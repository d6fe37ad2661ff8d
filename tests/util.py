"""Shared tolerances for the parity tests.

bf16 carries 8 significant bits, so two correct bf16 results of the same fp32 value can differ by one ulp
(2^-8 relative) when the fp32 values straddle a rounding boundary.  The bar used everywhere a floating-point
kernel is compared with the oracle (north_star: "within 1e-3 relative for bf16/FP8"):
  * relative L2 error over the tensor   <= 1e-3
  * every element within `ulps` bf16 ulps of the oracle (default 1; accumulation-order noise)
Integer / copy / index work is compared with torch.equal (bit-exact).

Attention: the reference ladder (FlashInfer) rounds the softmax numerators P to bf16 before the PV tensor-core
product, relative to whatever running maximum the tile order produced, so two correct implementations with a
different tile / split order differ by independent 2^-9-relative perturbations of every p_j.  For
o_d = sum_j p_j v_jd that is a forward error of up to ~1e-3 * sum_j p_j |v_jd| - NOT 1e-3 * |o_d|, which on the
synthetic N(0,1) KV of SURVEY 8d is ~sqrt(kv_len) smaller because of cancellation.  `assert_close_attention`
therefore states the bar in the standard dot-product sense: |err_d| <= 2e-3 * sum_j p_j |v_jd| + 1 bf16 ulp (two
independent 2^-9 roundings of every p_j - the oracle's and the kernel's - i.e. 1e-3 each; checked over millions of elements),
with the scale sum_j p_j |v_jd| computed by the oracle itself (same attention with |V|).
"""
import torch


REL_L2_LOG = []      # (what, rel-L2) of every attention comparison of the session (printed by conftest at exit)


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    a = x.abs().to(torch.float32).clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def assert_close_bf16(got: torch.Tensor, ref: torch.Tensor, ulps: float = 1.0, rel_l2: float = 1e-3, what: str = "",
                      atol: float = 0.0):
    g, r = got.detach().cpu().to(torch.float32), ref.detach().cpu().to(torch.float32)
    assert g.shape == r.shape, f"{what}: shape {g.shape} vs {r.shape}"
    assert torch.isfinite(g).all(), f"{what}: non-finite output"
    err = (g - r).abs()
    den = r.norm().item()
    l2 = (g - r).norm().item() / den if den > 0 else (g - r).norm().item()
    assert l2 <= rel_l2, f"{what}: relative L2 error {l2:.3e} > {rel_l2:.1e}"
    bound = ulps * torch.maximum(bf16_ulp(r), bf16_ulp(g)) + atol
    bad = err > bound
    assert not bad.any(), (f"{what}: {int(bad.sum())} / {bad.numel()} elements beyond {ulps} bf16 ulp; "
                           f"worst |err|={err.max().item():.3e} at ref={r.flatten()[err.argmax()].item():.4e}")
    return l2


def assert_close_attention(got, ref, abs_scale, rtol: float = 2e-3, what: str = "", rel_l2: float = 3e-3):
    """|got - ref| <= rtol * (sum_j p_j |v_j|) + 1 bf16 ulp(ref), elementwise (see module docstring), AND relative L2
    error over the tensor <= rel_l2, so that a regression in the accumulation ladder is visible long before it trips
    the forward-error bound.  rel_l2=None disables it.

    Why 3e-3 and not the north-star's 1e-3: the reference ladder (FlashInfer) rounds every softmax numerator p_j to bf16
    (8 significant bits: relative error uniform in +-2^-8/m, m the significand in [1,2) - RMS 2^-8 * sqrt(E[1/m^2]/3) =
    1.66e-3).  On synthetic N(0,1) V the output o = sum p_j v_j has the same magnitude as the error-carrying sum, so ONE
    implementation of the reference ladder sits 1.66e-3 (relative L2) from the un-rounded result, and two independent
    implementations (different tile / split order => different running maxima => independent roundings) sit
    sqrt(2) * 1.66e-3 = 2.35e-3 apart before the bf16 rounding of o itself; the reference's own two decode paths (CUDA-core
    and tensor-core FlashInfer) differ from each other by as much.  The single-implementation
    distance is asserted separately against the fp32-P oracle (test_paged_decode_distance_from_exact_math).

    The same bound with rtol = 1e-5 is used for fp32-accumulated dot products (linears): two correct summation orders
    of sum_k x_k w_k differ by O(eps_fp32 * sqrt(K)) * sum_k |x_k w_k|, which is many bf16 ulps of an output that
    happens to cancel to ~0, so the absolute term has to be relative to sum_k |x_k w_k| (computed by the oracle)."""
    g, r = got.detach().cpu().to(torch.float32), ref.detach().cpu().to(torch.float32)
    sc = abs_scale.detach().cpu().to(torch.float32)
    assert g.shape == r.shape == sc.shape, f"{what}: shapes {g.shape} {r.shape} {sc.shape}"
    assert torch.isfinite(g).all(), f"{what}: non-finite output"
    err = (g - r).abs()
    if rel_l2 is not None and r.norm().item() > 0:
        l2 = (g - r).norm().item() / r.norm().item()
        REL_L2_LOG.append((what, l2))
        assert l2 <= rel_l2, f"{what}: relative L2 error {l2:.3e} > {rel_l2:.1e}"
    bound = rtol * sc + torch.maximum(bf16_ulp(r), bf16_ulp(g))
    bad = err > bound
    assert not bad.any(), (f"{what}: {int(bad.sum())} / {bad.numel()} elements beyond {rtol:.0e} * sum p|v| + 1 ulp; "
                           f"worst err/bound = {(err / bound).max().item():.2f}")
    return (err / sc.clamp_min(1e-30)).max().item()


assert_close_sum = assert_close_attention
