"""GPU parity of the exact-dequant form of the W4A16 decode kernels (xb_set_w4_decode_form(1), spec form 2 of
oracle/quant.py): integer nibbles on the tensor core, scale / zero applied once per (row, group) in fp32.
  (a) against the exact-form oracle (float64) within the fp32 dot-product bound,
  (b) against the bf16-weight form within the rounding of w that form makes (2^-9 per weight),
  (c) the fused epilogues (SiLU*mul, RoPE + KV scatter, residual + statistics) and the staged-x variants under this form:
      the proofs of tests/test_gpu_fused_gemv.py re-run (fused == plain kernel + separate kernel, bit-exact),
  (d) a whole decode step."""
import pytest
import torch

from oracle import quant as Q
from tests import test_gpu_fused_gemv as F
from tests.util import assert_close_bf16, assert_close_sum

pytestmark = [pytest.mark.gpu, pytest.mark.w4_exact]
BF16 = torch.bfloat16
DEV = "cuda"

SHAPES = [(4608, 3584), (3584, 3584), (37888, 3584), (3584, 18944), (1152, 896)]


@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("M", [1, 4, 8])
@pytest.mark.parametrize("sym", [False, True])
def test_linear_w4a16_exact_form(M, N, K, sym, built_lib):
    from xllm_b200 import ops, quant
    if sym and N * K > 5e7:
        pytest.skip("full-size covered asym")
    gs = 128 if K % 128 == 0 else 64
    g = torch.Generator().manual_seed(2026)
    w = (torch.randn(N, K, generator=g) * 0.02).to(BF16)
    q, s, z = Q.quantize(w, 4, gs, sym=sym)
    x = torch.randn(M, K, generator=g).to(BF16)
    b = torch.randn(N, generator=g).to(BF16) if N == 4608 else None
    qw, meta = quant.pack_w4(q, s, z, gs)
    y = ops.w4a16_linear_small_m(x.to(DEV), qw.to(DEV), meta.to(DEV), gs, b.to(DEV) if b is not None else None)
    wd = Q.dequantize(q, s, z, gs)
    scale = x.float().abs() @ wd.float().abs().t() + (b.float().abs() if b is not None else 0)
    # (a) the form's own oracle.  The kernel accumulates sum x (128 + q) and subtracts (128 + z) sum x per group: its fp32
    # dot products run over terms |x| (128 + q) s, ~30x larger than |x||w|, so the honest fp32 bound (1e-5 of the sum of
    # the magnitudes of the terms actually added, tests/util.py) is stated on THAT sum - the price of the form: about one
    # bf16 ulp of a typical down_proj output.
    sg = s.float().repeat_interleave(gs, dim=1)
    scale_off = x.float().abs() @ ((q.float() + 128.0) * sg).t() + (b.float().abs() if b is not None else 0)
    assert_close_sum(y, Q.linear_wna16(x, q, s, z, gs, b, form="exact"), scale_off, rtol=1e-5, what=f"w4 exact M={M} N={N} K={K}")
    # (b) the other form: every weight rounded to bf16 first (<= 2^-9 relative per product).  Expected relative L2
    # distance: the rounding of w (RMS 1.66e-3 of every product, tests/util.py) and the two independent bf16 roundings of
    # the outputs (1.1e-3 each) -> sqrt(1.66^2 + 2 * 1.1^2) e-3 = 2.3e-3 (measured 2.0-2.4e-3)
    ref_b = Q.linear_wna16(x, q, s, z, gs, b)
    assert_close_sum(y, ref_b, scale, rtol=2.0 ** -9, rel_l2=3e-3, what="exact form vs bf16-weight form")


def test_exact_form_is_selected_and_differs(built_lib):
    """the switch is live: the two forms give different bits on a case where the bf16 rounding of w matters."""
    from xllm_b200 import ops, quant
    g = torch.Generator().manual_seed(7)
    N, K, gs = 512, 1024, 128
    w = (torch.randn(N, K, generator=g) * 0.02).to(BF16)
    q, s, z = Q.quantize(w, 4, gs)
    x = torch.randn(2, K, generator=g).to(BF16).to(DEV)
    qw, meta = quant.pack_w4(q, s, z, gs)
    qw, meta = qw.to(DEV), meta.to(DEV)
    y1 = ops.w4a16_linear_small_m(x, qw, meta, gs)
    old = ops.set_w4_decode_form(0)
    assert old == 1
    y0 = ops.w4a16_linear_small_m(x, qw, meta, gs)
    ops.set_w4_decode_form(1)
    assert not torch.equal(y0, y1)
    assert_close_bf16(y1, y0, ulps=1e9, rel_l2=3e-3, what="forms agree to bf16 rounding of w")


@pytest.mark.parametrize("nh,nkv,D,K", [(28, 4, 128, 3584), (14, 2, 64, 896)])
@pytest.mark.parametrize("M", [1, 8])
def test_exact_fused_rope_epilogue(M, nh, nkv, D, K, built_lib):
    F.test_fused_rope_epilogue_equals_gemv_then_rope(M, nh, nkv, D, K, True, built_lib, oracle_form="exact")


@pytest.mark.parametrize("N,K", [(3584, 3584), (3584, 18944), (37888, 3584)])
def test_exact_staged_x_is_bit_identical(N, K, built_lib):
    F.test_staged_x_is_bit_identical(N, K, built_lib)


@pytest.mark.parametrize("M", [1, 8])
def test_exact_gate_up_act_and_residual_stats(M, built_lib):
    """gate_up with the SiLU*mul epilogue and down_proj with the residual + statistics epilogue, exact form, against the
    exact-form oracle followed by the reference elementwise ops."""
    from oracle import ops as O
    from xllm_b200 import ops, quant
    g = torch.Generator().manual_seed(3)
    H, I, gs = 896, 2432, 64
    qg, sg, zg, _ = F._w4(2 * I, H, gs, 31, bias=False)
    x = torch.randn(M, H, generator=g).to(BF16)
    qw, meta, _ = quant.pack_w4_gate_up(qg, sg, zg, gs, None)
    act = ops.w4a16_gate_up_act(x.to(DEV), qw.to(DEV), meta.to(DEV), gs, "silu", None)
    ref = O.act_and_mul(Q.linear_wna16(x, qg, sg, zg, gs, None, form="exact"), "silu")
    assert_close_bf16(act, ref, ulps=4, rel_l2=3e-3, what="gate_up + act (exact form)", atol=2.0 ** -12)
    qd, sd, zd, _ = F._w4(H, I, gs, 32, bias=False)
    a = torch.randn(M, I, generator=g).to(BF16)
    res = torch.randn(M, H, generator=g).to(BF16)
    qw1, m1 = quant.pack_w4(qd, sd, zd, gs)
    res_out = torch.empty(M, H, dtype=BF16, device=DEV)
    stats = torch.full((H // 16, 8), -1.0, dtype=torch.float32, device=DEV)
    ops.w4a16_decode_fused(a.to(DEV), qw1.to(DEV), m1.to(DEV), gs, None, None, epilogue="residual_stats", residual_in=res.to(DEV),
                           residual_out=res_out, norm_stats_out=stats)
    torch.cuda.synchronize()
    r_ref = (Q.linear_wna16(a, qd, sd, zd, gs, None, form="exact").float() + res.float()).to(BF16)
    assert_close_bf16(res_out, r_ref, ulps=2, rel_l2=1e-3, what="residual stream (exact form)", atol=2.0 ** -8)
    tile_sq = (res_out.cpu().float() ** 2).view(M, H // 16, 16).sum(-1).t()
    assert torch.allclose(stats.cpu()[:, :M], tile_sq, rtol=1e-6, atol=0)


@pytest.mark.parametrize("use_graph", [True, False])
def test_decode_step_exact_form(use_graph, built_lib):
    from tests.model_parity import run_decode_parity
    from tests.test_gpu_model import _small
    cfg = _small("w4a16")
    logits, ref_logits, nxt, ref_next, _, _ = run_decode_parity(cfg, [37, 300, 1], use_graph, True)
    assert_close_bf16(logits, ref_logits, ulps=1e9, rel_l2=2e-2, what="decode-step logits (exact W4 form)")
    assert torch.equal(nxt.long().cpu()[:3], ref_next), "greedy tokens differ"
