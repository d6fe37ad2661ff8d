"""Edges of the weight-only and bf16 decode linears that the shape-driven suites do not reach.

  (a) group sizes from 256 up to K (one group per row) on every weight-only entry point: the meta row is then recomputed
      from the k index (>> log2(k64 tiles per group) >= 2) instead of advancing one row per ring slot or k block;
  (b) the exact-dequant form serves groups of 64 / 128 only and must fall back to the bf16-weight form bit for bit above;
  (c) group sizes the kernels cannot index are rejected before any launch (the host-only cases: test_group_size_checks_cpu);
  (d) the bf16 small-M kernel's per-warp cp.async ring: k32 tile counts below the warp count, not a multiple of 8, one
      ring and one ring + 1 per warp; N < 16; strided x and y; the Qwen2 lm_heads;
  (e) the W4 small-M launch geometry: grids of 1 CTA and around 1, 2, 3 x the SM count (where the shared-memory padding
      changes), a last CTA with idle row tiles, K = 64.
References are the spec of oracle/quant.py and oracle/ops.py, accumulated in float64 on the device."""
import re

import pytest
import torch

from oracle import ops as O
from oracle import quant as Q
from tests import test_gpu_fused_gemv as F
from tests.group_probe import w4_probe
from tests.util import assert_close_bf16, assert_close_sum

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"

# (N, K, gs): Qwen2-7B o_proj and down_proj at groups of 256 / 512, a Llama-3-70B TP8 o_proj shard at 256 / 1024 / K, and a
# narrow channelwise projection
LARGE_GROUPS = [(3584, 3584, 256), (3584, 3584, 512), (3584, 18944, 256), (3584, 18944, 512), (1024, 8192, 256),
                (1024, 8192, 1024), (1024, 8192, 8192), (64, 1024, 1024)]
SMALL_M = [1, 8, 9, 16, 17, 33, 64]      # every token-tile bucket of the small-M kernels and its edges


def _full_size(N, K):
    return N * K > 5e7


def _qsz(N, K, gs, bits, seed):
    """random logical weight-only tensors on the device: q over the whole range, scales and zeros per group"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randint(0, 1 << bits, (N, K), generator=g, device=DEV, dtype=torch.uint8)
    s = (torch.rand(N, K // gs, generator=g, device=DEV) * 0.01 + 0.001).to(BF16)
    z = torch.randint(0, 1 << bits, (N, K // gs), generator=g, device=DEV, dtype=torch.uint8)
    return q, s, z


def _ref(x, w, b=None):
    """spec linear on the bf16 weight w, accumulated in float64: (y rounded to bf16, sum_k |x w| + |b|)"""
    xd, wd = x.double(), w.double()
    y = xd @ wd.t()
    mag = xd.abs() @ wd.abs().t()
    if b is not None:
        y, mag = y + b.double(), mag + b.double().abs()
    return y.float().to(BF16), mag


def _check(y, ref, mag, what):
    assert_close_sum(y, ref, mag, rtol=1e-5, what=what)
    assert_close_bf16(y, ref, ulps=1e9, rel_l2=1e-3, what=what + " rel L2")


# ---- (a) group sizes 256 .. K ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("N,K,gs", LARGE_GROUPS)
@pytest.mark.parametrize("M", SMALL_M)
def test_w4a16_small_m_large_groups(M, N, K, gs, built_lib):
    from xllm_b200 import ops, quant
    if M > 1 and _full_size(N, K):
        pytest.skip("full size at M = 1")
    q, s, z = _qsz(N, K, gs, 4, seed=N + K + gs)
    g = torch.Generator(device=DEV).manual_seed(M)
    x = torch.randn(M, K, generator=g, device=DEV).to(BF16)
    b = torch.randn(N, generator=g, device=DEV).to(BF16) if N == 1024 else None
    qw, meta = quant.pack_w4(q, s, z, gs)
    y = ops.w4a16_linear_small_m(x, qw, meta, gs, b)
    ref, mag = _ref(x, Q.dequantize(q, s, z, gs), b)
    _check(y, ref, mag, f"w4a16 small-M M={M} N={N} K={K} gs={gs}")


@pytest.mark.parametrize("I,K,gs", [(18944, 3584, 512), (1024, 8192, 1024), (512, 8192, 8192), (512, 1024, 256)])
@pytest.mark.parametrize("M", [1, 8, 9, 16, 40])
def test_w4a16_gate_up_act_large_groups(M, I, K, gs, built_lib):
    """M <= 16: the GEMV with the SiLU*mul epilogue; M = 40: the wgmma GEMM + act_and_mul over the interleaved columns"""
    from xllm_b200 import ops, quant
    if M > 1 and _full_size(2 * I, K):
        pytest.skip("full size at M = 1")
    q, s, z = _qsz(2 * I, K, gs, 4, seed=I + K + gs)
    g = torch.Generator(device=DEV).manual_seed(M)
    x = torch.randn(M, K, generator=g, device=DEV).to(BF16)
    qw, meta, _ = quant.pack_w4_gate_up(q, s, z, gs)
    y = ops.w4a16_gate_up_act(x, qw, meta, gs, "silu")
    lin, mag = _ref(x, Q.dequantize(q, s, z, gs))
    lin, mag = lin.cpu(), mag.cpu().float()
    ref = O.act_and_mul(lin, "silu")
    # act(gate)*up of two 1-ulp-accurate linears (the bar of test_gpu_linear.py::test_w4a16_gate_up_act_fused: 4 ulps), plus
    # the fp32 summation-order error of each linear (1e-5 of sum |x w|, tests/util.py), which a gate or up value that cancels
    # to far below sum |x w| carries into the product: |silu'| <= 1.1, so by at most 1.1 |up| e_gate + |silu(gate)| e_up
    e = 1e-5 * mag
    gate, up = lin[:, :I].float(), lin[:, I:].float()
    carried = 1.1 * up.abs() * e[:, :I] + (gate * torch.sigmoid(gate)).abs() * e[:, I:] + e[:, :I] * e[:, I:]
    assert_close_bf16(y, ref, ulps=4, rel_l2=2e-3, what=f"gate_up_act M={M} I={I} K={K} gs={gs}", atol=carried + 1e-4)


@pytest.mark.parametrize("nh,nkv,D,K,gs", [(28, 4, 128, 3584, 256), (28, 4, 128, 3584, 512), (8, 1, 128, 8192, 1024),
                                           (8, 1, 128, 8192, 8192)])
@pytest.mark.parametrize("M", [1, 8])
@pytest.mark.parametrize("staged", [False, True])
def test_decode_fused_rope_large_groups(M, nh, nkv, D, K, gs, staged, built_lib):
    F.test_fused_rope_epilogue_equals_gemv_then_rope(M, nh, nkv, D, K, staged, built_lib, gs=gs)


@pytest.mark.parametrize("N,K,epi,gs", [(4608, 3584, "none", 256), (4608, 3584, "none", 512), (37888, 3584, "act_mul", 512),
                                        (1024, 8192, "none", 1024), (1024, 8192, "none", 8192)])
@pytest.mark.parametrize("M", [1, 4])
def test_decode_fused_norm_prologue_large_groups(M, N, K, epi, gs, built_lib):
    if M > 1 and _full_size(N, K):
        pytest.skip("full size at M = 1")
    F.test_fused_norm_prologue(M, N, K, epi, True, built_lib, gs=gs)


@pytest.mark.parametrize("H,Kin,Nout,epi,gs", [(3584, 3584, 4608, "none", 256), (3584, 3584, 4608, "none", 512),
                                               (3584, 18944, 37888, "act_mul", 512), (8192, 8192, 1280, "none", 1024),
                                               (8192, 8192, 1280, "none", 8192)])
@pytest.mark.parametrize("M", [1, 3])
def test_decode_fused_split_norm_large_groups(M, H, Kin, Nout, epi, gs, built_lib):
    if M > 1 and (_full_size(H, Kin) or _full_size(Nout, H)):
        pytest.skip("full size at M = 1")
    F.test_split_rms_norm_producer_and_consumer(M, H, Kin, Nout, epi, built_lib, gs=gs)


@pytest.mark.parametrize("N,K,gs", [(3584, 3584, 512), (3584, 18944, 256), (1024, 8192, 8192)])
def test_decode_fused_staged_x_large_groups(N, K, gs, built_lib):
    F.test_staged_x_is_bit_identical(N, K, built_lib, gs=gs)


@pytest.mark.parametrize("M,N,K,gs", [(17, 1024, 8192, 256), (300, 3584, 3584, 256), (333, 3584, 3584, 512),
                                      (200, 3584, 18944, 512), (130, 1024, 8192, 1024), (65, 1024, 8192, 8192),
                                      (100, 64, 1024, 1024), (1024, 20480, 4096, 4096)])
def test_w4a16_gemm_large_groups(M, N, K, gs, built_lib):
    """the wgmma dequant-GEMM (meta row of k block kb = kb >> log2(k64 tiles per group)), directly and through w4a16_linear,
    which takes it above 16 tokens unless the projection is narrow enough for the streaming kernel"""
    from xllm_b200 import ops, quant
    q, s, z = _qsz(N, K, gs, 4, seed=M + N + K + gs)
    g = torch.Generator(device=DEV).manual_seed(M)
    x = torch.randn(M, K, generator=g, device=DEV).to(BF16)
    b = torch.randn(N, generator=g, device=DEV).to(BF16) if M % 2 == 0 else None
    qw, meta = quant.pack_w4(q, s, z, gs)
    ref, mag = _ref(x, Q.dequantize(q, s, z, gs), b)
    _check(ops.gemm_w4a16(x, qw, meta, gs, b), ref, mag, f"gemm_w4a16 {M}x{N}x{K} gs={gs}")
    _check(ops.w4a16_linear(x, qw, meta, gs, b), ref, mag, f"w4a16_linear {M}x{N}x{K} gs={gs}")


@pytest.mark.parametrize("N,K,gs", LARGE_GROUPS)
@pytest.mark.parametrize("M", [1, 9, 33, 64, 200])
def test_w8a16_large_groups(M, N, K, gs, built_lib):
    """W8A16: the streaming kernel up to 64 tokens, the wgmma dequant-GEMM at 200"""
    from xllm_b200 import ops, quant
    if M > 1 and _full_size(N, K):
        pytest.skip("full size at M = 1")
    q, s, z = _qsz(N, K, gs, 8, seed=N + K + gs)
    s = (s.float() * 0.0625).to(BF16)                   # (q - z) spans +-255: keep the outputs near unit size
    g = torch.Generator(device=DEV).manual_seed(M)
    x = torch.randn(M, K, generator=g, device=DEV).to(BF16)
    b = torch.randn(N, generator=g, device=DEV).to(BF16) if N == 1024 else None
    qw, meta = quant.pack_w8(q, s, z, gs)
    ref, mag = _ref(x, Q.dequantize(q, s, z, gs), b)
    if M <= 64:
        _check(ops.w8a16_linear_small_m(x, qw, meta, gs, b), ref, mag, f"w8a16 small-M M={M} N={N} K={K} gs={gs}")
    else:
        _check(ops.gemm_w8a16(x, qw, meta, gs, b), ref, mag, f"gemm_w8a16 {M}x{N}x{K} gs={gs}")


# ---- (b) the exact-dequant form at large groups ------------------------------------------------------------------------

@pytest.mark.w4_exact
@pytest.mark.parametrize("gs", [64, 128, 256, 512, 4096])
def test_w4a16_dequant_is_bit_exact_exact_form(gs, built_lib):
    """the group-index probe under the exact-dequant form: 8 one-hot tokens per launch and K = 4096, so that x and its
    group sums fit the shared-memory stage and the form applies (groups of 64 / 128; above, the fallback).  With one non-zero
    x per token, s * ((128 + q) - (128 + z) * 1) is bf16((q - z) s) exactly.  N = 8448 keeps the k split at 4, so every
    split streams more groups than its ring holds."""
    w4_probe(gs, rows=8, N=8448, K=4096)


@pytest.mark.w4_exact
@pytest.mark.parametrize("N,K,gs", [(3584, 3584, 256), (1024, 8192, 1024), (3584, 18944, 512), (64, 1024, 1024)])
@pytest.mark.parametrize("M", [1, 8])
def test_exact_form_falls_back_above_128(M, N, K, gs, built_lib):
    """the exact-dequant form serves groups of 64 / 128; above, the decode kernels compute the bf16-weight form, bit for
    bit, with and without the shared-memory x stage (test_gpu_w4_exact.py shows the forms differ where both apply)"""
    from xllm_b200 import ops, quant
    q, s, z = _qsz(N, K, gs, 4, seed=7)
    g = torch.Generator(device=DEV).manual_seed(M)
    x = torch.randn(M, K, generator=g, device=DEV).to(BF16)
    qw, meta = quant.pack_w4(q, s, z, gs)
    staged = ops.w4a16_decode_fused_fits(M, K)
    y1 = ops.w4a16_linear_small_m(x, qw, meta, gs)
    f1 = ops.w4a16_decode_fused(x, qw, meta, gs, stage_x=staged)
    old = ops.set_w4_decode_form(0)
    assert old == 1
    try:
        y0 = ops.w4a16_linear_small_m(x, qw, meta, gs)
        f0 = ops.w4a16_decode_fused(x, qw, meta, gs, stage_x=staged)
    finally:
        ops.set_w4_decode_form(1)
    assert torch.equal(y1, y0), "w4a16_linear_small_m: the exact form did not fall back to the bf16-weight form"
    assert torch.equal(f1, f0), "w4a16_decode_fused: the exact form did not fall back to the bf16-weight form"


# ---- (c) rejections that need the device ---------------------------------------------------------------------------

def _raises_naming(fn, gs):
    from xllm_b200._lib import XllmB200Error
    with pytest.raises(XllmB200Error) as e:
        fn()
    assert re.search(rf"group_size {gs}\b|\(got {gs}\)", str(e.value)), str(e.value)


def test_w4_small_m_rejects_group_192(built_lib):
    """192 = 3 k64 tiles: a multiple of 64 dividing K = 384, but not a power-of-two number of tiles (checked after the
    device's SM count is read, hence on the device)"""
    from xllm_b200 import ops
    K, N, gs = 384, 128, 192
    x = torch.randn(1, K, device=DEV).to(BF16)
    qw = torch.zeros(N // 16, K // 64, 32, 4, dtype=torch.int32, device=DEV)
    meta = torch.zeros(K // gs, N, dtype=torch.int32, device=DEV)
    _raises_naming(lambda: ops.w4a16_linear_small_m(x, qw, meta, gs), gs)
    _raises_naming(lambda: ops.w4a16_gate_up_act(x, qw, meta, gs), gs)
    _raises_naming(lambda: ops.w4a16_decode_fused(x, qw, meta, gs, stage_x=True), gs)
    torch.cuda.synchronize()


@pytest.mark.parametrize("K,gs", [(384, 96), (960, 160)])
def test_prefill_linears_reject_groups_not_a_multiple_of_64(K, gs, built_lib):
    """a prefill batch (M = 300) must be refused like the decode batch, not computed with 64 / 128-wide groups"""
    from xllm_b200 import ops
    M, N = 300, 128
    x = torch.randn(M, K, device=DEV).to(BF16)
    meta = torch.zeros(K // gs, N, dtype=torch.int32, device=DEV)
    out = torch.full((M, N), 3.0, dtype=BF16, device=DEV)
    _raises_naming(lambda: ops.w4a16_linear(x, torch.zeros(N // 16, K // 64, 32, 4, dtype=torch.int32, device=DEV), meta, gs,
                                            out=out), gs)
    _raises_naming(lambda: ops.w8a16_linear(x, torch.zeros(N // 16, K // 64, 32, 8, dtype=torch.int32, device=DEV), meta, gs,
                                            out=out), gs)
    torch.cuda.synchronize()
    assert torch.all(out == 3.0), "a rejected call wrote its output"


# ---- (d) bf16 small-M ring edges -----------------------------------------------------------------------------------

# k32 tiles: 1, 2, 3 (warps without tiles), 7, 9 (not a multiple of 8), 23, 64 (one 8-slot ring per warp), 72 (one ring + 1),
# 256
RING_K = [32, 64, 96, 224, 288, 736, 2048, 2304, 8192]
RING_N = [1, 8, 15, 16, 17, 1007]
RING_M = [1, 8, 9, 16, 17, 32, 33, 64]


@pytest.mark.parametrize("K", RING_K)
@pytest.mark.parametrize("strided", [False, True])
def test_bf16_small_m_ring_edges(K, strided, built_lib):
    """every (N, bias, M) of the grid at this K; strided: x is a column slice of a wider buffer and y a column slice of a
    wider output filled with a sentinel that must survive"""
    from xllm_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(K)
    sentinel = -7.0
    for N in RING_N:
        w = (torch.randn(N, K, generator=g, device=DEV) * K ** -0.5).to(BF16)
        for bias in (False, True):
            b = torch.randn(N, generator=g, device=DEV).to(BF16) if bias else None
            for M in RING_M:
                if strided:
                    xbuf = torch.randn(M, K + 24, generator=g, device=DEV).to(BF16)
                    x = xbuf[:, 8:8 + K]
                    obuf = torch.full((M, N + 11), sentinel, dtype=BF16, device=DEV)
                    y = ops.matmul_small_m(x, w, b, out=obuf[:, 5:5 + N])
                else:
                    x = torch.randn(M, K, generator=g, device=DEV).to(BF16)
                    y = ops.matmul_small_m(x, w, b)
                ref, mag = _ref(x, w, b)
                _check(y, ref, mag, f"bf16 small-M M={M} N={N} K={K} bias={bias} strided={strided}")
                if strided:
                    assert torch.all(obuf[:, :5] == sentinel) and torch.all(obuf[:, 5 + N:] == sentinel), \
                        f"M={M} N={N} K={K}: columns outside the output slice were written"


@pytest.mark.parametrize("N,K", [(151936, 896), (151936, 3584)])
def test_bf16_small_m_qwen2_lm_heads(N, K, built_lib):
    from xllm_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(N + K)
    w = (torch.randn(N, K, generator=g, device=DEV) * 0.02).to(BF16)
    x = torch.randn(1, K, generator=g, device=DEV).to(BF16)
    y = ops.matmul_small_m(x, w)
    refs, mags = zip(*(_ref(x, w[n0:n0 + 16384]) for n0 in range(0, N, 16384)))
    _check(y, torch.cat(refs, 1), torch.cat(mags, 1), f"lm_head {N}x{K}")


# ---- (e) W4 small-M launch geometry ----------------------------------------------------------------------------------

def _w4_grid(N, K, sms):
    """the launch geometry w4_small_m_impl picks (csrc/linear_small_m.cu): the k split and the CTAs over N/16 row tiles"""
    ntiles, ktiles = N // 16, K // 64
    split = 1
    while split < 8 and ntiles * split < sms * 16 and ktiles // (split * 2) >= 3:
        split *= 2
    per_cta = 8 // split
    return (ntiles + per_cta - 1) // per_cta, per_cta


def _geometry_ns(K, sms):
    """N values whose grids are 1 CTA and sms * j + {-1, 0, 1} CTAs (j = 1, 2, 3): for every k split that gives such a
    grid, the fewest and the most row tiles that do (the fewest leaves idle row tiles in the last CTA wherever a CTA holds
    several)"""
    want = {1} | {j * sms + d for j in (1, 2, 3) for d in (-1, 0, 1)}
    lo, hi = {}, {}
    for nt in range(1, 8 * (3 * sms + 2)):
        grid, per_cta = _w4_grid(16 * nt, K, sms)
        if grid in want:
            lo.setdefault((grid, per_cta), nt)
            hi[grid, per_cta] = nt
    assert {grid for grid, _ in lo} == want, f"grids not reachable at K={K}"
    return sorted({16 * nt for nt in list(lo.values()) + list(hi.values())})


@pytest.mark.parametrize("K", [64, 3584, 18944])
def test_w4_small_m_launch_geometry(K, built_lib):
    from xllm_b200 import ops, quant
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ns = _geometry_ns(K, sms)
    assert any(_w4_grid(n, K, sms)[1] > 1 and (n // 16) % _w4_grid(n, K, sms)[1] for n in ns), "no CTA with idle row tiles"
    gs = 64 if K == 64 else 128
    nmax = ns[-1]
    # one weight for the widest N; narrower Ns use its leading row tiles.  Built in row chunks to bound the temporaries.
    qws, metas, wds = [], [], []
    for n0 in range(0, nmax, 8192):
        q, s, z = _qsz(min(8192, nmax - n0), K, gs, 4, seed=K + n0)
        qw, meta = quant.pack_w4(q, s, z, gs)
        qws.append(qw); metas.append(meta); wds.append(Q.dequantize(q, s, z, gs))
        del q
    qw_all, meta_all = torch.cat(qws), torch.cat(metas, 1)
    del qws, metas
    g = torch.Generator(device=DEV).manual_seed(K)
    for M in (1, 8):
        x = torch.randn(M, K, generator=g, device=DEV).to(BF16)
        refs, mags = zip(*(_ref(x, wd) for wd in wds))
        ref_all, mag_all = torch.cat(refs, 1), torch.cat(mags, 1)
        for N in ns:
            qw, meta = qw_all[:N // 16], meta_all[:, :N].contiguous()
            obuf = torch.full((2, M, N + 32), -7.0, dtype=BF16, device=DEV)
            y0 = ops.w4a16_linear_small_m(x, qw, meta, gs, out=obuf[0, :, 16:16 + N])
            y1 = ops.w4a16_linear_small_m(x, qw, meta, gs, out=obuf[1, :, 16:16 + N])
            grid, per_cta = _w4_grid(N, K, sms)
            what = f"W4 small-M M={M} N={N} K={K} ({grid} CTAs of {per_cta} row tiles)"
            _check(y0, ref_all[:, :N], mag_all[:, :N], what)
            assert torch.equal(y0, y1), f"{what}: two calls differ"
            assert torch.all(obuf[:, :, :16] == -7.0) and torch.all(obuf[:, :, 16 + N:] == -7.0), \
                f"{what}: columns outside the output slice were written"
