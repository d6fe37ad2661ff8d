"""GPU parity of the 8-bit linears: W8A16 weight-only (streaming decode kernel + wgmma dequant-GEMM, spec
oracle/quant.py with bits = 8) and the FP8 W8A8 small-M (swap-AB streaming) kernel behind cutlass_scaled_mm."""
import pytest
import torch

from oracle import ops as O
from oracle import quant as Q
from tests.group_probe import group_probe_weights
from tests.util import assert_close_bf16, assert_close_sum

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
E4M3 = torch.float8_e4m3fn
DEV = "cuda"

# Qwen2-7B projections + Qwen2-0.5B qkv + Llama-3-70B TP8 shards
SHAPES = [(4608, 3584), (3584, 3584), (37888, 3584), (3584, 18944), (1152, 896), (1280, 8192)]


def _abs_scale(x, w, b=None):
    s = x.float().abs() @ w.float().abs().t()
    return s + (b.float().abs() if b is not None else 0)


@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("M", [1, 5, 8, 16, 40, 64])
@pytest.mark.parametrize("sym", [False, True])
def test_linear_w8a16_small_m(M, N, K, sym, built_lib):
    from xllm_b200 import ops, quant
    if (M > 8 or sym) and N * K > 5e7:
        pytest.skip("full-size covered at M<=8 asym")
    gs = 128 if K % 128 == 0 else 64
    g = torch.Generator().manual_seed(2026)
    w = (torch.randn(N, K, generator=g) * 0.02).to(BF16)
    q, s, z = Q.quantize(w, 8, gs, sym=sym)
    x = torch.randn(M, K, generator=g).to(BF16)
    b = torch.randn(N, generator=g).to(BF16) if N == 4608 else None
    ref = Q.linear_wna16(x, q, s, z, gs, b)
    qw, meta = quant.pack_w8(q, s, z, gs)
    y = ops.w8a16_linear_small_m(x.to(DEV), qw.to(DEV), meta.to(DEV), gs, b.to(DEV) if b is not None else None)
    assert_close_sum(y, ref, _abs_scale(x, Q.dequantize(q, s, z, gs), b), rtol=1e-5, what=f"w8a16 M={M} N={N} K={K} sym={sym}")
    assert_close_bf16(y, ref, ulps=1e9, rel_l2=1e-3, what="w8a16 rel L2")


def test_w8a16_dequant_is_bit_exact(built_lib):
    """identity activations read single weights back: every one of the 256 levels, zero points across the 8-bit range
    and both kernels (streaming and wgmma converter) must reproduce bf16((q - z) * s) bit for bit, at every group size from
    64 to K; scales and zeros differ from group to group, so reading another group's meta row shows."""
    from xllm_b200 import ops, quant
    N, K = 256, 2048
    eye = torch.eye(K, dtype=BF16, device=DEV)
    for gs in (64, 128, 256, 512, K):
        q, s, z = group_probe_weights(N, K, gs, 8, seed=11)             # zero points (n + 7 g) mod 256: the whole range
        q[0, :256] = torch.arange(256, dtype=torch.uint8)              # all levels in one row
        wd = Q.dequantize(q, s, z, gs)
        qw, meta = quant.pack_w8(q, s, z, gs)
        assert torch.equal(qw, quant.pack_w8_c(q)), "torch and C packers disagree"
        qw, meta = qw.to(DEV), meta.to(DEV)
        for k0 in range(0, K, 64):
            y = ops.w8a16_linear_small_m(eye[k0:k0 + 64], qw, meta, gs)
            assert torch.equal(y.cpu(), wd[:, k0:k0 + 64].t().contiguous()), \
                f"streaming kernel: dequant mismatch in k block {k0} at group size {gs}"
        y = ops.gemm_w8a16(eye, qw, meta, gs)
        assert torch.equal(y.cpu(), wd.t().contiguous()), f"wgmma converter: dequant mismatch at group size {gs}"


@pytest.mark.parametrize("M,N,K", [(128, 4608, 3584), (333, 3584, 3584), (2048, 37888, 3584), (512, 3584, 18944), (17, 1152, 896),
                                   (100, 1280, 8192)])
def test_gemm_w8a16(M, N, K, built_lib):
    from xllm_b200 import ops, quant
    gs = 128 if K % 128 == 0 else 64
    g = torch.Generator().manual_seed(2026)
    w = (torch.randn(N, K, generator=g) * 0.02).to(BF16)
    q, s, z = Q.quantize(w, 8, gs)
    x = torch.randn(M, K, generator=g).to(BF16)
    b = torch.randn(N, generator=g).to(BF16) if N == 4608 else None
    qw, meta = quant.pack_w8(q, s, z, gs)
    y = ops.gemm_w8a16(x.to(DEV), qw.to(DEV), meta.to(DEV), gs, b.to(DEV) if b is not None else None)
    wd = Q.dequantize(q, s, z, gs)
    if M * N * K > 2e10:      # full size: against the bf16 wgmma GEMM on the dequantised weight (the CPU oracle takes minutes)
        ref = ops.gemm_bf16(x.to(DEV), wd.to(DEV), b.to(DEV) if b is not None else None).cpu()
    else:
        ref = Q.linear_wna16(x, q, s, z, gs, b)
    assert_close_sum(y, ref, _abs_scale(x, wd, b), rtol=1e-5, what=f"gemm_w8a16 {M}x{N}x{K}")
    assert_close_bf16(y, ref, ulps=1e9, rel_l2=1e-3, what="gemm_w8a16 rel L2")


def test_w8a16_decode_and_prefill_kernels_agree(built_lib):
    from xllm_b200 import ops, quant
    g = torch.Generator().manual_seed(13)
    N, K, gs, M = 4608, 3584, 128, 16
    q = torch.randint(0, 256, (N, K), dtype=torch.uint8, generator=g)
    s = (torch.rand(N, K // gs, generator=g) * 0.001 + 0.0001).to(BF16)
    z = torch.randint(100, 156, (N, K // gs), dtype=torch.uint8, generator=g)
    qw, meta = quant.pack_w8(q, s, z, gs)
    x = torch.randn(M, K, generator=g).to(BF16).to(DEV)
    y1 = ops.gemm_w8a16(x, qw.to(DEV), meta.to(DEV), gs)
    y2 = ops.w8a16_linear_small_m(x, qw.to(DEV), meta.to(DEV), gs)
    assert_close_sum(y1, y2, _abs_scale(x.cpu(), Q.dequantize(q, s, z, gs)), rtol=1e-5, what="w8 prefill vs decode kernel")


# ---- FP8 W8A8 small-M ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,K", [(4608, 3584), (3584, 18944), (10240, 8192), (1024, 3584), (1008, 512)])
@pytest.mark.parametrize("M", [1, 7, 16, 32, 64])
@pytest.mark.parametrize("per_row", [False, True])
def test_fp8_small_m_matches_oracle(M, N, K, per_row, built_lib):
    """the streaming swap-AB kernel behind cutlass_scaled_mm at decode sizes (M <= 64) against the oracle's
    fp8_scaled_matmul (scaled_mm_entry.cu:55-108 semantics) and against the FP8 GEMM on the same inputs."""
    from xllm_b200 import ops
    if N * K > 5e7 and M not in (1, 32):
        pytest.skip("full size at M = 1 and 32")
    g = torch.Generator().manual_seed(2026)
    a = torch.randn(M, K, generator=g).clamp(-3, 3).to(E4M3)
    b = torch.randn(N, K, generator=g).clamp(-3, 3).to(E4M3)
    a_s = (torch.rand(M if per_row else 1, generator=g) * 0.05 + 0.01).float()
    b_s = (torch.rand(N if per_row else 1, generator=g) * 0.05 + 0.01).float()
    bias = torch.randn(N, generator=g).to(BF16) if N == 4608 else None
    ref = O.fp8_scaled_matmul(a, b, a_s, b_s, bias)
    c = torch.empty(M, N, dtype=BF16, device=DEV)
    ops.fp8_scaled_mm_small_m(c, a.to(DEV), b.to(DEV).t(), a_s.to(DEV), b_s.to(DEV), bias.to(DEV) if bias is not None else None)
    scale = (a.float().abs() @ b.float().abs().t()) * a_s.view(-1, 1) * b_s.view(1, -1) + (bias.float().abs() if bias is not None else 0)
    assert_close_sum(c, ref, scale, rtol=1e-5, what=f"fp8 small-M {M}x{N}x{K} per_row={per_row}")
    assert_close_bf16(c, ref, ulps=1e9, rel_l2=1e-3, what="fp8 small-M rel L2")
    if N % 64 == 0:
        # the wgmma kernel on the same inputs (forced by calling the GEMM entry point directly)
        from xllm_b200._lib import c_i32, c_i64, check, lib
        c2 = torch.empty_like(c)
        ad, bd, asd, bsd = a.to(DEV), b.to(DEV), a_s.to(DEV), b_s.to(DEV)
        bi = bias.to(DEV) if bias is not None else None
        check(lib().xb_gemm_fp8_scaled(ops._p(c2), c_i64(c2.stride(0)), ops._p(ad), c_i64(ad.stride(0)), ops._p(bd), ops._p(asd),
                                       c_i32(asd.numel()), ops._p(bsd), c_i32(bsd.numel()), ops._p(bi), c_i32(M), c_i32(N), c_i32(K),
                                       ops._stream()), "gemm_fp8_scaled")
        assert_close_sum(c, c2, scale, rtol=1e-5, what="fp8 small-M vs wgmma GEMM")


def test_fp8_small_m_exact_products(built_lib):
    """e4m3 x e4m3 products are exact in fp32 and small sums too: with power-of-two scales the kernel must reproduce an
    integer-valued reference bit for bit (checks the k permutation of the two operands slot by slot)."""
    from xllm_b200 import ops
    g = torch.Generator().manual_seed(5)
    M, N, K = 8, 64, 128
    a = torch.randint(-4, 5, (M, K), generator=g).float().to(E4M3)
    b = torch.randint(-4, 5, (N, K), generator=g).float().to(E4M3)
    one = torch.ones(1, dtype=torch.float32, device=DEV)
    c = torch.empty(M, N, dtype=BF16, device=DEV)
    ops.fp8_scaled_mm_small_m(c, a.to(DEV), b.to(DEV).t(), one, one * 0.5, None)
    ref = (a.float() @ b.float().t() * 0.5).to(BF16)
    assert torch.equal(c.cpu(), ref)


@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (300, 512, 256), (1024, 3584, 3584)])
def test_gemm_w8a16_prefill_shapes(M, N, K, built_lib):
    """the kind-W8 wgmma kernel at prefill-sized M: converter warps dequantise the int8 tiles into the MMA's B stages."""
    from xllm_b200 import ops, quant
    gs = 128
    g = torch.Generator().manual_seed(2026)
    w = (torch.randn(N, K, generator=g) * 0.02).to(BF16)
    q, s, z = Q.quantize(w, 8, gs)
    x = torch.randn(M, K, generator=g).to(BF16)
    qw, meta = quant.pack_w8(q, s, z, gs)
    y = ops.gemm_w8a16(x.to(DEV), qw.to(DEV), meta.to(DEV), gs)
    wd = Q.dequantize(q, s, z, gs)
    ref = Q.linear_wna16(x, q, s, z, gs, None)
    assert_close_sum(y, ref, _abs_scale(x, wd, None), rtol=1e-5, what=f"gemm_w8a16 {M}x{N}x{K}")
