"""GPU parity: wgmma GEMMs (bf16, FP8 W8A8, W4A16 dequant-GEMM) through the C ABI vs the oracle."""
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


def _abs_scale(x, w, b=None):
    s = x.float().abs() @ w.float().abs().t()
    return s + (b.float().abs() if b is not None else 0)


# (M, N, K): tile-aligned, ragged M / N / K, multi-tile persistent, Qwen2-7B projections at chunk sizes
BF16_SHAPES = [(128, 128, 64), (128, 128, 512), (256, 384, 1024), (100, 136, 200), (1, 64, 64), (333, 4608, 3584),
               (2048, 3584, 3584), (512, 37888, 3584), (300, 3584, 18944), (129, 1152, 896), (256, 256, 64), (256, 256, 512),
               (384, 512, 1024), (300, 768, 200), (1024, 3584, 3584), (2049, 4608, 3584), (256, 37888, 512)]


@pytest.mark.parametrize("M,N,K", BF16_SHAPES)
def test_gemm_bf16(M, N, K, built_lib):
    from xllm_b200 import ops
    g = torch.Generator().manual_seed(2026)
    a = torch.randn(M, K, generator=g).to(BF16)
    w = (torch.randn(N, K, generator=g) * 0.02).to(BF16)
    b = torch.randn(N, generator=g).to(BF16) if N % 3 == 0 else None
    ref = O.linear(a, w, b)
    y = ops.gemm_bf16(a.to(DEV), w.to(DEV), b.to(DEV) if b is not None else None)
    assert_close_sum(y, ref, _abs_scale(a, w, b), rtol=1e-5, what=f"gemm_bf16 {M}x{N}x{K}")
    assert_close_bf16(y, ref, ulps=1e9, rel_l2=1e-3, what="gemm_bf16 rel L2")


def test_gemm_bf16_strided_a_and_out(built_lib):
    """A is a column slice of a wider buffer (like attn_out views) and C a slice of a wider output."""
    from xllm_b200 import ops
    g = torch.Generator().manual_seed(1)
    big = torch.randn(200, 1024, generator=g).to(BF16)
    w = (torch.randn(256, 512, generator=g) * 0.05).to(BF16)
    ref = O.linear(big[:, 256:768], w)
    outbuf = torch.zeros(200, 640, dtype=BF16, device=DEV)
    y = ops.gemm_bf16(big.to(DEV)[:, 256:768], w.to(DEV), None, outbuf[:, 128:384])
    assert_close_sum(y, ref, _abs_scale(big[:, 256:768], w), rtol=1e-5, what="strided gemm")
    assert torch.all(outbuf[:, :128] == 0) and torch.all(outbuf[:, 384:] == 0)


def test_gemm_bf16_matches_small_m_kernel_bitwise_spec(built_lib):
    """decode and prefill paths of the same linear agree (same spec, different kernels)."""
    from xllm_b200 import ops
    g = torch.Generator().manual_seed(3)
    a = torch.randn(16, 3584, generator=g).to(BF16).to(DEV)
    w = (torch.randn(4608, 3584, generator=g) * 0.02).to(BF16).to(DEV)
    y1 = ops.gemm_bf16(a, w)
    y2 = ops.matmul_small_m(a, w)
    assert_close_sum(y1, y2, _abs_scale(a.cpu(), w.cpu()), rtol=1e-5, what="gemm vs small-m")


# reference's own test grid: tests/core/kernels/cuda/cutlass_scaled_mm_test.cpp:44-296 (up to 512x1024x768, per-tensor,
# per-token x per-channel, bias) - there checked loosely (max diff < 2, mean < 0.5 vs fp32 matmul); here vs the oracle.
FP8_CASES = [(16, 128, 128, False, False, False), (64, 256, 512, False, False, True), (512, 1024, 768, True, True, True),
             (100, 272, 400, True, False, False), (300, 4608, 3584, False, True, True), (2048, 3584, 3584, False, False, False),
             (300, 256, 400, True, False, False), (1024, 4608, 3584, True, True, False), (384, 37888, 3584, False, True, True)]


@pytest.mark.parametrize("M,N,K,per_token,per_channel,use_bias", FP8_CASES)
def test_cutlass_scaled_mm(M, N, K, per_token, per_channel, use_bias, built_lib):
    from xllm_b200 import ops
    if K % 16:
        pytest.skip("K%16 required")
    g = torch.Generator().manual_seed(2026)
    a = torch.randn(M, K, generator=g).clamp(-3, 3).to(E4M3)
    w = torch.randn(N, K, generator=g).clamp(-3, 3).to(E4M3)
    a_s = (torch.rand(M if per_token else 1, generator=g) * 0.1 + 0.01).float()
    b_s = (torch.rand(N if per_channel else 1, generator=g) * 0.1 + 0.01).float()
    bias = torch.randn(N, generator=g).to(BF16) if use_bias else None
    ref = O.fp8_scaled_matmul(a, w, a_s, b_s, bias)
    c = torch.empty(M, N, dtype=BF16, device=DEV)
    ops.cutlass_scaled_mm(c, a.to(DEV), w.to(DEV).t(), a_s.to(DEV), b_s.to(DEV), bias.to(DEV) if bias is not None else None)
    scale = (a.float().abs() @ w.float().abs().t()) * a_s.reshape(-1, 1) * b_s.reshape(1, -1)
    if bias is not None:
        scale = scale + bias.float().abs()
    assert_close_sum(c, ref, scale, rtol=1e-5, what=f"cutlass_scaled_mm {M}x{N}x{K}")
    assert_close_bf16(c, ref, ulps=1e9, rel_l2=1e-3, what="fp8 rel L2")


def test_cutlass_scaled_mm_argument_checks(built_lib):
    """same rejections as the reference's TORCH_CHECKs (cutlass_scaled_mm_test.cpp:279-295)."""
    from xllm_b200 import ops
    from xllm_b200._lib import XllmB200Error
    a = torch.zeros(16, 128, dtype=E4M3, device=DEV)
    w = torch.zeros(64, 128, dtype=E4M3, device=DEV)
    s1 = torch.ones(1, device=DEV)
    c = torch.empty(16, 64, dtype=BF16, device=DEV)
    with pytest.raises(XllmB200Error):
        ops.cutlass_scaled_mm(c, a, w, s1, s1)                      # b not column-major
    with pytest.raises(XllmB200Error):
        ops.cutlass_scaled_mm(c, a, w.t(), torch.ones(3, device=DEV), s1)   # bad scale numel
    with pytest.raises(XllmB200Error):
        ops.cutlass_scaled_mm(torch.empty(16, 32, dtype=BF16, device=DEV), a, w.t(), s1, s1)   # shape mismatch


def test_fp8_linear_static_and_dynamic(built_lib):
    """fp8_linear_forward (linear.cpp:137-182): quantise activations (static / dynamic scale) then scaled matmul."""
    from xllm_b200 import ops
    g = torch.Generator().manual_seed(5)
    x = torch.randn(96, 1024, generator=g).to(BF16)
    w8 = (torch.randn(512, 1024, generator=g)).clamp(-2, 2).to(E4M3)
    w_s = torch.tensor([0.02])
    for in_scale in (torch.tensor([0.01]), None):
        ref = O.fp8_linear(x, w8, w_s, in_scale)
        q, s = ops.fp8_scaled_quantize(x.to(DEV), None, in_scale.to(DEV) if in_scale is not None else None)
        y = ops.fp8_scaled_matmul(q, w8.to(DEV), s, w_s.to(DEV))
        assert_close_bf16(y, ref, ulps=1, rel_l2=1e-3, what="fp8 linear")


W4_SHAPES = [(128, 128, 128), (64, 64, 64), (100, 192, 256), (333, 4608, 3584), (1024, 3584, 3584), (256, 37888, 3584),
             (200, 3584, 18944), (17, 1152, 896), (256, 256, 128), (300, 512, 256), (512, 37888, 3584), (400, 3584, 18944),
             (1024, 4608, 3584)]


@pytest.mark.parametrize("M,N,K", W4_SHAPES)
def test_gemm_w4a16(M, N, K, built_lib):
    from xllm_b200 import ops, quant
    gs = 128 if K % 128 == 0 else 64
    g = torch.Generator().manual_seed(2026)
    w = (torch.randn(N, K, generator=g) * 0.02).to(BF16)
    q, s, z = Q.quantize(w, 4, gs)
    x = torch.randn(M, K, generator=g).to(BF16)
    b = torch.randn(N, generator=g).to(BF16) if N == 4608 else None
    ref = Q.linear_wna16(x, q, s, z, gs, b)
    qw, meta = quant.pack_w4(q, s, z, gs)
    y = ops.gemm_w4a16(x.to(DEV), qw.to(DEV), meta.to(DEV), gs, b.to(DEV) if b is not None else None)
    assert_close_sum(y, ref, _abs_scale(x, Q.dequantize(q, s, z, gs), b), rtol=1e-5, what=f"gemm_w4a16 {M}x{N}x{K}")
    assert_close_bf16(y, ref, ulps=1e9, rel_l2=1e-3, what="gemm_w4a16 rel L2")


def test_gemm_w4a16_dequant_bit_exact(built_lib):
    """identity activations read the dequantised weights back out of the tensor-core path bit-for-bit, at every group size
    from 64 to K; scales and zeros differ from group to group, so a k block that reads another group's meta row shows."""
    from xllm_b200 import ops, quant
    N, K = 256, 2048
    x = torch.eye(K, dtype=BF16, device=DEV)
    for gs in (64, 128, 256, 512, K):
        q, s, z = group_probe_weights(N, K, gs, 4, seed=11)
        wd = Q.dequantize(q, s, z, gs)
        qw, meta = quant.pack_w4(q, s, z, gs)
        y = ops.gemm_w4a16(x, qw.to(DEV), meta.to(DEV), gs)
        assert torch.equal(y.cpu(), wd.t().contiguous()), f"dequant mismatch at group size {gs}"


def test_w4a16_decode_and_prefill_kernels_agree(built_lib):
    from xllm_b200 import ops, quant
    g = torch.Generator().manual_seed(13)
    N, K, gs, M = 4608, 3584, 128, 16
    q = torch.randint(0, 16, (N, K), dtype=torch.uint8, generator=g)
    s = (torch.rand(N, K // gs, generator=g) * 0.01 + 0.001).to(BF16)
    z = torch.randint(0, 16, (N, K // gs), dtype=torch.uint8, generator=g)
    qw, meta = quant.pack_w4(q, s, z, gs)
    x = torch.randn(M, K, generator=g).to(BF16).to(DEV)
    y1 = ops.gemm_w4a16(x, qw.to(DEV), meta.to(DEV), gs)
    y2 = ops.w4a16_linear_small_m(x, qw.to(DEV), meta.to(DEV), gs)
    wd = Q.dequantize(q, s, z, gs)
    assert_close_sum(y1, y2, _abs_scale(x.cpu(), wd), rtol=1e-5, what="w4 prefill vs decode kernel")


@pytest.mark.parametrize("M,N,K,per_token,per_channel,use_bias", [(1, 256, 128, False, False, False), (32, 1280, 8192, True, True, True),
                                                                  (17, 8192, 1024, False, True, False), (64, 7168, 8192, True, False, True),
                                                                  (33, 1000, 416, False, False, False)])
def test_cutlass_scaled_mm_swap_ab(M, N, K, per_token, per_channel, use_bias, built_lib):
    """decode-sized M through the wgmma kernel with the weight rows in the MMA M slot (xb_set_fp8_swap_max_m): same spec."""
    from xllm_b200 import ops
    g = torch.Generator().manual_seed(2026)
    a = torch.randn(M, K, generator=g).clamp(-3, 3).to(E4M3)
    w = torch.randn(N, K, generator=g).clamp(-3, 3).to(E4M3)
    a_s = (torch.rand(M if per_token else 1, generator=g) * 0.1 + 0.01).float()
    b_s = (torch.rand(N if per_channel else 1, generator=g) * 0.1 + 0.01).float()
    bias = torch.randn(N, generator=g).to(BF16) if use_bias else None
    ref = O.fp8_scaled_matmul(a, w, a_s, b_s, bias)
    c = torch.zeros(M, N, dtype=BF16, device=DEV)
    old = ops.set_fp8_swap_max_m(64)
    try:
        ops.gemm_fp8_scaled(c, a.to(DEV), w.to(DEV), a_s.to(DEV), b_s.to(DEV), bias.to(DEV) if bias is not None else None)
        torch.cuda.synchronize()
    finally:
        ops.set_fp8_swap_max_m(old)
    scale = (a.float().abs() @ w.float().abs().t()) * a_s.reshape(-1, 1) * b_s.reshape(1, -1)
    if bias is not None:
        scale = scale + bias.float().abs()
    assert_close_sum(c, ref, scale, rtol=1e-5, what=f"fp8 swap-AB {M}x{N}x{K}")


@pytest.mark.parametrize("M,N,K,per_token,per_channel,use_bias", [(32, 1280, 8192, True, True, True), (17, 8192, 1024, False, True, False),
                                                                  (64, 7168, 8192, True, False, True), (5, 256, 4736, False, False, False),
                                                                  (32, 8192, 3584, False, False, False), (1, 128, 28672, True, True, True)])
def test_cutlass_scaled_mm_swap_ab_split_k(M, N, K, per_token, per_channel, use_bias, built_lib):
    """swap-AB FP8 GEMM with K cut into ranges over otherwise idle SMs (xb_set_gemm_splitk_workspace): same spec, the same bits
    on every call (partials are summed in split order; the arrival tickets reset themselves), and back to the unsplit kernel
    when the workspace is withdrawn."""
    from xllm_b200 import ops
    g = torch.Generator().manual_seed(77)
    a = torch.randn(M, K, generator=g).clamp(-3, 3).to(E4M3)
    w = torch.randn(N, K, generator=g).clamp(-3, 3).to(E4M3)
    a_s = (torch.rand(M if per_token else 1, generator=g) * 0.1 + 0.01).float()
    b_s = (torch.rand(N if per_channel else 1, generator=g) * 0.1 + 0.01).float()
    bias = torch.randn(N, generator=g).to(BF16) if use_bias else None
    ref = O.fp8_scaled_matmul(a, w, a_s, b_s, bias)
    ad, wd, asd, bsd = a.to(DEV), w.to(DEV), a_s.to(DEV), b_s.to(DEV)
    bd = bias.to(DEV) if bias is not None else None
    outs = []
    ops.enable_fp8_splitk(DEV)
    try:
        for _ in range(3):
            c = torch.zeros(M, N, dtype=BF16, device=DEV)
            ops.gemm_fp8_scaled(c, ad, wd, asd, bsd, bd)
            torch.cuda.synchronize()
            outs.append(c.cpu())
    finally:
        ops.disable_fp8_splitk()
    c1 = torch.zeros(M, N, dtype=BF16, device=DEV)
    ops.gemm_fp8_scaled(c1, ad, wd, asd, bsd, bd)
    torch.cuda.synchronize()
    scale = (a.float().abs() @ w.float().abs().t()) * a_s.reshape(-1, 1) * b_s.reshape(1, -1)
    if bias is not None:
        scale = scale + bias.float().abs()
    assert_close_sum(outs[0], ref, scale, rtol=1e-5, what=f"fp8 swap-AB split-K {M}x{N}x{K}")
    assert_close_sum(c1, ref, scale, rtol=1e-5, what=f"fp8 swap-AB unsplit {M}x{N}x{K}")
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2]), "split-K result changed between calls"
