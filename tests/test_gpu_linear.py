"""GPU parity: small-M linears (bf16 and W4A16) through the C ABI vs the oracle."""
import pytest
import torch

from oracle import ops as O
from oracle import quant as Q
from tests.group_probe import PROBE_K, w4_probe
from tests.util import assert_close_bf16, assert_close_sum


def _abs_scale(x, w, b=None):
    s = x.float().abs() @ w.float().abs().t()
    return s + (b.float().abs() if b is not None else 0)

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"

# Qwen2-7B projections (qkv, o, gate_up, down) + Qwen2-0.5B qkv + an lm_head slice
SHAPES = [(4608, 3584), (3584, 3584), (37888, 3584), (3584, 18944), (1152, 896), (16000, 3584)]


@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("M", [1, 5, 8, 9, 33, 64])
def test_linear_bf16_small_m(M, N, K, built_lib):
    from xllm_b200 import ops
    if M > 8 and N * K > 5e7:
        pytest.skip("large-M full-size cases covered by M<=8 and the smaller shapes")
    g = torch.Generator().manual_seed(2026)
    w = (torch.randn(N, K, generator=g) * 0.02).to(BF16)
    x = torch.randn(M, K, generator=g).to(BF16)
    b = torch.randn(N, generator=g).to(BF16) if N % 3 == 0 else None
    ref = O.linear(x, w, b)
    y = ops.matmul_small_m(x.to(DEV), w.to(DEV), b.to(DEV) if b is not None else None)
    assert_close_sum(y, ref, _abs_scale(x, w, b), rtol=1e-5, what=f"linear_bf16 M={M} N={N} K={K}")
    assert_close_bf16(y, ref, ulps=1e9, rel_l2=1e-3, what="linear_bf16 rel L2")


def test_linear_bf16_ragged_n(built_lib):
    from xllm_b200 import ops
    g = torch.Generator().manual_seed(3)
    N, K, M = 1000 + 7, 256, 3                      # N not a multiple of 16
    w = (torch.randn(N, K, generator=g) * 0.05).to(BF16)
    x = torch.randn(M, K, generator=g).to(BF16)
    y = ops.matmul_small_m(x.to(DEV), w.to(DEV))
    assert_close_sum(y, O.linear(x, w), _abs_scale(x, w), rtol=1e-5, what="ragged N")


@pytest.mark.parametrize("N,K", SHAPES[:5])
@pytest.mark.parametrize("M", [1, 4, 8, 16, 40, 64])
@pytest.mark.parametrize("sym", [False, True])
def test_linear_w4a16_small_m(M, N, K, sym, built_lib):
    from xllm_b200 import ops, quant
    if (M > 8 or sym) and N * K > 5e7:
        pytest.skip("full-size covered at M<=8 asym")
    gs = 128 if K % 128 == 0 else 64
    g = torch.Generator().manual_seed(2026)
    w = (torch.randn(N, K, generator=g) * 0.02).to(BF16)
    q, s, z = Q.quantize(w, 4, gs, sym=sym)
    x = torch.randn(M, K, generator=g).to(BF16)
    b = torch.randn(N, generator=g).to(BF16) if N == 4608 else None
    ref = Q.linear_wna16(x, q, s, z, gs, b)
    qw, meta = quant.pack_w4(q, s, z, gs)
    y = ops.w4a16_linear_small_m(x.to(DEV), qw.to(DEV), meta.to(DEV), gs, b.to(DEV) if b is not None else None)
    wd = Q.dequantize(q, s, z, gs)
    assert_close_sum(y, ref, _abs_scale(x, wd, b), rtol=1e-5, what=f"w4a16 M={M} N={N} K={K} sym={sym}")
    assert_close_bf16(y, ref, ulps=1e9, rel_l2=1e-3, what="w4a16 rel L2")


def test_w4a16_dequant_is_bit_exact(built_lib):
    """x = identity rows picks out single weights: y[m, n] = bf16(w[n, k_m]) must equal the spec's dequantised
    weight bit-for-bit (one rounding in (q-z)*s), at every group size from 64 to K (tests/group_probe.py)."""
    for gs in (64, 128, 256, 512, PROBE_K):
        w4_probe(gs)


def test_linear_linearity_full_size(built_lib):
    """Property at BASELINE size (gate_up, M=64): f(x1 + x2) == f(x1) + f(x2) up to fp32 accumulation order when
    x1, x2 have disjoint support (exact split of the K sum)."""
    from xllm_b200 import ops, quant
    g = torch.Generator().manual_seed(5)
    N, K, M, gs = 37888, 3584, 64, 128
    q = torch.randint(0, 16, (N, K), dtype=torch.uint8, generator=g)
    s = (torch.rand(N, K // gs, generator=g) * 0.01 + 0.001).to(BF16)
    z = torch.randint(0, 16, (N, K // gs), dtype=torch.uint8, generator=g)
    qw, meta = quant.pack_w4(q, s, z, gs)
    qw, meta = qw.to(DEV), meta.to(DEV)
    x = torch.randn(M, K, generator=g).to(BF16).to(DEV)
    x1, x2 = x.clone(), x.clone()
    x1[:, K // 2:] = 0
    x2[:, :K // 2] = 0
    y = ops.w4a16_linear_small_m(x, qw, meta, gs).float()
    y12 = ops.w4a16_linear_small_m(x1, qw, meta, gs).float() + ops.w4a16_linear_small_m(x2, qw, meta, gs).float()
    rel = ((y - y12).norm() / y.norm()).item()
    assert rel < 4e-3, f"linearity violated: {rel:.3e}"   # two extra bf16 output roundings


@pytest.mark.parametrize("M", [1, 7, 8, 16, 40])
@pytest.mark.parametrize("I,K,bias", [(18944, 3584, False), (512, 256, True), (4864, 896, False)])
def test_w4a16_gate_up_act_fused(M, I, K, bias, built_lib):
    """gate_up linear + SiLU*mul in one kernel (interleaved gate/up packing) == act_and_mul(linear(x)) of the oracle."""
    from xllm_b200 import ops, quant
    if M > 8 and I * K > 5e7:
        pytest.skip("full size covered at M<=8")
    gs = 128 if K % 128 == 0 else 64
    g = torch.Generator().manual_seed(2026)
    w = (torch.randn(2 * I, K, generator=g) * 0.05).to(BF16)
    q, s, z = Q.quantize(w, 4, gs)
    b = (torch.randn(2 * I, generator=g) * 0.1).to(BF16) if bias else None
    x = torch.randn(M, K, generator=g).to(BF16)
    ref = O.act_and_mul(Q.linear_wna16(x, q, s, z, gs, b), "silu")
    qw, meta, bi = quant.pack_w4_gate_up(q, s, z, gs, b)
    y = ops.w4a16_gate_up_act(x.to(DEV), qw.to(DEV), meta.to(DEV), gs, "silu", bi.to(DEV) if bi is not None else None)
    # act(gate)*up of two 1-ulp-accurate linears: a flip in either input moves the product by up to ~2 ulps
    assert_close_bf16(y, ref, ulps=4, rel_l2=2e-3, what=f"gate_up_act M={M} I={I}", atol=1e-4)
    frac = (y.cpu() != ref).float().mean().item()
    assert frac < 0.05, f"{frac:.3f} of elements differ"


def test_interleave_index_is_a_permutation():
    from xllm_b200 import quant
    idx = quant.interleave_gate_up_index(64)
    assert sorted(idx.tolist()) == list(range(128))
    assert idx[:16].tolist() == list(range(8)) + list(range(64, 72))


@pytest.mark.parametrize("fmt", ["awq", "gptq"])
def test_checkpoint_layout_tensor_through_the_kernels(fmt, built_lib):
    """SURVEY 8f n1 end to end on the GPU: tensors in the AutoAWQ / AutoGPTQ checkpoint layout -> from_awq / from_gptq ->
    kernel layout (xb_w4_pack_rows) -> the decode GEMV and the wgmma dequant-GEMM, against the oracle on the logical form."""
    from tests.test_checkpoint_surface import _logical, _pack_awq, _pack_seq_lastdim
    from xllm_b200 import ops, quant
    N, K, gs = 1152, 1024, 128
    q, z, s = _logical(N=N, K=K, gs=gs, seed=4)
    if fmt == "awq":
        q2, s2, z2 = quant.from_awq(_pack_awq(q.t().contiguous()), _pack_awq(z.t().contiguous()), s.t().contiguous(), gs)
    else:
        qw_ckpt = _pack_seq_lastdim(q).t().contiguous()
        qz_ckpt = _pack_seq_lastdim((z.t().to(torch.int16) - 1).contiguous())
        g_idx = torch.arange(K, dtype=torch.int32) // gs
        q2, s2, z2 = quant.from_gptq(qw_ckpt, qz_ckpt, s.t().contiguous(), g_idx, gs)
    assert torch.equal(q2, q) and torch.equal(z2, z)
    qw, meta = quant.pack_w4(q2, s2, z2, gs)
    g = torch.Generator().manual_seed(8)
    for M in (1, 7, 300):
        x = torch.randn(M, K, generator=g).to(BF16)
        ref = Q.linear_wna16(x, q2, s2, z2, gs, None)
        y = ops.w4a16_linear(x.to(DEV), qw.to(DEV), meta.to(DEV), gs) if hasattr(ops, "w4a16_linear") else \
            (ops.w4a16_linear_small_m if M <= 64 else ops.gemm_w4a16)(x.to(DEV), qw.to(DEV), meta.to(DEV), gs)
        assert_close_sum(y, ref, _abs_scale(x, Q.dequantize(q2, s2, z2, gs)), rtol=1e-5, what=f"{fmt} checkpoint M={M}")
