"""GPU parity: MoE router top-k (integer ids bit-exact, fp32 weights to expf rounding) and the decode-sized gated expert MLP
through the C ABI vs oracle/moe.py; FusedMoE layer composition incl. the expert-parallel split."""
import pytest
import torch

from oracle import moe as OM
from oracle import ops as O
from tests.util import assert_close_bf16

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"


@pytest.mark.parametrize("T,E,k", [(1, 8, 2), (5, 64, 6), (33, 128, 8), (3, 256, 8), (7, 60, 4), (2, 512, 32)])
@pytest.mark.parametrize("scoring,renorm,with_bias", [("softmax", True, False), ("softmax", False, False), ("sigmoid", True, True),
                                                      ("sigmoid", False, False)])
@pytest.mark.parametrize("dtype", [torch.float32, BF16])
def test_moe_fused_topk(T, E, k, scoring, renorm, with_bias, dtype, built_lib):
    from xllm_b200 import ops
    g = torch.Generator().manual_seed(T * 1000 + E + k)
    x = (torch.randn(T, E, generator=g) * 2).to(dtype)
    if T > 1:
        x[1, 3] = x[1, min(E - 1, 9)] = x[1].float().max().to(dtype) + 1          # exact tie: lower index first
    bias = (torch.randn(E, generator=g) * 0.5).float() if with_bias else None
    w_ref, id_ref = OM.moe_fused_topk(x, k, renorm, bias, scoring)
    w, ids = ops.moe_fused_topk(x.to(DEV), k, renorm, bias.to(DEV) if bias is not None else None, scoring)
    torch.cuda.synchronize()
    ids, w = ids.cpu(), w.cpu()
    same = ids == id_ref
    if not bool(same.all()):
        # a selection may differ only where two candidates are within the rounding of expf (never on exact ties)
        for t, kk in (~same).nonzero().tolist():
            a, b = int(ids[t, kk]), int(id_ref[t, kk])
            xa, xb = float(x[t, a]), float(x[t, b])
            assert xa != xb and abs(xa - xb) < 1e-5 * max(1.0, abs(xa)), (t, kk, a, b, xa, xb)
    assert torch.allclose(w[same], w_ref[same], rtol=2e-6, atol=1e-9)
    if T > 1:
        assert ids[1, 0] == 3 or scoring == "sigmoid" and with_bias


@pytest.mark.parametrize("T,k,E,H,I", [(1, 2, 4, 256, 128), (4, 8, 64, 1024, 512), (3, 6, 16, 2048, 1408), (16, 2, 8, 512, 96)])
def test_cutlass_fused_moe_decode(T, k, E, H, I, built_lib):
    from xllm_b200 import ops
    g = torch.Generator().manual_seed(E + H)
    x = torch.randn(T, H, generator=g).to(BF16)
    fc1 = (torch.randn(E, 2 * I, H, generator=g) * H ** -0.5).to(BF16)
    fc2 = (torch.randn(E, H, I, generator=g) * I ** -0.5).to(BF16)
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)]).to(torch.int32)
    sc = torch.rand(T, k, generator=g).float()
    ref, mag = OM.fused_moe(x, ids, sc, fc1, fc2, return_abs=True)
    out = ops.cutlass_fused_moe(x.to(DEV), ids.to(DEV), sc.to(DEV), fc1.to(DEV), fc2.to(DEV))
    torch.cuda.synchronize()
    # three roundings to bf16 (activation, expert output, final): a 1-ulp flip of one expert output y2_k moves the weighted
    # sum by an ulp of THAT term, which can exceed an ulp of a sum that cancels: bound on sum_k scale_k |y2_k|
    err = (out.float().cpu() - ref.float()).abs()
    bound = 2.0 ** -7 * mag + 2.0 ** -7 * ref.float().abs() + 2.0 ** -10
    assert bool((err <= bound).all()), f"fused_moe T={T} k={k} E={E}: worst err/bound {(err / bound).max():.2f}"
    assert float((out.float().cpu() - ref.float()).norm() / ref.float().norm()) <= 3e-3
    # expert parallelism: two ranks' partial outputs add up to the full result
    half = E // 2
    lo = ops.cutlass_fused_moe(x.to(DEV), ids.to(DEV), sc.to(DEV), fc1[:half].contiguous().to(DEV), fc2[:half].contiguous().to(DEV),
                               ep_size=2, ep_rank=0)
    hi = ops.cutlass_fused_moe(x.to(DEV), ids.to(DEV), sc.to(DEV), fc1[half:].contiguous().to(DEV), fc2[half:].contiguous().to(DEV),
                               ep_size=2, ep_rank=1)
    # each half is rounded to bf16 on its own before the all-reduce adds them: where the halves cancel, the error is an ulp of
    # the (larger) halves, not of the sum
    both = lo.float().cpu() + hi.float().cpu()
    err = (both - ref.float()).abs()
    bound = 2.0 ** -7 * (lo.float().abs().cpu() + hi.float().abs().cpu() + ref.float().abs()) + 2.0 ** -9
    assert bool((err <= bound).all()), f"EP halves: worst err/bound {(err / bound).max():.2f}"
    assert float((both - ref.float()).norm() / ref.float().norm()) <= 5e-3


def test_fused_moe_layer(built_lib):
    """gate -> top-k -> experts, against the oracle fed with the same router logits."""
    from xllm_b200.moe import FusedMoE
    g = torch.Generator().manual_seed(9)
    T, H, I, E, k = 5, 512, 256, 32, 4
    x = torch.randn(T, H, generator=g).to(BF16)
    gate = (torch.randn(E, H, generator=g) * H ** -0.5).to(BF16)
    w13 = (torch.randn(E, 2 * I, H, generator=g) * H ** -0.5).to(BF16)
    w2 = (torch.randn(E, H, I, generator=g) * I ** -0.5).to(BF16)
    layer = FusedMoE(gate.to(DEV), w13.to(DEV), w2.to(DEV), k, renormalize=True, scoring_func="softmax")
    y = layer.forward(x.to(DEV))
    torch.cuda.synchronize()
    logits = O.linear(x, gate)
    sc, ids = OM.moe_fused_topk(logits, k, True, None, "softmax")
    ref = OM.fused_moe(x, ids, sc, w13, w2)
    assert_close_bf16(y, ref, ulps=6, rel_l2=5e-3, what="FusedMoE layer", atol=2.0 ** -9)


@pytest.mark.parametrize("T,k,E,H,I,gs", [(1, 2, 4, 256, 128, 64), (4, 8, 32, 1024, 512, 128), (3, 6, 16, 2048, 1408, 128),
                                            (3, 4, 8, 1024, 512, 256), (64, 2, 4, 512, 512, 512), (2, 2, 4, 2048, 1024, 1024)])
def test_fused_moe_w4a16_decode(T, k, E, H, I, gs, built_lib):
    """W4A16 experts (additive, BASELINE configs[4]): per-expert tile-packed int4 weights through the expert-indexed GEMVs vs the
    oracle MoE on the dequantised weights (spec form 1 of oracle/quant.py: w = bf16((q - z) s))."""
    from oracle import quant as Q
    from xllm_b200 import ops, quant
    g = torch.Generator().manual_seed(E * 7 + H)
    x = torch.randn(T, H, generator=g).to(BF16)
    fc1 = (torch.randn(E, 2 * I, H, generator=g) * H ** -0.5).to(BF16)
    fc2 = (torch.randn(E, H, I, generator=g) * I ** -0.5).to(BF16)
    q1w, m1, q2w, m2, d1, d2 = [], [], [], [], [], []
    for e in range(E):
        q, s, z = Q.quantize(fc1[e], 4, gs)
        a, b = quant.pack_w4(q, s, z, gs)
        q1w.append(a); m1.append(b); d1.append(Q.dequantize(q, s, z, gs))
        q, s, z = Q.quantize(fc2[e], 4, gs)
        a, b = quant.pack_w4(q, s, z, gs)
        q2w.append(a); m2.append(b); d2.append(Q.dequantize(q, s, z, gs))
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)]).to(torch.int32)
    sc = torch.rand(T, k, generator=g).float()
    ref, mag = OM.fused_moe(x, ids, sc, torch.stack(d1), torch.stack(d2), return_abs=True)
    out = ops.fused_moe_w4a16(x.to(DEV), ids.to(DEV), sc.to(DEV), torch.stack(q1w).to(DEV), torch.stack(m1).to(DEV),
                              torch.stack(q2w).to(DEV), torch.stack(m2).to(DEV), gs)
    torch.cuda.synchronize()
    err = (out.float().cpu() - ref.float()).abs()
    bound = 2.0 ** -7 * mag + 2.0 ** -7 * ref.float().abs() + 2.0 ** -10
    assert bool((err <= bound).all()), f"fused_moe_w4a16 T={T} k={k} E={E}: worst err/bound {(err / bound).max():.2f}"
    assert float((out.float().cpu() - ref.float()).norm() / ref.float().norm()) <= 3e-3
