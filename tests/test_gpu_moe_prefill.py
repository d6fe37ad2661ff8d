"""GPU parity of the MoE prefill path (T >= 65): device-side routing + grouped wgmma GEMMs behind ops.cutlass_fused_moe and
ops.fused_moe_w4a16, against tests/moe_grouped_ref.py::fused_moe_grouped (pinned to oracle.moe.fused_moe on the CPU), checked
in two steps (_run_checked) with the bounds of test_gpu_moe.py.  Also: skewed routing, ids outside the local range, expert
parallelism, more than 65535 pairs, determinism, CUDA-graph replay with new routing, the FusedMoE layer and the C++ shim's
cutlass_fused_moe."""
import pytest
import torch

from oracle import moe as OM
from tests.moe_grouped_ref import fused_moe_grouped

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"


def _weights(g, E, H, I):
    fc1 = (torch.randn(E, 2 * I, H, generator=g) * H ** -0.5).to(BF16)
    fc2 = (torch.randn(E, H, I, generator=g) * I ** -0.5).to(BF16)
    return fc1, fc2


def _random_ids(g, T, k, E):
    return torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)]).to(torch.int32)


class _W4:
    """per-expert tile-packed int4 experts and their dequantised bf16 weights (the spec the kernels are checked against)"""

    def __init__(self, fc1, fc2, gs):
        from oracle import quant as Q
        from xllm_b200 import quant
        q1w, m1, q2w, m2, d1, d2 = [], [], [], [], [], []
        for e in range(fc1.size(0)):
            q, s, z = Q.quantize(fc1[e], 4, gs)
            a, b = quant.pack_w4(q, s, z, gs)
            q1w.append(a); m1.append(b); d1.append(Q.dequantize(q, s, z, gs))
            q, s, z = Q.quantize(fc2[e], 4, gs)
            a, b = quant.pack_w4(q, s, z, gs)
            q2w.append(a); m2.append(b); d2.append(Q.dequantize(q, s, z, gs))
        self.gs = gs
        self.dev = [torch.stack(t).to(DEV) for t in (q1w, m1, q2w, m2)]
        self.fc1, self.fc2 = torch.stack(d1), torch.stack(d2)


def _run(kind, x, ids, sc, w, **kw):
    from xllm_b200 import ops
    if kind == "bf16":
        fc1, fc2 = w
        return ops.cutlass_fused_moe(x.to(DEV), ids.to(DEV), sc.to(DEV), fc1.to(DEV), fc2.to(DEV), **kw)
    return ops.fused_moe_w4a16(x.to(DEV), ids.to(DEV), sc.to(DEV), *w.dev, w.gs, **kw)


def _spec_weights(kind, w):
    return w if kind == "bf16" else (w.fc1, w.fc2)


def _check(out, ref, mag, what):
    err = (out.float().cpu() - ref.float()).abs()
    bound = 2.0 ** -7 * mag + 2.0 ** -7 * ref.float().abs() + 2.0 ** -10
    assert bool((err <= bound).all()), f"{what}: worst err/bound {(err / bound).max():.2f}"
    den = ref.float().norm()
    if float(den) > 0:
        assert float((out.float().cpu() - ref.float()).norm() / den) <= 3e-3, what


def _act_of_pairs(ws, T, k, H, I, n_local):
    """the activations the grouped path left in its workspace (include/xllm_b200_ops.h: header, row_of_pair, pair_of_row,
    sorted input, act, y2), back in pair order [T, k, I]; zero for pairs of other experts"""
    P = T * k
    m = (4 * P + 255) // 256 * 256
    pair_of_row = ws[8192 + m:8192 + m + 4 * P].view(torch.int32)[:n_local].long()
    off = 8192 + 2 * m + P * H * 2
    act = ws[off:off + P * I * 2].view(BF16).view(P, I)[:n_local]
    out = torch.zeros(P, I, dtype=BF16, device=ws.device)
    out[pair_of_row] = act
    return out.view(T, k, I).cpu()


def _run_checked(kind, x, ids, sc, w, what, expert_begin=0, **kw):
    """run the grouped path and check it in two steps, each against one bf16 rounding: the activations against the reference's
    (the fp32 sums of GEMM1 differ in their last bits, so an activation may round the other way: <= 1 ulp, plus a floor for
    activations that cancel to ~0), then the output against the reference's GEMM2 + combine run from the same activations.
    Every activation that rounds the other way moves a whole y2 row by |fc2 column| x 1 ulp, which the end-to-end bound of
    test_gpu_moe.py does not allow for; the end-to-end result is held to its rel-L2 bar."""
    from xllm_b200 import ops
    T, k = ids.shape
    H = x.size(1)
    fc1, fc2 = _spec_weights(kind, w)
    El, I = fc1.size(0), fc2.size(2)
    ws = torch.empty(int(ops.lib().xb_moe_experts_workspace_bytes(T, k, H, I)), dtype=torch.uint8, device=DEV)
    out = _run(kind, x, ids, sc, w, workspace=ws, **kw)
    torch.cuda.synchronize()
    ref, _, act_ref = fused_moe_grouped(x, ids, sc, fc1, fc2, expert_begin, return_abs=True, return_act=True)
    n_local = int(((ids >= expert_begin) & (ids < expert_begin + El)).sum())
    act = _act_of_pairs(ws, T, k, H, I, n_local)
    da = (act.float() - act_ref.float()).abs()
    assert bool((da <= 2.0 ** -7 * act_ref.float().abs() + 2.0 ** -16).all()), f"{what}: activations"
    ref2, mag2 = fused_moe_grouped(x, ids, sc, fc1, fc2, expert_begin, return_abs=True, act=act)
    _check(out, ref2, mag2, what)
    den = ref.float().norm()
    if float(den) > 0:
        assert float((out.float().cpu() - ref.float()).norm() / den) <= 3e-3, what
    return out, act


def _problem(kind, seed, T, k, E, H, I, gs=128):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, H, generator=g).to(BF16)
    fc1, fc2 = _weights(g, E, H, I)
    w = (fc1, fc2) if kind == "bf16" else _W4(fc1, fc2, gs)
    return g, x, w


def test_the_default_boundary_is_65_tokens(built_lib):
    from xllm_b200 import ops
    assert ops.moe_experts_describe("bf16", 64, 8, 7168, 2048, 32) == "bf16 gemv"
    assert ops.moe_experts_describe("w4", 65, 8, 7168, 2048, 32).startswith("w4 grouped")


@pytest.mark.parametrize("T", [65, 256, 1000])
@pytest.mark.parametrize("E,k,H,I", [(8, 2, 512, 96), (60, 4, 1024, 1408), (32, 8, 256, 160)])
def test_grouped_bf16(T, E, k, H, I, built_lib):
    g, x, w = _problem("bf16", T * 31 + E, T, k, E, H, I)
    ids = _random_ids(g, T, k, E)
    sc = torch.rand(T, k, generator=g).float()
    _run_checked("bf16", x, ids, sc, w, f"bf16 T={T} E={E} k={k} H={H} I={I}")


@pytest.mark.parametrize("T", [65, 256, 1000])
@pytest.mark.parametrize("E,k,H,I,gs", [(8, 2, 512, 128, 64), (8, 4, 512, 1408, 128), (4, 2, 7168, 128, 128), (8, 2, 1024, 512, 256),
                                         (4, 2, 512, 512, 512)])
def test_grouped_w4a16(T, E, k, H, I, gs, built_lib):
    g, x, w = _problem("w4", T * 37 + E, T, k, E, H, I, gs)
    ids = _random_ids(g, T, k, E)
    sc = torch.rand(T, k, generator=g).float()
    _run_checked("w4", x, ids, sc, w, f"w4 T={T} E={E} k={k} H={H} I={I} g={gs}")


def _skewed_routings(g, E):
    """(name, ids [T, k]) with k = 1 or 2"""
    out = [("one expert", torch.full((300, 1), 3, dtype=torch.int32))]
    # segments of 1, 127, 128 and 129 rows on experts 0..3, experts 4.. empty, tokens in shuffled order
    seg = torch.cat([torch.full((n,), e, dtype=torch.int32) for e, n in enumerate((1, 127, 128, 129))])
    out.append(("segments 1/127/128/129", seg[torch.randperm(seg.numel(), generator=g)].view(-1, 1)))
    # ids outside [0, E): negative and too large, mixed with local ones
    ids = torch.randint(-3, E + 3, (200, 2), generator=g, dtype=torch.int32)
    ids[:5] = -1
    ids[5:10] = E
    out.append(("foreign ids", ids))
    return out


@pytest.mark.parametrize("kind", ["bf16", "w4"])
def test_skewed_routing(kind, built_lib):
    E, H, I = 8, 256, 128
    g, x_all, w = _problem(kind, 5, 385, 2, E, H, I)
    for name, ids in _skewed_routings(g, E):
        T, k = ids.shape
        x = x_all[:T].contiguous()
        sc = torch.rand(T, k, generator=g).float()
        out, _ = _run_checked(kind, x, ids, sc, w, f"{kind} {name}")
        if name == "foreign ids":
            only_foreign = ((ids < 0) | (ids >= E)).all(1)
            assert bool(only_foreign[:10].all()) and torch.equal(out[:10].cpu(), torch.zeros(10, H, dtype=BF16))


def test_expert_parallel_halves_add_up(built_lib):
    T, k, E, H, I = 256, 4, 16, 512, 256
    g, x, (fc1, fc2) = _problem("bf16", 11, T, k, E, H, I)
    ids = _random_ids(g, T, k, E)
    sc = torch.rand(T, k, generator=g).float()
    half = E // 2
    lo, act_lo = _run_checked("bf16", x, ids, sc, (fc1[:half].contiguous(), fc2[:half].contiguous()), "EP rank 0", 0,
                              ep_size=2, ep_rank=0)
    hi, act_hi = _run_checked("bf16", x, ids, sc, (fc1[half:].contiguous(), fc2[half:].contiguous()), "EP rank 1", half,
                              ep_size=2, ep_rank=1)
    # the full layer from the same activations (each pair's activations come from the rank that owns its expert)
    ref = fused_moe_grouped(x, ids, sc, fc1, fc2, act=act_lo.float() + act_hi.float())
    both = lo.float().cpu() + hi.float().cpu()
    err = (both - ref.float()).abs()
    bound = 2.0 ** -7 * (lo.float().abs().cpu() + hi.float().abs().cpu() + ref.float().abs()) + 2.0 ** -9
    assert bool((err <= bound).all()), f"EP halves: worst err/bound {(err / bound).max():.2f}"
    assert float((both - ref.float()).norm() / ref.float().norm()) <= 5e-3


def test_more_than_65535_pairs(built_lib):
    """a full default prefill batch at DeepSeek-V3's top-8 (10240 x 8 pairs), which the GEMV path cannot take"""
    T, k, E, H, I = 10240, 8, 16, 128, 64
    g, x, w = _problem("bf16", 13, T, k, E, H, I)
    ids = _random_ids(g, T, k, E)
    sc = torch.rand(T, k, generator=g).float()
    _run_checked("bf16", x, ids, sc, w, "10240 x 8 pairs")


def test_deterministic(built_lib):
    T, k, E, H, I = 1000, 4, 16, 512, 256
    g, x, w = _problem("bf16", 17, T, k, E, H, I)
    ids = _random_ids(g, T, k, E)
    sc = torch.rand(T, k, generator=g).float()
    a = _run("bf16", x, ids, sc, w)
    b = _run("bf16", x, ids, sc, w)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_cuda_graph_replays_with_new_routing(built_lib):
    from xllm_b200 import ops
    T, k, E, H, I = 512, 4, 16, 512, 256
    g, x, (fc1, fc2) = _problem("bf16", 19, T, k, E, H, I)
    x, fc1, fc2 = x.to(DEV), fc1.to(DEV), fc2.to(DEV)
    routings = [(_random_ids(g, T, k, E).to(DEV), torch.rand(T, k, generator=g).float().to(DEV)) for _ in range(4)]
    ids, sc = routings[0][0].clone(), routings[0][1].clone()
    out = torch.empty(T, H, dtype=BF16, device=DEV)
    ws = torch.empty(int(ops.lib().xb_moe_experts_workspace_bytes(T, k, H, I)), dtype=torch.uint8, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.cutlass_fused_moe(x, ids, sc, fc1, fc2, output=out, workspace=ws)      # warm-up outside capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.cutlass_fused_moe(x, ids, sc, fc1, fc2, output=out, workspace=ws)
    results = []
    for r_ids, r_sc in routings[1:]:
        ids.copy_(r_ids)
        sc.copy_(r_sc)
        graph.replay()
        results.append(out.clone())
    torch.cuda.synchronize()
    for (r_ids, r_sc), got in zip(routings[1:], results):
        eager = ops.cutlass_fused_moe(x, r_ids, r_sc, fc1, fc2)
        torch.cuda.synchronize()
        assert torch.equal(got, eager)
    assert not torch.equal(results[0], results[1])


def test_fused_moe_layer_prefill(built_lib):
    """gate -> top-k -> experts at T = 512: the router against the oracle's on the same logits, the layer bit for bit against
    the composition of the ops, and the experts against the grouped reference (two-step check)"""
    from xllm_b200 import ops
    from xllm_b200.moe import FusedMoE
    g = torch.Generator().manual_seed(23)
    T, H, I, E, k = 512, 512, 256, 32, 4
    x = torch.randn(T, H, generator=g).to(BF16)
    gate = (torch.randn(E, H, generator=g) * H ** -0.5).to(BF16)
    w13, w2 = _weights(g, E, H, I)
    layer = FusedMoE(gate.to(DEV), w13.to(DEV), w2.to(DEV), k, renormalize=True, scoring_func="softmax")
    y = layer.forward(x.to(DEV))
    logits = ops.matmul(x.to(DEV), gate.to(DEV))
    sc_dev, ids_dev = ops.moe_fused_topk(logits, k, True, None, "softmax")
    torch.cuda.synchronize()
    sc, ids = OM.moe_fused_topk(logits.cpu(), k, True, None, "softmax")
    same = (ids_dev.cpu() == ids).all(1)
    assert int(same.sum()) >= T - 2          # a selection may differ only within the rounding of expf (test_gpu_moe.py)
    assert torch.allclose(sc_dev.cpu()[same], sc[same], rtol=2e-6, atol=1e-9)
    out, _ = _run_checked("bf16", x, ids_dev.cpu(), sc_dev.cpu(), (w13, w2), "FusedMoE experts T=512")
    assert torch.equal(y, out)


def test_shim_cutlass_fused_moe_matches_ops(built_lib):
    from xllm_b200 import build_shim, ops
    shim = build_shim.load_py()
    T, k, E, H, I = 512, 4, 16, 512, 256
    g, x, (fc1, fc2) = _problem("bf16", 29, T, k, E, H, I)
    ids = _random_ids(g, T, k, E).to(DEV)
    sc = torch.rand(T, k, generator=g).float().to(DEV)
    x, fc1, fc2 = x.to(DEV), fc1.to(DEV), fc2.to(DEV)
    a = shim.cutlass_fused_moe(x, ids, sc, fc1, fc2)
    b = ops.cutlass_fused_moe(x, ids, sc, fc1, fc2)
    half = E // 2
    c = shim.cutlass_fused_moe(x, ids, sc, fc1[half:].contiguous(), fc2[half:].contiguous(), 2, 1)
    d = ops.cutlass_fused_moe(x, ids, sc, fc1[half:].contiguous(), fc2[half:].contiguous(), ep_size=2, ep_rank=1)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(c, d)
