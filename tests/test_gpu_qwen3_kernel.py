"""GPU: xb_qk_norm_rope_and_cache_bf16 (K10+K12 in one launch) against the two-launch pair fused_qk_norm_rope +
reshape_paged_cache (bit for bit in qkv and both caches) and against the oracle (1 bf16 ulp)."""
import pytest
import torch

from oracle import ops as O
from tests.util import assert_close_bf16

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"
MAX_POS = 8192
BS = 16


def _case(T, HQ, HKV, D, seed):
    """qkv rows, norm weights, table, positions (some at the end of the table), slots: a scattered permutation with slot -1
    tokens and, from T >= 3 on, decode padding rows (same row, position 0, slot 0) at the end"""
    g = torch.Generator().manual_seed(seed)
    heads = HQ + 2 * HKV
    # per-head magnitudes spread over two decades so that the norm matters
    qkv = (torch.randn(T, heads, D, generator=g) * torch.exp(torch.randn(T, heads, 1, generator=g))).to(BF16).view(T, -1)
    qw = (1 + 0.1 * torch.randn(D, generator=g)).to(BF16)
    kw = (1 + 0.1 * torch.randn(D, generator=g)).to(BF16)
    cs = O.compute_cos_sin_cache(D, MAX_POS, 1000000.0, BF16)
    pos = torch.randint(0, MAX_POS, (T,), generator=g)
    pos[: max(1, T // 8)] = MAX_POS - 1 - torch.arange(max(1, T // 8)) % 4
    nblocks = (T + BS - 1) // BS + 4
    slots = (torch.randperm(nblocks * BS - BS, generator=g)[:T] + BS).to(torch.int32)   # block 0 kept for padding
    if T >= 3:
        slots[1::7] = -1
        npad = max(1, T // 16)
        qkv[T - npad:] = qkv[T - npad]
        pos[T - npad:] = 0
        slots[T - npad:] = 0
    kc = torch.randn(nblocks, BS, HKV, D, generator=g).to(BF16)
    vc = torch.randn(nblocks, BS, HKV, D, generator=g).to(BF16)
    return qkv, qw, kw, cs, pos, slots, kc, vc


def _pair(qkv, HQ, HKV, D, qw, kw, cs, pos, slots, kc, vc):
    from xllm_b200 import ops
    T, qs, kvs = qkv.size(0), HQ * D, HKV * D
    ops.fused_qk_norm_rope(qkv, HQ, HKV, HKV, D, 1e-6, qw, kw, cs, False, pos)
    ops.reshape_paged_cache(slots, qkv[:, qs:qs + kvs].view(T, HKV, D), qkv[:, qs + kvs:].view(T, HKV, D), kc, vc)


def _fused(qkv, HQ, HKV, D, qw, kw, cs, pos, slots, kc, vc):
    from xllm_b200 import ops
    ops.qk_norm_rope_and_cache(qkv, HQ, HKV, D, 1e-6, qw, kw, cs, pos, slots, kc, vc)


HEADS = [(32, 8, 128), (16, 8, 128), (64, 8, 128), (8, 2, 64), (4, 1, 64)]


@pytest.mark.parametrize("T", [1, 3, 37, 4096])
@pytest.mark.parametrize("HQ,HKV,D", HEADS)
def test_qk_norm_rope_and_cache_matches_pair_and_oracle(HQ, HKV, D, T, built_lib):
    qkv, qw, kw, cs, pos, slots, kc, vc = _case(T, HQ, HKV, D, seed=T * 131 + HQ)
    dev = [t.to(DEV) for t in (qw, kw, cs, pos, slots)]
    a = [qkv.to(DEV), kc.to(DEV), vc.to(DEV)]
    b = [t.clone() for t in a]
    _pair(a[0], HQ, HKV, D, *dev[:4], dev[4], a[1], a[2])
    _fused(b[0], HQ, HKV, D, *dev[:4], dev[4], b[1], b[2])
    torch.cuda.synchronize()
    for name, x, y in zip(("qkv", "k_cache", "v_cache"), a, b):
        assert torch.equal(x, y), f"{name} differs from fused_qk_norm_rope + reshape_paged_cache"
    # cache rows of slots no token wrote are untouched
    written = torch.zeros(kc.shape[0] * BS, dtype=torch.bool)
    written[slots[slots >= 0].long()] = True
    for name, got, init in (("k_cache", b[1], kc), ("v_cache", b[2], vc)):
        g = got.cpu().view(-1, HKV * D)
        assert torch.equal(g[~written], init.view(-1, HKV * D)[~written]), f"{name}: an untouched row changed"
    ref = O.fused_qk_norm_rope(qkv, HQ, HKV, HKV, D, 1e-6, qw, kw, cs, False, pos)
    # the fp32 rotation x*c - y*s may contract to an FMA on the GPU and not in torch: the two differ by ~1e-7, which is
    # more than a bf16 ulp only for results below ~3e-5 (cancellation); measured on 24 of 25M elements at T = 4096
    assert_close_bf16(b[0], ref, ulps=1, atol=2.0 ** -18, what=f"qk_norm_rope_and_cache {HQ}/{HKV}x{D} T={T}")
    qs, kvs = HQ * D, HKV * D
    g = b[1].cpu().view(-1, HKV * D)
    live = slots >= 0
    assert torch.equal(g[slots[live].long()], b[0].cpu()[live, qs:qs + kvs]), "k_cache rows are not the normalised k"
    assert torch.equal(b[2].cpu().view(-1, HKV * D)[slots[live].long()], qkv[live, qs + kvs:]), "v_cache rows are not v"


def test_qk_norm_rope_and_cache_under_graph_capture(built_lib):
    HQ, HKV, D, T = 32, 8, 128, 37
    qkv, qw, kw, cs, pos, slots, kc, vc = _case(T, HQ, HKV, D, seed=5)
    dev = [t.to(DEV) for t in (qw, kw, cs, pos, slots)]
    a = [qkv.to(DEV), kc.to(DEV), vc.to(DEV)]
    b = [t.clone() for t in a]
    _fused(a[0], HQ, HKV, D, *dev[:4], dev[4], a[1], a[2])
    src = qkv.to(DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            _fused(b[0], HQ, HKV, D, *dev[:4], dev[4], b[1], b[2])
    torch.cuda.current_stream().wait_stream(s)
    b[0].copy_(src)
    graph.replay()
    torch.cuda.synchronize()
    for name, x, y in zip(("qkv", "k_cache", "v_cache"), a, b):
        assert torch.equal(x, y), f"{name}: graph replay differs from the eager launch"


def test_qk_norm_rope_and_cache_rejects_bad_arguments(built_lib):
    from xllm_b200 import ops
    from xllm_b200._lib import XllmB200Error
    qkv, qw, kw, cs, pos, slots, kc, vc = _case(3, 8, 2, 64, seed=1)
    d = [t.to(DEV) for t in (qkv, qw, kw, cs, pos, slots, kc, vc)]
    with pytest.raises(XllmB200Error, match="int64"):
        ops.qk_norm_rope_and_cache(d[0], 8, 2, 64, 1e-6, d[1], d[2], d[3], d[4].int(), d[5], d[6], d[7])
    with pytest.raises(XllmB200Error, match="full rotary"):
        ops.qk_norm_rope_and_cache(d[0], 8, 2, 64, 1e-6, d[1], d[2], d[3][:, :32], d[4], d[5], d[6], d[7])
    with pytest.raises(XllmB200Error, match="contiguous"):
        ops.qk_norm_rope_and_cache(d[0].t(), 8, 2, 64, 1e-6, d[1], d[2], d[3], d[4], d[5], d[6], d[7])
