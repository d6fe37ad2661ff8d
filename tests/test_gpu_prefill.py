"""GPU parity: prefill (ragged) and chunked-prefill (paged) attention on wgmma vs the oracle."""
import math

import pytest
import torch

from oracle import ops as O
from tests.util import assert_close_attention

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"


def _ragged_case(lens, HQ, HKV, D, seed=2026):
    g = torch.Generator().manual_seed(seed)
    T = sum(lens)
    qkv = torch.randn(T, (HQ + 2 * HKV) * D, generator=g).to(BF16)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0).tolist()), dtype=torch.int32)
    return qkv, cu


RAGGED = [
    ([128], 28, 4, 128), ([128, 128], 16, 8, 128), ([32, 64, 128], 16, 8, 128), ([2048], 28, 4, 128),
    ([1, 5, 300, 17], 28, 4, 128), ([333, 700], 14, 2, 64), ([257], 8, 8, 128), ([513, 40], 32, 2, 128), ([130], 4, 4, 64),
    ([2048, 2048], 28, 4, 128), ([4096], 32, 8, 128),
]


@pytest.mark.parametrize("lens,HQ,HKV,D", RAGGED)
def test_batch_prefill_ragged(lens, HQ, HKV, D, built_lib):
    from xllm_b200 import ops
    qkv, cu = _ragged_case(lens, HQ, HKV, D)
    T = qkv.shape[0]
    q = qkv[:, :HQ * D].reshape(T, HQ, D)
    k = qkv[:, HQ * D:(HQ + HKV) * D].reshape(T, HKV, D)
    v = qkv[:, (HQ + HKV) * D:].reshape(T, HKV, D)
    sc = 1.0 / math.sqrt(D)
    ref = O.ragged_prefill_attention(q, k, v, cu, cu, sc, causal=True)
    scale = O.ragged_prefill_attention(q, k, v.abs(), cu, cu, sc, causal=True)
    d = qkv.to(DEV)
    out = torch.empty(T, HQ, D, dtype=BF16, device=DEV)
    lse = torch.empty(T, HQ, dtype=torch.float32, device=DEV)
    ops.batch_prefill(d[:, :HQ * D].view(T, HQ, D), d[:, HQ * D:(HQ + HKV) * D].view(T, HKV, D),
                      d[:, (HQ + HKV) * D:].view(T, HKV, D), cu.to(DEV), cu.to(DEV), sc, out, lse, max_qo_len=max(lens))
    assert_close_attention(out, ref, scale, what=f"batch_prefill {lens}")
    # first token of every request attends only to itself: output == its V row bit-exactly
    for b in range(len(lens)):
        t0 = int(cu[b])
        assert torch.equal(out[t0].cpu(), v[t0].repeat_interleave(HQ // HKV, 0)), "token 0 must return its own V"


def _paged_case(q_lens, kv_lens, HQ, HKV, D, page, seed=7):
    g = torch.Generator().manual_seed(seed)
    B = len(q_lens)
    npages = [(n + page - 1) // page for n in kv_lens]
    total = sum(npages)
    nblocks = total + 4
    perm = (torch.randperm(nblocks - 1, generator=g) + 1)[:total].to(torch.int32)
    indptr = torch.tensor([0] + list(torch.tensor(npages).cumsum(0).tolist()), dtype=torch.int32)
    last = torch.tensor([(n - 1) % page + 1 for n in kv_lens], dtype=torch.int32)
    kc = torch.randn(nblocks, page, HKV, D, generator=g).to(BF16)
    vc = torch.randn(nblocks, page, HKV, D, generator=g).to(BF16)
    q = torch.randn(sum(q_lens), HQ, D, generator=g).to(BF16)
    qo = torch.tensor([0] + list(torch.tensor(q_lens).cumsum(0).tolist()), dtype=torch.int32)
    return q, kc, vc, qo, indptr, perm, last


PAGED = [
    # q_lens,            kv_lens,             HQ, HKV, D, page, causal
    ([128],              [128],               28, 4, 128, 128, True),
    ([64, 200, 1],       [300, 200, 77],      28, 4, 128, 16, True),     # chunked prefill: kv_len >= qo_len
    ([512],              [2048],              28, 4, 128, 128, True),
    ([100, 30],          [1000, 30],          14, 2, 64, 32, True),
    ([1, 1, 1],          [500, 17, 4096],     28, 4, 128, 128, False),   # decode on tensor cores (causal = False)
    ([9, 4, 1, 4],       [9, 8, 16, 8],       16, 8, 128, 4, True),      # the BatchTest.Basic batch (block_size 4)
    ([40],               [333],               32, 2, 128, 64, True),
]


@pytest.mark.parametrize("q_lens,kv_lens,HQ,HKV,D,page,causal", PAGED)
def test_batch_chunked_prefill_paged(q_lens, kv_lens, HQ, HKV, D, page, causal, built_lib):
    from xllm_b200 import ops
    q, kc, vc, qo, indptr, perm, last = _paged_case(q_lens, kv_lens, HQ, HKV, D, page)
    sc = 1.0 / math.sqrt(D)
    ref, ref_lse = O.paged_attention(q, kc, vc, qo, indptr, perm, last, sc, causal=causal, return_lse=True)
    scale = O.paged_attention(q, kc, vc.abs(), qo, indptr, perm, last, sc, causal=causal)
    out = torch.empty_like(q, device=DEV)
    lse = torch.empty(q.shape[0], HQ, dtype=torch.float32, device=DEV)
    ops.batch_chunked_prefill(q.to(DEV), kc.to(DEV), vc.to(DEV), indptr.to(DEV), perm.to(DEV), last.to(DEV), sc, out, lse,
                              qo.to(DEV), causal, max_qo_len=max(q_lens))
    assert_close_attention(out, ref, scale, what=f"batch_chunked_prefill q={q_lens} kv={kv_lens}")
    # l sums bf16-rounded P relative to the running maximum of the tile order: log2(l) moves by ~2^-9 / ln 2
    assert torch.allclose(lse.cpu(), ref_lse, rtol=1e-4, atol=5e-3), "base-2 LSE mismatch"


def test_prefill_decode_kernels_agree(built_lib):
    """the tensor-core paged kernel with q_len = 1 and the streaming decode kernel implement the same function."""
    from xllm_b200 import ops
    q, kc, vc, qo, indptr, perm, last = _paged_case([1, 1], [777, 4096], 28, 4, 128, 128)
    sc = 1.0 / math.sqrt(128)
    o1 = torch.empty_like(q, device=DEV)
    o2 = torch.empty_like(q, device=DEV)
    args = (kc.to(DEV), vc.to(DEV), indptr.to(DEV), perm.to(DEV), last.to(DEV))
    ops.batch_chunked_prefill(q.to(DEV), *args, sc, o1, None, qo.to(DEV), False, max_qo_len=1)
    plan = ops.DecodePlan(2, 28, 4, 128, 128, 32, DEV)
    ops.batch_decode(plan, q.to(DEV), *args, sc, o2)
    scale = O.paged_attention(q, kc, vc.abs(), qo, indptr, perm, last, sc, causal=False)
    assert_close_attention(o1, o2, scale, what="prefill-kernel decode vs decode kernel")


@pytest.mark.parametrize("q_lens,kv_lens,page", [([16], [4096], 128), ([64, 8, 1], [3000, 8192, 700], 16), ([128], [2048], 128)])
@pytest.mark.parametrize("splits", [2, 5, 8])
def test_chunked_prefill_split_kv_matches_oracle_and_unsplit(q_lens, kv_lens, page, splits, built_lib):
    """short query chunk over a long paged KV: the split-KV path (fp32 partials + merge kernel; the reference's planner
    splits the same cases, flashinfer_planinfo.cpp:168-247) against the oracle and against the unsplit kernel."""
    from xllm_b200 import ops
    HQ, HKV, D = 28, 4, 128
    g = torch.Generator().manual_seed(17)
    B = len(q_lens)
    npg = [(n + page - 1) // page for n in kv_lens]
    nblocks = sum(npg) + 3
    perm = (torch.randperm(nblocks - 1, generator=g) + 1)[:sum(npg)].to(torch.int32)
    indptr = torch.tensor([0] + list(torch.tensor(npg).cumsum(0).tolist()), dtype=torch.int32)
    last = torch.tensor([(n - 1) % page + 1 for n in kv_lens], dtype=torch.int32)
    qo = torch.tensor([0] + list(torch.tensor(q_lens).cumsum(0).tolist()), dtype=torch.int32)
    T = sum(q_lens)
    q = torch.randn(T, HQ, D, generator=g).to(BF16)
    kc = torch.randn(nblocks, page, HKV, D, generator=g).to(BF16)
    vc = torch.randn(nblocks, page, HKV, D, generator=g).to(BF16)
    sc = 1.0 / math.sqrt(D)
    ref, ref_lse = O.paged_attention(q, kc, vc, qo, indptr, perm, last, sc, causal=True, return_lse=True)
    scale = O.paged_attention(q, kc, vc.abs(), qo, indptr, perm, last, sc, causal=True)
    args = (q.to(DEV), kc.to(DEV), vc.to(DEV), indptr.to(DEV), perm.to(DEV), last.to(DEV), sc)
    out = torch.empty(T, HQ, D, dtype=BF16, device=DEV)
    lse = torch.empty(T, HQ, dtype=torch.float32, device=DEV)
    ops.batch_chunked_prefill(*args, out, lse, qo.to(DEV), True, max(q_lens), kv_splits=splits)
    base = torch.empty_like(out)
    ops.batch_chunked_prefill(*args, base, None, qo.to(DEV), True, max(q_lens))
    torch.cuda.synchronize()
    assert_close_attention(out, ref, scale, what=f"split-KV chunked prefill q={q_lens} kv={kv_lens} splits={splits}")
    assert_close_attention(out, base, scale, what="split vs unsplit kernel")
    assert torch.allclose(lse.cpu(), ref_lse, rtol=1e-4, atol=5e-3), "base-2 LSE of the merged result"


def test_prefill_plan_splits_rule(built_lib):
    from xllm_b200 import ops
    assert ops.prefill_plan_splits(1, 2048, 2048, 28, 4) == 1          # 112 q tiles x 4 heads: plenty of CTAs
    assert ops.prefill_plan_splits(1, 16, 8192, 28, 4) == 16           # 1 x 4 CTAs: min(132 / 4 = 33, 8192 / 512 = 16)
    assert ops.prefill_plan_splits(1, 16, 600, 28, 4) == 1             # short KV: not worth a merge pass
    assert ops.prefill_plan_splits(8, 18, 4096, 28, 4) == 4            # 8 x 4 = 32 CTAs -> 132 / 32 = 4
