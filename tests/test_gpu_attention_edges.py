"""Exact-answer probes of paged decode, ragged prefill, paged prefill and split-KV paged prefill attention, at the GQA
groups, page sizes and split / cluster geometries where an index or mask error hides from the random-data parity tests.

On N(0,1) data one extra or missing key moves an output by about |v| / kv_len, far inside the bf16-P tolerance of
tests/util.py at long context.  These probes make the right answer exact instead (float64 arithmetic on the probe's own
construction, no attention oracle):
  * needle: every visible key is 0 in the query's direction except one, K = BIG e_d, and the query is C e_d.  Its base-2
    score (260 or more) flushes every other weight to 0, so the output is that key's V row bit for bit, through any split
    or cluster merge.  Each head of a group gets its own direction and needle where D allows.
  * poison: every slot the kernel must not read (slack past last_page_len, unused blocks, block 0, other requests' keys,
    future tokens) scores higher still and carries V = +-1000, so any leak dominates the output.  Requests own disjoint
    query directions; a request's keys hold the poison value in every other request's directions.
  * count: with all visible scores 0 the base-2 LSE is log2(#visible keys) (to 1e-5: an off-by-one shows up to ~1e5
    keys) and the output is the mean of V.  V is integer-valued in [-8, 8], so the fp32 sums are exact: the output is
    within 1 bf16 ulp of the float64 mean, and bit-exact when nothing merges and the count is a power of two.
"""
import math

import numpy as np
import pytest
import torch

from tests.util import bf16_ulp

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
F32 = torch.float32
DEV = "cuda"

BIG = 64.0          # needle key value in its direction
C = 32.0            # query value in its direction: BIG * C * sm_scale * log2(e) >= 261 for D <= 128
POISON_K = 128.0    # unreadable keys: score 2 * BIG * C against every query
POISON_V = 1000.0
MERGE_ATOL = 2.0 ** -16   # fp32 rounding of the split weights when partial means are merged (|V| <= 8)
DECODE_ENV = ("XB_DECODE_CLUSTER", "XB_DECODE_PARTS", "XB_DECODE_WARPS", "XB_DECODE_CHUNK")


def _needle_lse(D):
    """base-2 score of the needle as the kernels form it: fp32(BIG * C) * fp32(fp32(sm_scale) * fp32(log2 e))."""
    scale_log2 = np.float32(np.float32(1.0 / math.sqrt(D)) * np.float32(1.44269504088896340736))
    return float(np.float32(BIG * C) * scale_log2)


def _dirs(B, G, D):
    """query directions per request: request b owns [b * nd, (b + 1) * nd), head h of a group uses b * nd + h % nd."""
    nd = max(1, min(G, D // B))
    assert B * nd <= D
    return nd


class _Layout:
    """paged KV layout: pages of every request are a random permutation of physical blocks 1.., block 0 and a few
    trailing blocks stay unused; rows[b][t] = physical row (block * page + slot) of token t of request b."""

    def __init__(self, kv_lens, page, g, extra=3):
        self.kv_lens, self.page = list(kv_lens), page
        self.npages = [(n + page - 1) // page for n in kv_lens]
        total = sum(self.npages)
        self.nblocks = total + 1 + extra
        self.indices = (torch.randperm(self.nblocks - 1, generator=g) + 1)[:total].to(torch.int32)
        self.indptr = torch.tensor([0] + np.cumsum(self.npages).tolist(), dtype=torch.int32)
        self.last = torch.tensor([(n - 1) % page + 1 if n > 0 else 0 for n in kv_lens], dtype=torch.int32)
        self.rows = []
        for b, n in enumerate(kv_lens):
            idx = self.indices[int(self.indptr[b]):int(self.indptr[b + 1])].long()
            t = torch.arange(n)
            self.rows.append(idx[t // page] * page + t % page)


def _kv_values(n_rows, valid_rows, HKV, D, g):
    """V: integers in [-8, 8] on the valid rows, +-1000 everywhere else."""
    sign = torch.where(torch.arange(D) % 2 == 0, 1.0, -1.0)
    v = (POISON_V * sign).expand(n_rows, HKV, D).clone()
    v[valid_rows] = torch.randint(-8, 9, (valid_rows.numel(), HKV, D), generator=g).float()
    return v


def _kv_keys(n_rows, rows_per_req, HKV, D, nd):
    """K without needles: POISON_K everywhere, and on a request's own rows 0 except in the other requests' directions."""
    k = torch.full((n_rows, HKV, D), POISON_K)
    B = len(rows_per_req)
    for b, rows in enumerate(rows_per_req):
        own = torch.full((D,), POISON_K)
        own[b * nd:(b + 1) * nd] = 0.0
        own[B * nd:] = 0.0                 # directions no request owns
        k[rows] = own
    return k


def _queries(q_lens, G, HKV, D, nd):
    """[sum(q_lens), HKV * G, D]: head h of every kv head of request b is C e_(b * nd + h % nd)."""
    q = torch.zeros(sum(q_lens), HKV, G, D)
    h = torch.arange(G)
    t0 = 0
    for b, n in enumerate(q_lens):
        q[t0:t0 + n, :, h, b * nd + h % nd] = C
        t0 += n
    return q.reshape(-1, HKV * G, D)


def _candidates(n, page, chunk=None, tile=None):
    """key positions where index arithmetic goes wrong: ends, page / 16-block / split-chunk / 128-tile boundaries +-1."""
    c = {0, 1, n - 1, n - 2}
    for step in {page, 16, chunk or 16, tile or 16}:
        ks = sorted({1, 2, n // step // 2, n // step - 1, n // step})
        for k in ks:
            c.update((k * step - 1, k * step, k * step + 1))
    return sorted(x for x in c if 0 <= x < n)


def _assert_probe(out, lse, exp_out, exp_lse, needle, exact, atol, what):
    """out [..., D] bf16 and lse [...] against float64 expectations.  needle: rows whose answer is one V row (bit-exact,
    LSE = the needle score); exact: mean rows that must match bit for bit; the other rows within 1 bf16 ulp + atol."""
    out, lse = out.cpu().float(), lse.cpu()
    ref = exp_out.to(BF16).float()
    assert torch.isfinite(out).all(), f"{what}: non-finite output (unwritten or poisoned rows)"
    bit = needle | exact
    if bit.any():
        bad = (out != ref).any(-1) & bit
        assert not bad.any(), (f"{what}: {int(bad.sum())} exact rows differ, first at {bad.nonzero()[0].tolist()}: "
                               f"got {out[bad][0, :4].tolist()} want {ref[bad][0, :4].tolist()}")
    err = (out.double() - exp_out).abs()
    bound = bf16_ulp(torch.maximum(exp_out.abs(), out.double().abs()).float()).double() + atol
    bad = (err > bound).any(-1)
    assert not bad.any(), (f"{what}: {int(bad.sum())} rows beyond 1 bf16 ulp of the float64 mean, first at "
                           f"{bad.nonzero()[0].tolist()}: worst |err| {err.max().item():.3e}")
    fin = torch.isfinite(exp_lse)
    assert torch.equal(torch.isfinite(lse), fin) and (lse[~fin] == -math.inf).all(), f"{what}: LSE finiteness differs"
    d = (lse.double() - exp_lse).abs()[fin]
    tol = torch.where(needle[fin], 1e-4, 1e-5)
    assert (d <= tol).all(), (f"{what}: base-2 LSE off by {d.max().item():.3e} (count rows resolve an off-by-one "
                              f"at 1e-5)")


# ================================================ decode ================================================

def _split_chunk(n, S):
    """the live split size paged_decode_kernel derives from kv_len and the launched split count (min_chunk 64)."""
    return max(64, ((n + S - 1) // S + 15) // 16 * 16) if S > 0 else n


def _clear_decode_env(monkeypatch, env):
    for k in DECODE_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, str(v))


def _decode_probe(kv_lens, G, HKV, D, page, *, num_sms=None, halves=False, seed=0, expect_cluster=None):
    """needle rounds until every candidate position of every request has been a needle, then the count probe; every
    geometry is launched twice on one workspace and must give the same bits."""
    from xllm_b200 import _lib, ops
    B, HQ = len(kv_lens), G * HKV
    g = torch.Generator().manual_seed(seed)
    lay = _Layout(kv_lens, page, g)
    nd = _dirs(B, G, D)
    n_rows = lay.nblocks * page
    rows_all = torch.cat(lay.rows) if sum(kv_lens) else torch.zeros(0, dtype=torch.long)
    V = _kv_values(n_rows, rows_all, HKV, D, g)
    K0 = _kv_keys(n_rows, lay.rows, HKV, D, nd)
    q = _queries([1] * B, G, HKV, D, nd).to(BF16).to(DEV)
    plan = ops.DecodePlan(B, HQ, HKV, D, page, max(lay.npages + [1]), DEV, num_sms=num_sms)
    S = plan.max_splits
    if halves:      # K and V as the two halves of one [blocks, 2, page, Hkv, D] tensor: page stride 2 * page * Hkv * D
        kv = torch.empty(lay.nblocks, 2, page, HKV, D, dtype=BF16, device=DEV)
        kc, vc = kv[:, 0], kv[:, 1]
    else:
        kc = torch.empty(lay.nblocks, page, HKV, D, dtype=BF16, device=DEV)
        vc = torch.empty_like(kc)
    vc.copy_(V.view(lay.nblocks, page, HKV, D))
    meta = (lay.indptr.to(DEV), lay.indices.to(DEV), lay.last.to(DEV))
    sc = 1.0 / math.sqrt(D)
    what = f"decode kv={kv_lens} G={G} Hkv={HKV} D={D} page={page} splits={S} cluster={plan.cluster}"

    def launch():
        res = []
        for _ in range(2):
            out = torch.full((B, HQ, D), float("nan"), dtype=BF16, device=DEV)
            lse = torch.full((B, HQ), float("nan"), dtype=F32, device=DEV)
            ops.batch_decode(plan, q, kc, vc, *meta, sc, out, lse)
            res.append((out, lse))
        torch.cuda.synchronize()
        if expect_cluster is not None:
            assert _lib.lib().xb_debug_last_decode_cluster() == expect_cluster, \
                f"{what}: launched cluster {_lib.lib().xb_debug_last_decode_cluster()}, planned {expect_cluster}"
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]), \
            f"{what}: relaunch on the same workspace changed the bits"
        return res[0][0].view(B, HKV, G, D), res[0][1].view(B, HKV, G)

    cands = [_candidates(n, page, _split_chunk(n, S)) for n in kv_lens]
    rounds = max([(len(c) + nd - 1) // nd for c in cands] + [1])
    h = torch.arange(G)
    s_needle = _needle_lse(D)
    Vr = [V[r].double() for r in lay.rows]          # [n, HKV, D] per request
    K0d = K0.view(lay.nblocks, page, HKV, D).to(BF16).to(DEV)
    for r in range(rounds):
        exp_out = torch.zeros(B, HKV, G, D, dtype=torch.float64)
        exp_lse = torch.full((B, HKV, G), -math.inf, dtype=torch.float64)
        at = []                                     # (physical row, kv head, direction) of every needle
        for b, n in enumerate(kv_lens):
            if n == 0:
                continue
            for kvh in range(HKV):
                js = torch.tensor([cands[b][(r * nd + s + kvh * 5) % len(cands[b])] for s in range(nd)])
                at.append(torch.stack([lay.rows[b][js], torch.full((nd,), kvh), b * nd + torch.arange(nd)]))
                exp_out[b, kvh] = Vr[b][js[h % nd], kvh]
                exp_lse[b, kvh] = s_needle
        kc.copy_(K0d)
        if at:
            row, kvh_i, d_i = torch.cat(at, 1).to(DEV)
            kc[row // page, row % page, kvh_i, d_i] = BIG
        out, lse = launch()
        needle = torch.isfinite(exp_lse)
        _assert_probe(out, lse, exp_out, exp_lse, needle, ~needle, 0.0, f"{what} needle round {r}")
    # count probe
    kc.copy_(K0d)
    out, lse = launch()
    exp_out = torch.zeros(B, HKV, G, D, dtype=torch.float64)
    exp_lse = torch.full((B, HKV, G), -math.inf, dtype=torch.float64)
    exact = torch.zeros(B, HKV, G, dtype=torch.bool)
    for b, n in enumerate(kv_lens):
        if n == 0:
            exact[b] = True             # empty request: output 0, LSE -inf, as the oracle defines it
            continue
        exp_out[b] = Vr[b].mean(0)[:, None, :]
        exp_lse[b] = math.log2(n)
        single = (n + _split_chunk(n, S) - 1) // _split_chunk(n, S) <= 1
        exact[b] = single and (n & (n - 1)) == 0
    merged = S > 1
    _assert_probe(out, lse, exp_out, exp_lse, torch.zeros_like(exact), exact, MERGE_ATOL if merged else 0.0,
                  f"{what} count")
    return plan


PAGES = (1, 3, 16, 48, 128, 256)
GROUPS = (1, 3, 5, 6, 7, 8, 12, 16, 20, 24, 48, 128)


def _group_cases():
    cases = []
    for i, (G, D) in enumerate((G, D) for G in GROUPS for D in (64, 128)):
        k = 10 + 17 * i
        lens = [16 * k - 1, 16 * k, 16 * k + 1]
        if i % 3 == 0:
            lens.insert(1, 0)           # an empty request inside a batch with splits
        cases.append((lens, G, 2 if G <= 24 else 1, D, PAGES[i % len(PAGES)]))
    return cases


@pytest.mark.parametrize("kv_lens,G,HKV,D,page", _group_cases())
def test_decode_probes_groups_pages(kv_lens, G, HKV, D, page, monkeypatch, built_lib):
    _clear_decode_env(monkeypatch, None)
    plan = _decode_probe(kv_lens, G, HKV, D, page)
    assert plan.max_splits > 1, "every geometry here must merge splits"


@pytest.mark.parametrize("kv_lens,G,HKV,D,page,num_sms,splits", [
    ([16 * 1024 + 17], 8, 1, 128, 16, 1 << 20, 256),      # the 2 * head_dim cap: 4 batches of 64 per team lane
    ([8200, 5000], 5, 1, 64, 48, 1 << 20, 128),           # cap at D = 64, one request with idle splits
    ([6500], 16, 1, 128, 128, 100, 100),                  # 100 partials: a second, partly filled batch
    ([4400, 33], 20, 1, 128, 3, 4 * 70, 69),              # two head tiles, 69 splits (the 64-token floor of by_len)
    ([4160, 0, 4100], 7, 1, 128, 256, 3 * 65, 65),        # one past 64
])
def test_decode_probes_team_merge_beyond_64(kv_lens, G, HKV, D, page, num_sms, splits, monkeypatch, built_lib):
    _clear_decode_env(monkeypatch, None)
    plan = _decode_probe(kv_lens, G, HKV, D, page, num_sms=num_sms)
    assert plan.max_splits == splits and plan.cluster == 1


# (env, kv_lens, G, HKV, D, page, num_sms, cluster, splits); units = len(kv_lens) * HKV * head tiles, want = num_sms / units
CLUSTER_CASES = [
    ({"XB_DECODE_CLUSTER": 2}, [3000, 900], 4, 2, 128, 16, 4 * 2, 2, 2),                # one cluster of 2
    ({"XB_DECODE_CLUSTER": 2}, [3000, 900], 4, 2, 128, 16, 4 * 10, 2, 10),              # five clusters of 2
    ({"XB_DECODE_CLUSTER": 8}, [3000, 1], 8, 1, 128, 128, 2 * 8, 8, 8),                 # one cluster of 8
    ({"XB_DECODE_CLUSTER": 8}, [3000, 1000], 6, 1, 64, 48, 2 * 24, 8, 24),              # three clusters of 8
    ({"XB_DECODE_CLUSTER": 16}, [4000], 7, 2, 128, 16, 2 * 16, 16, 16),                 # one cluster of 16
    ({"XB_DECODE_CLUSTER": 16}, [9000, 5000], 5, 1, 128, 256, 2 * 64, 16, 64),          # four clusters of 16
    ({"XB_DECODE_CLUSTER": 16, "XB_DECODE_PARTS": 2}, [4000], 7, 2, 128, 1, 2 * 16, 8, 16),   # forced: two of 8
    ({"XB_DECODE_CLUSTER": 16, "XB_DECODE_PARTS": 3}, [6000, 2], 3, 1, 64, 16, 2 * 48, 16, 48),  # forced: three of 16
    ({"XB_DECODE_CLUSTER": 16}, [3000], 12, 1, 64, 16, 1 * 16, 16, 16),                 # group 12: 16-head CTAs
    ({"XB_DECODE_CLUSTER": 8}, [5000, 700], 24, 1, 128, 16, 2 * 2 * 16, 8, 16),         # group 24: two head tiles
    ({"XB_DECODE_CLUSTER": 8, "XB_DECODE_WARPS": 4}, [3000], 7, 1, 128, 16, 16, 8, 16),  # 4-warp CTAs in clusters
]


@pytest.mark.parametrize("env,kv_lens,G,HKV,D,page,num_sms,cluster,splits", CLUSTER_CASES)
def test_decode_probes_cluster_merge(env, kv_lens, G, HKV, D, page, num_sms, cluster, splits, monkeypatch, built_lib):
    """splits merged through distributed shared memory; the launched cluster size is asserted, so a fall-back to
    per-CTA partials (cluster 1) fails instead of passing as the plain path."""
    _clear_decode_env(monkeypatch, env)
    plan = _decode_probe(kv_lens, G, HKV, D, page, num_sms=num_sms, expect_cluster=cluster)
    assert (plan.cluster, plan.max_splits) == (cluster, splits)


@pytest.mark.parametrize("env,kv_lens,G,HKV,D,page", [
    ({"XB_DECODE_WARPS": 4}, [2000, 47, 0], 7, 2, 128, 16),
    ({"XB_DECODE_WARPS": 4}, [1500, 1], 16, 1, 64, 3),
    ({"XB_DECODE_WARPS": 4}, [3000], 24, 1, 128, 128),
    ({"XB_DECODE_CHUNK": 16}, [1000, 64, 65], 5, 1, 128, 16),     # nominal 16: the kernel's 64-token floor applies
    ({"XB_DECODE_CHUNK": 200}, [3000, 191, 193], 6, 2, 64, 48),
])
def test_decode_probes_warps_and_chunk(env, kv_lens, G, HKV, D, page, monkeypatch, built_lib):
    _clear_decode_env(monkeypatch, env)
    _decode_probe(kv_lens, G, HKV, D, page)


@pytest.mark.parametrize("kv_lens,G,HKV,D,page", [([700, 4096, 1], 7, 4, 128, 16), ([300, 129], 6, 2, 64, 128)])
def test_decode_probes_kv_halves_of_one_tensor(kv_lens, G, HKV, D, page, monkeypatch, built_lib):
    """K and V as views [:, 0] / [:, 1] of one [blocks, 2, page, Hkv, D] tensor (a page stride of 2 * page * Hkv * D)."""
    _clear_decode_env(monkeypatch, None)
    _decode_probe(kv_lens, G, HKV, D, page, halves=True)


@pytest.mark.parametrize("HQ,HKV,D,page,kv_lens", [(28, 4, 128, 16, [300, 17, 4096, 1]), (12, 2, 64, 128, [129, 2000]),
                                                   (40, 8, 128, 16, [64, 65])])
def test_decode_product_step(HQ, HKV, D, page, kv_lens, monkeypatch, built_lib):
    """what a decode step runs per layer: rope_and_cache writes the newest token of every request, then, on the same
    stream with PDL on, batch_decode with an early-prefetch plan reads q as a strided slice of the packed qkv and writes
    a view of a wider buffer.  The newest key is the needle, so the output must be the newest V row exactly; a block
    prefetched before the write would hold the stale slot (poison).  The plain plan must agree bit for bit."""
    from xllm_b200 import _lib, ops
    from oracle import ops as O
    _clear_decode_env(monkeypatch, None)
    _lib.set_pdl(True)
    B, G = len(kv_lens), HQ // HKV
    g = torch.Generator().manual_seed(11)
    lay = _Layout(kv_lens, page, g)
    nd = _dirs(B, G, D)
    n_rows = lay.nblocks * page
    old = [r[:-1] for r in lay.rows]
    V = _kv_values(n_rows, torch.cat(old), HKV, D, g)
    K = _kv_keys(n_rows, old, HKV, D, nd)              # the newest slots keep the poison until rope_and_cache writes them
    kc = K.view(lay.nblocks, page, HKV, D).to(BF16).to(DEV)
    vc = V.view(lay.nblocks, page, HKV, D).to(BF16).to(DEV)
    q_size, kv_size = HQ * D, HKV * D
    qkv = torch.zeros(B, q_size + 2 * kv_size)
    qkv[:, :q_size] = _queries([1] * B, G, HKV, D, nd).reshape(B, -1)
    knew = torch.zeros(B, HKV, D)
    for b in range(B):
        knew[b, :, b * nd:(b + 1) * nd] = BIG
    vnew = torch.randint(-8, 9, (B, HKV, D), generator=g).float()
    qkv[:, q_size:q_size + kv_size] = knew.reshape(B, -1)
    qkv[:, q_size + kv_size:] = vnew.reshape(B, -1)
    qkv = qkv.to(BF16).to(DEV)
    # position 0 makes RoPE the identity, so q and the new key stay on their probe directions; the slot written is
    # still each request's newest one
    positions = torch.zeros(B, dtype=torch.int64, device=DEV)
    slots = torch.stack([r[-1] for r in lay.rows]).to(torch.int32).to(DEV)
    cs = O.compute_cos_sin_cache(D, 64, 1000000, BF16).to(DEV)
    wide = torch.full((B, q_size + 64), 7.0, dtype=BF16, device=DEV)
    out = wide[:, :q_size].view(B, HQ, D)
    plan = ops.DecodePlan(B, HQ, HKV, D, page, max(lay.npages), DEV, early_prefetch=True)
    meta = (lay.indptr.to(DEV), lay.indices.to(DEV), lay.last.to(DEV))
    sc = D ** -0.5
    torch.cuda.synchronize()
    ops.rope_and_cache(positions, qkv[:, :q_size], qkv[:, q_size:q_size + kv_size], qkv[:, q_size + kv_size:], cs, slots,
                       kc, vc, True)
    ops.batch_decode(plan, qkv[:, :q_size].view(-1, HQ, D), kc, vc, *meta, sc, out)
    torch.cuda.synchronize()
    exp = vnew[:, :, None, :].expand(B, HKV, G, D).reshape(B, HQ, D).to(BF16)
    got = out.cpu()
    bad = (got != exp).any(-1)
    assert not bad.any(), f"early-prefetch decode after rope_and_cache: {int(bad.sum())} heads are not the newest V row"
    assert (wide[:, q_size:] == 7.0).all(), "wrote past the output view"
    plain = ops.DecodePlan(B, HQ, HKV, D, page, max(lay.npages), DEV)
    out2 = torch.empty(B, HQ, D, dtype=BF16, device=DEV)
    ops.batch_decode(plain, qkv[:, :q_size].view(-1, HQ, D), kc, vc, *meta, sc, out2)
    assert torch.equal(out2, out), "early-prefetch and plain plans disagree on the same inputs"


def test_batch_decode_rejects_inputs_that_do_not_match_the_plan(monkeypatch, built_lib):
    """every bad case raises before launch and leaves the output untouched; the valid call still computes."""
    from xllm_b200 import ops
    from xllm_b200._lib import XllmB200Error
    _clear_decode_env(monkeypatch, None)
    B, HQ, HKV, D, page, nb = 2, 8, 2, 64, 16, 6
    plan = ops.DecodePlan(B, HQ, HKV, D, page, 2, DEV)
    kc = torch.randn(nb, page, HKV, D, device=DEV).to(BF16)
    vc = torch.randn(nb, page, HKV, D, device=DEV).to(BF16)
    q = torch.randn(B, HQ, D, device=DEV).to(BF16)
    meta = (torch.tensor([0, 2, 3], dtype=torch.int32, device=DEV), torch.tensor([1, 2, 3], dtype=torch.int32, device=DEV),
            torch.tensor([5, 16], dtype=torch.int32, device=DEV))
    out = torch.full((B, HQ, D), 3.0, dtype=BF16, device=DEV)

    def strided_last(t):            # same shape, last dimension with stride 2
        return torch.empty(*t.shape, 2, dtype=BF16, device=DEV)[..., 0].copy_(t)

    v_other_layout = torch.empty(nb, HKV, page, D, dtype=BF16, device=DEV).transpose(1, 2).copy_(vc)
    kv_halves = torch.empty(nb, 2, page, HKV, D, dtype=BF16, device=DEV)
    bad = {
        "v strides differ from k (other layout)": (q, kc, v_other_layout, out),
        "v strides differ from k (half of a kv tensor)": (q, kc, kv_halves[:, 1], out),
        "k strides differ from v (half of a kv tensor)": (q, kv_halves[:, 0], vc, out),
        "q last dim strided": (strided_last(q), kc, vc, out),
        "cache last dim strided": (q, strided_last(kc), strided_last(vc), out),
        "q with fewer rows than the plan": (q[:1], kc, vc, out),
        "q with more rows than the plan": (torch.cat([q, q]), kc, vc, out),
        "q with other head count": (q[:, :HQ - 1], kc, vc, out),
        "q head_dim 128": (torch.zeros(B, HQ, 128, dtype=BF16, device=DEV), kc, vc, out),
        "cache page 128 for a page-16 plan": (q, torch.zeros(1, 128, HKV, D, dtype=BF16, device=DEV),
                                              torch.zeros(1, 128, HKV, D, dtype=BF16, device=DEV), out),
        "cache with other kv head count": (q, kc[:, :, :1], vc[:, :, :1], out),
        "v with fewer blocks than k": (q, kc, vc[:-1], out),
        "cache without block dimension": (q, kc[0], vc[0], out),
    }
    for name, (qq, kk, vv, oo) in bad.items():
        with pytest.raises(XllmB200Error):
            ops.batch_decode(plan, qq, kk, vv, *meta, 0.125, oo)
        torch.cuda.synchronize()
        assert (out == 3.0).all(), f"{name}: rejected call wrote the output"
    out_strided = strided_last(out)
    with pytest.raises(XllmB200Error):
        ops.batch_decode(plan, q, kc, vc, *meta, 0.125, out_strided)
    with pytest.raises(XllmB200Error):
        ops.batch_decode(plan, q, kc, vc, *meta, 0.125, out[:1])
    torch.cuda.synchronize()
    assert (out == 3.0).all() and (out_strided == 3.0).all()
    ops.batch_decode(plan, q, kc, vc, *meta, 0.125, out)
    torch.cuda.synchronize()
    assert not (out == 3.0).all(), "the valid call must compute"


# ================================================ prefill ================================================

def _prefill_expected(q_lens, kv_lens, G, HKV, D, nd, needles, V_req, causal):
    """per request: [q_len, HKV, G, D] float64 output, [q_len, HKV, G] LSE and the needle-row mask."""
    s_needle = _needle_lse(D)
    h = torch.arange(G)
    res = []
    for b, (nq, nk) in enumerate(zip(q_lens, kv_lens)):
        if nq == 0:
            res.append((torch.zeros(0, HKV, G, D, dtype=torch.float64), torch.zeros(0, HKV, G, dtype=torch.float64),
                        torch.zeros(0, HKV, G, dtype=torch.bool), torch.zeros(0, dtype=torch.long)))
            continue
        off = nk - nq
        lims = (torch.arange(nq) + off + 1).clamp(max=nk) if causal else torch.full((nq,), nk)
        assert (lims >= 1).all()
        Vb = V_req[b]                                            # [nk, HKV, D]
        mean = Vb.cumsum(0)[lims - 1] / lims[:, None, None]      # [nq, HKV, D]
        js = needles[b][:, h % nd]                               # [HKV, G]
        vis = js[None] < lims[:, None, None]                     # [nq, HKV, G]
        nv = Vb[js, torch.arange(HKV)[:, None]]                  # [HKV, G, D]
        out = torch.where(vis[..., None], nv[None], mean[:, :, None, :])
        lse = torch.where(vis, s_needle, torch.log2(lims.double())[:, None, None].expand(nq, HKV, G))
        res.append((out, lse, vis, lims))
    return res


def _prefill_needles(kv_lens, HKV, nd, page, tpt, g):
    """[HKV, nd] needle positions per request: boundary candidates, different for every kv head and direction."""
    out = []
    for n in kv_lens:
        c = _candidates(n, page, tpt, 128) or [0]
        pick = torch.randperm(max(len(c), HKV * nd), generator=g)[:HKV * nd] % len(c)
        out.append(torch.tensor(c)[pick].view(HKV, nd))
    return out


def _prefill_probe(q_lens, kv_lens, G, HKV, D, *, causal=True, page=None, kv_splits=1, seed=0):
    """page None: ragged batch_prefill (K / V rows of all requests back to back); else paged batch_chunked_prefill."""
    from xllm_b200 import ops
    B, HQ = len(q_lens), G * HKV
    tpt = 128 // G
    g = torch.Generator().manual_seed(seed)
    nd = _dirs(B, G, D)
    if page is None:
        cu_kv = np.cumsum([0] + list(kv_lens))
        rows = [torch.arange(int(cu_kv[b]), int(cu_kv[b + 1])) for b in range(B)]
        n_rows = int(cu_kv[-1])
    else:
        lay = _Layout(kv_lens, page, g)
        rows, n_rows = lay.rows, lay.nblocks * page
    V = _kv_values(n_rows, torch.cat(rows), HKV, D, g)
    K = _kv_keys(n_rows, rows, HKV, D, nd)
    needles = _prefill_needles(kv_lens, HKV, nd, page or 16, tpt, g)
    for b in range(B):
        for kvh in range(HKV):
            if kv_lens[b]:
                K[rows[b][needles[b][kvh]], kvh, b * nd + torch.arange(nd)] = BIG
    q = _queries(q_lens, G, HKV, D, nd).to(BF16).to(DEV)
    T = q.shape[0]
    out = torch.full((T, HQ, D), float("nan"), dtype=BF16, device=DEV)
    lse = torch.full((T, HQ), float("nan"), dtype=F32, device=DEV)
    qo = torch.tensor(np.cumsum([0] + list(q_lens)), dtype=torch.int32, device=DEV)
    sc = 1.0 / math.sqrt(D)
    kind = "ragged" if page is None else f"paged page={page} splits={kv_splits}"
    what = f"prefill {kind} q={q_lens} kv={kv_lens} G={G} Hkv={HKV} D={D} causal={causal}"
    if page is None:
        kvc = torch.tensor(cu_kv, dtype=torch.int32, device=DEV)
        ops.batch_prefill(q, K.to(BF16).to(DEV), V.to(BF16).to(DEV), qo, kvc, sc, out, lse, max_qo_len=max(q_lens),
                          causal=causal)
    else:
        shape = (lay.nblocks, page, HKV, D)
        ops.batch_chunked_prefill(q, K.view(shape).to(BF16).to(DEV), V.view(shape).to(BF16).to(DEV), lay.indptr.to(DEV),
                                  lay.indices.to(DEV), lay.last.to(DEV), sc, out, lse, qo, causal, max(q_lens),
                                  kv_splits=kv_splits)
    torch.cuda.synchronize()
    exp = _prefill_expected(q_lens, kv_lens, G, HKV, D, nd, needles, [V[r].double() for r in rows], causal)
    exp_out = torch.cat([e[0] for e in exp])
    exp_lse = torch.cat([e[1] for e in exp])
    needle = torch.cat([e[2] for e in exp])
    lims = torch.cat([e[3] for e in exp])[:, None, None].expand_as(needle)
    exact = ((lims & (lims - 1)) == 0) if kv_splits == 1 else torch.zeros_like(needle)
    _assert_probe(out.view(T, HKV, G, D), lse.view(T, HKV, G), exp_out, exp_lse, needle, exact,
                  MERGE_ATOL if kv_splits > 1 else 0.0, what)


PREFILL_GROUPS = (3, 5, 6, 8, 12, 24, 32, 48, 64, 96, 128)


def _tile_lens(G):
    tpt = 128 // G
    return [tpt - 1, tpt, tpt + 1, 2 * tpt]


@pytest.mark.parametrize("G", PREFILL_GROUPS)
def test_prefill_probes_groups_ragged(G, built_lib):
    """q lengths one below, at and one above the tokens a q tile packs (128 // group), and two tiles; kv_len = q_len
    and kv_len > q_len (end-aligned causal: offsets 126, 3, 200 put a first-row limit 1 below a 128-key tile edge)."""
    D = 128 if PREFILL_GROUPS.index(G) % 2 == 0 else 64
    HKV = 2 if G <= 24 else 1
    q_lens = _tile_lens(G)
    _prefill_probe(q_lens, q_lens, G, HKV, D, seed=G)
    _prefill_probe(q_lens, [n + o for n, o in zip(q_lens, (126, 0, 3, 200))], G, HKV, D, seed=G + 1)


@pytest.mark.parametrize("G", PREFILL_GROUPS)
def test_prefill_probes_groups_paged(G, built_lib):
    D = 64 if PREFILL_GROUPS.index(G) % 2 == 0 else 128
    HKV = 2 if G <= 24 else 1
    q_lens = _tile_lens(G)
    pages = (1, 2, 8, 16, 128, 256, 512)
    page = pages[PREFILL_GROUPS.index(G) % len(pages)]
    _prefill_probe(q_lens, [n + o for n, o in zip(q_lens, (300, 126, 0, 129))], G, HKV, D, page=page, seed=G + 2)


@pytest.mark.parametrize("G,HKV,D", [(7, 4, 128), (5, 1, 64), (1, 2, 128)])
def test_prefill_probes_ragged_long_kv_and_noncausal(G, HKV, D, built_lib):
    q_lens = [1, 130, 40, 300]
    kv_lens = [700, 130, 40 + 126, 1000]
    _prefill_probe(q_lens, kv_lens, G, HKV, D, causal=True, seed=3)
    _prefill_probe(q_lens, kv_lens, G, HKV, D, causal=False, seed=4)
    _prefill_probe([17, 5], [17, 300], G, HKV, D, causal=False, seed=5)


@pytest.mark.parametrize("page", [1, 2, 8, 256, 512])
@pytest.mark.parametrize("causal", [True, False])
def test_prefill_probes_paged_page_sizes(page, causal, built_lib):
    """pages that divide 128 (several TMA boxes per tile) and pages above 128 (tile rows at t0 % page inside a page)."""
    _prefill_probe([40, 1, 128], [1300, 700, 128 + 126], 7, 2, 128, causal=causal, page=page, seed=page)


@pytest.mark.parametrize("G", [5, 16])
@pytest.mark.parametrize("splits_from_tiles", [-1, 0, 1, None])
def test_prefill_probes_split_kv(G, splits_from_tiles, built_lib):
    """split-KV counts around the number of 128-key tiles of the longest request (8 here), and 64: splits past the tile
    count get no tiles and must merge as empty partials."""
    kv_lens = [1000, 700, 129]
    n_tiles = (max(kv_lens) + 127) // 128
    splits = 64 if splits_from_tiles is None else n_tiles + splits_from_tiles
    tpt = 128 // G
    _prefill_probe([tpt, 3, 1], kv_lens, G, 2, 128, page=16, kv_splits=splits, seed=splits)
    _prefill_probe([2 * tpt + 1, 1, 129], kv_lens, G, 1, 64, page=16, kv_splits=splits, seed=splits + 1)
