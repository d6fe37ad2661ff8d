"""The NVLink exchange kernels (csrc/allreduce.cu) on ONE GPU, with every rank of a world emulated on the same device.

The kernels see their peers only through two host arrays of device pointers, peer_data[r] and peer_flags[r].  Here those
name W ordinary buffers of this device, and the exchange is launched once as each rank in turn, one launch after the other
on one stream (never concurrently).  That runs everything but the waiting half of the barrier and cross-GPU visibility,
which stay with tests/test_gpu_tp.py under torchrun: the fixed-order fp32 sum and its one rounding, bit-identity across
calling ranks, the fused residual add + RMSNorm, which flag slot each CTA signals, the epoch kept in device memory for
CUDA-graph replays, and the grid capped at max_ctas.

Emulated world: W partial buffers; per rank an `out`, a `residual` and an epoch array; and for every launch (calling rank r)
its own W signal pads pads[r][p], each [slots][8] int32, so that no launch ever reads a slot another launch wrote.

Hang-proof arming.  A launch spins only while (int32)(flag - target) < 0, where target = epoch[b] + 1.  Right before every
launch as rank r, all of pads[r] (guard rows included) is filled with ARMED = e0 + 2^30, e0 being the launch's starting
epoch, and the launch holds no pointer to any other pad.  The launch writes only `target` into slots, so every slot it can
wait on holds either ARMED (>= target) or the target it just wrote itself, whatever store or load index the kernel uses.
Guard epoch entries hold SENTINEL(b) = e0 + 2^29 + b, whose targets are below ARMED too.  e0 = -2 makes the targets cross
2^32 (-1, 0, 1 over three graph replays), exercising the signed comparison.

Guard room.  Epoch arrays and pads have GUARD entries past max_ctas, as many as the uncapped grid of the largest exchange
here (64 tokens x 16384 = 256 CTAs of 4096 elements): a CTA launched past the cap changes a sentinel instead of writing
out of bounds.
"""
import ctypes

import pytest
import torch

from oracle import ops as O
from tests.util import bf16_ulp

pytestmark = pytest.mark.gpu
BF16, I16, I32, F32 = torch.bfloat16, torch.int16, torch.int32, torch.float32
DEV = "cuda"
MAX_CTAS = 64                     # PeerExchange.MAX_CTAS
GUARD = 64 * 16384 // (8 * 512)    # the uncapped grid of the largest exchange here
TAIL = 64                         # sentinel elements past numel
EPS = 1e-6
OUT_SENTINEL = 0x7FA5             # a NaN bit pattern no exchange produces


def i32(v):
    return (v + 2 ** 31) % 2 ** 32 - 2 ** 31


E0 = i32(-2)
ARMED = i32(E0 + 2 ** 30)


def sentinel(b):
    return i32(E0 + 2 ** 29 + b)


@pytest.fixture(scope="module")
def L(built_lib):
    from xllm_b200 import _lib
    return _lib.lib()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _vp(t):
    return ctypes.c_void_p(t.data_ptr())


def bits(t):
    return t.detach().cpu().contiguous().view(I16)


def sentinel_bf16(*shape):
    return torch.full(shape, OUT_SENTINEL, dtype=I16, device=DEV).view(BF16)


class World:
    """Epochs and signal pads of W emulated ranks (see the module docstring)."""

    def __init__(self, W, max_ctas=MAX_CTAS):
        self.W, self.max_ctas, self.slots = W, max_ctas, max_ctas + GUARD
        self.pads = torch.empty(W, W, self.slots, 8, dtype=I32, device=DEV)    # pads[r][p]: peer p's pad as launch r sees it
        self.epoch = self.initial_epoch().to(DEV).expand(W, -1).contiguous()
        self.pads.fill_(ARMED)

    def initial_epoch(self):
        e = torch.full((self.slots,), E0, dtype=I32)
        e[self.max_ctas:] = torch.tensor([sentinel(b) for b in range(self.max_ctas, self.slots)], dtype=I32)
        return e

    def peers(self, r, data, world=None):
        """ctypes arrays of the partial buffers data[p] and of launch r's pads (W entries, or `world` for a bad world)."""
        n = world if world is not None and world > 0 else self.W
        pd = (ctypes.c_void_p * n)(*[data[p % self.W].data_ptr() for p in range(n)])
        pf = (ctypes.c_void_p * n)(*[self.pads[r, p % self.W].data_ptr() for p in range(n)])
        return pd, pf

    def oneshot(self, L, r, out, data, numel, world=None, max_ctas=None, rank=None):
        self.pads[r].fill_(ARMED)
        pd, pf = self.peers(r, data, world)
        return L.xb_oneshot_allreduce_bf16(_vp(out), pd, pf, _vp(self.epoch[r]), ctypes.c_int(r if rank is None else rank),
                                           ctypes.c_int(self.W if world is None else world), ctypes.c_int64(numel),
                                           ctypes.c_int(self.max_ctas if max_ctas is None else max_ctas), _stream())

    def fused(self, L, r, out, residual, weight, data, tokens, hidden, world=None, rank=None):
        self.pads[r].fill_(ARMED)
        pd, pf = self.peers(r, data, world)
        return L.xb_allreduce_add_rms_norm_bf16(_vp(out), _vp(residual), _vp(weight), pd, pf, _vp(self.epoch[r]),
                                                ctypes.c_int(r if rank is None else rank),
                                                ctypes.c_int(self.W if world is None else world), ctypes.c_float(EPS),
                                                ctypes.c_int(tokens), ctypes.c_int(hidden), ctypes.c_int(self.max_ctas),
                                                _stream())

    def check_signals(self, r, ctas, k=1):
        """after k exchanges as rank r with `ctas` CTAs: epoch[b] advanced by k for exactly those CTAs, slot pads[r][p][b][r]
        holds e0 + k for every peer p and launched b, and every other slot of launch r's pads still holds ARMED."""
        torch.cuda.synchronize()
        want_e = self.initial_epoch()
        want_e[:ctas] = i32(E0 + k)
        got_e = self.epoch[r].cpu()
        bad = (got_e != want_e).nonzero().flatten().tolist()
        assert not bad, f"rank {r}: epoch entries {bad[:8]} hold {got_e[bad[:8]].tolist()}, want {want_e[bad[:8]].tolist()}"
        want_p = torch.full((self.W, self.slots, 8), ARMED, dtype=I32)
        want_p[:, :ctas, r] = i32(E0 + k)
        got_p = self.pads[r].cpu()
        bad = (got_p != want_p).nonzero().tolist()
        assert not bad, (f"rank {r}: {len(bad)} signal slots wrong, first [peer, cta, column] {bad[:4]} hold "
                         f"{[got_p[tuple(i)].item() for i in bad[:4]]}")


def seq_sum(parts, order=None):
    """fp32 sum over ranks in `order` (default 0..W-1) starting from +0.0, as the kernel sums: never torch.sum."""
    acc = torch.zeros(parts.shape[1:], dtype=F32)
    for r in (range(parts.shape[0]) if order is None else order):
        acc = acc + parts[r].float()
    return acc


def assert_sum_bound(got, parts):
    """|bf16 result - float64 sum| <= half a bf16 ulp + W * 2^-24 * sum |p_r| (fp32 accumulation, then one rounding)."""
    p = parts.double()
    err = (got.double() - p.sum(0)).abs()
    tol = 0.5 * bf16_ulp(got).double() + parts.shape[0] * 2.0 ** -24 * p.abs().sum(0)
    assert (err <= tol).all(), f"{int((err > tol).sum())} elements beyond the float64 bound, worst {(err - tol).max():.3e}"


def assert_norm_close(got, s, res, w):
    """`got` against the oracle's fused_add_rms_norm(s, res, w): within one bf16 ulp, plus one ulp of bf16(z * rstd) times
    the weight.  The oracle sums the squares in torch's order, so its rstd can differ in the last bit and move that
    intermediate rounding by one ulp, which the weight then scales (observed: 2 output ulps).  The strict check of the
    fused kernel's norm is its bit-identity to the library's composition."""
    ref, _ = O.fused_add_rms_norm(s, res, w, EPS)
    normed, _ = O.fused_add_rms_norm(s, res, torch.ones_like(w), EPS)      # bf16(z * rstd): a weight of 1 is exact
    err = (got.float() - ref.float()).abs()
    tol = torch.maximum(bf16_ulp(ref), bf16_ulp(got)) + w.float().abs() * bf16_ulp(normed)
    assert (err <= tol).all(), f"out beyond the oracle's bound at {int((err > tol).sum())} elements, worst {err.max().item():.3e}"


def _partials(W, shape, seed):
    g = torch.Generator().manual_seed(seed)
    scale = torch.exp2(torch.randint(-6, 7, (W,) + tuple(shape), generator=g).float())
    return (torch.randn((W,) + tuple(shape), generator=g) * scale).to(BF16)


def _run_oneshot(L, W, parts, numel, max_ctas=MAX_CTAS):
    """exchange as every rank; checks the signals and the sentinels past numel; returns the W outputs [W, numel]."""
    world = World(W, max_ctas)
    d = torch.zeros(W, numel + TAIL, dtype=BF16, device=DEV)
    d[:, :numel] = parts.reshape(W, numel).to(DEV)
    outs = sentinel_bf16(W, numel + TAIL)
    ctas = min(-(-numel // (8 * 512)), max_ctas)
    for r in range(W):
        n0 = L.xb_launch_count()
        rc = world.oneshot(L, r, outs[r], d, numel)
        assert rc == 0, L.xb_last_error()
        assert L.xb_launch_count() == n0 + 1
        world.check_signals(r, ctas)
    o = bits(outs)
    assert (o[:, numel:] == OUT_SENTINEL).all(), "oneshot_allreduce wrote past numel"
    return outs[:, :numel].cpu()


# ---------------------------------------------------------------------------------------------------------------------
# xb_oneshot_allreduce_bf16
# ---------------------------------------------------------------------------------------------------------------------
ONESHOT_SHAPES = [(n, c) for n in (8, 8 * 512, 8 * 512 + 8, 3584 * 64) for c in (1, 64)]
# four CTAs each stride over 512 vectors three times, and a partial fourth pass
ONESHOT_SHAPES += [(8 * 512 * 4 * 3 + 8, c) for c in (1, 4, 64)]


@pytest.mark.parametrize("numel,max_ctas", ONESHOT_SHAPES)
@pytest.mark.parametrize("W", range(1, 9))
def test_oneshot_allreduce(W, numel, max_ctas, L):
    parts = _partials(W, (numel,), seed=W * 1000 + numel % 997 + max_ctas)
    outs = _run_oneshot(L, W, parts, numel, max_ctas)
    ref = seq_sum(parts).to(BF16)
    for r in range(W):
        assert torch.equal(bits(outs[r]), bits(ref)), f"rank {r}: {int((bits(outs[r]) != bits(ref)).sum())} elements differ"
    assert_sum_bound(outs[0], parts)


def test_oneshot_allreduce_empty_launches_nothing(L):
    world = World(2)
    d = torch.randn(2, 64, device=DEV).to(BF16)
    out = sentinel_bf16(64)
    n0 = L.xb_launch_count()
    assert world.oneshot(L, 0, out, d, 0) == 0
    assert L.xb_launch_count() == n0
    assert (bits(out) == OUT_SENTINEL).all()
    world.check_signals(0, 0)


# ---------------------------------------------------------------------------------------------------------------------
# xb_allreduce_add_rms_norm_bf16
# ---------------------------------------------------------------------------------------------------------------------
def _composition(L, W, d, res0, w, T, H):
    """the library's unfused path on the same partials: xb_oneshot_allreduce_bf16, then xb_fused_add_rms_norm_bf16 -
    what _row_parallel computes with NCCL (pg.allreduce + add_norm).  Returns (out, residual, bf16 sum)."""
    from xllm_b200 import ops
    x = torch.empty(T, H, dtype=BF16, device=DEV)
    assert World(W).oneshot(L, 0, x, d, T * H) == 0, L.xb_last_error()
    s = x.clone()
    res = res0.clone()
    ops.fused_add_rms_norm(x, res, w, EPS)
    return x.cpu(), res.cpu(), s.cpu()


def _run_fused(L, world, d, res0, w, T, H, rows):
    """fused exchange as every rank into its own out / residual (`rows` >= T rows, sentinels past T); returns them."""
    W = world.W
    outs = sentinel_bf16(W, rows, H)
    resid = sentinel_bf16(W, rows, H)
    resid[:, :T] = res0
    for r in range(W):
        n0 = L.xb_launch_count()
        rc = world.fused(L, r, outs[r], resid[r], w, d, T, H)
        assert rc == 0, L.xb_last_error()
        assert L.xb_launch_count() == n0 + 1
        world.check_signals(r, T)
    assert (bits(outs[:, T:]) == OUT_SENTINEL).all(), "allreduce_add_rms_norm wrote out rows past num_tokens"
    assert (bits(resid[:, T:]) == OUT_SENTINEL).all(), "allreduce_add_rms_norm wrote residual rows past num_tokens"
    return outs[:, :T].cpu(), resid[:, :T].cpu()


# 1032 = 129 vectors (a part-filled last warp); 8200 is the first hidden whose vectors need the second kMaxVec pass of a
# 1024-thread CTA; 16384 is the largest accepted
FUSED_HIDDEN = [8, 64, 896, 1032, 3584, 5120, 7168, 8192, 8200, 16384]


@pytest.mark.parametrize("T", [1, 7, MAX_CTAS])
@pytest.mark.parametrize("H", FUSED_HIDDEN)
@pytest.mark.parametrize("W", [1, 2, 3, 4, 8])
def test_allreduce_add_rms_norm(W, H, T, L):
    """Bit-identical to the library's own composition (oneshot exchange, then fused_add_rms_norm).  For up to 255 tokens
    both kernels run ceil(H/8/32)*32 threads (at most 1024) per token and thread t owns vectors t and t + blockDim, so
    their fp32 sums of squares add the same terms in the same order: any difference is a rounding the fused kernel does
    differently.  The residual is also checked bit-exact against bf16(float(bf16 sum) + residual), and the output against
    the oracle's fused_add_rms_norm."""
    g = torch.Generator().manual_seed(W * 100000 + H * 10 + T)
    parts = _partials(W, (T, H), seed=W * 7919 + H + T)
    res0 = torch.randn(T, H, generator=g).to(BF16)
    w = (1 + 0.1 * torch.randn(H, generator=g)).to(BF16)
    d, res0_d, w_d = parts.to(DEV), res0.to(DEV), w.to(DEV)
    outs, resid = _run_fused(L, World(W), d, res0_d, w_d, T, H, T + 2)

    c_out, c_res, c_sum = _composition(L, W, d, res0_d, w_d, T, H)
    s = seq_sum(parts).to(BF16)
    assert torch.equal(bits(c_sum), bits(s)), "oneshot_allreduce differs from the sequential fp32 sum"
    ref_res = (s.float() + res0.float()).to(BF16)
    for r in range(W):
        nres = int((bits(resid[r]) != bits(ref_res)).sum())
        assert nres == 0, f"rank {r}: {nres} residual elements differ from bf16(bf16 sum + residual)"
        nout = int((bits(outs[r]) != bits(c_out)).sum())
        assert nout == 0, f"rank {r}: {nout} / {c_out.numel()} outputs differ from oneshot_allreduce + fused_add_rms_norm"
    assert torch.equal(bits(c_res), bits(ref_res))
    assert_norm_close(outs[0], s, res0, w)


# ---------------------------------------------------------------------------------------------------------------------
# probes: inputs whose exact answer exposes a skipped, repeated or reordered rank, or a lost sign / subnormal
# ---------------------------------------------------------------------------------------------------------------------
PROBE_T, PROBE_H = 4, 1024


def _probe_both_kernels(L, parts):
    """runs the probe partials [W, PROBE_T, PROBE_H] through both kernels as every rank (residual 0) and checks each result
    bit for bit against the sequential fp32 sum; returns that sum rounded to bf16."""
    W = parts.shape[0]
    ref = seq_sum(parts).to(BF16)
    outs = _run_oneshot(L, W, parts, PROBE_T * PROBE_H)
    for r in range(W):
        n = int((bits(outs[r].reshape(PROBE_T, PROBE_H)) != bits(ref)).sum())
        assert n == 0, f"oneshot_allreduce as rank {r}: {n} elements differ"
    zero = torch.zeros(PROBE_T, PROBE_H, dtype=BF16, device=DEV)
    w = torch.ones(PROBE_H, dtype=BF16, device=DEV)
    _, resid = _run_fused(L, World(W), parts.to(DEV), zero, w, PROBE_T, PROBE_H, PROBE_T)
    want = (ref.float() + 0.0).to(BF16)
    for r in range(W):
        n = int((bits(resid[r]) != bits(want)).sum())
        assert n == 0, f"allreduce_add_rms_norm as rank {r}: {n} residual elements differ"
    return ref


@pytest.mark.parametrize("W", [1, 2, 3, 5, 8])
def test_probe_rank_mask(W, L):
    """partial r = +-2^r: the sum is exactly +-(2^W - 1), so a rank skipped or counted twice changes the bits."""
    g = torch.Generator().manual_seed(W)
    sign = torch.randint(0, 2, (PROBE_T, PROBE_H), generator=g).float() * 2 - 1
    parts = torch.stack([sign * 2.0 ** r for r in range(W)]).to(BF16)
    ref = _probe_both_kernels(L, parts)
    assert torch.equal(ref.float(), sign * (2 ** W - 1))


@pytest.mark.parametrize("W", [3, 4, 5, 8])
def test_probe_summation_order(W, L):
    """rows whose fp32 sum depends on the order of the ranks, e.g. (2^25, 1, -2^25, 1, ...) sums to 1 in rank order but to
    0 reversed.  (Two-term sums are commutative, so the probe starts at W = 3.)"""
    g = torch.Generator().manual_seed(40 + W)
    vals = torch.tensor([2.0 ** 25, -2.0 ** 25, 2.0 ** 24, 1.0, -1.0, 3.0, 0.5])
    parts = vals[torch.randint(0, len(vals), (W, PROBE_T, PROBE_H), generator=g)]
    pattern = torch.tensor([2.0 ** 25, 1.0, -2.0 ** 25, 1.0])
    parts[:, 0, :] = pattern[torch.arange(W) % 4].unsqueeze(1)
    parts = parts.to(BF16)
    ref = _probe_both_kernels(L, parts)
    # the probe must catch a wrong order: the calling rank first, or the ranks reversed, give other bits
    orders = {f"from rank {r}": list(range(r, W)) + list(range(r)) for r in range(1, W)}
    orders["reversed"] = list(range(W))[::-1]
    for what, order in orders.items():
        assert not torch.equal(bits(seq_sum(parts, order).to(BF16)), bits(ref)), f"probe blind to the order {what}"


@pytest.mark.parametrize("W", [2, 3, 5, 8])
def test_probe_cancellation(W, L):
    """sums that cancel to +0 (also from all -0 partials: the sum starts from +0.0), to tiny normals and to subnormals
    (2^-132: a flush-to-zero add would give 0)."""
    g = torch.Generator().manual_seed(70 + W)
    n = PROBE_T * PROBE_H
    parts = torch.zeros(W, n)
    parts[:, :] = torch.where(torch.rand(W, n, generator=g) < 0.5, -0.0, 0.0)
    kind = torch.arange(n) % 4
    x = torch.exp2(torch.randint(-20, 20, (n,), generator=g).float()) * (1 + torch.randint(0, 127, (n,), generator=g) / 128)
    i, j = torch.arange(n) % W, (torch.arange(n) + 1) % W
    cols = torch.arange(n)
    # kind 0: all +-0; kind 1: x and -x on two ranks; kind 2: (1 + 2^-7) and -1 -> 2^-7; kind 3: 3*2^-133 and -2^-133
    parts[i[kind == 1], cols[kind == 1]] = x[kind == 1]
    parts[j[kind == 1], cols[kind == 1]] = -x[kind == 1]
    parts[i[kind == 2], cols[kind == 2]] = 1 + 2.0 ** -7
    parts[j[kind == 2], cols[kind == 2]] = -1.0
    parts[i[kind == 3], cols[kind == 3]] = 3 * 2.0 ** -133
    parts[j[kind == 3], cols[kind == 3]] = -(2.0 ** -133)
    parts = parts.to(BF16).view(W, PROBE_T, PROBE_H)
    ref = _probe_both_kernels(L, parts).flatten()
    assert (bits(ref[kind <= 1]) == 0).all(), "the probe expects +0 from cancellation"
    assert (ref[kind == 2].float() == 2.0 ** -7).all() and (ref[kind == 3].float() == 2.0 ** -132).all()


# ---------------------------------------------------------------------------------------------------------------------
# CUDA graph: the epoch lives in device memory, so replays keep signalling fresh targets
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["oneshot", "fused"])
def test_graph_replays_advance_the_epoch(kind, L):
    W, T, H, replays = 4, 7, 3584, 3
    parts = _partials(W, (T, H), seed=5)
    g = torch.Generator().manual_seed(6)
    res0 = torch.randn(T, H, generator=g).to(BF16)
    w = (1 + 0.1 * torch.randn(H, generator=g)).to(BF16)
    d, w_d = parts.to(DEV), w.to(DEV)
    world = World(W)
    outs = sentinel_bf16(W, T, H)
    resid = res0.to(DEV).expand(W, T, H).contiguous()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for r in range(W):                                     # each launch arms its pads inside the graph
            if kind == "oneshot":
                rc = world.oneshot(L, r, outs[r], d, T * H)
            else:
                rc = world.fused(L, r, outs[r], resid[r], w_d, d, T, H)
            assert rc == 0, L.xb_last_error()
    for _ in range(replays):
        graph.replay()
    torch.cuda.synchronize()
    ctas = min(-(-T * H // (8 * 512)), MAX_CTAS) if kind == "oneshot" else T
    for r in range(W):
        world.check_signals(r, ctas, k=replays)
    s = seq_sum(parts).to(BF16)
    res_in = want_res = res0                                   # residual before / after the last replay
    if kind == "fused":
        for _ in range(replays):
            res_in, want_res = want_res, (s.float() + want_res.float()).to(BF16)
    for r in range(W):
        assert torch.equal(bits(resid[r]), bits(want_res)), f"rank {r}: residual after {replays} replays"
        got = outs[r].cpu()
        if kind == "oneshot":
            assert torch.equal(bits(got), bits(s)), f"rank {r}: output after {replays} replays"
        else:
            assert_norm_close(got, s, res_in, w)


# ---------------------------------------------------------------------------------------------------------------------
# the product's order: the row-parallel linear writes the partial, the fused exchange follows it under PDL
# ---------------------------------------------------------------------------------------------------------------------
def test_pdl_linear_then_fused_exchange(L):
    """As _row_parallel: xb_linear_bf16_small_m writes the calling rank's partial straight into its exchange buffer, and
    the fused kernel follows it with PDL.  The buffer first holds the negated partial, so a kernel that read it before the
    linear finished would give other bits.  K = 18944 (Qwen2-7B down_proj) keeps the linear running for a while."""
    from xllm_b200 import _lib, ops
    W, T, H, K = 4, 4, 3584, 18944
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(W, T, K, generator=g)).to(BF16).to(DEV)
    wl = (torch.randn(H, K, generator=g) * 0.02).to(BF16).to(DEV)
    res0 = torch.randn(T, H, generator=g).to(BF16).to(DEV)
    wn = (1 + 0.1 * torch.randn(H, generator=g)).to(BF16).to(DEV)
    y = torch.stack([ops.matmul_small_m(x[p], wl) for p in range(W)])    # every rank's partial, made by the same linear
    torch.cuda.synchronize()

    def run(pdl):
        _lib.set_pdl(pdl)
        world = World(W)
        outs = torch.empty(W, T, H, dtype=BF16, device=DEV)
        resid = res0.expand(W, T, H).contiguous()
        for r in range(W):
            d = y.clone()
            d[r].copy_(-y[r])                                    # stale contents of the calling rank's buffer
            ops.matmul_small_m(x[r], wl, out=d[r])               # the partial lands in the exchange buffer
            rc = world.fused(L, r, outs[r], resid[r], wn, d, T, H)
            assert rc == 0, L.xb_last_error()
            torch.cuda.synchronize()                             # d is freed at the end of the iteration
        for r in range(W):
            world.check_signals(r, T)
        return outs.cpu(), resid.cpu()

    try:
        out_pdl, res_pdl = run(True)
        out_plain, res_plain = run(False)
    finally:
        _lib.set_pdl(True)
    c_out, c_res, _ = _composition(L, W, y, res0, wn, T, H)
    s = seq_sum(y.cpu()).to(BF16)
    ref_res = (s.float() + res0.cpu().float()).to(BF16)
    for r in range(W):
        assert torch.equal(bits(out_pdl[r]), bits(out_plain[r])) and torch.equal(bits(res_pdl[r]), bits(res_plain[r])), \
            f"rank {r}: PDL changes the result"
        assert torch.equal(bits(out_pdl[r]), bits(c_out)), f"rank {r}: output differs from the composition"
        assert torch.equal(bits(res_pdl[r]), bits(ref_res)), f"rank {r}: residual differs from the reference"


# ---------------------------------------------------------------------------------------------------------------------
# refusals with real, armed buffers: an error, no launch, nothing written
# ---------------------------------------------------------------------------------------------------------------------
W_REJ, H_REJ, T_REJ = 4, 896, 4
REFUSED = [
    ("oneshot", dict(numel=12), r"numel 12\b"),
    ("oneshot", dict(numel=-8), r"numel -8\b"),
    ("oneshot", dict(max_ctas=0), r"max_ctas 0\b"),
    ("oneshot", dict(max_ctas=-1), r"max_ctas -1\b"),
    ("oneshot", dict(world=0), r"world 0\b"),
    ("oneshot", dict(world=9), r"world 9\b"),
    ("oneshot", dict(rank=W_REJ), rf"rank {W_REJ}\b"),
    ("oneshot", dict(rank=-1), r"rank -1\b"),
    ("fused", dict(hidden=12), r"hidden 12\b"),
    ("fused", dict(hidden=16392), r"hidden 16392\b"),
    ("fused", dict(hidden=0), r"hidden 0\b"),
    ("fused", dict(hidden=-8), r"hidden -8\b"),
    ("fused", dict(tokens=MAX_CTAS + 1), rf"{MAX_CTAS + 1} tokens exceed\b"),
    ("fused", dict(tokens=-1), r"num_tokens -1\b"),
    ("fused", dict(world=0), r"world 0\b"),
    ("fused", dict(world=9), r"world 9\b"),
    ("fused", dict(rank=W_REJ), rf"rank {W_REJ}\b"),
    ("fused", dict(rank=-1), r"rank -1\b"),
]


@pytest.mark.parametrize("kind,bad,pattern", REFUSED, ids=[f"{k}-{list(b)[0]}={list(b.values())[0]}" for k, b, _ in REFUSED])
def test_bad_arguments_are_refused_with_real_buffers(kind, bad, pattern, L):
    from xllm_b200._lib import XllmB200Error, check
    rows = MAX_CTAS + 1                                          # room for every token count tried
    world = World(W_REJ)
    d = torch.randn(W_REJ, rows, H_REJ, device=DEV).to(BF16)
    out = sentinel_bf16(rows, H_REJ)
    resid = torch.randn(rows, H_REJ, device=DEV).to(BF16)
    w = torch.ones(H_REJ, dtype=BF16, device=DEV)
    world.pads[0].fill_(ARMED)
    before = [t.clone() for t in (out, resid, world.pads, world.epoch)]
    n0 = L.xb_launch_count()
    with pytest.raises(XllmB200Error, match=pattern):
        if kind == "oneshot":
            check(world.oneshot(L, 0, out, d, bad.get("numel", T_REJ * H_REJ), world=bad.get("world"),
                                max_ctas=bad.get("max_ctas"), rank=bad.get("rank")), "oneshot_allreduce")
        else:
            check(world.fused(L, 0, out, resid, w, d, bad.get("tokens", T_REJ), bad.get("hidden", H_REJ),
                              world=bad.get("world"), rank=bad.get("rank")), "allreduce_add_rms_norm")
    torch.cuda.synchronize()
    assert L.xb_launch_count() == n0
    for name, a, b in zip(("out", "residual", "pads", "epoch"), before, (out, resid, world.pads, world.epoch)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"{name} changed"
