"""MLA on the GPU: the latent cache writer (against the reference composition, and bit-exact against the library's own
unfused kernels) and paged absorbed-MLA attention (against tests/mla_ref.py on the attention error bound of tests/util.py),
split-KV determinism, one CUDA graph replayed over changing batches, and the shim binding."""
import math

import pytest
import torch

from oracle import ops as O
from tests import mla_ref as R
from tests.util import assert_close_attention, assert_close_bf16
from xllm_b200 import ops

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"
SCALE = (192 ** -0.5)      # qk_head_dim^-0.5 of DeepSeek-V3 (128 nope + 64 rope); mscale 1
# Elementwise factor of the attention bound.  The kernel rounds P to bf16 against the running row maximum of its kv tile
# order, the reference against the final maximum, so the two carry independent P roundings (as any two implementations
# of the ladder do).  These cases check 1e6 - 3.4e7 outputs each (512 wide), 10-100x more than the GQA attention tests,
# and the tail of that difference reaches 1.15x the 2e-3 factor on up to 20 elements; the relative-L2 bar (3e-3) is
# unchanged and holds with margin (<= 1.5e-3 measured).
RTOL = 2.5e-3


def _latent_case(T, page, seed, n_pages=None):
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(T, 640, generator=g).to(BF16)
    latent = base[:, 8:8 + 576]                               # strided view (row stride 640, 16-byte aligned)
    gamma = (1 + 0.1 * torch.randn(512, generator=g)).to(BF16)
    positions = torch.randint(0, 4096, (T,), generator=g, dtype=torch.int64)
    n_pages = n_pages or (T + page - 1) // page + 2
    slots = torch.randperm(n_pages * page, generator=g)[:T].to(torch.int32)
    slots[::5] = -1
    cs = O.compute_cos_sin_cache(64, 4096, 10000)
    return base, latent, gamma, positions, slots, cs, n_pages


@pytest.mark.parametrize("interleaved", [True, False])
@pytest.mark.parametrize("page", [1, 16, 64, 128])
def test_cache_writer(interleaved, page):
    T, eps = 300, 1e-6
    base, latent, gamma, pos, slots, cs, n_pages = _latent_case(T, page, seed=page + 7 * interleaved)
    ckv_ref = torch.zeros(n_pages, page, 512, dtype=BF16)
    kpe_ref = torch.zeros(n_pages, page, 64, dtype=BF16)
    R.mla_cache_latent(latent, gamma, eps, pos, cs, slots, ckv_ref, kpe_ref, interleaved)

    d_base = base.to(DEV)
    d_lat = d_base[:, 8:8 + 576]
    args = (gamma.to(DEV), eps, pos.to(DEV), cs.to(DEV), slots.to(DEV))
    ckv = torch.zeros(n_pages, page, 512, dtype=BF16, device=DEV)
    kpe = torch.zeros(n_pages, page, 64, dtype=BF16, device=DEV)
    n0 = ops.lib().xb_launch_count()
    ops.mla_cache_latent(d_lat, args[0], eps, args[2], args[3], args[4], ckv, kpe, interleaved=interleaved)
    assert ops.lib().xb_launch_count() - n0 == 1
    torch.cuda.synchronize()
    # RoPE has no reduction: bit-exact with the reference ladder.  The norm's fp32 sum of squares is ordered differently on
    # the CPU, so rstd may differ in its last bit and flip the bf16 rounding of x * rstd; the product with gamma rounds
    # again, so a flipped element can sit 2 ulps away.
    assert torch.equal(kpe.cpu(), kpe_ref)
    assert_close_bf16(ckv, ckv_ref, ulps=2, what=f"mla writer ckv page={page}")

    # the four launches the writer replaces, on the same inputs
    normed = torch.empty(T, 512, dtype=BF16, device=DEV)
    ops.rms_norm(normed, d_lat[:, :512], args[0], eps)
    k_pe = d_lat[:, 512:].clone().view(T, 1, 64)
    ops.rotary_embedding(args[2], k_pe, None, args[3], is_neox=not interleaved)
    ckv4, kpe4 = torch.zeros_like(ckv), torch.zeros_like(kpe)
    ops.reshape_paged_cache(args[4], normed.view(T, 1, 512), normed.view(T, 1, 512), ckv4.view(n_pages, page, 1, 512),
                            torch.zeros_like(ckv4).view(n_pages, page, 1, 512))
    ops.reshape_paged_cache(args[4], k_pe, k_pe, kpe4.view(n_pages, page, 1, 64), torch.zeros_like(kpe4).view(n_pages, page, 1, 64))
    torch.cuda.synchronize()
    assert torch.equal(ckv, ckv4) and torch.equal(kpe, kpe4)
    assert torch.equal(d_base, base.to(DEV)), "the writer must not modify its input"


def make_mla_case(kv_lens, qo_lens, H, page=16, seed=0, extra_pages=5):
    """random caches with pages handed out as a random permutation; q in both forms (split / packed 576)."""
    g = torch.Generator().manual_seed(seed)
    B = len(kv_lens)
    n_pages_req = [(k + page - 1) // page for k in kv_lens]
    n_pages = sum(n_pages_req) + extra_pages
    perm = torch.randperm(n_pages, generator=g).to(torch.int32)
    indptr = torch.tensor([0] + list(torch.tensor(n_pages_req).cumsum(0).tolist()), dtype=torch.int32)
    indices = perm[:int(indptr[-1])].clone()
    last = torch.tensor([(k - (n - 1) * page) if n > 0 else 0 for k, n in zip(kv_lens, n_pages_req)], dtype=torch.int32)
    qo_indptr = torch.tensor([0] + list(torch.tensor(qo_lens).cumsum(0).tolist()), dtype=torch.int32)
    T = int(qo_indptr[-1])
    ckv = torch.randn(n_pages, page, 512, generator=g).to(BF16)
    kpe = torch.randn(n_pages, page, 64, generator=g).to(BF16)
    q_input = torch.randn(T, H, 576, generator=g).to(BF16)
    return dict(q_input=q_input, ckv=ckv, kpe=kpe, qo_indptr=qo_indptr, kv_indptr=indptr, kv_indices=indices, last=last,
                B=B, T=T, H=H, page=page, max_pages=max(max(n_pages_req), 1), max_qo=max(qo_lens))


def _dev(c):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in c.items()}


def run_mla(c, causal, packed=True, splits=None, plan=None):
    d = _dev(c)
    q = d["q_input"]
    if packed:
        q_nope, q_pe = q[..., :512], q[..., 512:]
    else:
        q_nope, q_pe = q[..., :512].contiguous(), q[..., 512:].contiguous()
    plan = plan or ops.MlaPlan(c["B"], c["H"], c["max_qo"], c["page"], c["max_pages"], DEV, splits=splits)
    out = torch.full((c["T"], c["H"], 512), float("nan"), dtype=BF16, device=DEV)
    ops.mla_paged_attention(plan, q_nope, q_pe, d["ckv"], d["kpe"], d["qo_indptr"], d["kv_indptr"], d["kv_indices"],
                            d["last"], SCALE, out, causal=causal)
    torch.cuda.synchronize()
    return out, plan


def ref_mla(c, causal):
    d = _dev(c)
    q = d["q_input"]
    a = (q[..., :512], q[..., 512:], d["ckv"], d["kpe"], d["qo_indptr"], d["kv_indptr"], d["kv_indices"], d["last"], SCALE,
         causal)
    return R.mla_paged_attention(*a), R.mla_paged_attention(*a, abs_value=True)


DECODE_LENS = [0, 1, 127, 128, 129, 4096]


@pytest.mark.parametrize("H", [8, 16, 32, 128])
@pytest.mark.parametrize("B", [1, 7, 64])
def test_mla_decode_vs_reference(H, B):
    kv = [DECODE_LENS[(i * 5 + H) % len(DECODE_LENS)] for i in range(B)]
    if B == 1:
        kv = [33000]
    c = make_mla_case(kv, [1] * B, H, page=16 if B != 7 else 1, seed=H * 100 + B)
    ref, sc = ref_mla(c, causal=False)
    for packed in (True, False):
        out, _ = run_mla(c, causal=False, packed=packed)
        assert_close_attention(out, ref, sc, rtol=RTOL, what=f"mla decode H={H} B={B} packed={packed}")
    rows0 = [b for b in range(B) if kv[b] == 0]
    assert all(out[b].abs().max().item() == 0 for b in rows0), "kv_len 0 must give zero rows"


@pytest.mark.parametrize("H", [16, 128])
@pytest.mark.parametrize("qo", [2, 3, 4])
def test_mla_speculative_causal(H, qo):
    kv = [qo + k for k in (5, 300, 4096, 0, 77, 1000, 31)]
    c = make_mla_case(kv, [qo] * len(kv), H, page=64, seed=qo * 10 + H)
    ref, sc = ref_mla(c, causal=True)
    out, _ = run_mla(c, causal=True)
    assert_close_attention(out, ref, sc, rtol=RTOL, what=f"mla mtp H={H} qo={qo}")


@pytest.mark.parametrize("H,qo,hist", [(16, 2048, 0), (16, 2048, 8192), (128, 300, 8192), (128, 512, 0)])
def test_mla_chunked_prefill(H, qo, hist):
    c = make_mla_case([hist + qo, 40 + 7], [qo, 7], H, page=128, seed=hist + qo + H)
    ref, sc = ref_mla(c, causal=True)
    out, _ = run_mla(c, causal=True)
    assert_close_attention(out, ref, sc, rtol=RTOL, what=f"mla prefill H={H} qo={qo} hist={hist}")


def test_mla_forced_splits_and_determinism():
    c = make_mla_case([4096, 1, 129, 2500, 0], [1] * 5, 16, seed=5)
    ref, sc = ref_mla(c, causal=False)
    for s in (1, 2, 3, 7, 32):
        out, plan = run_mla(c, causal=False, splits=s)
        assert plan.splits == s
        assert_close_attention(out, ref, sc, rtol=RTOL, what=f"mla splits={s}")
        again, _ = run_mla(c, causal=False, plan=plan)
        assert torch.equal(out, again), f"splits={s}: two runs of one plan differ"
    c = make_mla_case([1500, 900], [3, 2], 128, seed=6)
    ref, sc = ref_mla(c, causal=True)
    for s in (1, 5):
        out, _ = run_mla(c, causal=True, splits=s)
        assert_close_attention(out, ref, sc, rtol=RTOL, what=f"mla mtp splits={s}")


def test_mla_graph_replay_writer_and_attention():
    """one graph of writer + attention captured once at batch 8, replayed over three batches whose paged triplet and
    slots are refreshed on the device by xb_decode_metadata_update; each replay equals the eager result."""
    H, page, B_cap, max_pages, n_pages = 16, 16, 8, 80, 8 * 80 + 1
    g = torch.Generator().manual_seed(11)
    ckv = torch.randn(n_pages, page, 512, generator=g).to(BF16).to(DEV)
    kpe = torch.randn(n_pages, page, 64, generator=g).to(BF16).to(DEV)
    gamma = (1 + 0.1 * torch.randn(512, generator=g)).to(BF16).to(DEV)
    cs = O.compute_cos_sin_cache(64, 8192, 10000).to(DEV)
    latent = torch.zeros(B_cap, 576, dtype=BF16, device=DEV)
    q = torch.zeros(B_cap, H, 576, dtype=BF16, device=DEV)
    pos64 = torch.zeros(B_cap, dtype=torch.int64, device=DEV)
    st = {k: torch.zeros(n, dtype=torch.int32, device=DEV) for k, n in
          (("tokens", B_cap), ("positions", B_cap), ("slots", B_cap), ("kv_seq_lens", B_cap + 1), ("delta", B_cap),
           ("indptr", B_cap + 1), ("indices", B_cap * max_pages), ("last", B_cap))}
    qo_indptr = torch.arange(B_cap + 1, dtype=torch.int32, device=DEV)
    out = torch.zeros(B_cap, H, 512, dtype=BF16, device=DEV)
    plan = ops.MlaPlan(B_cap, H, 1, page, max_pages, DEV)

    def step():
        ops.mla_cache_latent(latent, gamma, 1e-6, pos64, cs, st["slots"], ckv, kpe, interleaved=True)
        ops.mla_paged_attention(plan, q[..., :512], q[..., 512:], ckv, kpe, qo_indptr, st["indptr"], st["indices"],
                                st["last"], SCALE, out, causal=False)

    def refresh(kv_lens):
        """host-side step inputs for len(kv_lens) live requests (the rest of the captured batch padded with empty
        requests), copied into the graph's buffers on the device."""
        B = len(kv_lens)
        perm = torch.randperm(n_pages - 1, generator=g)[:sum((k + page - 1) // page for k in kv_lens)] + 1
        npg = [(k + page - 1) // page for k in kv_lens] + [0] * (B_cap - B)
        indptr = torch.tensor([0] + list(torch.tensor(npg).cumsum(0).tolist()), dtype=torch.int32)
        last = torch.tensor([k - (n - 1) * page if n else 0 for k, n in zip(kv_lens + [0] * (B_cap - B), npg)], dtype=torch.int32)
        slots = torch.full((B_cap,), -1, dtype=torch.int32)
        for b, k in enumerate(kv_lens):      # the newest token of each live request is written this step
            slots[b] = int(perm[int(indptr[b]) + (k - 1) // page]) * page + (k - 1) % page
        pos = torch.tensor([k - 1 for k in kv_lens] + [0] * (B_cap - B), dtype=torch.int32)
        src = [torch.zeros(B_cap, dtype=torch.int32), pos, slots, torch.zeros(B_cap + 1, dtype=torch.int32), indptr,
               perm.to(torch.int32), last]
        src = [s.to(DEV) for s in src]
        rc = ops.lib().xb_decode_metadata_update(
            *[ops._p(s) for s in src], ops._p(st["tokens"]), ops._p(st["positions"]), ops._p(st["slots"]),
            ops._p(st["kv_seq_lens"]), ops._p(st["delta"]), ops._p(st["indptr"]), ops._p(st["indices"]), ops._p(st["last"]),
            ops.c_i64(B_cap), ops.c_i64(B_cap), ops.c_i64(B_cap), ops.c_i64(perm.numel()), ops.c_ptr(0), ops.c_i64(0),
            ops._stream())
        assert rc == 0
        pos64.copy_(st["positions"].to(torch.int64))
        latent.copy_(torch.randn(B_cap, 576, generator=g).to(BF16))
        q.copy_(torch.randn(B_cap, H, 576, generator=g).to(BF16))

    refresh([10] * B_cap)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    for kv_lens in ([17, 1000, 3, 1279, 64, 65, 900, 1], [1270, 5], [300, 301, 302, 640, 2]):
        refresh(kv_lens)
        ckv0, kpe0 = ckv.clone(), kpe.clone()
        graph.replay()
        torch.cuda.synchronize()
        got, ckv_g, kpe_g = out.clone(), ckv.clone(), kpe.clone()
        ckv.copy_(ckv0)
        kpe.copy_(kpe0)
        step()
        torch.cuda.synchronize()
        assert torch.equal(got, out) and torch.equal(ckv_g, ckv) and torch.equal(kpe_g, kpe), f"replay at {kv_lens}"
        assert all(out[b].abs().max().item() == 0 for b in range(len(kv_lens), B_cap))


def test_mla_shim_binding():
    from xllm_b200 import build_shim
    shim = build_shim.load_py()
    T, page, eps = 40, 16, 1e-6
    base, latent, gamma, pos, slots, cs, n_pages = _latent_case(T, page, seed=3)
    d_lat = base.to(DEV)[:, 8:8 + 576]
    ckv = torch.zeros(n_pages, page, 1, 512, dtype=BF16, device=DEV)
    kpe = torch.zeros(n_pages, page, 1, 64, dtype=BF16, device=DEV)
    shim.fused_mla_kv(d_lat, cs.to(DEV), pos.to(DEV), gamma.to(DEV), ckv, kpe, slots.to(DEV), "none", eps, True)
    ckv_ref = torch.zeros(n_pages, page, 512, dtype=BF16)
    kpe_ref = torch.zeros(n_pages, page, 64, dtype=BF16)
    R.mla_cache_latent(latent, gamma, eps, pos, cs, slots, ckv_ref, kpe_ref, True)
    assert torch.equal(ckv.cpu()[:, :, 0], ckv_ref) and torch.equal(kpe.cpu()[:, :, 0], kpe_ref)
    with pytest.raises(RuntimeError, match="quant_mode"):
        shim.fused_mla_kv(d_lat, cs.to(DEV), pos.to(DEV), gamma.to(DEV), ckv, kpe, slots.to(DEV), "dynamic_per_token", eps, True)

    c = make_mla_case([700, 3, 0], [2, 1, 1], 16, seed=9)
    d = _dev(c)
    out = torch.empty(c["T"], 16, 512, dtype=BF16, device=DEV)
    shim.mla_paged_attention(d["q_input"][..., :512], d["q_input"][..., 512:], d["ckv"], d["kpe"], d["qo_indptr"],
                             d["kv_indptr"], d["kv_indices"], d["last"], c["max_qo"], SCALE, True, out)
    torch.cuda.synchronize()
    ref, sc = ref_mla(c, causal=True)
    assert_close_attention(out, ref, sc, rtol=RTOL, what="mla shim")
    # wrong shapes raise c10::Error before any launch
    with pytest.raises(RuntimeError, match="shapes"):
        shim.fused_mla_kv(d_lat, cs.to(DEV), pos.to(DEV), gamma.to(DEV), ckv[..., :256], kpe, slots.to(DEV), "none", eps, True)
    q = d["q_input"]
    with pytest.raises(RuntimeError, match="equal T and H"):
        shim.mla_paged_attention(q[..., :512], q[:, :8, 512:], d["ckv"], d["kpe"], d["qo_indptr"], d["kv_indptr"],
                                 d["kv_indices"], d["last"], c["max_qo"], SCALE, True, out)
    with pytest.raises(RuntimeError, match="ckv_cache row"):
        shim.mla_paged_attention(q[..., :512], q[..., 512:], d["ckv"][..., :256], d["kpe"], d["qo_indptr"], d["kv_indptr"],
                                 d["kv_indices"], d["last"], c["max_qo"], SCALE, True, out)


_fi_probe = {}


def flashinfer_mla_or_skip():
    """FlashInfer's fa2 batch_mla module (pre-built by tools/build_flashinfer_cache.py into baseline/_fi, or JIT-built here
    within 300 s); skips only when it cannot be built."""
    if "skip" in _fi_probe:
        pytest.skip(_fi_probe["skip"])
    if "mod" in _fi_probe:
        return _fi_probe["mod"]
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tools"))
    import build_flashinfer_cache as FIC
    FIC.set_env()
    try:
        import flashinfer
        from flashinfer.jit import core as jc
        spec = FIC.mla_specs()[0]
    except Exception as e:  # pragma: no cover
        _fi_probe["skip"] = f"flashinfer not importable: {e}"
        pytest.skip(_fi_probe["skip"])
    if not spec.jit_library_path.exists():
        r = subprocess.run(["timeout", "300", sys.executable, os.path.join(root, "tools", "build_flashinfer_cache.py"), "mla"],
                           capture_output=True, text=True)
        if r.returncode != 0 or not spec.jit_library_path.exists():
            _fi_probe["skip"] = "FlashInfer batch_mla module not pre-built and JIT did not finish in 300 s"
            pytest.skip(_fi_probe["skip"])
    if not getattr(jc.JitSpec, "_xb_patched", False):
        orig = jc.JitSpec.build

        def build(self, verbose, need_lock=True):      # a pre-built library is loaded as is
            if self.jit_library_path.exists():
                return None
            return orig(self, verbose, need_lock)
        jc.JitSpec.build = build
        jc.JitSpec._xb_patched = True
    _fi_probe["mod"] = flashinfer
    return flashinfer


@pytest.mark.parametrize("H,kv,qo,page", [(16, [4096, 1, 129, 700, 33000], 1, 16), (128, [4096, 17, 1000], 1, 64),
                                          (16, [2 + k for k in (5, 300, 4096, 77)], 2, 64),
                                          (128, [4 + k for k in (31, 1000)], 4, 16),
                                          (16, [8192 + 2048, 47], [2048, 7], 128)])
def test_mla_vs_flashinfer(H, kv, qo, page):
    """the same inputs through FlashInfer's BatchMLAPagedAttentionWrapper (fa2), held to the same bound as the reference"""
    fi = flashinfer_mla_or_skip()
    qo_lens = qo if isinstance(qo, list) else [qo] * len(kv)
    causal = max(qo_lens) > 1
    c = make_mla_case(kv, qo_lens, H, page=page, seed=H + len(kv) + page)
    d = _dev(c)
    ws = torch.empty(128 << 20, dtype=torch.uint8, device=DEV)
    w = fi.mla.BatchMLAPagedAttentionWrapper(ws, backend="fa2")
    w.plan(d["qo_indptr"], d["kv_indptr"], d["kv_indices"], torch.tensor(kv, dtype=torch.int32, device=DEV), H, 512, 64,
           page, causal, SCALE, BF16, BF16)
    q = d["q_input"]
    theirs = w.run(q[..., :512].contiguous(), q[..., 512:].contiguous(), d["ckv"], d["kpe"])
    ours, _ = run_mla(c, causal=causal)
    _, sc = ref_mla(c, causal)
    assert_close_attention(ours, theirs, sc, rtol=RTOL, what=f"mla vs flashinfer H={H} qo={qo}")
