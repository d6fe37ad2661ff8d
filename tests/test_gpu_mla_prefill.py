"""Expanded MLA prefill on the GPU (xb_mla_prefill_expanded_bf16): the up-projection against the oracle's linear, the
192 / 128 attention against tests/mla_expanded_ref.py on the attention bound of tests/util.py, the whole DeepSeek-V3
attention layer in both forms, repeatability, FlashInfer's ragged 192 / 128 prefill on the same inputs, and that lengths
beyond the plan never write past the workspace."""
import pytest
import torch

from oracle import ops as O
from tests import mla_expanded_ref as E
from tests import mla_ref as R
from tests.util import assert_close_attention, assert_close_bf16, assert_close_sum
from xllm_b200 import ops

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"
SCALE = 192 ** -0.5
QO = [1, 37, 128, 300, 1024]
# Elementwise factor of the attention bound, as in tests/test_gpu_mla.py: the kernel and the reference round P to bf16
# against different running maxima, and these cases check 9e6 - 7e7 outputs each, 10-100x more than the GQA attention
# tests, so the tail of that difference reaches past the 2e-3 factor on single elements (1.06x on 1 of 9.2e6 at H = 16,
# page 1); the relative-L2 bar (3e-3) is unchanged.
RTOL = 2.5e-3
HIST = [0, 17, 2000]


def make_case(qo_lens, hists, H, page, seed):
    """paged caches (pages handed out as a random permutation) holding history + the step's tokens, q [T, H, 192],
    kv_b_proj [H * 256, 512]; all on the GPU"""
    g = torch.Generator().manual_seed(seed)
    kv_lens = [q + h for q, h in zip(qo_lens, hists)]
    npg = [(k + page - 1) // page for k in kv_lens]
    n_pages = sum(npg) + 3
    perm = torch.randperm(n_pages, generator=g).to(torch.int32)
    indptr = torch.tensor([0] + torch.tensor(npg).cumsum(0).tolist(), dtype=torch.int32)
    last = torch.tensor([k - (n - 1) * page for k, n in zip(kv_lens, npg)], dtype=torch.int32)
    qo_indptr = torch.tensor([0] + torch.tensor(qo_lens).cumsum(0).tolist(), dtype=torch.int32)
    T = int(qo_indptr[-1])
    c = dict(ckv=torch.randn(n_pages, page, 512, generator=g).to(BF16), kpe=torch.randn(n_pages, page, 64, generator=g).to(BF16),
             q=torch.randn(T, H, 192, generator=g).to(BF16), w=(torch.randn(H * 256, 512, generator=g) * 512 ** -0.5).to(BF16),
             qo_indptr=qo_indptr, kv_indptr=indptr, kv_indices=perm[:int(indptr[-1])].clone(), last=last)
    c = {k: v.to(DEV) for k, v in c.items()}
    c.update(H=H, T=T, qo_lens=qo_lens, kv_lens=kv_lens)
    return c


def run(c, plan=None, ws=None):
    plan = plan or ops.MlaExpandedPlan(c["H"], c["qo_lens"], c["kv_lens"], DEV)
    if ws is None:
        ws = plan.workspace if plan.workspace is not None else torch.empty(plan.workspace_bytes, dtype=torch.uint8, device=DEV)
    out = torch.full((c["T"], c["H"], 128), float("nan"), dtype=BF16, device=DEV)
    ops.mla_prefill_expanded(plan, c["q"], c["ckv"], c["kpe"], c["qo_indptr"], c["kv_indptr"], c["kv_indices"], c["last"],
                             c["w"], SCALE, out, workspace=ws)
    torch.cuda.synchronize()
    return out, plan, ws


def workspace_views(plan, ws):
    """kv_up [total_kv, H, 256] and kpe [total_kv, 64] at the offsets include/xllm_b200_ops.h documents"""
    n, H = plan.total_kv, plan.num_heads
    a = lambda x: (x + 255) // 256 * 256
    kv_up = ws[:n * H * 512].view(BF16).view(n, H, 256)
    off = a(n * H * 512) + a(n * 1024)
    return kv_up, ws[off:off + n * 128].view(BF16).view(n, 64)


@pytest.mark.parametrize("page", [1, 16, 64])
@pytest.mark.parametrize("H", [16, 128])
def test_expanded_vs_reference(H, page):
    qo_lens = [q for q in QO for _ in HIST]
    hists = [h for _ in QO for h in HIST]
    c = make_case(qo_lens, hists, H, page, seed=H + page)
    out, plan, ws = run(c)
    kv_up, kpe = workspace_views(plan, ws)
    ckv_r, kpe_r, cu = E.gather_latent(c["ckv"], c["kpe"], c["kv_indptr"], c["kv_indices"], c["last"])
    assert torch.equal(kpe, kpe_r), "gathered k_pe rows"
    up_r = E.up_project(ckv_r, c["w"], H)
    w_abs = c["w"].float().abs().t()
    for r0 in range(0, up_r.shape[0], 2048):      # the |x| |w| scale of the GEMM bound, 2048 rows at a time
        r1 = min(r0 + 2048, up_r.shape[0])
        assert_close_sum(kv_up[r0:r1], up_r[r0:r1], (ckv_r[r0:r1].float().abs() @ w_abs).view(r1 - r0, H, 256), rtol=1e-5,
                         what=f"kv_up rows {r0}.. H={H} page={page}")
    assert_close_bf16(kv_up, up_r, ulps=1e9, rel_l2=1e-3, what=f"kv_up rel L2 H={H} page={page}")
    cu = cu.to(DEV)
    ref = E.expanded_attention(c["q"], kv_up, kpe, c["qo_indptr"], cu, SCALE)
    sc = E.expanded_attention(c["q"], kv_up, kpe, c["qo_indptr"], cu, SCALE, abs_value=True)
    assert_close_attention(out, ref, sc, rtol=RTOL, what=f"expanded attention H={H} page={page}")
    again, _, _ = run(c, plan, ws)
    assert torch.equal(out, again), "two runs of one plan differ"


def test_workspace_bound_when_lengths_exceed_the_plan():
    """a plan made for shorter histories than the device's: nothing past plan.workspace_bytes is written"""
    c = make_case([300, 37], [2000, 17], 16, 16, seed=3)
    small = ops.MlaExpandedPlan(16, [300, 37], [1200, 40], DEV)
    ws = torch.full((small.workspace_bytes + 65536,), 0xA5, dtype=torch.uint8, device=DEV)
    out = torch.zeros(c["T"], 16, 128, dtype=BF16, device=DEV)
    ops.mla_prefill_expanded(small, c["q"], c["ckv"], c["kpe"], c["qo_indptr"], c["kv_indptr"], c["kv_indices"], c["last"],
                             c["w"], SCALE, out, workspace=ws[:small.workspace_bytes])
    torch.cuda.synchronize()
    assert bool((ws[small.workspace_bytes:] == 0xA5).all()), "the sentinels past the workspace were overwritten"


def test_wrapper_rejects_token_counts_other_than_the_plans():
    """q and output must hold the plan's tokens: the attention's q tensor map is sized from the plan"""
    c = make_case([300, 37], [2000, 17], 16, 16, seed=4)
    plan = ops.MlaExpandedPlan(16, c["qo_lens"], c["kv_lens"], DEV)
    out = torch.zeros(c["T"], 16, 128, dtype=BF16, device=DEV)
    args = (c["ckv"], c["kpe"], c["qo_indptr"], c["kv_indptr"], c["kv_indices"], c["last"], c["w"], SCALE)
    with pytest.raises(ops.XllmB200Error, match="tokens"):
        ops.mla_prefill_expanded(plan, c["q"][:-1], *args, out)
    with pytest.raises(ops.XllmB200Error, match="tokens"):
        ops.mla_prefill_expanded(plan, c["q"], *args, out[:-1])


def _layer_weights(H, hidden, q_lora, g):
    w = {"q_a_proj": torch.randn(q_lora, hidden, generator=g) * hidden ** -0.5,
         "q_a_layernorm": 1 + 0.1 * torch.randn(q_lora, generator=g),
         "q_b_proj": torch.randn(H * 192, q_lora, generator=g) * q_lora ** -0.5,
         "kv_a_proj_with_mqa": torch.randn(576, hidden, generator=g) * hidden ** -0.5,
         "kv_a_layernorm": 1 + 0.1 * torch.randn(512, generator=g),
         "kv_b_proj": torch.randn(H * 256, 512, generator=g) * 512 ** -0.5,
         "o_proj": torch.randn(hidden, H * 128, generator=g) * (H * 128) ** -0.5}
    return {k: v.to(BF16) for k, v in w.items()}


def _gpu_layer(w, x, pos, cs, slots, ckv, kpe, qo_indptr, indptr, indices, last, H, eps, qo_lens, kv_lens, form):
    """the DeepSeek-V3 attention layer on the library's kernels: projections on xb_gemm_bf16 (oracle-equal linears),
    writer, then the expanded form (raw q, o_proj on o) or the absorbed one (q_nope W_UK, o W_UV)"""
    T = x.shape[0]
    lin = _gemm
    qa = torch.empty(T, w["q_a_proj"].shape[0], dtype=BF16, device=DEV)
    ops.rms_norm(qa, lin(x, w["q_a_proj"]), w["q_a_layernorm"], eps)
    q = lin(qa, w["q_b_proj"]).view(T, H, 192)
    ops.rotary_embedding(pos, q[..., 128:], None, cs, is_neox=False)
    ops.mla_cache_latent(lin(x, w["kv_a_proj_with_mqa"]), w["kv_a_layernorm"], eps, pos, cs, slots, ckv, kpe, interleaved=True)
    if form == "expanded":
        plan = ops.MlaExpandedPlan(H, qo_lens, kv_lens, DEV)
        o = torch.empty(T, H, 128, dtype=BF16, device=DEV)
        ws = torch.empty(plan.workspace_bytes, dtype=torch.uint8, device=DEV)
        ops.mla_prefill_expanded(plan, q, ckv, kpe, qo_indptr, indptr, indices, last, w["kv_b_proj"], SCALE, o, workspace=ws)
        return lin(o.view(T, H * 128), w["o_proj"])
    kv_b = w["kv_b_proj"].view(H, 256, 512)
    q_abs = torch.bmm(q[..., :128].transpose(0, 1).float(), kv_b[:, :128].float()).transpose(0, 1).to(BF16)
    plan = ops.MlaPlan(len(qo_lens), H, max(qo_lens), ckv.shape[1], max(-(-k // ckv.shape[1]) for k in kv_lens), DEV)
    o = torch.empty(T, H, 512, dtype=BF16, device=DEV)
    ops.mla_paged_attention(plan, q_abs, q[..., 128:], ckv, kpe, qo_indptr, indptr, indices, last, SCALE, o, causal=True)
    ov = torch.bmm(o.transpose(0, 1).float(), kv_b[:, 128:].float().transpose(1, 2)).transpose(0, 1).to(BF16)
    return lin(ov.reshape(T, H * 128), w["o_proj"])


def _gemm(a, b):
    a = a.contiguous()
    y = torch.empty(a.shape[0], b.shape[0], dtype=BF16, device=DEV)
    ops.check(ops.lib().xb_gemm_bf16(ops._p(y), ops.c_i64(b.shape[0]), ops._p(a), ops.c_i64(a.shape[1]), ops._p(b),
                                     ops.c_ptr(0), ops.c_i32(a.shape[0]), ops.c_i32(b.shape[0]), ops.c_i32(a.shape[1]),
                                     ops._stream()), "gemm")
    return y


def test_layer_both_forms_vs_reference():
    """a ragged prompt batch and a chunk over history through the whole layer on the GPU, in both forms, against the CPU
    reference layers (tests.mla_ref / tests.mla_expanded_ref) and against each other; bounds of
    tests/test_mla_expanded_cpu.py (both bf16 forms sit about 5e-3 from the fp32 layer)"""
    H, hidden, page, eps = 16, 512, 16, 1e-6
    g = torch.Generator().manual_seed(21)
    w = _layer_weights(H, hidden, 256, g)
    cs = O.compute_cos_sin_cache(64, 4096, 10000)
    hist, qo_lens = [0, 0, 700], [300, 129, 200]
    kv_lens = [h + q for h, q in zip(hist, qo_lens)]
    npg = [-(-k // page) for k in kv_lens]
    pages = torch.randperm(sum(npg) + 2, generator=g)[:sum(npg)].to(torch.int32)
    indptr = torch.tensor([0] + torch.tensor(npg).cumsum(0).tolist(), dtype=torch.int32)
    last = torch.tensor([k - (n - 1) * page for k, n in zip(kv_lens, npg)], dtype=torch.int32)
    qo_indptr = torch.tensor([0] + torch.tensor(qo_lens).cumsum(0).tolist(), dtype=torch.int32)
    ckv0 = torch.randn(sum(npg) + 2, page, 512, generator=g).to(BF16)     # request 2's history is already cached
    kpe0 = torch.randn(sum(npg) + 2, page, 64, generator=g).to(BF16)
    x = torch.randn(sum(qo_lens), hidden, generator=g).to(BF16)
    pos = torch.tensor([p for h, q in zip(hist, qo_lens) for p in range(h, h + q)], dtype=torch.int64)
    slots = torch.tensor([int(pages[int(indptr[b]) + p // page]) * page + p % page
                          for b, (h, q) in enumerate(zip(hist, qo_lens)) for p in range(h, h + q)], dtype=torch.int32)
    args = (qo_indptr, indptr, pages, last, H, 128, 128, eps, SCALE)
    ref = {}
    for form, fn in (("absorbed", R.mla_attention_layer), ("expanded", E.mla_attention_layer_expanded)):
        ref[form] = fn(w, x, pos, cs, slots, ckv0.clone(), kpe0.clone(), *args).float()
    d = lambda t: t.to(DEV)
    got = {}
    for form in ("expanded", "absorbed"):
        got[form] = _gpu_layer({k: d(v) for k, v in w.items()}, d(x), d(pos), d(cs), d(slots), d(ckv0), d(kpe0),
                               d(qo_indptr), d(indptr), d(pages), d(last), H, eps, qo_lens, kv_lens, form).float().cpu()
    rel = lambda a, b: ((a - b).norm() / b.norm()).item()
    bf16_form = rel(ref["expanded"], ref["absorbed"])       # the two reference forms' own bf16 difference
    assert bf16_form < 1e-2
    print("layer rel-L2: forms (reference)", bf16_form, "gpu vs reference", {f: rel(got[f], ref[f]) for f in got},
          "gpu forms", rel(got["expanded"], got["absorbed"]))
    for form in ("expanded", "absorbed"):
        assert rel(got[form], ref[form]) <= bf16_form, (form, rel(got[form], ref[form]), bf16_form)
    assert rel(got["expanded"], got["absorbed"]) <= 1.1 * bf16_form, (rel(got["expanded"], got["absorbed"]), bf16_form)


def flashinfer_ragged_or_skip():
    """FlashInfer's fa2 ragged prefill module with head_dim_qk 192 / head_dim_vo 128 (pre-built by
    tools/build_flashinfer_cache.py, or JIT-built here within 300 s); skips only when it cannot be built"""
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
        spec = FIC.mla_prefill_specs()[0]
    except Exception as e:  # pragma: no cover
        pytest.skip(f"flashinfer not importable: {e}")
    if not spec.jit_library_path.exists():
        r = subprocess.run(["timeout", "300", sys.executable, os.path.join(root, "tools", "build_flashinfer_cache.py"),
                            "mla_prefill"], capture_output=True, text=True)
        if r.returncode != 0 or not spec.jit_library_path.exists():
            pytest.skip("FlashInfer ragged 192/128 prefill module not pre-built and JIT did not finish in 300 s")
    if not getattr(jc.JitSpec, "_xb_patched", False):
        orig = jc.JitSpec.build

        def build(self, verbose, need_lock=True):      # a pre-built library is loaded as is
            if self.jit_library_path.exists():
                return None
            return orig(self, verbose, need_lock)
        jc.JitSpec.build = build
        jc.JitSpec._xb_patched = True
    return flashinfer


@pytest.mark.parametrize("H", [16, 128])
def test_expanded_vs_flashinfer(H):
    """the same inputs through FlashInfer's BatchPrefillWithRaggedKVCacheWrapper (fa2, qk 192 / vo 128), fed
    K = [k_nope | broadcast k_pe] and V from the kernel's own up-projection; held to the reference bound"""
    fi = flashinfer_ragged_or_skip()
    c = make_case([1024, 37, 300], [0, 2000, 17], H, 16, seed=40 + H)
    out, plan, ws = run(c)
    kv_up, kpe = workspace_views(plan, ws)
    k = torch.cat([kv_up[..., :128], kpe[:, None].expand(-1, H, -1)], -1).contiguous()
    v = kv_up[..., 128:].contiguous()
    _, _, cu = E.gather_latent(c["ckv"], c["kpe"], c["kv_indptr"], c["kv_indices"], c["last"])
    cu = cu.to(DEV)
    wrapper = fi.BatchPrefillWithRaggedKVCacheWrapper(torch.empty(128 << 20, dtype=torch.uint8, device=DEV), "NHD",
                                                      backend="fa2")
    wrapper.plan(c["qo_indptr"], cu, H, H, 192, head_dim_vo=128, causal=True, sm_scale=SCALE, q_data_type=BF16)
    theirs = wrapper.run(c["q"], k, v)
    sc = E.expanded_attention(c["q"], kv_up, kpe, c["qo_indptr"], cu, SCALE, abs_value=True)
    assert_close_attention(out, theirs, sc, rtol=RTOL, what=f"expanded vs flashinfer H={H}")
