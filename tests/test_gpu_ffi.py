"""GPU parity THROUGH the run-time boundary xLLM uses: the TVM-FFI modules are loaded from the FlashInfer-style
"$OPS/<uri>/<uri>.so" layout and called with the reference's exact argument lists (batch_decode.cpp:64-84,
flashinfer_planinfo.cpp:318-335, batch_prefill.cpp:100-128, batch_chunked_prefill.cpp:63-91)."""
import math
import os

import pytest
import torch

from oracle import ops as O
from tests.test_gpu_decode import make_case
from tests.util import assert_close_attention

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"


def _load(kind, head_dim):
    import tvm_ffi
    from xllm_b200 import build_ffi
    ops_dir = build_ffi.build()
    dec, pre = build_ffi.uris()
    uri = [u for u in (dec if kind == "decode" else pre) if f"head_dim_qk_{head_dim}_" in u][0]
    return tvm_ffi.load_module(os.path.join(ops_dir, uri, uri + ".so"))


def test_ffi_decode_plan_run(built_lib):
    import tvm_ffi
    mod = _load("decode", 128)
    kv_lens, HQ, HKV, D, page = [700, 4096, 1], 28, 4, 128, 128
    q, kc, vc, indptr, indices, last = make_case(kv_lens, HQ, HKV, D, page)
    B = len(kv_lens)
    float_ws = torch.empty(128 << 20, dtype=torch.uint8, device=DEV)          # flashinfer_workspace.cpp:25-39 sizes
    int_ws = torch.empty(8 << 20, dtype=torch.uint8, device=DEV)
    pinned = torch.empty(8 << 20, dtype=torch.uint8).pin_memory()
    empty = torch.empty(0, dtype=BF16, device=DEV)
    out = torch.empty(B, HQ, D, dtype=BF16, device=DEV)
    with tvm_ffi.use_torch_stream():
        plan = mod["plan"](float_ws, int_ws, pinned, indptr, B, HQ, HKV, page, False, -1, 0.0, D, D, empty, empty)
        mod["run"](float_ws, int_ws, plan, q.to(DEV), kc.to(DEV), vc.to(DEV), indptr.to(DEV), indices.to(DEV), last.to(DEV),
                   out, None, 0, -1, True, None, 0.0, 1.0 / math.sqrt(D), 1.0, 1.0 / 10000.0)
    torch.cuda.synchronize()
    qo = torch.arange(B + 1, dtype=torch.int32)
    ref = O.paged_attention(q, kc, vc, qo, indptr, indices, last, 1.0 / math.sqrt(D), causal=False)
    scale = O.paged_attention(q, kc, vc.abs(), qo, indptr, indices, last, 1.0 / math.sqrt(D), causal=False)
    assert_close_attention(out, ref, scale, what="FFI decode run")


def test_ffi_prefill_ragged_and_paged(built_lib):
    import tvm_ffi
    mod = _load("prefill", 128)
    HQ, HKV, D = 28, 4, 128
    g = torch.Generator().manual_seed(3)
    lens = [100, 257]
    T = sum(lens)
    qkv = torch.randn(T, (HQ + 2 * HKV) * D, generator=g).to(BF16)
    cu = torch.tensor([0, 100, 357], dtype=torch.int32)
    q = qkv[:, :HQ * D].reshape(T, HQ, D)
    k = qkv[:, HQ * D:(HQ + HKV) * D].reshape(T, HKV, D)
    v = qkv[:, (HQ + HKV) * D:].reshape(T, HKV, D)
    sc = 1.0 / math.sqrt(D)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    pinned = torch.empty(1 << 20, dtype=torch.uint8).pin_memory()
    d = qkv.to(DEV)
    out = torch.empty(T, HQ, D, dtype=BF16, device=DEV)
    kv_len_arr = torch.tensor(lens, dtype=torch.int32)
    with tvm_ffi.use_torch_stream():
        plan = mod["plan"](ws, ws, pinned, cu, cu, kv_len_arr, T, 2, HQ, HKV, 1, False, D, D, True, -1, -1, False, 0)
        mod["ragged_run"](ws, ws, plan, d[:, :HQ * D].view(T, HQ, D), d[:, HQ * D:(HQ + HKV) * D].view(T, HKV, D),
                          d[:, (HQ + HKV) * D:].view(T, HKV, D), cu.to(DEV), cu.to(DEV), out, None, 1, 0, -1, True,
                          None, None, None, None, None, None, 0.0, sc, 1.0, 1.0 / 10000.0, 0)
    torch.cuda.synchronize()
    ref = O.ragged_prefill_attention(q, k, v, cu, cu, sc, causal=True)
    scale = O.ragged_prefill_attention(q, k, v.abs(), cu, cu, sc, causal=True)
    assert_close_attention(out, ref, scale, what="FFI ragged_run")
    # paged_run: chunked prefill of 64 new tokens on top of 300 cached ones, page_size 16
    page, kv_len, qn = 16, 364, 64
    npg = (kv_len + page - 1) // page
    kc = torch.randn(npg + 3, page, HKV, D, generator=g).to(BF16)
    vc = torch.randn(npg + 3, page, HKV, D, generator=g).to(BF16)
    idx = (torch.randperm(npg + 2, generator=g) + 1)[:npg].to(torch.int32)
    indptr = torch.tensor([0, npg], dtype=torch.int32)
    last = torch.tensor([(kv_len - 1) % page + 1], dtype=torch.int32)
    qo = torch.tensor([0, qn], dtype=torch.int32)
    q2 = torch.randn(qn, HQ, D, generator=g).to(BF16)
    out2 = torch.empty(qn, HQ, D, dtype=BF16, device=DEV)
    with tvm_ffi.use_torch_stream():
        plan = mod["plan"](ws, ws, pinned, qo, indptr, torch.tensor([kv_len], dtype=torch.int32), qn, 1, HQ, HKV, page, False, D,
                           D, True, -1, -1, False, 0)
        mod["paged_run"](ws, ws, plan, q2.to(DEV), kc.to(DEV), vc.to(DEV), qo.to(DEV), indptr.to(DEV), idx.to(DEV), last.to(DEV),
                         out2, None, 1, 0, -1, True, None, None, None, None, None, None, 0.0, sc, 1.0, 1.0 / 10000.0, 0)
    torch.cuda.synchronize()
    ref2 = O.paged_attention(q2, kc, vc, qo, indptr, idx, last, sc, causal=True)
    scale2 = O.paged_attention(q2, kc, vc.abs(), qo, indptr, idx, last, sc, causal=True)
    assert_close_attention(out2, ref2, scale2, what="FFI paged_run")


def test_ffi_prefill_sm90_ragged_run(built_lib):
    """the "_sm90" ragged-prefill module an sm90a device asks for (backend "fa3"): plan without the split arguments
    (flashinfer_planinfo.cpp:119-137) and ragged_run with FlashInfer's FA3 argument list (batch_prefill.cpp:135-158)."""
    import tvm_ffi
    from xllm_b200 import build_ffi
    ops_dir = build_ffi.build()
    HQ, HKV, D = 28, 4, 128
    uri = [u for u in build_ffi.uris_sm90() if f"head_dim_qk_{D}_" in u][0]
    mod = tvm_ffi.load_module(os.path.join(ops_dir, uri, uri + ".so"))
    g = torch.Generator().manual_seed(4)
    lens = [300, 1, 777]
    T = sum(lens)
    qkv = torch.randn(T, (HQ + 2 * HKV) * D, generator=g).to(BF16)
    cu = torch.tensor([0, 300, 301, 1078], dtype=torch.int32)
    q = qkv[:, :HQ * D].reshape(T, HQ, D)
    k = qkv[:, HQ * D:(HQ + HKV) * D].reshape(T, HKV, D)
    v = qkv[:, (HQ + HKV) * D:].reshape(T, HKV, D)
    sc = 1.0 / math.sqrt(D)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    pinned = torch.empty(1 << 20, dtype=torch.uint8).pin_memory()
    d = qkv.to(DEV)
    out = torch.empty(T, HQ, D, dtype=BF16, device=DEV)
    lse = torch.empty(T, HQ, dtype=torch.float32, device=DEV)
    with tvm_ffi.use_torch_stream():
        plan = mod["plan"](ws, ws, pinned, cu, cu, torch.tensor(lens, dtype=torch.int32), T, len(lens), HQ, HKV, 1, False, D, D,
                           True, -1)
        mod["ragged_run"](ws, ws, plan, d[:, :HQ * D].view(T, HQ, D), d[:, HQ * D:(HQ + HKV) * D].view(T, HKV, D),
                          d[:, (HQ + HKV) * D:].view(T, HKV, D), cu.to(DEV), cu.to(DEV), out, lse, 1, 0, -1, True,
                          None, None, None, None, 0.0, sc, 1.0, 0)
    torch.cuda.synchronize()
    ref = O.ragged_prefill_attention(q, k, v, cu, cu, sc, causal=True)
    scale = O.ragged_prefill_attention(q, k, v.abs(), cu, cu, sc, causal=True)
    assert_close_attention(out, ref, scale, what="FFI sm90 ragged_run")
    assert torch.isfinite(lse).all()


def _ws():
    float_ws = torch.empty(128 << 20, dtype=torch.uint8, device=DEV)          # flashinfer_workspace.cpp:25-39 sizes
    int_ws = torch.empty(8 << 20, dtype=torch.uint8, device=DEV)
    pinned = torch.empty(8 << 20, dtype=torch.uint8).pin_memory()
    return float_ws, int_ws, pinned


def _time_us(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def test_ffi_paged_run_one_row_is_the_decode_kernel(built_lib):
    """The unmodified reference serves Qwen2-7B decode (GQA group 7 >= 4) through the PREFILL module:
    batch_decode.cpp:43-60 -> batch_chunked_prefill.cpp:63-91 with qo_indptr = arange and causal=False.  That call must
    land on the split-KV streaming kernel: same result as the oracle, and within 1.3x of the decode module's `run`."""
    import tvm_ffi
    dec, pre = _load("decode", 128), _load("prefill", 128)
    kv_lens, HQ, HKV, D, page = [4096], 28, 4, 128, 128
    q, kc, vc, indptr, indices, last = make_case(kv_lens, HQ, HKV, D, page)
    B = 1
    sc = 1.0 / math.sqrt(D)
    f1, i1, pin = _ws()
    f2, i2, _ = _ws()
    empty = torch.empty(0, dtype=BF16, device=DEV)
    qd, kcd, vcd = q.to(DEV), kc.to(DEV), vc.to(DEV)
    ipd, ixd, lad = indptr.to(DEV), indices.to(DEV), last.to(DEV)
    qo = torch.arange(B + 1, dtype=torch.int32)
    qod = qo.to(DEV)
    out_d = torch.empty(B, HQ, D, dtype=BF16, device=DEV)
    out_p = torch.empty(B, HQ, D, dtype=BF16, device=DEV)
    kv_len_arr = torch.tensor(kv_lens, dtype=torch.int32)
    with tvm_ffi.use_torch_stream():
        plan_d = dec["plan"](f1, i1, pin, indptr, B, HQ, HKV, page, False, -1, 0.0, D, D, empty, empty)
        plan_p = pre["plan"](f2, i2, pin, qo, indptr, kv_len_arr, B, B, HQ, HKV, page, False, D, D, False, -1, -1, False, 0)
        assert len(plan_p) == 14 and plan_p[5] == 1, "one-row batches must be planned for the decode kernel"
        run_d = lambda: dec["run"](f1, i1, plan_d, qd, kcd, vcd, ipd, ixd, lad, out_d, None, 0, -1, True, None, 0.0, sc, 1.0, 1e-4)
        run_p = lambda: pre["paged_run"](f2, i2, plan_p, qd, kcd, vcd, qod, ipd, ixd, lad, out_p, None, 0, 0, -1, True,
                                         None, None, None, None, None, None, 0.0, sc, 1.0, 1e-4, 0)
        run_d(); run_p()
        torch.cuda.synchronize()
        t_d, t_p = _time_us(run_d), _time_us(run_p)
    ref = O.paged_attention(q, kc, vc, qo, indptr, indices, last, sc, causal=False)
    scale = O.paged_attention(q, kc, vc.abs(), qo, indptr, indices, last, sc, causal=False)
    assert_close_attention(out_p, ref, scale, what="FFI paged_run one-row (decode through the prefill module)")
    assert torch.equal(out_p, out_d), "paged_run(one row) and run must be the same kernel on the same plan"
    assert t_p <= 1.3 * t_d + 2.0, f"paged_run one-row {t_p:.1f} us vs decode run {t_d:.1f} us"


@pytest.mark.parametrize("module", ["decode", "prefill"])
def test_ffi_plan_under_cuda_graph_serves_longer_contexts(module, built_lib):
    """The reference plans once at CUDA-graph capture and replays `run` for later steps with longer contexts
    (flashinfer_attention.cpp:306-311, cuda_graph_executor_impl.cpp:751-822).  Plan at ctx 512 with
    enable_cuda_graph=True, run at ctx 4096 (and at ctx 40): the result must equal the oracle - the kernel derives the
    split size from the live kv_len, nothing is baked in at plan time."""
    import tvm_ffi
    mod = _load(module, 128)
    HQ, HKV, D, page = 28, 4, 128, 128
    sc = 1.0 / math.sqrt(D)
    B = 2
    fws, iws, pin = _ws()
    empty = torch.empty(0, dtype=BF16, device=DEV)
    qo = torch.arange(B + 1, dtype=torch.int32)
    plan_lens = [512, 300]
    _, _, _, indptr_plan, _, _ = make_case(plan_lens, HQ, HKV, D, page)
    with tvm_ffi.use_torch_stream():
        if module == "decode":
            plan = mod["plan"](fws, iws, pin, indptr_plan, B, HQ, HKV, page, True, -1, 0.0, D, D, empty, empty)
        else:
            plan = mod["plan"](fws, iws, pin, qo, indptr_plan, torch.tensor(plan_lens, dtype=torch.int32), B, B, HQ, HKV, page,
                               True, D, D, False, -1, -1, False, 0)
        for kv_lens in ([4096, 1000], [40, 2], [8192, 129]):
            q, kc, vc, indptr, indices, last = make_case(kv_lens, HQ, HKV, D, page)
            out = torch.empty(B, HQ, D, dtype=BF16, device=DEV)
            args = (q.to(DEV), kc.to(DEV), vc.to(DEV))
            for rep in range(2):                      # twice: the split tickets must be restored between launches
                if module == "decode":
                    mod["run"](fws, iws, plan, *args, indptr.to(DEV), indices.to(DEV), last.to(DEV), out, None, 0, -1, True,
                               None, 0.0, sc, 1.0, 1e-4)
                else:
                    mod["paged_run"](fws, iws, plan, *args, qo.to(DEV), indptr.to(DEV), indices.to(DEV), last.to(DEV), out, None,
                                     0, 0, -1, True, None, None, None, None, None, None, 0.0, sc, 1.0, 1e-4, 0)
            torch.cuda.synchronize()
            ref = O.paged_attention(q, kc, vc, qo, indptr, indices, last, sc, causal=False)
            scale = O.paged_attention(q, kc, vc.abs(), qo, indptr, indices, last, sc, causal=False)
            assert_close_attention(out, ref, scale, what=f"{module} module, graph-time plan at {plan_lens}, run at {kv_lens}")


def test_ffi_paged_run_splits_kv_for_short_chunks(built_lib):
    """chunked prefill of a 16-token chunk over 6000 cached tokens through the prefill module: `plan` must decide a
    KV split (the reference's planner does, flashinfer_planinfo.cpp:168-247) and `paged_run` must match the oracle."""
    import tvm_ffi
    mod = _load("prefill", 128)
    HQ, HKV, D, page = 28, 4, 128, 16
    g = torch.Generator().manual_seed(23)
    kv_len, qn = 6016, 16
    npg = (kv_len + page - 1) // page
    kc = torch.randn(npg + 3, page, HKV, D, generator=g).to(BF16)
    vc = torch.randn(npg + 3, page, HKV, D, generator=g).to(BF16)
    idx = (torch.randperm(npg + 2, generator=g) + 1)[:npg].to(torch.int32)
    indptr = torch.tensor([0, npg], dtype=torch.int32)
    last = torch.tensor([(kv_len - 1) % page + 1], dtype=torch.int32)
    qo = torch.tensor([0, qn], dtype=torch.int32)
    q = torch.randn(qn, HQ, D, generator=g).to(BF16)
    out = torch.empty(qn, HQ, D, dtype=BF16, device=DEV)
    sc = 1.0 / math.sqrt(D)
    fws, iws, pin = _ws()
    with tvm_ffi.use_torch_stream():
        plan = mod["plan"](fws, iws, pin, qo, indptr, torch.tensor([kv_len], dtype=torch.int32), qn, 1, HQ, HKV, page, False, D, D,
                           True, -1, -1, False, 0)
        assert len(plan) == 7 and plan[5] == 0 and plan[6] > 1, f"expected a KV split for 4 CTAs of work, plan = {list(plan)}"
        mod["paged_run"](fws, iws, plan, q.to(DEV), kc.to(DEV), vc.to(DEV), qo.to(DEV), indptr.to(DEV), idx.to(DEV), last.to(DEV),
                         out, None, 1, 0, -1, True, None, None, None, None, None, None, 0.0, sc, 1.0, 1.0 / 10000.0, 0)
    torch.cuda.synchronize()
    ref = O.paged_attention(q, kc, vc, qo, indptr, idx, last, sc, causal=True)
    scale = O.paged_attention(q, kc, vc.abs(), qo, indptr, idx, last, sc, causal=True)
    assert_close_attention(out, ref, scale, what="FFI paged_run with split KV")
