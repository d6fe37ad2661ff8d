"""Pins the attention kernels against FlashInfer itself - the library whose fa2 kernels the reference dlopen()s for
batch_decode / batch_prefill / batch_chunked_prefill (xllm/core/kernels/cuda/utils.cpp:371-450; reference pin v0.6.2,
this image ships flashinfer-python 0.6.11 with the same fa2 templates).  The oracle's attention ladder is a restatement
of FlashInfer's published algorithm; on a GPU box this test replaces "parity unpinned" (DESIGN.md section 2) by a direct
comparison on the same seeded inputs.

Gate = capability probe, not an environment switch: the FlashInfer modules are pre-built with nvcc on the authoring
machine into baseline/_fi/ (tools/build_flashinfer_cache.py; git-ignored, travels with the snapshot).  If a module is
absent the probe tries to JIT it under `timeout 300`; the test skips only if that cannot build.
"""
import math
import os
import subprocess
import sys

import pytest
import torch

from oracle import ops as O
from tests.test_gpu_decode import make_case
from tests.util import assert_close_attention

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import build_flashinfer_cache as FIC  # noqa: E402

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"
_probe = {}


def flashinfer_or_skip(head_dim):
    """import flashinfer with its JIT workspace pointed at baseline/_fi and make sure the fa2 decode + prefill modules of
    this head_dim exist (pre-built, or JIT-able within 300 s)."""
    if head_dim in _probe:
        if _probe[head_dim] is not None:
            pytest.skip(_probe[head_dim])
        import flashinfer
        return flashinfer
    FIC.set_env()
    try:
        import flashinfer
        from flashinfer.jit import core as jc
    except Exception as e:  # pragma: no cover
        _probe[head_dim] = f"flashinfer not importable: {e}"
        pytest.skip(_probe[head_dim])
    missing = [s for s in FIC.specs((head_dim,)) if not s.jit_library_path.exists()]
    if missing:
        r = subprocess.run(["timeout", "300", sys.executable, os.path.join(ROOT, "tools", "build_flashinfer_cache.py"),
                            str(head_dim)], capture_output=True, text=True)
        if r.returncode != 0 or any(not s.jit_library_path.exists() for s in missing):
            _probe[head_dim] = f"FlashInfer fa2 modules (head_dim {head_dim}) not pre-built and JIT did not finish in 300 s"
            pytest.skip(_probe[head_dim])
    if not getattr(jc.JitSpec, "_xb_patched", False):
        orig = jc.JitSpec.build

        def build(self, verbose, need_lock=True):      # a pre-built library is loaded as is (no ninja re-check on the box)
            if self.jit_library_path.exists():
                return None
            return orig(self, verbose, need_lock)
        jc.JitSpec.build = build
        jc.JitSpec._xb_patched = True
    _probe[head_dim] = None
    return flashinfer


def _p_abs_v_scale(q, kc, vc, indptr, indices, last, sm_scale):
    """sum_j p_j |v_j| per output element (the forward-error scale of tests/util.py): the oracle run on |V|."""
    qo = torch.arange(q.shape[0] + 1, dtype=torch.int32)
    return O.paged_attention(q, kc, vc.abs(), qo, indptr, indices, last, sm_scale, causal=False)


@pytest.mark.parametrize("kv_lens,HQ,HKV,D,page", [([4096], 28, 4, 128, 128), ([17, 700, 1, 129, 2048], 28, 4, 128, 16),
                                                   ([1000, 31], 8, 8, 128, 32), ([333, 64], 14, 2, 64, 16)])
@pytest.mark.parametrize("tensor_cores", [False, True])
def test_decode_matches_flashinfer(kv_lens, HQ, HKV, D, page, tensor_cores, built_lib):
    """tensor_cores=True is the path the reference takes for GQA group >= 4 (utils.cpp:349-367 -> batch_decode.cpp:43-60:
    decode served by the fa2 prefill kernel, causal=False); tensor_cores=False is FlashInfer's CUDA-core decode kernel."""
    flashinfer = flashinfer_or_skip(D)
    from xllm_b200 import ops
    if not tensor_cores and HQ // HKV not in (1, 2, 3, 4, 8):
        pytest.skip(f"FlashInfer's CUDA-core decode kernel is not instantiated for GQA group {HQ // HKV} (batch_decode.cu: "
                    "'Unsupported group_size') - the reference never takes that path for such models (utils.cpp:349-367)")
    q, kc, vc, indptr, indices, last = make_case(kv_lens, HQ, HKV, D, page)
    B = len(kv_lens)
    sm_scale = 1.0 / math.sqrt(D)
    qd, kcd, vcd = q.to(DEV), kc.to(DEV), vc.to(DEV)
    ws = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    w = flashinfer.BatchDecodeWithPagedKVCacheWrapper(ws, "NHD", use_tensor_cores=tensor_cores)
    w.plan(indptr.to(DEV), indices.to(DEV), last.to(DEV), HQ, HKV, D, page, pos_encoding_mode="NONE", q_data_type=BF16,
           kv_data_type=BF16, sm_scale=sm_scale)
    ref = w.run(qd, (kcd, vcd))
    max_pages = int((indptr[1:] - indptr[:-1]).max())
    plan = ops.DecodePlan(B, HQ, HKV, D, page, max_pages, DEV)
    out = torch.empty(B, HQ, D, dtype=BF16, device=DEV)
    ops.batch_decode(plan, qd, kcd, vcd, indptr.to(DEV), indices.to(DEV), last.to(DEV), sm_scale, out, None)
    torch.cuda.synchronize()
    scale = _p_abs_v_scale(q, kc, vc, indptr, indices, last, sm_scale)
    # FlashInfer's CUDA-core decode kernel keeps P in fp32 (no bf16 rounding of P), its tensor-core path rounds P like
    # ours: both are within the same forward-error bound of our result
    # two different kernels, each with its own bf16 roundings of P (and FlashInfer's own split-KV merge): see tests/util.py
    # for the 2.35e-3 analytic floor of two independent implementations
    assert_close_attention(out, ref, scale, rtol=2e-3, rel_l2=4e-3, what=f"decode vs flashinfer {kv_lens} (tensor_cores={tensor_cores})")
    # and the oracle agrees with FlashInfer to the same bar: this is what pins the oracle's attention ladder
    qo = torch.arange(B + 1, dtype=torch.int32)
    orc = O.paged_attention(q, kc, vc, qo, indptr, indices, last, sm_scale, causal=False)
    assert_close_attention(orc, ref, scale, rtol=2e-3, rel_l2=4e-3, what=f"oracle vs flashinfer {kv_lens} (tensor_cores={tensor_cores})")


@pytest.mark.parametrize("lens,HQ,HKV,D", [([2048], 28, 4, 128), ([128, 77, 300], 28, 4, 128), ([1024], 14, 2, 64)])
def test_ragged_prefill_matches_flashinfer(lens, HQ, HKV, D, built_lib):
    flashinfer = flashinfer_or_skip(D)
    from xllm_b200 import ops
    g = torch.Generator().manual_seed(2026)
    T = sum(lens)
    q = torch.randn(T, HQ, D, generator=g).to(BF16)
    k = torch.randn(T, HKV, D, generator=g).to(BF16)
    v = torch.randn(T, HKV, D, generator=g).to(BF16)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0).tolist()), dtype=torch.int32)
    sm_scale = 1.0 / math.sqrt(D)
    ws = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    w = flashinfer.BatchPrefillWithRaggedKVCacheWrapper(ws, "NHD", backend="fa2")
    w.plan(cu.to(DEV), cu.to(DEV), HQ, HKV, D, causal=True, pos_encoding_mode="NONE", sm_scale=sm_scale, q_data_type=BF16,
           kv_data_type=BF16)
    ref = w.run(q.to(DEV), k.to(DEV), v.to(DEV))
    out = torch.empty(T, HQ, D, dtype=BF16, device=DEV)
    ops.batch_prefill(q.to(DEV), k.to(DEV), v.to(DEV), cu.to(DEV), cu.to(DEV), sm_scale, out, None, max_qo_len=max(lens))
    torch.cuda.synchronize()
    scale = O.ragged_prefill_attention(q, k, v.abs(), cu, cu, sm_scale, causal=True)
    assert_close_attention(out, ref, scale, rtol=2e-3, what=f"ragged prefill vs flashinfer {lens}")
    orc = O.ragged_prefill_attention(q, k, v, cu, cu, sm_scale, causal=True)
    assert_close_attention(orc, ref, scale, rtol=2e-3, what=f"oracle ragged prefill vs flashinfer {lens}")
