"""This library's elementwise kernels against the REFERENCE'S OWN CUDA kernels (activation.cu, norm.cu, rope.cu,
reshape_paged_cache.cu, fp8_quant.cu, fused_qknorm_rope.cu, fp8_scaled_quantize.cpp, moe/moe_fused_topk.cu,
llm_decode_metadata_update.cu).  Their outputs on the seeded inputs of tools/ref_kernel_parity.py are stored as fixed samples
in tests/golden/ref_kernels.npz (made with `python tools/ref_kernel_parity.py --save-golden ...` against the reference's kernels
compiled by oracle/build_ref.py on an H100); the tool reruns this library's kernels on the same inputs in its own process (a
fault inside a kernel must not take the session's CUDA context with it) and reports the comparison per op."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_kernels.npz")
OPS = ["rms_norm", "fused_add_rms_norm", "rms_norm_static_fp8_quant", "fused_add_rms_norm_static_fp8_quant", "static_scaled_fp8_quant",
       "act_and_mul", "rotary_embedding", "reshape_paged_cache", "fused_qk_norm_rope", "fp8_scaled_quantize", "moe_fused_topk_ids",
       "update_llm_decode_metadata"]


@pytest.fixture(scope="module")
def parity(built_lib):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ref_kernel_parity.py"), "--check-golden", GOLDEN], cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert r.returncode == 0 and lines, f"reference-kernel comparison failed (rc {r.returncode}): {r.stderr[-1500:]}"
    d = json.loads(lines[-1])
    assert d["complete"] and d["mode"] == "stored"
    return d["ops"]


@pytest.mark.parametrize("op", OPS)
def test_kernel_is_bit_identical_to_the_reference_kernel(op, parity):
    r = parity[op]
    assert r["cases"] > 0 and not r.get("errors"), f"{op}: {r.get('errors')}"
    assert r["bit_identical"] == r["cases"], f"{op}: {r['bit_identical']} / {r['cases']} cases bit-identical; worst {r['worst']}"


def test_router_weights_match_the_reference_kernel(parity):
    """fp32 routing weights: the reference has two softmax kernels (fused for power-of-two expert counts, generic otherwise) whose
    reductions sum in different orders, so the floating-point bar is 1e-6 relative rather than bit identity (the expert ids - index
    work - are held to identity above)."""
    r = parity["moe_fused_topk_weights"]
    assert r["cases"] > 0 and not r.get("errors"), r.get("errors")
    assert r["bit_identical"] == r["cases"] or r["max_rel_diff"] <= 1e-6, r
