"""The shipped library really contains sm_90a tensor-core / TMA code (no GPU needed): cuobjdump of the in-tree
libxllm_b200_ops.so must show the SASS forms of wgmma (HGMMA), TMA tensor loads (UTMALDG),
mbarrier traffic (SYNCS) and the cp.async staging of the small-M kernels (LDGSTS) - in the kernels that are supposed to
use them - and it must be built for sm_90a only."""
import re
import shutil
import subprocess

import pytest

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def _sass_by_kernel(lib):
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    kernels, cur = {}, None
    for line in out.split("\n"):
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = []
        elif cur is not None:
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]+)", line)
            if m:
                kernels[cur].append(m.group(1).split(".")[0])
    return kernels


@pytest.fixture(scope="module")
def sass(built_lib):
    if not shutil.which(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    return _sass_by_kernel(built_lib)


def _ops(sass, name_part):
    sel = {k: set(v) for k, v in sass.items() if name_part in k}
    assert sel, f"no kernel matching {name_part}"
    return sel


def test_built_for_sm90a_only(built_lib):
    out = subprocess.run([CUOBJDUMP, "-lelf", built_lib], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_gemm_kernels_use_wgmma_tma(sass):
    kernels = _ops(sass, "gemm_wgmma_kernel")
    for name, ops in kernels.items():
        assert "HGMMA" in ops, f"{name}: no wgmma"
        assert "UTMALDG" in ops, f"{name}: no TMA tensor load"
        assert "SYNCS" in ops, f"{name}: no mbarrier pipeline"
        assert "HMMA" not in ops, f"{name}: legacy mma.sync in a wgmma kernel"
    fp8 = [k for k in kernels if "gemm_wgmma_kernelILi1E" in k]
    assert fp8, "the FP8 GEMM instantiations must be in the library"
    for k in fp8:
        # converter warps widen e4m3 to fp16 (exact) for the fp32-accumulating fp16 wgmma
        assert "F2FP" in kernels[k], f"{k}: no e4m3 -> f16 conversion"


def test_prefill_attention_uses_wgmma(sass):
    for name, ops in _ops(sass, "prefill_attention_kernel").items():
        assert "HGMMA" in ops and "HMMA" not in ops, name            # S = Q K^T and O += P V both on wgmma
        assert "UTMALDG" in ops and "MUFU" in ops, name


def test_streaming_kernels_shape(sass):
    # HBM-bound small-M kernels: register-resident mma.sync fragments; the W4 kernel stages through cp.async
    for name, ops in _ops(sass, "linear_w4a16_small_m_kernel").items():
        assert "HMMA" in ops and "LDGSTS" in ops and "DEPBAR" in ops, f"{name}: expected mma.sync + cp.async groups"
        assert not (ops & {"HGMMA", "QGMMA"}), name
    for name, ops in _ops(sass, "paged_decode_kernel").items():
        assert "HMMA" in ops and "MUFU" in ops, name
    for name, ops in _ops(sass, "allreduce").items():
        assert not (ops & {"HMMA", "HGMMA"}), name
