"""Group sizes the weight-only linears cannot index are refused before any CUDA call (no device needed: the C ABI is called
with null data pointers).  A group must be a power-of-two number of k64 tiles dividing K (and hidden / inter for the
experts); anything else would have the kernels apply scales on 64- or 128-wide groups and read meta rows past K / group.
192 on the W4 small-M entry is refused only after the device's SM count is read: tests/test_gpu_linear_edges.py."""
import ctypes
import re

import pytest

NULL = ctypes.c_void_p(0)
# (group_size, K): not positive, below 64, not a multiple of 64 (96 and 160 pass every other check), not a power-of-two
# number of k64 tiles, not dividing K
BAD_GROUPS = [(0, 384), (-1, 384), (32, 384), (96, 384), (160, 960), (192, 384), (256, 384)]


@pytest.fixture(scope="module")
def L(built_lib):
    from xllm_b200 import _lib
    return _lib.lib()


def _linear(fn):
    return lambda M, N, K, gs: fn(NULL, ctypes.c_int64(N), NULL, ctypes.c_int64(K), NULL, NULL, NULL, M, N, K, gs, NULL)


def _moe(L):
    def call(M, N, K, gs):
        return L.xb_moe_experts_w4a16(NULL, ctypes.c_int64(K), NULL, ctypes.c_int64(K), NULL, NULL, NULL, NULL, NULL, NULL, gs,
                                      M, 2, K, K, 4, 0, NULL, ctypes.c_int64(0), NULL)
    return call


ENTRIES = {
    "xb_linear_w4a16_small_m": (lambda L: _linear(L.xb_linear_w4a16_small_m), 1),
    "xb_linear_w8a16_small_m": (lambda L: _linear(L.xb_linear_w8a16_small_m), 1),
    "xb_gemm_w4a16": (lambda L: _linear(L.xb_gemm_w4a16), 300),
    "xb_gemm_w8a16": (lambda L: _linear(L.xb_gemm_w8a16), 300),
    "xb_moe_experts_w4a16 (expert GEMVs)": (_moe, 3),
    "xb_moe_experts_w4a16 (grouped GEMMs)": (_moe, 300),
}


@pytest.mark.parametrize("gs,K", BAD_GROUPS)
@pytest.mark.parametrize("entry", list(ENTRIES))
def test_bad_group_size_is_rejected(entry, gs, K, L):
    from xllm_b200._lib import XllmB200Error, check
    if entry == "xb_linear_w4a16_small_m" and gs == 192:
        pytest.skip("refused after the SM count is read: tests/test_gpu_linear_edges.py::test_w4_small_m_rejects_group_192")
    make, M = ENTRIES[entry]
    n0 = L.xb_launch_count()
    with pytest.raises(XllmB200Error) as e:
        check(make(L)(M, 128, K, gs), entry)
    msg = str(e.value)
    assert re.search(rf"group_size {gs}\b|\(got {gs}\)", msg), f"{entry}: the message does not name the group size: {msg}"
    assert L.xb_launch_count() == n0
