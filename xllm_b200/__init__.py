"""xllm_b200: H100-native (sm_90a) implementation of xLLM's per-layer inference hot path.

The product is the C-ABI library `xllm_b200/lib/libxllm_b200_ops.so`
(include/xllm_b200_ops.h).  This package is the host-side mirror of the
reference's operator interface (`xllm::kernel::cuda::*`,
xllm/core/kernels/cuda/cuda_ops_api.h) on top of that C ABI: same names,
argument meaning and error behaviour, torch tensors only as device-memory
handles.  There is no CPU fallback: every op raises if the library is missing
or the tensors are not on a CUDA device.
"""
from . import _lib  # noqa: F401

__all__ = ["_lib"]
