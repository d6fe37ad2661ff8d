"""The NVLink exchange entry points refuse arguments their kernels cannot run on before any launch (no device needed: the
C ABI is called with fake device pointers that nothing dereferences).  The kernels move data as uint4 and signals as
uint32, so a misaligned pointer would fault the GPU; a negative size or an empty flag pad would launch a kernel that
signals on slots the caller does not own.  Each refusal must name the offending value and launch nothing.

Cases a missing check would let through to a launch on fake pointers are skipped where a GPU is present, since there that
launch would fault instead of returning an error.  tests/test_gpu_peer_exchange.py checks the size refusals with real
buffers; the alignment refusals are checked only here."""
import ctypes
import re

import pytest
import torch

NULL = ctypes.c_void_p(0)
DATA, FLAGS, EPOCH, OUT, RES, WEIGHT = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
W = 4


@pytest.fixture(scope="module")
def L(built_lib):
    from xllm_b200 import _lib
    return _lib.lib()


def _arrays(world, data=None, flags=None):
    n = max(world, 1)
    d = [DATA + 0x1000 * r for r in range(n)]
    f = [FLAGS + 0x1000 * r for r in range(n)]
    for r, p in (data or {}).items():
        d[r] = p
    for r, p in (flags or {}).items():
        f[r] = p
    return (ctypes.c_void_p * n)(*d), (ctypes.c_void_p * n)(*f)


def oneshot(L, out=OUT, epoch=EPOCH, rank=0, world=W, numel=4096, max_ctas=64, data=None, flags=None):
    pd, pf = _arrays(world, data, flags)
    return L.xb_oneshot_allreduce_bf16(ctypes.c_void_p(out), pd, pf, ctypes.c_void_p(epoch), ctypes.c_int(rank),
                                       ctypes.c_int(world), ctypes.c_int64(numel), ctypes.c_int(max_ctas), NULL)


def fused(L, out=OUT, residual=RES, weight=WEIGHT, epoch=EPOCH, rank=0, world=W, tokens=4, hidden=896, max_ctas=64,
          data=None, flags=None):
    pd, pf = _arrays(world, data, flags)
    return L.xb_allreduce_add_rms_norm_bf16(ctypes.c_void_p(out), ctypes.c_void_p(residual), ctypes.c_void_p(weight), pd, pf,
                                            ctypes.c_void_p(epoch), ctypes.c_int(rank), ctypes.c_int(world),
                                            ctypes.c_float(1e-6), ctypes.c_int(tokens), ctypes.c_int(hidden),
                                            ctypes.c_int(max_ctas), NULL)


# (id, entry, arguments, regex the message must match, refused by the parent commit's checks)
CASES = [
    ("oneshot numel 12", oneshot, dict(numel=12), r"numel 12\b", True),
    ("oneshot world 0", oneshot, dict(world=0), r"world 0\b", True),
    ("oneshot world 9", oneshot, dict(world=9), r"world 9\b", True),
    ("oneshot rank -1", oneshot, dict(rank=-1), r"rank -1\b", True),
    ("oneshot rank == world", oneshot, dict(rank=W), rf"rank {W}\b", True),
    ("oneshot numel -8", oneshot, dict(numel=-8), r"numel -8\b", False),
    ("oneshot max_ctas 0", oneshot, dict(max_ctas=0), r"max_ctas 0\b", False),
    ("oneshot max_ctas -1", oneshot, dict(max_ctas=-1), r"max_ctas -1\b", False),
    ("oneshot out 0x1002", oneshot, dict(out=0x1002), r"out 0x1002\b", False),
    ("oneshot out 0x40008", oneshot, dict(out=0x40008), r"out 0x40008\b", False),
    ("oneshot peer_data[3] 0x1002", oneshot, dict(data={3: 0x1002}), r"peer_data\[3\] 0x1002\b", False),
    ("oneshot peer_data[0] 0x10008", oneshot, dict(data={0: 0x10008}), r"peer_data\[0\] 0x10008\b", False),
    ("oneshot peer_flags[2] 0x20002", oneshot, dict(flags={2: 0x20002}), r"peer_flags\[2\] 0x20002\b", False),
    ("oneshot epoch 0x30001", oneshot, dict(epoch=0x30001), r"epoch 0x30001\b", False),
    ("fused hidden 12", fused, dict(hidden=12), r"hidden 12\b", True),
    ("fused hidden 16392", fused, dict(hidden=16392), r"hidden 16392\b", True),
    ("fused tokens > max_ctas", fused, dict(tokens=65), r"65 tokens exceed the 64\b", True),
    ("fused world 0", fused, dict(world=0), r"world 0\b", True),
    ("fused world 9", fused, dict(world=9), r"world 9\b", True),
    ("fused rank -1", fused, dict(rank=-1), r"rank -1\b", True),
    ("fused rank == world", fused, dict(rank=W), rf"rank {W}\b", True),
    ("fused hidden 0", fused, dict(hidden=0), r"hidden 0\b", False),
    ("fused hidden -8", fused, dict(hidden=-8), r"hidden -8\b", False),
    ("fused num_tokens -1", fused, dict(tokens=-1), r"num_tokens -1\b", False),
    ("fused out 0x1002", fused, dict(out=0x1002), r"out 0x1002\b", False),
    ("fused residual 0x50008", fused, dict(residual=0x50008), r"residual 0x50008\b", False),
    ("fused weight 0x60004", fused, dict(weight=0x60004), r"weight 0x60004\b", False),
    ("fused peer_data[3] 0x1002", fused, dict(data={3: 0x1002}), r"peer_data\[3\] 0x1002\b", False),
    ("fused peer_flags[1] 0x20001", fused, dict(flags={1: 0x20001}), r"peer_flags\[1\] 0x20001\b", False),
    ("fused epoch 0x30002", fused, dict(epoch=0x30002), r"epoch 0x30002\b", False),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_bad_argument_is_refused_before_launch(case, L):
    from xllm_b200._lib import XllmB200Error, check
    name, entry, kwargs, pattern, checked_before = case
    if not checked_before and torch.cuda.is_available():
        pytest.skip("without this check the call would launch a kernel on fake pointers")
    n0 = L.xb_launch_count()
    with pytest.raises(XllmB200Error) as e:
        check(entry(L, **kwargs), name)
    assert re.search(pattern, str(e.value)), f"{name}: the message does not name the value: {e.value}"
    assert L.xb_launch_count() == n0


def test_empty_exchange_launches_nothing(L):
    """numel == 0 and num_tokens == 0 return before any check or launch, whatever the pointers."""
    n0 = L.xb_launch_count()
    assert oneshot(L, out=0x1002, numel=0) == 0
    assert fused(L, out=0x1002, tokens=0) == 0
    assert L.xb_launch_count() == n0
