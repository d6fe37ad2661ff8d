import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")
    config.addinivalue_line("markers", "w4_exact: run with the exact-dequant form of the W4A16 decode kernels "
                                       "(xb_set_w4_decode_form(1)); every other GPU test pins the bf16-weight form")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def built_lib():
    """Make sure the C-ABI library exists (builds it with nvcc if not)."""
    from xllm_b200 import build
    return build.build()


@pytest.fixture(autouse=True)
def _pin_w4_decode_form(request):
    """The W4A16 decode kernels have two arithmetic forms (oracle/quant.py).  Every GPU test states which one it checks:
    the bf16-weight form unless marked `w4_exact` - independent of the library's default."""
    import torch
    if "gpu" not in request.keywords or not torch.cuda.is_available():
        yield
        return
    from xllm_b200 import build, ops
    build.build()
    old = ops.set_w4_decode_form(1 if "w4_exact" in request.keywords else 0)
    yield
    ops.set_w4_decode_form(old)
    if ops._splitk_ws is not None:
        # an FP8 runner registered the process-wide split-K workspace: withdraw it so that the next test's FP8 GEMMs do not
        # depend on which tests ran before it
        torch.cuda.synchronize()
        ops.disable_fp8_splitk()


def pytest_sessionfinish(session, exitstatus):
    """keep the measured rel-L2 of every attention / dot-product comparison of the session (the bar is asserted in
    tests/util.py; the log shows the margin)."""
    try:
        from tests.util import REL_L2_LOG
        if REL_L2_LOG:
            os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
            with open(os.path.join(ROOT, "gpurun_out", "rel_l2_log.txt"), "a") as f:
                for what, l2 in REL_L2_LOG:
                    f.write(f"{l2:.3e}\t{what}\n")
    except Exception:
        pass
