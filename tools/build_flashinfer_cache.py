"""Pre-builds (nvcc, no GPU needed) the FlashInfer fa2 modules that tests/test_gpu_flashinfer_pin.py and bench.py's
GPU comparators load, into baseline/_fi/ (git-ignored, travels to the GPU box with the snapshot like our own .so files).

FlashInfer is LIBRARY code here: it is the implementation the reference dlopen()s for batch_decode / batch_prefill /
batch_chunked_prefill (xllm/core/kernels/cuda/utils.cpp:371-450; reference pin v0.6.2, this image ships 0.6.11 with
the same fa2 templates).  It is used only as a checker (tests) and as a same-box comparator (bench), never on the
product path.  On a fresh GPU box the JIT would otherwise spend minutes of charged box time in nvcc per variant.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FI_BASE = os.path.join(ROOT, "baseline", "_fi")


def set_env():
    os.environ["FLASHINFER_WORKSPACE_BASE"] = FI_BASE
    os.environ["FLASHINFER_CUDA_ARCH_LIST"] = "9.0a"


def specs(head_dims=(128, 64)):
    import torch
    from flashinfer.jit.attention.modules import gen_batch_decode_module, gen_batch_prefill_module
    bf, i32 = torch.bfloat16, torch.int32
    out = []
    for d in head_dims:
        out.append(gen_batch_decode_module(bf, bf, bf, i32, d, d, 0, False, False))
        out.append(gen_batch_prefill_module("fa2", bf, bf, bf, i32, d, d, 0, False, False, False))
    return out


def mla_specs():
    """the fa2 batch_mla module BatchMLAPagedAttentionWrapper(backend="fa2") loads for DeepSeek-V2/V3 (ckv 512, kpe 64):
    the comparator of tests/test_gpu_mla.py and tools/mla_sweep.py"""
    import torch
    from flashinfer.jit.attention.modules import gen_batch_mla_module
    bf = torch.bfloat16
    return [gen_batch_mla_module("fa2", bf, bf, bf, torch.int32, 512, 64, False)]


def mla_prefill_specs():
    """the fa2 ragged prefill module BatchPrefillWithRaggedKVCacheWrapper(backend="fa2") loads for DeepSeek-V3's expanded
    MLA prefill (head_dim_qk 192, head_dim_vo 128): the comparator of tests/test_gpu_mla_prefill.py and tools/mla_sweep.py"""
    import torch
    from flashinfer.jit.attention.modules import gen_batch_prefill_module
    bf = torch.bfloat16
    return [gen_batch_prefill_module("fa2", bf, bf, bf, torch.int32, 192, 128, 0, False, False, False)]


def main():
    set_env()
    os.makedirs(FI_BASE, exist_ok=True)
    if sys.argv[1:] == ["mla"]:
        todo = mla_specs()
    elif sys.argv[1:] == ["mla_prefill"]:
        todo = mla_prefill_specs()
    else:
        todo = specs(tuple(int(a) for a in sys.argv[1:]) or (128, 64)) + (mla_specs() + mla_prefill_specs() if not sys.argv[1:] else [])
    for s in todo:
        print("building", s.name, flush=True)
        s.build(verbose=False)
        print("  ->", s.jit_library_path, os.path.getsize(s.jit_library_path) >> 20, "MiB", flush=True)


if __name__ == "__main__":
    main()
