"""Host logic of the split-K decision for the decode-sized FP8 GEMM (xb_gemm_fp8_split_k: no device needed): the shapes of the
Llama-3-70B shards, and the invariants the kernel relies on (one wave, no empty k range, >= 12 k blocks per range)."""
import ctypes
import random

import pytest


@pytest.fixture(scope="module")
def L(built_lib):
    lib = ctypes.CDLL(built_lib)
    lib.xb_gemm_fp8_split_k.restype = ctypes.c_int
    lib.xb_gemm_fp8_split_k.argtypes = [ctypes.c_int] * 4
    return lib


def test_split_k_of_the_llama70b_shards(L):
    f = lambda M, N, K: L.xb_gemm_fp8_split_k(M, N, K, 132)
    assert f(32, 1280, 8192) == 5          # qkv TP8 shard: 10 tiles, 64 k blocks -> 5 ranges of 13 (64 / 12 caps it)
    assert f(32, 8192, 1024) == 1          # o_proj TP8 shard: 8 k blocks - splitting measured slower
    assert f(32, 8192, 2048) == 1          # o_proj TP4 shard
    assert f(32, 7168, 8192) == 2          # gate_up TP8 shard: 56 tiles
    assert f(32, 8192, 3584) == 2          # down TP8 shard: 64 tiles, 28 k blocks
    assert f(32, 8192, 28672) == 2         # down unsharded
    assert f(32, 57344, 8192) == 1         # gate_up unsharded: 448 tiles already fill the SMs
    assert f(32, 10240, 8192) == 1         # qkv unsharded: 80 tiles, 2 x 80 > 132
    assert f(65, 1280, 8192) == 1 and f(32, 64, 8192) == 1 and f(0, 1280, 8192) == 1     # not a swap-AB shape


def test_split_k_invariants(L):
    rng = random.Random(2026)
    for _ in range(2000):
        M = rng.randint(1, 64)
        N = rng.choice([128, 256, 1000, 1280, 2560, 4096, 7168, 8192, 14336, 20000])
        K = 16 * rng.randint(1, 4096)
        sms = rng.choice([8, 74, 132, 148, 160])
        s = L.xb_gemm_fp8_split_k(M, N, K, sms)
        assert 1 <= s <= 8
        if s > 1:
            tiles, num_kb = (N + 127) // 128, (K + 127) // 128
            kb_per = (num_kb + s - 1) // s
            assert tiles * s <= sms, "more than one wave"
            assert (s - 1) * kb_per < num_kb, "empty k range"
            assert kb_per >= 12, "range shorter than the TMA ring needs"


def _describe(L, kind, M, N, K, sms=132):
    buf = ctypes.create_string_buffer(96)
    n = L.xb_gemm_describe(kind, M, N, K, sms, buf, 96)
    assert n > 0
    return buf.value.decode()


def test_gemm_dispatch_of_the_baseline_shapes(L):
    """which wgmma variant the GEMM entry points pick (xb_gemm_describe, host-only).  Qwen2-7B prefill at M = 8192 (BASELINE
    configs[2]): 128-column tiles; decode-sized FP8 (configs[3] shards): swap-AB, split-K on the narrow shards."""
    BF16, FP8, W4, W8 = 0, 1, 2, 3
    for kind, name in ((BF16, "bf16"), (FP8, "fp8"), (W4, "w4"), (W8, "w8")):
        assert _describe(L, kind, 8192, 4608, 3584) == f"{name} bn=128"        # qkv
        assert _describe(L, kind, 8192, 37888, 3584) == f"{name} bn=128"       # gate_up
        assert _describe(L, kind, 8192, 3584, 3584) == f"{name} bn=128"        # o
        assert _describe(L, kind, 8192, 3584, 18944) == f"{name} bn=128"       # down
    # too few 128 x 128 tiles to cover the SMs: 64-column tiles
    assert _describe(L, BF16, 300, 4608, 3584) == "bf16 bn=64"
    assert _describe(L, W4, 2048, 1000, 512) == "w4 bn=64"                    # N % 128 != 0
    assert _describe(L, BF16, 17, 152064, 3584) == "bf16 bn=128"              # lm_head of a small batch
    # Llama-3-70B FP8 decode, batch 32
    assert _describe(L, FP8, 32, 1280, 8192) == "fp8 swap-AB bn=32 split_k=5"        # qkv TP8 shard
    assert _describe(L, FP8, 64, 8192, 28672) == "fp8 swap-AB bn=64 split_k=2"       # down unsharded, batch 64
    assert _describe(L, FP8, 32, 57344, 8192) == "fp8 swap-AB bn=32 split_k=1"       # gate_up unsharded
    assert _describe(L, FP8, 65, 8192, 8192) == "fp8 bn=64"                          # above the swap-AB bucket
    assert L.xb_gemm_describe(7, 1, 1, 1, 132, ctypes.create_string_buffer(8), 8) == -1
