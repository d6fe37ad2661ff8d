"""Host side of the MoE prefill (grouped-GEMM) path, no device needed: which path the expert entries take for a token count
(xb_moe_experts_describe) and its setter, the workspace each path needs, argument errors of the grouped path reported through
xb_last_error before any launch, and the per-expert vectorised reference (tests/moe_grouped_ref.py::fused_moe_grouped) against
oracle.moe.fused_moe."""
import ctypes

import pytest
import torch

from oracle import moe as OM
from tests.moe_grouped_ref import fused_moe_grouped

BF16 = torch.bfloat16


@pytest.fixture(scope="module")
def L(built_lib):
    lib = ctypes.CDLL(built_lib)
    lib.xb_moe_experts_workspace_bytes.restype = ctypes.c_int64
    lib.xb_moe_experts_workspace_bytes.argtypes = [ctypes.c_int] * 4
    lib.xb_last_error.restype = ctypes.c_char_p
    return lib


def _describe(L, kind, T, k, H, I, E):
    buf = ctypes.create_string_buffer(96)
    n = L.xb_moe_experts_describe(kind, T, k, H, I, E, buf, 96)
    assert n > 0
    return buf.value.decode()


def _grouped_bytes(T, k, H, I):
    P = T * k
    return 8192 + 2 * ((4 * P + 255) // 256 * 256) + P * (2 * H + I) * 2


def test_path_follows_the_token_count(L):
    for kind, name in ((0, "bf16"), (2, "w4")):
        for T in (1, 16, 63, 64):
            assert _describe(L, kind, T, 8, 7168, 2048, 32) == f"{name} gemv"
        for T in (65, 128, 1000, 10240):
            assert _describe(L, kind, T, 8, 7168, 2048, 32).startswith(f"{name} grouped bn=128")
    # upper bound of the m tiles: ceil(P / 128) + one partial tile per local expert
    assert _describe(L, 0, 256, 2, 4096, 14336, 8) == "bf16 grouped bn=128 m_tiles<=12"
    assert L.xb_moe_experts_describe(1, 100, 2, 256, 128, 4, ctypes.create_string_buffer(8), 8) == -1
    assert L.xb_moe_experts_describe(0, 100, 2, 256, 128, 4, None, 8) == -1


def test_setter_moves_the_boundary_and_restores_it(L):
    old = L.xb_set_moe_grouped_min_tokens(17)
    try:
        assert old == 65
        assert _describe(L, 0, 16, 2, 256, 128, 4) == "bf16 gemv"
        assert _describe(L, 0, 17, 2, 256, 128, 4).startswith("bf16 grouped")
        assert L.xb_moe_experts_workspace_bytes(17, 2, 256, 128) == _grouped_bytes(17, 2, 256, 128)
        assert L.xb_set_moe_grouped_min_tokens(0) == -1 and b"out of range" in L.xb_last_error()
    finally:
        assert L.xb_set_moe_grouped_min_tokens(old) == 17
    assert _describe(L, 0, 64, 2, 256, 128, 4) == "bf16 gemv" and _describe(L, 0, 65, 2, 256, 128, 4).startswith("bf16 grouped")


def test_workspace_query(L):
    # T <= 64: the GEMV path's act + y2, unchanged
    for T, k, H, I in ((1, 2, 256, 128), (16, 2, 512, 96), (64, 8, 7168, 2048), (33, 8, 1024, 512)):
        assert L.xb_moe_experts_workspace_bytes(T, k, H, I) == T * k * (I + H) * 2
    # T >= 65: routing header, the two pair maps, sorted input, act, y2
    for T, k, H, I in ((65, 2, 4096, 14336), (1000, 4, 2048, 1408), (10240, 8, 7168, 2048), (10240, 8, 64, 32)):
        assert L.xb_moe_experts_workspace_bytes(T, k, H, I) == _grouped_bytes(T, k, H, I)
    assert L.xb_moe_experts_workspace_bytes(10240, 8, 7168, 2048) > 2 ** 31          # int64 sizes


def _bf16_call(L, T=128, k=2, H=256, I=128, E=4, input_ptr=1 << 20, ws_bytes=1 << 40):
    p = ctypes.c_void_p
    return L.xb_moe_experts_bf16(p(1 << 21), ctypes.c_int64(H), p(input_ptr), ctypes.c_int64(H), p(1 << 22), p(1 << 23),
                                 p(1 << 24), p(1 << 25), T, k, H, I, E, 0, p(1 << 26), ctypes.c_int64(ws_bytes), None)


def _w4_call(L, gs=128, T=128, k=2, H=256, I=128, E=4, meta_ptr=1 << 27):
    p = ctypes.c_void_p
    return L.xb_moe_experts_w4a16(p(1 << 21), ctypes.c_int64(H), p(1 << 20), ctypes.c_int64(H), p(1 << 22), p(1 << 23),
                                  p(1 << 24), p(meta_ptr), p(1 << 25), p(1 << 28), gs, T, k, H, I, E, 0, p(1 << 26),
                                  ctypes.c_int64(1 << 40), None)


def test_grouped_path_argument_errors_without_a_device(L):
    """every check of the grouped path runs before the first launch (the pointers here are never dereferenced)"""
    assert _bf16_call(L, input_ptr=(1 << 20) + 2) != 0 and b"16-byte alignment" in L.xb_last_error()
    assert _w4_call(L, gs=96) != 0 and b"group_size 96" in L.xb_last_error()
    assert _w4_call(L, gs=192, H=384, I=384) != 0 and b"power of two" in L.xb_last_error()
    assert _w4_call(L, meta_ptr=(1 << 27) + 4) != 0 and b"meta" in L.xb_last_error()
    assert _bf16_call(L, ws_bytes=_grouped_bytes(128, 2, 256, 128) - 1) != 0 and b"workspace too small" in L.xb_last_error()
    assert _bf16_call(L, T=70000) != 0 and b"grouped path" in L.xb_last_error()
    assert _bf16_call(L, E=513) != 0 and b"grouped path" in L.xb_last_error()
    assert _bf16_call(L, k=33) != 0 and b"grouped path" in L.xb_last_error()
    assert _bf16_call(L, H=100) != 0 and b"multiples of 32" in L.xb_last_error()
    # the GEMV path keeps its own pair limit
    assert _bf16_call(L, T=64, k=1024) != 0 and b"decode-sized path" in L.xb_last_error()


def _problem(seed, T, k, E, H, I, id_lo=0, id_hi=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, H, generator=g).to(BF16)
    fc1 = (torch.randn(E, 2 * I, H, generator=g) * H ** -0.5).to(BF16)
    fc2 = (torch.randn(E, H, I, generator=g) * I ** -0.5).to(BF16)
    ids = torch.randint(id_lo, E if id_hi is None else id_hi, (T, k), generator=g, dtype=torch.int32)
    sc = torch.rand(T, k, generator=g).float()
    return x, ids, sc, fc1, fc2


def _within_one_ulp(a, b):
    """|a - b| <= one bf16 ulp of max(|a|, |b|) (exact for zeros)"""
    a, b = a.float(), b.float()
    m = torch.maximum(a.abs(), b.abs())
    ulp = torch.where(m > 0, 2.0 ** (torch.floor(torch.log2(m.clamp_min(2.0 ** -126))) - 7), torch.zeros_like(m))
    return bool(((a - b).abs() <= ulp).all())


@pytest.mark.parametrize("T,k,E,H,I", [(9, 2, 4, 64, 32), (17, 4, 6, 128, 96), (5, 3, 8, 96, 64)])
def test_grouped_reference_matches_fused_moe(T, k, E, H, I):
    x, ids, sc, fc1, fc2 = _problem(T + E, T, k, E, H, I)
    ref, mag = OM.fused_moe(x, ids, sc, fc1, fc2, return_abs=True)
    out, mag2 = fused_moe_grouped(x, ids, sc, fc1, fc2, return_abs=True)
    assert _within_one_ulp(out, ref)
    assert torch.allclose(mag, mag2, rtol=1e-2, atol=1e-6)


def test_grouped_reference_ep_slices_and_foreign_ids():
    T, k, E, H, I = 11, 3, 6, 64, 32
    # ids from -2 to E + 2: negative and too-large ids belong to no rank and contribute zero
    x, ids, sc, fc1, fc2 = _problem(7, T, k, E, H, I, id_lo=-2, id_hi=E + 3)
    assert bool((ids < 0).any()) and bool((ids >= E).any())
    full = OM.fused_moe(x, ids, sc, fc1, fc2)
    assert _within_one_ulp(fused_moe_grouped(x, ids, sc, fc1, fc2), full)
    for lo, hi in ((0, 3), (3, 6), (2, 5)):
        ref = OM.fused_moe(x, ids, sc, fc1[lo:hi], fc2[lo:hi], expert_begin=lo)
        assert _within_one_ulp(fused_moe_grouped(x, ids, sc, fc1[lo:hi], fc2[lo:hi], expert_begin=lo), ref)
    # a slice that owns none of the ids: exact zeros
    none = fused_moe_grouped(x, torch.full_like(ids, 100), sc, fc1, fc2)
    assert torch.equal(none, torch.zeros_like(none))
