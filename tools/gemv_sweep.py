"""Development aid (not the bench contract): device timings of the W4A16 decode GEMV variants on the four Qwen2-7B
projection shapes - plain, x staged in shared memory, add+RMSNorm prologue, act / rope epilogues - each as isolated
launches and as PDL-chained back-to-back launches over rotating weight copies (> L2)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xllm_b200 import ops  # noqa: E402

DEV, BF16 = "cuda", torch.bfloat16
PEAK = 6482.4


def chained(fns, reps=5):
    for f in fns:
        f()
    torch.cuda.synchronize()
    torch.cuda._sleep(int(20e6))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        for f in fns:
            f()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (reps * len(fns))


def graph_time(fns, iters=20):
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for f in fns:
            f()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for f in fns:
                f()
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters / len(fns)


def weights(N, K, gs, copies):
    ws = []
    for _ in range(copies):
        qw = torch.randint(-2 ** 31, 2 ** 31 - 1, (N // 16, K // 64, 32, 4), dtype=torch.int32, device=DEV)
        s = (torch.rand(K // gs, N, device=DEV) * 0.01 + 0.001).to(BF16).view(torch.int16).to(torch.int32) & 0xFFFF
        ws.append((qw, (s | (0x4308 << 16)).contiguous()))
    return ws


def run(name, N, K, M=1, gs=128, heads=None):
    copies = max(2, int(400e6 / (N * K / 2)) + 1)
    ws = weights(N, K, gs, copies)
    x = torch.randn(M, K, device=DEV, dtype=BF16)
    res = torch.randn(M, K, device=DEV, dtype=BF16)
    res_out = torch.empty_like(res)
    nw = torch.ones(K, device=DEV, dtype=BF16)
    y = torch.empty(M, N, device=DEV, dtype=BF16)
    nbytes = N * K // 2 + (K // gs) * N * 4 + M * K * 2 + M * N * 2
    variants = [("plain", lambda i: ops.w4a16_linear_small_m(x, ws[i][0], ws[i][1], gs, None, y)),
                ("x staged", lambda i: ops.w4a16_decode_fused(x, ws[i][0], ws[i][1], gs, None, y, stage_x=True)),
                ("norm prologue", lambda i: ops.w4a16_decode_fused(x, ws[i][0], ws[i][1], gs, None, y, norm_weight=nw, residual_in=res,
                                                                   residual_out=res_out))]
    if name == "gate_up":
        ya = torch.empty(M, N // 2, device=DEV, dtype=BF16)
        variants += [("act epilogue", lambda i: ops.w4a16_gate_up_act(x, ws[i][0], ws[i][1], gs, "silu", None, ya)),
                     ("norm + act", lambda i: ops.w4a16_decode_fused(x, ws[i][0], ws[i][1], gs, None, ya, norm_weight=nw, residual_in=res,
                                                                     residual_out=res_out, epilogue="act_mul"))]
    if heads:
        nh, nkv, D = heads
        pos = torch.full((M,), 4095, dtype=torch.int64, device=DEV)
        cs = torch.randn(8192, D, device=DEV, dtype=BF16)
        slots = torch.arange(M, dtype=torch.int32, device=DEV) + 128
        kc = torch.zeros(8, 128, nkv, D, device=DEV, dtype=BF16)
        vc = torch.zeros_like(kc)
        variants += [("rope/cache epilogue", lambda i: ops.w4a16_decode_fused(x, ws[i][0], ws[i][1], gs, None, y, epilogue="rope_cache",
                                                                              positions=pos, cos_sin_cache=cs, slot_ids=slots,
                                                                              key_cache=kc, value_cache=vc, num_heads=nh,
                                                                              num_kv_heads=nkv, head_dim=D))]
        variants += [("norm + rope/cache", lambda i: ops.w4a16_decode_fused(x, ws[i][0], ws[i][1], gs, None, y, norm_weight=nw, residual_in=res,
                                                                            residual_out=res_out, epilogue="rope_cache", positions=pos,
                                                                            cos_sin_cache=cs, slot_ids=slots, key_cache=kc, value_cache=vc,
                                                                            num_heads=nh, num_kv_heads=nkv, head_dim=D))]
    if os.environ.get("XB_SWEEP_FEW"):          # A/B of the two arithmetic forms: only the variants the step launches
        variants = [v for v in variants if v[0] in ("plain", "x staged", "act epilogue", "rope/cache epilogue")]
    for vn, fn in variants:
        fns = [lambda i=i: fn(i) for i in range(copies)]
        t_c, t_g = chained(fns), graph_time(fns)
        print(f"{name:8s} N={N:6d} K={K:6d} M={M} {vn:18s} chained {t_c:7.2f} us ({nbytes / t_c / 1e3 / PEAK:5.1%})  graph {t_g:7.2f} us "
              f"({nbytes / t_g / 1e3 / PEAK:5.1%})", flush=True)


def run_q8(name, N, K, M):
    """W8A16 and FP8 W8A8 streaming kernels, and the small-M / wgmma crossover of the three weight formats."""
    gs = 128
    copies = max(2, int(400e6 / (N * K)) + 1)
    x = torch.randn(M, K, device=DEV, dtype=BF16)
    y = torch.empty(M, N, device=DEV, dtype=BF16)
    w8 = []
    for _ in range(copies):
        qw = torch.randint(-2 ** 31, 2 ** 31 - 1, (N // 16, K // 64, 32, 8), dtype=torch.int32, device=DEV)
        sc = (torch.rand(K // gs, N, device=DEV) * 0.001 + 0.0001).to(BF16).view(torch.int16).to(torch.int32) & 0xFFFF
        w8.append((qw, (sc | (128 << 16)).contiguous()))
    nb = N * K + (K // gs) * N * 4 + M * K * 2 + M * N * 2
    fns = [lambda i=i: ops.w8a16_linear_small_m(x, w8[i][0], w8[i][1], gs, None, y) for i in range(copies)]
    t = graph_time(fns)
    print(f"{name:8s} N={N:6d} K={K:6d} M={M:2d} w8a16 streaming      graph {t:7.2f} us ({nb / t / 1e3 / PEAK:5.1%})", flush=True)
    if M > 16:
        fns = [lambda i=i: ops.gemm_w8a16(x, w8[i][0], w8[i][1], gs, None, y) for i in range(copies)]
        t = graph_time(fns)
        print(f"{name:8s} N={N:6d} K={K:6d} M={M:2d} w8a16 wgmma GEMM   graph {t:7.2f} us ({nb / t / 1e3 / PEAK:5.1%})", flush=True)
    del w8
    f8 = [torch.randn(N, K, device=DEV).clamp(-3, 3).to(torch.float8_e4m3fn) for _ in range(copies)]
    a8 = torch.randn(M, K, device=DEV).clamp(-3, 3).to(torch.float8_e4m3fn)
    one = torch.ones(1, device=DEV)
    nb = N * K + M * K + M * N * 2
    fns = [lambda i=i: ops.fp8_scaled_mm_small_m(y, a8, f8[i].t(), one, one, None) for i in range(copies)]
    t = graph_time(fns)
    print(f"{name:8s} N={N:6d} K={K:6d} M={M:2d} fp8 streaming (M<=64) graph {t:7.2f} us ({nb / t / 1e3 / PEAK:5.1%})", flush=True)
    from xllm_b200._lib import c_i32, c_i64, check, lib
    fns = [lambda i=i: check(lib().xb_gemm_fp8_scaled(ops._p(y), c_i64(y.stride(0)), ops._p(a8), c_i64(a8.stride(0)), ops._p(f8[i]),
                                                      ops._p(one), c_i32(1), ops._p(one), c_i32(1), ops._p(None), c_i32(M), c_i32(N),
                                                      c_i32(K), ops._stream()), "gemm_fp8") for i in range(copies)]
    t = graph_time(fns)
    print(f"{name:8s} N={N:6d} K={K:6d} M={M:2d} fp8 wgmma GEMM      graph {t:7.2f} us ({nb / t / 1e3 / PEAK:5.1%})", flush=True)
    del f8
    # W4 crossover
    ws = weights(N, K, gs, max(2, int(400e6 / (N * K / 2)) + 1))
    nb = N * K // 2 + (K // gs) * N * 4 + M * K * 2 + M * N * 2
    fns = [lambda i=i: ops.w4a16_linear_small_m(x, ws[i][0], ws[i][1], gs, None, y) for i in range(len(ws))]
    t = graph_time(fns)
    print(f"{name:8s} N={N:6d} K={K:6d} M={M:2d} w4a16 streaming      graph {t:7.2f} us ({nb / t / 1e3 / PEAK:5.1%})", flush=True)
    if M > 16:
        fns = [lambda i=i: ops.gemm_w4a16(x, ws[i][0], ws[i][1], gs, None, y) for i in range(len(ws))]
        t = graph_time(fns)
        print(f"{name:8s} N={N:6d} K={K:6d} M={M:2d} w4a16 wgmma GEMM   graph {t:7.2f} us ({nb / t / 1e3 / PEAK:5.1%})", flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "q8":
        for M in (1, 32, 64):
            run_q8("qkv70b", 10240, 8192, M)
            run_q8("down", 3584, 18944, M)
            run_q8("gate_up", 37888, 3584, M)
        sys.exit(0)
    Ms = [int(a) for a in sys.argv[1:]] or [1]
    print("W4 decode form:", "exact-dequant" if os.environ.get("XB_W4_EXACT", "0") not in ("0", "") else "bf16-weight (or library default)")
    for M in Ms:
        run("qkv", 4608, 3584, M, heads=(28, 4, 128))
        run("o", 3584, 3584, M)
        run("gate_up", 37888, 3584, M)
        run("down", 3584, 18944, M)
