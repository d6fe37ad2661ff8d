"""Development probe: FP8 W8A8 linears at decode batch sizes (M = 32 tokens) - the shipped dispatch (tokens in the 128-row MMA M
slot, wgmma BLOCK_N 64 / streaming kernel) against the wgmma kernel in swap-AB mode (weight rows in the M slot, tokens as a
32 / 64-column N tile, transposed store: xb_set_fp8_swap_max_m).  Shapes: Llama-3-70B projections, unsharded and
the TP8 shard.  us per call from CUDA-graph replay over rotating weight copies (> L2)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xllm_b200 import ops  # noqa: E402

DEV, BF16, E4M3 = "cuda", torch.bfloat16, torch.float8_e4m3fn
PEAK = 6482.4


def graph_time(fns, iters=10):
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


def main():
    M = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    shapes = {"qkv tp8": (1280, 8192), "o tp8": (8192, 1024), "gate_up tp8": (7168, 8192), "down tp8": (8192, 3584),
              "qkv tp1": (10240, 8192), "o tp1": (8192, 8192), "gate_up tp1": (57344, 8192), "down tp1": (8192, 28672)}
    one = torch.ones(1, device=DEV)
    for name, (N, K) in shapes.items():
        copies = max(2, int(300e6 / (N * K)) + 1)
        ws = [torch.randn(N, K, device=DEV).clamp(-3, 3).to(E4M3) for _ in range(copies)]
        x = torch.randn(M, K, device=DEV).clamp(-3, 3).to(E4M3)
        y = torch.empty(M, N, device=DEV, dtype=BF16)
        nb = N * K + M * K + M * N * 2
        t_cur = graph_time([lambda i=i: ops.cutlass_scaled_mm(y, x, ws[i].t(), one, one, None) for i in range(copies)])
        t_small = graph_time([lambda i=i: ops.fp8_scaled_mm_small_m(y, x, ws[i].t(), one, one, None) for i in range(copies)])
        old = ops.set_fp8_swap_max_m(64)
        t_swap = graph_time([lambda i=i: ops.gemm_fp8_scaled(y, x, ws[i], one, one, None) for i in range(copies)])
        ref = (x.float() @ ws[0].float().t())
        ops.gemm_fp8_scaled(y, x, ws[0], one, one, None)
        ops.set_fp8_swap_max_m(old)
        err = float((y.float() - ref).abs().max() / ref.abs().max())
        print(f"{name:12s} N={N:6d} K={K:6d} M={M}: shipped dispatch {t_cur:7.2f} us ({nb / t_cur / 1e3 / PEAK:5.1%})  streaming {t_small:7.2f} us "
              f"({nb / t_small / 1e3 / PEAK:5.1%})  swapped wgmma {t_swap:7.2f} us ({nb / t_swap / 1e3 / PEAK:5.1%})  rel err {err:.1e}", flush=True)
        del ws


if __name__ == "__main__":
    main()
