"""MoE expert layer (fc1 -> SwiGLU -> fc2 -> combine) at decode and prefill token counts: the grouped-GEMM path against the
expert-GEMV path, on an H100.

    python tools/moe_prefill_sweep.py --out DIR [--shapes mixtral,qwen,dsv3] [--tokens 16,32,...]

For every shape and token count it checks the grouped path's output against the GEMV path's (where both can run) before
timing, warms both up, times each with CUDA events over enough launches to fill --min-seconds, and writes one JSON file
(DIR/moe_prefill_sweep.json) with a row per (shape, T):
  - time of each path (ms), the grouped path's speed-up;
  - algorithmic FLOPs of the local pairs, 2 * P_local * 3 * I * H, as TFLOP/s and as a share of the 989 TFLOP/s dense bf16
    data-sheet rate of the H100 SXM;
  - for T <= 256, the bytes of the expert weights the step touches (every expert with at least one local pair) over each
    path's time, as a share of the 3.35 TB/s HBM3 data-sheet bandwidth;
  - bf16 shapes: torch._grouped_mm on the same two GEMMs (same expert-sorted rows), and one dense xb_gemm_bf16 of equal
    M * N * K (M = P_local, N = 3I, K = H).
The card's name and power limit are printed and stored with the numbers.  Needs a CUDA device; there is no CPU fallback.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from xllm_b200 import ops  # noqa: E402

BF16 = torch.bfloat16
PEAK_BF16_TFLOPS = 989.0
PEAK_HBM_TBS = 3.35
SHAPES = {
    # name: kind, E (all experts), E_local, k, H, I, group size
    "mixtral": ("bf16", 8, 8, 2, 4096, 14336, None),       # Mixtral-8x7B-like
    "qwen": ("bf16", 60, 60, 4, 2048, 1408, None),         # Qwen1.5-MoE-A2.7B-like
    "dsv3": ("w4", 256, 32, 8, 7168, 2048, 128),           # DeepSeek-V3 routed experts, one EP8 shard, W4A16 g = 128
}
TOKENS = [16, 32, 64, 65, 128, 256, 1024, 4096, 10240]
GEMV_MAX_PAIRS = 65535


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:       # the numbers still carry torch's device name
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def make_weights(kind, El, H, I, gs, g):
    if kind == "bf16":
        fc1 = (torch.randn(El, 2 * I, H, device="cuda", generator=g) * H ** -0.5).to(BF16)
        fc2 = (torch.randn(El, H, I, device="cuda", generator=g) * I ** -0.5).to(BF16)
        return fc1, fc2

    # random int4 codes with per-group bf16 scale ~ 1/8 of the bf16 weights' spread and zero point 8
    def packed(rows, K, s):
        q = torch.randint(-2 ** 31, 2 ** 31 - 1, (El, rows // 16, K // 64, 32, 4), device="cuda", dtype=torch.int64,
                          generator=g).to(torch.int32)
        scale = (torch.rand(El, K // gs, rows, device="cuda", generator=g) * s + s / 2).to(BF16)
        meta = scale.view(torch.int16).to(torch.int32) & 0xFFFF
        meta = meta | (torch.tensor(136.0, dtype=BF16).view(torch.int16).to(torch.int32) << 16)
        return q, meta.contiguous()
    q1, m1 = packed(2 * I, H, H ** -0.5 / 4)
    q2, m2 = packed(H, I, I ** -0.5 / 4)
    return q1, m1, q2, m2


def run_moe(kind, x, ids, sc, w, gs, El, ws, out):
    if kind == "bf16":
        return ops.cutlass_fused_moe(x, ids, sc, w[0], w[1], output=out, workspace=ws)
    return ops.fused_moe_w4a16(x, ids, sc, *w, gs, output=out, workspace=ws)


def timed(fn, min_seconds, max_iters=200):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    one = time.perf_counter() - t0
    iters = int(max(3, min(max_iters, min_seconds / max(one, 1e-6))))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters, iters


def with_min_tokens(v, fn):
    old = ops.set_moe_grouped_min_tokens(v)
    try:
        return fn()
    finally:
        ops.set_moe_grouped_min_tokens(old)


def sweep_shape(name, tokens, min_seconds, rows):
    kind, E, El, k, H, I, gs = SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(2026)
    w = make_weights(kind, El, H, I, gs, g)
    for T in tokens:
        x = torch.randn(T, H, device="cuda", generator=g).to(BF16)
        ids = torch.rand(T, E, device="cuda", generator=g).topk(k, dim=1).indices.to(torch.int32).contiguous()
        sc = torch.rand(T, k, device="cuda", generator=g).softmax(1).contiguous()
        local = (ids < El)
        p_local = int(local.sum())
        touched = int(torch.unique(ids[local]).numel()) if p_local else 0
        flops = 2.0 * p_local * 3 * I * H
        wbytes_expert = 3 * I * H * (2 if kind == "bf16" else 0.5) + (0 if kind == "bf16" else 3 * I * H // gs * 4)
        row = {"shape": name, "kind": kind, "T": T, "k": k, "E": E, "E_local": El, "H": H, "I": I, "group_size": gs,
               "pairs_local": p_local, "experts_touched": touched, "gflop": flops / 1e9}
        out_g = torch.empty(T, H, dtype=BF16, device="cuda")
        out_v = torch.empty(T, H, dtype=BF16, device="cuda")
        ws_g = torch.empty(with_min_tokens(1, lambda: int(ops.lib().xb_moe_experts_workspace_bytes(T, k, H, I))),
                           dtype=torch.uint8, device="cuda")
        row["path_default"] = ops.moe_experts_describe(kind, T, k, H, I, El)
        grouped = lambda: with_min_tokens(1, lambda: run_moe(kind, x, ids, sc, w, gs, El, ws_g, out_g))
        both = T * k <= GEMV_MAX_PAIRS
        if both:
            ws_v = torch.empty(T * k * (I + H) * 2, dtype=torch.uint8, device="cuda")
            gemv = lambda: with_min_tokens(1 << 30, lambda: run_moe(kind, x, ids, sc, w, gs, El, ws_v, out_v))
            grouped()
            gemv()
            torch.cuda.synchronize()
            d = (out_g.float() - out_v.float())
            rel = float(d.norm() / out_v.float().norm().clamp_min(1e-30))
            row["grouped_vs_gemv_rel_l2"] = rel
            row["grouped_vs_gemv_max_abs"] = float(d.abs().max())
            assert rel <= 1e-2, f"{name} T={T}: grouped path differs from the GEMV path (rel-L2 {rel:.2e})"
        row["grouped_ms"], row["grouped_iters"] = timed(grouped, min_seconds)
        row["grouped_tflops"] = flops / row["grouped_ms"] / 1e9
        row["grouped_share_of_989"] = row["grouped_tflops"] / PEAK_BF16_TFLOPS
        if both:
            row["gemv_ms"], row["gemv_iters"] = timed(gemv, min_seconds)
            row["gemv_tflops"] = flops / row["gemv_ms"] / 1e9
            row["speedup_grouped_over_gemv"] = row["gemv_ms"] / row["grouped_ms"]
        if T <= 256:
            wb = touched * wbytes_expert
            row["weight_bytes_touched"] = wb
            row["grouped_weight_share_of_3.35TBs"] = wb / (row["grouped_ms"] * 1e-3) / (PEAK_HBM_TBS * 1e12)
            if both:
                row["gemv_weight_share_of_3.35TBs"] = wb / (row["gemv_ms"] * 1e-3) / (PEAK_HBM_TBS * 1e12)
        if kind == "bf16" and p_local:
            comparators(row, x, ids, w, El, k, H, I, p_local, flops, min_seconds)
        rows.append(row)
        print(json.dumps(row), flush=True)
        del x, ids, sc, out_g, out_v, ws_g


def comparators(row, x, ids, w, El, k, H, I, p_local, flops, min_seconds):
    fc1, fc2 = w
    flat = ids.view(-1).long()
    order = torch.sort(flat, stable=True).indices[:p_local]
    a = x[order // k].contiguous()
    counts = torch.bincount(flat[flat < El], minlength=El)
    offs = torch.cumsum(counts, 0).to(torch.int32)
    act = torch.randn(p_local, I, device="cuda").to(BF16)
    try:
        b1, b2 = fc1.transpose(1, 2), fc2.transpose(1, 2)
        gm = lambda: (torch._grouped_mm(a, b1, offs=offs), torch._grouped_mm(act, b2, offs=offs))
        row["torch_grouped_mm_ms"], _ = timed(gm, min_seconds)
        row["torch_grouped_mm_tflops"] = flops / row["torch_grouped_mm_ms"] / 1e9
    except Exception as e:
        row["torch_grouped_mm_error"] = str(e).splitlines()[0][:200]
    wd = torch.randn(3 * I, H, device="cuda").to(BF16) * H ** -0.5
    c = torch.empty(p_local, 3 * I, dtype=BF16, device="cuda")
    dense = lambda: ops.matmul(a, wd, None, c)
    row["dense_gemm_equal_mnk_ms"], _ = timed(dense, min_seconds)
    row["dense_gemm_tflops"] = flops / row["dense_gemm_equal_mnk_ms"] / 1e9
    row["grouped_over_dense_throughput"] = row["dense_gemm_equal_mnk_ms"] / row["grouped_ms"]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True, help="output directory (moe_prefill_sweep.json)")
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--tokens", default=",".join(map(str, TOKENS)))
    ap.add_argument("--min-seconds", type=float, default=0.3, help="timed window per measurement")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("moe_prefill_sweep needs a CUDA device")
    name = card()
    print("card:", name, flush=True)
    rows = []
    for s in args.shapes.split(","):
        sweep_shape(s, [int(t) for t in args.tokens.split(",")], args.min_seconds, rows)
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "moe_prefill_sweep.json")
    with open(path, "w") as f:
        json.dump({"card": name, "torch": torch.__version__, "rows": rows}, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()
