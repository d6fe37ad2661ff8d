"""Qwen3 measurements on one GPU; writes OUT/qwen3_decode_sweep.json.

  python tools/qwen3_decode_sweep.py OUT

1. kernel: qk_norm_rope_and_cache (K10+K12, one launch) vs fused_qk_norm_rope + reshape_paged_cache (two launches) at the
   Qwen3-8B heads (32 / 8 x 128) over T tokens: CUDA-graph replays of many launches timed with CUDA events, three repetitions
   with the two forms alternated; the outputs of one eager call of each form are compared bit for bit in the same run.
2. step: the Qwen3-8B W4A16 decode step (synthetic weights, batch 1 and 16, every request at ctx 4096) as one CUDA-graph
   replay: tokens/s, and the step's bytes (weights + KV cache read + KV rows written, computed from shapes) over 3.35 TB/s,
   the H100 SXM data-sheet HBM3 bandwidth - a whole-step share, not a kernel share.
3. the same step with the two-launch pair in place of the fused kernel (Qwen2DecodeRunner(fused_rope_cache=False)), runs
   alternated with (2), logits compared bit for bit.
The card's name, power limit and max SM clock come from a read-only nvidia-smi query in the same run."""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

HBM_BPS = 3.35e12
HQ, HKV, D = 32, 8, 128
TOKENS = [1, 8, 64, 512, 4096, 16384]


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"error": f"nvidia-smi query failed: {e}"}


def graph_of(fn, n):
    """one CUDA graph of n calls of fn (warmed up eagerly first)"""
    fn()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(n):
                fn()
    torch.cuda.current_stream().wait_stream(s)
    return g


def time_replays(g, replays):
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / replays


def kernel_sweep(ops):
    from xllm_b200.qwen2 import Qwen2Config, make_cos_sin_cache
    cfg = Qwen2Config.qwen3_8b()
    cs = make_cos_sin_cache(cfg, "cuda")
    qs, kvs = HQ * D, HKV * D
    rows = []
    for T in TOKENS:
        g = torch.Generator(device="cuda").manual_seed(T)
        bs = 128
        nblocks = (T + bs - 1) // bs + 1
        qkv0 = torch.randn(T, (HQ + 2 * HKV) * D, generator=g, device="cuda").to(torch.bfloat16)
        qw = (1 + 0.1 * torch.randn(D, generator=g, device="cuda")).to(torch.bfloat16)
        kw = (1 + 0.1 * torch.randn(D, generator=g, device="cuda")).to(torch.bfloat16)
        pos = torch.randint(0, cfg.max_position_embeddings, (T,), generator=g, device="cuda")
        slots = (torch.randperm(nblocks * bs - bs, generator=g, device="cuda")[:T] + bs).to(torch.int32)
        kc0 = torch.zeros(nblocks, bs, HKV, D, dtype=torch.bfloat16, device="cuda")
        bufs = {k: (qkv0.clone(), kc0.clone(), kc0.clone()) for k in ("fused", "pair")}

        def fused(b=bufs["fused"]):
            ops.qk_norm_rope_and_cache(b[0], HQ, HKV, D, cfg.rms_norm_eps, qw, kw, cs, pos, slots, b[1], b[2])

        def pair(b=bufs["pair"]):
            ops.fused_qk_norm_rope(b[0], HQ, HKV, HKV, D, cfg.rms_norm_eps, qw, kw, cs, False, pos)
            ops.reshape_paged_cache(slots, b[0][:, qs:qs + kvs].view(T, HKV, D), b[0][:, qs + kvs:].view(T, HKV, D),
                                    b[1], b[2])
        fused()
        pair()
        torch.cuda.synchronize()
        same = all(torch.equal(x, y) for x, y in zip(bufs["fused"], bufs["pair"]))
        n = 200 if T <= 512 else 20
        graphs = {"fused": graph_of(fused, n), "pair": graph_of(pair, n)}
        us = {"fused": [], "pair": []}
        for _ in range(3):
            for k in ("fused", "pair"):
                us[k].append(time_replays(graphs[k], 10) * 1e3 / n)
        # fused kernel traffic: read q|k|v, write q|k back, write the k and v cache rows
        nbytes = T * ((HQ + 2 * HKV) + (HQ + HKV) + 2 * HKV) * D * 2
        row = {"T": T, "bit_identical": same, "launches_per_graph": n, "fused_us": us["fused"], "pair_us": us["pair"],
               "fused_us_median": statistics.median(us["fused"]), "pair_us_median": statistics.median(us["pair"]),
               "fused_bytes": nbytes, "fused_GBps": nbytes / (statistics.median(us["fused"]) * 1e-6) / 1e9}
        row["speedup"] = row["pair_us_median"] / row["fused_us_median"]
        print(json.dumps(row), flush=True)
        rows.append(row)
        del graphs, bufs
        torch.cuda.empty_cache()
    return rows


def step_sweep(ops, ctx=4096, batches=(1, 16), replays=50):
    from xllm_b200 import _lib
    from xllm_b200.qwen2 import Qwen2Config, Qwen2DecodeRunner, Qwen2Weights
    cfg = Qwen2Config.qwen3_8b()
    w = Qwen2Weights.synthetic(cfg, "cuda", seed=2026)
    out = []
    for B in batches:
        bs = cfg.block_size
        npg = (ctx + bs - 1) // bs
        runners, launches = {}, {}
        for k, fused in (("fused", True), ("pair", False)):
            r = Qwen2DecodeRunner(cfg, w, max_batch=B, max_ctx=ctx, device="cuda", fused_rope_cache=fused)
            g = torch.Generator(device="cuda").manual_seed(7)
            for li in range(cfg.num_layers):
                r.k_caches[li].normal_(generator=g)
                r.v_caches[li].normal_(generator=g)
            pages = list(range(1, B * npg + 1))
            slots = [pages[b * npg + (ctx - 1) // bs] * bs + (ctx - 1) % bs for b in range(B)]
            r.set_inputs_host([1234 + b for b in range(B)], [ctx - 1] * B, slots, [b * npg for b in range(B + 1)], pages,
                              [(ctx - 1) % bs + 1] * B)
            r.step()
            n0 = _lib.launch_count()
            r.launch_step()
            torch.cuda.synchronize()
            launches[k] = _lib.launch_count() - n0
            r.capture()
            runners[k] = r
        ms = {"fused": [], "pair": []}
        for _ in range(3):
            for k, r in runners.items():
                ms[k].append(time_replays(r.graph, replays))
        same = torch.equal(runners["fused"].logits, runners["pair"].logits)
        kv_read = B * ctx * cfg.num_layers * 2 * cfg.n_kv_heads * cfg.head_dim * 2
        step_bytes = w.weight_bytes() + kv_read + B * cfg.num_layers * 2 * cfg.kv_size * 2
        row = {"batch": B, "ctx": ctx, "step_bytes": step_bytes, "weight_bytes": w.weight_bytes(), "kv_read_bytes": kv_read,
               "logits_bit_identical": same}
        for k in ("fused", "pair"):
            m = statistics.median(ms[k])
            row[k] = {"ms_per_step": ms[k], "ms_median": m, "tokens_per_s": B / (m / 1e3), "launches_per_step": launches[k],
                      "step_bytes_over_hbm_peak": step_bytes / HBM_BPS / (m / 1e3)}
        print(json.dumps(row), flush=True)
        out.append(row)
        del runners
        torch.cuda.empty_cache()
    return out


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    assert torch.cuda.is_available(), "this tool measures on a GPU"
    from xllm_b200 import ops
    res = {"card": card(), "kernel": kernel_sweep(ops), "step": step_sweep(ops),
           "timing": "CUDA events around CUDA-graph replays; three repetitions, the two forms alternated"}
    os.makedirs(sys.argv[1], exist_ok=True)
    path = os.path.join(sys.argv[1], "qwen3_decode_sweep.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()
