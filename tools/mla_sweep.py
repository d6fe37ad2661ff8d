"""Times the MLA kernels on the GPU: paged absorbed-MLA attention (decode, speculative, prefill shapes of DeepSeek-V3
at TP8 / TP1 head counts) and the latent cache writer against the four launches it replaces.  Prefill shapes also run in the expanded form
(xb_mla_prefill_expanded_bf16: gather + kv_b_proj up-projection + 192 / 128 attention, timed as one call) and, with
--flashinfer, through FlashInfer's ragged prefill with head_dim_qk 192 / head_dim_vo 128 fed K = [k_nope | broadcast
k_pe] and V from the same up-projection (its attention only).  --prefill times only those forms plus the selector grid:
a chunk of qo tokens over a history at H = 16 and 128, absorbed against expanded, with the form xb_mla_expanded_plan
picks, which calibrates the selector's constant (expanded FLOP = 2 H pairs (192 + 128) + 2 * 512 * 256 H kv tokens).

Kernel time = CUDA events around replays of a CUDA graph holding `--iters` launches (see time_it).  Bytes and FLOP are counted from the shapes here:
  bytes = sum over requests of kv_len * 1152 (c_kv 1024 + k_pe 128) + q (T*H*576*2) + o (T*H*512*2) + page indices
  FLOP  = 2 * H * (visible (q, kv) pairs) * (576 + 512)
Share of peak = the larger of bytes / 3.35 TB/s and FLOP / 989 TFLOP/s (H100 SXM data sheet, 700 W) over kernel time;
the line says which of the two binds.  The card's name and power limit are read in the same run.

    python tools/mla_sweep.py [--iters 50] [--warmup 10] [--flashinfer] [--prefill] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
BF16_PEAK = 989e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def time_it(fn, iters, warmup):
    """seconds per call of fn: `iters` calls captured into one CUDA graph, the graph replayed after warm-up, CUDA events
    around the replays - the host's per-call cost (argument checks, ctypes) stays out of the kernel time.  Returns
    (seconds, "graph"), or (seconds, "eager") when fn cannot be captured."""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    try:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(iters):
                fn()
        g.replay()
        torch.cuda.synchronize()
        reps = 3
        a.record()
        for _ in range(reps):
            g.replay()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / (reps * iters) * 1e-3, "graph"
    except Exception:
        torch.cuda.synchronize()
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / iters * 1e-3, "eager"


def attention_case(B, H, qo, kv, page=64, seed=0):
    import torch
    from xllm_b200 import ops
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(seed)
    npg = (kv + page - 1) // page
    n_pages = B * npg + 1
    ckv = torch.randn(n_pages, page, 512, device=dev, generator=g).to(torch.bfloat16)
    kpe = torch.randn(n_pages, page, 64, device=dev, generator=g).to(torch.bfloat16)
    indices = (torch.randperm(n_pages - 1, device=dev, generator=g)[:B * npg] + 1).to(torch.int32)
    indptr = torch.arange(B + 1, device=dev, dtype=torch.int32) * npg
    last = torch.full((B,), kv - (npg - 1) * page, dtype=torch.int32, device=dev)
    qo_indptr = torch.arange(B + 1, device=dev, dtype=torch.int32) * qo
    T = B * qo
    q = torch.randn(T, H, 576, device=dev, generator=g).to(torch.bfloat16)
    out = torch.empty(T, H, 512, dtype=torch.bfloat16, device=dev)
    plan = ops.MlaPlan(B, H, qo, page, npg, dev)
    causal = qo > 1

    def run():
        ops.mla_paged_attention(plan, q[..., :512], q[..., 512:], ckv, kpe, qo_indptr, indptr, indices, last, 192 ** -0.5,
                                out, causal=causal)
    pairs = B * (qo * (kv - qo) + qo * (qo + 1) // 2 if causal else qo * kv)
    bytes_ = B * kv * 1152 + T * H * (576 + 512) * 2 + B * npg * 4
    flop = 2 * H * pairs * (576 + 512)
    return run, bytes_, flop, plan.splits, dict(q=q, ckv=ckv, kpe=kpe, qo_indptr=qo_indptr, indptr=indptr, indices=indices,
                                                last=last, page=page, out=out, causal=causal)


def flashinfer_mla(d, B, H, qo, kv):
    """FlashInfer's BatchMLAPagedAttentionWrapper on the same inputs, or None when its module is not available."""
    try:
        import torch
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        import build_flashinfer_cache as FIC
        FIC.set_env()
        import flashinfer
        ws = torch.empty(128 << 20, dtype=torch.uint8, device="cuda")
        w = flashinfer.mla.BatchMLAPagedAttentionWrapper(ws, backend="fa2")
        kv_lens = torch.full((B,), kv, dtype=torch.int32, device="cuda")
        w.plan(d["qo_indptr"], d["indptr"], d["indices"], kv_lens, H, 512, 64, d["page"], d["causal"], 192 ** -0.5,
               torch.bfloat16, torch.bfloat16)
        q = d["q"]
        qn, qp = q[..., :512].contiguous(), q[..., 512:].contiguous()
        out = torch.empty_like(d["out"])

        def run():
            w.run(qn, qp, d["ckv"], d["kpe"], out=out)
        run()
        return run
    except Exception as e:  # the comparator is optional: report why it is absent
        return str(e).splitlines()[0][:120] if str(e) else type(e).__name__


def expanded_case(d, B, H, qo, kv, seed=0):
    """the expanded form on attention_case's inputs (q_input's first 192 columns as q, a random kv_b_proj); returns
    (run, plan, workspace, kv_b_proj, FLOP)"""
    import torch
    from xllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    w = (torch.randn(H * 256, 512, device="cuda", generator=g) * 512 ** -0.5).to(torch.bfloat16)
    q = d["q"][..., :192]
    plan = ops.MlaExpandedPlan(H, [qo] * B, [kv] * B, "cuda")
    ws = plan.workspace if plan.workspace is not None else torch.empty(plan.workspace_bytes, dtype=torch.uint8, device="cuda")
    out = torch.empty(B * qo, H, 128, dtype=torch.bfloat16, device="cuda")

    def run():
        ops.mla_prefill_expanded(plan, q, d["ckv"], d["kpe"], d["qo_indptr"], d["indptr"], d["indices"], d["last"], w,
                                 192 ** -0.5, out, workspace=ws)
    pairs = B * (qo * (kv - qo) + qo * (qo + 1) // 2)
    return run, plan, ws, out, 2 * H * pairs * (192 + 128) + 2 * 512 * 256 * H * B * kv


def flashinfer_ragged(d, plan, ws, H, B, qo, kv):
    """FlashInfer's BatchPrefillWithRaggedKVCacheWrapper (fa2, qk 192 / vo 128) on the expanded form's q and
    up-projection, or the reason it is unavailable"""
    try:
        import torch
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        import build_flashinfer_cache as FIC
        FIC.set_env()
        import flashinfer
        n = plan.total_kv
        kv_up = ws[:n * H * 512].view(torch.bfloat16).view(n, H, 256)
        off = (n * H * 512 + 255) // 256 * 256 + (n * 1024 + 255) // 256 * 256
        kpe = ws[off:off + n * 128].view(torch.bfloat16).view(n, 64)
        k = torch.cat([kv_up[..., :128], kpe[:, None].expand(-1, H, -1)], -1).contiguous()
        v = kv_up[..., 128:].contiguous()
        q = d["q"][..., :192].contiguous()
        kv_cu = torch.arange(B + 1, device="cuda", dtype=torch.int32) * kv
        w = flashinfer.BatchPrefillWithRaggedKVCacheWrapper(torch.empty(128 << 20, dtype=torch.uint8, device="cuda"), "NHD",
                                                            backend="fa2")
        w.plan(d["qo_indptr"], kv_cu, H, H, 192, head_dim_vo=128, causal=True, sm_scale=192 ** -0.5,
               q_data_type=torch.bfloat16)
        out = torch.empty(B * qo, H, 128, dtype=torch.bfloat16, device="cuda")

        def run():
            w.run(q, k, v, out=out)
        run()
        return run
    except Exception as e:  # the comparator is optional: report why it is absent
        return str(e).splitlines()[0][:120] if str(e) else type(e).__name__


GRID = [(H, qo, hist) for H in (16, 128) for qo in (16, 128, 512, 1024, 4096) for hist in (0, 4096, 32768)]


def prefill_forms(a, rows):
    """the README's prefill rows in the expanded / absorbed / FlashInfer forms, then the selector grid"""
    import torch
    for kind, H, B, qo, kv in [s for s in ATTN_SHAPES if s[0] == "prefill"]:
        run, _, fl, _, d = attention_case(B, H, qo, kv)
        iters = max(3, a.iters // 20)
        t_abs, _ = time_it(run, iters, a.warmup)
        erun, plan, ws, _, efl = expanded_case(d, B, H, qo, kv)
        t_exp, how = time_it(erun, iters, a.warmup)
        row = dict(kind="prefill-forms", H=H, B=B, qo=qo, kv=kv, absorbed_us=t_abs * 1e6, expanded_us=t_exp * 1e6,
                   expanded_TFLOPs=efl / t_exp / 1e12, selector="expanded" if plan.expanded else "absorbed", timing=how)
        fi = flashinfer_ragged(d, plan, ws, H, B, qo, kv) if a.flashinfer else None
        if callable(fi):
            row["flashinfer_us"] = time_it(fi, iters, a.warmup)[0] * 1e6
        elif fi is not None:
            row["flashinfer"] = f"unavailable: {fi}"
        rows.append(row)
        fi_s = f"  flashinfer ragged 192/128 {row['flashinfer_us']:9.1f} us" if "flashinfer_us" in row else f"  {row.get('flashinfer', '')}"
        print(f"prefill  H={H:3d} qo={qo:4d} kv={kv:6d}  absorbed {t_abs * 1e6:9.1f} us  expanded {t_exp * 1e6:9.1f} us "
              f"({efl / t_exp / 1e12:5.1f} TFLOP/s, x{t_abs / t_exp:.2f})  selector: {row['selector']}{fi_s}")
        del d, ws
        torch.cuda.empty_cache()
    for H, qo, hist in GRID:
        run, _, fl, _, d = attention_case(1, H, qo, qo + hist)
        iters = 3
        t_abs, _ = time_it(run, iters, a.warmup // 5 + 1)
        erun, plan, ws, _, efl = expanded_case(d, 1, H, qo, qo + hist)
        t_exp, _ = time_it(erun, iters, a.warmup // 5 + 1)
        rows.append(dict(kind="selector-grid", H=H, qo=qo, hist=hist, absorbed_us=t_abs * 1e6, expanded_us=t_exp * 1e6,
                         absorbed_flop=fl, expanded_flop=efl, selector="expanded" if plan.expanded else "absorbed"))
        # the constant that would put this point on the boundary: absorbed FLOP / expanded FLOP at equal times
        print(f"grid     H={H:3d} qo={qo:4d} hist={hist:6d}  absorbed {t_abs * 1e6:9.1f} us  expanded {t_exp * 1e6:9.1f} us  "
              f"faster: {'expanded' if t_exp < t_abs else 'absorbed'}  selector: {rows[-1]['selector']}  "
              f"break-even constant {fl / efl * t_exp / t_abs:.2f}")
        del d, ws
        torch.cuda.empty_cache()
    calibrate([r for r in rows if r["kind"] == "selector-grid"])


def calibrate(grid):
    """The selector's constant C (expanded when absorbed FLOP / expanded FLOP > C): for each interval between the grid's
    FLOP ratios, the total time of the grid with the forms C picks, and the worst slowdown against the faster form.  The
    constant is taken from the middle of the interval with the least total time."""
    ratios = sorted({r["absorbed_flop"] / r["expanded_flop"] for r in grid})
    cuts = [0.0] + ratios + [ratios[-1] * 2]
    best = None
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        c = (lo + hi) / 2
        times = [r["expanded_us"] if r["absorbed_flop"] / r["expanded_flop"] > c else r["absorbed_us"] for r in grid]
        total = sum(times)
        worst = max(t / min(r["expanded_us"], r["absorbed_us"]) for t, r in zip(times, grid))
        print(f"calibrate C in [{lo:.3f}, {hi:.3f}): grid total {total:10.1f} us  worst slowdown x{worst:.2f}")
        if best is None or total < best[0]:
            best = (total, lo, hi, worst)
    print(f"calibrate least total time: C in [{best[1]:.3f}, {best[2]:.3f}), total {best[0]:.1f} us, "
          f"worst slowdown x{best[3]:.2f}")


def writer_case(T, page=64, seed=0):
    import torch
    from oracle import ops as O
    from xllm_b200 import ops
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(seed)
    latent = torch.randn(T, 576, device=dev, generator=g).to(torch.bfloat16)
    gamma = torch.ones(512, dtype=torch.bfloat16, device=dev)
    pos = torch.arange(T, device=dev, dtype=torch.int64) % 4096
    cs = O.compute_cos_sin_cache(64, 4096, 10000).to(dev)
    n_pages = (T + page - 1) // page + 1
    slots = torch.randperm(n_pages * page, device=dev, generator=g)[:T].to(torch.int32)
    ckv = torch.zeros(n_pages, page, 512, dtype=torch.bfloat16, device=dev)
    kpe = torch.zeros(n_pages, page, 64, dtype=torch.bfloat16, device=dev)
    normed = torch.empty(T, 512, dtype=torch.bfloat16, device=dev)
    k_pe = latent[:, 512:].view(T, 1, 64)      # RoPE in place on the projection output, as the unfused layer does
    dummy_c, dummy_k = torch.empty_like(ckv), torch.empty_like(kpe)

    def fused():
        ops.mla_cache_latent(latent, gamma, 1e-6, pos, cs, slots, ckv, kpe, interleaved=True)

    def four():
        ops.rms_norm(normed, latent[:, :512], gamma, 1e-6)
        ops.rotary_embedding(pos, k_pe, None, cs, is_neox=False)
        ops.reshape_paged_cache(slots, normed.view(T, 1, 512), normed.view(T, 1, 512), ckv.view(n_pages, page, 1, 512),
                                dummy_c.view(n_pages, page, 1, 512))
        ops.reshape_paged_cache(slots, k_pe, k_pe, kpe.view(n_pages, page, 1, 64), dummy_k.view(n_pages, page, 1, 64))
    return fused, four, T * (576 * 2 + 576 * 2 + 8 + 4)


ATTN_SHAPES = ([("decode", 16, b, 1, ctx) for ctx in (4096, 32768) for b in (1, 16, 64, 128)] +
               [("decode", 128, b, 1, 4096) for b in (1, 16, 64)] +
               [("mtp", 16, 64, 2, 4096)] +
               [("prefill", h, 1, 4096, 4096 + hist) for h in (16, 128) for hist in (0, 8192)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    ap.add_argument("--flashinfer", action="store_true", help="also time FlashInfer's MLA wrapper (JIT-builds its module if absent)")
    ap.add_argument("--prefill", action="store_true", help="time only the prefill forms and the selector grid")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "mla_sweep measures on the GPU; there is no CPU timing"
    dev_card = card()
    print(f"# card: {dev_card}")
    rows = []
    prefill_forms(a, rows)
    for kind, H, B, qo, kv in ([] if a.prefill else ATTN_SHAPES):
        run, by, fl, splits, d = attention_case(B, H, qo, kv)
        iters = max(3, a.iters // (20 if kind == "prefill" else 1))
        t, how = time_it(run, iters, a.warmup)
        t_mem, t_fl = by / HBM, fl / BF16_PEAK
        bound = "HBM" if t_mem >= t_fl else "BF16"
        row = dict(kind=kind, H=H, B=B, qo=qo, kv=kv, splits=splits, us=t * 1e6, TBps=by / t / 1e12, TFLOPs=fl / t / 1e12,
                   bound=bound, share=max(t_mem, t_fl) / t, timing=how)
        fi = flashinfer_mla(d, B, H, qo, kv) if a.flashinfer else None
        if callable(fi):
            t_fi, how_fi = time_it(fi, iters, a.warmup)
            row["flashinfer_us"], row["flashinfer_timing"] = t_fi * 1e6, how_fi
        elif fi is not None:
            row["flashinfer"] = f"unavailable: {fi}"
        rows.append(row)
        fi_s = (f"  flashinfer {row['flashinfer_us']:9.1f} us ({row['flashinfer_timing']}, ours / theirs "
                f"{t * 1e6 / row['flashinfer_us']:.2f})" if "flashinfer_us" in row else f"  {row.get('flashinfer', '')}")
        print(f"{kind:8s} H={H:3d} B={B:3d} qo={qo:4d} kv={kv:6d} splits={splits:3d}  {t * 1e6:9.1f} us  "
              f"{row['TBps']:5.2f} TB/s  {row['TFLOPs']:6.1f} TFLOP/s  {100 * row['share']:5.1f}% of {bound} bound ({how}){fi_s}")
        del d
        torch.cuda.empty_cache()
    for T in (() if a.prefill else (1, 64, 8192)):
        fused, four, by = writer_case(T)
        (tf, _), (t4, _) = time_it(fused, a.iters, a.warmup), time_it(four, a.iters, a.warmup)
        rows.append(dict(kind="writer", T=T, us=tf * 1e6, four_launch_us=t4 * 1e6))
        print(f"writer   T={T:5d}  fused {tf * 1e6:7.2f} us   four launches {t4 * 1e6:7.2f} us   ({by / tf / 1e9:.0f} GB/s fused)")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=dev_card, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
