"""GPU parity of this library's elementwise kernels against the REFERENCE'S OWN kernels (activation.cu, norm.cu, rope.cu,
reshape_paged_cache.cu, fp8_quant.cu, fused_qknorm_rope.cu, moe/moe_fused_topk.cu, llm_decode_metadata_update.cu), on the same
seeded inputs.  Prints one JSON object: per op the number of cases, how many were bit-identical, the largest difference in units
of the output format's last place (max_ulps) and the worst case otherwise.  Runs in its own process so that a fault inside a
kernel cannot take the test session with it.
  python tools/ref_kernel_parity.py [out.json]                          live: against oracle/_ref (built by oracle/build_ref.py)
  python tools/ref_kernel_parity.py --save-golden tests/golden/ref_kernels.npz [out.json]
                                                                        live, and store seeded samples of the reference outputs
  python tools/ref_kernel_parity.py --check-golden tests/golden/ref_kernels.npz [out.json]
                                                                        against the stored samples (no reference library needed;
                                                                        tests/test_gpu_zzz_ref_kernels.py)"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DEV, BF16, E4M3 = "cuda", torch.bfloat16, torch.float8_e4m3fn
SAMPLES = 512          # stored elements per output tensor (all of it when smaller)
MANTISSA = {BF16: 7, E4M3: 3, torch.float32: 23}


def _sample_index(n):
    """fixed, seeded positions of a flattened output of n elements"""
    import numpy as np
    if n <= SAMPLES:
        return torch.arange(n)
    return torch.from_numpy(np.sort(np.random.RandomState(n % (2 ** 31)).choice(n, SAMPLES, replace=False)))


class _NoReference:
    """stands in for the reference library in --check-golden mode: its outputs come from the stored samples"""

    def fp8_scaled_quantize(self, x, *_):
        return torch.zeros_like(x, dtype=E4M3), torch.zeros(1, device=x.device)

    def moe_fused_topk(self, logits, k, *_):
        return torch.zeros(logits.size(0), k, device=logits.device), torch.zeros(logits.size(0), k, dtype=torch.int32,
                                                                                 device=logits.device)

    def __getattr__(self, name):
        return lambda *a, **k: None


def main():
    import numpy as np
    from xllm_b200 import ops
    args = sys.argv[1:]
    save = check = None
    if args[:1] == ["--save-golden"]:
        save, args = args[1], args[2:]
    elif args[:1] == ["--check-golden"]:
        check, args = args[1], args[2:]
    if check:
        ref, golden = _NoReference(), dict(np.load(check))
    else:
        from oracle import build_ref
        ref, golden = build_ref.load(), {}
        if ref is None:
            print(json.dumps({"unavailable": "oracle/_ref is not built and the reference tree is absent"}))
            return 1
    stored = {}
    g = torch.Generator(device=DEV).manual_seed(2026)
    res = {}

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g, device=DEV) * scale).to(BF16)

    def record(op, case, pairs):
        """pairs of (this library's output, the reference's output); both are compared on the stored sample positions"""
        r = res.setdefault(op, {"cases": 0, "bit_identical": 0, "worst": None, "errors": [], "max_ulps": 0.0, "max_rel_diff": 0.0})
        r["cases"] += 1
        same, d, n = True, 0.0, 0
        for i, (a, b) in enumerate(pairs):
            key = f"{op}|{case}|{i}"
            idx = _sample_index(a.numel()).to(a.device)
            va = a.reshape(-1)[idx].float()
            if check:
                if key not in golden:
                    raise KeyError(f"no stored reference output {key}")
                vb = torch.from_numpy(golden[key]).to(a.device)
            else:
                vb = b.reshape(-1)[idx].float()
                stored[key] = vb.cpu().numpy().astype(np.float32)
            diff = (va - vb).abs()
            if bool((diff > 0).any()) or bool(torch.isnan(va).ne(torch.isnan(vb)).any()):
                same = False
                d, n = max(d, diff.max().item()), n + int((diff > 0).sum())
            m = MANTISSA.get(a.dtype)
            if m is not None:
                ulp = torch.exp2(torch.floor(torch.log2(vb.abs().clamp_min(2.0 ** -126))) - m)
                r["max_ulps"] = max(r["max_ulps"], (diff / ulp).max().item())
                r["max_rel_diff"] = max(r["max_rel_diff"], (diff / vb.abs().clamp_min(1e-30)).max().item())
            elif bool((diff > 0).any()):
                r["max_ulps"] = float("inf")            # integer / index output: any difference is a mismatch
        if same:
            r["bit_identical"] += 1
        elif r["worst"] is None or d > r["worst"]["max_abs_diff"]:
            r["worst"] = {"case": case, "max_abs_diff": d, "elements_differing": n}

    out_path = args[0] if args else None

    def dump():
        """partial results after every comparison: if a later kernel takes the process down, what ran before is still on disk"""
        if out_path:
            with open(out_path, "w") as f:
                json.dump({"device": torch.cuda.get_device_name(0), "ops": res, "complete": False}, f, indent=1)

    def guarded(op, case, fn):
        """one comparison; an exception of either implementation (unsupported shape, failed check) is recorded, not fatal"""
        try:
            fn()
        except Exception as e:                                             # noqa: BLE001
            r = res.setdefault(op, {"cases": 0, "bit_identical": 0, "worst": None, "errors": []})
            r["cases"] += 1
            r["errors"].append(f"{case}: {type(e).__name__}: {str(e)[:160]}")
        try:
            torch.cuda.synchronize()
            dump()
        except Exception:                                                  # noqa: BLE001
            pass

    for T, H in ((7, 3584), (64, 4096), (1, 256), (33, 1024), (300, 8192)):
        x, r0, w = rnd(T, H), rnd(T, H), (1 + 0.1 * torch.randn(H, generator=g, device=DEV)).to(BF16)
        s = torch.tensor([0.05], device=DEV)
        case = f"{T}x{H}"

        def norm():
            a, b = torch.empty_like(x), torch.empty_like(x)
            ops.rms_norm(a, x, w, 1e-6)
            ref.rms_norm(b, x, w, 1e-6)
            record("rms_norm", case, [(a, b)])

        def add_norm():
            x1, r1, x2, r2 = x.clone(), r0.clone(), x.clone(), r0.clone()
            ops.fused_add_rms_norm(x1, r1, w, 1e-6)
            ref.fused_add_rms_norm(x2, r2, w, 1e-6)
            record("fused_add_rms_norm", case, [(x1, x2), (r1, r2)])

        def norm_q():
            q1, q2 = torch.empty(T, H, dtype=E4M3, device=DEV), torch.empty(T, H, dtype=E4M3, device=DEV)
            ops.rms_norm_static_fp8_quant(q1, x, w, s, 1e-6)
            ref.rms_norm_static_fp8_quant(q2, x, w, s, 1e-6)
            record("rms_norm_static_fp8_quant", case, [(q1, q2)])

        def add_norm_q():
            q1, q2 = torch.empty(T, H, dtype=E4M3, device=DEV), torch.empty(T, H, dtype=E4M3, device=DEV)
            x1, r1, x2, r2 = x.clone(), r0.clone(), x.clone(), r0.clone()
            ops.fused_add_rms_norm_static_fp8_quant(q1, x1, r1, w, s, 1e-6)
            ref.fused_add_rms_norm_static_fp8_quant(q2, x2, r2, w, s, 1e-6)
            record("fused_add_rms_norm_static_fp8_quant", case, [(q1, q2), (r1, r2)])

        def quant():
            big = rnd(T, H, scale=5.0)
            big[0, 0] = 3000.0
            for sv in (0.5, 0.02):
                sc = torch.tensor([sv], device=DEV)
                q1, q2 = torch.empty(T, H, dtype=E4M3, device=DEV), torch.empty(T, H, dtype=E4M3, device=DEV)
                ops.static_scaled_fp8_quant(q1, big, sc)
                ref.static_scaled_fp8_quant(q2, big, sc)
                record("static_scaled_fp8_quant", f"{case} scale {sv}", [(q1, q2)])
        for op, fn in (("rms_norm", norm), ("fused_add_rms_norm", add_norm), ("rms_norm_static_fp8_quant", norm_q),
                       ("fused_add_rms_norm_static_fp8_quant", add_norm_q), ("static_scaled_fp8_quant", quant)):
            guarded(op, case, fn)
    for T, d in ((7, 18944), (4 * 7, 64), (28, 129), (33, 1024)):
        gu = rnd(T, 2 * d, scale=0.5)
        for mode in ("silu", "gelu", "gelu_tanh"):
            def act():
                o1, o2 = torch.empty(T, d, dtype=BF16, device=DEV), torch.empty(T, d, dtype=BF16, device=DEV)
                ops.act_and_mul(o1, gu, mode)
                ref.act_and_mul(o2, gu, mode)
                record("act_and_mul", f"{T}x{d} {mode}", [(o1, o2)])
            guarded("act_and_mul", f"{T}x{d} {mode}", act)
    from xllm_b200.qwen2 import Qwen2Config, make_cos_sin_cache
    for T, HQ, HKV, D, neox in ((6, 8, 2, 16, True), (5, 6, 2, 8, False), (33, 28, 4, 128, True), (128, 32, 8, 64, True), (1, 64, 8, 128, True),
                                (7, 8, 2, 64, False)):
        def rope():
            cfg = Qwen2Config(hidden_size=HQ * D, num_layers=1, n_heads=HQ, n_kv_heads=HKV, head_dim=D, intermediate_size=64, vocab_size=64,
                              max_position_embeddings=max(64, T + 8), block_size=16, quant="bf16", name="rope")
            cache = make_cos_sin_cache(cfg, DEV)
            pos = torch.tensor([(i * 3 + 1) % cache.size(0) for i in range(T)], dtype=torch.int64, device=DEV)
            q, k = rnd(T, HQ * D), rnd(T, HKV * D)
            q1, k1, q2, k2 = q.clone(), k.clone(), q.clone(), k.clone()
            ops.rotary_embedding(pos, q1, k1, cache, neox)
            ref.rotary_embedding(pos, q2, k2, cache, neox)
            record("rotary_embedding", f"T{T} {HQ}/{HKV}x{D} neox={neox}", [(q1, q2), (k1, k2)])
        guarded("rotary_embedding", f"T{T} {HQ}/{HKV}x{D} neox={neox}", rope)
    for n_tokens, n_blocks, bs, hkv, D in ((4, 1, 16, 1, 64), (32, 8, 16, 4, 128), (64, 4, 64, 8, 128), (256, 16, 64, 8, 128), (1, 4, 16, 4, 128)):
        def scatter():
            keys, vals = rnd(n_tokens, hkv, D), rnd(n_tokens, hkv, D)
            slots = torch.randperm(n_blocks * bs, generator=g, device=DEV)[:n_tokens].to(torch.int32)
            kc1 = torch.zeros(n_blocks, bs, hkv, D, dtype=BF16, device=DEV)
            vc1, kc2, vc2 = torch.zeros_like(kc1), torch.zeros_like(kc1), torch.zeros_like(kc1)
            ops.reshape_paged_cache(slots, keys, vals, kc1, vc1)
            ref.reshape_paged_cache(slots, keys, vals, kc2, vc2)
            record("reshape_paged_cache", f"{n_tokens} tokens {n_blocks}x{bs} blocks {hkv}x{D}", [(kc1, kc2), (vc1, vc2)])
        guarded("reshape_paged_cache", f"{n_tokens} tokens", scatter)
    for T, hq, hk, D, maxpos, inter in ((17, 8, 4, 128, 512, False), (11, 6, 2, 64, 256, True), (3, 16, 2, 128, 64, False)):
        def qknorm():
            qkv = rnd(T, (hq + 2 * hk) * D, scale=0.2)
            qw, kw = rnd(D), rnd(D)
            cache = torch.randn(maxpos, D, generator=g, device=DEV).to(BF16)
            pos = torch.randint(0, maxpos, (T,), generator=g, device=DEV)
            a, b = qkv.clone(), qkv.clone()
            ops.fused_qk_norm_rope(a, hq, hk, hk, D, 1e-6, qw, kw, cache, inter, pos)
            ref.fused_qk_norm_rope(b, hq, hk, hk, D, 1e-6, qw, kw, cache, inter, pos)
            record("fused_qk_norm_rope", f"T{T} {hq}/{hk}x{D} interleaved={inter}", [(a, b)])
        guarded("fused_qk_norm_rope", f"T{T} {hq}/{hk}x{D} interleaved={inter}", qknorm)
    # dynamic per-tensor FP8 quantisation (fp8_scaled_quantize.cpp:36-41: the scale is formed in the tensor's dtype, then cast)
    for T, H, sc_ in ((7, 3584, 1.0), (32, 8192, 5.0), (1, 256, 0.01), (64, 1024, 40.0)):
        def dyn():
            x = rnd(T, H, scale=sc_)
            q1, s1 = ops.fp8_scaled_quantize(x)
            q2, s2 = ref.fp8_scaled_quantize(x, None, None)
            record("fp8_scaled_quantize", f"{T}x{H} x{sc_}", [(q1, q2), (s1.reshape(-1).float(), s2.reshape(-1).float())])
        guarded("fp8_scaled_quantize", f"{T}x{H} x{sc_}", dyn)
    # MoE router (n4): moe_fused_topk.cu + moe_topk_{softmax,sigmoid}_kernels.cuh
    for T, E, k, dt in ((7, 16, 2, torch.float32), (33, 64, 8, torch.float32), (512, 16, 2, BF16), (5, 256, 8, BF16), (1, 8, 1, torch.float32)):
        logits = (torch.randn(T, E, generator=g, device=DEV) * 3).to(dt)
        bias = torch.randn(E, generator=g, device=DEV) * 0.1
        for scoring, use_bias in (("softmax", False), ("sigmoid", False), ("sigmoid", True)):
            for renorm in (True, False):
                name = f"{T}x{E} top{k} {str(dt).split('.')[-1]} {scoring} bias={use_bias} renorm={renorm}"

                def router():
                    w1, i1 = ops.moe_fused_topk(logits, k, renorm, bias if use_bias else None, scoring)
                    w2, i2 = ref.moe_fused_topk(logits.clone(), k, renorm, bias if use_bias else None, scoring)
                    record("moe_fused_topk_ids", name, [(i1.to(torch.int64), i2.to(torch.int64))])          # index work: must be identical
                    record("moe_fused_topk_weights", name, [(w1.float(), w2.float())])                      # fp32: 1e-6 relative stated in the test
                guarded("moe_fused_topk_ids", name, router)
    # CUDA-graph decode metadata refresh (n3): llm_decode_metadata_update.cu - integer work, every destination buffer compared whole
    I32 = torch.int32
    FIELDS = ("tokens", "positions", "new_cache_slots", "kv_seq_lens", "paged_kv_indptr", "paged_kv_indices", "paged_kv_last_page_len")
    DFIELDS = ("tokens", "positions", "new_cache_slots", "kv_seq_lens", "kv_seq_lens_delta", "paged_kv_indptr", "paged_kv_indices",
               "paged_kv_last_page_len")
    for n_tok, padded, batch, n_idx in ((5, 8, 5, 37), (1, 1, 1, 1), (64, 64, 64, 4000), (3, 16, 3, 0), (300, 512, 300, 70000)):
        def metadata():
            ri = lambda n, hi=100000: torch.randint(0, hi, (n,), generator=g, device=DEV, dtype=I32)
            zero = torch.zeros(1, dtype=I32, device=DEV)
            src = dict(tokens=ri(n_tok), positions=ri(n_tok), new_cache_slots=ri(n_tok),
                       kv_seq_lens=torch.cat([zero, ri(batch, 500).cumsum(0).to(I32)]),
                       paged_kv_indptr=torch.cat([zero, ri(batch, 40).cumsum(0).to(I32)]), paged_kv_indices=ri(max(n_idx, 1)),
                       paged_kv_last_page_len=ri(max(batch, 1), 128) + 1)
            cap_tok, cap_batch, cap_idx = max(padded, n_tok) + 7, batch + 5, n_idx + 11
            dst = dict(tokens=ri(cap_tok), positions=ri(cap_tok), new_cache_slots=ri(cap_tok), kv_seq_lens=ri(cap_batch + 1),
                       kv_seq_lens_delta=ri(cap_batch), paged_kv_indptr=ri(cap_batch + 1), paged_kv_indices=ri(cap_idx),
                       paged_kv_last_page_len=ri(cap_batch))
            d1 = {k_: v.clone() for k_, v in dst.items()}
            d2 = {k_: v.clone() for k_, v in dst.items()}
            ops.update_llm_decode_metadata(src, d1, n_tok, padded, batch, n_idx)
            ref.update_llm_decode_metadata([src[f] for f in FIELDS], [d2[f] for f in DFIELDS], n_tok, padded, batch, n_idx)
            record("update_llm_decode_metadata", f"tokens {n_tok}/{padded} batch {batch} indices {n_idx}", [(d1[f], d2[f]) for f in DFIELDS])
        guarded("update_llm_decode_metadata", f"tokens {n_tok}/{padded} batch {batch}", metadata)
    torch.cuda.synchronize()
    if save:
        np.savez_compressed(save, **stored)
    out = {"device": torch.cuda.get_device_name(0), "ops": res, "complete": True, "mode": "stored" if check else "live"}
    print(json.dumps(out))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
