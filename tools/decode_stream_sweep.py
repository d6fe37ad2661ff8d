"""Development aid (not the bench contract): where the decode step's weight stream goes, at bench.py's shapes (Qwen2-7B
W4A16, batch 1, group 128).

  python tools/decode_stream_sweep.py OUT [name=path/to/libxllm_b200_ops.so ...]

prints the card and its power limit, then times qkv (rope epilogue), o, gate_up (SiLU*mul epilogue), down and the bf16
lm_head as 28 PDL-chained launches over 28 layers' weights (4 copies of the lm_head; both far past L2) and as isolated
launches, for the library in the tree and every library given (e.g. one built from another commit), alternating them,
three repetitions each.  It checks that every library computes the same bits as the first one and writes the results to
OUT/sweep.json.  Give only libraries built from sources whose bf16 small-M kernel takes no dynamic shared memory next
to the one in the tree: with two such libraries in one process the second one's lm_head launches failed with an
invalid argument (most likely both libraries' identically named template functions resolve to the first library's).
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TBS = 3.35        # H100 SXM data sheet, HBM3
LAYERS = 28
H, I, NH, NKV, D, V, GS = 3584, 18944, 28, 4, 128, 152064, 128


def run(out, extra):
    import torch
    from xllm_b200 import _lib, ops
    dev, bf16 = "cuda", torch.bfloat16
    libs = {"shipped": _lib.LIB_PATH}
    for a in extra:
        k, v = a.split("=", 1)
        libs[k] = os.path.abspath(v)
    handles = {}

    def use(name):          # every ops.* call goes through _lib.lib(): point it at one library
        if name not in handles:
            _lib._lib, _lib.LIB_PATH = None, libs[name]
            handles[name] = _lib.lib()
        _lib._lib = handles[name]

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "times": {}, "equal": {}}
    print("gpu:", smi, flush=True)
    torch.manual_seed(0)

    def w4(N, K):
        qw = torch.randint(-2 ** 31, 2 ** 31 - 1, (N // 16, K // 64, 32, 4), dtype=torch.int32, device=dev)
        s = (torch.rand(K // GS, N, device=dev) * 0.01 + 0.001).to(bf16).view(torch.int16).to(torch.int32) & 0xFFFF
        return qw, (s | (0x4308 << 16)).contiguous()

    x_h, x_i = torch.randn(1, H, device=dev, dtype=bf16), torch.randn(1, I, device=dev, dtype=bf16)
    pos = torch.full((1,), 4095, dtype=torch.int64, device=dev)
    cs = torch.randn(8192, D, device=dev, dtype=bf16)
    slots = torch.tensor([130], dtype=torch.int32, device=dev)
    kc = torch.zeros(2, 128, NKV, D, device=dev, dtype=bf16)
    vc = torch.zeros_like(kc)
    shapes = {  # name: (N, K, x, out columns, epilogue)
        "qkv": ((NH + 2 * NKV) * D, H, x_h, (NH + 2 * NKV) * D, 2),
        "o": (H, H, x_h, H, 0),
        "gate_up": (2 * I, H, x_h, I, 1),
        "down": (H, I, x_i, H, 0),
    }

    def timed(fns):
        """(chained us per launch, isolated us per launch)"""
        for f in fns:
            f()
        torch.cuda.synchronize()
        torch.cuda._sleep(int(20e6))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 5
        a.record()
        for _ in range(reps):
            for f in fns:
                f()
        b.record()
        torch.cuda.synchronize()
        ch = a.elapsed_time(b) * 1e3 / (reps * len(fns))
        iso = []
        for f in fns:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            iso.append(e0.elapsed_time(e1) * 1e3)
        iso.sort()
        return ch, iso[len(iso) // 2]

    def measure(name, nbytes, make_fns, outs):
        ref = None
        for rep in range(3):
            for ln in libs:
                use(ln)
                fns = make_fns()
                ch, iso = timed(fns)
                res["times"].setdefault(f"{name}/{ln}", []).append({"chained_us": ch, "isolated_us": iso})
                print(f"{name:8s} {ln:8s} rep {rep} chained {ch:8.2f} us ({nbytes / ch / 1e6 / PEAK_TBS:6.1%})  isolated {iso:8.2f} us "
                      f"({nbytes / iso / 1e6 / PEAK_TBS:6.1%})", flush=True)
                if rep == 0:
                    for o in outs:
                        o.fill_(0)
                    fns[0]()
                    torch.cuda.synchronize()
                    got = [o.clone() for o in outs]
                    if ref is None:
                        ref = got
                    eq = all(torch.equal(p, q) for p, q in zip(ref, got))
                    res["equal"][f"{name}/{ln}"] = eq
                    np_dir = os.path.join(out, "outputs", ln)
                    os.makedirs(np_dir, exist_ok=True)
                    torch.save([g.cpu() for g in got], os.path.join(np_dir, f"{name}.pt"))
                    print(f"{name:8s} {ln:8s} output equal to {next(iter(libs))}: {eq}", flush=True)

    for name, (N, K, x, ncol, epi) in shapes.items():
        ws = [w4(N, K) for _ in range(LAYERS)]
        y = torch.empty(1, ncol, dtype=bf16, device=dev)
        nbytes = N * K // 2 + (K // GS) * N * 4 + K * 2 + ncol * 2
        if epi == 2:
            def make(ws=ws, y=y, x=x):
                return [lambda w=w: ops.w4a16_decode_fused(x, w[0], w[1], GS, None, y, epilogue="rope_cache", positions=pos,
                                                           cos_sin_cache=cs, slot_ids=slots, key_cache=kc, value_cache=vc,
                                                           num_heads=NH, num_kv_heads=NKV, head_dim=D) for w in ws]
            outs = [y, kc, vc]
        elif epi == 1:
            def make(ws=ws, y=y, x=x):
                return [lambda w=w: ops.w4a16_gate_up_act(x, w[0], w[1], GS, "silu", None, y) for w in ws]
            outs = [y]
        else:
            def make(ws=ws, y=y, x=x):
                return [lambda w=w: ops.w4a16_linear(x, w[0], w[1], GS, None, y) for w in ws]
            outs = [y]
        measure(name, nbytes, make, outs)
        del ws
        torch.cuda.empty_cache()
    # lm_head: 4 copies of the bf16 [V, H] weight (4.4 GB, far past L2)
    lm = [(torch.randn(V, H, device=dev) * 0.02).to(bf16) for _ in range(4)]
    logits = torch.empty(1, V, dtype=bf16, device=dev)
    measure("lm_head", V * H * 2 + H * 2 + V * 2, lambda: [lambda w=w: ops.matmul_small_m(x_h, w, None, logits) for w in lm], [logits])
    with open(os.path.join(out, "sweep.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    os.makedirs(sys.argv[1], exist_ok=True)
    run(sys.argv[1], sys.argv[2:])
