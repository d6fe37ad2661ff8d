"""Qwen3 dense (Qwen2Config.qk_norm): the oracle composition and the runner-side helpers of tests/model_parity.py with the
per-head q / k RMSNorm of Qwen2AttentionImpl's is_qwen3_style_ branch (qwen2_attention.cpp:40-80, 132-193): no qkv bias,
head_dim independent of hidden / n_heads, fused_qk_norm_rope (NeoX) in place of rotary_embedding (:147-171).
Used by tests/test_qwen3_*_cpu.py and tests/test_gpu_qwen3_*.py."""
import torch

from oracle import layer as OL
from oracle import ops as O
from tests import model_parity as MP

BF16 = torch.bfloat16


class Qwen3AttentionOracle(OL.Qwen2AttentionOracle):
    """Qwen2AttentionOracle with the Qwen3 q / k norm: qkv -> fused_qk_norm_rope (per-head RMSNorm with q_norm_w / k_norm_w,
    then NeoX RoPE, fused_qknorm_rope.cu:84-300) -> KV scatter + attention -> o_proj."""

    def __init__(self, n_heads, n_kv_heads, head_dim, cos_sin_cache, q_norm_w, k_norm_w, eps, linear, o_linear):
        super().__init__(None, None, None, n_heads, n_kv_heads, head_dim, cos_sin_cache, linear=linear, o_linear=o_linear)
        self.q_norm_w, self.k_norm_w, self.eps = q_norm_w, k_norm_w, eps

    def forward(self, positions, hidden, meta, k_cache, v_cache):
        qkv = self.linear(hidden, self.qkv_w, self.qkv_b)
        hq, hkv, D = self.n_heads, self.n_kv_heads, self.head_dim
        qkv = O.fused_qk_norm_rope(qkv.contiguous(), hq, hkv, hkv, D, self.eps, self.q_norm_w, self.k_norm_w,
                                   self.cos_sin_cache, False, positions)
        qs, kvs = hq * D, hkv * D
        out = OL.attention_forward(meta, qkv[:, :qs].contiguous(), qkv[:, qs:qs + kvs].contiguous(),
                                   qkv[:, qs + kvs:].contiguous(), k_cache, v_cache, self.scale, hq, hkv, D)
        return self.o_linear(out, self.o_w, None)


def build_case(cfg, B, kv_lens, seed=2026, w_std=0.05):
    """tests/model_parity.build_case plus per-layer q_norm / k_norm [head_dim] (drawn from their own generator, so the rest
    of the case is the Qwen2 helper's)."""
    assert cfg.qk_norm and not cfg.qkv_bias
    W, kcs, vcs, meta = MP.build_case(cfg, B, kv_lens, seed, w_std)
    g = torch.Generator().manual_seed(seed + 1)
    for L in W["layers"]:
        L["q_norm"] = (1 + 0.1 * torch.randn(cfg.head_dim, generator=g)).to(BF16)
        L["k_norm"] = (1 + 0.1 * torch.randn(cfg.head_dim, generator=g)).to(BF16)
    return W, kcs, vcs, meta


def _cos_sin(cfg):
    return O.compute_cos_sin_cache(cfg.head_dim, cfg.max_position_embeddings, cfg.rope_theta, BF16)


def decoder_layer(cfg, L, cs):
    attn = Qwen3AttentionOracle(cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, cs, L["q_norm"], L["k_norm"], cfg.rms_norm_eps,
                                MP._olin(L["qkv"]), MP._olin(L["o"]))
    return OL.Qwen2DecoderLayerOracle(attn, L["input_norm"], L["post_norm"], cfg.rms_norm_eps, MP._olin(L["gate_up"]),
                                      MP._olin(L["down"]))


def _decode_meta(meta):
    B = len(meta["tokens"])
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)
    return OL.AttnMeta(False, False, torch.arange(B + 1, dtype=torch.int32), None, i32(meta["slots"]), i32(meta["indptr"]),
                       i32(meta["indices"]), i32(meta["last"]))


def _model(cfg, W, kcs, vcs, tokens, positions, am):
    cs = _cos_sin(cfg)
    x, residual = W["embed"][torch.tensor(tokens)], None
    for li, L in enumerate(W["layers"]):
        x, residual = decoder_layer(cfg, L, cs).forward(x, residual, positions, am, kcs[li], vcs[li])
    x, _ = O.fused_add_rms_norm(x, residual, W["final_norm"], cfg.rms_norm_eps)
    return x


def oracle_step(cfg, W, kcs, vcs, meta):
    """one decode step of the oracle (caches updated in place): (logits bf16 [B, vocab], next tokens)."""
    x = _model(cfg, W, kcs, vcs, meta["tokens"], torch.tensor(meta["positions"]), _decode_meta(meta))
    logits = O.linear(x, W["lm_head"])
    return logits, logits.to(torch.float32).argmax(-1)


def oracle_prefill(cfg, W, kcs, vcs, tokens, meta, chunked):
    """ragged (chunked=False) or chunked prefill of the oracle; meta: oracle.batch.PagedMeta.  Last-token logits [B, vocab]."""
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)
    am = OL.AttnMeta(True, chunked, i32(meta.q_cu_seq_lens), i32(meta.kv_cu_seq_lens), i32(meta.new_cache_slots),
                     i32(meta.paged_kv_indptr), i32(meta.paged_kv_indices), i32(meta.paged_kv_last_page_len))
    x = _model(cfg, W, kcs, vcs, tokens, torch.tensor(meta.positions), am)
    return O.linear(x[torch.tensor(meta.q_cu_seq_lens[1:]) - 1], W["lm_head"])


def upload(cfg, W, device="cuda"):
    """tests/model_parity.upload with the qkv projection in the plain layout (the rope-pair order of the W4 decode GEMV's
    RoPE epilogue does not apply under QK-norm) and the q_norm / k_norm weights."""
    from xllm_b200 import quant
    from xllm_b200.qwen2 import Linear
    w = MP.upload(cfg, W, device)
    for L, d in zip(w.layers, W["layers"]):
        L["q_norm"], L["k_norm"] = d["q_norm"].to(device), d["k_norm"].to(device)
        if cfg.quant == "w4a16":
            q = d["qkv"]
            lin = Linear(cfg.q_size + 2 * cfg.kv_size, cfg.hidden_size, "w4a16", cfg.group_size)
            qw, meta = quant.pack_w4(q["q"], q["s"], q["z"], cfg.group_size)
            lin.qweight, lin.meta = qw.to(device), meta.to(device)
            L["qkv"] = lin
    return w


def _runner(cfg, W, kcs, vcs, meta, kv_lens, fused=True):
    from xllm_b200.qwen2 import Qwen2DecodeRunner
    runner = Qwen2DecodeRunner(cfg, upload(cfg, W), len(kv_lens), max(kv_lens), num_blocks=meta["nblocks"],
                               fused_rope_cache=fused)
    for li in range(cfg.num_layers):
        runner.k_caches[li].copy_(kcs[li])
        runner.v_caches[li].copy_(vcs[li])
    runner.set_inputs_host(meta["tokens"], meta["positions"], meta["slots"], meta["indptr"], meta["indices"], meta["last"])
    return runner


def run_decode_parity(cfg, kv_lens, use_graph=True, fused=True, seed=2026):
    """tests/model_parity.run_decode_parity for Qwen3: (logits, oracle logits, tokens, oracle tokens, runner, caches)."""
    W, kcs, vcs, meta = build_case(cfg, len(kv_lens), kv_lens, seed)
    runner = _runner(cfg, W, kcs, vcs, meta, kv_lens, fused)
    if use_graph:
        runner.step()            # eager once (module load), then capture
        for li in range(cfg.num_layers):
            runner.k_caches[li].copy_(kcs[li])
            runner.v_caches[li].copy_(vcs[li])
        runner.capture()
    nxt = runner.step().clone()
    logits = runner.logits.cpu()
    ref_logits, ref_next = oracle_step(cfg, W, kcs, vcs, meta)
    return logits, ref_logits, nxt, ref_next, runner, (kcs, vcs)


def run_layerwise_parity(cfg, kv_lens, seed=2026, w_std=0.05):
    """tests/model_parity.run_layerwise_parity for Qwen3: every oracle layer is fed the GPU's own state before that layer.
    Returns a list of (gpu_h, ref_h, gpu_res, ref_res) per layer."""
    W, kcs, vcs, meta = build_case(cfg, len(kv_lens), kv_lens, seed, w_std)
    runner = _runner(cfg, W, kcs, vcs, meta, kv_lens)
    for d, h in ((runner.token_ids, runner.h_token_ids), (runner.positions, runner.h_positions), (runner.slots, runner.h_slots),
                 (runner.kv_indptr, runner.h_kv_indptr), (runner.kv_indices, runner.h_kv_indices), (runner.kv_last, runner.h_kv_last)):
        d.copy_(h)
    trace = []
    runner.launch_step(trace)
    torch.cuda.synchronize()
    cs, am, positions = _cos_sin(cfg), _decode_meta(meta), torch.tensor(meta["positions"])
    res_in = W["embed"][torch.tensor(meta["tokens"])]
    h_in = O.rms_norm(res_in, W["layers"][0]["input_norm"], cfg.rms_norm_eps)
    out = []
    for li, L in enumerate(W["layers"]):
        # the runner's state convention: (normalised layer input, residual stream) -> the next layer's
        a = decoder_layer(cfg, L, cs).attn.forward(positions, h_in, am, kcs[li].clone(), vcs[li].clone())
        h_mid, res_mid = O.fused_add_rms_norm(a, res_in, L["post_norm"], cfg.rms_norm_eps)
        down = MP._olin(L["down"])(O.act_and_mul(MP._olin(L["gate_up"])(h_mid), "silu"))
        next_w = W["layers"][li + 1]["input_norm"] if li + 1 < cfg.num_layers else W["final_norm"]
        ref_h, ref_res = O.fused_add_rms_norm(down, res_mid, next_w, cfg.rms_norm_eps)
        gh, gres = trace[li][0].cpu(), trace[li][1].cpu()
        out.append((gh, ref_h, gres, ref_res))
        h_in, res_in = gh, gres          # teacher forcing
    return out
