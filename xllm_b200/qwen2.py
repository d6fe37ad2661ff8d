"""Decode-step driver for the Qwen2 decoder stack on top of the C-ABI ops.

Mirrors the reference composition (call stack B of SURVEY.md section 3):
  LlmModelImplBase::forward            xllm/models/llm/llm_model_base.h:60-131
  Qwen2DecoderLayerImpl::forward       xllm/core/layers/qwen2_decoder_layer.cpp:89-112
  Qwen2AttentionImpl::forward          xllm/core/layers/common/qwen2_attention.cpp:132-193
  DenseMLPImpl::forward                xllm/core/layers/common/dense_mlp.cpp:97-118
with the per-layer launches of this library.  One decode step = one replay of
a CUDA graph made only of libxllm_b200_ops launches chained with PDL.
The integer inputs of a step (token ids, positions, new_cache_slots, the paged
triplet) are exactly the reference's ForwardInput integers
(batch_input_builder.cpp:739-831) and are copied from pinned host memory.
"""
from dataclasses import dataclass
from typing import List, Optional

import os

import torch

from . import ops, quant

BF16 = torch.bfloat16


@dataclass
class Qwen2Config:
    hidden_size: int = 3584
    num_layers: int = 28
    n_heads: int = 28
    n_kv_heads: int = 4
    head_dim: int = 128
    intermediate_size: int = 18944
    vocab_size: int = 152064
    rope_theta: float = 1000000.0
    rms_norm_eps: float = 1e-6
    max_position_embeddings: int = 32768
    block_size: int = 128                 # kv_cache_config.cpp:21
    quant: str = "w4a16"                  # "w4a16" | "w8a16" | "bf16" | "fp8" (W8A8 per-tensor static, linear.cpp:137-182)
    group_size: int = 128
    tie_word_embeddings: bool = False
    qkv_bias: bool = True                 # qwen2_attention.cpp:52; Llama: False
    # Llama-3.1 "rope_scaling" {"rope_type": "llama3", factor, low_freq_factor, high_freq_factor,
    # original_max_position_embeddings}; None = plain rope_theta.  (The reference's llama.h parses these fields,
    # models/llm/npu/llama.h:341-346, but builds its table from rope_theta alone, :77-106; the CUDA registry entry of
    # integration/patches/0002 applies them.)
    rope_scaling: Optional[dict] = None
    # Qwen3: per-head RMSNorm of q and k (weights q_norm / k_norm [head_dim]) before RoPE (qwen2_attention.cpp:147-171)
    qk_norm: bool = False
    name: str = "Qwen2-7B"

    @staticmethod
    def qwen2_7b(**kw):
        return Qwen2Config(**kw)

    @staticmethod
    def qwen2_0_5b(**kw):
        d = dict(hidden_size=896, num_layers=24, n_heads=14, n_kv_heads=2, head_dim=64, intermediate_size=4864,
                 vocab_size=151936, quant="bf16", tie_word_embeddings=True, name="Qwen2-0.5B")
        d.update(kw)
        return Qwen2Config(**d)

    @staticmethod
    def llama3_70b(**kw):
        """BASELINE configs[3] architecture (the reference registers Llama only under models/llm/npu/llama3.h; the layer
        graph is Qwen2's without the qkv bias).  Llama-3-70B itself has no rope_scaling; pass
        rope_scaling=dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
        original_max_position_embeddings=8192) for the 3.1 checkpoints."""
        d = dict(hidden_size=8192, num_layers=80, n_heads=64, n_kv_heads=8, head_dim=128, intermediate_size=28672,
                 vocab_size=128256, rope_theta=500000.0, rms_norm_eps=1e-5, quant="fp8", qkv_bias=False,
                 max_position_embeddings=8192, name="Llama-3-70B")
        d.update(kw)
        return Qwen2Config(**d)

    @staticmethod
    def qwen3_8b(**kw):
        """Qwen3-8B (published config.json): head_dim 128 is not hidden / n_heads; no qkv bias, QK-norm."""
        d = dict(hidden_size=4096, num_layers=36, n_heads=32, n_kv_heads=8, head_dim=128, intermediate_size=12288,
                 vocab_size=151936, rope_theta=1000000.0, rms_norm_eps=1e-6, max_position_embeddings=40960,
                 qkv_bias=False, qk_norm=True, name="Qwen3-8B")
        d.update(kw)
        return Qwen2Config(**d)

    @staticmethod
    def qwen3_0_6b(**kw):
        """Qwen3-0.6B (published config.json): q_size 2048 over hidden 1024, tied embeddings."""
        d = dict(hidden_size=1024, num_layers=28, n_heads=16, n_kv_heads=8, head_dim=128, intermediate_size=3072,
                 vocab_size=151936, rope_theta=1000000.0, rms_norm_eps=1e-6, max_position_embeddings=40960,
                 qkv_bias=False, qk_norm=True, tie_word_embeddings=True, name="Qwen3-0.6B")
        d.update(kw)
        return Qwen2Config(**d)

    @property
    def q_size(self):
        return self.n_heads * self.head_dim

    @property
    def kv_size(self):
        return self.n_kv_heads * self.head_dim


class Linear:
    """One of qkv_proj / o_proj / gate_up_proj / down_proj / lm_head: y = x W^T (+b)."""

    def __init__(self, out_features, in_features, kind, group_size=128):
        self.N, self.K, self.kind, self.group_size = out_features, in_features, kind, group_size
        self.weight = None      # bf16 [N,K] (or e4m3 [N,K] for kind "fp8")
        self.qweight = None     # int32 tiles
        self.meta = None        # int32 [K/g, N]
        self.bias = None
        self.gate_up_interleaved = False   # w4a16 gate_up packed with quant.pack_w4_gate_up: activation fuses into the GEMV
        self.qkv_rope_packed = False       # w4a16 qkv packed with quant.pack_w4_qkv_rope: RoPE + KV scatter fuse into the GEMV
        self.weight_scale = None   # fp8: float32 [1] per-tensor weight scale
        self.input_scale = None    # fp8: float32 [1] static activation scale (None -> dynamic per-tensor)
        self._x8 = None

    def weight_bytes(self):
        if self.kind == "bf16":
            return self.weight.numel() * 2
        if self.kind == "fp8":
            return self.weight.numel()
        return self.qweight.numel() * 4 + self.meta.numel() * 4

    def forward(self, x, out):
        """M <= 16: HBM-bound streaming kernels; larger M: wgmma GEMMs.  fp8 follows fp8_linear_forward
        (linear.cpp:137-182): quantise the activation (static scale if present) then the scaled matmul."""
        if self.kind == "bf16":
            ops.matmul(x, self.weight, self.bias, out)
        elif self.kind == "fp8" and x.dtype == torch.float8_e4m3fn:
            # already quantised by the norm in front (RMSNormImpl::forward_fp8): fp8_linear_forward skips its own
            # quantisation and uses input_scale directly (linear.cpp:150-157)
            if self.input_scale is None:
                raise ValueError("input_scale must be provided when input is already FP8")
            ops.fp8_scaled_matmul(x, self.weight, self.input_scale, self.weight_scale, BF16, self.bias, out)
        elif self.kind == "fp8":
            if self._x8 is None or self._x8.shape != x.shape:
                self._x8 = torch.empty(x.shape, dtype=torch.float8_e4m3fn, device=x.device)
            x8, sc = ops.fp8_scaled_quantize(x, self._x8, self.input_scale)
            ops.fp8_scaled_matmul(x8, self.weight, sc, self.weight_scale, BF16, self.bias, out)
        elif self.kind == "w8a16":
            ops.w8a16_linear(x, self.qweight, self.meta, self.group_size, self.bias, out)
        else:
            ops.w4a16_linear(x, self.qweight, self.meta, self.group_size, self.bias, out)
        return out


class Qwen2Weights:
    def __init__(self, cfg: Qwen2Config):
        self.cfg = cfg
        self.embed = None
        self.lm_head: Optional[Linear] = None
        self.final_norm = None
        self.layers: List[dict] = []

    @staticmethod
    def _synthetic_linear(N, K, kind, gs, gen, device, bias=False, std=0.02):
        lin = Linear(N, K, kind, gs)
        if kind == "bf16":
            lin.weight = (torch.randn(N, K, generator=gen, device=device) * std).to(BF16)
        elif kind == "fp8":
            lin.weight = (torch.randn(N, K, generator=gen, device=device)).clamp(-3, 3).to(torch.float8_e4m3fn)
            lin.weight_scale = torch.full((1,), std, dtype=torch.float32, device=device)
            lin.input_scale = torch.full((1,), 0.05, dtype=torch.float32, device=device)
        elif kind == "w8a16":
            lin.qweight = torch.randint(-2 ** 31, 2 ** 31 - 1, (N // 16, K // 64, 32, 8), generator=gen, device=device,
                                        dtype=torch.int32)
            s = (torch.rand(K // gs, N, generator=gen, device=device) * 0.5 + 0.75) * (std * 3.0 / 127.5)
            z = torch.randint(120, 136, (K // gs, N), generator=gen, device=device)
            s_bits = s.to(BF16).view(torch.int16).to(torch.int32) & 0xFFFF
            lin.meta = (s_bits | (z.to(torch.int32) << 16)).contiguous()
        else:
            # uniform nibbles + scales such that w ~ N(0, std^2)-like spread; generated directly in packed form
            lin.qweight = torch.randint(-2 ** 31, 2 ** 31 - 1, (N // 16, K // 64, 32, 4), generator=gen, device=device,
                                        dtype=torch.int32)
            s = (torch.rand(K // gs, N, generator=gen, device=device) * 0.5 + 0.75) * (std * 3.0 / 7.5)
            z = torch.randint(6, 10, (K // gs, N), generator=gen, device=device)
            s_bits = s.to(BF16).view(torch.int16).to(torch.int32) & 0xFFFF
            z_bits = (z.float() + 128.0).to(BF16).view(torch.int16).to(torch.int32) & 0xFFFF
            lin.meta = (s_bits | (z_bits << 16)).contiguous()
        if bias:
            lin.bias = (torch.randn(N, generator=gen, device=device) * std).to(BF16)
        return lin

    @staticmethod
    def synthetic(cfg: Qwen2Config, device="cuda", seed=2026, tp_rank: int = 0, tp: int = 1):
        """random-init weights of the named architecture (no checkpoints offline), generated on device.  With tp > 1 the
        shapes are this rank's shards (column-parallel qkv / gate_up / lm_head, row-parallel o / down).  Tensors that the
        reference REPLICATES across a TP group (embedding table, every RMSNorm weight) come from a generator seeded by
        `seed` alone, so all ranks of a group hold identical copies; shards are seeded per rank."""
        from .parallel import partition_heads
        g_rep = torch.Generator(device=device).manual_seed(seed)
        g = torch.Generator(device=device).manual_seed(seed + 7919 * (tp_rank + 1)) if tp > 1 else g_rep
        w = Qwen2Weights(cfg)
        H, I = cfg.hidden_size, cfg.intermediate_size // tp
        hp = partition_heads(cfg.n_heads, cfg.n_kv_heads, tp_rank, tp)
        q_size, kv_size = hp.num_heads * cfg.head_dim, hp.num_kv_heads * cfg.head_dim
        w.embed = (torch.randn(cfg.vocab_size, H, generator=g_rep, device=device) * 0.02).to(BF16)
        w.final_norm = (1.0 + 0.05 * torch.randn(H, generator=g_rep, device=device)).to(BF16)
        vs = cfg.vocab_size // tp
        w.lm_head = Linear(vs, H, "bf16")                   # lm_head stays unquantised (linear.cpp:512-520)
        w.lm_head.weight = w.embed if (cfg.tie_word_embeddings and tp == 1) else \
            (torch.randn(vs, H, generator=g, device=device) * 0.02).to(BF16)
        for _ in range(cfg.num_layers):
            mk = lambda n, k, b=False: Qwen2Weights._synthetic_linear(n, k, cfg.quant, cfg.group_size, g, device, b)
            w.layers.append(dict(
                input_norm=(1.0 + 0.05 * torch.randn(H, generator=g_rep, device=device)).to(BF16),
                post_norm=(1.0 + 0.05 * torch.randn(H, generator=g_rep, device=device)).to(BF16),
                qkv=mk(q_size + 2 * kv_size, H, cfg.qkv_bias), o=mk(H, q_size),
                gate_up=mk(2 * I, H), down=mk(H, I)))
            if cfg.qk_norm:
                w.layers[-1]["q_norm"] = (1.0 + 0.05 * torch.randn(cfg.head_dim, generator=g_rep, device=device)).to(BF16)
                w.layers[-1]["k_norm"] = (1.0 + 0.05 * torch.randn(cfg.head_dim, generator=g_rep, device=device)).to(BF16)
            # synthetic packed nibbles are random anyway: declare the gate_up rows interleaved so the fused epilogue runs.
            # The rope-pair qkv order serves only the GEMV's RoPE epilogue, which cannot normalise a head: plain under qk_norm.
            w.layers[-1]["gate_up"].gate_up_interleaved = cfg.quant == "w4a16"
            w.layers[-1]["qkv"].qkv_rope_packed = cfg.quant == "w4a16" and not cfg.qk_norm
        return w

    def weight_bytes(self):
        n = self.lm_head.weight_bytes()
        for l in self.layers:
            n += sum(l[k].weight_bytes() for k in ("qkv", "o", "gate_up", "down"))
        return n


def llama3_scale_inv_freq(inv_freq: torch.Tensor, factor: float, low_freq_factor: float, high_freq_factor: float,
                          original_max_position_embeddings: int) -> torch.Tensor:
    """Llama-3.1 frequency scaling (the published "llama3" rope_type): wavelengths above original_max / low_freq_factor
    are slowed by `factor`, below original_max / high_freq_factor kept, the band between interpolated."""
    import math
    low_wl = original_max_position_embeddings / low_freq_factor
    high_wl = original_max_position_embeddings / high_freq_factor
    wavelen = 2.0 * math.pi / inv_freq
    smooth = (original_max_position_embeddings / wavelen - low_freq_factor) / (high_freq_factor - low_freq_factor)
    mid = (1.0 - smooth) * inv_freq / factor + smooth * inv_freq
    scaled = torch.where(wavelen > low_wl, inv_freq / factor, inv_freq)
    return torch.where((wavelen <= low_wl) & (wavelen >= high_wl), mid, scaled)


def make_cos_sin_cache(cfg: Qwen2Config, device):
    """[max_pos, head_dim] = [cos_half | sin_half] in bf16 - the pre-sliced layout the CUDA kernel reads
    (rotary_embedding.cpp:31-52, rotary_embedding_util.cpp:115-144,303-310; rope_theta passes through int64)."""
    rot = cfg.head_dim
    sl = torch.arange(0, rot, 2, dtype=torch.float32)
    inv_freq = 1.0 / torch.pow(torch.tensor(float(int(cfg.rope_theta)), dtype=torch.float32), sl / float(rot))
    rs = cfg.rope_scaling
    if rs is not None:
        if rs.get("rope_type", rs.get("type")) != "llama3":
            raise ValueError(f"unsupported rope_scaling {rs}")
        inv_freq = llama3_scale_inv_freq(inv_freq, float(rs["factor"]), float(rs["low_freq_factor"]),
                                         float(rs["high_freq_factor"]), int(rs["original_max_position_embeddings"]))
    t = torch.arange(cfg.max_position_embeddings, dtype=torch.float32)
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    return torch.cat([freqs.cos(), freqs.sin()], dim=-1).to(BF16).to(device)


class Qwen2DecodeRunner:
    """Batched single-token decode over a paged KV cache (continuous-batching decode step of the reference)."""

    def __init__(self, cfg: Qwen2Config, weights: Qwen2Weights, max_batch: int, max_ctx: int, device="cuda",
                 num_blocks: Optional[int] = None, fused_rope_cache: bool = True, pg=None, exchange: str = "peer",
                 fuse_gemv: bool = False):
        """pg: xllm_b200.parallel.ProcessGroup for tensor parallelism (weights must already be this rank's shards);
        exchange: "peer" = NVLink one-shot all-reduce fused with add+RMSNorm, "nccl" = c10d all-reduce (baseline);
        fuse_gemv: W4A16 decode with batch <= 8 splits add+RMSNorm between the o / down epilogues and the qkv / gate_up
        prologues (5 launches per layer instead of 7).  OFF by default: the 200-launch step's small add+RMSNorm kernels
        overlap the next GEMV's weight prefetch under PDL, while folded into the GEMVs they sit on every CTA's critical path.  RoPE + KV scatter (qkv epilogue) and SiLU*mul (gate_up epilogue) ride in the
        GEMVs either way.  Always off for qk_norm (Qwen3) configs: it needs the rope-pair packed qkv epilogue, which cannot
        normalise a head.
        fused_rope_cache: qk_norm configs run qk_norm_rope_and_cache (one launch) when True, fused_qk_norm_rope +
        reshape_paged_cache when False; other configs rope_and_cache vs rotary_embedding + reshape_paged_cache."""
        self.cfg, self.w, self.B, self.device = cfg, weights, max_batch, device
        self.pg = pg if (pg is not None and pg.world_size > 1) else None
        self.tp = self.pg.world_size if self.pg else 1
        self.tp_rank = self.pg.rank if self.pg else 0
        from .parallel import partition_heads
        hp = partition_heads(cfg.n_heads, cfg.n_kv_heads, self.tp_rank, self.tp)
        self.nh, self.nkv = hp.num_heads, hp.num_kv_heads
        self.q_size, self.kv_size = self.nh * cfg.head_dim, self.nkv * cfg.head_dim
        self.inter = cfg.intermediate_size // self.tp
        self.exchange = None
        self.exchange_mode = exchange
        bs = cfg.block_size
        self.max_pages = (max_ctx + bs - 1) // bs
        self.num_blocks = num_blocks or (max_batch * self.max_pages + 1)     # block 0 reserved (block_manager_impl.cpp:71-73)
        self.fused_rope_cache = fused_rope_cache
        H, I = cfg.hidden_size, cfg.intermediate_size
        B = max_batch
        dev = device
        self.k_caches = [torch.zeros(self.num_blocks, bs, self.nkv, cfg.head_dim, dtype=BF16, device=dev)
                         for _ in range(cfg.num_layers)]
        self.v_caches = [torch.zeros_like(k) for k in self.k_caches]
        self.cos_sin = make_cos_sin_cache(cfg, dev)
        # step inputs (device) + pinned host mirrors
        n_idx = B * self.max_pages
        self.token_ids = torch.zeros(B, dtype=torch.int32, device=dev)
        self.positions = torch.zeros(B, dtype=torch.int64, device=dev)
        self.slots = torch.zeros(B, dtype=torch.int32, device=dev)
        self.kv_indptr = torch.zeros(B + 1, dtype=torch.int32, device=dev)
        self.kv_indices = torch.zeros(n_idx, dtype=torch.int32, device=dev)
        self.kv_last = torch.ones(B, dtype=torch.int32, device=dev)
        self.h_token_ids = torch.zeros(B, dtype=torch.int32).pin_memory()
        self.h_positions = torch.zeros(B, dtype=torch.int64).pin_memory()
        self.h_slots = torch.zeros(B, dtype=torch.int32).pin_memory()
        self.h_kv_indptr = torch.zeros(B + 1, dtype=torch.int32).pin_memory()
        self.h_kv_indices = torch.zeros(n_idx, dtype=torch.int32).pin_memory()
        self.h_kv_last = torch.ones(B, dtype=torch.int32).pin_memory()
        self.h_next = torch.zeros(B, dtype=torch.int32).pin_memory()
        # activations
        self.hidden = torch.empty(B, H, dtype=BF16, device=dev)
        self.residual = torch.empty(B, H, dtype=BF16, device=dev)
        self.normed = torch.empty(B, H, dtype=BF16, device=dev)
        # `hidden` carries the residual stream from layer 0 on (it aliases the embedding output);
        # o_proj writes buf_a, down_proj writes buf_b
        self.buf_a = torch.empty(B, H, dtype=BF16, device=dev)
        self.buf_b = torch.empty(B, H, dtype=BF16, device=dev)
        self.qkv = torch.empty(B, self.q_size + 2 * self.kv_size, dtype=BF16, device=dev)
        self.qkv_raw = torch.empty_like(self.qkv)       # rope-pair packed projection output when RoPE is not fused
        self.res_pp = [torch.empty(B, H, dtype=BF16, device=dev) for _ in range(2)]   # residual stream ping-pong (fused GEMVs)
        self.norm_stats = [torch.zeros(H // 16, 8, dtype=torch.float32, device=dev) for _ in range(2)]   # split-RMSNorm partials
        w4 = cfg.quant == "w4a16" and all(L["qkv"].kind == "w4a16" for L in weights.layers)
        import os
        if os.environ.get("XB_FUSE_GEMV") is not None:          # A/B measurements
            fuse_gemv = os.environ["XB_FUSE_GEMV"] != "0"
        if cfg.qk_norm and any(L["qkv"].qkv_rope_packed for L in weights.layers):
            raise ValueError("qk_norm needs the plain qkv weight layout: the rope-pair packed one cannot normalise a head")
        self.fuse_gemv = bool(fuse_gemv and w4 and B <= 8 and ops.w4a16_decode_fused_fits(B, H) and not cfg.qk_norm)
        # post-attention add+RMSNorm folded into the gate_up GEMV's prologue only (XB_FUSE_MLP_NORM=1; experiment): the wide
        # gate_up launch hides the prologue (+0.5 us measured) while the separate add+norm kernel costs ~2.2 us
        self.fuse_mlp_norm = bool(os.environ.get("XB_FUSE_MLP_NORM", "0") != "0" and w4 and B <= 8 and
                                  ops.w4a16_decode_fused_fits(B, H) and not self.fuse_gemv)
        self.attn_out = torch.empty(B, self.q_size, dtype=BF16, device=dev)
        self.gate_up = torch.empty(B, 2 * self.inter, dtype=BF16, device=dev)
        self.act = torch.empty(B, self.inter, dtype=BF16, device=dev)
        self.logits = torch.empty(B, cfg.vocab_size, dtype=BF16, device=dev)
        self.logits_local = torch.empty(B, cfg.vocab_size // self.tp, dtype=BF16, device=dev) if self.pg else self.logits
        if self.pg and exchange == "peer":
            from .parallel import PeerExchange
            try:
                self.exchange = PeerExchange(self.pg, B, H, dev)
            except Exception as e:          # no P2P mapping available: the NCCL exchange is the baseline path
                import warnings
                warnings.warn(f"NVLink peer exchange unavailable ({e}); falling back to NCCL all-reduce")
                self.exchange, self.exchange_mode = None, "nccl (peer exchange unavailable)"
        self.next_tokens = torch.zeros(B, dtype=torch.int32, device=dev)
        # norm + static FP8 quantisation in one kernel where the consumer is an FP8 linear with a static input scale (the
        # reference's composition for such checkpoints).  Not under the one-shot NVLink exchange, whose fused add+norm emits bf16.
        self.fp8_norm_quant = (cfg.quant == "fp8" and os.environ.get("XB_FP8_NORM_QUANT", "1") != "0" and
                               all(L[k].input_scale is not None for L in weights.layers for k in ("qkv", "gate_up")))
        self.normed8 = torch.empty(B, H, dtype=torch.float8_e4m3fn, device=dev) if cfg.quant == "fp8" else None
        if cfg.quant == "fp8" and os.environ.get("XB_FP8_SPLITK", "1") != "0":
            # decode-sized FP8 linears: K split over otherwise idle SMs (shard-sized N leaves 10-64 weight tiles for 132 SMs)
            ops.enable_fp8_splitk(dev)
        self.embed_local = torch.empty(B, weights.embed.size(1), dtype=BF16, device=dev) if weights.embed.size(1) != H else None
        self.plan = ops.DecodePlan(B, self.nh, self.nkv, cfg.head_dim, bs, self.max_pages, dev, early_prefetch=True)
        self.graph = None
        self.h2d_bytes = sum(t.numel() * t.element_size() for t in
                             (self.h_token_ids, self.h_positions, self.h_slots, self.h_kv_indptr, self.h_kv_indices,
                              self.h_kv_last))
        self.d2h_bytes = self.h_next.numel() * 4

    # -- one decode step worth of launches (capturable) -----------------------------------
    def _row_parallel(self, lin, x, which, norm_w, out, fp8_scale=None):
        """row-parallel linear + exchange + the fused add+RMSNorm that follows it in the layer
        (linear.cpp:1405-1522 + qwen2_decoder_layer.cpp:103-109).  Returns the normalised activations.  fp8_scale: static
        input scale of the linear that consumes them - the norm then emits e4m3 directly, as the reference's apply_norm does
        for FP8 checkpoints (qwen2_decoder_layer.cpp:64-84 -> RMSNormImpl::forward_fp8, rms_norm.cpp:94-128)."""
        cfg = self.cfg

        def add_norm():
            if fp8_scale is not None:
                ops.fused_add_rms_norm_static_fp8_quant(self.normed8, out, self.residual, norm_w, fp8_scale, cfg.rms_norm_eps)
                return self.normed8
            ops.fused_add_rms_norm(out, self.residual, norm_w, cfg.rms_norm_eps)
            return out
        if self.pg is None:
            lin.forward(x, out)
            return add_norm()
        if self.exchange is not None and x.size(0) <= self.exchange.MAX_CTAS:
            part = self.exchange.partial_buffer(which, x.size(0))
            lin.forward(x, part)                                    # partial straight into the symmetric buffer
            self.exchange.allreduce_add_rms_norm(which, out, self.residual, norm_w, cfg.rms_norm_eps, x.size(0))
            return out
        lin.forward(x, out)
        self.pg.allreduce(out)                                      # NCCL baseline
        return add_norm()

    def _qkv_and_rope(self, L, li, h, norm_w=None, res_in=None, res_out=None, stats_in=None):
        """qkv_proj + RoPE + KV scatter of layer li (qwen2_attention.cpp:147-176, flashinfer_attention.cpp:128-131);
        with norm_w the add+RMSNorm in front of it rides in the same launch.  Leaves q | k | v (logical) in self.qkv."""
        cfg = self.cfg
        qs, kvs = self.q_size, self.kv_size
        lin = L["qkv"]
        packed = lin.kind == "w4a16" and lin.qkv_rope_packed
        if packed and h.size(0) <= 8 and (self.fuse_gemv or norm_w is None):
            ops.w4a16_decode_fused(h, lin.qweight, lin.meta, lin.group_size, lin.bias, self.qkv, norm_weight=norm_w,
                                   eps=cfg.rms_norm_eps, residual_in=res_in, residual_out=res_out, stage_x=self.fuse_gemv,
                                   norm_stats_in=stats_in, epilogue="rope_cache", positions=self.positions, cos_sin_cache=self.cos_sin,
                                   slot_ids=self.slots, key_cache=self.k_caches[li], value_cache=self.v_caches[li],
                                   num_heads=self.nh, num_kv_heads=self.nkv, head_dim=cfg.head_dim)
            return
        assert norm_w is None
        if cfg.qk_norm:
            lin.forward(h, self.qkv)
            if self.fused_rope_cache:
                ops.qk_norm_rope_and_cache(self.qkv, self.nh, self.nkv, cfg.head_dim, cfg.rms_norm_eps, L["q_norm"], L["k_norm"],
                                           self.cos_sin, self.positions, self.slots, self.k_caches[li], self.v_caches[li])
            else:
                ops.fused_qk_norm_rope(self.qkv, self.nh, self.nkv, self.nkv, cfg.head_dim, cfg.rms_norm_eps, L["q_norm"],
                                       L["k_norm"], self.cos_sin, False, self.positions)
                k, v = self.qkv[:, qs:qs + kvs], self.qkv[:, qs + kvs:]
                ops.reshape_paged_cache(self.slots, k.view(-1, self.nkv, cfg.head_dim), v.view(-1, self.nkv, cfg.head_dim),
                                        self.k_caches[li], self.v_caches[li])
            return
        if packed:
            lin.forward(h, self.qkv_raw)
            ops.rope_and_cache_packed(self.positions, self.qkv_raw, self.qkv, self.cos_sin, self.slots, self.k_caches[li],
                                      self.v_caches[li], self.nh, self.nkv, cfg.head_dim)
            return
        lin.forward(h, self.qkv)
        q, k, v = self.qkv[:, :qs], self.qkv[:, qs:qs + kvs], self.qkv[:, qs + kvs:]
        if self.fused_rope_cache:
            ops.rope_and_cache(self.positions, q, k, v, self.cos_sin, self.slots, self.k_caches[li], self.v_caches[li], True)
        else:
            ops.rotary_embedding(self.positions, q, k, self.cos_sin, True)
            ops.reshape_paged_cache(self.slots, k.view(-1, self.nkv, cfg.head_dim), v.view(-1, self.nkv, cfg.head_dim),
                                    self.k_caches[li], self.v_caches[li])

    def _attention(self, li):
        cfg = self.cfg
        ops.batch_decode(self.plan, self.qkv[:, :self.q_size].view(-1, self.nh, cfg.head_dim), self.k_caches[li],
                         self.v_caches[li], self.kv_indptr, self.kv_indices, self.kv_last, cfg.head_dim ** -0.5,
                         self.attn_out.view(-1, self.nh, cfg.head_dim))

    def _launch_step_fused(self):
        """TP = 1, W4A16, batch <= 8: five launches per layer, RMSNorm split between producer and consumer linears.
        The reference runs residual-add + RMSNorm as its own kernel after o_proj / down_proj
        (qwen2_decoder_layer.cpp:89-112).  Here the row-parallel projection's epilogue adds the residual, writes the
        updated residual stream and per-tile partial sums of its squares ("residual_stats"); the NEXT linear (qkv /
        gate_up) takes the residual stream as its x, sums the partials in a fixed order and normalises while it stages x in
        shared memory; RoPE + KV scatter ride in the qkv epilogue, SiLU*mul in the gate_up epilogue.  The residual stream
        ping-pongs between two buffers (the producer's CTAs read the old one while they write the new one)."""
        cfg, w = self.cfg, self.w
        eps = cfg.rms_norm_eps
        ops.embedding(self.hidden, self.token_ids, w.embed)
        # layer 0's input norm has no producer linear: the plain kernel (one launch per step)
        ops.rms_norm(self.normed, self.hidden, w.layers[0]["input_norm"], eps)
        res, pp, stats = self.hidden, 0, None
        B = self.hidden.size(0)
        for li, L in enumerate(w.layers):
            if li == 0:
                self._qkv_and_rope(L, li, self.normed)
            else:
                self._qkv_and_rope(L, li, res, L["input_norm"], stats_in=stats)
            self._attention(li)
            o, gu, dn = L["o"], L["gate_up"], L["down"]
            ops.w4a16_decode_fused(self.attn_out, o.qweight, o.meta, o.group_size, o.bias, self.buf_a, epilogue="residual_stats",
                                   residual_in=res, residual_out=self.res_pp[pp], norm_stats_out=self.norm_stats[0])
            res, pp = self.res_pp[pp], pp ^ 1
            epi = "act_mul" if gu.gate_up_interleaved else "none"
            ops.w4a16_decode_fused(res, gu.qweight, gu.meta, gu.group_size, gu.bias, self.act if epi == "act_mul" else self.gate_up,
                                   norm_weight=L["post_norm"], eps=eps, norm_stats_in=self.norm_stats[0], epilogue=epi,
                                   act_mode="silu")
            if epi == "none":
                ops.act_and_mul(self.act, self.gate_up, "silu")
            ops.w4a16_decode_fused(self.act, dn.qweight, dn.meta, dn.group_size, dn.bias, self.buf_b, epilogue="residual_stats",
                                   residual_in=res, residual_out=self.res_pp[pp], norm_stats_out=self.norm_stats[1],
                                   stage_x=ops.w4a16_decode_fused_fits(B, dn.K))
            res, pp, stats = self.res_pp[pp], pp ^ 1, self.norm_stats[1]
        self.residual = res
        ops.rms_norm(self.normed, res, w.final_norm, eps)
        w.lm_head.forward(self.normed, self.logits_local)
        ops.argmax(self.next_tokens, self.logits)

    def _embed(self):
        """token embedding into self.hidden; a table sharded along the hidden dimension (word_embedding_impl.cpp:48-56: each
        rank holds H / tp columns) is looked up locally and all-gathered."""
        w = self.w
        if self.pg is not None and w.embed.size(1) != self.cfg.hidden_size:
            from .parallel import gather
            ops.embedding(self.embed_local, self.token_ids, w.embed)
            self.hidden.copy_(gather(self.embed_local, self.pg, dim=-1))
        else:
            ops.embedding(self.hidden, self.token_ids, w.embed)

    def _launch_step_mlp_norm(self):
        """TP = 1, W4A16, batch <= 8: the shipped step, except that the post-attention add+RMSNorm
        (qwen2_decoder_layer.cpp:89-101) rides in the gate_up GEMV's prologue (every CTA recomputes the 7 KB row); the residual
        stream ping-pongs between two buffers because the prologue's CTAs read the old one while CTA 0 writes the new one."""
        cfg, w = self.cfg, self.w
        eps = cfg.rms_norm_eps
        ops.embedding(self.hidden, self.token_ids, w.embed)
        res, pp = self.hidden, 0
        ops.rms_norm(self.normed, self.hidden, w.layers[0]["input_norm"], eps)
        h = self.normed
        n_layers = len(w.layers)
        for li, L in enumerate(w.layers):
            self._qkv_and_rope(L, li, h)
            self._attention(li)
            L["o"].forward(self.attn_out, self.buf_a)
            gu, dn = L["gate_up"], L["down"]
            # x = o_proj output, residual_in = stream; residual_out = stream + x; act = silu(gate) * up of the normed row
            ops.w4a16_decode_fused(self.buf_a, gu.qweight, gu.meta, gu.group_size, gu.bias, self.act, norm_weight=L["post_norm"],
                                   eps=eps, residual_in=res, residual_out=self.res_pp[pp], epilogue="act_mul", act_mode="silu")
            res, pp = self.res_pp[pp], pp ^ 1
            dn.forward(self.act, self.buf_b)
            next_w = w.layers[li + 1]["input_norm"] if li + 1 < n_layers else w.final_norm
            ops.fused_add_rms_norm(self.buf_b, res, next_w, eps)       # buf_b := normed, res := res + down output (in place)
            h = self.buf_b
        self.residual = res
        w.lm_head.forward(h, self.logits_local)
        ops.argmax(self.next_tokens, self.logits)

    def launch_step(self, trace=None):
        """trace (eager only): list that receives (normed layer output, residual) clones after every decoder layer."""
        cfg, w = self.cfg, self.w
        if self.fuse_gemv and self.pg is None and trace is None:
            return self._launch_step_fused()
        if self.fuse_mlp_norm and self.pg is None and trace is None:
            return self._launch_step_mlp_norm()
        self._embed()
        # apply_norm, first layer (qwen2_decoder_layer.cpp:72-79): the residual stream aliases the embedding output
        self.residual = self.hidden
        # FP8 checkpoints with static activation scales: every norm in front of a quantised linear emits e4m3 with that
        # linear's input scale (get_fp8_input_scale: qwen2_attention.cpp:204-209, dense_mlp.cpp:137-142)
        nq = self.fp8_norm_quant

        def in_scale(lin):
            return lin.input_scale if (nq and lin.kind == "fp8") else None
        if in_scale(w.layers[0]["qkv"]) is not None:
            ops.rms_norm_static_fp8_quant(self.normed8, self.hidden, w.layers[0]["input_norm"], w.layers[0]["qkv"].input_scale,
                                          cfg.rms_norm_eps)
            h = self.normed8
        else:
            ops.rms_norm(self.normed, self.hidden, w.layers[0]["input_norm"], cfg.rms_norm_eps)
            h = self.normed
        n_layers = len(w.layers)
        for li, L in enumerate(w.layers):
            self._qkv_and_rope(L, li, h)
            self._attention(li)
            # o_proj (+ all-reduce) + post-attention add+norm
            h = self._row_parallel(L["o"], self.attn_out, 0, L["post_norm"], self.buf_a, in_scale(L["gate_up"]))
            gu = L["gate_up"]
            if gu.kind == "w4a16" and gu.gate_up_interleaved:
                # gate_up GEMV with SiLU*mul in its epilogue (one launch instead of two)
                ops.w4a16_gate_up_act(h, gu.qweight, gu.meta, gu.group_size, "silu", gu.bias, self.act, self.gate_up)
            else:
                gu.forward(h, self.gate_up)
                ops.act_and_mul(self.act, self.gate_up, "silu")
            # down_proj (+ all-reduce) + the NEXT layer's input add+norm (or the final norm)
            next_w = w.layers[li + 1]["input_norm"] if li + 1 < n_layers else w.final_norm
            h = self._row_parallel(L["down"], self.act, 1, next_w, self.buf_b,
                                   in_scale(w.layers[li + 1]["qkv"]) if li + 1 < n_layers else None)
            if trace is not None:
                trace.append((h.clone(), self.residual.clone()))
        w.lm_head.forward(h, self.logits_local)
        if self.pg is not None:
            # column-parallel lm_head with gather_output (linear.cpp:712-714 -> parallel_state.cpp:89-102)
            from .parallel import gather
            self.logits.copy_(gather(self.logits_local, self.pg, dim=-1))
        ops.argmax(self.next_tokens, self.logits)

    def capture(self):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self.launch_step()          # warm-up (sets func attributes, loads modules)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                self.launch_step()
        torch.cuda.current_stream().wait_stream(s)
        self.graph = g
        return g

    def run_device_only(self):
        """replay with whatever step inputs are resident on the device."""
        if self.graph is None:
            self.launch_step()
        else:
            self.graph.replay()

    def set_inputs_host(self, token_ids, positions, slots, kv_indptr, kv_indices, kv_last):
        """Step inputs of `n <= max_batch` live requests.  The captured graph always processes max_batch rows, so rows
        n..B-1 are padded EXACTLY as the reference pads a decode batch (padding_decode_batch_size,
        batch_input_builder.cpp:833-875): token 0, position 0, slot 0 and one page = block 0 (the reserved padding block,
        block_manager_impl.cpp:71-73) with last_page_len 1.  Stale rows from a previous, larger batch would otherwise
        scatter K/V into slots the block manager may have handed to another request."""
        n, B = len(token_ids), self.B
        if n > B:
            raise ValueError(f"{n} requests exceed max_batch {B}")
        kv_indptr, kv_indices = list(kv_indptr), list(kv_indices)
        if len(kv_indptr) != n + 1 or kv_indptr[-1] != len(kv_indices):
            raise ValueError("paged_kv_indptr / paged_kv_indices are inconsistent")
        pad = B - n
        if len(kv_indices) + pad > self.h_kv_indices.numel():
            raise ValueError("paged_kv_indices exceed the runner's page budget")
        self.h_token_ids[:n] = torch.as_tensor(token_ids, dtype=torch.int32)
        self.h_positions[:n] = torch.as_tensor(positions, dtype=torch.int64)
        self.h_slots[:n] = torch.as_tensor(slots, dtype=torch.int32)
        self.h_kv_indptr[:n + 1] = torch.as_tensor(kv_indptr, dtype=torch.int32)
        self.h_kv_indices[:len(kv_indices)] = torch.as_tensor(kv_indices, dtype=torch.int32)
        self.h_kv_last[:n] = torch.as_tensor(kv_last, dtype=torch.int32)
        if pad:
            self.h_token_ids[n:] = 0
            self.h_positions[n:] = 0
            self.h_slots[n:] = 0
            base = kv_indptr[-1]
            self.h_kv_indices[base:base + pad] = 0
            self.h_kv_indptr[n + 1:] = torch.arange(base + 1, base + pad + 1, dtype=torch.int32)
            self.h_kv_last[n:] = 1

    def step(self):
        """end-to-end step: H2D of the pinned step inputs, graph replay, D2H of the sampled tokens."""
        self.token_ids.copy_(self.h_token_ids, non_blocking=True)
        self.positions.copy_(self.h_positions, non_blocking=True)
        self.slots.copy_(self.h_slots, non_blocking=True)
        self.kv_indptr.copy_(self.h_kv_indptr, non_blocking=True)
        self.kv_indices.copy_(self.h_kv_indices, non_blocking=True)
        self.kv_last.copy_(self.h_kv_last, non_blocking=True)
        self.run_device_only()
        self.h_next.copy_(self.next_tokens, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self.h_next
