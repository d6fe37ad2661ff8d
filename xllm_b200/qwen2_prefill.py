"""Prefill / chunked-prefill step of the Qwen2 (Llama-family) stack over a ragged batch: the composition the reference
runs in LlmModelImplBase::forward (xllm/models/llm/llm_model_base.h:60-131) over Qwen2DecoderLayerImpl::forward
(layers/qwen2_decoder_layer.cpp:64-112), Qwen2AttentionImpl::forward (layers/common/qwen2_attention.cpp:132-193),
FlashInferAttentionImpl::forward (layers/cuda/flashinfer_attention.cpp:112-157: scatter K/V first, then ragged prefill
or paged chunked prefill) and DenseMLPImpl::forward (layers/common/dense_mlp.cpp:97-118).

Eager library launches through the C ABI (token counts change every step, so no graph); it shares weights, KV caches
and the cos/sin table with a Qwen2DecodeRunner, which takes over after the prompt.  Logits are produced for the LAST
token of every sequence only (the rows the sampler reads).

Tensor parallel (the reference reduces [T, H] after every row-parallel linear at any T: layers/common/linear.cpp:1518-1520):
heads / intermediate columns are this rank's shards, o_proj and down_proj outputs are all-reduced over the TP group
(NCCL: prefill-sized messages) before the add+RMSNorm, the column-parallel lm_head is gathered; an embedding table sharded
along the hidden dimension (word_embedding_impl.cpp:48-56) is gathered after the lookup.

Composition exercised on CPU with the oracle ops swapped in (tests/test_prefill_composition_cpu.py), end to end on the GPU
(tests/test_gpu_model_prefill.py) and under TP by tp_check.tp_prefill_parity (tests/test_gpu_tp.py).
"""
from typing import Optional, Tuple

import torch

from . import qwen2 as _q

BF16 = torch.bfloat16


class Qwen2PrefillRunner:
    def __init__(self, cfg, weights, k_caches, v_caches, cos_sin, device="cuda", pg=None):
        self.cfg, self.w, self.device = cfg, weights, device
        self.k_caches, self.v_caches, self.cos_sin = k_caches, v_caches, cos_sin
        self.pg = pg if (pg is not None and pg.world_size > 1) else None
        tp = self.pg.world_size if self.pg else 1
        from .parallel import partition_heads
        hp = partition_heads(cfg.n_heads, cfg.n_kv_heads, self.pg.rank if self.pg else 0, tp)
        self.nh, self.nkv = hp.num_heads, hp.num_kv_heads
        self.q_size, self.kv_size = self.nh * cfg.head_dim, self.nkv * cfg.head_dim
        self.inter = cfg.intermediate_size // tp
        self.tp = tp

    @classmethod
    def from_decode_runner(cls, r):
        """same weights (this rank's shards) / caches / rope table / TP group as the decode runner."""
        return cls(r.cfg, r.w, r.k_caches, r.v_caches, r.cos_sin, r.device, pg=r.pg)

    def forward(self, token_ids, positions, slots, q_cu_seq_lens, kv_cu_seq_lens=None, paged_kv_indptr=None,
                paged_kv_indices=None, paged_kv_last_page_len=None, chunked: bool = False,
                max_qo_len: Optional[int] = None, trace=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """token_ids int32 [T], positions int64 [T], slots int32 [T] (new_cache_slots), q_cu_seq_lens int32 [B+1].
        chunked=False: first chunk of every request (no KV history): ragged attention over the fresh k/v, needs
        kv_cu_seq_lens (= q_cu_seq_lens).  chunked=True: attention over the paged cache (history + this chunk), needs
        the paged triplet describing the cache AFTER this chunk was appended.  Returns (logits [B, vocab], tokens [B])."""
        ops = _q.ops
        cfg, w = self.cfg, self.w
        dev = token_ids.device
        T = token_ids.numel()
        B = q_cu_seq_lens.numel() - 1
        H, D = cfg.hidden_size, cfg.head_dim
        qs, kvs = self.q_size, self.kv_size
        scale = D ** -0.5
        if max_qo_len is None:
            max_qo_len = int((q_cu_seq_lens[1:] - q_cu_seq_lens[:-1]).max().item())
        if not chunked and kv_cu_seq_lens is None:
            kv_cu_seq_lens = q_cu_seq_lens
        hidden = torch.empty(T, H, dtype=BF16, device=dev)
        normed = torch.empty(T, H, dtype=BF16, device=dev)
        buf_a = torch.empty(T, H, dtype=BF16, device=dev)
        buf_b = torch.empty(T, H, dtype=BF16, device=dev)
        qkv = torch.empty(T, qs + 2 * kvs, dtype=BF16, device=dev)
        qkv_raw = torch.empty_like(qkv) if any(L["qkv"].qkv_rope_packed for L in w.layers) else None
        attn_out = torch.empty(T, qs, dtype=BF16, device=dev)
        inter = self.inter
        gate_up = torch.empty(T, 2 * inter, dtype=BF16, device=dev)
        act = torch.empty(T, inter, dtype=BF16, device=dev)

        if self.pg is not None and w.embed.size(1) != H:
            # embedding sharded along the hidden dimension: local lookup + all-gather (word_embedding_impl.cpp:48-56)
            from .parallel import gather
            local = torch.empty(T, w.embed.size(1), dtype=BF16, device=dev)
            ops.embedding(local, token_ids, w.embed)
            hidden.copy_(gather(local, self.pg, dim=-1))
        else:
            ops.embedding(hidden, token_ids, w.embed)
        residual = hidden                                   # apply_norm, first layer (qwen2_decoder_layer.cpp:72-79)
        ops.rms_norm(normed, hidden, w.layers[0]["input_norm"], cfg.rms_norm_eps)
        h = normed
        n_layers = len(w.layers)
        for li, L in enumerate(w.layers):
            q, k, v = qkv[:, :qs], qkv[:, qs:qs + kvs], qkv[:, qs + kvs:]
            # RoPE on q/k and the KV scatter of this chunk (flashinfer_attention.cpp:128-131 scatters before attending)
            if cfg.qk_norm:
                # Qwen3: per-head q / k RMSNorm + RoPE in place, then the scatter; the ragged path reads the normalised k from qkv
                L["qkv"].forward(h, qkv)
                ops.qk_norm_rope_and_cache(qkv, self.nh, self.nkv, D, cfg.rms_norm_eps, L["q_norm"], L["k_norm"], self.cos_sin,
                                           positions, slots, self.k_caches[li], self.v_caches[li])
            elif L["qkv"].qkv_rope_packed:
                # decode-layout weights (rows in rope-pair order): the GEMM output is un-permuted by the rope kernel
                L["qkv"].forward(h, qkv_raw)
                ops.rope_and_cache_packed(positions, qkv_raw, qkv, self.cos_sin, slots, self.k_caches[li], self.v_caches[li],
                                          self.nh, self.nkv, D)
            else:
                L["qkv"].forward(h, qkv)
                ops.rope_and_cache(positions, q, k, v, self.cos_sin, slots, self.k_caches[li], self.v_caches[li], True)
            q3, o3 = q.view(T, self.nh, D), attn_out.view(T, self.nh, D)
            if chunked:
                ops.batch_chunked_prefill(q3, self.k_caches[li], self.v_caches[li], paged_kv_indptr, paged_kv_indices,
                                          paged_kv_last_page_len, scale, o3, None, q_cu_seq_lens, True, max_qo_len)
            else:
                ops.batch_prefill(q3, k.view(T, self.nkv, D), v.view(T, self.nkv, D), q_cu_seq_lens, kv_cu_seq_lens, scale,
                                  o3, None, max_qo_len, True)
            L["o"].forward(attn_out, buf_a)
            if self.pg is not None:
                self.pg.allreduce(buf_a)                      # row-parallel o_proj (linear.cpp:1518-1520)
            ops.fused_add_rms_norm(buf_a, residual, L["post_norm"], cfg.rms_norm_eps)
            gu = L["gate_up"]
            if gu.kind == "w4a16" and gu.gate_up_interleaved:
                ops.w4a16_gate_up_act(buf_a, gu.qweight, gu.meta, gu.group_size, "silu", gu.bias, act, gate_up)
            else:
                gu.forward(buf_a, gate_up)
                ops.act_and_mul(act, gate_up, "silu")
            L["down"].forward(act, buf_b)
            if self.pg is not None:
                self.pg.allreduce(buf_b)                      # row-parallel down_proj
            next_w = w.layers[li + 1]["input_norm"] if li + 1 < n_layers else w.final_norm
            ops.fused_add_rms_norm(buf_b, residual, next_w, cfg.rms_norm_eps)
            h = buf_b
            if trace is not None:
                trace.append((h.clone(), residual.clone()))
        # logits only where the sampler looks: the last token of every sequence (llm_model_base.h: selected token idxes)
        last = (q_cu_seq_lens[1:].to(torch.int64) - 1)
        h_last = h.index_select(0, last).contiguous()
        logits = torch.empty(B, cfg.vocab_size, dtype=BF16, device=dev)
        if self.pg is not None:
            # column-parallel lm_head with gather_output (linear.cpp:712-714 -> parallel_state.cpp:89-102)
            from .parallel import gather
            local = torch.empty(B, cfg.vocab_size // self.tp, dtype=BF16, device=dev)
            w.lm_head.forward(h_last, local)
            logits.copy_(gather(local, self.pg, dim=-1))
        else:
            w.lm_head.forward(h_last, logits)
        tokens = torch.zeros(B, dtype=torch.int32, device=dev)
        ops.argmax(tokens, logits)
        return logits, tokens
