"""CPU reference of the MLA ops (test infrastructure): the latent cache writer as the composition of the oracle's
rms_norm / rotary_embedding / scatter, and absorbed MLA attention on the oracle's attention ladder (fp32 scores,
base-2 softmax with sm_scale*log2(e), P rounded to bf16, denominator = sum of the rounded P, fp32 PV), with the value
width taken from v (512) rather than from q (576)."""
import math

import torch

from oracle.ops import BF16, F32, LOG2E, _r, gather_paged_kv, rms_norm, rotary_embedding

KV_LORA_RANK = 512
ROPE_DIM = 64


def mla_cache_latent(latent, gamma, eps, positions, cos_sin_cache, slot_ids, ckv_cache, kpe_cache, interleaved=True):
    """In place on ckv_cache [pages, page_size, 512] / kpe_cache [pages, page_size, 64]; slot < 0 skipped."""
    ckv = rms_norm(latent[:, :KV_LORA_RANK], gamma, eps)
    kpe = rotary_embedding(positions, latent[:, None, KV_LORA_RANK:].clone(), None, cos_sin_cache,
                           is_neox=not interleaved)[0][:, 0]
    bs = ckv_cache.shape[1]
    for t, slot in enumerate(slot_ids.tolist()):
        if slot >= 0:
            ckv_cache[slot // bs, slot % bs] = ckv[t]
            kpe_cache[slot // bs, slot % bs] = kpe[t]


def attend_mla(q, k, v, sm_scale, causal, round_p=True):
    """q [Lq, H, Dk], k [Lk, Dk], v [Lk, Dv] (one kv head) -> [Lq, H, Dv] in q's dtype."""
    Lq, H, _ = q.shape
    Lk, Dv = k.shape[0], v.shape[-1]
    if Lk == 0:
        return torch.zeros(Lq, H, Dv, dtype=q.dtype, device=q.device)
    s = torch.einsum("qhd,kd->qhk", q.to(F32), k.to(F32)) * (sm_scale * LOG2E)
    if causal:
        allowed = torch.arange(Lk, device=q.device)[None, :] <= (Lk - Lq + torch.arange(Lq, device=q.device))[:, None]
        s = s.masked_fill(~allowed[:, None, :], -math.inf)
    m = s.max(-1, keepdim=True).values
    m_safe = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    p = torch.exp2(s - m_safe)
    if round_p:
        p = _r(p)
    l = p.sum(-1, keepdim=True)
    o = torch.einsum("qhk,kd->qhd", p, v.to(F32)) / torch.where(l > 0, l, torch.ones_like(l))
    return o.to(q.dtype)


def mla_paged_attention(q_nope, q_pe, ckv_cache, kpe_cache, qo_indptr, kv_indptr, kv_indices, kv_last_page_len, sm_scale,
                        causal, round_p=True, abs_value=False, out_dtype=None):
    """q_nope [T, H, 512], q_pe [T, H, 64]; caches [pages, page_size, 512 | 64] -> [T, H, 512] bf16 (runs on the tensors'
    device).  abs_value=True attends to |c_kv| (sum_j p_j |v_j|, the scale of the attention error bound), in fp32."""
    q = torch.cat([q_nope, q_pe], -1)
    dt = out_dtype or (F32 if abs_value else q.dtype)
    out = torch.zeros(q.shape[0], q.shape[1], KV_LORA_RANK, dtype=dt, device=q.device)
    for b in range(len(kv_indptr) - 1):
        q0, q1 = int(qo_indptr[b]), int(qo_indptr[b + 1])
        if q1 == q0:
            continue
        ckv = gather_paged_kv(ckv_cache[:, :, None], kv_indptr, kv_indices, kv_last_page_len, b)[:, 0]
        kpe = gather_paged_kv(kpe_cache[:, :, None], kv_indptr, kv_indices, kv_last_page_len, b)[:, 0]
        v = ckv.to(F32).abs() if abs_value else ckv
        out[q0:q1] = attend_mla(q[q0:q1].to(dt), torch.cat([ckv, kpe], -1), v, sm_scale, causal, round_p=round_p).to(dt)
    return out



def mla_attention_layer(w, x, positions, cos_sin_cache, slot_ids, ckv_cache, kpe_cache, qo_indptr, kv_indptr, kv_indices,
                        kv_last_page_len, num_heads, qk_nope_head_dim, v_head_dim, eps, sm_scale):
    """DeepSeek-V3 attention in the absorbed form the reference composes (layers/mlu/deepseek_v2_attention.cpp:200-240,
    444-496): q_a_proj / q_a_layernorm / q_b_proj -> split -> q_nope W_kc, interleaved RoPE on q_pe; kv_a_proj_with_mqa ->
    cache writer -> attention over the caches -> W_vc -> o_proj.  w: bf16 weights under the checkpoint's names.
    x [T, hidden] bf16 -> [T, hidden] bf16; writes the step's latent rows into the caches."""
    from oracle.ops import linear
    T, H, dn, dv = x.shape[0], num_heads, qk_nope_head_dim, v_head_dim
    q = linear(rms_norm(linear(x, w["q_a_proj"]), w["q_a_layernorm"], eps), w["q_b_proj"]).view(T, H, dn + ROPE_DIM)
    kv_b = w["kv_b_proj"].view(H, dn + dv, KV_LORA_RANK)
    w_kc, w_vc = kv_b[:, :dn], kv_b[:, dn:]                                     # [H, dn, 512], [H, dv, 512]
    q_nope = torch.einsum("thd,hdc->thc", q[..., :dn].to(F32), w_kc.to(F32)).to(BF16)
    q_pe = rotary_embedding(positions, q[..., dn:].contiguous(), None, cos_sin_cache, is_neox=False)[0]
    latent = linear(x, w["kv_a_proj_with_mqa"])
    mla_cache_latent(latent, w["kv_a_layernorm"], eps, positions, cos_sin_cache, slot_ids, ckv_cache, kpe_cache, True)
    o = mla_paged_attention(q_nope, q_pe, ckv_cache, kpe_cache, qo_indptr, kv_indptr, kv_indices, kv_last_page_len,
                            sm_scale, causal=True)
    ov = torch.einsum("thc,hdc->thd", o.to(F32), w_vc.to(F32)).to(BF16)
    return linear(ov.reshape(T, H * dv), w["o_proj"])
