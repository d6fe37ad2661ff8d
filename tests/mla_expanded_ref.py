"""CPU reference of expanded MLA prefill (test infrastructure), beside tests/mla_ref.py: the latent gather through the page
table, kv_b_proj as the oracle's `linear`, and causal attention on the oracle's ladder (fp32 scores, base-2 softmax with
sm_scale*log2(e), P rounded to bf16, denominator = sum of the rounded P, fp32 PV) with per-head K = [k_nope | k_pe shared
by all heads] and per-head V."""
import math

import torch

from oracle.ops import BF16, F32, LOG2E, _r, gather_paged_kv, linear, rms_norm, rotary_embedding
from tests.mla_ref import ROPE_DIM, mla_cache_latent


def gather_latent(ckv_cache, kpe_cache, kv_indptr, kv_indices, kv_last_page_len):
    """-> ckv [total_kv, 512], kpe [total_kv, 64] in request order (on the caches' device), kv_cu [batch + 1] (CPU)"""
    ckv, kpe, cu = [], [], [0]
    for b in range(len(kv_indptr) - 1):
        ckv.append(gather_paged_kv(ckv_cache[:, :, None], kv_indptr, kv_indices, kv_last_page_len, b)[:, 0])
        kpe.append(gather_paged_kv(kpe_cache[:, :, None], kv_indptr, kv_indices, kv_last_page_len, b)[:, 0])
        cu.append(cu[-1] + ckv[-1].shape[0])
    return torch.cat(ckv), torch.cat(kpe), torch.tensor(cu, dtype=torch.int32)


def up_project(ckv, kv_b_proj, num_heads):
    """kv_up [total_kv, H, dn + dv] = ckv . kv_b_proj^T (bf16 out, fp32 accumulation)"""
    return linear(ckv, kv_b_proj).view(ckv.shape[0], num_heads, -1)


def attend_expanded(q, k_nope, k_pe, v, sm_scale, round_p=True):
    """causal, end-aligned.  q [Lq, H, dn + dr], k_nope [Lk, H, dn], k_pe [Lk, dr], v [Lk, H, dv] -> [Lq, H, dv] fp32"""
    Lq, H, _ = q.shape
    Lk, dn = k_nope.shape[0], k_nope.shape[-1]
    if Lk == 0:
        return torch.zeros(Lq, H, v.shape[-1], dtype=F32, device=q.device)
    s = (torch.einsum("qhd,khd->qhk", q[..., :dn].to(F32), k_nope.to(F32)) +
         torch.einsum("qhd,kd->qhk", q[..., dn:].to(F32), k_pe.to(F32))) * (sm_scale * LOG2E)
    allowed = torch.arange(Lk, device=q.device)[None, :] <= (Lk - Lq + torch.arange(Lq, device=q.device))[:, None]
    s = s.masked_fill(~allowed[:, None, :], -math.inf)
    m = s.max(-1, keepdim=True).values
    p = torch.exp2(s - torch.where(torch.isinf(m), torch.zeros_like(m), m))
    if round_p:
        p = _r(p)
    l = p.sum(-1, keepdim=True)
    return torch.einsum("qhk,khd->qhd", p, v.to(F32)) / torch.where(l > 0, l, torch.ones_like(l))


def expanded_attention(q, kv_up, kpe, qo_indptr, kv_cu, sm_scale, qk_nope_head_dim=128, abs_value=False):
    """ragged: q [T, H, dn + 64], kv_up [total_kv, H, dn + dv], kpe [total_kv, 64] -> [T, H, dv] bf16 (abs_value: fp32
    attention to |v|, the scale of the attention error bound)"""
    dn = qk_nope_head_dim
    out = torch.zeros(q.shape[0], q.shape[1], kv_up.shape[-1] - dn, dtype=F32 if abs_value else BF16, device=q.device)
    for b in range(len(qo_indptr) - 1):
        q0, q1, k0, k1 = int(qo_indptr[b]), int(qo_indptr[b + 1]), int(kv_cu[b]), int(kv_cu[b + 1])
        if q1 == q0:
            continue
        v = kv_up[k0:k1, :, dn:]
        o = attend_expanded(q[q0:q1], kv_up[k0:k1, :, :dn], kpe[k0:k1], v.to(F32).abs() if abs_value else v, sm_scale)
        out[q0:q1] = o.to(out.dtype)
    return out


def mla_prefill_expanded(q, ckv_cache, kpe_cache, qo_indptr, kv_indptr, kv_indices, kv_last_page_len, kv_b_proj, sm_scale,
                         qk_nope_head_dim=128):
    """-> (o [T, H, dv] bf16, kv_up, kpe, kv_cu)"""
    ckv, kpe, cu = gather_latent(ckv_cache, kpe_cache, kv_indptr, kv_indices, kv_last_page_len)
    kv_up = up_project(ckv, kv_b_proj, q.shape[1])
    return expanded_attention(q, kv_up, kpe, qo_indptr, cu, sm_scale, qk_nope_head_dim), kv_up, kpe, cu


def mla_attention_layer_expanded(w, x, positions, cos_sin_cache, slot_ids, ckv_cache, kpe_cache, qo_indptr, kv_indptr,
                                 kv_indices, kv_last_page_len, num_heads, qk_nope_head_dim, v_head_dim, eps, sm_scale):
    """DeepSeek-V3 attention in the expanded form (transformers' DeepseekV3Attention): same arguments and result as
    tests.mla_ref.mla_attention_layer; q = [q_nope | rope(q_pe)] is used as is, the latent is up-projected through
    kv_b_proj, and the attention output goes straight into o_proj."""
    T, H, dn = x.shape[0], num_heads, qk_nope_head_dim
    q = linear(rms_norm(linear(x, w["q_a_proj"]), w["q_a_layernorm"], eps), w["q_b_proj"]).view(T, H, dn + ROPE_DIM)
    q_pe = rotary_embedding(positions, q[..., dn:].contiguous(), None, cos_sin_cache, is_neox=False)[0]
    q = torch.cat([q[..., :dn], q_pe], -1)
    latent = linear(x, w["kv_a_proj_with_mqa"])
    mla_cache_latent(latent, w["kv_a_layernorm"], eps, positions, cos_sin_cache, slot_ids, ckv_cache, kpe_cache, True)
    o = mla_prefill_expanded(q, ckv_cache, kpe_cache, qo_indptr, kv_indptr, kv_indices, kv_last_page_len, w["kv_b_proj"],
                             sm_scale, dn)[0]
    return linear(o.reshape(T, H * v_head_dim), w["o_proj"])
