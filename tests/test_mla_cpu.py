"""MLA without a GPU: the plan's host arithmetic, argument errors of the C ABI (raised before any launch), the shim's
dtype checks, and the absorbed form of the attention against the un-absorbed one in fp32."""
import ctypes

import pytest
import torch

from tests import mla_ref as R
from xllm_b200 import _lib

c_i64 = ctypes.c_int64


def plan(batch, H, max_qo, page, max_pages, sms=132, dc=512, dr=64):
    arr = (ctypes.c_int64 * 8)()
    rc = _lib.lib().xb_mla_plan(arr, batch, H, dc, dr, max_qo, page, max_pages, sms)
    return rc, arr


@pytest.mark.parametrize("B,H,qo,ctx", [(1, 16, 1, 4096), (1, 16, 1, 32768), (16, 16, 1, 4096), (64, 16, 1, 4096),
                                        (128, 16, 1, 4096), (1, 128, 1, 4096), (64, 128, 1, 4096), (64, 16, 2, 4096),
                                        (1, 16, 4096, 12288), (1, 128, 4096, 4096)])
def test_plan_covers_sms_and_sizes_workspace(B, H, qo, ctx):
    page = 64
    rc, p = plan(B, H, qo, page, ctx // page)
    assert rc == 0
    splits, ws, rg, m_tiles = p[0], p[1], p[7] & 0xFF, p[6]
    rows = qo * H
    assert rg == (1 if rows <= 16 else 4) and m_tiles == -(-rows // (16 * rg))
    slots = 132 * (2 if rg == 1 else 1)
    ctas = B * m_tiles
    assert 1 <= splits <= 128 and splits <= max(1, -(-ctx // 256))
    if ctas < slots and ctx >= 256 * 2:
        assert ctas * splits <= slots and ctas * (splits + 1) > slots or splits == min(128, -(-ctx // 256))
    else:
        assert splits == 1
    assert ws == (splits * B * qo * H * 513 * 4 if splits > 1 else 0)
    assert _lib.lib().xb_mla_plan_set_splits(p, 5) == 0 and p[0] == 5 and p[1] == 5 * B * qo * H * 513 * 4


def _err():
    return _lib.lib().xb_last_error().decode()


def test_plan_rejects_bad_arguments():
    assert plan(1, 16, 1, 16, 8, dc=256)[0] != 0 and "kv_lora_rank" in _err()
    assert plan(1, 16, 1, 16, 8, dr=128)[0] != 0 and "qk_rope_head_dim" in _err()
    assert plan(1, 0, 1, 16, 8)[0] != 0 and "num_heads" in _err()
    assert plan(1, 129, 1, 16, 8)[0] != 0 and "num_heads" in _err()
    assert plan(0, 16, 1, 16, 8)[0] != 0 and "batch" in _err()
    assert plan(1, 16, 1, 0, 8)[0] != 0 and "page" in _err()
    assert _lib.lib().xb_mla_plan(None, 1, 16, 512, 64, 1, 16, 8, 132) != 0 and "null" in _err()
    rc, p = plan(1, 16, 1, 16, 8)
    assert _lib.lib().xb_mla_plan_set_splits(p, 0) != 0 and "splits" in _err()
    assert _lib.lib().xb_mla_plan_set_splits(p, 129) != 0 and "splits" in _err()


def _attn(p, ptr=16, ws=None, ws_bytes=0):
    """a call whose pointers are never dereferenced: every case is rejected before any launch"""
    v = ctypes.c_void_p(ptr) if ptr else None
    i32 = ctypes.cast(v, ctypes.POINTER(ctypes.c_int32)) if ptr else None
    return _lib.lib().xb_mla_paged_attention_bf16(
        p, v, c_i64(576 * 16), c_i64(576), v, c_i64(576 * 16), c_i64(576), v, c_i64(16 * 512), c_i64(512), v,
        c_i64(16 * 64), c_i64(64), i32, i32, i32, i32, 0, v, c_i64(512 * 16), c_i64(512), ctypes.c_float(0.07),
        ws, c_i64(ws_bytes), None)


def test_attention_rejects_bad_arguments():
    rc, p = plan(1, 16, 1, 16, 4096, sms=132)
    assert rc == 0 and p[0] > 1
    assert _attn(None) != 0 and "plan" in _err()
    assert _attn(p, ptr=0) != 0 and "null" in _err()
    assert _attn(p) != 0 and "workspace" in _err()                               # split plan without a workspace
    assert _attn(p, ws=ctypes.c_void_p(4096), ws_bytes=p[1] - 1) != 0 and "workspace" in _err()
    assert _attn(p, ptr=18) != 0 and "aligned" in _err()
    bad = (ctypes.c_int64 * 8)(*p)
    bad[7] = 1
    assert _attn(bad) != 0 and "MLA plan" in _err()


def test_writer_rejects_bad_arguments():
    L = _lib.lib()
    v = ctypes.c_void_p(16)
    i64 = ctypes.cast(v, ctypes.POINTER(ctypes.c_int64))
    i32 = ctypes.cast(v, ctypes.POINTER(ctypes.c_int32))

    def call(dc=512, dr=64, latent=v, T=4, page=16):
        return L.xb_mla_cache_latent_bf16(latent, c_i64(576), v, ctypes.c_float(1e-6), i64, v, 1, i32, v, c_i64(16 * 512),
                                          c_i64(512), v, c_i64(16 * 64), c_i64(64), dc, dr, page, T, None)
    assert call(dc=576) != 0 and "kv_lora_rank" in _err()
    assert call(dr=32) != 0 and "qk_rope_head_dim" in _err()
    assert call(latent=None) != 0 and "null" in _err()
    assert call(page=0) != 0 and "page_size" in _err()
    assert call(latent=ctypes.c_void_p(18)) != 0 and "aligned" in _err()
    assert call(T=0, latent=None) == 0                                          # nothing to do


def test_shim_rejects_wrong_dtype():
    from xllm_b200 import build_shim
    shim = build_shim.load_py()
    f32 = torch.zeros(4, 576)
    with pytest.raises(RuntimeError, match="bfloat16"):
        shim.fused_mla_kv(f32, f32, torch.zeros(4, dtype=torch.int64), f32, f32, f32, torch.zeros(4, dtype=torch.int32),
                          "none", 1e-6, True)
    with pytest.raises(RuntimeError, match="quant_mode"):
        shim.fused_mla_kv(f32, f32, torch.zeros(4, dtype=torch.int64), f32, f32, f32, torch.zeros(4, dtype=torch.int32),
                          "static_per_channel", 1e-6, True)
    q = torch.zeros(2, 16, 512)
    i32 = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="bfloat16"):
        shim.mla_paged_attention(q, q, q, q, i32, i32, i32, i32, 1, 0.07, True, q)


def test_absorbed_equals_unabsorbed_fp32():
    """softmax(s [q_nope W_kc | q_pe] [c_kv | k_pe]^T) c_kv W_vc^T == standard MLA with k_nope = c_kv W_kc^T,
    v = c_kv W_vc^T, to fp32 rounding: the absorbed form the kernels compute is the model's attention."""
    g = torch.Generator().manual_seed(0)
    H, dn, dv, Lq, Lk = 4, 128, 128, 5, 37
    q_nope, q_pe = torch.randn(Lq, H, dn, generator=g), torch.randn(Lq, H, 64, generator=g)
    ckv, kpe = torch.randn(Lk, 512, generator=g), torch.randn(Lk, 64, generator=g)
    w_kc, w_vc = torch.randn(H, dn, 512, generator=g) * 0.05, torch.randn(H, dv, 512, generator=g) * 0.05
    scale = (dn + 64) ** -0.5
    k_nope, v = torch.einsum("kc,hdc->khd", ckv, w_kc), torch.einsum("kc,hdc->khd", ckv, w_vc)
    s = (torch.einsum("qhd,khd->hqk", q_nope, k_nope) + torch.einsum("qhd,kd->hqk", q_pe, kpe)) * scale
    allowed = torch.arange(Lk)[None, :] <= (Lk - Lq + torch.arange(Lq))[:, None]
    p = torch.softmax(s.masked_fill(~allowed, float("-inf")), -1)
    ref = torch.einsum("hqk,khd->qhd", p, v)
    q_abs = torch.einsum("qhd,hdc->qhc", q_nope, w_kc)
    o = R.attend_mla(torch.cat([q_abs, q_pe], -1), torch.cat([ckv, kpe], -1), ckv, scale, causal=True, round_p=False)
    got = torch.einsum("qhc,hdc->qhd", o, w_vc)
    assert ((got - ref).norm() / ref.norm()).item() < 1e-5


def test_absorbed_layer_vs_transformers_deepseek_v3():
    """tests/mla_ref.mla_attention_layer (projections, q_a/kv_a layernorms, interleaved RoPE, cache writer, absorbed paged
    attention, W_vc, o_proj) against transformers' own DeepseekV3Attention (eager, rope_interleave=True, no rope scaling)
    on the same bf16 weights: a ragged prompt batch, then one decode step against the caches.

    Bound: the two bf16 forms round different intermediates (the absorbed one rounds q_nope W_kc [T, H, 512] and the
    512-wide attention output, the un-absorbed one k_nope / v per head), so neither is closer to the exact result than
    bf16 allows.  Measured against the same layer run in fp32 (the model's definition without bf16 roundings), the
    absorbed form must be as accurate as transformers' bf16 forward (within 10 %), and its distance from that forward must
    stay within transformers' own bf16 error.  Both sit ~5e-3 from fp32 here (1 bf16 ulp = 3.9e-3 relative), which is why the
    3e-3 bar of the Qwen2 layer comparison does not apply to this deeper chain."""
    from transformers import DeepseekV3Config
    from transformers.models.deepseek_v3 import modeling_deepseek_v3 as M
    from oracle import ops as O
    BF16 = torch.bfloat16
    H, dn, dv, page, eps = 4, 32, 32, 4, 1e-6
    cfg = DeepseekV3Config(hidden_size=256, num_attention_heads=H, num_key_value_heads=H, q_lora_rank=96, kv_lora_rank=512,
                           qk_rope_head_dim=64, qk_nope_head_dim=dn, v_head_dim=dv, rope_interleave=True,
                           max_position_embeddings=256, attention_bias=False, rms_norm_eps=eps)
    cfg._attn_implementation = "eager"
    torch.manual_seed(0)
    att = M.DeepseekV3Attention(cfg, 0)
    with torch.no_grad():
        for n, p in att.named_parameters():
            p.copy_(1 + 0.1 * torch.randn_like(p) if "layernorm" in n else torch.randn_like(p) * p.shape[1] ** -0.5)
    att = att.to(BF16).eval()
    rot = M.DeepseekV3RotaryEmbedding(cfg)
    w = {n[:-len(".weight")]: p.detach() for n, p in att.named_parameters()}
    lens = [5, 9]
    xs = [torch.randn(L + 1, 256).to(BF16) for L in lens]            # prompt + the decode step's token

    def hf(dtype):
        m = att.to(dtype)
        out = []
        for x in xs:
            L = x.shape[0]
            cos, sin = rot(x[None].to(dtype), torch.arange(L)[None])
            mask = torch.full((L, L), float("-inf")).triu(1)[None, None].to(dtype)
            with torch.no_grad():
                out.append(m(x[None].to(dtype), (cos, sin), mask)[0][0].float())
        return out

    hf32, hf16 = hf(torch.float32), hf(BF16)

    cs = O.compute_cos_sin_cache(64, 256, 10000)
    npg = [(L + 1 + page - 1) // page for L in lens]
    ckv = torch.zeros(sum(npg) + 1, page, 512, dtype=BF16)
    kpe = torch.zeros(sum(npg) + 1, page, 64, dtype=BF16)
    pages = [list(range(1 + sum(npg[:b]), 1 + sum(npg[:b + 1])))[::-1] for b in range(2)]   # pages out of order

    def step(x_rows, pos_lists, kv_lens):
        pos = torch.tensor(sum(pos_lists, []), dtype=torch.int64)
        slots = torch.tensor([pages[b][p // page] * page + p % page for b, pl in enumerate(pos_lists) for p in pl],
                             dtype=torch.int32)
        qo = torch.tensor([0] + torch.tensor([len(p) for p in pos_lists]).cumsum(0).tolist(), dtype=torch.int32)
        n = [(k + page - 1) // page for k in kv_lens]
        indices = torch.tensor(pages[0][:n[0]] + pages[1][:n[1]], dtype=torch.int32)
        indptr = torch.tensor([0] + torch.tensor(n).cumsum(0).tolist(), dtype=torch.int32)
        last = torch.tensor([k - (m - 1) * page for k, m in zip(kv_lens, n)], dtype=torch.int32)
        return R.mla_attention_layer(w, torch.cat(x_rows), pos, cs, slots, ckv, kpe, qo, indptr, indices, last, H, dn, dv,
                                     eps, (dn + 64) ** -0.5).float()

    prefill = step([x[:L] for x, L in zip(xs, lens)], [list(range(L)) for L in lens], lens)
    decode = step([x[L:] for x, L in zip(xs, lens)], [[L] for L in lens], [L + 1 for L in lens])
    ours = torch.cat([prefill[:lens[0]], decode[:1], prefill[lens[0]:], decode[1:]])
    r32, r16 = torch.cat(hf32), torch.cat(hf16)

    def rel(a, b):
        return ((a - b).norm() / b.norm()).item()
    hf_err = rel(r16, r32)
    assert rel(ours, r32) <= 1.1 * hf_err, (rel(ours, r32), hf_err)
    assert rel(ours, r16) <= hf_err, (rel(ours, r16), hf_err)
    assert hf_err < 1e-2
