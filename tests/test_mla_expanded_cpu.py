"""Expanded MLA prefill without a GPU: the expanded reference layer against transformers' DeepseekV3Attention and against
the absorbed reference layer, the plan's arithmetic and form selector, and argument errors of the C ABI (raised before
any launch)."""
import ctypes

import torch

from tests import mla_expanded_ref as E
from tests import mla_ref as R
from xllm_b200 import _lib

c_i64 = ctypes.c_int64
# the selector's constant (include/xllm_b200_ops.h, xb_mla_expanded_plan)
EXPANDED_COST = 0.5


def plan(qo, kv, H=16):
    arr = (ctypes.c_int64 * 8)()
    rc = _lib.lib().xb_mla_expanded_plan(arr, len(qo), H, (ctypes.c_int32 * len(qo))(*qo), (ctypes.c_int32 * len(kv))(*kv))
    return rc, arr


def _err():
    return _lib.lib().xb_last_error().decode()


def _a(x):
    return (x + 255) // 256 * 256


def test_plan_sizes_workspace_and_counts():
    for qo, kv, H in (([4096], [4096], 128), ([300, 1, 37], [2300, 18, 37], 16), ([16], [32768], 1)):
        rc, p = plan(qo, kv, H)
        assert rc == 0
        n = sum(kv)
        assert p[5] == n and p[2] == len(qo) and p[3] == H and p[4] == max(qo) and p[6] == max(kv)
        assert p[7] & ((1 << 40) - 1) == sum(qo)
        assert p[1] == _a(n * H * 512) + _a(n * 1024) + _a(n * 128) + _a((len(qo) + 1) * 4)


def _expanded_by_rule(qo, kv):
    pairs = sum(q * (k - q) + q * (q + 1) // 2 for q, k in zip(qo, kv))
    absorbed = 2 * (576 + 512) * pairs
    expanded = 2 * (192 + 128) * pairs + 2 * 512 * 256 * sum(kv)
    return max(qo) > 1 and absorbed > EXPANDED_COST * expanded


def test_selector():
    assert plan([1] * 64, [4096] * 64)[1][0] == 0                 # decode: absorbed
    assert plan([1], [1])[1][0] == 0
    assert plan([4096], [4096])[1][0] == 1                        # a prompt: expanded
    assert plan([4096], [4096], H=128)[1][0] == 1
    assert plan([16], [32768])[1][0] == 0                         # a short chunk over a long history: absorbed
    # both sides of the boundary, over history 0 .. 32 K
    for hist in (0, 1024, 8192, 32768):
        flips = [qo for qo in range(2, 4097) if _expanded_by_rule([qo], [qo + hist])]
        assert flips, hist
        q = flips[0]
        assert plan([q], [q + hist])[1][0] == 1 and plan([q - 1], [q - 1 + hist])[1][0] == (1 if q - 1 in flips else 0)
        assert all(plan([x], [x + hist])[1][0] == int(x in flips) for x in (q - 1, q, q + 1, 2 * q, 4096) if x >= 1)


def test_plan_rejects_bad_arguments():
    assert plan([5], [4], 16)[0] != 0 and "qo_len" in _err()
    assert plan([5], [8], 0)[0] != 0 and "num_heads" in _err()
    assert plan([5], [8], 129)[0] != 0 and "num_heads" in _err()
    assert _lib.lib().xb_mla_expanded_plan(None, 1, 16, None, None) != 0 and "null" in _err()
    arr = (ctypes.c_int64 * 8)()
    assert _lib.lib().xb_mla_expanded_plan(arr, 0, 16, None, None) != 0 and "batch" in _err()
    assert _lib.lib().xb_mla_expanded_plan(arr, 1, 16, None, None) != 0 and "null" in _err()


def _run(p, ptr=16, ws_bytes=None, page=16):
    """a call whose pointers are never dereferenced: every case is rejected before any launch"""
    v = ctypes.c_void_p(ptr) if ptr else None
    i32 = ctypes.cast(v, ctypes.POINTER(ctypes.c_int32)) if ptr else None
    return _lib.lib().xb_mla_prefill_expanded_bf16(
        p, v, c_i64(16 * 192), c_i64(192), v, c_i64(16 * 512), c_i64(512), v, c_i64(16 * 64), c_i64(64), page, i32, i32, i32,
        i32, v, v, c_i64(16 * 128), c_i64(128), ctypes.c_float(0.07), ctypes.c_void_p(4096),
        c_i64(1 << 40 if ws_bytes is None else ws_bytes), None)


def test_prefill_rejects_bad_arguments():
    rc, p = plan([300, 37], [2300, 37], 16)
    assert rc == 0
    assert _run(None) != 0 and "plan" in _err()
    assert _run(p, ptr=0) != 0 and "null" in _err()
    assert _run(p, ws_bytes=p[1] - 1) != 0 and "workspace" in _err()
    assert _run(p, ptr=18) != 0 and "aligned" in _err()
    assert _run(p, page=0) != 0 and "page_size" in _err()
    bad = (ctypes.c_int64 * 8)(*p)
    bad[1] += 256
    assert _run(bad) != 0 and "corrupt" in _err()
    absorbed = (ctypes.c_int64 * 8)()
    assert _lib.lib().xb_mla_plan(absorbed, 1, 16, 512, 64, 1, 16, 8, 132) == 0
    assert _run(absorbed) != 0 and "expanded MLA plan" in _err()


def test_expanded_layer_vs_transformers_deepseek_v3():
    """tests/mla_expanded_ref.mla_attention_layer_expanded against transformers' DeepseekV3Attention (eager,
    rope_interleave=True), on a ragged prompt batch and then a chunk of 3 tokens per request over that history, with the
    bounds of test_absorbed_layer_vs_transformers_deepseek_v3: as accurate as transformers' bf16 forward against its fp32
    forward (within 10 %), and within transformers' own bf16 error of it.  The expanded and the absorbed reference layers
    round different intermediates, so they must agree within that same bf16 error."""
    from transformers import DeepseekV3Config
    from transformers.models.deepseek_v3 import modeling_deepseek_v3 as M
    from oracle import ops as O
    BF16 = torch.bfloat16
    H, dn, dv, page, eps, chunk = 4, 32, 32, 4, 1e-6, 3
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
    xs = [torch.randn(L + chunk, 256).to(BF16) for L in lens]        # prompt + the chunk's tokens

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
    npg = [(L + chunk + page - 1) // page for L in lens]
    pages = [list(range(1 + sum(npg[:b]), 1 + sum(npg[:b + 1])))[::-1] for b in range(2)]   # pages out of order

    def run(layer):
        ckv = torch.zeros(sum(npg) + 1, page, 512, dtype=BF16)
        kpe = torch.zeros(sum(npg) + 1, page, 64, dtype=BF16)

        def step(x_rows, pos_lists, kv_lens):
            pos = torch.tensor(sum(pos_lists, []), dtype=torch.int64)
            slots = torch.tensor([pages[b][p // page] * page + p % page for b, pl in enumerate(pos_lists) for p in pl],
                                 dtype=torch.int32)
            qo = torch.tensor([0] + torch.tensor([len(p) for p in pos_lists]).cumsum(0).tolist(), dtype=torch.int32)
            n = [(k + page - 1) // page for k in kv_lens]
            indices = torch.tensor(pages[0][:n[0]] + pages[1][:n[1]], dtype=torch.int32)
            indptr = torch.tensor([0] + torch.tensor(n).cumsum(0).tolist(), dtype=torch.int32)
            last = torch.tensor([k - (m - 1) * page for k, m in zip(kv_lens, n)], dtype=torch.int32)
            return layer(w, torch.cat(x_rows), pos, cs, slots, ckv, kpe, qo, indptr, indices, last, H, dn, dv, eps,
                         (dn + 64) ** -0.5).float()

        prefill = step([x[:L] for x, L in zip(xs, lens)], [list(range(L)) for L in lens], lens)
        chunked = step([x[L:] for x, L in zip(xs, lens)], [list(range(L, L + chunk)) for L in lens],
                       [L + chunk for L in lens])
        return torch.cat([prefill[:lens[0]], chunked[:chunk], prefill[lens[0]:], chunked[chunk:]])

    ours, absorbed = run(E.mla_attention_layer_expanded), run(R.mla_attention_layer)
    r32, r16 = torch.cat(hf32), torch.cat(hf16)

    def rel(a, b):
        return ((a - b).norm() / b.norm()).item()
    hf_err = rel(r16, r32)
    assert rel(ours, r32) <= 1.1 * hf_err, (rel(ours, r32), hf_err)
    assert rel(ours, r16) <= hf_err, (rel(ours, r16), hf_err)
    assert rel(ours, absorbed) <= hf_err, (rel(ours, absorbed), hf_err)
    assert hf_err < 1e-2


def test_expanded_attention_equals_absorbed_fp32():
    """the expanded reference attention on kv_b_proj's up-projection equals the absorbed one followed by W_UV, in fp32
    (un-rounded P): the two forms compute the same attention"""
    g = torch.Generator().manual_seed(1)
    H, Lq, Lk = 4, 5, 37
    q = torch.randn(Lq, H, 192, generator=g)
    ckv, kpe = torch.randn(Lk, 512, generator=g), torch.randn(Lk, 64, generator=g)
    w = torch.randn(H * 256, 512, generator=g) * 0.05
    kv_up = (ckv @ w.t()).view(Lk, H, 256)
    o = E.attend_expanded(q, kv_up[..., :128], kpe, kv_up[..., 128:], 192 ** -0.5, round_p=False)
    w_kc, w_vc = w.view(H, 256, 512)[:, :128], w.view(H, 256, 512)[:, 128:]
    q_abs = torch.einsum("qhd,hdc->qhc", q[..., :128], w_kc)
    oa = R.attend_mla(torch.cat([q_abs, q[..., 128:]], -1), torch.cat([ckv, kpe], -1), ckv, 192 ** -0.5, causal=True,
                      round_p=False)
    ref = torch.einsum("qhc,hdc->qhd", oa, w_vc)
    assert ((o - ref).norm() / ref.norm()).item() < 1e-5
