"""GPU parity of the decode-step form of the W4A16 linears (xb_linear_w4a16_decode_fused): add+RMSNorm prologue and the
RoPE + KV-scatter epilogue folded into the GEMV launch.  Decomposition of the proof:
  (a) rope_and_cache_packed (elementwise, packed column order) == oracle rotary_embedding + reshape_paged_cache, bit-exact
  (b) fused rope epilogue == plain GEMV on the same packed weights followed by (a), bit-exact (same accumulation order)
  (c) the plain GEMV itself vs the oracle linear: tests/test_gpu_linear.py
  (d) norm prologue: residual_out bit-exact; y vs oracle(fused_add_rms_norm -> linear) within the dot-product bound
  (e) staging x in shared memory alone changes nothing, bit-exact
"""
import math

import pytest
import torch

from oracle import ops as O
from oracle import quant as Q
from tests.util import assert_close_bf16, assert_close_sum

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"

HEADS = [(28, 4, 128), (14, 2, 64), (8, 1, 128)]     # Qwen2-7B, Qwen2-0.5B, Llama-3-70B TP8 per-GPU


def _packed_from_logical(t, nh, nkv, D):
    from xllm_b200 import quant
    return t[:, quant.qkv_rope_index(nh, nkv, D)]


def _rope_case(T, nh, nkv, D, page=16, seed=5):
    g = torch.Generator().manual_seed(seed)
    N = (nh + 2 * nkv) * D
    qkv = torch.randn(T, N, generator=g).to(BF16)
    pos = torch.randint(0, 4000, (T,), generator=g, dtype=torch.int64)
    nblk = T + 3
    slots = (torch.randperm(nblk * page - page, generator=g)[:T] + page).to(torch.int32)
    if T > 2:
        slots[1] = -1                                                    # skipped token
    cs = O.compute_cos_sin_cache(D, 4096, 1000000.0, BF16)
    kc = torch.randn(nblk, page, nkv, D, generator=g).to(BF16)
    vc = torch.randn(nblk, page, nkv, D, generator=g).to(BF16)
    return qkv, pos, slots, cs, kc, vc


def _oracle_rope_cache(qkv, pos, slots, cs, kc, vc, nh, nkv, D):
    qs, kvs = nh * D, nkv * D
    T = qkv.shape[0]
    q, k, v = qkv[:, :qs].reshape(T, nh, D), qkv[:, qs:qs + kvs].reshape(T, nkv, D), qkv[:, qs + kvs:].reshape(T, nkv, D)
    q2, k2 = O.rotary_embedding(pos, q, k, cs, is_neox=True)
    kc2, vc2 = kc.clone(), vc.clone()
    O.reshape_paged_cache(slots, k2, v, kc2, vc2)
    return torch.cat([q2.reshape(T, -1), k2.reshape(T, -1), v.reshape(T, -1)], dim=1), kc2, vc2


@pytest.mark.parametrize("nh,nkv,D", HEADS)
@pytest.mark.parametrize("T", [1, 5, 40])
def test_rope_and_cache_packed_bit_exact(T, nh, nkv, D, built_lib):
    from xllm_b200 import ops
    qkv, pos, slots, cs, kc, vc = _rope_case(T, nh, nkv, D)
    ref, kc_ref, vc_ref = _oracle_rope_cache(qkv, pos, slots, cs, kc, vc, nh, nkv, D)
    packed = _packed_from_logical(qkv, nh, nkv, D).contiguous().to(DEV)
    out = torch.empty_like(packed)
    kcd, vcd = kc.to(DEV), vc.to(DEV)
    ops.rope_and_cache_packed(pos.to(DEV), packed, out, cs.to(DEV), slots.to(DEV), kcd, vcd, nh, nkv, D)
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), ref), "q | k | v after RoPE (logical order)"
    assert torch.equal(kcd.cpu(), kc_ref) and torch.equal(vcd.cpu(), vc_ref), "paged caches after the scatter"


def _w4(N, K, gs, seed, bias):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(N, K, generator=g) * 0.02).to(BF16)
    q, s, z = Q.quantize(w, 4, gs)
    b = (torch.randn(N, generator=g) * 0.1).to(BF16) if bias else None
    return q, s, z, b


@pytest.mark.parametrize("nh,nkv,D,K", [(28, 4, 128, 3584), (14, 2, 64, 896), (8, 1, 128, 8192)])
@pytest.mark.parametrize("M", [1, 3, 8])
@pytest.mark.parametrize("staged", [False, True])
def test_fused_rope_epilogue_equals_gemv_then_rope(M, nh, nkv, D, K, staged, built_lib, oracle_form="bf16w", gs=None):
    from xllm_b200 import ops, quant
    N = (nh + 2 * nkv) * D
    gs = gs or (128 if K % 128 == 0 else 64)
    if staged and not ops.w4a16_decode_fused_fits(M, K):
        pytest.skip("activation block does not fit the shared-memory stage (the runner falls back to the unstaged kernel)")
    q, s, z, b = _w4(N, K, gs, 11, bias=True)
    qw, meta, bp = quant.pack_w4_qkv_rope(q, s, z, nh, nkv, D, gs, b)
    qw, meta, bp = qw.to(DEV), meta.to(DEV), bp.to(DEV)
    _, pos, slots, cs, kc, vc = _rope_case(M, nh, nkv, D, seed=3)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(M, K, generator=g).to(BF16).to(DEV)
    # reference path on the device: plain GEMV (packed column order) -> packed rope kernel
    raw = ops.w4a16_linear_small_m(x, qw, meta, gs, bp)
    ref = torch.empty_like(raw)
    kc1, vc1 = kc.to(DEV), vc.to(DEV)
    ops.rope_and_cache_packed(pos.to(DEV), raw, ref, cs.to(DEV), slots.to(DEV), kc1, vc1, nh, nkv, D)
    # fused
    out = torch.empty_like(raw)
    kc2, vc2 = kc.to(DEV), vc.to(DEV)
    ops.w4a16_decode_fused(x, qw, meta, gs, bp, out, stage_x=staged, epilogue="rope_cache", positions=pos.to(DEV),
                           cos_sin_cache=cs.to(DEV), slot_ids=slots.to(DEV), key_cache=kc2, value_cache=vc2, num_heads=nh,
                           num_kv_heads=nkv, head_dim=D)
    torch.cuda.synchronize()
    assert torch.equal(out, ref), "fused RoPE epilogue differs from GEMV + rope kernel"
    assert torch.equal(kc2, kc1) and torch.equal(vc2, vc1), "fused KV scatter differs"
    # and against the oracle end to end (linear on the logical rows -> RoPE), within the linear's 1-ulp noise:
    # a 1-ulp flip of one linear output moves a rotated value by at most that ulp (|cos|, |sin| <= 1)
    y = Q.linear_wna16(x.cpu(), q, s, z, gs, b, form=oracle_form)
    full, _, _ = _oracle_rope_cache(y, pos, slots, cs, kc, vc, nh, nkv, D)
    qs = nh * D
    mag = y.float().abs()
    half = D // 2
    pair = mag.view(M, -1, 2, half)
    bound = (pair[:, :, 0] + pair[:, :, 1]).repeat_interleave(2, dim=1).reshape(M, -1) * 2.0 ** -7 + 2.0 ** -9
    err = (out.cpu().float() - full.float()).abs()
    assert (err <= bound).all(), f"fused qkv vs oracle: worst err/bound {(err / bound).max():.2f}"


@pytest.mark.parametrize("N,K,epi", [(4608, 3584, "none"), (37888, 3584, "act_mul"), (1024, 8192, "none"), (2432, 896, "none")])
@pytest.mark.parametrize("M", [1, 4, 8])
@pytest.mark.parametrize("with_res", [True, False])
def test_fused_norm_prologue(M, N, K, epi, with_res, built_lib, gs=None):
    from xllm_b200 import ops, quant
    if M * (K + 8) * 2 + 256 > 72 * 1024:
        assert not ops.w4a16_decode_fused_fits(M, K)
        pytest.skip("activation block does not fit the shared-memory stage (the runner falls back to separate launches)")
    assert ops.w4a16_decode_fused_fits(M, K)
    gs = gs or (128 if K % 128 == 0 else 64)
    q, s, z, b = _w4(N, K, gs, 21, bias=(N == 4608))
    g = torch.Generator().manual_seed(31)
    x = torch.randn(M, K, generator=g).to(BF16)
    res = torch.randn(M, K, generator=g).to(BF16) if with_res else None
    nw = (1 + 0.1 * torch.randn(K, generator=g)).to(BF16)
    eps = 1e-6
    if with_res:
        normed, res_ref = O.fused_add_rms_norm(x, res, nw, eps)
    else:
        normed, res_ref = O.rms_norm(x, nw, eps), x
    if epi == "act_mul":
        qw, meta, bp = quant.pack_w4_gate_up(q, s, z, gs, b)
        ref = O.act_and_mul(Q.linear_wna16(normed, q, s, z, gs, b), "silu")
    else:
        qw, meta = quant.pack_w4(q, s, z, gs)
        bp = b
        ref = Q.linear_wna16(normed, q, s, z, gs, b)
    res_out = torch.full((M, K), 7.0, dtype=BF16, device=DEV)
    y = ops.w4a16_decode_fused(x.to(DEV), qw.to(DEV), meta.to(DEV), gs, bp.to(DEV) if bp is not None else None,
                               norm_weight=nw.to(DEV), eps=eps, residual_in=res.to(DEV) if with_res else None,
                               residual_out=res_out, epilogue=epi, act_mode="silu")
    torch.cuda.synchronize()
    assert torch.equal(res_out.cpu(), res_ref), "updated residual stream must be bit-exact (one bf16 add)"
    if epi == "act_mul":
        # act(gate)*up of two 1-ulp-accurate linears (same bar as test_w4a16_gate_up_act_fused)
        assert_close_bf16(y, ref, ulps=4, rel_l2=3e-3, what=f"norm + gate_up + act M={M}", atol=2.0 ** -12)
    else:
        wd = Q.dequantize(q, s, z, gs)
        scale = normed.float().abs() @ wd.float().abs().t() + (b.float().abs() if b is not None else 0)
        # rstd is summed in a different order than the oracle's: an occasional 1-ulp flip of a normalised activation
        # perturbs the dot product by 2^-8 of ONE term - covered by 3e-5 of the sum of the terms
        assert_close_sum(y, ref, scale, rtol=3e-5, what=f"norm prologue + linear M={M} N={N} K={K}")


@pytest.mark.parametrize("N,K", [(3584, 3584), (3584, 18944), (37888, 3584)])
def test_staged_x_is_bit_identical(N, K, built_lib, gs=128):
    from xllm_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(1)
    qw = torch.randint(-2 ** 31, 2 ** 31 - 1, (N // 16, K // 64, 32, 4), generator=g, device=DEV, dtype=torch.int32)
    sc = (torch.rand(K // gs, N, generator=g, device=DEV) * 0.01 + 0.001).to(BF16).view(torch.int16).to(torch.int32) & 0xFFFF
    meta = (sc | (0x4308 << 16)).contiguous()
    for M in (1, 2, 8):
        if not ops.w4a16_decode_fused_fits(M, K):
            continue
        x = torch.randn(M, K, generator=g, device=DEV).to(BF16)
        y0 = ops.w4a16_linear_small_m(x, qw, meta, gs)
        y1 = ops.w4a16_decode_fused(x, qw, meta, gs, stage_x=True)
        torch.cuda.synchronize()
        assert torch.equal(y0, y1), f"M={M}: staging x in shared memory changed the result"


@pytest.mark.parametrize("H,Kin,Nout,epi", [(3584, 3584, 4608, "none"), (3584, 18944, 37888, "act_mul"), (896, 896, 1152, "none"),
                                            (8192, 8192, 1280, "none")])
@pytest.mark.parametrize("M", [1, 3, 8])
def test_split_rms_norm_producer_and_consumer(M, H, Kin, Nout, epi, built_lib, gs=None):
    """RMSNorm split over two linears: the row-parallel projection (producer, epilogue "residual_stats") adds the
    residual and emits the updated residual stream + per-tile partial sums of its squares; the next linear (consumer,
    norm_stats_in) normalises that stream while staging it.  Checked against fused_add_rms_norm -> linear of the oracle:
    (a) residual stream vs bf16(bf16(linear) + residual) within the linear's 1-ulp noise, (b) the partials sum to the sum of
    squares of the stream the kernel wrote, (c) the consumer against the oracle fed with the kernel's own stream."""
    from xllm_b200 import ops, quant
    if not ops.w4a16_decode_fused_fits(M, H):
        pytest.skip("the consumer's activation block does not fit the shared-memory stage")
    gs = gs or (128 if Kin % 128 == 0 and H % 128 == 0 else 64)
    g = torch.Generator().manual_seed(41)
    q1, s1, z1, _ = _w4(H, Kin, gs, 5, bias=False)               # producer: [H, Kin] (o_proj / down_proj)
    q2, s2, z2, b2 = _w4(Nout, H, gs, 6, bias=(Nout == 4608))    # consumer: [Nout, H] (qkv / gate_up)
    x = torch.randn(M, Kin, generator=g).to(BF16)
    res = torch.randn(M, H, generator=g).to(BF16)
    nw = (1 + 0.1 * torch.randn(H, generator=g)).to(BF16)
    eps = 1e-6
    qw1, m1 = quant.pack_w4(q1, s1, z1, gs)
    res_out = torch.empty(M, H, dtype=BF16, device=DEV)
    stats = torch.full((H // 16, 8), -1.0, dtype=torch.float32, device=DEV)
    ops.w4a16_decode_fused(x.to(DEV), qw1.to(DEV), m1.to(DEV), gs, None, None, epilogue="residual_stats", residual_in=res.to(DEV),
                           residual_out=res_out, norm_stats_out=stats, stage_x=ops.w4a16_decode_fused_fits(M, Kin))
    torch.cuda.synchronize()
    y1 = Q.linear_wna16(x, q1, s1, z1, gs, None)
    r_ref = (y1.float() + res.float()).to(BF16)
    assert_close_bf16(res_out, r_ref, ulps=2, rel_l2=1e-3, what="residual stream of the producer", atol=2.0 ** -8)
    r = res_out.cpu()
    ss = stats.cpu()
    assert torch.all(ss[:, M:] == 0), "partials of absent tokens must be zero"
    tile_sq = (r.float() ** 2).view(M, H // 16, 16).sum(-1).t()          # [H/16, M]
    assert torch.allclose(ss[:, :M], tile_sq, rtol=1e-6, atol=0), "per-tile partial sums of squares"
    # consumer on the kernel's own stream
    if epi == "act_mul":
        qw2, m2, bp = quant.pack_w4_gate_up(q2, s2, z2, gs, b2)
    else:
        qw2, m2 = quant.pack_w4(q2, s2, z2, gs)
        bp = b2
    y = ops.w4a16_decode_fused(res_out, qw2.to(DEV), m2.to(DEV), gs, bp.to(DEV) if bp is not None else None, norm_weight=nw.to(DEV),
                               eps=eps, norm_stats_in=stats, epilogue=epi, act_mode="silu")
    torch.cuda.synchronize()
    normed = O.rms_norm(r, nw, eps)
    ref = Q.linear_wna16(normed, q2, s2, z2, gs, b2)
    if epi == "act_mul":
        assert_close_bf16(y, O.act_and_mul(ref, "silu"), ulps=4, rel_l2=3e-3, what="split norm + gate_up + act", atol=2.0 ** -12)
    else:
        wd = Q.dequantize(q2, s2, z2, gs)
        scale = normed.float().abs() @ wd.float().abs().t() + (b2.float().abs() if b2 is not None else 0)
        assert_close_sum(y, ref, scale, rtol=3e-5, what=f"split norm consumer M={M} N={Nout} K={H}")
