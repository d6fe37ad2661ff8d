"""Checkpoint-side packing of weight-only quantised linears into the kernel layout.

Logical form (AWQ/GPTQ-like, oracle/quant.py spec): q uint8 [N,K] in 0..15, scales bf16 [N,K/g], zeros uint8 [N,K/g].
Kernel form: qweight int32 [N/16, K/64, 32, 4] (tile-packed nibbles, see csrc/linear_small_m.cu) and
meta int32 [K/g, N] = bf16(scale) | bf16(128+zero) << 16.  Packing runs on the host (C routine
xb_w4_pack_rows through ctypes, or the vectorised torch path below) - it is load-time work, not the hot path.
"""
import ctypes

import torch

from ._lib import check, lib


def pack_w4(q: torch.Tensor, scales: torch.Tensor, zeros: torch.Tensor, group_size: int = 128):
    """-> (qweight int32 [N/16,K/64,32,4], meta int32 [K/g,N]) on q's device."""
    N, K = q.shape
    assert N % 16 == 0 and K % 64 == 0 and K % group_size == 0 and group_size % 64 == 0
    qq = q.to(torch.int32).view(N // 16, 2, 8, K // 64, 4, 4, 4)          # [nt, half(r0/r1), g, kt, t, j, s]
    r0, r1 = qq[:, 0], qq[:, 1]                                           # [nt, g, kt, t, j, s]
    w = (r0[..., 0] | (r0[..., 1] << 16) | (r1[..., 0] << 4) | (r1[..., 1] << 20) |
         (r0[..., 2] << 8) | (r0[..., 3] << 24) | (r1[..., 2] << 12) | (r1[..., 3] << 28))   # [nt, g, kt, t, j]
    # int32 overflow of bit 31 wraps as intended
    qweight = w.permute(0, 2, 1, 3, 4).reshape(N // 16, K // 64, 32, 4).contiguous()
    s_bits = scales.to(torch.bfloat16).view(torch.int16).to(torch.int32) & 0xFFFF
    z_bits = (zeros.to(torch.float32) + 128.0).to(torch.bfloat16).view(torch.int16).to(torch.int32) & 0xFFFF
    meta = (s_bits | (z_bits << 16)).t().contiguous()
    return qweight, meta


def interleave_gate_up_index(intermediate: int, device=None) -> torch.Tensor:
    """Row permutation of a fused gate_up projection [2I, K] (gate rows then up rows) into the layout the fused
    gate_up+activation kernel expects: per 16-row tile, 8 gate rows followed by the matching 8 up rows."""
    assert intermediate % 8 == 0
    t = torch.arange(intermediate // 8, device=device).repeat_interleave(16)
    i = torch.arange(16, device=device).repeat(intermediate // 8)
    return torch.where(i < 8, 8 * t + i, intermediate + 8 * t + (i - 8))


def pack_w4_gate_up(q, scales, zeros, group_size=128, bias=None):
    """pack a fused gate_up weight with interleaved rows -> (qweight, meta, bias_interleaved)."""
    idx = interleave_gate_up_index(q.shape[0] // 2, q.device)
    qw, meta = pack_w4(q[idx], scales[idx], zeros[idx], group_size)
    return qw, meta, (bias[idx].contiguous() if bias is not None else None)


def qkv_rope_index(num_heads: int, num_kv_heads: int, head_dim: int, device=None) -> torch.Tensor:
    """Row permutation of a fused qkv projection [(Hq + 2 Hkv) * D, K] into the layout the rope-fused GEMV epilogue
    expects (csrc/linear_small_m.cu, epilogue 2): inside every head, 16-row tile j holds dims 8j..8j+7 followed by
    D/2 + 8j..D/2 + 8j+7 - the two halves of 8 NeoX rotary pairs sit in rows g and g+8 of one tile."""
    assert head_dim % 16 == 0
    half = head_dim // 2
    j = torch.arange(head_dim // 16, device=device).repeat_interleave(16)
    i = torch.arange(16, device=device).repeat(head_dim // 16)
    within = torch.where(i < 8, 8 * j + i, half + 8 * j + (i - 8))                     # [D] permuted -> logical dim
    heads = torch.arange(num_heads + 2 * num_kv_heads, device=device).unsqueeze(1) * head_dim
    return (heads + within.unsqueeze(0)).reshape(-1)


def pack_w4_qkv_rope(q, scales, zeros, num_heads, num_kv_heads, head_dim, group_size=128, bias=None):
    """pack a fused qkv weight with the rope-pair row order -> (qweight, meta, bias_permuted)."""
    idx = qkv_rope_index(num_heads, num_kv_heads, head_dim, q.device)
    assert idx.numel() == q.shape[0]
    qw, meta = pack_w4(q[idx], scales[idx], zeros[idx], group_size)
    return qw, meta, (bias[idx].contiguous() if bias is not None else None)


def pack_w8(q: torch.Tensor, scales: torch.Tensor, zeros: torch.Tensor, group_size: int = 128):
    """W8A16: q uint8 [N,K] in 0..255 -> (qweight int32 [N/16,K/64,32,8], meta int32 [K/g,N] = bf16 scale | zero << 16).
    Lane 4g+t of a 16x64 tile holds rows g (words 0..3) and g+8 (words 4..7), k in [16t, 16t+16) ascending
    (csrc/linear_q8_small_m.cu; the same tensor feeds the wgmma GEMM kind W8)."""
    N, K = q.shape
    assert N % 16 == 0 and K % 64 == 0 and K % group_size == 0 and group_size % 64 == 0
    qq = q.to(torch.int32).view(N // 16, 2, 8, K // 64, 4, 4, 4)          # [nt, half, g, kt, t, j, byte]
    w = qq[..., 0] | (qq[..., 1] << 8) | (qq[..., 2] << 16) | (qq[..., 3] << 24)     # [nt, half, g, kt, t, j]
    qweight = w.permute(0, 3, 2, 4, 1, 5).reshape(N // 16, K // 64, 32, 8).contiguous()   # [nt, kt, g, t, half, j]
    s_bits = scales.to(torch.bfloat16).view(torch.int16).to(torch.int32) & 0xFFFF
    meta = (s_bits | (zeros.to(torch.int32) << 16)).t().contiguous()
    return qweight, meta


def pack_w8_c(q: torch.Tensor) -> torch.Tensor:
    """byte packing through the C routine (tests pin the two packers against each other)."""
    N, K = q.shape
    qc = q.cpu().contiguous()
    out = torch.empty(N // 16, K // 64, 32, 8, dtype=torch.int32)
    check(lib().xb_w8_pack_rows(ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(qc.data_ptr()), ctypes.c_int(N),
                                ctypes.c_int(K)), "w8_pack_rows")
    return out


def pack_w4_c(q: torch.Tensor) -> torch.Tensor:
    """Same nibble packing through the C routine (used by tests to pin the two packers against each other)."""
    N, K = q.shape
    qc = q.cpu().contiguous()
    out = torch.empty(N // 16, K // 64, 32, 4, dtype=torch.int32)
    check(lib().xb_w4_pack_rows(ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(qc.data_ptr()), ctypes.c_int(N),
                                ctypes.c_int(K)), "w4_pack_rows")
    return out


# ---------------------------------------------------------------------------------------------------------------
# checkpoint surface (SURVEY 8f n1): AutoAWQ / AutoGPTQ tensors -> the logical (q, scales, zeros) form above.
# The reference parses `bits / group_size / sym / desc_act` into QuantArgs (framework/quant_args.h:36-60,
# hf_model_loader.cpp:384-440) but loads no qweight/qzeros/scales; these converters are what its loader would call.
# Formats (published conventions of the two libraries):
#   AWQ  (GEMM):  qweight int32 [K, N/8], qzeros int32 [K/g, N/8], scales fp16 [K/g, N]; the 8 nibbles of a word hold
#                 columns 8j + [0, 2, 4, 6, 1, 3, 5, 7] from the low nibble up ("order_map"); w = (q - z) * s.
#   GPTQ (v1):    qweight int32 [K/8, N] (8 consecutive k per word, low nibble first), qzeros int32 [K/g, N/8]
#                 (8 consecutive n per word) storing z - 1, scales fp16 [K/g, N], g_idx int32 [K]; w = (q - (qz + 1)) * s.
# ---------------------------------------------------------------------------------------------------------------
_AWQ_ORDER = [0, 2, 4, 6, 1, 3, 5, 7]


def _unpack_nibbles_lastdim(t: torch.Tensor, order=None) -> torch.Tensor:
    """int32 [..., C] -> uint8 [..., 8C]: nibble i of a word goes to position order[i] within its group of 8."""
    shifts = torch.arange(0, 32, 4, dtype=torch.int32, device=t.device)
    nib = ((t.unsqueeze(-1) >> shifts) & 0xF).to(torch.uint8)            # [..., C, 8] nibble-position order
    if order is not None:
        out = torch.empty_like(nib)
        out[..., torch.tensor(order, device=t.device)] = nib              # position i -> column order[i]
        nib = out
    return nib.reshape(*t.shape[:-1], t.shape[-1] * 8)


def from_awq(qweight: torch.Tensor, qzeros: torch.Tensor, scales: torch.Tensor, group_size: int = 128):
    """AutoAWQ GEMM tensors -> (q uint8 [N,K], scales bf16 [N,K/g], zeros uint8 [N,K/g])."""
    K = qweight.shape[0]
    q = _unpack_nibbles_lastdim(qweight, _AWQ_ORDER)                       # [K, N]
    z = _unpack_nibbles_lastdim(qzeros, _AWQ_ORDER)                        # [K/g, N]
    if K % group_size != 0 or z.shape[0] != K // group_size:
        raise ValueError("AWQ tensors do not match group_size")
    return q.t().contiguous(), scales.to(torch.bfloat16).t().contiguous(), z.t().contiguous()


def from_gptq(qweight: torch.Tensor, qzeros: torch.Tensor, scales: torch.Tensor, g_idx=None, group_size: int = 128,
              zeros_plus_one: bool = True):
    """AutoGPTQ 4-bit tensors -> (q uint8 [N,K], scales bf16 [N,K/g], zeros uint8 [N,K/g]).
    desc_act (a g_idx that is not k // group_size) permutes K and is not supported by the kernels."""
    K8, N = qweight.shape
    K = K8 * 8
    q = _unpack_nibbles_lastdim(qweight.t().contiguous()).reshape(N, K)    # words along K: [N, K/8] -> [N, K]
    z = _unpack_nibbles_lastdim(qzeros).to(torch.int16)                    # [K/g, N]
    if zeros_plus_one:
        z = z + 1
    if g_idx is not None:
        expect = torch.arange(K, device=g_idx.device, dtype=g_idx.dtype) // group_size
        if not torch.equal(g_idx, expect):
            raise ValueError("desc_act / act-order checkpoints (non-monotonic g_idx) are not supported")
    if (z < 0).any() or (z > 15).any():
        raise ValueError("zero points out of the 4-bit range after the +1 correction")
    return q.contiguous(), scales.to(torch.bfloat16).t().contiguous(), z.to(torch.uint8).t().contiguous()
