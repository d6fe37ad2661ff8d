"""Host-side mirror of `xllm::kernel::cuda::*` (xllm/core/kernels/cuda/cuda_ops_api.h:31-216).

Same function names, argument order and in-place/out conventions as the
reference; tensors are torch CUDA tensors used purely as device-memory handles.
Everything routes through the C ABI (include/xllm_b200_ops.h); errors raise
XllmB200Error (the reference aborts via glog CHECK / throws c10::Error).
"""
import ctypes
from typing import Optional, Tuple

import torch

from ._lib import XllmB200Error, c_f32, c_i32, c_i64, c_ptr, check, lib

BF16 = torch.bfloat16
E4M3 = torch.float8_e4m3fn


def _stream():
    return c_ptr(torch.cuda.current_stream().cuda_stream)


def _p(t: Optional[torch.Tensor]):
    return c_ptr(0) if t is None else c_ptr(t.data_ptr())


def _need(cond, msg):
    if not cond:
        raise XllmB200Error(msg)


def _cuda_bf16(t, name):
    _need(t.is_cuda, f"{name} must be a CUDA tensor (no CPU path)")
    _need(t.dtype == BF16, f"{name} must be bfloat16, got {t.dtype}")


# Streaming (small-M) kernels vs the 128-row GEMMs: the GEMMs launch one CTA per 128-row output tile, so with few output
# columns most SMs idle, while the streaming kernels spread every weight row over the SMs.  Weight-only: streaming up to
# M = 16 always, up to M = 64 when N <= 16384.  FP8: streaming only up to M = 8 and N <= 16384 (the FP8 GEMM's swap-AB
# form already streams 1 byte per weight).  The crossovers have not been re-measured on the H100 (tools/gemv_sweep.py q8).
FP8_SMALL_M_MAX = 8
WQ_SMALL_M_MAX = 16
WQ_SMALL_M_MAX_NARROW = 64      # ... when the projection has at most SMALL_N_MAX output columns
SMALL_N_MAX = 16384


# ---- K7 ---------------------------------------------------------------------
def rms_norm(output: torch.Tensor, input: torch.Tensor, weight: torch.Tensor, eps: float) -> None:
    """cuda_ops_api.h:157-160 / norm.cu:430-460."""
    _cuda_bf16(input, "input"); _cuda_bf16(output, "output"); _cuda_bf16(weight, "weight")
    _need(input.stride(-1) == 1, "input last dim must be contiguous")
    H = input.size(-1)
    x2 = input.reshape(-1, H) if input.dim() != 2 else input
    _need(output.is_contiguous(), "output must be contiguous")
    check(lib().xb_rms_norm_bf16(_p(output), _p(x2), c_i64(x2.stride(0)), _p(weight), c_f32(eps),
                                 c_i32(x2.size(0)), c_i32(H), _stream()), "rms_norm")


def fused_add_rms_norm(input: torch.Tensor, residual: torch.Tensor, weight: torch.Tensor, epsilon: float) -> None:
    """cuda_ops_api.h:162-165 / norm.cu:462-515: in place on input and residual."""
    _cuda_bf16(input, "input"); _cuda_bf16(residual, "residual"); _cuda_bf16(weight, "weight")
    _need(input.stride(-1) == 1 and residual.is_contiguous(), "input/residual layout")
    H = input.size(-1)
    T = input.numel() // H
    stride = input.stride(-2) if input.dim() >= 2 else H
    check(lib().xb_fused_add_rms_norm_bf16(_p(input), c_i64(stride), _p(residual), _p(weight), c_f32(epsilon),
                                           c_i32(T), c_i32(H), _stream()), "fused_add_rms_norm")


# ---- K8 ---------------------------------------------------------------------
def rms_norm_static_fp8_quant(out, input, weight, scale, epsilon) -> None:
    """cuda_ops_api.h:203-209."""
    _cuda_bf16(input, "input"); _need(out.dtype == E4M3 and out.is_contiguous(), "out must be contiguous e4m3")
    H = input.size(-1)
    T = input.numel() // H
    check(lib().xb_rms_norm_static_fp8_quant_bf16(_p(out), _p(input), c_i64(input.stride(-2) if input.dim() >= 2 else H),
                                                  _p(weight), _p(scale), c_f32(epsilon), c_i32(T), c_i32(H), _stream()),
          "rms_norm_static_fp8_quant")


def fused_add_rms_norm_static_fp8_quant(out, input, residual, weight, scale, epsilon) -> None:
    """cuda_ops_api.h:214-221."""
    _cuda_bf16(input, "input"); _cuda_bf16(residual, "residual")
    _need(out.dtype == E4M3 and out.is_contiguous(), "out must be contiguous e4m3")
    H = input.size(-1)
    T = input.numel() // H
    check(lib().xb_fused_add_rms_norm_static_fp8_quant_bf16(
        _p(out), _p(input), c_i64(input.stride(-2) if input.dim() >= 2 else H), _p(residual), _p(weight), _p(scale),
        c_f32(epsilon), c_i32(T), c_i32(H), _stream()), "fused_add_rms_norm_static_fp8_quant")


# ---- K6 ---------------------------------------------------------------------
def static_scaled_fp8_quant(out, input, scale) -> None:
    """cuda_ops_api.h:182-186 / fp8_quant.cu:114-153."""
    _cuda_bf16(input, "input")
    _need(input.stride(-1) == 1, "last dimension of input must be contiguous")
    _need(out.stride(-1) == 1, "last dimension of output must be contiguous")
    H = input.size(-1)
    T = input.numel() // H
    check(lib().xb_static_scaled_fp8_quant_bf16(_p(out), c_i64(out.stride(-2) if out.dim() >= 2 else H), _p(input),
                                                c_i64(input.stride(-2) if input.dim() >= 2 else H), _p(scale),
                                                c_i32(T), c_i32(H), _stream()), "static_scaled_fp8_quant")


def fp8_scaled_quantize(input, output=None, scale=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """cuda_ops_api.h:188-193 / fp8_scaled_quantize.cpp:20-48.  Dynamic scale is computed on device (no host sync)."""
    out = output if output is not None else torch.empty_like(input, dtype=E4M3)
    if scale is not None:
        static_scaled_fp8_quant(out, input, scale)
        return out, scale
    _cuda_bf16(input, "input")
    s = torch.empty(1, dtype=torch.float32, device=input.device)
    H = input.size(-1)
    T = input.numel() // H
    check(lib().xb_dynamic_scaled_fp8_quant_bf16(_p(out), c_i64(out.stride(-2) if out.dim() >= 2 else H), _p(input),
                                                 c_i64(input.stride(-2) if input.dim() >= 2 else H), _p(s), c_i32(T),
                                                 c_i32(H), _stream()), "fp8_scaled_quantize")
    return out, s


# ---- K9 ---------------------------------------------------------------------
def rotary_embedding(positions, query, key, cos_sin_cache, is_neox: bool) -> None:
    """cuda_ops_api.h:31-37 / rope.cu:156-250: in place; positions int64 [T]; query [T, Hq*D] or [T, Hq, D]."""
    _cuda_bf16(query, "query"); _cuda_bf16(cos_sin_cache, "cos_sin_cache")
    _need(positions.dtype == torch.int64, "positions must be int64 (forward_params.h:200-206)")
    head_size = cos_sin_cache.size(-1)
    T = positions.numel()
    _need(query.size(0) == T and (key is None or key.size(0) == T),
          "query, key and positions must have the same number of tokens")
    qh = query.numel() // T
    kh = key.numel() // T if key is not None else 0
    _need(qh % head_size == 0 and kh % head_size == 0, "hidden size must be a multiple of head_size")
    nh, nkv = qh // head_size, (kh // head_size if key is not None else qh // head_size)
    _need(nh % nkv == 0, "num_heads must be a multiple of num_kv_heads")
    head_stride = query.stride(-2) if query.dim() == 3 else head_size
    check(lib().xb_rotary_embedding_bf16(_p(positions), _p(query), _p(key), _p(cos_sin_cache),
                                         c_i32(cos_sin_cache.size(1)), c_i64(query.stride(0)),
                                         c_i64(key.stride(0) if key is not None else 0), c_i64(head_stride), c_i32(nh),
                                         c_i32(nkv), c_i32(head_size), c_i32(1 if is_neox else 0), c_i32(T), _stream()),
          "rotary_embedding")


# ---- K12 --------------------------------------------------------------------
def reshape_paged_cache(slot_ids, keys, values, key_cache, value_cache) -> None:
    """cuda_ops_api.h:44-49 / reshape_paged_cache.cu:64-99."""
    _cuda_bf16(keys, "keys"); _cuda_bf16(values, "values"); _cuda_bf16(key_cache, "key_cache")
    _need(slot_ids.dtype == torch.int32, "slot_ids must be int32")
    _need(keys.stride(-1) == 1 and keys.stride(-2) == keys.size(-1), "keys must be contiguous in (heads, dim)")
    _need(values.stride(-1) == 1 and values.stride(-2) == values.size(-1), "values must be contiguous in (heads, dim)")
    _need(key_cache.is_contiguous() and value_cache.is_contiguous(), "caches must be contiguous")
    T, Hkv, D = keys.size(-3), keys.size(-2), keys.size(-1)
    check(lib().xb_reshape_paged_cache_bf16(_p(slot_ids), _p(keys), _p(values), _p(key_cache), _p(value_cache),
                                            c_i64(keys.stride(-3)), c_i64(values.stride(-3)), c_i32(Hkv), c_i32(D),
                                            c_i32(key_cache.size(-3)), c_i32(T), _stream()), "reshape_paged_cache")


def rope_and_cache(positions, query, key, value, cos_sin_cache, slot_ids, key_cache, value_cache, is_neox=True) -> None:
    """Fused K9+K12 (one launch); bit-identical to rotary_embedding + reshape_paged_cache."""
    _cuda_bf16(query, "query"); _cuda_bf16(key, "key"); _cuda_bf16(value, "value")
    _need(positions.dtype == torch.int64 and slot_ids.dtype == torch.int32, "positions int64 / slot_ids int32")
    D = key_cache.size(-1)
    T = positions.numel()
    nh, nkv = query.numel() // T // D, key.numel() // T // D
    check(lib().xb_rope_and_cache_bf16(_p(positions), _p(query), _p(key), _p(value), _p(cos_sin_cache), _p(slot_ids),
                                       _p(key_cache), _p(value_cache), c_i32(cos_sin_cache.size(1)),
                                       c_i64(query.stride(0)), c_i64(key.stride(0)), c_i64(value.stride(0)), c_i32(nh),
                                       c_i32(nkv), c_i32(D), c_i32(key_cache.size(-3)), c_i32(1 if is_neox else 0),
                                       c_i32(T), _stream()), "rope_and_cache")


# ---- K10 --------------------------------------------------------------------
def fused_qk_norm_rope(qkv, num_heads_q, num_heads_k, num_heads_v, head_dim, eps, q_weight, k_weight, cos_sin_cache,
                       interleaved, position_ids) -> None:
    """cuda_ops_api.h:252-266 / fused_qknorm_rope.cu:388-471."""
    _cuda_bf16(qkv, "qkv")
    _need(qkv.is_contiguous(), "qkv must be contiguous")
    _need(position_ids.dtype == torch.int64, "position_ids must be int64")
    T = qkv.size(0)
    check(lib().xb_fused_qk_norm_rope_bf16(_p(qkv), c_i32(num_heads_q), c_i32(num_heads_k), c_i32(num_heads_v),
                                           c_i32(head_dim), c_f32(eps), _p(q_weight), _p(k_weight), _p(cos_sin_cache),
                                           c_i32(cos_sin_cache.size(-1)), c_i32(1 if interleaved else 0),
                                           _p(position_ids), c_i32(T), _stream()), "fused_qk_norm_rope")


def qk_norm_rope_and_cache(qkv, num_heads_q, num_heads_kv, head_dim, eps, q_weight, k_weight, cos_sin_cache, position_ids,
                           slot_ids, key_cache, value_cache) -> None:
    """Fused K10+K12 (one launch): per-head RMSNorm + NeoX RoPE of q and k in place in qkv [T, (Hq+2Hkv)*D], then the new
    k and v rows into the paged caches (slot < 0 skipped); bit-identical to fused_qk_norm_rope + reshape_paged_cache."""
    _cuda_bf16(qkv, "qkv"); _cuda_bf16(key_cache, "key_cache"); _cuda_bf16(value_cache, "value_cache")
    _need(qkv.is_contiguous(), "qkv must be contiguous")
    _need(key_cache.is_contiguous() and value_cache.is_contiguous(), "caches must be contiguous")
    _need(position_ids.dtype == torch.int64, "position_ids must be int64")
    _need(slot_ids.dtype == torch.int32, "slot_ids must be int32")
    _need(cos_sin_cache.size(-1) == head_dim, "full rotary only (cos_sin_cache rows of head_dim)")
    T = qkv.size(0)
    check(lib().xb_qk_norm_rope_and_cache_bf16(_p(qkv), c_i32(num_heads_q), c_i32(num_heads_kv), c_i32(head_dim), c_f32(eps),
                                               _p(q_weight), _p(k_weight), _p(cos_sin_cache), _p(position_ids),
                                               _p(slot_ids), _p(key_cache), _p(value_cache), c_i32(T), _stream()),
          "qk_norm_rope_and_cache")


# ---- K11 --------------------------------------------------------------------
_ACT = {"silu": 0, "gelu": 1, "gelu_tanh": 2, "gelu_pytorch_tanh": 2}


def act_and_mul(out, input, act_mode: str) -> None:
    """cuda_ops_api.h:39-42 / activation.cu:158-186."""
    if act_mode not in _ACT:
        raise XllmB200Error(f"Unsupported act mode: {act_mode}, only support silu, gelu, gelu_tanh, gelu_pytorch_tanh")
    _cuda_bf16(input, "input"); _cuda_bf16(out, "out")
    _need(input.is_contiguous() and out.is_contiguous(), "act_and_mul tensors must be contiguous")
    d = input.size(-1) // 2
    T = input.numel() // input.size(-1)
    check(lib().xb_act_and_mul_bf16(_p(out), _p(input), c_i32(d), c_i32(T), c_i32(_ACT[act_mode]), _stream()),
          "act_and_mul")


# ---- K1: paged decode attention ------------------------------------------------
class DecodePlan:
    """Opaque plan (the reference deep-copies FlashInfer's plan_info: flashinfer_planinfo.cpp:37-62)."""

    def __init__(self, batch, num_qo_heads, num_kv_heads, head_dim, page_size, max_pages_per_request, device,
                 num_sms: Optional[int] = None, early_prefetch: bool = False):
        if num_sms is None:
            num_sms = torch.cuda.get_device_properties(device).multi_processor_count
        self.arr = (ctypes.c_int64 * 8)()
        check(lib().xb_decode_plan(self.arr, c_i32(batch), c_i32(num_qo_heads), c_i32(num_kv_heads), c_i32(head_dim),
                                   c_i32(page_size), c_i32(max_pages_per_request), c_i32(num_sms)), "decode_plan")
        # the shapes batch_decode's tensors must have: query / output, and a cache without its block dimension
        self.q_shape = (batch, num_qo_heads, head_dim)
        self.page_shape = (page_size, num_kv_heads, head_dim)
        # chunk_tokens: nominal split size at the planned maximum context (the kernel derives the live one on the device);
        # max_splits: splits launched per (request, kv head) = clusters x cluster size
        self.chunk_tokens, self.max_splits = int(self.arr[0]), int(self.arr[1])
        self.cluster = int(self.arr[7] >> 44) & 0x1F
        self.float_ws = torch.empty(int(self.arr[2]), dtype=torch.uint8, device=device)
        self.int_ws = torch.zeros(int(self.arr[3]) & 0xFFFFFFFF, dtype=torch.uint8, device=device)
        if early_prefetch:
            # only inside a decode step: nothing in flight writes old KV rows or the paged triplet
            check(lib().xb_decode_plan_set_flags(self.arr, c_i32(1)), "decode_plan_set_flags")


def batch_decode(plan: DecodePlan, query, k_cache, v_cache, paged_kv_indptr, paged_kv_indices,
                 paged_kv_last_page_len, sm_scale: float, output, output_lse=None) -> None:
    """xllm::kernel::cuda::batch_decode (cuda_ops_api.h:130-147, batch_decode.cpp:26-86), NHD layout.
    query/output [B, Hq, D]; caches [n_blocks, block_size, Hkv, D]."""
    _cuda_bf16(query, "query"); _cuda_bf16(k_cache, "k_cache"); _cuda_bf16(v_cache, "v_cache"); _cuda_bf16(output, "output")
    for t, n in ((paged_kv_indptr, "paged_kv_indptr"), (paged_kv_indices, "paged_kv_indices"),
                 (paged_kv_last_page_len, "paged_kv_last_page_len")):
        _need(t.dtype == torch.int32 and t.is_cuda, f"{n} must be int32 on device")
    # The kernel takes the plan's geometry and one set of strides for both caches: anything else would be read with the
    # wrong layout, or past the end of a tensor, without an error.  (Messages are formatted only on failure: this runs
    # once per layer and step.)
    if query.shape != plan.q_shape or output.shape != plan.q_shape:
        raise XllmB200Error(f"query {tuple(query.shape)} and output {tuple(output.shape)} must be "
                            f"[batch, num_qo_heads, head_dim] = {list(plan.q_shape)} of the plan")
    if k_cache.shape[1:] != plan.page_shape or v_cache.shape != k_cache.shape:
        raise XllmB200Error(f"k_cache {tuple(k_cache.shape)} and v_cache {tuple(v_cache.shape)} must be [blocks, page_size, "
                            f"num_kv_heads, head_dim] with [page_size, num_kv_heads, head_dim] = {list(plan.page_shape)} "
                            "of the plan")
    kv_stride = k_cache.stride()
    if v_cache.stride() != kv_stride:
        raise XllmB200Error(f"v_cache strides {v_cache.stride()} differ from k_cache strides {kv_stride}")
    _need(query.stride(2) == 1 and output.stride(2) == 1 and kv_stride[3] == 1,
          "the last dimension of query, output and the caches must be unit-stride")
    check(lib().xb_paged_decode_bf16(plan.arr, _p(query), c_i64(query.stride(0)), c_i64(query.stride(1)), _p(k_cache),
                                     _p(v_cache), c_i64(kv_stride[0]), c_i64(kv_stride[1]),
                                     c_i64(kv_stride[2]), _p(paged_kv_indptr), _p(paged_kv_indices),
                                     _p(paged_kv_last_page_len), _p(output), c_i64(output.stride(0)),
                                     c_i64(output.stride(1)), _p(output_lse), c_f32(sm_scale), _p(plan.float_ws),
                                     _p(plan.int_ws), _stream()), "batch_decode")


# ---- MLA (DeepSeek-V2/V3): latent cache writer + paged absorbed attention --------
MLA_KV_LORA_RANK = 512
MLA_ROPE_DIM = 64


def mla_cache_latent(latent, gamma, eps: float, positions, cos_sin_cache, slot_ids, ckv_cache, kpe_cache,
                     interleaved: bool = True) -> None:
    """fused_mla_kv (kernels/param.h:1105-1180), quant_mode "none", CUDA two-cache layout: ckv_cache[slot] =
    rms_norm(latent[:, :512], gamma), kpe_cache[slot] = rope(latent[:, 512:]); slot < 0 skipped.
    latent [T, 576] (row stride allowed); caches [pages, page_size, 512] / [pages, page_size, 64] (or with a
    singleton kv-head dim)."""
    for t, n in ((latent, "latent"), (gamma, "gamma"), (cos_sin_cache, "cos_sin_cache"), (ckv_cache, "ckv_cache"),
                 (kpe_cache, "kpe_cache")):
        _cuda_bf16(t, n)
    _need(positions.dtype == torch.int64 and slot_ids.dtype == torch.int32, "positions int64 / slot_ids int32")
    _need(latent.dim() == 2 and latent.stride(1) == 1, "latent must be [T, 576] with unit column stride")
    T = latent.size(0)
    _need(positions.numel() == T and slot_ids.numel() == T, "positions / slot_ids need one entry per latent row")
    ckv, kpe = ckv_cache.reshape(ckv_cache.size(0), ckv_cache.size(1), -1), kpe_cache.reshape(kpe_cache.size(0), kpe_cache.size(1), -1)
    _need(ckv.stride(2) == 1 and kpe.stride(2) == 1, "cache rows must be contiguous")
    _need(latent.size(1) == ckv.size(2) + kpe.size(2) and cos_sin_cache.size(-1) == kpe.size(2),
          "latent must be [T, kv_lora_rank + rope_dim], cos_sin_cache [max_pos, rope_dim]")
    check(lib().xb_mla_cache_latent_bf16(_p(latent), c_i64(latent.stride(0)), _p(gamma), c_f32(eps), _p(positions),
                                         _p(cos_sin_cache), c_i32(1 if interleaved else 0), _p(slot_ids), _p(ckv),
                                         c_i64(ckv.stride(0)), c_i64(ckv.stride(1)), _p(kpe), c_i64(kpe.stride(0)),
                                         c_i64(kpe.stride(1)), c_i32(ckv.size(2)), c_i32(kpe.size(2)), c_i32(ckv.size(1)), c_i32(T), _stream()),
          "mla_cache_latent")


class MlaPlan:
    """Host-only plan of mla_paged_attention (split count + workspace); valid for any later context length."""

    def __init__(self, batch, num_heads, max_qo_len, page_size, max_pages_per_request, device,
                 num_sms: Optional[int] = None, splits: Optional[int] = None):
        if num_sms is None:
            num_sms = torch.cuda.get_device_properties(device).multi_processor_count
        self.arr = (ctypes.c_int64 * 8)()
        check(lib().xb_mla_plan(self.arr, c_i32(batch), c_i32(num_heads), c_i32(MLA_KV_LORA_RANK), c_i32(MLA_ROPE_DIM),
                                c_i32(max_qo_len), c_i32(page_size), c_i32(max_pages_per_request), c_i32(num_sms)),
              "mla_plan")
        if splits is not None:
            check(lib().xb_mla_plan_set_splits(self.arr, c_i32(splits)), "mla_plan_set_splits")
        self.splits, self.workspace_bytes = int(self.arr[0]), int(self.arr[1])
        self.workspace = torch.empty(max(self.workspace_bytes, 16), dtype=torch.uint8, device=device)


def mla_paged_attention(plan: MlaPlan, q_nope, q_pe, ckv_cache, kpe_cache, qo_indptr, paged_kv_indptr, paged_kv_indices,
                        paged_kv_last_page_len, sm_scale: float, output, causal: bool = True) -> None:
    """Absorbed MLA over the paged latent caches: q_nope [T, H, 512], q_pe [T, H, 64] (separate strides: split tensors
    or views of a packed [T, H, 576] q_input), output [T, H, 512]."""
    for t, n in ((q_nope, "q_nope"), (q_pe, "q_pe"), (ckv_cache, "ckv_cache"), (kpe_cache, "kpe_cache"), (output, "output")):
        _cuda_bf16(t, n)
    for t, n in ((qo_indptr, "qo_indptr"), (paged_kv_indptr, "paged_kv_indptr"), (paged_kv_indices, "paged_kv_indices"),
                 (paged_kv_last_page_len, "paged_kv_last_page_len")):
        _need(t.dtype == torch.int32 and t.is_cuda, f"{n} must be int32 on device")
    _need(q_nope.dim() == 3 and q_pe.dim() == 3 and output.dim() == 3, "q_nope / q_pe / output must be [T, H, D]")
    _need(q_nope.size(2) == MLA_KV_LORA_RANK and q_pe.size(2) == MLA_ROPE_DIM and output.size(2) == MLA_KV_LORA_RANK,
          "MLA dims are kv_lora_rank 512 / qk_rope_head_dim 64")
    _need(q_nope.stride(2) == 1 and q_pe.stride(2) == 1 and output.stride(2) == 1, "last dims must be contiguous")
    ckv, kpe = ckv_cache.reshape(ckv_cache.size(0), ckv_cache.size(1), -1), kpe_cache.reshape(kpe_cache.size(0), kpe_cache.size(1), -1)
    _need(ckv.stride(2) == 1 and kpe.stride(2) == 1, "cache rows must be contiguous")
    check(lib().xb_mla_paged_attention_bf16(
        plan.arr, _p(q_nope), c_i64(q_nope.stride(0)), c_i64(q_nope.stride(1)), _p(q_pe), c_i64(q_pe.stride(0)),
        c_i64(q_pe.stride(1)), _p(ckv), c_i64(ckv.stride(0)), c_i64(ckv.stride(1)), _p(kpe), c_i64(kpe.stride(0)),
        c_i64(kpe.stride(1)), _p(qo_indptr), _p(paged_kv_indptr), _p(paged_kv_indices), _p(paged_kv_last_page_len),
        c_i32(1 if causal else 0), _p(output), c_i64(output.stride(0)), c_i64(output.stride(1)), c_f32(sm_scale),
        _p(plan.workspace), c_i64(plan.workspace.numel()), _stream()), "mla_paged_attention")


MLA_UP_HEAD_DIM = 256          # kv_b_proj rows per head: qk_nope_head_dim 128 | v_head_dim 128


class MlaExpandedPlan:
    """Host-only plan of one MLA prefill step from its host-side lengths (qo_lens: the step's q tokens, kv_lens: history +
    the step's tokens).  `.expanded` is the form the step should take (mla_prefill_expanded when True, the absorbed
    mla_paged_attention otherwise); `.workspace` is allocated only for the expanded form."""

    def __init__(self, num_heads, qo_lens, kv_lens, device):
        qo = (ctypes.c_int32 * len(qo_lens))(*qo_lens)
        kv = (ctypes.c_int32 * len(kv_lens))(*kv_lens)
        _need(len(qo_lens) == len(kv_lens), "qo_lens and kv_lens need one entry per request")
        self.arr = (ctypes.c_int64 * 8)()
        check(lib().xb_mla_expanded_plan(self.arr, c_i32(len(qo_lens)), c_i32(num_heads), qo, kv), "mla_expanded_plan")
        self.expanded = bool(self.arr[0])
        self.workspace_bytes, self.total_kv, self.num_heads = int(self.arr[1]), int(self.arr[5]), num_heads
        self.total_q = int(self.arr[7]) & ((1 << 40) - 1)
        self.workspace = torch.empty(self.workspace_bytes, dtype=torch.uint8, device=device) if self.expanded else None


def mla_prefill_expanded(plan: MlaExpandedPlan, q, ckv_cache, kpe_cache, qo_indptr, paged_kv_indptr, paged_kv_indices,
                         paged_kv_last_page_len, kv_b_proj, sm_scale: float, output, workspace=None) -> None:
    """Expanded MLA prefill (causal): q [T, H, 192] = [q_nope | roped q_pe], caches as in mla_paged_attention, kv_b_proj
    [H * 256, 512], output [T, H, 128] (o_proj's input).  workspace: plan.workspace unless given (at least
    plan.workspace_bytes, layout in include/xllm_b200_ops.h)."""
    ws = plan.workspace if workspace is None else workspace
    _need(ws is not None, "mla_prefill_expanded: the plan chose the absorbed form and holds no workspace; pass one")
    for t, n in ((q, "q"), (ckv_cache, "ckv_cache"), (kpe_cache, "kpe_cache"), (kv_b_proj, "kv_b_proj"), (output, "output")):
        _cuda_bf16(t, n)
    for t, n in ((qo_indptr, "qo_indptr"), (paged_kv_indptr, "paged_kv_indptr"), (paged_kv_indices, "paged_kv_indices"),
                 (paged_kv_last_page_len, "paged_kv_last_page_len")):
        _need(t.dtype == torch.int32 and t.is_cuda, f"{n} must be int32 on device")
    H = plan.num_heads
    _need(q.dim() == 3 and q.size(1) == H and q.size(2) == 128 + MLA_ROPE_DIM and q.stride(2) == 1,
          f"q must be [T, {H}, 192] with contiguous rows")
    _need(output.dim() == 3 and output.size(1) == H and output.size(2) == 128 and output.stride(2) == 1,
          f"output must be [T, {H}, 128] with contiguous rows")
    # the kernels read plan.total_q rows of q and write the rows qo_indptr names into output
    _need(q.size(0) == plan.total_q and output.size(0) == plan.total_q,
          f"q and output need the plan's {plan.total_q} tokens (got {q.size(0)} / {output.size(0)})")
    _need(tuple(kv_b_proj.shape) == (H * MLA_UP_HEAD_DIM, MLA_KV_LORA_RANK) and kv_b_proj.is_contiguous(),
          f"kv_b_proj must be a contiguous [{H * MLA_UP_HEAD_DIM}, {MLA_KV_LORA_RANK}] weight")
    ckv, kpe = ckv_cache.reshape(ckv_cache.size(0), ckv_cache.size(1), -1), kpe_cache.reshape(kpe_cache.size(0), kpe_cache.size(1), -1)
    _need(ckv.size(2) == MLA_KV_LORA_RANK and kpe.size(2) == MLA_ROPE_DIM and ckv.stride(2) == 1 and kpe.stride(2) == 1,
          "caches must be [pages, page_size, 512] / [pages, page_size, 64] with contiguous rows")
    _need(ws.is_cuda and ws.numel() * ws.element_size() >= plan.workspace_bytes, "workspace is smaller than the plan's")
    check(lib().xb_mla_prefill_expanded_bf16(
        plan.arr, _p(q), c_i64(q.stride(0)), c_i64(q.stride(1)), _p(ckv), c_i64(ckv.stride(0)), c_i64(ckv.stride(1)),
        _p(kpe), c_i64(kpe.stride(0)), c_i64(kpe.stride(1)), c_i32(ckv.size(1)), _p(paged_kv_indptr), _p(paged_kv_indices),
        _p(paged_kv_last_page_len), _p(qo_indptr), _p(kv_b_proj), _p(output), c_i64(output.stride(0)),
        c_i64(output.stride(1)), c_f32(sm_scale), _p(ws), c_i64(ws.numel() * ws.element_size()), _stream()),
        "mla_prefill_expanded")


# ---- linears ------------------------------------------------------------------
def matmul_small_m(a, b, bias=None, out=None):
    """xllm::kernel::cuda::matmul (cuda_ops_api.h:167-169, matmul.cpp:20-24) for M <= 64: a [M,K], b [N,K]."""
    _cuda_bf16(a, "a"); _cuda_bf16(b, "b")
    M, K = a.shape
    N = b.size(0)
    _need(b.is_contiguous() and a.stride(1) == 1, "a/b layout")
    y = out if out is not None else torch.empty(M, N, dtype=BF16, device=a.device)
    check(lib().xb_linear_bf16_small_m(_p(y), c_i64(y.stride(0)), _p(a), c_i64(a.stride(0)), _p(b), _p(bias), c_i32(M),
                                       c_i32(N), c_i32(K), _stream()), "matmul_small_m")
    return y


def w4a16_linear_small_m(x, qweight, meta, group_size, bias=None, out=None):
    """additive boundary (SURVEY 8b-3): y = x . dequant(W)^T (+bias), M <= 64.  qweight/meta from quant.pack_w4."""
    _cuda_bf16(x, "x")
    _need(qweight.dtype == torch.int32 and meta.dtype == torch.int32, "qweight/meta must be int32 storage")
    M, K = x.shape
    N = meta.size(1)
    y = out if out is not None else torch.empty(M, N, dtype=BF16, device=x.device)
    check(lib().xb_linear_w4a16_small_m(_p(y), c_i64(y.stride(0)), _p(x), c_i64(x.stride(0)), _p(qweight), _p(meta),
                                        _p(bias), c_i32(M), c_i32(N), c_i32(K), c_i32(group_size), _stream()),
          "w4a16_linear_small_m")
    return y


# ---- step boundary -------------------------------------------------------------
def embedding(out, token_ids, table) -> None:
    """WordEmbeddingImpl::forward (word_embedding_impl.cpp:33-56), TP=1."""
    _cuda_bf16(table, "table"); _cuda_bf16(out, "out")
    _need(token_ids.dtype == torch.int32, "token_ids must be int32")
    check(lib().xb_embedding_bf16(_p(out), _p(token_ids), _p(table), c_i32(token_ids.numel()), c_i32(table.size(1)),
                                  c_i32(table.size(0)), _stream()), "embedding")


def update_llm_decode_metadata(src: dict, dst: dict, actual_num_tokens: int, padded_num_tokens: int, actual_batch_size: int,
                               actual_indices_size: int, plan_counters=None) -> None:
    """xllm::kernel::cuda::update_llm_decode_metadata (llm_decode_metadata_update.h:35-58): src / dst are dicts of int32
    CUDA tensors with the fields of LlmDecodeMetadataUpdateParams (src: tokens, positions, new_cache_slots, kv_seq_lens,
    paged_kv_indptr, paged_kv_indices, paged_kv_last_page_len; dst: the same + kv_seq_lens_delta).  plan_counters: optional
    int32 workspace of a DecodePlan to re-zero in the same launch."""
    for d in (src, dst):
        for k, t in d.items():
            _need(t.is_cuda and t.dtype == torch.int32 and t.is_contiguous(), f"{k} must be a contiguous int32 CUDA tensor")
    nc = plan_counters.numel() if plan_counters is not None else 0
    check(lib().xb_decode_metadata_update(
        _p(src["tokens"]), _p(src["positions"]), _p(src["new_cache_slots"]), _p(src["kv_seq_lens"]), _p(src["paged_kv_indptr"]),
        _p(src["paged_kv_indices"]), _p(src["paged_kv_last_page_len"]), _p(dst["tokens"]), _p(dst["positions"]),
        _p(dst["new_cache_slots"]), _p(dst["kv_seq_lens"]), _p(dst["kv_seq_lens_delta"]), _p(dst["paged_kv_indptr"]),
        _p(dst["paged_kv_indices"]), _p(dst["paged_kv_last_page_len"]), c_i64(actual_num_tokens), c_i64(padded_num_tokens),
        c_i64(actual_batch_size), c_i64(actual_indices_size), _p(plan_counters), c_i64(nc), _stream()),
        "update_llm_decode_metadata")


def argmax(out, logits) -> None:
    """greedy sampling: out int32 [rows]."""
    _cuda_bf16(logits, "logits")
    _need(out.dtype == torch.int32, "out must be int32")
    check(lib().xb_argmax_bf16(_p(out), _p(logits), c_i64(logits.stride(0)), c_i32(logits.size(0)),
                               c_i32(logits.size(1)), _stream()), "argmax")


# ---- wgmma GEMMs ---------------------------------------------------------------
def matmul(a, b, bias=None, out=None):
    """xllm::kernel::cuda::matmul (cuda_ops_api.h:167-169): F::linear(a, b, bias); a [M,K], b [N,K] bf16.
    M <= 16 streams the weight once through the small-M kernel; larger M runs the wgmma GEMM."""
    _cuda_bf16(a, "a"); _cuda_bf16(b, "b")
    M, K = a.shape
    N = b.size(0)
    _need(b.is_contiguous() and a.stride(1) == 1, "a/b layout")
    y = out if out is not None else torch.empty(M, N, dtype=BF16, device=a.device)
    if M <= 16 and K % 32 == 0:
        return matmul_small_m(a, b, bias, y)
    check(lib().xb_gemm_bf16(_p(y), c_i64(y.stride(0)), _p(a), c_i64(a.stride(0)), _p(b), _p(bias), c_i32(M), c_i32(N),
                             c_i32(K), _stream()), "matmul")
    return y


def set_fp8_swap_max_m(max_m: int) -> int:
    """largest M for which xb_gemm_fp8_scaled runs swap-AB (weight rows in the MMA M slot); 0 = never.  Returns the old value."""
    return int(lib().xb_set_fp8_swap_max_m(c_i32(max_m)))


_splitk_ws = None


def enable_fp8_splitk(device=None) -> None:
    """register a split-K workspace for the decode-sized (swap-AB) FP8 GEMMs (xb_set_gemm_splitk_workspace); idempotent.  The
    buffer lives as long as the process (the library keeps the pointer)."""
    global _splitk_ws
    if _splitk_ws is not None:
        return
    import ctypes
    L = lib()
    L.xb_gemm_splitk_workspace_bytes.restype = ctypes.c_size_t
    n = int(L.xb_gemm_splitk_workspace_bytes())
    ws = torch.empty(n, dtype=torch.uint8, device=device if device is not None else torch.cuda.current_device())
    check(L.xb_set_gemm_splitk_workspace(_p(ws), ctypes.c_size_t(n)), "set_gemm_splitk_workspace")
    _splitk_ws = ws


def disable_fp8_splitk() -> None:
    global _splitk_ws
    import ctypes
    check(lib().xb_set_gemm_splitk_workspace(None, ctypes.c_size_t(0)), "set_gemm_splitk_workspace")
    _splitk_ws = None


def set_fp8_splitk_max(max_split: int) -> int:
    return int(lib().xb_set_fp8_splitk_max(c_i32(max_split)))


def gemm_fp8_scaled(c, a, w, a_scales, b_scales, bias=None) -> None:
    """the wgmma FP8 kernel directly (no small-M dispatch): a [M,K] e4m3, w [N,K] e4m3 (the reference's weight layout)."""
    M, K = a.shape
    N = w.size(0)
    check(lib().xb_gemm_fp8_scaled(_p(c), c_i64(c.stride(0)), _p(a), c_i64(a.stride(0)), _p(w), _p(a_scales),
                                   c_i32(a_scales.numel()), _p(b_scales), c_i32(b_scales.numel()), _p(bias), c_i32(M),
                                   c_i32(N), c_i32(K), _stream()), "gemm_fp8_scaled")


def gemm_bf16(a, b, bias=None, out=None):
    """always the wgmma kernel (tests / benchmarks)."""
    _cuda_bf16(a, "a"); _cuda_bf16(b, "b")
    M, K = a.shape
    N = b.size(0)
    y = out if out is not None else torch.empty(M, N, dtype=BF16, device=a.device)
    check(lib().xb_gemm_bf16(_p(y), c_i64(y.stride(0)), _p(a), c_i64(a.stride(0)), _p(b), _p(bias), c_i32(M), c_i32(N),
                             c_i32(K), _stream()), "gemm_bf16")
    return y


def cutlass_scaled_mm(c, a, b, a_scales, b_scales, bias=None) -> None:
    """xllm::kernel::cuda::cutlass_scaled_mm (cuda_ops_api.h:171-176): c [M,N] bf16 = a_s * b_s * (a @ b) + bias with
    a [M,K] e4m3 row-major and b [K,N] e4m3 COLUMN-major (the reference passes weight.t(): fp8_scaled_matmul.cpp:20-45)."""
    _need(a.dtype == E4M3 and b.dtype == E4M3, "a and b must be float8_e4m3fn")
    _need(c.dtype == BF16, "c must be bfloat16")
    _need(a.dim() == 2 and b.dim() == 2 and c.dim() == 2, "2-D tensors expected")
    _need(c.size(0) == a.size(0) and a.size(1) == b.size(0) and b.size(1) == c.size(1), "shape mismatch")
    _need(a.stride(1) == 1 and c.stride(1) == 1, "a and c must be row major")
    _need(b.stride(0) == 1, "b must be column major")
    _need(c.stride(0) % 16 == 0 and b.stride(1) % 16 == 0, "row strides must be multiples of 16")
    _need(a_scales.is_contiguous() and b_scales.is_contiguous(), "scales must be contiguous")
    _need(a_scales.dtype == torch.float32 and b_scales.dtype == torch.float32, "scales must be float32")
    M, K = a.shape
    N = b.size(1)
    _need(b.stride(1) == K, "b must be a dense column-major [K,N] view of a [N,K] weight")
    _need(a_scales.numel() in (1, M) and b_scales.numel() in (1, N), "scale numel must be 1 or M / N")
    if bias is not None:
        _need(bias.numel() == N and bias.is_contiguous() and bias.dim() == 1 and bias.dtype == BF16, "bias must be [N] bf16")
    if M <= FP8_SMALL_M_MAX and N <= SMALL_N_MAX and K % 64 == 0:
        return fp8_scaled_mm_small_m(c, a, b, a_scales, b_scales, bias)
    check(lib().xb_gemm_fp8_scaled(_p(c), c_i64(c.stride(0)), _p(a), c_i64(a.stride(0)), _p(b), _p(a_scales),
                                   c_i32(a_scales.numel()), _p(b_scales), c_i32(b_scales.numel()), _p(bias), c_i32(M),
                                   c_i32(N), c_i32(K), _stream()), "cutlass_scaled_mm")


def fp8_scaled_mm_small_m(c, a, b, a_scales, b_scales, bias=None) -> None:
    """the streaming swap-AB form of cutlass_scaled_mm for M <= 64 (same arguments: b is the [K, N] column-major view of
    the [N, K] weight): weights streamed once, tokens in the n8 slot of mma.sync e4m3 (the reference's M <= 16 / <= 64
    buckets, scaled_mm_sm100_fp8_dispatch.cuh:148-287)."""
    M, K = a.shape
    N = b.size(1)
    _need(b.stride(0) == 1 and b.stride(1) == K, "b must be a dense column-major [K,N] view of a [N,K] weight")
    check(lib().xb_linear_fp8_small_m(_p(c), c_i64(c.stride(0)), _p(a), c_i64(a.stride(0)), _p(b), _p(a_scales),
                                      c_i32(a_scales.numel()), _p(b_scales), c_i32(b_scales.numel()), _p(bias),
                                      c_i32(M), c_i32(N), c_i32(K), _stream()), "fp8_scaled_mm_small_m")


def fp8_scaled_matmul(a, b, a_scale, b_scale, output_dtype=BF16, bias=None, output=None):
    """xllm::kernel::cuda::fp8_scaled_matmul (cuda_ops_api.h:223-233, fp8_scaled_matmul.cpp:20-45): b is the [N,K] weight."""
    _need(output_dtype == BF16, "only bfloat16 output is implemented")
    M, N = a.size(0), b.size(0)
    out = output if output is not None else torch.empty(M, N, dtype=BF16, device=a.device)
    cutlass_scaled_mm(out, a, b.t(), a_scale, b_scale, bias)
    return out


def w4a16_linear(x, qweight, meta, group_size, bias=None, out=None):
    """weight-only linear for any M: small-M streaming kernel up to 16 tokens, wgmma dequant-GEMM above."""
    _cuda_bf16(x, "x")
    M, K = x.shape
    N = meta.size(1)
    y = out if out is not None else torch.empty(M, N, dtype=BF16, device=x.device)
    if M <= WQ_SMALL_M_MAX or (M <= WQ_SMALL_M_MAX_NARROW and N <= SMALL_N_MAX):
        return w4a16_linear_small_m(x, qweight, meta, group_size, bias, y)
    check(lib().xb_gemm_w4a16(_p(y), c_i64(y.stride(0)), _p(x), c_i64(x.stride(0)), _p(qweight), _p(meta), _p(bias),
                              c_i32(M), c_i32(N), c_i32(K), c_i32(group_size), _stream()), "w4a16_linear")
    return y


def gemm_w4a16(x, qweight, meta, group_size, bias=None, out=None):
    """always the wgmma dequant-GEMM (tests / benchmarks)."""
    _cuda_bf16(x, "x")
    M, K = x.shape
    N = meta.size(1)
    y = out if out is not None else torch.empty(M, N, dtype=BF16, device=x.device)
    check(lib().xb_gemm_w4a16(_p(y), c_i64(y.stride(0)), _p(x), c_i64(x.stride(0)), _p(qweight), _p(meta), _p(bias),
                              c_i32(M), c_i32(N), c_i32(K), c_i32(group_size), _stream()), "gemm_w4a16")
    return y


# ---- K3 / K2 prefill attention ------------------------------------------------------

def batch_prefill(query, key, value, q_cu_seq_lens, kv_cu_seq_lens, sm_scale, output, output_lse=None, max_qo_len=None,
                  causal=True) -> None:
    """xllm::kernel::cuda::batch_prefill (cuda_ops_api.h:52-66, batch_prefill.cpp:21-163): contiguous ragged q/k/v.
    query [T, Hq, D] (may be a strided view of the packed qkv), key/value [T_kv, Hkv, D]."""
    _cuda_bf16(query, "query"); _cuda_bf16(key, "key"); _cuda_bf16(value, "value"); _cuda_bf16(output, "output")
    _need(q_cu_seq_lens.dtype == torch.int32 and kv_cu_seq_lens.dtype == torch.int32, "cu_seq_lens must be int32")
    _need(key.stride(0) == value.stride(0), "key/value must share the token stride")
    T, Hq, D = query.shape
    Hkv = key.size(1)
    _need(key.stride(1) == D and value.stride(1) == D, "kv heads must be contiguous")
    if max_qo_len is None:
        max_qo_len = int((q_cu_seq_lens[1:] - q_cu_seq_lens[:-1]).max().item())   # host sync; pass it to avoid
    check(lib().xb_prefill_ragged_bf16(_p(query), c_i64(query.stride(0)), c_i64(query.stride(1)), _p(key), _p(value),
                                       c_i64(key.stride(0)), _p(q_cu_seq_lens), _p(kv_cu_seq_lens), _p(output),
                                       c_i64(output.stride(0)), c_i64(output.stride(1)), _p(output_lse),
                                       c_i32(q_cu_seq_lens.numel() - 1), c_i64(T), c_i64(key.size(0)), c_i32(max_qo_len),
                                       c_i32(Hq), c_i32(Hkv), c_i32(D), c_i32(1 if causal else 0), c_f32(sm_scale), _stream()),
          "batch_prefill")


def prefill_plan_splits(batch, max_qo_len, max_kv_len, num_qo_heads, num_kv_heads, num_sms=132) -> int:
    """host-side split-KV decision for a short query chunk over a long KV (what the reference's prefill `plan` decides,
    flashinfer_planinfo.cpp:168-247)."""
    return int(lib().xb_prefill_plan_splits(c_i32(batch), c_i32(max_qo_len), c_i64(max_kv_len), c_i32(num_qo_heads),
                                            c_i32(num_kv_heads), c_i32(num_sms)))


def batch_chunked_prefill(query, k_cache, v_cache, paged_kv_indptr, paged_kv_indices, paged_kv_last_page_len, sm_scale,
                          output, output_lse=None, qo_indptr=None, causal=True, max_qo_len=None, kv_splits=1,
                          workspace=None) -> None:
    """xllm::kernel::cuda::batch_chunked_prefill (cuda_ops_api.h:110-128, batch_chunked_prefill.cpp:26-92).
    kv_splits > 1 (from prefill_plan_splits): split-KV kernel + merge; workspace = uint8/float CUDA buffer (allocated
    here when absent)."""
    _cuda_bf16(query, "query"); _cuda_bf16(k_cache, "k_cache"); _cuda_bf16(v_cache, "v_cache"); _cuda_bf16(output, "output")
    _need(k_cache.is_contiguous() and v_cache.is_contiguous(), "caches must be contiguous NHD")
    T, Hq, D = query.shape
    B = paged_kv_indptr.numel() - 1
    if qo_indptr is None:
        qo_indptr = torch.arange(B + 1, dtype=torch.int32, device=query.device)
        max_qo_len = 1
    if max_qo_len is None:
        max_qo_len = int((qo_indptr[1:] - qo_indptr[:-1]).max().item())
    if kv_splits > 1:
        need = int(lib().xb_prefill_split_workspace_bytes(c_i32(kv_splits), c_i64(T), c_i32(Hq), c_i32(D)))
        if workspace is None:
            workspace = torch.empty(need, dtype=torch.uint8, device=query.device)
        check(lib().xb_prefill_paged_split_bf16(
            _p(query), c_i64(query.stride(0)), c_i64(query.stride(1)), _p(k_cache), _p(v_cache), c_i64(k_cache.size(0)),
            c_i32(k_cache.size(1)), _p(qo_indptr), _p(paged_kv_indptr), _p(paged_kv_indices), _p(paged_kv_last_page_len),
            _p(output), c_i64(output.stride(0)), c_i64(output.stride(1)), _p(output_lse), c_i32(B), c_i64(T), c_i32(max_qo_len),
            c_i32(Hq), c_i32(k_cache.size(2)), c_i32(D), c_i32(1 if causal else 0), c_f32(sm_scale), c_i32(kv_splits),
            _p(workspace), c_i64(workspace.numel() * workspace.element_size()), _stream()), "batch_chunked_prefill (split KV)")
        return
    check(lib().xb_prefill_paged_bf16(_p(query), c_i64(query.stride(0)), c_i64(query.stride(1)), _p(k_cache), _p(v_cache),
                                      c_i64(k_cache.size(0)), c_i32(k_cache.size(1)), _p(qo_indptr), _p(paged_kv_indptr),
                                      _p(paged_kv_indices), _p(paged_kv_last_page_len), _p(output), c_i64(output.stride(0)),
                                      c_i64(output.stride(1)), _p(output_lse), c_i32(B), c_i64(T), c_i32(max_qo_len),
                                      c_i32(Hq), c_i32(k_cache.size(2)), c_i32(D), c_i32(1 if causal else 0),
                                      c_f32(sm_scale), _stream()), "batch_chunked_prefill")


def w4a16_gate_up_act(x, qweight, meta, group_size, act_mode="silu", bias=None, out=None, gate_up_buf=None):
    """DenseMLPImpl's gate_up linear + act_and_mul (dense_mlp.cpp:97-118) with the INTERLEAVED gate/up packing
    (quant.pack_w4_gate_up).  M <= 16: one fused kernel (activation in the GEMV epilogue); larger M: wgmma
    dequant-GEMM into `gate_up_buf` + act_and_mul over the interleaved columns."""
    _cuda_bf16(x, "x")
    if act_mode not in _ACT:
        raise XllmB200Error(f"Unsupported act mode: {act_mode}")
    M, K = x.shape
    N = meta.size(1)
    y = out if out is not None else torch.empty(M, N // 2, dtype=BF16, device=x.device)
    if M <= 16:
        check(lib().xb_linear_w4a16_gate_up_act_small_m(_p(y), c_i64(y.stride(0)), _p(x), c_i64(x.stride(0)), _p(qweight),
                                                        _p(meta), _p(bias), c_i32(M), c_i32(N), c_i32(K), c_i32(group_size),
                                                        c_i32(_ACT[act_mode]), _stream()), "w4a16_gate_up_act")
        return y
    gu = gate_up_buf if gate_up_buf is not None else torch.empty(M, N, dtype=BF16, device=x.device)
    gemm_w4a16(x, qweight, meta, group_size, bias, gu)
    check(lib().xb_act_and_mul_interleaved8_bf16(_p(y), _p(gu), c_i32(N // 2), c_i32(M), c_i32(_ACT[act_mode]), _stream()),
          "act_and_mul_interleaved8")
    return y


def set_w4_decode_form(form: int) -> int:
    """0: bf16-weight form, 1: exact-dequant form (oracle/quant.py) of the W4A16 decode kernels; returns the old form."""
    return int(lib().xb_set_w4_decode_form(c_i32(form)))


def w4a16_decode_fused_fits(M: int, K: int) -> bool:
    """whether w4a16_decode_fused can stage an [M, K] activation block in shared memory."""
    return bool(lib().xb_linear_w4a16_decode_fused_fits(c_i32(M), c_i32(K)))


def w4a16_decode_fused(x, qweight, meta, group_size, bias=None, out=None, *, norm_weight=None, eps=1e-6, residual_in=None,
                       residual_out=None, stage_x=False, epilogue="none", act_mode="silu", positions=None,
                       cos_sin_cache=None, slot_ids=None, key_cache=None, value_cache=None, num_heads=0, num_kv_heads=0,
                       head_dim=0, norm_stats_in=None, norm_stats_out=None):
    """Decode-step form of a weight-only linear (M <= 8): the launches the reference makes around the GEMV ride in it.
      prologue  norm_weight: x := RMSNorm(x (+ residual_in)) * norm_weight  (rms_norm / fused_add_rms_norm,
                cuda_ops_api.h:157-165); residual_out receives x + residual_in (must be a different buffer)
      epilogue  "none" | "act_mul" (DenseMLP's act_and_mul on interleaved gate/up rows, out [M, N/2]) |
                "rope_cache" (rotary_embedding + reshape_paged_cache of qwen2_attention.cpp:147-171 /
                flashinfer_attention.cpp:128-131; rows packed by quant.pack_w4_qkv_rope, out [M, N] logical order) |
                "residual_stats" (row-parallel projection as producer of a split RMSNorm: residual_out = bf16(y +
                residual_in), norm_stats_out [N/16, 8] f32 = partial sums of its squares; `out` is not written)
      split-norm consumer: norm_stats_in (+ norm_weight): x is the residual stream, the prologue only normalises"""
    _cuda_bf16(x, "x")
    _need(qweight.dtype == torch.int32 and meta.dtype == torch.int32, "qweight/meta must be int32 storage")
    epi = {"none": 0, "act_mul": 1, "rope_cache": 2, "residual_stats": 3}.get(epilogue)
    _need(epi is not None, f"unknown epilogue {epilogue}")
    if epi == 1 and act_mode not in _ACT:
        raise XllmB200Error(f"Unsupported act mode: {act_mode}")
    M, K = x.shape
    N = meta.size(1)
    n_out = N // 2 if epi == 1 else N
    y = out if out is not None else (x if epi == 3 else torch.empty(M, n_out, dtype=BF16, device=x.device))
    for t, n in ((norm_stats_in, "norm_stats_in"), (norm_stats_out, "norm_stats_out")):
        if t is not None:
            _need(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), f"{n} must be a contiguous float32 CUDA tensor")
    for t, n in ((norm_weight, "norm_weight"), (residual_in, "residual_in"), (residual_out, "residual_out")):
        if t is not None:
            _cuda_bf16(t, n)
            _need(t.is_contiguous(), f"{n} must be contiguous")
    if epi == 2:
        _need(positions is not None and positions.dtype == torch.int64 and slot_ids is not None and
              slot_ids.dtype == torch.int32, "positions int64 / slot_ids int32")
        _cuda_bf16(cos_sin_cache, "cos_sin_cache"); _cuda_bf16(key_cache, "key_cache"); _cuda_bf16(value_cache, "value_cache")
        _need(key_cache.is_contiguous() and value_cache.is_contiguous(), "caches must be contiguous NHD")
        _need(cos_sin_cache.size(-1) == head_dim, "full rotary only (rot_dim == head_dim)")
    check(lib().xb_linear_w4a16_decode_fused(
        _p(y), c_i64(y.stride(0)), _p(x), c_i64(x.stride(0)), _p(qweight), _p(meta), _p(bias), c_i32(M), c_i32(N), c_i32(K),
        c_i32(group_size), _p(norm_weight), c_f32(eps), _p(residual_in), _p(residual_out), c_i32(1 if stage_x else 0),
        c_i32(epi), c_i32(_ACT.get(act_mode, 0)), _p(positions), _p(cos_sin_cache), _p(slot_ids), _p(key_cache),
        _p(value_cache), c_i32(num_heads), c_i32(num_kv_heads), c_i32(head_dim), _p(norm_stats_in), _p(norm_stats_out),
        _stream()), "w4a16_decode_fused")
    return y


def rope_and_cache_packed(positions, qkv_packed, qkv_out, cos_sin_cache, slot_ids, key_cache, value_cache, num_heads,
                          num_kv_heads, head_dim) -> None:
    """rotary_embedding + reshape_paged_cache for a qkv projection in the rope-pair packed column order
    (quant.pack_w4_qkv_rope) that ran as a plain GEMM: qkv_out receives q | k | v in logical order."""
    _cuda_bf16(qkv_packed, "qkv_packed"); _cuda_bf16(qkv_out, "qkv_out"); _cuda_bf16(cos_sin_cache, "cos_sin_cache")
    _need(positions.dtype == torch.int64 and slot_ids.dtype == torch.int32, "positions int64 / slot_ids int32")
    _need(qkv_packed.stride(-1) == 1 and qkv_out.stride(-1) == 1 and key_cache.is_contiguous() and value_cache.is_contiguous(),
          "layout")
    _need(cos_sin_cache.size(-1) == head_dim, "full rotary only (rot_dim == head_dim)")
    T = positions.numel()
    check(lib().xb_rope_and_cache_packed_bf16(_p(positions), _p(qkv_packed), c_i64(qkv_packed.stride(0)), _p(qkv_out),
                                              c_i64(qkv_out.stride(0)), _p(cos_sin_cache), _p(slot_ids), _p(key_cache),
                                              _p(value_cache), c_i32(num_heads), c_i32(num_kv_heads), c_i32(head_dim),
                                              c_i32(T), _stream()), "rope_and_cache_packed")


# ---- W8A16 ------------------------------------------------------------------------------------------------------
def w8a16_linear_small_m(x, qweight, meta, group_size, bias=None, out=None):
    """additive boundary (SURVEY 8b-3): y = x . dequant(W8)^T (+bias), M <= 64.  qweight/meta from quant.pack_w8."""
    _cuda_bf16(x, "x")
    _need(qweight.dtype == torch.int32 and meta.dtype == torch.int32, "qweight/meta must be int32 storage")
    M, K = x.shape
    N = meta.size(1)
    y = out if out is not None else torch.empty(M, N, dtype=BF16, device=x.device)
    check(lib().xb_linear_w8a16_small_m(_p(y), c_i64(y.stride(0)), _p(x), c_i64(x.stride(0)), _p(qweight), _p(meta),
                                        _p(bias), c_i32(M), c_i32(N), c_i32(K), c_i32(group_size), _stream()),
          "w8a16_linear_small_m")
    return y


def gemm_w8a16(x, qweight, meta, group_size, bias=None, out=None):
    """always the wgmma dequant-GEMM (tests / benchmarks)."""
    _cuda_bf16(x, "x")
    M, K = x.shape
    N = meta.size(1)
    y = out if out is not None else torch.empty(M, N, dtype=BF16, device=x.device)
    check(lib().xb_gemm_w8a16(_p(y), c_i64(y.stride(0)), _p(x), c_i64(x.stride(0)), _p(qweight), _p(meta), _p(bias),
                              c_i32(M), c_i32(N), c_i32(K), c_i32(group_size), _stream()), "gemm_w8a16")
    return y


def w8a16_linear(x, qweight, meta, group_size, bias=None, out=None):
    """weight-only int8 linear for any M: streaming kernel for decode batches, wgmma dequant-GEMM above."""
    M, N = x.shape[0], meta.size(1)
    if M <= WQ_SMALL_M_MAX or (M <= WQ_SMALL_M_MAX_NARROW and N <= SMALL_N_MAX):
        return w8a16_linear_small_m(x, qweight, meta, group_size, bias, out)
    return gemm_w8a16(x, qweight, meta, group_size, bias, out)


# ---- mixture of experts (SURVEY 8f n4) ------------------------------------------------
def moe_fused_topk(gating_output, topk: int, renormalize: bool, correction_bias=None, scoring_func: str = "softmax"):
    """xllm::kernel::cuda::moe_fused_topk (cuda_ops_api.h:251-256): -> (topk_weights fp32 [T, k], topk_ids int32 [T, k])."""
    _need(gating_output.is_cuda and gating_output.dim() == 2 and gating_output.stride(1) == 1, "gating_output [T, E] on device")
    _need(gating_output.dtype in (torch.float32, BF16), "gating_output must be float32 or bfloat16")
    if scoring_func not in ("softmax", "sigmoid"):
        raise XllmB200Error(f"Unsupported scoring function for moe topk: {scoring_func}")
    if correction_bias is not None:
        _need(correction_bias.dtype == torch.float32 and correction_bias.is_contiguous(), "correction_bias must be float32")
        if scoring_func == "softmax":
            correction_bias = None          # the reference drops it on the softmax path (moe_fused_topk.cu:36-43)
    T, E = gating_output.shape
    w = torch.empty(T, topk, dtype=torch.float32, device=gating_output.device)
    ids = torch.empty(T, topk, dtype=torch.int32, device=gating_output.device)
    check(lib().xb_moe_fused_topk(_p(w), _p(ids), _p(gating_output), c_i32(1 if gating_output.dtype == BF16 else 0),
                                  c_i64(gating_output.stride(0)), _p(correction_bias), c_i32(T), c_i32(E), c_i32(topk),
                                  c_i32(1 if renormalize else 0), c_i32(1 if scoring_func == "sigmoid" else 0), _stream()),
          "moe_fused_topk")
    return w, ids


def set_moe_grouped_min_tokens(min_tokens: int) -> int:
    """smallest token count for which the MoE expert entries take the grouped-GEMM path (default 65, i.e. T <= 64 runs the
    expert GEMVs); for tests and sweeps.  Returns the old value."""
    old = int(lib().xb_set_moe_grouped_min_tokens(c_i32(min_tokens)))
    _need(old >= 1, f"set_moe_grouped_min_tokens: {lib().xb_last_error().decode()}")
    return old


def moe_experts_describe(kind: str, T: int, k: int, H: int, I: int, E_local: int) -> str:
    """host-only: the path the MoE expert entries take for a shape ("bf16 gemv", "w4 grouped bn=128 m_tiles<=40");
    kind "bf16" or "w4"."""
    buf = ctypes.create_string_buffer(96)
    n = lib().xb_moe_experts_describe(c_i32({"bf16": 0, "w4": 2}[kind]), c_i32(T), c_i32(k), c_i32(H), c_i32(I), c_i32(E_local),
                                      buf, c_i32(96))
    _need(n > 0, "moe_experts_describe failed")
    return buf.value.decode()


def cutlass_fused_moe(input, token_selected_experts, token_final_scales, fc1_expert_weights, fc2_expert_weights, ep_size: int = 1,
                      ep_rank: int = 0, output=None, workspace=None):
    """xllm::kernel::cuda::cutlass_fused_moe (cuda_ops_api.h:260-289) for unquantised bf16 experts at any token count:
    fc1 [E_local, 2I, H] ([up | gate]), fc2 [E_local, H, I]; experts of other EP ranks contribute zero.  T <= 64 runs one
    expert GEMV per (token, expert) pair (decode); T >= 65 sorts the pairs by expert on the device and runs grouped wgmma
    GEMMs (prefill).  No host synchronisation either way, so the call can be captured in a CUDA graph."""
    _cuda_bf16(input, "input"); _cuda_bf16(fc1_expert_weights, "fc1_expert_weights"); _cuda_bf16(fc2_expert_weights, "fc2_expert_weights")
    _need(token_selected_experts.dtype == torch.int32 and token_final_scales.dtype == torch.float32, "ids int32 / scales float32")
    _need(token_selected_experts.is_contiguous() and token_final_scales.is_contiguous() and fc1_expert_weights.is_contiguous() and
          fc2_expert_weights.is_contiguous(), "contiguous ids / scales / expert weights")
    T, H = input.shape
    k = token_selected_experts.size(1)
    El, I2, _ = fc1_expert_weights.shape
    inter = I2 // 2
    _need(tuple(fc2_expert_weights.shape) == (El, H, inter), "fc2_expert_weights must be [E_local, H, I]")
    out = output if output is not None else torch.empty(T, H, dtype=BF16, device=input.device)
    need = int(lib().xb_moe_experts_workspace_bytes(c_i32(T), c_i32(k), c_i32(H), c_i32(inter)))
    ws = workspace if workspace is not None and workspace.numel() >= need else torch.empty(need, dtype=torch.uint8, device=input.device)
    check(lib().xb_moe_experts_bf16(_p(out), c_i64(out.stride(0)), _p(input), c_i64(input.stride(0)), _p(token_selected_experts),
                                    _p(token_final_scales), _p(fc1_expert_weights), _p(fc2_expert_weights), c_i32(T), c_i32(k),
                                    c_i32(H), c_i32(inter), c_i32(El), c_i32(ep_rank * El), _p(ws), c_i64(ws.numel()), _stream()),
          "cutlass_fused_moe")
    return out


def fused_moe_w4a16(input, token_selected_experts, token_final_scales, fc1_qweight, fc1_meta, fc2_qweight, fc2_meta, group_size,
                    ep_size: int = 1, ep_rank: int = 0, output=None, workspace=None):
    """W4A16 experts (additive; BASELINE configs[4]): fc1 [E_local, 2I/16, H/64, 32, 4] + meta [E_local, H/g, 2I] ([up | gate]
    rows, quant.pack_w4 per expert), fc2 [E_local, H/16, I/64, 32, 4] + meta [E_local, I/g, H].  Same two paths as
    cutlass_fused_moe: expert GEMVs for T <= 64, grouped wgmma GEMMs with the int4 dequantisation fused in above."""
    _cuda_bf16(input, "input")
    for t_, n in ((fc1_qweight, "fc1_qweight"), (fc1_meta, "fc1_meta"), (fc2_qweight, "fc2_qweight"), (fc2_meta, "fc2_meta")):
        _need(t_.is_cuda and t_.dtype == torch.int32 and t_.is_contiguous(), f"{n} must be contiguous int32 storage on device")
    _need(token_selected_experts.dtype == torch.int32 and token_final_scales.dtype == torch.float32 and
          token_selected_experts.is_contiguous() and token_final_scales.is_contiguous(), "ids int32 / scales float32, contiguous")
    T, H = input.shape
    k = token_selected_experts.size(1)
    El = fc1_qweight.size(0)
    inter = fc1_meta.size(2) // 2
    _need(tuple(fc2_meta.shape[:1]) == (El,) and fc2_meta.size(2) == H, "fc2_meta must be [E_local, I/g, H]")
    out = output if output is not None else torch.empty(T, H, dtype=BF16, device=input.device)
    need = int(lib().xb_moe_experts_workspace_bytes(c_i32(T), c_i32(k), c_i32(H), c_i32(inter)))
    ws = workspace if workspace is not None and workspace.numel() >= need else torch.empty(need, dtype=torch.uint8, device=input.device)
    check(lib().xb_moe_experts_w4a16(_p(out), c_i64(out.stride(0)), _p(input), c_i64(input.stride(0)), _p(token_selected_experts),
                                     _p(token_final_scales), _p(fc1_qweight), _p(fc1_meta), _p(fc2_qweight), _p(fc2_meta),
                                     c_i32(group_size), c_i32(T), c_i32(k), c_i32(H), c_i32(inter), c_i32(El), c_i32(ep_rank * El),
                                     _p(ws), c_i64(ws.numel()), _stream()), "fused_moe_w4a16")
    return out
