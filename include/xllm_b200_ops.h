/*
 * xllm_b200_ops.h -- C-ABI of libxllm_b200_ops.so
 *
 * H100-native (sm_90a) replacement for the per-layer inference hot path of
 * jd-opensource/xllm (reference @ 87e8d6e, v0.9.0).  Every entry point takes
 * plain device pointers, sizes, element strides and a cudaStream_t (passed as
 * void*); none takes a torch type.  Each one cites the reference interface it
 * replaces (paths relative to the reference checkout, file:line).
 *
 * Conventions
 *   - return value: 0 on success, non-zero on error; xb_last_error() returns a
 *     thread-local message (the reference aborts through glog CHECK/TORCH_CHECK:
 *     the C++ shim in xllm_b200/csrc/xllm_cuda_ops.cpp turns a non-zero code
 *     into TORCH_CHECK(false, msg)).
 *   - all tensors are borrowed; nothing is allocated or freed by the callee;
 *     scratch comes from caller-provided workspaces; no host synchronisation
 *     (every launcher is CUDA-graph-capturable).
 *   - bf16 = __nv_bfloat16 storage (uint16), e4m3 = __nv_fp8_e4m3 storage (uint8).
 *   - strides are in ELEMENTS unless the name ends in _bytes.
 */
#ifndef XLLM_B200_OPS_H_
#define XLLM_B200_OPS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XB_ABI_VERSION 1

typedef void* xb_stream_t; /* cudaStream_t */

/* ---- library ------------------------------------------------------------
 * library-level entries (no reference counterpart): ABI version, the message of the last failed call on this thread (the
 * reference reports through glog CHECK / c10::Error; a C ABI returns a code + this string), launch counter for the benches. */
int xb_abi_version(void);
const char* xb_last_error(void);
/* library-level: number of kernels this library has launched in this process (all threads);
 * bench.py reports the delta over the timed region as "gpu_launches". */
uint64_t xb_launch_count(void);
/* enable (1) / disable (0) programmatic dependent launch on our launches.
 * Mirrors support_pdl() -> Platform::is_enable_pdl()
 * (xllm/core/kernels/cuda/utils.cpp:370, batch_decode.cpp:79). */
void xb_set_pdl(int enable);

/* ---- K7: RMSNorm ---------------------------------------------------------
 * replaces xllm::kernel::cuda::rms_norm          (cuda_ops_api.h:157-160,
 *          norm.cu:43-78,430-460) and
 *          xllm::kernel::cuda::fused_add_rms_norm (cuda_ops_api.h:162-165,
 *          norm.cu:80-173,462-515).
 * out[t,:] = bf16( bf16(x[t,:] * rstd_t) * w ),  rstd_t = rsqrt(mean_f32(x^2)+eps)
 * fused:  residual <- bf16(input + residual); input <- norm(residual) (in place). */
int xb_rms_norm_bf16(void* out, const void* input, int64_t input_stride,
                     const void* weight, float eps, int num_tokens,
                     int hidden_size, xb_stream_t stream);
int xb_fused_add_rms_norm_bf16(void* input, int64_t input_stride, void* residual,
                               const void* weight, float eps, int num_tokens,
                               int hidden_size, xb_stream_t stream);

/* ---- K8: RMSNorm + static FP8 quant ---------------------------------------
 * replaces rms_norm_static_fp8_quant / fused_add_rms_norm_static_fp8_quant
 * (cuda_ops_api.h:203-221, norm.cu:228-423,517-600).  scale: device float[1]. */
int xb_rms_norm_static_fp8_quant_bf16(void* out_e4m3, const void* input,
                                      int64_t input_stride, const void* weight,
                                      const float* scale, float eps,
                                      int num_tokens, int hidden_size,
                                      xb_stream_t stream);
int xb_fused_add_rms_norm_static_fp8_quant_bf16(
    void* out_e4m3, void* input, int64_t input_stride, void* residual,
    const void* weight, const float* scale, float eps, int num_tokens,
    int hidden_size, xb_stream_t stream);

/* ---- K6: static scaled FP8 quant -----------------------------------------
 * replaces static_scaled_fp8_quant (cuda_ops_api.h:182-186, fp8_quant.cu:78-153):
 * out = sat_e4m3(x * (1/scale)), RNE, saturating at +-448. */
int xb_static_scaled_fp8_quant_bf16(void* out_e4m3, int64_t out_stride,
                                    const void* input, int64_t input_stride,
                                    const float* scale, int num_tokens,
                                    int hidden_size, xb_stream_t stream);
/* dynamic per-tensor scale = max(amax/448, 1e-12) (fp8_scaled_quantize.cpp:36-41),
 * computed on device into scale_out[1] (no host sync), then quantised. */
int xb_dynamic_scaled_fp8_quant_bf16(void* out_e4m3, int64_t out_stride,
                                     const void* input, int64_t input_stride,
                                     float* scale_out, int num_tokens,
                                     int hidden_size, xb_stream_t stream);

/* ---- K9: rotary embedding -------------------------------------------------
 * replaces xllm::kernel::cuda::rotary_embedding (cuda_ops_api.h:31-37,
 * rope.cu:27-250).  In place on query/key; cos_sin_cache[max_pos, rot_dim] =
 * [cos(rot/2) | sin(rot/2)] in bf16; all arithmetic in bf16 with a rounding
 * after every multiply/add, as the reference does with scalar_t = BFloat16.
 * key may be NULL.  positions are int64. */
int xb_rotary_embedding_bf16(const int64_t* positions, void* query, void* key,
                             const void* cos_sin_cache, int rot_dim,
                             int64_t query_stride, int64_t key_stride,
                             int64_t head_stride, int num_heads,
                             int num_kv_heads, int head_size, int is_neox,
                             int num_tokens, xb_stream_t stream);

/* ---- K12: KV-cache scatter -----------------------------------------------
 * replaces xllm::kernel::cuda::reshape_paged_cache (cuda_ops_api.h:44-49,
 * reshape_paged_cache.cu:23-99).  cache layout [n_blocks, block_size,
 * n_kv_heads, head_dim]; slot<0 is skipped.  Bit-exact copy. */
int xb_reshape_paged_cache_bf16(const int32_t* slot_ids, const void* keys,
                                const void* values, void* key_cache,
                                void* value_cache, int64_t k_stride,
                                int64_t v_stride, int n_kv_heads, int head_dim,
                                int block_size, int num_tokens,
                                xb_stream_t stream);

/* ---- K9+K12 fused: RoPE (q,k in place) + scatter of rotated k and v --------
 * one launch instead of rotary_embedding + reshape_paged_cache
 * (qwen2_attention.cpp:173-176 + flashinfer_attention.cpp:128-131).
 * Results are bit-identical to calling the two ops in sequence. */
int xb_rope_and_cache_bf16(const int64_t* positions, void* query, void* key,
                           const void* value, const void* cos_sin_cache,
                           const int32_t* slot_ids, void* key_cache,
                           void* value_cache, int rot_dim, int64_t query_stride,
                           int64_t key_stride, int64_t value_stride,
                           int num_heads, int num_kv_heads, int head_size,
                           int block_size, int is_neox, int num_tokens,
                           xb_stream_t stream);

/* additive (no reference counterpart; same arithmetic as rope.cu:27-54 + reshape_paged_cache.cu:23-62): the same two ops on a
 * qkv projection whose output columns are in the rope-pair packed order of the weight-only decode layout (quant.pack_w4_qkv_rope; the decode GEMV does this work in its epilogue, see
 * xb_linear_w4a16_decode_fused): reads qkv_packed [T, (Hq+2Hkv)*D], writes q | k | v in LOGICAL order to qkv_out
 * (a different buffer) and the new k / v rows to the paged caches.  NeoX halves, full rotary. */
int xb_rope_and_cache_packed_bf16(const int64_t* positions, const void* qkv_packed,
                                  int64_t in_stride, void* qkv_out, int64_t out_stride,
                                  const void* cos_sin_cache, const int32_t* slot_ids,
                                  void* key_cache, void* value_cache, int num_heads,
                                  int num_kv_heads, int head_size, int num_tokens,
                                  xb_stream_t stream);

/* ---- K10: fused per-head QK RMSNorm + RoPE (Qwen3) -------------------------
 * replaces xllm::kernel::cuda::fused_qk_norm_rope (cuda_ops_api.h:252-266,
 * fused_qknorm_rope.cu:84-471). qkv packed [T,(hq+hk+hv)*d], in place. */
int xb_fused_qk_norm_rope_bf16(void* qkv, int num_heads_q, int num_heads_k,
                               int num_heads_v, int head_dim, float eps,
                               const void* q_weight, const void* k_weight,
                               const void* cos_sin_cache, int rot_dim,
                               int interleaved, const int64_t* position_ids,
                               int num_tokens, xb_stream_t stream);

/* ---- K10+K12 fused: QK-norm + RoPE (q,k in place) + scatter of k and v -----
 * one launch instead of fused_qk_norm_rope + reshape_paged_cache
 * (qwen2_attention.cpp:147-171 + flashinfer_attention.cpp:128-131).
 * qkv contiguous [T,(hq+2*hkv)*d], d = 64 or 128; NeoX halves, full rotary
 * (cos_sin_cache [max_pos, d]); caches NHD [n_blocks, block_size, hkv, d];
 * slot<0 skips the cache writes only.  qkv and both caches are bit-identical
 * to calling the two ops in sequence.  Other head_dim and NULL weights or
 * table are rejected before any device access; num_tokens == 0 is a no-op. */
int xb_qk_norm_rope_and_cache_bf16(void* qkv, int num_heads_q, int num_heads_kv,
                                   int head_dim, float eps, const void* q_weight,
                                   const void* k_weight,
                                   const void* cos_sin_cache,
                                   const int64_t* positions,
                                   const int32_t* slot_ids, void* key_cache,
                                   void* value_cache, int num_tokens,
                                   xb_stream_t stream);

/* ---- K11: act_and_mul ------------------------------------------------------
 * replaces xllm::kernel::cuda::act_and_mul (cuda_ops_api.h:39-42,
 * activation.cu:45-186).  out[t,:] = bf16( bf16(act(x[t,:d])) * x[t,d:] ).
 * act_mode: 0 silu, 1 gelu (erf), 2 gelu_tanh. */
int xb_act_and_mul_bf16(void* out, const void* input, int d, int num_tokens,
                        int act_mode, xb_stream_t stream);

/* ---- K1/K2-decode: paged decode attention ----------------------------------
 * replaces the FlashInfer decode module the reference dlopen()s
 * (xllm/core/kernels/cuda/batch_decode.cpp:26-86 `run`; planner
 * layers/cuda/flashinfer_planinfo.cpp:249-337 `plan`).
 *
 * q   [batch, num_qo_heads, head_dim] bf16 (q_stride_n / q_stride_h elements)
 * k_cache, v_cache: paged, element strides (page, token, head); NHD layout of
 *     the reference = (block_size*H_kv*D, H_kv*D, D).
 * kv_indptr[batch+1], kv_indices[], kv_last_page_len[batch]: the reference's
 *     paged triplet (batch_input_builder.cpp:790-801), int32, on device.
 * o   [batch, num_qo_heads, head_dim] bf16; lse (optional) [batch, num_qo_heads]
 *     f32, base-2 log-sum-exp of sm_scale*log2(e)*q.k like FlashInfer's state.
 *
 * xb_decode_plan is host-only arithmetic (no device access, no sync): given an
 * upper bound of pages per request it picks how many KV splits to launch so
 * that batch*num_kv_heads*splits covers the SMs (and how many of them form one
 * thread-block cluster), and returns workspace needs.  The split SIZE is not
 * part of the plan: the kernel derives it from the live kv_len and the launched
 * grid, so a plan made at CUDA-graph capture stays correct for any later
 * context length (the reference replays a captured `run`:
 * layers/cuda/flashinfer_attention.cpp:306-311).
 * The plan is opaque int64[8] (plan_info is opaque to xLLM too:
 * flashinfer_planinfo.cpp:37-62).  workspace_f32 needs plan[2] bytes,
 * workspace_i32 needs plan[3] & 0xffffffff bytes and MUST be zero-initialised
 * once (the kernel restores it to zero). */
int xb_decode_plan(int64_t* plan8, int batch, int num_qo_heads, int num_kv_heads,
                   int head_dim, int page_size, int max_pages_per_request,
                   int num_sms);
/* additive (no reference counterpart).  flags bit 0 ("early prefetch"): the caller guarantees that no kernel still in flight writes KV rows other than the
 * newest token of each request, nor the paged triplet (true inside a decode step); the kernel then streams KV before
 * its programmatic-dependent-launch wait, overlapping the producer kernel's tail. */
int xb_decode_plan_set_flags(int64_t* plan8, int flags);
/* debug aid: the next xb_paged_decode_bf16 launches write per-CTA stage timestamps (%globaltimer, ns) to
 * buf = uint64[grid CTAs][8] (device memory); null switches it off. */
int xb_debug_set_decode_trace(void* buf);
/* debug aid: number of thread-block clusters of `cluster` CTAs of the paged decode kernel the current device can run
 * concurrently (cudaOccupancyMaxActiveClusters), -1 if that cluster size cannot be launched. */
int xb_debug_max_active_clusters(int cluster);
/* debug aid: cluster size the most recent xb_paged_decode_bf16 launch of this process used (1 when the launcher fell
 * back from the planned size because the device cannot co-schedule it), 0 before the first launch. */
int xb_debug_last_decode_cluster(void);
int xb_paged_decode_bf16(const int64_t* plan8, const void* q, int64_t q_stride_n,
                         int64_t q_stride_h, const void* k_cache,
                         const void* v_cache, int64_t kv_stride_page,
                         int64_t kv_stride_token, int64_t kv_stride_head,
                         const int32_t* kv_indptr, const int32_t* kv_indices,
                         const int32_t* kv_last_page_len, void* o,
                         int64_t o_stride_n, int64_t o_stride_h, float* lse,
                         float sm_scale, void* workspace_f32,
                         void* workspace_i32, xb_stream_t stream);

/* ---- MLA (DeepSeek-V2/V3, Kimi-K2): latent cache writer + absorbed attention --
 * additive (the reference runs MLA on MLU/NPU only; its CUDA cache layout is
 * framework/kv_cache/kv_cache_shape.cpp:242-257,273-288): two paged caches,
 * ckv_cache [pages, page_size, 512] = RMSNorm(c_kv) and kpe_cache
 * [pages, page_size, 64] = RoPE(k_pe), element strides (page, token).
 * Fixed dims kv_lora_rank = 512, qk_rope_head_dim = 64; others are rejected.
 *
 * xb_mla_cache_latent_bf16: fused_mla_kv with quant_mode "none"
 * (kernels/param.h:1105-1180; non-fused form deepseek_v2_attention.cpp:223-240)
 * in one launch.  latent [T, 576] (row stride) = kv_a_proj_with_mqa output
 * [c_kv | k_pe]; gamma [512] = kv_a_layernorm; positions int64 [T];
 * cos_sin_cache [max_pos, 64] = [cos | sin]; interleaved = 1 pairs (2i, 2i+1)
 * (DeepSeek), 0 pairs (i, i+32) (NeoX); slot_ids int32 [T], slot < 0 skipped.
 * Bit-identical to xb_rms_norm_bf16 + xb_rotary_embedding_bf16 + two
 * xb_reshape_paged_cache_bf16 on the same inputs. */
int xb_mla_cache_latent_bf16(const void* latent, int64_t latent_stride, const void* gamma, float eps,
                             const int64_t* positions, const void* cos_sin_cache, int interleaved,
                             const int32_t* slot_ids, void* ckv_cache, int64_t ckv_stride_page,
                             int64_t ckv_stride_token, void* kpe_cache, int64_t kpe_stride_page,
                             int64_t kpe_stride_token, int kv_lora_rank, int qk_rope_head_dim, int page_size,
                             int num_tokens, xb_stream_t stream);
/* xb_mla_plan: host-only arithmetic like xb_decode_plan.  Picks the KV-split
 * count for batch requests of up to max_qo_len q tokens and num_heads heads
 * (1..128) and returns the float workspace size in plan[1] bytes (0 without
 * splits).  The split SIZE is derived on the device from the live kv_len, so a
 * plan captured into a CUDA graph stays correct at later context lengths.
 * xb_mla_plan_set_splits overrides the split count (1..128) and updates plan[1].
 *
 * xb_mla_paged_attention_bf16: absorbed MLA (layers/mlu/attention.cpp:65-155)
 * over the paged caches: per q row, key = [c_kv | k_pe] of one kv head,
 * value = c_kv; o = softmax(sm_scale [q_nope | q_pe] key^T) value.
 * q_nope [T, H, 512] and q_pe [T, H, 64] take separate strides (the split form,
 * or views of a packed q_input [T, H, 576]); o [T, H, 512] bf16.  Ragged q
 * through qo_indptr [batch+1] (qo_len <= the plan's max_qo_len: q rows past
 * it are not computed, and nothing is written outside o and the workspace); the paged
 * triplet as in xb_paged_decode_bf16.  causal: q row i of a request sees
 * kv <= kv_len - qo_len + i.  Serves decode (qo_len 1), speculative steps and
 * chunked prefill; requests with kv_len 0 produce zero rows.  No allocation,
 * no host synchronisation, capturable. */
int xb_mla_plan(int64_t* plan8, int batch, int num_heads, int kv_lora_rank, int qk_rope_head_dim, int max_qo_len,
                int page_size, int max_pages_per_request, int num_sms);
int xb_mla_plan_set_splits(int64_t* plan8, int splits);
int xb_mla_paged_attention_bf16(const int64_t* plan8, const void* q_nope, int64_t q_nope_stride_t,
                                int64_t q_nope_stride_h, const void* q_pe, int64_t q_pe_stride_t, int64_t q_pe_stride_h,
                                const void* ckv_cache, int64_t ckv_stride_page, int64_t ckv_stride_token,
                                const void* kpe_cache, int64_t kpe_stride_page, int64_t kpe_stride_token,
                                const int32_t* qo_indptr, const int32_t* kv_indptr, const int32_t* kv_indices,
                                const int32_t* kv_last_page_len, int causal, void* o, int64_t o_stride_t,
                                int64_t o_stride_h, float sm_scale, void* workspace, int64_t workspace_bytes,
                                xb_stream_t stream);
/* Expanded MLA prefill (DeepSeek-V3 attention as transformers' DeepseekV3Attention
 * computes it): the latent rows are up-projected through kv_b_proj into per-head
 * k_nope / v, then ordinary causal attention runs with 192-wide QK
 * ([q_nope | q_pe] . [k_nope | k_pe], k_pe shared by all heads) and 128-wide V.
 * qk_nope_head_dim = v_head_dim = 128 (kv_b_proj [H * 256, 512]), kv_lora_rank 512,
 * qk_rope_head_dim 64.
 *
 * xb_mla_expanded_plan: host-only.  qo_lens_host / kv_lens_host [batch] are the
 * step's q lengths and the total kv lengths (history + the step's tokens,
 * qo_len <= kv_len).  plan8: [0] use_expanded, [1] workspace bytes, [2] batch,
 * [3] num_heads, [4] max_qo_len, [5] total_kv, [6] max_kv_len, [7] total_q | tag.
 *   use_expanded = max_qo_len > 1 and  F_abs > 0.5 * (F_up + F_exp), with per
 *   head F_abs = 2 (576 + 512) P, F_exp = 2 (192 + 128) P, F_up = 2 * 512 * 256 *
 *   total_kv, P = the causal (q, kv) pairs: one FLOP of the expanded path is
 *   taken to cost as much as 0.5 FLOP of the absorbed kernel.  The constant
 *   gives the least total time over the selector grid of tools/mla_sweep.py
 *   (README).  Decode steps and short chunks over long histories come out
 *   absorbed (xb_mla_paged_attention_bf16); long prompts expanded.  The form and
 *   the sizes do not depend on the SM count, so the plan takes none.
 *   The selector looks at FLOPs only: the workspace grows as total_kv * H * 512
 *   bytes (8.9 GB for 4096 new tokens over 128 K of history at H = 128); a
 *   caller short of memory compares plan[1] with what it can spare and runs
 *   the absorbed form instead.
 *   Workspace layout, every part 256-byte aligned:
 *     kv_up [total_kv, H, 256] bf16 (per head k_nope | v) at byte 0,
 *     ckv   [total_kv, 512] bf16 at align256(total_kv * H * 512),
 *     kpe   [total_kv, 64] bf16 after it (align256(total_kv * 1024) further),
 *     kv_cu int32 [batch + 1] after it (align256(total_kv * 128) further).
 *
 * xb_mla_prefill_expanded_bf16: three launches, no allocation, no host
 * synchronisation.  q [T, H, 192] = [q_nope | roped q_pe] (row / head strides);
 * the caches and the paged triplet as in xb_mla_paged_attention_bf16, holding
 * the history and the step's tokens; qo_indptr [batch + 1]; kv_b_proj
 * [H * 256, 512] (the checkpoint's kv_b_proj.weight); o [T, H, 128] = o_proj's
 * input.  Causal: q row i of a request sees kv <= kv_len - qo_len + i.
 *   1. gather: each request's c_kv / k_pe rows into the workspace's ckv / kpe,
 *      row offsets from the device's lengths; rows past the plan's total_kv are
 *      not written (the workspace is never written outside plan[1] bytes);
 *   2. xb_gemm_bf16: kv_up = ckv . kv_b_proj^T;
 *   3. attention on the 192 / 128 wgmma prefill kernel. */
int xb_mla_expanded_plan(int64_t* plan8, int batch, int num_heads, const int32_t* qo_lens_host,
                         const int32_t* kv_lens_host);
int xb_mla_prefill_expanded_bf16(const int64_t* plan8, const void* q, int64_t q_stride_t, int64_t q_stride_h,
                                 const void* ckv_cache, int64_t ckv_stride_page, int64_t ckv_stride_token,
                                 const void* kpe_cache, int64_t kpe_stride_page, int64_t kpe_stride_token, int page_size,
                                 const int32_t* kv_indptr, const int32_t* kv_indices, const int32_t* kv_last_page_len,
                                 const int32_t* qo_indptr, const void* kv_b_proj, void* o, int64_t o_stride_t,
                                 int64_t o_stride_h, float sm_scale, void* workspace, int64_t workspace_bytes,
                                 xb_stream_t stream);

/* ---- weight-only / dense linears for small M (decode) ----------------------
 * y[M,N] = x[M,K] . W^T (+ bias).  HBM-bound streaming kernels for M <= 64.
 * (reference: ColumnParallelLinearImpl/RowParallelLinearImpl::forward,
 *  layers/common/linear.cpp:616-716,1405-1522 -> kernels/cuda/matmul.cpp:20-24.)
 *
 * bf16: W is the reference's [N,K] row-major bf16 weight, untouched.
 * w4a16: NEW additive boundary (SURVEY 8b-3; the reference has no weight-only
 *   kernel).  Spec (oracle/quant.py): w[n,k] = bf16( (q[n,k]-z[n,k/g]) * s[n,k/g] )
 *   with q,z in 0..15, s bf16, g = group_size (multiple of 64; 128 default);
 *   y = bf16( sum_k f32(x)*f32(w) (+bias) ), fp32 accumulation.
 *   qweight is the tile-packed layout produced by xb_w4_pack_rows() /
 *   xllm_b200.quant.pack_w4: [N/16][K/64][32 lanes][4] uint32; meta[K/g][N]
 *   uint32 = (bf16 scale) | (bf16(128+zero) << 16). N%16==0, K%64==0. */
int xb_linear_bf16_small_m(void* y, int64_t y_stride, const void* x,
                           int64_t x_stride, const void* w, const void* bias,
                           int M, int N, int K, xb_stream_t stream);
int xb_linear_w4a16_small_m(void* y, int64_t y_stride, const void* x,
                            int64_t x_stride, const uint32_t* qweight,
                            const uint32_t* meta, const void* bias, int M, int N,
                            int K, int group_size, xb_stream_t stream);
/* gate_up_proj with SiLU*mul (or GELU*mul) fused into the epilogue (DenseMLPImpl::forward, dense_mlp.cpp:97-118 =
 * gate_up linear + act_and_mul): qweight / meta / bias rows in the interleaved order of
 * xllm_b200.quant.interleave_gate_up (per 16-row tile 8 gate rows then the matching 8 up rows); y [M, N/2]; M <= 16.
 * Same rounding ladder as the two separate ops (both linear outputs -> bf16, bf16(act(gate)) * up -> bf16). */
int xb_linear_w4a16_gate_up_act_small_m(void* y, int64_t y_stride, const void* x, int64_t x_stride,
                                        const uint32_t* qweight, const uint32_t* meta,
                                        const void* bias, int M, int N, int K, int group_size,
                                        int act_mode, xb_stream_t stream);
/* decode-step form of a weight-only linear (M <= 8): the work the step does right before and after the GEMV rides in
 * the same launch (north-star "RMSNorm+RoPE as a single fused epilogue"):
 *   prologue  norm_weight != NULL: x := RMSNorm(x (+ residual_in)) * norm_weight  (fused_add_rms_norm / rms_norm,
 *             xllm/core/kernels/cuda/norm.cu:43-136); residual_out (may be NULL, must not alias residual_in)
 *             receives the updated residual stream.  stage_x != 0 stages x in shared memory without a norm.
 *   epilogue  0: +bias; 1: act(gate)*up on interleaved rows, y [M, N/2] (activation.cu:45-130);
 *             2: qkv_proj: +bias, NeoX RoPE on q / k heads (rope.cu:27-137) and scatter of the new k / v rows into
 *                the paged caches (reshape_paged_cache.cu:23-62); weight rows packed by quant.pack_w4_qkv_rope;
 *                y [M, N] in logical [q | k | v] order.
 *             3: row-parallel projection (o_proj / down_proj) as the PRODUCER of a split RMSNorm:
 *                r = bf16(bf16(y) + residual_in) -> residual_out, per-(16-row tile, token) sums of r^2 ->
 *                norm_stats_out [N/16][8] f32 (fixed order, no atomics); y is not written.
 *   split norm consumer: norm_stats_in != NULL (with norm_weight): x is the residual stream r, the K/16 partials are
 *             summed in a fixed order and x is normalised while it is staged - one L2 round trip in the prologue.
 * xb_linear_w4a16_decode_fused_fits(M, K) tells whether the [M, K] activation block fits the shared-memory stage. */
int xb_linear_w4a16_decode_fused(void* y, int64_t y_stride, const void* x, int64_t x_stride,
                                 const uint32_t* qweight, const uint32_t* meta, const void* bias,
                                 int M, int N, int K, int group_size, const void* norm_weight, float eps,
                                 const void* residual_in, void* residual_out, int stage_x, int epilogue,
                                 int act_mode, const int64_t* positions, const void* cos_sin_cache,
                                 const int32_t* slot_ids, void* k_cache, void* v_cache, int num_heads,
                                 int num_kv_heads, int head_dim, const float* norm_stats_in,
                                 float* norm_stats_out, xb_stream_t stream);
int xb_linear_w4a16_decode_fused_fits(int M, int K);
/* additive (the reference has no weight-only kernel, SURVEY 8b-3).  Arithmetic form of the W4A16 decode kernels (M <= 8; group_size
 * 64 / 128), both defined in oracle/quant.py:
 *   0  bf16-weight form: w = bf16((q - z) * s) per weight, then the bf16 linear (what the wgmma prefill GEMM computes)
 *   1  exact-dequant form: y = bf16(sum_g s_g * sum_{k in g} x_k (q_k - z_g) + b), fp32 - the integer nibbles go to the
 *      tensor core unscaled and scale / zero are applied once per (row, group); differs from form 0 only by the bf16
 *      rounding of w that form 0 makes (<= 2^-9 relative per weight).
 * Returns the previous form. */
int xb_set_w4_decode_form(int form);

/* ---- W8A16 weight-only linears (north-star "W4A16 / W8A16 / FP8"; additive boundary, SURVEY 8b-3) -------------
 * spec oracle/quant.py with bits = 8: w = bf16((q - z) * s), y = bf16(sum_k f32(x) f32(w) + b).
 * qweight: tile-packed bytes [N/16][K/64][32 lanes][8 words] (xb_w8_pack_rows / quant.pack_w8): lane 4g+t holds rows
 * n0+g (words 0..3) and n0+g+8 (words 4..7), k in [k0+16t, k0+16t+16) ascending; meta [K/g][N] = bf16 scale | zero<<16.
 * xb_linear_w8a16_small_m: M <= 64 streaming kernel (decode); xb_gemm_w8a16: wgmma GEMM with the int8 -> bf16
 * unpack fused into the MMA main loop (prefill). */
int xb_linear_w8a16_small_m(void* y, int64_t y_stride, const void* x, int64_t x_stride,
                            const uint32_t* qweight, const uint32_t* meta, const void* bias,
                            int M, int N, int K, int group_size, xb_stream_t stream);
int xb_gemm_w8a16(void* c, int64_t ldc, const void* a, int64_t lda, const uint32_t* qweight,
                  const uint32_t* meta, const void* bias, int M, int N, int K, int group_size,
                  xb_stream_t stream);
int xb_w8_pack_rows(uint32_t* out, const uint8_t* q, int N, int K);

/* ---- FP8 W8A8 small-M (decode) --------------------------------------------------------------------------------
 * cutlass_scaled_mm for M <= 64 (the reference buckets M <= 16 / <= 64 into swap-AB tiles:
 * cutlass_w8a8/c3x/scaled_mm_sm100_fp8_dispatch.cuh:148-287): c [M,N] bf16 = a_s * (b_s * (a . b^T)) + bias,
 * a [M,K] e4m3 (lda bytes), b [N,K] e4m3 dense (the reference's weight layout), scales f32 with numel 1 or M / N.
 * HBM-streaming kernel: weight rows in the M slot of mma.sync m16n8k32.e4m3, tokens in the n8 slot. */
int xb_linear_fp8_small_m(void* c, int64_t ldc, const void* a, int64_t lda, const void* b,
                          const float* a_scale, int a_scale_numel, const float* b_scale,
                          int b_scale_numel, const void* bias, int M, int N, int K,
                          xb_stream_t stream);

/* additive (arithmetic of activation.cu:97-125): act_and_mul over that interleaved column layout (prefill path sharing the same
 * packed weight):
 * out[t, 8j+i] = act(x[t, 16j+i]) * x[t, 16j+8+i]. */
int xb_act_and_mul_interleaved8_bf16(void* out, const void* input, int d, int num_tokens,
                                     int act_mode, xb_stream_t stream);
/* additive, host-side packer (plain C, no CUDA; layout spec: oracle/quant.py, SURVEY 8b-3): q[N,K] uint8 (0..15) -> qweight tiles. */
int xb_w4_pack_rows(uint32_t* qweight_out, const uint8_t* q, int N, int K);

/* ---- K3 / K2: prefill and chunked-prefill attention (wgmma + TMA) ------------------------------------
 * ragged: replaces the FlashInfer `ragged_run` module behind xllm::kernel::cuda::batch_prefill
 *   (cuda_ops_api.h:52-66, batch_prefill.cpp:21-163): q [total_q, Hq, D], k/v [total_kv, Hkv, D] contiguous ragged,
 *   q_cu_seq_lens / kv_cu_seq_lens int32 [batch+1] on device, causal self-attention.
 * paged:  replaces `paged_run` behind xllm::kernel::cuda::batch_chunked_prefill (cuda_ops_api.h:110-128,
 *   batch_chunked_prefill.cpp:26-92): ragged q (qo_indptr) over the NHD paged cache [pages, page_size, Hkv, D]
 *   (contiguous) with the paged triplet; causal => query i of a chunk sees kv_idx <= kv_len - qo_len + i.
 * o [total_q, Hq, D] bf16; lse optional [total_q, Hq] f32 (base 2).  max_qo_len: host upper bound of the longest
 * request's query length (grid sizing; the reference planner has it from qo_indptr_host). head_dim 64 | 128. */
int xb_prefill_ragged_bf16(const void* q, int64_t q_stride_n, int64_t q_stride_h,
                           const void* k, const void* v, int64_t kv_stride_n,
                           const int32_t* q_cu_seq_lens, const int32_t* kv_cu_seq_lens,
                           void* o, int64_t o_stride_n, int64_t o_stride_h, float* lse,
                           int batch, int64_t total_q, int64_t total_kv, int max_qo_len,
                           int num_qo_heads, int num_kv_heads, int head_dim, int causal,
                           float sm_scale, xb_stream_t stream);
int xb_prefill_paged_bf16(const void* q, int64_t q_stride_n, int64_t q_stride_h,
                          const void* k_cache, const void* v_cache, int64_t num_pages,
                          int page_size, const int32_t* qo_indptr, const int32_t* kv_indptr,
                          const int32_t* kv_indices, const int32_t* kv_last_page_len,
                          void* o, int64_t o_stride_n, int64_t o_stride_h, float* lse,
                          int batch, int64_t total_q, int max_qo_len, int num_qo_heads,
                          int num_kv_heads, int head_dim, int causal, float sm_scale,
                          xb_stream_t stream);
/* split-KV form of paged_run for a short query chunk over a long KV (the reference's planner decides split_kv,
 * layers/cuda/flashinfer_planinfo.cpp:168-247): the kv tiles of every (q tile, kv head, request) are divided over
 * kv_splits CTAs, fp32 partials + LSEs go to workspace_f32 (xb_prefill_split_workspace_bytes) and a merge kernel
 * finishes.  xb_prefill_plan_splits is the host-side decision (pure arithmetic); kv_splits == 1 is xb_prefill_paged_bf16. */
int xb_prefill_paged_split_bf16(const void* q, int64_t q_stride_n, int64_t q_stride_h,
                                const void* k_cache, const void* v_cache, int64_t num_pages,
                                int page_size, const int32_t* qo_indptr, const int32_t* kv_indptr,
                                const int32_t* kv_indices, const int32_t* kv_last_page_len, void* o,
                                int64_t o_stride_n, int64_t o_stride_h, float* lse, int batch,
                                int64_t total_q, int max_qo_len, int num_qo_heads, int num_kv_heads,
                                int head_dim, int causal, float sm_scale, int kv_splits,
                                void* workspace_f32, int64_t workspace_bytes, xb_stream_t stream);
int64_t xb_prefill_split_workspace_bytes(int kv_splits, int64_t total_q, int num_qo_heads, int head_dim);
int xb_prefill_plan_splits(int batch, int max_qo_len, int64_t max_kv_len, int num_qo_heads,
                           int num_kv_heads, int num_sms);

/* ---- wgmma GEMMs for prefill-sized M (any M; TMA zero-fills ragged edges) -----------------------
 * C[M,N] = A[M,K] . B[N,K]^T (+ bias), fp32 accumulation in registers, bf16 output.
 * bf16:  replaces xllm::kernel::cuda::matmul (cuda_ops_api.h:167-169, matmul.cpp:20-24 -> F::linear).
 * fp8:   replaces xllm::kernel::cuda::cutlass_scaled_mm (cuda_ops_api.h:171-176,
 *        cutlass_w8a8/scaled_mm_entry.cu:55-108): a,b e4m3 [M,K] / [N,K] (b is the reference's b.t() view),
 *        C = a_scale * (b_scale * acc) (+ bias); scales fp32 with numel 1 (per-tensor) or M / N.
 * w4a16: the weight-only GEMM (SURVEY 8b-3): same packed operands as xb_linear_w4a16_small_m, int4->bf16
 *        unpack fused into the wgmma main loop. */
int xb_gemm_bf16(void* c, int64_t ldc, const void* a, int64_t lda, const void* b,
                 const void* bias, int M, int N, int K, xb_stream_t stream);
int xb_gemm_fp8_scaled(void* c, int64_t ldc, const void* a_e4m3, int64_t lda,
                       const void* b_e4m3, const float* a_scale, int a_scale_numel,
                       const float* b_scale, int b_scale_numel, const void* bias,
                       int M, int N, int K, xb_stream_t stream);
int xb_gemm_w4a16(void* c, int64_t ldc, const void* a, int64_t lda,
                  const uint32_t* qweight, const uint32_t* meta, const void* bias,
                  int M, int N, int K, int group_size, xb_stream_t stream);
/* xb_gemm_fp8_scaled with M <= max_m (<= 64) runs swap-AB: the weight rows take the 128-row MMA M slot and the tokens the
 * N tile (what the reference's M <= 16 / M <= 64 buckets of its fp8 dispatch do), so a
 * decode-sized batch streams every weight tile on its own CTA.  0 = never.  Returns the old value. */
int xb_set_fp8_swap_max_m(int max_m);
/* split-K for the swap-AB FP8 GEMM: a decode-sized GEMM has only N/128 weight tiles (10 for a TP8 qkv shard of Llama-3-70B), so
 * each tile's K is cut into up to `max_split` ranges walked by different CTAs; fp32 partials meet in a caller-owned workspace
 * and the last CTA to arrive sums them in split order (bit-reproducible) and runs the epilogue.  Off until a workspace of
 * xb_gemm_splitk_workspace_bytes() is registered (the library never allocates); the first 4 KB are zeroed by the setter
 * (cudaMemset: call it outside stream capture) and reset themselves afterwards, so CUDA-graph replays need no memset.
 * Launches that share the workspace must be stream-ordered.  ws = NULL switches split-K off again. */
size_t xb_gemm_splitk_workspace_bytes(void);
int xb_set_gemm_splitk_workspace(void* ws, size_t bytes);
/* host-only query (no device needed): k ranges xb_gemm_fp8_scaled uses for [M,K] x [N,K]^T on a device with sm_count SMs once a
 * workspace is registered (1 = unsplit): fill the SMs once, >= 12 k blocks of 128 per range, no empty range. */
int xb_gemm_fp8_split_k(int M, int N, int K, int sm_count);
/* host-only (no device needed): the kernel variant the GEMM entry points pick for a shape, as text ("bf16 bn=128",
 * "fp8 swap-AB bn=32 split_k=5", "w4 bn=64").  kind: 0 bf16 | 1 fp8 | 2 w4a16 | 3 w8a16.  Returns the length, -1 on a bad
 * kind.  For capacity planning and the dispatch tests (tests/test_splitk_host_cpu.py). */
int xb_gemm_describe(int kind, int M, int N, int K, int sm_count, char* buf, int buf_len);
int xb_set_fp8_splitk_max(int max_split);   /* 1 = never split .. 32; default 8 (XB_FP8_SPLITK_MAX); returns the old value */

/* ---- tensor-parallel exchange over NVLink peer memory (decode-sized messages) ---------------------------------
 * replaces parallel_state::reduce -> ProcessGroup::allreduce (framework/parallel_state/parallel_state.cpp:183-192,
 * process_group.cpp:97-107) after the row-parallel linears (layers/common/linear.cpp:1518-1520).
 * peer_data[r] / peer_flags[r]: device pointers, valid on THIS GPU, to rank r's symmetric partial buffer and signal
 * pad ([max_ctas][8] uint32, zero-initialised once); epoch: local uint32[max_ctas], zero-initialised once.
 * Sum order is rank 0..world-1 in fp32, one rounding: bit-identical on all ranks.
 * out / residual / weight / peer_data[r] must be 16-byte aligned, peer_flags[r] / epoch 4-byte aligned; numel >= 0,
 * max_ctas >= 1, 0 < hidden <= 16384, 0 <= num_tokens <= max_ctas.  Anything else is refused before any launch.
 * xb_allreduce_add_rms_norm_bf16 fuses the exchange with the fused_add_rms_norm that follows every row-parallel
 * linear: residual <- bf16(allreduce(partials)) + residual; out <- rms_norm(residual) * weight. */
int xb_oneshot_allreduce_bf16(void* out, const void* const* peer_data, void* const* peer_flags,
                              void* epoch, int rank, int world, int64_t numel, int max_ctas,
                              xb_stream_t stream);
int xb_allreduce_add_rms_norm_bf16(void* out, void* residual, const void* weight,
                                   const void* const* peer_data, void* const* peer_flags,
                                   void* epoch, int rank, int world, float eps, int num_tokens,
                                   int hidden, int max_ctas, xb_stream_t stream);

/* ---- step boundary helpers ---------------------------------------------------
 * embedding row gather (WordEmbeddingImpl::forward, layers/common/word_embedding_impl.cpp:33-56,
 * TP=1) and greedy argmax over logits rows (ties -> lowest index). */
int xb_embedding_bf16(void* out, const int32_t* token_ids, const void* table,
                      int num_tokens, int hidden, int vocab, xb_stream_t stream);
int xb_argmax_bf16(int32_t* out, const void* logits, int64_t stride, int rows,
                   int vocab, xb_stream_t stream);

/* ---- Mixture of experts (SURVEY 8f n4) ------------------------------------------------------------------------------------
 * xb_moe_fused_topk replaces xllm::kernel::cuda::moe_fused_topk (cuda_ops_api.h:251-256, moe/moe_fused_topk.cu:22-58):
 *   gating_output [T, E] fp32 or bf16 (row stride in elements), scoring softmax (scoring_sigmoid = 0) or sigmoid with an
 *   optional fp32 correction bias [E] (added for the selection, subtracted from the returned weight), top-k with ties to the
 *   lower expert index, optional renormalisation by the sum of the selected weights; outputs topk_weights fp32 [T, k],
 *   topk_ids int32 [T, k].  E <= 512, k <= 32.
 * xb_moe_experts_bf16 replaces xllm::kernel::cuda::cutlass_fused_moe (cuda_ops_api.h:260-289, moe/fused_moe.cpp:23-124) for
 *   unquantised bf16 experts (all the reference's CUDA FusedMoE accepts, layers/cuda/fused_moe.cpp:39-42): fc1 [E_local, 2I, H]
 *   in [up | gate] row order, fc2 [E_local, H, I]; out[t] = bf16(sum_k scale[t,k] * bf16(fc2_e . bf16(silu(gate) * up))).
 *   Experts outside [expert_begin, expert_begin + num_local_experts) contribute zero, whatever the id, negative ids included
 *   (expert parallelism: the caller all-reduces, layers/cuda/fused_moe.cpp:116-117).
 * The expert entries take one of two paths by the token count T alone (P = T * topk pairs):
 *   T <= 64 (decode): one expert-indexed GEMV per pair, each streaming its expert's weights; P <= 65535.
 *   T >= 65 (prefill): the local pairs are sorted by expert on the device (stable), their input rows gathered, and two grouped
 *     wgmma GEMMs over the stacked expert weights run fc1 + SwiGLU and fc2, tensor-core bound; T <= 65535, topk <= 32,
 *     num_local_experts <= 512.  No host synchronisation: one captured CUDA graph replays with any routing.
 * workspace: xb_moe_experts_workspace_bytes(T, topk, H, I) bytes, 16-byte aligned, scratch only (no state between calls):
 *   T <= 64:  P * (I + H) * 2                                         (act, y2)
 *   T >= 65:  8192 + 2 * round_up(4 * P, 256) + P * (2H + I) * 2     (routing header for up to 512 experts, row_of_pair and
 *             pair_of_row maps, the expert-sorted input rows, act, y2)
 * xb_moe_experts_describe (host-only, no device): the path the entries take for a shape, as text ("bf16 gemv",
 *   "w4 grouped bn=128 m_tiles<=40"); kind 0 bf16 | 2 w4a16 (the codes of xb_gemm_describe).  Returns the length, -1 on a bad
 *   kind.  xb_set_moe_grouped_min_tokens: the smallest T that takes the grouped path (>= 1; default 65, env
 *   XB_MOE_GROUPED_MIN_TOKENS), for tests and sweeps; returns the old value, -1 on a bad value. */
int xb_moe_fused_topk(float* topk_weights, int32_t* topk_ids, const void* gating_output, int gating_is_bf16,
                      int64_t gating_stride, const float* correction_bias, int num_tokens, int num_experts, int topk,
                      int renormalize, int scoring_sigmoid, xb_stream_t stream);
int64_t xb_moe_experts_workspace_bytes(int num_tokens, int topk, int hidden, int inter);
int xb_moe_experts_describe(int kind, int num_tokens, int topk, int hidden, int inter, int num_local_experts, char* buf,
                            int buf_len);
int xb_set_moe_grouped_min_tokens(int min_tokens);
int xb_moe_experts_bf16(void* out, int64_t out_stride, const void* input, int64_t in_stride,
                        const int32_t* token_selected_experts, const float* token_final_scales,
                        const void* fc1_weights, const void* fc2_weights, int num_tokens, int topk, int hidden,
                        int inter, int num_local_experts, int expert_begin, void* workspace,
                        int64_t workspace_bytes, xb_stream_t stream);

/* W4A16 experts (BASELINE configs[4] "MoE W4A16"; additive like the dense weight-only linears): per expert the tile-packed
 * int4 layout of xb_linear_w4a16_small_m - fc1 qweight [E_local, 2I/16, H/64, 32, 4] u32 + meta [E_local, H/g, 2I] u32 (rows
 * [up | gate]), fc2 qweight [E_local, H/16, I/64, 32, 4] + meta [E_local, I/g, H]; same arithmetic and the same two paths as
 * xb_moe_experts_bf16 on the dequantised weights w = bf16((q - z) * s).  The grouped path also needs 16-byte aligned meta. */
int xb_moe_experts_w4a16(void* out, int64_t out_stride, const void* input, int64_t in_stride,
                         const int32_t* token_selected_experts, const float* token_final_scales,
                         const uint32_t* fc1_qweight, const uint32_t* fc1_meta, const uint32_t* fc2_qweight,
                         const uint32_t* fc2_meta, int group_size, int num_tokens, int topk, int hidden, int inter,
                         int num_local_experts, int expert_begin, void* workspace, int64_t workspace_bytes,
                         xb_stream_t stream);

/* ---- CUDA-graph decode metadata refresh (SURVEY 8f n3) ---------------------------------------------------------------
 * replaces xllm::kernel::cuda::update_llm_decode_metadata (kernels/cuda/llm_decode_metadata_update.h:35-58,
 * llm_decode_metadata_update.cu:29-96; caller runtime/cuda_graph_executor_impl.cpp:218-258): same fields, same padding
 * rule (tokens / slots of rows actual..padded are zeroed, positions are left), kv_seq_lens_delta[i] = kv_seq_lens[i+1] -
 * kv_seq_lens[i].  plan_counters / n_counter_words (optional): the int workspace words of this library's decode plan to
 * re-zero in the same launch - with them the host-side `plan` the reference re-runs before every replay
 * (cuda_graph_executor_impl.cpp:751-822) is not needed for this library's attention modules: their split geometry is
 * derived on the device from the refreshed paged triplet. */
int xb_decode_metadata_update(const int32_t* src_tokens, const int32_t* src_positions,
                              const int32_t* src_new_cache_slots, const int32_t* src_kv_seq_lens,
                              const int32_t* src_paged_kv_indptr, const int32_t* src_paged_kv_indices,
                              const int32_t* src_paged_kv_last_page_len, int32_t* dst_tokens,
                              int32_t* dst_positions, int32_t* dst_new_cache_slots, int32_t* dst_kv_seq_lens,
                              int32_t* dst_kv_seq_lens_delta, int32_t* dst_paged_kv_indptr,
                              int32_t* dst_paged_kv_indices, int32_t* dst_paged_kv_last_page_len,
                              int64_t actual_num_tokens, int64_t padded_num_tokens, int64_t actual_batch_size,
                              int64_t actual_indices_size, int32_t* plan_counters, int64_t n_counter_words,
                              xb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* XLLM_B200_OPS_H_ */
