// HBM-bound elementwise ops between the linears and attention:
//   K7/K8 RMSNorm(+residual)(+static FP8 quant), K6 FP8 quant, K9 RoPE,
//   K12 KV scatter, K9+K12 fused, K10 QK-norm+RoPE, K10+K12 fused, K11 act_and_mul.
// Rounding order follows the reference kernels exactly (see each kernel).
// All kernels: 16-byte vectorised accesses, one CTA (or a few warps) per token,
// PDL-aware (griddepcontrol) so they chain inside a CUDA graph without bubbles.
#include <type_traits>

#include "common.cuh"

namespace xb {

// ---------------------------------------------------------------------------
// RMSNorm family.  Reference: xllm/core/kernels/cuda/norm.cu
//   rms_norm_kernel                         :43-78
//   fused_add_rms_norm_kernel (width 8)     :80-136
//   rms_norm_static_fp8_quant_kernel        :228-270
//   fused_add_rms_norm_static_fp8_quant     :283-345 (width 8), :350-396 generic
// kVec: 8 bf16 per thread per step, row kept in registers (<= kMaxVec steps),
// otherwise re-read from L2 (rows > 16K elements).
// ---------------------------------------------------------------------------

template <bool kFusedAdd, bool kFp8Out, bool kRoundBeforeFp8>
__global__ void __launch_bounds__(1024)
rms_norm_vec_kernel(void* __restrict__ out_, __nv_bfloat16* __restrict__ input,
                    int64_t input_stride, __nv_bfloat16* __restrict__ residual,
                    const __nv_bfloat16* __restrict__ weight,
                    const float* __restrict__ fp8_scale, float eps,
                    int hidden_size) {
  constexpr int kMaxVec = 2;
  __shared__ float red[33];
  const int64_t tok = blockIdx.x;
  const int nvec = hidden_size >> 3;
  uint4* in_v = reinterpret_cast<uint4*>(input + tok * input_stride);
  uint4* res_v = kFusedAdd ? reinterpret_cast<uint4*>(residual + tok * (int64_t)hidden_size) : nullptr;
  const uint4* w_v = reinterpret_cast<const uint4*>(weight);

  // weights do not depend on the producer kernel: fetch before the PDL wait
  uint4 wreg[kMaxVec];
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    int idx = threadIdx.x + i * blockDim.x;
    if (idx < nvec) wreg[i] = __ldg(w_v + idx);
  }
  pdl_launch_dependents();  // consumer prologues (weight / KV prefetch) may start now
  pdl_wait();

  uint4 xr[kMaxVec];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    int idx = threadIdx.x + i * blockDim.x;
    if (idx < nvec) {
      uint4 x = in_v[idx];
      if (kFusedAdd) {
        x = add_bf16x8(x, res_v[idx]);
        res_v[idx] = x;
      }
      ss = sumsq_bf16x8(ss, x);
      xr[i] = x;
    }
  }
  // tail beyond the register-cached part (very wide rows): accumulate only
  for (int idx = threadIdx.x + kMaxVec * blockDim.x; idx < nvec; idx += blockDim.x) {
    uint4 x = in_v[idx];
    if (kFusedAdd) {
      x = add_bf16x8(x, res_v[idx]);
      res_v[idx] = x;
    }
    ss = sumsq_bf16x8(ss, x);
  }
  const float rstd = rms_rstd(block_sum(ss, red), hidden_size, eps);
  pdl_launch_dependents();

  float inv_scale = 0.f;
  if (kFp8Out) inv_scale = 1.0f / __ldg(fp8_scale);

  auto emit = [&](int idx, const uint4& x, const uint4& w) {
    const uint32_t* xp = &x.x;
    const uint32_t* wp = &w.x;
    if (!kFp8Out) {
      const uint4 o = rms_apply_bf16x8(x, w, rstd);
      uint4* dst = kFusedAdd ? in_v : reinterpret_cast<uint4*>(
                                          reinterpret_cast<__nv_bfloat16*>(out_) + tok * (int64_t)hidden_size);
      dst[idx] = o;
    } else {
      uint8_t q[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float a = rms_norm_x(bf16lo(xp[j]), rstd) * bf16lo(wp[j]);
        float b = rms_norm_x(bf16hi(xp[j]), rstd) * bf16hi(wp[j]);
        if (kRoundBeforeFp8) {  // width-8 fused path rounds to bf16 first (norm.cu:333-343)
          a = round_bf16(a);
          b = round_bf16(b);
        }
        q[2 * j] = scaled_fp8_e4m3(a, inv_scale);
        q[2 * j + 1] = scaled_fp8_e4m3(b, inv_scale);
      }
      uint2* dst = reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(out_) + tok * (int64_t)hidden_size);
      dst[idx] = *reinterpret_cast<uint2*>(q);
    }
  };

#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    int idx = threadIdx.x + i * blockDim.x;
    if (idx < nvec) emit(idx, xr[i], wreg[i]);
  }
  for (int idx = threadIdx.x + kMaxVec * blockDim.x; idx < nvec; idx += blockDim.x) {
    uint4 x = kFusedAdd ? res_v[idx] : in_v[idx];
    emit(idx, x, __ldg(w_v + idx));
  }
}

// scalar fallback (unaligned / hidden % 8 != 0); same rounding, generic kernels
// norm.cu:43-78,139-173,228-270,350-396 (fp8 from the un-rounded fp32 product).
template <bool kFusedAdd, bool kFp8Out>
__global__ void __launch_bounds__(1024)
rms_norm_scalar_kernel(void* __restrict__ out_, __nv_bfloat16* __restrict__ input,
                       int64_t input_stride, __nv_bfloat16* __restrict__ residual,
                       const __nv_bfloat16* __restrict__ weight,
                       const float* __restrict__ fp8_scale, float eps, int hidden_size) {
  __shared__ float red[33];
  const int64_t tok = blockIdx.x;
  __nv_bfloat16* in = input + tok * input_stride;
  __nv_bfloat16* res = kFusedAdd ? residual + tok * (int64_t)hidden_size : nullptr;
  pdl_launch_dependents();  // consumer prologues (weight / KV prefetch) may start now
  pdl_wait();
  float ss = 0.f;
  for (int i = threadIdx.x; i < hidden_size; i += blockDim.x) {
    float x = __bfloat162float(in[i]);
    if (kFusedAdd) {
      x = add_bf16(x, __bfloat162float(res[i]));
      res[i] = __float2bfloat16_rn(x);
    }
    ss += x * x;
  }
  const float rstd = rms_rstd(block_sum(ss, red), hidden_size, eps);
  pdl_launch_dependents();
  float inv_scale = kFp8Out ? 1.0f / __ldg(fp8_scale) : 0.f;
  for (int i = threadIdx.x; i < hidden_size; i += blockDim.x) {
    float x = __bfloat162float(kFusedAdd ? res[i] : in[i]);
    float y = rms_norm_x(x, rstd) * __bfloat162float(weight[i]);
    if (kFp8Out) {
      reinterpret_cast<uint8_t*>(out_)[tok * (int64_t)hidden_size + i] = scaled_fp8_e4m3(y, inv_scale);
    } else if (kFusedAdd) {
      in[i] = __float2bfloat16_rn(y);
    } else {
      reinterpret_cast<__nv_bfloat16*>(out_)[tok * (int64_t)hidden_size + i] = __float2bfloat16_rn(y);
    }
  }
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <bool kFusedAdd, bool kFp8Out>
static int launch_rms_norm(void* out, void* input, int64_t input_stride, void* residual,
                           const void* weight, const float* scale, float eps, int num_tokens,
                           int hidden_size, cudaStream_t stream) {
  if (num_tokens == 0) return 0;
  XB_CHECK(hidden_size > 0 && num_tokens > 0, "rms_norm: bad shape T=%d H=%d", num_tokens, hidden_size);
  const bool vec = (hidden_size % 8 == 0) && (input_stride % 8 == 0) && aligned16(input) &&
                   aligned16(weight) && (!kFusedAdd || aligned16(residual)) &&
                   (kFp8Out ? (reinterpret_cast<uintptr_t>(out) % 8 == 0) : (kFusedAdd || aligned16(out)));
  auto* in = reinterpret_cast<__nv_bfloat16*>(input);
  auto* res = reinterpret_cast<__nv_bfloat16*>(residual);
  auto* w = reinterpret_cast<const __nv_bfloat16*>(weight);
  if (vec) {
    int nvec = hidden_size / 8;
    // smaller CTAs when there are many tokens (more CTAs resident per SM)
    int max_threads = num_tokens < 256 ? 1024 : 256;
    int threads = ((nvec + 31) / 32) * 32;
    if (threads > max_threads) threads = max_threads;
    // the width-8 fused fp8 path rounds through bf16 (norm.cu:333-343); the
    // non-fused fp8 kernel never does (norm.cu:262-268)
    constexpr bool kRound = kFusedAdd && kFp8Out;
    XB_CUDA_OK(launch(rms_norm_vec_kernel<kFusedAdd, kFp8Out, kRound>, dim3(num_tokens), dim3(threads), 0,
                      stream, true, out, in, input_stride, res, w, scale, eps, hidden_size));
  } else {
    int threads = hidden_size < 1024 ? ((hidden_size + 31) / 32) * 32 : 1024;
    XB_CUDA_OK(launch(rms_norm_scalar_kernel<kFusedAdd, kFp8Out>, dim3(num_tokens), dim3(threads), 0, stream,
                      true, out, in, input_stride, res, w, scale, eps, hidden_size));
  }
  return 0;
}

// ---------------------------------------------------------------------------
// K6 static / dynamic FP8 quant.  fp8_quant.cu:78-153, fp8_scaled_quantize.cpp:36-41
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
fp8_quant_kernel(uint8_t* __restrict__ out, int64_t out_stride, const __nv_bfloat16* __restrict__ in,
                 int64_t in_stride, const float* __restrict__ scale, int hidden_size, bool vec) {
  const int64_t tok = blockIdx.x;
  pdl_launch_dependents();  // consumer prologues (weight / KV prefetch) may start now
  pdl_wait();
  const float inv_scale = 1.0f / __ldg(scale);
  const __nv_bfloat16* src = in + tok * in_stride;
  uint8_t* dst = out + tok * out_stride;
  if (vec) {
    const uint4* sv = reinterpret_cast<const uint4*>(src);
    uint2* dv = reinterpret_cast<uint2*>(dst);
    for (int i = threadIdx.x; i < hidden_size / 8; i += blockDim.x) {
      uint4 x = sv[i];
      const uint32_t* xp = &x.x;
      uint8_t q[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        q[2 * j] = scaled_fp8_e4m3(bf16lo(xp[j]), inv_scale);
        q[2 * j + 1] = scaled_fp8_e4m3(bf16hi(xp[j]), inv_scale);
      }
      dv[i] = *reinterpret_cast<uint2*>(q);
    }
  } else {
    for (int i = threadIdx.x; i < hidden_size; i += blockDim.x)
      dst[i] = scaled_fp8_e4m3(__bfloat162float(src[i]), inv_scale);
  }
  pdl_launch_dependents();
}

// amax over the whole tensor -> scale_out[0] = max(amax/448, 1e-12).
// Two tiny launches (init + atomicMax on the non-negative float bit pattern).
__global__ void fp8_scale_init_kernel(float* scale_out) { scale_out[0] = 0.f; }
__global__ void __launch_bounds__(256)
fp8_amax_kernel(const __nv_bfloat16* __restrict__ in, int64_t in_stride, int hidden_size, float* amax_bits) {
  __shared__ float red[33];
  const __nv_bfloat16* src = in + (int64_t)blockIdx.x * in_stride;
  float m = 0.f;
  for (int i = threadIdx.x; i < hidden_size; i += blockDim.x) m = fmaxf(m, fabsf(__bfloat162float(src[i])));
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_max(t);
    if (threadIdx.x == 0) atomicMax(reinterpret_cast<int*>(amax_bits), __float_as_int(t));
  }
}
__global__ void fp8_scale_finish_kernel(float* scale_out) {
  // (amax / 448).clamp_min(1e-12) evaluated in bf16 like the reference's 0-dim bf16 tensor math
  scale_out[0] = fmaxf(round_bf16(scale_out[0] / 448.0f), round_bf16(1e-12f));
}

// ---------------------------------------------------------------------------
// K9 rotary embedding.  rope.cu:27-137: scalar_t arithmetic => every product
// and the final add/sub are rounded to bf16 (rope_pair).
// ---------------------------------------------------------------------------

template <bool kNeox>
__global__ void __launch_bounds__(512)
rotary_embedding_kernel(const int64_t* __restrict__ positions, __nv_bfloat16* __restrict__ query,
                        __nv_bfloat16* __restrict__ key, const __nv_bfloat16* __restrict__ cos_sin_cache,
                        int rot_dim, int64_t query_stride, int64_t key_stride, int64_t head_stride,
                        int num_heads, int num_kv_heads) {
  const int64_t tok = blockIdx.x;
  pdl_launch_dependents();  // consumer prologues (weight / KV prefetch) may start now
  pdl_wait();
  const int64_t pos = positions[tok];
  const __nv_bfloat16* cache = cos_sin_cache + pos * rot_dim;
  const int embed = rot_dim / 2;
  const int nq = num_heads * embed;
  const int nk = key ? num_kv_heads * embed : 0;
  for (int i = threadIdx.x; i < nq + nk; i += blockDim.x) {
    const bool is_k = i >= nq;
    const int j = is_k ? i - nq : i;
    const int head = j / embed, r = j % embed;
    __nv_bfloat16* arr = (is_k ? key + tok * key_stride : query + tok * query_stride) + head * head_stride;
    const float c = __bfloat162float(cache[r]);
    const float s = __bfloat162float(cache[embed + r]);
    if (kNeox) rope_pair(arr, r, embed + r, c, s);
    else rope_pair(arr, 2 * r, 2 * r + 1, c, s);
  }
  pdl_launch_dependents();
}

// ---------------------------------------------------------------------------
// K12 KV scatter.  reshape_paged_cache.cu:23-62.  16-byte copies when aligned.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
reshape_paged_cache_kernel(const int32_t* __restrict__ slot_ids, const __nv_bfloat16* __restrict__ keys,
                           const __nv_bfloat16* __restrict__ values, __nv_bfloat16* __restrict__ key_cache,
                           __nv_bfloat16* __restrict__ value_cache, int64_t k_stride, int64_t v_stride,
                           int row_elems /* n_kv_heads*head_dim */, bool vec) {
  const int64_t tok = blockIdx.x;
  pdl_launch_dependents();  // consumer prologues (weight / KV prefetch) may start now
  pdl_wait();
  const int64_t slot = slot_ids[tok];
  if (slot < 0) return;
  // cache row of a slot: [block, offset] flattened == slot * row_elems
  const int64_t dst = slot * row_elems;
  if (vec) {
    const uint4* ks = reinterpret_cast<const uint4*>(keys + tok * k_stride);
    const uint4* vs = reinterpret_cast<const uint4*>(values + tok * v_stride);
    uint4* kd = reinterpret_cast<uint4*>(key_cache + dst);
    uint4* vd = reinterpret_cast<uint4*>(value_cache + dst);
    for (int i = threadIdx.x; i < row_elems / 8; i += blockDim.x) {
      kd[i] = ks[i];
      vd[i] = vs[i];
    }
  } else {
    for (int i = threadIdx.x; i < row_elems; i += blockDim.x) {
      key_cache[dst + i] = keys[tok * k_stride + i];
      value_cache[dst + i] = values[tok * v_stride + i];
    }
  }
  pdl_launch_dependents();
}

// ---------------------------------------------------------------------------
// K9+K12 fused: rotate q and k in place, then scatter rotated k and v.
// One CTA per token; thread i owns rotation pair i so no intra-CTA hazard
// between the rotate and the copy of k (each pair is copied by its owner).
// ---------------------------------------------------------------------------
template <bool kNeox>
__global__ void __launch_bounds__(512)
rope_and_cache_kernel(const int64_t* __restrict__ positions, __nv_bfloat16* __restrict__ query,
                      __nv_bfloat16* __restrict__ key, const __nv_bfloat16* __restrict__ value,
                      const __nv_bfloat16* __restrict__ cos_sin_cache, const int32_t* __restrict__ slot_ids,
                      __nv_bfloat16* __restrict__ key_cache, __nv_bfloat16* __restrict__ value_cache,
                      int rot_dim, int64_t query_stride, int64_t key_stride, int64_t value_stride,
                      int num_heads, int num_kv_heads, int head_size) {
  const int64_t tok = blockIdx.x;
  pdl_launch_dependents();  // consumer prologues (weight / KV prefetch) may start now
  pdl_wait();
  const int64_t pos = positions[tok];
  const int64_t slot = slot_ids[tok];
  const __nv_bfloat16* cache = cos_sin_cache + pos * rot_dim;
  const int embed = rot_dim / 2;
  const int nq = num_heads * embed, nk = num_kv_heads * embed;
  const int row_elems = num_kv_heads * head_size;
  __nv_bfloat16* kc = key_cache + slot * row_elems;
  __nv_bfloat16* vc = value_cache + slot * row_elems;
  for (int i = threadIdx.x; i < nq + nk; i += blockDim.x) {
    const bool is_k = i >= nq;
    const int j = is_k ? i - nq : i;
    const int head = j / embed, r = j % embed;
    __nv_bfloat16* arr = (is_k ? key + tok * key_stride : query + tok * query_stride) + (int64_t)head * head_size;
    const float c = __bfloat162float(cache[r]);
    const float s = __bfloat162float(cache[embed + r]);
    const int xi = kNeox ? r : 2 * r, yi = kNeox ? embed + r : 2 * r + 1;
    rope_pair(arr, xi, yi, c, s);
    if (is_k && slot >= 0) {
      kc[head * head_size + xi] = arr[xi];
      kc[head * head_size + yi] = arr[yi];
    }
  }
  if (slot >= 0) {
    // un-rotated tail of k (rot_dim < head_size) and all of v
    if (rot_dim < head_size) {
      const int tail = head_size - rot_dim;
      for (int i = threadIdx.x; i < num_kv_heads * tail; i += blockDim.x) {
        const int head = i / tail, d = rot_dim + i % tail;
        kc[head * head_size + d] = key[tok * key_stride + head * head_size + d];
      }
    }
    const __nv_bfloat16* vs = value + tok * value_stride;
    if ((row_elems % 8 == 0) && (value_stride % 8 == 0) && ((reinterpret_cast<uintptr_t>(value) & 15) == 0) &&
        ((reinterpret_cast<uintptr_t>(value_cache) & 15) == 0)) {
      const uint4* sv = reinterpret_cast<const uint4*>(vs);
      uint4* dv = reinterpret_cast<uint4*>(vc);
      for (int i = threadIdx.x; i < row_elems / 8; i += blockDim.x) dv[i] = sv[i];
    } else {
      for (int i = threadIdx.x; i < row_elems; i += blockDim.x) vc[i] = vs[i];
    }
  }
  pdl_launch_dependents();
}

// ---------------------------------------------------------------------------
// K9+K12 on a qkv projection whose output columns are in the ROPE-PAIR packed order of quant.pack_w4_qkv_rope (inside
// every head, packed column 16j+i holds dim 8j+i for i < 8 and dim D/2 + 8j + (i-8) otherwise): the decode GEMV
// applies RoPE + scatter in its own epilogue; this kernel serves the same weights when the projection ran as a plain
// GEMM (prefill, decode batches > 8).  Reads the packed row, writes q / k / v in LOGICAL order to qkv_out and the new
// k / v rows into the paged caches, with the GEMV epilogue's qkv_rope_store.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(512)
rope_and_cache_packed_kernel(const int64_t* __restrict__ positions, const __nv_bfloat16* __restrict__ qkv_packed,
                             int64_t in_stride, __nv_bfloat16* __restrict__ qkv_out, int64_t out_stride,
                             const __nv_bfloat16* __restrict__ cos_sin_cache, const int32_t* __restrict__ slot_ids,
                             __nv_bfloat16* __restrict__ key_cache, __nv_bfloat16* __restrict__ value_cache,
                             int num_heads, int num_kv_heads, int head_size) {
  const int64_t tok = blockIdx.x;
  pdl_launch_dependents();
  pdl_wait();
  const QkvRopeCache p{positions, cos_sin_cache, slot_ids, key_cache, value_cache, num_heads, num_kv_heads, head_size};
  const __nv_bfloat16* in = qkv_packed + tok * in_stride;
  const int pairs = (num_heads + 2 * num_kv_heads) * (head_size >> 1);
  for (int i = threadIdx.x; i < pairs; i += blockDim.x) {
    const int nt = i >> 3, r = i & 7;   // packed columns 16 nt + r and 16 nt + r + 8
    qkv_rope_store(p, qkv_out, out_stride, (int)tok, nt, r, __bfloat162float(in[16 * nt + r]),
                   __bfloat162float(in[16 * nt + r + 8]));
  }
  pdl_launch_dependents();
}

// ---------------------------------------------------------------------------
// K10 fused per-head RMSNorm(q,k) + RoPE (Qwen3).  fused_qknorm_rope.cu:84-300:
// one warp per (token, head); fp32 norm: x*rstd*w kept in fp32, RoPE in fp32,
// single rounding to bf16 at the store.
// ---------------------------------------------------------------------------
template <int kHeadDim, bool kInterleave>
__global__ void __launch_bounds__(256)
fused_qk_norm_rope_kernel(__nv_bfloat16* __restrict__ qkv, int num_heads_q, int num_heads_k, int num_heads_v,
                          float eps, const __nv_bfloat16* __restrict__ q_weight,
                          const __nv_bfloat16* __restrict__ k_weight,
                          const __nv_bfloat16* __restrict__ cos_sin_cache, int rot_dim,
                          const int64_t* __restrict__ position_ids, int num_tokens) {
  constexpr int kPerLane = kHeadDim / 32;
  const int warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int heads_qk = num_heads_q + num_heads_k;
  const int tok = warp_global / heads_qk;
  const int head = warp_global % heads_qk;
  if (tok >= num_tokens) return;
  pdl_launch_dependents();  // consumer prologues (weight / KV prefetch) may start now
  pdl_wait();
  const bool is_q = head < num_heads_q;
  const int total_heads = num_heads_q + num_heads_k + num_heads_v;
  __nv_bfloat16* ptr = qkv + ((int64_t)tok * total_heads + head) * kHeadDim;
  const __nv_bfloat16* w = is_q ? q_weight : k_weight;
  float e[kPerLane], wf[kPerLane];
  // lane owns kPerLane consecutive elements
#pragma unroll
  for (int i = 0; i < kPerLane; ++i) {
    e[i] = __bfloat162float(ptr[lane * kPerLane + i]);
    wf[i] = __bfloat162float(w[lane * kPerLane + i]);
  }
  qk_norm_rope_warp<kHeadDim, kInterleave>(e, wf, eps, cos_sin_cache + position_ids[tok] * rot_dim, rot_dim, lane);
#pragma unroll
  for (int i = 0; i < kPerLane; ++i) ptr[lane * kPerLane + i] = __float2bfloat16_rn(e[i]);
  pdl_launch_dependents();
}

// ---------------------------------------------------------------------------
// K10+K12 fused (Qwen3): per-head RMSNorm + NeoX RoPE of q and k in place, then the normalised, rotated k row and the
// untouched v row into the NHD paged caches (slot < 0: no cache write).  One warp per (token, head) over
// Hq + 2 Hkv heads; v-head warps only copy.  Norm + RoPE are qk_norm_rope_warp and the store rounds once, as
// fused_qk_norm_rope_kernel does, so qkv and both caches are bit-identical to K10 followed by K12.
// ---------------------------------------------------------------------------
template <int kHeadDim>
__global__ void __launch_bounds__(256)
qk_norm_rope_and_cache_kernel(__nv_bfloat16* __restrict__ qkv, int num_heads_q, int num_heads_kv, float eps,
                              const __nv_bfloat16* __restrict__ q_weight, const __nv_bfloat16* __restrict__ k_weight,
                              const __nv_bfloat16* __restrict__ cos_sin_cache, const int64_t* __restrict__ positions,
                              const int32_t* __restrict__ slot_ids, __nv_bfloat16* __restrict__ key_cache,
                              __nv_bfloat16* __restrict__ value_cache, int num_tokens) {
  constexpr int kPerLane = kHeadDim / 32;   // 2 or 4 bf16: one 4- or 8-byte access per lane
  using Vec = typename std::conditional<kPerLane == 4, uint2, uint32_t>::type;
  const int warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int heads = num_heads_q + 2 * num_heads_kv;
  const int tok = warp_global / heads;
  const int head = warp_global % heads;
  if (tok >= num_tokens) return;
  const bool is_q = head < num_heads_q, is_v = head >= num_heads_q + num_heads_kv;
  // norm weights do not depend on the producer kernel: fetch before the PDL wait
  float w[kPerLane];
  if (!is_v) {
    const __nv_bfloat16* wp = (is_q ? q_weight : k_weight) + lane * kPerLane;
#pragma unroll
    for (int i = 0; i < kPerLane; ++i) w[i] = __bfloat162float(wp[i]);
  }
  pdl_launch_dependents();  // consumer prologues (weight / KV prefetch) may start now
  pdl_wait();
  Vec* ptr = reinterpret_cast<Vec*>(qkv + ((int64_t)tok * heads + head) * kHeadDim) + lane;
  const int64_t slot = slot_ids[tok];
  const int kvh = is_v ? head - num_heads_q - num_heads_kv : head - num_heads_q;
  const int64_t crow = (slot * num_heads_kv + kvh) * kHeadDim;
  if (is_v) {
    if (slot >= 0) reinterpret_cast<Vec*>(value_cache + crow)[lane] = *ptr;
    return;
  }
  const Vec x = *ptr;
  const uint32_t* xp = reinterpret_cast<const uint32_t*>(&x);
  float e[kPerLane];
#pragma unroll
  for (int j = 0; j < kPerLane / 2; ++j) {
    e[2 * j] = bf16lo(xp[j]);
    e[2 * j + 1] = bf16hi(xp[j]);
  }
  qk_norm_rope_warp<kHeadDim, false>(e, w, eps, cos_sin_cache + positions[tok] * kHeadDim, kHeadDim, lane);
  Vec y;
  uint32_t* yp = reinterpret_cast<uint32_t*>(&y);
#pragma unroll
  for (int j = 0; j < kPerLane / 2; ++j) yp[j] = pack_bf16x2(e[2 * j], e[2 * j + 1]);
  *ptr = y;
  if (!is_q && slot >= 0) reinterpret_cast<Vec*>(key_cache + crow)[lane] = y;
  pdl_launch_dependents();
}

// ---------------------------------------------------------------------------
// K11 act_and_mul.  activation.cu:45-130: act in fp32, rounded to bf16, then a
// bf16 multiply (second rounding).
// ---------------------------------------------------------------------------

template <int kAct>
__global__ void __launch_bounds__(1024)
act_and_mul_kernel(__nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ in, int d, bool vec) {
  const int64_t tok = blockIdx.y;
  const __nv_bfloat16* x = in + tok * 2 * (int64_t)d;
  const __nv_bfloat16* y = x + d;
  __nv_bfloat16* o = out + tok * (int64_t)d;
  pdl_launch_dependents();  // consumer prologues (weight / KV prefetch) may start now
  pdl_wait();
  if (vec) {
    const uint4* xv = reinterpret_cast<const uint4*>(x);
    const uint4* yv = reinterpret_cast<const uint4*>(y);
    uint4* ov = reinterpret_cast<uint4*>(o);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d / 8; i += gridDim.x * blockDim.x) {
      uint4 a = xv[i], b = yv[i], r;
      const uint32_t* ap = &a.x;
      const uint32_t* bp = &b.x;
      uint32_t* rp = &r.x;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float lo = round_bf16(act_fn<kAct>(bf16lo(ap[j]))) * bf16lo(bp[j]);
        float hi = round_bf16(act_fn<kAct>(bf16hi(ap[j]))) * bf16hi(bp[j]);
        rp[j] = pack_bf16x2(lo, hi);
      }
      ov[i] = r;
    }
  } else {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d; i += gridDim.x * blockDim.x)
      o[i] = __float2bfloat16_rn(round_bf16(act_fn<kAct>(__bfloat162float(x[i]))) * __bfloat162float(y[i]));
  }
  pdl_launch_dependents();
}

// act_and_mul over the INTERLEAVED gate/up layout the fused decode GEMV uses (per 16 columns: 8 gate then 8 up), so the
// prefill GEMM can share the same packed gate_up weight: out[t, 8j + i] = act(x[t, 16j + i]) * x[t, 16j + 8 + i].
template <int kAct>
__global__ void __launch_bounds__(256)
act_and_mul_interleaved8_kernel(__nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ in, int d /* out cols */) {
  const int64_t tok = blockIdx.y;
  const uint4* x = reinterpret_cast<const uint4*>(in + tok * 2 * (int64_t)d);
  uint4* o = reinterpret_cast<uint4*>(out + tok * (int64_t)d);
  pdl_launch_dependents();
  pdl_wait();
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < d / 8; j += gridDim.x * blockDim.x) {
    const uint4 a = x[2 * j], b = x[2 * j + 1];
    const uint32_t* ap = &a.x;
    const uint32_t* bp = &b.x;
    uint4 r;
    uint32_t* rp = &r.x;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      rp[i] = pack_bf16x2(round_bf16(act_fn<kAct>(bf16lo(ap[i]))) * bf16lo(bp[i]),
                          round_bf16(act_fn<kAct>(bf16hi(ap[i]))) * bf16hi(bp[i]));
    o[j] = r;
  }
}

// ---------------------------------------------------------------------------
// MLA latent cache writer (DeepSeek-V2/V3): the kv_a_proj_with_mqa row [c_kv 512 | k_pe 64] ->
//   ckv_cache[slot] = RMSNorm(c_kv) (kv_a_layernorm), kpe_cache[slot] = RoPE(k_pe); slot < 0 skipped.
// One launch for what rms_norm + rotary_embedding + two reshape_paged_cache do (fused_mla_kv with quant_mode "none",
// kernels/param.h:1105-1180; non-fused form layers/mlu/deepseek_v2_attention.cpp:223-240).  64 threads per token: the
// norm uses the thread mapping, accumulation order and rounding of rms_norm_vec_kernel at hidden size 512 (64 threads
// of 8 elements) and RoPE is rope_pair, so both halves are bit-identical to the unfused kernels.
// ---------------------------------------------------------------------------
template <bool kNeox>
__global__ void __launch_bounds__(64)
mla_cache_latent_kernel(const __nv_bfloat16* __restrict__ latent, int64_t latent_stride,
                        const __nv_bfloat16* __restrict__ gamma, float eps, const int64_t* __restrict__ positions,
                        const __nv_bfloat16* __restrict__ cos_sin_cache, const int32_t* __restrict__ slot_ids,
                        __nv_bfloat16* __restrict__ ckv_cache, int64_t ckv_stride_page, int64_t ckv_stride_token,
                        __nv_bfloat16* __restrict__ kpe_cache, int64_t kpe_stride_page, int64_t kpe_stride_token,
                        int page_size) {
  constexpr int kDc = 512, kRot = 64;
  __shared__ float red[33];
  const int64_t tok = blockIdx.x;
  const uint4 w = __ldg(reinterpret_cast<const uint4*>(gamma) + threadIdx.x);  // weights before the PDL wait
  pdl_launch_dependents();
  pdl_wait();
  const int64_t slot = slot_ids[tok];
  if (slot < 0) return;  // uniform over the CTA
  const __nv_bfloat16* row = latent + tok * latent_stride;
  const uint4 x = reinterpret_cast<const uint4*>(row)[threadIdx.x];
  const float rstd = rms_rstd(block_sum(sumsq_bf16x8(0.f, x), red), kDc, eps);
  const int64_t page = slot / page_size, off = slot % page_size;
  reinterpret_cast<uint4*>(ckv_cache + page * ckv_stride_page + off * ckv_stride_token)[threadIdx.x] =
      rms_apply_bf16x8(x, w, rstd);
  if (threadIdx.x < kRot / 2) {
    const int r = threadIdx.x;
    const __nv_bfloat16* cs = cos_sin_cache + positions[tok] * kRot;
    const float c = __bfloat162float(cs[r]), sn = __bfloat162float(cs[kRot / 2 + r]);
    __nv_bfloat16* dst = kpe_cache + page * kpe_stride_page + off * kpe_stride_token;
    if (kNeox) rope_pair(row + kDc, dst, r, kRot / 2 + r, c, sn);
    else rope_pair(row + kDc, dst, 2 * r, 2 * r + 1, c, sn);
  }
  pdl_launch_dependents();
}

}  // namespace xb

// ===========================================================================
// C ABI
// ===========================================================================
using namespace xb;

extern "C" int xb_rms_norm_bf16(void* out, const void* input, int64_t input_stride, const void* weight,
                                float eps, int num_tokens, int hidden_size, xb_stream_t stream) {
  return launch_rms_norm<false, false>(out, const_cast<void*>(input), input_stride, nullptr, weight, nullptr, eps,
                                       num_tokens, hidden_size, (cudaStream_t)stream);
}
extern "C" int xb_fused_add_rms_norm_bf16(void* input, int64_t input_stride, void* residual, const void* weight,
                                          float eps, int num_tokens, int hidden_size, xb_stream_t stream) {
  return launch_rms_norm<true, false>(nullptr, input, input_stride, residual, weight, nullptr, eps, num_tokens,
                                      hidden_size, (cudaStream_t)stream);
}
extern "C" int xb_rms_norm_static_fp8_quant_bf16(void* out, const void* input, int64_t input_stride,
                                                 const void* weight, const float* scale, float eps, int num_tokens,
                                                 int hidden_size, xb_stream_t stream) {
  return launch_rms_norm<false, true>(out, const_cast<void*>(input), input_stride, nullptr, weight, scale, eps,
                                      num_tokens, hidden_size, (cudaStream_t)stream);
}
extern "C" int xb_fused_add_rms_norm_static_fp8_quant_bf16(void* out, void* input, int64_t input_stride,
                                                           void* residual, const void* weight, const float* scale,
                                                           float eps, int num_tokens, int hidden_size,
                                                           xb_stream_t stream) {
  return launch_rms_norm<true, true>(out, input, input_stride, residual, weight, scale, eps, num_tokens,
                                     hidden_size, (cudaStream_t)stream);
}

extern "C" int xb_static_scaled_fp8_quant_bf16(void* out, int64_t out_stride, const void* input,
                                               int64_t input_stride, const float* scale, int num_tokens,
                                               int hidden_size, xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  const bool vec = hidden_size % 8 == 0 && input_stride % 8 == 0 && out_stride % 8 == 0 && aligned16(input) &&
                   (reinterpret_cast<uintptr_t>(out) % 8 == 0);
  XB_CUDA_OK(launch(fp8_quant_kernel, dim3(num_tokens), dim3(256), 0, (cudaStream_t)stream, true,
                    reinterpret_cast<uint8_t*>(out), out_stride, reinterpret_cast<const __nv_bfloat16*>(input),
                    input_stride, scale, hidden_size, vec));
  return 0;
}
extern "C" int xb_dynamic_scaled_fp8_quant_bf16(void* out, int64_t out_stride, const void* input,
                                                int64_t input_stride, float* scale_out, int num_tokens,
                                                int hidden_size, xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  XB_CUDA_OK(launch(fp8_scale_init_kernel, dim3(1), dim3(1), 0, s, false, scale_out));
  XB_CUDA_OK(launch(fp8_amax_kernel, dim3(num_tokens), dim3(256), 0, s, false,
                    reinterpret_cast<const __nv_bfloat16*>(input), input_stride, hidden_size, scale_out));
  XB_CUDA_OK(launch(fp8_scale_finish_kernel, dim3(1), dim3(1), 0, s, false, scale_out));
  return xb_static_scaled_fp8_quant_bf16(out, out_stride, input, input_stride, scale_out, num_tokens, hidden_size,
                                         stream);
}

extern "C" int xb_rotary_embedding_bf16(const int64_t* positions, void* query, void* key, const void* cos_sin_cache,
                                        int rot_dim, int64_t query_stride, int64_t key_stride, int64_t head_stride,
                                        int num_heads, int num_kv_heads, int head_size, int is_neox, int num_tokens,
                                        xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  XB_CHECK(rot_dim > 0 && rot_dim % 2 == 0 && rot_dim <= head_size, "rotary_embedding: bad rot_dim %d (head %d)",
           rot_dim, head_size);
  XB_CHECK(num_kv_heads > 0 && num_heads % num_kv_heads == 0, "rotary_embedding: heads %d %% kv heads %d != 0",
           num_heads, num_kv_heads);
  int work = (num_heads + (key ? num_kv_heads : 0)) * rot_dim / 2;
  int threads = work < 512 ? ((work + 31) / 32) * 32 : 512;
  auto* q = reinterpret_cast<__nv_bfloat16*>(query);
  auto* k = reinterpret_cast<__nv_bfloat16*>(key);
  auto* cs = reinterpret_cast<const __nv_bfloat16*>(cos_sin_cache);
  if (is_neox)
    XB_CUDA_OK(launch(rotary_embedding_kernel<true>, dim3(num_tokens), dim3(threads), 0, (cudaStream_t)stream, true,
                      positions, q, k, cs, rot_dim, query_stride, key_stride, head_stride, num_heads, num_kv_heads));
  else
    XB_CUDA_OK(launch(rotary_embedding_kernel<false>, dim3(num_tokens), dim3(threads), 0, (cudaStream_t)stream, true,
                      positions, q, k, cs, rot_dim, query_stride, key_stride, head_stride, num_heads, num_kv_heads));
  return 0;
}

extern "C" int xb_reshape_paged_cache_bf16(const int32_t* slot_ids, const void* keys, const void* values,
                                           void* key_cache, void* value_cache, int64_t k_stride, int64_t v_stride,
                                           int n_kv_heads, int head_dim, int block_size, int num_tokens,
                                           xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  (void)block_size;  // [block, offset] flattens to slot * row_elems for the contiguous reference layout
  const int row = n_kv_heads * head_dim;
  const bool vec = row % 8 == 0 && k_stride % 8 == 0 && v_stride % 8 == 0 && aligned16(keys) && aligned16(values) &&
                   aligned16(key_cache) && aligned16(value_cache);
  int threads = vec ? row / 8 : row;
  threads = threads < 32 ? 32 : (threads > 256 ? 256 : ((threads + 31) / 32) * 32);
  XB_CUDA_OK(launch(reshape_paged_cache_kernel, dim3(num_tokens), dim3(threads), 0, (cudaStream_t)stream, true,
                    slot_ids, reinterpret_cast<const __nv_bfloat16*>(keys),
                    reinterpret_cast<const __nv_bfloat16*>(values), reinterpret_cast<__nv_bfloat16*>(key_cache),
                    reinterpret_cast<__nv_bfloat16*>(value_cache), k_stride, v_stride, row, vec));
  return 0;
}

extern "C" int xb_rope_and_cache_bf16(const int64_t* positions, void* query, void* key, const void* value,
                                      const void* cos_sin_cache, const int32_t* slot_ids, void* key_cache,
                                      void* value_cache, int rot_dim, int64_t query_stride, int64_t key_stride,
                                      int64_t value_stride, int num_heads, int num_kv_heads, int head_size,
                                      int block_size, int is_neox, int num_tokens, xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  (void)block_size;
  XB_CHECK(rot_dim > 0 && rot_dim % 2 == 0 && rot_dim <= head_size, "rope_and_cache: bad rot_dim %d", rot_dim);
  int work = (num_heads + num_kv_heads) * rot_dim / 2;
  int threads = work < 512 ? ((work + 31) / 32) * 32 : 512;
  auto* q = reinterpret_cast<__nv_bfloat16*>(query);
  auto* k = reinterpret_cast<__nv_bfloat16*>(key);
  auto* v = reinterpret_cast<const __nv_bfloat16*>(value);
  auto* cs = reinterpret_cast<const __nv_bfloat16*>(cos_sin_cache);
  auto* kc = reinterpret_cast<__nv_bfloat16*>(key_cache);
  auto* vc = reinterpret_cast<__nv_bfloat16*>(value_cache);
  if (is_neox)
    XB_CUDA_OK(launch(rope_and_cache_kernel<true>, dim3(num_tokens), dim3(threads), 0, (cudaStream_t)stream, true,
                      positions, q, k, v, cs, slot_ids, kc, vc, rot_dim, query_stride, key_stride, value_stride,
                      num_heads, num_kv_heads, head_size));
  else
    XB_CUDA_OK(launch(rope_and_cache_kernel<false>, dim3(num_tokens), dim3(threads), 0, (cudaStream_t)stream, true,
                      positions, q, k, v, cs, slot_ids, kc, vc, rot_dim, query_stride, key_stride, value_stride,
                      num_heads, num_kv_heads, head_size));
  return 0;
}

extern "C" int xb_rope_and_cache_packed_bf16(const int64_t* positions, const void* qkv_packed, int64_t in_stride,
                                             void* qkv_out, int64_t out_stride, const void* cos_sin_cache,
                                             const int32_t* slot_ids, void* key_cache, void* value_cache,
                                             int num_heads, int num_kv_heads, int head_size, int num_tokens,
                                             xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  XB_CHECK(head_size % 16 == 0 && num_heads > 0 && num_kv_heads > 0, "rope_and_cache_packed: bad heads %d/%d x %d",
           num_heads, num_kv_heads, head_size);
  XB_CHECK(qkv_packed != qkv_out, "rope_and_cache_packed: out of place only (the permutation is not in-place safe)");
  const int work = (num_heads + 2 * num_kv_heads) * head_size / 2;
  const int threads = work < 512 ? ((work + 31) / 32) * 32 : 512;
  XB_CUDA_OK(launch(rope_and_cache_packed_kernel, dim3(num_tokens), dim3(threads), 0, (cudaStream_t)stream, true, positions,
                    reinterpret_cast<const __nv_bfloat16*>(qkv_packed), in_stride, reinterpret_cast<__nv_bfloat16*>(qkv_out),
                    out_stride, reinterpret_cast<const __nv_bfloat16*>(cos_sin_cache), slot_ids,
                    reinterpret_cast<__nv_bfloat16*>(key_cache), reinterpret_cast<__nv_bfloat16*>(value_cache), num_heads,
                    num_kv_heads, head_size));
  return 0;
}

extern "C" int xb_fused_qk_norm_rope_bf16(void* qkv, int num_heads_q, int num_heads_k, int num_heads_v, int head_dim,
                                          float eps, const void* q_weight, const void* k_weight,
                                          const void* cos_sin_cache, int rot_dim, int interleaved,
                                          const int64_t* position_ids, int num_tokens, xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  XB_CHECK(head_dim == 64 || head_dim == 128 || head_dim == 256, "fused_qk_norm_rope: head_dim %d unsupported",
           head_dim);
  {
    const int per_lane = head_dim / 32, rl = rot_dim / per_lane;
    XB_CHECK(rot_dim > 0 && rot_dim <= head_dim && rot_dim % (2 * per_lane) == 0 && (rl & (rl - 1)) == 0,
             "fused_qk_norm_rope: rotary_dim %d unsupported for head_dim %d", rot_dim, head_dim);
  }
  const int warps = num_tokens * (num_heads_q + num_heads_k);
  const int wpb = 8;
  dim3 grid((warps + wpb - 1) / wpb), block(wpb * 32);
  auto* p = reinterpret_cast<__nv_bfloat16*>(qkv);
  auto* qw = reinterpret_cast<const __nv_bfloat16*>(q_weight);
  auto* kw = reinterpret_cast<const __nv_bfloat16*>(k_weight);
  auto* cs = reinterpret_cast<const __nv_bfloat16*>(cos_sin_cache);
  cudaStream_t s = (cudaStream_t)stream;
#define XB_QKNR(D, I)                                                                                              \
  XB_CUDA_OK(launch(fused_qk_norm_rope_kernel<D, I>, grid, block, 0, s, true, p, num_heads_q, num_heads_k,        \
                    num_heads_v, eps, qw, kw, cs, rot_dim, position_ids, num_tokens))
  if (head_dim == 64) { if (interleaved) XB_QKNR(64, true); else XB_QKNR(64, false); }
  else if (head_dim == 128) { if (interleaved) XB_QKNR(128, true); else XB_QKNR(128, false); }
  else { if (interleaved) XB_QKNR(256, true); else XB_QKNR(256, false); }
#undef XB_QKNR
  return 0;
}

extern "C" int xb_qk_norm_rope_and_cache_bf16(void* qkv, int num_heads_q, int num_heads_kv, int head_dim, float eps,
                                              const void* q_weight, const void* k_weight, const void* cos_sin_cache,
                                              const int64_t* positions, const int32_t* slot_ids, void* key_cache,
                                              void* value_cache, int num_tokens, xb_stream_t stream) {
  XB_CHECK(head_dim == 64 || head_dim == 128, "qk_norm_rope_and_cache: head_dim %d unsupported (64 or 128)", head_dim);
  XB_CHECK(num_heads_q > 0 && num_heads_kv > 0 && num_tokens >= 0, "qk_norm_rope_and_cache: bad heads %d/%d or tokens %d",
           num_heads_q, num_heads_kv, num_tokens);
  XB_CHECK(q_weight && k_weight && cos_sin_cache, "qk_norm_rope_and_cache: null q_weight, k_weight or cos_sin_cache");
  if (num_tokens == 0) return 0;
  XB_CHECK(qkv && positions && slot_ids && key_cache && value_cache, "qk_norm_rope_and_cache: null pointer argument");
  const uintptr_t align = (uintptr_t)head_dim / 16;   // one 4- / 8-byte access per lane
  XB_CHECK((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(key_cache) |
            reinterpret_cast<uintptr_t>(value_cache)) % align == 0,
           "qk_norm_rope_and_cache: qkv and caches must be %d-byte aligned", (int)align);
  const int64_t warps = (int64_t)num_tokens * (num_heads_q + 2 * num_heads_kv);
  const int wpb = 8;
  XB_CHECK(warps <= (int64_t)INT32_MAX - wpb, "qk_norm_rope_and_cache: %lld (token, head) pairs", (long long)warps);
  dim3 grid((unsigned)((warps + wpb - 1) / wpb)), block(wpb * 32);
  auto* p = reinterpret_cast<__nv_bfloat16*>(qkv);
  auto* qw = reinterpret_cast<const __nv_bfloat16*>(q_weight);
  auto* kw = reinterpret_cast<const __nv_bfloat16*>(k_weight);
  auto* cs = reinterpret_cast<const __nv_bfloat16*>(cos_sin_cache);
  auto* kc = reinterpret_cast<__nv_bfloat16*>(key_cache);
  auto* vc = reinterpret_cast<__nv_bfloat16*>(value_cache);
  auto kern = head_dim == 64 ? qk_norm_rope_and_cache_kernel<64> : qk_norm_rope_and_cache_kernel<128>;
  XB_CUDA_OK(launch(kern, grid, block, 0, (cudaStream_t)stream, true, p, num_heads_q, num_heads_kv, eps, qw, kw, cs,
                    positions, slot_ids, kc, vc, num_tokens));
  return 0;
}

extern "C" int xb_act_and_mul_bf16(void* out, const void* input, int d, int num_tokens, int act_mode,
                                   xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  XB_CHECK(act_mode >= 0 && act_mode <= 2, "act_and_mul: unsupported act mode %d (silu|gelu|gelu_tanh)", act_mode);
  const bool vec = d % 8 == 0 && aligned16(input) && aligned16(out);
  const int work = vec ? d / 8 : d;
  int threads = work < 256 ? ((work + 31) / 32) * 32 : 256;
  // few tokens: spread one row over several CTAs so a decode step is not one-SM bound
  int bx = (work + threads - 1) / threads;
  if (num_tokens >= 512) bx = 1;
  else if (bx > 32) bx = 32;
  dim3 grid(bx, num_tokens), block(threads);
  auto* o = reinterpret_cast<__nv_bfloat16*>(out);
  auto* in = reinterpret_cast<const __nv_bfloat16*>(input);
  cudaStream_t s = (cudaStream_t)stream;
  if (act_mode == 0) XB_CUDA_OK(launch(act_and_mul_kernel<0>, grid, block, 0, s, true, o, in, d, vec));
  else if (act_mode == 1) XB_CUDA_OK(launch(act_and_mul_kernel<1>, grid, block, 0, s, true, o, in, d, vec));
  else XB_CUDA_OK(launch(act_and_mul_kernel<2>, grid, block, 0, s, true, o, in, d, vec));
  return 0;
}

extern "C" int xb_act_and_mul_interleaved8_bf16(void* out, const void* input, int d, int num_tokens, int act_mode,
                                                xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  XB_CHECK(act_mode >= 0 && act_mode <= 2, "act_and_mul_interleaved8: unsupported act mode %d", act_mode);
  XB_CHECK(d % 8 == 0 && aligned16(input) && aligned16(out), "act_and_mul_interleaved8: d %% 8 and 16-byte alignment required");
  int bx = (d / 8 + 255) / 256;
  if (num_tokens >= 512) bx = 1;
  dim3 grid(bx, num_tokens), block(256);
  auto* o = reinterpret_cast<__nv_bfloat16*>(out);
  auto* in = reinterpret_cast<const __nv_bfloat16*>(input);
  cudaStream_t s = (cudaStream_t)stream;
  if (act_mode == 0) XB_CUDA_OK(launch(act_and_mul_interleaved8_kernel<0>, grid, block, 0, s, true, o, in, d));
  else if (act_mode == 1) XB_CUDA_OK(launch(act_and_mul_interleaved8_kernel<1>, grid, block, 0, s, true, o, in, d));
  else XB_CUDA_OK(launch(act_and_mul_interleaved8_kernel<2>, grid, block, 0, s, true, o, in, d));
  return 0;
}

extern "C" int xb_mla_cache_latent_bf16(const void* latent, int64_t latent_stride, const void* gamma, float eps,
                                        const int64_t* positions, const void* cos_sin_cache, int interleaved,
                                        const int32_t* slot_ids, void* ckv_cache, int64_t ckv_stride_page,
                                        int64_t ckv_stride_token, void* kpe_cache, int64_t kpe_stride_page,
                                        int64_t kpe_stride_token, int kv_lora_rank, int qk_rope_head_dim, int page_size,
                                        int num_tokens, xb_stream_t stream) {
  XB_CHECK(kv_lora_rank == 512 && qk_rope_head_dim == 64,
           "mla_cache_latent: kv_lora_rank %d / qk_rope_head_dim %d unsupported (512 / 64)", kv_lora_rank,
           qk_rope_head_dim);
  XB_CHECK(num_tokens >= 0 && page_size >= 1, "mla_cache_latent: bad num_tokens %d or page_size %d", num_tokens,
           page_size);
  if (num_tokens == 0) return 0;
  XB_CHECK(latent && gamma && positions && cos_sin_cache && slot_ids && ckv_cache && kpe_cache,
           "mla_cache_latent: null pointer argument");
  XB_CHECK(aligned16(latent) && aligned16(gamma) && aligned16(ckv_cache) && aligned16(kpe_cache) &&
               latent_stride % 8 == 0 && ckv_stride_page % 8 == 0 && ckv_stride_token % 8 == 0,
           "mla_cache_latent: latent, gamma and ckv_cache rows must be 16-byte aligned");
  auto* lat = reinterpret_cast<const __nv_bfloat16*>(latent);
  auto* g = reinterpret_cast<const __nv_bfloat16*>(gamma);
  auto* cs = reinterpret_cast<const __nv_bfloat16*>(cos_sin_cache);
  auto* ckv = reinterpret_cast<__nv_bfloat16*>(ckv_cache);
  auto* kpe = reinterpret_cast<__nv_bfloat16*>(kpe_cache);
  auto kern = interleaved ? mla_cache_latent_kernel<false> : mla_cache_latent_kernel<true>;
  XB_CUDA_OK(launch(kern, dim3(num_tokens), dim3(64), 0, (cudaStream_t)stream, true, lat, latent_stride, g, eps,
                    positions, cs, slot_ids, ckv, ckv_stride_page, ckv_stride_token, kpe, kpe_stride_page,
                    kpe_stride_token, page_size));
  return 0;
}
