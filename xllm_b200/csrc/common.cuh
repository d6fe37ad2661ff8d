// Shared device/host helpers for libxllm_b200_ops (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <utility>

#include "../../include/xllm_b200_ops.h"

namespace xb {

// ---- error plumbing (thread-local message, C-ABI returns non-zero) ----------
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launch_count;
extern std::atomic<int> g_pdl_enabled;

#define XB_CHECK(cond, ...)          \
  do {                               \
    if (!(cond)) {                   \
      ::xb::set_error(__VA_ARGS__);  \
      return 1;                      \
    }                                \
  } while (0)

#define XB_CUDA_OK(expr)                                                      \
  do {                                                                        \
    cudaError_t _e = (expr);                                                  \
    if (_e != cudaSuccess) {                                                  \
      ::xb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                      __FILE__, __LINE__);                                    \
      return 2;                                                               \
    }                                                                         \
  } while (0)

// SM count of the device current at the first call, cached for the process.
int device_sm_count();

// Launch helper: counts launches, optionally attaches the PDL attribute, launches thread-block clusters of cluster_x CTAs
// along grid x (1 = plain launch).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                  bool pdl, int cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (pdl && g_pdl_enabled.load(std::memory_order_relaxed)) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                          Args&&... args) {
  return launch_cluster(kernel, grid, block, smem, stream, pdl, 1, std::forward<Args>(args)...);
}

// Raises kKernel's dynamic shared-memory limit to `bytes` once per process, on the device current at the first call;
// every call returns the result of that one attempt.
template <auto kKernel>
inline cudaError_t set_max_dynamic_smem_once(int bytes) {
  static const cudaError_t err = cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  return err;
}

// ---- device helpers ---------------------------------------------------------
#ifdef __CUDACC__

// PDL: wait for the producer grid's memory to be visible / let the consumer
// grid start its prologue early.  No-ops when not launched with the attribute.
__device__ __forceinline__ void pdl_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

__device__ __forceinline__ float bf16_bits_to_f32(uint32_t bits16) {
  return __uint_as_float(bits16 << 16);
}
__device__ __forceinline__ float bf16lo(uint32_t packed) {
  return __uint_as_float(packed << 16);
}
__device__ __forceinline__ float bf16hi(uint32_t packed) {
  return __uint_as_float(packed & 0xffff0000u);
}
// round-to-nearest-even float -> bf16 bits (NaN-safe via intrinsic)
__device__ __forceinline__ uint32_t f32_to_bf16_bits(float x) {
  return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(x));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// bf16 value rounded through bf16 and back (models `static_cast<scalar_t>(f)`)
__device__ __forceinline__ float round_bf16(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

// 2^x on the SFU, one MUFU.EX2 (flush-to-zero, ~2 ulp): the softmax inner loops are MUFU-throughput bound
// (16 ex2 / clk / SM), the range/denormal fix-up code of exp2f() would only add issue slots
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// 128-bit streaming loads/stores.  KV pages and weights are read exactly once
// per step: keep them out of L1 (L1::no_allocate) so x / q stay resident.
__device__ __forceinline__ uint4 ldg_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 ldg_cached(const void* p) {
  return __ldg(reinterpret_cast<const uint4*>(p));
}

// Ampere-style async copies global -> shared.  Used by the HBM-streaming small-M kernels as a per-lane private
// staging ring: completion is tracked in ORDER by commit groups (wait_group N = "all but the N youngest"), which a
// register ring of plain LDGs cannot express - ptxas puts every in-flight LDG of a loop on one scoreboard and a wait
// on the oldest load then waits for the youngest too, so the prefetch depth silently collapses to zero.
__device__ __forceinline__ uint32_t smem_addr_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src) {   // L2 only (streamed once)
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_4(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int kPending>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(kPending) : "memory");
}
__device__ __forceinline__ uint4 lds_128(uint32_t addr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr) : "memory");
  return r;
}
__device__ __forceinline__ uint32_t lds_32(uint32_t addr) {
  uint32_t r;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(addr) : "memory");
  return r;
}
__device__ __forceinline__ void sts_128(uint32_t addr, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint2 lds_64(uint32_t addr) {
  uint2 r;
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(addr) : "memory");
  return r;
}

// sat_e4m3(x*inv_scale): fp8_quant_utils.cuh:112-129 (clamp to +-448, then
// __nv_cvt_float_to_fp8(..., __NV_SATFINITE, __NV_E4M3) = RNE).
__device__ __forceinline__ uint8_t scaled_fp8_e4m3(float v, float inv_scale) {
  float x = v * inv_scale;
  float r = fmaxf(-448.0f, fminf(x, 448.0f));
  return (uint8_t)__nv_cvt_float_to_fp8(r, __NV_SATFINITE, __NV_E4M3);
}

__device__ __forceinline__ uint32_t hmul2_bf16x2(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}
__device__ __forceinline__ uint32_t hsub2_bf16x2(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("sub.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}
// int4 weight-only dequant (oracle/quant.py, bits = 4) of the tile-packed W4 layout described in linear_small_m.cu.
// W4 meta word (bf16 scale | bf16(128 + zero) << 16) -> bf16x2 scale, bf16x2 (128 + zero)
__device__ __forceinline__ void w4_meta(uint32_t m, uint32_t& s2, uint32_t& z2) {
  s2 = __byte_perm(m, 0, 0x1010);
  z2 = __byte_perm(m, 0, 0x3232);
}
// one packed word -> the four bf16x2 mma A-fragment registers as exact bf16 integers 128 + q: (w >> 4i) & 0x000f000f | 0x4300
// in each half; q[0] / q[2] are row g, q[1] / q[3] row g+8
__device__ __forceinline__ void w4_nibbles(uint32_t w, uint32_t (&q)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
    asm("lop3.b32 %0, %1, %2, %3, 0xea;" : "=r"(q[i]) : "r"(w >> (4 * i)), "r"(0x000f000fu), "r"(0x43004300u));  // (a & b) | c
}
// w = bf16((q - z) * s), bit-exact with the spec: (128 + q) - (128 + z) is exact, the product by s rounds once.
// a[0] / a[2] are row g (scale s0, zero z0), a[1] / a[3] row g+8 (s1, z1).
__device__ __forceinline__ void w4_dequant_word(uint32_t w, uint32_t z0, uint32_t s0, uint32_t z1, uint32_t s1,
                                                uint32_t (&a)[4]) {
  uint32_t q[4];
  w4_nibbles(w, q);
  a[0] = hmul2_bf16x2(hsub2_bf16x2(q[0], z0), s0);
  a[1] = hmul2_bf16x2(hsub2_bf16x2(q[1], z1), s1);
  a[2] = hmul2_bf16x2(hsub2_bf16x2(q[2], z0), s0);
  a[3] = hmul2_bf16x2(hsub2_bf16x2(q[3], z1), s1);
}
// int8 weight-only dequant (oracle/quant.py, bits = 8): four unsigned bytes of one weight row (k ascending) -> two bf16x2
// registers bf16((q - z) * s), bit-exact with the spec: 0x4B0000qq is float(2^23 + q), adding neg_mz = -(2^23 + z) gives
// q - z exactly, the bf16x2 pack is exact for |q - z| <= 255 and the product by s rounds once.
__device__ __forceinline__ void w8_dequant_word(uint32_t w, float neg_mz, uint32_t s2, uint32_t& lo, uint32_t& hi) {
  const float f0 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7650)) + neg_mz;
  const float f1 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7651)) + neg_mz;
  const float f2 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7652)) + neg_mz;
  const float f3 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7653)) + neg_mz;
  lo = hmul2_bf16x2(pack_bf16x2(f0, f1), s2);
  hi = hmul2_bf16x2(pack_bf16x2(f2, f3), s2);
}
// W8 meta word (bf16 scale | zero << 16) -> bf16x2 scale, -(2^23 + zero)
__device__ __forceinline__ void w8_meta(uint32_t m, uint32_t& s2, float& neg_mz) {
  s2 = __byte_perm(m, 0, 0x1010);
  neg_mz = __uint_as_float(0xCB000000u + (m >> 16));
}

// mma.sync m16n8k32 e4m3 x e4m3 -> f32 (register-resident fragments; FP8 W8A8 small-M kernel)
__device__ __forceinline__ void mma_e4m3_16832(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.f32.e4m3.e4m3.f32 "
      "{%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// mma.sync m16n8k16 bf16 x bf16 -> f32 (register-resident fragments; used by
// the HBM-bound small-M kernels where no smem staging is wanted).
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0,
                                               uint32_t a1, uint32_t a2,
                                               uint32_t a3, uint32_t b0,
                                               uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 "
      "{%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// C fragment of lane (g, t) of an m16n8 mma into a row-major 16 x 8 fp32 tile:
// c0 (g, 2t), c1 (g, 2t+1), c2 (g+8, 2t), c3 (g+8, 2t+1)
__device__ __forceinline__ void store_c_frag(float* tile16x8, const float (&c)[4], int g, int t) {
  tile16x8[g * 8 + 2 * t] = c[0];
  tile16x8[g * 8 + 2 * t + 1] = c[1];
  tile16x8[(g + 8) * 8 + 2 * t] = c[2];
  tile16x8[(g + 8) * 8 + 2 * t + 1] = c[3];
}

// ---- reference arithmetic ---------------------------------------------------
// The rounding order of the reference's RMSNorm (xllm/core/kernels/cuda/norm.cu), RoPE (rope.cu) and gated activations
// (activation.cu).  Every kernel that normalises, rotates or gates a row calls these, which keeps the fused forms
// bit-identical to the unfused kernels.

// block-wide sum (<= 1024 threads, smem[33]); stands in for the cub::BlockReduce of norm.cu:60-62
__device__ __forceinline__ float block_sum(float v, float* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  const int nwarps = (blockDim.x + 31) >> 5;
  if (warp == 0) {
    float t = lane < nwarps ? smem[lane] : 0.f;
    t = warp_sum(t);
    if (lane == 0) smem[32] = t;
  }
  __syncthreads();
  return smem[32];
}

// bf16 residual add, one rounding per element (norm.cu:112, _f16Vec::operator+= of type_convert.cuh:150-169)
__device__ __forceinline__ float add_bf16(float x, float r) {
  return round_bf16(x + r);
}
__device__ __forceinline__ uint4 add_bf16x8(const uint4 x, const uint4 r) {
  const uint32_t* xp = &x.x;
  const uint32_t* rp = &r.x;
  uint4 o;
  uint32_t* op = &o.x;
#pragma unroll
  for (int j = 0; j < 4; ++j) op[j] = pack_bf16x2(bf16lo(xp[j]) + bf16lo(rp[j]), bf16hi(xp[j]) + bf16hi(rp[j]));
  return o;
}

// ss + sum of squares of the 8 bf16 of x, fp32 in element order (_f16Vec::sum_squares, type_convert.cuh:213-228)
__device__ __forceinline__ float sumsq_bf16x8(float ss, const uint4 x) {
  const uint32_t* xp = &x.x;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float a = bf16lo(xp[j]), b = bf16hi(xp[j]);
    ss += a * a + b * b;
  }
  return ss;
}

// 1 / RMS of a row of n elements from its sum of squares (norm.cu:65,122)
__device__ __forceinline__ float rms_rstd(float sumsq, int n, float eps) {
  return rsqrtf(sumsq / (float)n + eps);
}

// normalised value bf16(x * rstd); the output is that times the weight, the product left in fp32 for the caller's
// rounding (norm.cu:72,130-131)
__device__ __forceinline__ float rms_norm_x(float x, float rstd) {
  return round_bf16(x * rstd);
}
__device__ __forceinline__ uint4 rms_apply_bf16x8(const uint4 x, const uint4 w, float rstd) {
  const uint32_t* xp = &x.x;
  const uint32_t* wp = &w.x;
  uint4 o;
  uint32_t* op = &o.x;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float a = rms_norm_x(bf16lo(xp[j]), rstd) * bf16lo(wp[j]);
    const float b = rms_norm_x(bf16hi(xp[j]), rstd) * bf16hi(wp[j]);
    op[j] = pack_bf16x2(a, b);
  }
  return o;
}

// rotary pair in bf16 arithmetic, (x, y) -> (rope_x, rope_y): every product and the add / subtract rounded to bf16
// (rope.cu:52-53)
__device__ __forceinline__ float rope_x(float x, float y, float c, float s) {
  return round_bf16(x * c) - round_bf16(y * s);
}
__device__ __forceinline__ float rope_y(float x, float y, float c, float s) {
  return round_bf16(y * c) + round_bf16(x * s);
}
// rotated pair (in[xi], in[yi]) -> (out[xi], out[yi]); in place when in == out
__device__ __forceinline__ void rope_pair(const __nv_bfloat16* in, __nv_bfloat16* out, int xi, int yi, float c, float s) {
  const float x = __bfloat162float(in[xi]);
  const float y = __bfloat162float(in[yi]);
  out[xi] = __float2bfloat16_rn(rope_x(x, y, c, s));
  out[yi] = __float2bfloat16_rn(rope_y(x, y, c, s));
}
__device__ __forceinline__ void rope_pair(__nv_bfloat16* arr, int xi, int yi, float c, float s) {
  rope_pair(arr, arr, xi, yi, c, s);
}

// Qwen3 per-head RMSNorm + RoPE on one warp (fused_qknorm_rope.cu:84-300): lane owns the kHeadDim / 32 consecutive
// elements e of one head and the matching weights w.  Norm in fp32 (e *= rstd * w, :197-202), rotation in fp32 over the
// first rot_dim elements of the [cos | sin] row `cache`, no rounding: the caller rounds once at the store.
template <int kHeadDim, bool kInterleave>
__device__ __forceinline__ void qk_norm_rope_warp(float (&e)[kHeadDim / 32], const float (&w)[kHeadDim / 32], float eps,
                                                  const __nv_bfloat16* cache, int rot_dim, int lane) {
  constexpr int kPerLane = kHeadDim / 32;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kPerLane; ++i) ss += e[i] * e[i];
  ss = warp_sum(ss);
  const float rstd = rsqrtf(ss / (float)kHeadDim + eps);
#pragma unroll
  for (int i = 0; i < kPerLane; ++i) e[i] *= rstd * w[i];
  const int embed = rot_dim / 2;
  if (kInterleave) {
    // pairs (2r, 2r+1) are both inside the lane (kPerLane even)
#pragma unroll
    for (int i = 0; i < kPerLane; i += 2) {
      const int d = lane * kPerLane + i;
      if (d < rot_dim) {
        const float c = __bfloat162float(cache[d / 2]), s = __bfloat162float(cache[embed + d / 2]);
        const float x = e[i], y = e[i + 1];
        e[i] = x * c - y * s;
        e[i + 1] = y * c + x * s;
      }
    }
  } else {
    // NeoX: pair (r, r+embed); partner lives in lane ^ (embed / kPerLane) when rot_dim == head_dim
    const int lanes_half = embed / kPerLane;
#pragma unroll
    for (int i = 0; i < kPerLane; ++i) {
      const int d = lane * kPerLane + i;
      const float partner = __shfl_xor_sync(0xffffffffu, e[i], lanes_half);
      if (d < rot_dim) {
        const int r = d < embed ? d : d - embed;
        const float c = __bfloat162float(cache[r]), s = __bfloat162float(cache[embed + r]);
        e[i] = d < embed ? e[i] * c - partner * s : e[i] * c + partner * s;
      }
    }
  }
}

// Output side of a qkv projection whose columns are in the rope-pair packed order of quant.pack_w4_qkv_rope (inside every
// head, packed column 16j+i holds dim 8j+i for i < 8 and dim D/2 + 8j + (i-8) otherwise).
struct QkvRopeCache {
  const int64_t* positions;
  const __nv_bfloat16* cos_sin;   // [max_pos, head_dim] = [cos half | sin half]
  const int32_t* slots;           // negative: the token is not cached
  __nv_bfloat16* k_cache;
  __nv_bfloat16* v_cache;
  int num_heads, num_kv_heads, head_dim;
};
// Packed columns 16 nt + r and 16 nt + r + 8 (r < 8) of token tok, with fp32 values lo / hi: the pair (dims d and
// d + D/2 of one head), rounded to bf16 as the linear's output, is rotated for q and k heads (rope_x / rope_y, NeoX
// halves, full rotary), written to row tok of y in logical [q | k | v] column order and, for k / v heads, into the paged
// caches (reshape_paged_cache.cu:23-62).
__device__ __forceinline__ void qkv_rope_store(const QkvRopeCache& p, __nv_bfloat16* y, int64_t y_stride, int tok, int nt,
                                               int r, float lo, float hi) {
  const int D = p.head_dim, half = D >> 1, tiles_per_head = D >> 4;
  const int hd = nt / tiles_per_head, d = (nt % tiles_per_head) * 8 + r;
  float v1 = round_bf16(lo), v2 = round_bf16(hi);
  const bool is_q = hd < p.num_heads, is_k = !is_q && hd < p.num_heads + p.num_kv_heads;
  if (is_q || is_k) {
    const __nv_bfloat16* cs = p.cos_sin + p.positions[tok] * (int64_t)D;
    const float c = __bfloat162float(cs[d]), sn = __bfloat162float(cs[half + d]);
    const float o1 = rope_x(v1, v2, c, sn);
    const float o2 = rope_y(v1, v2, c, sn);
    v1 = o1;
    v2 = o2;
  }
  const __nv_bfloat16 b1 = __float2bfloat16_rn(v1), b2 = __float2bfloat16_rn(v2);
  __nv_bfloat16* yr = y + (int64_t)tok * y_stride + (int64_t)hd * D;
  yr[d] = b1;
  yr[half + d] = b2;
  if (!is_q) {
    const int64_t slot = p.slots[tok];
    if (slot >= 0) {
      const int kvh = is_k ? hd - p.num_heads : hd - p.num_heads - p.num_kv_heads;
      __nv_bfloat16* row = (is_k ? p.k_cache : p.v_cache) + (slot * p.num_kv_heads + kvh) * (int64_t)D;
      row[d] = b1;
      row[half + d] = b2;
    }
  }
}

// gate activation in fp32 (activation.cu:97-125); kAct 0 silu, 1 gelu, 2 gelu_tanh.  The bf16 gated form is
// bf16(act(gate)) * up on bf16 gate and up (activation.cu:35).
template <int kAct>
__device__ __forceinline__ float act_fn(float f) {
  if (kAct == 0) return f / (1.0f + expf(-f));
  if (kAct == 1) return f * 0.5f * (1.0f + erff(f * 0.70710678118654752440f));
  const float kBeta = 0.79788456080286535588f;                       // sqrt(2)*2/sqrt(pi)*0.5
  const float inner = kBeta * (f + 0.044715f * f * f * f);
  return 0.5f * f * (1.0f + tanhf(inner));
}
__device__ __forceinline__ float act_fn(int act_mode, float f) {
  if (act_mode == 0) return act_fn<0>(f);
  if (act_mode == 1) return act_fn<1>(f);
  return act_fn<2>(f);
}

// SwiGLU on fp32 sums, rounded once by the caller: the MoE experts' form (the fused MoE's fc1 epilogue behind
// kernels/cuda/moe/fused_moe.cpp:23-124 gates the fp32 accumulators)
__device__ __forceinline__ float silu_mul_f32(float gate, float up) {
  return act_fn<0>(gate) * up;
}

#endif  // __CUDACC__
}  // namespace xb
