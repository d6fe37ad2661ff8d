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

#endif  // __CUDACC__
}  // namespace xb
