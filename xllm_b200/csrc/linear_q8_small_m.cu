// Small-M (decode, M <= 64) linears with 8-bit weights: HBM-bound weight-streaming kernels, the 8-bit siblings of
// linear_small_m.cu.
//
//  W8A16 (north-star "W4A16 / W8A16 / FP8"; spec oracle/quant.py with bits = 8; additive boundary SURVEY 8b-3, the
//  reference parses `bits` into QuantArgs - framework/quant_args.h:36-39 - but has no kernel):
//     w = bf16((q - z) * s), y = bf16(sum_k f32(x) f32(w) + b).  Weights are tile-packed like the W4 layout, one byte per
//     weight: qweight8[N/16][K/64][32 lanes][8 words]; lane (g,t) owns rows n0+g (words 0..3) and n0+g+8 (words 4..7),
//     k in [k0+16t, k0+16t+16), bytes ascending in k.  meta[K/g][N] = bf16 scale | zero << 16.  Dequant per 4 weights:
//     4 PRMT + 4 FADD + 2 CVT.BF16X2 + 2 HMUL2.BF16 (bit-exact, see w8_dequant_word), 4 legacy HMMAs per k64 tile.
//     The same packed tensor feeds the wgmma prefill GEMM (gemm_wgmma.cu kind W8).
//
//  FP8 W8A8 (fp8_linear_forward, xllm/core/layers/common/linear.cpp:137-182 -> cutlass_scaled_mm,
//  kernels/cuda/cutlass_w8a8/scaled_mm_entry.cu:55-108; the reference buckets M <= 16 / <= 64 into swap-AB tiles,
//  c3x/scaled_mm_sm100_fp8_dispatch.cuh:148-287): C = a_s * (b_s * (A8 . B8^T)) + bias with A8 [M,K] e4m3 activations and
//     B8 [N,K] e4m3 weights in the reference layout, untouched.  Weight rows ride in the M slot of mma.sync
//     m16n8k32.e4m3 (swap-AB), the <= 8 tokens of a tile in the n8 slot; a lane reads 16 bytes of rows n0+g and n0+g+8
//     per k64 tile, the k order inside a tile is permuted identically for both operands.  ~10 instructions per KB of
//     weights: the kernel is bandwidth-bound like the bf16 one.
#include <cstdlib>

#include "common.cuh"

namespace xb {

constexpr int kQ8Warps = 8;

// ---------------------------------------------------------------------------------------------------------------
// W8A16: warps of a CTA split K (interleaved k64 tiles) and reduce through shared memory; grid tiles N by 16 rows.
// Per-lane private cp.async ring (see linear_small_m.cu for why not a register ring).
// ---------------------------------------------------------------------------------------------------------------
template <int kMT, int kDepth>
__global__ void __launch_bounds__(kQ8Warps * 32, kMT >= 8 ? 1 : 2)
linear_w8a16_small_m_kernel(__nv_bfloat16* __restrict__ y, int64_t y_stride, const __nv_bfloat16* __restrict__ x,
                            int64_t x_stride, const uint4* __restrict__ qweight, const uint32_t* __restrict__ meta,
                            const __nv_bfloat16* __restrict__ bias, int M, int N, int K, int gshift /* log2(k64 tiles per group) */) {
  __shared__ float red[kQ8Warps][kMT][16 * 8];
  extern __shared__ __align__(16) uint8_t ring_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int ntile = blockIdx.x;
  const int n0 = ntile * 16;
  const int ktiles = K >> 6;
  // warp w owns k tiles [kb, ke): contiguous ranges (a quantisation group stays inside one warp when it can)
  const int per = (ktiles + kQ8Warps - 1) / kQ8Warps;
  const int kb = min(ktiles, warp * per), ke = min(ktiles, kb + per);
  constexpr int kSlotBytes = 1024 + 256;    // one k64 tile (32 lanes x 32 B) + 32 lanes x 2 meta words
  const uint32_t ring_w = smem_addr_u32(ring_smem) + warp * (kDepth * kSlotBytes) + lane * 32;
  const uint32_t ring_m = smem_addr_u32(ring_smem) + warp * (kDepth * kSlotBytes) + 1024 + lane * 8;
  const uint4* wp = qweight + ((int64_t)ntile * ktiles + kb) * 64 + lane * 2;
  const uint32_t* mbase = meta + n0 + g;
  auto issue = [&](int slot, int kt) {
    const uint4* src = wp + (int64_t)(kt - kb) * 64;
    cp_async_16(ring_w + slot * kSlotBytes, src);
    cp_async_16(ring_w + slot * kSlotBytes + 16, src + 1);
    const uint32_t* msrc = mbase + (int64_t)(kt >> gshift) * N;
    cp_async_4(ring_m + slot * kSlotBytes, msrc);
    cp_async_4(ring_m + slot * kSlotBytes + 4, msrc + 8);
  };
#pragma unroll
  for (int i = 0; i < kDepth; ++i) {
    if (kb + i < ke) issue(i, kb + i);
    cp_async_commit();
  }
  pdl_wait();   // x comes from the producer kernel

  float acc[kMT][4];
#pragma unroll
  for (int m = 0; m < kMT; ++m)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[m][i] = 0.f;
  const __nv_bfloat16* xp[kMT];
#pragma unroll
  for (int m = 0; m < kMT; ++m) xp[m] = x + (int64_t)min(m * 8 + g, M - 1) * x_stride + (int64_t)kb * 64 + 16 * t;

  auto consume = [&](int slot) {
    const uint4 w0 = lds_128(ring_w + slot * kSlotBytes), w1 = lds_128(ring_w + slot * kSlotBytes + 16);
    const uint2 mt = lds_64(ring_m + slot * kSlotBytes);
    uint32_t s0, s1;
    float nz0, nz1;
    w8_meta(mt.x, s0, nz0);
    w8_meta(mt.y, s1, nz1);
    uint32_t lo[8], hi[8];    // row g / row g+8: 16 bf16 = 8 packed registers, k ascending
    const uint32_t* a = &w0.x;
    const uint32_t* b = &w1.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      w8_dequant_word(a[j], nz0, s0, lo[2 * j], lo[2 * j + 1]);
      w8_dequant_word(b[j], nz1, s1, hi[2 * j], hi[2 * j + 1]);
    }
#pragma unroll
    for (int m = 0; m < kMT; ++m) {
      const uint4 xl = *reinterpret_cast<const uint4*>(xp[m]);
      const uint4 xh = *reinterpret_cast<const uint4*>(xp[m] + 8);
      xp[m] += 64;
      // k16 step i uses registers 2i, 2i+1 of both rows and of x (same k permutation on both operands)
      mma_bf16_16816(acc[m], lo[0], hi[0], lo[1], hi[1], xl.x, xl.y);
      mma_bf16_16816(acc[m], lo[2], hi[2], lo[3], hi[3], xl.z, xl.w);
      mma_bf16_16816(acc[m], lo[4], hi[4], lo[5], hi[5], xh.x, xh.y);
      mma_bf16_16816(acc[m], lo[6], hi[6], lo[7], hi[7], xh.z, xh.w);
    }
  };
  int kt = kb;
  for (; kt + kDepth <= ke; kt += kDepth) {
#pragma unroll
    for (int i = 0; i < kDepth; ++i) {
      cp_async_wait<kDepth - 1>();
      consume(i);
      if (kt + i + kDepth < ke) issue(i, kt + i + kDepth);
      cp_async_commit();
    }
  }
  cp_async_wait<0>();
#pragma unroll
  for (int i = 0; i < kDepth; ++i)
    if (kt + i < ke) consume(i);
  pdl_launch_dependents();

#pragma unroll
  for (int m = 0; m < kMT; ++m) store_c_frag(red[warp][m], acc[m], g, t);
  __syncthreads();
  for (int i = threadIdx.x; i < kMT * 128; i += blockDim.x) {
    const int m = i >> 7, r = (i & 127) >> 3, c = i & 7;
    const int tok = m * 8 + c;
    if (tok < M) {
      float s = 0.f;
#pragma unroll
      for (int ww = 0; ww < kQ8Warps; ++ww) s += red[ww][m][r * 8 + c];
      if (bias) s += __bfloat162float(bias[n0 + r]);
      y[(int64_t)tok * y_stride + n0 + r] = __float2bfloat16_rn(s);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// FP8 W8A8 (per-tensor or per-token / per-channel scales), weights [N,K] e4m3 row-major.
// ---------------------------------------------------------------------------------------------------------------
template <int kMT, int kUnroll>
__global__ void __launch_bounds__(kQ8Warps * 32)
linear_fp8_small_m_kernel(__nv_bfloat16* __restrict__ y, int64_t y_stride, const uint8_t* __restrict__ a8, int64_t a_stride,
                          const uint8_t* __restrict__ b8, const float* __restrict__ a_scale, int a_per_row,
                          const float* __restrict__ b_scale, int b_per_col, const __nv_bfloat16* __restrict__ bias, int M,
                          int N, int K) {
  __shared__ float red[kQ8Warps][kMT][16 * 8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int n0 = blockIdx.x * 16;
  const int ktiles = K >> 6;   // k64 tiles: 64 bytes per row
  const bool r0_ok = (n0 + g) < N, r1_ok = (n0 + g + 8) < N;
  const uint8_t* w0 = b8 + (int64_t)(n0 + g) * K + 16 * t;
  const uint8_t* w1 = b8 + (int64_t)(n0 + g + 8) * K + 16 * t;
  float acc[kMT][4];
#pragma unroll
  for (int m = 0; m < kMT; ++m)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[m][i] = 0.f;

  for (int kt0 = warp; kt0 < ktiles; kt0 += kQ8Warps * kUnroll) {
    uint4 wa[kUnroll], wb[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int kt = kt0 + u * kQ8Warps;
      wa[u] = make_uint4(0, 0, 0, 0);
      wb[u] = make_uint4(0, 0, 0, 0);
      if (kt < ktiles) {
        if (r0_ok) wa[u] = ldg_stream(w0 + (kt << 6));
        if (r1_ok) wb[u] = ldg_stream(w1 + (kt << 6));
      }
    }
    if (kt0 == warp) pdl_wait();   // weights are requested before the dependency wait, activations after it
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int kt = kt0 + u * kQ8Warps;
      if (kt < ktiles) {
#pragma unroll
        for (int m = 0; m < kMT; ++m) {
          const int tok = m * 8 + g;
          uint4 xv = make_uint4(0, 0, 0, 0);
          if (tok < M) xv = *reinterpret_cast<const uint4*>(a8 + (int64_t)tok * a_stride + (kt << 6) + 16 * t);
          // words (0,1) and (2,3) of the lane's 16-byte run fill the two k halves of one k32 step, on both operands
          mma_e4m3_16832(acc[m], wa[u].x, wb[u].x, wa[u].y, wb[u].y, xv.x, xv.y);
          mma_e4m3_16832(acc[m], wa[u].z, wb[u].z, wa[u].w, wb[u].w, xv.z, xv.w);
        }
      }
    }
  }
  if (ktiles <= warp) pdl_wait();
  pdl_launch_dependents();
#pragma unroll
  for (int m = 0; m < kMT; ++m) store_c_frag(red[warp][m], acc[m], g, t);
  __syncthreads();
  for (int i = threadIdx.x; i < kMT * 128; i += blockDim.x) {
    const int m = i >> 7, r = (i & 127) >> 3, c = i & 7;
    const int tok = m * 8 + c, n = n0 + r;
    if (tok < M && n < N) {
      float s = 0.f;
#pragma unroll
      for (int ww = 0; ww < kQ8Warps; ++ww) s += red[ww][m][r * 8 + c];
      // same order as the FP8 GEMM epilogue and the oracle: a_s * (b_s * acc) + bias
      const float as = a_scale[a_per_row ? tok : 0], bs = b_scale[b_per_col ? n : 0];
      float v = as * (bs * s);
      if (bias) v += __bfloat162float(bias[n]);
      y[(int64_t)tok * y_stride + n] = __float2bfloat16_rn(v);
    }
  }
}

}  // namespace xb

using namespace xb;

extern "C" int xb_linear_w8a16_small_m(void* y, int64_t y_stride, const void* x, int64_t x_stride, const uint32_t* qweight,
                                       const uint32_t* meta, const void* bias, int M, int N, int K, int group_size,
                                       xb_stream_t stream) {
  if (M == 0) return 0;
  XB_CHECK(M > 0 && M <= 64, "linear_w8a16_small_m: M=%d out of range (1..64); use the wgmma GEMM", M);
  XB_CHECK(N % 16 == 0 && K % 64 == 0, "linear_w8a16_small_m: N=%d must be %%16, K=%d %%64", N, K);
  XB_CHECK(group_size >= 64 && group_size % 64 == 0 && K % group_size == 0,
           "linear_w8a16_small_m: group_size %d must be a multiple of 64 dividing K=%d", group_size, K);
  const int tpg = group_size / 64;
  XB_CHECK((tpg & (tpg - 1)) == 0, "linear_w8a16_small_m: group_size/64 must be a power of two (got %d)", group_size);
  XB_CHECK(x_stride % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0, "linear_w8a16_small_m: x not 16B aligned");
  int gshift = 0;
  while ((1 << gshift) < tpg) ++gshift;
  auto* yy = reinterpret_cast<__nv_bfloat16*>(y);
  auto* xx = reinterpret_cast<const __nv_bfloat16*>(x);
  auto* qw = reinterpret_cast<const uint4*>(qweight);
  auto* bb = reinterpret_cast<const __nv_bfloat16*>(bias);
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid(N / 16), block(kQ8Warps * 32);
  constexpr int kDepth = 6;    // 6 KB of weights in flight per warp, 96 KB per SM at 2 CTAs
  constexpr size_t smem = (size_t)kQ8Warps * kDepth * (1024 + 256);
#define XB_W8(MT)                                                                                                   \
  {                                                                                                                 \
    constexpr auto kern = linear_w8a16_small_m_kernel<MT, kDepth>;                                                  \
    XB_CUDA_OK(set_max_dynamic_smem_once<kern>((int)smem));                                                         \
    XB_CUDA_OK(launch(kern, grid, block, smem, s, true, yy, y_stride, xx, x_stride, qw, meta, bb, M, N, K, gshift)); \
  }
  if (M <= 8) XB_W8(1)
  else if (M <= 16) XB_W8(2)
  else if (M <= 32) XB_W8(4)
  else XB_W8(8)
#undef XB_W8
  return 0;
}

extern "C" int xb_linear_fp8_small_m(void* c, int64_t ldc, const void* a, int64_t lda, const void* b, const float* a_scale,
                                     int a_scale_numel, const float* b_scale, int b_scale_numel, const void* bias, int M,
                                     int N, int K, xb_stream_t stream) {
  if (M == 0 || N == 0) return 0;
  XB_CHECK(M > 0 && M <= 64, "linear_fp8_small_m: M=%d out of range (1..64); use the wgmma GEMM", M);
  XB_CHECK(K % 64 == 0 && lda % 16 == 0, "linear_fp8_small_m: K=%d / lda=%lld must be multiples of 64 / 16", K, (long long)lda);
  XB_CHECK(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0, "linear_fp8_small_m: a / b not 16B aligned");
  XB_CHECK(a_scale_numel == 1 || a_scale_numel == M, "linear_fp8_small_m: a_scales must have numel 1 or M");
  XB_CHECK(b_scale_numel == 1 || b_scale_numel == N, "linear_fp8_small_m: b_scales must have numel 1 or N");
  auto* cc = reinterpret_cast<__nv_bfloat16*>(c);
  auto* aa = reinterpret_cast<const uint8_t*>(a);
  auto* bq = reinterpret_cast<const uint8_t*>(b);
  auto* bi = reinterpret_cast<const __nv_bfloat16*>(bias);
  dim3 grid((N + 15) / 16), block(kQ8Warps * 32);
  cudaStream_t s = (cudaStream_t)stream;
#define XB_F8(MT, U)                                                                                                   \
  XB_CUDA_OK(launch(linear_fp8_small_m_kernel<MT, U>, grid, block, 0, s, true, cc, ldc, aa, lda, bq, a_scale,           \
                    a_scale_numel > 1 ? 1 : 0, b_scale, b_scale_numel > 1 ? 1 : 0, bi, M, N, K))
  if (M <= 8) XB_F8(1, 8);
  else if (M <= 16) XB_F8(2, 4);
  else if (M <= 32) XB_F8(4, 2);
  else XB_F8(8, 1);
#undef XB_F8
  return 0;
}

// Host-side packer (plain C++): q[N,K] (one 8-bit value per byte) -> tile layout [N/16][K/64][32 lanes][8 words].
extern "C" int xb_w8_pack_rows(uint32_t* out, const uint8_t* q, int N, int K) {
  XB_CHECK(N % 16 == 0 && K % 64 == 0, "w8_pack_rows: N=%d must be %%16, K=%d %%64", N, K);
  const int ktiles = K / 64;
  for (int nt = 0; nt < N / 16; ++nt)
    for (int kt = 0; kt < ktiles; ++kt)
      for (int lane = 0; lane < 32; ++lane) {
        const int g = lane >> 2, t = lane & 3;
        for (int half = 0; half < 2; ++half) {
          const uint8_t* r = q + (size_t)(nt * 16 + g + 8 * half) * K + kt * 64 + 16 * t;
          for (int j = 0; j < 4; ++j) {
            const uint32_t w = (uint32_t)r[4 * j] | ((uint32_t)r[4 * j + 1] << 8) | ((uint32_t)r[4 * j + 2] << 16) |
                               ((uint32_t)r[4 * j + 3] << 24);
            out[(((size_t)nt * ktiles + kt) * 32 + lane) * 8 + half * 4 + j] = w;
          }
        }
      }
  return 0;
}
