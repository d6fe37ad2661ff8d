// Mixture of experts (SURVEY 8f n4): router top-k and the gated expert MLP at any token count.
//   xb_moe_fused_topk        replaces xllm::kernel::cuda::moe_fused_topk (kernels/cuda/moe/moe_fused_topk.cu:22-58 ->
//                            moe_topk_softmax_kernels.cuh / moe_topk_sigmoid_kernels.cuh): softmax or sigmoid scores in fp32,
//                            optional correction bias (added for the SELECTION, subtracted again from the returned weight,
//                            moe_topk_sigmoid_kernels.cuh:66-71,131-139), top-k by value with ties to the lower expert index
//                            (the ordering tests/core/kernels/cuda/moe/moe_topk_test.cu:31-55 pins), optional
//                            renormalisation by the sum of the k selected weights taken in selection order.
//   xb_moe_experts_bf16      replaces xllm::kernel::cuda::cutlass_fused_moe (kernels/cuda/moe/fused_moe.cpp:23-124 -> FlashInfer
//                            fused_moe_100) for unquantised bf16 experts - the only kind the reference's CUDA FusedMoE accepts
//                            (layers/cuda/fused_moe.cpp:39-42): fc1 [E, 2I, H] in [up | gate] row order (fused_moe.cpp /
//                            layers/cuda/fused_moe.cpp:124-126 "CUTLASS SwiGLU consumes fc1 as [linear, gate]"), fc2 [E, H, I].
// Two paths with the same arithmetic, chosen by the token count alone (moe_layout below):
//   decode, T < 65 (HBM-bound): every (token, selected expert) pair streams its expert's weights once with the register-
//     fragment GEMV of linear_small_m.cu; fc1 computes the up rows and the matching gate rows in one CTA and applies
//     silu(gate) * up on the fp32 sums (one rounding to bf16), fc2 writes bf16 rows per pair.
//   prefill, T >= 65 (tensor-core bound): the route kernel sorts the local pairs by expert on the device, the gather kernel
//     copies their x rows into that order, and two grouped wgmma GEMMs (gemm_wgmma.cu, kGroupFc1 / kGroupFc2) read each
//     expert's weights once per 128-row m tile: fc1 applies SwiGLU to the fp32 sums in its epilogue, fc2 stores its rows
//     back in pair order.
// Both end in the combine kernel: sum_k scale_k * y2_k in fp32 in selection order.  Experts outside [expert_begin,
// expert_end) (expert parallelism: fused_moe.cpp ep_rank / ep_size) contribute zero, as in the reference where the EP
// all-reduce adds the other ranks.
#include <climits>
#include <cstdlib>

#include "tc_common.cuh"

namespace xb {

// ---------------------------------------------------------------------------------------------------------------------
// router: one warp per token, up to 32 * kPerLane experts
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kTopkPerLane = 16;   // experts per lane: E <= 512

template <typename T>
__device__ __forceinline__ float to_f32(T v);
template <>
__device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__global__ void __launch_bounds__(128)
moe_fused_topk_kernel(float* __restrict__ weights, int32_t* __restrict__ ids, const T* __restrict__ gating, int64_t g_stride,
                      const float* __restrict__ bias, int num_tokens, int E, int k, int renormalize, int sigmoid) {
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tok = blockIdx.x * 4 + warp;
  if (tok >= num_tokens) return;
  const T* row = gating + (int64_t)tok * g_stride;
  float sc[kTopkPerLane];      // selection score of expert lane + 32 * i (-inf beyond E)
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < kTopkPerLane; ++i) {
    const int e = lane + 32 * i;
    sc[i] = e < E ? to_f32(row[e]) : -INFINITY;
    mx = fmaxf(mx, sc[i]);
  }
  if (sigmoid) {
#pragma unroll
    for (int i = 0; i < kTopkPerLane; ++i) {
      const int e = lane + 32 * i;
      if (e < E) {
        float v = 1.0f / (1.0f + expf(-sc[i]));
        if (bias) v = v + bias[e];
        sc[i] = v;
      }
    }
  } else {
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < kTopkPerLane; ++i) {
      const int e = lane + 32 * i;
      if (e < E) {
        sc[i] = expf(sc[i] - mx);
        sum += sc[i];
      }
    }
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
#pragma unroll
    for (int i = 0; i < kTopkPerLane; ++i)
      if (lane + 32 * i < E) sc[i] = sc[i] * inv;
  }
  float row_sum = 0.f;
  float my_w = 0.f;            // lane j keeps the j-th selected weight
  int my_id = 0;
  for (int kk = 0; kk < k; ++kk) {
    // lane-local best (ties: lower expert index = lower i), then the warp's best (ties: lower expert index)
    float bv = -INFINITY;
    int be = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < kTopkPerLane; ++i) {
      const int e = lane + 32 * i;
      if (e < E && (sc[i] > bv || (sc[i] == bv && e < be))) {
        bv = sc[i];
        be = e;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oe = __shfl_xor_sync(0xffffffffu, be, o);
      if (ov > bv || (ov == bv && oe < be)) {
        bv = ov;
        be = oe;
      }
    }
    // remove the winner from the candidates
    if ((be & 31) == lane) {
#pragma unroll
      for (int i = 0; i < kTopkPerLane; ++i)
        if (i == (be >> 5)) sc[i] = -INFINITY;
    }
    float w = bv;
    if (sigmoid && bias) w -= bias[be];
    row_sum += w;
    if (lane == kk) {
      my_w = w;
      my_id = be;
    }
  }
  if (lane < k) {
    if (renormalize) my_w = my_w * (1.0f / row_sum);
    weights[(int64_t)tok * k + lane] = my_w;
    ids[(int64_t)tok * k + lane] = my_id;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// expert-indexed GEMV: y[pair] = W[expert(pair)] . x[row(pair)]   (bf16 weights [E][N][K] row-major, M = 1 per pair)
//   kSwiGLU: W is fc1 [E][2I][K] in [up | gate] order; the CTA owns up rows n0.. and gate rows I + n0.. and writes
//            a[pair][n0 + r] = bf16(silu(gate) * up), both from the fp32 sums.
// lane (g, t) reads rows n0+g and n0+g+8, 16 bytes per k32 tile (the layout of linear_bf16_small_m_kernel); the token sits
// in column 0 of the n8 slot.
// ---------------------------------------------------------------------------------------------------------------------
template <bool kSwiGLU>
__global__ void __launch_bounds__(256)
moe_expert_gemv_kernel(__nv_bfloat16* __restrict__ y, int64_t y_stride, const __nv_bfloat16* __restrict__ x, int64_t x_stride,
                       int x_row_div /* x row = pair / x_row_div */, const __nv_bfloat16* __restrict__ w,
                       const int32_t* __restrict__ expert_ids, int N /* output rows per expert (I for SwiGLU) */, int K,
                       int expert_begin, int expert_end) {
  constexpr int kW = 8;
  __shared__ float red[kW][kSwiGLU ? 2 : 1][16];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int pair = blockIdx.y;
  const int n0 = blockIdx.x * 16;
  pdl_launch_dependents();
  pdl_wait();
  const int e_glob = expert_ids[pair];
  const bool mine = e_glob >= expert_begin && e_glob < expert_end;
  const int e = e_glob - expert_begin;
  const int rows_per_expert = kSwiGLU ? 2 * N : N;
  const __nv_bfloat16* we = w + (int64_t)(mine ? e : 0) * rows_per_expert * K;
  const __nv_bfloat16* xr = x + (int64_t)(pair / x_row_div) * x_stride;
  const int ktiles = K >> 5;
  float acc[kSwiGLU ? 2 : 1][4];
#pragma unroll
  for (int h = 0; h < (kSwiGLU ? 2 : 1); ++h)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[h][i] = 0.f;
  if (mine) {
    const bool r0 = n0 + g < N, r1 = n0 + g + 8 < N;
    constexpr int kU = 4;
    for (int kt0 = warp; kt0 < ktiles; kt0 += kW * kU) {
      uint4 wa[kSwiGLU ? 2 : 1][kU], wb[kSwiGLU ? 2 : 1][kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int kt = kt0 + u * kW;
#pragma unroll
        for (int h = 0; h < (kSwiGLU ? 2 : 1); ++h) {
          wa[h][u] = make_uint4(0, 0, 0, 0);
          wb[h][u] = make_uint4(0, 0, 0, 0);
          if (kt < ktiles) {
            const __nv_bfloat16* base = we + (int64_t)(h * N + n0) * K + (kt << 5) + 8 * t;
            if (r0) wa[h][u] = ldg_stream(base + (int64_t)g * K);
            if (r1) wb[h][u] = ldg_stream(base + (int64_t)(g + 8) * K);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int kt = kt0 + u * kW;
        if (kt < ktiles) {
          uint4 xv = make_uint4(0, 0, 0, 0);
          if (g == 0) xv = *reinterpret_cast<const uint4*>(xr + (kt << 5) + 8 * t);   // token in column 0 only
#pragma unroll
          for (int h = 0; h < (kSwiGLU ? 2 : 1); ++h) {
            mma_bf16_16816(acc[h], wa[h][u].x, wb[h][u].x, wa[h][u].y, wb[h][u].y, xv.x, xv.y);
            mma_bf16_16816(acc[h], wa[h][u].z, wb[h][u].z, wa[h][u].w, wb[h][u].w, xv.z, xv.w);
          }
        }
      }
    }
  }
  // C fragment: c0 = (row g, col 2t), c2 = (row g+8, col 2t); the token is column 0 -> lanes with t == 0
  if (t == 0) {
#pragma unroll
    for (int h = 0; h < (kSwiGLU ? 2 : 1); ++h) {
      red[warp][h][g] = acc[h][0];
      red[warp][h][g + 8] = acc[h][2];
    }
  }
  __syncthreads();
  if (threadIdx.x < 16) {
    const int r = threadIdx.x;
    if (n0 + r < N) {
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int ww = 0; ww < kW; ++ww) {
        s0 += red[ww][0][r];
        if (kSwiGLU) s1 += red[ww][1][r];
      }
      float out = s0;
      if (kSwiGLU) out = silu_mul_f32(s1, s0);
      y[(int64_t)pair * y_stride + n0 + r] = __float2bfloat16_rn(mine ? out : 0.f);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// W4A16 experts (SURVEY cfg[4] "MoE W4A16"; additive like the dense W4A16 linears - the reference's CUDA FusedMoE takes
// unquantised experts only): the same expert-indexed GEMV over the tile-packed int4 layout of linear_small_m.cu, one
// [rows/16][K/64][32][4] weight and one [K/g][rows] meta block per expert, dequantised by w4_dequant_word (common.cuh)
// right before the mma.
// ---------------------------------------------------------------------------------------------------------------------

template <bool kSwiGLU>
__global__ void __launch_bounds__(256)
moe_expert_gemv_w4_kernel(__nv_bfloat16* __restrict__ y, int64_t y_stride, const __nv_bfloat16* __restrict__ x, int64_t x_stride,
                          int x_row_div, const uint4* __restrict__ qweight, const uint32_t* __restrict__ meta,
                          const int32_t* __restrict__ expert_ids, int N /* output rows per expert (I for SwiGLU) */, int K,
                          int gshift /* log2(k64 tiles per quantisation group) */, int expert_begin, int expert_end) {
  constexpr int kW = 8, kH = kSwiGLU ? 2 : 1;
  __shared__ float red[kW][kH][16];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int pair = blockIdx.y;
  const int n0 = blockIdx.x * 16;
  pdl_launch_dependents();
  pdl_wait();
  const int e_glob = expert_ids[pair];
  const bool mine = e_glob >= expert_begin && e_glob < expert_end;
  const int e = mine ? e_glob - expert_begin : 0;
  const int rows = kSwiGLU ? 2 * N : N;
  const int ktiles = K >> 6;
  const uint4* qe = qweight + (int64_t)e * (rows >> 4) * ktiles * 32;
  const uint32_t* me = meta + (int64_t)e * ((ktiles >> gshift) * (int64_t)rows);
  const __nv_bfloat16* xr = x + (int64_t)(pair / x_row_div) * x_stride;
  float acc[kH][4];
#pragma unroll
  for (int h = 0; h < kH; ++h)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[h][i] = 0.f;
  if (mine && n0 < N) {
    constexpr int kU = 4;
    for (int kt0 = warp; kt0 < ktiles; kt0 += kW * kU) {
      uint4 wq[kH][kU];
      uint32_t m0[kH][kU], m1[kH][kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int kt = kt0 + u * kW;
#pragma unroll
        for (int h = 0; h < kH; ++h) {
          wq[h][u] = make_uint4(0, 0, 0, 0);
          m0[h][u] = m1[h][u] = 0;
          if (kt < ktiles) {
            const int row0 = h * N + n0;                       // up rows, then the matching gate rows
            wq[h][u] = ldg_stream(qe + ((int64_t)(row0 >> 4) * ktiles + kt) * 32 + lane);
            const uint32_t* mr = me + (int64_t)(kt >> gshift) * rows + row0;
            m0[h][u] = __ldg(mr + g);
            m1[h][u] = __ldg(mr + g + 8);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int kt = kt0 + u * kW;
        if (kt < ktiles) {
          uint4 xlo = make_uint4(0, 0, 0, 0), xhi = make_uint4(0, 0, 0, 0);
          if (g == 0) {                                        // the token sits in column 0 of the n8 slot
            const uint4* xp = reinterpret_cast<const uint4*>(xr + (kt << 6) + 16 * t);
            xlo = xp[0];
            xhi = xp[1];
          }
#pragma unroll
          for (int h = 0; h < kH; ++h) {
            uint32_t s0, z0, s1, z1;
            w4_meta(m0[h][u], s0, z0);
            w4_meta(m1[h][u], s1, z1);
            const uint32_t* wv = &wq[h][u].x;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              uint32_t a[4];
              w4_dequant_word(wv[j], z0, s0, z1, s1, a);
              const uint32_t* xv = j < 2 ? &xlo.x : &xhi.x;
              mma_bf16_16816(acc[h], a[0], a[1], a[2], a[3], xv[(j & 1) * 2], xv[(j & 1) * 2 + 1]);
            }
          }
        }
      }
    }
  }
  if (t == 0) {
#pragma unroll
    for (int h = 0; h < kH; ++h) {
      red[warp][h][g] = acc[h][0];
      red[warp][h][g + 8] = acc[h][2];
    }
  }
  __syncthreads();
  if (threadIdx.x < 16) {
    const int r = threadIdx.x;
    if (n0 + r < N) {
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int ww = 0; ww < kW; ++ww) {
        s0 += red[ww][0][r];
        if (kSwiGLU) s1 += red[ww][1][r];
      }
      float out = s0;
      if (kSwiGLU) out = silu_mul_f32(s1, s0);
      y[(int64_t)pair * y_stride + n0 + r] = __float2bfloat16_rn(mine ? out : 0.f);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// grouped (prefill) path: device-side routing.  The route kernel sorts the local pairs by expert (stable: pair order within
// an expert) and writes the workspace header the grouped GEMMs schedule from; the gather kernel copies the x rows into that
// order, because TMA loads boxes of consecutive rows and cannot gather.  Nothing is read back to the host, and the header is
// rewritten from scratch by every call, so one captured CUDA graph serves any routing.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kMoeMaxExperts = 512;           // local experts of the grouped path (the router's limit)
constexpr int kHdrRowStart = 0;               // [E + 1] first sorted row of each local expert (exclusive scan of the counts)
constexpr int kHdrMtileStart = 520;           // [E + 1] first 128-row m tile of each local expert
constexpr int kHdrCounts = 1040;              // [E] local pairs of each expert
constexpr int64_t kMoeHeaderBytes = 8192;

__global__ void __launch_bounds__(1024)
moe_route_kernel(int32_t* __restrict__ hdr, int32_t* __restrict__ row_of_pair, int32_t* __restrict__ pair_of_row,
                 const int32_t* __restrict__ expert_ids, int P, int E, int expert_begin, int expert_end) {
  __shared__ int next_row[kMoeMaxExperts];                 // pairs per local expert, then the next free row of each
  __shared__ uint8_t round_cnt[32][kMoeMaxExperts];       // pairs of the current 1024-pair round per (warp, expert)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_launch_dependents();
  for (int i = tid; i < kMoeMaxExperts; i += blockDim.x) next_row[i] = 0;
  for (int i = tid; i < 32 * kMoeMaxExperts / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(round_cnt)[i] = 0;
  __syncthreads();
  pdl_wait();                                              // ids come from the router; the previous call is done with hdr
  auto local_expert = [&](int p) {
    const int id = expert_ids[p];
    return id >= expert_begin && id < expert_end ? id - expert_begin : -1;
  };
  for (int p = tid; p < P; p += blockDim.x) {
    const int e = local_expert(p);
    if (e >= 0) atomicAdd(&next_row[e], 1);
  }
  __syncthreads();
  if (warp == 0) {
    // exclusive scans of the rows and of the 128-row m tiles; lane l owns experts 16 l .. 16 l + 15
    constexpr int kPer = kMoeMaxExperts / 32;
    int c[kPer], rows = 0, tiles = 0;
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
      const int e = lane * kPer + i;
      c[i] = e < E ? next_row[e] : 0;
      rows += c[i];
      tiles += (c[i] + 127) >> 7;
    }
    int rows_inc = rows, tiles_inc = tiles;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int r = __shfl_up_sync(0xffffffffu, rows_inc, o), t = __shfl_up_sync(0xffffffffu, tiles_inc, o);
      if (lane >= o) {
        rows_inc += r;
        tiles_inc += t;
      }
    }
    int r = rows_inc - rows, t = tiles_inc - tiles;
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
      const int e = lane * kPer + i;
      if (e < E) {
        hdr[kHdrCounts + e] = c[i];
        hdr[kHdrRowStart + e] = r;
        hdr[kHdrMtileStart + e] = t;
        next_row[e] = r;
      }
      r += c[i];
      t += (c[i] + 127) >> 7;
    }
    if (lane == 31) {
      hdr[kHdrRowStart + E] = rows_inc;
      hdr[kHdrMtileStart + E] = tiles_inc;
    }
  }
  __syncthreads();
  // stable placement, 1024 pairs per round: row = the expert's next free row + its pairs in lower warps of this round + its
  // pairs in lower lanes of this warp
  for (int base = 0; base < P; base += blockDim.x) {
    const int p = base + tid;
    const int e = p < P ? local_expert(p) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, e);
    const bool leader = lane == __ffs(peers) - 1;
    if (e >= 0 && leader) round_cnt[warp][e] = (uint8_t)__popc(peers);
    __syncthreads();
    if (e >= 0) {
      int row = next_row[e] + __popc(peers & ((1u << lane) - 1u));
      for (int w = 0; w < warp; ++w) row += round_cnt[w][e];
      row_of_pair[p] = row;
      pair_of_row[row] = p;
    } else if (p < P) {
      row_of_pair[p] = -1;
    }
    __syncthreads();
    if (e >= 0 && leader) {
      atomicAdd(&next_row[e], __popc(peers));
      round_cnt[warp][e] = 0;
    }
    __syncthreads();
  }
}

// a_sorted[row_of_pair[p]] = x[p / k] for the local pairs; y2[p] = 0 for the others, so the combine can read every pair
__global__ void __launch_bounds__(256)
moe_gather_kernel(__nv_bfloat16* __restrict__ a_sorted, __nv_bfloat16* __restrict__ y2, const __nv_bfloat16* __restrict__ x,
                  int64_t x_stride, const int32_t* __restrict__ row_of_pair, int k, int H) {
  pdl_launch_dependents();
  pdl_wait();
  const int p = blockIdx.x;
  const int row = row_of_pair[p];
  const int chunks = H / 8;                                // 16-byte chunks per row
  if (row >= 0) {
    const uint4* src = reinterpret_cast<const uint4*>(x + (int64_t)(p / k) * x_stride);
    uint4* dst = reinterpret_cast<uint4*>(a_sorted + (int64_t)row * H);
    for (int i = threadIdx.x; i < chunks; i += blockDim.x) dst[i] = src[i];
  } else {
    uint4* dst = reinterpret_cast<uint4*>(y2 + (int64_t)p * H);
    for (int i = threadIdx.x; i < chunks; i += blockDim.x) dst[i] = make_uint4(0, 0, 0, 0);
  }
}

// out[t] = bf16( sum_k scale[t,k] * y2[t*k + kk] ), fp32, selection order
__global__ void __launch_bounds__(256)
moe_combine_kernel(__nv_bfloat16* __restrict__ out, int64_t out_stride, const __nv_bfloat16* __restrict__ y2, const float* __restrict__ scales,
                   int k, int H) {
  pdl_launch_dependents();
  pdl_wait();
  const int tok = blockIdx.y;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < H / 2; c += gridDim.x * blockDim.x) {
    float a0 = 0.f, a1 = 0.f;
    for (int kk = 0; kk < k; ++kk) {
      const float s = scales[(int64_t)tok * k + kk];
      const uint32_t v = reinterpret_cast<const uint32_t*>(y2 + ((int64_t)tok * k + kk) * H)[c];
      a0 = fmaf(s, bf16lo(v), a0);
      a1 = fmaf(s, bf16hi(v), a1);
    }
    reinterpret_cast<uint32_t*>(out + (int64_t)tok * out_stride)[c] = pack_bf16x2(a0, a1);
  }
}

}  // namespace xb

using namespace xb;

extern "C" int xb_moe_fused_topk(float* topk_weights, int32_t* topk_ids, const void* gating_output, int gating_is_bf16,
                                 int64_t gating_stride, const float* correction_bias, int num_tokens, int num_experts,
                                 int topk, int renormalize, int scoring_sigmoid, xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  XB_CHECK(num_experts >= 1 && num_experts <= 32 * kTopkPerLane, "moe_fused_topk: %d experts unsupported (1..%d)", num_experts,
           32 * kTopkPerLane);
  XB_CHECK(topk >= 1 && topk <= 32 && topk <= num_experts, "moe_fused_topk: topk %d out of range (1..min(32, experts))", topk);
  XB_CHECK(scoring_sigmoid || correction_bias == nullptr, "moe_fused_topk: correction_bias goes with sigmoid scoring");
  dim3 grid((num_tokens + 3) / 4), block(128);
  if (gating_is_bf16)
    XB_CUDA_OK(launch(moe_fused_topk_kernel<__nv_bfloat16>, grid, block, 0, (cudaStream_t)stream, true, topk_weights, topk_ids,
                      reinterpret_cast<const __nv_bfloat16*>(gating_output), gating_stride, correction_bias, num_tokens,
                      num_experts, topk, renormalize, scoring_sigmoid));
  else
    XB_CUDA_OK(launch(moe_fused_topk_kernel<float>, grid, block, 0, (cudaStream_t)stream, true, topk_weights, topk_ids,
                      reinterpret_cast<const float*>(gating_output), gating_stride, correction_bias, num_tokens, num_experts,
                      topk, renormalize, scoring_sigmoid));
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// path choice and workspace layout: the one host rule the entry points, the workspace query and xb_moe_experts_describe share
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kMoeGemvMaxPairs = 65535;        // GEMV path: one CTA row per pair in grid.y
constexpr int kMoeGroupedMaxTokens = 65535;    // grouped path: the combine kernel's grid.y
constexpr int kMoeGroupedMaxTopk = 32;         // the router's limit

// smallest token count that takes the grouped path.  65 by default: T <= 64 is the decode range, the same M <= 64 boundary as
// the dense linears' streaming kernels.  XB_MOE_GROUPED_MIN_TOKENS / xb_set_moe_grouped_min_tokens move it (tests, sweeps).
static std::atomic<int> g_moe_grouped_min_tokens{-1};
static int moe_grouped_min_tokens() {
  int v = g_moe_grouped_min_tokens.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("XB_MOE_GROUPED_MIN_TOKENS");
    v = e ? atoi(e) : 65;
    if (v < 1) v = 65;
    g_moe_grouped_min_tokens.store(v, std::memory_order_relaxed);
  }
  return v;
}

// GEMV:    act [P][I] | y2 [P][H]                                              (P = T * k pairs)
// grouped: header (8 KB) | row_of_pair [P] i32 | pair_of_row [P] i32 (each padded to 256 bytes) | x_sorted [P][H] | act [P][I]
//          | y2 [P][H], all bf16 except the maps
struct MoeLayout {
  bool grouped;
  int64_t bytes, row_of_pair, pair_of_row, x_sorted, act, y2;   // byte offsets
};
static MoeLayout moe_layout(int num_tokens, int topk, int hidden, int inter) {
  MoeLayout l{};
  const int64_t P = (int64_t)num_tokens * topk;
  l.grouped = num_tokens >= moe_grouped_min_tokens();
  if (!l.grouped) {
    l.act = 0;
    l.y2 = P * inter * 2;
    l.bytes = (int64_t)num_tokens * topk * ((int64_t)inter + hidden) * 2;
    return l;
  }
  const int64_t map = (P * 4 + 255) / 256 * 256;
  l.row_of_pair = kMoeHeaderBytes;
  l.pair_of_row = l.row_of_pair + map;
  l.x_sorted = l.pair_of_row + map;
  l.act = l.x_sorted + P * hidden * 2;
  l.y2 = l.act + P * inter * 2;
  l.bytes = l.y2 + P * hidden * 2;
  return l;
}

// shape limits of the grouped path (int64 byte offsets throughout; TMA coordinates are int32)
static int moe_grouped_check(const char* name, int num_tokens, int topk, int hidden, int inter, int num_local_experts) {
  XB_CHECK(num_tokens <= kMoeGroupedMaxTokens && topk <= kMoeGroupedMaxTopk && num_local_experts <= kMoeMaxExperts,
           "%s: %d tokens x top-%d over %d local experts exceed the grouped path (tokens <= %d, topk <= %d, experts <= %d)", name,
           num_tokens, topk, num_local_experts, kMoeGroupedMaxTokens, kMoeGroupedMaxTopk, kMoeMaxExperts);
  XB_CHECK((int64_t)num_local_experts * 2 * inter <= INT_MAX && (int64_t)num_local_experts * hidden <= INT_MAX,
           "%s: %d experts x (hidden %d, 2 x inter %d) weight rows exceed int32", name, num_local_experts, hidden, inter);
  return 0;
}

static int moe_grouped_run(bool w4, void* out, int64_t out_stride, const void* input, int64_t in_stride,
                           const int32_t* token_selected_experts, const float* token_final_scales, const void* fc1,
                           const uint32_t* fc1_meta, const void* fc2, const uint32_t* fc2_meta, int gshift, int group_size,
                           int num_tokens, int topk, int hidden, int inter, int num_local_experts, int expert_begin,
                           void* workspace, const MoeLayout& l, cudaStream_t s) {
  const int pairs = num_tokens * topk;
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  auto* hdr = reinterpret_cast<int32_t*>(ws);
  auto* row_of_pair = reinterpret_cast<int32_t*>(ws + l.row_of_pair);
  auto* pair_of_row = reinterpret_cast<int32_t*>(ws + l.pair_of_row);
  auto* x_sorted = reinterpret_cast<__nv_bfloat16*>(ws + l.x_sorted);
  auto* act = reinterpret_cast<__nv_bfloat16*>(ws + l.act);
  auto* y2 = reinterpret_cast<__nv_bfloat16*>(ws + l.y2);
  XB_CUDA_OK(launch(moe_route_kernel, dim3(1), dim3(1024), 0, s, true, hdr, row_of_pair, pair_of_row, token_selected_experts,
                    pairs, num_local_experts, expert_begin, expert_begin + num_local_experts));
  XB_CUDA_OK(launch(moe_gather_kernel, dim3(pairs), dim3(256), 0, s, true, x_sorted, y2,
                    reinterpret_cast<const __nv_bfloat16*>(input), in_stride, row_of_pair, topk, hidden));
  if (int rc = tc::moe_grouped_gemm(w4, 0, act, x_sorted, fc1, fc1_meta, gshift, group_size, hdr + kHdrRowStart,
                                    hdr + kHdrMtileStart, pair_of_row, pairs, hidden, inter, num_local_experts, s))
    return rc;
  if (int rc = tc::moe_grouped_gemm(w4, 1, y2, act, fc2, fc2_meta, gshift, group_size, hdr + kHdrRowStart,
                                    hdr + kHdrMtileStart, pair_of_row, pairs, hidden, inter, num_local_experts, s))
    return rc;
  const int cx = (hidden / 2 + 255) / 256;
  XB_CUDA_OK(launch(moe_combine_kernel, dim3(cx, num_tokens), dim3(256), 0, s, true, reinterpret_cast<__nv_bfloat16*>(out),
                    out_stride, reinterpret_cast<const __nv_bfloat16*>(y2), token_final_scales, topk, hidden));
  return 0;
}

extern "C" int xb_set_moe_grouped_min_tokens(int min_tokens) {
  if (min_tokens < 1) {
    set_error("set_moe_grouped_min_tokens: %d out of range (>= 1)", min_tokens);
    return -1;
  }
  const int old = moe_grouped_min_tokens();
  g_moe_grouped_min_tokens.store(min_tokens, std::memory_order_relaxed);
  return old;
}

extern "C" int xb_moe_experts_describe(int kind, int num_tokens, int topk, int hidden, int inter, int num_local_experts,
                                       char* buf, int buf_len) {
  if ((kind != 0 && kind != 2) || buf == nullptr || buf_len <= 0) return -1;
  const char* name = kind == 0 ? "bf16" : "w4";
  if (!moe_layout(num_tokens, topk, hidden, inter).grouped) return snprintf(buf, (size_t)buf_len, "%s gemv", name);
  // upper bound of the grouped GEMMs' tiles: every local expert adds at most one partial 128-row m tile
  const int64_t m_tiles = ((int64_t)num_tokens * topk + 127) / 128 + (num_local_experts > 0 ? num_local_experts : 0);
  return snprintf(buf, (size_t)buf_len, "%s grouped bn=128 m_tiles<=%lld", name, (long long)m_tiles);
}

extern "C" int64_t xb_moe_experts_workspace_bytes(int num_tokens, int topk, int hidden, int inter) {
  return moe_layout(num_tokens, topk, hidden, inter).bytes;
}

extern "C" int xb_moe_experts_bf16(void* out, int64_t out_stride, const void* input, int64_t in_stride,
                                   const int32_t* token_selected_experts, const float* token_final_scales,
                                   const void* fc1_weights, const void* fc2_weights, int num_tokens, int topk, int hidden,
                                   int inter, int num_local_experts, int expert_begin, void* workspace,
                                   int64_t workspace_bytes, xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  XB_CHECK(hidden % 32 == 0 && inter % 32 == 0, "moe_experts: hidden %d / inter %d must be multiples of 32", hidden, inter);
  XB_CHECK(topk >= 1 && num_local_experts >= 1, "moe_experts: bad topk %d / experts %d", topk, num_local_experts);
  const MoeLayout l = moe_layout(num_tokens, topk, hidden, inter);
  if (l.grouped) {
    if (int rc = moe_grouped_check("moe_experts", num_tokens, topk, hidden, inter, num_local_experts)) return rc;
  } else {
    XB_CHECK((int64_t)num_tokens * topk <= kMoeGemvMaxPairs,
             "moe_experts: %d x %d (token, expert) pairs exceed the decode-sized path (65535)", num_tokens, topk);
  }
  XB_CHECK(workspace != nullptr && workspace_bytes >= l.bytes, "moe_experts: workspace too small (need %lld bytes)",
           (long long)l.bytes);
  XB_CHECK(in_stride % 8 == 0 && out_stride % 2 == 0 &&
               ((reinterpret_cast<uintptr_t>(input) | reinterpret_cast<uintptr_t>(fc1_weights) |
                 reinterpret_cast<uintptr_t>(fc2_weights) | reinterpret_cast<uintptr_t>(workspace)) & 15) == 0,
           "moe_experts: 16-byte alignment");
  cudaStream_t s = (cudaStream_t)stream;
  if (l.grouped)
    return moe_grouped_run(false, out, out_stride, input, in_stride, token_selected_experts, token_final_scales, fc1_weights,
                           nullptr, fc2_weights, nullptr, 0, 0, num_tokens, topk, hidden, inter, num_local_experts,
                           expert_begin, workspace, l, s);
  const int pairs = num_tokens * topk;
  auto* act = reinterpret_cast<__nv_bfloat16*>(workspace);                 // [pairs][inter]
  auto* y2 = act + (int64_t)pairs * inter;                                 // [pairs][hidden]
  XB_CUDA_OK(launch(moe_expert_gemv_kernel<true>, dim3((inter + 15) / 16, pairs), dim3(256), 0, s, true, act, (int64_t)inter,
                    reinterpret_cast<const __nv_bfloat16*>(input), in_stride, topk,
                    reinterpret_cast<const __nv_bfloat16*>(fc1_weights), token_selected_experts, inter, hidden, expert_begin,
                    expert_begin + num_local_experts));
  XB_CUDA_OK(launch(moe_expert_gemv_kernel<false>, dim3((hidden + 15) / 16, pairs), dim3(256), 0, s, true, y2, (int64_t)hidden,
                    reinterpret_cast<const __nv_bfloat16*>(act), (int64_t)inter, 1,
                    reinterpret_cast<const __nv_bfloat16*>(fc2_weights), token_selected_experts, hidden, inter, expert_begin,
                    expert_begin + num_local_experts));
  const int cx = (hidden / 2 + 255) / 256;
  XB_CUDA_OK(launch(moe_combine_kernel, dim3(cx, num_tokens), dim3(256), 0, s, true, reinterpret_cast<__nv_bfloat16*>(out),
                    out_stride, reinterpret_cast<const __nv_bfloat16*>(y2), token_final_scales, topk, hidden));
  return 0;
}

extern "C" int xb_moe_experts_w4a16(void* out, int64_t out_stride, const void* input, int64_t in_stride,
                                    const int32_t* token_selected_experts, const float* token_final_scales,
                                    const uint32_t* fc1_qweight, const uint32_t* fc1_meta, const uint32_t* fc2_qweight,
                                    const uint32_t* fc2_meta, int group_size, int num_tokens, int topk, int hidden, int inter,
                                    int num_local_experts, int expert_begin, void* workspace, int64_t workspace_bytes,
                                    xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  XB_CHECK(hidden % 64 == 0 && inter % 64 == 0, "moe_experts_w4a16: hidden %d / inter %d must be multiples of 64", hidden, inter);
  XB_CHECK(group_size >= 64 && group_size % 64 == 0 && hidden % group_size == 0 && inter % group_size == 0,
           "moe_experts_w4a16: group_size %d must be a multiple of 64 dividing hidden and inter", group_size);
  const int tpg = group_size / 64;
  XB_CHECK((tpg & (tpg - 1)) == 0, "moe_experts_w4a16: group_size / 64 must be a power of two (got %d)", group_size);
  int gshift = 0;
  while ((1 << gshift) < tpg) ++gshift;
  const MoeLayout l = moe_layout(num_tokens, topk, hidden, inter);
  if (l.grouped) {
    XB_CHECK(topk >= 1 && num_local_experts >= 1, "moe_experts_w4a16: bad topk %d / experts %d", topk, num_local_experts);
    if (int rc = moe_grouped_check("moe_experts_w4a16", num_tokens, topk, hidden, inter, num_local_experts)) return rc;
  } else {
    XB_CHECK(topk >= 1 && num_local_experts >= 1 && (int64_t)num_tokens * topk <= kMoeGemvMaxPairs,
             "moe_experts_w4a16: bad topk / experts / pairs");
  }
  XB_CHECK(workspace != nullptr && workspace_bytes >= l.bytes, "moe_experts_w4a16: workspace too small (need %lld bytes)",
           (long long)l.bytes);
  XB_CHECK(in_stride % 8 == 0 && out_stride % 2 == 0 &&
               ((reinterpret_cast<uintptr_t>(input) | reinterpret_cast<uintptr_t>(fc1_qweight) |
                 reinterpret_cast<uintptr_t>(fc2_qweight) | reinterpret_cast<uintptr_t>(workspace)) & 15) == 0,
           "moe_experts_w4a16: 16-byte alignment");
  cudaStream_t s = (cudaStream_t)stream;
  if (l.grouped) {
    // the grouped GEMMs load the meta words with TMA as well
    XB_CHECK(((reinterpret_cast<uintptr_t>(fc1_meta) | reinterpret_cast<uintptr_t>(fc2_meta)) & 15) == 0,
             "moe_experts_w4a16: 16-byte alignment of the meta words");
    return moe_grouped_run(true, out, out_stride, input, in_stride, token_selected_experts, token_final_scales, fc1_qweight,
                           fc1_meta, fc2_qweight, fc2_meta, gshift, group_size, num_tokens, topk, hidden, inter,
                           num_local_experts, expert_begin, workspace, l, s);
  }
  const int pairs = num_tokens * topk;
  auto* act = reinterpret_cast<__nv_bfloat16*>(workspace);
  auto* y2 = act + (int64_t)pairs * inter;
  XB_CUDA_OK(launch(moe_expert_gemv_w4_kernel<true>, dim3(inter / 16, pairs), dim3(256), 0, s, true, act, (int64_t)inter,
                    reinterpret_cast<const __nv_bfloat16*>(input), in_stride, topk, reinterpret_cast<const uint4*>(fc1_qweight),
                    fc1_meta, token_selected_experts, inter, hidden, gshift, expert_begin, expert_begin + num_local_experts));
  XB_CUDA_OK(launch(moe_expert_gemv_w4_kernel<false>, dim3(hidden / 16, pairs), dim3(256), 0, s, true, y2, (int64_t)hidden,
                    reinterpret_cast<const __nv_bfloat16*>(act), (int64_t)inter, 1, reinterpret_cast<const uint4*>(fc2_qweight),
                    fc2_meta, token_selected_experts, hidden, inter, gshift, expert_begin, expert_begin + num_local_experts));
  const int cx = (hidden / 2 + 255) / 256;
  XB_CUDA_OK(launch(moe_combine_kernel, dim3(cx, num_tokens), dim3(256), 0, s, true, reinterpret_cast<__nv_bfloat16*>(out),
                    out_stride, reinterpret_cast<const __nv_bfloat16*>(y2), token_final_scales, topk, hidden));
  return 0;
}
