// Small-M (decode, M <= 64) linears: y[M,N] = x[M,K] . W^T (+bias).
//
// These are HBM-bound weight-streaming kernels: every weight byte is read once
// with 16-byte coalesced loads straight into mma.sync fragments (no shared
// memory staging of W), the M<=8 token columns ride in the n8 slot of
// m16n8k16, fp32 accumulation.  The warps of a CTA split K and reduce through
// shared memory; the CTA grid tiles N.  Weight loads are issued BEFORE the PDL
// dependency wait (they do not depend on the producer kernel), so in a chained
// decode step the HBM stream of layer i+1 starts while layer i drains.
//
// W4A16 spec (oracle/quant.py): w = bf16((q - z) * s); dequant is 1 LOP3
// (+1 SHF) + HSUB2.BF16 + HMUL2.BF16 per weight PAIR, bit-exact with the spec:
//   (q | 0x4300) is bf16(128+q) exactly; (128+q)-(128+z) is exact; one rounding
//   in the multiply by s.
//
// Tile-packed W4 layout (shared with the wgmma prefill GEMM, which writes the
// same per-thread 16-element k runs as 16-byte swizzled smem chunks):
//   qweight[N/16][K/64][lane 0..31][word 0..3]  (uint32)
//   lane = 4*g + t owns rows n0+g and n0+g+8, k in [k0+16t, k0+16t+16).
//   word j holds k = k0+16t+4j+{0,1,2,3} for both rows; nibble positions
//     [0]=(g,s0) [4]=(g,s1) [1]=(g+8,s0) [5]=(g+8,s1)
//     [2]=(g,s2) [6]=(g,s3) [3]=(g+8,s2) [7]=(g+8,s3)
//   so (w >> 4i) & 0x000f000f yields the bf16x2 mma A-fragment register a_i.
// The mma k index is a permutation of physical k (dot products do not care);
// the x fragment is gathered with the same permutation.
#include <cstdlib>

#include "common.cuh"

namespace xb {

constexpr int kWarps = 8;

// m16n8k16 with a zero accumulator input (opens a fresh accumulation chain without clearing registers)
__device__ __forceinline__ void mma_bf16_16816_zero(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                    uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 "
      "{%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
      : "=f"(c[0]), "=f"(c[1]), "=f"(c[2]), "=f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "f"(0.f));
}

// x fragment for one k64 tile (4 k16 steps) and one n8 token tile:
// lane (g,t) needs x[tok = tile*8+g][k0 + 16t .. +16) = 32 bytes.
struct XFrag {
  uint4 lo, hi;  // k 0..7, 8..15 of the lane's run
};
__device__ __forceinline__ XFrag load_x(const __nv_bfloat16* x, int64_t x_stride, int tok, int M, int k) {
  XFrag f;
  if (tok < M) {
    const uint4* p = reinterpret_cast<const uint4*>(x + (int64_t)tok * x_stride + k);
    f.lo = p[0];
    f.hi = p[1];
  } else {
    f.lo = make_uint4(0, 0, 0, 0);
    f.hi = make_uint4(0, 0, 0, 0);
  }
  return f;
}

// ---------------------------------------------------------------------------
// W4A16.  Work unit = (16-row tile, k split).  A warp owns one unit and streams its k range with a
// register ring of kDepth slots (one slot = kTG k64 tiles = kTG 16-byte loads + the group's scale/zero
// words) that is refilled as it is consumed: the HBM pipe never drains between tiles.  kSplit warps of a
// CTA share a row tile and reduce through shared memory; with kSplit == 1 (wide N, e.g. gate_up) a warp
// owns its rows outright and writes them directly.  The inner loop runs several lane-ops per HBM byte, so it is
// instruction-bound next to HBM: addresses are running pointers, the group index is a shift, and the
// per-weight work is exactly LOP3(+SHF) / HSUB2 / HMUL2 per bf16 PAIR plus one HMMA per 8 weights.
// ---------------------------------------------------------------------------
template <int kMT>
struct XRing {
  uint4 lo[kMT], hi[kMT];
};

// Work the decode step does right before / after a weight-only linear, folded into the GEMV launch
// (north-star: "RMSNorm+RoPE as a single fused epilogue"; SURVEY call stack B, qwen2_decoder_layer.cpp:89-112):
//   prologue (kXs): x := RMSNorm(x (+ residual)) * norm_w - fused_add_rms_norm / rms_norm (norm.cu:43-136), computed
//       by EVERY CTA into its shared memory (the activation row is K*2 bytes: recomputing it is cheaper than a
//       launch); CTA 0 also writes the updated residual stream to res_out (a different buffer than res_in: other
//       CTAs still read res_in).  With norm_w == nullptr x is only staged in shared memory.
//   epilogue 1: act(gate) * up on interleaved gate/up rows (activation.cu:45-130)
//   epilogue 2: qkv_proj -> bias, RoPE on q and k (rope.cu:27-137, NeoX halves), KV scatter of the rotated k and of v
//       into the paged cache (reshape_paged_cache.cu:23-62).  Rows of every head are packed so that dims d and
//       d + head_dim/2 are rows g and g+8 of one 16-row tile (quant.pack_w4_qkv_rope): a thread that owns an output
//       pair owns a whole rotary pair.
struct W4Fuse {
  const __nv_bfloat16* norm_w;
  const __nv_bfloat16* res_in;
  __nv_bfloat16* res_out;
  float eps;
  // split RMSNorm: the PRODUCER linear (epilogue 3: o_proj / down_proj) adds the residual, writes the updated residual
  // stream r = bf16(bf16(y) + residual) to res_out and the per-(16-row tile, token) sums of r^2 to stats_out
  // [N/16][8]; the CONSUMER linear (stats_in != null: qkv / gate_up) reads r as its x, sums the K/16 partials in a
  // fixed order and normalises x once it is staged in shared memory - no reduction over K in any CTA.
  const float* stats_in;
  float* stats_out;
  QkvRopeCache rope;   // epilogue 2
};

template <int kMT /* n8 token tiles: M <= 8*kMT */, int kSplit /* 1,2,4,8 warps per row tile */, int kDepth,
          int kTG /* k64 tiles per ring slot: 2 when group_size >= 128, else 1 */, int kOcc = 2 /* CTAs per SM */,
          int kEpi = 0 /* 0: bias; 1: gate/up rows interleaved, act(gate)*up; 2: rope + KV scatter (qkv);
                          3: + residual -> residual stream and sum-of-squares partials (producer of a split RMSNorm) */,
          bool kXs = false /* x staged (and optionally normalised) in shared memory by the prologue */,
          bool kExact = false /* exact-dequant form: integer nibbles on the tensor core, scale / zero once per group */>
__global__ void __launch_bounds__(kWarps * 32, kMT >= 8 ? 1 : kOcc)
linear_w4a16_small_m_kernel(__nv_bfloat16* __restrict__ y, int64_t y_stride, const __nv_bfloat16* __restrict__ x,
                            int64_t x_stride, const uint4* __restrict__ qweight, const uint32_t* __restrict__ meta,
                            const __nv_bfloat16* __restrict__ bias, int M, int N, int K, int gshift /* log2(tiles per group) */,
                            int act_mode, const W4Fuse fz) {
  constexpr bool kGateUp = kEpi == 1;
  constexpr bool kPair = kEpi == 1 || kEpi == 2;    // rows g / g+8 of a tile form an output pair
  // kExact ("exact" form of the spec, oracle/quant.py): y = sum_g s_g * ( sum_{k in g} x_k (128 + q_k) - (128 + z_g) X_g ),
  // X_g = sum_{k in g} x_k.  The nibbles go to the tensor core as the exact bf16 integers 128 + q (LOP3 only: no HSUB2 /
  // HMUL2 per weight pair), X_g is formed ONCE per CTA while x is staged in shared memory (it is the same for every
  // row), and scale / zero are applied in fp32 once per (row, group): ~50 instead of 83 warp instructions per 512-byte
  // tile.  Serves one token tile with a ring slot = one quantisation group (group_size 64 / 128).
  static_assert(!kExact || (kMT == 1 && kXs), "the exact-dequant form stages x (and the group sums) in shared memory");
  static_assert(kEpi != 3 || (kSplit > 1 && kMT == 1), "the residual + statistics epilogue lives in the k-split reduction");
  constexpr int kTilesPerCta = kWarps / kSplit;
  __shared__ float red[kSplit > 1 ? kWarps : 1][kMT][16 * 8];
  __shared__ float s_ss[kXs ? kWarps : 1][8];
  __shared__ float s_sq[kEpi == 3 ? kTilesPerCta : 1][16][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int ntiles = N >> 4;
  const int ntile = blockIdx.x * kTilesPerCta + warp / kSplit;
  const int split = warp % kSplit;
  const bool live = ntile < ntiles;
  const int n0 = ntile * 16;
  const int ktiles = K >> 6;
  const int nslots = ktiles / kTG;
  const int per = (nslots + kSplit - 1) / kSplit;
  const int s_begin = split * per;
  const int s_end = live ? min(nslots, s_begin + per) : s_begin;

  // kAcc independent accumulator sets (one per k16 step of a tile when registers allow): legacy HMMA has a long
  // issue-to-result latency, a single chain per warp leaves the scheduler with nothing eligible
  constexpr int kAcc = kMT == 1 ? 4 : (kMT == 2 ? 2 : 1);
  float accj[kAcc][kMT][4];
#pragma unroll
  for (int a = 0; a < kAcc; ++a)
#pragma unroll
    for (int m = 0; m < kMT; ++m)
#pragma unroll
      for (int i = 0; i < 4; ++i) accj[a][m][i] = 0.f;

  // running pointers (one 64-bit add per slot instead of a multiply per tile)
  const uint4* wp = qweight + ((int64_t)ntile * ktiles + (int64_t)s_begin * kTG) * 32 + lane;
  const uint32_t* mbase = meta + n0 + g;

  // ---- staging ring: per-lane PRIVATE shared-memory slots filled with cp.async ------------------------------
  // Every lane copies exactly the 16 bytes (and the two scale/zero words) it will consume itself and reads them
  // back with LDS: no cross-lane hand-off, so no barrier - only the in-order commit-group wait.  (A register ring
  // of LDGs looks equivalent but is not: ptxas tracks all in-flight LDGs of the loop on one scoreboard, so waiting
  // for the oldest slot waits for the refill issued a moment ago and the HBM latency is exposed on every slot.)
  extern __shared__ __align__(16) uint8_t ring_smem[];
  constexpr int kSlotBytes = kTG * 512 + 256;          // kTG k64 tiles (32 lanes x 16 B) + 32 lanes x 2 meta words
  const uint32_t ring_w = smem_addr_u32(ring_smem) + warp * (kDepth * kSlotBytes) + lane * 16;
  const uint32_t ring_m = smem_addr_u32(ring_smem) + warp * (kDepth * kSlotBytes) + kTG * 512 + lane * 8;
  auto issue = [&](int i, const uint4* wsrc, const uint32_t* msrc) {
#pragma unroll
    for (int u = 0; u < kTG; ++u) cp_async_16(ring_w + i * kSlotBytes + u * 512, wsrc + u * 32);
    cp_async_4(ring_m + i * kSlotBytes, msrc);
    cp_async_4(ring_m + i * kSlotBytes + 4, msrc + 8);
  };

  // ---- prologue: fill the ring (weights + scale/zero words do not depend on the producer kernel) ----
#pragma unroll
  for (int i = 0; i < kDepth; ++i) {
    if (s_begin + i < s_end) issue(i, wp + i * kTG * 32, mbase + (int64_t)(((s_begin + i) * kTG) >> gshift) * N);
    cp_async_commit();     // one group per slot, empty or not: group n <-> slot n of this warp
  }
  wp += kDepth * kTG * 32;   // next slot to prefetch
  pdl_wait();  // x (and bias) come from the producer kernel

  // ---- x: either staged (+ normalised) in shared memory by all threads of the CTA, or read through L1 per tile ----
  // shared layout: [M rows][K + 8] bf16 (the 16-byte pad spreads the rows of a token tile over the banks), 128 bytes
  // of slack after the last row: the one-tile-ahead fragment prefetch may read past a warp's k range
  const int xs_stride = K + 8;
  __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(ring_smem + kWarps * kDepth * kSlotBytes);
  // kExact: X_g per (group, token) as [K / group][8] fp32 behind the x stage (16-byte aligned: rows are K + 8 bf16)
  float* gsum = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(xs) + (((size_t)M * (K + 8) * 2 + 256 + 15) & ~size_t(15)));
  if constexpr (kXs) {
    const int nvec = K >> 3;
    const bool do_norm = fz.norm_w != nullptr;
    // split RMSNorm consumer: x IS the residual stream and sum(x^2) per token arrives as K/16 partials
    const bool split_norm = fz.stats_in != nullptr;
    for (int tok = 0; tok < M; ++tok) {
      const uint4* src = reinterpret_cast<const uint4*>(x + (int64_t)tok * x_stride);
      // (under epilogue 3 the residual pointers belong to the EPILOGUE - the [M, N] residual stream - not to x)
      const uint4* rsrc = (kEpi != 3 && fz.res_in) ? reinterpret_cast<const uint4*>(fz.res_in + (int64_t)tok * K) : nullptr;
      uint4* rdst = (kEpi != 3 && fz.res_out && blockIdx.x == 0) ? reinterpret_cast<uint4*>(fz.res_out + (int64_t)tok * K) : nullptr;
      uint4* dst = reinterpret_cast<uint4*>(xs + (int64_t)tok * xs_stride);
      float ss = 0.f;
      if constexpr (kExact) {
        // stage x and form the group sums X_g: a group is kTG * 8 consecutive 16-byte vectors = consecutive lanes
        constexpr int kVecPerGroup = kTG * 8;
        for (int base = 0; base < nvec; base += kWarps * 32) {     // warp-uniform trip count (full-warp shuffles)
          const int idx = base + threadIdx.x;
          float part = 0.f;
          if (idx < nvec) {
            const uint4 v = src[idx];
            const uint32_t* vp = &v.x;
#pragma unroll
            for (int j = 0; j < 4; ++j) part += bf16lo(vp[j]) + bf16hi(vp[j]);
            dst[idx] = v;
          }
#pragma unroll
          for (int o = kVecPerGroup / 2; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
          if (idx < nvec && (lane & (kVecPerGroup - 1)) == 0) gsum[(idx / kVecPerGroup) * 8 + tok] = part;
        }
        continue;
      }
      for (int idx = threadIdx.x; idx < nvec; idx += kWarps * 32) {
        uint4 v = src[idx];
        if (rsrc) v = add_bf16x8(v, rsrc[idx]);
        if (rdst) rdst[idx] = v;
        ss = sumsq_bf16x8(ss, v);
        dst[idx] = v;
      }
      if (do_norm && !split_norm) {
        ss = warp_sum(ss);
        if (lane == 0) s_ss[warp][tok] = ss;
      }
    }
    if (split_norm) {
      float part[8];
#pragma unroll
      for (int tk = 0; tk < 8; ++tk) part[tk] = 0.f;
      for (int i = threadIdx.x; i < (K >> 4); i += kWarps * 32) {      // fixed assignment -> every CTA gets the same bits
        const float4 a = __ldcg(reinterpret_cast<const float4*>(fz.stats_in + (int64_t)i * 8));
        const float4 b = __ldcg(reinterpret_cast<const float4*>(fz.stats_in + (int64_t)i * 8 + 4));
        part[0] += a.x; part[1] += a.y; part[2] += a.z; part[3] += a.w;
        part[4] += b.x; part[5] += b.y; part[6] += b.z; part[7] += b.w;
      }
#pragma unroll
      for (int tk = 0; tk < 8; ++tk) {
        const float v = warp_sum(part[tk]);
        if (lane == 0) s_ss[warp][tk] = v;
      }
    }
    if (do_norm) {
      __syncthreads();
      const uint4* wv = reinterpret_cast<const uint4*>(fz.norm_w);
      for (int tok = 0; tok < M; ++tok) {
        float var = 0.f;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) var += s_ss[w][tok];       // fixed order: every CTA gets the same rstd
        const float rstd = rms_rstd(var, K, fz.eps);
        uint4* dst = reinterpret_cast<uint4*>(xs + (int64_t)tok * xs_stride);
        for (int idx = threadIdx.x; idx < nvec; idx += kWarps * 32)   // same elements this thread staged above
          dst[idx] = rms_apply_bf16x8(dst[idx], __ldg(wv + idx), rstd);
      }
    }
    __syncthreads();
  }

  // x fragments: lane (g,t) needs x[tok = 8m+g][k0 + 16t .. +16) per tile
  // token columns past M read the last valid token instead of zeros: their accumulator columns are
  // finite garbage that is never stored, and the loads need neither a predicate nor a zero fill
  const __nv_bfloat16* xp[kMT];
  uint32_t xsa[kMT];
#pragma unroll
  for (int m = 0; m < kMT; ++m) {
    const int tok = min(m * 8 + g, M - 1);
    xp[m] = x + (int64_t)tok * x_stride + (int64_t)s_begin * kTG * 64 + 16 * t;
    xsa[m] = smem_addr_u32(xs) + (uint32_t)((tok * xs_stride + s_begin * kTG * 64 + 16 * t) * 2);
  }
  auto load_xtile = [&](XRing<kMT>& d) {
#pragma unroll
    for (int m = 0; m < kMT; ++m) {
      if constexpr (kXs) {
        d.lo[m] = lds_128(xsa[m]);
        d.hi[m] = lds_128(xsa[m] + 16);
        xsa[m] += 128;
      } else {
        d.lo[m] = *reinterpret_cast<const uint4*>(xp[m]);   // L1 hits, hidden by the other warps
        d.hi[m] = *reinterpret_cast<const uint4*>(xp[m] + 8);
        xp[m] += 64;
      }
    }
  };
  // kXs: fragments are prefetched ONE TILE AHEAD into the other half of a two-deep register buffer (shared-memory
  // loads return in order and in tens of cycles, so the prefetch never exposes more than that)
  XRing<kMT> xbuf[2];
  if constexpr (kXs) load_xtile(xbuf[0]);

  auto consume = [&](int i) {
    uint4 wq[kTG];
#pragma unroll
    for (int u = 0; u < kTG; ++u) wq[u] = lds_128(ring_w + i * kSlotBytes + u * 512);
    const uint2 mt = lds_64(ring_m + i * kSlotBytes);
    uint32_t s0, z0, s1, z1;
    w4_meta(mt.x, s0, z0);
    w4_meta(mt.y, s1, z1);
#pragma unroll
    for (int u = 0; u < kTG; ++u) {
      const int par = (i * kTG + u) & 1;       // compile-time after unrolling (kDepth * kTG is even)
      if constexpr (kXs) load_xtile(xbuf[par ^ 1]);
      else load_xtile(xbuf[0]);
      const XRing<kMT>& xf = kXs ? xbuf[par] : xbuf[0];
      const uint32_t* wv = &wq[u].x;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint32_t a[4];
        w4_dequant_word(wv[j], z0, s0, z1, s1, a);
#pragma unroll
        for (int m = 0; m < kMT; ++m) {
          // lane run element 4j+{0,1} -> b0, 4j+{2,3} -> b1
          const uint32_t* xv = j < 2 ? &xf.lo[m].x : &xf.hi[m].x;
          mma_bf16_16816(accj[j % kAcc][m], a[0], a[1], a[2], a[3], xv[(j & 1) * 2], xv[(j & 1) * 2 + 1]);
        }
      }
    }
  };

  // kExact: one ring slot = one quantisation group.  Two accumulation chains per group (opened with a zero-C MMA), then
  // yacc += s * (c - (128 + z) * X_g) in fp32; rows g / g+8 use meta words x / y, token columns 2t / 2t+1 use X_g[2t..].
  float yacc[4] = {0.f, 0.f, 0.f, 0.f};
  const uint32_t gsum_a = smem_addr_u32(gsum) + t * 8;
  auto consume_exact = [&](int i, int slot_abs) {
    uint4 wq[kTG];
#pragma unroll
    for (int u = 0; u < kTG; ++u) wq[u] = lds_128(ring_w + i * kSlotBytes + u * 512);
    const uint2 mt = lds_64(ring_m + i * kSlotBytes);
    float c0[4], c1[4];
#pragma unroll
    for (int u = 0; u < kTG; ++u) {
      const int par = (i * kTG + u) & 1;
      load_xtile(xbuf[par ^ 1]);
      const XRing<kMT>& xf = xbuf[par];
      const uint32_t* wv = &wq[u].x;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint32_t q[4];
        w4_nibbles(wv[j], q);
        const uint32_t* xv = j < 2 ? &xf.lo[0].x : &xf.hi[0].x;
        const uint32_t b0 = xv[(j & 1) * 2], b1 = xv[(j & 1) * 2 + 1];
        if (u == 0 && j == 0) mma_bf16_16816_zero(c0, q[0], q[1], q[2], q[3], b0, b1);
        else if (u == 0 && j == 1) mma_bf16_16816_zero(c1, q[0], q[1], q[2], q[3], b0, b1);
        else if (j & 1) mma_bf16_16816(c1, q[0], q[1], q[2], q[3], b0, b1);
        else mma_bf16_16816(c0, q[0], q[1], q[2], q[3], b0, b1);
      }
    }
    const uint2 sxb = lds_64(gsum_a + (uint32_t)slot_abs * 32u);
    const float sx0 = __uint_as_float(sxb.x), sx1 = __uint_as_float(sxb.y);
    const float s0 = bf16lo(mt.x), nz0 = -bf16hi(mt.x), s1 = bf16lo(mt.y), nz1 = -bf16hi(mt.y);   // scale, -(128 + zero)
    yacc[0] = fmaf(s0, fmaf(nz0, sx0, c0[0] + c1[0]), yacc[0]);
    yacc[1] = fmaf(s0, fmaf(nz0, sx1, c0[1] + c1[1]), yacc[1]);
    yacc[2] = fmaf(s1, fmaf(nz1, sx0, c0[2] + c1[2]), yacc[2]);
    yacc[3] = fmaf(s1, fmaf(nz1, sx1, c0[3] + c1[3]), yacc[3]);
  };

  // Meta words: when a ring slot is exactly one quantisation group (group 128 with kTG 2, group 64 with kTG 1) the
  // row pointer just advances by N per slot; otherwise it is recomputed from the slot index.
  const bool slot_is_group = (1 << gshift) == kTG;
  const uint32_t* mp = mbase + (int64_t)(((s_begin + kDepth) * kTG) >> gshift) * N;   // next slot to prefetch

  int sl = s_begin;
  // full rounds: every ring slot is consumed, then (while data remains) refilled kDepth slots ahead.  The LDS of a
  // slot have returned before the HMMAs that use them issue, so the refill that follows cannot overtake them.
  for (; sl + kDepth <= s_end; sl += kDepth) {
#pragma unroll
    for (int i = 0; i < kDepth; ++i) {
      cp_async_wait<kDepth - 1>();
      if constexpr (kExact) consume_exact(i, sl + i);
      else consume(i);
      if (sl + i + kDepth < s_end)
        issue(i, wp, slot_is_group ? mp : mbase + (int64_t)(((sl + i + kDepth) * kTG) >> gshift) * N);
      cp_async_commit();
      wp += kTG * 32;
      mp += N;
    }
  }
  // tail: fewer than kDepth slots left, all already in flight
  cp_async_wait<0>();
#pragma unroll
  for (int i = 0; i < kDepth; ++i) {
    if (sl + i < s_end) {
      if constexpr (kExact) consume_exact(i, sl + i);
      else consume(i);
    }
  }
  pdl_launch_dependents();
  float acc[kMT][4];
#pragma unroll
  for (int m = 0; m < kMT; ++m)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float v = accj[0][m][i];
#pragma unroll
      for (int a = 1; a < kAcc; ++a) v += accj[a][m][i];
      acc[m][i] = kExact ? yacc[i] : v;
    }

  // c0:(row g, tok 2t) c1:(g, 2t+1) c2:(g+8, 2t) c3:(g+8, 2t+1)
  // kGateUp: row g of the tile is gate row 8*ntile+g and row g+8 the matching up row, so SiLU*mul (activation.cu:45-130:
  // both linear outputs rounded to bf16, bf16(act(gate)) * up rounded again) is applied right here and only
  // N/2 values per token are written - the separate act_and_mul launch and its 3*N bytes of traffic disappear.
  auto gate_up = [&](float gate, float up) -> __nv_bfloat16 {
    const float gr = round_bf16(gate), ur = round_bf16(up);
    return __float2bfloat16_rn(round_bf16(act_fn(act_mode, gr)) * ur);
  };
  if constexpr (kSplit == 1) {
    if (live) {
#pragma unroll
      for (int m = 0; m < kMT; ++m) {
        if constexpr (kPair) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int tok = m * 8 + 2 * t + e;
            if (tok < M) {
              float gv = acc[m][e], uv = acc[m][2 + e];
              if (bias) { gv += __bfloat162float(bias[n0 + g]); uv += __bfloat162float(bias[n0 + g + 8]); }
              if constexpr (kGateUp) y[(int64_t)tok * y_stride + ntile * 8 + g] = gate_up(gv, uv);
              else qkv_rope_store(fz.rope, y, y_stride, tok, ntile, g, gv, uv);
            }
          }
        } else {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int tok = m * 8 + 2 * t + (i & 1), r = g + (i >> 1) * 8;
            if (tok < M) {
              float v = acc[m][i];
              if (bias) v += __bfloat162float(bias[n0 + r]);
              y[(int64_t)tok * y_stride + n0 + r] = __float2bfloat16_rn(v);
            }
          }
        }
      }
    }
    return;
  } else {
#pragma unroll
    for (int m = 0; m < kMT; ++m) store_c_frag(red[warp][m], acc[m], g, t);
    __syncthreads();
    for (int i = threadIdx.x; i < kTilesPerCta * kMT * 128; i += blockDim.x) {
      const int tl = i / (kMT * 128), rem = i % (kMT * 128);
      const int m = rem >> 7, r = (rem & 127) >> 3, c = rem & 7;
      const int tok = m * 8 + c;
      const int nt = blockIdx.x * kTilesPerCta + tl;
      if (tok < M && nt < ntiles) {
        float sum = 0.f;
#pragma unroll
        for (int w = 0; w < kSplit; ++w) sum += red[tl * kSplit + w][m][r * 8 + c];
        if (bias) sum += __bfloat162float(bias[nt * 16 + r]);
        if constexpr (kPair) {
          if (r < 8) {
            float up = 0.f;
#pragma unroll
            for (int w = 0; w < kSplit; ++w) up += red[tl * kSplit + w][m][(r + 8) * 8 + c];
            if (bias) up += __bfloat162float(bias[nt * 16 + r + 8]);
            if constexpr (kGateUp) y[(int64_t)tok * y_stride + nt * 8 + r] = gate_up(sum, up);
            else qkv_rope_store(fz.rope, y, y_stride, tok, nt, r, sum, up);
          }
        } else if constexpr (kEpi == 3) {
          // producer half of the split RMSNorm (fused_add_rms_norm, norm.cu:80-136): r = bf16(bf16(y) + residual)
          const int n = nt * 16 + r;
          const float rr = add_bf16(round_bf16(sum), __bfloat162float(fz.res_in[(int64_t)tok * N + n]));
          fz.res_out[(int64_t)tok * N + n] = __float2bfloat16_rn(rr);
          s_sq[tl][r][c] = rr * rr;
        } else {
          y[(int64_t)tok * y_stride + nt * 16 + r] = __float2bfloat16_rn(sum);
        }
      } else if constexpr (kEpi == 3) {
        if (tl < kTilesPerCta) s_sq[tl][r][c] = 0.f;
      }
    }
    if constexpr (kEpi == 3) {
      __syncthreads();
      // per (row tile, token): the 16 squares in row order - fixed order, no atomics: bit-reproducible statistics
      for (int i = threadIdx.x; i < kTilesPerCta * 8; i += blockDim.x) {
        const int tl = i >> 3, c = i & 7;
        const int nt = blockIdx.x * kTilesPerCta + tl;
        if (nt < ntiles) {
          float ssum = 0.f;
#pragma unroll
          for (int r = 0; r < 16; ++r) ssum += s_sq[tl][r][c];
          fz.stats_out[(int64_t)nt * 8 + c] = ssum;
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------
// bf16 weights [N,K] row-major (the reference layout, untouched).
// lane (g,t) reads rows n0+g and n0+g+8, 16 bytes each per k32 tile:
// k in [k0+8t, k0+8t+8) -> two k16 steps (elements 0..3 -> step 0, 4..7 -> 1).
// Warp w owns the k32 tiles w, w + 8, w + 16, ... and streams them through a per-lane private cp.async ring of
// kBf16Ring slots in shared memory (the W4 kernel's scheme): the ring is refilled as it is consumed, so the weight
// stream stays full until the warp's last tile.
// ---------------------------------------------------------------------------
constexpr int kBf16Ring = 8;
template <int kMT>
__global__ void __launch_bounds__(kWarps * 32)
linear_bf16_small_m_kernel(__nv_bfloat16* __restrict__ y, int64_t y_stride, const __nv_bfloat16* __restrict__ x,
                           int64_t x_stride, const __nv_bfloat16* __restrict__ w,
                           const __nv_bfloat16* __restrict__ bias, int M, int N, int K) {
  __shared__ float red[kWarps][kMT][16 * 8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int n0 = blockIdx.x * 16;
  const int ktiles = K >> 5;  // k32 tiles
  const int nt = ktiles > warp ? (ktiles - warp + kWarps - 1) / kWarps : 0;   // tiles of this warp
  // rows past N read row N - 1: a row of the mma's A operand only reaches its own output row, which is not stored
  const __nv_bfloat16* w0 = w + (int64_t)min(n0 + g, N - 1) * K + 8 * t + (warp << 5);
  const __nv_bfloat16* w1 = w + (int64_t)min(n0 + g + 8, N - 1) * K + 8 * t + (warp << 5);

  float acc[kMT][4];
#pragma unroll
  for (int m = 0; m < kMT; ++m)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[m][i] = 0.f;

  // slot = [row g chunks of the 32 lanes | row g+8 chunks]: 1 KB per warp and slot
  extern __shared__ __align__(16) uint8_t ring_smem[];
  const uint32_t ring = smem_addr_u32(ring_smem) + warp * (kBf16Ring * 1024) + lane * 16;
  auto issue = [&](int j) {
    const uint32_t dst = ring + (j & (kBf16Ring - 1)) * 1024;
    cp_async_16(dst, w0 + (int64_t)j * (kWarps << 5));
    cp_async_16(dst + 512, w1 + (int64_t)j * (kWarps << 5));
  };
#pragma unroll
  for (int j = 0; j < kBf16Ring; ++j) {
    if (j < nt) issue(j);
    cp_async_commit();     // one group per slot, empty or not
  }
  pdl_wait();  // x (and bias) come from the producer kernel
  const __nv_bfloat16* xp[kMT];
#pragma unroll
  for (int m = 0; m < kMT; ++m) xp[m] = x + (int64_t)min(m * 8 + g, M - 1) * x_stride + 8 * t + (warp << 5);
#pragma unroll 1
  for (int j = 0; j < nt; ++j) {
    cp_async_wait<kBf16Ring - 1>();
    const uint32_t src = ring + (j & (kBf16Ring - 1)) * 1024;
    const uint4 wa = lds_128(src), wb = lds_128(src + 512);
#pragma unroll
    for (int m = 0; m < kMT; ++m) {
      uint4 xv = *reinterpret_cast<const uint4*>(xp[m] + (int64_t)j * (kWarps << 5));
      if (m * 8 + g >= M) xv = make_uint4(0, 0, 0, 0);
      mma_bf16_16816(acc[m], wa.x, wb.x, wa.y, wb.y, xv.x, xv.y);
      mma_bf16_16816(acc[m], wa.z, wb.z, wa.w, wb.w, xv.z, xv.w);
    }
    // the LDS of this slot have returned before the HMMAs that use them issue: the refill cannot overtake them
    if (j + kBf16Ring < nt) issue(j + kBf16Ring);
    cp_async_commit();
  }
  pdl_launch_dependents();

#pragma unroll
  for (int m = 0; m < kMT; ++m) store_c_frag(red[warp][m], acc[m], g, t);
  __syncthreads();
  for (int i = threadIdx.x; i < kMT * 128; i += blockDim.x) {
    const int m = i >> 7, r = (i & 127) >> 3, c = i & 7;
    const int tok = m * 8 + c;
    if (tok < M && n0 + r < N) {
      float s = 0.f;
#pragma unroll
      for (int ww = 0; ww < kWarps; ++ww) s += red[ww][m][r * 8 + c];
      if (bias) s += __bfloat162float(bias[n0 + r]);
      y[(int64_t)tok * y_stride + n0 + r] = __float2bfloat16_rn(s);
    }
  }
}

}  // namespace xb

using namespace xb;

// dynamic shared memory of the W4 kernel: kWarps private rings of `depth` slots (kTG tiles + meta words each)
static constexpr size_t w4_ring_bytes(int depth, int tg) { return (size_t)kWarps * depth * (tg * 512 + 256); }
// largest activation block ([M][K + 8] bf16 + slack) the kXs variants stage in shared memory next to the ring
static constexpr size_t kXsMaxBytes = 72 * 1024;
static inline size_t w4_xs_bytes(int M, int K) { return (size_t)M * (K + 8) * 2 + 256; }
// exact-dequant form: the group sums X_g [K / group][8] fp32 live behind the x stage
static inline size_t w4_gsum_bytes(int K, int group_size) { return (size_t)(K / group_size) * 32 + 16; }
// 0: bf16-weight form (w = bf16((q - z) s), the prefill GEMM's form); 1: exact-dequant form for M <= 8, group 64 / 128
static std::atomic<int> g_w4_decode_form{-1};
static int w4_decode_form() {
  int f = g_w4_decode_form.load(std::memory_order_relaxed);
  if (f < 0) {
    const char* e = getenv("XB_W4_EXACT");
    f = e ? atoi(e) : 0;
    if (f < 0 || f > 1) f = 0;
    g_w4_decode_form.store(f, std::memory_order_relaxed);
  }
  return f;
}
extern "C" int xb_set_w4_decode_form(int form) {
  if (form < 0 || form > 1) {
    set_error("set_w4_decode_form: form %d (0 bf16-weight | 1 exact-dequant)", form);
    return -1;
  }
  const int old = w4_decode_form();
  g_w4_decode_form.store(form, std::memory_order_relaxed);
  return old;
}

// ring depth: 8 k64 tiles (4 KB) per warp in flight = 64 KB per SM at 2 CTAs/SM, ~1.5x the HBM latency-bandwidth
// product; the ring lives in shared memory, so the depth no longer competes with the accumulators for registers
// (a 12-tile ring measured the same as 8 tiles on every decode shape)
static constexpr int kW4RingTiles = 8;

// The kernel arguments of one W4 launch and the runtime choices of w4_small_m_impl that select its instantiation.
struct W4Launch {
  __nv_bfloat16* y;
  int64_t y_stride;
  const __nv_bfloat16* x;
  int64_t x_stride;
  const uint4* qw;
  const uint32_t* meta;
  const __nv_bfloat16* bias;
  int M, N, K, gshift, act_mode;
  W4Fuse fz;
  cudaStream_t stream;
  size_t xs_bytes;
  int split, epi;
  bool tg2, xs, exact;
};

// What padding the shared memory of a W4 launch needs: the CTAs of `kern` an SM holds at `smem` bytes of dynamic shared
// memory, the kernel's static shared memory and the device's per-SM / per-CTA-reserved shared memory.  Also lets the
// kernel take up to half an SM's shared memory dynamically.
struct W4Residency {
  cudaError_t err;
  int resident, static_smem, smem_per_sm, reserved_per_cta;
};
template <typename K>
static W4Residency w4_residency(K kern, int smem) {
  W4Residency r{cudaSuccess, 0, 0, 0, 0};
  cudaFuncAttributes fa{};
  int dev = 0;
  if ((r.err = cudaGetDevice(&dev)) != cudaSuccess ||
      (r.err = cudaDeviceGetAttribute(&r.smem_per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev)) != cudaSuccess ||
      (r.err = cudaDeviceGetAttribute(&r.reserved_per_cta, cudaDevAttrReservedSharedMemoryPerBlock, dev)) != cudaSuccess ||
      (r.err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, r.smem_per_sm / 2)) != cudaSuccess ||
      (r.err = cudaFuncGetAttributes(&fa, kern)) != cudaSuccess ||
      (r.err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&r.resident, kern, kWarps * 32, smem)) != cudaSuccess)
    return r;
  r.static_smem = (int)fa.sharedSizeBytes;
  return r;
}

template <int kMT, int kSplit, int kTG, int kEpi, bool kXs, bool kExact>
static int w4_launch(const W4Launch& l) {
  constexpr int kDepth = kW4RingTiles / kTG;
  constexpr auto kern = linear_w4a16_small_m_kernel<kMT, kSplit, kDepth, kTG, 2, kEpi, kXs, kExact>;
  const dim3 grid((l.N / 16 + kWarps / kSplit - 1) / (kWarps / kSplit)), block(kWarps * 32);
  size_t smem = w4_ring_bytes(kDepth, kTG) + l.xs_bytes;
  if constexpr (kXs) {
    // static reduction scratch + ring + x stage may exceed the default 48 KB
    XB_CUDA_OK(set_max_dynamic_smem_once<kern>((int)(w4_ring_bytes(kDepth, kTG) + kXsMaxBytes)));
  } else {
    // The block scheduler does not spread a one-wave grid evenly when SMs have room for more CTAs than the even share:
    // o_proj / down_proj of Qwen2-7B (224 CTAs on 132 SMs that hold 3 each) stream like SMs holding 3 CTAs.  Padding
    // the shared memory so that an SM holds at most ceil(grid / SMs) CTAs took down_proj from 18.0 to 15.9 us (H100).
    // The carveout preference is left to the driver: forcing the maximum shared carveout as well measured 445 instead
    // of 459 decode tokens/s.
    static const W4Residency res = w4_residency(kern, (int)smem);
    XB_CUDA_OK(res.err);
    const int per_sm = ((int)grid.x + device_sm_count() - 1) / device_sm_count();
    if (per_sm < res.resident)
      smem = std::max(smem, (size_t)(res.smem_per_sm / (per_sm + 1) + 128 - res.reserved_per_cta - res.static_smem));
  }
  XB_CUDA_OK(launch(kern, grid, block, smem, l.stream, true, l.y, l.y_stride, l.x,
                    l.x_stride, l.qw, l.meta, l.bias, l.M, l.N, l.K, l.gshift, l.act_mode, l.fz));
  return 0;
}

// Runtime choices -> template arguments, instantiating only the supported variants: the staged-x, exact-dequant, rope
// and residual forms serve one token tile (M <= 8), and the residual epilogue (3) lives in the k-split reduction.
template <int kMT, int kSplit, int kEpi, bool kXs, bool kExact>
static int w4_pick_tg(const W4Launch& l) {
  return l.tg2 ? w4_launch<kMT, kSplit, 2, kEpi, kXs, kExact>(l) : w4_launch<kMT, kSplit, 1, kEpi, kXs, kExact>(l);
}
template <int kMT, int kSplit, bool kXs, bool kExact>
static int w4_pick_epi(const W4Launch& l) {
  if constexpr (kMT == 1) {
    if (l.epi == 3) {
      if constexpr (kSplit > 1) return w4_pick_tg<1, kSplit, 3, kXs, kExact>(l);
      return 0;   // not reached: w4_small_m_impl gives epilogue 3 a split of at least 2
    }
    if (l.epi == 2) return w4_pick_tg<1, kSplit, 2, kXs, kExact>(l);
  }
  return l.epi == 1 ? w4_pick_tg<kMT, kSplit, 1, kXs, kExact>(l) : w4_pick_tg<kMT, kSplit, 0, kXs, kExact>(l);
}
template <int kMT, int kSplit>
static int w4_pick_form(const W4Launch& l) {
  if constexpr (kMT == 1) {
    if (l.exact) return w4_pick_epi<1, kSplit, true, true>(l);
    if (l.xs) return w4_pick_epi<1, kSplit, true, false>(l);
  }
  return w4_pick_epi<kMT, kSplit, false, false>(l);
}
template <int kMT>
static int w4_pick_split(const W4Launch& l) {
  switch (l.split) {
    case 1: return w4_pick_form<kMT, 1>(l);
    case 2: return w4_pick_form<kMT, 2>(l);
    case 4: return w4_pick_form<kMT, 4>(l);
    default: return w4_pick_form<kMT, 8>(l);
  }
}

// epi: 0 plain (+bias), 1 gate/up + activation (act_mode), 2 qkv rope + KV scatter (fz).  xs: stage x in shared memory
// (required for the norm prologue).  fz may be null when neither the prologue nor epilogue 2 is used.
static int w4_small_m_impl(void* y, int64_t y_stride, const void* x, int64_t x_stride, const uint32_t* qweight,
                           const uint32_t* meta, const void* bias, int M, int N, int K, int group_size, int epi,
                           int act_mode, bool xs, const W4Fuse* fzp, xb_stream_t stream) {  // (xs is forced on by the exact form)
  if (M == 0) return 0;
  XB_CHECK(M > 0 && M <= 64, "linear_w4a16_small_m: M=%d out of range (1..64); use the wgmma GEMM", M);
  XB_CHECK(N % 16 == 0 && K % 64 == 0, "linear_w4a16_small_m: N=%d must be %%16, K=%d %%64", N, K);
  XB_CHECK(group_size >= 64 && group_size % 64 == 0 && K % group_size == 0,
           "linear_w4a16_small_m: group_size %d must be a multiple of 64 dividing K=%d", group_size, K);
  XB_CHECK(x_stride % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0, "linear_w4a16_small_m: x not 16B aligned");
  XB_CHECK(!(xs || epi >= 2) || M <= 8, "linear_w4a16_small_m: the fused prologue / epilogues serve M <= 8 (got %d)", M);
  XB_CHECK(!xs || w4_xs_bytes(M, K) <= kXsMaxBytes, "linear_w4a16_small_m: M=%d x K=%d does not fit the shared-memory x stage", M, K);
  W4Fuse fz{};
  if (fzp) fz = *fzp;
  // pick the k split so that (row tiles x splits) covers ~16 warps on each of the device's SMs
  const int ntiles = N / 16, ktiles = K / 64;
  int split = 1;
  while (split < 8 && ntiles * split < device_sm_count() * 16 && ktiles / (split * 2) >= 3) split *= 2;
  if (epi == 3 && split < 2) split = 2;   // the residual + statistics epilogue lives in the k-split reduction
  const int tpg = group_size / 64;   // k64 tiles per quantisation group
  XB_CHECK((tpg & (tpg - 1)) == 0, "linear_w4a16_small_m: group_size/64 must be a power of two (got %d)", group_size);
  int gshift = 0;
  while ((1 << gshift) < tpg) ++gshift;
  const bool tg2 = tpg >= 2;
  // exact-dequant form: one token tile, ring slot = one group, no norm prologue, x + group sums fit the shared-memory stage
  const bool exact = w4_decode_form() == 1 && M <= 8 && (tpg == 1 || tpg == 2) && fz.norm_w == nullptr &&
                     w4_xs_bytes(M, K) + w4_gsum_bytes(K, group_size) <= kXsMaxBytes;
  if (exact) xs = true;
  const size_t xs_bytes = (xs ? w4_xs_bytes(M, K) : 0) + (exact ? w4_gsum_bytes(K, group_size) : 0);
  XB_CHECK(!(epi == 1 && M > 16), "linear_w4a16_gate_up_act_small_m: M=%d > 16, use the GEMM + act_and_mul_interleaved8", M);
  const W4Launch l{reinterpret_cast<__nv_bfloat16*>(y), y_stride, reinterpret_cast<const __nv_bfloat16*>(x), x_stride,
                   reinterpret_cast<const uint4*>(qweight), meta, reinterpret_cast<const __nv_bfloat16*>(bias),
                   M, N, K, gshift, act_mode, fz, (cudaStream_t)stream, xs_bytes, split, epi, tg2, xs, exact};
  if (M <= 8) return w4_pick_split<1>(l);
  if (M <= 16) return w4_pick_split<2>(l);
  if (M <= 32) return w4_pick_split<4>(l);
  return w4_pick_split<8>(l);
}

extern "C" int xb_linear_w4a16_small_m(void* y, int64_t y_stride, const void* x, int64_t x_stride,
                                       const uint32_t* qweight, const uint32_t* meta, const void* bias, int M, int N,
                                       int K, int group_size, xb_stream_t stream) {
  return w4_small_m_impl(y, y_stride, x, x_stride, qweight, meta, bias, M, N, K, group_size, 0, -1, false, nullptr, stream);
}

// gate_up_proj with the activation fused into the epilogue.  qweight / meta / bias rows must be in the interleaved
// order produced by xllm_b200.quant.interleave_gate_up (per 16-row tile: 8 gate rows then the matching 8 up rows).
// y [M, N/2].  act_mode: 0 silu, 1 gelu, 2 gelu_tanh.
extern "C" int xb_linear_w4a16_gate_up_act_small_m(void* y, int64_t y_stride, const void* x, int64_t x_stride,
                                                   const uint32_t* qweight, const uint32_t* meta, const void* bias,
                                                   int M, int N, int K, int group_size, int act_mode, xb_stream_t stream) {
  XB_CHECK(act_mode >= 0 && act_mode <= 2, "gate_up_act: unsupported act mode %d", act_mode);
  return w4_small_m_impl(y, y_stride, x, x_stride, qweight, meta, bias, M, N, K, group_size, 1, act_mode, false, nullptr, stream);
}

// The decode-step form of a weight-only linear (M <= 8): optional add + RMSNorm prologue, optional epilogue.
//   prologue: norm_weight != null: x := RMSNorm(x (+ residual_in)) * norm_weight (fused_add_rms_norm / rms_norm); the
//             updated residual stream x + residual_in goes to residual_out (must not alias residual_in; null = not
//             wanted).  norm_weight == null with stage_x != 0 only stages x in shared memory.
//             Split form: norm_stats_in != null: x IS the residual stream and sum(x^2) per token arrives as K/16
//             partials [K/16][8] written by the producer linear's epilogue 3 - the consumer only normalises.
//   epilogue: 3 (o_proj / down_proj): r = bf16(bf16(y) + residual_in) -> residual_out, sum of r^2 per (16-row tile,
//             token) -> norm_stats_out [N/16][8]; y is not written.
//   epilogue: 0 bias; 1 act(gate) * up (act_mode; interleaved rows; y [M, N/2]); 2 RoPE (NeoX) on the q and k heads +
//             scatter of the new k / v rows into the paged caches (rows packed by quant.pack_w4_qkv_rope; y [M, N] in
//             logical [q | k | v] order; positions int64 [M], cos_sin_cache [max_pos, head_dim] bf16, slot_ids int32
//             [M] (negative = skip), caches [blocks, block_size, num_kv_heads, head_dim]).
extern "C" int xb_linear_w4a16_decode_fused(void* y, int64_t y_stride, const void* x, int64_t x_stride,
                                            const uint32_t* qweight, const uint32_t* meta, const void* bias, int M, int N,
                                            int K, int group_size, const void* norm_weight, float eps,
                                            const void* residual_in, void* residual_out, int stage_x, int epilogue,
                                            int act_mode, const int64_t* positions, const void* cos_sin_cache,
                                            const int32_t* slot_ids, void* k_cache, void* v_cache, int num_heads,
                                            int num_kv_heads, int head_dim, const float* norm_stats_in,
                                            float* norm_stats_out, xb_stream_t stream) {
  XB_CHECK(epilogue >= 0 && epilogue <= 3, "linear_w4a16_decode_fused: epilogue %d unknown", epilogue);
  XB_CHECK(epilogue != 1 || (act_mode >= 0 && act_mode <= 2), "linear_w4a16_decode_fused: unsupported act mode %d", act_mode);
  XB_CHECK(M >= 0 && M <= 8, "linear_w4a16_decode_fused: M=%d out of range (0..8)", M);
  W4Fuse fz{};
  fz.norm_w = reinterpret_cast<const __nv_bfloat16*>(norm_weight);
  fz.res_in = reinterpret_cast<const __nv_bfloat16*>(residual_in);
  fz.res_out = reinterpret_cast<__nv_bfloat16*>(residual_out);
  fz.eps = eps;
  fz.stats_in = norm_stats_in;
  fz.stats_out = norm_stats_out;
  if (epilogue == 3) {
    XB_CHECK(residual_in && residual_out && norm_stats_out && !norm_weight,
             "linear_w4a16_decode_fused: epilogue 3 needs residual_in, residual_out and norm_stats_out (and no norm prologue)");
    XB_CHECK((reinterpret_cast<uintptr_t>(norm_stats_out) & 15) == 0, "linear_w4a16_decode_fused: norm_stats_out must be 16-byte aligned");
  } else {
    XB_CHECK(!norm_stats_out, "linear_w4a16_decode_fused: norm_stats_out belongs to epilogue 3");
    XB_CHECK(!(residual_in || residual_out) || norm_weight, "linear_w4a16_decode_fused: a residual needs the norm prologue");
  }
  if (norm_stats_in) {
    XB_CHECK(norm_weight && !residual_in && !residual_out && K % 16 == 0 &&
                 (reinterpret_cast<uintptr_t>(norm_stats_in) & 15) == 0,
             "linear_w4a16_decode_fused: norm_stats_in goes with norm_weight, x = the residual stream and no residual pointers");
  }
  XB_CHECK(!residual_in || residual_in != residual_out, "linear_w4a16_decode_fused: residual_out must not alias residual_in");
  XB_CHECK(!norm_weight || ((reinterpret_cast<uintptr_t>(norm_weight) | reinterpret_cast<uintptr_t>(residual_in) |
                             reinterpret_cast<uintptr_t>(residual_out)) & 15) == 0,
           "linear_w4a16_decode_fused: norm weight / residuals must be 16-byte aligned");
  if (epilogue == 2) {
    XB_CHECK(positions && cos_sin_cache && slot_ids && k_cache && v_cache, "linear_w4a16_decode_fused: rope epilogue needs positions, cos/sin, slots and caches");
    XB_CHECK((head_dim == 64 || head_dim == 128) && num_heads > 0 && num_kv_heads > 0 &&
                 N == (num_heads + 2 * num_kv_heads) * head_dim,
             "linear_w4a16_decode_fused: N=%d is not (%d + 2*%d) heads of %d", N, num_heads, num_kv_heads, head_dim);
    fz.rope = QkvRopeCache{positions, reinterpret_cast<const __nv_bfloat16*>(cos_sin_cache), slot_ids,
                           reinterpret_cast<__nv_bfloat16*>(k_cache), reinterpret_cast<__nv_bfloat16*>(v_cache),
                           num_heads, num_kv_heads, head_dim};
  }
  const bool xs = norm_weight != nullptr || stage_x != 0;
  return w4_small_m_impl(y, y_stride, x, x_stride, qweight, meta, bias, M, N, K, group_size, epilogue, act_mode, xs, &fz, stream);
}

// 1 when xb_linear_w4a16_decode_fused can stage an [M, K] activation block in shared memory (host-side query)
extern "C" int xb_linear_w4a16_decode_fused_fits(int M, int K) {
  return M >= 1 && M <= 8 && w4_xs_bytes(M, K) <= kXsMaxBytes ? 1 : 0;
}

template <int kMT>
static int bf16_small_m_launch(__nv_bfloat16* y, int64_t y_stride, const __nv_bfloat16* x, int64_t x_stride,
                               const __nv_bfloat16* w, const __nv_bfloat16* bias, int M, int N, int K, cudaStream_t s) {
  constexpr auto kern = linear_bf16_small_m_kernel<kMT>;
  constexpr int kRingBytes = kWarps * kBf16Ring * 1024;
  XB_CUDA_OK(set_max_dynamic_smem_once<kern>(kRingBytes));
  XB_CUDA_OK(launch(kern, dim3((N + 15) / 16), dim3(kWarps * 32), kRingBytes, s, true, y, y_stride, x, x_stride, w, bias,
                    M, N, K));
  return 0;
}

extern "C" int xb_linear_bf16_small_m(void* y, int64_t y_stride, const void* x, int64_t x_stride, const void* w,
                                      const void* bias, int M, int N, int K, xb_stream_t stream) {
  if (M == 0) return 0;
  XB_CHECK(M > 0 && M <= 64, "linear_bf16_small_m: M=%d out of range (1..64); use the wgmma GEMM", M);
  XB_CHECK(K % 32 == 0, "linear_bf16_small_m: K=%d must be a multiple of 32", K);
  XB_CHECK(x_stride % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
               (reinterpret_cast<uintptr_t>(w) & 15) == 0,
           "linear_bf16_small_m: x / w not 16B aligned");
  auto* yy = reinterpret_cast<__nv_bfloat16*>(y);
  auto* xx = reinterpret_cast<const __nv_bfloat16*>(x);
  auto* ww = reinterpret_cast<const __nv_bfloat16*>(w);
  auto* bb = reinterpret_cast<const __nv_bfloat16*>(bias);
  if (M <= 8) return bf16_small_m_launch<1>(yy, y_stride, xx, x_stride, ww, bb, M, N, K, (cudaStream_t)stream);
  if (M <= 16) return bf16_small_m_launch<2>(yy, y_stride, xx, x_stride, ww, bb, M, N, K, (cudaStream_t)stream);
  if (M <= 32) return bf16_small_m_launch<4>(yy, y_stride, xx, x_stride, ww, bb, M, N, K, (cudaStream_t)stream);
  return bf16_small_m_launch<8>(yy, y_stride, xx, x_stride, ww, bb, M, N, K, (cudaStream_t)stream);
}

// Host-side packer (plain C++): q[N,K] (one 4-bit value per byte) -> tile layout.
extern "C" int xb_w4_pack_rows(uint32_t* out, const uint8_t* q, int N, int K) {
  XB_CHECK(N % 16 == 0 && K % 64 == 0, "w4_pack_rows: N=%d must be %%16, K=%d %%64", N, K);
  const int ktiles = K / 64;
  for (int nt = 0; nt < N / 16; ++nt)
    for (int kt = 0; kt < ktiles; ++kt)
      for (int lane = 0; lane < 32; ++lane) {
        const int g = lane >> 2, t = lane & 3;
        const uint8_t* r0 = q + (size_t)(nt * 16 + g) * K + kt * 64 + 16 * t;
        const uint8_t* r1 = q + (size_t)(nt * 16 + g + 8) * K + kt * 64 + 16 * t;
        for (int j = 0; j < 4; ++j) {
          uint32_t w = 0;
          w |= (uint32_t)(r0[4 * j + 0] & 15) << 0;
          w |= (uint32_t)(r0[4 * j + 1] & 15) << 16;
          w |= (uint32_t)(r1[4 * j + 0] & 15) << 4;
          w |= (uint32_t)(r1[4 * j + 1] & 15) << 20;
          w |= (uint32_t)(r0[4 * j + 2] & 15) << 8;
          w |= (uint32_t)(r0[4 * j + 3] & 15) << 24;
          w |= (uint32_t)(r1[4 * j + 2] & 15) << 12;
          w |= (uint32_t)(r1[4 * j + 3] & 15) << 28;
          out[(((size_t)nt * ktiles + kt) * 32 + lane) * 4 + j] = w;
        }
      }
  return 0;
}
