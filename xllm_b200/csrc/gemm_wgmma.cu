// wgmma / TMA GEMM for the prefill-sized linears:  C[M,N] = A[M,K] . B[N,K]^T (+bias)
//   kind BF16 : A, B bf16 (K-major, as the reference stores activations [T,in] and weights [out,in])
//               replaces xllm::kernel::cuda::matmul -> F::linear (kernels/cuda/matmul.cpp:20-24)
//   kind FP8  : A, B e4m3, C = a_scale * (b_scale * acc) + bias, per-tensor or per-token / per-channel scales
//               replaces cutlass_scaled_mm (cutlass_w8a8/scaled_mm_entry.cu:55-108).  Converter warps widen both e4m3 tiles
//               to fp16 (exact) in the swizzled stage buffers the MMA reads: Hopper's e4m3 wgmma adds its products with
//               fewer than fp32's mantissa bits, which leaves results more than one bf16 ulp from the fp32-accumulated
//               spec, while fp16 wgmma accumulates in full fp32.
//   kind W4   : B is the tile-packed int4 weight of linear_small_m.cu; converter warps dequantise bf16((q-z)*s)
//               (bit-exact with the spec) straight into the 128B-swizzled K-major stage buffer the MMA reads, so the
//               unpack is fused into the wgmma main loop (no bf16 copy of W ever exists in HBM).  W8: the same with int8.
//
// One persistent CTA per SM, warp-specialised:
//   warp 0        TMA producer (A tiles, and B tiles / packed-B tiles), one elected lane
//   warps 4..11   two consumer warpgroups: warpgroup g owns rows 64 g .. 64 g + 63 of the 128-row tile, issues
//                 wgmma m64 x BLOCK_N x 16 (bf16, or fp16 for FP8) with fp32 register accumulators, then runs the
//                 epilogue (scale / bias -> bf16 -> global) from those registers
//   warps 12..15  (W4 / W8 / FP8) converters: packed int4 / int8 / e4m3 smem -> swizzled bf16 / fp16 smem -> fence.proxy.async
// Pipelines are mbarrier rings: smem full/empty (TMA <-> MMA), packed full / B ready / B empty (TMA <-> converters <-> MMA).
#include "tc_common.cuh"

namespace xb {
namespace tc {

EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess) p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_bytes, uint32_t box_rows,
                 uint32_t box_cols, int elem_bytes) {
  EncodeTiledFn enc = get_encode_tiled();
  XB_CHECK(enc != nullptr, "cuTensorMapEncodeTiled is not available from this driver");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMapDataType dt = elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8;
  CUresult r = enc(out, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  XB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d (rows %llu cols %llu pitch %llu)", (int)r,
           (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)pitch_bytes);
  return 0;
}

int make_tmap_2d_raw(CUtensorMap* out, const void* base, int dtype, uint64_t rows, uint64_t cols, uint64_t pitch_bytes,
                     uint32_t box_rows, uint32_t box_cols, int swizzle) {
  EncodeTiledFn enc = get_encode_tiled();
  XB_CHECK(enc != nullptr, "cuTensorMapEncodeTiled is not available from this driver");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, (CUtensorMapDataType)dtype, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, (CUtensorMapSwizzle)swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  XB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(raw) failed with CUresult %d", (int)r);
  return 0;
}

int make_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                      uint64_t stride2_bytes, uint32_t b0, uint32_t b1, uint32_t b2) {
  EncodeTiledFn enc = get_encode_tiled();
  XB_CHECK(enc != nullptr, "cuTensorMapEncodeTiled is not available from this driver");
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  XB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(3d) failed with CUresult %d", (int)r);
  return 0;
}


enum { kKindBF16 = 0, kKindFP8 = 1, kKindW4 = 2, kKindW8 = 3 };
constexpr bool kind_is_wq(int kind) { return kind == kKindW4 || kind == kKindW8; }   // weight-only: packed B + converter warps
constexpr bool kind_converts(int kind) { return kind != kKindBF16; }   // converter warps fill the MMA's operand ring

struct GemmParams {
  __nv_bfloat16* c;
  int64_t ldc;
  const __nv_bfloat16* bias;   // [N] or null
  const float* a_scale;        // fp8: [1] or [M]
  const float* b_scale;        // fp8: [1] or [N]
  int a_scale_per_row, b_scale_per_col;
  int gshift;                  // W4 / W8: log2(k64 tiles per quantisation group)
  int M, N, K;
  // swap-AB (decode-sized M): the WEIGHT rows ride in the 128-row MMA M slot and the tokens are the N tile, so every CTA
  // streams 128 weight rows instead of idling most of a 128-token tile.  M / N / a_scale / b_scale are already in the
  // swapped roles (M = output channels, N = tokens, a_scale per channel, b_scale per token); the epilogue indexes bias by
  // row, keeps the reference's product order token_scale * (channel_scale * acc) and stores C transposed: c[col][row]
  int swap_ab;
  // split-K (swap-AB FP8 only): a decode-sized GEMM has N/128 tiles - 10 for a TP8 qkv shard - so most SMs would idle while a
  // few CTAs stream all of K.  Each output tile is cut into split_k k-ranges walked by different CTAs; every CTA leaves its
  // fp32 partial in splitk_ws, takes a ticket (self-resetting atomicInc, so graph replays need no memset), and the LAST
  // arriver sums the partials in split order (deterministic) and runs the epilogue.  Nobody waits, so no co-residency
  // requirement.  Workspace: caller-owned (xb_set_gemm_splitk_workspace).
  int split_k;
  float* splitk_ws;            // [tiles][split_k][kBlockN][128] fp32
  unsigned int* splitk_tickets;  // [tiles], zero at rest
  // grouped MoE experts (kGroup != 0, the prefill path of moe.cu): A is the expert-sorted activation buffer [M = pairs, K],
  // B the local experts' weights stacked along N.  The tile count and every tile's expert come from the routing header the
  // route kernel wrote on the device (no host read).  fc1 (kGroupFc1): a tile loads up rows n0.. and gate rows I + n0.. as
  // two half boxes and the epilogue writes c[row][n0 + c] = bf16(silu(gate) * up) from the fp32 sums; fc2 (kGroupFc2): the
  // epilogue stores sorted row r to c[pair_of_row[r]], back in pair order.  N is I (fc1) or H (fc2).
  const int* grp_row_start;    // [E + 1] first sorted row of each local expert
  const int* grp_mtile_start;  // [E + 1] first 128-row m tile of each local expert
  const int* grp_pair_of_row;  // fc2: the pair (y2 row) of each sorted row
  int grp_experts;
  int grp_b_rows;              // weight rows per expert: 2I (fc1) or H (fc2)
  int grp_half;                // fc1: offset of the gate rows (I)
  int grp_meta_rows;           // W4: meta rows per expert (K / group_size)
};

enum { kGroupNone = 0, kGroupFc1 = 1, kGroupFc2 = 2 };

constexpr int kBlockM = 128;
constexpr int kConsumerWGs = 2;                 // 64 rows each
constexpr int kConsumerThreads = kConsumerWGs * 128;

template <int kKind, int kBlockN>
struct GemmCfg {
  static constexpr int kBlockK = 64;                               // k elements per stage: one 128-byte row of 16-bit operands
  static constexpr int kMmaK = 16;
  static constexpr int kElemA = kKind == kKindFP8 ? 1 : 2;
  static constexpr int kABytes = kBlockM * kBlockK * kElemA;      // A tile as TMA lands it (FP8: unswizzled 64-byte rows)
  static constexpr int kBBytes = kBlockN * 128;                    // 16-bit B tile the MMA reads (128B-swizzled)
  static constexpr int kPackedBytes = kKind == kKindW4 ? kBlockN * kBlockK / 2 : (kKind == kKindW8 ? kBlockN * kBlockK :
                                      (kKind == kKindFP8 ? kBlockN * kBlockK : 0));
  static constexpr int kMetaBytes = kind_is_wq(kKind) ? kBlockN * 4 : 0;
  // BF16: a stage holds the A and B tiles.  W4 / W8: A + the PACKED B tile + its scale/zero words; FP8: both e4m3 tiles.  The
  // packed stages are small, so the TMA ring can be deep enough to cover HBM latency; the 16-bit operands the converters
  // write live in a separate 2-deep ring (FP8: A and B, W4 / W8: B).
  static constexpr int kPackedRegion = ((kPackedBytes + 1023) / 1024) * 1024;      // stages stay 1024-byte aligned (SW128)
  static constexpr int kStageBytes = kind_converts(kKind) ? kABytes + kPackedRegion + ((kMetaBytes + 1023) / 1024) * 1024
                                                          : kABytes + kBBytes;
  static constexpr int kRingABytes = kKind == kKindFP8 ? kBlockM * 128 : 0;
  static constexpr int kRingBytes = kRingABytes + kBBytes;
  static_assert(kStageBytes % 1024 == 0 && kBBytes % 1024 == 0 && kABytes % 1024 == 0, "SW128 tiles need 1024-byte alignment");
  static constexpr int kBStages = kind_converts(kKind) ? 2 : 0;
  static constexpr int kBRing = 2;                                  // barriers of the ring (dummies when unused)
  static constexpr int kConvWarps = kind_converts(kKind) ? 4 : 0;
  static constexpr int kBudget = 227 * 1024 - 1024 - 512 - kBStages * kRingBytes;
  static constexpr int kStages = kBudget / kStageBytes > 8 ? 8 : kBudget / kStageBytes;
  static constexpr int kThreads = 128 + kConsumerThreads + kConvWarps * 32;
  static constexpr int kAcc = kBlockN / 2;                          // fp32 accumulators per consumer thread
  static constexpr int kSmemBytes = kStages * kStageBytes + kBStages * kRingBytes + 1024 /*align*/ + 512 /*barriers*/;
};

// One k block of wgmma m64 x BLOCK_N x 16 into the fp32 accumulators (committed and waited for by the caller)
template <int kKind, int kBlockN>
__device__ __forceinline__ void gemm_mma(float (&acc)[kBlockN / 2], uint32_t a_addr, uint32_t b_addr, bool accumulate) {
  using Cfg = GemmCfg<kKind, kBlockN>;
#pragma unroll
  for (int k = 0; k < Cfg::kBlockK / Cfg::kMmaK; ++k) {
    const uint64_t da = gmma_desc_sw128(a_addr + k * 32), db = gmma_desc_sw128(b_addr + k * 32);
    const uint32_t scale_d = (accumulate || k > 0) ? 1u : 0u;
    if constexpr (kKind == kKindFP8) wgmma_f16<kBlockN>(acc, da, db, scale_d);
    else wgmma_bf16<kBlockN>(acc, da, db, scale_d);
  }
}

// four e4m3 (k ascending) -> two f16x2, exact
__device__ __forceinline__ void e4m3x4_to_f16(uint32_t w, uint32_t& lo, uint32_t& hi) {
  asm("{\n.reg .b16 l, h;\nmov.b32 {l, h}, %2;\ncvt.rn.f16x2.e4m3x2 %0, l;\ncvt.rn.f16x2.e4m3x2 %1, h;\n}\n"
      : "=r"(lo), "=r"(hi) : "r"(w));
}

// grouped mode: linear tile index -> (local expert, m block within the expert, n block).  Expert e owns the tiles
// [mtile_start[e] * n_blocks, mtile_start[e + 1] * n_blocks), m fastest, so the m blocks of one expert run next to each other
// and share every B tile through L2.  Experts without rows own no tiles.
struct GroupTile {
  int e, m_blk, n_blk;
  int a_row;   // first sorted row of the tile
  int rows;    // rows of the tile that belong to expert e (the rest are the next expert's or past the end: masked)
};
__device__ __forceinline__ GroupTile group_tile(const GemmParams& p, int tile, int n_blocks) {
  const int* ms = p.grp_mtile_start;
  int lo = 0, hi = p.grp_experts;   // ms[lo] * n_blocks <= tile < ms[hi] * n_blocks
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (ms[mid] * n_blocks <= tile) lo = mid;
    else hi = mid;
  }
  GroupTile g;
  const int mt = ms[lo + 1] - ms[lo];
  const int local = tile - ms[lo] * n_blocks;
  g.e = lo;
  g.n_blk = local / mt;
  g.m_blk = local - g.n_blk * mt;
  g.a_row = p.grp_row_start[lo] + g.m_blk * kBlockM;
  g.rows = min(kBlockM, p.grp_row_start[lo + 1] - g.a_row);
  return g;
}

template <int kKind, int kBlockN, int kGroup = kGroupNone>
__global__ void __launch_bounds__(GemmCfg<kKind, kBlockN>::kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_m, const GemmParams p) {
  using Cfg = GemmCfg<kKind, kBlockN>;
  constexpr int kStages = Cfg::kStages;
  static_assert(kGroup == kGroupNone || kKind == kKindBF16 || kKind == kKindW4, "grouped mode: bf16 and W4 only");
  constexpr int kTileCols = kGroup == kGroupFc1 ? kBlockN / 2 : kBlockN;   // output columns of a tile (fc1: up | gate halves)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* bbuf = smem + kStages * Cfg::kStageBytes;                  // [kBStages][kRingBytes] converted operand ring
  uint8_t* bar_mem = bbuf + Cfg::kBStages * Cfg::kRingBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bar_mem);          // [kStages] TMA -> MMA (A, and B for BF16); FP8: -> converters
  uint64_t* empty_bar = full_bar + kStages;                           // [kStages] MMA (FP8: converters) -> TMA
  uint64_t* packed_bar = empty_bar + kStages;                         // [kStages] TMA -> converters (W4 / W8)
  uint64_t* bready_bar = packed_bar + kStages;                        // [kBRing] converters -> MMA
  uint64_t* bempty_bar = bready_bar + Cfg::kBRing;                    // [kBRing] MMA -> converters
  volatile uint32_t* ticket_flag = reinterpret_cast<volatile uint32_t*>(bempty_bar + Cfg::kBRing);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blocks = (p.M + kBlockM - 1) / kBlockM;
  const int n_blocks = (p.N + kTileCols - 1) / kTileCols;
  const int num_kb = (p.K + Cfg::kBlockK - 1) / Cfg::kBlockK;
  // split-K exists in the swap-AB FP8 instantiations only (compile-time off elsewhere)
  constexpr bool kSplitOK = kKind == kKindFP8 && kBlockN <= 64;
  const int split_k = kSplitOK ? p.split_k : 1;
  const int kb_per = (num_kb + split_k - 1) / split_k;
  int num_tiles = m_blocks * n_blocks * split_k;      // work units: (output tile, k range); the splits of a tile are adjacent

  auto stage_a = [&](int s) { return smem + s * Cfg::kStageBytes; };
  auto stage_b = [&](int s) { return smem + s * Cfg::kStageBytes + Cfg::kABytes; };               // BF16
  auto stage_packed = [&](int s) { return smem + s * Cfg::kStageBytes + Cfg::kABytes; };          // W4 / W8 / FP8 (e4m3 B)
  auto stage_meta = [&](int s) { return smem + s * Cfg::kStageBytes + Cfg::kABytes + Cfg::kPackedRegion; };
  auto ring_a = [&](int bs) { return bbuf + bs * Cfg::kRingBytes; };                               // FP8: fp16 A
  auto b_ring = [&](int bs) { return bbuf + bs * Cfg::kRingBytes + Cfg::kRingABytes; };

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar + s, 1);
      mbar_init(empty_bar + s, kKind == kKindFP8 ? Cfg::kConvWarps : kConsumerThreads / 32);   // one arrive per reading warp
      mbar_init(packed_bar + s, 1);
    }
    for (int s = 0; s < Cfg::kBRing; ++s) {
      mbar_init(bready_bar + s, Cfg::kConvWarps > 0 ? Cfg::kConvWarps : 1);
      mbar_init(bempty_bar + s, kConsumerThreads / 32);
    }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (kind_is_wq(kKind)) tma_prefetch_desc(&tmap_m);
  }
  __syncthreads();

  pdl_launch_dependents();
  pdl_wait();   // A (activations) comes from the producer kernel
  if constexpr (kGroup != kGroupNone) num_tiles = p.grp_mtile_start[p.grp_experts] * n_blocks;   // written by the route kernel

  if (warp == 0) {
    // ======================= TMA producer =======================
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int otile = tile / split_k, ks = tile - otile * split_k;
        const int m_blk = otile % m_blocks, n_blk = otile / m_blocks;
        const int kb0 = ks * kb_per, kb1 = min(num_kb, kb0 + kb_per);
        // first A row, first B (weight) row and first meta row / column of the tile; grouped: offset to the tile's expert
        int a_row = m_blk * kBlockM, b_row = n_blk * kBlockN, meta_row = 0, meta_col = n_blk * kBlockN;
        if constexpr (kGroup != kGroupNone) {
          const GroupTile gt = group_tile(p, tile, n_blocks);
          a_row = gt.a_row;
          b_row = gt.e * p.grp_b_rows + gt.n_blk * kTileCols;
          meta_row = gt.e * p.grp_meta_rows;
          meta_col = gt.n_blk * kTileCols;
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(empty_bar + s, ph ^ 1);
          if (kind_is_wq(kKind)) {
            // packed B: the kBlockN/16 row tiles of this k tile are one 2-D TMA box (tensor [N/16][K/64 * 128 words],
            // box [kBlockN/16][128 words], no swizzle), plus the group's scale/zero words for these rows (tensor [K/g][N])
            mbar_expect_tx(packed_bar + s, Cfg::kPackedBytes + Cfg::kMetaBytes);
            // (W8: one byte per weight - 256 words per row tile and k tile instead of 128)
            tma_load_2d(stage_packed(s), &tmap_b, packed_bar + s, kb * (kKind == kKindW8 ? 256 : 128), b_row / 16);
            tma_load_2d(stage_meta(s), &tmap_m, packed_bar + s, meta_col, meta_row + (kb >> p.gshift));
            if constexpr (kGroup == kGroupFc1) {   // the matching gate rows: second half of the packed tile and of the meta
              tma_load_2d(stage_packed(s) + Cfg::kPackedBytes / 2, &tmap_b, packed_bar + s, kb * 128, (b_row + p.grp_half) / 16);
              tma_load_2d(stage_meta(s) + Cfg::kMetaBytes / 2, &tmap_m, packed_bar + s, meta_col + p.grp_half,
                          meta_row + (kb >> p.gshift));
            }
            mbar_expect_tx(full_bar + s, Cfg::kABytes);
            tma_load_2d(stage_a(s), &tmap_a, full_bar + s, kb * Cfg::kBlockK, a_row);
          } else if (kKind == kKindFP8) {
            mbar_expect_tx(full_bar + s, Cfg::kABytes + Cfg::kPackedBytes);
            tma_load_2d(stage_a(s), &tmap_a, full_bar + s, kb * Cfg::kBlockK, a_row);
            tma_load_2d(stage_packed(s), &tmap_b, full_bar + s, kb * Cfg::kBlockK, b_row);
          } else {
            mbar_expect_tx(full_bar + s, Cfg::kABytes + Cfg::kBBytes);
            tma_load_2d(stage_a(s), &tmap_a, full_bar + s, kb * Cfg::kBlockK, a_row);
            tma_load_2d(stage_b(s), &tmap_b, full_bar + s, kb * Cfg::kBlockK, b_row);
            if constexpr (kGroup == kGroupFc1)      // gate rows into the second half of the B tile
              tma_load_2d(stage_b(s) + Cfg::kBBytes / 2, &tmap_b, full_bar + s, kb * Cfg::kBlockK, b_row + p.grp_half);
          }
          if (++s == kStages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp >= 4 && warp < 4 + kConsumerThreads / 32) {
    // ======================= consumers: wgmma main loop + epilogue =======================
    const int wg = (warp - 4) >> 2;            // 64-row half of the tile
    const int wq = warp & 3;                   // 16-row slice of the warpgroup's half
    const int ctid = threadIdx.x - 128;        // 0 .. 255
    float acc[Cfg::kAcc];
    int s = 0;
    uint32_t ph = 0;
    int bs = 0;
    uint32_t bph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int otile = tile / split_k, ks = tile - otile * split_k;
      const int m_blk = otile % m_blocks, n_blk = otile / m_blocks;
      const int kb0 = ks * kb_per, kb1 = min(num_kb, kb0 + kb_per);
      int prev_s = -1, prev_bs = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        if (kKind != kKindFP8) mbar_wait(full_bar + s, ph);
        if (kind_converts(kKind)) mbar_wait(bready_bar + bs, bph);
        const uint32_t a_addr = smem_u32(kKind == kKindFP8 ? ring_a(bs) : stage_a(s)) + wg * 64 * 128;
        const uint32_t b_addr = smem_u32(kind_converts(kKind) ? b_ring(bs) : stage_b(s));
        wgmma_fence();
        gemm_mma<kKind, kBlockN>(acc, a_addr, b_addr, kb > kb0);
        wgmma_commit();
        wgmma_wait<1>();                       // the MMAs of the previous k block have read their operands
        if (prev_s >= 0 && lane == 0) {
          if (kKind != kKindFP8) mbar_arrive(empty_bar + prev_s);
          if (kind_converts(kKind)) mbar_arrive(bempty_bar + prev_bs);
        }
        prev_s = s;
        prev_bs = bs;
        if (++s == kStages) { s = 0; ph ^= 1; }
        if (kind_converts(kKind) && ++bs == Cfg::kBRing) { bs = 0; bph ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_operands(acc);
      if (prev_s >= 0 && lane == 0) {
        if (kKind != kKindFP8) mbar_arrive(empty_bar + prev_s);
        if (kind_converts(kKind)) mbar_arrive(bempty_bar + prev_bs);
      }

      // ---- epilogue: fragment element d[4j + 2h + e] is (row r0 + 8h, column c0 + 8j + e) of the tile ----
      const int r_loc = wg * 64 + wq * 16 + (lane >> 2);
      const int c_loc = 2 * (lane & 3);
      if constexpr (kGroup != kGroupNone) {
        // rows past the expert's segment are masked; N (I or H) is a multiple of 32, so a column pair is in or out together
        const GroupTile gt = group_tile(p, tile, n_blocks);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int rr = r_loc + 8 * h;
          if (rr >= gt.rows) continue;
          const int row = gt.a_row + rr;
          if constexpr (kGroup == kGroupFc1) {
            // up column c is fragment column group j < kBlockN / 16, its gate column c + kBlockN / 2 is group j + kBlockN / 16
            __nv_bfloat16* crow = p.c + (int64_t)row * p.ldc;
#pragma unroll
            for (int j = 0; j < Cfg::kAcc / 8; ++j) {
              const int col = gt.n_blk * kTileCols + 8 * j + c_loc;
              if (col >= p.N) continue;
              float o[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float up = acc[4 * j + 2 * h + e], gate = acc[4 * (j + Cfg::kAcc / 8) + 2 * h + e];
                o[e] = silu_mul_f32(gate, up);
              }
              *reinterpret_cast<uint32_t*>(crow + col) = pack_bf16x2(o[0], o[1]);
            }
          } else {
            __nv_bfloat16* crow = p.c + (int64_t)p.grp_pair_of_row[row] * p.ldc;   // back to pair order
#pragma unroll
            for (int j = 0; j < Cfg::kAcc / 4; ++j) {
              const int col = gt.n_blk * kBlockN + 8 * j + c_loc;
              if (col >= p.N) continue;
              *reinterpret_cast<uint32_t*>(crow + col) = pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
          }
        }
        continue;
      }
      if (kSplitOK && split_k > 1) {
        // leave this k range's fp32 partial in the workspace ([split][column][row]), take a ticket; the last arriver sums
        // the partials in split order (the same order whichever CTA arrived last: bit-reproducible)
        float* wp = p.splitk_ws + ((size_t)otile * split_k + ks) * (kBlockN * kBlockM);
#pragma unroll
        for (int i = 0; i < Cfg::kAcc; ++i) {
          const int j = i >> 2, h = (i >> 1) & 1, e = i & 1;
          __stcg(wp + (c_loc + 8 * j + e) * kBlockM + r_loc + 8 * h, acc[i]);
        }
        __threadfence();
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
        if (ctid == 0) *ticket_flag = atomicInc(p.splitk_tickets + otile, (unsigned)split_k - 1u);
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
        const bool last = *ticket_flag == (uint32_t)split_k - 1u;
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");   // the flag is read before the next tile's ticket
        if (!last) continue;
        __threadfence();
        const float* ws_tile = p.splitk_ws + (size_t)otile * split_k * (kBlockN * kBlockM);
#pragma unroll
        for (int i = 0; i < Cfg::kAcc; ++i) {
          const int j = i >> 2, h = (i >> 1) & 1, e = i & 1;
          const int off = (c_loc + 8 * j + e) * kBlockM + r_loc + 8 * h;
          float v = __ldcg(ws_tile + off);
          for (int sp = 1; sp < split_k; ++sp) v += __ldcg(ws_tile + (size_t)sp * (kBlockN * kBlockM) + off);
          acc[i] = v;
        }
      }
      const bool pair_store = !p.swap_ab && (p.ldc % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.c) & 3) == 0);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m_blk * kBlockM + r_loc + 8 * h;
        if (row >= p.M) continue;
        float a_s = 1.f, b_s_uniform = 1.f;
        if (kKind == kKindFP8) {
          a_s = p.a_scale[p.a_scale_per_row ? row : 0];
          b_s_uniform = p.b_scale[0];
        }
        const float bias_row = (p.bias && p.swap_ab) ? __bfloat162float(p.bias[row]) : 0.f;
#pragma unroll
        for (int j = 0; j < Cfg::kAcc / 4; ++j) {
          const int col = n_blk * kBlockN + 8 * j + c_loc;
          if (col >= p.N) continue;
          float x[2] = {acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int cc = min(col + e, p.N - 1);
            if (kKind == kKindFP8) {
              const float b = p.b_scale_per_col ? p.b_scale[cc] : b_s_uniform;
              // ScaledEpilogue order scale_a * (scale_b * acc); swap-AB: rows = channels (scale_b), columns = tokens
              x[e] = p.swap_ab ? b * (a_s * x[e]) : a_s * (b * x[e]);
            }
            if (p.bias) x[e] += p.swap_ab ? bias_row : __bfloat162float(p.bias[cc]);
          }
          if (p.swap_ab) {
            p.c[(int64_t)col * p.ldc + row] = __float2bfloat16_rn(x[0]);
            if (col + 1 < p.N) p.c[(int64_t)(col + 1) * p.ldc + row] = __float2bfloat16_rn(x[1]);
          } else if (pair_store && col + 1 < p.N) {
            *reinterpret_cast<uint32_t*>(p.c + (int64_t)row * p.ldc + col) = pack_bf16x2(x[0], x[1]);
          } else {
            p.c[(int64_t)row * p.ldc + col] = __float2bfloat16_rn(x[0]);
            if (col + 1 < p.N) p.c[(int64_t)row * p.ldc + col + 1] = __float2bfloat16_rn(x[1]);
          }
        }
      }
    }
  } else if (kKind == kKindFP8 && warp >= 4 + kConsumerThreads / 32) {
    // ======================= FP8 converters (warps 12..15) =======================
    // e4m3 A [128][64] and B [kBlockN][64] (unswizzled 64-byte rows) -> fp16 rows of 128 bytes in the 128B-swizzled ring
    // (16-byte chunk c of row r at chunk c ^ (r & 7)); a thread widens one 16-byte run (16 elements) per step
    const int cw = warp - (4 + kConsumerThreads / 32);
    int s = 0, bs = 0;
    uint32_t ph = 0, bph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int ks = tile % split_k;
      const int kb0 = ks * kb_per, kb1 = min(num_kb, kb0 + kb_per);
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(full_bar + s, ph);            // both e4m3 tiles landed
        mbar_wait(bempty_bar + bs, bph ^ 1);    // the MMAs have finished reading this ring slot
        const uint32_t sa = smem_u32(stage_a(s)), sb = smem_u32(stage_packed(s));
        const uint32_t ra = smem_u32(ring_a(bs)), rb = smem_u32(b_ring(bs));
#pragma unroll 4
        for (int i = cw * 32 + lane; i < (kBlockM + kBlockN) * 4; i += Cfg::kConvWarps * 32) {
          const int r = i >> 2, c = i & 3;
          const bool is_a = r < kBlockM;
          const int rr = is_a ? r : r - kBlockM;
          const uint4 v = lds_128((is_a ? sa : sb) + rr * 64 + c * 16);
          uint32_t h[8];
          e4m3x4_to_f16(v.x, h[0], h[1]);
          e4m3x4_to_f16(v.y, h[2], h[3]);
          e4m3x4_to_f16(v.z, h[4], h[5]);
          e4m3x4_to_f16(v.w, h[6], h[7]);
          const uint32_t dst = (is_a ? ra : rb) + rr * 128;
          sts_128(dst + (((2 * c) ^ (rr & 7)) << 4), make_uint4(h[0], h[1], h[2], h[3]));
          sts_128(dst + (((2 * c + 1) ^ (rr & 7)) << 4), make_uint4(h[4], h[5], h[6], h[7]));
        }
        fence_proxy_async_smem();     // generic-proxy stores -> visible to the tensor core's async-proxy reads
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(bready_bar + bs);
          mbar_arrive(empty_bar + s);   // the e4m3 stage may be refilled
        }
        if (++s == kStages) { s = 0; ph ^= 1; }
        if (++bs == Cfg::kBRing) { bs = 0; bph ^= 1; }
      }
    }
  } else if (kind_is_wq(kKind) && warp >= 4 + kConsumerThreads / 32) {
    // ======================= W4 / W8 converters (warps 12..15) =======================
    // converter warp cw handles row tiles cw, cw+4, ... of the stage; a lane's 16 bytes of packed data are
    // rows (g, g+8) x k in [16t, 16t+16) of its row tile  ->  four 16-byte chunks of the swizzled bf16 tile.
    const int cw = warp - (4 + kConsumerThreads / 32);
    const int g = lane >> 2, t = lane & 3;
    int it = 0;                                  // k blocks since kernel start
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int s = it % kStages, bs = it % Cfg::kBRing;
        const uint32_t ph = (it / kStages) & 1, bph = (it / Cfg::kBRing) & 1;
        mbar_wait(packed_bar + s, ph);          // packed tile + meta landed
        mbar_wait(bempty_bar + bs, bph ^ 1);    // the MMAs have finished reading this B buffer
        // explicit shared-space addresses: through generic pointers these compile to LD.E / ST.E (address-space
        // resolution per access) instead of LDS / STS
        const uint32_t pk = smem_u32(stage_packed(s));
        const uint32_t mt = smem_u32(stage_meta(s));
        const uint32_t bt = smem_u32(b_ring(bs));
#pragma unroll
        for (int r = cw; r < kBlockN / 16; r += Cfg::kConvWarps) {
          uint32_t lo[8], hi[8];   // row g / row g+8: 16 bf16 = 8 packed registers, k ascending
          const uint32_t m0 = lds_32(mt + (r * 16 + g) * 4), m1 = lds_32(mt + (r * 16 + g + 8) * 4);
          if constexpr (kKind == kKindW8) {
            // int8 tile: 32 bytes per lane (row g then row g+8), meta = bf16 scale | zero << 16 (common.cuh w8_dequant_word)
            const uint4 wa = lds_128(pk + r * 1024 + lane * 32);
            const uint4 wb = lds_128(pk + r * 1024 + lane * 32 + 16);
            uint32_t s0, s1;
            float nz0, nz1;
            w8_meta(m0, s0, nz0);
            w8_meta(m1, s1, nz1);
            const uint32_t* av = &wa.x;
            const uint32_t* bv = &wb.x;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              w8_dequant_word(av[j], nz0, s0, lo[2 * j], lo[2 * j + 1]);
              w8_dequant_word(bv[j], nz1, s1, hi[2 * j], hi[2 * j + 1]);
            }
          } else {
            // int4 tile: 16 bytes per lane in the layout of linear_small_m.cu (common.cuh w4_dequant_word)
            const uint4 wq = lds_128(pk + r * 512 + lane * 16);
            uint32_t s0, z0, s1, z1;
            w4_meta(m0, s0, z0);
            w4_meta(m1, s1, z1);
            const uint32_t* wv = &wq.x;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              uint32_t a[4];
              w4_dequant_word(wv[j], z0, s0, z1, s1, a);
              lo[2 * j] = a[0];
              hi[2 * j] = a[1];
              lo[2 * j + 1] = a[2];
              hi[2 * j + 1] = a[3];
            }
          }
          // swizzled K-major tile: row n at n*128 bytes, 16-byte chunk c stored at chunk (c ^ (n & 7))
          const int n_lo = r * 16 + g, n_hi = n_lo + 8;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int c = 2 * t + h;
            sts_128(bt + n_lo * 128 + ((c ^ (n_lo & 7)) << 4), make_uint4(lo[4 * h], lo[4 * h + 1], lo[4 * h + 2], lo[4 * h + 3]));
            sts_128(bt + n_hi * 128 + ((c ^ (n_hi & 7)) << 4), make_uint4(hi[4 * h], hi[4 * h + 1], hi[4 * h + 2], hi[4 * h + 3]));
          }
        }
        fence_proxy_async_smem();     // generic-proxy stores -> visible to the tensor core's async-proxy reads
        __syncwarp();
        if (lane == 0) mbar_arrive(bready_bar + bs);
      }
    }
  }
}

template <int kKind, int kBlockN, int kGroup = kGroupNone>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, GemmParams p, cudaStream_t stream,
                       const CUtensorMap* tm = nullptr) {
  using Cfg = GemmCfg<kKind, kBlockN>;
  constexpr auto kern = gemm_wgmma_kernel<kKind, kBlockN, kGroup>;
  XB_CUDA_OK(set_max_dynamic_smem_once<kern>(Cfg::kSmemBytes));
  const int max_ctas = device_sm_count();     // persistent CTAs: one per SM
  if (p.split_k < 1) p.split_k = 1;
  // grouped: the tile count is only known on the device; every expert adds at most one partial m tile
  constexpr int kTileCols = kGroup == kGroupFc1 ? kBlockN / 2 : kBlockN;
  const int64_t m_units = (p.M + kBlockM - 1) / kBlockM + (kGroup != kGroupNone ? p.grp_experts : 0);
  const int64_t units = m_units * ((p.N + kTileCols - 1) / kTileCols) * p.split_k;
  dim3 grid(units < max_ctas ? (unsigned)units : (unsigned)max_ctas), block(Cfg::kThreads);
  XB_CUDA_OK(launch(kern, grid, block, (size_t)Cfg::kSmemBytes, stream, true, ta, tb, tm ? *tm : ta, p));
  return 0;
}

// grouped expert GEMMs of the MoE prefill path (declared in tc_common.cuh, called by moe.cu after the routing kernels).  Shapes
// and alignment are validated by the MoE entry points.
//   fc1: c = act [P, I],  act[r] = bf16(silu(a[r] . gate_e) * (a[r] . up_e)),  a [P, H];  b = fc1 stacked [E * 2I, H]
//   fc2: c = y2 [P, H],   y2[pair_of_row[r]] = bf16(a[r] . fc2_e),              a = act [P, I];  b = fc2 stacked [E * H, I]
// W4: b is the stacked tile-packed qweight [E * rows / 16, K / 64 * 128] u32 and meta the stacked [E * K / g, rows] words.
// BLOCK_N is 128 throughout: fc1 tiles then cover 64 output columns (64 up + 64 gate rows of B).
int moe_grouped_gemm(int w4, int fc2, void* c, const void* a, const void* b, const uint32_t* meta, int gshift, int group_size,
                     const int* row_start, const int* mtile_start, const int* pair_of_row, int P, int H, int I, int E,
                     cudaStream_t stream) {
  constexpr int kBN = 128;
  const int N = fc2 ? H : I, K = fc2 ? I : H;
  const int rows = fc2 ? H : 2 * I;             // weight rows per expert
  const uint32_t box_rows = fc2 ? kBN : kBN / 2;
  GemmParams p{};
  p.c = reinterpret_cast<__nv_bfloat16*>(c);
  p.ldc = N;
  p.M = P; p.N = N; p.K = K;
  p.gshift = gshift;
  p.grp_row_start = row_start;
  p.grp_mtile_start = mtile_start;
  p.grp_pair_of_row = pair_of_row;
  p.grp_experts = E;
  p.grp_b_rows = rows;
  p.grp_half = I;
  p.grp_meta_rows = w4 ? K / group_size : 0;
  CUtensorMap ta, tb, tm;
  if (make_tmap_2d(&ta, a, P, K, (uint64_t)K * 2, kBlockM, 64, 2)) return 1;
  if (!w4) {
    if (make_tmap_2d(&tb, b, (uint64_t)E * rows, K, (uint64_t)K * 2, box_rows, 64, 2)) return 1;
    return fc2 ? launch_gemm<kKindBF16, kBN, kGroupFc2>(ta, tb, p, stream)
               : launch_gemm<kKindBF16, kBN, kGroupFc1>(ta, tb, p, stream);
  }
  const uint64_t ktiles = K / 64;
  if (make_tmap_2d_raw(&tb, b, CU_TENSOR_MAP_DATA_TYPE_UINT32, (uint64_t)E * rows / 16, ktiles * 128, ktiles * 512, box_rows / 16,
                       128, CU_TENSOR_MAP_SWIZZLE_NONE))
    return 1;
  if (make_tmap_2d_raw(&tm, meta, CU_TENSOR_MAP_DATA_TYPE_UINT32, (uint64_t)E * (K / group_size), rows, (uint64_t)rows * 4, 1,
                       box_rows, CU_TENSOR_MAP_SWIZZLE_NONE))
    return 1;
  return fc2 ? launch_gemm<kKindW4, kBN, kGroupFc2>(ta, tb, p, stream, &tm)
             : launch_gemm<kKindW4, kBN, kGroupFc1>(ta, tb, p, stream, &tm);
}

}  // namespace tc
}  // namespace xb

using namespace xb;
using namespace xb::tc;

// e4m3 operand [rows, K] as the FP8 converters read it: boxes of box_rows x 64 bytes, unswizzled
static int make_tmap_fp8(CUtensorMap* out, const void* base, uint64_t rows, uint64_t K, uint64_t pitch, uint32_t box_rows) {
  return make_tmap_2d_raw(out, base, CU_TENSOR_MAP_DATA_TYPE_UINT8, rows, K, pitch, box_rows, 64, CU_TENSOR_MAP_SWIZZLE_NONE);
}

// pick BLOCK_N so that small problems still spread over the SMs: 128-column tiles once there are enough of them to fill
// the 132 SMs about once, 64-column tiles below that (the reference buckets by M the same way)
static int pick_block_n(int M, int N) {
  const int m_blocks = (M + kBlockM - 1) / kBlockM;
  if ((int64_t)m_blocks * ((N + 127) / 128) >= 120) return 128;
  return 64;
}

static std::atomic<int> g_fp8_swap_max_m{-1};
static int fp8_swap_max_m() {
  int v = g_fp8_swap_max_m.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("XB_FP8_SWAP_MAX_M");
    v = e ? atoi(e) : 64;
    if (v < 0 || v > 64) v = 64;
    g_fp8_swap_max_m.store(v, std::memory_order_relaxed);
  }
  return v;
}

// split-K workspace of the swap-AB FP8 GEMM (caller-owned device memory; every split-K launch uses it, so launches that share
// it must be stream-ordered - the decode step's are).  Layout: 4 KB of tickets (zeroed here, self-resetting afterwards), then
// the fp32 partials.
static std::atomic<void*> g_splitk_ws{nullptr};
static std::atomic<size_t> g_splitk_bytes{0};
static std::atomic<int> g_splitk_device{-1};     // the device the workspace lives on: GEMMs on another device run unsplit
static std::atomic<int> g_splitk_max{-1};
constexpr size_t kSplitKTicketBytes = 4096;
static int splitk_max() {
  int v = g_splitk_max.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("XB_FP8_SPLITK_MAX");
    v = e ? atoi(e) : 8;
    if (v < 1 || v > 32) v = 8;
    g_splitk_max.store(v, std::memory_order_relaxed);
  }
  return v;
}
// k ranges for `tiles` output tiles over `num_kb` k blocks: fill the SMs once (tiles * split <= sm_count), keep >= 12 k blocks
// per range (shorter ranges spend more on filling the TMA ring and the ticket round trip than the extra CTAs win) and no
// empty range
static int split_k_for(int tiles, int num_kb, int sms) {
  int split = sms / tiles;
  if (split > splitk_max()) split = splitk_max();
  if (split > num_kb / 12) split = num_kb / 12;
  if (split < 2) return 1;
  const int kb_per = (num_kb + split - 1) / split;
  split = (num_kb + kb_per - 1) / kb_per;
  return split < 2 ? 1 : split;
}
static int pick_split_k(int tiles, int num_kb, int tokens_bn, size_t* need_bytes) {
  *need_bytes = 0;
  if (g_splitk_ws.load(std::memory_order_relaxed) == nullptr) return 1;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev != g_splitk_device.load(std::memory_order_relaxed)) {
    cudaGetLastError();
    return 1;
  }
  int split = split_k_for(tiles, num_kb, device_sm_count());
  if (split < 2) return 1;
  const size_t need = kSplitKTicketBytes + (size_t)tiles * split * tokens_bn * kBlockM * sizeof(float);
  if ((size_t)tiles * sizeof(unsigned) > kSplitKTicketBytes || need > g_splitk_bytes.load(std::memory_order_relaxed)) return 1;
  *need_bytes = need;
  return split;
}

// host-only query (no device needed): the number of k ranges xb_gemm_fp8_scaled would use for an [M, K] x [N, K]^T product on a
// device with `sm_count` SMs once a workspace is registered; 1 = unsplit.  For capacity planning and the CPU tests.
extern "C" int xb_gemm_fp8_split_k(int M, int N, int K, int sm_count) {
  if (M <= 0 || N < 128 || K <= 0 || sm_count <= 0 || M > 64 || M > fp8_swap_max_m()) return 1;
  return split_k_for((N + kBlockM - 1) / kBlockM, (K + 127) / 128, sm_count);
}

// host-only (no device needed): which kernel variant the GEMM entry points pick for a shape, as text, e.g.
// "bf16 bn=128", "fp8 swap-AB bn=32 split_k=5", "w4 bn=64".  kind: 0 bf16 | 1 fp8 | 2 w4a16 | 3 w8a16.  Mirrors the decision
// order of xb_gemm_bf16 / xb_gemm_fp8_scaled / xb_gemm_w4a16 / xb_gemm_w8a16 below (keep the two in step); split_k is what a
// registered workspace would allow on a device with sm_count SMs.  Returns the length written, -1 on a bad kind.
extern "C" int xb_gemm_describe(int kind, int M, int N, int K, int sm_count, char* buf, int buf_len) {
  static const char* names[] = {"bf16", "fp8", "w4", "w8"};
  if (kind < 0 || kind > 3 || buf == nullptr || buf_len <= 0) return -1;
  if (kind == 1 && M <= fp8_swap_max_m() && M <= 64 && N >= 128)
    return snprintf(buf, (size_t)buf_len, "fp8 swap-AB bn=%d split_k=%d", M <= 32 ? 32 : 64, xb_gemm_fp8_split_k(M, N, K, sm_count));
  int bn = pick_block_n(M, N);
  if (kind >= 2 && N % 128 != 0) bn = 64;
  return snprintf(buf, (size_t)buf_len, "%s bn=%d", names[kind], bn);
}

extern "C" size_t xb_gemm_splitk_workspace_bytes(void) {
  // one wave of 132 CTAs (H100 SXM) x the largest token tile (64) is the most the heuristic asks for there; on a device with
  // more SMs a split that would not fit runs unsplit
  return kSplitKTicketBytes + (size_t)132 * 64 * kBlockM * sizeof(float);
}

extern "C" int xb_set_gemm_splitk_workspace(void* ws, size_t bytes) {
  if (ws != nullptr && (bytes <= kSplitKTicketBytes || (reinterpret_cast<uintptr_t>(ws) & 15) != 0)) {
    set_error("set_gemm_splitk_workspace: need a 16-byte aligned buffer of more than %zu bytes", kSplitKTicketBytes);
    return -1;
  }
  int dev = -1;
  if (ws != nullptr) {
    XB_CUDA_OK(cudaMemset(ws, 0, kSplitKTicketBytes));
    cudaPointerAttributes attr{};
    if (cudaPointerGetAttributes(&attr, ws) == cudaSuccess) dev = attr.device;
    else { cudaGetLastError(); cudaGetDevice(&dev); }
  }
  g_splitk_device.store(dev, std::memory_order_relaxed);
  g_splitk_ws.store(ws, std::memory_order_relaxed);
  g_splitk_bytes.store(ws ? bytes : 0, std::memory_order_relaxed);
  return 0;
}

extern "C" int xb_set_fp8_splitk_max(int max_split) {
  if (max_split < 1 || max_split > 32) {
    set_error("set_fp8_splitk_max: %d out of range (1 = never split .. 32)", max_split);
    return -1;
  }
  const int old = splitk_max();
  g_splitk_max.store(max_split, std::memory_order_relaxed);
  return old;
}

extern "C" int xb_set_fp8_swap_max_m(int max_m) {
  if (max_m < 0 || max_m > 64) {
    set_error("set_fp8_swap_max_m: %d out of range (0 = never swap .. 64)", max_m);
    return -1;
  }
  const int old = fp8_swap_max_m();
  g_fp8_swap_max_m.store(max_m, std::memory_order_relaxed);
  return old;
}

extern "C" int xb_gemm_bf16(void* c, int64_t ldc, const void* a, int64_t lda, const void* b, const void* bias, int M, int N,
                            int K, xb_stream_t stream) {
  if (M == 0 || N == 0) return 0;
  XB_CHECK(K % 8 == 0 && lda % 8 == 0, "gemm_bf16: K=%d and lda=%lld must be multiples of 8 (16-byte rows for TMA)", K,
           (long long)lda);
  XB_CHECK((reinterpret_cast<uintptr_t>(a) & 15) == 0 && (reinterpret_cast<uintptr_t>(b) & 15) == 0, "gemm_bf16: a/b alignment");
  GemmParams p{};
  p.c = reinterpret_cast<__nv_bfloat16*>(c);
  p.ldc = ldc;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.M = M; p.N = N; p.K = K;
  const int bn = pick_block_n(M, N);
  CUtensorMap ta, tb;
  if (make_tmap_2d(&ta, a, M, K, (uint64_t)lda * 2, kBlockM, 64, 2)) return 1;
  if (make_tmap_2d(&tb, b, N, K, (uint64_t)K * 2, bn, 64, 2)) return 1;
  return bn == 128 ? launch_gemm<kKindBF16, 128>(ta, tb, p, (cudaStream_t)stream)
                   : launch_gemm<kKindBF16, 64>(ta, tb, p, (cudaStream_t)stream);
}

extern "C" int xb_gemm_fp8_scaled(void* c, int64_t ldc, const void* a, int64_t lda, const void* b, const float* a_scale,
                                  int a_scale_numel, const float* b_scale, int b_scale_numel, const void* bias, int M, int N,
                                  int K, xb_stream_t stream) {
  if (M == 0 || N == 0) return 0;
  // same argument checks as cutlass_scaled_mm (scaled_mm_entry.cu:62-85)
  XB_CHECK(K % 16 == 0 && lda % 16 == 0, "cutlass_scaled_mm: K=%d / lda=%lld must be multiples of 16", K, (long long)lda);
  XB_CHECK(ldc % 8 == 0, "cutlass_scaled_mm: c.stride(0) %% 16 bytes != 0");
  XB_CHECK(a_scale_numel == 1 || a_scale_numel == M, "cutlass_scaled_mm: a_scales must have numel 1 or M");
  XB_CHECK(b_scale_numel == 1 || b_scale_numel == N, "cutlass_scaled_mm: b_scales must have numel 1 or N");
  GemmParams p{};
  p.c = reinterpret_cast<__nv_bfloat16*>(c);
  p.ldc = ldc;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.a_scale = a_scale; p.b_scale = b_scale;
  p.a_scale_per_row = a_scale_numel > 1; p.b_scale_per_col = b_scale_numel > 1;
  p.M = M; p.N = N; p.K = K;
  // decode-sized M: swap-AB (see GemmParams::swap_ab).  XB_FP8_SWAP_MAX_M: largest M that swaps (0 disables).
  if (M <= fp8_swap_max_m() && M <= 64 && N >= 128) {
    p.swap_ab = 1;
    p.M = N; p.N = M;
    p.a_scale = b_scale; p.b_scale = a_scale;          // per-row = channel scales, per-column = token scales
    p.a_scale_per_row = b_scale_numel > 1; p.b_scale_per_col = a_scale_numel > 1;
    {
      size_t need = 0;
      const int split = pick_split_k((N + kBlockM - 1) / kBlockM, (K + 127) / 128, M <= 32 ? 32 : 64, &need);
      if (split > 1) {
        uint8_t* ws = static_cast<uint8_t*>(g_splitk_ws.load(std::memory_order_relaxed));
        p.split_k = split;
        p.splitk_tickets = reinterpret_cast<unsigned int*>(ws);
        p.splitk_ws = reinterpret_cast<float*>(ws + kSplitKTicketBytes);
      }
    }
    CUtensorMap tw, tx;
    if (make_tmap_fp8(&tw, b, N, K, (uint64_t)K, kBlockM)) return 1;
    if (M <= 32) {
      if (make_tmap_fp8(&tx, a, M, K, (uint64_t)lda, 32)) return 1;
      return launch_gemm<kKindFP8, 32>(tw, tx, p, (cudaStream_t)stream);
    }
    if (make_tmap_fp8(&tx, a, M, K, (uint64_t)lda, 64)) return 1;
    return launch_gemm<kKindFP8, 64>(tw, tx, p, (cudaStream_t)stream);
  }
  const int bn = pick_block_n(M, N);
  CUtensorMap ta, tb;
  if (make_tmap_fp8(&ta, a, M, K, (uint64_t)lda, kBlockM)) return 1;
  if (make_tmap_fp8(&tb, b, N, K, (uint64_t)K, bn)) return 1;
  return bn == 128 ? launch_gemm<kKindFP8, 128>(ta, tb, p, (cudaStream_t)stream)
                   : launch_gemm<kKindFP8, 64>(ta, tb, p, (cudaStream_t)stream);
}

extern "C" int xb_gemm_w4a16(void* c, int64_t ldc, const void* a, int64_t lda, const uint32_t* qweight, const uint32_t* meta,
                             const void* bias, int M, int N, int K, int group_size, xb_stream_t stream) {
  if (M == 0 || N == 0) return 0;
  XB_CHECK(N % 64 == 0 && K % 64 == 0, "gemm_w4a16: N=%d and K=%d must be multiples of 64", N, K);
  XB_CHECK(group_size >= 64 && group_size % 64 == 0 && K % group_size == 0,
           "gemm_w4a16: group_size %d must be a multiple of 64 dividing K=%d", group_size, K);
  const int tpg = group_size / 64;
  XB_CHECK((tpg & (tpg - 1)) == 0, "gemm_w4a16: group_size/64 must be a power of two (got %d)", group_size);
  XB_CHECK(lda % 8 == 0 && (reinterpret_cast<uintptr_t>(a) & 15) == 0, "gemm_w4a16: a alignment");
  GemmParams p{};
  p.c = reinterpret_cast<__nv_bfloat16*>(c);
  p.ldc = ldc;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.gshift = 0;
  while ((1 << p.gshift) < tpg) ++p.gshift;
  p.M = M; p.N = N; p.K = K;
  const int bn = N % 128 == 0 ? pick_block_n(M, N) : 64;
  CUtensorMap ta, tb, tm;
  if (make_tmap_2d(&ta, a, M, K, (uint64_t)lda * 2, kBlockM, 64, 2)) return 1;
  const uint64_t ktiles = K / 64;
  if (make_tmap_2d_raw(&tb, qweight, CU_TENSOR_MAP_DATA_TYPE_UINT32, N / 16, ktiles * 128, ktiles * 512, bn / 16, 128,
                       CU_TENSOR_MAP_SWIZZLE_NONE))
    return 1;
  if (make_tmap_2d_raw(&tm, meta, CU_TENSOR_MAP_DATA_TYPE_UINT32, K / group_size, N, (uint64_t)N * 4, 1, bn,
                       CU_TENSOR_MAP_SWIZZLE_NONE))
    return 1;
  return bn == 128 ? launch_gemm<kKindW4, 128>(ta, tb, p, (cudaStream_t)stream, &tm)
                   : launch_gemm<kKindW4, 64>(ta, tb, p, (cudaStream_t)stream, &tm);
}

// kind W8: B is the tile-packed int8 weight of linear_q8_small_m.cu ([N/16][K/64][32 lanes][8 words]); same pipeline as W4
// with a 1 KB packed row tile per k64 step and the int8 converter (w8_dequant_word).
extern "C" int xb_gemm_w8a16(void* c, int64_t ldc, const void* a, int64_t lda, const uint32_t* qweight, const uint32_t* meta,
                             const void* bias, int M, int N, int K, int group_size, xb_stream_t stream) {
  if (M == 0 || N == 0) return 0;
  XB_CHECK(N % 64 == 0 && K % 64 == 0, "gemm_w8a16: N=%d and K=%d must be multiples of 64", N, K);
  XB_CHECK(group_size >= 64 && group_size % 64 == 0 && K % group_size == 0,
           "gemm_w8a16: group_size %d must be a multiple of 64 dividing K=%d", group_size, K);
  const int tpg = group_size / 64;
  XB_CHECK((tpg & (tpg - 1)) == 0, "gemm_w8a16: group_size/64 must be a power of two (got %d)", group_size);
  XB_CHECK(lda % 8 == 0 && (reinterpret_cast<uintptr_t>(a) & 15) == 0, "gemm_w8a16: a alignment");
  GemmParams p{};
  p.c = reinterpret_cast<__nv_bfloat16*>(c);
  p.ldc = ldc;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.gshift = 0;
  while ((1 << p.gshift) < tpg) ++p.gshift;
  p.M = M; p.N = N; p.K = K;
  const int bn = N % 128 == 0 ? pick_block_n(M, N) : 64;
  CUtensorMap ta, tb, tm;
  if (make_tmap_2d(&ta, a, M, K, (uint64_t)lda * 2, kBlockM, 64, 2)) return 1;
  const uint64_t ktiles = K / 64;
  if (make_tmap_2d_raw(&tb, qweight, CU_TENSOR_MAP_DATA_TYPE_UINT32, N / 16, ktiles * 256, ktiles * 1024, bn / 16, 256,
                       CU_TENSOR_MAP_SWIZZLE_NONE))
    return 1;
  if (make_tmap_2d_raw(&tm, meta, CU_TENSOR_MAP_DATA_TYPE_UINT32, K / group_size, N, (uint64_t)N * 4, 1, bn,
                       CU_TENSOR_MAP_SWIZZLE_NONE))
    return 1;
  return bn == 128 ? launch_gemm<kKindW8, 128>(ta, tb, p, (cudaStream_t)stream, &tm)
                   : launch_gemm<kKindW8, 64>(ta, tb, p, (cudaStream_t)stream, &tm);
}
