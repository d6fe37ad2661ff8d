// Prefill / chunked-prefill attention on wgmma tensor cores with TMA staging.
// Replaces the FlashInfer fa2 (mma.sync) modules the reference dlopen()s:
//   ragged_run  - xllm::kernel::cuda::batch_prefill          (kernels/cuda/batch_prefill.cpp:21-163): contiguous ragged q/k/v
//   paged_run   - xllm::kernel::cuda::batch_chunked_prefill  (kernels/cuda/batch_chunked_prefill.cpp:26-92): ragged q over the
//                 paged KV cache (chunked prefill with causal offset; also "decode on tensor cores", causal = false)
//
// One CTA per (q tile, kv head, request).  A q tile packs (token, head-of-the-GQA-group) pairs into 128 rows
// (tokens_per_tile = 128 / group), so every K/V tile is fetched once per kv head for the whole group.
//   warp 0      TMA producer: Q tile once (3-D tensor map token x head x d), then K and V tiles through 2-stage rings.
//               Paged KV: one 2-D TMA per page fragment, the row coordinate comes from the page table.
//   warps 4..11 two consumer warpgroups, warpgroup g owns rows 64 g .. 64 g + 63 of the tile:
//               S = Q K^T (wgmma m64 x 128 x 16, both operands K-major in smem, fp32 in registers), base-2 online
//               softmax (sm_scale*log2e folded; causal / length mask only on tiles that need it), P rounded to bf16
//               (denominator summed from the ROUNDED P like the reference ladder) and kept in registers as the A operand
//               of O += P V (V straight from its [kv, d] TMA tile as an MN-major operand - no transpose pass), final
//               O / l -> bf16 -> global.
// kDQK != kDV (192 / 128: expanded MLA prefill, group 1, ragged, kv_splits 1): Q [T, H, 192] is three 64-column sub-tiles;
// a K tile is two 64-column sub-tiles of k_nope from tmap_k at column kvh * kv_head_stride plus one sub-tile of k_pe from
// tmap_kr at column kvh * kr_head_stride (0: one k_pe row shared by all heads); a V tile is two sub-tiles from tmap_v at
// column kvh * kv_head_stride + v_col_off.  So k_nope and v are read as strided views of the up-projection [N, H, 256].
#include <type_traits>

#include "tc_common.cuh"

namespace xb {
namespace tc {

struct PrefillParams {
  const int32_t* qo_indptr;
  const int32_t* kv_indptr;        // paged: page indptr; ragged: kv_cu_seq_lens
  const int32_t* kv_indices;       // paged only
  const int32_t* kv_last_page_len; // paged only
  int paged, page_size;
  __nv_bfloat16* o;
  int64_t o_stride_n, o_stride_h;
  float* lse;                      // [T, Hq] base-2, optional
  float scale_log2;
  int num_qo_heads, num_kv_heads, group, tokens_per_tile, causal;
  int box_rows;                    // kv rows per TMA load (min(page_size, 128) or 128 for ragged)
  // split-KV (short q over a long KV: chunked prefill of a small chunk, flashinfer_planinfo.cpp:168-247 split_kv): the kv
  // tiles of a work item are divided over kv_splits CTAs (blockIdx.z = request * kv_splits + split); each writes a
  // normalised fp32 partial + base-2 LSE, prefill_merge_kernel combines them.  kv_splits == 1: direct output.
  int kv_splits;
  float* part_o;                   // [kv_splits][total_q][Hq][D]
  float* part_lse;                 // [kv_splits][total_q][Hq]
  int64_t total_q;
};

// kDQK != kDV only: column offsets (elements) of a head's K / V parts, see the header comment
struct KvColumns {
  int kv_head_stride, v_col_off, kr_head_stride;
};

constexpr int kKT = 128;   // kv tile
constexpr int kPrefillThreads = 384;

template <int kDQK, int kDV>
struct PrefillCfg {
  static constexpr int kHalves = kDQK / 64;                        // sub-tiles of a Q or K tile
  static constexpr int kVHalves = kDV / 64;
  static constexpr int kSub = 128 * 128;                           // one [128 rows x 64 elems] swizzled sub-tile
  static constexpr int kQBytes = kHalves * kSub;
  static constexpr int kKBytes = kHalves * kSub;
  static constexpr int kVBytes = kVHalves * kSub;
  static constexpr int kSmemBytes = kQBytes + 2 * kKBytes + 2 * kVBytes + 1024 + 256;
};

// tmap_kr (the shared k_pe rows) and kc are read only when kDQK != kDV.  They follow p, and PrefillParams keeps its
// layout, so the kDQK == kDV instantiations compile to the code they had before the 192 / 128 variant existed.
template <int kDQK, int kDV>
__global__ void __launch_bounds__(kPrefillThreads, 1)
prefill_attention_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                         const __grid_constant__ CUtensorMap tmap_v, const PrefillParams p,
                         const __grid_constant__ CUtensorMap tmap_kr, const KvColumns kc) {
  static_assert((kDQK == 64 && kDV == 64) || (kDQK == 128 && kDV == 128) || (kDQK == 192 && kDV == 128),
                "prefill attention: QK / V widths 64 / 64, 128 / 128 or 192 / 128");
  using Cfg = PrefillCfg<kDQK, kDV>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* q_s = smem;
  uint8_t* k_s = q_s + Cfg::kQBytes;                // [2][kKBytes]
  uint8_t* v_s = k_s + 2 * Cfg::kKBytes;            // [2][kVBytes]
  uint64_t* bars = reinterpret_cast<uint64_t*>(v_s + 2 * Cfg::kVBytes);
  uint64_t* q_full = bars;            // 1
  uint64_t* k_full = bars + 1;        // 2
  uint64_t* k_empty = bars + 3;       // 2
  uint64_t* v_full = bars + 5;        // 2
  uint64_t* v_empty = bars + 7;       // 2

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.z / p.kv_splits, split = blockIdx.z - b * p.kv_splits, kvh = blockIdx.y;
  const int ti = gridDim.x - 1 - blockIdx.x;          // heavy (late, causal) tiles first

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(k_full + i, 1);
      mbar_init(k_empty + i, 8);      // one arrive per consumer warp
      mbar_init(v_full + i, 1);
      mbar_init(v_empty + i, 8);
    }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    if constexpr (kDQK != kDV) tma_prefetch_desc(&tmap_kr);
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  // ---- work item geometry (uniform across the CTA) ------------------------------------------------------------
  const int q0 = __ldg(p.qo_indptr + b);
  const int qo_len = __ldg(p.qo_indptr + b + 1) - q0;
  const int tq0 = ti * p.tokens_per_tile;              // first q token of this tile (request-local)
  int kv_len, kv_base = 0, indptr0 = 0, n_pages = 0;
  if (p.paged) {
    indptr0 = __ldg(p.kv_indptr + b);
    n_pages = __ldg(p.kv_indptr + b + 1) - indptr0;
    kv_len = n_pages > 0 ? (n_pages - 1) * p.page_size + __ldg(p.kv_last_page_len + b) : 0;
  } else {
    kv_base = __ldg(p.kv_indptr + b);
    kv_len = __ldg(p.kv_indptr + b + 1) - kv_base;
  }
  const bool live = tq0 < qo_len;
  const int tq_last = min(qo_len, tq0 + p.tokens_per_tile) - 1;
  const int kv_off = kv_len - qo_len;                  // causal offset of chunked prefill (prefill.cuh:1017 semantics)
  int kv_limit = p.causal ? min(kv_len, tq_last + kv_off + 1) : kv_len;
  if (kv_limit < 0) kv_limit = 0;
  const int n_tiles_all = live ? (kv_limit + kKT - 1) / kKT : 0;
  // this CTA's share of the kv tiles; j below counts LOCAL tiles (ring phases), j0 + j is the kv tile
  const int per_split = (n_tiles_all + p.kv_splits - 1) / p.kv_splits;
  const int j0 = split * per_split;
  const int n_tiles = max(0, min(per_split, n_tiles_all - j0));
  const int rows_used = p.tokens_per_tile * p.group;

  // 192 / 128: the consumers' 128 fp32 accumulators and the wider Q / K addressing do not fit the 168 registers that
  // __launch_bounds__(384, 1) leaves (65536 / 384, rounded down to 8), so warpgroup 0, which only issues TMA, hands
  // registers to the two consumer warpgroups: 128 x 40 + 256 x 232 = 384 x 168.
  if (warp == 0) {
    if constexpr (kDQK != kDV) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    // ============================== TMA producer ==============================
    if (lane == 0 && n_tiles > 0) {
      mbar_expect_tx(q_full, rows_used * kDQK * 2);
#pragma unroll
      for (int h = 0; h < Cfg::kHalves; ++h)
        tma_load_3d(q_s + h * Cfg::kSub, &tmap_q, q_full, h * 64, kvh * p.group, q0 + tq0);
      const int loads = kKT / p.box_rows;
      for (int j = 0; j < n_tiles; ++j) {
        const int st = j & 1;
        const uint32_t par = ((j >> 1) & 1) ^ 1;
        if constexpr (kDQK == kDV) {
          for (int kv = 0; kv < 2; ++kv) {           // kv = 0: K tile, 1: V tile
            uint64_t* full = kv ? v_full + st : k_full + st;
            mbar_wait(kv ? v_empty + st : k_empty + st, par);
            mbar_expect_tx(full, kKT * kDQK * 2);
            uint8_t* dst = (kv ? v_s : k_s) + st * Cfg::kKBytes;
            const CUtensorMap* map = kv ? &tmap_v : &tmap_k;
            for (int i = 0; i < loads; ++i) {
              const int t0 = (j0 + j) * kKT + i * p.box_rows;
              int row;
              if (p.paged) {
                int pg = t0 / p.page_size;
                if (pg >= n_pages) pg = n_pages - 1;    // beyond the request: masked anyway, keep the address valid
                row = __ldg(p.kv_indices + indptr0 + pg) * p.page_size + (t0 % p.page_size);
              } else {
                row = kv_base + t0;
              }
#pragma unroll
              for (int h = 0; h < Cfg::kHalves; ++h)
                tma_load_2d(dst + h * Cfg::kSub + i * p.box_rows * 128, map, full, kvh * kDQK + h * 64, row);
            }
          }
        } else {                                     // ragged, one 128-row box per sub-tile
          const int row = kv_base + (j0 + j) * kKT;
          mbar_wait(k_empty + st, par);
          mbar_expect_tx(k_full + st, kKT * kDQK * 2);
          uint8_t* dst = k_s + st * Cfg::kKBytes;
#pragma unroll
          for (int h = 0; h < Cfg::kHalves - 1; ++h)     // k_nope, then the 64 k_pe columns as the last sub-tile
            tma_load_2d(dst + h * Cfg::kSub, &tmap_k, k_full + st, kvh * kc.kv_head_stride + h * 64, row);
          tma_load_2d(dst + (Cfg::kHalves - 1) * Cfg::kSub, &tmap_kr, k_full + st, kvh * kc.kr_head_stride, row);
          mbar_wait(v_empty + st, par);
          mbar_expect_tx(v_full + st, kKT * kDV * 2);
          dst = v_s + st * Cfg::kVBytes;
#pragma unroll
          for (int h = 0; h < Cfg::kVHalves; ++h)
            tma_load_2d(dst + h * Cfg::kSub, &tmap_v, v_full + st, kvh * kc.kv_head_stride + kc.v_col_off + h * 64, row);
        }
      }
    }
  } else if (warp >= 4) {
    if constexpr (kDQK != kDV) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    // ============================== consumers: S, softmax, O ==============================
    // thread (warp w of warpgroup g, lane l) holds rows rr[h] = 64 g + 16 w + l / 4 + 8 h (h = 0, 1) and columns
    // 8 j + 2 (l % 4) + e of every accumulator (tc_common.cuh fragment layout)
    const int wg = (warp - 4) >> 2, wq = warp & 3;
    const int cq = 2 * (lane & 3);
    int my_lim[2];
    bool row_valid[2];
    int q_idx[2], head_local[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
      const int tok_local = r / p.group;
      head_local[h] = r - tok_local * p.group;
      q_idx[h] = tq0 + tok_local;
      row_valid[h] = live && r < rows_used && q_idx[h] < qo_len;
      my_lim[h] = p.causal ? min(kv_len, q_idx[h] + kv_off + 1) : kv_len;        // #visible keys of the row
    }
    const int lim_first = p.causal ? min(kv_len, tq0 + kv_off + 1) : kv_len;      // smallest limit in the tile
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};            // l_run: this thread's columns only
    float o[kDV / 2];
#pragma unroll
    for (int i = 0; i < kDV / 2; ++i) o[i] = 0.f;
    float s[kKT / 2];
    if (n_tiles > 0) mbar_wait(q_full, 0);

    for (int j = 0; j < n_tiles; ++j) {
      const int st = j & 1;
      const uint32_t par = (j >> 1) & 1;
      // ---- S = Q K^T ----
      mbar_wait(k_full + st, par);
      {
        const uint32_t qa = smem_u32(q_s) + wg * 64 * 128, ka = smem_u32(k_s + st * Cfg::kKBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kDQK / 16; ++k) {
          const uint32_t off = (k >> 2) * Cfg::kSub + (k & 3) * 32;
          wgmma_bf16<kKT>(s, gmma_desc_sw128(qa + off), gmma_desc_sw128(ka + off), k > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(s);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(k_empty + st);
      const bool need_mask = (j0 + j + 1) * kKT > lim_first;
      // ---- online softmax (the four lanes of a row reduce with shuffles) ----
      float alpha[2], m_safe[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int col_lim = my_lim[h] - (j0 + j) * kKT;      // columns >= col_lim are masked
        float mx = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < kKT / 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float v = s[4 * jj + 2 * h + e];
            mx = fmaxf(mx, (!need_mask || 8 * jj + cq + e < col_lim) ? v : -INFINITY);
          }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run[h], mx * p.scale_log2);
        m_safe[h] = m_new == -INFINITY ? 0.f : m_new;
        alpha[h] = fast_exp2(m_run[h] - m_safe[h]);
        m_run[h] = m_new;
        float psum = 0.f;
#pragma unroll
        for (int jj = 0; jj < kKT / 8; ++jj) {
          const int i0 = 4 * jj + 2 * h;
          float p0 = fast_exp2(s[i0] * p.scale_log2 - m_safe[h]);
          float p1 = fast_exp2(s[i0 + 1] * p.scale_log2 - m_safe[h]);
          if (need_mask) {
            if (8 * jj + cq >= col_lim) p0 = 0.f;
            if (8 * jj + cq + 1 >= col_lim) p1 = 0.f;
          }
          const uint32_t pp = pack_bf16x2(p0, p1);
          s[i0] = __uint_as_float(pp);                 // the bf16 pair, as the A fragment of P V below
          psum += bf16lo(pp) + bf16hi(pp);             // denominator from the ROUNDED P (reference ladder)
        }
        l_run[h] = l_run[h] * alpha[h] + psum;
      }
#pragma unroll
      for (int jj = 0; jj < kDV / 8; ++jj)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          o[4 * jj + 2 * h] *= alpha[h];
          o[4 * jj + 2 * h + 1] *= alpha[h];
        }
      // ---- O += P V: A fragment of k step kk = S columns 16 kk .. 16 kk + 15 (rows h = 0, 1; column halves 0, 1) ----
      mbar_wait(v_full + st, par);
      {
        const uint32_t va = smem_u32(v_s + st * Cfg::kVBytes);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kKT / 16; ++kk) {
          const uint32_t a[4] = {__float_as_uint(s[8 * kk + 0]), __float_as_uint(s[8 * kk + 2]), __float_as_uint(s[8 * kk + 4]),
                                 __float_as_uint(s[8 * kk + 6])};
          wgmma_bf16_rs_tb<kDV>(o, a, gmma_desc_sw128_mn(va + kk * 2048, Cfg::kSub, 1024), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(o);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(v_empty + st);
    }
    // ---- epilogue: O / l -> bf16 -> global ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float l = l_run[h];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      if (!row_valid[h]) continue;
      const float inv = l > 0.f ? 1.0f / l : 0.f;
      const int64_t tq = q0 + q_idx[h];
      const int head = kvh * p.group + head_local[h];
      const float lse2 = l > 0.f ? m_run[h] + log2f(l) : -INFINITY;
      if (p.kv_splits == 1) {
        __nv_bfloat16* dst = p.o + tq * p.o_stride_n + (int64_t)head * p.o_stride_h;
        if (p.lse && (lane & 3) == 0) p.lse[tq * p.num_qo_heads + head] = lse2;
#pragma unroll
        for (int jj = 0; jj < kDV / 8; ++jj)
          *reinterpret_cast<uint32_t*>(dst + 8 * jj + cq) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
      } else {
        const int64_t slot = ((int64_t)split * p.total_q + tq) * p.num_qo_heads + head;
        float* pdst = p.part_o + slot * kDV;
        if ((lane & 3) == 0) p.part_lse[slot] = lse2;
#pragma unroll
        for (int jj = 0; jj < kDV / 8; ++jj)
          *reinterpret_cast<float2*>(pdst + 8 * jj + cq) = make_float2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
      }
    }
  } else if constexpr (kDQK != kDV) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");   // warps 1..3 of warpgroup 0
  }
}

// Combines the kv_splits partials of every (q row, head): weights 2^(lse_s - max) / sum, fixed split order.
__global__ void __launch_bounds__(128)
prefill_merge_kernel(const PrefillParams p, int head_dim) {
  const int64_t tq = blockIdx.x;
  const int head = blockIdx.y;
  pdl_launch_dependents();
  pdl_wait();
  float mx = -INFINITY;
  for (int s = 0; s < p.kv_splits; ++s) mx = fmaxf(mx, p.part_lse[((int64_t)s * p.total_q + tq) * p.num_qo_heads + head]);
  const float m_safe = mx == -INFINITY ? 0.f : mx;
  float wsum = 0.f;
  for (int s = 0; s < p.kv_splits; ++s) wsum += fast_exp2(p.part_lse[((int64_t)s * p.total_q + tq) * p.num_qo_heads + head] - m_safe);
  const float inv = wsum > 0.f ? 1.0f / wsum : 0.f;
  for (int d = threadIdx.x; d < head_dim; d += blockDim.x) {
    float acc = 0.f;
    for (int s = 0; s < p.kv_splits; ++s) {
      const int64_t slot = ((int64_t)s * p.total_q + tq) * p.num_qo_heads + head;
      acc += p.part_o[slot * head_dim + d] * fast_exp2(p.part_lse[slot] - m_safe);
    }
    p.o[tq * p.o_stride_n + (int64_t)head * p.o_stride_h + d] = __float2bfloat16_rn(acc * inv);
  }
  if (p.lse && threadIdx.x == 0) p.lse[tq * p.num_qo_heads + head] = wsum > 0.f ? mx + log2f(wsum) : -INFINITY;
}

template <int kDQK, int kDV>
static int launch_prefill(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const PrefillParams& p,
                          int batch, int q_tiles, cudaStream_t stream, const CUtensorMap& tkr = {},
                          const KvColumns& kc = {}) {
  using Cfg = PrefillCfg<kDQK, kDV>;
  constexpr auto kern = prefill_attention_kernel<kDQK, kDV>;
  XB_CUDA_OK(set_max_dynamic_smem_once<kern>(Cfg::kSmemBytes));
  dim3 grid(q_tiles, p.num_kv_heads, batch * p.kv_splits), block(kPrefillThreads);
  XB_CUDA_OK(launch(kern, grid, block, (size_t)Cfg::kSmemBytes, stream, true, tq, tk, tv, p, tkr, kc));
  if (p.kv_splits > 1)
    XB_CUDA_OK(launch(prefill_merge_kernel, dim3((unsigned)p.total_q, p.num_qo_heads), dim3(kDV < 128 ? kDV : 128), 0, stream, true, p, kDV));
  return 0;
}
}  // namespace tc
}  // namespace xb

using namespace xb;
using namespace xb::tc;

// Shared host path of ragged_run / paged_run.
static int prefill_common(const void* q, int64_t q_stride_n, int64_t q_stride_h, int64_t total_q, const void* k,
                          const void* v, int64_t kv_rows, int64_t kv_row_stride, int paged, int page_size,
                          const int32_t* qo_indptr, const int32_t* kv_indptr, const int32_t* kv_indices,
                          const int32_t* kv_last_page_len, void* o, int64_t o_stride_n, int64_t o_stride_h, float* lse,
                          int batch, int max_qo_len, int num_qo_heads, int num_kv_heads, int head_dim, int causal,
                          float sm_scale, cudaStream_t stream, int kv_splits = 1, void* workspace_f32 = nullptr,
                          int64_t workspace_bytes = 0) {
  if (batch == 0 || total_q == 0 || max_qo_len == 0) return 0;
  XB_CHECK(kv_splits >= 1 && kv_splits <= 64, "prefill attention: kv_splits %d out of range (1..64)", kv_splits);
  if (kv_splits > 1) {
    const int64_t need = (int64_t)kv_splits * total_q * num_qo_heads * (head_dim + 1) * 4;
    XB_CHECK(workspace_f32 != nullptr && workspace_bytes >= need && (reinterpret_cast<uintptr_t>(workspace_f32) & 15) == 0,
             "prefill attention: split-KV needs a 16-byte aligned float workspace of %lld bytes (got %lld)", (long long)need,
             (long long)workspace_bytes);
  }
  XB_CHECK(head_dim == 64 || head_dim == 128, "prefill attention: head_dim %d unsupported (64|128)", head_dim);
  XB_CHECK(num_kv_heads > 0 && num_qo_heads % num_kv_heads == 0, "prefill attention: bad head counts %d/%d", num_qo_heads,
           num_kv_heads);
  const int group = num_qo_heads / num_kv_heads;
  XB_CHECK(group <= 128, "prefill attention: GQA group %d > 128", group);
  XB_CHECK(q_stride_h == head_dim, "prefill attention: q heads must be contiguous (stride %lld)", (long long)q_stride_h);
  XB_CHECK(q_stride_n % 8 == 0 && kv_row_stride % 8 == 0 && o_stride_n % 8 == 0 && o_stride_h % 8 == 0,
           "prefill attention: strides must keep 16-byte alignment");
  XB_CHECK(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
             reinterpret_cast<uintptr_t>(o)) & 15) == 0, "prefill attention: pointers must be 16-byte aligned");
  PrefillParams p{};
  p.qo_indptr = qo_indptr;
  p.kv_indptr = kv_indptr;
  p.kv_indices = kv_indices;
  p.kv_last_page_len = kv_last_page_len;
  p.paged = paged;
  p.page_size = page_size;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.o_stride_n = o_stride_n;
  p.o_stride_h = o_stride_h;
  p.lse = lse;
  p.scale_log2 = sm_scale * 1.44269504088896340736f;
  p.num_qo_heads = num_qo_heads;
  p.num_kv_heads = num_kv_heads;
  p.group = group;
  p.tokens_per_tile = 128 / group;
  p.causal = causal;
  p.kv_splits = kv_splits;
  p.total_q = total_q;
  p.part_o = reinterpret_cast<float*>(workspace_f32);
  p.part_lse = p.part_o ? p.part_o + (int64_t)kv_splits * total_q * num_qo_heads * head_dim : nullptr;
  if (paged) {
    XB_CHECK(page_size > 0 && ((page_size <= 128 && 128 % page_size == 0) || page_size % 128 == 0),
             "prefill attention: page_size %d must divide 128 or be a multiple of it", page_size);
    p.box_rows = page_size < 128 ? page_size : 128;
  } else {
    p.box_rows = 128;
  }
  CUtensorMap tq, tk, tv;
  if (make_tmap_3d_bf16(&tq, q, head_dim, num_qo_heads, total_q, (uint64_t)q_stride_h * 2, (uint64_t)q_stride_n * 2, 64,
                        group, p.tokens_per_tile))
    return 1;
  if (make_tmap_2d(&tk, k, kv_rows, (uint64_t)num_kv_heads * head_dim, (uint64_t)kv_row_stride * 2, p.box_rows, 64, 2)) return 1;
  if (make_tmap_2d(&tv, v, kv_rows, (uint64_t)num_kv_heads * head_dim, (uint64_t)kv_row_stride * 2, p.box_rows, 64, 2)) return 1;
  const int q_tiles = (max_qo_len + p.tokens_per_tile - 1) / p.tokens_per_tile;
  return head_dim == 128 ? launch_prefill<128, 128>(tq, tk, tv, p, batch, q_tiles, stream)
                         : launch_prefill<64, 64>(tq, tk, tv, p, batch, q_tiles, stream);
}

// Expanded MLA prefill attention (ragged, causal, group 1, kv_splits 1): q [total_q, H, 192] (row / head strides),
// kv_up [total_kv, H, 256] contiguous = per head [k_nope 128 | v 128], kpe [total_kv, 64] contiguous (one k_pe row per kv
// token, shared by all heads), kv_cu_seq_lens [batch + 1] on the device; o [T, H, 128].
int xb::mla_expanded_attention(const void* q, int64_t q_stride_n, int64_t q_stride_h, int64_t total_q, const void* kv_up,
                               const void* kpe, int64_t total_kv, const int32_t* qo_indptr, const int32_t* kv_cu_seq_lens,
                               void* o, int64_t o_stride_n, int64_t o_stride_h, int batch, int max_qo_len, int num_heads,
                               float sm_scale, cudaStream_t stream) {
  constexpr int kDQK = 192, kDV = 128, kKvW = 256;
  if (batch == 0 || total_q == 0 || max_qo_len == 0) return 0;
  PrefillParams p{};
  p.qo_indptr = qo_indptr;
  p.kv_indptr = kv_cu_seq_lens;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.o_stride_n = o_stride_n;
  p.o_stride_h = o_stride_h;
  p.scale_log2 = sm_scale * 1.44269504088896340736f;
  p.num_qo_heads = num_heads;
  p.num_kv_heads = num_heads;
  p.group = 1;
  p.tokens_per_tile = 128;
  p.causal = 1;
  p.kv_splits = 1;
  p.total_q = total_q;
  p.box_rows = 128;
  CUtensorMap tq, tk, tkr;
  if (make_tmap_3d_bf16(&tq, q, kDQK, num_heads, total_q, (uint64_t)q_stride_h * 2, (uint64_t)q_stride_n * 2, 64, 1, 128))
    return 1;
  if (make_tmap_2d(&tk, kv_up, total_kv, (uint64_t)num_heads * kKvW, (uint64_t)num_heads * kKvW * 2, 128, 64, 2)) return 1;
  if (make_tmap_2d(&tkr, kpe, total_kv, 64, 128, 128, 64, 2)) return 1;
  const int q_tiles = (max_qo_len + 127) / 128;
  // k_nope at column 256 h, v at 256 h + 128 of the same rows; one k_pe row for every head
  return launch_prefill<kDQK, kDV>(tq, tk, tk, p, batch, q_tiles, stream, tkr, KvColumns{kKvW, kDV, 0});
}

extern "C" int xb_prefill_ragged_bf16(const void* q, int64_t q_stride_n, int64_t q_stride_h, const void* k, const void* v,
                                      int64_t kv_stride_n, const int32_t* q_cu_seq_lens, const int32_t* kv_cu_seq_lens,
                                      void* o, int64_t o_stride_n, int64_t o_stride_h, float* lse, int batch,
                                      int64_t total_q, int64_t total_kv, int max_qo_len, int num_qo_heads, int num_kv_heads,
                                      int head_dim, int causal, float sm_scale, xb_stream_t stream) {
  return prefill_common(q, q_stride_n, q_stride_h, total_q, k, v, total_kv, kv_stride_n, 0, 1, q_cu_seq_lens, kv_cu_seq_lens,
                        nullptr, nullptr, o, o_stride_n, o_stride_h, lse, batch, max_qo_len, num_qo_heads, num_kv_heads,
                        head_dim, causal, sm_scale, (cudaStream_t)stream);
}

extern "C" int xb_prefill_paged_bf16(const void* q, int64_t q_stride_n, int64_t q_stride_h, const void* k_cache,
                                     const void* v_cache, int64_t num_pages, int page_size, const int32_t* qo_indptr,
                                     const int32_t* kv_indptr, const int32_t* kv_indices, const int32_t* kv_last_page_len,
                                     void* o, int64_t o_stride_n, int64_t o_stride_h, float* lse, int batch, int64_t total_q,
                                     int max_qo_len, int num_qo_heads, int num_kv_heads, int head_dim, int causal,
                                     float sm_scale, xb_stream_t stream) {
  // NHD cache [pages, page_size, Hkv, D] contiguous: a 2-D [pages*page_size, Hkv*D] row tensor
  return prefill_common(q, q_stride_n, q_stride_h, total_q, k_cache, v_cache, num_pages * page_size,
                        (int64_t)num_kv_heads * head_dim, 1, page_size, qo_indptr, kv_indptr, kv_indices, kv_last_page_len, o,
                        o_stride_n, o_stride_h, lse, batch, max_qo_len, num_qo_heads, num_kv_heads, head_dim, causal, sm_scale,
                        (cudaStream_t)stream);
}

// paged_run with the KV range of every work item divided over kv_splits CTAs (chunked prefill of a short chunk over a
// long history: flashinfer_planinfo.cpp:168-247 decides split_kv; kernels/cuda/batch_chunked_prefill.cpp:63-91 runs it).
// workspace_f32: kv_splits * total_q * num_qo_heads * (head_dim + 1) floats (xb_prefill_split_workspace_bytes).
extern "C" int xb_prefill_paged_split_bf16(const void* q, int64_t q_stride_n, int64_t q_stride_h, const void* k_cache,
                                           const void* v_cache, int64_t num_pages, int page_size, const int32_t* qo_indptr,
                                           const int32_t* kv_indptr, const int32_t* kv_indices,
                                           const int32_t* kv_last_page_len, void* o, int64_t o_stride_n, int64_t o_stride_h,
                                           float* lse, int batch, int64_t total_q, int max_qo_len, int num_qo_heads,
                                           int num_kv_heads, int head_dim, int causal, float sm_scale, int kv_splits,
                                           void* workspace_f32, int64_t workspace_bytes, xb_stream_t stream) {
  return prefill_common(q, q_stride_n, q_stride_h, total_q, k_cache, v_cache, num_pages * page_size,
                        (int64_t)num_kv_heads * head_dim, 1, page_size, qo_indptr, kv_indptr, kv_indices, kv_last_page_len, o,
                        o_stride_n, o_stride_h, lse, batch, max_qo_len, num_qo_heads, num_kv_heads, head_dim, causal, sm_scale,
                        (cudaStream_t)stream, kv_splits, workspace_f32, workspace_bytes);
}

extern "C" int64_t xb_prefill_split_workspace_bytes(int kv_splits, int64_t total_q, int num_qo_heads, int head_dim) {
  return kv_splits > 1 ? (int64_t)kv_splits * total_q * num_qo_heads * (head_dim + 1) * 4 : 0;
}

// Host-side split decision (pure arithmetic): how many KV splits make a short-q / long-kv batch fill the SMs.
// grid = q tiles x kv heads x requests CTAs; split only when that leaves more than half of the SMs idle and the longest
// KV spans several 128-token tiles; never more splits than 512-token pieces of the longest KV.
extern "C" int xb_prefill_plan_splits(int batch, int max_qo_len, int64_t max_kv_len, int num_qo_heads, int num_kv_heads,
                                      int num_sms) {
  if (batch <= 0 || max_qo_len <= 0 || num_kv_heads <= 0 || num_qo_heads % num_kv_heads != 0) return 1;
  if (num_sms <= 0) num_sms = 132;
  const int group = num_qo_heads / num_kv_heads;
  const int tokens_per_tile = group <= 128 ? 128 / group : 1;
  const int64_t q_tiles = (max_qo_len + tokens_per_tile - 1) / tokens_per_tile;
  const int64_t grid = q_tiles * num_kv_heads * batch;
  if (grid * 2 > num_sms || max_kv_len < 1024) return 1;
  int64_t splits = num_sms / grid;
  const int64_t by_len = (max_kv_len + 511) / 512;
  if (splits > by_len) splits = by_len;
  if (splits > 32) splits = 32;
  return splits < 1 ? 1 : (int)splits;
}
