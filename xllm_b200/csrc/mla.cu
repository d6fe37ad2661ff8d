// Paged absorbed-MLA attention (DeepSeek-V2/V3, Kimi-K2) over FlashInfer's two-cache CUDA layout
// (framework/kv_cache/kv_cache_shape.cpp:242-257,273-288): ckv_cache [pages, page_size, 512] holds the normalised latent
// c_kv, kpe_cache [pages, page_size, 64] the roped k_pe.  One kv head; per q row the key is [c_kv | k_pe] (576) and the
// value is c_kv (512): the math of layers/mlu/attention.cpp:65-155 on the absorbed q_input = [q_nope W_kc | rope(q_pe)].
//
// Tiling: one CTA per (m-tile, kv split, request).  The rows of one request are (q token, head) pairs, head minor,
// packed into the M dimension (kM = 16 or 64 rows).  Every kv token is streamed once per m-tile: a 1024-byte c_kv row and
// a 128-byte k_pe row, gathered through the page table by cp.async into a kStages-deep ring of kN-token tiles.  The V
// operand is the c_kv part of the same tile, read transposed by ldmatrix, so nothing is loaded twice.
// Warps come in pairs per 16-row group: S = [q_nope | q_pe] [c_kv | k_pe]^T is split by kv token (16 each, 36 k16
// steps), the pair exchanges row maxima and the bf16 P tile through shared memory, and each warp accumulates half of the
// 512 output columns (128 fp32 registers).  Softmax ladder of the other attention kernels: base-2 with sm_scale log2(e),
// P rounded to bf16, denominator = sum of the rounded P, fp32 PV.
// Split-KV: the plan fixes the split COUNT; the split size is derived here from the live kv_len, so a plan captured into
// a CUDA graph stays valid at later context lengths.  Partials (normalised fp32 O + base-2 LSE) meet in a separate merge
// kernel that sums them in split order (run-to-run bit-identical), as prefill_attention.cu does.
//
// Expanded prefill (xb_mla_prefill_expanded_bf16): the latent rows are gathered into a contiguous workspace, up-projected
// through kv_b_proj into per-head [k_nope | v] by the wgmma GEMM, and attended by the 192 / 128 instantiation of the
// prefill attention kernel: 2 (192 + 128) FLOP per (q, kv, head) instead of the absorbed form's 2 (576 + 512).
#include "tc_common.cuh"

namespace xb {
namespace {

constexpr int kMlaDc = 512;              // kv_lora_rank: c_kv = V = output width
constexpr int kMlaDr = 64;               // qk_rope_head_dim
constexpr int kMlaD = kMlaDc + kMlaDr;   // 576 = 36 k16 steps
constexpr int kMlaChunks = kMlaD / 8;    // 16-byte chunks per row
constexpr int kMlaLd = kMlaD + 8;        // shared row pitch: 1168 bytes = 16 mod 128, ldmatrix rows hit distinct banks
constexpr int kMlaN = 32;                // kv tokens per pipeline stage
constexpr int kMlaPLd = kMlaN + 8;       // P tile pitch (80 bytes, conflict-free for ldmatrix)
constexpr int kMlaMaxSplits = 128;
constexpr int kMlaMinSplitTokens = 256;  // a split streams at least this many tokens at the planned maximum context
constexpr int64_t kMlaPlanTag = 0x4D4C41;  // "MLA": plan8[7] >> 8

struct MlaParams {
  const __nv_bfloat16* q_nope;
  int64_t qn_stride_t, qn_stride_h;
  const __nv_bfloat16* q_pe;
  int64_t qp_stride_t, qp_stride_h;
  const __nv_bfloat16* ckv;
  int64_t ckv_stride_page, ckv_stride_token;
  const __nv_bfloat16* kpe;
  int64_t kpe_stride_page, kpe_stride_token;
  const int32_t* qo_indptr;
  const int32_t* kv_indptr;
  const int32_t* kv_indices;
  const int32_t* kv_last_page_len;
  __nv_bfloat16* o;
  int64_t o_stride_t, o_stride_h;
  float scale_log2;
  int num_heads, page_size, causal, splits, max_qo_len, batch;
  int64_t part_rows;  // batch * max_qo_len: row capacity of the partial buffers
  float* part_o;      // [splits][part_rows][num_heads][512]
  float* part_lse;    // [splits][part_rows][num_heads]
};

template <int kRG>
struct MlaCfg {
  static constexpr int kM = 16 * kRG;
  static constexpr int kThreads = 64 * kRG;
  static constexpr int kStages = kRG == 1 ? 2 : 3;  // kRG 1: two CTAs per SM, 4 stages in flight per SM either way
  static constexpr int kQBytes = kM * kMlaLd * 2;
  static constexpr int kStageBytes = kMlaN * kMlaLd * 2;
  static constexpr int kPBytes = kRG * 16 * kMlaPLd * 2;
  static constexpr int kRedBytes = kRG * 2 * 16 * 4;
  static constexpr int kSmemBytes = kQBytes + kStages * kStageBytes + kPBytes + 2 * kRedBytes;
};

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
// the two warps of one 16-row group
__device__ __forceinline__ void pair_sync(int rg) {
  asm volatile("bar.sync %0, 64;" ::"r"(1 + rg) : "memory");
}

template <int kRG>
__global__ void __launch_bounds__(64 * kRG, 1)
mla_attention_kernel(const MlaParams p) {
  using Cfg = MlaCfg<kRG>;
  constexpr int kM = Cfg::kM, kThreads = Cfg::kThreads, kStages = Cfg::kStages;
  extern __shared__ __align__(128) uint8_t smem[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem);
  __nv_bfloat16* sKV = reinterpret_cast<__nv_bfloat16*>(smem + Cfg::kQBytes);
  __nv_bfloat16* sP = reinterpret_cast<__nv_bfloat16*>(smem + Cfg::kQBytes + kStages * Cfg::kStageBytes);
  float* sMax = reinterpret_cast<float*>(smem + Cfg::kQBytes + kStages * Cfg::kStageBytes + Cfg::kPBytes);  // [kRG][2][16]
  float* sSum = sMax + kRG * 32;

  const int mt = blockIdx.x, split = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rg = warp >> 1, ch = warp & 1;  // 16-row group, output-column half / kv-token half
  const int g = lane >> 2, t4 = lane & 3;

  pdl_launch_dependents();
  pdl_wait();
  const int q0 = p.qo_indptr[b];
  const int qo_len = min(p.qo_indptr[b + 1] - q0, p.max_qo_len);
  const int H = p.num_heads;
  const int rows = qo_len * H;
  const int m0 = mt * kM;
  if (m0 >= rows) return;  // uniform over the CTA
  const int p0 = p.kv_indptr[b];
  const int n_pages = p.kv_indptr[b + 1] - p0;
  const int kv_len = n_pages > 0 ? (n_pages - 1) * p.page_size + p.kv_last_page_len[b] : 0;
  // this split's token range, derived from the live kv_len
  const int tiles_all = (kv_len + kMlaN - 1) / kMlaN;
  const int per_split = (tiles_all + p.splits - 1) / p.splits;
  const int kv_lo = min(kv_len, split * per_split * kMlaN);
  int kv_hi = min(kv_len, kv_lo + per_split * kMlaN);
  const int diag = kv_len - qo_len;  // causal: q row qi sees kv <= diag + qi
  if (p.causal) kv_hi = min(kv_hi, max(kv_lo, diag + (min(m0 + kM, rows) - 1) / H + 1));
  const int n_tiles = (kv_hi - kv_lo + kMlaN - 1) / kMlaN;

  // ---- Q tile: row r = (q token, head), [q_nope | q_pe]; rows past the request are zero ----
  for (int c = tid; c < kM * kMlaChunks; c += kThreads) {
    const int r = c / kMlaChunks, k = c % kMlaChunks;
    const int row = m0 + r;
    const uint32_t dst = smem_addr_u32(sQ + r * kMlaLd + k * 8);
    if (row < rows) {
      const int64_t tq = q0 + row / H;
      const int h = row % H;
      cp_async_16(dst, k < kMlaDc / 8 ? p.q_nope + tq * p.qn_stride_t + h * p.qn_stride_h + k * 8
                                      : p.q_pe + tq * p.qp_stride_t + h * p.qp_stride_h + (k - kMlaDc / 8) * 8);
    } else {
      sts_128(dst, make_uint4(0u, 0u, 0u, 0u));
    }
  }
  // ---- kv tile loader: kTPT threads per token, kCPT chunks each ----
  constexpr int kTPT = kThreads / kMlaN;
  constexpr int kCPT = kMlaChunks / kTPT;
  static_assert(kMlaChunks % kTPT == 0, "kv chunks split evenly over a token's threads");
  const int ld_tok = tid / kTPT, ld_sub = tid % kTPT;
  auto load_tile = [&](int j) {
    // tokens past the range load a real row (the last one): their scores are masked, their V rows meet P = 0
    const int kv = min(kv_lo + j * kMlaN + ld_tok, kv_hi - 1);
    const int64_t pg = p.kv_indices[p0 + kv / p.page_size];
    const int64_t off = kv % p.page_size;
    const __nv_bfloat16* ck = p.ckv + pg * p.ckv_stride_page + off * p.ckv_stride_token;
    const __nv_bfloat16* kp = p.kpe + pg * p.kpe_stride_page + off * p.kpe_stride_token;
    const uint32_t dst = smem_addr_u32(sKV + ((j % kStages) * kMlaN + ld_tok) * kMlaLd);
#pragma unroll
    for (int i = 0; i < kCPT; ++i) {
      const int k = ld_sub + i * kTPT;
      cp_async_16(dst + k * 16, k < kMlaDc / 8 ? ck + k * 8 : kp + (k - kMlaDc / 8) * 8);
    }
  };
  if (n_tiles > 0) load_tile(0);
  cp_async_commit();
#pragma unroll
  for (int s = 1; s < kStages - 1; ++s) {
    if (s < n_tiles) load_tile(s);
    cp_async_commit();
  }

  const bool active = m0 + rg * 16 < rows;  // this pair's 16 rows hold at least one live row (uniform per pair)
  int qi_row[2];                            // q index of rows g and g + 8
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) qi_row[hh] = (m0 + rg * 16 + g + 8 * hh) / H;
  float o[32][4];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  const uint32_t a_q = smem_addr_u32(sQ + (rg * 16 + (lane & 15)) * kMlaLd + (lane >> 4) * 8);
  const uint32_t a_p = smem_addr_u32(sP + (rg * 16 + (lane & 15)) * kMlaPLd + (lane >> 4) * 8);
  for (int j = 0; j < n_tiles; ++j) {
    cp_async_wait<kStages - 2>();
    __syncthreads();  // tile j landed for every thread; the ring slot of tile j - 1 and sMax / sP are free
    if (j + kStages - 1 < n_tiles) load_tile(j + kStages - 1);
    cp_async_commit();
    if (!active) continue;
    const __nv_bfloat16* kv_s = sKV + (j % kStages) * kMlaN * kMlaLd;
    // S: this warp's 16 rows x kv tokens [16 ch, 16 ch + 16) of the tile
    float s[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    const uint32_t b_k = smem_addr_u32(kv_s + (ch * 16 + (lane & 7) + (lane >> 4) * 8) * kMlaLd + ((lane >> 3) & 1) * 8);
#pragma unroll 12
    for (int k = 0; k < kMlaD / 16; ++k) {
      uint32_t a[4], bk[4];
      ldsm_x4(a, a_q + k * 32);
      ldsm_x4(bk, b_k + k * 32);
      mma_bf16_16816(s[0], a[0], a[1], a[2], a[3], bk[0], bk[1]);
      mma_bf16_16816(s[1], a[0], a[1], a[2], a[3], bk[2], bk[3]);
    }
    const int kv_base = kv_lo + j * kMlaN + ch * 16 + 2 * t4;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hh = e >> 1, kv = kv_base + nt * 8 + (e & 1);
        const bool ok = kv < kv_hi && (!p.causal || kv <= diag + qi_row[hh]);
        s[nt][e] = ok ? s[nt][e] * p.scale_log2 : -INFINITY;
        mx[hh] = fmaxf(mx[hh], s[nt][e]);
      }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
    }
    if (t4 == 0) {
      sMax[(rg * 2 + ch) * 16 + g] = mx[0];
      sMax[(rg * 2 + ch) * 16 + g + 8] = mx[1];
    }
    pair_sync(rg);
    float alpha[2], m_safe[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const float m_new = fmaxf(m_run[hh], fmaxf(mx[hh], sMax[(rg * 2 + (ch ^ 1)) * 16 + g + 8 * hh]));
      m_safe[hh] = m_new == -INFINITY ? 0.f : m_new;
      alpha[hh] = fast_exp2(m_run[hh] - m_safe[hh]);  // 0 while m_run is -inf
      m_run[hh] = m_new;
      l_run[hh] *= alpha[hh];
    }
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const uint32_t pp = pack_bf16x2(fast_exp2(s[nt][2 * hh] - m_safe[hh]), fast_exp2(s[nt][2 * hh + 1] - m_safe[hh]));
        l_run[hh] += bf16lo(pp) + bf16hi(pp);  // denominator = sum of the ROUNDED P
        *reinterpret_cast<uint32_t*>(sP + (rg * 16 + g + 8 * hh) * kMlaPLd + ch * 16 + nt * 8 + 2 * t4) = pp;
      }
    pair_sync(rg);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      o[i][0] *= alpha[0]; o[i][1] *= alpha[0];
      o[i][2] *= alpha[1]; o[i][3] *= alpha[1];
    }
    // O[:, 256 ch : 256 ch + 256] += P (16 x 32) V (32 x 256), V = c_kv rows of the tile read transposed
    const uint32_t b_v = smem_addr_u32(kv_s + ((lane & 7) + ((lane >> 3) & 1) * 8) * kMlaLd + ch * 256 + (lane >> 4) * 8);
#pragma unroll
    for (int ks = 0; ks < kMlaN / 16; ++ks) {
      uint32_t a[4];
      ldsm_x4(a, a_p + ks * 32);
#pragma unroll
      for (int np = 0; np < 16; ++np) {
        uint32_t bv[4];
        ldsm_x4_trans(bv, b_v + ks * 16 * kMlaLd * 2 + np * 32);
        mma_bf16_16816(o[2 * np], a[0], a[1], a[2], a[3], bv[0], bv[1]);
        mma_bf16_16816(o[2 * np + 1], a[0], a[1], a[2], a[3], bv[2], bv[3]);
      }
    }
  }
  cp_async_wait<0>();
  if (!active) return;

  // ---- epilogue: full row sums (quad, then the pair), normalise, store ----
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l_run[hh] += __shfl_xor_sync(0xffffffffu, l_run[hh], 1);
    l_run[hh] += __shfl_xor_sync(0xffffffffu, l_run[hh], 2);
  }
  if (t4 == 0) {
    sSum[(rg * 2 + ch) * 16 + g] = l_run[0];
    sSum[(rg * 2 + ch) * 16 + g + 8] = l_run[1];
  }
  pair_sync(rg);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = m0 + rg * 16 + g + 8 * hh;
    if (row >= rows) continue;
    const float l = l_run[hh] + sSum[(rg * 2 + (ch ^ 1)) * 16 + g + 8 * hh];
    const float inv = l > 0.f ? 1.0f / l : 0.f;
    const int64_t tq = q0 + row / H;
    const int h = row % H;
    if (p.splits == 1) {
      __nv_bfloat16* dst = p.o + tq * p.o_stride_t + h * p.o_stride_h + ch * 256 + 2 * t4;
#pragma unroll
      for (int nt = 0; nt < 32; ++nt)
        *reinterpret_cast<uint32_t*>(dst + nt * 8) = pack_bf16x2(o[nt][2 * hh] * inv, o[nt][2 * hh + 1] * inv);
    } else if (tq < p.part_rows) {  // a qo_indptr past the plan's batch * max_qo_len never writes outside its split
      const int64_t slot = ((int64_t)split * p.part_rows + tq) * H + h;
      float* dst = p.part_o + slot * kMlaDc + ch * 256 + 2 * t4;
#pragma unroll
      for (int nt = 0; nt < 32; ++nt)
        *reinterpret_cast<float2*>(dst + nt * 8) = make_float2(o[nt][2 * hh] * inv, o[nt][2 * hh + 1] * inv);
      if (ch == 0 && t4 == 0) p.part_lse[slot] = l > 0.f ? m_run[hh] + log2f(l) : -INFINITY;
    }
  }
}

// Combines the split partials of one (q token, head): weights 2^(lse_s - max) / sum, fixed split order.
__global__ void __launch_bounds__(128)
mla_merge_kernel(const MlaParams p) {
  const int64_t tq = blockIdx.x;
  const int h = blockIdx.y;
  pdl_launch_dependents();
  pdl_wait();
  if (tq >= p.qo_indptr[p.batch]) return;
  const int64_t stride = p.part_rows * p.num_heads;
  const int64_t slot0 = tq * p.num_heads + h;
  float mx = -INFINITY;
  for (int s = 0; s < p.splits; ++s) mx = fmaxf(mx, p.part_lse[slot0 + s * stride]);
  const float m_safe = mx == -INFINITY ? 0.f : mx;
  float wsum = 0.f;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  const int d = threadIdx.x * 4;
  for (int s = 0; s < p.splits; ++s) {
    const int64_t slot = slot0 + s * stride;
    const float w = fast_exp2(p.part_lse[slot] - m_safe);
    const float4 v = __ldcg(reinterpret_cast<const float4*>(p.part_o + slot * kMlaDc + d));
    wsum += w;
    acc.x += v.x * w; acc.y += v.y * w; acc.z += v.z * w; acc.w += v.w * w;
  }
  const float inv = wsum > 0.f ? 1.0f / wsum : 0.f;
  uint2 ob;
  ob.x = pack_bf16x2(acc.x * inv, acc.y * inv);
  ob.y = pack_bf16x2(acc.z * inv, acc.w * inv);
  *reinterpret_cast<uint2*>(p.o + tq * p.o_stride_t + h * p.o_stride_h + d) = ob;
}

template <int kRG>
int launch_mla(const MlaParams& p, int m_tiles, cudaStream_t stream) {
  constexpr auto kern = mla_attention_kernel<kRG>;
  XB_CUDA_OK(set_max_dynamic_smem_once<kern>(MlaCfg<kRG>::kSmemBytes));
  XB_CUDA_OK(launch(kern, dim3(m_tiles, p.splits, p.batch), dim3(MlaCfg<kRG>::kThreads),
                    (size_t)MlaCfg<kRG>::kSmemBytes, stream, true, p));
  if (p.splits > 1)
    XB_CUDA_OK(launch(mla_merge_kernel, dim3((unsigned)p.part_rows, p.num_heads), dim3(kMlaDc / 4), 0, stream, true, p));
  return 0;
}

int64_t mla_workspace_bytes(int64_t splits, int64_t part_rows, int num_heads) {
  return splits > 1 ? splits * part_rows * num_heads * (kMlaDc + 1) * (int64_t)sizeof(float) : 0;
}

// ---- expanded prefill ------------------------------------------------------------------------------------------
constexpr int kMlaUpW = 256;                 // kv_b_proj rows per head: k_nope 128 | v 128
constexpr int kMlaGatherTokens = 32;
constexpr int kMlaGatherThreads = 256;
constexpr int64_t kMlaExpTag = 0x4D4C45;     // "MLE": plan8[7] >> 40
// Selector: expanded when  absorbed FLOP > kMlaExpandedCost * (up-projection FLOP + expanded attention FLOP), i.e. one
// FLOP of the expanded path costs as much time as kMlaExpandedCost FLOP of the absorbed kernel.  Criterion: the least total
// time over the selector grid of tools/mla_sweep.py (H100 80GB HBM3, 700 W; README).  Every constant from 0.13 to 0.80
// reaches it (63.84 ms; the qo = 128 / history 0 points, FLOP ratio 0.463, split that range and move the total by 1.6 us),
// and 0.5 lies amid the break-even ratios measured for chunks of 512+ tokens (0.37-0.68).  Worst point: a 128-token
// chunk over 32 K history at H = 16 runs expanded, 1.40x slower than absorbed.
constexpr double kMlaExpandedCost = 0.5;

struct MlaGatherParams {
  const __nv_bfloat16* ckv;
  int64_t ckv_stride_page, ckv_stride_token;
  const __nv_bfloat16* kpe;
  int64_t kpe_stride_page, kpe_stride_token;
  const int32_t* kv_indptr;
  const int32_t* kv_indices;
  const int32_t* kv_last_page_len;
  int page_size;
  int64_t total_kv;       // the plan's row capacity of ckv_out / kpe_out
  __nv_bfloat16* ckv_out; // [total_kv, 512]
  __nv_bfloat16* kpe_out; // [total_kv, 64]
  int32_t* kv_cu;         // [batch + 1] ragged offsets of the gathered rows
};

__device__ __forceinline__ int64_t mla_kv_len(const MlaGatherParams& g, int b) {
  const int n_pages = g.kv_indptr[b + 1] - g.kv_indptr[b];
  return n_pages > 0 ? (int64_t)(n_pages - 1) * g.page_size + g.kv_last_page_len[b] : 0;
}

// One CTA per (32 kv tokens, request).  The request's first row is the sum of the live kv lengths before it; rows at or
// past the plan's total_kv are not written, and kv_cu is clamped to total_kv, so lengths beyond the plan stay inside the
// workspace.
__global__ void __launch_bounds__(kMlaGatherThreads)
mla_gather_latent_kernel(const MlaGatherParams g) {
  __shared__ int64_t red[kMlaGatherThreads / 32];
  const int b = blockIdx.y;
  pdl_launch_dependents();
  pdl_wait();
  int64_t part = 0;
  for (int i = threadIdx.x; i < b; i += kMlaGatherThreads) part += mla_kv_len(g, i);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
  __syncthreads();
  int64_t off = 0;
#pragma unroll
  for (int w = 0; w < kMlaGatherThreads / 32; ++w) off += red[w];
  const int64_t kv_len = mla_kv_len(g, b);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    g.kv_cu[b + 1] = (int32_t)min(off + kv_len, g.total_kv);
    if (b == 0) g.kv_cu[0] = 0;
  }
  const int p0 = g.kv_indptr[b];
  constexpr int kChunks = kMlaD / 8;  // 16-byte pieces of [c_kv | k_pe]
  for (int c = threadIdx.x; c < kMlaGatherTokens * kChunks; c += kMlaGatherThreads) {
    const int64_t t = (int64_t)blockIdx.x * kMlaGatherTokens + c / kChunks;
    const int k = c % kChunks;
    const int64_t row = off + t;
    if (t >= kv_len || row >= g.total_kv) continue;
    const int64_t pg = g.kv_indices[p0 + t / g.page_size], in_pg = t % g.page_size;
    if (k < kMlaDc / 8)
      *reinterpret_cast<uint4*>(g.ckv_out + row * kMlaDc + k * 8) =
          *reinterpret_cast<const uint4*>(g.ckv + pg * g.ckv_stride_page + in_pg * g.ckv_stride_token + k * 8);
    else
      *reinterpret_cast<uint4*>(g.kpe_out + row * kMlaDr + (k - kMlaDc / 8) * 8) =
          *reinterpret_cast<const uint4*>(g.kpe + pg * g.kpe_stride_page + in_pg * g.kpe_stride_token + (k - kMlaDc / 8) * 8);
  }
}

int64_t align256(int64_t x) { return (x + 255) & ~int64_t(255); }

// workspace layout (bytes): kv_up [total_kv, H, 256] bf16 at 0 | ckv [total_kv, 512] bf16 | kpe [total_kv, 64] bf16 |
// kv_cu int32 [batch + 1]; each part starts on a 256-byte boundary
struct MlaExpLayout {
  int64_t ckv, kpe, kv_cu, bytes;
};
MlaExpLayout mla_exp_layout(int64_t total_kv, int num_heads, int batch) {
  MlaExpLayout l;
  l.ckv = align256(total_kv * num_heads * kMlaUpW * 2);
  l.kpe = l.ckv + align256(total_kv * kMlaDc * 2);
  l.kv_cu = l.kpe + align256(total_kv * kMlaDr * 2);
  l.bytes = l.kv_cu + align256((int64_t)(batch + 1) * 4);
  return l;
}

}  // namespace
}  // namespace xb

using namespace xb;

// plan8: [0] splits  [1] float workspace bytes  [2] batch  [3] num_heads  [4] max_qo_len  [5] page_size
//        [6] m-tiles per request  [7] rows per m-tile / 16 (1 | 4) | tag << 8
extern "C" int xb_mla_plan(int64_t* plan8, int batch, int num_heads, int kv_lora_rank, int qk_rope_head_dim,
                           int max_qo_len, int page_size, int max_pages_per_request, int num_sms) {
  XB_CHECK(plan8 != nullptr, "mla_plan: plan8 is null");
  XB_CHECK(kv_lora_rank == kMlaDc && qk_rope_head_dim == kMlaDr,
           "mla_plan: kv_lora_rank %d / qk_rope_head_dim %d unsupported (512 / 64)", kv_lora_rank, qk_rope_head_dim);
  XB_CHECK(num_heads >= 1 && num_heads <= 128, "mla_plan: num_heads %d unsupported (1..128)", num_heads);
  XB_CHECK(batch >= 1 && batch <= 65535, "mla_plan: batch %d out of range (1..65535)", batch);
  XB_CHECK(max_qo_len >= 1 && (int64_t)batch * max_qo_len <= INT32_MAX, "mla_plan: bad max_qo_len %d", max_qo_len);
  XB_CHECK(page_size >= 1 && max_pages_per_request >= 1, "mla_plan: bad page geometry (page_size %d, max pages %d)",
           page_size, max_pages_per_request);
  if (num_sms <= 0) num_sms = 132;
  const int64_t rows = (int64_t)max_qo_len * num_heads;
  const int rg = rows <= 16 ? 1 : 4;
  const int64_t m_tiles = (rows + 16 * rg - 1) / (16 * rg);
  XB_CHECK(m_tiles <= INT32_MAX, "mla_plan: %lld m-tiles", (long long)m_tiles);
  // one wave: CTAs resident per SM (two of the 16-row kernel, one of the 64-row kernel) over the CTAs without splits
  const int64_t slots = (int64_t)num_sms * (rg == 1 ? 2 : 1);
  int64_t splits = slots / ((int64_t)batch * m_tiles);
  const int64_t max_kv = (int64_t)max_pages_per_request * page_size;
  const int64_t by_len = (max_kv + kMlaMinSplitTokens - 1) / kMlaMinSplitTokens;
  if (splits > by_len) splits = by_len;
  if (splits > kMlaMaxSplits) splits = kMlaMaxSplits;
  if (splits < 1) splits = 1;
  const int64_t part_rows = (int64_t)batch * max_qo_len;
  plan8[0] = splits;
  plan8[1] = mla_workspace_bytes(splits, part_rows, num_heads);
  plan8[2] = batch;
  plan8[3] = num_heads;
  plan8[4] = max_qo_len;
  plan8[5] = page_size;
  plan8[6] = m_tiles;
  plan8[7] = rg | (kMlaPlanTag << 8);
  return 0;
}

extern "C" int xb_mla_plan_set_splits(int64_t* plan8, int splits) {
  XB_CHECK(plan8 != nullptr && (plan8[7] >> 8) == kMlaPlanTag, "mla_plan_set_splits: not an MLA plan");
  XB_CHECK(splits >= 1 && splits <= kMlaMaxSplits, "mla_plan_set_splits: splits %d out of range (1..%d)", splits,
           kMlaMaxSplits);
  plan8[0] = splits;
  plan8[1] = mla_workspace_bytes(splits, plan8[2] * plan8[4], (int)plan8[3]);
  return 0;
}

extern "C" int xb_mla_paged_attention_bf16(const int64_t* plan8, const void* q_nope, int64_t q_nope_stride_t,
                                           int64_t q_nope_stride_h, const void* q_pe, int64_t q_pe_stride_t,
                                           int64_t q_pe_stride_h, const void* ckv_cache, int64_t ckv_stride_page,
                                           int64_t ckv_stride_token, const void* kpe_cache, int64_t kpe_stride_page,
                                           int64_t kpe_stride_token, const int32_t* qo_indptr, const int32_t* kv_indptr,
                                           const int32_t* kv_indices, const int32_t* kv_last_page_len, int causal,
                                           void* o, int64_t o_stride_t, int64_t o_stride_h, float sm_scale,
                                           void* workspace, int64_t workspace_bytes, xb_stream_t stream) {
  XB_CHECK(plan8 != nullptr && (plan8[7] >> 8) == kMlaPlanTag, "mla_paged_attention: plan is not an MLA plan (xb_mla_plan)");
  XB_CHECK(q_nope && q_pe && ckv_cache && kpe_cache && o, "mla_paged_attention: null q_nope / q_pe / cache / o pointer");
  XB_CHECK(qo_indptr && kv_indptr && kv_indices && kv_last_page_len, "mla_paged_attention: null qo_indptr / paged kv pointer");
  const auto a16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  XB_CHECK(a16(q_nope) && a16(q_pe) && a16(ckv_cache) && a16(kpe_cache) && (reinterpret_cast<uintptr_t>(o) & 7) == 0 &&
               q_nope_stride_t % 8 == 0 && q_nope_stride_h % 8 == 0 && q_pe_stride_t % 8 == 0 && q_pe_stride_h % 8 == 0 &&
               ckv_stride_page % 8 == 0 && ckv_stride_token % 8 == 0 && kpe_stride_page % 8 == 0 &&
               kpe_stride_token % 8 == 0 && o_stride_t % 4 == 0 && o_stride_h % 4 == 0,
           "mla_paged_attention: q / cache rows must be 16-byte aligned, o rows 8-byte aligned");
  MlaParams p{};
  p.splits = (int)plan8[0];
  p.batch = (int)plan8[2];
  p.num_heads = (int)plan8[3];
  p.max_qo_len = (int)plan8[4];
  p.page_size = (int)plan8[5];
  const int m_tiles = (int)plan8[6];
  const int rg = (int)(plan8[7] & 0xff);
  p.part_rows = plan8[2] * plan8[4];
  XB_CHECK(p.splits >= 1 && p.splits <= kMlaMaxSplits && (rg == 1 || rg == 4), "mla_paged_attention: corrupt plan");
  XB_CHECK(plan8[1] == mla_workspace_bytes(p.splits, p.part_rows, p.num_heads), "mla_paged_attention: corrupt plan");
  XB_CHECK(p.splits == 1 || (workspace != nullptr && workspace_bytes >= plan8[1]),
           "mla_paged_attention: workspace of %lld bytes is smaller than the plan's %lld", (long long)workspace_bytes,
           (long long)plan8[1]);
  XB_CHECK(p.splits == 1 || (reinterpret_cast<uintptr_t>(workspace) & 15) == 0,
           "mla_paged_attention: workspace must be 16-byte aligned");
  p.q_nope = reinterpret_cast<const __nv_bfloat16*>(q_nope);
  p.qn_stride_t = q_nope_stride_t;
  p.qn_stride_h = q_nope_stride_h;
  p.q_pe = reinterpret_cast<const __nv_bfloat16*>(q_pe);
  p.qp_stride_t = q_pe_stride_t;
  p.qp_stride_h = q_pe_stride_h;
  p.ckv = reinterpret_cast<const __nv_bfloat16*>(ckv_cache);
  p.ckv_stride_page = ckv_stride_page;
  p.ckv_stride_token = ckv_stride_token;
  p.kpe = reinterpret_cast<const __nv_bfloat16*>(kpe_cache);
  p.kpe_stride_page = kpe_stride_page;
  p.kpe_stride_token = kpe_stride_token;
  p.qo_indptr = qo_indptr;
  p.kv_indptr = kv_indptr;
  p.kv_indices = kv_indices;
  p.kv_last_page_len = kv_last_page_len;
  p.causal = causal ? 1 : 0;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.o_stride_t = o_stride_t;
  p.o_stride_h = o_stride_h;
  p.scale_log2 = sm_scale * 1.44269504088896340736f;
  p.part_o = reinterpret_cast<float*>(workspace);
  p.part_lse = p.part_o ? p.part_o + (int64_t)p.splits * p.part_rows * p.num_heads * kMlaDc : nullptr;
  cudaStream_t s = (cudaStream_t)stream;
  return rg == 1 ? launch_mla<1>(p, m_tiles, s) : launch_mla<4>(p, m_tiles, s);
}

// plan8: [0] use_expanded  [1] workspace bytes  [2] batch  [3] num_heads  [4] max_qo_len  [5] total_kv  [6] max_kv_len
//        [7] total_q | tag << 40
extern "C" int xb_mla_expanded_plan(int64_t* plan8, int batch, int num_heads, const int32_t* qo_lens_host,
                                    const int32_t* kv_lens_host) {
  XB_CHECK(plan8 != nullptr, "mla_expanded_plan: plan8 is null");
  XB_CHECK(num_heads >= 1 && num_heads <= 128, "mla_expanded_plan: num_heads %d unsupported (1..128)", num_heads);
  XB_CHECK(batch >= 1 && batch <= 65535, "mla_expanded_plan: batch %d out of range (1..65535)", batch);
  XB_CHECK(qo_lens_host != nullptr && kv_lens_host != nullptr, "mla_expanded_plan: null qo_lens / kv_lens");
  int64_t total_q = 0, total_kv = 0, pairs = 0;
  int max_qo = 0, max_kv = 0;
  for (int b = 0; b < batch; ++b) {
    const int64_t qo = qo_lens_host[b], kv = kv_lens_host[b];
    XB_CHECK(qo >= 0 && kv >= qo, "mla_expanded_plan: request %d has qo_len %lld > kv_len %lld (or a negative length)", b,
             (long long)qo, (long long)kv);
    total_q += qo;
    total_kv += kv;
    pairs += qo * (kv - qo) + qo * (qo + 1) / 2;  // causal (q, kv) pairs
    max_qo = qo > max_qo ? (int)qo : max_qo;
    max_kv = kv > max_kv ? (int)kv : max_kv;
  }
  XB_CHECK(total_q <= INT32_MAX && total_kv <= INT32_MAX, "mla_expanded_plan: %lld q / %lld kv tokens exceed int32",
           (long long)total_q, (long long)total_kv);
  // FLOP per head: absorbed 2 (576 + 512) per pair; expanded 2 (192 + 128) per pair + 2 * 512 * 256 per kv token
  const double absorbed = 2.0 * (kMlaD + kMlaDc) * (double)pairs;
  const double expanded = 2.0 * (192 + 128) * (double)pairs + 2.0 * kMlaDc * kMlaUpW * (double)total_kv;
  plan8[0] = max_qo > 1 && absorbed > kMlaExpandedCost * expanded ? 1 : 0;
  plan8[1] = mla_exp_layout(total_kv, num_heads, batch).bytes;
  plan8[2] = batch;
  plan8[3] = num_heads;
  plan8[4] = max_qo;
  plan8[5] = total_kv;
  plan8[6] = max_kv;
  plan8[7] = total_q | (kMlaExpTag << 40);
  return 0;
}

extern "C" int xb_mla_prefill_expanded_bf16(const int64_t* plan8, const void* q, int64_t q_stride_t, int64_t q_stride_h,
                                            const void* ckv_cache, int64_t ckv_stride_page, int64_t ckv_stride_token,
                                            const void* kpe_cache, int64_t kpe_stride_page, int64_t kpe_stride_token,
                                            int page_size, const int32_t* kv_indptr, const int32_t* kv_indices,
                                            const int32_t* kv_last_page_len, const int32_t* qo_indptr,
                                            const void* kv_b_proj, void* o, int64_t o_stride_t, int64_t o_stride_h,
                                            float sm_scale, void* workspace, int64_t workspace_bytes,
                                            xb_stream_t stream) {
  XB_CHECK(plan8 != nullptr && (plan8[7] >> 40) == kMlaExpTag,
           "mla_prefill_expanded: plan is not an expanded MLA plan (xb_mla_expanded_plan)");
  const int batch = (int)plan8[2], num_heads = (int)plan8[3], max_qo = (int)plan8[4], max_kv = (int)plan8[6];
  const int64_t total_kv = plan8[5], total_q = plan8[7] & ((int64_t(1) << 40) - 1);
  XB_CHECK(batch >= 1 && num_heads >= 1 && num_heads <= 128 && total_kv >= 0 && max_kv >= 0 &&
               plan8[1] == mla_exp_layout(total_kv, num_heads, batch).bytes,
           "mla_prefill_expanded: corrupt plan");
  XB_CHECK(q && ckv_cache && kpe_cache && kv_b_proj && o, "mla_prefill_expanded: null q / cache / kv_b_proj / o pointer");
  XB_CHECK(qo_indptr && kv_indptr && kv_indices && kv_last_page_len,
           "mla_prefill_expanded: null qo_indptr / paged kv pointer");
  XB_CHECK(page_size >= 1, "mla_prefill_expanded: page_size %d", page_size);
  XB_CHECK(workspace != nullptr && workspace_bytes >= plan8[1],
           "mla_prefill_expanded: workspace of %lld bytes is smaller than the plan's %lld", (long long)workspace_bytes,
           (long long)plan8[1]);
  const auto a16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  XB_CHECK(a16(q) && a16(ckv_cache) && a16(kpe_cache) && a16(kv_b_proj) && a16(workspace) &&
               (reinterpret_cast<uintptr_t>(o) & 3) == 0 && q_stride_t % 8 == 0 && q_stride_h % 8 == 0 &&
               ckv_stride_page % 8 == 0 && ckv_stride_token % 8 == 0 && kpe_stride_page % 8 == 0 &&
               kpe_stride_token % 8 == 0 && o_stride_t % 2 == 0 && o_stride_h % 2 == 0,
           "mla_prefill_expanded: q / cache / kv_b_proj / workspace rows must be 16-byte aligned, o rows 4-byte aligned");
  if (total_q == 0) return 0;
  const MlaExpLayout l = mla_exp_layout(total_kv, num_heads, batch);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  auto* kv_up = reinterpret_cast<__nv_bfloat16*>(ws);
  MlaGatherParams g{};
  g.ckv = reinterpret_cast<const __nv_bfloat16*>(ckv_cache);
  g.ckv_stride_page = ckv_stride_page;
  g.ckv_stride_token = ckv_stride_token;
  g.kpe = reinterpret_cast<const __nv_bfloat16*>(kpe_cache);
  g.kpe_stride_page = kpe_stride_page;
  g.kpe_stride_token = kpe_stride_token;
  g.kv_indptr = kv_indptr;
  g.kv_indices = kv_indices;
  g.kv_last_page_len = kv_last_page_len;
  g.page_size = page_size;
  g.total_kv = total_kv;
  g.ckv_out = reinterpret_cast<__nv_bfloat16*>(ws + l.ckv);
  g.kpe_out = reinterpret_cast<__nv_bfloat16*>(ws + l.kpe);
  g.kv_cu = reinterpret_cast<int32_t*>(ws + l.kv_cu);
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned chunks = (unsigned)((max_kv + kMlaGatherTokens - 1) / kMlaGatherTokens);
  XB_CUDA_OK(launch(mla_gather_latent_kernel, dim3(chunks > 0 ? chunks : 1, batch), dim3(kMlaGatherThreads), 0, s, true, g));
  // kv_up [total_kv, H * 256] = ckv [total_kv, 512] . kv_b_proj [H * 256, 512]^T
  if (xb_gemm_bf16(kv_up, (int64_t)num_heads * kMlaUpW, g.ckv_out, kMlaDc, kv_b_proj, nullptr, (int)total_kv,
                   num_heads * kMlaUpW, kMlaDc, stream))
    return 1;
  return mla_expanded_attention(q, q_stride_t, q_stride_h, total_q, kv_up, g.kpe_out, total_kv, qo_indptr, g.kv_cu, o,
                                o_stride_t, o_stride_h, batch, max_qo, num_heads, sm_scale, s);
}
