// Paged decode attention (q_len = 1 per request) over the block-table KV cache.
// Replaces the FlashInfer decode module behind xllm::kernel::cuda::batch_decode
// (xllm/core/kernels/cuda/batch_decode.cpp:26-86; planner
//  xllm/core/layers/cuda/flashinfer_planinfo.cpp:249-337).
//
// Design (HBM-bound):
//   grid = (kv splits, kv heads, batch).  One CTA streams one KV chunk of one
//   (request, kv head): all GQA query heads of that kv head share the chunk, so
//   every KV byte is read exactly once.  Per 16-token block a thread issues 16
//   independent 16-byte loads (8 K + 8 V) straight into mma.sync fragments -
//   rows are gathered through the page table, each K/V row is a contiguous
//   head_dim*2-byte segment (128-byte coalesced sectors), no shared-memory
//   staging.  The head-dim / token permutations the fragment layout implies are
//   absorbed by loading q with the same permutation (a dot product does not
//   care about the order of its terms).
//     S[head, tok]  = Q[16 heads x d] . K^T        (m16n8k16, heads in M)
//     O[head, d]   += P[16 heads x 16 tok] . V     (C-fragments of S feed A of PV)
//   fp32 online softmax in base 2 (sm_scale*log2(e) folded into one FMUL), P is
//   rounded to bf16 for the PV MMA, fp32 accumulation - the same ladder as the
//   FlashInfer tensor-core decode path the reference selects for GQA >= 4
//   (utils.cpp:349-367).
//   Warps of a CTA split the chunk's 16-token blocks and merge their
//   (m, l, O) states through shared memory.  The splits of one (request, kv
//   head) are merged in up to two more levels, both inside this launch:
//     * thread-block CLUSTER (<= 16 CTAs along the split axis): every CTA keeps
//       its normalised partial + base-2 LSE in shared memory; after one
//       cluster barrier CTA r merges slice r of the (head, d) items of all
//       peers through distributed shared memory (reduce-scatter: 215-cycle
//       DSMEM loads instead of a round trip through L2) and writes it out;
//     * if one request's splits span K > 1 clusters, the cluster results go to
//       the float workspace and the LAST CTA to arrive (atomic ticket in the
//       int workspace) merges the K partials.
//   No second launch, no host sync, CUDA-graph safe: the split size is derived
//   ON THE DEVICE from the live kv_len and the launched grid, so a plan made at
//   graph capture serves any later context length (flashinfer_attention.cpp:
//   306-311 replays a captured `run`); clusters past the live split count exit.
#include "common.cuh"

namespace xb {

struct DecodeParams {
  const __nv_bfloat16* q;
  int64_t q_stride_n, q_stride_h;
  const __nv_bfloat16* k_cache;
  const __nv_bfloat16* v_cache;
  int64_t stride_page, stride_token, stride_head;
  const int32_t* kv_indptr;
  const int32_t* kv_indices;
  const int32_t* kv_last_page_len;
  __nv_bfloat16* o;
  int64_t o_stride_n, o_stride_h;
  float* lse;  // optional [batch, num_qo_heads]
  float scale_log2;
  float* part_o;    // [batch, num_qo_heads, max_parts, D]
  float* part_lse;  // [batch, num_qo_heads, max_parts]
  int32_t* counters;  // [batch, num_kv_heads * head_tiles][2]: word 0 = self-resetting arrival counter (word 1 unused)
  int num_qo_heads, num_kv_heads, group, head_tiles;
  int page_size, page_shift;  // page_shift >= 0 when page_size is a power of two
  int min_chunk;              // smallest KV chunk a split may get (multiple of 16)
  int max_parts;              // stride of the partial buffers (>= gridDim.x / cluster)
  int cluster;                // CTAs per cluster along the split axis (1 = no cluster launch)
  int early_prefetch;  // KV rows of old tokens + the paged triplet are not written by any in-flight kernel
  unsigned long long* trace;  // debug: per-CTA stage timestamps (xb_debug_set_decode_trace), else null
};

// ---- thread-block cluster primitives (sm_90+): rank, barrier, distributed shared memory loads ----
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_arrive_release() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_wait_acquire() {
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t dsmem_addr(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ float ld_dsmem_f1(uint32_t addr) {
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ const __nv_bfloat16* kv_row(const DecodeParams& p, const __nv_bfloat16* cache,
                                                       int indptr0, int tok, int kvh) {
  int page_idx, off;
  if (p.page_shift >= 0) {
    page_idx = tok >> p.page_shift;
    off = tok & (p.page_size - 1);
  } else {
    page_idx = tok / p.page_size;
    off = tok - page_idx * p.page_size;
  }
  const int64_t page = __ldg(p.kv_indices + indptr0 + page_idx);
  return cache + page * p.stride_page + (int64_t)off * p.stride_token + (int64_t)kvh * p.stride_head;
}

constexpr int kTeam = 8;   // CTAs that share the final merge of one (request, kv head)

template <int kD, int kGT /*1: <=8 heads per CTA, 2: <=16*/, int kWarpsT>
__global__ void __launch_bounds__(kWarpsT * 32, 1)
paged_decode_kernel(const DecodeParams p) {
  constexpr int kChunks = kD / 32;  // 16-byte K chunks per lane per token
  constexpr int kNT = kD / 8;       // n8 tiles of the output
  constexpr int kVC = kD / 64;      // V chunk loads per token per lane
  constexpr int kHeads = 8 * kGT;
  constexpr int kRS = kD + 4;       // padded smem row (floats)
  extern __shared__ __align__(16) float smem[];
  float* sm_o = smem;                              // [warps][kHeads][kRS]
  float* sm_m = sm_o + kWarpsT * kHeads * kRS;      // [warps][kHeads]
  float* sm_l = sm_m + kWarpsT * kHeads;           // [warps][kHeads]
  float* sm_co = sm_l + kWarpsT * kHeads;          // [kHeads][kD]  this CTA's normalised partial (read by cluster peers)
  float* sm_clse = sm_co + kHeads * kD;            // [kHeads]      its base-2 LSE
  __shared__ int s_ticket;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int split = blockIdx.x;
  const int kvh = blockIdx.y / p.head_tiles, htile = blockIdx.y % p.head_tiles;
  const int b = blockIdx.z;

  pdl_launch_dependents();  // let the consumer's prologue (weight prefetch) start as early as possible
  if (!p.early_prefetch) pdl_wait();
  const int cta_lin = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  auto stamp = [&](int i) {
    if (p.trace && threadIdx.x == 0) p.trace[(size_t)cta_lin * 8 + i] = globaltimer_ns();
  };
  stamp(0);

  const int indptr0 = __ldg(p.kv_indptr + b);
  const int n_pages = __ldg(p.kv_indptr + b + 1) - indptr0;
  const int kv_len = n_pages > 0 ? (n_pages - 1) * p.page_size + __ldg(p.kv_last_page_len + b) : 0;
  // Split geometry is derived HERE from the live kv_len and the launched grid (not baked into the plan): any context
  // length is covered by gridDim.x splits of whole 16-token blocks, so a plan / CUDA graph made for a short context
  // stays correct when replayed on a longer one.
  const int S = gridDim.x, C = p.cluster;
  int chunk = (((kv_len + S - 1) / S) + 15) & ~15;
  if (chunk < p.min_chunk) chunk = p.min_chunk;
  int n_splits = (kv_len + chunk - 1) / chunk;
  if (n_splits < 1) n_splits = 1;
  const int n_parts = (n_splits + C - 1) / C;     // live clusters (= partials that reach the workspace) of this unit
  const int part = split / C;
  if (part >= n_parts) return;                    // uniform over the whole cluster: nobody waits for this CTA
  stamp(1);
  const int t_begin = min(split * chunk, kv_len);
  const int t_end = min(kv_len, t_begin + chunk);
  const int head0 = kvh * p.group + htile * kHeads;            // first qo head of this CTA
  const int nheads = min(kHeads, p.group - htile * kHeads);    // live heads in this CTA
  const int nblk = (t_end - t_begin + 15) >> 4;
  const int last_tok = kv_len - 1;

  struct KVFrag {
    uint4 kf[2][kChunks];
    uint4 vf[4][kVC];
  };
  // 16 independent 16-byte loads of one 16-token block, straight into MMA fragment registers
  auto load_block = [&](KVFrag& f, int blk) {
    const int tb = t_begin + (blk << 4);
#pragma unroll
    for (int tile = 0; tile < 2; ++tile) {
      const int tok = min(tb + tile * 8 + g, last_tok);
      const __nv_bfloat16* row = kv_row(p, p.k_cache, indptr0, tok, kvh);
#pragma unroll
      for (int i = 0; i < kChunks; ++i) f.kf[tile][i] = ldg_stream(row + (4 * i + t) * 8);
    }
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int tok = min(tb + (s >> 1) * 8 + 2 * t + (s & 1), last_tok);
      const __nv_bfloat16* row = kv_row(p, p.v_cache, indptr0, tok, kvh);
#pragma unroll
      for (int c = 0; c < kVC; ++c) f.vf[s][c] = ldg_stream(row + (c * 8 + g) * 8);
    }
  };

  int blk = warp;
  bool have = blk < nblk;
  KVFrag cur;
  // With early_prefetch the first block of every warp is fetched while the producer kernel (RoPE + KV scatter of the
  // NEWEST token) may still be running - except the block that holds that newest token.
  const bool early = p.early_prefetch && have && (t_begin + (blk << 4) + 16 <= last_tok);
  if (early) load_block(cur, blk);
  if (p.early_prefetch) pdl_wait();

  // ---- Q fragments (chunk 4i+t of head g / g+8, same permutation as K) -------
  uint4 qa[kChunks], qb[kChunks];
  {
    const __nv_bfloat16* qrow = p.q + (int64_t)b * p.q_stride_n;
#pragma unroll
    for (int i = 0; i < kChunks; ++i) {
      qa[i] = make_uint4(0, 0, 0, 0);
      qb[i] = make_uint4(0, 0, 0, 0);
      if (g < nheads) qa[i] = *reinterpret_cast<const uint4*>(qrow + (int64_t)(head0 + g) * p.q_stride_h + (4 * i + t) * 8);
      if (kGT == 2 && g + 8 < nheads)
        qb[i] = *reinterpret_cast<const uint4*>(qrow + (int64_t)(head0 + g + 8) * p.q_stride_h + (4 * i + t) * 8);
    }
  }
  if (have && !early) load_block(cur, blk);

  float o_acc[kNT][4];
#pragma unroll
  for (int j = 0; j < kNT; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) o_acc[j][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};  // head g, head g+8
  float l_run[2] = {0.f, 0.f};              // per-thread partial sums

  while (have) {
    const int tb = t_begin + (blk << 4);
    // ---- prefetch the warp's next block while this one is consumed -----------
    const int nblk_next = blk + kWarpsT;
    const bool have_next = nblk_next < nblk;
    KVFrag nxt;
    if (have_next) load_block(nxt, nblk_next);
    const uint4 (&kf)[2][kChunks] = cur.kf;
    const uint4 (&vf)[4][kVC] = cur.vf;
    // ---- S = Q K^T ----------------------------------------------------------
    float s_acc[2][4];
#pragma unroll
    for (int tile = 0; tile < 2; ++tile) {
#pragma unroll
      for (int i = 0; i < 4; ++i) s_acc[tile][i] = 0.f;
#pragma unroll
      for (int i = 0; i < kChunks; ++i) {
        mma_bf16_16816(s_acc[tile], qa[i].x, qb[i].x, qa[i].y, qb[i].y, kf[tile][i].x, kf[tile][i].y);
        mma_bf16_16816(s_acc[tile], qa[i].z, qb[i].z, qa[i].w, qb[i].w, kf[tile][i].z, kf[tile][i].w);
      }
    }
    if (p.trace && blk == warp && warp == 0 && s_acc[0][0] != 12345.678f) stamp(7);   // first K block has arrived
    // ---- online softmax (base 2) ---------------------------------------------
    uint32_t pa[4];  // A fragment of P: a0 (g, tile0) a1 (g+8, tile0) a2 (g, tile1) a3 (g+8, tile1)
#pragma unroll
    for (int hh = 0; hh < kGT; ++hh) {
      float sv[4];
#pragma unroll
      for (int tile = 0; tile < 2; ++tile)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int tok = tb + tile * 8 + 2 * t + e;
          const float s = s_acc[tile][hh * 2 + e] * p.scale_log2;
          sv[tile * 2 + e] = tok < t_end ? s : -INFINITY;
        }
      float mx = fmaxf(fmaxf(sv[0], sv[1]), fmaxf(sv[2], sv[3]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[hh], mx);
      const float m_safe = m_new == -INFINITY ? 0.f : m_new;
      const float alpha = fast_exp2(m_run[hh] - m_safe);
      float pv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) pv[i] = fast_exp2(sv[i] - m_safe);
      // P is rounded to bf16 for the PV MMA and the denominator sums the ROUNDED values
      // (FlashInfer prefill.cuh compute_sfm_v: rowsum over s_frag_f16), so the weights stay normalised.
      const uint32_t p01 = pack_bf16x2(pv[0], pv[1]), p23 = pack_bf16x2(pv[2], pv[3]);
      const float ps = (bf16lo(p01) + bf16hi(p01)) + (bf16lo(p23) + bf16hi(p23));
      l_run[hh] = l_run[hh] * alpha + ps;
      m_run[hh] = m_new;
#pragma unroll
      for (int j = 0; j < kNT; ++j) {
        o_acc[j][hh * 2] *= alpha;
        o_acc[j][hh * 2 + 1] *= alpha;
      }
      pa[hh] = p01;
      pa[2 + hh] = p23;
    }
    if (kGT == 1) {
      pa[1] = 0;
      pa[3] = 0;
    }
    // ---- O += P V -----------------------------------------------------------
#pragma unroll
    for (int c = 0; c < kVC; ++c) {
      const uint32_t* v0 = &vf[0][c].x;
      const uint32_t* v1 = &vf[1][c].x;
      const uint32_t* v2 = &vf[2][c].x;
      const uint32_t* v3 = &vf[3][c].x;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const uint32_t b0e = __byte_perm(v0[r], v1[r], 0x5410), b1e = __byte_perm(v2[r], v3[r], 0x5410);
        const uint32_t b0o = __byte_perm(v0[r], v1[r], 0x7632), b1o = __byte_perm(v2[r], v3[r], 0x7632);
        mma_bf16_16816(o_acc[c * 8 + 2 * r], pa[0], pa[1], pa[2], pa[3], b0e, b1e);
        mma_bf16_16816(o_acc[c * 8 + 2 * r + 1], pa[0], pa[1], pa[2], pa[3], b0o, b1o);
      }
    }
    if (have_next) cur = nxt;
    blk = nblk_next;
    have = have_next;
  }

  // ---- publish warp state ------------------------------------------------------
#pragma unroll
  for (int hh = 0; hh < kGT; ++hh) {
    float l = l_run[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int h = g + 8 * hh;
    if (t == 0) {
      sm_m[warp * kHeads + h] = m_run[hh];
      sm_l[warp * kHeads + h] = l;
    }
    // lane (g,t) holds, for head h, d in [64c+16t, 64c+16t+16): n-tile j=8c+jj, column
    // 2t+e  <->  d = 64c + 8*(2t+e) + jj.  Two float4 stores per (c,e).
    float* orow = sm_o + ((warp * kHeads + h) * kRS);
#pragma unroll
    for (int c = 0; c < kVC; ++c)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float* dst = orow + 64 * c + 16 * t + 8 * e;
        *reinterpret_cast<float4*>(dst) = make_float4(o_acc[c * 8 + 0][hh * 2 + e], o_acc[c * 8 + 1][hh * 2 + e],
                                                      o_acc[c * 8 + 2][hh * 2 + e], o_acc[c * 8 + 3][hh * 2 + e]);
        *reinterpret_cast<float4*>(dst + 4) = make_float4(o_acc[c * 8 + 4][hh * 2 + e], o_acc[c * 8 + 5][hh * 2 + e],
                                                          o_acc[c * 8 + 6][hh * 2 + e], o_acc[c * 8 + 7][hh * 2 + e]);
      }
  }
  __syncthreads();

  stamp(2);
  // ---- merge warps; each thread owns (head, 4 consecutive d) items ---------------
  constexpr int kItems = kHeads * (kD / 4);
  const bool single = C == 1 && n_splits == 1;
  for (int it = threadIdx.x; it < kItems; it += kWarpsT * 32) {
    const int h = it / (kD / 4), d4 = (it % (kD / 4)) * 4;
    if (h >= nheads) continue;
    float m_tot = -INFINITY;
#pragma unroll
    for (int w = 0; w < kWarpsT; ++w) m_tot = fmaxf(m_tot, sm_m[w * kHeads + h]);
    const float m_safe = m_tot == -INFINITY ? 0.f : m_tot;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    float l_tot = 0.f;
#pragma unroll
    for (int w = 0; w < kWarpsT; ++w) {
      const float sc = fast_exp2(sm_m[w * kHeads + h] - m_safe);
      l_tot += sm_l[w * kHeads + h] * sc;
      const float4 v = *reinterpret_cast<const float4*>(sm_o + ((w * kHeads + h) * kRS) + d4);
      acc.x += v.x * sc;
      acc.y += v.y * sc;
      acc.z += v.z * sc;
      acc.w += v.w * sc;
    }
    const float inv = l_tot > 0.f ? 1.0f / l_tot : 0.f;
    acc.x *= inv; acc.y *= inv; acc.z *= inv; acc.w *= inv;
    const float lse2 = l_tot > 0.f ? m_tot + log2f(l_tot) : -INFINITY;
    const int qh = head0 + h;
    if (single) {
      uint2 ob;
      ob.x = pack_bf16x2(acc.x, acc.y);
      ob.y = pack_bf16x2(acc.z, acc.w);
      *reinterpret_cast<uint2*>(p.o + (int64_t)b * p.o_stride_n + (int64_t)qh * p.o_stride_h + d4) = ob;
      if (p.lse && d4 == 0) p.lse[(int64_t)b * p.num_qo_heads + qh] = lse2;
    } else if (C == 1) {
      const int64_t slot = ((int64_t)b * p.num_qo_heads + qh) * p.max_parts + part;
      *reinterpret_cast<float4*>(p.part_o + slot * kD + d4) = acc;
      if (d4 == 0) p.part_lse[slot] = lse2;
    } else {
      *reinterpret_cast<float4*>(sm_co + h * kD + d4) = acc;
      if (d4 == 0) sm_clse[h] = lse2;
    }
  }
  if (single) return;
  stamp(3);

  // ---- cluster level: reduce-scatter of the C partials through distributed shared memory ---------------------------
  if (C > 1) {
    cluster_arrive_release();
    cluster_wait_acquire();          // every peer's sm_co / sm_clse is complete and visible
    const int rank = (int)cluster_ctarank();
    const int per = (kItems + C - 1) / C;
    const int first = rank * per, lim = min(kItems, first + per);
    const int sub = threadIdx.x & 15, grp = threadIdx.x >> 4;     // 16 lanes = the (up to 16) peers of one item
    const uint32_t co_base = smem_addr_u32(sm_co), clse_base = smem_addr_u32(sm_clse);
    for (int base = first; base < lim; base += kWarpsT * 2) {
      const int it = base + grp;
      const bool item_ok = it < lim;
      const int h = item_ok ? it / (kD / 4) : 0, d4 = item_ok ? (it % (kD / 4)) * 4 : 0;
      const bool head_ok = item_ok && h < nheads;
      float ls = -INFINITY;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (head_ok && sub < C) {
        ls = ld_dsmem_f1(dsmem_addr(clse_base + h * 4, (uint32_t)sub));
        v = ld_dsmem_f4(dsmem_addr(co_base + (h * kD + d4) * 4, (uint32_t)sub));
      }
      float mx = ls;
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float m_safe = mx == -INFINITY ? 0.f : mx;
      const float w = fast_exp2(ls - m_safe);                     // 0 for empty / padding peers
      float wsum = w;
      float4 acc = make_float4(v.x * w, v.y * w, v.z * w, v.w * w);
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {
        wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o);
        acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o);
        acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
      }
      if (head_ok && sub == 0) {
        const float inv = wsum > 0.f ? 1.0f / wsum : 0.f;
        acc.x *= inv; acc.y *= inv; acc.z *= inv; acc.w *= inv;
        const float lse2 = wsum > 0.f ? mx + log2f(wsum) : -INFINITY;
        const int qh = head0 + h;
        if (n_parts == 1) {
          uint2 ob;
          ob.x = pack_bf16x2(acc.x, acc.y);
          ob.y = pack_bf16x2(acc.z, acc.w);
          *reinterpret_cast<uint2*>(p.o + (int64_t)b * p.o_stride_n + (int64_t)qh * p.o_stride_h + d4) = ob;
          if (p.lse && d4 == 0) p.lse[(int64_t)b * p.num_qo_heads + qh] = lse2;
        } else {
          const int64_t slot = ((int64_t)b * p.num_qo_heads + qh) * p.max_parts + part;
          *reinterpret_cast<float4*>(p.part_o + slot * kD + d4) = acc;
          if (d4 == 0) p.part_lse[slot] = lse2;
        }
      }
    }
    cluster_arrive_release();        // this CTA no longer reads its peers' shared memory
    stamp(4);
    if (n_parts == 1) {
      cluster_wait_acquire();        // ... and may exit once no peer reads ITS shared memory any more
      return;
    }
  }

  // ---- the LAST few CTAs of this (request, kv head, head tile) to arrive merge the n_parts partials as a team ------
  // One last-arriver merging everything alone reads n_parts x kHeads x kD floats through a single SM (130 KB for the
  // BASELINE shape: ~4 us).  Instead the last R arrivers (ticket order) each take 1/R of the (head, d) items; the ones
  // that are not the very last spin until the ticket shows every partial published.  Forward progress: at most half of
  // a unit's CTAs ever spin (R <= (n + 1) / 2), the others never wait, and CTAs are dispatched in index order, so the
  // CTAs a spinner waits for are resident or ahead of every spinner in the dispatch queue (the assumption CUB's
  // decoupled look-back makes).
  __syncthreads();
  // One arrival counter per unit, SELF-RESETTING: atomicInc wraps to 0 on the n_arrive-th arrival, so the launch leaves
  // the workspace as it found it without a second atomic on the completion path.  A waiting member sees "everyone has
  // arrived" as "the counter is no longer above my own ticket" (before the wrap it is always >= ticket + 1; the next
  // launch cannot touch it before this grid has completed).
  uint32_t* counter = reinterpret_cast<uint32_t*>(p.counters) + 2 * ((int64_t)b * gridDim.y + blockIdx.y);
  const int n_arrive = n_parts * C;
  if (threadIdx.x == 0) {
    __threadfence();       // one fence after the CTA barrier publishes every thread's partials (cumulativity)
    s_ticket = (int)atomicInc(counter, (uint32_t)(n_arrive - 1));
  }
  __syncthreads();
  const int team = min(kTeam, (n_arrive + 1) >> 1);
  const int member = s_ticket - (n_arrive - team);
  if (member < 0) {
    if (C > 1) cluster_wait_acquire();
    return;
  }
  if (threadIdx.x == 0 && s_ticket != n_arrive - 1) {
    uint32_t seen;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter) : "memory");
    } while (seen > (uint32_t)s_ticket);
  }
  __syncthreads();
  stamp(5);
  // This member's slice of the (head, 4 d) items.  8 lanes share an item and stride over the partials: every lane loads
  // the LSEs and the partial outputs of ITS partials together (all addresses known up front: ONE round trip to L2),
  // the softmax weights across partials are then formed with 8-lane shuffles - no shared memory, no second pass.
  {
    const int n_splits_m = n_parts;
    const int live_items = nheads * (kD / 4);
    const int per = (live_items + team - 1) / team;
    const int first = member * per, lim = min(live_items, first + per);
    const int sub = threadIdx.x & 7, grp = threadIdx.x >> 3;
    for (int base_it = first; base_it < lim; base_it += kWarpsT * 4) {
      const int it = base_it + grp;
      const bool ok = it < lim;
      const int h = ok ? it / (kD / 4) : 0, d4 = ok ? (it % (kD / 4)) * 4 : 0;
      const int qh = head0 + h;
      const int64_t slot0 = ((int64_t)b * p.num_qo_heads + qh) * p.max_parts;
      const float4* src = reinterpret_cast<const float4*>(p.part_o + slot0 * kD + d4);
      const float* lsrc = p.part_lse + slot0;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      float mx = -INFINITY, wsum = 0.f;
      // pass over this lane's partials in batches of 8 (all loads of a batch in flight together: up to 64 partials per
      // item in ONE round trip to L2), keeping a running maximum like the main loop
      constexpr int kB = 8;
      for (int s0 = sub; s0 < n_splits_m; s0 += 8 * kB) {
        float4 v[kB];
        float ls[kB];
#pragma unroll
        for (int u = 0; u < kB; ++u) {
          const int sidx = s0 + 8 * u;
          const bool live = ok && sidx < n_splits_m;
          ls[u] = live ? __ldcg(lsrc + sidx) : -INFINITY;
          v[u] = live ? __ldcg(src + (int64_t)sidx * (kD / 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float m_new = mx;
#pragma unroll
        for (int u = 0; u < kB; ++u) m_new = fmaxf(m_new, ls[u]);
        const float m_safe = m_new == -INFINITY ? 0.f : m_new;
        const float alpha = fast_exp2(mx - m_safe);          // 0 when mx was -inf
        acc.x *= alpha; acc.y *= alpha; acc.z *= alpha; acc.w *= alpha;
        wsum *= alpha;
#pragma unroll
        for (int u = 0; u < kB; ++u) {
          const float w = fast_exp2(ls[u] - m_safe);          // 0 for absent / empty partials
          wsum += w;
          acc.x += v[u].x * w; acc.y += v[u].y * w; acc.z += v[u].z * w; acc.w += v[u].w * w;
        }
        mx = m_new;
      }
      // combine the 8 lanes of the item (fixed xor order: deterministic)
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) {
        const float m_o = __shfl_xor_sync(0xffffffffu, mx, o);
        const float w_o = __shfl_xor_sync(0xffffffffu, wsum, o);
        float4 a_o;
        a_o.x = __shfl_xor_sync(0xffffffffu, acc.x, o);
        a_o.y = __shfl_xor_sync(0xffffffffu, acc.y, o);
        a_o.z = __shfl_xor_sync(0xffffffffu, acc.z, o);
        a_o.w = __shfl_xor_sync(0xffffffffu, acc.w, o);
        const float m_new = fmaxf(mx, m_o);
        const float m_safe = m_new == -INFINITY ? 0.f : m_new;
        const float sa = fast_exp2(mx - m_safe), sb = fast_exp2(m_o - m_safe);
        acc.x = acc.x * sa + a_o.x * sb;
        acc.y = acc.y * sa + a_o.y * sb;
        acc.z = acc.z * sa + a_o.z * sb;
        acc.w = acc.w * sa + a_o.w * sb;
        wsum = wsum * sa + w_o * sb;
        mx = m_new;
      }
      if (ok && sub == 0) {
        const float inv = wsum > 0.f ? 1.0f / wsum : 0.f;
        uint2 ob;
        ob.x = pack_bf16x2(acc.x * inv, acc.y * inv);
        ob.y = pack_bf16x2(acc.z * inv, acc.w * inv);
        *reinterpret_cast<uint2*>(p.o + (int64_t)b * p.o_stride_n + (int64_t)qh * p.o_stride_h + d4) = ob;
        if (p.lse && d4 == 0) p.lse[(int64_t)b * p.num_qo_heads + qh] = wsum > 0.f ? mx + log2f(wsum) : -INFINITY;
      }
    }
  }
  stamp(6);
  if (C > 1) cluster_wait_acquire();
}

namespace {
unsigned long long* g_decode_trace = nullptr;   // debug only (xb_debug_set_decode_trace)
std::atomic<int> g_last_decode_cluster{0};       // debug only (xb_debug_last_decode_cluster)
}

template <int kD, int kGT, int kW>
static int launch_decode_w(DecodeParams& p, int batch, int splits, cudaStream_t stream) {
  constexpr int kHeads = 8 * kGT;
  constexpr size_t smem = ((size_t)kW * kHeads * (kD + 4 + 2) + (size_t)kHeads * (kD + 1) + 3) * sizeof(float);
  constexpr auto kern = paged_decode_kernel<kD, kGT, kW>;
  XB_CUDA_OK(set_max_dynamic_smem_once<kern>((int)smem));
  // largest cluster size this device can co-schedule for this kernel (probed once per instantiation)
  static const int max_cluster = [] {
    // clusters of more than 8 CTAs are "non-portable": allowed explicitly, then verified with an occupancy query
    cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    int max_c = 1;
    for (int c : {16, 8, 4, 2}) {
      cudaLaunchConfig_t cfg{};
      cfg.gridDim = dim3(c, 1, 1);
      cfg.blockDim = dim3(kW * 32);
      cfg.dynamicSmemBytes = smem;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = c;
      at[0].val.clusterDim.y = 1;
      at[0].val.clusterDim.z = 1;
      cfg.attrs = at;
      cfg.numAttrs = 1;
      int n = 0;
      if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) == cudaSuccess && n > 0) {
        max_c = c;
        break;
      }
    }
    cudaGetLastError();   // a failed probe must not poison the next launch's error state
    return max_c;
  }();
  // the plan's cluster size is a request: fall back to per-CTA partials (cluster 1) when the device cannot co-schedule it
  if (p.cluster > max_cluster || splits % p.cluster != 0) p.cluster = 1;
  g_last_decode_cluster.store(p.cluster, std::memory_order_relaxed);
  p.trace = g_decode_trace;
  dim3 grid(splits, p.num_kv_heads * p.head_tiles, batch), block(kW * 32);
  XB_CUDA_OK(launch_cluster(kern, grid, block, smem, stream, true, p.cluster, p));
  return 0;
}

template <int kD, int kGT>
static int launch_decode(DecodeParams& p, int batch, int splits, int cta_warps, cudaStream_t stream) {
  return cta_warps == 4 ? launch_decode_w<kD, kGT, 4>(p, batch, splits, stream)
                        : launch_decode_w<kD, kGT, 8>(p, batch, splits, stream);
}

}  // namespace xb

using namespace xb;

// plan8: [0]=nominal chunk tokens at the planned maximum context (informational: the kernel derives the live value)
//        [1]=splits launched per (request, kv head, head tile) = gridDim.x = clusters x cluster size
//        [2]=float ws bytes [3]=int ws bytes | flags << 32
//        [4]=batch [5]=num_qo_heads [6]=num_kv_heads
//        [7]=head_dim | page_size<<16 | cta_warps<<40 | cluster size<<44
extern "C" int xb_decode_plan(int64_t* plan8, int batch, int num_qo_heads, int num_kv_heads, int head_dim,
                              int page_size, int max_pages_per_request, int num_sms) {
  XB_CHECK(batch > 0 && num_kv_heads > 0 && num_qo_heads % num_kv_heads == 0,
           "decode_plan: bad heads %d/%d or batch %d", num_qo_heads, num_kv_heads, batch);
  XB_CHECK(head_dim == 64 || head_dim == 128, "decode_plan: head_dim %d unsupported (64|128)", head_dim);
  XB_CHECK(page_size > 0 && page_size < 65536 && max_pages_per_request > 0, "decode_plan: bad page geometry");
  if (num_sms <= 0) num_sms = 132;
  const int group = num_qo_heads / num_kv_heads;
  const int head_tiles = (group + 15) / 16;
  const int64_t units = (int64_t)batch * num_kv_heads * head_tiles;
  const int64_t max_kv = (int64_t)max_pages_per_request * page_size;
  const int64_t kMinChunk = 64;
  // one resident CTA per SM; aim for one full wave, chunks are whole 16-token blocks of at least kMinChunk tokens
  int64_t want = num_sms / units;
  if (want < 1) want = 1;
  const int64_t by_len = (max_kv + kMinChunk - 1) / kMinChunk;
  if (want > by_len) want = by_len;
  const int64_t max_splits = 2 * head_dim;   // final-merge scratch in shared memory
  if (want > max_splits) want = max_splits;
  const char* env = getenv("XB_DECODE_CHUNK");     // tuning / tests: force the nominal chunk
  if (env && atoi(env) >= 16) {
    const int64_t chunk = (atoi(env) / 16) * 16;
    want = (max_kv + chunk - 1) / chunk;
    if (want > max_splits) want = max_splits;
  }
  // Cluster geometry: up to 16 splits merge through distributed shared memory inside one cluster; more splits than
  // that use K = ceil(want / 16) clusters whose K results meet in the workspace (last-arriver merge).
  int64_t cluster = 1, parts = want;
  const char* envc = getenv("XB_DECODE_CLUSTER");  // 0 / 1: no clusters (every split is a workspace partial)
  // Default 1 (no clusters): GPCs are unevenly populated, so the device co-schedules fewer large clusters than its SM count
  // suggests and cluster geometries that fill the SMs can run in two waves (tools/decode_sweep.py measures it).  The path
  // stays available.
  const int64_t cmax = envc ? atoi(envc) : 1;
  if (want > 1 && cmax > 1) {
    parts = (want + cmax - 1) / cmax;
    const char* envp = getenv("XB_DECODE_PARTS");  // tuning: force the number of clusters per (request, kv head)
    if (envp && atoi(envp) >= 1 && atoi(envp) <= want) parts = atoi(envp);
    cluster = want / parts;
    if (cluster > cmax) cluster = cmax;
  }
  const int64_t splits = parts * cluster;
  int64_t chunk = (((max_kv + splits - 1) / splits + 15) / 16) * 16;
  if (chunk < kMinChunk) chunk = kMinChunk;
  plan8[0] = chunk;
  plan8[1] = splits;
  // sized for one partial per split so that the launcher may fall back to cluster size 1 on any device
  plan8[2] = splits > 1 ? (int64_t)batch * num_qo_heads * splits * (head_dim + 1) * 4 : 16;
  plan8[3] = units * 8;  // low 32 bits: int workspace bytes (arrival + team-done counter per unit); bit 32: early-prefetch flag (xb_decode_plan_set_flags)
  plan8[4] = batch;
  plan8[5] = num_qo_heads;
  plan8[6] = num_kv_heads;
  // warps per CTA: 8 by default; 4 leaves register room for a co-resident consumer CTA under PDL (XB_DECODE_WARPS)
  int cta_warps = 8;
  const char* envw = getenv("XB_DECODE_WARPS");
  if (envw && atoi(envw) == 4) cta_warps = 4;
  plan8[7] = (int64_t)head_dim | ((int64_t)page_size << 16) | ((int64_t)cta_warps << 40) | (cluster << 44);
  return 0;
}

extern "C" int xb_paged_decode_bf16(const int64_t* plan8, const void* q, int64_t q_stride_n, int64_t q_stride_h,
                                    const void* k_cache, const void* v_cache, int64_t kv_stride_page,
                                    int64_t kv_stride_token, int64_t kv_stride_head, const int32_t* kv_indptr,
                                    const int32_t* kv_indices, const int32_t* kv_last_page_len, void* o,
                                    int64_t o_stride_n, int64_t o_stride_h, float* lse, float sm_scale,
                                    void* workspace_f32, void* workspace_i32, xb_stream_t stream) {
  XB_CHECK(plan8 != nullptr, "paged_decode: plan is null (call xb_decode_plan first)");
  DecodeParams p{};
  const int batch = (int)plan8[4];
  const int head_dim = (int)(plan8[7] & 0xffff);
  p.page_size = (int)((plan8[7] >> 16) & 0xffffff);
  const int cta_warps = (int)((plan8[7] >> 40) & 0xf);
  p.cluster = (int)((plan8[7] >> 44) & 0x1f);
  if (p.cluster < 1) p.cluster = 1;
  p.page_shift = -1;
  if ((p.page_size & (p.page_size - 1)) == 0) {
    int s = 0;
    while ((1 << s) < p.page_size) ++s;
    p.page_shift = s;
  }
  p.num_qo_heads = (int)plan8[5];
  p.num_kv_heads = (int)plan8[6];
  p.group = p.num_qo_heads / p.num_kv_heads;
  p.head_tiles = (p.group + 15) / 16;
  p.min_chunk = 64;
  const int splits = (int)plan8[1];
  p.max_parts = splits;
  XB_CHECK(q_stride_h % 8 == 0 && q_stride_n % 8 == 0 && kv_stride_token % 8 == 0 && kv_stride_head % 8 == 0 &&
               kv_stride_page % 8 == 0 && o_stride_h % 4 == 0 && o_stride_n % 4 == 0,
           "paged_decode: strides must keep 16-byte alignment");
  XB_CHECK(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k_cache) |
             reinterpret_cast<uintptr_t>(v_cache)) & 15) == 0 && (reinterpret_cast<uintptr_t>(o) & 7) == 0,
           "paged_decode: q/k_cache/v_cache must be 16-byte aligned");
  XB_CHECK(splits >= 1 && splits % p.cluster == 0, "paged_decode: corrupt plan (splits %d, cluster %d)", splits, p.cluster);
  XB_CHECK(splits == 1 || (workspace_f32 && workspace_i32), "paged_decode: split-KV needs both workspaces");
  XB_CHECK(splits <= 2 * head_dim, "paged_decode: %d KV splits exceed the merge buffer (max %d)", splits, 2 * head_dim);
  p.q = reinterpret_cast<const __nv_bfloat16*>(q);
  p.q_stride_n = q_stride_n;
  p.q_stride_h = q_stride_h;
  p.k_cache = reinterpret_cast<const __nv_bfloat16*>(k_cache);
  p.v_cache = reinterpret_cast<const __nv_bfloat16*>(v_cache);
  p.stride_page = kv_stride_page;
  p.stride_token = kv_stride_token;
  p.stride_head = kv_stride_head;
  p.kv_indptr = kv_indptr;
  p.kv_indices = kv_indices;
  p.kv_last_page_len = kv_last_page_len;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.o_stride_n = o_stride_n;
  p.o_stride_h = o_stride_h;
  p.lse = lse;
  p.scale_log2 = sm_scale * 1.44269504088896340736f;
  p.part_o = reinterpret_cast<float*>(workspace_f32);
  p.part_lse = p.part_o ? p.part_o + (int64_t)batch * p.num_qo_heads * p.max_parts * head_dim : nullptr;
  p.counters = reinterpret_cast<int32_t*>(workspace_i32);
  p.early_prefetch = (int)(plan8[3] >> 32) & 1;
  cudaStream_t s = (cudaStream_t)stream;
  const bool wide = p.group > 8;
  if (head_dim == 128)
    return wide ? launch_decode<128, 2>(p, batch, splits, cta_warps, s) : launch_decode<128, 1>(p, batch, splits, cta_warps, s);
  if (head_dim == 64)
    return wide ? launch_decode<64, 2>(p, batch, splits, cta_warps, s) : launch_decode<64, 1>(p, batch, splits, cta_warps, s);
  XB_CHECK(false, "paged_decode: head_dim %d unsupported", head_dim);
  return 1;
}

// flags bit 0: early prefetch - the caller guarantees that KV rows other than the newest token of each request, and the
// paged triplet, are not written by any kernel still in flight when this one is launched (true for the decode step:
// the only producer in flight is RoPE+scatter of the newest token).  The kernel then fetches KV before the PDL wait.
extern "C" int xb_decode_plan_set_flags(int64_t* plan8, int flags) {
  XB_CHECK(plan8 != nullptr, "decode_plan_set_flags: null plan");
  plan8[3] = (plan8[3] & 0xffffffffll) | ((int64_t)(flags & 1) << 32);
  return 0;
}

// debug: how many clusters of `cluster` CTAs of the (head_dim 128, group <= 8, 8 warps) kernel the device co-schedules.
extern "C" int xb_debug_max_active_clusters(int cluster) {
  auto kern = paged_decode_kernel<128, 1, 8>;
  const size_t smem = ((size_t)8 * 8 * (128 + 4 + 2) + (size_t)8 * (128 + 1) + 3) * sizeof(float);
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cluster, 1, 1);
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = cluster;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) {
    cudaGetLastError();
    return -1;
  }
  return n;
}

// debug: cluster size (CTAs along the split axis) of the most recent paged_decode launch of this process, after the
// fall-back to 1 when the device cannot co-schedule the planned size; 0 before the first launch.
extern "C" int xb_debug_last_decode_cluster() { return g_last_decode_cluster.load(std::memory_order_relaxed); }

// debug: per-CTA stage timestamps (%globaltimer, ns) of the next paged_decode launches: buf = uint64[ctas][8], or null.
extern "C" int xb_debug_set_decode_trace(void* buf) {
  g_decode_trace = reinterpret_cast<unsigned long long*>(buf);
  return 0;
}
