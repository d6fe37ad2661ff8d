// Tensor-parallel exchange for the row-parallel linears (o_proj, down_proj) over NVLink peer memory.
// Replaces parallel_state::reduce -> ProcessGroup::allreduce (c10d NCCL) at
//   xllm/core/layers/common/linear.cpp:1518-1520 -> framework/parallel_state/parallel_state.cpp:183-192
// for decode-sized messages, where 2 x L NCCL launches per step are latency-, not bandwidth-, bound.
//
// Every rank's row-parallel GEMV writes its partial [T, H] straight into a SYMMETRIC buffer (same allocation on every
// GPU, peer-mapped through NVLink/NVSwitch).  Two kernels consume it:
//   * allreduce_add_rms_norm : ONE kernel = flag barrier + pull the `world` partials over NVLink + sum (fixed rank
//     order, fp32: bit-identical on every rank) + residual add + RMSNorm (+ the next layer's input).  The all-reduce is
//     fused into the fused_add_rms_norm that follows every row-parallel linear in the decoder layer
//     (qwen2_decoder_layer.cpp:103-109), so TP adds NO launches to the step.
//   * oneshot_allreduce      : the plain exchange (same barrier + pull + sum), for call sites without a norm.
// Barrier: CTA b of rank r stores an increasing epoch into flag[b][r] of every peer (st.release.sys) and spins on its
// own flag[b][p] (ld.acquire.sys).  The epoch lives in device memory, so CUDA-graph replays keep working.  Buffers are
// reused safely without a trailing barrier because consecutive exchanges alternate between two symmetric buffers
// (o_proj -> A, down_proj -> B): a rank can only overwrite A again after it has passed the barrier of the exchange
// on B, which every peer enters only after finishing its reads of A.
// Large (prefill) messages stay on NCCL (ring / NVLS moves 2(P-1)/P of the payload instead of (P-1) x).
#include "common.cuh"

namespace xb {

constexpr int kMaxRanks = 8;

struct PeerPtrs {
  const __nv_bfloat16* data[kMaxRanks];   // peer-mapped partial buffers (index = rank)
  uint32_t* flags[kMaxRanks];             // peer-mapped signal pads: [max_ctas][kMaxRanks] uint32
  uint32_t* epoch;                        // local: [max_ctas]
  int rank, world;
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// all ranks have launched this exchange (=> their producer kernels have completed and their partials are visible)
__device__ __forceinline__ void peer_barrier(const PeerPtrs& pp) {
  __shared__ uint32_t s_target;
  if (threadIdx.x == 0) {
    const uint32_t target = pp.epoch[blockIdx.x] + 1;
    pp.epoch[blockIdx.x] = target;
    s_target = target;
  }
  __syncthreads();
  const uint32_t target = s_target;
  if (threadIdx.x < pp.world) {
    const int peer = threadIdx.x;
    st_release_sys(pp.flags[peer] + blockIdx.x * kMaxRanks + pp.rank, target);
    const uint32_t* mine = pp.flags[pp.rank] + blockIdx.x * kMaxRanks + peer;
    while ((int32_t)(ld_acquire_sys(mine) - target) < 0) {
    }
  }
  __syncthreads();
}

__device__ __forceinline__ void sum_peers(const PeerPtrs& pp, int64_t elem_off, float (&acc)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  uint4 v[kMaxRanks];
#pragma unroll
  for (int r = 0; r < kMaxRanks; ++r)
    if (r < pp.world) v[r] = *reinterpret_cast<const uint4*>(pp.data[r] + elem_off);   // NVLink loads, all in flight
#pragma unroll
  for (int r = 0; r < kMaxRanks; ++r)
    if (r < pp.world) {
      const uint32_t* w = &v[r].x;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[2 * j] += bf16lo(w[j]);
        acc[2 * j + 1] += bf16hi(w[j]);
      }
    }
}

__global__ void __launch_bounds__(512)
oneshot_allreduce_kernel(__nv_bfloat16* __restrict__ out, const PeerPtrs pp, int64_t n_vec /* 8-element vectors */) {
  pdl_launch_dependents();
  pdl_wait();
  peer_barrier(pp);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_vec; i += (int64_t)gridDim.x * blockDim.x) {
    float acc[8];
    sum_peers(pp, i * 8, acc);
    uint4 o;
    o.x = pack_bf16x2(acc[0], acc[1]);
    o.y = pack_bf16x2(acc[2], acc[3]);
    o.z = pack_bf16x2(acc[4], acc[5]);
    o.w = pack_bf16x2(acc[6], acc[7]);
    reinterpret_cast<uint4*>(out)[i] = o;
  }
}

// out[t,:] = rms_norm( bf16(sum_r partial_r[t,:]) + residual[t,:] ) ; residual <- that sum (fused_add_rms_norm semantics,
// norm.cu:80-136, applied to the all-reduced row).  One CTA per token, hidden % 8 == 0.
__global__ void __launch_bounds__(1024)
allreduce_add_rms_norm_kernel(__nv_bfloat16* __restrict__ out, __nv_bfloat16* __restrict__ residual,
                              const __nv_bfloat16* __restrict__ weight, const PeerPtrs pp, float eps, int hidden) {
  __shared__ float red[33];
  pdl_launch_dependents();
  pdl_wait();
  peer_barrier(pp);
  const int64_t tok = blockIdx.x;
  const int nvec = hidden >> 3;
  constexpr int kMaxVec = 2;
  uint4 zr[kMaxVec];
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < kMaxVec; ++k) {
    const int idx = threadIdx.x + k * blockDim.x;
    if (idx < nvec) {
      float acc[8];
      sum_peers(pp, tok * hidden + (int64_t)idx * 8, acc);
      const uint4 rv = reinterpret_cast<const uint4*>(residual + tok * hidden)[idx];
      const uint32_t* rp = &rv.x;
      uint4 z;
      uint32_t* zp = &z.x;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        // all-reduce result rounded to bf16 (what the reference's NCCL sum returns), then the bf16 residual add
        const float a = round_bf16(acc[2 * j]) + bf16lo(rp[j]);
        const float b = round_bf16(acc[2 * j + 1]) + bf16hi(rp[j]);
        zp[j] = pack_bf16x2(a, b);
        const float za = bf16lo(zp[j]), zb = bf16hi(zp[j]);
        ss += za * za + zb * zb;
      }
      reinterpret_cast<uint4*>(residual + tok * hidden)[idx] = z;
      zr[k] = z;
    }
  }
  // the residual add, squares and block sum above are add_bf16x8 / sumsq_bf16x8 / block_sum written out on the fp32
  // all-reduce sums (through the helpers this kernel compiles to different code); tests/test_gpu_peer_exchange.py holds
  // it bit-identical to oneshot_allreduce followed by fused_add_rms_norm
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < ((blockDim.x + 31) >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) red[32] = t;
  }
  __syncthreads();
  const float rstd = rms_rstd(red[32], hidden, eps);
#pragma unroll
  for (int k = 0; k < kMaxVec; ++k) {
    const int idx = threadIdx.x + k * blockDim.x;
    if (idx < nvec) {
      reinterpret_cast<uint4*>(out + tok * hidden)[idx] =
          rms_apply_bf16x8(zr[k], __ldg(reinterpret_cast<const uint4*>(weight) + idx), rstd);
    }
  }
}

}  // namespace xb

using namespace xb;

static inline bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// The kernels move data as uint4 and signals / epochs as uint32: a misaligned pointer would fault the GPU, so it is refused.
static int fill_peers(PeerPtrs& pp, const void* const* peer_data, void* const* peer_flags, void* epoch, int rank, int world) {
  XB_CHECK(world >= 1 && world <= kMaxRanks && rank >= 0 && rank < world, "allreduce: bad rank %d / world %d", rank, world);
  for (int r = 0; r < world; ++r) {
    XB_CHECK(aligned(peer_data[r], 16), "allreduce: peer_data[%d] %p is not 16-byte aligned", r, peer_data[r]);
    XB_CHECK(aligned(peer_flags[r], 4), "allreduce: peer_flags[%d] %p is not 4-byte aligned", r, peer_flags[r]);
  }
  XB_CHECK(aligned(epoch, 4), "allreduce: epoch %p is not 4-byte aligned", epoch);
  for (int r = 0; r < kMaxRanks; ++r) {
    pp.data[r] = r < world ? reinterpret_cast<const __nv_bfloat16*>(peer_data[r]) : nullptr;
    pp.flags[r] = r < world ? reinterpret_cast<uint32_t*>(peer_flags[r]) : nullptr;
  }
  pp.epoch = reinterpret_cast<uint32_t*>(epoch);
  pp.rank = rank;
  pp.world = world;
  return 0;
}

extern "C" int xb_oneshot_allreduce_bf16(void* out, const void* const* peer_data, void* const* peer_flags, void* epoch,
                                         int rank, int world, int64_t numel, int max_ctas, xb_stream_t stream) {
  if (numel == 0) return 0;
  XB_CHECK(numel % 8 == 0, "oneshot_allreduce: numel %lld must be a multiple of 8", (long long)numel);
  XB_CHECK(numel > 0, "oneshot_allreduce: numel %lld must not be negative", (long long)numel);
  XB_CHECK(max_ctas >= 1, "oneshot_allreduce: max_ctas %d must be at least 1", max_ctas);
  PeerPtrs pp;
  if (fill_peers(pp, peer_data, peer_flags, epoch, rank, world)) return 1;
  XB_CHECK(aligned(out, 16), "oneshot_allreduce: out %p is not 16-byte aligned", out);
  int64_t n_vec = numel / 8;
  int ctas = (int)((n_vec + 511) / 512);
  if (ctas > max_ctas) ctas = max_ctas;
  XB_CUDA_OK(launch(oneshot_allreduce_kernel, dim3(ctas), dim3(512), 0, (cudaStream_t)stream, true,
                    reinterpret_cast<__nv_bfloat16*>(out), pp, n_vec));
  return 0;
}

extern "C" int xb_allreduce_add_rms_norm_bf16(void* out, void* residual, const void* weight, const void* const* peer_data,
                                              void* const* peer_flags, void* epoch, int rank, int world, float eps,
                                              int num_tokens, int hidden, int max_ctas, xb_stream_t stream) {
  if (num_tokens == 0) return 0;
  XB_CHECK(hidden > 0 && hidden % 8 == 0 && hidden <= 16384,
           "allreduce_add_rms_norm: hidden %d must be a positive multiple of 8 and <= 16384", hidden);
  XB_CHECK(num_tokens <= max_ctas, "allreduce_add_rms_norm: %d tokens exceed the %d flag slots (use NCCL for prefill-sized messages)",
           num_tokens, max_ctas);
  XB_CHECK(num_tokens > 0, "allreduce_add_rms_norm: num_tokens %d must not be negative", num_tokens);
  PeerPtrs pp;
  if (fill_peers(pp, peer_data, peer_flags, epoch, rank, world)) return 1;
  XB_CHECK(aligned(out, 16) && aligned(residual, 16) && aligned(weight, 16),
           "allreduce_add_rms_norm: out %p / residual %p / weight %p must be 16-byte aligned", out, residual, weight);
  int threads = ((hidden / 8 + 31) / 32) * 32;
  if (threads > 1024) threads = 1024;
  XB_CUDA_OK(launch(allreduce_add_rms_norm_kernel, dim3(num_tokens), dim3(threads), 0, (cudaStream_t)stream, true,
                    reinterpret_cast<__nv_bfloat16*>(out), reinterpret_cast<__nv_bfloat16*>(residual),
                    reinterpret_cast<const __nv_bfloat16*>(weight), pp, eps, hidden));
  return 0;
}
