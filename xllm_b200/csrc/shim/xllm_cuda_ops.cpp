// Link-time drop-in for the reference's CUDA operator namespace:
//   namespace xllm::kernel::cuda  --  xllm/core/kernels/cuda/cuda_ops_api.h:31-216
// Same function names, argument order, in-place / returned-tensor conventions and error behaviour (TORCH_CHECK ->
// c10::Error, as the reference tests rely on: tests/core/kernels/cuda/cutlass_scaled_mm_test.cpp:279-295).  Each
// function unwraps the borrowed torch::Tensor arguments (data_ptr / strides / current CUDA stream) and forwards to the
// C ABI of libxllm_b200_ops.so (include/xllm_b200_ops.h).  To use it, drop this file into xllm/core/kernels/cuda/ in
// place of {norm,rope,activation,reshape_paged_cache,fp8_quant}.cu, matmul.cpp, fp8_scaled_{quantize,matmul}.cpp and
// cutlass_w8a8/, and link libxllm_b200_ops.so (see INTEGRATION.md).  Attention is served through the TVM-FFI modules
// (csrc/ffi/tvm_ffi_modules.cc), which needs no source change in xLLM at all.
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAGraphsUtils.cuh>
#include <c10/cuda/CUDAGuard.h>
#include <torch/torch.h>

#include <algorithm>
#include <optional>
#include <string>
#include <tuple>
#include <vector>

#include "../../../include/xllm_b200_ops.h"

namespace xllm::kernel::cuda {

namespace {
inline void* stream() { return at::cuda::getCurrentCUDAStream().stream(); }
inline void ok(int rc, const char* what) { TORCH_CHECK(rc == 0, what, ": ", xb_last_error()); }
// The reference dispatches on fp16 / bf16 / fp32 (DISPATCH_FLOATING_TYPES); this library implements the serving dtype
// only, so every tensor argument is checked and an unsupported dtype raises instead of being reinterpreted.
inline void need_bf16(const torch::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kBFloat16, name,
              " must be a CUDA bfloat16 tensor (xllm_b200 implements bfloat16 only), got ", t.scalar_type());
}
inline void need_dtype(const torch::Tensor& t, torch::ScalarType st, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == st, name, " must be a CUDA tensor of ", st, ", got ", t.scalar_type());
}
#define XB_GUARD(t) const at::cuda::OptionalCUDAGuard device_guard(device_of(t))
}  // namespace

// cuda_ops_api.h:31-37
void rotary_embedding(torch::Tensor& positions, torch::Tensor& query, std::optional<torch::Tensor> key,
                      torch::Tensor& cos_sin_cache, bool is_neox) {
  need_bf16(query, "query");
  need_bf16(cos_sin_cache, "cos_sin_cache");
  if (key.has_value()) need_bf16(*key, "key");
  const int64_t head_size = cos_sin_cache.size(-1);
  const int64_t num_tokens = positions.numel();
  TORCH_CHECK(positions.scalar_type() == torch::kInt64, "positions must be int64");
  TORCH_CHECK(query.size(0) == positions.size(0) && (!key.has_value() || key->size(0) == positions.size(0)),
              "query, key and positions must have the same number of tokens");
  const int64_t q_hidden = query.numel() / num_tokens;
  const int64_t k_hidden = key.has_value() ? key->numel() / num_tokens : 0;
  TORCH_CHECK(q_hidden % head_size == 0 && k_hidden % head_size == 0);
  const int num_heads = q_hidden / head_size;
  const int num_kv_heads = key.has_value() ? k_hidden / head_size : num_heads;
  const int64_t head_stride = query.dim() == positions.dim() + 2 ? query.stride(-2) : head_size;
  const at::cuda::OptionalCUDAGuard guard(device_of(query));
  ok(xb_rotary_embedding_bf16(positions.data_ptr<int64_t>(), query.data_ptr(), key.has_value() ? key->data_ptr() : nullptr,
                              cos_sin_cache.data_ptr(), (int)cos_sin_cache.size(1), query.stride(positions.dim() - 1),
                              key.has_value() ? key->stride(positions.dim() - 1) : 0, head_stride, num_heads, num_kv_heads,
                              (int)head_size, is_neox ? 1 : 0, (int)num_tokens, stream()),
     "rotary_embedding");
}

// cuda_ops_api.h:39-42
void act_and_mul(torch::Tensor out, torch::Tensor input, const std::string& act_mode) {
  int mode = act_mode == "silu" ? 0 : act_mode == "gelu" ? 1 : (act_mode == "gelu_tanh" || act_mode == "gelu_pytorch_tanh") ? 2 : -1;
  TORCH_CHECK(mode >= 0, "Unsupported act mode: ", act_mode, ", only support silu, gelu, gelu_tanh, gelu_pytorch_tanh");
  need_bf16(input, "input");
  need_bf16(out, "out");
  TORCH_CHECK(input.is_contiguous() && out.is_contiguous(), "act_and_mul: tensors must be contiguous");
  const int d = input.size(-1) / 2;
  const int64_t tokens = input.numel() / input.size(-1);
  const at::cuda::OptionalCUDAGuard guard(device_of(input));
  ok(xb_act_and_mul_bf16(out.data_ptr(), input.data_ptr(), d, (int)tokens, mode, stream()), "act_and_mul");
}

// cuda_ops_api.h:44-49
void reshape_paged_cache(torch::Tensor slot_ids, torch::Tensor keys, torch::Tensor values, torch::Tensor key_cache,
                         torch::Tensor value_cache) {
  need_bf16(keys, "keys");
  need_bf16(values, "values");
  need_bf16(key_cache, "key_cache");
  need_bf16(value_cache, "value_cache");
  need_dtype(slot_ids, torch::kInt32, "slot_ids");
  TORCH_CHECK(key_cache.is_contiguous() && value_cache.is_contiguous(), "caches must be contiguous");
  XB_GUARD(keys);
  TORCH_CHECK(keys.stride(-1) == 1 && keys.stride(-2) == keys.size(-1));
  TORCH_CHECK(values.stride(-1) == 1 && values.stride(-2) == values.size(-1));
  ok(xb_reshape_paged_cache_bf16(slot_ids.data_ptr<int>(), keys.data_ptr(), values.data_ptr(), key_cache.data_ptr(),
                                 value_cache.data_ptr(), keys.stride(-3), values.stride(-3), (int)keys.size(-2),
                                 (int)keys.size(-1), (int)key_cache.size(-3), (int)keys.size(-3), stream()),
     "reshape_paged_cache");
}

// cuda_ops_api.h:157-160
void rms_norm(torch::Tensor output, torch::Tensor input, torch::Tensor weight, double eps) {
  need_bf16(input, "input");
  need_bf16(output, "output");
  need_bf16(weight, "weight");
  TORCH_CHECK(output.is_contiguous(), "output must be contiguous");
  TORCH_CHECK(input.stride(-1) == 1);
  // norm.cu:436-441: inputs with more than 2 dims are made contiguous so that one row stride describes them
  if (input.dim() > 2 && !input.is_contiguous()) input = input.contiguous();
  XB_GUARD(input);
  const int hidden = input.size(-1);
  ok(xb_rms_norm_bf16(output.data_ptr(), input.data_ptr(), input.dim() >= 2 ? input.stride(-2) : hidden, weight.data_ptr(), (float)eps,
                      (int)(input.numel() / hidden), hidden, stream()),
     "rms_norm");
}

// cuda_ops_api.h:162-165
void fused_add_rms_norm(torch::Tensor& input, torch::Tensor& residual, torch::Tensor& weight, double epsilon) {
  need_bf16(input, "input");
  need_bf16(residual, "residual");
  need_bf16(weight, "weight");
  TORCH_CHECK(input.stride(-1) == 1 && residual.is_contiguous());
  TORCH_CHECK(input.dim() <= 2 || input.is_contiguous(), "fused_add_rms_norm: input with more than 2 dims must be contiguous");
  XB_GUARD(input);
  const int hidden = input.size(-1);
  ok(xb_fused_add_rms_norm_bf16(input.data_ptr(), input.stride(-2), residual.data_ptr(), weight.data_ptr(), (float)epsilon,
                                (int)(input.numel() / hidden), hidden, stream()),
     "fused_add_rms_norm");
}

// cuda_ops_api.h:167-169 (matmul.cpp:20-24: F::linear)
torch::Tensor matmul(torch::Tensor a, torch::Tensor b, std::optional<torch::Tensor> bias) {
  need_bf16(a, "a");
  need_bf16(b, "b");
  if (bias.has_value() && bias->defined()) need_bf16(*bias, "bias");
  TORCH_CHECK(b.dim() == 2 && b.is_contiguous() && a.size(-1) == b.size(1), "matmul: b must be a contiguous [N, K] weight");
  XB_GUARD(a);
  auto a2 = a.reshape({-1, a.size(-1)});
  if (a2.stride(-1) != 1) a2 = a2.contiguous();
  const int64_t M = a2.size(0), K = a2.size(1), N = b.size(0);
  auto out = torch::empty({M, N}, a.options());
  const void* bp = bias.has_value() && bias->defined() ? bias->data_ptr() : nullptr;
  if (M <= 16 && K % 32 == 0)
    ok(xb_linear_bf16_small_m(out.data_ptr(), N, a2.data_ptr(), a2.stride(0), b.data_ptr(), bp, (int)M, (int)N, (int)K, stream()),
       "matmul");
  else
    ok(xb_gemm_bf16(out.data_ptr(), N, a2.data_ptr(), a2.stride(0), b.data_ptr(), bp, (int)M, (int)N, (int)K, stream()), "matmul");
  auto shape = a.sizes().vec();
  shape.back() = N;
  return out.view(shape);
}

// cuda_ops_api.h:171-176 (cutlass_w8a8/scaled_mm_entry.cu:55-108)
void cutlass_scaled_mm(torch::Tensor& c, torch::Tensor const& a, torch::Tensor const& b, torch::Tensor const& a_scales,
                       torch::Tensor const& b_scales, std::optional<torch::Tensor> const& bias) {
  TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && c.dim() == 2);
  TORCH_CHECK(c.size(0) == a.size(0) && a.size(1) == b.size(0) && b.size(1) == c.size(1));
  TORCH_CHECK(a.stride(1) == 1 && c.stride(1) == 1);  // Row-major
  TORCH_CHECK(b.stride(0) == 1);                      // Column-major
  TORCH_CHECK(c.stride(0) % 16 == 0 && b.stride(1) % 16 == 0);
  // the C ABI takes the weight as a dense [N, K] matrix (ldb == K): a padded column-major b is rejected, not misread
  TORCH_CHECK(b.stride(1) == a.size(1), "cutlass_scaled_mm: b must be a dense column-major [K, N] view (stride(1) == K), got ",
              b.stride(1));
  TORCH_CHECK(a_scales.is_contiguous() && b_scales.is_contiguous());
  need_dtype(a_scales, torch::kFloat32, "a_scales");
  need_dtype(b_scales, torch::kFloat32, "b_scales");
  TORCH_CHECK((a_scales.numel() == 1 || a_scales.numel() == a.size(0)) && (b_scales.numel() == 1 || b_scales.numel() == b.size(1)),
              "scale numel must be 1 or M / N");
  if (bias) need_bf16(*bias, "bias");
  if (bias) TORCH_CHECK(bias->numel() == b.size(1) && bias->is_contiguous() && bias->dim() == 1);
  TORCH_CHECK(a.scalar_type() == torch::kFloat8_e4m3fn && b.scalar_type() == torch::kFloat8_e4m3fn, "fp8 e4m3 inputs expected");
  TORCH_CHECK(c.scalar_type() == torch::kBFloat16, "only bfloat16 output is implemented");
  const at::cuda::OptionalCUDAGuard guard(device_of(a));
  {
    // split-K workspace of the decode-sized GEMM: owned here, registered once per process (xLLM runs one process per GPU) on
    // the first call that is not inside a stream capture (the setter clears the ticket words with a synchronous memset)
    static torch::Tensor splitk_ws;
    if (!splitk_ws.defined() && a.size(0) <= 64 &&
        at::cuda::currentStreamCaptureStatus() == at::cuda::CaptureStatus::None) {
      const auto bytes = (int64_t)xb_gemm_splitk_workspace_bytes();
      splitk_ws = torch::empty({bytes}, torch::TensorOptions().dtype(torch::kUInt8).device(a.device()));
      ok(xb_set_gemm_splitk_workspace(splitk_ws.data_ptr(), (size_t)bytes), "cutlass_scaled_mm (split-K workspace)");
    }
  }
  if (a.size(0) <= 8 && b.size(1) <= 16384 && a.size(1) % 64 == 0) {
    // decode on a narrow projection: the HBM-streaming swap-AB kernel (the reference's small-M buckets,
    // c3x/scaled_mm_sm100_fp8_dispatch.cuh:148-287); measured crossover in xllm_b200/ops.py
    ok(xb_linear_fp8_small_m(c.data_ptr(), c.stride(0), a.data_ptr(), a.stride(0), b.data_ptr(), a_scales.data_ptr<float>(),
                             (int)a_scales.numel(), b_scales.data_ptr<float>(), (int)b_scales.numel(),
                             bias ? bias->data_ptr() : nullptr, (int)a.size(0), (int)b.size(1), (int)a.size(1), stream()),
       "cutlass_scaled_mm");
    return;
  }
  ok(xb_gemm_fp8_scaled(c.data_ptr(), c.stride(0), a.data_ptr(), a.stride(0), b.data_ptr(), a_scales.data_ptr<float>(),
                        (int)a_scales.numel(), b_scales.data_ptr<float>(), (int)b_scales.numel(),
                        bias ? bias->data_ptr() : nullptr, (int)a.size(0), (int)b.size(1), (int)a.size(1), stream()),
     "cutlass_scaled_mm");
}

// cuda_ops_api.h:182-186
void static_scaled_fp8_quant(torch::Tensor& out, torch::Tensor const& input, torch::Tensor const& scale) {
  TORCH_CHECK(input.stride(-1) == 1, "last dimension of input must be contiguous");
  TORCH_CHECK(out.stride(-1) == 1, "last dimension of output must be contiguous");
  need_bf16(input, "input");
  need_dtype(out, torch::kFloat8_e4m3fn, "out");
  need_dtype(scale, torch::kFloat32, "scale");
  TORCH_CHECK(input.dim() >= 2 && out.dim() >= 2, "static_scaled_fp8_quant: [tokens, hidden] tensors expected");
  XB_GUARD(input);
  const int hidden = input.size(-1);
  ok(xb_static_scaled_fp8_quant_bf16(out.data_ptr(), out.stride(-2), input.data_ptr(), input.stride(-2),
                                     scale.data_ptr<float>(), (int)(input.numel() / hidden), hidden, stream()),
     "static_scaled_fp8_quant");
}

// cuda_ops_api.h:188-193 (fp8_scaled_quantize.cpp:20-48) - the dynamic scale is computed on the device, no host sync
std::tuple<torch::Tensor, torch::Tensor> fp8_scaled_quantize(const torch::Tensor& input, const std::optional<torch::Tensor>& output,
                                                             const std::optional<torch::Tensor>& scale) {
  torch::Tensor out = output.has_value() && output->defined() ? *output
                                                              : torch::empty_like(input, input.options().dtype(torch::kFloat8_e4m3fn));
  if (scale.has_value() && scale->defined()) {
    static_scaled_fp8_quant(out, input, *scale);
    return {out, *scale};
  }
  need_bf16(input, "input");
  need_dtype(out, torch::kFloat8_e4m3fn, "output");
  TORCH_CHECK(input.stride(-1) == 1 && out.stride(-1) == 1 && input.dim() >= 2, "fp8_scaled_quantize: [tokens, hidden] row-major tensors expected");
  XB_GUARD(input);
  auto s = torch::empty({1}, input.options().dtype(torch::kFloat32));
  const int hidden = input.size(-1);
  ok(xb_dynamic_scaled_fp8_quant_bf16(out.data_ptr(), out.stride(-2), input.data_ptr(), input.stride(-2), s.data_ptr<float>(),
                                      (int)(input.numel() / hidden), hidden, stream()),
     "fp8_scaled_quantize");
  return {out, s};
}

// cuda_ops_api.h:203-221
void rms_norm_static_fp8_quant(torch::Tensor& out, torch::Tensor& input, torch::Tensor& weight, torch::Tensor& scale, double epsilon) {
  need_bf16(input, "input");
  need_bf16(weight, "weight");
  need_dtype(out, torch::kFloat8_e4m3fn, "out");
  need_dtype(scale, torch::kFloat32, "scale");
  TORCH_CHECK(out.is_contiguous() && input.stride(-1) == 1 && input.dim() >= 2);
  XB_GUARD(input);
  const int hidden = input.size(-1);
  ok(xb_rms_norm_static_fp8_quant_bf16(out.data_ptr(), input.data_ptr(), input.stride(-2), weight.data_ptr(),
                                       scale.data_ptr<float>(), (float)epsilon, (int)(input.numel() / hidden), hidden, stream()),
     "rms_norm_static_fp8_quant");
}
void fused_add_rms_norm_static_fp8_quant(torch::Tensor& out, torch::Tensor& input, torch::Tensor& residual, torch::Tensor& weight,
                                         torch::Tensor& scale, double epsilon) {
  need_bf16(input, "input");
  need_bf16(residual, "residual");
  need_bf16(weight, "weight");
  need_dtype(out, torch::kFloat8_e4m3fn, "out");
  need_dtype(scale, torch::kFloat32, "scale");
  TORCH_CHECK(out.is_contiguous() && residual.is_contiguous() && input.stride(-1) == 1 && input.dim() >= 2);
  XB_GUARD(input);
  const int hidden = input.size(-1);
  ok(xb_fused_add_rms_norm_static_fp8_quant_bf16(out.data_ptr(), input.data_ptr(), input.stride(-2), residual.data_ptr(),
                                                 weight.data_ptr(), scale.data_ptr<float>(), (float)epsilon,
                                                 (int)(input.numel() / hidden), hidden, stream()),
     "fused_add_rms_norm_static_fp8_quant");
}

// cuda_ops_api.h:223-233 (fp8_scaled_matmul.cpp:20-45)
torch::Tensor fp8_scaled_matmul(const torch::Tensor& a, const torch::Tensor& b, const torch::Tensor& a_scale,
                                const torch::Tensor& b_scale, torch::ScalarType output_dtype,
                                const std::optional<torch::Tensor>& bias, const std::optional<torch::Tensor>& output) {
  TORCH_CHECK(output_dtype == torch::kBFloat16, "only bfloat16 output is implemented");
  torch::Tensor out = output.has_value() && output->defined() ? *output : torch::empty({a.size(0), b.size(0)}, a.options().dtype(output_dtype));
  cutlass_scaled_mm(out, a, b.t(), a_scale, b_scale, bias);
  return out;
}

// cuda_ops_api.h:252-266
void fused_qk_norm_rope(torch::Tensor& qkv, int64_t num_heads_q, int64_t num_heads_k, int64_t num_heads_v, int64_t head_dim,
                        double eps, const torch::Tensor& q_weight, const torch::Tensor& k_weight, const torch::Tensor& cos_sin_cache,
                        bool interleaved, const torch::Tensor& position_ids) {
  need_bf16(qkv, "qkv");
  need_bf16(q_weight, "q_weight");
  need_bf16(k_weight, "k_weight");
  need_bf16(cos_sin_cache, "cos_sin_cache");
  TORCH_CHECK(qkv.is_contiguous() && position_ids.scalar_type() == torch::kInt64);
  XB_GUARD(qkv);
  ok(xb_fused_qk_norm_rope_bf16(qkv.data_ptr(), (int)num_heads_q, (int)num_heads_k, (int)num_heads_v, (int)head_dim, (float)eps,
                                q_weight.data_ptr(), k_weight.data_ptr(), cos_sin_cache.data_ptr(), (int)cos_sin_cache.size(-1),
                                interleaved ? 1 : 0, position_ids.data_ptr<int64_t>(), (int)qkv.size(0), stream()),
     "fused_qk_norm_rope");
}

// ---- additive boundary (SURVEY 8b-3): weight-only linears; the reference has no such op ---------------------------
torch::Tensor w4a16_linear(const torch::Tensor& x, const torch::Tensor& qweight, const torch::Tensor& meta, int64_t group_size,
                           const std::optional<torch::Tensor>& bias) {
  need_bf16(x, "x");
  need_dtype(qweight, torch::kInt32, "qweight");
  need_dtype(meta, torch::kInt32, "meta");
  if (bias.has_value() && bias->defined()) need_bf16(*bias, "bias");
  XB_GUARD(x);
  auto x2 = x.reshape({-1, x.size(-1)});
  if (x2.stride(-1) != 1) x2 = x2.contiguous();
  const int64_t M = x2.size(0), K = x2.size(1), N = meta.size(1);
  auto out = torch::empty({M, N}, x.options());
  const void* bp = bias.has_value() && bias->defined() ? bias->data_ptr() : nullptr;
  auto* qw = reinterpret_cast<const uint32_t*>(qweight.data_ptr());
  auto* mt = reinterpret_cast<const uint32_t*>(meta.data_ptr());
  if (M <= 16)
    ok(xb_linear_w4a16_small_m(out.data_ptr(), N, x2.data_ptr(), x2.stride(0), qw, mt, bp, (int)M, (int)N, (int)K, (int)group_size, stream()),
       "w4a16_linear");
  else
    ok(xb_gemm_w4a16(out.data_ptr(), N, x2.data_ptr(), x2.stride(0), qw, mt, bp, (int)M, (int)N, (int)K, (int)group_size, stream()),
       "w4a16_linear");
  auto shape = x.sizes().vec();
  shape.back() = N;
  return out.view(shape);
}

torch::Tensor w8a16_linear(const torch::Tensor& x, const torch::Tensor& qweight, const torch::Tensor& meta, int64_t group_size,
                           const std::optional<torch::Tensor>& bias) {
  need_bf16(x, "x");
  need_dtype(qweight, torch::kInt32, "qweight");
  need_dtype(meta, torch::kInt32, "meta");
  if (bias.has_value() && bias->defined()) need_bf16(*bias, "bias");
  XB_GUARD(x);
  auto x2 = x.reshape({-1, x.size(-1)});
  if (x2.stride(-1) != 1) x2 = x2.contiguous();
  const int64_t M = x2.size(0), K = x2.size(1), N = meta.size(1);
  auto out = torch::empty({M, N}, x.options());
  const void* bp = bias.has_value() && bias->defined() ? bias->data_ptr() : nullptr;
  auto* qw = reinterpret_cast<const uint32_t*>(qweight.data_ptr());
  auto* mt = reinterpret_cast<const uint32_t*>(meta.data_ptr());
  if (M <= 16)
    ok(xb_linear_w8a16_small_m(out.data_ptr(), N, x2.data_ptr(), x2.stride(0), qw, mt, bp, (int)M, (int)N, (int)K, (int)group_size, stream()),
       "w8a16_linear");
  else
    ok(xb_gemm_w8a16(out.data_ptr(), N, x2.data_ptr(), x2.stride(0), qw, mt, bp, (int)M, (int)N, (int)K, (int)group_size, stream()),
       "w8a16_linear");
  auto shape = x.sizes().vec();
  shape.back() = N;
  return out.view(shape);
}


// ---- kernels/cuda/llm_decode_metadata_update.h:35-58 (same struct, same entry point) -------------------------------------
struct LlmDecodeMetadataUpdateParams {
  const int32_t* src_tokens;
  const int32_t* src_positions;
  const int32_t* src_new_cache_slots;
  const int32_t* src_kv_seq_lens;
  const int32_t* src_paged_kv_indptr;
  const int32_t* src_paged_kv_indices;
  const int32_t* src_paged_kv_last_page_len;
  int32_t* dst_tokens;
  int32_t* dst_positions;
  int32_t* dst_new_cache_slots;
  int32_t* dst_kv_seq_lens;
  int32_t* dst_kv_seq_lens_delta;
  int32_t* dst_paged_kv_indptr;
  int32_t* dst_paged_kv_indices;
  int32_t* dst_paged_kv_last_page_len;
  int64_t actual_num_tokens;
  int64_t padded_num_tokens;
  int64_t actual_batch_size;
  int64_t actual_indices_size;
};
using LlmDecodeMetadataUpdateStream = cudaStream_t;

void update_llm_decode_metadata(const LlmDecodeMetadataUpdateParams& p, LlmDecodeMetadataUpdateStream stream) {
  ok(xb_decode_metadata_update(p.src_tokens, p.src_positions, p.src_new_cache_slots, p.src_kv_seq_lens, p.src_paged_kv_indptr,
                               p.src_paged_kv_indices, p.src_paged_kv_last_page_len, p.dst_tokens, p.dst_positions,
                               p.dst_new_cache_slots, p.dst_kv_seq_lens, p.dst_kv_seq_lens_delta, p.dst_paged_kv_indptr,
                               p.dst_paged_kv_indices, p.dst_paged_kv_last_page_len, p.actual_num_tokens, p.padded_num_tokens,
                               p.actual_batch_size, p.actual_indices_size, nullptr, 0, (xb_stream_t)stream),
     "update_llm_decode_metadata");
}


// ---- cuda_ops_api.h:251-256 ------------------------------------------------------------------------------------------------
std::tuple<torch::Tensor, torch::Tensor> moe_fused_topk(torch::Tensor& gating_output, int64_t topk, bool renormalize,
                                                        const std::optional<torch::Tensor>& correction_bias,
                                                        const std::string& scoring_func) {
  TORCH_CHECK(scoring_func == "softmax" || scoring_func == "sigmoid", "Unsupported scoring function for moe topk: ", scoring_func,
              "only softmax and sigmoid are supported");
  TORCH_CHECK(gating_output.is_cuda() && gating_output.dim() == 2 && gating_output.stride(1) == 1, "gating_output [tokens, experts]");
  const bool is_bf16 = gating_output.scalar_type() == torch::kBFloat16;
  TORCH_CHECK(is_bf16 || gating_output.scalar_type() == torch::kFloat32, "moe_fused_topk: gating_output must be float32 or bfloat16");
  XB_GUARD(gating_output);
  const int64_t T = gating_output.size(0);
  auto w = torch::empty({T, topk}, torch::dtype(torch::kFloat32).device(gating_output.device()));
  auto ids = torch::empty({T, topk}, torch::dtype(torch::kInt32).device(gating_output.device()));
  const bool sig = scoring_func == "sigmoid";
  const float* bias = nullptr;
  if (sig && correction_bias.has_value() && correction_bias->defined()) {       // dropped on the softmax path (moe_fused_topk.cu:36-43)
    TORCH_CHECK(correction_bias->scalar_type() == torch::kFloat32 && correction_bias->is_contiguous(), "correction_bias must be float32");
    bias = correction_bias->data_ptr<float>();
  }
  ok(xb_moe_fused_topk(w.data_ptr<float>(), ids.data_ptr<int32_t>(), gating_output.data_ptr(), is_bf16 ? 1 : 0, gating_output.stride(0),
                       bias, (int)T, (int)gating_output.size(1), (int)topk, renormalize ? 1 : 0, sig ? 1 : 0, stream()),
     "moe_fused_topk");
  return std::make_tuple(w, ids);
}

// ---- cuda_ops_api.h:260-289 (utils.h:61-71 ActivationType) -------------------------------------------------------------------
enum class ActivationType : int8_t { GELU = 0, RELU = 1, SILU = 2, SWIGLU = 3, GEGLU = 4, SWIGLU_BIAS = 5, RELU2 = 6, IDENTITY = 7, INVALID_TYPE = 8 };

torch::Tensor cutlass_fused_moe(const torch::Tensor& input, const torch::Tensor& token_selected_experts,
                                const torch::Tensor& token_final_scales, const torch::Tensor& fc1_expert_weights,
                                const torch::Tensor& fc2_expert_weights, torch::ScalarType output_dtype,
                                const std::vector<torch::Tensor>& quant_scales, int32_t tp_size, int32_t tp_rank, int32_t ep_size,
                                int32_t ep_rank, int32_t cluster_size, int32_t cluster_rank,
                                const std::optional<torch::Tensor>& fc1_expert_biases, const std::optional<torch::Tensor>& fc2_expert_biases,
                                const std::optional<torch::Tensor>& input_sf, const std::optional<torch::Tensor>& swiglu_alpha,
                                const std::optional<torch::Tensor>& swiglu_beta, const std::optional<torch::Tensor>& swiglu_limit,
                                const std::optional<torch::Tensor>& output, bool enable_alltoall, bool use_deepseek_fp8_block_scale,
                                bool use_w4_group_scaling, bool use_mxfp8_act_scaling, bool min_latency_mode, bool use_packed_weights,
                                int32_t /*tune_max_num_tokens*/, ActivationType activation_type) {
  // what layers/cuda/fused_moe.cpp:97-115 asks for: bf16 experts, no quant scales, SwiGLU, result reduction by the caller
  TORCH_CHECK(quant_scales.empty() && !use_deepseek_fp8_block_scale && !use_w4_group_scaling && !use_mxfp8_act_scaling &&
                  !use_packed_weights && !input_sf.has_value(),
              "cutlass_fused_moe: only unquantized bf16 experts are supported");
  TORCH_CHECK(!fc1_expert_biases.has_value() && !fc2_expert_biases.has_value() && !swiglu_alpha.has_value() &&
                  !swiglu_beta.has_value() && !swiglu_limit.has_value(),
              "cutlass_fused_moe: expert biases / swiglu alpha, beta, limit are not supported");
  TORCH_CHECK(activation_type == ActivationType::SWIGLU, "cutlass_fused_moe: only SWIGLU experts are supported");
  TORCH_CHECK(!enable_alltoall && !min_latency_mode && cluster_size == 1 && cluster_rank == 0, "cutlass_fused_moe: unsupported mode");
  TORCH_CHECK(output_dtype == torch::kBFloat16 && input.scalar_type() == torch::kBFloat16 &&
                  fc1_expert_weights.scalar_type() == torch::kBFloat16 && fc2_expert_weights.scalar_type() == torch::kBFloat16,
              "cutlass_fused_moe: bf16 only");
  TORCH_CHECK(token_selected_experts.scalar_type() == torch::kInt32 && token_final_scales.scalar_type() == torch::kFloat32,
              "cutlass_fused_moe: ids int32 / scales float32");
  TORCH_CHECK(input.dim() == 2 && input.stride(1) == 1 && fc1_expert_weights.is_contiguous() && fc2_expert_weights.is_contiguous() &&
                  token_selected_experts.is_contiguous() && token_final_scales.is_contiguous(),
              "cutlass_fused_moe: layout");
  (void)tp_size; (void)tp_rank;            // the intermediate dimension is already this rank's slice (load_experts)
  XB_GUARD(input);
  const int64_t T = input.size(0), H = fc2_expert_weights.size(1), I = fc2_expert_weights.size(2), El = fc1_expert_weights.size(0);
  const int64_t k = token_selected_experts.size(1);
  torch::Tensor out = (output.has_value() && output->defined()) ? *output : torch::empty({T, H}, input.options());
  const int64_t need = xb_moe_experts_workspace_bytes((int)T, (int)k, (int)H, (int)I);
  auto ws = torch::empty({need}, torch::dtype(torch::kUInt8).device(input.device()));
  ok(xb_moe_experts_bf16(out.data_ptr(), out.stride(0), input.data_ptr(), input.stride(0), token_selected_experts.data_ptr<int32_t>(),
                         token_final_scales.data_ptr<float>(), fc1_expert_weights.data_ptr(), fc2_expert_weights.data_ptr(), (int)T,
                         (int)k, (int)H, (int)I, (int)El, (int)(ep_rank * El), ws.data_ptr(), need, stream()),
     "cutlass_fused_moe");
  (void)ep_size;
  return out;
}

// ---- MLA (additive: the CUDA two-cache layout of kv_cache_shape.cpp:242-257,273-288) ----------------------------------------
// fused_mla_kv (ops_api.h:112, FusedMlaKVParams param.h:1105-1180) for quant_mode "none" and a paged cache: input_kv
// [T, 576] = [c_kv | k_pe], gamma [512], position_id int64 [T], the [cos | sin] table [max_pos, 64] the CUDA RoPE ops use,
// k_cache = ckv_cache [blocks, block_size, (1,) 512], v_cache = kpe_cache [blocks, block_size, (1,) 64].
void fused_mla_kv(const torch::Tensor& input_kv, const torch::Tensor& cos_sin_cache, const torch::Tensor& position_id,
                  const torch::Tensor& gamma, torch::Tensor& k_cache, torch::Tensor& v_cache, const torch::Tensor& slot_mapping,
                  const std::string& quant_mode, double eps, bool interleaved) {
  TORCH_CHECK(quant_mode == "none", "fused_mla_kv: only quant_mode \"none\" is supported, got ", quant_mode);
  need_bf16(input_kv, "input_kv");
  need_bf16(cos_sin_cache, "cos_sin_cache");
  need_bf16(gamma, "gamma");
  need_bf16(k_cache, "k_cache");
  need_bf16(v_cache, "v_cache");
  need_dtype(position_id, torch::kInt64, "position_id");
  need_dtype(slot_mapping, torch::kInt32, "slot_mapping");
  const auto in = input_kv.reshape({-1, input_kv.size(-1)});
  TORCH_CHECK(in.stride(1) == 1, "fused_mla_kv: input_kv rows must be contiguous");
  const int64_t T = in.size(0);
  TORCH_CHECK(position_id.numel() == T && slot_mapping.numel() == T, "fused_mla_kv: position_id / slot_mapping need one entry per token");
  const auto ckv = k_cache.reshape({k_cache.size(0), k_cache.size(1), -1});
  const auto kpe = v_cache.reshape({v_cache.size(0), v_cache.size(1), -1});
  TORCH_CHECK(ckv.stride(2) == 1 && kpe.stride(2) == 1 && in.size(1) == ckv.size(2) + kpe.size(2) &&
                  cos_sin_cache.size(-1) == kpe.size(2) && gamma.numel() == ckv.size(2),
              "fused_mla_kv: shapes: input_kv [T, ", in.size(1), "], k_cache rows ", ckv.size(2), ", v_cache rows ", kpe.size(2));
  XB_GUARD(input_kv);
  ok(xb_mla_cache_latent_bf16(in.data_ptr(), in.stride(0), gamma.data_ptr(), (float)eps, position_id.data_ptr<int64_t>(),
                              cos_sin_cache.data_ptr(), interleaved ? 1 : 0, slot_mapping.data_ptr<int32_t>(), ckv.data_ptr(),
                              ckv.stride(0), ckv.stride(1), kpe.data_ptr(), kpe.stride(0), kpe.stride(1), (int)ckv.size(2),
                              (int)kpe.size(2), (int)ckv.size(1), (int)T, stream()),
     "fused_mla_kv");
}

// Absorbed MLA attention over the two paged caches: q_nope [T, H, 512], q_pe [T, H, 64] (any strides with unit last dim),
// the ragged q / paged kv quadruple int32 on device, output [T, H, 512].  Plans (host-only) for max_qo_len and allocates
// the split workspace when the plan asks for one; layers that capture graphs call the C ABI with a persistent plan.
void mla_paged_attention(const torch::Tensor& q_nope, const torch::Tensor& q_pe, const torch::Tensor& ckv_cache,
                         const torch::Tensor& kpe_cache, const torch::Tensor& qo_indptr, const torch::Tensor& paged_kv_indptr,
                         const torch::Tensor& paged_kv_indices, const torch::Tensor& paged_kv_last_page_len, int64_t max_qo_len,
                         double sm_scale, bool causal, torch::Tensor& output) {
  need_bf16(q_nope, "q_nope");
  need_bf16(q_pe, "q_pe");
  need_bf16(ckv_cache, "ckv_cache");
  need_bf16(kpe_cache, "kpe_cache");
  need_bf16(output, "output");
  need_dtype(qo_indptr, torch::kInt32, "qo_indptr");
  need_dtype(paged_kv_indptr, torch::kInt32, "paged_kv_indptr");
  need_dtype(paged_kv_indices, torch::kInt32, "paged_kv_indices");
  need_dtype(paged_kv_last_page_len, torch::kInt32, "paged_kv_last_page_len");
  TORCH_CHECK(q_nope.dim() == 3 && q_pe.dim() == 3 && output.dim() == 3 && q_nope.size(0) == q_pe.size(0) &&
                  q_nope.size(1) == q_pe.size(1) && output.size(0) == q_nope.size(0) && output.size(1) == q_nope.size(1),
              "mla_paged_attention: q_nope / q_pe / output must be [T, H, D] with equal T and H");
  TORCH_CHECK(q_nope.stride(2) == 1 && q_pe.stride(2) == 1 && output.stride(2) == 1, "mla_paged_attention: last dims must be contiguous");
  const auto ckv = ckv_cache.reshape({ckv_cache.size(0), ckv_cache.size(1), -1});
  const auto kpe = kpe_cache.reshape({kpe_cache.size(0), kpe_cache.size(1), -1});
  TORCH_CHECK(ckv.stride(2) == 1 && kpe.stride(2) == 1 && output.size(2) == ckv.size(2) && q_nope.size(2) == ckv.size(2) &&
                  q_pe.size(2) == kpe.size(2),
              "mla_paged_attention: q_nope / output width must equal the ckv_cache row, q_pe width the kpe_cache row");
  const int64_t batch = paged_kv_indptr.numel() - 1;
  TORCH_CHECK(batch >= 1 && qo_indptr.numel() == batch + 1 && paged_kv_last_page_len.numel() == batch,
              "mla_paged_attention: qo_indptr [B+1], paged_kv_indptr [B+1], paged_kv_last_page_len [B]");
  XB_GUARD(q_nope);
  int64_t plan[8];
  const int max_pages = (int)std::max<int64_t>(1, paged_kv_indices.numel());
  ok(xb_mla_plan(plan, (int)batch, (int)q_nope.size(1), (int)ckv.size(2), (int)kpe.size(2), (int)max_qo_len, (int)ckv.size(1),
                 max_pages, at::cuda::getCurrentDeviceProperties()->multiProcessorCount),
     "mla_paged_attention");
  torch::Tensor ws;
  if (plan[1] > 0) ws = torch::empty({plan[1]}, torch::dtype(torch::kUInt8).device(q_nope.device()));
  ok(xb_mla_paged_attention_bf16(plan, q_nope.data_ptr(), q_nope.stride(0), q_nope.stride(1), q_pe.data_ptr(), q_pe.stride(0),
                                 q_pe.stride(1), ckv.data_ptr(), ckv.stride(0), ckv.stride(1), kpe.data_ptr(), kpe.stride(0),
                                 kpe.stride(1), qo_indptr.data_ptr<int32_t>(), paged_kv_indptr.data_ptr<int32_t>(),
                                 paged_kv_indices.data_ptr<int32_t>(), paged_kv_last_page_len.data_ptr<int32_t>(), causal ? 1 : 0,
                                 output.data_ptr(), output.stride(0), output.stride(1), (float)sm_scale,
                                 ws.defined() ? ws.data_ptr() : nullptr, plan[1], stream()),
     "mla_paged_attention");
}

}  // namespace xllm::kernel::cuda
