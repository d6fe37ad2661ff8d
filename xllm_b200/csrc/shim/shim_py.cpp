// Test-side Python binding of the link-time drop-in (csrc/shim/xllm_cuda_ops.cpp): the xllm::kernel::cuda::* functions, called
// with torch tensors exactly as xLLM's layers call them, so that tests can exercise the C++ boundary itself - argument checks
// that raise c10::Error (the reference's tests rely on that: tests/core/kernels/cuda/cutlass_scaled_mm_test.cpp:279-295) and,
// on a GPU, the same launches as the ctypes driver.  Not part of the product; built by xllm_b200/build_shim.py::build_py().
#include <torch/extension.h>

#include <optional>
#include <string>
#include <tuple>

namespace xllm::kernel::cuda {
// declarations as in cuda_ops_api.h:31-266 (defined in xllm_cuda_ops.cpp)
void rotary_embedding(torch::Tensor& positions, torch::Tensor& query, std::optional<torch::Tensor> key, torch::Tensor& cos_sin_cache,
                      bool is_neox);
void act_and_mul(torch::Tensor out, torch::Tensor input, const std::string& act_mode);
void reshape_paged_cache(torch::Tensor slot_ids, torch::Tensor keys, torch::Tensor values, torch::Tensor key_cache,
                         torch::Tensor value_cache);
void rms_norm(torch::Tensor output, torch::Tensor input, torch::Tensor weight, double eps);
void fused_add_rms_norm(torch::Tensor& input, torch::Tensor& residual, torch::Tensor& weight, double epsilon);
torch::Tensor matmul(torch::Tensor a, torch::Tensor b, std::optional<torch::Tensor> bias);
void cutlass_scaled_mm(torch::Tensor& c, torch::Tensor const& a, torch::Tensor const& b, torch::Tensor const& a_scales,
                       torch::Tensor const& b_scales, std::optional<torch::Tensor> const& bias);
void static_scaled_fp8_quant(torch::Tensor& out, torch::Tensor const& input, torch::Tensor const& scale);
std::tuple<torch::Tensor, torch::Tensor> fp8_scaled_quantize(const torch::Tensor& input, const std::optional<torch::Tensor>& output,
                                                             const std::optional<torch::Tensor>& scale);
void rms_norm_static_fp8_quant(torch::Tensor& out, torch::Tensor& input, torch::Tensor& weight, torch::Tensor& scale, double epsilon);
void fused_add_rms_norm_static_fp8_quant(torch::Tensor& out, torch::Tensor& input, torch::Tensor& residual, torch::Tensor& weight,
                                         torch::Tensor& scale, double epsilon);
void fused_qk_norm_rope(torch::Tensor& qkv, int64_t num_heads_q, int64_t num_heads_k, int64_t num_heads_v, int64_t head_dim, double eps,
                        const torch::Tensor& q_weight, const torch::Tensor& k_weight, const torch::Tensor& cos_sin_cache,
                        bool interleaved, const torch::Tensor& position_ids);
std::tuple<torch::Tensor, torch::Tensor> moe_fused_topk(torch::Tensor& gating_output, int64_t topk, bool renormalize,
                                                        const std::optional<torch::Tensor>& correction_bias,
                                                        const std::string& scoring_func);
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
                                int32_t tune_max_num_tokens, ActivationType activation_type);
void fused_mla_kv(const torch::Tensor& input_kv, const torch::Tensor& cos_sin_cache, const torch::Tensor& position_id,
                  const torch::Tensor& gamma, torch::Tensor& k_cache, torch::Tensor& v_cache, const torch::Tensor& slot_mapping,
                  const std::string& quant_mode, double eps, bool interleaved);
void mla_paged_attention(const torch::Tensor& q_nope, const torch::Tensor& q_pe, const torch::Tensor& ckv_cache,
                         const torch::Tensor& kpe_cache, const torch::Tensor& qo_indptr, const torch::Tensor& paged_kv_indptr,
                         const torch::Tensor& paged_kv_indices, const torch::Tensor& paged_kv_last_page_len, int64_t max_qo_len,
                         double sm_scale, bool causal, torch::Tensor& output);
}  // namespace xllm::kernel::cuda

namespace xk = xllm::kernel::cuda;

PYBIND11_MODULE(xllm_b200_shim_py, m) {
  m.doc() = "xllm::kernel::cuda::* of libxllm_b200_shim.so (test binding)";
  m.def("rotary_embedding", [](torch::Tensor positions, torch::Tensor query, std::optional<torch::Tensor> key,
                               torch::Tensor cos_sin_cache, bool is_neox) { xk::rotary_embedding(positions, query, key, cos_sin_cache, is_neox); });
  m.def("act_and_mul", [](torch::Tensor out, torch::Tensor input, const std::string& mode) { xk::act_and_mul(out, input, mode); });
  m.def("reshape_paged_cache", [](torch::Tensor slot_ids, torch::Tensor keys, torch::Tensor values, torch::Tensor key_cache,
                                  torch::Tensor value_cache) { xk::reshape_paged_cache(slot_ids, keys, values, key_cache, value_cache); });
  m.def("rms_norm", [](torch::Tensor output, torch::Tensor input, torch::Tensor weight, double eps) { xk::rms_norm(output, input, weight, eps); });
  m.def("fused_add_rms_norm", [](torch::Tensor input, torch::Tensor residual, torch::Tensor weight, double eps) {
    xk::fused_add_rms_norm(input, residual, weight, eps);
  });
  m.def("matmul", [](torch::Tensor a, torch::Tensor b, std::optional<torch::Tensor> bias) { return xk::matmul(a, b, bias); });
  m.def("cutlass_scaled_mm", [](torch::Tensor c, torch::Tensor a, torch::Tensor b, torch::Tensor a_scales, torch::Tensor b_scales,
                                std::optional<torch::Tensor> bias) { xk::cutlass_scaled_mm(c, a, b, a_scales, b_scales, bias); });
  m.def("static_scaled_fp8_quant", [](torch::Tensor out, torch::Tensor input, torch::Tensor scale) { xk::static_scaled_fp8_quant(out, input, scale); });
  m.def("fp8_scaled_quantize", [](torch::Tensor input, std::optional<torch::Tensor> output, std::optional<torch::Tensor> scale) {
    return xk::fp8_scaled_quantize(input, output, scale);
  });
  m.def("rms_norm_static_fp8_quant", [](torch::Tensor out, torch::Tensor input, torch::Tensor weight, torch::Tensor scale, double eps) {
    xk::rms_norm_static_fp8_quant(out, input, weight, scale, eps);
  });
  m.def("fused_add_rms_norm_static_fp8_quant", [](torch::Tensor out, torch::Tensor input, torch::Tensor residual, torch::Tensor weight,
                                                  torch::Tensor scale, double eps) {
    xk::fused_add_rms_norm_static_fp8_quant(out, input, residual, weight, scale, eps);
  });
  m.def("fused_qk_norm_rope", [](torch::Tensor qkv, int64_t hq, int64_t hk, int64_t hv, int64_t head_dim, double eps, torch::Tensor qw,
                                 torch::Tensor kw, torch::Tensor cos_sin, bool interleaved, torch::Tensor pos) {
    xk::fused_qk_norm_rope(qkv, hq, hk, hv, head_dim, eps, qw, kw, cos_sin, interleaved, pos);
  });
  m.def("moe_fused_topk", [](torch::Tensor gating, int64_t topk, bool renormalize, std::optional<torch::Tensor> bias,
                             const std::string& scoring) { return xk::moe_fused_topk(gating, topk, renormalize, bias, scoring); });
  // the arguments layers/cuda/fused_moe.cpp:97-115 passes: bf16 experts, no quantisation, SwiGLU, the caller reduces over TP / EP
  m.def("cutlass_fused_moe", [](torch::Tensor input, torch::Tensor ids, torch::Tensor scales, torch::Tensor fc1, torch::Tensor fc2,
                                int64_t ep_size, int64_t ep_rank) {
    return xk::cutlass_fused_moe(input, ids, scales, fc1, fc2, torch::kBFloat16, {}, 1, 0, (int32_t)ep_size, (int32_t)ep_rank, 1, 0,
                                 std::nullopt, std::nullopt, std::nullopt, std::nullopt, std::nullopt, std::nullopt, std::nullopt,
                                 false, false, false, false, false, false, 0, xk::ActivationType::SWIGLU);
  }, pybind11::arg("input"), pybind11::arg("token_selected_experts"), pybind11::arg("token_final_scales"),
     pybind11::arg("fc1_expert_weights"), pybind11::arg("fc2_expert_weights"), pybind11::arg("ep_size") = 1,
     pybind11::arg("ep_rank") = 0);
  m.def("fused_mla_kv", [](torch::Tensor input_kv, torch::Tensor cos_sin_cache, torch::Tensor position_id, torch::Tensor gamma,
                           torch::Tensor k_cache, torch::Tensor v_cache, torch::Tensor slot_mapping, const std::string& quant_mode,
                           double eps, bool interleaved) {
    xk::fused_mla_kv(input_kv, cos_sin_cache, position_id, gamma, k_cache, v_cache, slot_mapping, quant_mode, eps, interleaved);
  });
  m.def("mla_paged_attention", [](torch::Tensor q_nope, torch::Tensor q_pe, torch::Tensor ckv_cache, torch::Tensor kpe_cache,
                                  torch::Tensor qo_indptr, torch::Tensor kv_indptr, torch::Tensor kv_indices, torch::Tensor kv_last_page_len,
                                  int64_t max_qo_len, double sm_scale, bool causal, torch::Tensor output) {
    xk::mla_paged_attention(q_nope, q_pe, ckv_cache, kpe_cache, qo_indptr, kv_indptr, kv_indices, kv_last_page_len, max_qo_len,
                            sm_scale, causal, output);
  });
}
