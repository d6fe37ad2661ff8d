// TVM-FFI SafeCall modules that xLLM dlopen()s IN PLACE OF FlashInfer's AOT modules
// (xllm/core/kernels/cuda/utils.cpp:371-374,526-564: "$FLASHINFER_OPS_PATH/<uri>/<uri>.so", symbols
//  __tvm_ffi_plan / __tvm_ffi_run / __tvm_ffi_paged_run / __tvm_ffi_ragged_run).
// Argument lists are FlashInfer v0.6.x's (flashinfer/data/csrc/batch_decode_jit_binding.cu:23-44,
// batch_prefill_jit_binding.cu:22-52) exactly as the reference passes them:
//   decode  plan : flashinfer_planinfo.cpp:318-335      run       : batch_decode.cpp:64-84
//   prefill plan : flashinfer_planinfo.cpp:145-164,227-245
//           ragged_run : batch_prefill.cpp:100-128      paged_run : batch_chunked_prefill.cpp:63-91
// Tensors arrive as borrowed DLPack views; the CUDA stream is the one the host bound with TVMFFIEnvSetStream
// (utils.h:147-161).  Everything forwards to the C ABI of libxllm_b200_ops.so; plan_info is opaque to xLLM
// (deep-copied only: flashinfer_planinfo.cpp:37-62), so it carries this library's own int64 layout.
// Build: see xllm_b200/build_ffi.py (decode, prefill and FA3-form prefill modules, installed under their URI directories).
#include <cuda_runtime.h>
#include <tvm/ffi/container/array.h>
#include <tvm/ffi/container/tensor.h>
#include <tvm/ffi/error.h>
#include <tvm/ffi/extra/c_env_api.h>
#include <tvm/ffi/function.h>
#include <tvm/ffi/optional.h>

#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstring>

#include "../../../include/xllm_b200_ops.h"

using tvm::ffi::Array;
using tvm::ffi::Optional;
using tvm::ffi::TensorView;

namespace {

inline cudaStream_t stream_of(const TensorView& t) {
  return static_cast<cudaStream_t>(TVMFFIEnvGetStream(t.device().device_type, t.device().device_id));
}
inline void* ptr(const TensorView& t) { return static_cast<char*>(t.data_ptr()) + t.byte_offset(); }
inline void check_rc(int rc, const char* what) {
  if (rc != 0) TVM_FFI_THROW(RuntimeError) << what << ": " << xb_last_error();
}
inline bool is_bf16(const TensorView& t) { return t.dtype().code == kDLBfloat && t.dtype().bits == 16; }

// ---------------------------------------------------------------------------------------------------------------
// decode planning shared by the decode module's `plan` and the prefill module's `plan` (the reference serves decode
// through the PREFILL module's paged_run when should_use_tensor_core() holds - GQA group >= 4, i.e. Qwen2-7B and
// Llama-3: kernels/cuda/utils.cpp:349-367, batch_decode.cpp:43-60)
// ---------------------------------------------------------------------------------------------------------------
void make_decode_plan(int64_t* plan, const TensorView& float_ws, const TensorView& int_ws, const int32_t* indptr_host,
                      int64_t batch_size, int64_t num_qo_heads, int64_t num_kv_heads, int64_t page_size, int64_t head_dim,
                      bool enable_cuda_graph) {
  int64_t max_pages = 1;
  for (int64_t b = 0; b < batch_size; ++b) max_pages = std::max<int64_t>(max_pages, indptr_host[b + 1] - indptr_host[b]);
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (enable_cuda_graph) {
    // The plan made at capture is replayed for later, longer steps (flashinfer_attention.cpp:306-311 skips `plan` under
    // replay; cuda_graph_executor_impl.cpp:751-822).  The kernel derives the split size from the live kv_len on the
    // device, so only the split COUNT is fixed here: size it for the SM count alone, as if the context were long.
    max_pages = std::max<int64_t>(max_pages, (int64_t)64 * sms / page_size + 1);
  }
  check_rc(xb_decode_plan(plan, (int)batch_size, (int)num_qo_heads, (int)num_kv_heads, (int)head_dim, (int)page_size,
                          (int)max_pages, sms), "decode plan");
  const int64_t need_f = plan[2], need_i = plan[3] & 0xffffffffll;
  if (need_f > float_ws.numel() * (float_ws.dtype().bits / 8))
    TVM_FFI_THROW(RuntimeError) << "float workspace too small: need " << need_f << " bytes";
  if (need_i > int_ws.numel() * (int_ws.dtype().bits / 8))
    TVM_FFI_THROW(RuntimeError) << "int workspace too small: need " << need_i << " bytes";
  // split tickets live at the start of the int workspace and must start at zero (the kernel restores them)
  cudaMemsetAsync(ptr(int_ws), 0, (size_t)need_i, stream_of(int_ws));
}

// ---------------------------------------------------------------------------------------------------------------
// decode module
// ---------------------------------------------------------------------------------------------------------------
Array<int64_t> DecodePlan(TensorView float_ws, TensorView int_ws, TensorView pinned_int_ws, TensorView indptr_host,
                          int64_t batch_size, int64_t num_qo_heads, int64_t num_kv_heads, int64_t page_size,
                          bool enable_cuda_graph, int64_t window_left, double logits_soft_cap, int64_t head_dim_qk,
                          int64_t head_dim_vo, TensorView empty_q, TensorView empty_kv) {
  (void)pinned_int_ws; (void)empty_q; (void)empty_kv;
  if (window_left >= 0) TVM_FFI_THROW(ValueError) << "sliding window attention is not implemented";
  if (logits_soft_cap > 0) TVM_FFI_THROW(ValueError) << "logits soft cap is not implemented";
  if (head_dim_qk != head_dim_vo) TVM_FFI_THROW(ValueError) << "head_dim_qk != head_dim_vo";
  const int32_t* ip = static_cast<const int32_t*>(ptr(indptr_host));   // host tensor (flashinfer_planinfo.cpp:310-311)
  int64_t plan[8];
  make_decode_plan(plan, float_ws, int_ws, ip, batch_size, num_qo_heads, num_kv_heads, page_size, head_dim_qk,
                   enable_cuda_graph);
  Array<int64_t> out;
  for (int i = 0; i < 8; ++i) out.push_back(plan[i]);
  return out;
}

void DecodeRun(TensorView float_ws, TensorView int_ws, Array<int64_t> plan_vec, TensorView q, TensorView k_cache,
               TensorView v_cache, TensorView kv_indptr, TensorView kv_indices, TensorView kv_last_page_len, TensorView o,
               Optional<TensorView> maybe_lse, int64_t kv_layout_code, int64_t window_left, bool enable_pdl,
               Optional<TensorView> maybe_alibi_slopes, double logits_soft_cap, double sm_scale, double rope_rcp_scale,
               double rope_rcp_theta) {
  (void)rope_rcp_scale; (void)rope_rcp_theta;
  if (plan_vec.size() != 8) TVM_FFI_THROW(ValueError) << "plan_info has " << plan_vec.size() << " entries, expected 8";
  if (!is_bf16(q) || !is_bf16(k_cache) || !is_bf16(o)) TVM_FFI_THROW(TypeError) << "only bf16 q/kv/o is implemented";
  if (maybe_alibi_slopes.has_value()) TVM_FFI_THROW(ValueError) << "alibi is not implemented";
  if (window_left >= 0 || logits_soft_cap > 0) TVM_FFI_THROW(ValueError) << "sliding window / soft cap not implemented";
  int64_t plan[8];
  for (int i = 0; i < 8; ++i) plan[i] = plan_vec[i];
  xb_set_pdl(enable_pdl ? 1 : 0);
  // kv_layout_code 0 = NHD [pages, page, heads, d], 1 = HND [pages, heads, page, d]
  const int64_t st_page = k_cache.stride(0);
  const int64_t st_tok = kv_layout_code == 0 ? k_cache.stride(1) : k_cache.stride(2);
  const int64_t st_head = kv_layout_code == 0 ? k_cache.stride(2) : k_cache.stride(1);
  float* lse = maybe_lse.has_value() ? static_cast<float*>(ptr(maybe_lse.value())) : nullptr;
  check_rc(xb_paged_decode_bf16(plan, ptr(q), q.stride(0), q.stride(1), ptr(k_cache), ptr(v_cache), st_page, st_tok, st_head,
                                static_cast<const int32_t*>(ptr(kv_indptr)), static_cast<const int32_t*>(ptr(kv_indices)),
                                static_cast<const int32_t*>(ptr(kv_last_page_len)), ptr(o), o.stride(0), o.stride(1), lse,
                                (float)sm_scale, ptr(float_ws), ptr(int_ws), stream_of(q)),
           "batch decode run");
}

// ---------------------------------------------------------------------------------------------------------------
// prefill module
// ---------------------------------------------------------------------------------------------------------------
// plan_info of the prefill module: [0] max_qo_len [1] batch [2] total rows [3] qo heads [4] causal
//   [5] 1 = every request has exactly one query row: paged_run is served by the split-KV decode kernel, whose plan8
//       follows in [6..13]; 0: [6] = kv_splits of the paged prefill kernel (1 = no split)  (a one-row query sees the whole KV under either mask mode: FlashInfer masks
//       kv_idx + qo_len > kv_len + q_idx, prefill.cuh:1017)
Array<int64_t> PrefillPlan(TensorView float_ws, TensorView int_ws, TensorView pinned_int_ws, TensorView qo_indptr_host,
                           TensorView kv_indptr_host, TensorView kv_len_arr_host, int64_t total_num_rows, int64_t batch_size,
                           int64_t num_qo_heads, int64_t num_kv_heads, int64_t page_size, bool enable_cuda_graph,
                           int64_t head_dim_qk, int64_t head_dim_vo, bool causal, int64_t window_left,
                           int64_t fixed_split_size, bool disable_split_kv, int64_t num_colocated_ctas) {
  (void)pinned_int_ws; (void)fixed_split_size; (void)num_colocated_ctas;
  if (window_left >= 0) TVM_FFI_THROW(ValueError) << "sliding window attention is not implemented";
  if (head_dim_qk != head_dim_vo) TVM_FFI_THROW(ValueError) << "head_dim_qk != head_dim_vo";
  const int32_t* qo = static_cast<const int32_t*>(ptr(qo_indptr_host));
  int64_t max_qo = 0, min_qo = INT64_MAX;
  for (int64_t b = 0; b < batch_size; ++b) {
    max_qo = std::max<int64_t>(max_qo, qo[b + 1] - qo[b]);
    min_qo = std::min<int64_t>(min_qo, qo[b + 1] - qo[b]);
  }
  const bool one_row = batch_size > 0 && max_qo == 1 && min_qo == 1 && total_num_rows == batch_size &&
                       (head_dim_qk == 64 || head_dim_qk == 128);
  Array<int64_t> out;
  out.push_back(max_qo);
  out.push_back(batch_size);
  out.push_back(total_num_rows);
  out.push_back(num_qo_heads);
  out.push_back(causal ? 1 : 0);
  out.push_back(one_row ? 1 : 0);
  if (!one_row) {
    // split-KV decision for short-q / long-kv chunked prefill (FlashInfer's planner decides split_kv here too:
    // flashinfer_planinfo.cpp:168-247): host arithmetic on the lengths the reference hands over
    const int32_t* kvl = static_cast<const int32_t*>(ptr(kv_len_arr_host));
    int64_t max_kv = 0;
    for (int64_t b = 0; b < batch_size; ++b) max_kv = std::max<int64_t>(max_kv, kvl[b]);
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int splits = (disable_split_kv || page_size <= 1) ? 1
                     : xb_prefill_plan_splits((int)batch_size, (int)max_qo, max_kv, (int)num_qo_heads, (int)num_kv_heads, sms);
    const int64_t ws_bytes = float_ws.numel() * (float_ws.dtype().bits / 8);
    while (splits > 1 && xb_prefill_split_workspace_bytes(splits, total_num_rows, (int)num_qo_heads, (int)head_dim_qk) > ws_bytes) --splits;
    out.push_back(splits);
  }
  if (one_row) {
    int64_t plan[8];
    // page_size 1 with kv_indptr = cu_seq_lens is how the reference plans ragged prefill; only real page tables land here
    make_decode_plan(plan, float_ws, int_ws, static_cast<const int32_t*>(ptr(kv_indptr_host)), batch_size, num_qo_heads,
                     num_kv_heads, page_size, head_dim_qk, enable_cuda_graph);
    for (int i = 0; i < 8; ++i) out.push_back(plan[i]);
  }
  return out;
}

void check_prefill_extras(const Optional<TensorView>& custom_mask, const Optional<TensorView>& alibi, int64_t window_left,
                          double logits_soft_cap) {
  if (custom_mask.has_value()) TVM_FFI_THROW(ValueError) << "custom masks are not implemented (VLM-only path)";
  if (alibi.has_value()) TVM_FFI_THROW(ValueError) << "alibi is not implemented";
  if (window_left >= 0 || logits_soft_cap > 0) TVM_FFI_THROW(ValueError) << "sliding window / soft cap not implemented";
}

void RaggedRun(TensorView float_ws, TensorView int_ws, Array<int64_t> plan_vec, TensorView q, TensorView k, TensorView v,
               TensorView qo_indptr, TensorView kv_indptr, TensorView o, Optional<TensorView> maybe_lse, int64_t mask_mode_code,
               int64_t layout, int64_t window_left, bool enable_pdl, Optional<TensorView> maybe_custom_mask,
               Optional<TensorView> maybe_mask_indptr, Optional<TensorView> maybe_alibi_slopes,
               Optional<TensorView> maybe_prefix_len_ptr, Optional<TensorView> maybe_token_pos_in_items_ptr,
               Optional<TensorView> maybe_max_item_len_ptr, double logits_soft_cap, double sm_scale, double rope_rcp_scale,
               double rope_rcp_theta, int64_t token_pos_in_items_len) {
  (void)float_ws; (void)int_ws; (void)maybe_mask_indptr; (void)maybe_prefix_len_ptr; (void)maybe_token_pos_in_items_ptr;
  (void)maybe_max_item_len_ptr; (void)rope_rcp_scale; (void)rope_rcp_theta; (void)token_pos_in_items_len; (void)layout;
  check_prefill_extras(maybe_custom_mask, maybe_alibi_slopes, window_left, logits_soft_cap);
  if (plan_vec.size() < 6) TVM_FFI_THROW(ValueError) << "plan_info too short";
  if (!is_bf16(q) || !is_bf16(k) || !is_bf16(o)) TVM_FFI_THROW(TypeError) << "only bf16 q/k/v/o is implemented";
  xb_set_pdl(enable_pdl ? 1 : 0);
  float* lse = maybe_lse.has_value() ? static_cast<float*>(ptr(maybe_lse.value())) : nullptr;
  check_rc(xb_prefill_ragged_bf16(ptr(q), q.stride(0), q.stride(1), ptr(k), ptr(v), k.stride(0),
                                  static_cast<const int32_t*>(ptr(qo_indptr)), static_cast<const int32_t*>(ptr(kv_indptr)),
                                  ptr(o), o.stride(0), o.stride(1), lse, (int)plan_vec[1], q.size(0), k.size(0),
                                  (int)plan_vec[0], (int)q.size(1), (int)k.size(1), (int)q.size(2), mask_mode_code == 1,
                                  (float)sm_scale, stream_of(q)),
           "batch prefill ragged_run");
}

void PagedRun(TensorView float_ws, TensorView int_ws, Array<int64_t> plan_vec, TensorView q, TensorView k_cache,
              TensorView v_cache, TensorView qo_indptr, TensorView kv_indptr, TensorView kv_indices,
              TensorView kv_last_page_len, TensorView o, Optional<TensorView> maybe_lse, int64_t mask_mode_code,
              int64_t layout, int64_t window_left, bool enable_pdl, Optional<TensorView> maybe_custom_mask,
              Optional<TensorView> maybe_mask_indptr, Optional<TensorView> maybe_alibi_slopes,
              Optional<TensorView> maybe_prefix_len_ptr, Optional<TensorView> maybe_token_pos_in_items_ptr,
              Optional<TensorView> maybe_max_item_len_ptr, double logits_soft_cap, double sm_scale, double rope_rcp_scale,
              double rope_rcp_theta, int64_t token_pos_in_items_len) {
  (void)maybe_mask_indptr; (void)maybe_prefix_len_ptr; (void)maybe_token_pos_in_items_ptr;
  (void)maybe_max_item_len_ptr; (void)rope_rcp_scale; (void)rope_rcp_theta; (void)token_pos_in_items_len;
  check_prefill_extras(maybe_custom_mask, maybe_alibi_slopes, window_left, logits_soft_cap);
  if (plan_vec.size() < 6) TVM_FFI_THROW(ValueError) << "plan_info too short";
  if (!is_bf16(q) || !is_bf16(k_cache) || !is_bf16(o)) TVM_FFI_THROW(TypeError) << "only bf16 q/kv/o is implemented";
  xb_set_pdl(enable_pdl ? 1 : 0);
  float* lse = maybe_lse.has_value() ? static_cast<float*>(ptr(maybe_lse.value())) : nullptr;
  if (plan_vec[5] == 1) {
    // decode served through the prefill module (batch_decode.cpp:43-60 -> batch_chunked_prefill.cpp:63-91 with
    // qo_indptr = arange): one query row per request -> the HBM-streaming split-KV decode kernel
    if (plan_vec.size() != 14) TVM_FFI_THROW(ValueError) << "plan_info has " << plan_vec.size() << " entries, expected 14";
    if (q.size(0) != plan_vec[1]) TVM_FFI_THROW(ValueError) << "paged_run: " << q.size(0) << " query rows, plan has " << plan_vec[1];
    int64_t plan[8];
    for (int i = 0; i < 8; ++i) plan[i] = plan_vec[6 + i];
    const int64_t st_page = k_cache.stride(0);
    const int64_t st_tok = layout == 0 ? k_cache.stride(1) : k_cache.stride(2);
    const int64_t st_head = layout == 0 ? k_cache.stride(2) : k_cache.stride(1);
    check_rc(xb_paged_decode_bf16(plan, ptr(q), q.stride(0), q.stride(1), ptr(k_cache), ptr(v_cache), st_page, st_tok,
                                  st_head, static_cast<const int32_t*>(ptr(kv_indptr)),
                                  static_cast<const int32_t*>(ptr(kv_indices)),
                                  static_cast<const int32_t*>(ptr(kv_last_page_len)), ptr(o), o.stride(0), o.stride(1), lse,
                                  (float)sm_scale, ptr(float_ws), ptr(int_ws), stream_of(q)),
             "batch prefill paged_run (one-row decode path)");
    return;
  }
  if (layout != 0) TVM_FFI_THROW(ValueError) << "paged_run: only the NHD cache layout is implemented";
  if (plan_vec.size() >= 7 && plan_vec[6] > 1) {
    check_rc(xb_prefill_paged_split_bf16(ptr(q), q.stride(0), q.stride(1), ptr(k_cache), ptr(v_cache), k_cache.size(0),
                                         (int)k_cache.size(1), static_cast<const int32_t*>(ptr(qo_indptr)),
                                         static_cast<const int32_t*>(ptr(kv_indptr)), static_cast<const int32_t*>(ptr(kv_indices)),
                                         static_cast<const int32_t*>(ptr(kv_last_page_len)), ptr(o), o.stride(0), o.stride(1), lse,
                                         (int)plan_vec[1], q.size(0), (int)plan_vec[0], (int)q.size(1), (int)k_cache.size(2),
                                         (int)q.size(2), mask_mode_code == 1, (float)sm_scale, (int)plan_vec[6], ptr(float_ws),
                                         float_ws.numel() * (float_ws.dtype().bits / 8), stream_of(q)),
             "batch prefill paged_run (split KV)");
    return;
  }
  check_rc(xb_prefill_paged_bf16(ptr(q), q.stride(0), q.stride(1), ptr(k_cache), ptr(v_cache), k_cache.size(0),
                                 (int)k_cache.size(1), static_cast<const int32_t*>(ptr(qo_indptr)),
                                 static_cast<const int32_t*>(ptr(kv_indptr)), static_cast<const int32_t*>(ptr(kv_indices)),
                                 static_cast<const int32_t*>(ptr(kv_last_page_len)), ptr(o), o.stride(0), o.stride(1), lse,
                                 (int)plan_vec[1], q.size(0), (int)plan_vec[0], (int)q.size(1), (int)k_cache.size(2),
                                 (int)q.size(2), mask_mode_code == 1, (float)sm_scale, stream_of(q)),
           "batch prefill paged_run");
}

// FA3 form of the ragged prefill module.  On an sm90a device the reference picks backend "fa3" for ragged prefill
// (utils.cpp:376-386), requests the URI with the "_sm90" suffix (utils.cpp:417), calls `plan` without fixed_split_size /
// disable_split_kv / num_colocated_ctas (flashinfer_planinfo.cpp:119-137) and `ragged_run` with FlashInfer's FA3 argument
// list (batch_prefill.cpp:129-158).  Both route to the same kernels as the fa2 entry points.
Array<int64_t> PrefillPlanSm90(TensorView float_ws, TensorView int_ws, TensorView pinned_int_ws, TensorView qo_indptr_host,
                               TensorView kv_indptr_host, TensorView kv_len_arr_host, int64_t total_num_rows,
                               int64_t batch_size, int64_t num_qo_heads, int64_t num_kv_heads, int64_t page_size,
                               bool enable_cuda_graph, int64_t head_dim_qk, int64_t head_dim_vo, bool causal,
                               int64_t window_left) {
  return PrefillPlan(float_ws, int_ws, pinned_int_ws, qo_indptr_host, kv_indptr_host, kv_len_arr_host, total_num_rows,
                     batch_size, num_qo_heads, num_kv_heads, page_size, enable_cuda_graph, head_dim_qk, head_dim_vo, causal,
                     window_left, -1, false, 0);
}

void RaggedRunSm90(TensorView float_ws, TensorView int_ws, Array<int64_t> plan_vec, TensorView q, TensorView k, TensorView v,
                   TensorView qo_indptr, TensorView kv_indptr, TensorView o, Optional<TensorView> maybe_lse,
                   int64_t mask_mode_code, int64_t layout, int64_t window_left, bool enable_pdl,
                   Optional<TensorView> maybe_prefix_len_ptr, Optional<TensorView> maybe_token_pos_in_items_ptr,
                   Optional<TensorView> maybe_max_item_len_ptr, Optional<TensorView> maybe_scale_v, double logits_soft_cap,
                   double sm_scale, double scale_v_scalar, int64_t token_pos_in_items_len) {
  // scale_v exists for fp8 K/V (batch_prefill.cpp:130-133); with bf16 K/V the reference passes no tensor and 1.0
  if (maybe_scale_v.has_value() || scale_v_scalar != 1.0) TVM_FFI_THROW(ValueError) << "fp8 V scaling is not implemented";
  RaggedRun(float_ws, int_ws, plan_vec, q, k, v, qo_indptr, kv_indptr, o, maybe_lse, mask_mode_code, layout, window_left,
            enable_pdl, Optional<TensorView>(), Optional<TensorView>(), Optional<TensorView>(), maybe_prefix_len_ptr,
            maybe_token_pos_in_items_ptr, maybe_max_item_len_ptr, logits_soft_cap, sm_scale, 1.0, 1.0 / 10000.0,
            token_pos_in_items_len);
}

// Optional capability probe (integration/patches/0003): a decode plan made under enable_cuda_graph depends only on the
// captured (padded) batch and the workspace sizes - the kernels derive the split geometry on the device from the live paged
// triplet and the arrival counters reset themselves - so a CUDA-graph executor may plan once and skip the host-side plan
// before every replay (cuda_graph_executor_impl.cpp:751-822).
int64_t PlanIsReplayInvariant() { return 1; }

}  // namespace

TVM_FFI_DLL_EXPORT_TYPED_FUNC(plan_is_replay_invariant, PlanIsReplayInvariant);
#if defined(XB_FFI_DECODE_MODULE)
TVM_FFI_DLL_EXPORT_TYPED_FUNC(plan, DecodePlan);
TVM_FFI_DLL_EXPORT_TYPED_FUNC(run, DecodeRun);
#elif defined(XB_FFI_PREFILL_SM90_MODULE)
TVM_FFI_DLL_EXPORT_TYPED_FUNC(plan, PrefillPlanSm90);
TVM_FFI_DLL_EXPORT_TYPED_FUNC(ragged_run, RaggedRunSm90);
#else
TVM_FFI_DLL_EXPORT_TYPED_FUNC(plan, PrefillPlan);
TVM_FFI_DLL_EXPORT_TYPED_FUNC(ragged_run, RaggedRun);
TVM_FFI_DLL_EXPORT_TYPED_FUNC(paged_run, PagedRun);
#endif
