// c_api.cc — the extern "C" boundary declared in include/ct2b200.h.  Every entry point converts C++
// exceptions into an error code + thread-local message (the reference surfaces std::invalid_argument /
// std::runtime_error through std::future::get(), src/cuda/utils.h:51-96).
#include <cuda_runtime.h>

#include <cstring>
#include <string>

#include "common.cuh"
#include "host/beam.h"
#include "host/dtw.h"
#include "host/engine.h"
#include "host/translator.h"
#include "kernels/beam_decide.h"
#include "kernels/kernels.h"
#include "kernels/philox.h"

using namespace ct2b200;

namespace {
thread_local std::string g_error;

template <typename F>
int guarded(F&& f) {
  try {
    f();
    return 0;
  } catch (const InvalidArgument& e) {
    g_error = std::string("invalid argument: ") + e.what();
    return 2;
  } catch (const std::invalid_argument& e) {
    g_error = std::string("invalid argument: ") + e.what();
    return 2;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 1;
  }
}

cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }

void require_device() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0)
    throw std::runtime_error("no CUDA device: ct2b200 has no CPU fallback");
}

// the num_hypotheses best hypotheses of every entry: out_ids [batch, num_hypotheses, max_length] (-1 padded), out_lens and
// out_scores [batch, num_hypotheses] (-1 and 0 for a hypothesis an entry does not have)
void copy_hypotheses(const std::vector<TranslationHypotheses>& res, int64_t batch, int num_hypotheses, int64_t max_length,
                     int32_t* out_ids, int32_t* out_lens, float* out_scores) {
  for (int64_t b = 0; b < batch; ++b)
    for (int h = 0; h < num_hypotheses; ++h) {
      int32_t* dst = out_ids + (b * num_hypotheses + h) * max_length;
      const bool have = h < static_cast<int>(res[b].tokens.size());
      const int64_t len = have ? static_cast<int64_t>(res[b].tokens[h].size()) : 0;
      for (int64_t i = 0; i < max_length; ++i) dst[i] = i < len ? res[b].tokens[h][i] : -1;
      out_lens[b * num_hypotheses + h] = have ? static_cast<int32_t>(len) : -1;
      out_scores[b * num_hypotheses + h] = have ? res[b].scores[h] : 0.f;
    }
}
}  // namespace

struct ct2b200_generator {
  std::unique_ptr<Generator> impl;
};
struct ct2b200_translator {
  std::unique_ptr<Translator> impl;
};
struct ct2b200_encoder {
  std::unique_ptr<Translator> impl;   // the encoder engine of the Translator in its encoder-only mode
};

extern "C" {

CT2B200_API const char* ct2b200_last_error(void) { return g_error.c_str(); }
CT2B200_API const char* ct2b200_version(void) { return "0.1.0 (sm_90a)"; }
CT2B200_API int64_t ct2b200_kernel_launch_count(void) { return g_kernel_launches.load(); }

CT2B200_API int ct2b200_device_info(int device, int* sm_count, int* cc_major, int* cc_minor, size_t* total_mem) {
  return guarded([&] {
    require_device();
    cudaDeviceProp p;
    CT2_CUDA_CHECK(cudaGetDeviceProperties(&p, device));
    if (sm_count) *sm_count = p.multiProcessorCount;
    if (cc_major) *cc_major = p.major;
    if (cc_minor) *cc_minor = p.minor;
    if (total_mem) *total_mem = p.totalGlobalMem;
  });
}

CT2B200_API int ct2b200_quantize_rows(const void* x, int dtype, int64_t rows, int64_t cols, int round_before_cast, int8_t* q,
                          float* scale, void* stream) {
  return guarded([&] {
    require_device();
    launch_quantize_rows(x, dtype, rows, cols, round_before_cast != 0, q, scale, S(stream));
  });
}

CT2B200_API int ct2b200_gemm_s8(const int8_t* a, const int8_t* b, int64_t m, int64_t n, int64_t k, int32_t* c, int impl,
                    void* stream) {
  return guarded([&] {
    require_device();
    DenseEpilogue e{nullptr, nullptr, nullptr, nullptr, nullptr, c, -1, n};
    gemm_s8(a, b, m, n, k, e, CT2B200_F32, impl, S(stream));
  });
}

CT2B200_API int ct2b200_dequantize_gemm_output(const int32_t* c, const float* a_scale, const float* b_scale, const void* bias,
                                   int act, int64_t m, int64_t n, void* y, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    DenseEpilogue e{a_scale, b_scale, bias, nullptr, y, nullptr, act, n};
    launch_dequantize_gemm_output(c, e, m, n, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_dequantize_rows(const int8_t* x, const float* scale, int64_t rows, int64_t cols, void* y, int dtype,
                            void* stream) {
  return guarded([&] {
    require_device();
    launch_dequantize_rows(x, scale, rows, cols, y, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_dense_s8(const int8_t* xq, const float* x_scale, const int8_t* w, const float* w_scale, const void* bias,
                     const void* residual, int act, int64_t m, int64_t n, int64_t k, void* y, int dtype, int impl,
                     void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(x_scale && w_scale, "dense_s8: scales are required");
    DenseEpilogue e{x_scale, w_scale, bias, residual, y, nullptr, act, n};
    gemm_s8(xq, w, m, n, k, e, dtype, impl, S(stream));
  });
}

CT2B200_API int ct2b200_dense_s8_glu(const int8_t* xq, const float* x_scale, const int8_t* w_gate, const float* w_gate_scale,
                         const int8_t* w_up, const float* w_up_scale, int act, int64_t m, int64_t n, int64_t k, void* h,
                         int dtype, int impl, void* stream) {
  return guarded([&] {
    require_device();
    GluEpilogue g{x_scale, w_gate_scale, w_up_scale, h, act, n};
    gemm_s8_glu(xq, w_gate, w_up, m, n, k, g, dtype, impl, S(stream));
  });
}

CT2B200_API int ct2b200_dense_s8_rows(const void* x, const void* gamma, float eps, const int8_t* w, const float* w_scale,
                          const void* bias, const void* residual, int act, int64_t m, int64_t n, int64_t k, void* y,
                          int dtype, int8_t* xq, float* x_scale, void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(x && w && w_scale && xq && x_scale, "dense_s8_rows: null argument");
    DenseEpilogue e{x_scale, w_scale, bias, residual, y, nullptr, act, n};
    rows_to_int8(x, gamma, eps, m, k, dtype, xq, x_scale, S(stream));
    gemm_s8(xq, w, m, n, k, e, dtype, CT2B200_GEMM_AUTO, S(stream));
  });
}

CT2B200_API int ct2b200_dense_s8_glu_rows(const void* x, const void* gamma, float eps, const int8_t* w_gate,
                              const float* w_gate_scale, const int8_t* w_up, const float* w_up_scale, int act, int64_t m,
                              int64_t n, int64_t k, void* h, int dtype, int8_t* xq, float* x_scale, void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(x && w_gate && w_up && xq && x_scale, "dense_s8_glu_rows: null argument");
    GluEpilogue g{x_scale, w_gate_scale, w_up_scale, h, act, n};
    rows_to_int8(x, gamma, eps, m, k, dtype, xq, x_scale, S(stream));
    gemm_s8_glu(xq, w_gate, w_up, m, n, k, g, dtype, CT2B200_GEMM_AUTO, S(stream));
  });
}

CT2B200_API int ct2b200_gemm_f16(const void* a, const void* b, const void* bias, const void* residual, int act, int64_t m,
                     int64_t n, int64_t k, void* c, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    gemm_f16_tc(a, b, bias, residual, act, m, n, k, c, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_rms_norm(const void* gamma, const void* x, int64_t rows, int64_t cols, float eps, int use_residual,
                     void* y, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    launch_rms_norm(gamma, x, rows, cols, eps, use_residual != 0, y, nullptr, nullptr, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_rms_norm_quantize(const void* gamma, const void* x, int64_t rows, int64_t cols, float eps,
                              int use_residual, int8_t* q, float* scale, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(q && scale, "rms_norm_quantize: outputs are required");
    launch_rms_norm(gamma, x, rows, cols, eps, use_residual != 0, nullptr, q, scale, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_rotary(const void* x, const void* sin, const void* cos, int64_t batch, int64_t time, int64_t depth,
                   int64_t ndims, int interleave, void* y, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(ndims <= depth && ndims % 2 == 0, "rotary: ndims must be even and <= depth");
    launch_rotary(x, sin, cos, batch, time, depth, ndims, interleave != 0, y, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_softmax(const void* x, const int32_t* lengths, int64_t rows, int64_t cols, int log, void* y, int dtype,
                    void* stream) {
  return guarded([&] {
    require_device();
    launch_softmax(x, lengths, rows, cols, log != 0, y, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_log_softmax_gather(const void* x, const int32_t* ids, int64_t rows, int64_t cols, float* y, int dtype,
                               void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(cols >= 1, "log_softmax_gather: empty rows");
    launch_log_softmax_gather(x, ids, rows, cols, y, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_topk(const void* x, int64_t rows, int64_t cols, int k, void* values, int32_t* indices, int dtype,
                 void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(k >= 1 && k <= 64 && k <= cols, "topk: k must be in [1, min(64, cols)]");
    launch_topk(x, rows, cols, k, values, indices, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_random_sample(const void* x, int64_t rows, int64_t cols, int k, float temperature, uint32_t seed,
                                      uint32_t counter, uint32_t step, int32_t* ids, float* logp, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    launch_random_sample(x, rows, cols, cols, k, temperature, seed, counter, step, ids, logp, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_set_random_seed(uint32_t seed) {
  return guarded([&] { set_random_seed(seed); });
}

CT2B200_API int ct2b200_philox4x32_host(const uint32_t* counter, const uint32_t* key, uint32_t* out) {
  return guarded([&] {
    CT2_REQUIRE(counter && key && out, "philox4x32_host: null argument");
    const Philox4 r = philox4x32_10(Philox4{{counter[0], counter[1], counter[2], counter[3]}}, key[0], key[1]);
    for (int i = 0; i < 4; ++i) out[i] = r.v[i];
  });
}

CT2B200_API int ct2b200_gather_rows(const void* data, const int32_t* ids, int64_t num_ids, int64_t row_bytes, void* out,
                        void* stream) {
  return guarded([&] {
    require_device();
    launch_gather_rows(data, ids, num_ids, row_bytes, out, S(stream));
  });
}

CT2B200_API int ct2b200_embedding_s8(const int8_t* w, const float* scale, const int32_t* ids, int64_t num_ids, int64_t depth,
                         void* y, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    launch_embedding_s8(w, scale, ids, num_ids, depth, y, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_mul_quantize(const void* gate, const void* up, int64_t rows, int64_t cols, int8_t* q, float* scale,
                         int dtype, void* stream) {
  return guarded([&] {
    require_device();
    launch_mul_quantize(gate, up, rows, cols, q, scale, dtype, S(stream));
  });
}

CT2B200_API size_t ct2b200_attention_decode_workspace(int64_t batch, int num_heads, int head_dim, int64_t max_len) {
  // 16 slots per (row, head) for the split-KV kernel + 64 for the persistent kernel (attention_decode.cu)
  (void)max_len;
  return attention_decode_workspace_bytes(batch, num_heads, head_dim, 80);
}

CT2B200_API int ct2b200_attention_decode(const void* qkv, void* k_cache, void* v_cache, const float* sin, const float* cos,
                             const int32_t* lens, int64_t batch, int num_heads, int num_heads_kv, int head_dim,
                             int64_t max_len, int rotary_interleave, float scale, void* out, void* workspace,
                             size_t workspace_bytes, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int splits = attention_decode_splits(batch, num_heads_kv, max_len, sms);
    launch_attention_decode(qkv, k_cache, v_cache, sin, cos, lens, batch, num_heads, num_heads_kv, head_dim, max_len,
                            rotary_interleave != 0, scale, out, workspace, workspace_bytes, splits, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_attention_prefill(const void* qkv, void* k_cache, void* v_cache, const float* sin, const float* cos,
                              const int32_t* lengths, int64_t batch, int64_t time, int64_t offset, int num_heads,
                              int num_heads_kv, int head_dim, int64_t max_len, int rotary_interleave, float scale,
                              void* out, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(offset + time <= max_len, "attention_prefill: offset + time exceeds max_len");
    launch_rope_append(const_cast<void*>(qkv), k_cache, v_cache, sin, cos, lengths, batch, time, offset, num_heads,
                       num_heads_kv, head_dim, max_len, rotary_interleave != 0, dtype, S(stream));
    launch_attention_prefill(qkv, k_cache, v_cache, lengths, batch, time, offset, num_heads, num_heads_kv, head_dim,
                             max_len, scale, out, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_attention_encoder(const void* qkv, const int32_t* lengths, int64_t batch, int keys, int H, int D,
                                          float scale, void* out, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(batch >= 0 && keys >= 0 && H > 0 && D > 0, "attention_encoder: bad shape");
    launch_attention_encoder(qkv, lengths, batch, keys, H, D, scale, out, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_attention_encoder_mma(const void* qkv, const int32_t* lengths, int64_t batch, int keys, int H, int D,
                                              float scale, void* out, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(batch >= 0 && keys >= 0 && H > 0 && D > 0, "attention_encoder_mma: bad shape");
    if (!launch_attention_encoder_mma(qkv, lengths, batch, keys, H, D, scale, out, dtype, S(stream)))
      throw std::invalid_argument("attention_encoder_mma: fp16 / bf16 with head_dim 64 or 128 only");
  });
}

CT2B200_API int ct2b200_attention_causal(const void* qkv, int64_t batch, int time, int H, int D, float scale, void* out, int dtype,
                                         void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(batch >= 0 && time >= 0 && H > 0 && D > 0, "attention_causal: bad shape");
    launch_attention_causal(qkv, batch, time, H, D, scale, out, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_attention_beam_self(const void* qkv, void* k_cache, void* v_cache, const int32_t* anc, const int32_t* step_d,
                                            int64_t rows, int max_len, int H, int D, float scale, void* out, int dtype,
                                            void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(rows >= 0 && max_len > 0 && H > 0 && D > 0, "attention_beam_self: bad shape");
    launch_attention_beam_self(qkv, k_cache, v_cache, anc, step_d, rows, max_len, H, D, scale, out, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_attention_cross(const void* q, const void* kv, const int32_t* lengths, int64_t rows, int beam, int keys,
                                        int H, int D, float scale, void* out, float* capture_out, const uint32_t* masks_d, int first,
                                        int total, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(rows >= 0 && beam > 0 && rows % beam == 0 && keys >= 0 && H > 0 && D > 0, "attention_cross: bad shape");
    if (!capture_out) {
      launch_attention_cross(q, kv, lengths, rows, beam, keys, H, D, scale, out, dtype, S(stream));
      return;
    }
    AttnCapture cap;
    cap.out = capture_out;
    cap.masks = masks_d;
    cap.first = first;
    cap.total = total;
    launch_attention_cross_capture(q, kv, lengths, rows, beam, keys, H, D, scale, out, cap, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_beam_rows(void* logits, const void* cum, int32_t* step_d, int batch, int beam, int vocab, int64_t vocab_ld,
                                  int min_length, const int32_t* end_ids_d, int num_end, void* row_scores, int32_t* row_ids,
                                  int dtype, void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(batch >= 0 && vocab > 0 && vocab_ld >= vocab && num_end >= 0 && (num_end == 0 || end_ids_d),
                "beam_rows: bad shape");
    BeamState s;
    s.batch = batch;
    s.beam = beam;
    s.vocab = vocab;
    s.vocab_ld = vocab_ld;
    s.min_length = min_length;
    s.end_ids = end_ids_d;
    s.num_end = num_end;
    s.step = step_d;
    launch_beam_rows(logits, cum, s, row_scores, row_ids, dtype, S(stream));
  });
}

CT2B200_API int ct2b200_awq_repack(const int32_t* qweight, const void* scales, const int32_t* qzeros, int layout, int group_size,
                       int64_t n, int64_t k, int32_t* wp, void* sc, void* zr, void* sz, void* stream) {
  return guarded([&] {
    require_device();
    awq_repack(qweight, scales, qzeros, layout, group_size, n, k, wp, sc, zr, S(stream));
    if (sz) {
      AwqNative w{wp, sc, zr, n, k, group_size};
      awq_build_group_major(w, sz, S(stream));
    }
  });
}

CT2B200_API int ct2b200_dense_awq(const void* x, const int32_t* wp, const void* sc, const void* zr, const void* sz,
                      int group_size, const void* bias, const void* residual, int act, int64_t m, int64_t n, int64_t k,
                      void* y, void* scratch_nk, void* stream) {
  return guarded([&] {
    require_device();
    AwqNative w{wp, sc, zr, n, k, group_size, sz};
    dense_awq(x, w, bias, residual, act, m, y, scratch_nk, S(stream));
  });
}

CT2B200_API int ct2b200_dense_awq_glu(const void* x, const int32_t* wp_gate, const void* sc_gate, const void* zr_gate,
                          const void* sz_gate, const int32_t* wp_up, const void* sc_up, const void* zr_up,
                          const void* sz_up, int group_size, int act, int64_t m, int64_t n, int64_t k, void* h,
                          void* scratch_nk, void* scratch_mn, void* stream) {
  return guarded([&] {
    require_device();
    AwqNative g{wp_gate, sc_gate, zr_gate, n, k, group_size, sz_gate}, u{wp_up, sc_up, zr_up, n, k, group_size, sz_up};
    dense_awq_glu(x, g, u, act, m, h, scratch_nk, scratch_mn, S(stream));
  });
}

CT2B200_API int ct2b200_dequantize_awq(const int32_t* qweight, const void* scales, const int32_t* qzeros, int layout,
                           int group_size, int64_t n, int64_t k, void* w, void* stream) {
  return guarded([&] {
    require_device();
    awq_dequantize_ref_layout(qweight, scales, qzeros, layout, group_size, n, k, w, S(stream));
  });
}

// ---- engine ----
CT2B200_API ct2b200_generator* ct2b200_generator_open(const char* model_dir, const ct2b200_generator_config* config) {
  ct2b200_generator* g = nullptr;
  const int rc = guarded([&] {
    require_device();
    CT2_REQUIRE(model_dir && config, "generator_open: null argument");
    auto holder = std::make_unique<ct2b200_generator>();
    holder->impl = std::make_unique<Generator>(model_dir, *config);
    g = holder.release();
  });
  return rc == 0 ? g : nullptr;
}

CT2B200_API void ct2b200_generator_close(ct2b200_generator* g) { delete g; }

CT2B200_API int ct2b200_generator_vocab_size(const ct2b200_generator* g) {
  return g ? static_cast<int>(g->impl->decoder().config().vocab) : -1;
}

CT2B200_API int ct2b200_generator_info(const ct2b200_generator* g, int* num_layers, int* num_heads, int* num_heads_kv, int* head_dim,
                           int* d_model, int64_t* weight_bytes) {
  return guarded([&] {
    CT2_REQUIRE(g, "null generator");
    const ModelConfig& c = g->impl->decoder().config();
    if (num_layers) *num_layers = c.num_layers;
    if (num_heads) *num_heads = c.num_heads;
    if (num_heads_kv) *num_heads_kv = c.num_heads_kv;
    if (head_dim) *head_dim = c.head_dim;
    if (d_model) *d_model = static_cast<int>(c.d_model);
    if (weight_bytes) *weight_bytes = c.weight_bytes;
  });
}

CT2B200_API int ct2b200_generate_batch(ct2b200_generator* g, const int32_t* prompt_ids, const int32_t* prompt_lens, int64_t batch,
                           int64_t max_prompt_len, int64_t max_length, int64_t min_length, const int32_t* end_ids,
                           int num_end_ids, int return_end_token, int32_t* out_ids, int32_t* out_lens) {
  return guarded([&] {
    CT2_REQUIRE(g && prompt_ids && prompt_lens && out_ids && out_lens, "generate_batch: null argument");
    GenerationRequest r;
    r.prompt_ids = prompt_ids;
    r.prompt_lens = prompt_lens;
    r.batch = batch;
    r.max_prompt_len = max_prompt_len;
    r.max_length = max_length;
    r.min_length = min_length;
    r.end_ids.assign(end_ids, end_ids + (end_ids ? num_end_ids : 0));
    r.return_end_token = return_end_token != 0;
    g->impl->generate(r, out_ids, out_lens);
  });
}

CT2B200_API int ct2b200_generate_batch_scores(ct2b200_generator* g, const int32_t* prompt_ids, const int32_t* prompt_lens,
                                              int64_t batch, int64_t max_prompt_len, int64_t max_length, int64_t min_length,
                                              const int32_t* end_ids, int num_end_ids, int return_end_token,
                                              float length_penalty, int32_t* out_ids, int32_t* out_lens, float* out_scores) {
  return guarded([&] {
    CT2_REQUIRE(g && prompt_ids && prompt_lens && out_ids && out_lens && out_scores, "generate_batch_scores: null argument");
    GenerationRequest r;
    r.prompt_ids = prompt_ids;
    r.prompt_lens = prompt_lens;
    r.batch = batch;
    r.max_prompt_len = max_prompt_len;
    r.max_length = max_length;
    r.min_length = min_length;
    r.end_ids.assign(end_ids, end_ids + (end_ids ? num_end_ids : 0));
    r.return_end_token = return_end_token != 0;
    r.return_scores = true;
    r.length_penalty = length_penalty;
    g->impl->generate(r, out_ids, out_lens, out_scores);
  });
}

CT2B200_API int ct2b200_generate_batch_beam(ct2b200_generator* g, const int32_t* prompt_ids, int64_t batch, int64_t prompt_len,
                                int64_t max_length, int64_t min_length, const int32_t* end_ids, int num_end_ids,
                                int return_end_token, int beam_size, float patience, float length_penalty, int num_hypotheses,
                                int32_t* out_ids, int32_t* out_lens, float* out_scores) {
  return guarded([&] {
    CT2_REQUIRE(g && prompt_ids && out_ids && out_lens && out_scores, "generate_batch_beam: null argument");
    std::vector<int32_t> lens(static_cast<size_t>(std::max<int64_t>(batch, 0)), static_cast<int32_t>(prompt_len));
    GenerationRequest r;
    r.prompt_ids = prompt_ids;
    r.prompt_lens = lens.data();
    r.batch = batch;
    r.max_prompt_len = prompt_len;
    r.max_length = max_length;
    r.min_length = min_length;
    r.end_ids.assign(end_ids, end_ids + (end_ids ? num_end_ids : 0));
    r.return_end_token = return_end_token != 0;
    r.beam_size = beam_size;
    r.patience = patience;
    r.length_penalty = length_penalty;
    r.num_hypotheses = num_hypotheses;
    copy_hypotheses(g->impl->generate_beam(r), batch, num_hypotheses, max_length, out_ids, out_lens, out_scores);
  });
}

CT2B200_API int ct2b200_forward_batch(ct2b200_generator* g, const int32_t* ids, int64_t batch, int64_t time, int return_log_probs,
                          float* logits) {
  return guarded([&] {
    CT2_REQUIRE(g && ids && logits, "forward_batch: null argument");
    g->impl->forward(ids, batch, time, return_log_probs != 0, logits);
  });
}

CT2B200_API int ct2b200_score_batch(ct2b200_generator* g, const int32_t* ids, const int32_t* lens, int64_t batch,
                        int64_t max_len, int64_t offset, float* out_scores) {
  return guarded([&] {
    CT2_REQUIRE(g && ids && lens && out_scores, "score_batch: null argument");
    g->impl->score(ids, lens, batch, max_len, offset, out_scores);
  });
}

CT2B200_API int ct2b200_bench_last_logits(ct2b200_generator* g, int64_t batch, float* logits_h, int64_t logits_len) {
  return guarded([&] {
    CT2_REQUIRE(g && logits_h, "null argument");
    g->impl->bench_last_logits(batch, logits_h, logits_len);
  });
}

CT2B200_API int ct2b200_bench_decode(ct2b200_generator* g, int64_t batch, int64_t prompt_len, int64_t steps, int64_t warmup,
                         float* prefill_ms, float* decode_ms, int64_t* kernel_launches) {
  return guarded([&] {
    CT2_REQUIRE(g, "null generator");
    g->impl->bench_decode(batch, prompt_len, steps, warmup, prefill_ms, decode_ms, kernel_launches);
  });
}

CT2B200_API int ct2b200_model_summary(const char* model_dir, char* json_out, size_t capacity) {
  return guarded([&] {
    CT2_REQUIRE(model_dir && json_out && capacity > 0, "model_summary: null argument");
    ModelFile file(model_dir);
    const ModelConfig mc = parse_model_config(file);
    char buf[1024];
    const int n = std::snprintf(
        buf, sizeof(buf),
        "{\"spec\": \"%s\", \"binary_version\": %u, \"revision\": %u, \"num_layers\": %d, \"num_heads\": %d, "
        "\"num_heads_kv\": %d, \"head_dim\": %d, \"d_model\": %lld, \"ffn_dim\": %lld, \"vocab_size\": %lld, "
        "\"weights\": \"%s\", \"float_type\": \"%s\", \"rotary_interleave\": %s, \"rotary_base\": %.9g, \"rotary_scaling_type\": %d, "
        "\"layer_norm_epsilon\": %.9g, \"activation\": %d}",
        file.spec_name.c_str(), file.binary_version, file.revision, mc.num_layers, mc.num_heads, mc.num_heads_kv, mc.head_dim,
        static_cast<long long>(mc.d_model), static_cast<long long>(mc.ffn_dim), static_cast<long long>(mc.vocab),
        mc.weights.c_str(), mc.float_type.c_str(), mc.rotary_interleave ? "true" : "false", static_cast<double>(mc.rotary_base),
        mc.rotary_scaling_type, static_cast<double>(mc.eps), mc.activation);
    CT2_REQUIRE(n > 0 && static_cast<size_t>(n) < capacity, "model_summary: output buffer too small");
    std::memcpy(json_out, buf, static_cast<size_t>(n) + 1);
  });
}

CT2B200_API int ct2b200_generator_tp_handle(ct2b200_generator* g, void* handle64_h) {
  return guarded([&] {
    CT2_REQUIRE(g && handle64_h, "null argument");
    g->impl->decoder().tp_handle(handle64_h);
  });
}
CT2B200_API int ct2b200_generator_tp_connect(ct2b200_generator* g, const void* handles_h, int num_handles) {
  return guarded([&] {
    CT2_REQUIRE(g && handles_h, "null argument");
    g->impl->decoder().tp_connect(handles_h, num_handles);
  });
}

// ---- encoder-decoder path ----
CT2B200_API int ct2b200_gemm_f32(const float* a, const float* b, const float* bias, const float* residual, int act, int64_t m,
                     int64_t n, int64_t k, float* c, void* stream) {
  return guarded([&] {
    require_device();
    gemm_f32(a, b, bias, residual, act, m, n, k, c, S(stream));
  });
}

CT2B200_API int ct2b200_layer_norm(const void* x, const void* gamma, const void* beta, int64_t rows, int64_t cols, float eps, void* y,
                       int8_t* q, float* scale, int round_before_cast, int dtype, void* stream) {
  return guarded([&] {
    require_device();
    CT2_REQUIRE(y || q, "layer_norm: no output requested");
    CT2_REQUIRE(!q || scale, "layer_norm: scale_d is required with q_d");
    launch_layer_norm(x, gamma, beta, rows, cols, eps, y, q, scale, round_before_cast != 0, dtype, S(stream));
  });
}

CT2B200_API ct2b200_translator* ct2b200_translator_open(const char* model_dir, const ct2b200_generator_config* config) {
  ct2b200_translator* t = nullptr;
  const int rc = guarded([&] {
    require_device();
    CT2_REQUIRE(model_dir && config, "translator_open: null argument");
    auto holder = std::make_unique<ct2b200_translator>();
    holder->impl = std::make_unique<Translator>(model_dir, *config);
    t = holder.release();
  });
  return rc == 0 ? t : nullptr;
}

CT2B200_API void ct2b200_translator_close(ct2b200_translator* t) { delete t; }

CT2B200_API int ct2b200_translator_info(const ct2b200_translator* t, int* encoder_layers, int* decoder_layers, int* num_heads,
                            int* d_model, int* source_vocab, int* target_vocab, int64_t* weight_bytes) {
  return guarded([&] {
    CT2_REQUIRE(t, "null translator");
    const Seq2SeqConfig& c = t->impl->config();
    if (encoder_layers) *encoder_layers = c.enc_layers;
    if (decoder_layers) *decoder_layers = c.dec_layers;
    if (num_heads) *num_heads = c.num_heads;
    if (d_model) *d_model = static_cast<int>(c.d_model);
    if (source_vocab) *source_vocab = static_cast<int>(c.src_vocab);
    if (target_vocab) *target_vocab = static_cast<int>(c.tgt_vocab);
    if (weight_bytes) *weight_bytes = c.weight_bytes;
  });
}

CT2B200_API int ct2b200_translator_positions(const ct2b200_translator* t, int64_t* encoder, int64_t* decoder) {
  return guarded([&] {
    CT2_REQUIRE(t && encoder && decoder, "translator_positions: null argument");
    *encoder = t->impl->encoder_positions();
    *decoder = t->impl->decoder_positions();
  });
}

CT2B200_API int ct2b200_translator_summary(const char* model_dir, char* json_out, size_t capacity) {
  return guarded([&] {
    CT2_REQUIRE(model_dir && json_out && capacity > 0, "translator_summary: null argument");
    ModelFile file(model_dir);
    const Seq2SeqConfig mc = parse_seq2seq_config(file);
    char buf[1024];
    const int n = std::snprintf(
        buf, sizeof(buf),
        "{\"spec\": \"%s\", \"binary_version\": %u, \"revision\": %u, \"encoder_layers\": %d, \"decoder_layers\": %d, "
        "\"num_heads\": %d, \"head_dim\": %d, \"d_model\": %lld, \"ffn_dim\": %lld, \"source_vocab\": %lld, "
        "\"target_vocab\": %lld, \"weights\": \"%s\", \"pre_norm\": %s, \"activation\": %d, \"embeddings_scale\": %.9g, "
        "\"layer_norm_epsilon\": %.9g, \"round_before_cast\": %s}",
        file.spec_name.c_str(), file.binary_version, file.revision, mc.enc_layers, mc.dec_layers, mc.num_heads, mc.head_dim,
        static_cast<long long>(mc.d_model), static_cast<long long>(mc.ffn_dim), static_cast<long long>(mc.src_vocab),
        static_cast<long long>(mc.tgt_vocab), mc.weights.c_str(), mc.dec_pre_norm ? "true" : "false", mc.dec_activation,
        static_cast<double>(mc.dec_emb_scale), static_cast<double>(mc.eps), mc.round_before_cast ? "true" : "false");
    CT2_REQUIRE(n > 0 && static_cast<size_t>(n) < capacity, "translator_summary: output buffer too small");
    std::memcpy(json_out, buf, static_cast<size_t>(n) + 1);
  });
}

namespace {
// the TranslationRequest of ct2b200_translate_batch's arguments (the logits processors left off)
TranslationRequest translation_request(const int32_t* source_ids, const int32_t* source_lens, int64_t batch, int64_t max_source_len,
                                       int beam_size, float patience, float length_penalty, int64_t max_decoding_length,
                                       int64_t min_decoding_length, int num_hypotheses, int32_t start_id, const int32_t* end_ids,
                                       int num_end_ids, int return_end_token) {
  TranslationRequest r;
  r.source_ids = source_ids;
  r.source_lens = source_lens;
  r.batch = batch;
  r.max_source_len = max_source_len;
  r.beam_size = beam_size;
  r.patience = patience;
  r.length_penalty = length_penalty;
  r.max_decoding_length = max_decoding_length;
  r.min_decoding_length = min_decoding_length;
  r.num_hypotheses = num_hypotheses;
  r.start_id = start_id;
  r.end_ids.assign(end_ids, end_ids + (end_ids ? num_end_ids : 0));
  r.return_end_token = return_end_token != 0;
  return r;
}
}  // namespace

CT2B200_API int ct2b200_translate_batch(ct2b200_translator* t, const int32_t* source_ids, const int32_t* source_lens, int64_t batch,
                            int64_t max_source_len, int beam_size, float patience, float length_penalty,
                            int64_t max_decoding_length, int64_t min_decoding_length, int num_hypotheses, int32_t start_id,
                            const int32_t* end_ids, int num_end_ids, int return_end_token, int32_t* out_ids, int32_t* out_lens,
                            float* out_scores) {
  return guarded([&] {
    CT2_REQUIRE(t && source_ids && source_lens && out_ids && out_lens && out_scores, "translate_batch: null argument");
    const TranslationRequest r = translation_request(source_ids, source_lens, batch, max_source_len, beam_size, patience,
                                                     length_penalty, max_decoding_length, min_decoding_length, num_hypotheses,
                                                     start_id, end_ids, num_end_ids, return_end_token);
    copy_hypotheses(t->impl->translate(r), batch, num_hypotheses, max_decoding_length, out_ids, out_lens, out_scores);
  });
}

CT2B200_API int ct2b200_translate_batch_attention(ct2b200_translator* t, const int32_t* source_ids, const int32_t* source_lens,
                            int64_t batch, int64_t max_source_len, int beam_size, float patience, float length_penalty,
                            int64_t max_decoding_length, int64_t min_decoding_length, int num_hypotheses, int32_t start_id,
                            const int32_t* end_ids, int num_end_ids, int return_end_token, float repetition_penalty,
                            int no_repeat_ngram_size, const int32_t* disable_ids, int num_disable_ids,
                            const int32_t* sequence_ids, const int32_t* sequence_offsets, int num_sequences,
                            float coverage_penalty, int32_t* out_ids, int32_t* out_lens, float* out_scores,
                            float* out_attention) {
  return guarded([&] {
    CT2_REQUIRE(t && source_ids && source_lens && out_ids && out_lens && out_scores, "translate_batch: null argument");
    CT2_REQUIRE(num_disable_ids >= 0 && num_sequences >= 0, "translate_batch: negative count");
    CT2_REQUIRE((num_disable_ids == 0 || disable_ids) && (num_sequences == 0 || sequence_offsets),
                "translate_batch: null processor table");
    CT2_REQUIRE(num_sequences <= kMaxSuppressSequences, "suppress_sequences: at most 4096 sequences");
    TranslationRequest r = translation_request(source_ids, source_lens, batch, max_source_len, beam_size, patience, length_penalty,
                                               max_decoding_length, min_decoding_length, num_hypotheses, start_id, end_ids,
                                               num_end_ids, return_end_token);
    r.repetition_penalty = repetition_penalty;
    r.no_repeat_ngram_size = no_repeat_ngram_size;
    r.disable_ids.assign(disable_ids, disable_ids + num_disable_ids);
    if (num_sequences > 0) {
      r.sequence_offsets.assign(sequence_offsets, sequence_offsets + num_sequences + 1);
      const int32_t total = r.sequence_offsets.back();
      CT2_REQUIRE(total >= 0 && total <= kMaxSuppressSequenceTokens && (total == 0 || sequence_ids),
                  "suppress_sequences: at most 65536 tokens in all");
      r.sequence_ids.assign(sequence_ids, sequence_ids + total);
    }
    r.coverage_penalty = coverage_penalty;
    r.attention = out_attention;
    copy_hypotheses(t->impl->translate(r), batch, num_hypotheses, max_decoding_length, out_ids, out_lens, out_scores);
  });
}

CT2B200_API int ct2b200_translate_batch_processors(ct2b200_translator* t, const int32_t* source_ids, const int32_t* source_lens,
                            int64_t batch, int64_t max_source_len, int beam_size, float patience, float length_penalty,
                            int64_t max_decoding_length, int64_t min_decoding_length, int num_hypotheses, int32_t start_id,
                            const int32_t* end_ids, int num_end_ids, int return_end_token, float repetition_penalty,
                            int no_repeat_ngram_size, const int32_t* disable_ids, int num_disable_ids,
                            const int32_t* sequence_ids, const int32_t* sequence_offsets, int num_sequences, int32_t* out_ids,
                            int32_t* out_lens, float* out_scores) {
  return ct2b200_translate_batch_attention(t, source_ids, source_lens, batch, max_source_len, beam_size, patience, length_penalty,
                                           max_decoding_length, min_decoding_length, num_hypotheses, start_id, end_ids,
                                           num_end_ids, return_end_token, repetition_penalty, no_repeat_ngram_size, disable_ids,
                                           num_disable_ids, sequence_ids, sequence_offsets, num_sequences, 0.f, out_ids,
                                           out_lens, out_scores, nullptr);
}

CT2B200_API int ct2b200_beam_decide_host(int beam_size, const int32_t* words, const int32_t* end_ids, int num_end_ids, int step,
                             int max_steps, int max_hyp, int max_candidates, int num_hypotheses, int early_exit, int include_eos,
                             int32_t* state_io, int32_t* active, int32_t* hyp_slot, int32_t* hyp_len) {
  return guarded([&] {
    CT2_REQUIRE(words && state_io && active && hyp_slot && hyp_len, "beam_decide_host: null argument");
    CT2_REQUIRE(beam_size >= 1 && beam_size <= kMaxBeam, "beam_size must be in [1, 32]");
    int w[2 * kMaxBeam];
    for (int i = 0; i < 2 * beam_size; ++i) w[i] = words[i];
    BeamDecision d;
    beam_decide(beam_size, w, end_ids, end_ids ? num_end_ids : 0, step, max_steps, state_io[2] != 0, state_io[1], state_io[0], max_hyp,
                max_candidates, num_hypotheses, early_exit, include_eos, d);
    if (!state_io[2]) {
      state_io[0] = d.num_hyp;
      state_io[1] = d.top_done;
      state_io[2] = d.finished;
    }
    for (int k = 0; k < beam_size; ++k) {
      active[k] = d.active[k];
      hyp_slot[k] = d.hyp_slot[k];
      hyp_len[k] = d.hyp_len[k];
    }
  });
}

CT2B200_API int ct2b200_translator_encode(ct2b200_translator* t, const int32_t* source_ids, const int32_t* source_lens, int64_t batch,
                              int64_t max_source_len, float* memory) {
  return guarded([&] {
    CT2_REQUIRE(t && source_ids && source_lens && memory, "translator_encode: null argument");
    t->impl->encode(source_ids, source_lens, batch, max_source_len, memory);
  });
}

CT2B200_API int ct2b200_translator_score_batch(ct2b200_translator* t, const int32_t* source_ids, const int32_t* source_lens,
                                   int64_t batch, int64_t max_source_len, const int32_t* target_ids, const int32_t* target_lens,
                                   int64_t max_target_len, int64_t offset, float* out_scores) {
  return guarded([&] {
    CT2_REQUIRE(t && source_ids && source_lens && target_ids && target_lens && out_scores, "translator_score_batch: null argument");
    t->impl->score(source_ids, source_lens, batch, max_source_len, target_ids, target_lens, max_target_len, offset, out_scores);
  });
}

CT2B200_API int ct2b200_bench_translate(ct2b200_translator* t, int64_t batch, int64_t source_len, int beam_size, int64_t steps,
                            int64_t warmup, float* encode_ms, float* decode_ms, int64_t* kernel_launches) {
  return guarded([&] {
    CT2_REQUIRE(t && encode_ms && decode_ms && kernel_launches, "bench_translate: null argument");
    t->impl->bench(batch, source_len, beam_size, steps, warmup, encode_ms, decode_ms, kernel_launches);
  });
}

// ---- Encoder ----
CT2B200_API ct2b200_encoder* ct2b200_encoder_open(const char* model_dir, const ct2b200_generator_config* config) {
  ct2b200_encoder* e = nullptr;
  const int rc = guarded([&] {
    require_device();
    CT2_REQUIRE(model_dir && config, "encoder_open: null argument");
    auto holder = std::make_unique<ct2b200_encoder>();
    holder->impl = std::make_unique<Translator>(model_dir, *config, true);
    e = holder.release();
  });
  return rc == 0 ? e : nullptr;
}

CT2B200_API void ct2b200_encoder_close(ct2b200_encoder* e) { delete e; }

CT2B200_API int ct2b200_encoder_summary(const char* model_dir, char* json_out, size_t capacity) {
  return guarded([&] {
    CT2_REQUIRE(model_dir && json_out && capacity > 0, "encoder_summary: null argument");
    ModelFile file(model_dir);
    const Seq2SeqConfig mc = parse_encoder_config(file);
    const HostVariable& pos = file.get("encoder/position_encodings/encodings");
    char buf[1024];
    const int n = std::snprintf(
        buf, sizeof(buf),
        "{\"spec\": \"%s\", \"binary_version\": %u, \"revision\": %u, \"num_layers\": %d, \"num_heads\": %d, "
        "\"head_dim\": %d, \"d_model\": %lld, \"ffn_dim\": %lld, \"vocab_size\": %lld, \"type_vocab_size\": %lld, "
        "\"max_positions\": %lld, \"weights\": \"%s\", \"pre_norm\": %s, \"activation\": %d, \"embeddings_scale\": %.9g, "
        "\"layernorm_embedding\": %s, \"final_norm\": %s, \"pooler\": %s, \"pooler_activation\": %d, "
        "\"layer_norm_epsilon\": %.9g, \"round_before_cast\": %s}",
        file.spec_name.c_str(), file.binary_version, file.revision, mc.enc_layers, mc.num_heads, mc.head_dim,
        static_cast<long long>(mc.d_model), static_cast<long long>(mc.ffn_dim), static_cast<long long>(mc.src_vocab),
        static_cast<long long>(mc.type_vocab), static_cast<long long>(pos.shape[0]), mc.weights.c_str(),
        mc.enc_pre_norm ? "true" : "false", mc.enc_activation, static_cast<double>(mc.enc_emb_scale),
        mc.has_emb_norm ? "true" : "false", mc.has_enc_final_norm ? "true" : "false", mc.has_pooler ? "true" : "false",
        mc.pooler_activation, static_cast<double>(mc.eps), mc.round_before_cast ? "true" : "false");
    CT2_REQUIRE(n > 0 && static_cast<size_t>(n) < capacity, "encoder_summary: output buffer too small");
    std::memcpy(json_out, buf, static_cast<size_t>(n) + 1);
  });
}

CT2B200_API int ct2b200_encoder_forward(ct2b200_encoder* e, const int32_t* ids, const int32_t* lengths, const int32_t* token_type_ids,
                                        int64_t batch, int64_t max_length, float* last_hidden_state, float* pooler_output) {
  return guarded([&] {
    CT2_REQUIRE(e && ids && lengths && last_hidden_state, "encoder_forward: null argument");
    e->impl->encoder_forward(ids, token_type_ids, lengths, batch, max_length, last_hidden_state, pooler_output);
  });
}

CT2B200_API int ct2b200_encoder_bench(ct2b200_encoder* e, const int32_t* lengths, int64_t batch, int64_t max_length, int64_t iters,
                                      int64_t warmup, float* median_ms) {
  return guarded([&] {
    CT2_REQUIRE(e && lengths && median_ms, "encoder_bench: null argument");
    e->impl->encoder_bench(lengths, batch, max_length, iters, warmup, median_ms);
  });
}

// ---- Whisper ----
CT2B200_API int ct2b200_whisper_info(const ct2b200_translator* t, int* n_mels, int* max_frames, int* d_model, int* vocab_size) {
  return guarded([&] {
    CT2_REQUIRE(t, "null translator");
    const Seq2SeqConfig& c = t->impl->config();
    CT2_REQUIRE(c.whisper, "not a Whisper model");
    if (n_mels) *n_mels = static_cast<int>(c.n_mels);
    if (max_frames) *max_frames = static_cast<int>(c.max_frames);
    if (d_model) *d_model = static_cast<int>(c.d_model);
    if (vocab_size) *vocab_size = static_cast<int>(c.tgt_vocab);
  });
}

CT2B200_API int ct2b200_whisper_encode(ct2b200_translator* t, const float* features, int64_t batch, int64_t frames, float* memory) {
  return guarded([&] {
    CT2_REQUIRE(t && features && memory, "whisper_encode: null argument");
    t->impl->whisper_encode(features, batch, frames, memory);
  });
}

namespace {
int whisper_generate(ct2b200_translator* t, const float* features, int64_t batch, int64_t frames, const int32_t* prompts,
                     int64_t prompt_len, int beam_size, float patience, float length_penalty, int64_t max_length, int num_hypotheses,
                     const int32_t* suppress_ids, int num_suppress, const int32_t* suppress_begin, int num_begin, int32_t sot_id,
                     int32_t eot_id, int32_t no_speech_id, int32_t no_timestamps_id, int max_initial_timestamp_index,
                     int sampling_topk, float sampling_temperature, int32_t* out_ids, int32_t* out_lens, float* out_scores,
                     float* no_speech) {
  return guarded([&] {
    CT2_REQUIRE(t && features && prompts && out_ids && out_lens && out_scores, "whisper_generate: null argument");
    WhisperRequest r;
    r.features = features;
    r.batch = batch;
    r.frames = frames;
    r.prompts = prompts;
    r.prompt_len = prompt_len;
    r.beam_size = beam_size;
    r.patience = patience;
    r.length_penalty = length_penalty;
    r.max_length = max_length;
    r.num_hypotheses = num_hypotheses;
    r.suppress_ids.assign(suppress_ids, suppress_ids + (suppress_ids ? num_suppress : 0));
    r.suppress_ids_begin.assign(suppress_begin, suppress_begin + (suppress_begin ? num_begin : 0));
    r.sot_id = sot_id;
    r.eot_id = eot_id;
    r.no_speech_id = no_speech_id;
    r.no_timestamps_id = no_timestamps_id;
    r.max_initial_timestamp_index = max_initial_timestamp_index;
    r.sampling_topk = sampling_topk;
    r.sampling_temperature = sampling_temperature;
    copy_hypotheses(t->impl->whisper_generate(r, no_speech), batch, num_hypotheses, max_length, out_ids, out_lens, out_scores);
  });
}
}  // namespace

CT2B200_API int ct2b200_whisper_generate(ct2b200_translator* t, const float* features, int64_t batch, int64_t frames,
                             const int32_t* prompts, int64_t prompt_len, int beam_size, float patience, float length_penalty,
                             int64_t max_length, int num_hypotheses, const int32_t* suppress_ids, int num_suppress,
                             const int32_t* suppress_begin, int num_begin, int32_t sot_id, int32_t eot_id, int32_t no_speech_id,
                             int32_t no_timestamps_id, int max_initial_timestamp_index, int32_t* out_ids, int32_t* out_lens,
                             float* out_scores, float* no_speech) {
  return whisper_generate(t, features, batch, frames, prompts, prompt_len, beam_size, patience, length_penalty, max_length,
                          num_hypotheses, suppress_ids, num_suppress, suppress_begin, num_begin, sot_id, eot_id, no_speech_id,
                          no_timestamps_id, max_initial_timestamp_index, 1, 1.f, out_ids, out_lens, out_scores, no_speech);
}

CT2B200_API int ct2b200_whisper_generate_sampling(ct2b200_translator* t, const float* features, int64_t batch, int64_t frames,
                                                  const int32_t* prompts, int64_t prompt_len, int beam_size, float patience,
                                                  float length_penalty, int64_t max_length, int num_hypotheses,
                                                  const int32_t* suppress_ids, int num_suppress, const int32_t* suppress_begin,
                                                  int num_begin, int32_t sot_id, int32_t eot_id, int32_t no_speech_id,
                                                  int32_t no_timestamps_id, int max_initial_timestamp_index, int sampling_topk,
                                                  float sampling_temperature, int32_t* out_ids, int32_t* out_lens,
                                                  float* out_scores, float* no_speech) {
  return whisper_generate(t, features, batch, frames, prompts, prompt_len, beam_size, patience, length_penalty, max_length,
                          num_hypotheses, suppress_ids, num_suppress, suppress_begin, num_begin, sot_id, eot_id, no_speech_id,
                          no_timestamps_id, max_initial_timestamp_index, sampling_topk, sampling_temperature, out_ids, out_lens,
                          out_scores, no_speech);
}

CT2B200_API int ct2b200_whisper_align(ct2b200_translator* t, const float* features, int64_t batch, int64_t frames,
                                      const int32_t* start_ids, int64_t start_len, const int32_t* text_ids, const int32_t* text_lens,
                                      int64_t max_text, const int32_t* num_frames, int median_filter_width, const int32_t* heads,
                                      int num_heads, int32_t no_timestamps_id, int32_t eot_id, int32_t* out_path,
                                      int32_t* out_path_lens, float* out_probs, float* matrix) {
  return guarded([&] {
    CT2_REQUIRE(t && features && start_ids && text_lens && num_frames && heads && out_path && out_path_lens && out_probs,
                "whisper_align: null argument");
    CT2_REQUIRE(max_text == 0 || text_ids, "whisper_align: null argument");
    WhisperAlignRequest r;
    r.features = features;
    r.batch = batch;
    r.frames = frames;
    r.start = start_ids;
    r.start_len = start_len;
    r.text = text_ids;
    r.text_lens = text_lens;
    r.max_text = max_text;
    r.num_frames = num_frames;
    r.median_filter_width = median_filter_width;
    for (int i = 0; i < num_heads; ++i) r.heads.emplace_back(heads[2 * i], heads[2 * i + 1]);
    r.no_timestamps_id = no_timestamps_id;
    r.eot_id = eot_id;
    const std::vector<WhisperAlignResult> res = t->impl->whisper_align(r, matrix);
    const int64_t max_path = max_text + 1 + (frames + 1) / 2;
    for (int64_t b = 0; b < batch; ++b) {
      const auto& p = res[b].path;
      CT2_REQUIRE(static_cast<int64_t>(p.size()) <= max_path, "whisper_align: path longer than expected");
      for (size_t i = 0; i < p.size(); ++i) {
        out_path[(b * max_path + i) * 2] = static_cast<int32_t>(p[i].first);
        out_path[(b * max_path + i) * 2 + 1] = static_cast<int32_t>(p[i].second);
      }
      out_path_lens[b] = static_cast<int32_t>(p.size());
      for (int64_t i = 0; i < max_text; ++i)
        out_probs[b * max_text + i] = i < static_cast<int64_t>(res[b].text_token_probs.size()) ? res[b].text_token_probs[i] : 0.f;
    }
  });
}

CT2B200_API int ct2b200_whisper_detect_language(ct2b200_translator* t, const float* features, int64_t batch, int64_t frames,
                                                int32_t sot_id, const int32_t* lang_ids, int num_langs, float* probs) {
  return guarded([&] {
    CT2_REQUIRE(t && features && lang_ids && probs, "whisper_detect_language: null argument");
    t->impl->whisper_detect_language(features, batch, frames, sot_id, std::vector<int32_t>(lang_ids, lang_ids + num_langs), probs);
  });
}

CT2B200_API int ct2b200_negative_dtw_host(const float* x, int64_t n, int64_t m, int32_t* out_path, int32_t* out_len) {
  return guarded([&] {
    CT2_REQUIRE(x && out_path && out_len && n >= 1 && m >= 1, "negative_dtw_host: bad argument");
    const auto p = negative_dtw(x, n, m);
    for (size_t i = 0; i < p.size(); ++i) {
      out_path[2 * i] = static_cast<int32_t>(p[i].first);
      out_path[2 * i + 1] = static_cast<int32_t>(p[i].second);
    }
    *out_len = static_cast<int32_t>(p.size());
  });
}

}  // extern "C"
