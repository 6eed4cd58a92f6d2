/* ct2b200.h — C-ABI of the H100-native (sm_90a) quantized-transformer decode path.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  CTranslate2 has no C plugin interface: its
 * boundary is the set of C++ `<Device::CUDA>` template specialisations listed below.  Every entry
 * point here is what one of those specialisations would call; the comment above each function cites
 * the reference interface it replaces (paths relative to the reference tree).  INTEGRATION.md shows
 * the reference-side shims.
 *
 * Conventions
 *  - plain pointers and sizes only; no torch / C++ types cross this boundary;
 *  - `*_d` pointers are DEVICE pointers, row-major, caller-owned, 16-byte aligned; `*_h` are HOST;
 *  - `stream` is a cudaStream_t passed as void* (0 = legacy default stream); op-level functions
 *    never allocate and never synchronise (split-K scratch comes from ct2b200_workspace_*);
 *  - every function returns 0 on success, non-zero on error; ct2b200_last_error() gives the
 *    message (thread-local).  Shape/argument errors mirror the reference's std::invalid_argument,
 *    CUDA failures its std::runtime_error (src/cuda/utils.h:51-96);
 *  - there is NO CPU fallback: without a CUDA device every compute call fails with an error.
 */
#ifndef CT2B200_H_
#define CT2B200_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define CT2B200_API __attribute__((visibility("default")))
#else
#define CT2B200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* include/ctranslate2/types.h:16-24 (DataType) — the float types activations may use. */
typedef enum { CT2B200_F32 = 0, CT2B200_F16 = 1, CT2B200_BF16 = 2 } ct2b200_dtype;

/* include/ctranslate2/ops/activation.h:9-17 (ActivationType), same order; -1 = none. */
typedef enum {
  CT2B200_ACT_NONE = -1, CT2B200_ACT_RELU = 0, CT2B200_ACT_GELU_TANH = 1, CT2B200_ACT_SWISH = 2,
  CT2B200_ACT_GELU = 3, CT2B200_ACT_GELU_SIGMOID = 4, CT2B200_ACT_TANH = 5, CT2B200_ACT_SIGMOID = 6
} ct2b200_activation;

/* INT8 GEMM implementation selector (diagnostics / tests; AUTO is what the engine uses). */
typedef enum { CT2B200_GEMM_AUTO = 0, CT2B200_GEMM_TCGEN05 = 1, CT2B200_GEMM_MMA_SYNC = 2 } ct2b200_gemm_impl;

CT2B200_API const char* ct2b200_last_error(void);
CT2B200_API const char* ct2b200_version(void);
/* Number of CUDA kernels this library has launched in the calling process (all threads). */
CT2B200_API int64_t ct2b200_kernel_launch_count(void);
/* Device properties the host side sizes grids with; fails when there is no sm_90 device. */
CT2B200_API int ct2b200_device_info(int device, int* sm_count, int* cc_major, int* cc_minor, size_t* total_mem);

/* ---------------------------------------------------------------------------------------------
 * Op level (SURVEY §8 a1-a5, a7, a9-a12, a14, a17)
 * ------------------------------------------------------------------------------------------- */

/* ops::Quantize::quantize<Device::CUDA,T,int8_t> — include/ctranslate2/ops/quantize.h:22-24,
 * src/ops/quantize_gpu.cu:57-105.  x [rows,cols] T -> q int8 [rows,cols], scale f32 [rows]. */
CT2B200_API int ct2b200_quantize_rows(const void* x_d, int dtype, int64_t rows, int64_t cols, int round_before_cast,
                          int8_t* q_d, float* scale_d, void* stream);

/* primitives<Device::CUDA>::gemm<int8_t,int32_t>(…trans_b=true, alpha=1, beta=0) —
 * include/ctranslate2/primitives.h:213-232, src/cuda/primitives.cu:571-597.
 * a [m,k] int8, b [n,k] int8 -> c [m,n] int32 (exact). k % 16 == 0. */
CT2B200_API int ct2b200_gemm_s8(const int8_t* a_d, const int8_t* b_d, int64_t m, int64_t n, int64_t k, int32_t* c_d,
                    int impl, void* stream);

/* ops::Dequantize::dequantize_gemm_output<Device::CUDA,T> — include/ctranslate2/ops/dequantize.h:19-25,
 * src/ops/dequantize_gpu.cu:30-144.  y = act(c / (a_scale[i]*b_scale[j]) + bias[j]).  bias may be NULL. */
CT2B200_API int ct2b200_dequantize_gemm_output(const int32_t* c_d, const float* a_scale_d, const float* b_scale_d,
                                   const void* bias_d, int act, int64_t m, int64_t n, void* y_d, int dtype,
                                   void* stream);

/* ops::Dequantize::dequantize<Device::CUDA,int8_t,T> (embedding rows) — src/ops/dequantize_gpu.cu:16-27:
 * y[i,:] = x[i,:] / scale[i]. */
CT2B200_API int ct2b200_dequantize_rows(const int8_t* x_d, const float* scale_d, int64_t rows, int64_t cols, void* y_d,
                            int dtype, void* stream);

/* layers::Dense::operator(), quantized arm, as ONE fused launch — src/layers/common.cc:353-401:
 *   y = act(gemm_s8(xq, w) / (x_scale[i]*w_scale[j]) + bias[j]) + residual[i,j]
 * xq [m,k] int8 with x_scale [m] (from ct2b200_quantize_rows / ct2b200_rms_norm_quantize),
 * w [n,k] int8 with w_scale [n]; bias [n] T or NULL; residual [m,n] T or NULL; y [m,n] T. */
CT2B200_API int ct2b200_dense_s8(const int8_t* xq_d, const float* x_scale_d, const int8_t* w_d, const float* w_scale_d,
                     const void* bias_d, const void* residual_d, int act, int64_t m, int64_t n, int64_t k,
                     void* y_d, int dtype, int impl, void* stream);

/* FeedForwardNetwork gate/up pair (src/layers/transformer.cc:21-51 with ffn_glu): fused
 *   h = act(dense(xq, w_gate)) * dense(xq, w_up)       h [m,n] T
 * replacing Dense(linear_0)+Dense(linear_0_noact)+ops::Mul. */
CT2B200_API int ct2b200_dense_s8_glu(const int8_t* xq_d, const float* x_scale_d, const int8_t* w_gate_d,
                         const float* w_gate_scale_d, const int8_t* w_up_d, const float* w_up_scale_d, int act,
                         int64_t m, int64_t n, int64_t k, void* h_d, int dtype, int impl, void* stream);

/* The whole quantized arm of layers::Dense::operator() INCLUDING its input side —
 * src/layers/common.cc:353-401 preceded by ops::Quantize (quantize.cc:21-50) or, with gamma_d, by the layer's pre-norm
 * ops::RMSNorm (rms_norm_gpu.cu:19-63):  xq, x_scale = Quantize([RMSNorm(x, gamma, eps)]);  y = dense_s8(xq, x_scale, ...).
 * x [m,k] T; xq_d [m,k] int8 and x_scale_d [m] are OUTPUTS (the same bits ct2b200_quantize_rows / ct2b200_rms_norm_quantize
 * produce).  Runs as the register-resident row kernel + the fused Dense under programmatic dependent launch. */
CT2B200_API int ct2b200_dense_s8_rows(const void* x_d, const void* gamma_d, float eps, const int8_t* w_d, const float* w_scale_d,
                          const void* bias_d, const void* residual_d, int act, int64_t m, int64_t n, int64_t k,
                          void* y_d, int dtype, int8_t* xq_d, float* x_scale_d, void* stream);
/* same for the gate/up pair: h = act(dense(xq, w_gate)) * dense(xq, w_up) */
CT2B200_API int ct2b200_dense_s8_glu_rows(const void* x_d, const void* gamma_d, float eps, const int8_t* w_gate_d,
                              const float* w_gate_scale_d, const int8_t* w_up_d, const float* w_up_scale_d, int act,
                              int64_t m, int64_t n, int64_t k, void* h_d, int dtype, int8_t* xq_d, float* x_scale_d,
                              void* stream);

/* primitives<Device::CUDA>::gemm<float16_t|bfloat16_t> (trans_b, alpha 1, beta 0) + ops::Gemm's
 * apply_bias_and_activation — src/cuda/primitives.cu:485-569, src/ops/gemm.cc:10-25.
 * a [m,k] T, b [n,k] T -> c [m,n] T, fp32 accumulation; dtype F16 or BF16. */
CT2B200_API int ct2b200_gemm_f16(const void* a_d, const void* b_d, const void* bias_d, const void* residual_d, int act,
                     int64_t m, int64_t n, int64_t k, void* c_d, int dtype, void* stream);

/* primitives<Device::CUDA>::gemm<float,float> (trans_b, alpha 1, beta 0) + apply_bias_and_activation —
 * src/cuda/primitives.cu:485-505 (cublasSgemm), src/ops/gemm.cc:10-25.  True fp32 FMAs (no TF32). */
CT2B200_API int ct2b200_gemm_f32(const float* a_d, const float* b_d, const float* bias_d, const float* residual_d, int act,
                     int64_t m, int64_t n, int64_t k, float* c_d, void* stream);

/* ops::LayerNorm::compute<Device::CUDA,T> (last axis) — include/ctranslate2/ops/layer_norm.h, src/ops/layer_norm_gpu.cu:33-66,
 * 169-206: y = (x - mean) * rsqrt(var + eps) * gamma + beta.  y_d may be NULL when only the quantized row is wanted;
 * q_d / scale_d non-NULL adds ops::Quantize of T(y) in the same launch (layers::LayerNorm + Dense's Quantize). */
CT2B200_API int ct2b200_layer_norm(const void* x_d, const void* gamma_d, const void* beta_d, int64_t rows, int64_t cols, float eps,
                       void* y_d, int8_t* q_d, float* scale_d, int round_before_cast, int dtype, void* stream);

/* ops::RMSNorm::compute<Device::CUDA,T> — include/ctranslate2/ops/rms_norm.h, src/ops/rms_norm_gpu.cu:19-63. */
CT2B200_API int ct2b200_rms_norm(const void* gamma_d, const void* x_d, int64_t rows, int64_t cols, float eps,
                     int use_residual, void* y_d, int dtype, void* stream);

/* RMSNorm followed by Quantize in one launch (layers::LayerNorm + Dense's Quantize,
 * src/layers/common.cc:464-472 + :392): q = quantize(T(rms_norm(x))). */
CT2B200_API int ct2b200_rms_norm_quantize(const void* gamma_d, const void* x_d, int64_t rows, int64_t cols, float eps,
                              int use_residual, int8_t* q_d, float* scale_d, int dtype, void* stream);

/* ops::Rotary::compute<Device::CUDA,T> — include/ctranslate2/ops/rotary.h, src/ops/rotary_gpu.cu:27-85.
 * x [batch, time, depth] rows (batch = b*h when transposed), sin/cos [time, ndims] T. */
CT2B200_API int ct2b200_rotary(const void* x_d, const void* sin_d, const void* cos_d, int64_t batch, int64_t time,
                   int64_t depth, int64_t ndims, int interleave, void* y_d, int dtype, void* stream);

/* ops::SoftMax::compute<Device::CUDA,T> (log=0) / LogSoftMax (log=1) — src/ops/softmax_gpu.cu:190-256.
 * lengths_d int32 [rows] or NULL. */
CT2B200_API int ct2b200_softmax(const void* x_d, const int32_t* lengths_d, int64_t rows, int64_t cols, int log, void* y_d,
                    int dtype, void* stream);

/* ops::LogSoftMax followed by ops::Gather(axis=-1, batch_dims=1) — src/scoring.cc:50-56, src/ops/softmax_gpu.cu:190-256,
 * src/ops/gather_gpu.cu — fused, without writing the log-probabilities: x_d [rows, cols] T (any width, any T-aligned
 * address), ids_d int32 [rows]; y_d f32 [rows] = float(T(x[r, ids[r]] - max_r - log(sum exp(x[r, :] - max_r)))), NaN for an
 * id outside [0, cols). */
CT2B200_API int ct2b200_log_softmax_gather(const void* x_d, const int32_t* ids_d, int64_t rows, int64_t cols, float* y_d,
                               int dtype, void* stream);

/* ops::TopK::compute<Device::CUDA,T,int32_t> — include/ctranslate2/ops/topk.h, src/ops/topk_gpu.cu:181-335.
 * Descending values; exact ties resolve lowest index first (SURVEY §8 a17).  k <= 64. */
CT2B200_API int ct2b200_topk(const void* x_d, int64_t rows, int64_t cols, int k, void* values_d, int32_t* indices_d,
                 int dtype, void* stream);

/* RandomSampler::sample (src/sampling.cc:34-101) on rows x_d [rows, cols] T: keep the top k of the row (value desc, index asc;
 * k = 0 or k = cols keeps all), weights exp((x - max) / temperature), one draw by inverse CDF in ascending index order against
 * u * sum, where u = philox_uniform(seed, counter, row, step) (csrc/kernels/philox.h).  ids_d int32 [rows] = the drawn ids,
 * logp_d f32 [rows] = T(LogSoftMax(x))[id], the log-probability of the unscaled row.  k in [0, cols], temperature > 0. */
CT2B200_API int ct2b200_random_sample(const void* x_d, int64_t rows, int64_t cols, int k, float temperature, uint32_t seed,
                                      uint32_t counter, uint32_t step, int32_t* ids_d, float* logp_d, int dtype, void* stream);
/* set_random_seed (src/random.cc): the process-wide seed of sampled searches; also resets the sampling-call counter, so the
 * same sequence of calls after the same seed gives the same results.  Without it a seed is drawn once from
 * std::random_device. */
CT2B200_API int ct2b200_set_random_seed(uint32_t seed);
/* Host only (no device): Philox4x32-10 of counter_h [4] under key_h [2] -> out_h [4], the generator of the sampling kernels. */
CT2B200_API int ct2b200_philox4x32_host(const uint32_t* counter_h, const uint32_t* key_h, uint32_t* out_h);

/* ops::Gather::compute<Device::CUDA,T>(axis 0) — src/ops/gather_gpu.cu:52-91.  Row copy of `row_bytes`. */
CT2B200_API int ct2b200_gather_rows(const void* data_d, const int32_t* ids_d, int64_t num_ids, int64_t row_bytes,
                        void* out_d, void* stream);

/* layers::Embeddings::operator() with INT8 weights — src/layers/common.cc:64-81
 * (Gather rows + Gather scales + Dequantize) in one launch: y[i,:] = w[ids[i],:] / scale[ids[i]]. */
CT2B200_API int ct2b200_embedding_s8(const int8_t* w_d, const float* scale_d, const int32_t* ids_d, int64_t num_ids,
                         int64_t depth, void* y_d, int dtype, void* stream);

/* ops::Mul + ops::Quantize of the SwiGLU product — q = quantize(T(gate*up)) (transformer.cc:31-37). */
CT2B200_API int ct2b200_mul_quantize(const void* gate_d, const void* up_d, int64_t rows, int64_t cols, int8_t* q_d,
                         float* scale_d, int dtype, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Attention (SURVEY §8 a8-a13): layers::MultiHeadAttention::operator() between the QKV Dense and
 * the output Dense — src/layers/attention.cc:485-602; FlashMultiHeadAttention src/layers/flash_attention.cc:18-137.
 *
 * KV cache layout (un-replicated GQA): k_cache / v_cache [batch_slots, num_heads_kv, max_len, head_dim] T.
 * qkv [rows, (H + 2*Hkv) * head_dim] T is the fused linear_0 output ([q | k | v]).
 * sin/cos tables [max_positions, head_dim] f32 (built like RotaryEmbeddings::initialize).
 * ------------------------------------------------------------------------------------------- */

/* Decode step (one new token per sequence): rotary(q,k) at position lens[b], append k/v at lens[b],
 * softmax(q k^T / sqrt(d)) v over positions 0..lens[b].  out [batch, H*head_dim] T.
 * lens_d int32 [batch] = tokens already cached per row (not modified).  head_dim must be 128 or 64 or 32.
 * The caches must hold finite values everywhere (zero-initialise them once): whole 64-key boxes are staged and the
 * keys past lens_d[b] are masked, not skipped.  workspace_d: ct2b200_attention_decode_workspace bytes, zeroed once. */
CT2B200_API int ct2b200_attention_decode(const void* qkv_d, void* k_cache_d, void* v_cache_d, const float* sin_d,
                             const float* cos_d, const int32_t* lens_d, int64_t batch, int num_heads,
                             int num_heads_kv, int head_dim, int64_t max_len, int rotary_interleave,
                             float scale, void* out_d, void* workspace_d, size_t workspace_bytes, int dtype,
                             void* stream);
CT2B200_API size_t ct2b200_attention_decode_workspace(int64_t batch, int num_heads, int head_dim, int64_t max_len);

/* Prefill (T new tokens per sequence starting at position `offset`, causal): qkv [batch*time, ...],
 * lengths_d int32 [batch] = valid new tokens per row (NULL = time).  out [batch*time, H*head_dim] T. */
CT2B200_API int ct2b200_attention_prefill(const void* qkv_d, void* k_cache_d, void* v_cache_d, const float* sin_d,
                              const float* cos_d, const int32_t* lengths_d, int64_t batch, int64_t time,
                              int64_t offset, int num_heads, int num_heads_kv, int head_dim, int64_t max_len,
                              int rotary_interleave, float scale, void* out_d, int dtype, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Encoder-decoder attention (layers::MultiHeadAttention of TransformerEncoder / TransformerDecoder, dot_product_attention,
 * src/layers/attention.cc:178-287): the kernel the Translator and Whisper run, exposed op by op.  Any head_dim; one warp per
 * (query row, head); scores T(scale * q.k), probabilities T(softmax), context T(sum p.v).  d = H * D, every row is T.
 * These calls fail with "invalid argument" when the per-warp score buffer (4 * (keys + D) floats) would exceed 200 KB.
 * ------------------------------------------------------------------------------------------- */

/* Encoder self-attention: qkv_d [batch * S, 3d] ([q | k | v]); row (b, t) attends to rows (b, j), j < lengths_d[b]
 * (NULL = S; a length of 0 gives a zero row).  out_d [batch * S, d]. */
CT2B200_API int ct2b200_attention_encoder(const void* qkv_d, const int32_t* lengths_d, int64_t batch, int S, int H, int D,
                                          float scale, void* out_d, int dtype, void* stream);
/* The same encoder self-attention on tensor cores (the kernel of encoder-only models, ct2b200_encoder_open): mma.sync
 * m16n8k16 tiles of 64 queries x 64 keys, fp32 online softmax, P rounded to T before P.V (flash-attention style instead of
 * the reference's MatMul + SoftMax + MatMul, src/layers/attention.cc:178-287).  fp16 / bf16 and head_dim 64 or 128 only
 * ("invalid argument" otherwise).  Key tiles past lengths_d[b] are not read; query tiles wholly past it are written as zeros,
 * the other rows past it attend like the valid ones. */
CT2B200_API int ct2b200_attention_encoder_mma(const void* qkv_d, const int32_t* lengths_d, int64_t batch, int S, int H, int D,
                                              float scale, void* out_d, int dtype, void* stream);
/* Teacher-forced causal decoder self-attention: qkv_d [batch * time, 3d]; row (b, t) attends to rows (b, j), j <= t.
 * out_d [batch * time, d]. */
CT2B200_API int ct2b200_attention_causal(const void* qkv_d, int64_t batch, int time, int H, int D, float scale, void* out_d,
                                         int dtype, void* stream);
/* One-token decoder self-attention over a beam-remapped cache: k_cache_d / v_cache_d [rows, max_len, d];
 * anc_d int32 [2][rows, max_len] (the table of parity *step_d & 1 is read); key j < step of row n lives at
 * (anc[n][j], j).  The row's new k / v (columns d.. and 2d.. of qkv_d [rows, 3d]) are written to (n, step).
 * step_d: int32 [1] on the device, step < max_len.  out_d [rows, d]. */
CT2B200_API int ct2b200_attention_beam_self(const void* qkv_d, void* k_cache_d, void* v_cache_d, const int32_t* anc_d,
                                            const int32_t* step_d, int64_t rows, int max_len, int H, int D, float scale,
                                            void* out_d, int dtype, void* stream);
/* Cross-attention: q_d [rows, d]; kv_d [batch * S, 2d] ([k | v]) with batch = rows / beam; row n attends to the first
 * lengths_d[n / beam] (NULL = S) rows of entry n / beam.  out_d [rows, d].  capture_out_d NULL: plain cross-attention.
 * Otherwise the scores T(scale * q.k) of the selected heads are also written, as f32, to
 * capture_out_d [batch, total, beam, S]: bit k of masks_d[h] (uint32 [H], device) sends head h to slot first + k, which must
 * be below total; positions at or past the entry's length are not written. */
CT2B200_API int ct2b200_attention_cross(const void* q_d, const void* kv_d, const int32_t* lengths_d, int64_t rows, int beam,
                                        int S, int H, int D, float scale, void* out_d, float* capture_out_d,
                                        const uint32_t* masks_d, int first, int total, int dtype, void* stream);
/* One beam-search step of every row (BeamSearch::search, src/decoding.cc:425-720): end ids disabled while *step_d <
 * min_length (in place in logits_d), LogSoftMax, + cum_d[row], then the row's best 2 * beam candidates ordered by
 * (score desc, index asc), ids flattened over [beam, vocab] (row % beam) and (-inf, -1) past the vocabulary.
 * logits_d [batch * beam, vocab_ld] T; cum_d [batch * beam] T; row_scores_d T / row_ids_d int32 [batch * beam, 2 * beam].
 * beam must be in [1, 8]. */
CT2B200_API int ct2b200_beam_rows(void* logits_d, const void* cum_d, int32_t* step_d, int batch, int beam, int vocab,
                                  int64_t vocab_ld, int min_length, const int32_t* end_ids_d, int num_end, void* row_scores_d,
                                  int32_t* row_ids_d, int dtype, void* stream);

/* ---------------------------------------------------------------------------------------------
 * AWQ-INT4 (SURVEY §8 a7): ops::GemmAwq / GemvAwq / DequantizeAwq — include/ctranslate2/ops/awq/{gemm,gemv,dequantize}.h,
 * src/ops/awq/{gemm,gemv,dequantize}_gpu.cu.  x [m,k] f16 -> y [m,n] f16.
 * layout 1 = AWQ_GEMM: qweight int32 [k, n/8], scales f16 [k/g, n], qzeros int32 [k/g, n/8]
 * layout 2 = AWQ_GEMV: qweight int32 [n, k/8], scales f16 [n, sf_w], qzeros int32 [n, zeros_w]
 * ------------------------------------------------------------------------------------------- */
/* One-time repack (Dense ctor / model load) of either reference layout into the native K-major layout:
 * wp int32 [n, k/8] (channel 8w+i of row n in nibble {0,4,1,5,2,6,3,7}[i] of word w), sc f16 [n, k/g], zr f16 [n, k/g],
 * and (sz_d non-NULL) the same {scale, zero} values as f16 pairs in group-major order sz [k/g, n][2]: the decode kernel
 * (m <= 64) stages the 128 pairs of a tile and group with one bulk copy and needs it; NULL = not produced. */
CT2B200_API int ct2b200_awq_repack(const int32_t* qweight_d, const void* scales_d, const int32_t* qzeros_d, int layout,
                       int group_size, int64_t n, int64_t k, int32_t* wp_d, void* sc_d, void* zr_d, void* sz_d,
                       void* stream);

/* ops::GemmAwq / GemvAwq + apply_bias_and_activation — src/ops/awq/gemm.cc:8-33, gemv.cc:9-37, on the native layout:
 * y = act(x . deq(W)^T + bias) + residual.  m <= 64: fused dequantize + wgmma GEMM (weight-streaming kernel with the
 * operand in registers when sz_d is given, the general kernel otherwise).  m > 64 (the reference's
 * DequantizeAwq + cuBLAS arm, src/layers/common.cc:409-420): needs scratch_nk_d, an fp16 [n,k] buffer. */
CT2B200_API int ct2b200_dense_awq(const void* x_d, const int32_t* wp_d, const void* sc_d, const void* zr_d, const void* sz_d,
                      int group_size, const void* bias_d, const void* residual_d, int act, int64_t m, int64_t n, int64_t k,
                      void* y_d, void* scratch_nk_d, void* stream);
/* gate/up pair of the gated FFN in one pass: h = act(x . deq(Wg)^T) * (x . deq(Wu)^T).  m > 64 also needs scratch_mn_d. */
CT2B200_API int ct2b200_dense_awq_glu(const void* x_d, const int32_t* wp_gate_d, const void* sc_gate_d, const void* zr_gate_d,
                          const void* sz_gate_d, const int32_t* wp_up_d, const void* sc_up_d, const void* zr_up_d,
                          const void* sz_up_d, int group_size, int act, int64_t m, int64_t n, int64_t k, void* h_d,
                          void* scratch_nk_d, void* scratch_mn_d, void* stream);
/* ops::DequantizeAwq — src/ops/awq/dequantize_gpu.cu:8-62: reference layout (1 or 2) -> W f16 [k, n]. */
CT2B200_API int ct2b200_dequantize_awq(const int32_t* qweight_d, const void* scales_d, const int32_t* qzeros_d, int layout,
                           int group_size, int64_t n, int64_t k, void* w_d /* f16 [k,n] */, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Engine level: models::Model::load + Generator (SURVEY §8 a16, a17, a20; §3.1).
 * ctranslate2::Generator — include/ctranslate2/generator.h:11-39; GenerationOptions generation.h:14-78.
 * Token strings <-> ids (Vocabulary) stay on the caller's side of the boundary; ids cross it.
 * ------------------------------------------------------------------------------------------- */
typedef struct ct2b200_generator ct2b200_generator;

/* Weight type requested by the compute type (models::Model::set_compute_type / ensure_dtype, src/models/model.cc:178-234,
 * 304-369): STORED = "default" (keep what model.bin holds), INT8 = the int8* compute types (float weights are quantized at
 * load: scale = 127 / amax per row, q = rint(w * scale)), FLOAT = float16 / bfloat16 (int8 weights are dequantized at load).
 * The conversion runs on the GPU.  AWQ-INT4 models ignore it (the reference pins ComputeType::FLOAT16, model.cc:750-757). */
typedef enum { CT2B200_WEIGHTS_STORED = 0, CT2B200_WEIGHTS_INT8 = 1, CT2B200_WEIGHTS_FLOAT = 2 } ct2b200_weight_type;

typedef struct {
  int device;               /* CUDA device ordinal */
  int compute_type;         /* ct2b200_dtype of activations / KV cache */
  int64_t max_batch;        /* batch slots to reserve */
  int64_t max_length;       /* max total positions (prompt + generated) per sequence */
  int tp_rank, tp_size;     /* tensor-parallel rank/size (1 = off); see ct2b200_generator_tp_connect */
  int use_cuda_graph;       /* capture the decode step in a CUDA graph */
  int gemm_impl;            /* ct2b200_gemm_impl */
  int weight_type;          /* ct2b200_weight_type: what Model::set_compute_type asks of the Dense / embedding weights */
} ct2b200_generator_config;

/* models::Model::load(model_dir, Device::CUDA, device, compute_type) + Generator ctor.
 * Reads model.bin (binary versions 2..6), config.json. */
CT2B200_API ct2b200_generator* ct2b200_generator_open(const char* model_dir, const ct2b200_generator_config* config);
CT2B200_API void ct2b200_generator_close(ct2b200_generator* g);
CT2B200_API int ct2b200_generator_vocab_size(const ct2b200_generator* g);
CT2B200_API int ct2b200_generator_info(const ct2b200_generator* g, int* num_layers, int* num_heads, int* num_heads_kv,
                           int* head_dim, int* d_model, int64_t* weight_bytes);

/* Host only (no device needed): what models::Model::load would find in `model_dir` — spec, binary version, decoder geometry
 * (layers, heads, kv heads, head_dim, d_model, ffn_dim, vocabulary) and the storage type of the linear layers, as a JSON
 * object written to json_out.  The same parser configures ct2b200_generator_open. */
CT2B200_API int ct2b200_model_summary(const char* model_dir, char* json_out, size_t capacity);

/* Generator::generate_batch_async(...).get(), greedy (beam_size 1, sampling_topk 1),
 * include_prompt_in_result=false.  HOST buffers:
 *   prompt_ids_h [batch, max_prompt_len] int32 (right-padded), prompt_lens_h [batch];
 *   end_ids_h [num_end_ids]; out_ids_h [batch, max_length] int32 (filled with -1 past the end),
 *   out_lens_h [batch].  max_length / min_length count generated tokens (generation.h:41-43). */
CT2B200_API int ct2b200_generate_batch(ct2b200_generator* g, const int32_t* prompt_ids_h, const int32_t* prompt_lens_h,
                           int64_t batch, int64_t max_prompt_len, int64_t max_length, int64_t min_length,
                           const int32_t* end_ids_h, int num_end_ids, int return_end_token,
                           int32_t* out_ids_h, int32_t* out_lens_h);

/* The same with GenerationOptions::return_scores = true: out_scores_h [batch] = sum of the log-probabilities of the
 * generated tokens (LogSoftMax of the processed logits, the end token's included) / length^length_penalty
 * (src/decoding.cc:875-923, 189-203; include/ctranslate2/generation.h:22-23, 55). */
CT2B200_API int ct2b200_generate_batch_scores(ct2b200_generator* g, const int32_t* prompt_ids_h, const int32_t* prompt_lens_h,
                           int64_t batch, int64_t max_prompt_len, int64_t max_length, int64_t min_length,
                           const int32_t* end_ids_h, int num_end_ids, int return_end_token, float length_penalty,
                           int32_t* out_ids_h, int32_t* out_lens_h, float* out_scores_h);

/* Generator::generate_batch_async with beam_size > 1 (BeamSearch::search, src/decoding.cc:425-720; GenerationOptions beam_size,
 * patience, length_penalty, num_hypotheses): prompts of equal length; out_ids_h [batch, num_hypotheses, max_length] (-1 padded),
 * out_lens_h / out_scores_h [batch, num_hypotheses] (length -1 = fewer hypotheses than asked); batch * beam_size <= max_batch.
 * Scores: cumulative log-probability / length^length_penalty, the end token counted (decoding.h:154). */
CT2B200_API int ct2b200_generate_batch_beam(ct2b200_generator* g, const int32_t* prompt_ids_h, int64_t batch, int64_t prompt_len,
                                int64_t max_length, int64_t min_length, const int32_t* end_ids_h, int num_end_ids,
                                int return_end_token, int beam_size, float patience, float length_penalty, int num_hypotheses,
                                int32_t* out_ids_h, int32_t* out_lens_h, float* out_scores_h);

/* Generator::forward_batch_async(ids, return_log_probs) — full-sequence forward from position 0.
 * ids_h [batch, time] int32 host; logits_h [batch, time, vocab] f32 host. */
CT2B200_API int ct2b200_forward_batch(ct2b200_generator* g, const int32_t* ids_h, int64_t batch, int64_t time,
                          int return_log_probs, float* logits_h);

/* Generator::score_batch_async (src/generator.cc:27-40; models/language_model.cc:38-52, 113-133; src/scoring.cc:6-66) with
 * ScoringOptions::offset: the log-probability of every token given its prefix, from one causal prompt pass over
 * ids[:, :-1], LogSoftMax in the compute type, Gather of ids[:, 1:].
 * ids_h [batch, max_len] int32 host, right-padded with valid ids; lens_h [batch] sequence lengths (<= max_len; a row
 * shorter than 2 scores nothing); max_len - 1 <= max_length of the generator.  out_scores_h [batch, max_len - 1] f32 host:
 * row b holds the scores of tokens offset + 1 .. lens_h[b] - 1, then zeros.  Truncation (Vocabulary::to_ids) and
 * re-batching (src/batch_reader.cc) are the caller's. */
CT2B200_API int ct2b200_score_batch(ct2b200_generator* g, const int32_t* ids_h, const int32_t* lens_h, int64_t batch,
                        int64_t max_len, int64_t offset, float* out_scores_h);

/* Split phases, device-timed, for bench.py: prefill `prompt_len-1` tokens then run `steps` decode
 * steps with inputs already resident in HBM.  Returns device milliseconds of each phase. */
CT2B200_API int ct2b200_bench_decode(ct2b200_generator* g, int64_t batch, int64_t prompt_len, int64_t steps, int64_t warmup,
                         float* prefill_ms, float* decode_ms, int64_t* kernel_launches);

/* The logits of the last decode step ct2b200_bench_decode ran: logits_h [batch, vocab] f32 host, of logits_len floats
 * (an error unless logits_len == batch * vocab of the model). */
CT2B200_API int ct2b200_bench_last_logits(ct2b200_generator* g, int64_t batch, float* logits_h, int64_t logits_len);

/* Tensor parallel (ct2b200_generator_config.tp_size > 1; one process per GPU; replaces ScopedMPISetter + the NCCL
 * communicator of src/devices.cc:141-217 and ops::ReduceAll / GatherAll, src/ops/nccl_ops_gpu.cu:52-85).
 * The collectives of the decoder are fused into its kernels over NVLink peer memory, so the bootstrap only has to
 * exchange one CUDA IPC handle per rank:
 *   1. every rank opens the generator with its tp_rank / tp_size (weights are sharded on load as in
 *      src/models/model.cc:662-743: QKV and gate/up by output channel, out-proj and down-proj by input channel);
 *   2. ct2b200_generator_tp_handle writes this rank's 64-byte cudaIpcMemHandle_t to handle64_h;
 *   3. the caller all-gathers the handles (torch.distributed, MPI, files ...) and passes the tp_size handles in rank
 *      order to ct2b200_generator_tp_connect.
 * Every rank must then issue the same generate_batch / forward_batch calls with the same inputs. */
CT2B200_API int ct2b200_generator_tp_handle(ct2b200_generator* g, void* handle64_h);
CT2B200_API int ct2b200_generator_tp_connect(ct2b200_generator* g, const void* handles_h, int num_handles);

/* ---------------------------------------------------------------------------------------------
 * Encoder-decoder path (SURVEY §8 f1): ctranslate2::Translator — include/ctranslate2/translator.h:20-60,
 * TranslationOptions include/ctranslate2/translation.h:14-98; models::TransformerModel (src/models/transformer.cc),
 * EncoderDecoderReplica::run_translation (src/models/sequence_to_sequence.cc:305-420), TransformerEncoder /
 * TransformerDecoder with cross-attention (src/layers/transformer.cc), BeamSearch::search (src/decoding.cc:425-720).
 * Serves pre- and post-norm LayerNorm Transformers with absolute (sinusoidal or stored) positions; model.bin versions 2..6.
 * ct2b200_generator_config: compute_type / weight_type / device / use_cuda_graph are honoured; max_length bounds the
 * positions reserved for sinusoidal encodings (>= 500); max_batch is a hint (arenas grow on demand).
 * ------------------------------------------------------------------------------------------- */
typedef struct ct2b200_translator ct2b200_translator;
CT2B200_API ct2b200_translator* ct2b200_translator_open(const char* model_dir, const ct2b200_generator_config* config);
CT2B200_API void ct2b200_translator_close(ct2b200_translator* t);
CT2B200_API int ct2b200_translator_info(const ct2b200_translator* t, int* encoder_layers, int* decoder_layers, int* num_heads,
                            int* d_model, int* source_vocab, int* target_vocab, int64_t* weight_bytes);
/* Positions the encoder / decoder position tables hold (stored tables, or the sinusoidal encodings reserved at open). */
CT2B200_API int ct2b200_translator_positions(const ct2b200_translator* t, int64_t* encoder, int64_t* decoder);
/* Host only: the geometry parse_seq2seq_config reads from `model_dir`, as JSON. */
CT2B200_API int ct2b200_translator_summary(const char* model_dir, char* json_out, size_t capacity);

/* Translator::translate_batch on ids (Vocabulary lookups stay on the caller's side).  HOST buffers:
 *   source_ids_h [batch, max_source_len] int32 right-padded (with_source_bos / eos already applied), source_lens_h [batch];
 *   out_ids_h [batch, num_hypotheses, max_decoding_length] (-1 padded), out_lens_h / out_scores_h [batch, num_hypotheses]
 *   (length -1 = fewer hypotheses than asked).  beam_size 1 = GreedySearch (identical results to the beam-of-one search).
 *   Scores are cumulative log-probabilities / length^length_penalty (finalize_result, decoding.cc:189-254). */
CT2B200_API int ct2b200_translate_batch(ct2b200_translator* t, const int32_t* source_ids_h, const int32_t* source_lens_h,
                            int64_t batch, int64_t max_source_len, int beam_size, float patience, float length_penalty,
                            int64_t max_decoding_length, int64_t min_decoding_length, int num_hypotheses, int32_t start_id,
                            const int32_t* end_ids_h, int num_end_ids, int return_end_token, int32_t* out_ids_h,
                            int32_t* out_lens_h, float* out_scores_h);
/* ct2b200_translate_batch with the logits processors of TranslationOptions (make_logits_processors, decoding.cc:1099-1112;
 * RepetitionPenalty, NoRepeatNgram, SuppressTokens and SuppressSequences of src/decoding_utils.cc:40-177; disable_unk and
 * suppress_sequences as SequenceToSequenceReplica::translate passes them, src/models/sequence_to_sequence.cc:341-362), applied
 * on the device inside every search step, on each beam's history of chosen tokens.  The penalty rewrites the logits first;
 * every disabled entry, the end ids below min_decoding_length included, is written last.
 *   repetition_penalty > 0 and finite (1 = off); no_repeat_ngram_size >= 0 (0 = off);
 *   disable_ids_h [num_disable_ids] target ids disabled at every step (disable_unk: the unknown-token id);
 *   sequence_offsets_h [num_sequences + 1] (0 .. total) into sequence_ids_h [total]: a one-token sequence is disabled at every
 *   step, the last token of a longer one when the history ends with the others, an empty one is ignored.
 * Every id must lie inside the target vocabulary.  At most 4096 disabled ids, 4096 sequences and 65536 sequence tokens in all
 * (the reference has no limit; larger tables are refused, not truncated).  With the processors off, the results are those of
 * ct2b200_translate_batch. */
CT2B200_API int ct2b200_translate_batch_processors(ct2b200_translator* t, const int32_t* source_ids_h,
                            const int32_t* source_lens_h, int64_t batch, int64_t max_source_len, int beam_size, float patience,
                            float length_penalty, int64_t max_decoding_length, int64_t min_decoding_length, int num_hypotheses,
                            int32_t start_id, const int32_t* end_ids_h, int num_end_ids, int return_end_token,
                            float repetition_penalty, int no_repeat_ngram_size, const int32_t* disable_ids_h, int num_disable_ids,
                            const int32_t* sequence_ids_h, const int32_t* sequence_offsets_h, int num_sequences,
                            int32_t* out_ids_h, int32_t* out_lens_h, float* out_scores_h);
/* ct2b200_translate_batch_processors with the alignment attention of TranslationOptions (return_attention, replace_unknowns and
 * coverage_penalty; DecodingResult::attention of BeamSearch::search, src/decoding.cc:425-720, and finalize_result, :176-254).
 * The attention of a step is the mean over heads [0, decoder/alignment_heads) of the softmax-normalised cross-attention of
 * layer decoder/alignment_layer (src/layers/transformer.cc:518-528, 811-838); the search keeps it for every beam on the
 * device and follows the beam reordering.
 *   coverage_penalty (finite; 0 = off): at finalize each score, after the length normalisation, gains
 *   coverage_penalty * sum over the source positions with coverage > 0 of log(min(coverage, 1)), coverage = the attention
 *   summed over every row of the hypothesis, end token included (compute_coverage_penalty, decoding.cc:176-187); the
 *   hypotheses are sorted after that, and early exit is off (:457).
 *   out_attention_h (null = not returned): [batch, num_hypotheses, max_decoding_length, max_source_len] f32, one row per
 *   returned token (row t from the decoder step that produced token t; the rows of stripped end tokens go with them,
 *   sequence_to_sequence.cc:381-391), zeros past the last row and past each entry's source length; the caller trims the
 *   columns to the source (:395-412).
 * Neither one asked: the results and the device work are those of ct2b200_translate_batch_processors. */
CT2B200_API int ct2b200_translate_batch_attention(ct2b200_translator* t, const int32_t* source_ids_h,
                            const int32_t* source_lens_h, int64_t batch, int64_t max_source_len, int beam_size, float patience,
                            float length_penalty, int64_t max_decoding_length, int64_t min_decoding_length, int num_hypotheses,
                            int32_t start_id, const int32_t* end_ids_h, int num_end_ids, int return_end_token,
                            float repetition_penalty, int no_repeat_ngram_size, const int32_t* disable_ids_h, int num_disable_ids,
                            const int32_t* sequence_ids_h, const int32_t* sequence_offsets_h, int num_sequences,
                            float coverage_penalty, int32_t* out_ids_h, int32_t* out_lens_h, float* out_scores_h,
                            float* out_attention_h);
/* Host only (no device): the per-entry bookkeeping of one BeamSearch::search step (decoding.cc:595-663) — the SAME function the
 * device kernel runs (csrc/kernels/beam_decide.h).  words_h [2 * beam_size] = the candidates' tokens in TopK order.  Outputs:
 * active_h [beam] (candidate each next beam continues), hyp_slot_h / hyp_len_h [beam] (hypothesis registered for candidate k, or
 * -1), state_io_h = {num_hyp, top_done, finished} updated in place. */
CT2B200_API int ct2b200_beam_decide_host(int beam_size, const int32_t* words_h, const int32_t* end_ids_h, int num_end_ids, int step,
                             int max_steps, int max_hyp, int max_candidates, int num_hypotheses, int early_exit,
                             int include_eos, int32_t* state_io_h, int32_t* active_h, int32_t* hyp_slot_h, int32_t* hyp_len_h);

/* TransformerEncoder::operator() — memory_h [batch, max_source_len, d_model] f32 host (padded positions are unspecified). */
CT2B200_API int ct2b200_translator_encode(ct2b200_translator* t, const int32_t* source_ids_h, const int32_t* source_lens_h,
                              int64_t batch, int64_t max_source_len, float* memory_h);
/* Translator::score_batch (python/cpp/translator.cc:504-531; EncoderDecoderReplica::run_scoring,
 * src/models/sequence_to_sequence.cc:235-261; src/scoring.cc:6-66) with ScoringOptions::offset: the log-probability of every
 * target token given the source and the target prefix, from one teacher-forced decoder pass over target_ids[:, :-1] with
 * causal self-attention, LogSoftMax in the compute type, Gather of target_ids[:, 1:].
 * source_ids_h [batch, max_source_len] int32 host, right-padded; source_lens_h [batch] in [1, max_source_len] (empty sources
 * are the caller's: skip_scoring gives them zeros).  target_ids_h [batch, max_target_len] int32 host = decoder start token (if
 * the model has one), target tokens, </s>, right-padded; target_lens_h [batch] in [0, max_target_len] (a row shorter than 2
 * scores nothing); max_target_len - 1 <= the decoder's position table.  out_scores_h [batch, max_target_len - 1] f32 host: row b
 * holds the scores of target tokens offset + 1 .. target_lens_h[b] - 1, then zeros.  Vocabulary lookup, truncation
 * (Vocabulary::to_ids) and re-batching (src/batch_reader.cc) are the caller's; pairs are run in the given order, split into
 * decoder passes of bounded size inside the call. */
CT2B200_API int ct2b200_translator_score_batch(ct2b200_translator* t, const int32_t* source_ids_h, const int32_t* source_lens_h,
                                   int64_t batch, int64_t max_source_len, const int32_t* target_ids_h,
                                   const int32_t* target_lens_h, int64_t max_target_len, int64_t offset, float* out_scores_h);
/* Device-timed phases for bench.py: one encoder pass of [batch, source_len], then `steps` beam-search steps of
 * batch * beam_size rows with inputs resident in HBM. */
CT2B200_API int ct2b200_bench_translate(ct2b200_translator* t, int64_t batch, int64_t source_len, int beam_size, int64_t steps,
                            int64_t warmup, float* encode_ms, float* decode_ms, int64_t* kernel_launches);

/* ---------------------------------------------------------------------------------------------
 * Whisper (SURVEY §8 f3): ctranslate2::models::Whisper — include/ctranslate2/models/whisper.h:86-190, src/models/whisper.cc,
 * WhisperEncoder / WhisperDecoder src/layers/whisper.cc, ops::Conv1D src/ops/conv1d_gpu.cu.  A WhisperSpec directory opens
 * with ct2b200_translator_open (same handle type; the encoder is the Conv1D front-end instead of source embeddings).
 * Served: encode, and generate for prompts made of previous-text tokens, <|startoftranscript|> and the task tokens (no text
 * after them), with the timestamp rules (whisper.cc:742-860) unless the last task token is <|notimestamps|>; detect_language
 * and align (word timings) from one teacher-forced decoder pass.  Already-encoded features are not accepted as input.
 * ------------------------------------------------------------------------------------------- */
CT2B200_API int ct2b200_whisper_info(const ct2b200_translator* t, int* n_mels, int* max_frames, int* d_model, int* vocab_size);
/* Whisper::encode: features_h [batch, n_mels, frames] f32 host -> memory_h [batch, (frames + 1) / 2, d_model] f32 host. */
CT2B200_API int ct2b200_whisper_encode(ct2b200_translator* t, const float* features_h, int64_t batch, int64_t frames,
                           float* memory_h);
/* Whisper::generate(features, prompts, WhisperOptions): prompts_h [batch, prompt_len] ids; suppress_ids_h = the resolved
 * WhisperOptions::suppress_tokens (config.json "suppress_ids" for -1), suppress_begin_h = "suppress_ids_begin" when
 * suppress_blank; out_ids_h [batch, num_hypotheses, max_length] (-1 padded; the decoder runs min(max_length / 2,
 * max_length - prompt_len + 1) steps, whisper.cc:299), out_lens_h / out_scores_h [batch, num_hypotheses];
 * no_speech_h [batch] or NULL (return_no_speech_prob; needs no_speech_id). */
CT2B200_API int ct2b200_whisper_generate(ct2b200_translator* t, const float* features_h, int64_t batch, int64_t frames,
                             const int32_t* prompts_h, int64_t prompt_len, int beam_size, float patience, float length_penalty,
                             int64_t max_length, int num_hypotheses, const int32_t* suppress_ids_h, int num_suppress,
                             const int32_t* suppress_begin_h, int num_begin, int32_t sot_id, int32_t eot_id,
                             int32_t no_speech_id, int32_t no_timestamps_id, int max_initial_timestamp_index,
                             int32_t* out_ids_h, int32_t* out_lens_h, float* out_scores_h, float* no_speech_h);
/* Whisper::generate with WhisperOptions::sampling_topk / sampling_temperature (src/models/whisper.cc:296-310, the sampler
 * choice of decoding.cc:1067-1074): the arguments of ct2b200_whisper_generate, plus the sampler.  sampling_topk == 1 or
 * sampling_temperature == 0 is the search of ct2b200_whisper_generate.  Otherwise beam_size must be 1 and every entry decodes
 * num_hypotheses (<= 32) independent sampled rows (GreedySearch, decoding.cc:751-971): each step keeps the top sampling_topk
 * (0 = all) of the processed logits, divides by the temperature and draws one token (ct2b200_random_sample, seeded by
 * ct2b200_set_random_seed); a row's score is the sum of the log-probabilities of its tokens (the end token included) over
 * length^length_penalty, and the rows of an entry come back best first.  sampling_topk in [0, vocab],
 * sampling_temperature >= 0. */
CT2B200_API int ct2b200_whisper_generate_sampling(ct2b200_translator* t, const float* features_h, int64_t batch, int64_t frames,
                                                  const int32_t* prompts_h, int64_t prompt_len, int beam_size, float patience,
                                                  float length_penalty, int64_t max_length, int num_hypotheses,
                                                  const int32_t* suppress_ids_h, int num_suppress, const int32_t* suppress_begin_h,
                                                  int num_begin, int32_t sot_id, int32_t eot_id, int32_t no_speech_id,
                                                  int32_t no_timestamps_id, int max_initial_timestamp_index, int sampling_topk,
                                                  float sampling_temperature, int32_t* out_ids_h, int32_t* out_lens_h,
                                                  float* out_scores_h, float* no_speech_h);
/* Whisper::align(features, start_sequence, text_tokens, num_frames, median_filter_width) — include/ctranslate2/models/whisper.h:
 * 135-140, src/models/whisper.cc:387-582: word-level timings from the cross-attention of the alignment heads.  Every entry is
 * start + <|notimestamps|> + text + <|endoftext|>, run through the decoder in one teacher-forced pass (the memory unmasked).
 * start_ids_h [start_len]; text_ids_h [batch, max_text] right-padded, text_lens_h [batch]; num_frames_h [batch] input frames
 * per entry (halved for the encoder stride); heads_h [num_heads][2] = (decoder layer, head), config.json's alignment_heads;
 * median_filter_width odd and <= 129, or <= 1 (no filter).  Outputs:
 *   out_path_h [batch, max_text + 1 + (frames + 1) / 2, 2] (text index, time index) pairs of negative_dtw (src/dtw.cc),
 *   out_path_lens_h [batch] (0 = empty alignment: no frames for the entry);
 *   out_probs_h [batch, max_text]: SoftMax over ids [0, eot_id) at position start_len + t, gathered at text[t] (0 for an id
 *   >= eot_id), then zeros;
 *   matrix_h [batch, max_text + 1, (frames + 1) / 2] f32 or NULL: the DTW input (standardised, median-filtered, head-averaged
 *   scores of rows start_len .. start_len + text_len), zeros past each entry's rows and frames. */
CT2B200_API int ct2b200_whisper_align(ct2b200_translator* t, const float* features_h, int64_t batch, int64_t frames,
                                      const int32_t* start_ids_h, int64_t start_len, const int32_t* text_ids_h,
                                      const int32_t* text_lens_h, int64_t max_text, const int32_t* num_frames_h,
                                      int median_filter_width, const int32_t* heads_h, int num_heads, int32_t no_timestamps_id,
                                      int32_t eot_id, int32_t* out_path_h, int32_t* out_path_lens_h, float* out_probs_h,
                                      float* matrix_h);
/* Whisper::detect_language(features) — include/ctranslate2/models/whisper.h:132-133, src/models/whisper.cc:584-652: one decoder
 * position per entry on <|startoftranscript|>, SoftMax over the logits of lang_ids_h [num_langs] in the compute type.
 * probs_h [batch, num_langs] f32 in lang_ids order (sorting is the caller's). */
CT2B200_API int ct2b200_whisper_detect_language(ct2b200_translator* t, const float* features_h, int64_t batch, int64_t frames,
                                                int32_t sot_id, const int32_t* lang_ids_h, int num_langs, float* probs_h);
/* Host only (no device): negative_dtw + backtrace (src/dtw.cc), the function whisper_align runs on its matrices.
 * x_h [n, m] f32; out_path_h [n + m, 2] (row, column) pairs, out_len_h = their count. */
CT2B200_API int ct2b200_negative_dtw_host(const float* x_h, int64_t n, int64_t m, int32_t* out_path_h, int32_t* out_len_h);

/* ---------------------------------------------------------------------------------------------
 * Encoder-only models: ctranslate2::Encoder — python/cpp/encoder.cc (forward_batch), models::EncoderReplica::forward_impl
 * (src/models/language_model.cc:302-400), TransformerEncoder (src/layers/transformer.cc:405-471).  Serves
 * TransformerEncoderSpec directories (BERT, DistilBERT, RoBERTa, XLM-R class): one token table or tokens + token types merged
 * by ADD, stored position encodings, optional layernorm_embedding, pre- or post-norm LayerNorm layers with ReLU / GELU /
 * GELUTanh, optional final norm, optional pooler_dense + pooler_activation on the first position.  Every other feature the
 * spec can hold is refused at open.  ct2b200_generator_config: device / compute_type / weight_type are honoured, the rest is
 * ignored (arenas grow on demand).  fp16 / bf16 compute with head_dim 64 or 128 runs ct2b200_attention_encoder_mma.
 * ------------------------------------------------------------------------------------------- */
typedef struct ct2b200_encoder ct2b200_encoder;
CT2B200_API ct2b200_encoder* ct2b200_encoder_open(const char* model_dir, const ct2b200_generator_config* config);
CT2B200_API void ct2b200_encoder_close(ct2b200_encoder* e);
/* Host only: the geometry parse_encoder_config reads from `model_dir`, as JSON (refuses what the engine cannot run). */
CT2B200_API int ct2b200_encoder_summary(const char* model_dir, char* json_out, size_t capacity);
/* Encoder::forward_batch on ids.  HOST buffers: ids_h [batch, max_length] int32 right-padded, lengths_h [batch] in
 * [1, max_length], token_type_ids_h [batch, max_length] or NULL (zeros, the reference's placeholder); max_length <= the
 * position table.  last_hidden_state_h [batch, max_length, d_model] f32 (positions past a row's length are unspecified);
 * pooler_output_h [batch, d_model] f32 or NULL (models with a pooler). */
CT2B200_API int ct2b200_encoder_forward(ct2b200_encoder* e, const int32_t* ids_h, const int32_t* lengths_h,
                                        const int32_t* token_type_ids_h, int64_t batch, int64_t max_length,
                                        float* last_hidden_state_h, float* pooler_output_h);
/* Device-timed encoder passes on resident synthetic ids of lengths_h [batch] (<= max_length): median_ms = the median of
 * `iters` passes after `warmup` untimed ones. */
CT2B200_API int ct2b200_encoder_bench(ct2b200_encoder* e, const int32_t* lengths_h, int64_t batch, int64_t max_length,
                                      int64_t iters, int64_t warmup, float* median_ms);

#ifdef __cplusplus
}
#endif
#endif /* CT2B200_H_ */
