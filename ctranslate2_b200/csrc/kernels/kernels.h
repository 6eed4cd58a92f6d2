// kernels.h — host-callable launchers of every CUDA kernel in csrc/kernels (one stream, no allocation
// except the lazily created split-K scratch, no synchronisation).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "../common.cuh"
#include "gemm_common.cuh"

namespace ct2b200 {

// rowwise.cu
void launch_quantize_rows(const void* x, int dtype, int64_t rows, int64_t cols, bool round, int8_t* q,
                          float* scale, cudaStream_t st);
void launch_rms_norm(const void* gamma, const void* x, int64_t rows, int64_t cols, float eps, bool use_residual,
                     void* y, int8_t* q, float* scale, int dtype, cudaStream_t st);
void launch_mul_quantize(const void* a, const void* b, int64_t rows, int64_t cols, int8_t* q, float* scale,
                         int dtype, cudaStream_t st);
void launch_dequantize_rows(const int8_t* x, const float* scale, int64_t rows, int64_t cols, void* y, int dtype,
                            cudaStream_t st, bool reciprocal = false);
void launch_dequantize_gemm_output(const int32_t* c, const DenseEpilogue& e, int64_t m, int64_t n, int dtype,
                                   cudaStream_t st);
void launch_embedding_s8(const int8_t* w, const float* scale, const int32_t* ids, int64_t num_ids, int64_t depth,
                         void* y, int dtype, cudaStream_t st);
void launch_gather_rows(const void* data, const int32_t* ids, int64_t num_ids, int64_t row_bytes, void* out,
                        cudaStream_t st);
void launch_rotary(const void* x, const void* sin, const void* cos, int64_t batch, int64_t time, int64_t depth,
                   int64_t ndims, bool interleave, void* y, int dtype, cudaStream_t st);
void launch_softmax(const void* x, const int32_t* lengths, int64_t rows, int64_t cols, bool log, void* y,
                    int dtype, cudaStream_t st);
// LogSoftMax + Gather fused: y [rows] f32 = T(x[r, ids[r]] - logsumexp(x[r, :])) (NaN for an id outside [0, cols)); row r
// starts at x + r * ld (ld = 0: cols)
void launch_log_softmax_gather(const void* x, const int32_t* ids, int64_t rows, int64_t cols, float* y, int dtype,
                               cudaStream_t st, int64_t ld = 0);
// SoftMax over the first `cols` elements of a row + Gather, the same row reduction: y [rows] f32 = T(exp(x[r, ids[r]] -
// logsumexp(x[r, :cols]))), 0 for an id outside [0, cols) (a masked softmax leaves 0 there); row r starts at x + r * ld
void launch_softmax_gather(const void* x, const int32_t* ids, int64_t rows, int64_t cols, int64_t ld, float* y, int dtype,
                           cudaStream_t st);
void launch_topk(const void* x, int64_t rows, int64_t cols, int k, void* values, int32_t* indices, int dtype,
                 cudaStream_t st);

// tp_rows.cu — tensor-parallel row kernels (collectives fused into their consumers over NVLink peer memory)
struct TpLink {
  int rank = 0, world = 1;
  const uint32_t* tick = nullptr;             // forward-pass counter of this rank (device)
  uint32_t* flags_local = nullptr;            // [2][8] epoch flags in this rank's exchange buffer (peers write them)
  uint32_t* flags_peer[8] = {};               // the same array inside every peer's buffer
  const void* parts[2][8] = {};               // partial buffer b ([rows, d_model] T) of rank r
  unsigned long long* amax_local = nullptr;   // [2][8][amax_rows] {epoch, amax} words in this rank's buffer
  unsigned long long* amax_peer[8] = {};
  int64_t amax_rows = 0;
};
void launch_tp_tick(uint32_t* tick, cudaStream_t st);
void launch_tp_reduce_norm_quantize(const TpLink& tp, int buf, int sync_idx, void* x, const void* gamma, int64_t rows,
                                    int64_t cols, float eps, int8_t* q, float* scale, int dtype, cudaStream_t st);
void launch_tp_reduce_norm(const TpLink& tp, int buf, int sync_idx, void* x, const void* gamma, int64_t rows, int64_t cols,
                           float eps, void* y, int dtype, cudaStream_t st);
void launch_tp_reduce(const TpLink& tp, int buf, int sync_idx, void* x, int64_t rows, int64_t cols, int dtype,
                      cudaStream_t st);
void launch_tp_quantize_rows(const TpLink& tp, int slot, int sync_idx, const void* x, int64_t rows, int64_t cols, int8_t* q,
                             float* scale, int dtype, cudaStream_t st);

// gemm_tc.cu (wgmma) — gemm_s8_mma.cu declarations live in gemm_common.cuh
void gemm_s8_tc(const int8_t* A, const int8_t* B, int64_t M, int64_t N, int64_t K, const DenseEpilogue& epi,
                int dtype, cudaStream_t st);
void gemm_s8_glu_tc(const int8_t* A, const int8_t* Bgate, const int8_t* Bup, int64_t M, int64_t N, int64_t K,
                    const GluEpilogue& glu, int dtype, cudaStream_t st);
void gemm_f16_tc(const void* A, const void* B, const void* bias, const void* residual, int act, int64_t M,
                 int64_t N, int64_t K, void* C, int dtype, cudaStream_t st);

// gemm_decode.cu (wgmma, m <= 64): false = shape not covered, use the general kernel
bool gemm_s8_decode(const int8_t* A, const int8_t* B, int64_t M, int64_t N, int64_t K, const DenseEpilogue& epi,
                    int dtype, cudaStream_t st);
bool gemm_s8_glu_decode(const int8_t* A, const int8_t* Bgate, const int8_t* Bup, int64_t M, int64_t N, int64_t K,
                        const GluEpilogue& glu, int dtype, cudaStream_t st);
bool gemm_f16_decode(const void* A, const void* B, const void* bias, const void* residual, int act, int64_t M,
                     int64_t N, int64_t K, void* C, int dtype, cudaStream_t st);

// gemm_prefill.cu (wgmma, m > 64, compute bound): false = shape not covered
bool gemm_s8_prefill(const int8_t* A, const int8_t* B, int64_t M, int64_t N, int64_t K, const DenseEpilogue& epi,
                     int dtype, cudaStream_t st);
bool gemm_s8_glu_prefill(const int8_t* A, const int8_t* Bgate, const int8_t* Bup, int64_t M, int64_t N, int64_t K,
                         const GluEpilogue& glu, int dtype, cudaStream_t st);
bool gemm_f16_prefill(const void* A, const void* B, const void* bias, const void* residual, int act, int64_t M,
                      int64_t N, int64_t K, void* C, int dtype, cudaStream_t st);

// dispatch by ct2b200_gemm_impl
void gemm_s8(const int8_t* A, const int8_t* B, int64_t M, int64_t N, int64_t K, const DenseEpilogue& epi,
             int dtype, int impl, cudaStream_t st);
void gemm_s8_glu(const int8_t* A, const int8_t* Bgate, const int8_t* Bup, int64_t M, int64_t N, int64_t K,
                 const GluEpilogue& glu, int dtype, int impl, cudaStream_t st);
void gemm_float(const void* A, const void* B, const void* bias, const void* residual, int act, int64_t M, int64_t N,
                int64_t K, void* C, int dtype, cudaStream_t st);

// awq.cu — AWQ-INT4 in the native (repacked, K-major) layout
struct AwqNative {
  const void* wp = nullptr;   // int32 [n, k/8]
  const void* sc = nullptr;   // f16 [n, k/group]
  const void* zr = nullptr;   // f16 [n, k/group]
  int64_t n = 0, k = 0;
  int group = 128;
  const void* sz = nullptr;   // optional: half2 {scale, zero} [k/group, n] (group-major: coalesced per-row fetches)
};
// {scale, zero} pairs of a repacked weight in group-major order (built once at load; awq_decode.cu reads it)
void awq_build_group_major(const AwqNative& w, void* sz_out /* half2 [k/group, n] */, cudaStream_t st);
// awq_decode.cu — lean decode kernel (m <= 64); false = shape not covered
bool dense_awq_decode(const void* x, const AwqNative& w, const void* bias, const void* residual, int act, int64_t m, void* y,
                      cudaStream_t st);
bool dense_awq_glu_decode(const void* x, const AwqNative& wg, const AwqNative& wu, int act, int64_t m, void* h,
                          cudaStream_t st);
// awq_gemv.cu — CUDA-core kernel for m <= 4 (no tensor cores, no barriers); false = not enabled / shape not covered
bool dense_awq_gemv(const void* x, const AwqNative& w, const void* bias, const void* residual, int act, int64_t m, void* y,
                    cudaStream_t st);
bool dense_awq_glu_gemv(const void* x, const AwqNative& wg, const AwqNative& wu, int act, int64_t m, void* h, cudaStream_t st);
void awq_repack(const int32_t* qweight, const void* scales, const int32_t* qzeros, int layout, int group, int64_t n,
                int64_t k, int32_t* wp, void* sc, void* zr, cudaStream_t st);
void awq_dequantize_ref_layout(const int32_t* qweight, const void* scales, const int32_t* qzeros, int layout, int group,
                               int64_t n, int64_t k, void* w_out, cudaStream_t st);
void awq_dequantize_native(const AwqNative& w, void* w_out, cudaStream_t st);
void dense_awq(const void* x, const AwqNative& w, const void* bias, const void* residual, int act, int64_t m, void* y,
               void* scratch_nk_f16, cudaStream_t st);
void dense_awq_glu(const void* x, const AwqNative& wg, const AwqNative& wu, int act, int64_t m, void* h,
                   void* scratch_nk_f16, void* scratch_mn_f16, cudaStream_t st);
void launch_mul_inplace_f16(void* a_inout, const void* b, int64_t n, cudaStream_t st);

// attention.cu
int attention_decode_splits(int64_t batch, int Hkv, int64_t max_len, int sm_count);
size_t attention_decode_workspace_bytes(int64_t batch, int H, int D, int splits);
void launch_attention_decode(const void* qkv, void* kc, void* vc, const float* sn, const float* cs,
                             const int32_t* lens, int64_t batch, int H, int Hkv, int D, int64_t max_len,
                             bool interleave, float scale, void* out, void* workspace, size_t workspace_bytes,
                             int splits, int dtype, cudaStream_t st);
void launch_rope_append(void* qkv, void* kc, void* vc, const float* sn, const float* cs, const int32_t* lengths,
                        int64_t batch, int64_t time, int64_t offset, int H, int Hkv, int D, int64_t max_len,
                        bool interleave, int dtype, cudaStream_t st);
void launch_attention_prefill_simple(const void* qkv, const void* kc, const void* vc, const int32_t* lengths,
                                     int64_t batch, int64_t time, int64_t offset, int H, int Hkv, int D,
                                     int64_t max_len, float scale, void* out, int dtype, cudaStream_t st);

// attention_mma.cu — tensor-core prefill attention (fp16/bf16, head_dim 64/128); false = shape not covered
bool launch_attention_prefill_mma(const void* qkv, const void* kc, const void* vc, int64_t batch, int64_t time,
                                  int64_t offset, int H, int Hkv, int D, int64_t max_len, float scale, void* out,
                                  int dtype, cudaStream_t st);
// encoder self-attention of launch_attention_encoder on tensor cores (fp16 / bf16, head_dim 64 or 128); false = not covered
bool launch_attention_encoder_mma(const void* qkv, const int32_t* lengths, int64_t batch, int S, int H, int D, float scale,
                                  void* out, int dtype, cudaStream_t st);
// attention_decode.cu — persistent work-balanced decode attention; false = shape not covered
bool launch_attention_decode_persistent(const void* qkv, void* kc, void* vc, const float* sn, const float* cs,
                                        const int32_t* lens, int64_t batch, int H, int Hkv, int D, int64_t max_len,
                                        bool interleave, float scale, void* out, float* partials, int32_t* tickets,
                                        int slots, int dtype, cudaStream_t st);
bool launch_attention_decode_mma(const void* qkv, void* kc, void* vc, const float* sn, const float* cs,
                                 const int32_t* lens, int64_t batch, int H, int Hkv, int D, int64_t max_len,
                                 bool interleave, float scale, void* out, float* partials, int32_t* tickets, int splits,
                                 int dtype, cudaStream_t st);
// picks the tensor-core kernel when it covers the shape (CT2B200_ATTN_PREFILL=simple forces the generic one)
void launch_attention_prefill(const void* qkv, const void* kc, const void* vc, const int32_t* lengths, int64_t batch,
                              int64_t time, int64_t offset, int H, int Hkv, int D, int64_t max_len, float scale,
                              void* out, int dtype, cudaStream_t st);

// decode_loop.cu
int sample_greedy_chunks(int64_t vocab);
void launch_sample_greedy(const void* logits, int64_t batch, int64_t vocab, const int32_t* gen, const int32_t* end_ids,
                          const int32_t* forced, int32_t* next_ids, int32_t* out_ids, int32_t* lens, float* part_v,
                          int32_t* part_i, int32_t* tickets, float* part_s, float* step_scores,
                          const int32_t* row_start, int32_t* attn_lens, int32_t* finished, int dtype, cudaStream_t st);
void launch_convert_to_f32(const void* x, int64_t n, float* y, int dtype, cudaStream_t st);
void launch_convert_from_f32(const float* x, int64_t n, void* y, int dtype, cudaStream_t st);
void launch_fill_i32(int32_t* p, int64_t n, int32_t v, cudaStream_t st);
void launch_mul_inplace(void* a_inout, const void* b, int64_t n, int dtype, cudaStream_t st);

// seq2seq.cu — encoder-decoder path (Translator): embeddings + positions, LayerNorm, head_dim-agnostic attention, beam search
void launch_embed_pos(const void* w, const float* w_scale, const int32_t* ids, int64_t rows, int64_t depth, float emb_scale,
                      const void* pos, int64_t time, const int32_t* step_ptr, bool zero_first, void* y, int dtype,
                      cudaStream_t st, const void* w2 = nullptr, const float* w2_scale = nullptr,
                      const int32_t* ids2 = nullptr);
void launch_layer_norm(const void* x, const void* gamma, const void* beta, int64_t rows, int64_t cols, float eps, void* y,
                       int8_t* q, float* scale, bool round, int dtype, cudaStream_t st);
void launch_attention_encoder(const void* qkv, const int32_t* lengths, int64_t batch, int S, int H, int D, float scale,
                              void* out, int dtype, cudaStream_t st);
void launch_attention_beam_self(const void* qkv, void* k_cache, void* v_cache, const int32_t* anc, const int32_t* step_ptr,
                                int64_t rows, int max_len, int H, int D, float scale, void* out, int dtype, cudaStream_t st);
void launch_attention_cross(const void* q, const void* kv, const int32_t* lengths, int64_t rows, int beam, int S, int H, int D,
                            float scale, void* out, int dtype, cudaStream_t st);
// The same cross-attention, also saving the pre-softmax scores T(scale * q.k) of selected heads (the attention a decoder
// returns with return_normalized_attention() == false, attention.cc:267-270): row n = (entry n / beam, position n % beam);
// masks [H] (device): bit k of masks[h] = head h goes to slot first + k of out [entries, total, beam, S] f32 (a head listed
// twice is written twice).
struct AttnCapture {
  float* out = nullptr;
  const uint32_t* masks = nullptr;
  int first = 0, total = 0;
};
void launch_attention_cross_capture(const void* q, const void* kv, const int32_t* lengths, int64_t rows, int beam, int S, int H,
                                    int D, float scale, void* out, const AttnCapture& cap, int dtype, cudaStream_t st);
// The same cross-attention, also writing the normalised probabilities of heads [0, heads) (what a Translator decoder returns,
// return_normalized_attention() == true) to probs [rows, heads, S] f32; keys past a row's entry length are not written.
void launch_attention_cross_align(const void* q, const void* kv, const int32_t* lengths, int64_t rows, int beam, int S, int H,
                                  int D, float scale, void* out, float* probs, int heads, int dtype, cudaStream_t st);
// the alignment attention of one decoding step (TransformerDecoder::decode, transformer.cc:811-838, averaged heads): row n of
// the history hist [rows, stride, S] f32 at position *step_ptr = T(the mean of probs [n, 0 .. heads, s]), summed in head
// order; exact zeros past the length of entry n / beam
void launch_align_mean(const float* probs, const int32_t* lengths, const int32_t* step_ptr, int64_t rows, int beam, int S,
                       int heads, int stride, float* hist, int dtype, cudaStream_t st);
// causal self-attention of `time` teacher-forced decoder positions per sequence: qkv [batch * time, 3d] (row b * time + t
// attends to rows b * time + j, j <= t), out [batch * time, d]; no cache is written
void launch_attention_causal(const void* qkv, int64_t batch, int time, int H, int D, float scale, void* out, int dtype,
                             cudaStream_t st);
// device state of BeamSearch::search (decoding.cc:425-720); N = batch * beam rows, `stride` = allocated steps per row
struct BeamState {
  int batch = 0, beam = 1, vocab = 0, stride = 0, max_steps = 0, max_hyp = 0, max_candidates = 1, num_hypotheses = 1;
  int64_t vocab_ld = 0;             // row stride of the logits (>= vocab; a multiple of 8 lets the kernels use 16-byte accesses)
  int early_exit = 0, num_end = 0, min_length = 0;
  int start_step = 0;               // absolute position of the first search step (prompt positions come before)
  int include_eos = 1;              // DecodingOptions::include_eos_in_hypotheses
  int num_disable = 0, num_begin = 0;
  const int32_t* disable_ids = nullptr;     // SuppressTokens: disabled at every step
  const int32_t* disable_begin = nullptr;   // SuppressTokensBegin: disabled at the first search step
  // The history-dependent logits processors (src/decoding_utils.cc:40-150), on each row's token history; zero = off.
  float rep_penalty = 0.f;          // RepetitionPenalty: x < 0 ? x * p : x / p on every token of the history, once each
  int no_repeat_ngram = 0;          // NoRepeatNgram: n-gram size
  int num_sequences = 0;            // SuppressSequences: sequence s = seq_ids[seq_offsets[s] .. seq_offsets[s + 1]) (non-empty)
  const int32_t* seq_ids = nullptr;
  const int32_t* seq_offsets = nullptr;   // [num_sequences + 1]
  // Whisper's ApplyTimestampRules (src/models/whisper.cc:742-860); ts_begin = 0 disables them
  int ts_begin = 0, ts_end = 0, ts_eot = 0, ts_no_timestamps = 0, ts_max_initial = 0;
  const int32_t* end_ids = nullptr;
  int32_t* step = nullptr;          // [1] current step, advanced by the update kernel
  int32_t* ticket = nullptr;        // [1]
  int32_t* num_finished = nullptr;  // [1] entries whose result is final (the host polls it)
  int32_t* finished = nullptr;      // [batch]
  int32_t* top_done = nullptr;      // [batch]
  int32_t* num_hyp = nullptr;       // [batch]
  int32_t* alive = nullptr;         // [2][N, stride] token history of the live beams (double-buffered by step parity)
  int32_t* anc = nullptr;           // [2][N, stride] cache slot holding position t of the row's history
  int32_t* next_ids = nullptr;      // [N] input ids of the next step
  int32_t* parent = nullptr;        // [N] or null: the row each next beam continues (gather index of Decoder::update_state)
  int32_t* hyp_tokens = nullptr;    // [batch, max_hyp, stride]
  int32_t* hyp_len = nullptr;       // [batch, max_hyp]
  float* hyp_score = nullptr;       // [batch, max_hyp] cumulative log-probability (not normalised)
  // [batch, max_hyp, stride] or null: the cache slot that computed each absolute position of a hypothesis, filled when it is
  // registered (its attention row t is then row hyp_anc[t] of the history at position t)
  int32_t* hyp_anc = nullptr;
  // Sampled search (GreedySearch with a RandomSampler, decoding.cc:751-971): sample_topk >= 0 selects it.  The `beam` rows of an
  // entry are its num_hypotheses independent samples; ancestry stays the identity and hypothesis slot h belongs to row h.
  int sample_topk = -1;             // 0 = the whole vocabulary
  float sample_temperature = 1.f;
  const uint32_t* rng = nullptr;    // [2] process seed, index of this sampling call (philox.h)
  int32_t* sample_ids = nullptr;    // [N] the step's sampled ids
  float* sample_logp = nullptr;     // [N] their log-probabilities
  float* row_score = nullptr;       // [N] cumulative log-probability of the row
  int32_t* row_done = nullptr;      // [N] the row's hypothesis is registered
};
void launch_beam_init(void* cum, int32_t* ids, int64_t rows, int beam, int start_id, int dtype, cudaStream_t st);
void launch_beam_logprobs(void* logits, const void* cum, const BeamState& s, int dtype, cudaStream_t st);
// beam <= 8: scores + the top 2 * beam of every ROW in one launch (row_scores T / row_ids int32 [batch * beam, 2 * beam], ids
// flattened over [beam, vocab]); launch_beam_update(per_row = true) merges the rows of an entry
void launch_beam_rows(void* logits, const void* cum, const BeamState& s, void* row_scores, int32_t* row_ids, int dtype,
                      cudaStream_t st);
// one prompt position without a search step: next ids = forced_next [rows], identity ancestry, step + 1
void launch_beam_force(const BeamState& s, const int32_t* forced_next, cudaStream_t st);
// sampled search step (s.sample_topk >= 0): beam_mask_row + RandomSampler::sample on every row of logits (modified in place)
// -> s.sample_ids / s.sample_logp, then the update: histories, row scores, hypothesis h of a row that ends, step + 1
void launch_beam_sample(void* logits, const BeamState& s, int dtype, cudaStream_t st);
void launch_beam_sample_update(const BeamState& s, cudaStream_t st);
// compute_coverage_penalty (decoding.cc:176-187) without its factor, for every registered hypothesis (s.hyp_anc set) over the
// attention history hist [N, s.stride, S]: out [batch, max_hyp] f32 (slots past num_hyp untouched)
void launch_hyp_coverage(const BeamState& s, const float* hist, int S, float* out, cudaStream_t st);
// out [batch, num, max_len, S] f32 = the attention rows of hypothesis slot sel[b * num + k] (device, -1 = none) of entry b,
// zeros past its length
void launch_hyp_attention_gather(const BeamState& s, const float* hist, int S, const int32_t* sel, int num, int max_len,
                                 float* out, cudaStream_t st);
// RandomSampler::sample on rows x [rows, ld] T of `vocab` logits: ids [rows], logp [rows] = T(LogSoftMax(x))[id]; the
// uniform of row r is philox_uniform(seed, call, r, step) (philox.h)
void launch_random_sample(const void* x, int64_t rows, int64_t vocab, int64_t ld, int k, float temperature, uint32_t seed,
                          uint32_t call, uint32_t step, int32_t* ids, float* logp, int dtype, cudaStream_t st);
// out[r] = softmax(logits[r * row_stride : +vocab])[token]
void launch_token_prob(const void* logits, int64_t rows, int64_t vocab, int64_t row_stride, int token, float* out, int dtype,
                       cudaStream_t st);
// whisper_align.cu — models::Whisper::align post-processing (whisper.cc:387-560) and detect_language (:584-652).
// scores [B, H, T, S] f32 (the captured T(scale * q.k)); nf [B] frames per entry (> 0 softmaxes), len [B] input lengths.
// 1. SoftMax of every row t < len[b] over its first nf[b] frames, in place, rounded to T.
void launch_align_softmax(float* scores, const int32_t* nf, const int32_t* len, int64_t batch, int heads, int64_t T, int64_t S,
                          int dtype, cudaStream_t st);
// 2. ops::LayerNorm(-2, 0) of every frame column over `rows` token rows (rows <= 0: len[b]; rows past len[b] - 1 read row
//    len[b] - 1, the padding the reference's Padder adds back), written for the DTW rows start .. start + ntext[b] to
//    norm [B, H, max_text + 1, F] f32 (T-rounded).
void launch_align_standardize(const float* scores, const int32_t* nf, const int32_t* len, const int32_t* ntext, int64_t batch,
                              int heads, int64_t T, int64_t S, int64_t rows, int64_t start, int64_t max_text, int64_t F,
                              float* norm, int dtype, cudaStream_t st);
// 3. ops::MedianFilter(width) along frames (mirrored edges; pass-through for width <= 1 or nf[b] <= width / 2), then
//    ops::Mean over the heads: matrix [B, max_text + 1, F] f32 (T-rounded; zeros past nf[b] and past ntext[b] + 1 rows).
void launch_align_median_mean(const float* norm, const int32_t* nf, const int32_t* ntext, int64_t batch, int heads,
                              int64_t max_text, int64_t F, int width, float* matrix, int dtype, cudaStream_t st);
// SoftMax over the logits of `n` ids (Gather then SoftMax, in T): probs [rows, n] f32 from rows of x at stride ld.
void launch_gather_softmax(const void* x, int64_t rows, int64_t ld, const int32_t* ids, int n, float* probs, int dtype,
                           cudaStream_t st);
// ops::Conv1D as im2col (+ the float Dense): cols [batch * Tout, Cin * K] T from x [batch, Cin, Tin] (channel_major) or [batch, Tin, Cin]
void launch_im2col(const void* x, bool x_is_f32, int64_t batch, int64_t Cin, int64_t Tin, int64_t Tout, int K, int stride,
                   int padding, bool channel_major, void* cols, int dtype, cudaStream_t st);
void launch_add_positions(void* x, const void* pos, int64_t rows, int64_t time, int64_t depth, int dtype, cudaStream_t st);
void launch_beam_update(const BeamState& s, const void* cand_scores, const int32_t* cand_ids, void* cum, bool per_row, int dtype,
                        cudaStream_t st);
// Decoder::update_state / replicate_state for the contiguous per-row caches of the decoder-only engine (decoder.cc:33-139):
// dst[row] = src[parent[row]] (parent == null: src[row / beam]) for positions [0, positions) of every kv head;
// caches [rows, Hkv, max_len, D] T
void launch_kv_gather(const void* src_k, const void* src_v, void* dst_k, void* dst_v, const int32_t* parent, int beam, int64_t rows,
                      int Hkv, int64_t max_len, int D, int64_t positions, int dtype, cudaStream_t st);
// float32 Dense (true fp32 FMAs): c [m,n] = a [m,k] . b [n,k]^T with bias / activation / residual
void gemm_f32(const float* A, const float* B, const float* bias, const float* residual, int act, int64_t M, int64_t N,
              int64_t K, float* C, cudaStream_t st);

}  // namespace ct2b200
