// translator.h — the encoder-decoder path behind ctranslate2::Translator (SURVEY §8 f1, BASELINE config 2): model loading for
// TransformerSpec directories (src/models/transformer.cc), TransformerEncoder (src/layers/transformer.cc:405-471),
// TransformerDecoder with cross-attention (:621-871, attention.cc:371-440) and BeamSearch::search (src/decoding.cc:425-720)
// resident on the device: the whole decoding step — embeddings to beam bookkeeping — is one CUDA graph, beams are
// reordered by an index remap of the K/V arena, and the host only polls a "finished entries" counter.
#pragma once

#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "beam.h"
#include "engine.h"

namespace ct2b200 {

struct Seq2SeqConfig {
  int enc_layers = 0, dec_layers = 0, num_heads = 8, head_dim = 0;
  int64_t d_model = 0, ffn_dim = 0, src_vocab = 0, tgt_vocab = 0;
  bool enc_pre_norm = true, dec_pre_norm = true;
  int enc_activation = CT2B200_ACT_RELU, dec_activation = CT2B200_ACT_RELU;
  float enc_emb_scale = 0.f, dec_emb_scale = 0.f;   // 0 = embeddings are not scaled
  float eps = 1e-5f;
  bool round_before_cast = true;                     // binary version >= 5 (model.h:87-89)
  bool has_enc_final_norm = false, has_dec_final_norm = false;
  bool start_from_zero_embedding = false;            // Marian / OPUS-MT decoders (transformer.cc:637-640)
  // the alignment attention a Translator returns (transformer.cc:518-528): the mean of the normalised cross-attention of
  // heads [0, align_heads) of decoder layer align_layer (the attributes' defaults: the last layer, one head)
  int align_layer = 0, align_heads = 1;
  bool whisper = false;                              // WhisperSpec: Conv1D front-end instead of source embeddings
  int64_t n_mels = 0, max_frames = 0;                // Whisper: input channels, encoder positions (frames / 2)
  // TransformerEncoderSpec (models::EncoderReplica, language_model.cc:302-400): the encoder alone, no decoder
  bool encoder_only = false;
  int64_t type_vocab = 0;                            // rows of the token-type embeddings merged by ADD (0 = none)
  bool has_emb_norm = false;                         // layernorm_embedding
  bool has_pooler = false;                           // pooler_dense on the first position
  int pooler_activation = CT2B200_ACT_TANH;
  int64_t weight_bytes = 0;
  std::string weights;                               // storage type of the linear layers
};

Seq2SeqConfig parse_seq2seq_config(const ModelFile& file);   // host only
Seq2SeqConfig parse_encoder_config(const ModelFile& file);   // host only; TransformerEncoderSpec directories

struct NormWeights {
  DeviceBuffer gamma, beta;
};
struct AttentionWeights {
  NormWeights norm;
  DenseWeights in;      // self-attention: fused q|k|v; cross-attention: q
  DenseWeights kv;      // cross-attention: fused k|v of the memory
  DenseWeights out;
};
struct FfnWeights {
  NormWeights norm;
  DenseWeights ff1, ff2;
};
struct EncoderLayerWeights {
  AttentionWeights self;
  FfnWeights ffn;
};
struct DecoderLayerWeights {
  AttentionWeights self, cross;
  FfnWeights ffn;
};

struct TranslationRequest {
  const int32_t* source_ids = nullptr;    // host [batch, max_source_len], right-padded
  const int32_t* source_lens = nullptr;   // host [batch]
  int64_t batch = 0, max_source_len = 0;
  int beam_size = 2;                      // TranslationOptions defaults (include/ctranslate2/translation.h)
  float patience = 1.f;
  float length_penalty = 1.f;
  int64_t max_decoding_length = 256, min_decoding_length = 1;
  int num_hypotheses = 1;
  int32_t start_id = 1;                   // decoder start token (<s>)
  std::vector<int32_t> end_ids;           // normally {</s>}
  bool return_end_token = false;
  // the logits processors (make_logits_processors, decoding.cc:1099-1112), applied on the device in every search step; the
  // defaults leave them off
  float repetition_penalty = 1.f;         // > 0 and finite
  int no_repeat_ngram_size = 0;
  std::vector<int32_t> disable_ids;       // SuppressTokens (disable_unk: the target vocabulary's unknown-token id)
  std::vector<int32_t> sequence_offsets;  // SuppressSequences: sequence s = sequence_ids[offsets[s] .. offsets[s + 1]);
  std::vector<int32_t> sequence_ids;      //   no offsets = no sequences
  // the alignment attention, kept on the device for every beam when either is asked (decoding.cc:176-254, 425-720)
  float coverage_penalty = 0.f;           // beta of the GNMT coverage term added at finalize (finite; 0 = off)
  float* attention = nullptr;             // host [batch, num_hypotheses, max_decoding_length, max_source_len] f32, or null
};
// The reference takes any number of suppressed sequences; this engine refuses more than these, never truncates.
constexpr int64_t kMaxSuppressSequences = 4096;      // sequences, and disabled ids
constexpr int64_t kMaxSuppressSequenceTokens = 65536;  // tokens of all sequences together

// models::Whisper::generate (include/ctranslate2/models/whisper.h:11-60, src/models/whisper.cc:232-390), prompts made of
// previous-text tokens, <|startoftranscript|> and the task tokens (no text after them); the timestamp rules
// (whisper.cc:742-860) apply unless the last task token is <|notimestamps|>
struct WhisperRequest {
  const float* features = nullptr;        // host [batch, n_mels, frames] f32
  int64_t batch = 0, frames = 0;
  const int32_t* prompts = nullptr;       // host [batch, prompt_len]
  int64_t prompt_len = 0;
  int beam_size = 5;
  float patience = 1.f, length_penalty = 1.f;
  int64_t max_length = 448;
  int num_hypotheses = 1;
  std::vector<int32_t> suppress_ids, suppress_ids_begin;
  int32_t sot_id = 0, eot_id = 0, no_speech_id = -1, no_timestamps_id = -1;
  int max_initial_timestamp_index = 50;
  bool return_no_speech_prob = false;
  // the sampler (decoding.cc:1067-1074): RandomSampler when sampling_topk != 1 and sampling_temperature != 0 (then beam_size 1
  // and num_hypotheses independent samples per entry), BestSampler otherwise
  int sampling_topk = 1;                  // 0 = the whole vocabulary
  float sampling_temperature = 1.f;
};
// models::Whisper::align (include/ctranslate2/models/whisper.h:135-140, src/models/whisper.cc:424-582) on ids: every entry is
// start + <|notimestamps|> + text + <|endoftext|>; heads = the (decoder layer, head) pairs of config.json's alignment_heads
struct WhisperAlignRequest {
  const float* features = nullptr;        // host [batch, n_mels, frames] f32
  int64_t batch = 0, frames = 0;
  const int32_t* start = nullptr;         // host [start_len]
  int64_t start_len = 0;
  const int32_t* text = nullptr;          // host [batch, max_text], right-padded
  const int32_t* text_lens = nullptr;     // host [batch]
  int64_t max_text = 0;
  const int32_t* num_frames = nullptr;    // host [batch]: input frames of each entry (halved here, whisper.cc:505-509)
  int median_filter_width = 7;
  std::vector<std::pair<int, int>> heads;
  int32_t no_timestamps_id = 0, eot_id = 0;
};

struct WhisperAlignResult {
  std::vector<std::pair<int64_t, int64_t>> path;   // (text index, time index)
  std::vector<float> text_token_probs;
};


class Translator {
 public:
  // encoder_only: a TransformerEncoderSpec directory (parse_encoder_config), served by encoder_forward / encoder_bench only
  Translator(const std::string& model_dir, const ct2b200_generator_config& cfg, bool encoder_only = false);
  ~Translator();
  const Seq2SeqConfig& config() const { return mc_; }
  int dtype() const { return dtype_; }
  int64_t encoder_positions() const { return enc_positions_; }
  int64_t decoder_positions() const { return dec_positions_; }

  // Translator::translate_batch on token ids
  std::vector<TranslationHypotheses> translate(const TranslationRequest& req);
  // TransformerEncoder::operator(): memory_h [batch, max_source_len, d_model] f32 host
  void encode(const int32_t* ids_h, const int32_t* lens_h, int64_t batch, int64_t max_source_len, float* memory_h);
  // WhisperEncoder::operator(): features_h [batch, n_mels, frames] f32 -> memory_h [batch, frames / 2, d_model] f32
  void whisper_encode(const float* features_h, int64_t batch, int64_t frames, float* memory_h);
  // Translator::score_batch on token ids (EncoderDecoderReplica::run_scoring, sequence_to_sequence.cc:235-261; scoring.cc:6-66):
  // sources [batch, max_source_len] right-padded (lengths >= 1), targets [batch, max_target_len] = start token .. </s>
  // right-padded; out_h [batch, max_target_len - 1] gets the log-probabilities of target tokens offset + 1 .. len - 1 of
  // each row, then zeros.  One teacher-forced pass of the decoder per group of pairs; nothing of the search state changes.
  void score(const int32_t* src_ids_h, const int32_t* src_lens_h, int64_t batch, int64_t max_source_len,
             const int32_t* tgt_ids_h, const int32_t* tgt_lens_h, int64_t max_target_len, int64_t offset, float* out_h);
  // models::Whisper::generate; no_speech_h [batch] or null
  std::vector<TranslationHypotheses> whisper_generate(const WhisperRequest& req, float* no_speech_h);
  // models::Whisper::align: one teacher-forced decoder pass per group of entries; matrix_h [batch, max_text + 1, (frames + 1)
  // / 2] (the DTW input, zeros past each entry's rows and frames) or null.  Like score, it leaves the search state alone.
  std::vector<WhisperAlignResult> whisper_align(const WhisperAlignRequest& req, float* matrix_h);
  // models::Whisper::detect_language: probs_h [batch, lang_ids.size()] = SoftMax over the logits of lang_ids at the first
  // decoder position (input <|startoftranscript|>), in lang_ids order
  void whisper_detect_language(const float* features_h, int64_t batch, int64_t frames, int32_t sot_id,
                               const std::vector<int32_t>& lang_ids, float* probs_h);
  // EncoderReplica::forward_impl (language_model.cc:349-400): ids_h / types_h (null: zeros) [batch, T] host, lens_h [batch]
  // in [1, T]; hidden_h [batch, T, d_model] f32 (positions past a row's length unspecified), pooled_h [batch, d_model] f32
  // (models with a pooler; ignored otherwise)
  void encoder_forward(const int32_t* ids_h, const int32_t* types_h, const int32_t* lens_h, int64_t batch, int64_t T,
                       float* hidden_h, float* pooled_h);
  // device-timed encoder-only passes over resident inputs of `batch` rows of lens_h[b] <= T tokens: the median of `iters`
  // passes after `warmup`
  void encoder_bench(const int32_t* lens_h, int64_t batch, int64_t T, int64_t iters, int64_t warmup, float* median_ms);
  // device-timed phases for bench.py: encoder pass, then `steps` decoding steps of batch * beam rows
  void bench(int64_t batch, int64_t source_len, int beam, int64_t steps, int64_t warmup, float* encode_ms, float* decode_ms,
             int64_t* launches);

 private:
  cudaStream_t stream() const { return gpu_.stream; }
  void load_norm(const ModelFile& f, const std::string& prefix, NormWeights& n);
  void drop_graph();            // synchronises and destroys the captured step (its buffers are about to move)
  void ensure_arena(int64_t batch, int64_t src_len, int beam, int64_t max_steps);
  void ensure_rows(int64_t entries, int64_t enc_rows, int64_t rows);
  // the Whisper front-end buffers (features, im2col columns, convolution output) for `batch` windows of S encoder positions;
  // the search state is not touched
  void ensure_whisper_frontend(int64_t batch, int64_t S);
  // Dense on T rows (quantizes them for int8 weights); `pre` = the LayerNorm applied first (fused with the quantization)
  void dense(const DenseWeights& w, const NormWeights* pre, const void* x, int64_t rows, const void* residual, int act, void* y,
             bool prequantized = false, int64_t ldy = 0);
  void set_logits_ld(BeamState& bs);
  bool post_norm(const NormWeights& n, void* x, int64_t rows, const DenseWeights* next);
  void run_encoder(int64_t batch, int64_t S);
  void run_encoder_layers(int64_t batch, int64_t S, const int32_t* lens_d);
  // the encoder-only model on src_ids_ / type_ids_ / src_lens_ -> memory_, and the pooler on its first positions -> pooled_
  void run_encoder_only(int64_t batch, int64_t S);
  // encoder positions of `frames` input frames; refuses a features shape the encoder cannot take
  int64_t whisper_positions(int64_t batch, int64_t frames) const;
  // the Whisper encoder on features_h [batch, n_mels, frames] f32 (host) -> memory_; src_lens_ = every position
  void encode_audio(const float* features_h, int64_t batch, int64_t frames);
  // memory_ [rows, d_model] -> memory_h f32 (host); synchronises
  void copy_memory_to_host(int64_t rows, float* memory_h);
  void run_search(const BeamState& bs, int64_t S, int64_t first_check);
  void project_memory(int64_t batch, int64_t S);
  // decoder embeddings of `rows` ids at positions 0 .. time - 1 (step_ptr null) or at *step_ptr (time 1) -> x_
  void embed_decoder(const int32_t* ids_d, int64_t rows, int64_t time, const int32_t* step_ptr);
  // the decoder layer stack on `rows` rows of x_; `self_attention(layer)` fills ctx_ from qkv_, and each run of
  // `rows_per_entry` rows attends to one memory entry.  Returns whether xq_ / xs_ hold Quantize(x_).
  // `capture` (one entry per layer, count 0 = none): the cross-attention also saves the scores of those heads
  // `align`: the alignment layer's cross-attention also writes the step's row of beam_'s attention history
  bool run_decoder_layers(int64_t rows, int rows_per_entry, int64_t S, const std::function<void(int)>& self_attention,
                          const std::vector<AttnCapture>* capture = nullptr, bool align = false);
  // the teacher-forced pass of score / whisper_align / whisper_detect_language: `entries` sequences of T decoder inputs ids_d
  // [entries * T] at positions 0 .. T - 1 with causal self-attention, each attending to its memory entry of S positions.
  // Returns whether xq_ / xs_ hold Quantize(x_).
  bool decode_teacher_forced(int64_t entries, int64_t T, int64_t S, const int32_t* ids_d,
                             const std::vector<AttnCapture>* capture = nullptr);
  // final norm + projection of n rows of x_ (rows_d [n]; null: the first n rows, at most one slab, with xq = what
  // decode_teacher_forced returned) in slabs of score_slab_rows_ into score_logits_; reduce(logits, first, count, ld) runs on
  // each slab's rows [first, first + count)
  void project_rows(const int32_t* rows_d, int64_t n, bool xq,
                    const std::function<void(const void*, int64_t, int64_t, int64_t)>& reduce);
  // the score slab, allocated on first use; returns the row stride of its logits
  int64_t ensure_score_slab();
  // copies `ids` into score_ids_ (grown as needed); `ids` must stay alive until the copy is done
  const int32_t* stage_ids(const std::vector<int32_t>& ids);
  // align: keep the step's alignment attention (a search with bs.hyp_anc set)
  void decoder_step(int64_t rows, int beam, int64_t batch, int64_t S, bool align = false);
  // one decoding step, captured as the graph of `key` (everything the capture bakes in) unless use_graph_ is off
  void launch_or_capture_step(const BeamState& bs, int64_t S, const std::vector<int64_t>& key);

  std::mutex mu_;                // translate / score / encode / bench are serialised per translator
  Seq2SeqConfig mc_;
  int dtype_ = CT2B200_F32;
  bool use_graph_ = true;

  DenseWeights enc_emb_, dec_emb_, projection_;
  DenseWeights type_emb_, pooler_;   // encoder-only models: token-type embeddings, pooler_dense
  NormWeights emb_norm_;             // encoder-only models: layernorm_embedding
  DeviceBuffer type_ids_, first_, pooled_;   // token types [rows]; first positions / pooler output [entries, d_model]
  int64_t cap_types_ = 0, cap_pooled_ = 0;
  DenseWeights conv1_, conv2_;   // Whisper: [d, n_mels * 3] / [d, d * 3] in T (+ bias)
  DeviceBuffer enc_pos_, dec_pos_;
  int64_t enc_positions_ = 0, dec_positions_ = 0;
  NormWeights enc_norm_, dec_norm_;
  std::vector<EncoderLayerWeights> enc_;
  std::vector<DecoderLayerWeights> dec_;

  // arena (grown on demand)
  int64_t cap_batch_ = 0, cap_src_ = 0, cap_steps_ = 0;          // search state
  int64_t cap_entries_ = 0, cap_enc_rows_ = 0, cap_rows_ = 0;     // encoder entries / rows, activation rows
  int cap_beam_ = 0;
  DeviceBuffer src_ids_, src_lens_, x_, xn_, xq_, xs_, qkv_, ctx_, h_, q_, memory_;
  std::vector<DeviceBuffer> mem_kv_, self_k_, self_v_;
  DeviceBuffer logits_;
  int64_t logits_ld_ = 0;                 // row stride of logits_ for the current search (set_logits_ld)
  BeamSearchArena beam_;         // search state: next ids, scores, histories, ancestry, hypotheses, counters
  DeviceBuffer features_, cols_, conv_out_, suppress_d_, forced_d_, no_speech_d_;   // Whisper
  int64_t cap_frames_ = 0;
  int64_t cap_fe_batch_ = 0, cap_fe_src_ = 0;                    // Whisper front-end buffers
  std::vector<int32_t> audio_lens_h_;    // source of encode_audio's src_lens_ copy, alive until the call synchronises
  int32_t* host_pinned_ = nullptr;
  size_t host_pinned_elems_ = 0;
  // score: logits slab [score_slab_rows_, vocab (padded)], per pass: decoder input ids | scored rows | their target ids, scores
  DeviceBuffer score_logits_, score_ids_, score_out_;
  int64_t score_slab_rows_ = 0;
  // whisper_align: captured scores [entries, heads, T, S], standardised DTW rows [entries, heads, text + 1, S], DTW matrix
  DeviceBuffer align_scores_, align_norm_, align_matrix_, align_masks_;

  StepGraph graph_;
  // last: it is destroyed first, so the stream is synchronised before any buffer above is freed
  EngineDevice gpu_;
};

}  // namespace ct2b200
