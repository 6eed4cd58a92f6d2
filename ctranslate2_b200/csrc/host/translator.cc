// translator.cc — see translator.h.  Reference counterparts: src/models/transformer.cc, src/models/sequence_to_sequence.cc
// (EncoderDecoderReplica::run_translation), src/layers/transformer.cc (TransformerEncoder / TransformerDecoder),
// src/layers/attention.cc, src/layers/common.cc (Embeddings, position encoders, LayerNorm, Dense), src/decoding.cc (BeamSearch).
#include "translator.h"

#include <cuda_profiler_api.h>

#include "dtw.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <numeric>

namespace ct2b200 {

// =============================================================================================
// configuration
// =============================================================================================
namespace {

const HostVariable* find_any(const ModelFile& f, std::initializer_list<std::string> names) {
  for (const auto& n : names)
    if (const HostVariable* v = f.find(n)) return v;
  return nullptr;
}

std::string embeddings_scope(const ModelFile& f, const std::string& scope) {
  if (f.find(scope + "/embeddings_0/weight")) {
    if (f.find(scope + "/embeddings_1/weight"))
      throw std::invalid_argument("models with several input features (embeddings_1) are not supported");
    return scope + "/embeddings_0";
  }
  return scope + "/embeddings";
}

// build_embeddings_scale (transformer.cc:380-402): the attribute is a flag or the scale itself
float embeddings_scale(const ModelFile& f, const std::string& scope, int64_t depth) {
  const HostVariable* s = find_any(f, {scope + "/scale_embeddings", scope + "/embeddings/multiply_by_sqrt_depth"});
  if (!s || (s->type_id == 1 && s->scalar() != 0.0)) return std::sqrt(static_cast<float>(depth));
  if (s->type_id != 1 && s->scalar() != 1.0) return static_cast<float>(s->scalar());
  return 0.f;
}

double scoped_attribute(const ModelFile& f, const std::string& scope, const std::string& name, double fallback) {
  // spec revisions < 5 keep the attribute at the top level (models/transformer.cc:67-79)
  const HostVariable* v = find_any(f, {scope + "/" + name, name});
  return v ? v->scalar() : fallback;
}

}  // namespace

Seq2SeqConfig parse_seq2seq_config(const ModelFile& f) {
  Seq2SeqConfig mc;
  if (!f.find("encoder/layer_0/self_attention/linear_0/weight") || !f.find("decoder/layer_0/attention/linear_0/weight"))
    throw std::invalid_argument("ct2b200 Translator serves encoder-decoder Transformer models (TransformerSpec, WhisperSpec); got " +
                                f.spec_name);
  while (f.find("encoder/layer_" + std::to_string(mc.enc_layers) + "/self_attention/linear_0/weight")) ++mc.enc_layers;
  while (f.find("decoder/layer_" + std::to_string(mc.dec_layers) + "/self_attention/linear_0/weight")) ++mc.dec_layers;
  const HostVariable& temb = f.get("decoder/embeddings/weight");
  mc.tgt_vocab = temb.shape[0];
  mc.d_model = temb.shape[1];
  mc.whisper = f.find("encoder/conv1/weight") != nullptr;
  if (mc.whisper) {
    // WhisperEncoder (layers/whisper.cc:8-23): Conv1D(k 3, stride 1, pad 1) + GELU, Conv1D(k 3, stride 2, pad 1) + GELU,
    // stored positions, pre-norm GELU layers
    const HostVariable& c1 = f.get("encoder/conv1/weight");
    const HostVariable& c2 = f.get("encoder/conv2/weight");
    CT2_REQUIRE(c1.shape.size() == 3 && c1.shape[2] == 3 && c2.shape.size() == 3 && c2.shape[2] == 3, "Whisper convolutions must have kernel size 3");
    CT2_REQUIRE(c1.shape[0] == mc.d_model && c2.shape[0] == mc.d_model && c2.shape[1] == mc.d_model, "unexpected convolution shapes");
    mc.n_mels = c1.shape[1];
    mc.max_frames = f.get("encoder/position_encodings/encodings").shape[0];
    CT2_REQUIRE(f.find("decoder/position_encodings/encodings") != nullptr, "Whisper decoders store their position encodings");
  } else {
    const HostVariable& semb = f.get(embeddings_scope(f, "encoder") + "/weight");
    mc.src_vocab = semb.shape[0];
    CT2_REQUIRE(semb.shape[1] == mc.d_model, "encoder and decoder depths differ");
  }
  // num_heads: attribute since revision 3; TransformerBase / TransformerBig imply 8 / 16 before (models/transformer.cc:62-65)
  mc.num_heads = static_cast<int>(scoped_attribute(f, "encoder", "num_heads", f.spec_name == "TransformerBig" ? 16 : 8));
  CT2_REQUIRE(static_cast<int>(scoped_attribute(f, "decoder", "num_heads", mc.num_heads)) == mc.num_heads,
              "encoder and decoder head counts differ");
  CT2_REQUIRE(mc.d_model % mc.num_heads == 0, "d_model must be divisible by num_heads");
  mc.head_dim = static_cast<int>(mc.d_model / mc.num_heads);
  mc.enc_pre_norm = scoped_attribute(f, "encoder", "pre_norm", 1.0) != 0.0;
  mc.dec_pre_norm = scoped_attribute(f, "decoder", "pre_norm", 1.0) != 0.0;
  mc.enc_activation = static_cast<int>(scoped_attribute(f, "encoder", "activation", 0.0));
  mc.dec_activation = static_cast<int>(scoped_attribute(f, "decoder", "activation", 0.0));
  if (mc.whisper) {
    mc.enc_pre_norm = true;
    mc.enc_activation = CT2B200_ACT_GELU;
  }
  mc.enc_emb_scale = mc.whisper ? 0.f : embeddings_scale(f, "encoder", mc.d_model);
  mc.dec_emb_scale = embeddings_scale(f, "decoder", mc.d_model);
  mc.ffn_dim = f.get("encoder/layer_0/ffn/linear_0/weight").shape[0];
  mc.round_before_cast = f.binary_version >= 5;
  mc.has_enc_final_norm = f.find("encoder/layer_norm/gamma") != nullptr;
  mc.has_dec_final_norm = f.find("decoder/layer_norm/gamma") != nullptr;
  const bool has_beta = f.find("encoder/layer_0/self_attention/layer_norm/beta") != nullptr;
  mc.eps = static_cast<float>(f.config_number("layer_norm_epsilon", has_beta ? 1e-5 : 1e-6));
  // what TransformerSpec can express and this engine does not compute: refuse instead of translating something else
  auto absent = [&](const std::string& name, const char* what) {
    if (f.find(name)) throw std::invalid_argument(std::string(what) + " (" + name + ") is not supported by the Translator engine");
  };
  CT2_REQUIRE(has_beta, "RMSNorm encoder-decoder models are not supported (LayerNorm with beta is)");
  for (const char* scope : {"encoder", "decoder"}) {
    const std::string s(scope);
    absent(s + "/layernorm_embedding/gamma", "layernorm_embedding");
    absent(s + "/layer_0/self_attention/relative_position_keys", "relative position representations");
    absent(s + "/layer_0/self_attention/relative_attention_bias", "relative attention bias");
    absent(s + "/layer_0/self_attention/rotary_dim", "rotary embeddings");
    absent(s + "/layer_0/self_attention/num_heads_kv", "grouped-query attention");
    absent(s + "/layer_0/ffn/linear_0_noact/weight", "gated feed-forward layers");
    absent(s + "/project_in/weight", "project_in");
    absent(s + "/project_out/weight", "project_out");
    if (scoped_attribute(f, s, "alibi", 0.0) != 0.0) throw std::invalid_argument("ALiBi is not supported by the Translator engine");
    if (scoped_attribute(f, s, "embeddings_merge", 0.0) != 0.0)
      throw std::invalid_argument("embeddings_merge other than CONCAT of one feature is not supported");
  }
  mc.start_from_zero_embedding = f.attribute("decoder/start_from_zero_embedding", 0.0) != 0.0;
  if (!mc.whisper) {
    // TransformerDecoder (transformer.cc:518-528): a negative layer counts from the end, 0 heads = every head
    int layer = static_cast<int>(scoped_attribute(f, "decoder", "alignment_layer", -1.0));
    int heads = static_cast<int>(scoped_attribute(f, "decoder", "alignment_heads", 1.0));
    if (layer < 0) layer += mc.dec_layers;
    if (heads == 0) heads = mc.num_heads;
    CT2_REQUIRE(layer >= 0 && layer < mc.dec_layers, "decoder/alignment_layer is outside the decoder's layers");
    CT2_REQUIRE(heads >= 1 && heads <= mc.num_heads, "decoder/alignment_heads must be in [0, num_heads]");
    mc.align_layer = layer;
    mc.align_heads = heads;
  }
  absent("decoder/scale_outputs", "scaled outputs");
  absent("decoder/layer_0/layer_scalar", "layer_scalar");
  absent("decoder/layer_0/self_attention/queries_scale", "a custom queries_scale");
  if (f.attribute("decoder/final_logit_softcapping", 0.0) != 0.0)
    throw std::invalid_argument("final logit soft-capping is not supported by the Translator engine");
  CT2_REQUIRE(f.revision != 1, "spec revision 1 (OpenNMT-tf variable names) is not supported");
  const HostVariable& w = f.get("encoder/layer_0/self_attention/linear_0/weight");
  mc.weights = w.type_id == 1 ? "int8" : w.type_id == 2 ? "int16" : w.type_id == 4 ? "float16" : w.type_id == 5 ? "bfloat16" : "float32";
  CT2_REQUIRE(w.type_id != 2, "int16 models are not supported (convert with int8 or a float type)");
  return mc;
}

// TransformerEncoderModelSpec (python/ctranslate2/specs/transformer_spec.py:771-812) read as TransformerEncoder
// (transformer.cc:405-471) + EncoderReplica's pooler (language_model.cc:335-345)
Seq2SeqConfig parse_encoder_config(const ModelFile& f) {
  Seq2SeqConfig mc;
  mc.encoder_only = true;
  if (f.spec_name != "TransformerEncoderSpec" || !f.find("encoder/layer_0/self_attention/linear_0/weight"))
    throw std::invalid_argument("ct2b200 Encoder serves Transformer encoder models (TransformerEncoderSpec); got " + f.spec_name);
  while (f.find("encoder/layer_" + std::to_string(mc.enc_layers) + "/self_attention/linear_0/weight")) ++mc.enc_layers;
  auto absent = [&](const std::string& name, const char* what) {
    if (f.find(name)) throw std::invalid_argument(std::string(what) + " (" + name + ") is not supported by the Encoder engine");
  };
  // ParallelEmbeddings (common.cc:84-148): one table, or the tokens and their types merged by ADD
  const bool parallel = f.find("encoder/embeddings_0/weight") != nullptr;
  const HostVariable& emb = f.get(parallel ? "encoder/embeddings_0/weight" : "encoder/embeddings/weight");
  mc.src_vocab = emb.shape[0];
  mc.d_model = emb.shape[1];
  if (parallel) {
    absent("encoder/embeddings_2/weight", "more than two input features");
    if (const HostVariable* types = f.find("encoder/embeddings_1/weight")) {
      if (f.attribute("encoder/embeddings_merge", 0.0) != 1.0)
        throw std::invalid_argument("embeddings_merge CONCAT is not supported by the Encoder engine (ADD is)");
      CT2_REQUIRE(types->shape.size() == 2 && types->shape[1] == mc.d_model, "token-type embeddings must have the model depth");
      mc.type_vocab = types->shape[0];
    }
  }
  mc.num_heads = static_cast<int>(f.attribute("encoder/num_heads", 8.0));
  CT2_REQUIRE(mc.num_heads > 0 && mc.d_model % mc.num_heads == 0, "d_model must be divisible by num_heads");
  mc.head_dim = static_cast<int>(mc.d_model / mc.num_heads);
  mc.enc_pre_norm = f.attribute("encoder/pre_norm", 1.0) != 0.0;
  mc.enc_activation = static_cast<int>(f.attribute("encoder/activation", 0.0));
  if (mc.enc_activation != CT2B200_ACT_RELU && mc.enc_activation != CT2B200_ACT_GELU && mc.enc_activation != CT2B200_ACT_GELU_TANH)
    throw std::invalid_argument("the Encoder engine runs ReLU, GELU and GELUTanh feed-forward layers; got activation " +
                                std::to_string(mc.enc_activation));
  mc.enc_emb_scale = embeddings_scale(f, "encoder", mc.d_model);
  mc.ffn_dim = f.get("encoder/layer_0/ffn/linear_0/weight").shape[0];
  mc.round_before_cast = f.binary_version >= 5;
  mc.has_enc_final_norm = f.find("encoder/layer_norm/gamma") != nullptr;
  mc.has_emb_norm = f.find("encoder/layernorm_embedding/gamma") != nullptr;
  mc.has_pooler = f.find("pooler_dense/weight") != nullptr;
  mc.pooler_activation = static_cast<int>(f.attribute("pooler_activation", static_cast<double>(CT2B200_ACT_TANH)));
  CT2_REQUIRE(mc.pooler_activation >= CT2B200_ACT_RELU && mc.pooler_activation <= CT2B200_ACT_SIGMOID, "unknown pooler_activation");
  const bool has_beta = f.find("encoder/layer_0/self_attention/layer_norm/beta") != nullptr;
  mc.eps = static_cast<float>(f.config_number("layer_norm_epsilon", has_beta ? 1e-5 : 1e-6));
  CT2_REQUIRE(has_beta, "RMSNorm encoder models are not supported (LayerNorm with beta is)");
  CT2_REQUIRE(f.find("encoder/position_encodings/encodings") != nullptr,
              "the Encoder engine needs stored position encodings (encoder/position_encodings/encodings)");
  const std::string a = "encoder/layer_0/self_attention/";
  absent(a + "relative_position_keys", "relative position representations");
  absent(a + "relative_asymmetric_position_keys", "relative position representations");
  absent(a + "relative_attention_bias", "relative attention bias");
  absent(a + "rotary_dim", "rotary embeddings");
  absent(a + "num_heads_kv", "grouped-query or multi-query attention");   // multi_query_attention stores num_heads_kv = 1
  absent(a + "head_dim", "a head_dim other than d_model / num_heads");
  absent(a + "sliding_window", "sliding-window attention");
  absent(a + "q_norm/gamma", "query / key normalisation");
  absent(a + "queries_scale", "a custom queries_scale");
  absent("encoder/sliding_window", "sliding-window attention");
  absent("encoder/layer_0/ffn/linear_0_noact/weight", "gated feed-forward layers");
  absent("encoder/layer_0/input_layer_norm/gamma", "pre-and-post layer norms");
  const HostVariable& w = f.get("encoder/layer_0/self_attention/linear_0/weight");
  mc.weights = w.type_id == 1 ? "int8" : w.type_id == 2 ? "int16" : w.type_id == 4 ? "float16" : w.type_id == 5 ? "bfloat16" : "float32";
  CT2_REQUIRE(w.type_id != 2, "int16 models are not supported (convert with int8 or a float type)");
  return mc;
}

// =============================================================================================
// loading
// =============================================================================================
void Translator::load_norm(const ModelFile& f, const std::string& prefix, NormWeights& n) {
  upload_as(n.gamma, f.get(prefix + "/gamma"), dtype_);
  upload_as(n.beta, f.get(prefix + "/beta"), dtype_);
}

namespace {
// generate_sinusoidal_position_encoding (common.cc:204-229): positions start at 1, [sin | cos] halves, fp32 then cast
std::vector<float> sinusoidal_positions(int64_t max_time, int64_t depth) {
  const float inc = std::log(10000.f) / static_cast<float>(depth / 2 - 1);
  std::vector<float> ts(depth / 2);
  for (int64_t i = 0; i < depth / 2; ++i) ts[i] = std::exp(-inc * static_cast<float>(i));
  std::vector<float> e(max_time * depth);
  for (int64_t t = 0; t < max_time; ++t)
    for (int64_t j = 0; j < depth / 2; ++j) {
      const float a = static_cast<float>(t + 1) * ts[j];
      e[t * depth + j] = std::sin(a);
      e[t * depth + depth / 2 + j] = std::cos(a);
    }
  return e;
}
}  // namespace

Translator::Translator(const std::string& model_dir, const ct2b200_generator_config& cfg, bool encoder_only)
    : gpu_(cfg.device) {
  dtype_ = cfg.compute_type;
  use_graph_ = cfg.use_cuda_graph != 0;
  CT2_REQUIRE(cfg.tp_size <= 1, "the Translator engine does not run tensor parallel");

  ModelFile f(model_dir);
  mc_ = encoder_only ? parse_encoder_config(f) : parse_seq2seq_config(f);
  // no AWQ arm here: AWQ weights are refused as an unsupported weight type
  const DenseLoad opt{dtype_, cfg.weight_type, stream()};
  auto load = [&](const std::string& prefix, DenseWeights& w) {
    mc_.weight_bytes += load_dense(f, prefix, opt, w);
    CT2_REQUIRE(w.kind != DenseWeights::INT8 || w.k % 16 == 0, "int8 Dense layers need an input size that is a multiple of 16");
  };
  if (mc_.encoder_only) {
    load(f.find("encoder/embeddings_0/weight") ? "encoder/embeddings_0" : "encoder/embeddings", enc_emb_);
    if (mc_.type_vocab) load("encoder/embeddings_1", type_emb_);
    if (mc_.has_emb_norm) load_norm(f, "encoder/layernorm_embedding", emb_norm_);
    if (mc_.has_pooler) load("pooler_dense", pooler_);
  } else if (mc_.whisper) {
    // the convolutions run as im2col + float Dense: weights [d, Cin, 3] flattened to [d, Cin * 3] in T (the reference keeps
    // them in float on CUDA too, model.cc:204-223; an int8-stored convolution is dequantized here: w = q / scale)
    auto load_conv = [&](const std::string& prefix, DenseWeights& w) {
      const HostVariable& wt = f.get(prefix + "/weight");
      HostVariable flat = wt;
      std::vector<float> deq;
      if (wt.type_id == 1) {
        const HostVariable& sc = f.get(prefix + "/weight_scale");
        CT2_REQUIRE(sc.type_id == 0 && (sc.size() == wt.shape[0] || sc.size() == 1), "unexpected convolution weight_scale");
        deq.resize(wt.size());
        const int64_t per = wt.size() / wt.shape[0];
        for (int64_t i = 0; i < wt.size(); ++i) {
          float scale;
          std::memcpy(&scale, sc.data + 4 * (sc.size() == 1 ? 0 : i / per), 4);
          deq[i] = static_cast<float>(reinterpret_cast<const int8_t*>(wt.data)[i]) / scale;
        }
        flat.type_id = 0;
        flat.data = reinterpret_cast<const uint8_t*>(deq.data());
        flat.nbytes = deq.size() * 4;
      }
      mc_.weight_bytes += upload_as(w.weight, flat, dtype_);
      w.kind = DenseWeights::FLOAT16;
      w.n = wt.shape[0];
      w.k = wt.shape[1] * wt.shape[2];
      if (const HostVariable* b = f.find(prefix + "/bias")) upload_as(w.bias, *b, dtype_);
    };
    CT2_REQUIRE(dtype_ == CT2B200_F32 || (mc_.n_mels * 3) % 8 == 0, "n_mels * 3 must be a multiple of 8 for float16 / bfloat16");
    load_conv("encoder/conv1", conv1_);
    load_conv("encoder/conv2", conv2_);
  } else {
    load(embeddings_scope(f, "encoder"), enc_emb_);
  }
  if (!mc_.encoder_only) {
    load("decoder/embeddings", dec_emb_);
    load("decoder/projection", projection_);
  }
  if (mc_.has_enc_final_norm) load_norm(f, "encoder/layer_norm", enc_norm_);
  if (mc_.has_dec_final_norm) load_norm(f, "decoder/layer_norm", dec_norm_);
  enc_.resize(mc_.enc_layers);
  for (int l = 0; l < mc_.enc_layers; ++l) {
    const std::string p = "encoder/layer_" + std::to_string(l) + "/";
    load_norm(f, p + "self_attention/layer_norm", enc_[l].self.norm);
    load(p + "self_attention/linear_0", enc_[l].self.in);
    load(p + "self_attention/linear_1", enc_[l].self.out);
    load_norm(f, p + "ffn/layer_norm", enc_[l].ffn.norm);
    load(p + "ffn/linear_0", enc_[l].ffn.ff1);
    load(p + "ffn/linear_1", enc_[l].ffn.ff2);
  }
  dec_.resize(mc_.dec_layers);
  for (int l = 0; l < mc_.dec_layers; ++l) {
    const std::string p = "decoder/layer_" + std::to_string(l) + "/";
    load_norm(f, p + "self_attention/layer_norm", dec_[l].self.norm);
    load(p + "self_attention/linear_0", dec_[l].self.in);
    load(p + "self_attention/linear_1", dec_[l].self.out);
    load_norm(f, p + "attention/layer_norm", dec_[l].cross.norm);
    load(p + "attention/linear_0", dec_[l].cross.in);
    load(p + "attention/linear_1", dec_[l].cross.kv);
    load(p + "attention/linear_2", dec_[l].cross.out);
    load_norm(f, p + "ffn/layer_norm", dec_[l].ffn.norm);
    load(p + "ffn/linear_0", dec_[l].ffn.ff1);
    load(p + "ffn/linear_1", dec_[l].ffn.ff2);
  }
  // position encodings: stored table (PositionEmbedding) or sinusoidal (SinusoidalPositionEncoder, 500 positions or more)
  auto load_positions = [&](const std::string& scope, DeviceBuffer& dst) -> int64_t {
    if (const HostVariable* e = f.find(scope + "/position_encodings/encodings")) {
      upload_as(dst, *e, dtype_);
      return e->shape[0];
    }
    const int64_t count = std::max<int64_t>(500, cfg.max_length);
    const std::vector<float> enc = sinusoidal_positions(count, mc_.d_model);
    HostVariable v;
    v.shape = {count, mc_.d_model};
    v.type_id = 0;
    v.data = reinterpret_cast<const uint8_t*>(enc.data());
    v.nbytes = enc.size() * 4;
    upload_as(dst, v, dtype_);
    return count;
  };
  enc_positions_ = load_positions("encoder", enc_pos_);
  if (!mc_.encoder_only) dec_positions_ = load_positions("decoder", dec_pos_);
  CT2_CUDA_CHECK(cudaDeviceSynchronize());
}

Translator::~Translator() {
  if (host_pinned_) cudaFreeHost(host_pinned_);
}

void Translator::drop_graph() {
  CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));
  graph_.reset();
}

// The search's state (beam arena, self-attention K/V, logits, Whisper front-end, host staging) is sized by batch x beam x
// steps; the encoder and activation buffers it shares with the scoring passes grow through ensure_rows.
void Translator::ensure_arena(int64_t batch, int64_t src_len, int beam, int64_t max_steps) {
  CT2_REQUIRE(src_len <= enc_positions_ && max_steps <= dec_positions_,
              "No position encodings are defined for positions this far (common.cc:157-161)");
  const size_t es = dtype_size(dtype_);
  if (batch > cap_batch_ || src_len > cap_src_ || beam > cap_beam_ || max_steps > cap_steps_) {
    drop_graph();
    cap_batch_ = std::max(cap_batch_, batch);
    cap_src_ = std::max(cap_src_, src_len);
    cap_beam_ = std::max(cap_beam_, beam);
    cap_steps_ = std::max(cap_steps_, max_steps);
    beam_.ensure(cap_batch_, cap_beam_, cap_steps_, es);          // same capacities: its stride is the K/V stride
    const int64_t B = cap_batch_, S = cap_src_, L = cap_steps_, N = B * cap_beam_;
    const int64_t d = mc_.d_model, V = mc_.tgt_vocab;
    self_k_.resize(mc_.dec_layers);
    self_v_.resize(mc_.dec_layers);
    for (int l = 0; l < mc_.dec_layers; ++l) {
      self_k_[l].alloc(N * L * d * es);
      self_v_[l].alloc(N * L * d * es);
    }
    logits_.alloc(N * ((V + 7) / 8 * 8) * es);
    if (mc_.whisper) ensure_whisper_frontend(B, S);
    const size_t need = static_cast<size_t>(B) * S + B + 64 + static_cast<size_t>(N) * 16 + 8192;
    if (need > host_pinned_elems_) {
      if (host_pinned_) cudaFreeHost(host_pinned_);
      CT2_CUDA_CHECK(cudaMallocHost(&host_pinned_, need * sizeof(int32_t)));
      host_pinned_elems_ = need;
    }
  }
  ensure_rows(cap_batch_, cap_batch_ * cap_src_, std::max(cap_batch_ * cap_src_, cap_batch_ * cap_beam_));
}

void Translator::ensure_whisper_frontend(int64_t batch, int64_t S) {
  if (batch <= cap_fe_batch_ && S <= cap_fe_src_) return;
  cap_fe_batch_ = std::max(cap_fe_batch_, batch);
  cap_fe_src_ = std::max(cap_fe_src_, S);
  const size_t es = dtype_size(dtype_);
  const int64_t B = cap_fe_batch_, frames = 2 * cap_fe_src_, d = mc_.d_model;   // conv2 halves the frames
  features_.alloc(B * mc_.n_mels * frames * 4);
  cols_.alloc(std::max(B * frames * mc_.n_mels * 3, B * cap_fe_src_ * d * 3) * es);
  conv_out_.alloc(B * frames * d * es);
}

// Encoder entries (source lengths), encoder rows (source ids, memory, memory keys / values: entries x padded source length)
// and activation rows (x_ .. h_: encoder rows, or decoder rows of a search step or of a scoring pass).
void Translator::ensure_rows(int64_t entries, int64_t enc_rows, int64_t rows) {
  if (entries <= cap_entries_ && enc_rows <= cap_enc_rows_ && rows <= cap_rows_) return;
  drop_graph();
  cap_entries_ = std::max(cap_entries_, entries);
  cap_enc_rows_ = std::max(cap_enc_rows_, enc_rows);
  cap_rows_ = std::max(cap_rows_, rows);
  const size_t es = dtype_size(dtype_);
  const int64_t E = cap_enc_rows_, R = cap_rows_, d = mc_.d_model, F = mc_.ffn_dim;
  src_ids_.alloc(E * 4);
  src_lens_.alloc(cap_entries_ * 4);
  x_.alloc(R * d * es);
  xn_.alloc(R * d * es);
  xq_.alloc(R * std::max(d, F));
  xs_.alloc(R * 4);
  qkv_.alloc(R * 3 * d * es);
  ctx_.alloc(R * d * es);
  h_.alloc(R * F * es);
  q_.alloc(R * d * es);
  memory_.alloc(E * d * es);
  mem_kv_.resize(mc_.dec_layers);
  for (int l = 0; l < mc_.dec_layers; ++l) mem_kv_[l].alloc(E * 2 * d * es);
}

// =============================================================================================
// layers
// =============================================================================================
void Translator::dense(const DenseWeights& w, const NormWeights* pre, const void* x, int64_t rows, const void* residual,
                       int act, void* y, bool prequantized, int64_t ldy) {
  const void* src = x;
  if (w.kind == DenseWeights::INT8) {
    if (prequantized)
      ;                                            // the post-norm kernel before this call left Quantize(x) in xq_ / xs_
    else if (pre)
      launch_layer_norm(x, pre->gamma.ptr, pre->beta.ptr, rows, w.k, mc_.eps, nullptr, xq_.as<int8_t>(), xs_.as<float>(),
                        mc_.round_before_cast, dtype_, stream());
    else
      launch_quantize_rows(x, dtype_, rows, w.k, mc_.round_before_cast, xq_.as<int8_t>(), xs_.as<float>(), stream());
  } else if (pre) {
    launch_layer_norm(x, pre->gamma.ptr, pre->beta.ptr, rows, w.k, mc_.eps, xn_.ptr, nullptr, nullptr, true, dtype_, stream());
    src = xn_.ptr;
  }
  dense_forward(w, xq_.as<int8_t>(), xs_.as<float>(), src, rows, residual, act, y, ldy, dtype_, CT2B200_GEMM_AUTO, nullptr,
                stream());
}

// Row stride of the logits for a search: INT8 projections write rows padded to a multiple of 8 elements (16-byte stores in the
// GEMM epilogue and 16-byte loads in the scoring kernel whatever the vocabulary size, e.g. 58101); the beam > 8 path runs
// ops::TopK over the flattened [beam * vocab] scores and needs them contiguous.
void Translator::set_logits_ld(BeamState& bs) {
  const int64_t V = mc_.tgt_vocab;
  logits_ld_ = (projection_.kind == DenseWeights::INT8 && bs.beam <= 8) ? (V + 7) / 8 * 8 : V;
  bs.vocab_ld = logits_ld_;
}

// Post-norm sublayer end (transformer.cc:35-38, attention.cc:603-606): x = LayerNorm(x).  When the consumer is an INT8 Dense
// the same launch also leaves its Quantize (of the rounded output, as the reference's separate op reads it) in xq_ / xs_;
// returns whether it did, for the `prequantized` argument of that Dense.
bool Translator::post_norm(const NormWeights& n, void* x, int64_t rows, const DenseWeights* next) {
  const bool q = next && next->kind == DenseWeights::INT8 && next->k == mc_.d_model;
  launch_layer_norm(x, n.gamma.ptr, n.beta.ptr, rows, mc_.d_model, mc_.eps, x, q ? xq_.as<int8_t>() : nullptr,
                    q ? xs_.as<float>() : nullptr, q ? mc_.round_before_cast : true, dtype_, stream());
  return q;
}

// TransformerEncoder::operator() (transformer.cc:427-471); rows = batch * S, padded positions are computed and ignored
void Translator::run_encoder(int64_t batch, int64_t S) {
  launch_embed_pos(enc_emb_.weight.ptr, enc_emb_.kind == DenseWeights::INT8 ? enc_emb_.scale.as<float>() : nullptr,
                   src_ids_.as<int32_t>(), batch * S, mc_.d_model, mc_.enc_emb_scale, enc_pos_.ptr, S, nullptr, false, x_.ptr,
                   dtype_, stream());
  run_encoder_layers(batch, S, src_lens_.as<int32_t>());
}

// the layer stack on x_ -> memory_ (lens_d = null: every position is valid)
void Translator::run_encoder_layers(int64_t batch, int64_t S, const int32_t* lens_d) {
  const int64_t rows = batch * S, d = mc_.d_model;
  const float scale = 1.f / std::sqrt(static_cast<float>(mc_.head_dim));
  const bool pre = mc_.enc_pre_norm;
  bool xq = false;                                 // xq_ / xs_ already hold Quantize(x_) (left by a post-norm launch)
  for (int l = 0; l < mc_.enc_layers; ++l) {
    EncoderLayerWeights& w = enc_[l];
    dense(w.self.in, pre ? &w.self.norm : nullptr, x_.ptr, rows, nullptr, -1, qkv_.ptr, xq);
    // encoder-only models run the tensor-core kernel where it covers the shape; the Translator and Whisper encoders keep
    // the generic one
    if (!mc_.encoder_only || !launch_attention_encoder_mma(qkv_.ptr, lens_d, batch, static_cast<int>(S), mc_.num_heads,
                                                           mc_.head_dim, scale, ctx_.ptr, dtype_, stream()))
      launch_attention_encoder(qkv_.ptr, lens_d, batch, static_cast<int>(S), mc_.num_heads, mc_.head_dim, scale, ctx_.ptr, dtype_,
                               stream());
    dense(w.self.out, nullptr, ctx_.ptr, rows, x_.ptr, -1, x_.ptr);
    xq = !pre && post_norm(w.self.norm, x_.ptr, rows, &w.ffn.ff1);
    dense(w.ffn.ff1, pre ? &w.ffn.norm : nullptr, x_.ptr, rows, nullptr, mc_.enc_activation, h_.ptr, xq);
    dense(w.ffn.ff2, nullptr, h_.ptr, rows, x_.ptr, -1, x_.ptr);
    xq = !pre && post_norm(w.ffn.norm, x_.ptr, rows, l + 1 < mc_.enc_layers ? &enc_[l + 1].self.in : nullptr);
  }
  if (mc_.has_enc_final_norm)
    launch_layer_norm(x_.ptr, enc_norm_.gamma.ptr, enc_norm_.beta.ptr, rows, d, mc_.eps, memory_.ptr, nullptr, nullptr, true, dtype_,
                      stream());
  else
    CT2_CUDA_CHECK(cudaMemcpyAsync(memory_.ptr, x_.ptr, rows * d * dtype_size(dtype_), cudaMemcpyDeviceToDevice, stream()));
}

// the memory keys / values of every decoder layer, once per batch (cached_attn_keys / values, attention.cc:385-428)
void Translator::project_memory(int64_t batch, int64_t S) {
  for (int l = 0; l < mc_.dec_layers; ++l)
    dense(dec_[l].cross.kv, nullptr, memory_.ptr, batch * S, nullptr, -1, mem_kv_[l].ptr);
}

// TransformerDecoder::decode's layer loop (transformer.cc:621-871), shared by the one-token step and the teacher-forced pass:
// only the self-attention differs.  Cross-attention: row n reads memory entry n / rows_per_entry.
bool Translator::run_decoder_layers(int64_t rows, int rows_per_entry, int64_t S, const std::function<void(int)>& self_attention,
                                    const std::vector<AttnCapture>* capture, bool align) {
  const float scale = 1.f / std::sqrt(static_cast<float>(mc_.head_dim));
  const bool pre = mc_.dec_pre_norm;
  bool xq = false;                                 // xq_ / xs_ already hold Quantize(x_) (left by a post-norm launch)
  for (int l = 0; l < mc_.dec_layers; ++l) {
    DecoderLayerWeights& w = dec_[l];
    dense(w.self.in, pre ? &w.self.norm : nullptr, x_.ptr, rows, nullptr, -1, qkv_.ptr, xq);
    self_attention(l);
    dense(w.self.out, nullptr, ctx_.ptr, rows, x_.ptr, -1, x_.ptr);
    xq = !pre && post_norm(w.self.norm, x_.ptr, rows, &w.cross.in);
    dense(w.cross.in, pre ? &w.cross.norm : nullptr, x_.ptr, rows, nullptr, -1, q_.ptr, xq);
    if (align && l == mc_.align_layer) {
      launch_attention_cross_align(q_.ptr, mem_kv_[l].ptr, src_lens_.as<int32_t>(), rows, rows_per_entry, static_cast<int>(S),
                                   mc_.num_heads, mc_.head_dim, scale, ctx_.ptr, beam_.attn_probs.as<float>(), mc_.align_heads,
                                   dtype_, stream());
      launch_align_mean(beam_.attn_probs.as<float>(), src_lens_.as<int32_t>(), beam_.counters.as<int32_t>(), rows, rows_per_entry,
                        static_cast<int>(S), mc_.align_heads, static_cast<int>(beam_.cap_steps), beam_.attn_hist.as<float>(),
                        dtype_, stream());
    } else if (capture && (*capture)[l].masks)
      launch_attention_cross_capture(q_.ptr, mem_kv_[l].ptr, src_lens_.as<int32_t>(), rows, rows_per_entry, static_cast<int>(S),
                                     mc_.num_heads, mc_.head_dim, scale, ctx_.ptr, (*capture)[l], dtype_, stream());
    else
      launch_attention_cross(q_.ptr, mem_kv_[l].ptr, src_lens_.as<int32_t>(), rows, rows_per_entry, static_cast<int>(S),
                             mc_.num_heads, mc_.head_dim, scale, ctx_.ptr, dtype_, stream());
    dense(w.cross.out, nullptr, ctx_.ptr, rows, x_.ptr, -1, x_.ptr);
    xq = !pre && post_norm(w.cross.norm, x_.ptr, rows, &w.ffn.ff1);
    dense(w.ffn.ff1, pre ? &w.ffn.norm : nullptr, x_.ptr, rows, nullptr, mc_.dec_activation, h_.ptr, xq);
    dense(w.ffn.ff2, nullptr, h_.ptr, rows, x_.ptr, -1, x_.ptr);
    xq = !pre && post_norm(w.ffn.norm, x_.ptr, rows,
                           l + 1 < mc_.dec_layers ? &dec_[l + 1].self.in : (mc_.has_dec_final_norm ? nullptr : &projection_));
  }
  return xq;
}

// with start_from_zero_embedding position 0 of every sequence is zeroed (transformer.cc:637-640)
void Translator::embed_decoder(const int32_t* ids_d, int64_t rows, int64_t time, const int32_t* step_ptr) {
  launch_embed_pos(dec_emb_.weight.ptr, dec_emb_.kind == DenseWeights::INT8 ? dec_emb_.scale.as<float>() : nullptr, ids_d, rows,
                   mc_.d_model, mc_.dec_emb_scale, dec_pos_.ptr, time, step_ptr, mc_.start_from_zero_embedding, x_.ptr, dtype_,
                   stream());
}

// TransformerDecoder::decode for one target position of every beam row (transformer.cc:621-871)
void Translator::decoder_step(int64_t rows, int beam, int64_t batch, int64_t S, bool align) {
  (void)batch;
  const float scale = 1.f / std::sqrt(static_cast<float>(mc_.head_dim));
  const int32_t* step_ptr = beam_.counters.as<int32_t>();
  embed_decoder(beam_.next_ids.as<int32_t>(), rows, 1, step_ptr);
  const bool xq = run_decoder_layers(rows, beam, S, [&](int l) {
    launch_attention_beam_self(qkv_.ptr, self_k_[l].ptr, self_v_[l].ptr, beam_.anc.as<int32_t>(), step_ptr, rows,
                               static_cast<int>(cap_steps_), mc_.num_heads, mc_.head_dim, scale, ctx_.ptr, dtype_, stream());
  }, nullptr, align);
  dense(projection_, mc_.has_dec_final_norm ? &dec_norm_ : nullptr, x_.ptr, rows, nullptr, -1, logits_.ptr, xq, logits_ld_);
}

void Translator::launch_or_capture_step(const BeamState& bs, int64_t S, const std::vector<int64_t>& key) {
  const int64_t rows = static_cast<int64_t>(bs.batch) * bs.beam;
  auto step = [&] {
    decoder_step(rows, bs.beam, bs.batch, S, bs.hyp_anc != nullptr);
    if (bs.sample_topk >= 0)
      beam_.sample_step(logits_.ptr, bs, dtype_, stream());
    else
      beam_.step(logits_.ptr, bs, dtype_, stream());
  };
  if (!use_graph_) {
    step();
    return;
  }
  graph_.capture(stream(), key, step);
  graph_.launch(stream());
}

// =============================================================================================
// the search (shared by translate_batch and Whisper::generate)
// =============================================================================================
// the decoding loop: one captured step per position; the host only polls the "finished entries" counter
void Translator::run_search(const BeamState& bs, int64_t S, int64_t first_check) {
  // everything the captured step bakes in (kernel arguments are values)
  uint32_t temperature_bits, penalty_bits;
  std::memcpy(&temperature_bits, &bs.sample_temperature, 4);
  std::memcpy(&penalty_bits, &bs.rep_penalty, 4);
  std::vector<int64_t> key = {bs.batch, bs.beam, S, bs.vocab_ld, bs.stride, bs.max_steps, bs.min_length, bs.max_hyp, bs.max_candidates,
                              bs.num_hypotheses, bs.early_exit, bs.num_end, bs.start_step, bs.include_eos, bs.num_disable,
                              bs.num_begin, bs.ts_begin, bs.ts_end, bs.ts_eot, bs.ts_no_timestamps, bs.ts_max_initial,
                              bs.sample_topk, temperature_bits, penalty_bits, bs.no_repeat_ngram, bs.num_sequences,
                              bs.hyp_anc != nullptr};
  const int64_t poll = eos_poll_interval();
  int32_t* hfin = beam_.host;
  for (int64_t s = 0; s < bs.max_steps; ++s) {
    launch_or_capture_step(bs, S, key);
    if (s + 1 == bs.max_steps) break;
    if (s >= first_check && (s - first_check) % poll == poll - 1) {
      CT2_CUDA_CHECK(cudaMemcpyAsync(hfin, bs.num_finished, 4, cudaMemcpyDeviceToHost, stream()));
      CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));
      if (*hfin >= bs.batch) break;
    }
  }
}

// =============================================================================================
// Translator::translate_batch
// =============================================================================================
std::vector<TranslationHypotheses> Translator::translate(const TranslationRequest& r) {
  std::lock_guard<std::mutex> lock(mu_);
  CT2_REQUIRE(!mc_.whisper, "this is a Whisper model: use whisper_generate");
  const int64_t B = r.batch, S = r.max_source_len, L = r.max_decoding_length;
  const int beam = r.beam_size;
  CT2_REQUIRE(B > 0 && S > 0, "translate_batch: empty batch");
  CT2_REQUIRE(beam >= 1 && beam <= 32, "beam_size must be in [1, 32]");
  CT2_REQUIRE(r.num_hypotheses >= 1 && r.num_hypotheses <= beam, "num_hypotheses must be in [1, beam_size]");   // decoding.cc:1046-1048
  CT2_REQUIRE(L >= 1 && r.min_decoding_length <= L, "min_decoding_length is greater than max_decoding_length");
  CT2_REQUIRE(r.patience > 0.f && r.patience <= 2.f, "patience must be in (0, 2]");
  CT2_REQUIRE(r.end_ids.size() <= 64, "at most 64 end tokens");
  CT2_REQUIRE(static_cast<int64_t>(2) * beam <= static_cast<int64_t>(beam) * mc_.tgt_vocab, "beam_size exceeds the vocabulary");
  for (int64_t b = 0; b < B; ++b) {
    CT2_REQUIRE(r.source_lens[b] >= 1 && r.source_lens[b] <= S, "translate_batch: source lengths must be in [1, max_source_len]");
    for (int64_t t = 0; t < r.source_lens[b]; ++t) {
      const int32_t id = r.source_ids[b * S + t];
      CT2_REQUIRE(id >= 0 && id < mc_.src_vocab, "translate_batch: source id out of range");
    }
  }
  CT2_REQUIRE(std::isfinite(r.repetition_penalty) && r.repetition_penalty > 0.f, "repetition_penalty must be positive and finite");
  CT2_REQUIRE(r.no_repeat_ngram_size >= 0, "no_repeat_ngram_size must be >= 0");
  const int64_t nseq = r.sequence_offsets.empty() ? 0 : static_cast<int64_t>(r.sequence_offsets.size()) - 1;
  CT2_REQUIRE(static_cast<int64_t>(r.disable_ids.size()) <= kMaxSuppressSequences && nseq <= kMaxSuppressSequences &&
                  static_cast<int64_t>(r.sequence_ids.size()) <= kMaxSuppressSequenceTokens,
              "suppress_sequences: at most 4096 ids, 4096 sequences and 65536 tokens in all");
  CT2_REQUIRE(r.sequence_offsets.empty() ? r.sequence_ids.empty()
                                         : r.sequence_offsets.front() == 0 &&
                                               r.sequence_offsets.back() == static_cast<int64_t>(r.sequence_ids.size()),
              "suppress_sequences: offsets must start at 0 and end at the number of ids");
  for (int64_t s = 0; s < nseq; ++s)
    CT2_REQUIRE(r.sequence_offsets[s] <= r.sequence_offsets[s + 1], "suppress_sequences: offsets must not decrease");
  for (const std::vector<int32_t>* ids : {&r.disable_ids, &r.sequence_ids})
    for (int32_t id : *ids) CT2_REQUIRE(id >= 0 && id < mc_.tgt_vocab, "suppressed token id outside the target vocabulary");
  CT2_REQUIRE(std::isfinite(r.coverage_penalty), "coverage_penalty must be finite");
  const bool keep_attention = r.attention || r.coverage_penalty != 0.f;
  ensure_arena(B, S, beam, L);
  if (keep_attention && beam_.ensure_attention(S, mc_.align_heads)) drop_graph();   // the step reads them through their address
  const size_t table = r.disable_ids.size() + r.sequence_offsets.size() + r.sequence_ids.size();
  if (table * 4 > beam_.processors.bytes) drop_graph();          // the captured step reads the tables through their address
  beam_.ensure_processors(table);

  // ---- inputs ----
  int32_t* hp = host_pinned_;
  for (int64_t b = 0; b < B; ++b)
    for (int64_t t = 0; t < S; ++t) hp[b * S + t] = t < r.source_lens[b] ? r.source_ids[b * S + t] : 0;
  int32_t* hl = hp + B * S;
  for (int64_t b = 0; b < B; ++b) hl[b] = r.source_lens[b];
  int32_t* hend = hl + B;
  for (size_t i = 0; i < r.end_ids.size(); ++i) hend[i] = r.end_ids[i];
  CT2_CUDA_CHECK(cudaMemcpyAsync(src_ids_.ptr, hp, B * S * 4, cudaMemcpyHostToDevice, stream()));
  CT2_CUDA_CHECK(cudaMemcpyAsync(src_lens_.ptr, hl, B * 4, cudaMemcpyHostToDevice, stream()));
  if (!r.end_ids.empty())
    CT2_CUDA_CHECK(cudaMemcpyAsync(beam_.end_ids.ptr, hend, r.end_ids.size() * 4, cudaMemcpyHostToDevice, stream()));

  // ---- encoder + memory projections ----
  run_encoder(B, S);
  project_memory(B, S);

  // ---- beam search: the earliest step at which an entry can be complete is min_decoding_length ----
  BeamState bs = beam_.state(B, beam, mc_.tgt_vocab, L, r.min_decoding_length, r.patience, r.length_penalty, r.num_hypotheses,
                             static_cast<int>(r.end_ids.size()));
  set_logits_ld(bs);
  beam_.set_processors(bs, r.repetition_penalty, r.no_repeat_ngram_size, r.disable_ids, r.sequence_offsets, r.sequence_ids,
                       stream());
  if (keep_attention) bs.hyp_anc = beam_.hyp_anc.as<int32_t>();
  if (r.coverage_penalty != 0.f) bs.early_exit = 0;               // decoding.cc:457: no early exit under a coverage penalty
  beam_.reset(bs, r.start_id, dtype_, stream());
  run_search(bs, S, std::max<int64_t>(0, r.min_decoding_length));
  return beam_.collect(bs, r.length_penalty, r.num_hypotheses, r.return_end_token ? std::vector<int32_t>{} : r.end_ids, stream(),
                       r.coverage_penalty, static_cast<int>(S), r.attention, L);
}

// =============================================================================================
// Translator::score_batch
// =============================================================================================
namespace {
constexpr int64_t kScorePassRows = 4096;   // decoder rows (and encoder rows) of one teacher-forced pass, one pair at least
constexpr int64_t kScoreSlabRows = 1024;   // scored positions projected at once; the slab also holds at most 256 MB of logits
}  // namespace

// The full-sequence decoder call (decoder.cc:13-26) shared by score, whisper_align and whisper_detect_language.  Uncaptured:
// the translate graph, the beam state and logits_ are not touched.
bool Translator::decode_teacher_forced(int64_t entries, int64_t T, int64_t S, const int32_t* ids_d,
                                       const std::vector<AttnCapture>* capture) {
  const float scale = 1.f / std::sqrt(static_cast<float>(mc_.head_dim));
  embed_decoder(ids_d, entries * T, T, nullptr);
  return run_decoder_layers(entries * T, static_cast<int>(T), S, [&](int) {
    launch_attention_causal(qkv_.ptr, entries, static_cast<int>(T), mc_.num_heads, mc_.head_dim, scale, ctx_.ptr, dtype_, stream());
  }, capture);
}

void Translator::project_rows(const int32_t* rows_d, int64_t n, bool xq,
                              const std::function<void(const void*, int64_t, int64_t, int64_t)>& reduce) {
  const int64_t ld = ensure_score_slab();
  CT2_REQUIRE(rows_d || n <= score_slab_rows_, "project_rows: rows projected in place must fit one slab");
  for (int64_t c = 0; c < n; c += score_slab_rows_) {
    const int64_t k = std::min(score_slab_rows_, n - c);
    if (rows_d) launch_gather_rows(x_.ptr, rows_d + c, k, mc_.d_model * dtype_size(dtype_), q_.ptr, stream());
    dense(projection_, mc_.has_dec_final_norm ? &dec_norm_ : nullptr, rows_d ? q_.ptr : x_.ptr, k, nullptr, -1,
          score_logits_.ptr, !rows_d && xq, ld);
    reduce(score_logits_.ptr, c, k, ld);
  }
}

const int32_t* Translator::stage_ids(const std::vector<int32_t>& ids) {
  const size_t bytes = ids.size() * sizeof(int32_t);
  if (score_ids_.bytes < bytes) score_ids_.alloc(bytes);
  CT2_CUDA_CHECK(cudaMemcpyAsync(score_ids_.ptr, ids.data(), bytes, cudaMemcpyHostToDevice, stream()));
  return score_ids_.as<int32_t>();
}

// EncoderDecoderReplica::run_scoring + score_sequences (sequence_to_sequence.cc:235-261, scoring.cc:6-66).  Consecutive pairs
// are grouped into passes of at most kScorePassRows rows.  A pass runs the encoder and the memory projections, then the
// teacher-forced decoder pass over all decoder inputs ids[:-1] of its pairs.  The rows of scored positions (offset <= t <
// len - 1, never padding) go through project_rows with the fused LogSoftMax + Gather; one float per scored position comes
// back to the host.
void Translator::score(const int32_t* src_ids_h, const int32_t* src_lens_h, int64_t batch, int64_t S, const int32_t* tgt_ids_h,
                       const int32_t* tgt_lens_h, int64_t T, int64_t offset, float* out_h) {
  std::lock_guard<std::mutex> lock(mu_);
  CT2_REQUIRE(!mc_.whisper, "this is a Whisper model: score_batch serves Translator models");
  CT2_REQUIRE(batch > 0 && S > 0 && T >= 1, "score_batch: empty batch");
  CT2_REQUIRE(offset >= 0, "score_batch: offset must be >= 0");
  CT2_REQUIRE(T - 1 <= dec_positions_, "No position encodings are defined for positions this far (common.cc:157-161)");
  for (int64_t b = 0; b < batch; ++b) {
    CT2_REQUIRE(src_lens_h[b] >= 1 && src_lens_h[b] <= S, "score_batch: source lengths must be in [1, max_source_len]");
    CT2_REQUIRE(src_lens_h[b] <= enc_positions_, "No position encodings are defined for positions this far (common.cc:157-161)");
    CT2_REQUIRE(tgt_lens_h[b] >= 0 && tgt_lens_h[b] <= T, "score_batch: target lengths must be in [0, max_target_len]");
    for (int64_t t = 0; t < src_lens_h[b]; ++t)
      CT2_REQUIRE(src_ids_h[b * S + t] >= 0 && src_ids_h[b * S + t] < mc_.src_vocab, "score_batch: source id out of range");
    for (int64_t t = 0; t < tgt_lens_h[b]; ++t)
      CT2_REQUIRE(tgt_ids_h[b * T + t] >= 0 && tgt_ids_h[b * T + t] < mc_.tgt_vocab, "score_batch: target id out of range");
  }
  const int64_t Tout = T - 1;
  std::fill(out_h, out_h + batch * Tout, 0.f);
  const int64_t V = mc_.tgt_vocab;
  for (int64_t p0 = 0; p0 < batch;) {
    // pairs p0 .. p1 - 1, padded to Sp source and Tp decoder positions
    int64_t p1 = p0 + 1, Sp = src_lens_h[p0], Tp = std::max<int64_t>(1, tgt_lens_h[p0] - 1);
    for (; p1 < batch; ++p1) {
      const int64_t s = std::max<int64_t>(Sp, src_lens_h[p1]), t = std::max<int64_t>(Tp, tgt_lens_h[p1] - 1);
      if ((p1 - p0 + 1) * std::max(s, t) > kScorePassRows) break;
      Sp = s;
      Tp = t;
    }
    const int64_t nb = p1 - p0, rows = nb * Tp;
    std::vector<int32_t> src(nb * Sp, 0), lens(nb), staged(rows, 0), picked, targets;   // staged: decoder inputs | picked | targets
    std::vector<int64_t> dest;                                                           // place of each scored position in out_h
    for (int64_t b = 0; b < nb; ++b) {
      const int64_t g = p0 + b, n = tgt_lens_h[g] - 1;
      lens[b] = src_lens_h[g];
      std::copy(src_ids_h + g * S, src_ids_h + g * S + lens[b], src.begin() + b * Sp);
      for (int64_t t = 0; t < n; ++t) staged[b * Tp + t] = tgt_ids_h[g * T + t];
      for (int64_t t = offset; t < n; ++t) {
        picked.push_back(static_cast<int32_t>(b * Tp + t));
        targets.push_back(tgt_ids_h[g * T + t + 1]);
        dest.push_back(g * Tout + t - offset);
      }
    }
    p0 = p1;
    const int64_t np = static_cast<int64_t>(picked.size());
    if (np == 0) continue;
    staged.insert(staged.end(), picked.begin(), picked.end());
    staged.insert(staged.end(), targets.begin(), targets.end());
    ensure_rows(nb, nb * Sp, std::max(rows, nb * Sp));     // no search state: the beam arena and self K/V keep their size
    if (score_out_.bytes < np * sizeof(float)) score_out_.alloc(np * sizeof(float));
    float* scores_d = score_out_.as<float>();
    CT2_CUDA_CHECK(cudaMemcpyAsync(src_ids_.ptr, src.data(), src.size() * 4, cudaMemcpyHostToDevice, stream()));
    CT2_CUDA_CHECK(cudaMemcpyAsync(src_lens_.ptr, lens.data(), nb * 4, cudaMemcpyHostToDevice, stream()));
    const int32_t* dec_d = stage_ids(staged);
    const int32_t* picked_d = dec_d + rows;
    const int32_t* targets_d = picked_d + np;

    run_encoder(nb, Sp);
    project_memory(nb, Sp);
    decode_teacher_forced(nb, Tp, Sp, dec_d);
    project_rows(picked_d, np, false, [&](const void* logits, int64_t c, int64_t k, int64_t ld) {
      launch_log_softmax_gather(logits, targets_d + c, k, V, scores_d + c, dtype_, stream(), ld);
    });
    std::vector<float> vals(np);
    CT2_CUDA_CHECK(cudaMemcpyAsync(vals.data(), scores_d, np * sizeof(float), cudaMemcpyDeviceToHost, stream()));
    CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));     // also keeps the staging vectors alive until their copies are done
    for (int64_t i = 0; i < np; ++i) out_h[dest[i]] = vals[i];
  }
}

int64_t Translator::ensure_score_slab() {
  const int64_t V = mc_.tgt_vocab;
  const size_t es = dtype_size(dtype_);
  // row stride of the logits: the INT8 epilogue stores 16-byte rows (set_logits_ld)
  const int64_t ld = projection_.kind == DenseWeights::INT8 ? (V + 7) / 8 * 8 : V;
  if (!score_logits_.ptr) {
    score_slab_rows_ = std::max<int64_t>(1, std::min<int64_t>(kScoreSlabRows, (static_cast<int64_t>(256) << 20) / (ld * es)));
    score_logits_.alloc(static_cast<size_t>(score_slab_rows_) * ld * es);
  }
  return ld;
}

void Translator::encode(const int32_t* ids_h, const int32_t* lens_h, int64_t batch, int64_t S, float* memory_h) {
  std::lock_guard<std::mutex> lock(mu_);
  CT2_REQUIRE(!mc_.whisper, "this is a Whisper model: use whisper_encode");
  CT2_REQUIRE(batch > 0 && S > 0, "encode: empty batch");
  ensure_arena(batch, S, 1, 1);
  int32_t* hp = host_pinned_;
  for (int64_t b = 0; b < batch; ++b) {
    CT2_REQUIRE(lens_h[b] >= 1 && lens_h[b] <= S, "encode: source lengths must be in [1, max_source_len]");
    for (int64_t t = 0; t < S; ++t) hp[b * S + t] = t < lens_h[b] ? ids_h[b * S + t] : 0;
  }
  CT2_CUDA_CHECK(cudaMemcpyAsync(src_ids_.ptr, hp, batch * S * 4, cudaMemcpyHostToDevice, stream()));
  CT2_CUDA_CHECK(cudaMemcpyAsync(src_lens_.ptr, lens_h, batch * 4, cudaMemcpyHostToDevice, stream()));
  run_encoder(batch, S);
  copy_memory_to_host(batch * S, memory_h);
}

void Translator::copy_memory_to_host(int64_t rows, float* memory_h) {
  DeviceBuffer f32(static_cast<size_t>(rows) * mc_.d_model * 4);
  launch_convert_to_f32(memory_.ptr, rows * mc_.d_model, f32.as<float>(), dtype_, stream());
  CT2_CUDA_CHECK(cudaMemcpyAsync(memory_h, f32.ptr, f32.bytes, cudaMemcpyDeviceToHost, stream()));
  CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));
}

void Translator::bench(int64_t batch, int64_t source_len, int beam, int64_t steps, int64_t warmup, float* encode_ms,
                       float* decode_ms, int64_t* launches) {
  std::lock_guard<std::mutex> lock(mu_);
  CT2_REQUIRE(!mc_.whisper, "bench_translate serves Translator models");
  const int64_t L = steps + warmup;
  ensure_arena(batch, source_len, beam, L);
  std::vector<int32_t> ids(batch * source_len), lens(batch, static_cast<int32_t>(source_len));
  for (size_t i = 0; i < ids.size(); ++i) ids[i] = static_cast<int32_t>((7919ull * i + 3) % mc_.src_vocab);
  CT2_CUDA_CHECK(cudaMemcpy(src_ids_.ptr, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice));
  CT2_CUDA_CHECK(cudaMemcpy(src_lens_.ptr, lens.data(), lens.size() * 4, cudaMemcpyHostToDevice));
  CT2_CUDA_CHECK(cudaDeviceSynchronize());      // pageable H2D: the DMA may still be running when cudaMemcpy returns (see upload())
  BeamState bs = beam_.state(batch, beam, mc_.tgt_vocab, L, 0, 1.f, 1.f, 1, 0);   // no end token: nothing finishes early
  set_logits_ld(bs);
  const std::vector<int64_t> key = {-1, batch, beam, source_len, bs.stride, L};
  cudaEvent_t e0, e1, e2, e3;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventCreate(&e2);
  cudaEventCreate(&e3);
  run_encoder(batch, source_len);      // warm-up (first-use kernel configuration)
  project_memory(batch, source_len);
  CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));
  cudaEventRecord(e0, stream());
  run_encoder(batch, source_len);
  project_memory(batch, source_len);
  cudaEventRecord(e1, stream());
  beam_.reset(bs, 1, dtype_, stream());
  for (int64_t s = 0; s < warmup; ++s) launch_or_capture_step(bs, source_len, key);
  CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));
  const int64_t l0 = g_kernel_launches.load();
  cudaProfilerStart();
  cudaEventRecord(e2, stream());
  for (int64_t s = 0; s < steps; ++s) launch_or_capture_step(bs, source_len, key);
  cudaEventRecord(e3, stream());
  CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));
  cudaProfilerStop();
  *launches = g_kernel_launches.load() - l0;
  cudaEventElapsedTime(encode_ms, e0, e1);
  cudaEventElapsedTime(decode_ms, e2, e3);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaEventDestroy(e2);
  cudaEventDestroy(e3);
}

// =============================================================================================
// Encoder (models::EncoderReplica, src/models/language_model.cc:302-400)
// =============================================================================================
// TransformerEncoder::operator() with the merged embeddings (transformer.cc:427-471): tokens + types (ADD in T), scale,
// positions, layernorm_embedding, the layers, output norm; then pooler_dense + activation on each row's first position
void Translator::run_encoder_only(int64_t batch, int64_t S) {
  const int64_t rows = batch * S, d = mc_.d_model;
  launch_embed_pos(enc_emb_.weight.ptr, enc_emb_.kind == DenseWeights::INT8 ? enc_emb_.scale.as<float>() : nullptr,
                   src_ids_.as<int32_t>(), rows, d, mc_.enc_emb_scale, enc_pos_.ptr, S, nullptr, false, x_.ptr, dtype_, stream(),
                   mc_.type_vocab ? type_emb_.weight.ptr : nullptr,
                   type_emb_.kind == DenseWeights::INT8 ? type_emb_.scale.as<float>() : nullptr, type_ids_.as<int32_t>());
  if (mc_.has_emb_norm)
    launch_layer_norm(x_.ptr, emb_norm_.gamma.ptr, emb_norm_.beta.ptr, rows, d, mc_.eps, x_.ptr, nullptr, nullptr, true, dtype_,
                      stream());
  run_encoder_layers(batch, S, src_lens_.as<int32_t>());
  if (mc_.has_pooler) {
    const size_t es = dtype_size(dtype_);
    CT2_CUDA_CHECK(cudaMemcpy2DAsync(first_.ptr, d * es, memory_.ptr, S * d * es, d * es, batch, cudaMemcpyDeviceToDevice, stream()));
    dense(pooler_, nullptr, first_.ptr, batch, nullptr, mc_.pooler_activation, pooled_.ptr);
  }
}

void Translator::encoder_forward(const int32_t* ids_h, const int32_t* types_h, const int32_t* lens_h, int64_t batch, int64_t T,
                                 float* hidden_h, float* pooled_h) {
  std::lock_guard<std::mutex> lock(mu_);
  CT2_REQUIRE(mc_.encoder_only, "forward_batch needs an encoder model (TransformerEncoderSpec)");
  CT2_REQUIRE(batch > 0 && T > 0, "forward_batch: empty batch");
  CT2_REQUIRE(T <= enc_positions_, "forward_batch: the sequences are longer than the position table");
  // padded positions get id 0 / type 0 so that every gathered row is in range
  std::vector<int32_t> ids(batch * T, 0), types(batch * T, 0);
  for (int64_t b = 0; b < batch; ++b) {
    CT2_REQUIRE(lens_h[b] >= 1 && lens_h[b] <= T, "forward_batch: lengths must be in [1, max_length]");
    for (int64_t t = 0; t < lens_h[b]; ++t) {
      const int32_t id = ids_h[b * T + t];
      CT2_REQUIRE(id >= 0 && id < mc_.src_vocab, "forward_batch: input id out of range");
      ids[b * T + t] = id;
      if (types_h) {
        const int32_t ty = types_h[b * T + t];
        CT2_REQUIRE(mc_.type_vocab > 0, "forward_batch: this model has no token-type embeddings");
        CT2_REQUIRE(ty >= 0 && ty < mc_.type_vocab, "forward_batch: token type id out of range");
        types[b * T + t] = ty;
      }
    }
  }
  ensure_rows(batch, batch * T, batch * T);
  const size_t es = dtype_size(dtype_);
  if (batch * T > cap_types_) {
    cap_types_ = batch * T;
    type_ids_.alloc(cap_types_ * 4);
  }
  if (mc_.has_pooler && batch > cap_pooled_) {
    cap_pooled_ = batch;
    first_.alloc(batch * mc_.d_model * es);
    pooled_.alloc(batch * mc_.d_model * es);
  }
  CT2_CUDA_CHECK(cudaMemcpyAsync(src_ids_.ptr, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice, stream()));
  CT2_CUDA_CHECK(cudaMemcpyAsync(type_ids_.ptr, types.data(), types.size() * 4, cudaMemcpyHostToDevice, stream()));
  CT2_CUDA_CHECK(cudaMemcpyAsync(src_lens_.ptr, lens_h, batch * 4, cudaMemcpyHostToDevice, stream()));
  run_encoder_only(batch, T);
  if (mc_.has_pooler && pooled_h) {
    DeviceBuffer f32(static_cast<size_t>(batch) * mc_.d_model * 4);
    launch_convert_to_f32(pooled_.ptr, batch * mc_.d_model, f32.as<float>(), dtype_, stream());
    CT2_CUDA_CHECK(cudaMemcpyAsync(pooled_h, f32.ptr, f32.bytes, cudaMemcpyDeviceToHost, stream()));
    CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));
  }
  copy_memory_to_host(batch * T, hidden_h);     // synchronises: ids / types may go
}

void Translator::encoder_bench(const int32_t* lens_h, int64_t batch, int64_t T, int64_t iters, int64_t warmup, float* median_ms) {
  CT2_REQUIRE(iters >= 1 && warmup >= 0, "encoder_bench: iters must be >= 1");
  std::vector<int32_t> ids(batch * T), types(batch * T, 0);
  for (size_t i = 0; i < ids.size(); ++i) ids[i] = static_cast<int32_t>((7919ull * i + 3) % mc_.src_vocab);
  std::vector<float> hidden(static_cast<size_t>(batch) * T * mc_.d_model), pooled(static_cast<size_t>(batch) * mc_.d_model);
  encoder_forward(ids.data(), mc_.type_vocab ? types.data() : nullptr, lens_h, batch, T, hidden.data(), pooled.data());
  std::lock_guard<std::mutex> lock(mu_);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  std::vector<float> ms;
  for (int64_t i = 0; i < warmup + iters; ++i) {
    cudaEventRecord(e0, stream());
    run_encoder_only(batch, T);
    cudaEventRecord(e1, stream());
    CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));
    float t = 0.f;
    cudaEventElapsedTime(&t, e0, e1);
    if (i >= warmup) ms.push_back(t);
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  std::sort(ms.begin(), ms.end());
  *median_ms = ms[ms.size() / 2];
}

// =============================================================================================
// Whisper (src/models/whisper.cc, src/layers/whisper.cc)
// =============================================================================================
int64_t Translator::whisper_positions(int64_t batch, int64_t frames) const {
  const int64_t S = (frames + 2 - 3) / 2 + 1;       // conv2: kernel 3, stride 2, padding 1
  CT2_REQUIRE(batch > 0 && frames >= 2 && S <= mc_.max_frames, "Invalid input features shape: too many frames for the encoder");
  return S;
}

// WhisperEncoder::operator(): conv1 + GELU, conv2 (stride 2) + GELU as im2col + float Dense (the GEMM output is already the
// transposed [batch, frames / 2, d] layout), stored positions, pre-norm GELU layers, LayerNorm
void Translator::encode_audio(const float* features_h, int64_t batch, int64_t frames) {
  const int64_t d = mc_.d_model, S = whisper_positions(batch, frames);
  audio_lens_h_.assign(batch, static_cast<int32_t>(S));
  CT2_CUDA_CHECK(cudaMemcpyAsync(features_.ptr, features_h, batch * mc_.n_mels * frames * 4, cudaMemcpyHostToDevice, stream()));
  CT2_CUDA_CHECK(cudaMemcpyAsync(src_lens_.ptr, audio_lens_h_.data(), batch * 4, cudaMemcpyHostToDevice, stream()));
  launch_im2col(features_.ptr, true, batch, mc_.n_mels, frames, frames, 3, 1, 1, true, cols_.ptr, dtype_, stream());
  gemm_float(cols_.ptr, conv1_.weight.ptr, conv1_.bias.ptr, nullptr, CT2B200_ACT_GELU, batch * frames, d, mc_.n_mels * 3,
             conv_out_.ptr, dtype_, stream());
  launch_im2col(conv_out_.ptr, false, batch, d, frames, S, 3, 2, 1, false, cols_.ptr, dtype_, stream());
  gemm_float(cols_.ptr, conv2_.weight.ptr, conv2_.bias.ptr, nullptr, CT2B200_ACT_GELU, batch * S, d, d * 3, x_.ptr, dtype_, stream());
  launch_add_positions(x_.ptr, enc_pos_.ptr, batch * S, S, d, dtype_, stream());
  run_encoder_layers(batch, S, nullptr);
}

void Translator::whisper_encode(const float* features_h, int64_t batch, int64_t frames, float* memory_h) {
  std::lock_guard<std::mutex> lock(mu_);
  CT2_REQUIRE(mc_.whisper, "whisper_encode needs a Whisper model");
  const int64_t S = whisper_positions(batch, frames);
  ensure_arena(batch, S, 1, 1);
  encode_audio(features_h, batch, frames);
  copy_memory_to_host(batch * S, memory_h);
}

std::vector<TranslationHypotheses> Translator::whisper_generate(const WhisperRequest& r, float* no_speech_h) {
  std::lock_guard<std::mutex> lock(mu_);
  CT2_REQUIRE(mc_.whisper, "whisper_generate needs a Whisper model");
  const int64_t B = r.batch, P = r.prompt_len, frames = r.frames;
  const int64_t S = whisper_positions(B, frames);
  CT2_REQUIRE(r.beam_size >= 1 && r.beam_size <= 32, "beam_size must be in [1, 32]");
  CT2_REQUIRE(r.sampling_topk >= 0 && r.sampling_temperature >= 0.f, "sampling_topk and sampling_temperature must be >= 0");
  const bool sampling = r.sampling_topk != 1 && r.sampling_temperature != 0.f;     // decoding.cc:1067-1074
  CT2_REQUIRE(!sampling || r.sampling_topk <= mc_.tgt_vocab, "sampling_topk is greater than the vocabulary size");
  CT2_REQUIRE(!sampling || r.beam_size == 1, "random sampling with beam_size > 1 (sampled beam search) is not supported");
  // a sampled call decodes num_hypotheses independent rows per entry, laid out like the rows of a beam
  const int beam = sampling ? r.num_hypotheses : r.beam_size;
  CT2_REQUIRE(r.num_hypotheses >= 1 && r.num_hypotheses <= (sampling ? 32 : r.beam_size),
              sampling ? "num_hypotheses must be in [1, 32] when sampling" : "num_hypotheses must be in [1, beam_size]");
  CT2_REQUIRE(r.patience > 0.f && r.patience <= 2.f, "patience must be in (0, 2]");
  CT2_REQUIRE(r.suppress_ids.size() + r.suppress_ids_begin.size() <= 4096, "too many suppressed tokens");
  // check_prompts (whisper.cc:168-197): <|startoftranscript|> at the same position in every prompt and the same number of
  // task tokens after it; this engine also requires the prompt to END with the task tokens (no text after them)
  CT2_REQUIRE(P >= 1 && P <= 16, "the prompt must hold <|startoftranscript|> and the task tokens (1 to 16 tokens)");
  CT2_REQUIRE(r.no_timestamps_id > r.sot_id && r.no_timestamps_id < mc_.tgt_vocab - 1, "no_timestamps_id must follow sot_id");
  int64_t sot_index = -1;
  for (int64_t b = 0; b < B; ++b) {
    int64_t idx = -1;
    for (int64_t t = 0; t < P; ++t) {
      const int32_t id = r.prompts[b * P + t];
      CT2_REQUIRE(id >= 0 && id < mc_.tgt_vocab, "prompt id out of range");
      if (id == r.sot_id && idx < 0) idx = t;
    }
    CT2_REQUIRE(idx >= 0, "<|startoftranscript|> token was not found in the prompt");
    CT2_REQUIRE(sot_index < 0 || idx == sot_index, "<|startoftranscript|> must be at the same position in all prompts");
    sot_index = idx;
    for (int64_t t = idx; t < P; ++t)                  // get_prompt_length (whisper.cc:156-166)
      CT2_REQUIRE(r.prompts[b * P + t] >= r.sot_id && r.prompts[b * P + t] <= r.no_timestamps_id,
                  "text after the task tokens (a decoding prefix) is not supported");
  }
  bool timestamps = r.prompts[P - 1] != r.no_timestamps_id;             // whisper.cc:325, decided on the first prompt
  const int64_t start_step = P - 1;
  const int64_t steps = std::min<int64_t>(r.max_length / 2, r.max_length - start_step);      // whisper.cc:299
  CT2_REQUIRE(steps >= 1, "max_length is too small for the prompt");
  ensure_arena(B, S, beam, start_step + steps);
  const int64_t N = B * beam;

  // ---- inputs ----
  int32_t* hp = host_pinned_;
  for (int64_t t = 0; t < P; ++t)                      // forced inputs [P, N]: prompt token t of the row's batch entry
    for (int64_t n = 0; n < N; ++n) hp[t * N + n] = r.prompts[(n / beam) * P + t];
  int32_t* hs = hp + P * N;
  for (size_t i = 0; i < r.suppress_ids.size(); ++i) hs[i] = r.suppress_ids[i];
  for (size_t i = 0; i < r.suppress_ids_begin.size(); ++i) hs[r.suppress_ids.size() + i] = r.suppress_ids_begin[i];
  hs[r.suppress_ids.size() + r.suppress_ids_begin.size()] = r.eot_id;
  const size_t nsup = r.suppress_ids.size() + r.suppress_ids_begin.size();
  forced_d_.alloc(P * N * 4);
  suppress_d_.alloc((nsup + 1) * 4);
  CT2_CUDA_CHECK(cudaMemcpyAsync(forced_d_.ptr, hp, P * N * 4, cudaMemcpyHostToDevice, stream()));
  CT2_CUDA_CHECK(cudaMemcpyAsync(suppress_d_.ptr, hs, (nsup + 1) * 4, cudaMemcpyHostToDevice, stream()));
  CT2_CUDA_CHECK(cudaMemcpyAsync(beam_.end_ids.ptr, suppress_d_.as<int32_t>() + nsup, 4, cudaMemcpyDeviceToDevice, stream()));
  CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));      // the pinned staging is reused below

  // ---- encoder + memory projections ----
  encode_audio(r.features, B, frames);
  project_memory(B, S);

  // ---- prompt: WhisperDecoder::forward_prompt on prompt[:-1], one position per step, no search ----
  BeamState bs = beam_.state(B, beam, mc_.tgt_vocab, steps, 0, r.patience, r.length_penalty, r.num_hypotheses, 1);
  set_logits_ld(bs);
  bs.start_step = static_cast<int>(start_step);
  bs.include_eos = 0;                                  // whisper.cc:309
  bs.num_disable = static_cast<int>(r.suppress_ids.size());
  bs.num_begin = static_cast<int>(r.suppress_ids_begin.size());
  bs.disable_ids = suppress_d_.as<int32_t>();
  bs.disable_begin = suppress_d_.as<int32_t>() + r.suppress_ids.size();
  if (timestamps) {
    bs.ts_begin = r.no_timestamps_id + 1;
    bs.ts_end = static_cast<int>(mc_.tgt_vocab) - 1;
    bs.ts_eot = r.eot_id;
    bs.ts_no_timestamps = r.no_timestamps_id;
    bs.ts_max_initial = bs.ts_begin + r.max_initial_timestamp_index;
  }
  beam_.reset(bs, r.prompts[0], dtype_, stream());
  if (sampling) beam_.reset_sampling(bs, r.sampling_topk, r.sampling_temperature, stream());
  CT2_CUDA_CHECK(cudaMemcpyAsync(beam_.next_ids.ptr, forced_d_.ptr, N * 4, cudaMemcpyDeviceToDevice, stream()));
  no_speech_d_.alloc(B * 4);
  for (int64_t t = 0; t < start_step; ++t) {
    decoder_step(N, beam, B, S);
    if (no_speech_h && t == sot_index) {
      CT2_REQUIRE(r.no_speech_id >= 0, "return_no_speech_prob needs the id of <|nospeech|>");
      launch_token_prob(logits_.ptr, B, mc_.tgt_vocab, static_cast<int64_t>(beam) * logits_ld_, r.no_speech_id,
                        no_speech_d_.as<float>(), dtype_, stream());
    }
    launch_beam_force(bs, forced_d_.as<int32_t>() + (t + 1) * N, stream());
  }
  CT2_REQUIRE(!no_speech_h || sot_index < start_step, "return_no_speech_prob with <|startoftranscript|> as the last prompt "
                                                      "token is not supported");

  // ---- search ----
  run_search(bs, S, 0);
  if (no_speech_h) {
    CT2_CUDA_CHECK(cudaMemcpyAsync(no_speech_h, no_speech_d_.ptr, B * 4, cudaMemcpyDeviceToHost, stream()));
    CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));
  }
  return beam_.collect(bs, r.length_penalty, r.num_hypotheses, {}, stream());
}

// =============================================================================================
// Whisper::align and Whisper::detect_language
// =============================================================================================
namespace {
constexpr int64_t kAlignScoreBytes = static_cast<int64_t>(256) << 20;   // captured scores of one pass (one entry at least)
constexpr int64_t kDetectPassEntries = 16;                              // entries encoded at once by detect_language
constexpr int64_t kAlignEncoderRows = 16 * 1500;                        // encoder rows of one pass: 16 windows of 30 s
}  // namespace

// WhisperReplica::align (whisper.cc:424-582) + compute_alignments (:387-422).  Entries are grouped into passes of at most
// kScorePassRows decoder rows and kAlignScoreBytes of captured scores.  A pass runs the encoder and the memory projections, then
// the teacher-forced decoder pass over every input start + <|notimestamps|> + text + <|endoftext|> (the memory is not masked),
// with the cross-attention of the alignment heads saving their scores.  The rows of the text positions go through
// project_rows with SoftMax over [0, <|endoftext|>) + Gather.  The scores go
// through SoftMax over the entry's frames, the standardisation of every frame column over the token rows (all T_max rows of
// the batch when every entry has the same frame count -- the rows past an input's length are copies of its last row, as the
// reference's Padder adds them back -- otherwise the entry's own rows), the median filter and the mean over the heads.  The
// DTW matrices come back to the host, where negative_dtw runs.  Uncaptured; the search state is not touched.
std::vector<WhisperAlignResult> Translator::whisper_align(const WhisperAlignRequest& r, float* matrix_h) {
  std::lock_guard<std::mutex> lock(mu_);
  CT2_REQUIRE(mc_.whisper, "whisper_align needs a Whisper model");
  const int64_t B = r.batch, frames = r.frames, s0 = r.start_len, Nt = r.max_text;
  const int64_t S = whisper_positions(B, frames);
  const int64_t V = mc_.tgt_vocab;
  CT2_REQUIRE(s0 >= 1 && Nt >= 0, "align: the start sequence must not be empty");
  CT2_REQUIRE(r.eot_id >= 1 && r.eot_id < V && r.no_timestamps_id >= 0 && r.no_timestamps_id < V, "align: special id out of range");
  const int width = r.median_filter_width;
  CT2_REQUIRE(width <= 1 || (width % 2 == 1 && width <= 129), "MedianFilter width must be odd and at most 129");
  const int Hs = static_cast<int>(r.heads.size());
  CT2_REQUIRE(Hs >= 1, "align: no alignment heads");
  // layer order, then list order (set_alignment_heads, transformer.cc:577-584): slot k of layer l's list -> bit k of the mask
  // of its head; layers without heads run the plain cross-attention
  const int H = mc_.num_heads;
  std::vector<int> count(mc_.dec_layers, 0);
  std::vector<uint32_t> masks(static_cast<size_t>(mc_.dec_layers) * H, 0);
  for (const auto& [layer, head] : r.heads) {
    CT2_REQUIRE(layer >= 0 && layer < mc_.dec_layers && head >= 0 && head < H, "align: alignment head out of range");
    CT2_REQUIRE(count[layer] < 32, "align: at most 32 alignment heads per layer");
    masks[static_cast<size_t>(layer) * H + head] |= 1u << count[layer]++;
  }
  if (align_masks_.bytes < masks.size() * 4) align_masks_.alloc(masks.size() * 4);
  CT2_CUDA_CHECK(cudaMemcpyAsync(align_masks_.ptr, masks.data(), masks.size() * 4, cudaMemcpyHostToDevice, stream()));
  std::vector<AttnCapture> capture(mc_.dec_layers);
  for (int l = 0, first = 0; l < mc_.dec_layers; ++l) {
    capture[l].masks = count[l] ? align_masks_.as<uint32_t>() + static_cast<size_t>(l) * H : nullptr;
    capture[l].first = first;
    capture[l].total = Hs;
    first += count[l];
  }
  for (int64_t t = 0; t < s0; ++t) CT2_REQUIRE(r.start[t] >= 0 && r.start[t] < V, "align: start id out of range");
  std::vector<int32_t> nf(B), len(B);
  int64_t Tg = 0;
  bool all_zero = true, equal = true;
  for (int64_t b = 0; b < B; ++b) {
    CT2_REQUIRE(r.text_lens[b] >= 0 && r.text_lens[b] <= Nt, "align: text lengths must be in [0, max_text]");
    for (int64_t t = 0; t < r.text_lens[b]; ++t)
      CT2_REQUIRE(r.text[b * Nt + t] >= 0 && r.text[b * Nt + t] < V, "align: text id out of range");
    CT2_REQUIRE(r.num_frames[b] >= 0, "align: num_frames must be >= 0");
    nf[b] = r.num_frames[b] / 2;                      // the second convolution has stride 2
    CT2_REQUIRE(nf[b] <= S, "align: num_frames exceeds the features' frames");
    len[b] = static_cast<int32_t>(s0 + r.text_lens[b] + 2);
    CT2_REQUIRE(len[b] <= dec_positions_, "No position encodings are defined for positions this far (common.cc:157-161)");
    Tg = std::max<int64_t>(Tg, len[b]);
    all_zero = all_zero && nf[b] == 0;
    equal = equal && nf[b] == nf[0];
  }
  std::vector<WhisperAlignResult> results(B);
  if (matrix_h) std::fill(matrix_h, matrix_h + B * (Nt + 1) * S, 0.f);
  for (int64_t p0 = 0; p0 < B;) {
    int64_t p1 = p0 + 1, Tp = len[p0];
    for (; p1 < B; ++p1) {
      const int64_t t = std::max<int64_t>(Tp, len[p1]), n = p1 - p0 + 1;
      if (n * t > kScorePassRows || n * S > kAlignEncoderRows || n * Hs * t * S * 4 > kAlignScoreBytes) break;
      Tp = t;
    }
    const int64_t nb = p1 - p0, rows = nb * Tp;
    // staged: decoder inputs [rows] | picked rows [np] | their text ids [np] | nf [nb] | len [nb] | text lengths [nb]
    std::vector<int32_t> staged(rows, 0), picked, targets;
    for (int64_t b = 0; b < nb; ++b) {
      const int64_t g = p0 + b, n = r.text_lens[g];
      int32_t* in = staged.data() + b * Tp;
      std::copy(r.start, r.start + s0, in);
      in[s0] = r.no_timestamps_id;
      std::copy(r.text + g * Nt, r.text + g * Nt + n, in + s0 + 1);
      in[s0 + 1 + n] = r.eot_id;
      for (int64_t t = 0; t < n; ++t) {                 // logits at position s0 + t, gathered at text[t] (whisper.cc:495-502)
        picked.push_back(static_cast<int32_t>(b * Tp + s0 + t));
        targets.push_back(r.text[g * Nt + t]);
      }
    }
    const int64_t np = static_cast<int64_t>(picked.size());
    staged.insert(staged.end(), picked.begin(), picked.end());
    staged.insert(staged.end(), targets.begin(), targets.end());
    staged.insert(staged.end(), nf.begin() + p0, nf.begin() + p1);
    staged.insert(staged.end(), len.begin() + p0, len.begin() + p1);
    for (int64_t b = p0; b < p1; ++b) staged.push_back(r.text_lens[b]);
    ensure_whisper_frontend(nb, S);
    ensure_rows(nb, nb * S, std::max(rows, nb * S));
    if (score_out_.bytes < std::max<int64_t>(np, 1) * sizeof(float)) score_out_.alloc(std::max<int64_t>(np, 1) * sizeof(float));
    const size_t score_bytes = static_cast<size_t>(nb) * Hs * Tp * S * 4, norm_bytes = static_cast<size_t>(nb) * Hs * (Nt + 1) * S * 4;
    const size_t matrix_bytes = static_cast<size_t>(nb) * (Nt + 1) * S * 4;
    if (align_scores_.bytes < score_bytes) align_scores_.alloc(score_bytes);
    if (align_norm_.bytes < norm_bytes) align_norm_.alloc(norm_bytes);
    if (align_matrix_.bytes < matrix_bytes) align_matrix_.alloc(matrix_bytes);
    const int32_t* dec_d = stage_ids(staged);
    const int32_t* picked_d = dec_d + rows;
    const int32_t* targets_d = picked_d + np;
    const int32_t* nf_d = targets_d + np;
    const int32_t* len_d = nf_d + nb;
    const int32_t* ntext_d = len_d + nb;
    float* probs_d = score_out_.as<float>();

    encode_audio(r.features + p0 * mc_.n_mels * frames, nb, frames);
    project_memory(nb, S);
    for (auto& c : capture) c.out = align_scores_.as<float>();
    decode_teacher_forced(nb, Tp, S, dec_d, &capture);
    project_rows(picked_d, np, false, [&](const void* logits, int64_t c, int64_t k, int64_t ld) {
      launch_softmax_gather(logits, targets_d + c, k, r.eot_id, ld, probs_d + c, dtype_, stream());
    });
    std::vector<float> probs(np), matrix;
    if (!all_zero) {
      float* sc = align_scores_.as<float>();
      launch_align_softmax(sc, nf_d, len_d, nb, Hs, Tp, S, dtype_, stream());
      launch_align_standardize(sc, nf_d, len_d, ntext_d, nb, Hs, Tp, S, equal ? Tg : 0, s0, Nt, S, align_norm_.as<float>(), dtype_,
                               stream());
      launch_align_median_mean(align_norm_.as<float>(), nf_d, ntext_d, nb, Hs, Nt, S, width, align_matrix_.as<float>(), dtype_,
                               stream());
      matrix.resize(nb * (Nt + 1) * S);
      CT2_CUDA_CHECK(cudaMemcpyAsync(matrix.data(), align_matrix_.ptr, matrix_bytes, cudaMemcpyDeviceToHost, stream()));
    }
    if (np) CT2_CUDA_CHECK(cudaMemcpyAsync(probs.data(), probs_d, np * sizeof(float), cudaMemcpyDeviceToHost, stream()));
    CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));     // also keeps the staging vectors alive until their copies are done
    int64_t k = 0;
    for (int64_t b = 0; b < nb; ++b) {
      const int64_t g = p0 + b, n = r.text_lens[g];
      results[g].text_token_probs.assign(probs.begin() + k, probs.begin() + k + n);
      k += n;
      if (all_zero || nf[g] == 0) continue;
      const float* mb = matrix.data() + b * (Nt + 1) * S;
      if (matrix_h) std::copy(mb, mb + (Nt + 1) * S, matrix_h + g * (Nt + 1) * S);
      std::vector<float> x((n + 1) * nf[g]);
      for (int64_t i = 0; i <= n; ++i) std::copy(mb + i * S, mb + i * S + nf[g], x.begin() + i * nf[g]);
      results[g].path = negative_dtw(x.data(), n + 1, nf[g]);
    }
    p0 = p1;
  }
  return results;
}

// WhisperReplica::detect_language (whisper.cc:584-652): one decoder position per entry on <|startoftranscript|>, Gather of the
// language ids' logits, SoftMax over them in T.  The caller sorts.
void Translator::whisper_detect_language(const float* features_h, int64_t batch, int64_t frames, int32_t sot_id,
                                         const std::vector<int32_t>& lang_ids, float* probs_h) {
  std::lock_guard<std::mutex> lock(mu_);
  CT2_REQUIRE(mc_.whisper, "detect_language needs a Whisper model");
  const int64_t S = whisper_positions(batch, frames), V = mc_.tgt_vocab;
  CT2_REQUIRE(sot_id >= 0 && sot_id < V, "detect_language: <|startoftranscript|> out of range");
  const int n = static_cast<int>(lang_ids.size());
  CT2_REQUIRE(n >= 1, "detect_language: no language ids");
  for (int32_t id : lang_ids) CT2_REQUIRE(id >= 0 && id < V, "detect_language: language id out of range");
  ensure_score_slab();
  const int64_t per_pass = std::min<int64_t>(score_slab_rows_, kDetectPassEntries);   // one slab: projected in place
  for (int64_t p0 = 0; p0 < batch; p0 += per_pass) {
    const int64_t nb = std::min(per_pass, batch - p0);
    ensure_whisper_frontend(nb, S);
    ensure_rows(nb, nb * S, nb * S);
    if (score_out_.bytes < nb * n * sizeof(float)) score_out_.alloc(nb * n * sizeof(float));
    std::vector<int32_t> staged(nb, sot_id);           // decoder inputs | language ids
    staged.insert(staged.end(), lang_ids.begin(), lang_ids.end());
    const int32_t* ids_d = stage_ids(staged);
    float* probs_d = score_out_.as<float>();
    encode_audio(features_h + p0 * mc_.n_mels * frames, nb, frames);
    project_memory(nb, S);
    const bool xq = decode_teacher_forced(nb, 1, S, ids_d);
    project_rows(nullptr, nb, xq, [&](const void* logits, int64_t c, int64_t k, int64_t ld) {
      launch_gather_softmax(logits, k, ld, ids_d + nb, n, probs_d + c * n, dtype_, stream());
    });
    CT2_CUDA_CHECK(cudaMemcpyAsync(probs_h + p0 * n, score_out_.ptr, nb * n * sizeof(float), cudaMemcpyDeviceToHost, stream()));
    CT2_CUDA_CHECK(cudaStreamSynchronize(stream()));
  }
}

}  // namespace ct2b200
