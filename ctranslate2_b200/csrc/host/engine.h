// engine.h — C++ host side above the kernels: model loading (models::Model::load), the Llama-class
// decoder driver (layers::TransformerDecoder), greedy search (GreedySearch::search) and the
// Generator entry points.  Names mirror the reference classes they stand for; every device
// operation goes through the launchers of kernels/*.cu on one CUDA stream.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../common.cuh"
#include "../kernels/kernels.h"

namespace ct2b200 {

// ---- model.bin (reference src/models/model.cc:561-660, writer model_spec.py:382-414) ----
struct HostVariable {
  std::vector<int64_t> shape;
  int type_id = 0;               // DataType enum order: f32, i8, i16, i32, f16, bf16 (include/ctranslate2/types.h)
  const uint8_t* data = nullptr; // points into the mapped file
  size_t nbytes = 0;
  int64_t size() const {
    int64_t n = 1;
    for (auto d : shape) n *= d;
    return n;
  }
  double scalar() const;         // value of a rank-0 attribute variable
};

class ModelFile {
 public:
  explicit ModelFile(const std::string& model_dir);
  ~ModelFile();
  const HostVariable* find(const std::string& name) const;
  const HostVariable& get(const std::string& name) const;
  double attribute(const std::string& name, double fallback) const;
  double config_number(const std::string& key, double fallback) const;   // config.json scalar
  std::string spec_name;
  uint32_t binary_version = 0, revision = 0;

 private:
  std::map<std::string, HostVariable> vars_;
  std::string config_json_;
  void* map_ = nullptr;
  size_t map_size_ = 0;
};

// ---- device tensors ----
struct DeviceBuffer {
  void* ptr = nullptr;
  size_t bytes = 0;
  DeviceBuffer() = default;
  explicit DeviceBuffer(size_t n) { alloc(n); }
  DeviceBuffer(const DeviceBuffer&) = delete;
  DeviceBuffer& operator=(const DeviceBuffer&) = delete;
  DeviceBuffer(DeviceBuffer&& o) noexcept : ptr(o.ptr), bytes(o.bytes) { o.ptr = nullptr; o.bytes = 0; }
  DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
    if (this != &o) { release(); ptr = o.ptr; bytes = o.bytes; o.ptr = nullptr; o.bytes = 0; }
    return *this;
  }
  ~DeviceBuffer() { release(); }
  void alloc(size_t n);
  void release();
  template <typename U> U* as() const { return static_cast<U*>(ptr); }
};

// layers::Dense weights (reference src/layers/common.cc:266-303)
struct DenseWeights {
  enum Kind { INT8, FLOAT16, AWQ_GEMM, AWQ_GEMV } kind = INT8;
  int64_t n = 0, k = 0;
  DeviceBuffer weight;          // int8 [n,k] | T [n,k] | packed int32
  DeviceBuffer scale;           // f32 [n] (INT8) | f16 scales (AWQ)
  DeviceBuffer zeros;           // AWQ qzeros
  DeviceBuffer scale_zero;      // AWQ: {scale, zero} pairs in group-major order [k/group, n] (awq_decode.cu)
  DeviceBuffer bias;            // T [n] or empty
  int group_size = 128;
};

// A decoding step captured once as a CUDA graph and replayed.  `key` holds everything the capture bakes in (kernel arguments
// are values): capture() with another key captures again.  Captured launches are counted when the graph is replayed, not
// when it is captured.
struct StepGraph {
  cudaGraphExec_t exec = nullptr;
  int64_t nodes = 0;
  std::vector<int64_t> key;
  StepGraph() = default;
  StepGraph(const StepGraph&) = delete;
  StepGraph& operator=(const StepGraph&) = delete;
  ~StepGraph() { reset(); }
  void reset();
  void capture(cudaStream_t st, const std::vector<int64_t>& key, const std::function<void()>& step);   // unless `key` is held
  void launch(cudaStream_t st);
};

// CT2B200_EOS_POLL: decoding steps between two looks of the host at the finished entries (default 4, at least 1)
int64_t eos_poll_interval();

// host-side conversion of a float variable to the compute dtype (gammas, biases, position encodings)
std::vector<uint8_t> convert_to_dtype(const HostVariable& v, int dtype);
void upload(DeviceBuffer& dst, const void* src, size_t n);
// convert_to_dtype + upload; returns the bytes uploaded
size_t upload_as(DeviceBuffer& dst, const HostVariable& v, int dtype);

// The device an engine runs on and its stream.  The constructor checks for compute capability 9, reads the SM count and
// creates a non-blocking stream with its split-K workspace (outside any graph capture); the destructor synchronises the
// stream, then releases the workspace and the stream.
struct EngineDevice {
  int device = 0, sm_count = 132;
  cudaStream_t stream = nullptr;
  explicit EngineDevice(int device);
  ~EngineDevice();
  EngineDevice(const EngineDevice&) = delete;
  EngineDevice& operator=(const EngineDevice&) = delete;
};

// how a Dense weight [n, k] is partitioned over the tensor-parallel ranks (models::Model::load, model.cc:662-743):
// column-parallel layers keep a slice of the output rows (fused QKV: this rank's query, key and value heads), row-parallel
// layers (COLS) a slice of K
enum class Shard { REPLICATED, ROWS, QKV_ROWS, COLS };
struct ShardPlan {
  std::vector<std::pair<int64_t, int64_t>> rows;   // output rows [b, e) kept, in order
  int64_t k0 = 0, k1 = 0;                          // input columns [k0, k1) kept
  int64_t n() const;
  int64_t k() const { return k1 - k0; }
};
// The part of a Dense weight [n, k] rank `rank` of `world` keeps (the whole weight for REPLICATED).  QKV_ROWS needs the head
// geometry; `group` > 0 (AWQ) must divide the K slice of a COLS shard.
ShardPlan shard_plan(Shard shard, int64_t n, int64_t k, int heads, int heads_kv, int head_dim, int rank, int world,
                     int64_t group = 0);

// How load_dense reads a Dense layer: the compute type and the weight type it asks for, the tensor-parallel shard, and
// whether AWQ-INT4 weights are accepted (otherwise they are refused as an unsupported weight type).
struct DenseLoad {
  int dtype = CT2B200_F16;
  int weight_type = CT2B200_WEIGHTS_STORED;
  cudaStream_t stream = nullptr;
  Shard shard = Shard::REPLICATED;
  int heads = 0, heads_kv = 0, head_dim = 0;   // QKV_ROWS: the unsharded head geometry
  int rank = 0, world = 1;
  bool awq = false;
};
// layers::Dense weights of `prefix`, converted on the GPU to what the compute type asks for (Model::set_compute_type) and cut
// to this rank's shard; returns the bytes of weight, scales and zeros (the bias is not counted)
int64_t load_dense(const ModelFile& f, const std::string& prefix, const DenseLoad& opt, DenseWeights& w);

AwqNative awq_view(const DenseWeights& w);
// [RMSNorm (gamma non-null) +] Quantize of m rows of k T values into xq / xs
void rows_to_int8(const void* x, const void* gamma, float eps, int64_t m, int64_t k, int dtype, int8_t* xq, float* xs,
                  cudaStream_t st);
// layers::Dense::operator() (src/layers/common.cc:339-442) on prepared inputs: INT8 weights read Quantize(x) from xq / xs,
// float and AWQ weights the T rows x (AWQ: awq_scratch as dense_awq's scratch_nk).  INT8 writes rows of stride ldy
// (0 = w.n); the float and AWQ arms write contiguous rows only.
void dense_forward(const DenseWeights& w, const int8_t* xq, const float* xs, const void* x, int64_t m, const void* residual,
                   int act, void* y, int64_t ldy, int dtype, int gemm_impl, void* awq_scratch, cudaStream_t st);

struct LayerWeights {
  DeviceBuffer attn_gamma, ffn_gamma;
  DenseWeights qkv, out, gate, up, down;
};

struct ModelConfig {
  int num_layers = 0, num_heads = 0, num_heads_kv = 0, head_dim = 0;
  int64_t d_model = 0, ffn_dim = 0, vocab = 0;
  float eps = 1e-6f;
  float rotary_base = 10000.f;
  bool rotary_interleave = true;
  int rotary_scaling_type = -1;
  float rotary_scaling_factor = 1.f, rotary_low_freq = 1.f, rotary_high_freq = 4.f;
  int original_max_positions = 0;
  int activation = CT2B200_ACT_SWISH;
  bool embeddings_int8 = true;
  int64_t weight_bytes = 0;
  std::string float_type;        // stored type of the non-weight float variables (decoder/layer_norm/gamma): what "default" keeps
  std::string weights;           // storage type of the linear layers: int8 | awq_gemm | awq_gemv | float16 | bfloat16 | float32
};

class ModelFile;
ModelConfig parse_model_config(const ModelFile& file);   // host only

// TransformerDecoder for pre-norm / RMSNorm / gated-FFN / rotary decoders (Llama family).
class LlamaDecoder {
 public:
  LlamaDecoder(const ModelFile& file, const ct2b200_generator_config& cfg);
  ~LlamaDecoder();

  const ModelConfig& config() const { return mc_; }
  int dtype() const { return dtype_; }
  cudaStream_t stream() const { return gpu_.stream; }
  int64_t max_batch() const { return max_batch_; }
  int64_t max_length() const { return max_len_; }

  // Forward `time` new tokens per row starting at position `offset` (same for every row, as in the
  // reference: decoder(step, ids, state)).  ids_d [batch, time] int32 on device.  When logits_rows_d is
  // non-null, rows listed there (indices into the flattened [batch*time] rows, `num_logit_rows` of them)
  // are projected to the vocabulary into logits_out_d ([num_logit_rows, vocab] T).
  void forward_prefill(const int32_t* ids_d, int64_t batch, int64_t time, int64_t offset, void* logits_out_d,
                       const int32_t* logits_rows_d, int64_t num_logit_rows);
  // One decode step for `batch` rows: ids_d [batch]; positions lens_d [batch] (device); logits [batch, vocab] T.
  void forward_step(const int32_t* ids_d, const int32_t* lens_d, int64_t batch, void* logits_out_d);

  // project rows (indices into the rows of the last forward_prefill) of the hidden state to the vocabulary
  void project_rows(const int32_t* rows_d, int64_t n, void* logits_out_d);
  // copy rows (indices into the rows of the last forward_prefill) of the hidden state to out_d [n, d_model] T
  void gather_hidden(const int32_t* rows_d, int64_t n, void* out_d);
  // final RMSNorm + lm_head of `rows` hidden rows x_rows_d [rows, d_model] T (at most prefill_chunk_rows()):
  // logits_out_d [rows, vocab] T
  void project_hidden(const void* x_rows_d, int64_t rows, void* logits_out_d);
  void* logits_buffer() const { return logits_.ptr; }       // [max_batch, vocab] T
  // Beam search on the contiguous per-row caches (Decoder::replicate_state / update_state, decoder.cc:33-139): the K/V rows are
  // re-gathered into a second cache set (allocated on first use) and the two sets swap roles.
  // parent_d == null: row r takes the first `positions` cached positions of row r / beam (replicate after the prompt pass);
  // otherwise of row parent_d[r] (reorder after a search step).
  void reorder_cache(const int32_t* parent_d, int beam, int64_t rows, int64_t positions);
  // after a beam search: the primary cache set is the one captured CUDA graphs point to (contents are dead by then)
  void restore_cache_orientation();
  // tensor parallel bootstrap (one process per GPU): this rank's exchange buffer as a cudaIpcMemHandle (64 bytes),
  // then the handles of all ranks in rank order
  int tp_size() const { return tp_.world; }
  void tp_handle(void* handle64) const;
  void tp_connect(const void* handles, int count);
  int64_t prefill_chunk_rows() const { return chunk_rows_; }
  void set_gemm_impl(int impl) { gemm_impl_ = impl; }

 private:
  void layers_forward_tp(int64_t rows, int64_t batch, int64_t time, int64_t offset, const int32_t* lens_d);
  void dense(const DenseWeights& w, const int8_t* xq, const float* xs, const void* x_float, int64_t m,
             const void* residual, int act, void* y);
  // INT8 Dense whose input rows are still in T: [RMSNorm +] Quantize (row kernel) + Dense
  void dense_from_rows(const DenseWeights& w, const void* x_rows, const void* gamma, int64_t cols, int64_t m,
                       const void* residual, int act, void* y);
  void glu_from_rows(const DenseWeights& gate, const DenseWeights& up, const void* x_rows, const void* gamma, int64_t m,
                     void* h);
  void layers_forward(int64_t rows, int64_t batch, int64_t time, int64_t offset, const int32_t* lens_d);
  void project(const void* x_rows, int64_t rows, void* logits_out);
  void embed(const int32_t* ids_d, int64_t rows);

  ModelConfig mc_;            // global (unsharded) geometry
  int heads_ = 0, heads_kv_ = 0;   // heads held by this rank
  int64_t ffn_ = 0;                // FFN columns held by this rank
  struct Tp {
    int rank = 0, world = 1;
    bool connected = false;
    DeviceBuffer exchange;      // flags | amax words | partial buffer 0 | partial buffer 1
    DeviceBuffer tick;
    size_t flags_off = 0, amax_off = 0, part_off[2] = {0, 0};
    void* peer[8] = {};         // mapped exchange buffers (peer[rank] = own)
    TpLink link;
  } tp_;
  int dtype_ = CT2B200_F16;
  int gemm_impl_ = CT2B200_GEMM_AUTO;
  int weight_type_ = CT2B200_WEIGHTS_STORED;
  int64_t max_batch_ = 0, max_len_ = 0, chunk_rows_ = 0;
  int attn_splits_ = 1;

  DenseWeights embeddings_;       // int8 [V,d] + scale, or T [V,d]
  DenseWeights projection_;
  DeviceBuffer final_gamma_;
  std::vector<LayerWeights> layers_;
  DeviceBuffer sin_, cos_;        // f32 [max_len, head_dim]
  std::vector<DeviceBuffer> k_cache_, v_cache_;   // per layer [max_batch, Hkv, max_len, D] T
  std::vector<DeviceBuffer> k_alt_, v_alt_;       // beam search: the other cache set (reorder_cache swaps them)
  bool cache_swapped_ = false;

  // activations (rows = max(chunk_rows, max_batch))
  DeviceBuffer x_, xq_, xs_, qkv_, attn_, h_, logits_, gathered_, attn_ws_;
  DeviceBuffer xn_, scratch_mn_, scratch_nk_;   // float/AWQ arms: normed activations, up-projection, dequantized weight
  // last: it is destroyed first, so the stream is synchronised before any buffer above is freed
  EngineDevice gpu_;
};

struct TranslationHypotheses;
struct GenerationRequest {
  const int32_t* prompt_ids = nullptr;     // host [batch, max_prompt_len]
  const int32_t* prompt_lens = nullptr;    // host [batch]
  int64_t batch = 0, max_prompt_len = 0, max_length = 0, min_length = 0;
  std::vector<int32_t> end_ids;
  bool return_end_token = false;
  bool return_scores = false;              // GenerationOptions::return_scores
  float length_penalty = 1.f;              // score / length^length_penalty (decoding.cc:189-203)
  int beam_size = 1;                       // > 1: BeamSearch::search (generate_beam)
  float patience = 1.f;
  int num_hypotheses = 1;
};

class Generator {
 public:
  Generator(const std::string& model_dir, const ct2b200_generator_config& cfg);
  ~Generator();
  LlamaDecoder& decoder() { return *decoder_; }
  // Generator::generate_batch (greedy): fills out_ids [batch, max_length] (-1 padded) and out_lens.
  void generate(const GenerationRequest& req, int32_t* out_ids, int32_t* out_lens, float* out_scores = nullptr);
  // Generator::generate_batch with beam_size > 1 (decoding.cc:425-720; prompt pass language_model.cc:217-238): prompts of equal
  // length; per entry the best num_hypotheses hypotheses (end token stripped unless return_end_token) and their scores
  std::vector<TranslationHypotheses> generate_beam(const GenerationRequest& req);
  // Generator::forward_batch
  void forward(const int32_t* ids_h, int64_t batch, int64_t time, bool log_probs, float* logits_h);
  // Generator::score_batch (src/scoring.cc:6-66): ids_h [batch, max_len] right-padded with valid ids, lens_h [batch] the
  // sequence lengths.  out_h [batch, max_len - 1]: row b holds log P(ids[b][t + 1] | ids[b][..t]) for
  // offset <= t < lens_h[b] - 1 at column t - offset, then zeros.
  void score(const int32_t* ids_h, const int32_t* lens_h, int64_t batch, int64_t max_len, int64_t offset, float* out_h);
  void bench_decode(int64_t batch, int64_t prompt_len, int64_t steps, int64_t warmup, float* prefill_ms,
                    float* decode_ms, int64_t* launches);
  void bench_last_logits(int64_t batch, float* logits_h, int64_t logits_len);

 private:
  // the prompt pass from position 0 in time chunks that fit the activation arena; after_chunk(t0, tc) runs once the hidden
  // state of positions [t0, t0 + tc) is complete, before the next chunk overwrites it
  void run_prefill(const int32_t* ids_d, int64_t batch, int64_t time,
                   const std::function<void(int64_t t0, int64_t tc)>& after_chunk = nullptr);
  void launch_step(int64_t batch);

  ct2b200_generator_config cfg_;
  std::mutex mu_;                          // generate / forward / bench_decode are serialised per generator
  std::unique_ptr<LlamaDecoder> decoder_;
  // decode-loop device state
  DeviceBuffer ids_d_, lens_d_, step_d_, forced_d_, out_d_, end_ids_d_, prompt_d_, sample_ws_, scores_d_, row_start_d_;
  DeviceBuffer attn_lens_d_, finished_d_;    // per row: cache length the attention kernel sees (0 once finished), finished flag
  bool want_scores_ = false;               // the step (and its CUDA graph) also writes per-step log-probabilities
  int32_t* host_pinned_ = nullptr;
  size_t host_pinned_elems_ = 0;
  std::unique_ptr<struct BeamSearchArena> beam_;   // created by the first beam search
  // score_batch, allocated by the first call: lm_head slab (logits [slab_rows, vocab] T | hidden rows [slab_rows, d_model] T),
  // per scored position its hidden-state row and target id (int32 [2, max_batch * max_length]), and its log-probability
  DeviceBuffer score_slab_, score_idx_d_, score_out_d_;
  int64_t score_slab_rows_ = 0;
  int32_t* score_pinned_ = nullptr;        // host staging of the row / target ids (pinned: the copies stay asynchronous)
  StepGraph graph_;                        // key: {batch, want_scores_}
};

}  // namespace ct2b200
