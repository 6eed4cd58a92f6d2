// beam.h — device-resident state of BeamSearch::search (src/decoding.cc:425-720) shared by the encoder-decoder engine
// (translator.cc) and the decoder-only Generator (engine.cc): buffers, the three kernels of a search step and
// finalize_result (decoding.cc:189-254) on the host.  The kernels live in kernels/seq2seq.cu.
#pragma once

#include <cstdint>
#include <vector>

#include "engine.h"

namespace ct2b200 {

struct TranslationHypotheses {            // per batch entry, best first
  std::vector<std::vector<int32_t>> tokens;
  std::vector<float> scores;
};

struct BeamSearchArena {
  int64_t cap_batch = 0, cap_steps = 0;
  int cap_beam = 0;
  DeviceBuffer cum, cand_scores, cand_ids, next_ids, end_ids, counters, finished, top_done, num_hyp, alive, anc, parent;
  DeviceBuffer hyp_tokens, hyp_len, hyp_score;
  DeviceBuffer rng, sample_ids, sample_logp, row_score, row_done;   // sampled search
  DeviceBuffer processors;                // logits processors: [disabled ids | sequence offsets | sequence ids] int32
  // the alignment attention, allocated by the first search that asks for it (return_attention, coverage_penalty): a step's
  // per-head probabilities [N, heads, S] f32, the history [N, steps, S] f32 (row n, absolute position, source position),
  // the hypotheses' ancestry [batch, max_hyp, steps]; at collect, the coverage terms [batch, max_hyp], the returned slots and
  // their gathered rows
  DeviceBuffer attn_probs, attn_hist, hyp_anc, attn_cov, attn_sel, attn_out;
  int64_t attn_rows = 0, attn_steps = 0, attn_src = 0, attn_heads = 0, attn_hyps = 0;
  int32_t* host = nullptr;                // pinned staging of the results
  size_t host_elems = 0;

  BeamSearchArena();
  ~BeamSearchArena();
  BeamSearchArena(const BeamSearchArena&) = delete;
  BeamSearchArena& operator=(const BeamSearchArena&) = delete;

  int64_t max_hyp() const { return 3 * static_cast<int64_t>(cap_beam); }   // round(beam * patience) + beam, patience <= 2
  // grows the buffers; true when something was reallocated (captured graphs over them are stale then)
  bool ensure(int64_t batch, int beam, int64_t steps, size_t elem_size);
  BeamState state(int64_t batch, int beam, int64_t vocab, int64_t max_steps, int64_t min_length, float patience,
                  float length_penalty, int num_hypotheses, int num_end) const;
  // grows `processors` to `elems` ids; true when it was reallocated (captured graphs over it are stale then)
  bool ensure_processors(size_t elems);
  // the history-dependent logits processors of a search (decoding_utils.cc:40-150): penalty 1 and n-gram size 0 are off;
  // disable_ids are disabled at every step (SuppressTokens); sequence s is sequence_ids[sequence_offsets[s] ..
  // sequence_offsets[s + 1]) (SuppressSequences; no offsets = none).  Uploads the tables on st into `processors`, which
  // ensure_processors has sized, and points bs at them.
  void set_processors(BeamState& bs, float repetition_penalty, int no_repeat_ngram_size, const std::vector<int32_t>& disable_ids,
                      const std::vector<int32_t>& sequence_offsets, const std::vector<int32_t>& sequence_ids, cudaStream_t st);
  // grows the attention buffers to the arena's capacities, `src_len` source positions and `heads` alignment heads; true when
  // something was reallocated (captured graphs over them are stale then)
  bool ensure_attention(int64_t src_len, int heads);
  // clears the counters / flags and starts every beam from start_id (beam 0 live, the others at the lowest score)
  void reset(const BeamState& bs, int32_t start_id, int dtype, cudaStream_t st);
  // one search step over logits [batch * beam, vocab] T (modified in place): log-probabilities + cumulative scores,
  // TopK of 2 * beam candidates per entry, bookkeeping; next_ids / cum / parent / histories are updated on the device
  void step(void* logits, const BeamState& bs, int dtype, cudaStream_t st);
  // sampled search (GreedySearch with a RandomSampler): turns bs into a sampled state and clears the row scores; the rows of
  // this call draw from (seed, call) of next_sampling_call()
  void reset_sampling(BeamState& bs, int topk, float temperature, cudaStream_t st);
  // one sampled step over logits [batch * beam, vocab] T (modified in place)
  void sample_step(void* logits, const BeamState& bs, int dtype, cudaStream_t st);
  // finalize_result; with bs.hyp_anc set (a search that kept the attention history of S source positions): coverage_penalty
  // adds beta * the coverage term before the sort, and attention (host, or null) gets [batch, num_hypotheses, max_len, S] f32,
  // the rows of the returned hypotheses (one per returned token), zeros past them
  std::vector<TranslationHypotheses> collect(const BeamState& bs, float length_penalty, int num_hypotheses,
                                             const std::vector<int32_t>& strip_ids, cudaStream_t st, float coverage_penalty = 0.f,
                                             int S = 0, float* attention = nullptr, int64_t max_len = 0);
};

// The process-wide random state of sampling (set_random_seed, src/random.cc): a seed, drawn once from std::random_device
// unless set, and the index of the next sampling call, which every sampled search advances and set_random_seed resets.
void set_random_seed(uint32_t seed);
struct SamplingCall {
  uint32_t seed, call;
};
SamplingCall next_sampling_call();

}  // namespace ct2b200
