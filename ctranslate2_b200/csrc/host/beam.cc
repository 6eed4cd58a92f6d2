// beam.cc — see beam.h.
#include "beam.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>
#include <numeric>
#include <random>

namespace ct2b200 {

BeamSearchArena::BeamSearchArena() {
  end_ids.alloc(64 * sizeof(int32_t));
  counters.alloc(64);
  rng.alloc(2 * sizeof(uint32_t));
  CT2_CUDA_CHECK(cudaMemset(counters.ptr, 0, 64));
  CT2_CUDA_CHECK(cudaDeviceSynchronize());   // legacy-stream memset vs the engine's non-blocking stream
}

BeamSearchArena::~BeamSearchArena() {
  if (host) cudaFreeHost(host);
}

bool BeamSearchArena::ensure(int64_t batch, int beam, int64_t steps, size_t es) {
  if (batch <= cap_batch && beam <= cap_beam && steps <= cap_steps) return false;
  cap_batch = std::max(cap_batch, batch);
  cap_beam = std::max(cap_beam, beam);
  cap_steps = std::max(cap_steps, steps);
  const int64_t B = cap_batch, L = cap_steps, N = B * cap_beam, maxh = max_hyp();
  cum.alloc(N * es);
  cand_scores.alloc(N * 2 * cap_beam * es);        // [B, 2 beam] (entry candidates) or [B * beam, 2 beam] (row candidates)
  cand_ids.alloc(N * 2 * cap_beam * 4);
  next_ids.alloc(N * 4);
  parent.alloc(N * 4);
  finished.alloc(B * 4);
  top_done.alloc(B * 4);
  num_hyp.alloc(B * 4);
  alive.alloc(2 * N * L * 4);
  anc.alloc(2 * N * L * 4);
  CT2_CUDA_CHECK(cudaMemset(anc.ptr, 0, anc.bytes));
  CT2_CUDA_CHECK(cudaDeviceSynchronize());   // legacy-stream memset vs the engine's non-blocking stream
  hyp_tokens.alloc(B * maxh * L * 4);
  hyp_len.alloc(B * maxh * 4);
  hyp_score.alloc(B * maxh * 4);
  sample_ids.alloc(N * 4);
  sample_logp.alloc(N * 4);
  row_score.alloc(N * 4);
  row_done.alloc(N * 4);
  const size_t need = static_cast<size_t>(B) * maxh * (L + 2) + B + 64;
  if (need > host_elems) {
    if (host) cudaFreeHost(host);
    CT2_CUDA_CHECK(cudaMallocHost(&host, need * sizeof(int32_t)));
    host_elems = need;
  }
  return true;
}

BeamState BeamSearchArena::state(int64_t batch, int beam, int64_t vocab, int64_t max_steps, int64_t min_length, float patience,
                                 float length_penalty, int num_hypotheses, int num_end) const {
  BeamState bs;
  bs.batch = static_cast<int>(batch);
  bs.beam = beam;
  bs.vocab = static_cast<int>(vocab);
  bs.vocab_ld = vocab;
  bs.stride = static_cast<int>(cap_steps);
  bs.max_steps = static_cast<int>(max_steps);
  bs.max_hyp = static_cast<int>(max_hyp());
  bs.min_length = static_cast<int>(min_length);
  bs.max_candidates = std::max(1, static_cast<int>(std::lround(beam * patience)));   // decoding.cc:415-418
  bs.num_hypotheses = num_hypotheses;
  bs.early_exit = length_penalty == 0.f ? 1 : 0;
  bs.num_end = num_end;
  bs.end_ids = end_ids.as<int32_t>();
  bs.step = counters.as<int32_t>();
  bs.ticket = bs.step + 1;
  bs.num_finished = bs.step + 2;
  bs.finished = finished.as<int32_t>();
  bs.top_done = top_done.as<int32_t>();
  bs.num_hyp = num_hyp.as<int32_t>();
  bs.alive = alive.as<int32_t>();
  bs.anc = anc.as<int32_t>();
  bs.next_ids = next_ids.as<int32_t>();
  bs.parent = parent.as<int32_t>();
  bs.hyp_tokens = hyp_tokens.as<int32_t>();
  bs.hyp_len = hyp_len.as<int32_t>();
  bs.hyp_score = hyp_score.as<float>();
  return bs;
}

bool BeamSearchArena::ensure_processors(size_t elems) {
  if (elems * 4 <= processors.bytes) return false;
  processors.alloc(std::max<size_t>(elems, 256) * 4);
  return true;
}

void BeamSearchArena::set_processors(BeamState& bs, float repetition_penalty, int no_repeat_ngram_size,
                                     const std::vector<int32_t>& disable_ids, const std::vector<int32_t>& sequence_offsets,
                                     const std::vector<int32_t>& sequence_ids, cudaStream_t st) {
  bs.rep_penalty = repetition_penalty != 1.f ? repetition_penalty : 0.f;
  bs.no_repeat_ngram = no_repeat_ngram_size;
  std::vector<int32_t> table(disable_ids);
  table.insert(table.end(), sequence_offsets.begin(), sequence_offsets.end());
  table.insert(table.end(), sequence_ids.begin(), sequence_ids.end());
  if (table.empty()) return;
  CT2_REQUIRE(table.size() * 4 <= processors.bytes, "set_processors: the table buffer was not grown");
  // pageable source: the call returns once the table is staged, so the vector may go
  CT2_CUDA_CHECK(cudaMemcpyAsync(processors.ptr, table.data(), table.size() * 4, cudaMemcpyHostToDevice, st));
  const int32_t* d = processors.as<int32_t>();
  bs.num_disable = static_cast<int>(disable_ids.size());
  bs.disable_ids = d;
  if (!sequence_offsets.empty()) {
    bs.num_sequences = static_cast<int>(sequence_offsets.size()) - 1;
    bs.seq_offsets = d + disable_ids.size();
    bs.seq_ids = bs.seq_offsets + sequence_offsets.size();
  }
}

bool BeamSearchArena::ensure_attention(int64_t src_len, int heads) {
  const int64_t N = cap_batch * cap_beam, hyps = cap_batch * max_hyp();
  if (N <= attn_rows && cap_steps <= attn_steps && src_len <= attn_src && heads <= attn_heads && hyps <= attn_hyps) return false;
  attn_rows = std::max(attn_rows, N);
  attn_steps = std::max(attn_steps, cap_steps);
  attn_src = std::max(attn_src, src_len);
  attn_heads = std::max<int64_t>(attn_heads, heads);
  attn_hyps = std::max(attn_hyps, hyps);
  attn_probs.alloc(attn_rows * attn_heads * attn_src * 4);
  attn_hist.alloc(attn_rows * attn_steps * attn_src * 4);
  hyp_anc.alloc(attn_hyps * attn_steps * 4);
  attn_cov.alloc(attn_hyps * 4);
  attn_sel.alloc(attn_hyps * 4);
  return true;
}

void BeamSearchArena::reset(const BeamState& bs, int32_t start_id, int dtype, cudaStream_t st) {
  CT2_CUDA_CHECK(cudaMemsetAsync(counters.ptr, 0, 64, st));
  CT2_CUDA_CHECK(cudaMemsetAsync(finished.ptr, 0, bs.batch * 4, st));
  CT2_CUDA_CHECK(cudaMemsetAsync(top_done.ptr, 0, bs.batch * 4, st));
  CT2_CUDA_CHECK(cudaMemsetAsync(num_hyp.ptr, 0, bs.batch * 4, st));
  launch_beam_init(cum.ptr, next_ids.as<int32_t>(), static_cast<int64_t>(bs.batch) * bs.beam, bs.beam, start_id, dtype, st);
}

void BeamSearchArena::step(void* logits, const BeamState& bs, int dtype, cudaStream_t st) {
  if (bs.beam <= 8) {                              // one pass over the logits, nothing written back
    launch_beam_rows(logits, cum.ptr, bs, cand_scores.ptr, cand_ids.as<int32_t>(), dtype, st);
    launch_beam_update(bs, cand_scores.ptr, cand_ids.as<int32_t>(), cum.ptr, true, dtype, st);
    return;
  }
  CT2_REQUIRE(bs.vocab_ld == bs.vocab, "beam search with beam_size > 8 needs contiguous logits rows");
  launch_beam_logprobs(logits, cum.ptr, bs, dtype, st);
  launch_topk(logits, bs.batch, static_cast<int64_t>(bs.beam) * bs.vocab, 2 * bs.beam, cand_scores.ptr, cand_ids.as<int32_t>(), dtype,
              st);
  launch_beam_update(bs, cand_scores.ptr, cand_ids.as<int32_t>(), cum.ptr, false, dtype, st);
}

void BeamSearchArena::reset_sampling(BeamState& bs, int topk, float temperature, cudaStream_t st) {
  bs.sample_topk = topk;
  bs.sample_temperature = temperature;
  bs.rng = rng.as<uint32_t>();
  bs.sample_ids = sample_ids.as<int32_t>();
  bs.sample_logp = sample_logp.as<float>();
  bs.row_score = row_score.as<float>();
  bs.row_done = row_done.as<int32_t>();
  const int64_t N = static_cast<int64_t>(bs.batch) * bs.beam;
  CT2_CUDA_CHECK(cudaMemsetAsync(row_score.ptr, 0, N * 4, st));
  CT2_CUDA_CHECK(cudaMemsetAsync(row_done.ptr, 0, N * 4, st));
  const SamplingCall c = next_sampling_call();
  int32_t words[2];
  std::memcpy(words, &c, sizeof(words));
  launch_fill_i32(rng.as<int32_t>(), 1, words[0], st);
  launch_fill_i32(rng.as<int32_t>() + 1, 1, words[1], st);
}

void BeamSearchArena::sample_step(void* logits, const BeamState& bs, int dtype, cudaStream_t st) {
  launch_beam_sample(logits, bs, dtype, st);
  launch_beam_sample_update(bs, st);
}

// finalize_result (decoding.cc:189-254): normalise by length^penalty, sort (stable: equal scores keep registration order), keep
// num_hypotheses, strip `strip_ids` from the tail
// (decoding.cc:189-254), and finalize_hypothesis_score's coverage penalty (:176-203) when asked
std::vector<TranslationHypotheses> BeamSearchArena::collect(const BeamState& bs, float length_penalty, int num_hypotheses,
                                                            const std::vector<int32_t>& strip_ids, cudaStream_t st,
                                                            float coverage_penalty, int S, float* attention, int64_t max_len) {
  const int64_t B = bs.batch, maxh = bs.max_hyp, stride = bs.stride;
  CT2_REQUIRE((coverage_penalty == 0.f && !attention) || bs.hyp_anc, "collect: the search kept no attention");
  std::vector<float> cov;
  if (coverage_penalty != 0.f) {
    cov.resize(B * maxh);
    launch_hyp_coverage(bs, attn_hist.as<float>(), S, attn_cov.as<float>(), st);
    CT2_CUDA_CHECK(cudaMemcpyAsync(cov.data(), attn_cov.ptr, B * maxh * 4, cudaMemcpyDeviceToHost, st));
  }
  int32_t* h_nh = host;
  int32_t* h_len = h_nh + B;
  float* h_score = reinterpret_cast<float*>(h_len + B * maxh);
  int32_t* h_tok = h_len + 2 * B * maxh;
  CT2_CUDA_CHECK(cudaMemcpyAsync(h_nh, num_hyp.ptr, B * 4, cudaMemcpyDeviceToHost, st));
  CT2_CUDA_CHECK(cudaMemcpyAsync(h_len, hyp_len.ptr, B * maxh * 4, cudaMemcpyDeviceToHost, st));
  CT2_CUDA_CHECK(cudaMemcpyAsync(h_score, hyp_score.ptr, B * maxh * 4, cudaMemcpyDeviceToHost, st));
  CT2_CUDA_CHECK(cudaMemcpyAsync(h_tok, hyp_tokens.ptr, B * maxh * stride * 4, cudaMemcpyDeviceToHost, st));
  CT2_CUDA_CHECK(cudaStreamSynchronize(st));
  std::vector<TranslationHypotheses> out(B);
  std::vector<int32_t> sel(attention ? B * num_hypotheses : 0, -1);   // the returned slots, best first
  for (int64_t b = 0; b < B; ++b) {
    const int nh = h_nh[b];
    std::vector<float> sc(nh);
    for (int j = 0; j < nh; ++j) {
      const float len = static_cast<float>(h_len[b * maxh + j]);
      sc[j] = h_score[b * maxh + j] / std::pow(len, length_penalty);
      if (coverage_penalty != 0.f) sc[j] += coverage_penalty * cov[b * maxh + j];
    }
    std::vector<int> order(nh);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int a, int c) { return sc[a] > sc[c]; });
    if (static_cast<int>(order.size()) > num_hypotheses) order.resize(num_hypotheses);
    for (size_t k = 0; k < order.size() && attention; ++k) sel[b * num_hypotheses + k] = order[k];
    for (int j : order) {
      const int32_t* t = h_tok + (b * maxh + j) * stride;
      std::vector<int32_t> toks(t, t + h_len[b * maxh + j]);
      while (!toks.empty() && std::find(strip_ids.begin(), strip_ids.end(), toks.back()) != strip_ids.end()) toks.pop_back();
      out[b].tokens.push_back(std::move(toks));
      out[b].scores.push_back(sc[j]);
    }
  }
  if (attention) {
    const size_t bytes = static_cast<size_t>(B) * num_hypotheses * max_len * S * 4;
    if (bytes > attn_out.bytes) attn_out.alloc(bytes);
    CT2_CUDA_CHECK(cudaMemcpyAsync(attn_sel.ptr, sel.data(), sel.size() * 4, cudaMemcpyHostToDevice, st));
    launch_hyp_attention_gather(bs, attn_hist.as<float>(), S, attn_sel.as<int32_t>(), num_hypotheses, static_cast<int>(max_len),
                                attn_out.as<float>(), st);
    CT2_CUDA_CHECK(cudaMemcpyAsync(attention, attn_out.ptr, bytes, cudaMemcpyDeviceToHost, st));
    CT2_CUDA_CHECK(cudaStreamSynchronize(st));
    // the rows of stripped end tokens go with them (sequence_to_sequence.cc:383-391)
    for (int64_t b = 0; b < B; ++b)
      for (size_t k = 0; k < out[b].tokens.size(); ++k) {
        const int32_t j = sel[b * num_hypotheses + k];
        const int64_t kept = static_cast<int64_t>(out[b].tokens[k].size()), len = std::min<int64_t>(h_len[b * maxh + j], max_len);
        if (len > kept)
          std::memset(attention + ((b * num_hypotheses + static_cast<int64_t>(k)) * max_len + kept) * S, 0, (len - kept) * S * 4);
      }
  }
  return out;
}

namespace {
std::mutex g_rng_mu;
bool g_rng_seeded = false;
SamplingCall g_rng{0, 0};
}  // namespace

void set_random_seed(uint32_t seed) {
  std::lock_guard<std::mutex> lock(g_rng_mu);
  g_rng = SamplingCall{seed, 0};
  g_rng_seeded = true;
}

SamplingCall next_sampling_call() {
  std::lock_guard<std::mutex> lock(g_rng_mu);
  if (!g_rng_seeded) {
    g_rng = SamplingCall{std::random_device{}(), 0};
    g_rng_seeded = true;
  }
  return SamplingCall{g_rng.seed, g_rng.call++};
}

}  // namespace ct2b200
