// seq2seq.cu — kernels of the encoder-decoder path (ctranslate2::Translator, SURVEY §8 f1): embeddings with scale and
// position encodings, LayerNorm (+ Quantize), a head_dim-agnostic attention (encoder self-attention with padding mask,
// single-token decoder self-attention over a beam-REMAPPED cache, cross-attention over the memory keys / values of the
// batch entry), and the device side of BeamSearch::search: log-softmax + cumulative scores, candidate bookkeeping,
// hypothesis registration and the beam reindex as an index remap (no K/V bytes move when beams are reordered).
// Reference kernels / functions these replace are cited per kernel (paths relative to the reference tree).
#include <algorithm>
#include <cfloat>
#include <type_traits>

#include "../common.cuh"
#include "beam_decide.h"
#include "kernels.h"
#include "philox.h"
#include "sample_row.cuh"

namespace ct2b200 {

namespace {

template <typename T> __device__ __forceinline__ float lowest_of();
template <> __device__ __forceinline__ float lowest_of<float>() { return -FLT_MAX; }
template <> __device__ __forceinline__ float lowest_of<__half>() { return -65504.f; }
template <> __device__ __forceinline__ float lowest_of<__nv_bfloat16>() { return -3.3895313892515355e38f; }

// ---------------------------------------------------------------------------------------------
// layers::Embeddings (+ int8 dequantization, common.cc:64-81) * embeddings scale (transformer.cc:382-402, ops::Mul in T)
// + PositionEncoder (common.cc:170-229, ops::Add in T).  Row r of [batch, time]: position = r % time, or *step_ptr for the
// single-token decoder step (device-resident so that the step is CUDA-graph capturable).  w2 (optional): a second table
// (token types) looked up with ids2 and merged by ADD in T before the scale (ParallelEmbeddings, common.cc:116-148).
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void embed_pos_kernel(const void* __restrict__ w, const float* __restrict__ w_scale, const int32_t* __restrict__ ids,
                                 int64_t depth, float emb_scale, const T* __restrict__ pos, int64_t time,
                                 const int32_t* __restrict__ step_ptr, bool zero_first, T* __restrict__ y,
                                 const void* __restrict__ w2, const float* __restrict__ w2_scale,
                                 const int32_t* __restrict__ ids2) {
  griddep_launch();
  griddep_wait();
  const int64_t r = blockIdx.x;
  const int64_t id = ids[r];
  const int64_t t = step_ptr ? static_cast<int64_t>(*step_ptr) : (r % time);
  const float es = round_to<T>(emb_scale);
  const bool zero = zero_first && t == 0;      // start_from_zero_embedding (transformer.cc:637-640): no token at step 0
  for (int64_t j = threadIdx.x; j < depth; j += blockDim.x) {
    float v;
    if (zero) v = 0.f;
    else if (w_scale) v = round_to<T>(__fdiv_rn(static_cast<float>(static_cast<const int8_t*>(w)[id * depth + j]), w_scale[id]));
    else v = to_f32(static_cast<const T*>(w)[id * depth + j]);
    if (w2) {
      const int64_t id2 = ids2[r];
      const float v2 = w2_scale ? round_to<T>(__fdiv_rn(static_cast<float>(static_cast<const int8_t*>(w2)[id2 * depth + j]), w2_scale[id2]))
                                : to_f32(static_cast<const T*>(w2)[id2 * depth + j]);
      v = round_to<T>(v2 + v);
    }
    if (emb_scale != 0.f && !zero) v = round_to<T>(v * es);
    if (pos) v = round_to<T>(v + to_f32(pos[t * depth + j]));
    y[r * depth + j] = from_f32<T>(v);
  }
}

// ---------------------------------------------------------------------------------------------
// ops::LayerNorm (src/ops/layer_norm_gpu.cu:169-206): mean = sum/n, var = max(sum(x^2)/n - mean^2, 0),
// y = T((x - mean) * rsqrt(var + eps) * gamma + beta); optionally followed by ops::Quantize of T(y) (quantize_gpu.cu:57-105;
// `round` = false reproduces models of binary version < 5, model.h:87-89).  y and (q, scale) may both be requested.
// ---------------------------------------------------------------------------------------------
// Rows of at most 8 * 256 elements: every thread keeps its (up to NV) elements and their normalised values in registers — one
// read of x, gamma and beta instead of four, same arithmetic and rounding points as the general kernel below.
template <typename T, int NV>
__global__ void __launch_bounds__(256) layer_norm_small_kernel(const T* __restrict__ x, const T* __restrict__ gamma,
                                                               const T* __restrict__ beta, int64_t cols, float eps,
                                                               T* __restrict__ y, int8_t* __restrict__ q, float* __restrict__ scale,
                                                               bool round) {
  __shared__ float red[32];
  griddep_launch();
  griddep_wait();
  const int64_t row = blockIdx.x;
  const T* xr = x + row * cols;
  float v[NV];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int64_t j = threadIdx.x + static_cast<int64_t>(i) * 256;
    v[i] = j < cols ? to_f32(xr[j]) : 0.f;
    s1 += v[i];
    s2 += v[i] * v[i];
  }
  s1 = block_reduce<false>(s1, red);
  s2 = block_reduce<false>(s2, red);
  const float inv_n = 1.f / static_cast<float>(cols);
  const float mean = s1 * inv_n;
  const float rstd = rsqrtf(fmaxf(s2 * inv_n - mean * mean, 0.f) + eps);
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int64_t j = threadIdx.x + static_cast<int64_t>(i) * 256;
    if (j < cols) {
      const float g = gamma ? to_f32(gamma[j]) : 1.f, b = beta ? to_f32(beta[j]) : 0.f;
      v[i] = round_to<T>((v[i] - mean) * rstd * g + b);
      amax = fmaxf(amax, fabsf(v[i]));
    }
  }
  if (q) {
    amax = block_reduce<true>(amax, red);
    const float s = amax != 0.f ? 127.f / amax : 1.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int64_t j = threadIdx.x + static_cast<int64_t>(i) * 256;
      if (j < cols) {
        const float w = v[i] * s;
        q[row * cols + j] = static_cast<int8_t>(round ? nearbyintf(w) : w);
      }
    }
    if (threadIdx.x == 0) scale[row] = s;
  }
  if (y) {
    T* yr = y + row * cols;   // y may alias x: every thread rewrites only the elements it read
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int64_t j = threadIdx.x + static_cast<int64_t>(i) * 256;
      if (j < cols) yr[j] = from_f32<T>(v[i]);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256) layer_norm_kernel(const T* __restrict__ x, const T* __restrict__ gamma,
                                                         const T* __restrict__ beta, int64_t cols, float eps,
                                                         T* __restrict__ y, int8_t* __restrict__ q, float* __restrict__ scale,
                                                         bool round) {
  __shared__ float red[32];
  griddep_launch();
  griddep_wait();
  const int64_t row = blockIdx.x;
  const T* xr = x + row * cols;
  float s1 = 0.f, s2 = 0.f;
  for (int64_t j = threadIdx.x; j < cols; j += blockDim.x) {
    const float v = to_f32(xr[j]);
    s1 += v;
    s2 += v * v;
  }
  s1 = block_reduce<false>(s1, red);
  s2 = block_reduce<false>(s2, red);
  const float inv_n = 1.f / static_cast<float>(cols);
  const float mean = s1 * inv_n;
  const float rstd = rsqrtf(fmaxf(s2 * inv_n - mean * mean, 0.f) + eps);
  auto normed = [&](int64_t j) {
    const float g = gamma ? to_f32(gamma[j]) : 1.f, b = beta ? to_f32(beta[j]) : 0.f;
    return round_to<T>((to_f32(xr[j]) - mean) * rstd * g + b);
  };
  if (q) {
    float amax = 0.f;
    for (int64_t j = threadIdx.x; j < cols; j += blockDim.x) amax = fmaxf(amax, fabsf(normed(j)));
    amax = block_reduce<true>(amax, red);
    const float s = amax != 0.f ? 127.f / amax : 1.f;
    for (int64_t j = threadIdx.x; j < cols; j += blockDim.x) {
      const float v = normed(j) * s;
      q[row * cols + j] = static_cast<int8_t>(round ? nearbyintf(v) : v);
    }
    if (threadIdx.x == 0) scale[row] = s;
  }
  if (y) {
    T* yr = y + row * cols;   // y may alias x: every thread rewrites only the elements it read last
    __syncthreads();
    for (int64_t j = threadIdx.x; j < cols; j += blockDim.x) yr[j] = from_f32<T>(normed(j));
  }
}

// ---------------------------------------------------------------------------------------------
// Attention for any head_dim (layers::MultiHeadAttention, attention.cc:178-287 dot_product_attention; the fused
// decode kernels of attention_mma.cu cover head_dim 64 / 128 with rotary positions — this one serves the
// encoder-decoder models: absolute positions, padding masks, beams).  One warp per (query row, head):
//   scores_j = T(scale * q . k_j)  (fp32 accumulate), probs = T(softmax over the valid keys) (fp32), out = T(sum_j p_j v_j).
// MODE 0  encoder self-attention: q, k, v = column blocks of qkv [B*S, 3d]; keys of row (b, t) = rows (b, j), j < lengths[b]
// MODE 1  decoder self-attention of ONE new token per row: the row's k / v (columns d.. / 2d.. of qkv [N, 3d]) are written to
//         the cache [N, max_len, d] at (row, step); key j < step lives in slot anc[row][j] — the beam ancestry table — so
//         reordering beams never copies K/V (Decoder::update_state, decoder.cc:33-55, gathers the whole state instead)
// MODE 2  cross-attention (attention.cc:371-440): q [N, d]; keys / values = column blocks of kv [B*S, 2d] of batch entry
//         row / beam, j < lengths[row / beam] (the beams of an entry share the memory: replicate_state copies it instead)
// MODE 3  decoder self-attention over T teacher-forced positions (the full-sequence decoder call of scoring, decoder.cc:13-26):
//         q, k, v = column blocks of qkv [B*T, 3d]; keys of row (b, t) = rows (b, j), j <= t (the causal mask; positions past
//         a sequence's length are computed and ignored, as in MODE 0); no cache is written
// ---------------------------------------------------------------------------------------------
struct AttnGeneric {
  const void* q;
  int64_t q_stride;
  const void* k;
  const void* v;
  int64_t kv_stride;
  void* out;
  int64_t out_stride;
  const int32_t* lengths;
  const int32_t* anc;        // MODE 1: [2][N, max_len] ancestry tables (read buffer = step & 1)
  const int32_t* step_ptr;   // MODE 1
  void* k_cache;             // MODE 1: [N, max_len, d]
  void* v_cache;
  int64_t rows;              // query rows
  int S;                     // keys per batch entry (MODE 0 / 2), max_len (MODE 1) or positions per sequence (MODE 3)
  int beam;
  int H, D;
  float scale;
  int max_keys;              // capacity of the per-warp score buffer
  bool vec_ok;               // every row start (q, k, v, caches, out) is 16-byte aligned
};

// The extra output of an instantiation and its argument: none (an empty one, so the parameter block keeps its size), the
// pre-softmax scores of selected heads (kCapture: Whisper::align) or the normalised probabilities of the alignment heads
// (kAlign: the attention a Translator returns, launch_attention_cross_align).
enum AttnExtra { kNoExtra = 0, kCapture = 1, kAlign = 2 };
struct NoCapture {};
struct AttnAlign {
  float* probs;              // [rows, heads, S]
  int heads;
};
template <int X>
using ExtraArg = std::conditional_t<X == kCapture, AttnCapture, std::conditional_t<X == kAlign, AttnAlign, NoCapture>>;

constexpr int kAttnWarps = 4;

// DT = head_dim known at compile time (64, 128: the loops over a key / value row unroll, so the 16-byte loads of a row are all
// in flight at once — with a run-time bound they are issued one L2 round trip at a time), 0 = any head_dim.  X = kCapture: also
// write the scores of the heads cap selects (Whisper::align); X = kAlign: also write the probabilities of heads
// [0, cap.heads); the other instantiations compile without either.
template <typename T, int MODE, int DT, int X = kNoExtra>
__global__ void __launch_bounds__(kAttnWarps * 32) attention_generic_kernel(AttnGeneric a, ExtraArg<X> cap) {
  extern __shared__ float smem_f[];
  griddep_launch();
  griddep_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t unit = static_cast<int64_t>(blockIdx.x) * kAttnWarps + warp;
  if (unit >= a.rows * a.H) return;
  const int64_t n = unit / a.H;
  const int h = static_cast<int>(unit % a.H);
  const int D = DT > 0 ? DT : a.D, d_model = a.H * D;
  float* qs = smem_f + static_cast<size_t>(warp) * (a.max_keys + D);
  float* sc = qs + D;
  const T* qrow = static_cast<const T*>(a.q) + n * a.q_stride + h * D;
  for (int i = lane; i < D; i += 32) qs[i] = to_f32(qrow[i]);

  int nkeys;
  int64_t base = 0;          // first key row (MODE 0 / 2 / 3)
  const int32_t* anc = nullptr;
  int step = 0;
  const T* kb = static_cast<const T*>(a.k);
  const T* vb = static_cast<const T*>(a.v);
  if constexpr (MODE == 0) {
    const int64_t b = n / a.S;
    nkeys = a.lengths ? min(a.lengths[b], a.S) : a.S;
    base = b * a.S;
  } else if constexpr (MODE == 3) {
    const int64_t b = n / a.S;
    nkeys = static_cast<int>(n - b * a.S) + 1;
    base = b * a.S;
  } else if constexpr (MODE == 2) {
    const int64_t b = n / a.beam;
    nkeys = a.lengths ? min(a.lengths[b], a.S) : a.S;
    base = b * a.S;
  } else {
    step = *a.step_ptr;
    nkeys = step + 1;
    anc = a.anc + static_cast<int64_t>(step & 1) * a.rows * a.S + n * a.S;
    // append this row's key / value at (row, step)
    T* kc = static_cast<T*>(a.k_cache) + (n * a.S + step) * d_model + h * D;
    T* vc = static_cast<T*>(a.v_cache) + (n * a.S + step) * d_model + h * D;
    const T* knew = static_cast<const T*>(a.q) + n * a.q_stride + d_model + h * D;
    const T* vnew = knew + d_model;
    for (int i = lane; i < D; i += 32) {
      kc[i] = knew[i];
      vc[i] = vnew[i];
    }
    kb = static_cast<const T*>(a.k_cache);
    vb = static_cast<const T*>(a.v_cache);
  }
  __syncwarp();
  auto key_row = [&](int j) -> int64_t {
    if constexpr (MODE == 1) return (j == step ? n : static_cast<int64_t>(anc[j])) * a.S + j;
    else return base + j;
  };
  // 16-byte loads of the key rows / paired loads of the value rows when the layout allows (head_dim 64, 128, ...: every model
  // this kernel serves); the accumulation order over a row is the same in both forms
  constexpr int NV = Vec16<T>::N;
  const bool vec = a.vec_ok && D % NV == 0;
  auto dot_row = [&](const T* kr) {
    float dot = 0.f;
    if (vec) {
      if constexpr (DT > 0) {
        Vec16<T> kk[DT / NV];
#pragma unroll
        for (int c = 0; c < DT / NV; ++c) kk[c] = ld16(kr + c * NV);
#pragma unroll
        for (int c = 0; c < DT / NV; ++c)
#pragma unroll
          for (int i = 0; i < NV; ++i) dot += qs[c * NV + i] * to_f32(kk[c].v[i]);
      } else {
        for (int c = 0; c < D; c += NV) {
          const Vec16<T> kk = ld16(kr + c);
#pragma unroll
          for (int i = 0; i < NV; ++i) dot += qs[c + i] * to_f32(kk.v[i]);
        }
      }
    } else {
      for (int i = 0; i < D; ++i) dot += qs[i] * to_f32(kr[i]);
    }
    return dot;
  };
  uint32_t cap_mask = 0;     // CAP: the slots this head is saved to, read once per warp
  if constexpr (X == kCapture) cap_mask = cap.masks[h];
  // scores: one key per lane
  float m = -INFINITY;
  for (int j = lane; j < nkeys; j += 32) {
    const T* kr = kb + key_row(j) * a.kv_stride + h * D;
    if constexpr (MODE == 1) {
      // own key: not necessarily visible through the cache pointer yet
      if (j == step) kr = static_cast<const T*>(a.q) + n * a.q_stride + d_model + h * D;
    }
    const float dot = dot_row(kr);
    const float s = round_to<T>(dot * a.scale);
    sc[j] = s;
    m = fmaxf(m, s);
    if constexpr (X == kCapture) {
      const int64_t e = n / a.beam, t = n - e * a.beam;
      for (uint32_t mk = cap_mask; mk; mk &= mk - 1)
        cap.out[((e * cap.total + cap.first + __ffs(mk) - 1) * a.beam + t) * a.S + j] = s;
    }
  }
  m = warp_max(m);
  float sum = 0.f;
  for (int j = lane; j < nkeys; j += 32) sum += expf(sc[j] - m);
  sum = warp_sum(sum);
  for (int j = lane; j < nkeys; j += 32) {
    sc[j] = round_to<T>(expf(sc[j] - m) / sum);
    if constexpr (X == kAlign) {
      if (h < cap.heads) cap.probs[(n * cap.heads + h) * a.S + j] = sc[j];
    }
  }
  __syncwarp();
  T* orow = static_cast<T*>(a.out) + n * a.out_stride + h * D;
  auto value_row = [&](int j) -> const T* {
    if constexpr (MODE == 1) {
      if (j == step) return static_cast<const T*>(a.q) + n * a.q_stride + 2 * d_model + h * D;
    }
    return vb + key_row(j) * a.kv_stride + h * D;
  };
  if (vec && sizeof(T) == 2 && D % 64 == 0) {
    // context: two adjacent output dimensions per lane, one 4-byte load per key (a warp reads 128 contiguous bytes)
    for (int i = 2 * lane; i < D; i += 64) {
      float a0 = 0.f, a1 = 0.f;
#pragma unroll 8
      for (int j = 0; j < nkeys; ++j) {              // unrolled: eight value rows in flight, sums in key order
        const T* vr = value_row(j);
        const uint32_t w = *reinterpret_cast<const uint32_t*>(vr + i);
        T e[2];
        *reinterpret_cast<uint32_t*>(e) = w;
        const float p = sc[j];
        a0 += p * to_f32(e[0]);
        a1 += p * to_f32(e[1]);
      }
      T o[2] = {from_f32<T>(a0), from_f32<T>(a1)};
      *reinterpret_cast<uint32_t*>(orow + i) = *reinterpret_cast<const uint32_t*>(o);
    }
    return;
  }
  // context: one output dimension per lane
  for (int i = lane; i < D; i += 32) {
    float acc = 0.f;
#pragma unroll 4
    for (int j = 0; j < nkeys; ++j) {
      const T* vr;
      if constexpr (MODE == 1) {
        vr = (j == step) ? static_cast<const T*>(a.q) + n * a.q_stride + 2 * d_model + h * D
                         : vb + key_row(j) * a.kv_stride + h * D;
      } else {
        vr = vb + key_row(j) * a.kv_stride + h * D;
      }
      acc += sc[j] * to_f32(vr[i]);
    }
    orow[i] = from_f32<T>(acc);
  }
}

// ---------------------------------------------------------------------------------------------
// BeamSearch::search, device side (src/decoding.cc:425-720).
// ---------------------------------------------------------------------------------------------
// Step 1 per row of [B*beam, V]: DisableTokens of the end ids while step < min_length (apply_min_length, decoding.cc:60-81),
// ops::LogSoftMax in fp32 -> T, then primitives::add_depth_broadcast of the beam's cumulative score IN T (decoding.cc:548-553).
// The logits processors of one row, in place, in the order of make_logits_processors (decoding.cc:1099-1112): the
// RepetitionPenalty rewrites values first; then DisableTokens (decoding_utils.h:20-60) writes every disabled entry — the end
// ids below min_length, NoRepeatNgram, SuppressTokens, SuppressTokensBegin at the first step, SuppressSequences — and
// Whisper's ApplyTimestampRules come last.  The history is the row's tokens chosen so far (alive, parity of the step).
// Ends with a block barrier.
template <typename T>
__device__ __forceinline__ void beam_mask_row(T* xr, const BeamState& st, int64_t row, int abs_step, float* red, int* s_check) {
  const int64_t vocab = st.vocab;
  const int step = abs_step - st.start_step;           // steps of the search (the prompt was forwarded before)
  const T lowest = from_f32<T>(lowest_of<T>());
  auto disable_range = [&](int lo, int hi) {           // [lo, hi)
    for (int j = lo + threadIdx.x; j < hi; j += blockDim.x) xr[j] = lowest;
  };
  const int64_t N = static_cast<int64_t>(st.batch) * st.beam;
  const int32_t* hist = st.alive + static_cast<int64_t>(abs_step & 1) * N * st.stride + row * st.stride;
  if (st.rep_penalty != 0.f && step > 0) {
    // RepetitionPenalty (decoding_utils.cc:40-67): the first occurrence of each token rewrites it from its unpenalised value;
    // the factor is the penalty rounded to T (cuda/primitives.cu:304-320), the arithmetic f32
    const float p = round_to<T>(st.rep_penalty);
    for (int t = threadIdx.x; t < step; t += blockDim.x) {
      const int32_t tok = hist[t];
      bool first = tok >= 0 && tok < vocab;
#pragma unroll 8
      for (int j = 0; j < t; ++j) first &= hist[j] != tok;
      if (first) {
        const float x = to_f32(xr[tok]);
        xr[tok] = from_f32<T>(x < 0.f ? x * p : x / p);
      }
    }
    __syncthreads();                                   // every disable below lands after the penalty
  }
  const int n = st.no_repeat_ngram;
  if (n > 0 && step >= n) {
    // NoRepeatNgram (:70-107): the token that completed an earlier occurrence of the last n - 1 tokens
    for (int q = threadIdx.x; q + n <= step; q += blockDim.x) {
      bool same = true;
      for (int j = 0; j + 1 < n && same; ++j) same = hist[q + j] == hist[step - n + 1 + j];
      const int32_t tok = hist[q + n - 1];
      if (same && tok >= 0 && tok < vocab) xr[tok] = lowest;
    }
  }
  for (int s = threadIdx.x; s < st.num_sequences; s += blockDim.x) {
    // SuppressSequences (:110-150): a single token always, else the last token when the history ends with the others; an
    // empty sequence is ignored
    const int32_t* seq = st.seq_ids + st.seq_offsets[s];
    const int k = st.seq_offsets[s + 1] - st.seq_offsets[s] - 1;
    bool match = k >= 0 && k <= step;
    for (int j = 0; j < k && match; ++j) match = hist[step - k + j] == seq[j];
    if (match && seq[k] >= 0 && seq[k] < vocab) xr[seq[k]] = lowest;
  }
  if (step < st.min_length)
    for (int e = threadIdx.x; e < st.num_end; e += blockDim.x)
      if (st.end_ids[e] >= 0 && st.end_ids[e] < vocab) xr[st.end_ids[e]] = lowest;
  for (int e = threadIdx.x; e < st.num_disable; e += blockDim.x)
    if (st.disable_ids[e] >= 0 && st.disable_ids[e] < vocab) xr[st.disable_ids[e]] = lowest;
  if (step == 0)
    for (int e = threadIdx.x; e < st.num_begin; e += blockDim.x)
      if (st.disable_begin[e] >= 0 && st.disable_begin[e] < vocab) xr[st.disable_begin[e]] = lowest;
  if (st.ts_begin > 0) {
    // ApplyTimestampRules (models/whisper.cc:764-838) on this row's history
    if (threadIdx.x == 0) {
      *s_check = 0;
      xr[st.ts_no_timestamps] = lowest;
    }
    __syncthreads();
    if (step == 0) {
      disable_range(0, st.ts_begin);                                   // a timestamp comes first,
      disable_range(st.ts_max_initial + 1, st.ts_end + 1);             // not later than max_initial_timestamp
    } else {
      const int last = hist[step - 1];
      if (last >= st.ts_begin) {
        const int penult = step - 1 > 0 ? hist[step - 2] : last;
        if (penult >= st.ts_begin) {
          disable_range(st.ts_begin, st.ts_end + 1);                   // timestamps come in pairs: text has to follow
        } else {
          disable_range(0, st.ts_eot);                                 // text cannot follow a single timestamp
          disable_range(st.ts_begin, last);
          if (threadIdx.x == 0) *s_check = 1;
        }
      } else {
        if (threadIdx.x == 0) *s_check = 1;
        int prev = -1;                                                 // timestamps do not decrease
        for (int t = step - 1; t >= 0; --t)
          if (hist[t] >= st.ts_begin) {
            prev = hist[t];
            break;
          }
        if (prev >= 0) disable_range(st.ts_begin, prev + 1);
      }
    }
    __syncthreads();
    if (*s_check) {
      // if the probability mass of the timestamps exceeds every text token, a timestamp is sampled (should_sample_timestamp)
      float m = -INFINITY;
      for (int64_t j = threadIdx.x; j < vocab; j += blockDim.x) m = fmaxf(m, to_f32(xr[j]));
      m = block_reduce<true>(m, red);
      float s = 0.f;
      for (int64_t j = threadIdx.x; j < vocab; j += blockDim.x) s += expf(to_f32(xr[j]) - m);
      s = block_reduce<false>(s, red);
      const float logs = logf(s);
      float tmax = -INFINITY, smax = -INFINITY;
      for (int j = threadIdx.x; j < st.ts_begin; j += blockDim.x) tmax = fmaxf(tmax, round_to<T>(to_f32(xr[j]) - m - logs));
      for (int j = st.ts_begin + threadIdx.x; j <= st.ts_end; j += blockDim.x) smax = fmaxf(smax, round_to<T>(to_f32(xr[j]) - m - logs));
      tmax = block_reduce<true>(tmax, red);
      smax = block_reduce<true>(smax, red);
      float ssum = 0.f;
      for (int j = st.ts_begin + threadIdx.x; j <= st.ts_end; j += blockDim.x) ssum += expf(round_to<T>(to_f32(xr[j]) - m - logs) - smax);
      ssum = block_reduce<false>(ssum, red);
      if (smax + logf(ssum) > tmax) disable_range(0, st.ts_begin);
    }
  }
  __syncthreads();
}

template <typename T>
__global__ void __launch_bounds__(256) beam_logprobs_kernel(T* __restrict__ logits, const T* __restrict__ cum, BeamState st) {
  __shared__ float red[32];
  __shared__ int s_check;
  griddep_launch();
  griddep_wait();
  const int64_t row = blockIdx.x, vocab = st.vocab;
  T* xr = logits + row * st.vocab_ld;
  beam_mask_row(xr, st, row, *st.step, red, &s_check);
  float m = -INFINITY;
  for (int64_t j = threadIdx.x; j < vocab; j += blockDim.x) m = fmaxf(m, to_f32(xr[j]));
  m = block_reduce<true>(m, red);
  float s = 0.f;
  for (int64_t j = threadIdx.x; j < vocab; j += blockDim.x) s += expf(to_f32(xr[j]) - m);
  s = block_reduce<false>(s, red);
  const float logs = logf(s);
  const float c = to_f32(cum[row]);
  for (int64_t j = threadIdx.x; j < vocab; j += blockDim.x)
    xr[j] = from_f32<T>(round_to<T>(to_f32(xr[j]) - m - logs) + c);
}

// Steps 1 + 2 in one pass over the logits (beam <= 8): the scores above are never written back.  A candidate of the entry's
// top 2 * beam (ops::TopK over the flattened [beam * vocab] scores, decoding.cc:556-563) is necessarily among the top
// 2 * beam of its own row, so every row selects its own — each thread keeps a sorted list of its best KT scores (the same
// T-rounded values the three-kernel path stores) and the lists are merged by 2 * beam block-wide arg-max rounds — and
// beam_update_kernel merges the beam rows of an entry.  Order everywhere: (score desc, flattened index asc), the order of
// topk_kernel (rowwise.cu).  Rows whose stride allows it are read with 16-byte loads.
constexpr int kRowsThreads = 512;
constexpr int kCandCap = 1024;         // elements a row may keep above its threshold before it falls back to the sorted lists

template <typename T, typename F>
__device__ __forceinline__ void for_row_elements(const T* xr, int64_t n, bool vec_ok, F f) {
  constexpr int N = Vec16<T>::N;
  if (vec_ok) {
    const int64_t nvec = n / N;
    for (int64_t vi = threadIdx.x; vi < nvec; vi += blockDim.x) {
      const Vec16<T> d = ld16(xr + vi * N);
#pragma unroll
      for (int i = 0; i < N; ++i) f(to_f32(d.v[i]), static_cast<int32_t>(vi * N + i));
    }
    for (int64_t j = nvec * N + threadIdx.x; j < n; j += blockDim.x) f(to_f32(xr[j]), static_cast<int32_t>(j));
  } else {
    for (int64_t j = threadIdx.x; j < n; j += blockDim.x) f(to_f32(xr[j]), static_cast<int32_t>(j));
  }
}

__device__ __forceinline__ bool score_better(float v, int32_t i, float bv, int32_t bi) { return v > bv || (v == bv && i < bi); }

template <typename T, int KT>
__global__ void __launch_bounds__(kRowsThreads) beam_rows_kernel(T* __restrict__ logits, const T* __restrict__ cum, BeamState st,
                                                                T* __restrict__ row_scores, int32_t* __restrict__ row_ids) {
  __shared__ float red[32];
  __shared__ int s_check;
  __shared__ float s_bv[2][kRowsThreads / 32];
  __shared__ int32_t s_bi[2][kRowsThreads / 32];
  __shared__ float s_tm[kRowsThreads];
  __shared__ float s_cv[kCandCap];
  __shared__ int32_t s_ci[kCandCap];
  __shared__ int s_cnt;
  griddep_launch();
  griddep_wait();
  const int64_t row = blockIdx.x, vocab = st.vocab;
  T* xr = logits + row * st.vocab_ld;
  beam_mask_row(xr, st, row, *st.step, red, &s_check);
  const bool vec_ok = (reinterpret_cast<uintptr_t>(xr) & 15) == 0;
  float tm = -INFINITY;                            // this thread's largest logit
  for_row_elements(xr, vocab, vec_ok, [&](float v, int32_t) { tm = fmaxf(tm, v); });
  const float m = block_reduce<true>(tm, red);
  float s = 0.f;
  // 2-byte logits: exp through ex2.approx (2 ulp of a sum that is rounded to 11 / 8 mantissa bits afterwards); float logits keep expf
  if constexpr (sizeof(T) == 2) {
    for_row_elements(xr, vocab, vec_ok, [&](float v, int32_t) { s += exp2f((v - m) * 1.4426950408889634f); });
  } else {
    for_row_elements(xr, vocab, vec_ok, [&](float v, int32_t) { s += expf(v - m); });
  }
  s = block_reduce<false>(s, red);
  const float logs = logf(s);
  const float c = to_f32(cum[row]);
  const int nc = 2 * st.beam, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = (row % st.beam) * vocab;
  auto score = [&](float x) { return round_to<T>(round_to<T>(x - m - logs) + c); };      // monotone in x

  // Fast path.  The score is a monotone map of the logit, so the nc-th largest of the 512 per-thread maxima is a lower bound V of
  // the row's nc-th best score: one more pass keeps the (few) elements with score >= V in shared memory and ranks them.  The
  // per-thread sorted lists below cost an insertion per element POSITION once any lane of the warp inserts; they remain the path of rows with more than kCandCap such elements
  // (ties: rows whose cumulative score is -inf at the first step).
  {
    const float mine = score(tm);
    s_tm[threadIdx.x] = mine;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    int greater = 0;
    for (int u = 0; u < kRowsThreads; ++u) greater += s_tm[u] > mine ? 1 : 0;
    const float vstar = -block_reduce<true>(greater < nc ? -mine : -INFINITY, red);
    if (vstar > -INFINITY) {                         // block-uniform
      for_row_elements(xr, vocab, vec_ok, [&](float x, int32_t j) {
        const float v = score(x);
        if (v >= vstar) {
          const int k = atomicAdd(&s_cnt, 1);
          if (k < kCandCap) { s_cv[k] = v; s_ci[k] = j; }
        }
      });
      __syncthreads();
      const int n = s_cnt;
      if (n <= kCandCap) {
        for (int t = threadIdx.x; t < n; t += kRowsThreads) {
          const float v = s_cv[t];
          const int32_t id = s_ci[t];
          int rank = 0;
          for (int u = 0; u < n; ++u) rank += score_better(s_cv[u], s_ci[u], v, id) ? 1 : 0;
          if (rank < nc) {
            row_scores[row * nc + rank] = from_f32<T>(v);
            row_ids[row * nc + rank] = static_cast<int32_t>(base + id);
          }
        }
        if (threadIdx.x == 0)
          for (int r = n; r < nc; ++r) {             // fewer elements than candidates (vocabulary < 2 * beam)
            row_scores[row * nc + r] = from_f32<T>(-INFINITY);
            row_ids[row * nc + r] = -1;
          }
        return;
      }
    }
    __syncthreads();
  }

  float tv[KT];
  int32_t ti[KT];
#pragma unroll
  for (int k = 0; k < KT; ++k) { tv[k] = -INFINITY; ti[k] = INT32_MAX; }
  for_row_elements(xr, vocab, vec_ok, [&](float x, int32_t j) {
    const float v = score(x);
    if (score_better(v, j, tv[KT - 1], ti[KT - 1])) {
      tv[KT - 1] = v;
      ti[KT - 1] = j;
#pragma unroll
      for (int k = KT - 1; k > 0; --k)
        if (score_better(tv[k], ti[k], tv[k - 1], ti[k - 1])) {
          const float fv = tv[k]; tv[k] = tv[k - 1]; tv[k - 1] = fv;
          const int32_t fi = ti[k]; ti[k] = ti[k - 1]; ti[k - 1] = fi;
        }
    }
  });
  // merge: 2 * beam rounds; the thread that owns the round's best pops it
  for (int r = 0; r < nc; ++r) {
    float bv = tv[0];
    int32_t bi = ti[0];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (score_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { s_bv[r & 1][warp] = bv; s_bi[r & 1][warp] = bi; }
    __syncthreads();
    bv = lane < kRowsThreads / 32 ? s_bv[r & 1][lane] : -INFINITY;
    bi = lane < kRowsThreads / 32 ? s_bi[r & 1][lane] : INT32_MAX;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (score_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (ti[0] == bi && bi != INT32_MAX) {            // indices are unique: exactly one owner
#pragma unroll
      for (int k = 0; k + 1 < KT; ++k) { tv[k] = tv[k + 1]; ti[k] = ti[k + 1]; }
      tv[KT - 1] = -INFINITY;
      ti[KT - 1] = INT32_MAX;
    }
    if (threadIdx.x == 0) {
      row_scores[row * nc + r] = from_f32<T>(bv);
      row_ids[row * nc + r] = bi == INT32_MAX ? -1 : static_cast<int32_t>(base + bi);
    }
  }
}

// Step 3 (step 2 = ops::TopK of 2 * beam candidates over the flattened [beam * vocab] scores, rowwise.cu): one CTA per batch
// entry walks the candidates exactly like decoding.cc:595-663 — a candidate among the first `beam` that ends (end token, or
// last step) is registered as a hypothesis and its slot refilled from the secondary list — then rebuilds the beam state:
// next ids, cumulative scores, token history (alive_seq) and the K/V ancestry table, both double-buffered by step parity.
// Finished entries keep decoding (their results are frozen); the last CTA to finish advances the step counter.
template <typename T>
__global__ void __launch_bounds__(128) beam_update_kernel(BeamState st, const T* __restrict__ cand_scores,
                                                          const int32_t* __restrict__ cand_ids, T* __restrict__ cum,
                                                          bool per_row) {
  __shared__ int s_origin[64], s_word[64], s_active[32], s_hyp[32];
  __shared__ float s_score[64];
  __shared__ float s_cv[128];
  __shared__ int32_t s_ci[128];
  __shared__ int s_last;
  griddep_launch();
  griddep_wait();
  const int i = blockIdx.x;
  const int beam = st.beam, nc = 2 * beam, L = st.stride;
  const int step = *st.step;                 // absolute position (indexes the K/V arena and the ancestry table)
  const int rel = step - st.start_step;      // step of the search (indexes the token history)
  const int N = st.batch * beam;
  if (per_row) {
    // candidates [beam rows][nc] of beam_rows_kernel: the entry's top nc by rank (the order is total: ids are unique)
    const int total = beam * nc;             // <= 128
    float v = -INFINITY;
    int32_t id = INT32_MAX;
    if (threadIdx.x < total) {
      v = to_f32(cand_scores[static_cast<int64_t>(i) * total + threadIdx.x]);
      id = cand_ids[static_cast<int64_t>(i) * total + threadIdx.x];
      if (id < 0) id = INT32_MAX;
    }
    s_cv[threadIdx.x] = v;
    s_ci[threadIdx.x] = id;
    __syncthreads();
    if (threadIdx.x < total && id != INT32_MAX) {
      int rank = 0;
      for (int j = 0; j < total; ++j) rank += score_better(s_cv[j], s_ci[j], v, id) ? 1 : 0;
      if (rank < nc) {
        s_origin[rank] = id / st.vocab;
        s_word[rank] = id % st.vocab;
        s_score[rank] = v;
      }
    }
  } else if (threadIdx.x < nc) {
    const int flat = cand_ids[i * nc + threadIdx.x];
    s_origin[threadIdx.x] = flat / st.vocab;
    s_word[threadIdx.x] = flat % st.vocab;
    s_score[threadIdx.x] = to_f32(cand_scores[i * nc + threadIdx.x]);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const bool was_finished = st.finished[i] != 0;
    BeamDecision d;
    beam_decide(beam, s_word, st.end_ids, st.num_end, rel, st.max_steps, was_finished, st.top_done[i], st.num_hyp[i], st.max_hyp,
                st.max_candidates, st.num_hypotheses, st.early_exit, st.include_eos, d);
    for (int k = 0; k < beam; ++k) {
      s_active[k] = d.active[k];
      s_hyp[k] = d.hyp_slot[k];
      if (d.hyp_slot[k] >= 0) {
        st.hyp_len[i * st.max_hyp + d.hyp_slot[k]] = d.hyp_len[k];
        st.hyp_score[i * st.max_hyp + d.hyp_slot[k]] = s_score[k];
      }
    }
    if (!was_finished) {
      st.num_hyp[i] = d.num_hyp;
      st.top_done[i] = d.top_done;
      if (d.finished) {
        st.finished[i] = 1;
        atomicAdd(st.num_finished, 1);
      }
    }
  }
  __syncthreads();
  const int32_t* alive_r = st.alive + static_cast<int64_t>(step & 1) * N * L;
  int32_t* alive_w = st.alive + static_cast<int64_t>((step + 1) & 1) * N * L;
  const int32_t* anc_r = st.anc + static_cast<int64_t>(step & 1) * N * L;
  int32_t* anc_w = st.anc + static_cast<int64_t>((step + 1) & 1) * N * L;
  // hypotheses registered this step: history of the candidate's origin beam + its word
  for (int k = 0; k < beam; ++k) {
    const int slot = s_hyp[k];
    if (slot < 0) continue;
    int32_t* dst = st.hyp_tokens + (static_cast<int64_t>(i) * st.max_hyp + slot) * L;
    const int32_t* src = alive_r + static_cast<int64_t>(i * beam + s_origin[k]) * L;
    for (int t = threadIdx.x; t < rel; t += blockDim.x) dst[t] = src[t];
    if (threadIdx.x == 0) dst[rel] = s_word[k];
    if (st.hyp_anc) {
      // the slots that computed its positions: the origin beam's ancestry, then the origin row itself
      int32_t* da = st.hyp_anc + (static_cast<int64_t>(i) * st.max_hyp + slot) * L;
      const int32_t* sa = anc_r + static_cast<int64_t>(i * beam + s_origin[k]) * L;
      for (int t = threadIdx.x; t < step; t += blockDim.x) da[t] = sa[t];
      if (threadIdx.x == 0) da[step] = i * beam + s_origin[k];
    }
  }
  // the next beams
  for (int k = 0; k < beam; ++k) {
    const int c = s_active[k];
    const int64_t row = static_cast<int64_t>(i) * beam + k, parent = static_cast<int64_t>(i) * beam + s_origin[c];
    for (int t = threadIdx.x; t < step; t += blockDim.x) {
      if (t < rel) alive_w[row * L + t] = alive_r[parent * L + t];
      anc_w[row * L + t] = anc_r[parent * L + t];
    }
    if (threadIdx.x == 0) {
      alive_w[row * L + rel] = s_word[c];
      anc_w[row * L + step] = static_cast<int32_t>(parent);
      st.next_ids[row] = s_word[c];
      if (st.parent) st.parent[row] = static_cast<int32_t>(parent);
      cum[row] = from_f32<T>(s_score[c]);
    }
  }
  // the last CTA advances the step (every CTA has read it by then)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = atomicAdd(st.ticket, 1) == static_cast<int>(gridDim.x) - 1;
    if (s_last) {
      *st.ticket = 0;
      *st.step = step + 1;
    }
  }
}

// One prompt position forwarded without a search step (WhisperDecoder::forward_prompt, layers/whisper.cc:66-75; the hard
// prefix of decode(), decoding.cc:1138-1170): every row keeps its own K/V slot, the next input is the next prompt token.
__global__ void beam_force_kernel(BeamState st, const int32_t* __restrict__ forced_next /* [rows] */) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  const int N = st.batch * st.beam;
  const int step = *st.step;
  if (row < N) {
    st.anc[static_cast<int64_t>(row) * st.stride + step] = row;                                  // both parities: identity
    st.anc[static_cast<int64_t>(N) * st.stride + static_cast<int64_t>(row) * st.stride + step] = row;
    st.next_ids[row] = forced_next[row];
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const bool last = atomicAdd(st.ticket, 1) == static_cast<int>(gridDim.x) - 1;
    if (last) {
      *st.ticket = 0;
      *st.step = step + 1;
    }
  }
}

// GreedySearch::search with a RandomSampler (decoding.cc:844-971), one CTA per row: the row's DisableTokens / timestamp rules,
// then the draw.  The seed and the call index come from device memory, so a replayed graph draws fresh numbers.
template <typename T>
__global__ void __launch_bounds__(kSampleThreads) beam_sample_kernel(T* __restrict__ logits, BeamState st) {
  __shared__ SampleShared sm;
  __shared__ int s_check;
  griddep_launch();
  griddep_wait();
  const int64_t row = blockIdx.x;
  const int step = *st.step;
  T* xr = logits + row * st.vocab_ld;
  beam_mask_row(xr, st, row, step, sm.red, &s_check);
  const float u = philox_uniform(st.rng[0], st.rng[1], static_cast<uint32_t>(row), static_cast<uint32_t>(step));
  sample_row(xr, st.vocab, st.sample_topk, st.sample_temperature, u, sm, st.sample_ids + row, st.sample_logp + row);
}

template <typename T>
__global__ void __launch_bounds__(kSampleThreads) random_sample_kernel(const T* __restrict__ x, int vocab, int64_t ld, int k,
                                                                       float temperature, uint32_t seed, uint32_t call,
                                                                       uint32_t step, int32_t* __restrict__ ids,
                                                                       float* __restrict__ logp) {
  __shared__ SampleShared sm;
  const int64_t row = blockIdx.x;
  const float u = philox_uniform(seed, call, static_cast<uint32_t>(row), step);
  sample_row(x + row * ld, vocab, k, temperature, u, sm, ids + row, logp + row);
}

// The bookkeeping of the sampled search, one thread per row (results[batch_id] of decoding.cc:910-960, with every entry
// repeated num_hypotheses times): the token joins the row's history, its log-probability the row's score; a row that samples
// an end token or reaches the last step registers hypothesis h (the end token counted in the score, left out of the
// hypothesis per include_eos).  An entry is finished when its rows all are.  The last CTA advances the step.
__global__ void beam_sample_update_kernel(BeamState st) {
  const int N = st.batch * st.beam, L = st.stride;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int step = *st.step, rel = step - st.start_step;
  if (n < N) {
    const int i = n / st.beam, h = n % st.beam;
    const int32_t tok = st.sample_ids[n];
    int32_t* hist0 = st.alive + static_cast<int64_t>(n) * L;
    int32_t* hist1 = hist0 + static_cast<int64_t>(N) * L;
    hist0[rel] = tok;                                  // identity ancestry: both parities hold the whole history
    hist1[rel] = tok;
    st.anc[static_cast<int64_t>(n) * L + step] = n;
    st.anc[static_cast<int64_t>(N) * L + static_cast<int64_t>(n) * L + step] = n;
    st.next_ids[n] = tok;
    if (!st.row_done[n]) {
      const float score = st.row_score[n] + st.sample_logp[n];
      st.row_score[n] = score;
      bool is_end = false;
      for (int e = 0; e < st.num_end; ++e) is_end |= st.end_ids[e] == tok;
      if (is_end || rel + 1 >= st.max_steps) {
        const int len = (is_end && !st.include_eos) ? rel : rel + 1;
        int32_t* dst = st.hyp_tokens + (static_cast<int64_t>(i) * st.max_hyp + h) * L;
        for (int t = 0; t < len; ++t) dst[t] = hist0[t];
        st.hyp_len[i * st.max_hyp + h] = len;
        st.hyp_score[i * st.max_hyp + h] = score;
        st.row_done[n] = 1;
        __threadfence();
        if (atomicAdd(st.num_hyp + i, 1) == st.beam - 1) {
          st.finished[i] = 1;
          atomicAdd(st.num_finished, 1);
        }
      }
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const bool last = atomicAdd(st.ticket, 1) == static_cast<int>(gridDim.x) - 1;
    if (last) {
      *st.ticket = 0;
      *st.step = step + 1;
    }
  }
}

// probability of one token under ops::SoftMax of the row (get_no_speech_probs_from_logits, models/whisper.cc:131-147)
template <typename T>
__global__ void __launch_bounds__(256) token_prob_kernel(const T* __restrict__ logits, int64_t vocab, int64_t row_stride,
                                                         int token, float* __restrict__ out) {
  __shared__ float red[32];
  const T* xr = logits + static_cast<int64_t>(blockIdx.x) * row_stride;
  float m = -INFINITY;
  for (int64_t j = threadIdx.x; j < vocab; j += blockDim.x) m = fmaxf(m, to_f32(xr[j]));
  m = block_reduce<true>(m, red);
  float s = 0.f;
  for (int64_t j = threadIdx.x; j < vocab; j += blockDim.x) s += expf(to_f32(xr[j]) - m);
  s = block_reduce<false>(s, red);
  if (threadIdx.x == 0) out[blockIdx.x] = round_to<T>(expf(to_f32(xr[token]) - m) / s);
}

// im2col of ops::Conv1D (src/ops/conv1d_gpu.cu; CPU form conv1d_cpu.cc:128-220): row (b, t) of cols = x[b, ci, t * stride + k -
// padding] in (ci, k) order, so that conv = cols . W^T with W [Cout, Cin * K] as stored.  channel_major: x is [B, Cin, Tin]
// (the input features); otherwise x is [B, Tin, Cin] (the previous convolution's GEMM output).
template <typename TIn, typename T>
__global__ void im2col_kernel(const TIn* __restrict__ x, int64_t Cin, int64_t Tin, int64_t Tout, int K, int stride, int padding,
                              bool channel_major, T* __restrict__ cols) {
  const int64_t r = blockIdx.x;                 // b * Tout + t
  const int64_t b = r / Tout, t = r % Tout;
  const int64_t width = Cin * K;
  for (int64_t j = threadIdx.x; j < width; j += blockDim.x) {
    const int64_t ci = j / K;
    const int k = static_cast<int>(j % K);
    const int64_t tt = t * stride + k - padding;
    float v = 0.f;
    if (tt >= 0 && tt < Tin) v = channel_major ? to_f32(x[(b * Cin + ci) * Tin + tt]) : to_f32(x[(b * Tin + tt) * Cin + ci]);
    cols[r * width + j] = from_f32<T>(v);
  }
}

// PositionEncoder::operator() (common.cc:150-172): x[b, t, :] += encodings[t, :], in T
template <typename T>
__global__ void add_positions_kernel(T* __restrict__ x, const T* __restrict__ pos, int64_t time, int64_t depth) {
  const int64_t r = blockIdx.x, t = r % time;
  for (int64_t j = threadIdx.x; j < depth; j += blockDim.x)
    x[r * depth + j] = from_f32<T>(to_f32(x[r * depth + j]) + to_f32(pos[t * depth + j]));
}

// rows of a contiguous K/V cache re-gathered after a search step (or replicated beam times after the prompt pass)
__global__ void kv_gather_kernel(const uint4* __restrict__ src_k, const uint4* __restrict__ src_v, uint4* __restrict__ dst_k,
                                 uint4* __restrict__ dst_v, const int32_t* __restrict__ parent, int beam, int Hkv,
                                 int64_t head_stride16, int64_t copy16) {
  const int64_t row = blockIdx.x / Hkv, h = blockIdx.x % Hkv;
  const int64_t from = parent ? parent[row] : row / beam;
  const int64_t so = (from * Hkv + h) * head_stride16, dof = (row * Hkv + h) * head_stride16;
  for (int64_t i = threadIdx.x + static_cast<int64_t>(blockIdx.y) * blockDim.x; i < copy16; i += static_cast<int64_t>(blockDim.x) * gridDim.y) {
    dst_k[dof + i] = src_k[so + i];
    dst_v[dof + i] = src_v[so + i];
  }
}

// initialize_beam_scores (decoding.cc:84-93): beam 0 of every entry starts at 0, the others at the lowest T
template <typename T>
__global__ void beam_init_kernel(T* cum, int32_t* ids, int n, int beam, int start_id) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  cum[r] = from_f32<T>((r % beam) == 0 ? 0.f : lowest_of<T>());
  ids[r] = start_id;
}

// ---------------------------------------------------------------------------------------------
// float32 Dense (primitives<CUDA>::gemm<float, float>, src/cuda/primitives.cu:485-505: cublasSgemm) — C[m,n] = A[m,k] . B[n,k]^T
// with the float epilogue of ops::Gemm (gemm.cc:10-25).  True fp32 FMAs on the CUDA cores (wgmma has no fp32 kind; TF32 would
// not meet the reference's 1e-5 class): 64 x 64 tiles, 16-deep K slices in shared memory, 4 x 4 outputs per thread.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gemm_f32_kernel(const float* __restrict__ A, const float* __restrict__ B, int64_t M, int64_t N,
                                                      int64_t K, FloatEpilogue e) {
  __shared__ float As[16][64 + 4], Bs[16][64 + 4];
  griddep_launch();
  griddep_wait();
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int64_t m0 = static_cast<int64_t>(blockIdx.y) * 64, n0 = static_cast<int64_t>(blockIdx.x) * 64;
  float acc[4][4] = {};
  for (int64_t k0 = 0; k0 < K; k0 += 16) {
    for (int idx = threadIdx.x; idx < 64 * 16; idx += 256) {
      const int r = idx / 16, c = idx % 16;
      As[c][r] = (m0 + r < M && k0 + c < K) ? A[(m0 + r) * K + k0 + c] : 0.f;
      Bs[c][r] = (n0 + r < N && k0 + c < K) ? B[(n0 + r) * K + k0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        a[i] = As[kk][ty * 4 + i];
        b[i] = Bs[kk][tx * 4 + i];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t r = m0 + ty * 4 + i, c = n0 + tx * 4 + j;
      if (r < M && c < N) float_epilogue_store<float>(e, acc[i][j], r, c);
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
void launch_embed_pos(const void* w, const float* w_scale, const int32_t* ids, int64_t rows, int64_t depth, float emb_scale,
                      const void* pos, int64_t time, const int32_t* step_ptr, bool zero_first, void* y, int dtype,
                      cudaStream_t st, const void* w2, const float* w2_scale, const int32_t* ids2) {
  if (rows == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (launch_pdl(embed_pos_kernel<T>, dim3(rows), dim3(128), 0, st, w, w_scale, ids, depth, emb_scale,
                                        static_cast<const T*>(pos), time, step_ptr, zero_first, static_cast<T*>(y), w2,
                                        w2_scale, ids2)));
  check_launch();
}

void launch_layer_norm(const void* x, const void* gamma, const void* beta, int64_t rows, int64_t cols, float eps, void* y,
                       int8_t* q, float* scale, bool round, int dtype, cudaStream_t st) {
  if (rows == 0) return;
  if (cols <= 512) {
    CT2_DISPATCH_DTYPE(dtype, (launch_pdl(layer_norm_small_kernel<T, 2>, dim3(rows), dim3(256), 0, st, static_cast<const T*>(x),
                                          static_cast<const T*>(gamma), static_cast<const T*>(beta), cols, eps,
                                          static_cast<T*>(y), q, scale, round)));
  } else if (cols <= 2048) {
    CT2_DISPATCH_DTYPE(dtype, (launch_pdl(layer_norm_small_kernel<T, 8>, dim3(rows), dim3(256), 0, st, static_cast<const T*>(x),
                                          static_cast<const T*>(gamma), static_cast<const T*>(beta), cols, eps,
                                          static_cast<T*>(y), q, scale, round)));
  } else {
    CT2_DISPATCH_DTYPE(dtype, (launch_pdl(layer_norm_kernel<T>, dim3(rows), dim3(256), 0, st, static_cast<const T*>(x),
                                          static_cast<const T*>(gamma), static_cast<const T*>(beta), cols, eps,
                                          static_cast<T*>(y), q, scale, round)));
  }
  check_launch();
}

namespace {
template <typename T, int MODE, int X = kNoExtra>
void launch_attn_mode(const AttnGeneric& a_in, cudaStream_t st, const ExtraArg<X>& cap = {}) {
  AttnGeneric a = a_in;
  {
    const size_t es = sizeof(T);
    auto al = [&](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    a.vec_ok = al(a.q) && al(a.k) && al(a.v) && al(a.out) && al(a.k_cache) && al(a.v_cache) && (a.q_stride * es) % 16 == 0 &&
               (a.kv_stride * es) % 16 == 0 && (a.out_stride * es) % 16 == 0 && (static_cast<size_t>(a.D) * es) % 16 == 0;
  }
  const size_t smem = static_cast<size_t>(kAttnWarps) * (a.max_keys + a.D) * sizeof(float);
  CT2_REQUIRE(smem <= 200 * 1024, "attention: too many keys for the generic kernel");
  auto kernel = a.D == 64 ? attention_generic_kernel<T, MODE, 64, X>
                : a.D == 128 ? attention_generic_kernel<T, MODE, 128, X> : attention_generic_kernel<T, MODE, 0, X>;
  if (smem > 48 * 1024) {
    // the attribute is per device: set it whenever the request grows (cheap, idempotent)
    CT2_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  }
  const int64_t units = a.rows * a.H;
  launch_pdl(kernel, dim3(static_cast<unsigned>((units + kAttnWarps - 1) / kAttnWarps)), dim3(kAttnWarps * 32), smem, st, a, cap);
  check_launch();
}
}  // namespace

void launch_attention_encoder(const void* qkv, const int32_t* lengths, int64_t batch, int S, int H, int D, float scale,
                              void* out, int dtype, cudaStream_t st) {
  if (batch * S == 0) return;
  const int64_t d = static_cast<int64_t>(H) * D;
  const size_t es = dtype_size(dtype);
  AttnGeneric a{};
  a.q = qkv;
  a.q_stride = 3 * d;
  a.k = static_cast<const uint8_t*>(qkv) + d * es;
  a.v = static_cast<const uint8_t*>(qkv) + 2 * d * es;
  a.kv_stride = 3 * d;
  a.out = out;
  a.out_stride = d;
  a.lengths = lengths;
  a.rows = batch * S;
  a.S = S;
  a.beam = 1;
  a.H = H;
  a.D = D;
  a.scale = scale;
  a.max_keys = S;
  CT2_DISPATCH_DTYPE(dtype, (launch_attn_mode<T, 0>(a, st)));
}

void launch_attention_causal(const void* qkv, int64_t batch, int time, int H, int D, float scale, void* out, int dtype,
                             cudaStream_t st) {
  if (batch * time == 0) return;
  const int64_t d = static_cast<int64_t>(H) * D;
  const size_t es = dtype_size(dtype);
  AttnGeneric a{};
  a.q = qkv;
  a.q_stride = 3 * d;
  a.k = static_cast<const uint8_t*>(qkv) + d * es;
  a.v = static_cast<const uint8_t*>(qkv) + 2 * d * es;
  a.kv_stride = 3 * d;
  a.out = out;
  a.out_stride = d;
  a.rows = batch * time;
  a.S = time;
  a.beam = 1;
  a.H = H;
  a.D = D;
  a.scale = scale;
  a.max_keys = time;
  CT2_DISPATCH_DTYPE(dtype, (launch_attn_mode<T, 3>(a, st)));
}

void launch_attention_beam_self(const void* qkv, void* k_cache, void* v_cache, const int32_t* anc, const int32_t* step_ptr,
                                int64_t rows, int max_len, int H, int D, float scale, void* out, int dtype, cudaStream_t st) {
  if (rows == 0) return;
  const int64_t d = static_cast<int64_t>(H) * D;
  AttnGeneric a{};
  a.q = qkv;
  a.q_stride = 3 * d;
  a.kv_stride = d;
  a.out = out;
  a.out_stride = d;
  a.anc = anc;
  a.step_ptr = step_ptr;
  a.k_cache = k_cache;
  a.v_cache = v_cache;
  a.rows = rows;
  a.S = max_len;
  a.beam = 1;
  a.H = H;
  a.D = D;
  a.scale = scale;
  a.max_keys = max_len;
  CT2_DISPATCH_DTYPE(dtype, (launch_attn_mode<T, 1>(a, st)));
}

void launch_attention_cross(const void* q, const void* kv, const int32_t* lengths, int64_t rows, int beam, int S, int H, int D,
                            float scale, void* out, int dtype, cudaStream_t st) {
  if (rows == 0) return;
  const int64_t d = static_cast<int64_t>(H) * D;
  const size_t es = dtype_size(dtype);
  AttnGeneric a{};
  a.q = q;
  a.q_stride = d;
  a.k = kv;
  a.v = static_cast<const uint8_t*>(kv) + d * es;
  a.kv_stride = 2 * d;
  a.out = out;
  a.out_stride = d;
  a.lengths = lengths;
  a.rows = rows;
  a.S = S;
  a.beam = beam;
  a.H = H;
  a.D = D;
  a.scale = scale;
  a.max_keys = S;
  CT2_DISPATCH_DTYPE(dtype, (launch_attn_mode<T, 2>(a, st)));
}

void launch_attention_cross_capture(const void* q, const void* kv, const int32_t* lengths, int64_t rows, int beam, int S, int H,
                                    int D, float scale, void* out, const AttnCapture& cap, int dtype, cudaStream_t st) {
  if (rows == 0) return;
  CT2_REQUIRE(cap.out && cap.masks && cap.first >= 0 && cap.first < cap.total, "attention capture: bad heads");
  const int64_t d = static_cast<int64_t>(H) * D;
  const size_t es = dtype_size(dtype);
  AttnGeneric a{};
  a.q = q;
  a.q_stride = d;
  a.k = kv;
  a.v = static_cast<const uint8_t*>(kv) + d * es;
  a.kv_stride = 2 * d;
  a.out = out;
  a.out_stride = d;
  a.lengths = lengths;
  a.rows = rows;
  a.S = S;
  a.beam = beam;
  a.H = H;
  a.D = D;
  a.scale = scale;
  a.max_keys = S;
  CT2_DISPATCH_DTYPE(dtype, (launch_attn_mode<T, 2, kCapture>(a, st, cap)));
}

void launch_attention_cross_align(const void* q, const void* kv, const int32_t* lengths, int64_t rows, int beam, int S, int H,
                                  int D, float scale, void* out, float* probs, int heads, int dtype, cudaStream_t st) {
  if (rows == 0) return;
  CT2_REQUIRE(probs && heads >= 1 && heads <= H, "attention alignment: bad heads");
  const int64_t d = static_cast<int64_t>(H) * D;
  const size_t es = dtype_size(dtype);
  AttnGeneric a{};
  a.q = q;
  a.q_stride = d;
  a.k = kv;
  a.v = static_cast<const uint8_t*>(kv) + d * es;
  a.kv_stride = 2 * d;
  a.out = out;
  a.out_stride = d;
  a.lengths = lengths;
  a.rows = rows;
  a.S = S;
  a.beam = beam;
  a.H = H;
  a.D = D;
  a.scale = scale;
  a.max_keys = S;
  const AttnAlign al{probs, heads};
  CT2_DISPATCH_DTYPE(dtype, (launch_attn_mode<T, 2, kAlign>(a, st, al)));
}

namespace {
// ops::Mean over the alignment heads (transformer.cc:826-829) of one decoding step, in a fixed head order: row n's entry of
// the attention history at the device-resident step; positions past the entry's length are exact zeros.
template <typename T>
__global__ void __launch_bounds__(128) align_mean_kernel(const float* __restrict__ probs, const int32_t* __restrict__ lengths,
                                                         const int32_t* __restrict__ step_ptr, int beam, int S, int heads,
                                                         int stride, float* __restrict__ hist) {
  griddep_launch();
  griddep_wait();
  const int64_t n = blockIdx.x;
  const int len = min(lengths[n / beam], S);
  float* out = hist + (n * stride + *step_ptr) * S;
  const float* p = probs + n * heads * S;
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    float v = 0.f;
    if (s < len) {
      for (int h = 0; h < heads; ++h) v += p[h * S + s];
      v = round_to<T>(v / static_cast<float>(heads));
    }
    out[s] = v;
  }
}

// The coverage term of compute_coverage_penalty (decoding.cc:176-187) of every registered hypothesis, one CTA per (entry,
// slot): sum over the columns with coverage > 0 of log(min(coverage, 1)), coverage = the column summed over the hypothesis's
// rows in order; beta is applied by the caller.
__global__ void __launch_bounds__(128) hyp_coverage_kernel(BeamState st, const float* __restrict__ hist, int S,
                                                           float* __restrict__ out) {
  __shared__ float red[32];
  const int i = blockIdx.x, j = blockIdx.y;
  if (j >= st.num_hyp[i]) return;
  const int64_t h = static_cast<int64_t>(i) * st.max_hyp + j;
  const int len = st.hyp_len[h];
  const int32_t* anc = st.hyp_anc + h * st.stride;
  float pen = 0.f;
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    float cov = 0.f;
    for (int t = 0; t < len; ++t) cov += hist[(static_cast<int64_t>(anc[t]) * st.stride + t) * S + s];
    if (cov > 0.f) pen += logf(fminf(cov, 1.f));
  }
  pen = block_reduce<false>(pen, red);
  if (threadIdx.x == 0) out[h] = pen;
}

// out [batch, num, max_len, S]: the attention rows of hypothesis slot sel[b * num + k] of entry b (-1: none), zeros past its
// length
__global__ void __launch_bounds__(128) hyp_attention_gather_kernel(BeamState st, const float* __restrict__ hist, int S,
                                                                   const int32_t* __restrict__ sel, int num, int max_len,
                                                                   float* __restrict__ out) {
  const int b = blockIdx.x / num;
  const int slot = sel[blockIdx.x];
  const int64_t h = static_cast<int64_t>(b) * st.max_hyp + slot;
  const int len = slot >= 0 ? min(st.hyp_len[h], max_len) : 0;
  float* o = out + static_cast<int64_t>(blockIdx.x) * max_len * S;
  for (int64_t e = threadIdx.x; e < static_cast<int64_t>(max_len) * S; e += blockDim.x) {
    const int t = static_cast<int>(e / S), s = static_cast<int>(e % S);
    o[e] = t < len ? hist[(static_cast<int64_t>(st.hyp_anc[h * st.stride + t]) * st.stride + t) * S + s] : 0.f;
  }
}
}  // namespace

void launch_align_mean(const float* probs, const int32_t* lengths, const int32_t* step_ptr, int64_t rows, int beam, int S,
                       int heads, int stride, float* hist, int dtype, cudaStream_t st) {
  if (rows == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (launch_pdl(align_mean_kernel<T>, dim3(static_cast<unsigned>(rows)), dim3(128), 0, st, probs, lengths,
                                        step_ptr, beam, S, heads, stride, hist)));
  check_launch();
}

void launch_hyp_coverage(const BeamState& s, const float* hist, int S, float* out, cudaStream_t st) {
  if (s.batch == 0) return;
  CT2_REQUIRE(s.hyp_anc, "hyp_coverage: no hypothesis ancestry");
  hyp_coverage_kernel<<<dim3(s.batch, s.max_hyp), 128, 0, st>>>(s, hist, S, out);
  check_launch();
}

void launch_hyp_attention_gather(const BeamState& s, const float* hist, int S, const int32_t* sel, int num, int max_len,
                                 float* out, cudaStream_t st) {
  if (s.batch == 0 || num == 0) return;
  CT2_REQUIRE(s.hyp_anc, "hyp_attention_gather: no hypothesis ancestry");
  hyp_attention_gather_kernel<<<s.batch * num, 128, 0, st>>>(s, hist, S, sel, num, max_len, out);
  check_launch();
}

void launch_beam_init(void* cum, int32_t* ids, int64_t rows, int beam, int start_id, int dtype, cudaStream_t st) {
  if (rows == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (beam_init_kernel<T><<<div_up(rows, 128), 128, 0, st>>>(static_cast<T*>(cum), ids,
                                                                                      static_cast<int>(rows), beam, start_id)));
  check_launch();
}

void launch_beam_logprobs(void* logits, const void* cum, const BeamState& s, int dtype, cudaStream_t st) {
  const int64_t rows = static_cast<int64_t>(s.batch) * s.beam;
  if (rows == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (launch_pdl(beam_logprobs_kernel<T>, dim3(rows), dim3(256), 0, st, static_cast<T*>(logits),
                                        static_cast<const T*>(cum), s)));
  check_launch();
}

void launch_beam_rows(void* logits, const void* cum, const BeamState& s, void* row_scores, int32_t* row_ids, int dtype,
                      cudaStream_t st) {
  const int64_t rows = static_cast<int64_t>(s.batch) * s.beam;
  if (rows == 0) return;
  CT2_REQUIRE(s.beam >= 1 && s.beam <= 8, "beam_rows: beam_size must be in [1, 8]");
  if (s.beam <= 4) {
    CT2_DISPATCH_DTYPE(dtype, (launch_pdl(beam_rows_kernel<T, 8>, dim3(rows), dim3(kRowsThreads), 0, st, static_cast<T*>(logits),
                                          static_cast<const T*>(cum), s, static_cast<T*>(row_scores), row_ids)));
  } else {
    CT2_DISPATCH_DTYPE(dtype, (launch_pdl(beam_rows_kernel<T, 16>, dim3(rows), dim3(kRowsThreads), 0, st, static_cast<T*>(logits),
                                          static_cast<const T*>(cum), s, static_cast<T*>(row_scores), row_ids)));
  }
  check_launch();
}

void launch_beam_force(const BeamState& s, const int32_t* forced_next, cudaStream_t st) {
  const int rows = s.batch * s.beam;
  beam_force_kernel<<<div_up(rows, 128), 128, 0, st>>>(s, forced_next);
  check_launch();
}

void launch_beam_sample(void* logits, const BeamState& s, int dtype, cudaStream_t st) {
  const int64_t rows = static_cast<int64_t>(s.batch) * s.beam;
  CT2_REQUIRE(s.sample_topk >= 0 && s.sample_topk <= s.vocab && s.sample_temperature > 0.f, "beam_sample: bad sampler");
  CT2_DISPATCH_DTYPE(dtype, (launch_pdl(beam_sample_kernel<T>, dim3(rows), dim3(kSampleThreads), 0, st, static_cast<T*>(logits),
                                        s)));
}

void launch_beam_sample_update(const BeamState& s, cudaStream_t st) {
  const int rows = s.batch * s.beam;
  beam_sample_update_kernel<<<div_up(rows, 128), 128, 0, st>>>(s);
  check_launch();
}

void launch_random_sample(const void* x, int64_t rows, int64_t vocab, int64_t ld, int k, float temperature, uint32_t seed,
                          uint32_t call, uint32_t step, int32_t* ids, float* logp, int dtype, cudaStream_t st) {
  CT2_REQUIRE(vocab >= 1 && vocab <= INT32_MAX && ld >= vocab, "random_sample: bad row shape");
  CT2_REQUIRE(k >= 0 && k <= vocab, "random_sample: sampling_topk must be in [0, vocab]");
  CT2_REQUIRE(temperature > 0.f, "random_sample: the temperature must be positive");
  if (rows == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (random_sample_kernel<T><<<static_cast<unsigned>(rows), kSampleThreads, 0, st>>>(
                                static_cast<const T*>(x), static_cast<int>(vocab), ld, k, temperature, seed, call, step, ids, logp)));
  check_launch();
}

void launch_token_prob(const void* logits, int64_t rows, int64_t vocab, int64_t row_stride, int token, float* out, int dtype,
                       cudaStream_t st) {
  if (rows == 0) return;
  CT2_REQUIRE(token >= 0 && token < vocab, "token_prob: token out of range");
  CT2_DISPATCH_DTYPE(dtype, (token_prob_kernel<T><<<rows, 256, 0, st>>>(static_cast<const T*>(logits), vocab, row_stride, token, out)));
  check_launch();
}

void launch_im2col(const void* x, bool x_is_f32, int64_t batch, int64_t Cin, int64_t Tin, int64_t Tout, int K, int stride,
                   int padding, bool channel_major, void* cols, int dtype, cudaStream_t st) {
  if (batch * Tout == 0) return;
  if (x_is_f32) {
    CT2_DISPATCH_DTYPE(dtype, (im2col_kernel<float, T><<<batch * Tout, 128, 0, st>>>(static_cast<const float*>(x), Cin, Tin, Tout, K,
                                                                                    stride, padding, channel_major,
                                                                                    static_cast<T*>(cols))));
  } else {
    CT2_DISPATCH_DTYPE(dtype, (im2col_kernel<T, T><<<batch * Tout, 128, 0, st>>>(static_cast<const T*>(x), Cin, Tin, Tout, K, stride,
                                                                                padding, channel_major, static_cast<T*>(cols))));
  }
  check_launch();
}

void launch_add_positions(void* x, const void* pos, int64_t rows, int64_t time, int64_t depth, int dtype, cudaStream_t st) {
  if (rows == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (add_positions_kernel<T><<<rows, 128, 0, st>>>(static_cast<T*>(x), static_cast<const T*>(pos), time, depth)));
  check_launch();
}

void launch_beam_update(const BeamState& s, const void* cand_scores, const int32_t* cand_ids, void* cum, bool per_row, int dtype,
                        cudaStream_t st) {
  CT2_REQUIRE(s.beam >= 1 && s.beam <= 32, "beam_size must be in [1, 32]");
  CT2_REQUIRE(!per_row || s.beam <= 8, "beam_update: per-row candidates need beam_size <= 8");
  CT2_DISPATCH_DTYPE(dtype, (launch_pdl(beam_update_kernel<T>, dim3(s.batch), dim3(128), 0, st, s,
                                        static_cast<const T*>(cand_scores), cand_ids, static_cast<T*>(cum), per_row)));
  check_launch();
}

void launch_kv_gather(const void* src_k, const void* src_v, void* dst_k, void* dst_v, const int32_t* parent, int beam, int64_t rows,
                      int Hkv, int64_t max_len, int D, int64_t positions, int dtype, cudaStream_t st) {
  if (rows == 0 || positions == 0) return;
  const size_t es = dtype_size(dtype);
  CT2_REQUIRE((static_cast<size_t>(D) * es) % 16 == 0, "kv_gather: head rows must be multiples of 16 bytes");
  const int64_t head_stride16 = max_len * D * es / 16, copy16 = positions * D * es / 16;
  const int chunks = static_cast<int>(std::min<int64_t>(8, (copy16 + 255) / 256));
  kv_gather_kernel<<<dim3(static_cast<unsigned>(rows * Hkv), chunks), 256, 0, st>>>(
      static_cast<const uint4*>(src_k), static_cast<const uint4*>(src_v), static_cast<uint4*>(dst_k), static_cast<uint4*>(dst_v),
      parent, beam, Hkv, head_stride16, copy16);
  check_launch();
}

void gemm_f32(const float* A, const float* B, const float* bias, const float* residual, int act, int64_t M, int64_t N,
              int64_t K, float* C, cudaStream_t st) {
  if (M == 0 || N == 0) return;
  FloatEpilogue e{bias, residual, C, act, N};
  launch_pdl(gemm_f32_kernel, dim3(div_up(N, 64), div_up(M, 64)), dim3(256), 0, st, A, B, M, N, K, e);
  check_launch();
}

}  // namespace ct2b200
