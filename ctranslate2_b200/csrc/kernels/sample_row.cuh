// sample_row.cuh — RandomSampler::sample (src/sampling.cc:34-101) for one row, run by one CTA of kSampleThreads threads:
//   1. max m and log-sum-exp of the row (the LogSoftMax the returned score comes from);
//   2. the top k by (value desc, index asc), the TopK order of the engine, as a radix select on order-preserving keys
//      (k = 0 or k >= vocab keeps the row);
//   3. weights exp((x - m) / temperature) over the kept set (m, the row's maximum, is always kept);
//   4. inverse CDF in ascending index order: the first kept index whose inclusive cumulative weight exceeds u * sum;
//   5. the id and T(x[id] - m - log sum exp(x - m)), the log-probability of the unscaled row.
// The row is read from global memory (L2-resident after the first pass); nothing is written back.
#pragma once

#include <cfloat>

#include "../common.cuh"

namespace ct2b200 {

constexpr int kSampleThreads = 512;
constexpr int kSampleWarps = kSampleThreads / 32;

struct SampleShared {
  float red[32];
  uint32_t hist[256];
  float gt_sum[kSampleWarps];      // per warp: weight of the kept elements above the threshold key
  int eq_cnt[kSampleWarps];        // per warp: elements equal to the threshold key
  float w_eq;                      // weight of an element equal to the threshold key
  uint32_t prefix;                 // threshold key (the k-th largest), built digit by digit
  int remaining;                   // elements equal to the threshold that are kept (lowest indices first)
  int sel_warp, eq_before;         // warp segment holding the draw, threshold-equal elements before it
  float target;                    // u * sum minus the kept weight before that segment
  int result;
};

// order-preserving key of a float (-0 ordered as +0); only the top 8 * SampleKey<T>::kDigits bits are compared, which decide
// the value for T (float: 32, half: 1 + 8 + 10 < 24, bfloat16: 16)
template <typename T> struct SampleKey { static constexpr int kDigits = 4; };
template <> struct SampleKey<__half> { static constexpr int kDigits = 3; };
template <> struct SampleKey<__nv_bfloat16> { static constexpr int kDigits = 2; };

__device__ __forceinline__ uint32_t float_order_key(float v) {
  const uint32_t b = __float_as_uint(v + 0.f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// All threads of the CTA call it; *id_out / *logp_out are written by thread 0.
template <typename T>
__device__ void sample_row(const T* __restrict__ xr, int vocab, int k, float temperature, float u, SampleShared& sm,
                           int32_t* id_out, float* logp_out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float m = -INFINITY;
  for (int j = threadIdx.x; j < vocab; j += kSampleThreads) m = fmaxf(m, to_f32(xr[j]));
  m = block_reduce<true>(m, sm.red);
  float s = 0.f;
  for (int j = threadIdx.x; j < vocab; j += kSampleThreads) s += expf(to_f32(xr[j]) - m);
  s = block_reduce<false>(s, sm.red);

  // ---- 2. radix select of the k-th largest key, 8 bits per pass from the top ----
  constexpr int kDigits = SampleKey<T>::kDigits;
  constexpr int kLow = 32 - 8 * kDigits;                 // key bits below the compared ones
  const bool select = k > 0 && k < vocab;
  if (threadIdx.x == 0) {
    sm.prefix = 0;
    sm.remaining = k;
  }
  __syncthreads();
  if (select) {
    for (int d = 0; d < kDigits; ++d) {
      const int shift = 24 - 8 * d;
      for (int b = threadIdx.x; b < 256; b += kSampleThreads) sm.hist[b] = 0;
      __syncthreads();
      const uint32_t prefix = sm.prefix;
      for (int base = 0; base < vocab; base += kSampleThreads) {   // every lane takes part in the match below
        const int j = base + threadIdx.x;
        const uint32_t key = j < vocab ? float_order_key(to_f32(xr[j])) : 0u;
        const bool in = j < vocab && (d == 0 || (key >> (shift + 8)) == (prefix >> (shift + 8)));
        const uint32_t digit = in ? (key >> shift) & 255u : 256u + lane;
        const unsigned peers = __match_any_sync(0xffffffffu, digit);
        if (in && lane == __ffs(peers) - 1) atomicAdd(&sm.hist[digit], static_cast<uint32_t>(__popc(peers)));
      }
      __syncthreads();
      if (warp == 0) {                                     // lane l owns digits 255 - 8l .. 248 - 8l (descending)
        int c[8], local = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          c[q] = static_cast<int>(sm.hist[255 - 8 * lane - q]);
          local += c[q];
        }
        int incl = local;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int v = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += v;
        }
        const int rem = sm.remaining;
        int above = incl - local;
        if (above < rem && rem <= incl) {                   // exactly one lane
          int q = 0;
          while (above + c[q] < rem) above += c[q++];
          sm.prefix = prefix | (static_cast<uint32_t>(255 - 8 * lane - q) << shift);
          sm.remaining = rem - above;
        }
      }
      __syncthreads();
    }
  }
  const uint32_t thr = sm.prefix >> kLow;
  const int need = sm.remaining;
  // 1 / temperature clamped: below 1 / FLT_MAX only the row's maxima keep a weight (0 * scale = 0, never inf * 0)
  const float scale = fminf(1.f / temperature, FLT_MAX);

  // ---- 3. kept weights per warp segment (contiguous, a multiple of 32 wide) ----
  const int seg = ((vocab + kSampleWarps - 1) / kSampleWarps + 31) & ~31;
  const int seg_lo = warp * seg, seg_hi = min(vocab, seg_lo + seg);
  // weight of element j (0 when not kept by value); eq = equal to the threshold (kept for the lowest `need` indices)
  auto weigh = [&](int j, bool& eq) {
    eq = false;
    if (j >= seg_hi) return 0.f;
    const float x = to_f32(xr[j]);
    if (select) {
      const uint32_t key = float_order_key(x) >> kLow;
      eq = key == thr;
      if (key < thr) return 0.f;
    }
    return expf((x - m) * scale);
  };
  float gt = 0.f;
  int eqn = 0;
  for (int base = seg_lo; base < seg_hi; base += 32) {
    bool eq;
    const float w = weigh(base + lane, eq);
    if (eq) sm.w_eq = w;                                    // every equal element has the same weight
    gt += eq ? 0.f : w;
    eqn += __popc(__ballot_sync(0xffffffffu, eq));
  }
  gt = warp_sum(gt);
  if (lane == 0) {
    sm.gt_sum[warp] = gt;
    sm.eq_cnt[warp] = eqn;
  }
  __syncthreads();

  // ---- 4. the segment holding u * sum ----
  if (threadIdx.x == 0) {
    float seg_w[kSampleWarps], total = 0.f;
    int eq_seen = 0;
    for (int w = 0; w < kSampleWarps; ++w) {
      const int kept_eq = select ? max(0, min(sm.eq_cnt[w], need - eq_seen)) : 0;
      seg_w[w] = sm.gt_sum[w] + (kept_eq ? kept_eq * sm.w_eq : 0.f);
      eq_seen += sm.eq_cnt[w];
      total += seg_w[w];
    }
    const float target = u * total;
    float before = 0.f;
    int sel = 0, sel_eq = 0;
    float sel_before = 0.f;
    eq_seen = 0;
    for (int w = 0; w < kSampleWarps; ++w) {               // the last non-empty segment starting at or below the target
      if (seg_w[w] > 0.f && before <= target) {
        sel = w;
        sel_before = before;
        sel_eq = eq_seen;
      }
      before += seg_w[w];
      eq_seen += sm.eq_cnt[w];
    }
    sm.sel_warp = sel;
    sm.target = target - sel_before;
    sm.eq_before = sel_eq;
    sm.result = -1;
  }
  __syncthreads();
  if (warp == sm.sel_warp) {
    const float target = sm.target;
    int eq_run = sm.eq_before, last = -1;
    float run = 0.f;
    for (int base = seg_lo; base < seg_hi; base += 32) {
      bool eq;
      float w = weigh(base + lane, eq);
      const unsigned eqm = __ballot_sync(0xffffffffu, eq);
      if (eq && eq_run + __popc(eqm & ((1u << lane) - 1u)) >= need) w = 0.f;
      float incl = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const unsigned hit = __ballot_sync(0xffffffffu, w > 0.f && run + incl > target);
      if (hit) {
        last = base + __ffs(hit) - 1;
        break;
      }
      const unsigned pos = __ballot_sync(0xffffffffu, w > 0.f);
      if (pos) last = base + 31 - __clz(pos);             // fall-back: the last kept element of the segment
      run += __shfl_sync(0xffffffffu, incl, 31);
      eq_run += __popc(eqm);
    }
    if (lane == 0) sm.result = last;
  }
  __syncthreads();
  int id = sm.result;
  if (id < 0) {
    // block-uniform: weights that are not finite (an infinite logit) leave the walk empty; the row's first maximum is kept
    // for every k, so it is the draw (index 0 when no element equals the maximum: a row without a finite or infinite value)
    float first = -INFINITY;
    for (int j = threadIdx.x; j < vocab; j += kSampleThreads)
      if (to_f32(xr[j]) == m) {
        first = -static_cast<float>(j);
        break;
      }
    first = block_reduce<true>(first, sm.red);
    id = first == -INFINITY ? 0 : static_cast<int>(-first);
  }
  if (threadIdx.x == 0) {
    *id_out = id;
    *logp_out = round_to<T>(to_f32(xr[id]) - m - logf(s));
  }
}

}  // namespace ct2b200
