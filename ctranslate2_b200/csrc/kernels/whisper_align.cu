// whisper_align.cu — the device side of models::Whisper::align after the decoder pass (src/models/whisper.cc:387-560) and the
// language probabilities of ::detect_language (:584-652).  The cross-attention scores of the alignment heads come from the CAP
// instantiation of attention_generic_kernel (seq2seq.cu) as f32 [B, heads, T, S]; everything here is memory-bound and rounds
// where the reference's ops round in T (SoftMax, LayerNorm, MedianFilter, Mean), with fp32 arithmetic in between.  DTW runs on
// the host (dtw.h), as in the reference (whisper.cc:403-405).
#include <cfloat>

#include "../common.cuh"
#include "kernels.h"

namespace ct2b200 {

namespace {

constexpr int kAlignWarps = 8;

// ops::SoftMax of the saved scores over the entry's frames (softmax_cpu: y = exp(x - max) * (1 / sum)): the equal-frames path
// trims the frames first (whisper.cc:553-554), the variable one masks them (:520-528); either way frames >= nf are not read
// again.  One warp per (entry, head, position) row; rows past the entry's input length are left alone.
template <typename T>
__global__ void __launch_bounds__(kAlignWarps * 32) align_softmax_kernel(float* __restrict__ sc, const int32_t* __restrict__ nf,
                                                                       const int32_t* __restrict__ len, int64_t units, int heads,
                                                                       int64_t T_, int64_t S) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t unit = static_cast<int64_t>(blockIdx.x) * kAlignWarps + warp;
  if (unit >= units) return;
  const int64_t b = unit / (heads * T_), t = unit % T_;
  const int n = nf[b];
  if (t >= len[b] || n <= 0) return;
  float* r = sc + unit * S;
  float m = -INFINITY;
  for (int j = lane; j < n; j += 32) m = fmaxf(m, r[j]);
  m = warp_max(m);
  float s = 0.f;
  for (int j = lane; j < n; j += 32) s += expf(r[j] - m);
  s = warp_sum(s);
  const float inv = 1.f / s;
  for (int j = lane; j < n; j += 32) r[j] = round_to<T>(expf(r[j] - m) * inv);
}

// ops::LayerNorm(axis -2, epsilon 0) without gamma / beta (layer_norm_axis, cpu/kernels.cc: mean = sum / n, var =
// max(sumsq / n - mean^2, 0), y = (x - mean) / sqrt(var)).  One thread per frame column, the token rows summed in order (the
// reference's order); neighbouring threads read neighbouring frames.  Only the rows the DTW matrix takes are written.
template <typename T>
__global__ void __launch_bounds__(128) align_standardize_kernel(const float* __restrict__ sc, const int32_t* __restrict__ nf,
                                                                const int32_t* __restrict__ len, const int32_t* __restrict__ ntext,
                                                                int heads, int64_t T_, int64_t S, int64_t rows, int64_t start,
                                                                int64_t max_text, int64_t F, float* __restrict__ norm) {
  const int64_t bh = blockIdx.y, b = bh / heads;
  const int64_t j = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= nf[b]) return;
  const int64_t last = len[b] - 1, R = rows > 0 ? rows : len[b];
  const float* col = sc + bh * T_ * S + j;
  float sum = 0.f, sq = 0.f;
  for (int64_t t = 0; t < R; ++t) {
    const float x = col[min(t, last) * S];
    sum += x;
    sq += x * x;
  }
  const float n = static_cast<float>(R);
  const float mean = sum / n;
  const float rstd = 1.f / sqrtf(fmaxf(sq / n - mean * mean, 0.f));
  float* out = norm + bh * (max_text + 1) * F + j;
  for (int64_t r = 0; r <= ntext[b]; ++r) out[r * F] = round_to<T>((col[(start + r) * S] - mean) * rstd);
}

// rank-th smallest of the window without storing it (width <= 129: no per-thread array): the element with fewer than rank + 1
// smaller ones and at least rank + 1 not greater; NaN when none qualifies (a NaN in the window)
__device__ __forceinline__ float window_select(const float* row, int j, int n, int rank) {
  auto at = [&](int k) {
    int read = abs(j + k);
    if (read >= n) read = 2 * n - read - 2;
    return row[read];
  };
  for (int c = -rank; c <= rank; ++c) {
    const float a = at(c);
    int less = 0, leq = 0;
    for (int k = -rank; k <= rank; ++k) {
      const float v = at(k);
      less += v < a;
      leq += v <= a;
    }
    if (less <= rank && rank < leq) return a;
  }
  return NAN;
}

// ops::MedianFilter (median_filter_cpu.cc: read = |j + k|, mirrored as depth - (read - depth) - 2) then ops::Mean(1) over the
// heads.  One CTA per (entry, DTW row); each head's row is staged in shared memory.
template <typename T>
__global__ void __launch_bounds__(256) align_median_mean_kernel(const float* __restrict__ norm, const int32_t* __restrict__ nf,
                                                                const int32_t* __restrict__ ntext, int heads, int64_t max_text,
                                                                int64_t F, int width, float* __restrict__ matrix) {
  extern __shared__ float smem[];
  float* row = smem;             // [F]
  float* acc = smem + F;         // [F]
  const int64_t b = blockIdx.x / (max_text + 1), r = blockIdx.x % (max_text + 1);
  const int n = nf[b];
  float* out = matrix + static_cast<int64_t>(blockIdx.x) * F;
  if (r > ntext[b] || n <= 0) {
    for (int64_t j = threadIdx.x; j < F; j += blockDim.x) out[j] = 0.f;
    return;
  }
  const int rank = width / 2;
  const bool pass = width <= 1 || n <= rank;
  for (int j = threadIdx.x; j < n; j += blockDim.x) acc[j] = 0.f;
  for (int h = 0; h < heads; ++h) {
    __syncthreads();
    const float* src = norm + ((b * heads + h) * (max_text + 1) + r) * F;
    for (int j = threadIdx.x; j < n; j += blockDim.x) row[j] = src[j];
    __syncthreads();
    for (int j = threadIdx.x; j < n; j += blockDim.x) acc[j] += pass ? row[j] : window_select(row, j, n, rank);
  }
  const float nh = static_cast<float>(heads);
  for (int64_t j = threadIdx.x; j < F; j += blockDim.x) out[j] = j < n ? round_to<T>(acc[j] / nh) : 0.f;
}

// ops::Gather(-1, 1) of the language ids then ops::SoftMax (whisper.cc:622-623), in T: one warp per row
template <typename T>
__global__ void __launch_bounds__(32) gather_softmax_kernel(const T* __restrict__ x, int64_t ld, const int32_t* __restrict__ ids,
                                                            int n, float* __restrict__ probs) {
  const int lane = threadIdx.x;
  const T* xr = x + static_cast<int64_t>(blockIdx.x) * ld;
  float m = -INFINITY;
  for (int k = lane; k < n; k += 32) m = fmaxf(m, to_f32(xr[ids[k]]));
  m = warp_max(m);
  float s = 0.f;
  for (int k = lane; k < n; k += 32) s += expf(to_f32(xr[ids[k]]) - m);
  s = warp_sum(s);
  const float inv = 1.f / s;
  for (int k = lane; k < n; k += 32) probs[static_cast<int64_t>(blockIdx.x) * n + k] = round_to<T>(expf(to_f32(xr[ids[k]]) - m) * inv);
}

}  // namespace

void launch_align_softmax(float* scores, const int32_t* nf, const int32_t* len, int64_t batch, int heads, int64_t time, int64_t S,
                          int dtype, cudaStream_t st) {
  const int64_t units = batch * heads * time;
  if (units == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (align_softmax_kernel<T><<<div_up(units, kAlignWarps), kAlignWarps * 32, 0, st>>>(scores, nf, len, units,
                                                                                                              heads, time, S)));
  check_launch();
}

void launch_align_standardize(const float* scores, const int32_t* nf, const int32_t* len, const int32_t* ntext, int64_t batch,
                              int heads, int64_t time, int64_t S, int64_t rows, int64_t start, int64_t max_text, int64_t F,
                              float* norm, int dtype, cudaStream_t st) {
  if (batch * heads == 0 || F == 0) return;
  CT2_REQUIRE(F <= S, "align_standardize: more frames than keys");
  const dim3 grid(div_up(F, 128), static_cast<unsigned>(batch * heads));
  CT2_DISPATCH_DTYPE(dtype, (align_standardize_kernel<T><<<grid, 128, 0, st>>>(scores, nf, len, ntext, heads, time, S, rows, start,
                                                                               max_text, F, norm)));
  check_launch();
}

void launch_align_median_mean(const float* norm, const int32_t* nf, const int32_t* ntext, int64_t batch, int heads,
                              int64_t max_text, int64_t F, int width, float* matrix, int dtype, cudaStream_t st) {
  if (batch == 0 || F == 0) return;
  CT2_REQUIRE(width <= 1 || (width % 2 == 1 && width <= 129), "MedianFilter width must be odd and at most 129");
  const size_t smem = 2 * static_cast<size_t>(F) * sizeof(float);
  CT2_REQUIRE(smem <= 48 * 1024, "align_median_mean: too many frames");
  CT2_DISPATCH_DTYPE(dtype, (align_median_mean_kernel<T><<<static_cast<unsigned>(batch * (max_text + 1)), 256, smem, st>>>(
                                norm, nf, ntext, heads, max_text, F, width, matrix)));
  check_launch();
}

void launch_gather_softmax(const void* x, int64_t rows, int64_t ld, const int32_t* ids, int n, float* probs, int dtype,
                           cudaStream_t st) {
  if (rows == 0 || n == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (gather_softmax_kernel<T><<<static_cast<unsigned>(rows), 32, 0, st>>>(static_cast<const T*>(x), ld, ids,
                                                                                                  n, probs)));
  check_launch();
}

}  // namespace ct2b200
