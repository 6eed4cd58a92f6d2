// rowwise.cu — the HBM/L2-bound row kernels of the decode path: Quantize, RMSNorm(+Quantize),
// Mul+Quantize, Dequantize (both forms), Rotary, SoftMax, TopK, Gather, INT8 Embeddings.
// One CTA per row (grid = rows); 16-byte vector accesses whenever the row pitch allows it.
// Reference kernels these replace are cited per launcher (paths relative to the reference tree).
#include <cstdlib>
#include <mutex>
#include <set>
#include <tuple>

#include "../common.cuh"
#include "row_ops.cuh"

namespace ct2b200 {

std::atomic<int64_t> g_kernel_launches{0};

bool mark_configured(const void* kernel, int tag) {
  static std::mutex mu;
  static std::set<std::tuple<const void*, int, int>> seen;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(mu);
  return seen.insert({kernel, tag, dev}).second;
}

namespace {
thread_local bool t_pdl_fence = false;
}

bool pdl_enabled() {
  static const bool on = [] {
    const char* e = std::getenv("CT2B200_PDL");
    return !(e && e[0] == '0');
  }();
  if (t_pdl_fence) {            // one launch on this thread with a full stream dependency (pdl_fence_next_launch)
    t_pdl_fence = false;
    return false;
  }
  return on;
}

void pdl_fence_next_launch() { t_pdl_fence = true; }

constexpr int kRowThreads = 256;

template <typename T>
__device__ __forceinline__ bool row_vec_ok(const void* p, int64_t cols) {
  return (cols % Vec16<T>::N == 0) && ((reinterpret_cast<uintptr_t>(p) & 15) == 0);
}

// quantize one row held in global memory `y(j)`: computes amax of |y|, the scale, writes int8.
// F(j) must return the value of element j (float, already rounded to T by the caller).
template <typename F>
__device__ __forceinline__ void quantize_row_generic(F value_at, int64_t cols, bool round, int8_t* q_row,
                                                     float* scale_out, float* red) {
  float amax = 0.f;
  for (int64_t j = threadIdx.x; j < cols; j += blockDim.x) amax = fmaxf(amax, fabsf(value_at(j)));
  amax = block_reduce<true>(amax, red);
  const float scale = amax != 0.f ? 127.f / amax : 1.f;
  for (int64_t j = threadIdx.x; j < cols; j += blockDim.x) {
    const float v = value_at(j) * scale;
    q_row[j] = static_cast<int8_t>(round ? nearbyintf(v) : v);
  }
  if (threadIdx.x == 0) *scale_out = scale;
}

// ---------------------------------------------------------------------------------------------
// ops::Quantize  (src/ops/quantize_gpu.cu:57-105)
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kRowThreads) quantize_rows_kernel(const T* __restrict__ x, int64_t cols,
                                                                    bool round, int8_t* __restrict__ q,
                                                                    float* __restrict__ scale) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const T* xr = x + row * cols;
  int8_t* qr = q + row * cols;
  if (row_vec_ok<T>(xr, cols) && (reinterpret_cast<uintptr_t>(qr) % (Vec16<T>::N) == 0)) {
    constexpr int N = Vec16<T>::N;
    const int64_t nv = cols / N;
    float amax = 0.f;
    for (int64_t v = threadIdx.x; v < nv; v += blockDim.x) {
      const Vec16<T> d = ld16(xr + v * N);
#pragma unroll
      for (int i = 0; i < N; ++i) amax = fmaxf(amax, fabsf(to_f32(d.v[i])));
    }
    amax = block_reduce<true>(amax, red);
    const float s = amax != 0.f ? 127.f / amax : 1.f;
    for (int64_t v = threadIdx.x; v < nv; v += blockDim.x) {
      const Vec16<T> d = ld16(xr + v * N);   // second read hits L1/L2
      int8_t out[N];
#pragma unroll
      for (int i = 0; i < N; ++i) {
        const float f = to_f32(d.v[i]) * s;
        out[i] = static_cast<int8_t>(round ? nearbyintf(f) : f);
      }
      if constexpr (N == 8) *reinterpret_cast<uint2*>(qr + v * N) = *reinterpret_cast<uint2*>(out);
      else *reinterpret_cast<uint32_t*>(qr + v * N) = *reinterpret_cast<uint32_t*>(out);
    }
    if (threadIdx.x == 0) scale[row] = s;
  } else {
    quantize_row_generic([&](int64_t j) { return to_f32(xr[j]); }, cols, round, qr, scale + row, red);
  }
}

// ---------------------------------------------------------------------------------------------
// ops::RMSNorm (src/ops/rms_norm_gpu.cu:19-63) and RMSNorm + Quantize fused
// ---------------------------------------------------------------------------------------------
template <typename T, bool kQuantize>
__global__ void __launch_bounds__(kRowThreads) rms_norm_kernel(const T* __restrict__ gamma,
                                                               const T* __restrict__ x, int64_t cols, float eps,
                                                               bool use_residual, T* __restrict__ y,
                                                               int8_t* __restrict__ q, float* __restrict__ scale) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const T* xr = x + row * cols;
  float ss = 0.f;
  for (int64_t j = threadIdx.x; j < cols; j += blockDim.x) {
    const float v = to_f32(xr[j]);
    ss += v * v;
  }
  ss = block_reduce<false>(ss, red);
  const float inv = rsqrtf(ss / static_cast<float>(cols) + eps);
  auto normed = [&](int64_t j) {
    const float g = to_f32(gamma[j]) + (use_residual ? 1.f : 0.f);
    return round_to<T>(to_f32(xr[j]) * inv * g);
  };
  if constexpr (!kQuantize) {
    T* yr = y + row * cols;
    for (int64_t j = threadIdx.x; j < cols; j += blockDim.x) yr[j] = from_f32<T>(normed(j));
  } else {
    quantize_row_generic(normed, cols, true, q + row * cols, scale + row, red);
  }
}

// ops::Mul + ops::Quantize of the SwiGLU product (transformer.cc:31-37)
template <typename T>
__global__ void __launch_bounds__(kRowThreads) mul_quantize_kernel(const T* __restrict__ a, const T* __restrict__ b,
                                                                   int64_t cols, int8_t* __restrict__ q,
                                                                   float* __restrict__ scale) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const T* ar = a + row * cols;
  const T* br = b + row * cols;
  quantize_row_generic([&](int64_t j) { return round_to<T>(to_f32(ar[j]) * to_f32(br[j])); }, cols, true,
                       q + row * cols, scale + row, red);
}

// ---------------------------------------------------------------------------------------------
// Register-resident fast path of the "-> int8 row" producers of the decode step (row_ops.cuh: MODE 0 Quantize, 1 RMSNorm +
// Quantize, 2 Mul + Quantize, 3 RMSNorm written as T).  One CTA of 128 threads per row, one global round trip.
// ---------------------------------------------------------------------------------------------
template <typename T, int MODE, int NV>
__global__ void __launch_bounds__(rowop::kThreads) row_to_int8_kernel(const T* __restrict__ x, const T* __restrict__ aux,
                                                                      int64_t cols, float eps, bool use_residual,
                                                                      int8_t* __restrict__ q, float* __restrict__ scale,
                                                                      T* __restrict__ y_out) {
  __shared__ float red[4];
  griddep_launch();
  griddep_wait();
  const int64_t row = blockIdx.x;
  const T* auxr = MODE == 2 ? aux + row * cols : aux;
  rowop::row_op_128<T, MODE, NV>(x + row * cols, auxr, cols, eps, use_residual, q ? q + row * cols : nullptr,
                             scale ? scale + row : nullptr, y_out ? y_out + row * cols : nullptr, red,
                             static_cast<int>(threadIdx.x), 1);
}

// returns false when the shape/alignment is not covered (caller falls back to the generic kernels)
template <typename T, int MODE>
bool launch_row_to_int8(const T* x, const T* aux, int64_t rows, int64_t cols, float eps, bool use_residual, int8_t* q,
                        float* scale, cudaStream_t st, T* y_out = nullptr) {
  if (!rowop::covers<T>(cols) || (reinterpret_cast<uintptr_t>(x) & 15) || (aux && (reinterpret_cast<uintptr_t>(aux) & 15)) ||
      (reinterpret_cast<uintptr_t>(q) & 7) || (reinterpret_cast<uintptr_t>(y_out) & 15))
    return false;
  if (rowop::nv_for<T>(cols) == 4)
    launch_pdl(row_to_int8_kernel<T, MODE, 4>, dim3(rows), dim3(rowop::kThreads), 0, st, x, aux, cols, eps, use_residual, q,
               scale, y_out);
  else
    launch_pdl(row_to_int8_kernel<T, MODE, rowop::kMaxNV>, dim3(rows), dim3(rowop::kThreads), 0, st, x, aux, cols, eps,
               use_residual, q, scale, y_out);
  return true;
}

// ---------------------------------------------------------------------------------------------
// ops::Dequantize  (src/ops/dequantize_gpu.cu:16-27 rows form, :30-144 GEMM-output form)
// ---------------------------------------------------------------------------------------------
// reciprocal = false: y = x / scale (the CUDA kernel of the reference, dequantize_gpu.cu:16-27); true: y = x * (1 / scale), the
// reference's CPU kernel (dequantize_cpu.cc:12-21), which is what converts int8 weights to float at load (model.cc:331-341)
template <typename T>
__global__ void dequantize_rows_kernel(const int8_t* __restrict__ x, const float* __restrict__ scale, int64_t cols,
                                       T* __restrict__ y, bool reciprocal) {
  const int64_t row = blockIdx.x;
  const float s = scale[row];
  const float r = __fdiv_rn(1.f, s);
  for (int64_t j = threadIdx.x; j < cols; j += blockDim.x) {
    const float v = static_cast<float>(x[row * cols + j]);
    y[row * cols + j] = from_f32<T>(reciprocal ? __fmul_rn(v, r) : __fdiv_rn(v, s));
  }
}

template <typename T>
__global__ void dequantize_gemm_output_kernel(const int32_t* __restrict__ c, DenseEpilogue e, int64_t n) {
  const int64_t i = blockIdx.x;
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) dense_epilogue_store<T>(e, c[i * n + j], i, j);
}

// layers::Embeddings with int8 weights (common.cc:64-81): gather row + scale, dequantize
template <typename T>
__global__ void embedding_s8_kernel(const int8_t* __restrict__ w, const float* __restrict__ scale,
                                    const int32_t* __restrict__ ids, int64_t depth, T* __restrict__ y) {
  griddep_launch();
  griddep_wait();
  const int64_t i = blockIdx.x;
  const int64_t id = ids[i];
  const float s = scale[id];
  const int8_t* wr = w + id * depth;
  for (int64_t j = threadIdx.x; j < depth; j += blockDim.x)
    y[i * depth + j] = from_f32<T>(__fdiv_rn(static_cast<float>(wr[j]), s));
}

// ops::Gather axis 0 (src/ops/gather_gpu.cu:52-91): copy rows of `row_bytes`
__global__ void gather_rows_kernel(const uint8_t* __restrict__ data, const int32_t* __restrict__ ids,
                                   int64_t row_bytes, uint8_t* __restrict__ out) {
  const int64_t i = blockIdx.x;
  const uint8_t* src = data + static_cast<int64_t>(ids[i]) * row_bytes;
  uint8_t* dst = out + i * row_bytes;
  if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst) | row_bytes) & 15) == 0) {
    for (int64_t j = threadIdx.x; j < row_bytes / 16; j += blockDim.x)
      reinterpret_cast<uint4*>(dst)[j] = reinterpret_cast<const uint4*>(src)[j];
  } else {
    for (int64_t j = threadIdx.x; j < row_bytes; j += blockDim.x) dst[j] = src[j];
  }
}

// ---------------------------------------------------------------------------------------------
// ops::Rotary (src/ops/rotary_gpu.cu:27-85): x rows [batch*time, depth], sin/cos [time, ndims] in T.
// The reference evaluates the rotation in T; we evaluate in fp32 and round once (closer to exact).
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void rotary_kernel(const T* __restrict__ x, const T* __restrict__ sin, const T* __restrict__ cos,
                              int64_t time, int64_t depth, int64_t ndims, bool interleave, T* __restrict__ y) {
  const int64_t row = blockIdx.x;
  const int64_t t = row % time;
  const T* xr = x + row * depth;
  T* yr = y + row * depth;
  const int64_t half = ndims / 2;
  for (int64_t i = threadIdx.x; i < depth; i += blockDim.x) {
    if (i >= ndims) {
      yr[i] = xr[i];
      continue;
    }
    float other;
    if (interleave) other = (i % 2 == 0) ? -to_f32(xr[i + 1]) : to_f32(xr[i - 1]);
    else other = (i < half) ? -to_f32(xr[i + half]) : to_f32(xr[i - half]);
    yr[i] = from_f32<T>(to_f32(xr[i]) * to_f32(cos[t * ndims + i]) + other * to_f32(sin[t * ndims + i]));
  }
}

// ---------------------------------------------------------------------------------------------
// ops::SoftMax / LogSoftMax with optional lengths (src/ops/softmax_gpu.cu:190-256)
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kRowThreads) softmax_kernel(const T* __restrict__ x,
                                                              const int32_t* __restrict__ lengths, int64_t cols,
                                                              bool log, T* __restrict__ y) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const T* xr = x + row * cols;
  T* yr = y + row * cols;
  const int64_t n = lengths ? min(static_cast<int64_t>(lengths[row]), cols) : cols;
  float m = -INFINITY;
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) m = fmaxf(m, to_f32(xr[j]));
  m = block_reduce<true>(m, red);
  float s = 0.f;
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) s += expf(to_f32(xr[j]) - m);
  s = block_reduce<false>(s, red);
  const float logs = logf(s);
  for (int64_t j = threadIdx.x; j < cols; j += blockDim.x) {
    float v = 0.f;
    if (j < n) v = log ? (to_f32(xr[j]) - m - logs) : expf(to_f32(xr[j]) - m) / s;
    yr[j] = from_f32<T>(v);
  }
}

// ---------------------------------------------------------------------------------------------
// ops::LogSoftMax + ops::Gather(axis -1, batch_dims 1) fused (src/scoring.cc:50-56): y[row] = float(T(x[id] - max -
// log(sum exp(x - max)))), the value softmax_kernel's log path stores at column id.  The row is read once: each thread keeps
// a running (max, sum) over 16-byte vectors (scalar head up to the first aligned element, scalar tail), the pairs are merged
// across the block, and the target element is read on its own.  The log-probabilities are never written back.  The exps of
// one vector are summed in fp32, the running sums and the final difference in fp64: the result is then within one unit of
// T's last place of the exact value also for fp32 rows of 128K columns, where an fp32 running sum is not.
// ---------------------------------------------------------------------------------------------
struct MaxSum { float m; double s; };
__device__ __forceinline__ MaxSum max_sum_merge(MaxSum a, MaxSum b) {
  const float m = fmaxf(a.m, b.m);
  if (m == -INFINITY) return {m, 0.0};
  return {m, a.s * expf(a.m - m) + b.s * expf(b.m - m)};
}
__device__ __forceinline__ MaxSum warp_max_sum(MaxSum v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v = max_sum_merge(v, {__shfl_xor_sync(0xffffffffu, v.m, o), __shfl_xor_sync(0xffffffffu, v.s, o)});
  return v;
}

// PROB: the probability T(exp(x[id] - logsumexp(x))) instead, 0 for an id outside the row (SoftMax over [0, cols) + Gather,
// models/whisper.cc:495-502, where the mask leaves 0 past the limit).
template <typename T, bool PROB = false>
__global__ void __launch_bounds__(kRowThreads) log_softmax_gather_kernel(const T* __restrict__ x,
                                                                         const int32_t* __restrict__ ids, int64_t cols,
                                                                         int64_t ld, float* __restrict__ y) {
  __shared__ MaxSum red[kRowThreads / 32];
  constexpr int N = Vec16<T>::N;
  const int64_t row = blockIdx.x;
  const T* xr = x + row * ld;
  // elements before the first 16-byte boundary (rows of an odd width start anywhere); T-aligned rows are assumed
  const int64_t head = min(cols, static_cast<int64_t>(((16 - (reinterpret_cast<uintptr_t>(xr) & 15)) & 15) / sizeof(T)));
  const int64_t nv = (cols - head) / N;
  const T* xv = xr + head;
  MaxSum acc{-INFINITY, 0.0};
  auto add = [&](float v) {               // one scalar element
    if (v > acc.m) {
      acc.s = acc.s * expf(acc.m - v) + 1.0;
      acc.m = v;
    } else if (v != -INFINITY) {
      acc.s += expf(v - acc.m);
    }
  };
  if (threadIdx.x < head) add(to_f32(xr[threadIdx.x]));
#pragma unroll 4
  for (int64_t v = threadIdx.x; v < nv; v += blockDim.x) {
    const Vec16<T> d = ld16(xv + v * N);
    float f[N];
    float vm = -INFINITY;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      f[i] = to_f32(d.v[i]);
      vm = fmaxf(vm, f[i]);
    }
    const float m = fmaxf(acc.m, vm);
    if (m == -INFINITY) continue;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < N; ++i) s += expf(f[i] - m);
    acc = {m, (m == acc.m ? acc.s : acc.s * expf(acc.m - m)) + s};
  }
  for (int64_t j = head + nv * N + threadIdx.x; j < cols; j += blockDim.x) add(to_f32(xr[j]));
  acc = warp_max_sum(acc);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (warp == 0) {
    acc = lane < kRowThreads / 32 ? red[lane] : MaxSum{-INFINITY, 0.0};
    acc = warp_max_sum(acc);
    if (lane == 0) {
      const int64_t id = ids[row];
      // an id outside the row has no log-probability: NaN rather than a read past the row
      const double v = static_cast<double>(to_f32(xr[id >= 0 && id < cols ? id : 0])) - acc.m - log(acc.s);
      if constexpr (PROB) y[row] = id >= 0 && id < cols ? round_to<T>(static_cast<float>(exp(v))) : 0.f;
      else y[row] = id >= 0 && id < cols ? round_to<T>(static_cast<float>(v)) : NAN;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// ops::TopK (src/ops/topk_gpu.cu:181-335).  k passes of a block arg-max over (value desc, index asc):
// a strict total order, so exact ties resolve lowest-index-first regardless of the reduction tree
// (the reference's cub tree does not guarantee that — SURVEY §8 a17).  The input is not mutated:
// pass p only considers elements strictly "after" the previous winner in that order.
// ---------------------------------------------------------------------------------------------
struct TopKItem { float v; int32_t i; };
__device__ __forceinline__ bool topk_better(float v1, int32_t i1, float v2, int32_t i2) {
  return v1 > v2 || (v1 == v2 && i1 < i2);
}
__device__ __forceinline__ TopKItem topk_warp_best(TopKItem a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v = __shfl_xor_sync(0xffffffffu, a.v, o);
    const int32_t i = __shfl_xor_sync(0xffffffffu, a.i, o);
    if (topk_better(v, i, a.v, a.i)) { a.v = v; a.i = i; }
  }
  return a;
}

template <typename T>
__global__ void __launch_bounds__(1024) topk_kernel(const T* __restrict__ x, int64_t cols, int k,
                                                    T* __restrict__ values, int32_t* __restrict__ indices) {
  __shared__ float sv[32];
  __shared__ int32_t si[32];
  __shared__ TopKItem prev_s;
  const int64_t row = blockIdx.x;
  const T* xr = x + row * cols;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  TopKItem prev{INFINITY, -1};
  for (int p = 0; p < k; ++p) {
    TopKItem best{-INFINITY, INT32_MAX};
    for (int64_t j = threadIdx.x; j < cols; j += blockDim.x) {
      const float v = to_f32(xr[j]);
      const int32_t jj = static_cast<int32_t>(j);
      // candidate must come strictly after `prev` in (value desc, index asc) order
      const bool after_prev = p == 0 || topk_better(prev.v, prev.i, v, jj);
      if (after_prev && topk_better(v, jj, best.v, best.i)) { best.v = v; best.i = jj; }
    }
    best = topk_warp_best(best);
    if (lane == 0) { sv[warp] = best.v; si[warp] = best.i; }
    __syncthreads();
    if (warp == 0) {
      TopKItem b{lane < nw ? sv[lane] : -INFINITY, lane < nw ? si[lane] : INT32_MAX};
      b = topk_warp_best(b);
      if (lane == 0) {
        prev_s = b;
        if (b.i != INT32_MAX) {
          values[row * k + p] = xr[b.i];
          indices[row * k + p] = b.i;
        }
      }
    }
    __syncthreads();
    prev = prev_s;
  }
}

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
void launch_quantize_rows(const void* x, int dtype, int64_t rows, int64_t cols, bool round, int8_t* q,
                          float* scale, cudaStream_t st) {
  if (rows == 0) return;
  bool done = false;
  if (round) CT2_DISPATCH_DTYPE(dtype, (done = launch_row_to_int8<T, 0>(static_cast<const T*>(x), nullptr, rows, cols, 0.f, false, q, scale, st)));
  if (!done)
    CT2_DISPATCH_DTYPE(dtype, (quantize_rows_kernel<T><<<rows, kRowThreads, 0, st>>>(
                                  static_cast<const T*>(x), cols, round, q, scale)));
  check_launch();
}

void launch_rms_norm(const void* gamma, const void* x, int64_t rows, int64_t cols, float eps, bool use_residual,
                     void* y, int8_t* q, float* scale, int dtype, cudaStream_t st) {
  if (rows == 0) return;
  if (q) {
    bool done = false;
    CT2_DISPATCH_DTYPE(dtype, (done = launch_row_to_int8<T, 1>(static_cast<const T*>(x), static_cast<const T*>(gamma), rows, cols, eps, use_residual, q, scale, st)));
    if (!done)
      CT2_DISPATCH_DTYPE(dtype, (rms_norm_kernel<T, true><<<rows, kRowThreads, 0, st>>>(
                                    static_cast<const T*>(gamma), static_cast<const T*>(x), cols, eps,
                                    use_residual, nullptr, q, scale)));
  } else {
    bool done = false;
    CT2_DISPATCH_DTYPE(dtype, (done = launch_row_to_int8<T, 3>(static_cast<const T*>(x), static_cast<const T*>(gamma), rows, cols, eps, use_residual, nullptr, nullptr, st, static_cast<T*>(y))));
    if (!done)
      CT2_DISPATCH_DTYPE(dtype, (rms_norm_kernel<T, false><<<rows, kRowThreads, 0, st>>>(
                                    static_cast<const T*>(gamma), static_cast<const T*>(x), cols, eps,
                                    use_residual, static_cast<T*>(y), nullptr, nullptr)));
  }
  check_launch();
}

void launch_mul_quantize(const void* a, const void* b, int64_t rows, int64_t cols, int8_t* q, float* scale,
                         int dtype, cudaStream_t st) {
  if (rows == 0) return;
  bool done = false;
  CT2_DISPATCH_DTYPE(dtype, (done = launch_row_to_int8<T, 2>(static_cast<const T*>(a), static_cast<const T*>(b), rows, cols, 0.f, false, q, scale, st)));
  if (!done)
    CT2_DISPATCH_DTYPE(dtype, (mul_quantize_kernel<T><<<rows, kRowThreads, 0, st>>>(
                                  static_cast<const T*>(a), static_cast<const T*>(b), cols, q, scale)));
  check_launch();
}

void launch_dequantize_rows(const int8_t* x, const float* scale, int64_t rows, int64_t cols, void* y, int dtype,
                            cudaStream_t st, bool reciprocal) {
  if (rows == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (dequantize_rows_kernel<T><<<rows, 256, 0, st>>>(x, scale, cols, static_cast<T*>(y), reciprocal)));
  check_launch();
}

void launch_dequantize_gemm_output(const int32_t* c, const DenseEpilogue& e, int64_t m, int64_t n, int dtype,
                                   cudaStream_t st) {
  if (m == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (dequantize_gemm_output_kernel<T><<<m, 256, 0, st>>>(c, e, n)));
  check_launch();
}

void launch_embedding_s8(const int8_t* w, const float* scale, const int32_t* ids, int64_t num_ids, int64_t depth,
                         void* y, int dtype, cudaStream_t st) {
  if (num_ids == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (launch_pdl(embedding_s8_kernel<T>, dim3(num_ids), dim3(256), 0, st, w, scale, ids, depth,
                                        static_cast<T*>(y))));
  check_launch();
}

void launch_gather_rows(const void* data, const int32_t* ids, int64_t num_ids, int64_t row_bytes, void* out,
                        cudaStream_t st) {
  if (num_ids == 0) return;
  gather_rows_kernel<<<num_ids, 256, 0, st>>>(static_cast<const uint8_t*>(data), ids, row_bytes,
                                              static_cast<uint8_t*>(out));
  check_launch();
}

void launch_rotary(const void* x, const void* sin, const void* cos, int64_t batch, int64_t time, int64_t depth,
                   int64_t ndims, bool interleave, void* y, int dtype, cudaStream_t st) {
  if (batch * time == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (rotary_kernel<T><<<batch * time, 128, 0, st>>>(
                                static_cast<const T*>(x), static_cast<const T*>(sin), static_cast<const T*>(cos),
                                time, depth, ndims, interleave, static_cast<T*>(y))));
  check_launch();
}

void launch_softmax(const void* x, const int32_t* lengths, int64_t rows, int64_t cols, bool log, void* y,
                    int dtype, cudaStream_t st) {
  if (rows == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (softmax_kernel<T><<<rows, kRowThreads, 0, st>>>(static_cast<const T*>(x), lengths,
                                                                           cols, log, static_cast<T*>(y))));
  check_launch();
}

void launch_log_softmax_gather(const void* x, const int32_t* ids, int64_t rows, int64_t cols, float* y, int dtype,
                               cudaStream_t st, int64_t ld) {
  if (rows == 0) return;
  CT2_DISPATCH_DTYPE(dtype, (log_softmax_gather_kernel<T><<<rows, kRowThreads, 0, st>>>(static_cast<const T*>(x), ids, cols,
                                                                                       ld > 0 ? ld : cols, y)));
  check_launch();
}

void launch_softmax_gather(const void* x, const int32_t* ids, int64_t rows, int64_t cols, int64_t ld, float* y, int dtype,
                           cudaStream_t st) {
  if (rows == 0) return;
  CT2_REQUIRE(cols >= 1 && ld >= cols, "softmax_gather: bad row width");
  CT2_DISPATCH_DTYPE(dtype, (log_softmax_gather_kernel<T, true><<<rows, kRowThreads, 0, st>>>(static_cast<const T*>(x), ids, cols,
                                                                                             ld, y)));
  check_launch();
}

void launch_topk(const void* x, int64_t rows, int64_t cols, int k, void* values, int32_t* indices, int dtype,
                 cudaStream_t st) {
  if (rows == 0) return;
  const int threads = cols >= 8192 ? 1024 : 256;
  CT2_DISPATCH_DTYPE(dtype, (topk_kernel<T><<<rows, threads, 0, st>>>(static_cast<const T*>(x), cols, k,
                                                                    static_cast<T*>(values), indices)));
  check_launch();
}

}  // namespace ct2b200
