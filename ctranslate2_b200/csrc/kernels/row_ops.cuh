// row_ops.cuh — the "-> int8 row" producers of the decode step as ONE device function of 128 threads, run by
// the row kernel of rowwise.cu (one CTA per row):
//   MODE 0: Quantize(x)                         ops::Quantize            src/ops/quantize_gpu.cu:57-105
//   MODE 1: Quantize(T(RMSNorm(x, gamma)))      ops::RMSNorm + Quantize  src/ops/rms_norm_gpu.cu:19-63
//   MODE 2: Quantize(T(a * b))                  ops::Mul + Quantize      src/layers/transformer.cc:31-37
//   MODE 3: T(RMSNorm(x, gamma)) written as T   (same summation order as MODE 1, so 1 == Quantize o 3 bit-exactly)
// The row is read ONCE with 16-byte loads and kept in registers in its storage type (NV vectors per thread; zero padding
// adds exact zeros, so every NV >= ceil(cols / (128 * N)) gives the same bits); the sum of squares is accumulated per
// thread in element order, then lanes (xor tree), then the four warps as (w0 + w1) + (w2 + w3).
#pragma once

#include "../common.cuh"

namespace ct2b200 {
namespace rowop {

constexpr int kThreads = 128;
constexpr int kMaxNV = 16;        // 128 threads x 16 vectors of 16 bytes: rows up to 16384 fp16 / 8192 fp32 elements

__device__ __forceinline__ void bar128(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// `red` = 4 floats of shared memory; t = thread index within the 128; result broadcast to the 128 threads
template <bool kMax>
__device__ __forceinline__ float reduce128(float v, float* red, int t, int bar_id) {
  v = kMax ? warp_max(v) : warp_sum(v);
  bar128(bar_id);                                   // protect `red` from a previous use
  if ((t & 31) == 0) red[t >> 5] = v;
  bar128(bar_id);
  const float r0 = red[0], r1 = red[1], r2 = red[2], r3 = red[3];
  return kMax ? fmaxf(fmaxf(r0, r1), fmaxf(r2, r3)) : ((r0 + r1) + (r2 + r3));
}

template <typename T>
__host__ __device__ inline bool covers(int64_t cols) {
  constexpr int N = 16 / static_cast<int>(sizeof(T));
  return cols % N == 0 && cols / N <= static_cast<int64_t>(kThreads) * kMaxNV;
}
// vectors per thread used for a row of `cols` elements: 4 (rows up to 4096 fp16) or kMaxNV
template <typename T>
__host__ __device__ inline int nv_for(int64_t cols) {
  constexpr int N = 16 / static_cast<int>(sizeof(T));
  return cols / N <= static_cast<int64_t>(kThreads) * 4 ? 4 : kMaxNV;
}

template <typename T, int MODE, int NV>
__device__ __forceinline__ void row_op_128(const T* __restrict__ xr, const T* __restrict__ aux, int64_t cols, float eps,
                                           bool use_residual, int8_t* __restrict__ qr, float* __restrict__ scale_out,
                                           T* __restrict__ y_row, float* red, int t, int bar_id) {
  constexpr int N = Vec16<T>::N;
  const int nv = static_cast<int>(cols / N);
  static_assert(NV <= kMaxNV, "NV");
  Vec16<T> d[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int vi = t + k * kThreads;
    if (vi < nv) {
      d[k] = ld16(xr + static_cast<int64_t>(vi) * N);
    } else {
#pragma unroll
      for (int i = 0; i < N; ++i) d[k].v[i] = from_f32<T>(0.f);
    }
  }
  if constexpr (MODE == 2) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int vi = t + k * kThreads;
      if (vi < nv) {
        const Vec16<T> b = ld16(aux + static_cast<int64_t>(vi) * N);
#pragma unroll
        for (int i = 0; i < N; ++i) d[k].v[i] = from_f32<T>(to_f32(d[k].v[i]) * to_f32(b.v[i]));
      }
    }
  }
  if constexpr (MODE == 1 || MODE == 3) {
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k)
#pragma unroll
      for (int i = 0; i < N; ++i) {
        const float v = to_f32(d[k].v[i]);
        ss += v * v;
      }
    ss = reduce128<false>(ss, red, t, bar_id);
    const float inv = rsqrtf(ss / static_cast<float>(cols) + eps);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int vi = t + k * kThreads;
      if (vi < nv) {
        const Vec16<T> g = ld16(aux + static_cast<int64_t>(vi) * N);
#pragma unroll
        for (int i = 0; i < N; ++i) {
          const float gg = to_f32(g.v[i]) + (use_residual ? 1.f : 0.f);
          d[k].v[i] = from_f32<T>(to_f32(d[k].v[i]) * inv * gg);
        }
      }
    }
  }
  if constexpr (MODE == 3) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int vi = t + k * kThreads;
      if (vi < nv) st16(y_row + static_cast<int64_t>(vi) * N, d[k]);
    }
    return;
  }
  float amax = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k)
#pragma unroll
    for (int i = 0; i < N; ++i) amax = fmaxf(amax, fabsf(to_f32(d[k].v[i])));
  amax = reduce128<true>(amax, red, t, bar_id);
  const float s = amax != 0.f ? 127.f / amax : 1.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int vi = t + k * kThreads;
    if (vi < nv) {
      int8_t out[N];
#pragma unroll
      for (int i = 0; i < N; ++i) out[i] = static_cast<int8_t>(nearbyintf(to_f32(d[k].v[i]) * s));
      int8_t* dst = qr + static_cast<int64_t>(vi) * N;
      if constexpr (N == 8) *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<uint2*>(out);
      else *reinterpret_cast<uint32_t*>(dst) = *reinterpret_cast<uint32_t*>(out);
    }
  }
  if (t == 0) *scale_out = s;
}

}  // namespace rowop
}  // namespace ct2b200
