// gemm_decode_common.cuh — pieces shared by the decode (weight-streaming) wgmma kernels: gemm_decode.cu (INT8 / f16
// weights) and awq_decode.cu (AWQ-INT4 weights): fused epilogue of one output channel, cluster barriers, planner helpers.
#pragma once

#include <algorithm>
#include <cstdlib>

#include "gemm_common.cuh"
#include "tc_common.cuh"

namespace ct2b200 {
namespace dec {

using namespace tc;

constexpr int kMaxStages = 10;

// defaults of the switchable kernels (1 = on)
#define CT2B200_DEFAULT_AWQ_DECODE 1
#define CT2B200_DEFAULT_AWQ_GEMV 1
#define CT2B200_DEFAULT_GEMM_DECODE_MAXM 64

struct DecParams {
  int64_t n;            // output channels (weight rows)
  int64_t m;            // activation rows
  int kb_total;         // K blocks of 128 bytes
  int tile_rows;        // weight rows per tile (multiple of 8, <= 128)
  int stages;           // operand ring depth
  // fused epilogue
  const float* a_scale;     // [m]   INT8: activation row scales
  const float* w_scale0;    // [n]   INT8: weight row scales (gate for GLU)
  const float* w_scale1;    // [n]   GLU: up scales
  const void* bias;         // [n] T or null
  const void* residual;     // [m, n] T or null
  void* y;                  // [m, n] T
  int act;
  int64_t ldy;
};


template <int KIND> struct Elem { static constexpr int bytes = KIND == 0 ? 1 : 2; };

static __device__ __noinline__ float dec_act(float x, int act) {
  if (act == CT2B200_ACT_SWISH) return __fdividef(x, 1.f + __expf(-x));
  return apply_act(x, act);
}

__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

// One thread finishes NC output elements of its channel `arow`: batch rows col0, col0 + cstep, ...
// r[w][j] = raw accumulators (int32 or fp32 bits).
template <typename T, int KIND, int NB, int NC>
__device__ __forceinline__ void dec_finish(const DecParams& p, const uint32_t (&r)[NB][NC], int64_t arow, int col0,
                                           int cstep, int nvalid, float sw0, float sw1, float bias_t) {
  T* yp = static_cast<T*>(p.y) + static_cast<int64_t>(col0) * p.ldy + arow;
  const T* rp = p.residual ? static_cast<const T*>(p.residual) + static_cast<int64_t>(col0) * p.ldy + arow : nullptr;
  const int64_t step = static_cast<int64_t>(cstep) * p.ldy;
  const int act = p.act;
  float res[NC];
  float sx[NC];
#pragma unroll
  for (int j = 0; j < NC; ++j) {                       // all loads first: one memory round trip
    const bool ok = j < nvalid && col0 + j * cstep < p.m;
    res[j] = (rp && ok) ? to_f32(rp[j * step]) : 0.f;
    if constexpr (KIND == 0) sx[j] = ok ? p.a_scale[col0 + j * cstep] : 1.f;   // plain load: may be written by this grid (pre-phase)
  }
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    if (j >= nvalid || col0 + j * cstep >= p.m) break;
    float v;
    if constexpr (NB == 2) {
      float gate, up;
      if constexpr (KIND == 0) {
        gate = __fdividef(static_cast<float>(static_cast<int32_t>(r[0][j])), sx[j] * sw0);
        up = __fdividef(static_cast<float>(static_cast<int32_t>(r[1][j])), sx[j] * sw1);
      } else {
        gate = __uint_as_float(r[0][j]);
        up = __uint_as_float(r[1][j]);
      }
      gate = round_to<T>(dec_act(round_to<T>(gate), act));
      v = gate * round_to<T>(up);
    } else {
      if constexpr (KIND == 0) v = __fdividef(static_cast<float>(static_cast<int32_t>(r[0][j])), sx[j] * sw0);
      else v = __uint_as_float(r[0][j]);
      // bias_t / res[j] are 0 when absent: adding them is exact, which keeps the unrolled code free of branch versions
      v = round_to<T>(round_to<T>(v) + bias_t);
      if (act >= 0) v = round_to<T>(dec_act(v, act));
      v = v + res[j];
    }
    yp[j * step] = from_f32<T>(v);
  }
}


inline int env_int(const char* name, int fallback) {
  const char* e = std::getenv(name);
  return e ? std::atoi(e) : fallback;
}

// co-resident clusters of `cs` CTAs of `kernel` (cs == 1: one CTA per SM)
template <typename K>
int max_clusters(K kernel, int cs, int threads, size_t smem, int sm_count) {
  if (cs == 1) return sm_count;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<unsigned>(cs * sm_count));
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) {
    cudaGetLastError();
    return sm_count / cs * 3 / 4;                      // conservative
  }
  return n;
}

inline int sm_count_of_current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  static int cached_dev = -1, cached = 132;
  if (cached_dev != dev) {
    cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev);
    cached_dev = dev;
  }
  return cached;
}

}  // namespace dec
}  // namespace ct2b200
