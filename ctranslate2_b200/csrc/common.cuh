// common.cuh — shared device/host helpers for the sm_90a kernels of ct2b200.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <utility>

#include "../../include/ct2b200.h"

namespace ct2b200 {

// ---- error handling (mirrors THROW_RUNTIME_ERROR / CUDA_CHECK, reference src/cuda/utils.h:51-96) ----
struct InvalidArgument : std::invalid_argument {
  using std::invalid_argument::invalid_argument;
};

#define CT2_CUDA_CHECK(expr)                                                                         \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    if (_e != cudaSuccess)                                                                           \
      throw std::runtime_error(std::string("CUDA failed with error ") + cudaGetErrorString(_e) +    \
                               " at " + __FILE__ + ":" + std::to_string(__LINE__));                \
  } while (0)

#define CT2_REQUIRE(cond, msg)                                   \
  do {                                                           \
    if (!(cond)) throw ::ct2b200::InvalidArgument(msg);          \
  } while (0)

extern std::atomic<int64_t> g_kernel_launches;
inline void count_launch(int n = 1) { g_kernel_launches.fetch_add(n, std::memory_order_relaxed); }
inline void check_launch() {
  count_launch();
  CT2_CUDA_CHECK(cudaGetLastError());
}

// ---- dtype helpers ----
template <typename T> struct DType;
template <> struct DType<float> { static constexpr int id = CT2B200_F32; };
template <> struct DType<__half> { static constexpr int id = CT2B200_F16; };
template <> struct DType<__nv_bfloat16> { static constexpr int id = CT2B200_BF16; };

inline size_t dtype_size(int dtype) { return dtype == CT2B200_F32 ? 4 : 2; }

#define CT2_DISPATCH_DTYPE(dtype, ...)                                          \
  switch (dtype) {                                                              \
    case CT2B200_F32: { using T = float; __VA_ARGS__; break; }                  \
    case CT2B200_F16: { using T = __half; __VA_ARGS__; break; }                 \
    case CT2B200_BF16: { using T = __nv_bfloat16; __VA_ARGS__; break; }         \
    default: throw ::ct2b200::InvalidArgument("unsupported dtype");             \
  }

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
// round a float through T (the reference materialises intermediates in T)
template <typename T> __device__ __forceinline__ float round_to(float v) { return to_f32(from_f32<T>(v)); }

// 16-byte vector of T
template <typename T> struct Vec16 { static constexpr int N = 16 / sizeof(T); T v[N]; };

template <typename T>
__device__ __forceinline__ Vec16<T> ld16(const T* p) {
  Vec16<T> r;
  *reinterpret_cast<uint4*>(&r) = *reinterpret_cast<const uint4*>(p);
  return r;
}
template <typename T>
__device__ __forceinline__ void st16(T* p, const Vec16<T>& r) {
  *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(&r);
}

// ---- reductions ----
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// block-wide reductions; `red` is >= 32 floats of shared memory; result broadcast to all threads
template <bool kMax>
__device__ __forceinline__ float block_reduce(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = kMax ? warp_max(v) : warp_sum(v);
  __syncthreads();  // protect `red` from a previous use
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = lane < nw ? red[lane] : (kMax ? -INFINITY : 0.f);
  r = kMax ? warp_max(r) : warp_sum(r);
  return r;
}

// ---- activations (reference src/cuda/helpers.h:244-305) ----
__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case CT2B200_ACT_RELU: return fmaxf(x, 0.f);
    case CT2B200_ACT_GELU_TANH: return 0.5f * x * (1.f + tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x)));
    case CT2B200_ACT_SWISH: return x / (1.f + expf(-x));
    case CT2B200_ACT_GELU: return 0.5f * x * (1.f + erff(0.7071067811865475f * x));
    case CT2B200_ACT_GELU_SIGMOID: return x / (1.f + expf(-1.702f * x));
    case CT2B200_ACT_TANH: return tanhf(x);
    case CT2B200_ACT_SIGMOID: return 1.f / (1.f + expf(-x));
    default: return x;
  }
}

// ---- fused Dense epilogue shared by every GEMM kernel ----
// y[i,j] = T( act( T( T(c / (sa[i]*sb[j])) + bias[j] ) ) ) (+ residual[i,j], added in T)
// rounding points follow the reference CUDA path (SURVEY §8 a'): dequantize_gpu.cu:43-53, common.cc:392-401.
struct DenseEpilogue {
  const float* a_scale;    // [m] or nullptr (=> raw accumulators are written to c_out)
  const float* b_scale;    // [n]
  const void* bias;        // [n] T or nullptr
  const void* residual;    // [m,n] T or nullptr
  void* y;                 // [m,n] T
  int32_t* c_out;          // [m,n] int32 raw output mode (when a_scale == nullptr)
  int act;
  int64_t ldy;             // row stride of y / residual / c_out (= n)
};

template <typename T>
__device__ __forceinline__ float dense_epilogue_value(const DenseEpilogue& e, int32_t acc, int64_t i, int64_t j) {
  float v = __fdiv_rn(static_cast<float>(acc), e.a_scale[i] * e.b_scale[j]);
  v = round_to<T>(v);
  if (e.bias) v = round_to<T>(v + to_f32(static_cast<const T*>(e.bias)[j]));
  if (e.act >= 0) v = round_to<T>(apply_act(v, e.act));
  return v;
}

template <typename T>
__device__ __forceinline__ void dense_epilogue_store(const DenseEpilogue& e, int32_t acc, int64_t i, int64_t j) {
  if (e.a_scale == nullptr) {
    e.c_out[i * e.ldy + j] = acc;
    return;
  }
  float v = dense_epilogue_value<T>(e, acc, i, j);
  if (e.residual) v = v + to_f32(static_cast<const T*>(e.residual)[i * e.ldy + j]);
  static_cast<T*>(e.y)[i * e.ldy + j] = from_f32<T>(v);
}

// ---- programmatic dependent launch (PDL) ----
// Every kernel of the decode step is launched with cudaLaunchAttributeProgrammaticStreamSerialization: it may start
// (be scheduled, run its prologue) while its predecessor is still draining; `griddep_wait()` blocks until all
// prerequisite grids have completed and their writes are visible, so it must precede the first access to data a
// previous kernel produced.  `griddep_launch()` lets the NEXT kernel's CTAs be scheduled early.
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

bool pdl_enabled();
// The next kernel this thread launches is a plain stream-ordered launch: it starts after EVERYTHING before it has completed.
// The step graphs get this boundary for free (consecutive graph launches are fully ordered); the eager decode loops ask for
// it at the first kernel of every step, so that programmatic overlap never spans two steps in either mode.
void pdl_fence_next_launch();
// true the first time (kernel, tag) is seen ON THE CURRENT DEVICE: function attributes (dynamic shared memory limit, carve-out)
// and occupancy queries are per device, and a process may open generators on several (tag 0 = carve-out, 1 = smem limit)
bool mark_configured(const void* kernel, int tag = 0);

// All kernels of the decode step ask for the maximum shared-memory carve-out: the wgmma GEMMs need ~200 KB of
// shared memory per SM, and alternating between kernels with different L1/shared splits forces the SMs to drain
// and reconfigure between launches.
template <typename K>
void prefer_max_shared(K kernel) {
  cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}

// cudaFuncAttributeMaxDynamicSharedMemorySize, once per kernel and device
template <typename K>
void allow_dynamic_smem(K kernel, size_t bytes) {
  if (mark_configured(reinterpret_cast<const void*>(kernel), 1))
    CT2_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes)));
}

// One launch with the attributes the kernels use: a thread-block cluster of `cs` CTAs when cs > 1, programmatic dependent
// launch when enabled.
template <typename... KArgs, typename... Args>
void launch_clustered(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, int cs, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (cs > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = cs;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  CT2_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...));
}

template <typename... KArgs, typename... Args>
void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  if (mark_configured(reinterpret_cast<const void*>(kernel))) prefer_max_shared(kernel);
  launch_clustered(kernel, grid, block, smem, 1, st, std::forward<Args>(args)...);
}

inline int div_up(int64_t a, int64_t b) { return static_cast<int>((a + b - 1) / b); }

}  // namespace ct2b200
