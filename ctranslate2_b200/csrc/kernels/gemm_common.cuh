// gemm_common.cuh — pieces shared by the INT8/FP16 GEMM kernels: the SwiGLU epilogue, the split-K
// scratch (zero-initialised once, self-cleaning) and the split heuristic.
#pragma once

#include <map>
#include <mutex>

#include "../common.cuh"

namespace ct2b200 {

// FeedForwardNetwork gate/up fusion (reference src/layers/transformer.cc:21-51 with ffn_glu):
//   gate = T(act(T(c_gate / (sa*sg)))) ; up = T(c_up / (sa*su)) ; h = T(gate * up)
struct GluEpilogue {
  const float* a_scale;      // [m]
  const float* gate_scale;   // [n]
  const float* up_scale;     // [n]
  void* h;                   // [m,n] T
  int act;
  int64_t ldh;
};

template <typename T>
__device__ __forceinline__ void glu_epilogue_store(const GluEpilogue& e, int32_t cg, int32_t cu, int64_t i, int64_t j) {
  const float sa = e.a_scale[i];
  float gate = round_to<T>(__fdiv_rn(static_cast<float>(cg), sa * e.gate_scale[j]));
  gate = round_to<T>(apply_act(gate, e.act));
  const float up = round_to<T>(__fdiv_rn(static_cast<float>(cu), sa * e.up_scale[j]));
  static_cast<T*>(e.h)[i * e.ldh + j] = from_f32<T>(gate * up);
}

// Float epilogue of the f16/bf16 GEMM (ops::Gemm::apply_bias_and_activation, reference src/ops/gemm.cc:10-25)
struct FloatEpilogue {
  const void* bias;
  const void* residual;
  void* y;
  int act;
  int64_t ldy;
};
template <typename T>
__device__ __forceinline__ void float_epilogue_store(const FloatEpilogue& e, float acc, int64_t i, int64_t j) {
  float v = round_to<T>(acc);
  if (e.bias) v = round_to<T>(v + to_f32(static_cast<const T*>(e.bias)[j]));
  if (e.act >= 0) v = round_to<T>(apply_act(v, e.act));
  if (e.residual) v = v + to_f32(static_cast<const T*>(e.residual)[i * e.ldy + j]);
  static_cast<T*>(e.y)[i * e.ldy + j] = from_f32<T>(v);
}


// SwiGLU over float accumulators (AWQ gate/up): h = T(act(T(gate))) * T(up)
struct FloatGluEpilogue {
  void* h;
  int act;
  int64_t ldh;
};
template <typename T>
__device__ __forceinline__ void float_glu_epilogue_store(const FloatGluEpilogue& e, float gate, float up, int64_t i, int64_t j) {
  const float g = round_to<T>(apply_act(round_to<T>(gate), e.act));
  static_cast<T*>(e.h)[i * e.ldh + j] = from_f32<T>(g * round_to<T>(up));
}

// Per-(device, stream) split-K scratch.  `accum` holds int32 (or fp32) partial sums and is all-zero
// between kernels; `counters` are per-tile arrival tickets, also zero between kernels.
struct SplitKWorkspace {
  int32_t* accum = nullptr;
  int32_t* counters = nullptr;
  int32_t* accum2 = nullptr;        // fully-overwritten partial slots of the float (f16/AWQ) kernels: never needs zeroing
  size_t accum_elems = 0;
  size_t num_counters = 0;
  int sm_count = 132;

  static constexpr size_t kAccumElems = size_t(16) << 20;  // 64 MiB of int32
  static constexpr size_t kCounters = 1 << 16;

  static std::mutex& mutex() {
    static std::mutex mu;
    return mu;
  }
  static std::map<std::pair<int, cudaStream_t>, SplitKWorkspace>& registry() {
    static std::map<std::pair<int, cudaStream_t>, SplitKWorkspace> all;
    return all;
  }
  // the owner of a stream (a decoder / translator) returns its scratch when it goes away
  static void release(cudaStream_t st) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return;
    std::lock_guard<std::mutex> lock(mutex());
    auto it = registry().find({dev, st});
    if (it == registry().end()) return;
    cudaFree(it->second.accum);
    cudaFree(it->second.counters);
    cudaFree(it->second.accum2);
    registry().erase(it);
  }

  static SplitKWorkspace& get(cudaStream_t st) {
    int dev = 0;
    CT2_CUDA_CHECK(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(mutex());
    auto& w = registry()[{dev, st}];
    if (!w.accum) {
      cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
      cudaStreamIsCapturing(st, &cs);
      if (cs != cudaStreamCaptureStatusNone)
        throw std::runtime_error("split-K workspace must be created before stream capture (call a GEMM once eagerly)");
      CT2_CUDA_CHECK(cudaMalloc(&w.accum, kAccumElems * sizeof(int32_t)));
      CT2_CUDA_CHECK(cudaMalloc(&w.counters, kCounters * sizeof(int32_t)));
      CT2_CUDA_CHECK(cudaMalloc(&w.accum2, kAccumElems * sizeof(int32_t)));
      CT2_CUDA_CHECK(cudaMemset(w.accum, 0, kAccumElems * sizeof(int32_t)));
      CT2_CUDA_CHECK(cudaMemset(w.counters, 0, kCounters * sizeof(int32_t)));
      CT2_CUDA_CHECK(cudaDeviceSynchronize());
      w.accum_elems = kAccumElems;
      w.num_counters = kCounters;
      CT2_CUDA_CHECK(cudaDeviceGetAttribute(&w.sm_count, cudaDevAttrMultiProcessorCount, dev));
    }
    return w;
  }
};

// SM count of the current device (cached per device)
inline int sm_count_of_current_device() {
  static std::mutex mu;
  static std::map<int, int> cache;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(dev);
  if (it == cache.end()) {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    it = cache.emplace(dev, sms).first;
  }
  return it->second;
}

// Number of K splits: enough CTAs to cover every SM about twice, while each split keeps >= 4 K-tiles
// and the partial planes fit the scratch.
inline int choose_splits(int tiles, int k_tiles, int64_t accum_elems_needed, const SplitKWorkspace& w) {
  if (tiles >= w.sm_count || k_tiles < 8) return 1;
  if (static_cast<size_t>(accum_elems_needed) > w.accum_elems || static_cast<size_t>(tiles) > w.num_counters) return 1;
  int want = (2 * w.sm_count + tiles - 1) / tiles;
  int max_by_k = k_tiles / 4;
  int s = want < max_by_k ? want : max_by_k;
  if (s < 1) s = 1;
  if (s > 16) s = 16;
  return s;
}

void gemm_s8_mma(const int8_t* A, const int8_t* B, int64_t M, int64_t N, int64_t K, const DenseEpilogue& epi,
                 int dtype, cudaStream_t st);
void gemm_s8_glu_mma(const int8_t* A, const int8_t* Bgate, const int8_t* Bup, int64_t M, int64_t N, int64_t K,
                     const GluEpilogue& glu, int dtype, cudaStream_t st);

}  // namespace ct2b200
