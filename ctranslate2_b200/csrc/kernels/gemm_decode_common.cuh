// gemm_decode_common.cuh — pieces shared by the decode (weight-streaming) wgmma kernels: gemm_decode.cu (INT8 / f16
// weights) and awq_decode.cu (AWQ-INT4 weights): the split-K cluster exchange with its fused epilogue of one output
// channel, and the planner / launch helpers.
#pragma once

#include <algorithm>
#include <cstdlib>
#include <map>
#include <mutex>
#include <tuple>
#include <type_traits>

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
    if constexpr (KIND == 0) sx[j] = ok ? p.a_scale[col0 + j * cstep] : 1.f;   // plain load: written by the previous kernel (build.py, NO_NC_LOADS)
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
      gate = round_to<T>(act_call(round_to<T>(gate), act));
      v = gate * round_to<T>(up);
    } else {
      if constexpr (KIND == 0) v = __fdividef(static_cast<float>(static_cast<int32_t>(r[0][j])), sx[j] * sw0);
      else v = __uint_as_float(r[0][j]);
      // bias_t / res[j] are 0 when absent: adding them is exact, which keeps the unrolled code free of branch versions
      v = round_to<T>(round_to<T>(v) + bias_t);
      if (act >= 0) v = round_to<T>(act_call(v, act));
      v = v + res[j];
    }
    yp[j * step] = from_f32<T>(v);
  }
}

// ---- the plan both kernels share: one tile per CTA, K split over a cluster of CS CTAs, reduced through DSMEM ----
// Split-K ownership: inside every 16-column chunk, column j belongs to rank j % CS (slot j / CS of that chunk).
constexpr int owned_per_chunk(int cs) { return (16 + cs - 1) / cs; }
// exchange buffer [cs source ranks][nb weights][(bn / 16) chunks x owned columns][128 channels] of 32-bit partials
constexpr size_t red_bytes(int cs, int nb, int bn) {
  return cs > 1 ? static_cast<size_t>(cs) * nb * (bn / 16) * owned_per_chunk(cs) * kTileM * 4 : 0;
}

// Epilogue with thread = output channel.  EVERY warp of the CTA calls it as the last thing it does: the consumer warps
// (kConsumer = true) once they have parked their accumulators (acc_store + epi_bar_sync), the producer warp once it has
// issued its last copy, because every thread of a cluster takes part in both phases of the cluster barrier.
// accs = [NB * BN columns][kAccPitch], red = exchange buffer of red_bytes(CS, NB, BN), a0 = first channel of the tile,
// crank = rank of this CTA in its cluster.
template <typename T, int KIND, int BN, int NB, int CS, bool kConsumer>
__device__ __forceinline__ void split_k_epilogue(const DecParams& p, const uint32_t* accs, uint32_t* red, int a0, int crank) {
  constexpr int cp16 = owned_per_chunk(CS);            // owned columns per chunk
  constexpr int cpr = (BN / 16) * cp16;                // owned column slots per rank
  const int rloc = threadIdx.x & 127;                  // consumer warps 0-3: channel of the tile
  const int64_t arow = static_cast<int64_t>(a0) + rloc;
  const bool row_ok = rloc < p.tile_rows && arow < p.n;
  float sw0 = 1.f, sw1 = 1.f, bias_t = 0.f;
  if constexpr (kConsumer) {
    griddep_wait();                                    // a_scale / residual come from the previous kernels
    if (row_ok) {
      if constexpr (KIND == 0) {
        sw0 = __ldg(p.w_scale0 + arow);
        if constexpr (NB == 2) sw1 = __ldg(p.w_scale1 + arow);
      }
      if (p.bias) bias_t = to_f32(static_cast<const T*>(p.bias)[arow]);
    }
    auto load_acc = [&](int c0, uint32_t (&r)[NB][16]) {
#pragma unroll
      for (int w = 0; w < NB; ++w) acc_load<16>(accs + (w * BN + c0) * kAccPitch, rloc, r[w]);
    };
    if constexpr (CS == 1) {
#pragma unroll 1
      for (int c0 = 0; c0 < BN; c0 += 16) {
        uint32_t r[NB][16];
        load_acc(c0, r);
        if (row_ok && c0 < p.m) dec_finish<T, KIND, NB, 16>(p, r, arow, c0, 1, 16, sw0, sw1, bias_t);
      }
    } else {
      // partial accumulators -> owner rank of each column
      cluster_wait();                                  // phase 1 complete: peers' shared memory may be written
      uint32_t peer[CS];                               // our source slot in every rank's buffer, at this thread's channel
#pragma unroll
      for (int o = 0; o < CS; ++o) {
        const uint32_t local = smem_u32(red + static_cast<size_t>(crank) * NB * cpr * kTileM + rloc);
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer[o]) : "r"(local), "r"(o));
      }
#pragma unroll 1
      for (int c0 = 0; c0 < BN; c0 += 16) {
        uint32_t r[NB][16];
        load_acc(c0, r);
        const uint32_t chunk_off = static_cast<uint32_t>((c0 / 16) * cp16 * kTileM * 4);
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int w = 0; w < NB; ++w) {
            const uint32_t off = static_cast<uint32_t>((w * cpr + j / CS) * kTileM * 4);
            asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(peer[j % CS] + chunk_off + off), "r"(r[w][j]) : "memory");
          }
      }
    }
  }
  if constexpr (CS > 1) {
    __syncwarp();
    if constexpr (!kConsumer) cluster_wait();                     // phase 1 (the consumer warps consumed it above)
    cluster_arrive();                                  // phase 2: all partials have landed in their owners
    cluster_wait();
    if constexpr (kConsumer) {
      const int nvalid = (16 - crank + CS - 1) / CS;   // columns of a chunk owned by this rank
#pragma unroll 1
      for (int ch = 0; ch < BN / 16; ++ch) {
        uint32_t r[NB][cp16];
#pragma unroll
        for (int w = 0; w < NB; ++w)
#pragma unroll
          for (int jj = 0; jj < cp16; ++jj) {
            uint32_t acc = 0u;
#pragma unroll
            for (int src = 0; src < CS; ++src) {       // fixed rank order: deterministic for the float kinds
              const uint32_t v = red[(static_cast<size_t>(src * NB + w) * cpr + ch * cp16 + jj) * kTileM + rloc];
              if constexpr (KIND == 0) acc += v;
              else acc = __float_as_uint(__uint_as_float(acc) + __uint_as_float(v));
            }
            r[w][jj] = acc;
          }
        const int col0 = ch * 16 + crank;
        if (row_ok && col0 < p.m) dec_finish<T, KIND, NB, cp16>(p, r, arow, col0, CS, nvalid, sw0, sw1, bias_t);
      }
    }
  }
}

inline int env_int(const char* name, int fallback) {
  const char* e = std::getenv(name);
  return e ? std::atoi(e) : fallback;
}

// ---- host side ----
constexpr size_t kMaxDynSmem = 226 * 1024;

// f(std::integral_constant<int, CS>) for the cluster sizes the kernels are instantiated for
template <typename F>
auto dispatch_cs(int cs, F&& f) {
  switch (cs) {
    case 1: return f(std::integral_constant<int, 1>());
    case 2: return f(std::integral_constant<int, 2>());
    case 3: return f(std::integral_constant<int, 3>());
    default: return f(std::integral_constant<int, 4>());
  }
}

// co-resident clusters of `cs` CTAs of `kernel` (cs == 1: one CTA per SM); the occupancy query is cached per device,
// kernel and shared-memory size.  The query fails for more than 48 KB of dynamic shared memory unless the kernel's limit
// has been raised first, hence allow_dynamic_smem here.
template <typename K>
int max_clusters(K kernel, int cs, int threads, size_t smem, int sm_count) {
  allow_dynamic_smem(kernel, kMaxDynSmem);
  if (cs == 1) return sm_count;
  static std::mutex mu;
  static std::map<std::tuple<int, const void*, size_t>, int> cache;
  int dev = 0;
  cudaGetDevice(&dev);
  const auto key = std::make_tuple(dev, reinterpret_cast<const void*>(kernel), smem);
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
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
    n = sm_count / cs * 3 / 4;                         // conservative
  }
  cache[key] = n;
  return n;
}

struct Plan {
  int cs = 0;            // 0 = shape not covered by the kernel
  int tile_rows = 128;
  int tiles = 0;
  int stages = 2;
};

// search(force_cs, force_rows) of a planner, cached per device, n and K blocks.  The cache is per call site: F is the
// closure type of the planner's lambda, so every planner instantiation has its own map.
// CT2B200_GEMM_CS / CT2B200_GEMM_ROWS pin the plan (tests sweep every cluster size and tile height with them); pinned
// plans, and those of a planner that reads further switches (`tunable`), are not cached.
template <typename F>
Plan cached_plan(int64_t n, int blocks, bool tunable, F&& search) {
  static std::mutex mu;
  static std::map<std::tuple<int, int64_t, int>, Plan> cache;
  int dev = 0;
  cudaGetDevice(&dev);
  const int force_cs = env_int("CT2B200_GEMM_CS", 0);
  const int force_rows = env_int("CT2B200_GEMM_ROWS", 0);
  if (force_cs != 0 || force_rows != 0 || tunable) return search(force_cs, force_rows);
  const auto key = std::make_tuple(dev, n, blocks);
  {
    std::lock_guard<std::mutex> lock(mu);
    auto it = cache.find(key);
    if (it != cache.end()) return it->second;
  }
  const Plan plan = search(0, 0);
  std::lock_guard<std::mutex> lock(mu);
  cache[key] = plan;
  return plan;
}

}  // namespace dec
}  // namespace ct2b200
