// gemm_decode.cu — weight-streaming GEMM of the decode step (m <= 64 activation rows) on wgmma.
//
// Replaces, for the Dense layers of one decode step, the reference chain
//   ops::Gemm (cuBLAS IMMA, int32 C in HBM) -> ops::Dequantize::dequantize_gemm_output -> ops::Add / ops::Mul
// (reference src/layers/common.cc:353-401, src/ops/gemm.cc:45-107, src/ops/dequantize_gpu.cu:30-144) by ONE kernel.
//
// Shape of the problem: y[m, n] = x[m, k] * W[n, k]^T with m <= 64: every weight byte is used once, so the kernel is a
// pure HBM stream and the only thing that matters is that all SMs stream the same number of bytes and that the
// fixed cost per launch (pipeline fill, epilogue, instruction fetch) is small.  Hence:
//   * "swap AB": the weights sit on the wgmma M side (two m64 instructions = 128 output channels), the activations on the
//     N side (BN = 16/32/64 columns), so a tiny m does not waste the 64-row MMA.
//   * the tile height (weight rows per CTA, a multiple of 8 <= 128) and the split of K over a thread-block cluster of
//     CS CTAs are chosen per shape so that tiles * CS ~ number of SMs, ONE tile per CTA, one wave (plan_decode).
//   * K split inside the cluster is reduced through distributed shared memory: rank r owns the output columns
//     j % CS == r, partial accumulators go to the owner with st.shared::cluster, one cluster barrier, no global traffic.
//   * the weights never depend on the previous kernel: the TMA producer fills the whole ring BEFORE
//     griddepcontrol.wait (programmatic dependent launch), so the stream overlaps the predecessor's tail.
//   * the code is kept small on purpose (one tile, compile-time CS, rolled 16-column chunks), so that the epilogue is not
//     bound by instruction fetch.
//
// Rounding points of the fused epilogue: DenseEpilogue / GluEpilogue / FloatEpilogue (common.cuh, gemm_common.cuh).
#include <algorithm>
#include <cstdlib>
#include <map>
#include <mutex>
#include <tuple>

#include "gemm_common.cuh"
#include "gemm_decode_common.cuh"
#include "kernels.h"
#include "row_ops.cuh"
#include "tc_common.cuh"

namespace ct2b200 {
namespace {

using namespace tc;
using namespace dec;

template <int BN, int NB>
struct DecSmem {
  static constexpr int kA = NB * kTileM * kSwizzleBytes;       // weight bytes per stage (always 128-row slots)
  static constexpr int kB = BN * kSwizzleBytes;                // activation bytes per stage
  static constexpr int kStage = kA + kB;
  static constexpr int kCtrl = 512;                            // barriers
  static constexpr int kAcc = acc_bytes(NB * BN);              // accumulators parked for the row-per-thread epilogue
  // per source rank and weight: (BN / 16) chunks x ceil(16 / cs) owned columns x 128 channels of 32-bit partials
  static size_t red_bytes(int cs) { return cs > 1 ? static_cast<size_t>(cs) * NB * (BN / 16) * ((16 + cs - 1) / cs) * kTileM * 4 : 0; }
  static size_t bytes(int stages, int cs) { return kAcc + static_cast<size_t>(stages) * kStage + kCtrl + red_bytes(cs) + 1024; }
};

// T = output dtype, KIND = 0 s8 / 1 f16 / 2 bf16, BN = wgmma N (activation rows, zero padded), NB = 2 for gate+up,
// CS = CTAs per tile (cluster size; K is split CS ways)
template <typename T, int KIND, int BN, int NB, int CS>
__global__ void __launch_bounds__(kTcThreads, 2)
    gemm_decode_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                       const __grid_constant__ CUtensorMap tm_w2, const DecParams p) {
  using S = DecSmem<BN, NB>;
  constexpr int kElem = Elem<KIND>::bytes;
  constexpr int BK = kSwizzleBytes / kElem;
  // split-K ownership: inside every 16-column chunk, column j belongs to rank j % CS (slot j / CS of that chunk)
  constexpr int cp16 = (16 + CS - 1) / CS;             // owned columns per chunk
  constexpr int cpr = (BN / 16) * cp16;                // owned column slots per rank

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nstages = p.stages;
  uint32_t* accs = reinterpret_cast<uint32_t*>(smem);                    // [NB * BN columns][kAccPitch]
  uint8_t* ring = smem + S::kAcc;
  uint8_t* ctrl = ring + nstages * S::kStage;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ctrl);               // [kMaxStages]
  uint64_t* empty_bar = full_bar + kMaxStages;                           // [kMaxStages]
  uint32_t* red = reinterpret_cast<uint32_t*>(ctrl + S::kCtrl);          // [CS src][NB][cpr][128] (CS > 1)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x / CS;
  const int crank = CS > 1 ? static_cast<int>(blockIdx.x % CS) : 0;
  const int kb_lo = crank * p.kb_total / CS, kb_hi = (crank + 1) * p.kb_total / CS;
  const int nkb = kb_hi - kb_lo;
  const int a0 = tile * p.tile_rows;

  if (threadIdx.x == 0) {
    for (int s = 0; s < nstages; ++s) {
      mbar_init(full_bar + s, 1);
      mbar_init(empty_bar + s, 4);                   // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  griddep_launch();
  if (CS > 1) cluster_arrive();                        // phase 1: every CTA of the cluster is alive

  if (warp == kProducerWarp) {
    // ===== TMA producer =====
    if (elect_one()) {
      const uint32_t stage_tx = static_cast<uint32_t>(NB * p.tile_rows * kSwizzleBytes + S::kB);
      auto weights = [&](int s, int kb) {
        uint8_t* sa = ring + s * S::kStage;
        tma_load_2d(sa, &tm_w, full_bar + s, kb * BK, a0, kEvictFirst);
        if (NB == 2) tma_load_2d(sa + kTileM * kSwizzleBytes, &tm_w2, full_bar + s, kb * BK, a0, kEvictFirst);
      };
      auto acts = [&](int s, int kb) {
        tma_load_2d(ring + s * S::kStage + S::kA, &tm_x, full_bar + s, kb * BK, 0, kEvictLast);
      };
      const int pre = min(nstages, nkb);
#pragma unroll 1
      for (int i = 0; i < pre; ++i) {                  // weights of the first ring fill: before the dependency wait
        mbar_expect_tx(full_bar + i, stage_tx);
        weights(i, kb_lo + i);
      }
      griddep_wait();
#pragma unroll 1
      for (int i = 0; i < pre; ++i) acts(i, kb_lo + i);
#pragma unroll 1
      for (int it = pre; it < nkb; ++it) {
        const int s = it % nstages;
        mbar_wait(empty_bar + s, ((it / nstages) & 1) ^ 1);
        mbar_expect_tx(full_bar + s, stage_tx);
        weights(s, kb_lo + it);
        acts(s, kb_lo + it);
      }
    }
  } else {
    // ===== consumer warpgroup: wgmma over this CTA's K blocks, then the epilogue with thread = output channel =====
    Acc<BN> acc[NB];
#pragma unroll 1
    for (int it = 0; it < nkb; ++it) {
      const int s = it % nstages;
      mbar_wait(full_bar + s, (it / nstages) & 1);
      const uint32_t sa = smem_u32(ring + s * S::kStage);
      wgmma_fence();
#pragma unroll
      for (int w = 0; w < NB; ++w) mma_block<KIND, BN>(acc[w], sa + w * kTileM * kSwizzleBytes, sa + S::kA, it == 0);
      wgmma_commit();
      wgmma_wait();
      if (lane == 0) mbar_arrive(empty_bar + s);       // this warp's share of the stage has been read
    }
#pragma unroll
    for (int w = 0; w < NB; ++w) acc_store<BN>(acc[w], accs + w * BN * kAccPitch);
    epi_bar_sync();
    const int q = warp & 3;
    const int rloc = q * 32 + lane;
    const int64_t arow = static_cast<int64_t>(a0) + rloc;
    const bool row_ok = rloc < p.tile_rows && arow < p.n;
    griddep_wait();                                    // a_scale / residual come from the previous kernels
    float sw0 = 1.f, sw1 = 1.f, bias_t = 0.f;
    if (row_ok) {
      if constexpr (KIND == 0) {
        sw0 = __ldg(p.w_scale0 + arow);
        if constexpr (NB == 2) sw1 = __ldg(p.w_scale1 + arow);
      }
      if (p.bias) bias_t = to_f32(static_cast<const T*>(p.bias)[arow]);
    }
    if constexpr (CS == 1) {
#pragma unroll 1
      for (int c0 = 0; c0 < BN; c0 += 16) {
        uint32_t r[NB][16];
#pragma unroll
        for (int w = 0; w < NB; ++w) acc_load<16>(accs + (w * BN + c0) * kAccPitch, rloc, r[w]);
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
#pragma unroll
        for (int w = 0; w < NB; ++w) acc_load<16>(accs + (w * BN + c0) * kAccPitch, rloc, r[w]);
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
    if (warp == kProducerWarp) cluster_wait();         // phase 1 (the consumer warps consumed it above)
    cluster_arrive();                                  // phase 2: all partials have landed in their owners
    cluster_wait();
    if (warp < kProducerWarp) {
      const int q = warp & 3;
      const int rloc = q * 32 + lane;
      const int64_t arow = static_cast<int64_t>(a0) + rloc;
      const bool row_ok = rloc < p.tile_rows && arow < p.n;
      float sw0 = 1.f, sw1 = 1.f, bias_t = 0.f;
      if (row_ok) {
        if constexpr (KIND == 0) {
          sw0 = __ldg(p.w_scale0 + arow);
          if constexpr (NB == 2) sw1 = __ldg(p.w_scale1 + arow);
        }
        if (p.bias) bias_t = to_f32(static_cast<const T*>(p.bias)[arow]);
      }
      const int nvalid = (16 - crank + CS - 1) / CS;    // columns of a chunk owned by this rank
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

// ---- host side ----
struct DecPlan {
  int cs = 0;            // 0 = shape not covered by this kernel
  int tile_rows = 128;
  int tiles = 0;
  int stages = 2;
};

template <typename T, int KIND, int BN, int NB, int CS>
void configure_once() {
  allow_dynamic_smem(gemm_decode_kernel<T, KIND, BN, NB, CS>, 226 * 1024);
}

template <typename T, int KIND, int BN, int NB, int CS>
int clusters_for(int stages, int sm_count) {
  configure_once<T, KIND, BN, NB, CS>();
  static std::mutex mu;
  static std::map<std::pair<int, int>, int> cache;       // (device, stages) -> clusters
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find({dev, stages});
  if (it != cache.end()) return it->second;
  const int n = max_clusters(gemm_decode_kernel<T, KIND, BN, NB, CS>, CS, kTcThreads, DecSmem<BN, NB>::bytes(stages, CS), sm_count);
  cache[{dev, stages}] = n;
  return n;
}

template <int BN, int NB>
int stages_for(int cs, int nkb) {
  using S = DecSmem<BN, NB>;
  const size_t cap = static_cast<size_t>(std::max(48, std::min(200, env_int("CT2B200_GEMM_SMEM_KB", 200)))) * 1024;
  int st = static_cast<int>((cap - S::kAcc - S::kCtrl - S::red_bytes(cs) - 1024) / S::kStage);
  st = std::max(2, std::min(st, kMaxStages));
  return std::max(2, std::min(st, std::max(nkb, 2)));
}

// Tile height and cluster size: one wave, every CTA streams (almost) the same number of weight bytes.
// cost = weight bytes per CTA (+ the DSMEM exchange, expressed in streamed-bytes equivalents).
template <typename T, int KIND, int BN, int NB>
DecPlan plan_decode(int64_t n, int kb_total, int sm_count) {
  static std::mutex mu;
  static std::map<std::tuple<int, int64_t, int>, DecPlan> cache;
  int dev = 0;
  cudaGetDevice(&dev);
  // CT2B200_GEMM_CS / CT2B200_GEMM_ROWS pin the plan (tests sweep every cluster size and tile height with them)
  const int force_cs = env_int("CT2B200_GEMM_CS", 0);
  const int force_rows = env_int("CT2B200_GEMM_ROWS", 0);
  const bool forced = force_cs != 0 || force_rows != 0 || std::getenv("CT2B200_GEMM_ROWSTEP") != nullptr;
  if (!forced) {
    std::lock_guard<std::mutex> lock(mu);
    auto it = cache.find({dev, n, kb_total});
    if (it != cache.end()) return it->second;
  }
  DecPlan best;
  double best_cost = 1e30;
  for (int cs = 1; cs <= 4; ++cs) {
    if (force_cs && cs != force_cs) continue;
    if (cs > 1 && kb_total < 2 * cs) continue;
    const int nkb = (kb_total + cs - 1) / cs;
    const int stages = stages_for<BN, NB>(cs, nkb);
    if (DecSmem<BN, NB>::bytes(stages, cs) > 226 * 1024) continue;      // wide activation tiles: the exchange buffer does not fit
    int maxc = 0;
    switch (cs) {
      case 1: maxc = clusters_for<T, KIND, BN, NB, 1>(stages, sm_count); break;
      case 2: maxc = clusters_for<T, KIND, BN, NB, 2>(stages, sm_count); break;
      case 3: maxc = clusters_for<T, KIND, BN, NB, 3>(stages, sm_count); break;
      default: maxc = clusters_for<T, KIND, BN, NB, 4>(stages, sm_count); break;
    }
    // tile heights need not be multiples of the 8-row swizzle atom: the TMA box simply ends inside an atom
    const int row_step = std::max(1, env_int("CT2B200_GEMM_ROWSTEP", 8));
    for (int rows = force_rows ? force_rows : 128; rows >= (force_rows ? force_rows : 64); rows -= row_step) {
      const int tiles = static_cast<int>((n + rows - 1) / rows);
      if (tiles > maxc) continue;
      const double cost = static_cast<double>(rows) * NB * nkb * kSwizzleBytes + (cs > 1 ? 48.0 * 1024 : 0.0) +
                          (128 - rows) * 16.0;          // mild preference for full-height tiles on ties
      if (cost < best_cost) {
        best_cost = cost;
        best.cs = cs;
        best.tile_rows = rows;
        best.tiles = tiles;
        best.stages = stages;
      }
    }
  }
  if (!forced) {
    std::lock_guard<std::mutex> lock(mu);
    cache[{dev, n, kb_total}] = best;
  }
  return best;
}

template <typename T, int KIND, int BN, int NB, int CS>
void launch_decode(const CUtensorMap& tmx, const CUtensorMap& tmw, const CUtensorMap& tmw2, const DecParams& p,
                   const DecPlan& plan, cudaStream_t st) {
  configure_once<T, KIND, BN, NB, CS>();
  auto kernel = gemm_decode_kernel<T, KIND, BN, NB, CS>;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<unsigned>(plan.tiles * CS));
  cfg.blockDim = dim3(kTcThreads);
  cfg.dynamicSmemBytes = DecSmem<BN, NB>::bytes(plan.stages, CS);
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (CS > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = CS;
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
  CT2_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, tmx, tmw, tmw2, p));
  check_launch();
}

template <typename T, int KIND, int BN, int NB>
bool run_decode(const void* x, const void* w, const void* w2, int64_t m, int64_t n, int64_t k, DecParams p,
                cudaStream_t st, const NextWeights* next = nullptr) {
  constexpr int elem = Elem<KIND>::bytes;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  {
    static std::mutex mu;
    static std::map<int, int> sm_cache;
    std::lock_guard<std::mutex> lock(mu);
    auto it = sm_cache.find(dev);
    if (it == sm_cache.end()) {
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
      sm_cache[dev] = sms;
    } else {
      sms = it->second;
    }
  }
  const int kb_total = div_up(k, kSwizzleBytes / elem);
  const DecPlan plan = plan_decode<T, KIND, BN, NB>(n, kb_total, sms);
  if (plan.cs == 0) return false;
  p.n = n;
  p.m = m;
  p.kb_total = kb_total;
  p.tile_rows = plan.tile_rows;
  p.stages = plan.stages;
  const CUtensorMap tmx = make_operand_map(x, m, k, elem, KIND, BN);
  const CUtensorMap tmw = make_operand_map(w, n, k, elem, KIND, plan.tile_rows);
  const CUtensorMap tmw2 = make_operand_map(w2 ? w2 : w, n, k, elem, KIND, plan.tile_rows);
  switch (plan.cs) {
    case 1: launch_decode<T, KIND, BN, NB, 1>(tmx, tmw, tmw2, p, plan, st); break;
    case 2: launch_decode<T, KIND, BN, NB, 2>(tmx, tmw, tmw2, p, plan, st); break;
    case 3: launch_decode<T, KIND, BN, NB, 3>(tmx, tmw, tmw2, p, plan, st); break;
    default: launch_decode<T, KIND, BN, NB, 4>(tmx, tmw, tmw2, p, plan, st); break;
  }
  return true;
}

template <typename T, int KIND, int NB>
bool run_decode_m(const void* x, const void* w, const void* w2, int64_t m, int64_t n, int64_t k, const DecParams& p,
                  cudaStream_t st, const NextWeights* next = nullptr) {
  if (m <= 16) return run_decode<T, KIND, 16, NB>(x, w, w2, m, n, k, p, st, next);
  if (m <= 32) return run_decode<T, KIND, 32, NB>(x, w, w2, m, n, k, p, st, next);
  if (m <= 64) return run_decode<T, KIND, 64, NB>(x, w, w2, m, n, k, p, st, next);
  if constexpr (KIND == 0 && NB == 1) {
    if (m <= 128) return run_decode<T, KIND, 128, NB>(x, w, w2, m, n, k, p, st, next);   // 128 accumulator registers per thread
  }
  return false;
}

// Rows this kernel takes.  Up to 64 it is the weight-streaming kernel of the decode step.  CT2B200_GEMM_DECODE_MAXM (up to 128: the accumulator registers of one warpgroup)
// also sends the small Dense layers of wide batches here (Transformer-base at batch x beam = 128: the whole weight matrix is a few
// hundred KB, the launch is latency-bound, and one lean tile per CTA on 8-32 SMs beats the persistent 128 x 256-tile kernel of
// gemm_prefill.cu on 4-16); only matrices of at most 4 M weights, so that compute-bound prompt GEMMs never come here.
int decode_max_m(int64_t n, int64_t k) {
  static const int max_m = std::max(64, std::min(128, env_int("CT2B200_GEMM_DECODE_MAXM", CT2B200_DEFAULT_GEMM_DECODE_MAXM)));
  return n * k <= (4 << 20) ? max_m : 64;
}

bool decode_kernel_enabled() {
  static const bool on = env_int("CT2B200_GEMM_DECODE", 1) != 0;
  return on;
}

}  // namespace

// The three entry points return false when the shape is not covered (m > 64, raw int32 output, more tiles than one
// wave holds): the caller then uses the general persistent kernel of gemm_tc.cu.
namespace {
// The row pre-phase ([RMSNorm +] Quantize of the activations inside this kernel, behind a grid barrier) is not implemented:
// callers that pass a RowPre get `false` and launch the row kernel themselves.
bool set_row_pre(DecParams&, const RowPre* pre, const int8_t*, const float*, int64_t, int) { return !pre || pre->mode == 0; }
}  // namespace

bool gemm_s8_decode(const int8_t* A, const int8_t* B, int64_t M, int64_t N, int64_t K, const DenseEpilogue& e, int dtype,
                    cudaStream_t st, const RowPre* pre, const NextWeights* next) {
  if (!decode_kernel_enabled() || M > decode_max_m(N, K) || M < 1 || e.a_scale == nullptr || K % 16 != 0) return false;
  DecParams p{};
  if (!set_row_pre(p, pre, A, e.a_scale, K, dtype)) return false;
  p.a_scale = e.a_scale;
  p.w_scale0 = e.b_scale;
  p.bias = e.bias;
  p.residual = e.residual;
  p.y = e.y;
  p.act = e.act;
  p.ldy = e.ldy;
  bool ok = false;
  CT2_DISPATCH_DTYPE(dtype, (ok = run_decode_m<T, 0, 1>(A, B, nullptr, M, N, K, p, st, next)));
  return ok;
}

bool gemm_s8_glu_decode(const int8_t* A, const int8_t* Bgate, const int8_t* Bup, int64_t M, int64_t N, int64_t K,
                        const GluEpilogue& g, int dtype, cudaStream_t st, const RowPre* pre, const NextWeights* next) {
  if (!decode_kernel_enabled() || M > 64 || M < 1 || K % 16 != 0) return false;
  DecParams p{};
  if (!set_row_pre(p, pre, A, g.a_scale, K, dtype)) return false;
  p.a_scale = g.a_scale;
  p.w_scale0 = g.gate_scale;
  p.w_scale1 = g.up_scale;
  p.y = g.h;
  p.act = g.act;
  p.ldy = g.ldh;
  bool ok = false;
  CT2_DISPATCH_DTYPE(dtype, (ok = run_decode_m<T, 0, 2>(A, Bgate, Bup, M, N, K, p, st, next)));
  return ok;
}

bool gemm_f16_decode(const void* A, const void* B, const void* bias, const void* residual, int act, int64_t M, int64_t N,
                     int64_t K, void* C, int dtype, cudaStream_t st) {
  if (!decode_kernel_enabled() || M > 64 || M < 1 || K % 8 != 0) return false;
  DecParams p{};
  p.bias = bias;
  p.residual = residual;
  p.y = C;
  p.act = act;
  p.ldy = N;
  if (dtype == CT2B200_F16) return run_decode_m<__half, 1, 1>(A, B, nullptr, M, N, K, p, st);
  if (dtype == CT2B200_BF16) return run_decode_m<__nv_bfloat16, 2, 1>(A, B, nullptr, M, N, K, p, st);
  return false;
}

}  // namespace ct2b200
