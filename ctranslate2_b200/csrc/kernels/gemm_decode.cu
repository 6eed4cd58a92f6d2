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

#include "gemm_common.cuh"
#include "gemm_decode_common.cuh"
#include "kernels.h"
#include "tc_common.cuh"

namespace ct2b200 {
namespace {

using namespace tc;
using namespace dec;

// The accumulators are parked for the epilogue in the operand ring: it has been consumed by then.
template <int BN, int NB>
struct DecSmem {
  static constexpr int kA = NB * kTileM * kSwizzleBytes;       // weight bytes per stage (always 128-row slots)
  static constexpr int kB = BN * kSwizzleBytes;                // activation bytes per stage
  static constexpr int kStage = kA + kB;
  static constexpr int kCtrl = 512;                            // barriers
  static constexpr int kAcc = acc_bytes(NB * BN);              // accumulators parked for the row-per-thread epilogue
  static __host__ __device__ int ring(int stages) { return stages * kStage > kAcc ? stages * kStage : kAcc; }
  static size_t bytes(int stages, int cs) { return ring(stages) + kCtrl + red_bytes(cs, NB, BN) + 1024; }
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

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nstages = p.stages;
  uint8_t* ring = smem;
  uint32_t* accs = reinterpret_cast<uint32_t*>(smem);                    // [NB * BN columns][kAccPitch], after the K loop
  uint8_t* ctrl = ring + S::ring(nstages);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ctrl);               // [kMaxStages]
  uint64_t* empty_bar = full_bar + kMaxStages;                           // [kMaxStages]
  uint32_t* red = reinterpret_cast<uint32_t*>(ctrl + S::kCtrl);          // split-K exchange buffer (CS > 1)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x / CS;
  const int crank = CS > 1 ? static_cast<int>(blockIdx.x % CS) : 0;
  const int kb_lo = crank * p.kb_total / CS, kb_hi = (crank + 1) * p.kb_total / CS;
  const int nkb = kb_hi - kb_lo;
  const int a0 = tile * p.tile_rows;

  ring_init<CS>(full_bar, empty_bar, nstages);

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
      produce(full_bar, empty_bar, nstages, stage_tx, kb_lo, nkb, weights, acts);
    }
    split_k_epilogue<T, KIND, BN, NB, CS, false>(p, accs, red, a0, crank);
  } else {
    // ===== consumer warpgroup: wgmma over this CTA's K blocks =====
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
    epi_bar_sync();                                    // every warp has read its last stage: the ring becomes `accs`
#pragma unroll
    for (int w = 0; w < NB; ++w) acc_store<BN>(acc[w], accs + w * BN * kAccPitch);
    epi_bar_sync();
    split_k_epilogue<T, KIND, BN, NB, CS, true>(p, accs, red, a0, crank);
  }
}

// ---- host side ----
// Ring depth.  Single-weight Dense layers (QKV, out, down) size the ring so that two CTAs fit on one SM, where three
// stages fit in 110 KB: the CTA of the next launch (programmatic dependent launch) then streams its weights while this
// one drains its ring and runs its epilogue, and split-K plans may place two CTAs per SM.  The fused gate/up GEMM keeps
// one CTA per SM with a ring of up to 200 KB: two co-resident gate/up CTAs of three stages each made the Llama-3-8B
// decode step slower, single-weight ones made it faster (README, "Measured").
template <int BN, int NB>
int stages_for(int cs, int nkb) {
  using S = DecSmem<BN, NB>;
  const size_t fixed = S::kCtrl + red_bytes(cs, NB, BN) + 1024;
  int st = static_cast<int>((110 * 1024 - fixed) / S::kStage);
  if (NB == 2 || st < 3 || S::bytes(st, cs) > 110 * 1024) st = static_cast<int>((200 * 1024 - fixed) / S::kStage);
  st = std::max(2, std::min(st, kMaxStages));
  return std::max(2, std::min(st, std::max(nkb, 2)));
}

// Tile height and cluster size: one wave, every CTA streams (almost) the same number of weight bytes.
// cost = weight bytes per CTA (+ the DSMEM exchange, expressed in streamed-bytes equivalents).
template <typename T, int KIND, int BN, int NB>
Plan plan_decode(int64_t n, int kb_total, int sm_count, int force_cs, int force_rows) {
  Plan best;
  double best_cost = 1e30;
  for (int cs = 1; cs <= 4; ++cs) {
    if (force_cs && cs != force_cs) continue;
    if (cs > 1 && kb_total < 2 * cs) continue;
    const int nkb = (kb_total + cs - 1) / cs;
    const int stages = stages_for<BN, NB>(cs, nkb);
    if (DecSmem<BN, NB>::bytes(stages, cs) > kMaxDynSmem) continue;      // wide activation tiles: the exchange buffer does not fit
    const int maxc = dispatch_cs(cs, [&](auto c) {
      return max_clusters(gemm_decode_kernel<T, KIND, BN, NB, decltype(c)::value>, cs, kTcThreads, DecSmem<BN, NB>::bytes(stages, cs), sm_count);
    });
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
  return best;
}

template <typename T, int KIND, int BN, int NB>
bool run_decode(const void* x, const void* w, const void* w2, int64_t m, int64_t n, int64_t k, DecParams p, cudaStream_t st) {
  constexpr int elem = Elem<KIND>::bytes;
  const int sms = sm_count_of_current_device();
  const int kb_total = div_up(k, kSwizzleBytes / elem);
  const Plan plan = cached_plan(n, kb_total, std::getenv("CT2B200_GEMM_ROWSTEP") != nullptr,
                                [&](int force_cs, int force_rows) { return plan_decode<T, KIND, BN, NB>(n, kb_total, sms, force_cs, force_rows); });
  if (plan.cs == 0) return false;
  p.n = n;
  p.m = m;
  p.kb_total = kb_total;
  p.tile_rows = plan.tile_rows;
  p.stages = plan.stages;
  const CUtensorMap tmx = make_operand_map(x, m, k, elem, KIND, BN);
  const CUtensorMap tmw = make_operand_map(w, n, k, elem, KIND, plan.tile_rows);
  const CUtensorMap tmw2 = make_operand_map(w2 ? w2 : w, n, k, elem, KIND, plan.tile_rows);
  dispatch_cs(plan.cs, [&](auto c) {
    auto kernel = gemm_decode_kernel<T, KIND, BN, NB, decltype(c)::value>;
    allow_dynamic_smem(kernel, kMaxDynSmem);
    launch_clustered(kernel, dim3(static_cast<unsigned>(plan.tiles * plan.cs)), dim3(kTcThreads), DecSmem<BN, NB>::bytes(plan.stages, plan.cs),
                     plan.cs, st, tmx, tmw, tmw2, p);
  });
  check_launch();
  return true;
}

template <typename T, int KIND, int NB>
bool run_decode_m(const void* x, const void* w, const void* w2, int64_t m, int64_t n, int64_t k, const DecParams& p,
                  cudaStream_t st) {
  if (m <= 16) return run_decode<T, KIND, 16, NB>(x, w, w2, m, n, k, p, st);
  if (m <= 32) return run_decode<T, KIND, 32, NB>(x, w, w2, m, n, k, p, st);
  if (m <= 64) return run_decode<T, KIND, 64, NB>(x, w, w2, m, n, k, p, st);
  if constexpr (KIND == 0 && NB == 1) {
    if (m <= 128) return run_decode<T, KIND, 128, NB>(x, w, w2, m, n, k, p, st);   // 128 accumulator registers per thread
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
bool gemm_s8_decode(const int8_t* A, const int8_t* B, int64_t M, int64_t N, int64_t K, const DenseEpilogue& e, int dtype,
                    cudaStream_t st) {
  if (!decode_kernel_enabled() || M > decode_max_m(N, K) || M < 1 || e.a_scale == nullptr || K % 16 != 0) return false;
  DecParams p{};
  p.a_scale = e.a_scale;
  p.w_scale0 = e.b_scale;
  p.bias = e.bias;
  p.residual = e.residual;
  p.y = e.y;
  p.act = e.act;
  p.ldy = e.ldy;
  bool ok = false;
  CT2_DISPATCH_DTYPE(dtype, (ok = run_decode_m<T, 0, 1>(A, B, nullptr, M, N, K, p, st)));
  return ok;
}

bool gemm_s8_glu_decode(const int8_t* A, const int8_t* Bgate, const int8_t* Bup, int64_t M, int64_t N, int64_t K,
                        const GluEpilogue& g, int dtype, cudaStream_t st) {
  if (!decode_kernel_enabled() || M > 64 || M < 1 || K % 16 != 0) return false;
  DecParams p{};
  p.a_scale = g.a_scale;
  p.w_scale0 = g.gate_scale;
  p.w_scale1 = g.up_scale;
  p.y = g.h;
  p.act = g.act;
  p.ldy = g.ldh;
  bool ok = false;
  CT2_DISPATCH_DTYPE(dtype, (ok = run_decode_m<T, 0, 2>(A, Bgate, Bup, M, N, K, p, st)));
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
