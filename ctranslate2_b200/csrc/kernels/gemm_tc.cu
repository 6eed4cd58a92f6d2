// gemm_tc.cu — the GENERAL wgmma GEMM (the fallback of the two specialised ones): wgmma (s8 / f16 / bf16) with
// TMA-staged, 128B-swizzled operand tiles in shared memory, accumulators in the registers of one warpgroup, fused
// Dense epilogue (one output row per thread, fed through a shared-memory transpose of the fragments).
//   * gemm_s8_tc / gemm_s8_glu_tc / gemm_f16_tc first try gemm_decode.cu (m <= 64, one tile per CTA, cluster/DSMEM
//     split-K) and gemm_prefill.cu (m > 64, two consumer warpgroups) and only land here for what those
//     do not cover: raw int32 output (ops::Gemm), N tiles beyond one wave at m <= 64 (the 128256-row lm_head),
//     unaligned rows.
//   * persistent stream-K over (tile, K block) units, "swap-AB" for m <= 64, stream-K / tile-partitioned / whole-tile
//     modes, deterministic slot-based reduction of shared tiles (no float atomics): the schedule of streamk.cuh, shared
//     with the AWQ kernel of awq.cu.
// Replaces cublasGemmEx s8/f16/bf16 (reference src/cuda/primitives.cu:485-597) + Dequantize epilogue
// (src/ops/dequantize_gpu.cu:30-121) + ops::Add/ops::Mul (src/layers/common.cc:392-401, transformer.cc:31-37).
//
// Warp roles (160 threads): warps 0..3 = consumer warpgroup (wgmma, then the epilogue: thread t owns tile row t),
// warp 4 = TMA producer (one elected lane).
#include <cuda.h>
#include <cudaTypedefs.h>

#include "../common.cuh"
#include "gemm_common.cuh"
#include "kernels.h"
#include "streamk.cuh"
#include "tc_common.cuh"

namespace ct2b200 {

namespace {

using namespace tc;

struct TcParams {
  int64_t rows_a;      // rows of the M-side operand (n when swapped, m otherwise)
  int64_t rows_b;      // rows of the N-side operand
  sk::Schedule sched;
  DenseEpilogue dense;
  GluEpilogue glu;
  FloatEpilogue fl;
  uint32_t* slots;     // partial-tile slots of the shared tiles [ctas][2][NB * 128 * BN]
  int32_t* counters;
};

template <int BN, int NB, bool kSwap>
struct TcSmem {
  static constexpr int kA = kTileM * kSwizzleBytes * (kSwap ? NB : 1);     // M-side bytes per stage
  static constexpr int kB = BN * kSwizzleBytes * (kSwap ? 1 : NB);         // N-side bytes per stage
  static constexpr int kStage = kA + kB;
  static constexpr int kAcc = acc_bytes(NB * BN);                          // accumulators parked for the epilogue
  static constexpr int kStages = ((200 * 1024 - kAcc) / kStage) > 8 ? 8 : ((200 * 1024 - kAcc) / kStage);
  static constexpr size_t kBytes = kAcc + static_cast<size_t>(kStages) * kStage + 1024 /*align*/ + 256 /*barriers*/;
};

// Epilogue of one thread over kCols (16) consecutive N-side rows of its M-side row `arow`.
//   kSwap: arow = output channel n, N-side rows = batch rows m;   !kSwap: arow = batch row m, N-side = channels n.
// Split in two so that the global loads (scales, bias, residual) can be issued early — before the accumulators are
// ready, or together with the scratch reads of the split-K fix-up — instead of adding a memory round trip:
//   epi_load:   all loads of the chunk, no dependent arithmetic;
//   epi_finish: arithmetic + stores (rounding points: see DenseEpilogue / GluEpilogue / FloatEpilogue).
template <int NB, int kCols>
struct EpiInputs {
  float st0, st1, bias_t;               // per-thread constants
  float sj0[kCols], sj1[NB == 2 ? kCols : 1], bj[kCols], resj[kCols];
  int ncols;                            // valid columns (0 => nothing to do)
};

template <typename T, int KIND, int NB, bool kSwap, int kCols>
__device__ __forceinline__ void epi_load(const TcParams& p, int64_t arow, int64_t brow0, EpiInputs<NB, kCols>& in) {
  const int64_t avail = p.rows_b > brow0 ? p.rows_b - brow0 : 0;      // N-side rows of the chunk inside the matrix
  in.ncols = arow < p.rows_a ? static_cast<int>(min(static_cast<int64_t>(kCols), avail)) : 0;
  in.st0 = in.st1 = 1.f;
  in.bias_t = 0.f;
  if (in.ncols == 0) return;
  if (KIND == 0 && NB == 1 && p.dense.a_scale == nullptr) return;      // raw int32 output needs no inputs
  const T* bias = static_cast<const T*>(KIND == 0 ? p.dense.bias : p.fl.bias);
  const T* residual = static_cast<const T*>(KIND == 0 ? p.dense.residual : p.fl.residual);
  const int64_t ldy = KIND == 0 ? (NB == 2 ? p.glu.ldh : p.dense.ldy) : p.fl.ldy;
  const int64_t base = kSwap ? brow0 * ldy + arow : arow * ldy + brow0;
  const int64_t step = kSwap ? ldy : 1;
  const float* x_scale = NB == 2 ? p.glu.a_scale : p.dense.a_scale;
  const float* w_scale0 = NB == 2 ? p.glu.gate_scale : p.dense.b_scale;
  const float* w_scale1 = p.glu.up_scale;
  if constexpr (KIND == 0) {
    if constexpr (kSwap) {
      in.st0 = __ldg(w_scale0 + arow);
      if constexpr (NB == 2) in.st1 = __ldg(w_scale1 + arow);
    } else {
      in.st0 = x_scale[arow];                   // activation scales come from the previous kernel: plain loads (build.py)
    }
  }
  if (bias && kSwap) in.bias_t = to_f32(bias[arow]);
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    const bool ok = j < in.ncols;
    if constexpr (KIND == 0) {
      if constexpr (kSwap) {
        in.sj0[j] = ok ? x_scale[brow0 + j] : 1.f;
      } else {
        in.sj0[j] = ok ? __ldg(w_scale0 + brow0 + j) : 1.f;
        if constexpr (NB == 2) in.sj1[j] = ok ? __ldg(w_scale1 + brow0 + j) : 1.f;
      }
    }
    in.bj[j] = (bias && !kSwap && ok) ? to_f32(bias[brow0 + j]) : in.bias_t;
    in.resj[j] = (residual && ok) ? to_f32(residual[base + j * step]) : 0.f;
  }
}

template <typename T, int KIND, int NB, bool kSwap, int kCols>
__device__ __forceinline__ void epi_finish(const TcParams& p, const uint32_t (&r)[NB][kCols], int64_t arow, int64_t brow0,
                                           const EpiInputs<NB, kCols>& in) {
  if (in.ncols == 0) return;
  const bool has_bias = (KIND == 0 ? p.dense.bias : p.fl.bias) != nullptr;
  const bool has_res = (KIND == 0 ? p.dense.residual : p.fl.residual) != nullptr;
  T* y = static_cast<T*>(KIND == 0 ? (NB == 2 ? p.glu.h : p.dense.y) : p.fl.y);
  const int64_t ldy = KIND == 0 ? (NB == 2 ? p.glu.ldh : p.dense.ldy) : p.fl.ldy;
  const int act = KIND == 0 ? (NB == 2 ? p.glu.act : p.dense.act) : p.fl.act;
  const int64_t base = kSwap ? brow0 * ldy + arow : arow * ldy + brow0;
  const int64_t step = kSwap ? ldy : 1;
  if (KIND == 0 && NB == 1 && p.dense.a_scale == nullptr) {      // raw int32 output (ops::Gemm int8)
#pragma unroll
    for (int j = 0; j < kCols; ++j)
      if (j < in.ncols) p.dense.c_out[base + j * step] = static_cast<int32_t>(r[0][j]);
    return;
  }
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    if (j >= in.ncols) break;
    float v;
    if constexpr (KIND != 0) {
      v = round_to<T>(__uint_as_float(r[0][j]));
      if (has_bias) v = round_to<T>(v + in.bj[j]);
      if (act >= 0) v = round_to<T>(act_call(v, act));
      if (has_res) v = v + in.resj[j];
    } else if constexpr (NB == 2) {
      const float sx = kSwap ? in.sj0[j] : in.st0;
      const float sg = kSwap ? in.st0 : in.sj0[j], su = kSwap ? in.st1 : in.sj1[j];
      float gate = round_to<T>(__fdividef(static_cast<float>(static_cast<int32_t>(r[0][j])), sx * sg));
      gate = round_to<T>(act_call(gate, act));
      const float up = round_to<T>(__fdividef(static_cast<float>(static_cast<int32_t>(r[1][j])), sx * su));
      v = gate * up;
    } else {
      const float sx = kSwap ? in.sj0[j] : in.st0, sw = kSwap ? in.st0 : in.sj0[j];
      v = round_to<T>(__fdividef(static_cast<float>(static_cast<int32_t>(r[0][j])), sx * sw));
      if (has_bias) v = round_to<T>(v + in.bj[j]);
      if (act >= 0) v = round_to<T>(act_call(v, act));
      if (has_res) v = v + in.resj[j];
    }
    y[base + j * step] = from_f32<T>(v);
  }
}

// Persistent stream-K GEMM over (output tile, K block) units (streamk.cuh): a tile whose K range is covered by one CTA is
// finished by that CTA straight from its accumulators, a shared tile by the last of its contributing CTAs.  The TMA
// producer runs ahead into the next segment while the warpgroup finishes the current one.
//
// T = output dtype, KIND = 0 s8 / 1 f16 / 2 bf16, BN = wgmma N (BN * NB <= 128 accumulator registers), NB = weight matrices (2 = GLU),
// kSwap = weights on the M side (decode).
template <typename T, int KIND, int BN, int NB, bool kSwap>
__global__ void __launch_bounds__(kTcThreads, 1)
    gemm_tc_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                   const __grid_constant__ CUtensorMap tm_w2, const TcParams p) {
  using S = TcSmem<BN, NB, kSwap>;
  constexpr int kElem = Elem<KIND>::bytes;
  constexpr int BK = kSwizzleBytes / kElem;            // elements of K per stage
  constexpr int kStages = S::kStages;
  static_assert(BN * NB <= 128 && kStages >= 2, "the accumulators of a tile live in the registers of one warpgroup");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint32_t* accs = reinterpret_cast<uint32_t*>(smem);                                 // [NB * BN columns][kAccPitch]
  uint8_t* ring = smem + S::kAcc;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ring + kStages * S::kStage);       // [kStages]
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int64_t u_begin, u_end;
  p.sched.range(blockIdx.x, u_begin, u_end);
  ring_init<1>(full_bar, empty_bar, kStages);

  if (warp == kProducerWarp) {
    // ===== TMA producer =====
    if (elect_one()) {
      sk::Cursor wc(p.sched, u_begin), xc = wc;      // unit of the next weight / activation copy
      auto weights = [&](int s, int) {
        uint8_t* sw = ring + s * S::kStage + (kSwap ? 0 : S::kA);
        const int row = kSwap ? wc.ta * kTileM : wc.tb * BN;
        tma_load_2d(sw, &tm_w, full_bar + s, wc.kb * BK, row, kEvictFirst);
        if (NB == 2) tma_load_2d(sw + (kSwap ? kTileM : BN) * kSwizzleBytes, &tm_w2, full_bar + s, wc.kb * BK, row, kEvictFirst);
        wc.next(p.sched);
      };
      auto acts = [&](int s, int) {
        uint8_t* sx = ring + s * S::kStage + (kSwap ? S::kA : 0);
        tma_load_2d(sx, &tm_x, full_bar + s, xc.kb * BK, kSwap ? xc.tb * BN : xc.ta * kTileM, kEvictLast);
        xc.next(p.sched);
      };
      produce(full_bar, empty_bar, kStages, S::kStage, static_cast<int>(u_begin), static_cast<int>(u_end - u_begin), weights, acts);
    }
  } else {
    // ===== consumer warpgroup: wgmma over a segment's K blocks, then its epilogue =====
    griddep_wait();                                 // scales / residual come from the previous kernels
    constexpr int kC = 16;                          // columns per chunk (rolled loop over chunks keeps the code small)
    const int rloc = threadIdx.x;                   // tile row owned by this thread
    int it = 0;
    auto mma = [&](int kb0, int kb1) {
      Acc<BN> acc[NB];
#pragma unroll 1
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % kStages;
        mbar_wait(full_bar + s, (it / kStages) & 1);
        const uint32_t sa = smem_u32(ring + s * S::kStage);
        const uint32_t sb = sa + S::kA;
        wgmma_fence();
#pragma unroll
        for (int w = 0; w < NB; ++w)
          mma_block<KIND, BN>(acc[w], sa + (kSwap ? w * kTileM * kSwizzleBytes : 0), sb + (kSwap ? 0 : w * BN * kSwizzleBytes), kb == kb0);
        wgmma_commit();
        wgmma_wait();
        if (lane == 0) mbar_arrive(empty_bar + s);  // this warp's share of the stage has been read
      }
      epi_bar_sync();                               // the previous segment's rows have been read out of accs
#pragma unroll
      for (int w = 0; w < NB; ++w) acc_store<BN>(acc[w], accs + w * BN * kAccPitch);
      epi_bar_sync();
    };
    auto load = [&](EpiInputs<NB, kC>& in, int64_t a0, int64_t b0) { epi_load<T, KIND, NB, kSwap, kC>(p, a0 + rloc, b0, in); };
    auto finish = [&](const EpiInputs<NB, kC>& in, const uint32_t (&r)[NB][kC], int64_t a0, int64_t b0) {
      epi_finish<T, KIND, NB, kSwap, kC>(p, r, a0 + rloc, b0, in);
    };
    sk::consume<NB, BN, kC, KIND == 0, EpiInputs<NB, kC>>(p.sched, blockIdx.x, u_begin, u_end, p.rows_b, accs, p.slots, p.counters, mma, load, finish);
  }
}

// ---- host side ----
template <typename T, int KIND, int BN, int NB, bool kSwap>
void launch_tc(const void* x, const void* w, const void* w2, int64_t m, int64_t n, int64_t k, TcParams p,
               cudaStream_t st) {
  using S = TcSmem<BN, NB, kSwap>;
  constexpr int elem = Elem<KIND>::bytes;
  auto kernel = gemm_tc_kernel<T, KIND, BN, NB, kSwap>;
  allow_dynamic_smem(kernel, S::kBytes);
  const CUtensorMap tmx = make_operand_map(x, m, k, elem, KIND, kSwap ? BN : kTileM);
  const CUtensorMap tmw = make_operand_map(w, n, k, elem, KIND, kSwap ? kTileM : BN);
  const CUtensorMap tmw2 = make_operand_map(w2 ? w2 : w, n, k, elem, KIND, kSwap ? kTileM : BN);
  p.rows_a = kSwap ? n : m;
  p.rows_b = kSwap ? m : n;
  SplitKWorkspace& wsp = SplitKWorkspace::get(st);
  p.sched = sk::choose(div_up(p.rows_a, kTileM), div_up(p.rows_b, BN), div_up(k, kSwizzleBytes / elem), NB * kTileM * BN, wsp);
  p.slots = reinterpret_cast<uint32_t*>(wsp.accum2);
  p.counters = wsp.counters;
  launch_pdl(kernel, dim3(static_cast<unsigned>(p.sched.ctas)), dim3(kTcThreads), S::kBytes, st, tmx, tmw, tmw2, p);
  check_launch();
}

template <typename T, int KIND, int NB>
void launch_tc_shape(const void* x, const void* w, const void* w2, int64_t m, int64_t n, int64_t k,
                     const TcParams& p, cudaStream_t st) {
  if (m <= 16) launch_tc<T, KIND, 16, NB, true>(x, w, w2, m, n, k, p, st);
  else if (m <= 32) launch_tc<T, KIND, 32, NB, true>(x, w, w2, m, n, k, p, st);
  else if (m <= 64) launch_tc<T, KIND, 64, NB, true>(x, w, w2, m, n, k, p, st);
  else if constexpr (NB == 2) launch_tc<T, KIND, 64, NB, false>(x, w, w2, m, n, k, p, st);
  else launch_tc<T, KIND, 128, NB, false>(x, w, w2, m, n, k, p, st);
}

}  // namespace

void gemm_s8_tc(const int8_t* A, const int8_t* B, int64_t M, int64_t N, int64_t K, const DenseEpilogue& epi,
                int dtype, cudaStream_t st) {
  if (M == 0 || N == 0) return;
  CT2_REQUIRE(K % 16 == 0, "gemm_s8: k must be a multiple of 16");
  if (gemm_s8_decode(A, B, M, N, K, epi, dtype, st)) return;
  if (gemm_s8_prefill(A, B, M, N, K, epi, dtype, st)) return;
  TcParams p{};
  p.dense = epi;
  CT2_DISPATCH_DTYPE(dtype, (launch_tc_shape<T, 0, 1>(A, B, nullptr, M, N, K, p, st)));
}

void gemm_s8_glu_tc(const int8_t* A, const int8_t* Bgate, const int8_t* Bup, int64_t M, int64_t N, int64_t K,
                    const GluEpilogue& glu, int dtype, cudaStream_t st) {
  if (M == 0 || N == 0) return;
  CT2_REQUIRE(K % 16 == 0, "gemm_s8: k must be a multiple of 16");
  if (gemm_s8_glu_decode(A, Bgate, Bup, M, N, K, glu, dtype, st)) return;
  if (gemm_s8_glu_prefill(A, Bgate, Bup, M, N, K, glu, dtype, st)) return;
  TcParams p{};
  p.glu = glu;
  CT2_DISPATCH_DTYPE(dtype, (launch_tc_shape<T, 0, 2>(A, Bgate, Bup, M, N, K, p, st)));
}

// a [m,k] T, b [n,k] T -> c [m,n] T (fp32 accumulate), T = f16 or bf16
void gemm_f16_tc(const void* A, const void* B, const void* bias, const void* residual, int act, int64_t M,
                 int64_t N, int64_t K, void* C, int dtype, cudaStream_t st) {
  if (M == 0 || N == 0) return;
  CT2_REQUIRE(K % 8 == 0, "gemm_f16: k must be a multiple of 8");
  CT2_REQUIRE(dtype == CT2B200_F16 || dtype == CT2B200_BF16, "gemm_f16: dtype must be float16 or bfloat16");
  if (gemm_f16_decode(A, B, bias, residual, act, M, N, K, C, dtype, st)) return;
  if (gemm_f16_prefill(A, B, bias, residual, act, M, N, K, C, dtype, st)) return;
  TcParams p{};
  p.fl = FloatEpilogue{bias, residual, C, act, N};
  if (dtype == CT2B200_F16) launch_tc_shape<__half, 1, 1>(A, B, nullptr, M, N, K, p, st);
  else launch_tc_shape<__nv_bfloat16, 2, 1>(A, B, nullptr, M, N, K, p, st);
}

}  // namespace ct2b200
