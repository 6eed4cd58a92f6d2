// gemm_tc.cu — the GENERAL wgmma GEMM (the fallback of the two specialised ones): wgmma (s8 / f16 / bf16) with
// TMA-staged, 128B-swizzled operand tiles in shared memory, accumulators in the registers of one warpgroup, fused
// Dense epilogue (one output row per thread, fed through a shared-memory transpose of the fragments).
//   * gemm_s8_tc / gemm_s8_glu_tc / gemm_f16_tc first try gemm_decode.cu (m <= 64, one tile per CTA, cluster/DSMEM
//     split-K) and gemm_prefill.cu (m > 64, two consumer warpgroups) and only land here for what those
//     do not cover: raw int32 output (ops::Gemm), N tiles beyond one wave at m <= 64 (the 128256-row lm_head),
//     unaligned rows.
//   * persistent stream-K over (tile, K block) units, "swap-AB" for m <= 64, cluster / partition / whole-tile modes,
//     deterministic slot-based reduction of shared tiles (no float atomics).
// Replaces cublasGemmEx s8/f16/bf16 (reference src/cuda/primitives.cu:485-597) + Dequantize epilogue
// (src/ops/dequantize_gpu.cu:30-121) + ops::Add/ops::Mul (src/layers/common.cc:392-401, transformer.cc:31-37).
//
// Warp roles (160 threads): warps 0..3 = consumer warpgroup (wgmma, then the epilogue: thread t owns tile row t),
// warp 4 = TMA producer (one elected lane).
#include <cuda.h>
#include <cudaTypedefs.h>

#include <algorithm>
#include <cstdlib>

#include "../common.cuh"
#include "gemm_common.cuh"
#include "kernels.h"
#include "tc_common.cuh"

namespace ct2b200 {

namespace {

using namespace tc;

struct TcParams {
  int64_t rows_a;      // rows of the M-side operand (n when swapped, m otherwise)
  int64_t rows_b;      // rows of the N-side operand
  int64_t k;           // elements
  int tiles_a;         // M-side tiles of 128 rows
  int tiles_b;         // N-side tiles of BN rows
  int kb_total;        // K blocks (128 bytes of K each) per output tile
  int whole_tiles;     // 1 = CTA ranges are aligned to whole tiles (no scratch needed)
  int cluster_s;       // >= 2: thread-block cluster of cluster_s CTAs per tile, split-K reduced through DSMEM
  int stages;          // smem ring depth actually used (<= TcSmem::kStages; smaller when the DSMEM buffer needs room)
  int part_lo;         // > 0: tile-partitioned split-K — every tile is owned by part_lo (or part_lo + 1) CTAs and every
  int part_rem;        //      CTA works on exactly ONE tile (one reduction round); the first part_rem tiles get +1 CTA
  DenseEpilogue dense;
  GluEpilogue glu;
  FloatEpilogue fl;
  int32_t* ws;
  float* fslots;       // float kinds: per-CTA partial-tile slots [ctas][2][128*BN] (deterministic reduction)
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
__device__ __forceinline__ void epi_load(const TcParams& p, int64_t arow, int64_t brow0, EpiInputs<NB, kCols>& in, int bstep = 1) {
  // N-side rows brow0, brow0 + bstep, ...: how many of the kCols are inside the matrix
  const int64_t avail = p.rows_b > brow0 ? (p.rows_b - brow0 + bstep - 1) / bstep : 0;
  in.ncols = arow < p.rows_a ? static_cast<int>(min(static_cast<int64_t>(kCols), avail)) : 0;
  in.st0 = in.st1 = 1.f;
  in.bias_t = 0.f;
  if (in.ncols == 0) return;
  if (KIND == 0 && NB == 1 && p.dense.a_scale == nullptr) return;      // raw int32 output needs no inputs
  const T* bias = static_cast<const T*>(KIND == 0 ? p.dense.bias : p.fl.bias);
  const T* residual = static_cast<const T*>(KIND == 0 ? p.dense.residual : p.fl.residual);
  const int64_t ldy = KIND == 0 ? (NB == 2 ? p.glu.ldh : p.dense.ldy) : p.fl.ldy;
  const int64_t base = kSwap ? brow0 * ldy + arow : arow * ldy + brow0;
  const int64_t step = (kSwap ? ldy : 1) * bstep;
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
        in.sj0[j] = ok ? x_scale[brow0 + j * bstep] : 1.f;
      } else {
        in.sj0[j] = ok ? __ldg(w_scale0 + brow0 + j * bstep) : 1.f;
        if constexpr (NB == 2) in.sj1[j] = ok ? __ldg(w_scale1 + brow0 + j * bstep) : 1.f;
      }
    }
    in.bj[j] = (bias && !kSwap && ok) ? to_f32(bias[brow0 + j * bstep]) : in.bias_t;
    in.resj[j] = (residual && ok) ? to_f32(residual[base + j * step]) : 0.f;
  }
}

template <typename T, int KIND, int NB, bool kSwap, int kCols>
__device__ __forceinline__ void epi_finish(const TcParams& p, const uint32_t (&r)[NB][kCols], int64_t arow, int64_t brow0,
                                           const EpiInputs<NB, kCols>& in, int bstep = 1) {
  if (in.ncols == 0) return;
  const bool has_bias = (KIND == 0 ? p.dense.bias : p.fl.bias) != nullptr;
  const bool has_res = (KIND == 0 ? p.dense.residual : p.fl.residual) != nullptr;
  T* y = static_cast<T*>(KIND == 0 ? (NB == 2 ? p.glu.h : p.dense.y) : p.fl.y);
  const int64_t ldy = KIND == 0 ? (NB == 2 ? p.glu.ldh : p.dense.ldy) : p.fl.ldy;
  const int act = KIND == 0 ? (NB == 2 ? p.glu.act : p.dense.act) : p.fl.act;
  const int64_t base = kSwap ? brow0 * ldy + arow : arow * ldy + brow0;
  const int64_t step = (kSwap ? ldy : 1) * bstep;
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

// Persistent "stream-K" GEMM: the work is the list of (output tile, K block) units, tile-major; CTA c of P
// owns the contiguous unit range [c*U/P, (c+1)*U/P), so every SM streams the same number of bytes and the TMA
// ring never drains between tiles.  A tile whose K range is covered by one CTA is finished by that CTA
// straight from its accumulators; a tile shared by several CTAs is reduced through the zeroed scratch (integer
// red.global.add => bit-exact, order independent) and finished by the last arriver (ticket).
// The TMA producer runs ahead into the next segment while the warpgroup finishes the current one.
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
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ring + p.stages * S::kStage);      // [kStages] (p.stages used)
  uint64_t* empty_bar = full_bar + kStages;
  __shared__ int s_last;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t KB = p.kb_total;
  const int64_t U = static_cast<int64_t>(p.tiles_a) * p.tiles_b * KB;
  const int64_t P = gridDim.x;
  const int64_t T_all = static_cast<int64_t>(p.tiles_a) * p.tiles_b;
  int64_t u_begin, u_end;
  int part_first = 0, part_n = 0;      // partition mode: first CTA and number of CTAs of this CTA's tile
  const int CS = p.cluster_s;          // cluster mode: CTAs per tile (= cluster size); rank = blockIdx.x % CS
  const int crank = CS >= 2 ? static_cast<int>(blockIdx.x % CS) : 0;
  const int nstages = p.stages;
  if (CS >= 2) {
    const int64_t t = blockIdx.x / CS;
    u_begin = t * KB + crank * KB / CS;
    u_end = t * KB + (crank + 1) * KB / CS;
  } else if (p.part_lo > 0) {
    const int big = p.part_rem * (p.part_lo + 1);
    int t, i;
    if (static_cast<int>(blockIdx.x) < big) {
      part_n = p.part_lo + 1;
      t = blockIdx.x / part_n;
      i = blockIdx.x % part_n;
      part_first = t * part_n;
    } else {
      part_n = p.part_lo;
      const int c2 = blockIdx.x - big;
      t = p.part_rem + c2 / part_n;
      i = c2 % part_n;
      part_first = big + (c2 / part_n) * part_n;
    }
    u_begin = t * KB + i * KB / part_n;
    u_end = t * KB + (i + 1) * KB / part_n;
  } else if (p.whole_tiles) {
    u_begin = (blockIdx.x * T_all / P) * KB;
    u_end = ((blockIdx.x + 1) * T_all / P) * KB;
  } else {
    u_begin = blockIdx.x * U / P;
    u_end = (blockIdx.x + 1) * U / P;
  }

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full_bar + s, 1);
      mbar_init(empty_bar + s, 4);                    // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  griddep_launch();                                 // the next kernel may be scheduled; it waits on our completion
  // cluster mode: reduction buffer behind the barriers; [src rank][plane][owned column][128 rows] of 32-bit partials
  uint32_t* red = reinterpret_cast<uint32_t*>(ring + nstages * S::kStage + 512);
  const int cpr = CS >= 2 ? (BN + CS - 1) / CS : 0;   // columns owned per rank (column j belongs to rank j % CS)
  if (CS >= 2) asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");   // peers are alive before DSMEM traffic

  const CUtensorMap* map_a0 = kSwap ? &tm_w : &tm_x;
  const CUtensorMap* map_a1 = &tm_w2;                   // only when kSwap && NB == 2
  const CUtensorMap* map_b0 = kSwap ? &tm_x : &tm_w;
  const CUtensorMap* map_b1 = &tm_w2;                   // only when !kSwap && NB == 2
  const uint64_t pol_a = kSwap ? kEvictFirst : kEvictLast;   // weights stream once; activations are reused
  const uint64_t pol_b = kSwap ? kEvictLast : kEvictFirst;

  if (warp == kProducerWarp) {
    // ===== TMA producer =====
    if (elect_one()) {
      int it = 0;
      int tile = static_cast<int>(u_begin / KB);
      int kb = static_cast<int>(u_begin - tile * KB);
      int a0 = (tile % p.tiles_a) * kTileM, b0 = (tile / p.tiles_a) * BN;
      // The weights never depend on the previous kernel: their tiles for the first ring fill are requested BEFORE
      // griddepcontrol.wait (so the pipeline fills during the predecessor's tail); the activation tiles after it.
      const int64_t prefill = min(static_cast<int64_t>(nstages), u_end - u_begin);
      auto issue = [&](int s, int kc, bool weights, bool acts) {
        uint8_t* sa = ring + s * S::kStage;
        uint8_t* sb = sa + S::kA;
        if (kSwap) {
          if (weights) {
            tma_load_2d(sa, &tm_w, full_bar + s, kc, a0, kEvictFirst);
            if (NB == 2) tma_load_2d(sa + kTileM * kSwizzleBytes, &tm_w2, full_bar + s, kc, a0, kEvictFirst);
          }
          if (acts) tma_load_2d(sb, &tm_x, full_bar + s, kc, b0, kEvictLast);
        } else {
          if (acts) tma_load_2d(sa, &tm_x, full_bar + s, kc, a0, kEvictLast);
          if (weights) {
            tma_load_2d(sb, &tm_w, full_bar + s, kc, b0, kEvictFirst);
            if (NB == 2) tma_load_2d(sb + BN * kSwizzleBytes, &tm_w2, full_bar + s, kc, b0, kEvictFirst);
          }
        }
      };
      {
        int t2 = tile, k2 = kb, a2 = a0, b2 = b0;
        for (int64_t i = 0; i < prefill; ++i, ++k2) {       // ring is empty at kernel start: no empty-wait needed
          if (k2 == KB) { k2 = 0; ++t2; a2 = (t2 % p.tiles_a) * kTileM; b2 = (t2 / p.tiles_a) * BN; }
          const int sv_a0 = a0, sv_b0 = b0;
          a0 = a2; b0 = b2;
          mbar_expect_tx(full_bar + i, S::kStage);
          issue(static_cast<int>(i), k2 * BK, true, false);
          a0 = sv_a0; b0 = sv_b0;
        }
      }
      griddep_wait();
      for (int64_t u = u_begin; u < u_end; ++u, ++it, ++kb) {
        if (kb == KB) {
          kb = 0;
          ++tile;
          a0 = (tile % p.tiles_a) * kTileM;
          b0 = (tile / p.tiles_a) * BN;
        }
        const int s = it % nstages;
        const uint32_t ph = (it / nstages) & 1;
        if (it < prefill) {
          issue(s, kb * BK, false, true);                   // weights of this stage are already in flight
        } else {
          mbar_wait(empty_bar + s, ph ^ 1);
          mbar_expect_tx(full_bar + s, S::kStage);
          issue(s, kb * BK, true, true);
        }
      }
    }
  } else {
    // ===== consumer warpgroup: wgmma over a segment's K blocks, then its epilogue =====
    griddep_wait();                                 // scales / residual come from the previous kernels
    const int q = warp & 3;
    const int et = threadIdx.x;                     // 0..127 among the consumer threads (== q * 32 + lane)
    const int64_t ldw = kSwap ? p.rows_a : p.rows_b;                 // row pitch of the [m, n] scratch plane
    const int64_t plane = p.rows_a * p.rows_b;
    constexpr int kC = 16;                          // columns per chunk (rolled loop over chunks keeps the code small)
    int it = 0;
    for (int64_t u = u_begin; u < u_end;) {
      const int64_t tile = u / KB;
      const int kb0 = static_cast<int>(u - tile * KB);
      const int kb1 = static_cast<int>(min(KB, static_cast<int64_t>(kb0) + (u_end - u)));
      u += kb1 - kb0;
      const int64_t a0 = (tile % p.tiles_a) * kTileM;
      const int64_t b0 = (tile / p.tiles_a) * BN;
      const bool direct = kb0 == 0 && kb1 == KB;
      const int rloc = q * 32 + lane;               // tile row owned by this thread
      const int64_t arow = a0 + rloc;
      // partial tiles are parked in per-CTA slots (plain coalesced stores: no atomics, nothing to re-zero, no
      // same-address contention) and summed by the last arriver in CTA order (deterministic for the float kinds)
      constexpr int64_t kSlot = static_cast<int64_t>(NB) * kTileM * BN;
      const int nb_valid = static_cast<int>(min(static_cast<int64_t>(BN), p.rows_b - b0));
      uint32_t* my_slot = reinterpret_cast<uint32_t*>(p.fslots) + (static_cast<int64_t>(blockIdx.x) * 2 + (kb0 > 0 ? 0 : 1)) * kSlot;
      int c_lo = 0, c_hi = 0;
      EpiInputs<NB, kC> ein;
      if (direct) epi_load<T, KIND, NB, kSwap, kC>(p, arow, b0, ein);   // issued while the MMAs of this segment run
      {
        Acc<BN> acc[NB];
#pragma unroll 1
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int s = it % nstages;
          mbar_wait(full_bar + s, (it / nstages) & 1);
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
      }
      // pass 0: accumulators -> epilogue (tile owned by this CTA alone) or -> scratch (shared tile);
      // pass 1 (last arriver of a shared tile only): reduced accumulators from the scratch -> epilogue.
#pragma unroll 1
      for (int pass = 0; pass < 2; ++pass) {
#pragma unroll 1
        for (int c0 = 0; c0 < BN; c0 += kC) {
          uint32_t r[NB][kC];
          if (pass == 0) {
            if (direct && c0 > 0) epi_load<T, KIND, NB, kSwap, kC>(p, arow, b0 + c0, ein);
#pragma unroll
            for (int w = 0; w < NB; ++w) acc_load<kC>(accs + (w * BN + c0) * kAccPitch, rloc, r[w]);
          } else {
            // the epilogue inputs and the reduced accumulators are requested together: one memory round trip
            epi_load<T, KIND, NB, kSwap, kC>(p, arow, b0 + c0, ein);
#pragma unroll
            for (int w = 0; w < NB; ++w)
#pragma unroll
              for (int j = 0; j < kC; ++j) r[w][j] = 0u;
            for (int c = c_lo; c <= c_hi; ++c) {        // fixed CTA order => run-to-run deterministic
              const uint32_t* sl = reinterpret_cast<const uint32_t*>(p.fslots) + (static_cast<int64_t>(c) * 2 + (c == c_lo ? 1 : 0)) * kSlot;
#pragma unroll
              for (int w = 0; w < NB; ++w)
#pragma unroll
                for (int j = 0; j < kC; ++j) {
                  if (c0 + j >= nb_valid) continue;
                  const uint32_t v = __ldcg(sl + (static_cast<int64_t>(w) * BN + c0 + j) * kTileM + rloc);
                  if constexpr (KIND == 0) r[w][j] += v;                                   // int32 (wrap-around add)
                  else r[w][j] = __float_as_uint(__uint_as_float(r[w][j]) + __uint_as_float(v));
                }
            }
          }
          if (direct || pass == 1) {
            epi_finish<T, KIND, NB, kSwap, kC>(p, r, arow, b0 + c0, ein);
          } else if (CS >= 2) {
            // cluster mode: column j goes to the CTA of rank j % CS (DSMEM store; the owner's own share stays local)
            if (c0 == 0) asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");   // start-up barrier
#pragma unroll
            for (int j = 0; j < kC; ++j) {
              const int col = c0 + j;
              if (col >= nb_valid) continue;
              const int owner = col % CS;
#pragma unroll
              for (int w = 0; w < NB; ++w) {
                uint32_t* dst = red + ((static_cast<int64_t>(crank) * NB + w) * cpr + col / CS) * kTileM + rloc;
                uint32_t raddr;
                asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(smem_u32(dst)), "r"(owner));
                asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(raddr), "r"(r[w][j]) : "memory");
              }
            }
          } else {
#pragma unroll
            for (int w = 0; w < NB; ++w)
#pragma unroll
              for (int j = 0; j < kC; ++j)       // [plane][N-side row][128 M-side rows]: a warp writes 128 contiguous bytes
                if (c0 + j < nb_valid) my_slot[(static_cast<int64_t>(w) * BN + c0 + j) * kTileM + rloc] = r[w][j];
          }
        }
        if (direct || pass == 1 || CS >= 2) break;
        // ---- shared tile: ticket; the last of the contributing CTAs finishes it ----
        __threadfence();
        epi_bar_sync();
        if (p.part_lo > 0) {
          c_lo = part_first;
          c_hi = part_first + part_n - 1;
        } else {
          c_lo = cta_of_unit(tile * KB, U, P);
          c_hi = cta_of_unit((tile + 1) * KB - 1, U, P);
        }
        if (et == 0) s_last = atomicAdd(p.counters + tile, 1) == c_hi - c_lo;
        epi_bar_sync();
        const bool last = s_last != 0;
        epi_bar_sync();                             // s_last is reused by the next shared tile
        if (!last) break;
        __threadfence();
        if (et == 0) p.counters[tile] = 0;
      }
    }
  }

  if (CS >= 2) {
    // every thread of the cluster meets here: all partials have landed in their owners' shared memory
    __syncwarp();
    if (warp == kProducerWarp || u_end <= u_begin) asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");     // pending start-up phase
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    if (warp < kProducerWarp && u_end > u_begin) {
      // each CTA finishes the columns it owns: sum the CS partials in rank order (deterministic), fused epilogue
      constexpr int kC2 = 16;
      const int q = warp & 3;
      const int rloc = q * 32 + lane;
      const int64_t tile = u_begin / KB;
      const int64_t a0 = (tile % p.tiles_a) * kTileM, b0 = (tile / p.tiles_a) * BN;
      const int64_t arow = a0 + rloc;
#pragma unroll 1
      for (int jj0 = 0; jj0 < cpr; jj0 += kC2) {          // owned columns jj0.. (global column = (jj0 + jj) * CS + crank)
        EpiInputs<NB, kC2> ein;
        const int64_t brow0 = b0 + crank + static_cast<int64_t>(jj0) * CS;
        epi_load<T, KIND, NB, kSwap, kC2>(p, arow, brow0, ein, CS);
        uint32_t r[NB][kC2];
#pragma unroll
        for (int w = 0; w < NB; ++w)
#pragma unroll
          for (int jj = 0; jj < kC2; ++jj) {
            uint32_t acc = 0u;
            if (jj < ein.ncols) {
              for (int src = 0; src < CS; ++src) {
                const uint32_t v = red[((static_cast<int64_t>(src) * NB + w) * cpr + jj0 + jj) * kTileM + rloc];
                if constexpr (KIND == 0) acc += v;
                else acc = __float_as_uint(__uint_as_float(acc) + __uint_as_float(v));
              }
            }
            r[w][jj] = acc;
          }
        epi_finish<T, KIND, NB, kSwap, kC2>(p, r, arow, brow0, ein, CS);
      }
    }
  }

}

// ---- host side ----
template <typename T, int KIND, int BN, int NB, bool kSwap>
void launch_tc(const void* x, const void* w, const void* w2, int64_t m, int64_t n, int64_t k, TcParams p,
               cudaStream_t st) {
  using S = TcSmem<BN, NB, kSwap>;
  constexpr int elem = Elem<KIND>::bytes;
  auto kernel = gemm_tc_kernel<T, KIND, BN, NB, kSwap>;
  allow_dynamic_smem(kernel, 226 * 1024);
  const CUtensorMap tmx = make_operand_map(x, m, k, elem, KIND, kSwap ? BN : kTileM);
  const CUtensorMap tmw = make_operand_map(w, n, k, elem, KIND, kSwap ? kTileM : BN);
  const CUtensorMap tmw2 = make_operand_map(w2 ? w2 : w, n, k, elem, KIND, kSwap ? kTileM : BN);
  p.rows_a = kSwap ? n : m;
  p.rows_b = kSwap ? m : n;
  p.k = k;
  p.tiles_a = div_up(p.rows_a, kTileM);
  p.tiles_b = div_up(p.rows_b, BN);
  p.kb_total = div_up(k, kSwizzleBytes / elem);
  SplitKWorkspace& wsp = SplitKWorkspace::get(st);
  const int64_t tiles = static_cast<int64_t>(p.tiles_a) * p.tiles_b;
  const int64_t units = tiles * p.kb_total;
  int64_t ctas = std::min<int64_t>(wsp.sm_count, units);
  // tiles shared between CTAs go through the scratch: fall back to whole tiles per CTA when it cannot hold them
  const bool scratch_ok = static_cast<size_t>(ctas) * 2 * NB * kTileM * BN <= wsp.accum_elems &&
                          static_cast<size_t>(tiles) <= wsp.num_counters;
  static const bool force_whole = [] { const char* e = std::getenv("CT2B200_GEMM_WHOLE"); return e && e[0] == '1'; }();
  p.whole_tiles = (scratch_ok && !force_whole) ? 0 : 1;
  if (p.whole_tiles) ctas = std::min<int64_t>(wsp.sm_count, tiles);   // tile-aligned CTA ranges
  p.part_lo = p.part_rem = 0;
  p.cluster_s = 0;
  // CT2B200_GEMM_SMEM_KB caps the operand ring of the decode (swap) kernels so that the CTAs of two consecutive GEMMs
  // fit on one SM together: the successor then prefetches its weights while the predecessor drains.
  static const int smem_cap_kb = [] { const char* e = std::getenv("CT2B200_GEMM_SMEM_KB"); return e ? std::atoi(e) : 0; }();
  int max_stages = S::kStages;
  if (kSwap && smem_cap_kb > 0) max_stages = std::max(2, std::min<int>(S::kStages, smem_cap_kb * 1024 / S::kStage));
  p.stages = max_stages;
  size_t smem_bytes = S::kAcc + static_cast<size_t>(max_stages) * S::kStage + 1024 + 256;
  static const int mode = [] { const char* e = std::getenv("CT2B200_GEMM_SPLIT"); return e ? std::atoi(e) : 0; }();   // 1 = stream-K, 2 = partition
  if (kSwap && !force_whole && mode == 0 && tiles < wsp.sm_count) {
    // Decode GEMMs (fewer tiles than SMs).  Split-K through global memory costs several dependent L2 round trips in
    // the tail of every CTA, which is comparable to streaming a whole small GEMM; so
    //  * >= 2 CTAs per tile: thread-block clusters of CS CTAs own one tile, K is split inside the cluster and the
    //    partial accumulators are exchanged through distributed shared memory (no global traffic, one cluster barrier);
    //  * otherwise whole tiles (no reduction at all) on as many SMs as there are tiles.
    int cs = static_cast<int>(wsp.sm_count / tiles);
    if (cs > 4) cs = 4;
    if (cs == 3 && tiles * 3 > wsp.sm_count / 4 * 4) cs = 2; // odd clusters do not tile the GPCs: leave a cluster of 4 SMs spare so all are co-resident (not measured on H100)
    while (cs >= 2 && p.kb_total < 2 * cs) --cs;
    if (cs >= 2) {
      const size_t red_bytes = static_cast<size_t>(cs) * NB * ((BN + cs - 1) / cs) * kTileM * 4;
      int stages = max_stages;
      while (stages > 2 && S::kAcc + static_cast<size_t>(stages) * S::kStage + 1024 + 512 + red_bytes > 226 * 1024) --stages;
      p.cluster_s = cs;
      p.stages = stages;
      p.whole_tiles = 0;
      ctas = tiles * cs;
      smem_bytes = S::kAcc + static_cast<size_t>(stages) * S::kStage + 1024 + 512 + red_bytes;
    } else {
      p.whole_tiles = 1;
      ctas = tiles;
    }
  } else if (!p.whole_tiles && mode != 1 && ctas >= 2 * tiles && p.kb_total >= 2 * ((ctas + tiles - 1) / tiles)) {
    // tile-partitioned split-K through the global slots: one reduction round per CTA
    p.part_lo = static_cast<int>(ctas / tiles);
    p.part_rem = static_cast<int>(ctas % tiles);
  }
  p.ws = wsp.accum;
  p.fslots = reinterpret_cast<float*>(wsp.accum2);
  p.counters = wsp.counters;
  if (p.cluster_s >= 2) {
    launch_clustered(kernel, dim3(static_cast<unsigned>(ctas)), dim3(kTcThreads), smem_bytes, p.cluster_s, st, tmx, tmw, tmw2, p);
    check_launch();
    return;
  }
  launch_pdl(kernel, dim3(static_cast<unsigned>(ctas)), dim3(kTcThreads), smem_bytes, st, tmx, tmw, tmw2, p);
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
