// streamk.cuh — the persistent stream-K schedule of the two general wgmma GEMMs, gemm_tc.cu (INT8 / f16 / bf16) and
// awq.cu (AWQ-INT4): which (output tile, K block) units each CTA works on, and how a tile shared by several CTAs is
// summed and finished.  The kernels pass in what is their own (wgmma loop, epilogue) as callbacks.
#pragma once

#include <algorithm>

#include "gemm_common.cuh"
#include "tc_common.cuh"

namespace ct2b200 {
namespace sk {

using namespace tc;

// The work is the list of (output tile, K block) units, tile-major: unit u = tile * kb + K block.  Tile t covers M-side
// tile t % tiles_a and N-side tile t / tiles_a.  Every CTA owns one contiguous unit range, in one of three modes:
//   * stream-K: CTA c of P owns [c*U/P, (c+1)*U/P), so every SM streams the same number of bytes and the TMA ring never
//     drains between tiles;
//   * tile-partitioned (part_lo > 0): every tile is owned by part_lo CTAs, the first part_rem tiles by part_lo + 1, and
//     every CTA works on exactly ONE tile (one reduction round);
//   * whole tiles: the ranges are aligned to tiles, so no tile is shared.
struct Schedule {
  int tiles_a;      // M-side tiles
  int tiles;        // output tiles
  int kb;           // K blocks per tile
  int ctas;         // grid size
  int part_lo;
  int part_rem;
  int whole;

  // unit range [lo, hi) of CTA c
  __device__ __forceinline__ void range(int c, int64_t& lo, int64_t& hi) const {
    const int64_t KB = kb;
    if (part_lo > 0) {
      const int big = part_rem * (part_lo + 1);             // CTAs of the tiles with part_lo + 1 owners
      const int n = c < big ? part_lo + 1 : part_lo;
      const int t = c < big ? c / n : part_rem + (c - big) / n;
      const int i = c < big ? c % n : (c - big) % n;
      lo = t * KB + i * KB / n;
      hi = t * KB + (i + 1) * KB / n;
    } else if (whole) {
      lo = (c * static_cast<int64_t>(tiles) / ctas) * KB;
      hi = ((c + 1) * static_cast<int64_t>(tiles) / ctas) * KB;
    } else {
      const int64_t U = tiles * KB;
      lo = c * U / ctas;
      hi = (c + 1) * U / ctas;
    }
  }

  // CTAs c_lo..c_hi whose ranges cover tile t (only the stream-K and tile-partitioned modes share tiles)
  __device__ __forceinline__ void contributors(int64_t t, int& c_lo, int& c_hi) const {
    if (part_lo > 0) {
      const bool big = t < part_rem;
      c_lo = static_cast<int>(big ? t * (part_lo + 1) : part_rem * (part_lo + 1) + (t - part_rem) * part_lo);
      c_hi = c_lo + (big ? part_lo : part_lo - 1);
    } else {
      const int64_t U = static_cast<int64_t>(tiles) * kb;
      auto cta_of_unit = [&](int64_t u) { return static_cast<int>(((u + 1) * ctas + U - 1) / U - 1); };
      c_lo = cta_of_unit(t * kb);
      c_hi = cta_of_unit((t + 1) * kb - 1);
    }
  }
};

// stream-K over min(SMs, units) CTAs
inline Schedule stream_k(int tiles_a, int tiles_b, int kb, int sm_count) {
  const int64_t tiles = static_cast<int64_t>(tiles_a) * tiles_b;
  const int64_t units = tiles * kb;
  CT2_REQUIRE(units < (int64_t(1) << 31), "gemm: more than 2^31 (tile, K block) units");
  Schedule s{};
  s.tiles_a = tiles_a;
  s.tiles = static_cast<int>(tiles);
  s.kb = kb;
  s.ctas = static_cast<int>(std::min<int64_t>(sm_count, units));
  return s;
}

// the partial-tile slots of every CTA ([ctas][2][slot_words]) and one ticket counter per tile fit the workspace
inline bool slots_fit(const Schedule& s, int64_t slot_words, const SplitKWorkspace& ws) {
  return static_cast<size_t>(s.ctas) * 2 * slot_words <= ws.accum_elems && static_cast<size_t>(s.tiles) <= ws.num_counters;
}

// The mode of gemm_tc.cu (awq.cu stays pure stream-K): whole tiles when the slots cannot hold the shared tiles;
// tile-partitioned split-K when every tile gets at least two CTAs with at least two K blocks each; stream-K otherwise.
inline Schedule choose(int tiles_a, int tiles_b, int kb, int64_t slot_words, const SplitKWorkspace& ws) {
  Schedule s = stream_k(tiles_a, tiles_b, kb, ws.sm_count);
  if (!slots_fit(s, slot_words, ws)) {
    s.whole = 1;
    s.ctas = std::min(ws.sm_count, s.tiles);
  } else if (s.ctas >= 2 * static_cast<int64_t>(s.tiles) && kb >= 2 * div_up(s.ctas, s.tiles)) {
    s.part_lo = s.ctas / s.tiles;
    s.part_rem = s.ctas % s.tiles;
  }
  return s;
}

// (M-side tile, N-side tile, K block) of a unit, advanced one unit per call (no division per step)
struct Cursor {
  int ta, tb, kb;
  __device__ __forceinline__ Cursor(const Schedule& s, int64_t u) {
    const int64_t t = u / s.kb;
    kb = static_cast<int>(u - t * s.kb);
    ta = static_cast<int>(t % s.tiles_a);
    tb = static_cast<int>(t / s.tiles_a);
  }
  __device__ __forceinline__ void next(const Schedule& s) {
    if (++kb == s.kb) {
      kb = 0;
      if (++ta == s.tiles_a) { ta = 0; ++tb; }
    }
  }
};

// The consumer warpgroup (threads 0..127, thread = M-side row of the tile) walks the units [lo, hi) of CTA `cta` one
// segment (the units of one tile) at a time:
//   mma(kb0, kb1):     the wgmma loop over K blocks [kb0, kb1); leaves the tile's accumulators in accs
//                      ([NB * BN columns][kAccPitch]) and ends with epi_bar_sync;
//   load(in, a0, b0):  issues the epilogue's global loads for the kC-column chunk at N-side row b0 of the tile at M-side
//                      row a0 into `in` (an Inputs of the segment);
//   finish(in, r, a0, b0): epilogue of that chunk, r[w][j] = raw accumulators (int32 or fp32 bits) of N-side row b0 + j.
// A tile covered by one segment is finished straight from its accumulators.  The partial tiles of a shared one are parked
// in per-CTA slots (plain coalesced stores: no atomics, nothing to re-zero, no same-address contention), and the last of
// its contributing CTAs (ticket on counters[tile], left at zero) sums the slots in CTA order, run-to-run deterministic:
// int32 wrap-around adds when kInt, fp32 adds from +0 otherwise.  rows_b = N-side rows of the matrix.
template <int NB, int BN, int kC, bool kInt, typename Inputs, typename Mma, typename Load, typename Finish>
__device__ __forceinline__ void consume(const Schedule& s, int cta, int64_t lo, int64_t hi, int64_t rows_b, const uint32_t* accs,
                                        uint32_t* slots, int32_t* counters, const Mma& mma, const Load& load, const Finish& finish) {
  __shared__ int s_last;
  constexpr int64_t kSlot = static_cast<int64_t>(NB) * kTileM * BN;      // [NB][BN N-side rows][128 M-side rows] words
  auto slot = [&](int c, bool first) { return slots + (static_cast<int64_t>(c) * 2 + (first ? 1 : 0)) * kSlot; };
  const int rloc = threadIdx.x;
  for (int64_t u = lo; u < hi;) {
    const int64_t tile = u / s.kb;
    const int kb0 = static_cast<int>(u - tile * s.kb);
    const int kb1 = static_cast<int>(min(static_cast<int64_t>(s.kb), static_cast<int64_t>(kb0) + (hi - u)));
    u += kb1 - kb0;
    const int64_t a0 = (tile % s.tiles_a) * kTileM;
    const int64_t b0 = (tile / s.tiles_a) * BN;
    const bool direct = kb0 == 0 && kb1 == s.kb;
    Inputs in;
    if (direct) load(in, a0, b0);                     // issued while the MMAs of this segment run
    mma(kb0, kb1);
    const int nb_valid = static_cast<int>(min(static_cast<int64_t>(BN), rows_b - b0));
    if (direct) {                                     // the tile is this CTA's alone: accumulators -> epilogue
#pragma unroll 1
      for (int c0 = 0; c0 < BN; c0 += kC) {
        uint32_t r[NB][kC];
        if (c0 > 0) load(in, a0, b0 + c0);
#pragma unroll
        for (int w = 0; w < NB; ++w) acc_load<kC>(accs + (w * BN + c0) * kAccPitch, rloc, r[w]);
        finish(in, r, a0, b0 + c0);
      }
      continue;
    }
    // ---- shared tile: park the partial tile in this CTA's slot ----
    uint32_t* my_slot = slot(cta, kb0 == 0);
#pragma unroll 1
    for (int c0 = 0; c0 < BN; c0 += kC) {
      uint32_t r[NB][kC];
#pragma unroll
      for (int w = 0; w < NB; ++w) acc_load<kC>(accs + (w * BN + c0) * kAccPitch, rloc, r[w]);
      uint32_t* dst = my_slot + c0 * kTileM + rloc;
#pragma unroll
      for (int w = 0; w < NB; ++w)
#pragma unroll
        for (int j = 0; j < kC; ++j)                  // a warp writes 128 contiguous bytes
          if (j < nb_valid - c0) dst[(w * BN + j) * kTileM] = r[w][j];
    }
    // ---- ticket: the last of the contributing CTAs finishes the tile ----
    __threadfence();
    epi_bar_sync();
    int c_lo, c_hi;
    s.contributors(tile, c_lo, c_hi);
    if (rloc == 0) s_last = atomicAdd(counters + tile, 1) == c_hi - c_lo;
    epi_bar_sync();
    const bool last = s_last != 0;
    epi_bar_sync();                                   // s_last is reused by the next shared tile
    if (!last) continue;
    __threadfence();
    if (rloc == 0) counters[tile] = 0;
#pragma unroll 1
    for (int c0 = 0; c0 < BN; c0 += kC) {
      uint32_t r[NB][kC];
      load(in, a0, b0 + c0);                          // requested together with the slots: one memory round trip
#pragma unroll
      for (int w = 0; w < NB; ++w)
#pragma unroll
        for (int j = 0; j < kC; ++j) r[w][j] = 0u;
      // one pointer walks the slots (c_lo's first-segment slot, then slot 0 of each later CTA), so that the loads below
      // are constant offsets from it
      const uint32_t* sl = slot(c_lo, true) + c0 * kTileM + rloc;
      for (int c = c_lo; c <= c_hi; ++c, sl += (c == c_lo + 1 ? 1 : 2) * kSlot) {
#pragma unroll
        for (int w = 0; w < NB; ++w)
#pragma unroll
          for (int j = 0; j < kC; ++j) {
            if (j >= nb_valid - c0) continue;
            const uint32_t v = __ldcg(sl + (w * BN + j) * kTileM);
            if constexpr (kInt) r[w][j] += v;
            else r[w][j] = __float_as_uint(__uint_as_float(r[w][j]) + __uint_as_float(v));
          }
      }
      finish(in, r, a0, b0 + c0);
    }
  }
}

}  // namespace sk
}  // namespace ct2b200
