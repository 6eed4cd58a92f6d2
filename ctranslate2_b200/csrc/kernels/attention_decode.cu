// attention_decode.cu — single-token (decode) attention as ONE persistent, work-balanced kernel.
//
// Replaces, per layer and step, the reference chain  Split(q,k,v) -> Rotary(q,k) -> Concat(cache,k/v) -> MatMul(QK^T)
// -> SoftMax -> MatMul(PV) -> combine_heads  (src/layers/attention.cc:442-615, 178-287; or the FA2 split-KV path
// src/ops/flash_attention_gpu.cu:195-366) by one launch that reads every cached K/V byte exactly once.
//
// Work decomposition.  A unit is one 64-key tile of one (batch row, KV head); units are numbered row-major
// (row, KV head, tile) and CTA c of P owns the contiguous range [c*U/P, (c+1)*U/P).  So every SM streams the same
// number of cache bytes whatever the batch size, the ragged lengths or the KV-head count (the split-KV grid of the
// previous kernel needed B*Hkv*splits to divide the SM count and paid its prologue/combine once per slice), the
// cp.async ring never drains between (row, head) pairs, and consecutive units of a CTA are consecutive cache lines.
//   * a pair that lies inside one CTA is normalised and written directly;
//   * a pair shared by several CTAs: the CTA that holds its HEAD combines.  The others (they meet the pair at the START
//     of their range) park fp32 partials (O, m, l) in their workspace slot — O and m first, then l with release
//     semantics, l > 0 doubling as the "ready" flag — and move on without waiting.  The head owner reaches the pair
//     at the END of its range, when the other parts are normally long done, folds them in slot order (deterministic)
//     and clears the flags for the next launch.  All CTAs of the grid are co-resident (grid = occupancy x SMs).
// Inner loop (per tile): the G query heads of the KV head are rows 0..G-1 of a 16-row MMA tile; warp w owns keys
// [16w, 16w+16): S = Q K^T (mma.sync m16n8k16, fp32), online softmax in fp32, O += P V.  K/V tiles are staged by TMA
// (64 keys x 128 B boxes, SWIZZLE_128B, one mbarrier per stage; 96 KB per CTA for D = 128, two CTAs per SM).
// The new token's rotated K and its V are appended to the cache by the CTA that owns the pair's last tile.
#include <cstdlib>
#include <string>

#include "../common.cuh"
#include "kernels.h"
#include "attention_tile.cuh"
#include "mma_common.cuh"
#include "tc_common.cuh"

namespace ct2b200 {
namespace {

using namespace mma;
using namespace attn;

constexpr int kThreads = 128;
constexpr int kTile = 64;            // keys per unit
constexpr int kStages = 3;
constexpr int kMaxBatch = 1024;      // rows whose tile counts fit the shared prefix table
constexpr int kSlots = 64;           // partial slots per (row, head) = max CTAs sharing one pair

template <typename T>
__device__ __forceinline__ float rope_elem(const T* x, const float* sin, const float* cos, int i, int D, bool interleave) {
  float other;
  if (interleave) other = (i & 1) ? to_f32(x[i - 1]) : -to_f32(x[i + 1]);
  else other = (i < D / 2) ? -to_f32(x[i + D / 2]) : to_f32(x[i - D / 2]);
  return to_f32(x[i]) * cos[i] + other * sin[i];
}

struct UnitCursor {                  // position in the (row, KV head, tile) enumeration
  int b, kvh, t, tiles;              // tiles = tiles of row b
};

template <typename T, int D, int G>
__global__ void __launch_bounds__(kThreads, 2)
    attention_decode_persistent_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                                       const T* __restrict__ qkv, T* __restrict__ k_cache, T* __restrict__ v_cache,
                                       const float* __restrict__ sin_t, const float* __restrict__ cos_t,
                                       const int32_t* __restrict__ lens, int batch, int H, int Hkv, int64_t max_len,
                                       bool interleave, float scale_log2, T* __restrict__ out,
                                       float* __restrict__ partials, int32_t* __restrict__ tickets) {
  constexpr int NW = kThreads / 32;
  constexpr int kTileElems = kTile * D;
  constexpr size_t PS = static_cast<size_t>(D) + 2;
  extern __shared__ uint8_t smem_dyn[];
  // TMA boxes (64 keys x 128 B, SWIZZLE_128B) need a 1024-byte aligned base
  uint8_t* smem_raw = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  T* sK = reinterpret_cast<T*>(smem_raw);                           // [stages][D/64 boxes][64 keys][128 B]
  T* sV = sK + kStages * kTileElems;
  float* s_q = reinterpret_cast<float*>(sV + kStages * kTileElems);  // [2][G][D] (current / next segment)
  int* s_pref = reinterpret_cast<int*>(s_q + 2 * G * D);             // [batch + 1] tiles before row b
  __shared__ float s_m[NW][G], s_l[NW][G];
  __shared__ __align__(8) uint64_t full_bar[kStages];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3;
  const int64_t row_w = static_cast<int64_t>(H + 2 * Hkv) * D;

  if (tid == 0) {
    for (int st = 0; st < kStages; ++st) tc::mbar_init(full_bar + st, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  griddep_launch();
  griddep_wait();                                 // qkv and lens come from the previous kernels

  // ---- tiles per row and their prefix sums ----
  if (warp == 0) {
    int carry = 0;
    for (int base = 0; base < batch; base += 32) {
      const int b = base + lane;
      int v = b < batch ? (lens[b] + 1 + kTile - 1) / kTile : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += n;
      }
      if (b < batch) s_pref[b + 1] = carry + v;
      carry += __shfl_sync(0xffffffffu, v, 31);
    }
    if (lane == 0) s_pref[0] = 0;
  }
  __syncthreads();
  const int64_t U = static_cast<int64_t>(s_pref[batch]) * Hkv;
  // no pair may be shared by more than kSlots CTAs: with fewer units than CTAs, use fewer CTAs
  int max_tiles = 0;
  for (int b = lane; b < batch; b += 32) max_tiles = max(max_tiles, s_pref[b + 1] - s_pref[b]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) max_tiles = max(max_tiles, __shfl_xor_sync(0xffffffffu, max_tiles, o));
  const int min_units = (max_tiles + kSlots - 2) / (kSlots - 1);    // units per CTA so that a pair spans < kSlots CTAs
  // every CTA must own at least one unit (the contributors of a pair are then consecutive CTAs)
  const int64_t P = min(static_cast<int64_t>(gridDim.x), max(static_cast<int64_t>(1), U / max(min_units, 1)));
  if (static_cast<int64_t>(blockIdx.x) >= P) return;
  const int64_t u0 = blockIdx.x * U / P, u1 = (blockIdx.x + 1) * U / P;
  if (u1 <= u0) return;

  auto cursor_at = [&](int64_t u) {
    // row b with s_pref[b]*Hkv <= u < s_pref[b+1]*Hkv (rows always have >= 1 tile)
    int lo = 0, hi = batch - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (static_cast<int64_t>(s_pref[mid]) * Hkv <= u) lo = mid; else hi = mid - 1;
    }
    UnitCursor c;
    c.b = lo;
    c.tiles = s_pref[lo + 1] - s_pref[lo];
    const int r = static_cast<int>(u - static_cast<int64_t>(s_pref[lo]) * Hkv);
    c.kvh = r / c.tiles;
    c.t = r - c.kvh * c.tiles;
    return c;
  };
  auto advance = [&](UnitCursor& c) {
    if (++c.t == c.tiles) {
      c.t = 0;
      if (++c.kvh == Hkv) {
        c.kvh = 0;
        ++c.b;
        c.tiles = c.b < batch ? s_pref[c.b + 1] - s_pref[c.b] : 1;
      }
    }
  };
  // first and last CTA of the pair that contains unit u (pair = units [base, base + tiles))
  auto cta_of = [&](int64_t u) { return static_cast<int>(((u + 1) * P - 1) / U); };

  // ---- append the new token's K (rotated) and V for every pair whose last tile is ours ----
  {
    UnitCursor c = cursor_at(u0);
    int64_t u = u0;
    while (u < u1) {
      const int64_t last = u + (c.tiles - 1 - c.t);               // unit of this pair's last tile
      if (last < u1) {
        const int pos = lens[c.b];
        const T* k_in = qkv + c.b * row_w + static_cast<int64_t>(H) * D + static_cast<int64_t>(c.kvh) * D;
        const T* v_in = k_in + static_cast<int64_t>(Hkv) * D;
        const float* sn = sin_t + static_cast<int64_t>(pos) * D;
        const float* cs = cos_t + static_cast<int64_t>(pos) * D;
        T* kc = k_cache + ((static_cast<int64_t>(c.b) * Hkv + c.kvh) * max_len + pos) * D;
        T* vc = v_cache + ((static_cast<int64_t>(c.b) * Hkv + c.kvh) * max_len + pos) * D;
        for (int i = tid; i < D; i += kThreads) {
          kc[i] = from_f32<T>(rope_elem(k_in, sn, cs, i, D, interleave));
          vc[i] = v_in[i];
        }
      }
      // jump to the first unit of the next pair
      u = last + 1;
      c.t = c.tiles - 1;
      advance(c);
    }
  }
  asm volatile("fence.proxy.async;" ::: "memory");   // the appended rows (generic proxy) before the TMA (async proxy) reads
  __syncthreads();

  // ---- K/V tile loads: TMA, one mbarrier per stage, issued by thread 0 ----
  using Ctx = TileCtx<T, D, true>;
  Ctx cx;
  cx.init(tid);
  const uint32_t sK_u32 = static_cast<uint32_t>(__cvta_generic_to_shared(sK));
  const uint32_t sV_u32 = static_cast<uint32_t>(__cvta_generic_to_shared(sV));
  auto load_unit = [&](int stage, const UnitCursor& c) {
    const int row = static_cast<int>((static_cast<int64_t>(c.b) * Hkv + c.kvh) * max_len) + c.t * kTile;
    tc::mbar_expect_tx(full_bar + stage, 2 * Ctx::kTileBytes);
#pragma unroll
    for (int h = 0; h < Ctx::kBoxes; ++h) {
      tc::tma_load_2d(reinterpret_cast<uint8_t*>(sK) + stage * Ctx::kTileBytes + h * Ctx::kBoxBytes, &tm_k, full_bar + stage,
                      h * 64, row, tc::kEvictFirst);
      tc::tma_load_2d(reinterpret_cast<uint8_t*>(sV) + stage * Ctx::kTileBytes + h * Ctx::kBoxBytes, &tm_v, full_bar + stage,
                      h * 64, row, tc::kEvictFirst);
    }
  };
  UnitCursor lc = cursor_at(u0);                   // load cursor (runs kStages - 1 units ahead)
  int64_t lu = u0;
#pragma unroll
  for (int s = 0; s < kStages - 1; ++s) {
    if (lu < u1) {
      if (warp == 0 && tc::elect_one()) load_unit(s, lc);
      advance(lc);
      ++lu;
    }
  }

  UnitCursor cc = cursor_at(u0);                   // compute cursor
  // ---- rotated, pre-scaled queries of a (row, KV head): raw loads first (prefetch), rotation + store later ----
  constexpr int QE = (G * D + kThreads - 1) / kThreads;            // query elements per thread
  float q_x[QE], q_o[QE], q_s[QE], q_c[QE];
  auto q_load = [&](const UnitCursor& c) {
    const int pos = lens[c.b];
    const T* q_in = qkv + c.b * row_w + static_cast<int64_t>(c.kvh) * G * D;
    const float* sn = sin_t + static_cast<int64_t>(pos) * D;
    const float* cs = cos_t + static_cast<int64_t>(pos) * D;
#pragma unroll
    for (int k = 0; k < QE; ++k) {
      const int e = tid + k * kThreads;
      if (e < G * D) {
        const int h = e / D, i = e % D;
        const T* x = q_in + h * D;
        q_x[k] = to_f32(x[i]);
        if (interleave) q_o[k] = (i & 1) ? to_f32(x[i - 1]) : -to_f32(x[i + 1]);
        else q_o[k] = (i < D / 2) ? -to_f32(x[i + D / 2]) : to_f32(x[i - D / 2]);
        q_s[k] = sn[i];
        q_c[k] = cs[i];
      }
    }
  };
  auto q_store = [&](float* dst) {
#pragma unroll
    for (int k = 0; k < QE; ++k) {
      const int e = tid + k * kThreads;
      if (e < G * D) dst[e] = (q_x[k] * q_c[k] + q_o[k] * q_s[k]) * scale_log2;
    }
  };
  int qb = 0;                                      // s_q buffer of the current segment
  q_load(cc);
  q_store(s_q);

  uint32_t qf[D / 16][2];                          // Q as A fragments: rows 0..G-1 = heads (a0, a2); rows 8..15 are zero
  WarpAcc<D> acc;
  acc.reset();
  bool seg_start = true;
  int seg_t0 = cc.t;                               // first tile of the current segment
  int it = 0;
  for (int64_t u = u0; u < u1; ++u, ++it) {
    const int stage = it % kStages;
    if (lu < u1) {                                 // refills the stage consumed in iteration it - 1 (trailing __syncthreads)
      if (warp == 0 && tc::elect_one()) load_unit((it + kStages - 1) % kStages, lc);
      advance(lc);
      ++lu;
    }
    const int nkeys = lens[cc.b] + 1;
    const bool pair_end = cc.t == cc.tiles - 1;
    const bool prefetch_q = pair_end && u + 1 < u1;   // the next unit opens a new (row, head): fetch its queries now
    if (prefetch_q) {
      UnitCursor nc = cc;
      advance(nc);
      q_load(nc);
    }
    if (seg_start) {
      __syncthreads();                             // s_q[qb] is complete
      const float* sq = s_q + qb * G * D;
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const float* qr = sq + (g < G ? g : 0) * D + kk * 16 + 2 * t4;
        const bool real = g < G;
        qf[kk][0] = real ? pack2<T>(qr[0], qr[1]) : 0u;
        qf[kk][1] = real ? pack2<T>(qr[8], qr[9]) : 0u;
      }
      acc.reset();
      seg_t0 = cc.t;
      seg_start = false;
    }
    tc::mbar_wait(full_bar + stage, (it / kStages) & 1);
    tile_step<T, D, true>(cx, sK_u32 + stage * Ctx::kTileBytes, sV_u32 + stage * Ctx::kTileBytes, warp, lane, qf, acc,
                          nkeys - cc.t * kTile);
    if (prefetch_q) q_store(s_q + (qb ^ 1) * G * D);   // read by the next iteration, after its __syncthreads
    __syncthreads();                               // the stage is free again (and may serve as scratch below)

    if (pair_end || u == u1 - 1) {
      // ---- end of a segment: merge the 4 warps; scratch = the stage just consumed (refilled only after the sync below)
      float* s_o = reinterpret_cast<float*>(sK + stage * kTileElems);      // [NW][G][D] fp32 <= 16 KB
      float ls = acc.l;
      ls += __shfl_xor_sync(0xffffffffu, ls, 1);
      ls += __shfl_xor_sync(0xffffffffu, ls, 2);
      if (g < G && t4 == 0) { s_m[warp][g] = acc.m; s_l[warp][g] = ls; }
      if (g < G) {
#pragma unroll
        for (int j = 0; j < D / 8; ++j)
          *reinterpret_cast<float2*>(s_o + (warp * G + g) * D + j * 8 + 2 * t4) = make_float2(acc.o[j][0], acc.o[j][1]);
      }
      __syncthreads();
      const bool head = seg_t0 == 0;               // this CTA holds the first tile of the pair
      const int64_t pair_base = u - cc.t;          // first unit of this pair
      const int c_first = cta_of(pair_base), c_last = cta_of(pair_base + cc.tiles - 1);
      const int nsplit = (head && pair_end) ? 1 : c_last - c_first + 1;
      const int slot = static_cast<int>(blockIdx.x) - c_first;
      float* part = partials + (static_cast<int64_t>(cc.b) * H + static_cast<int64_t>(cc.kvh) * G) * kSlots * PS;
      T* out_row = out + static_cast<int64_t>(cc.b) * H * D + static_cast<int64_t>(cc.kvh) * G * D;
      if (head && nsplit > 1) {
        // wait for the other parts (normally long complete): their l field turns non-zero
        for (int e = tid; e < G * (nsplit - 1); e += kThreads) {
          const int h = e / (nsplit - 1), sidx = 1 + e % (nsplit - 1);
          const float* lf = part + (static_cast<int64_t>(h) * kSlots + sidx) * PS + D + 1;
          float lv;
          do {
            asm volatile("ld.acquire.gpu.global.f32 %0, [%1];" : "=f"(lv) : "l"(lf) : "memory");
          } while (lv == 0.f);
        }
        __syncthreads();
      }
      for (int e = tid; e < G * D; e += kThreads) {
        const int h = e / D, i = e % D;
        float mm = -INFINITY;
#pragma unroll
        for (int w = 0; w < NW; ++w) mm = fmaxf(mm, s_m[w][h]);
        float ll = 0.f, a = 0.f;
#pragma unroll
        for (int w = 0; w < NW; ++w) {
          const float c = s_m[w][h] == -INFINITY ? 0.f : exp2f(s_m[w][h] - mm);
          ll += s_l[w][h] * c;
          a += s_o[(w * G + h) * D + i] * c;
        }
        if (head) {
          for (int sidx = 1; sidx < nsplit; ++sidx) {       // slot order: deterministic
            const float* ph = part + (static_cast<int64_t>(h) * kSlots + sidx) * PS;
            const float ms = __ldcg(ph + D), lsv = __ldcg(ph + D + 1), os = __ldcg(ph + i);
            const float nm = fmaxf(mm, ms);
            const float c0 = exp2f(mm - nm), c1 = exp2f(ms - nm);
            a = a * c0 + os * c1;
            ll = ll * c0 + lsv * c1;
            mm = nm;
          }
          out_row[e] = from_f32<T>(a * (1.f / ll));
        } else {
          float* ph = part + (static_cast<int64_t>(h) * kSlots + slot) * PS;
          ph[i] = a;
          if (i == 0) ph[D] = mm;
        }
      }
      if (head && nsplit > 1) {
        __syncthreads();                           // every thread has read the parts: clear the flags for the next launch
        for (int e = tid; e < G * (nsplit - 1); e += kThreads) {
          const int h = e / (nsplit - 1), sidx = 1 + e % (nsplit - 1);
          part[(static_cast<int64_t>(h) * kSlots + sidx) * PS + D + 1] = 0.f;
        }
      } else if (!head) {
        __threadfence();
        __syncthreads();                           // O and m of every head are written and fenced ...
        if (tid < G) {                             // ... then l, which publishes the record
          float mm = -INFINITY;
#pragma unroll
          for (int w = 0; w < NW; ++w) mm = fmaxf(mm, s_m[w][tid]);
          float ll = 0.f;
#pragma unroll
          for (int w = 0; w < NW; ++w) ll += s_l[w][tid] * (s_m[w][tid] == -INFINITY ? 0.f : exp2f(s_m[w][tid] - mm));
          float* lf = part + (static_cast<int64_t>(tid) * kSlots + slot) * PS + D + 1;
          asm volatile("st.release.gpu.global.f32 [%0], %1;" ::"l"(lf), "f"(ll) : "memory");
        }
      }
      // the scratch was written through the generic proxy; the next iteration refills this stage through the async proxy
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();                             // scratch stage released before the next iteration refills it
      seg_start = true;
      if (pair_end) qb ^= 1;
    }
    advance(cc);
  }
}

template <typename T, int D, int G>
void launch_persistent(const void* qkv, void* kc, void* vc, const float* sn, const float* cs, const int32_t* lens,
                       int64_t batch, int H, int Hkv, int64_t max_len, bool interleave, float scale, void* out,
                       float* partials, int32_t* tickets, int sm_count, cudaStream_t st) {
  auto kernel = attention_decode_persistent_kernel<T, D, G>;
  const size_t smem = static_cast<size_t>(2 * kStages * kTile * D) * sizeof(T) + static_cast<size_t>(2 * G) * D * sizeof(float) +
                      (static_cast<size_t>(batch) + 1) * sizeof(int) + 1024;
  const int kind = std::is_same<T, __half>::value ? 1 : 2;
  const CUtensorMap tmk = tc::make_operand_map(kc, batch * Hkv * max_len, D, 2, kind, kTile);
  const CUtensorMap tmv = tc::make_operand_map(vc, batch * Hkv * max_len, D, 2, kind, kTile);
  allow_dynamic_smem(kernel, 112 * 1024);
  static int occupancy = 0;                       // CTAs per SM: the grid must be fully co-resident (flag waits); the same on
  if (occupancy == 0) {                           // every device of a box
    int occ = 0;
    CT2_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kThreads, 112 * 1024));
    occupancy = std::max(1, std::min(occ, 2));
  }
  const int64_t max_units = batch * Hkv * ((max_len + kTile - 1) / kTile);
  const int64_t ctas = std::max<int64_t>(1, std::min<int64_t>(static_cast<int64_t>(occupancy) * sm_count, max_units));
  launch_pdl(kernel, dim3(static_cast<unsigned>(ctas)), dim3(kThreads), smem, st, tmk, tmv, static_cast<const T*>(qkv),
             static_cast<T*>(kc), static_cast<T*>(vc), sn, cs, lens, static_cast<int>(batch), H, Hkv, max_len, interleave,
             scale * 1.4426950408889634f, static_cast<T*>(out), partials, tickets);
  check_launch();
}

template <typename T, int D>
bool launch_persistent_g(const void* qkv, void* kc, void* vc, const float* sn, const float* cs, const int32_t* lens,
                         int64_t batch, int H, int Hkv, int64_t max_len, bool interleave, float scale, void* out,
                         float* partials, int32_t* tickets, int sm_count, cudaStream_t st) {
  switch (H / Hkv) {
    case 1: launch_persistent<T, D, 1>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, sm_count, st); return true;
    case 2: launch_persistent<T, D, 2>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, sm_count, st); return true;
    case 4: launch_persistent<T, D, 4>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, sm_count, st); return true;
    case 8: launch_persistent<T, D, 8>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, sm_count, st); return true;
    default: return false;
  }
}

}  // namespace

// fp16 / bf16, head_dim 64 or 128, G = H / Hkv in {1, 2, 4, 8}, batch <= 1024.  The workspace must hold kSlots (64)
// partial slots per (row, head) behind the 16 of the split-KV kernel: attention_decode_workspace_bytes(batch, H, D, 80).  false = shape not covered.
bool launch_attention_decode_persistent(const void* qkv, void* kc, void* vc, const float* sn, const float* cs,
                                        const int32_t* lens, int64_t batch, int H, int Hkv, int D, int64_t max_len,
                                        bool interleave, float scale, void* out, float* partials, int32_t* tickets,
                                        int slots, int dtype, cudaStream_t st) {
  // Policy (measured in the decode graph of Llama-3-8B, tools/ablate.py): while all (row, KV head) pairs fit in ONE wave
  // of the split-KV grid (attention_mma.cu) that kernel is 2-6 % faster per step (no prefix table, no cursor); beyond one
  // wave its second, partial wave costs up to 40 %, and the work-balanced persistent kernel wins.
  // CT2B200_ATTN_DECODE = persistent | split | simt pins the choice.
  // (read on every call: the tests pin each kernel in turn).  The two kernels never share partial records: the split-KV
  // kernel owns the first 16 slots' worth of the partial area, this one the next 64.
  int mode = 0;
  if (const char* e = std::getenv("CT2B200_ATTN_DECODE")) {
    const std::string v(e);
    mode = v == "persistent" ? 1 : (v == "split" || v == "simt") ? 2 : 0;
  }
  if (mode == 2 || dtype == CT2B200_F32 || (D != 128 && D != 64) || batch > kMaxBatch || slots < kSlots + 16) return false;
  partials += static_cast<size_t>(batch) * H * 16 * (static_cast<size_t>(D) + 2);
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  static int cached_dev = -1, cached_sms = 132;
  if (cached_dev != dev) {
    cudaDeviceGetAttribute(&cached_sms, cudaDevAttrMultiProcessorCount, dev);
    cached_dev = dev;
  }
  sms = cached_sms;
  if (mode == 0 && batch * Hkv <= 2 * static_cast<int64_t>(sms)) return false;
  if (dtype == CT2B200_F16) {
    return D == 128 ? launch_persistent_g<__half, 128>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, sms, st)
                    : launch_persistent_g<__half, 64>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, sms, st);
  }
  return D == 128 ? launch_persistent_g<__nv_bfloat16, 128>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, sms, st)
                  : launch_persistent_g<__nv_bfloat16, 64>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, sms, st);
}

}  // namespace ct2b200
