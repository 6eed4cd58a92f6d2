// awq.cu — AWQ-INT4 (SURVEY §8 a7): ops::GemmAwq / GemvAwq / DequantizeAwq re-designed for sm_90a.
//
// Reference: src/ops/awq/gemm_gpu.cu (mma.sync m16n8k16 + split-K=8 fp16 planes + ops::Sum),
// gemv_gpu.cu (one warp per output channel, fp32 FMA), dequantize_gpu.cu (+ cuBLAS when M >= 1024),
// dispatch in src/layers/common.cc:402-438.  Both reference layouts are accepted and repacked ONCE at load
// into a K-major "native" layout (SURVEY §7 step 5):
//   wp  int32 [N, K/8]  — word w of row n holds input channels 8w..8w+7; channel 8w+i sits in nibble
//                          kOrder[i] = {0,4,1,5,2,6,3,7}, so (w & 0x000f000f) / (w & 0x00f000f0) of w and w>>8
//                          yield the half2 pairs (k0,k1) (k2,k3) (k4,k5) (k6,k7) directly;
//   sc  f16   [N, K/G]  — group scales;   zr  f16 [N, K/G] — group zero points (0..15) as fp16.
// Decode GEMM (m <= 64): weight-streaming, HBM-bound.  TMA brings the packed tile [128 rows x 32 B] and the fp16
// activation tile; four transform warps dequantize ((q - z) * s, exact subtraction then one fp16 rounding — the
// arithmetic of the reference's dequantize_s4_to_fp16x2 + sub.f16x2 + fma.rn.f16x2) straight into the
// 128B-swizzled K-major wgmma operand layout; wgmma (f16) accumulates in registers (fp32); fused
// bias/activation/residual (or SwiGLU gate*up) epilogue.  Persistent stream-K over (tile, K-block) units like
// gemm_tc.cu; tiles shared by several CTAs are reduced DETERMINISTICALLY (per-CTA partial slots summed in CTA
// order by the last arriver — no float atomics).
// Prefill (m > 64): dequantize to fp16 [N,K] scratch + the f16 wgmma GEMM (the reference does the same above
// M >= 1024 with cuBLAS).
#include <algorithm>

#include "../common.cuh"
#include "awq_common.cuh"
#include "gemm_common.cuh"
#include "kernels.h"
#include "streamk.cuh"
#include "tc_common.cuh"

namespace ct2b200 {

namespace {

using namespace tc;

__device__ __constant__ int kOrderDev[8] = {0, 4, 1, 5, 2, 6, 3, 7};

// ---------------------------------------------------------------------------------------------
// repack (load time) and dequantize (op level / prefill)
// ---------------------------------------------------------------------------------------------
// layout 1 = AWQ_GEMM: qweight [K, N/8] (column 8c+i in nibble kOrder[i]), scales [K/G, N], qzeros [K/G, N/8]
// layout 2 = AWQ_GEMV: qweight [N, K/8] (channel 8w+i in nibble i), scales [N, sw], qzeros [N, zw] (nibble g%8 of word g/8)
__device__ __forceinline__ int awq_nibble(const int32_t* qweight, int layout, int64_t n, int64_t k, int64_t N, int64_t K) {
  if (layout == 1) {
    const uint32_t w = static_cast<uint32_t>(qweight[k * (N / 8) + n / 8]);
    return (w >> (4 * kOrderDev[n % 8])) & 0xF;
  }
  const uint32_t w = static_cast<uint32_t>(qweight[n * (K / 8) + k / 8]);
  return (w >> (4 * (k % 8))) & 0xF;
}
__device__ __forceinline__ int awq_zero(const int32_t* qzeros, int layout, int64_t n, int64_t g, int64_t N, int zw) {
  if (layout == 1) {
    const uint32_t w = static_cast<uint32_t>(qzeros[g * (N / 8) + n / 8]);
    return (w >> (4 * kOrderDev[n % 8])) & 0xF;
  }
  const uint32_t w = static_cast<uint32_t>(qzeros[n * zw + g / 8]);
  return (w >> (4 * (g % 8))) & 0xF;
}
__device__ __forceinline__ __half awq_scale(const __half* scales, int layout, int64_t n, int64_t g, int64_t N, int sw) {
  return layout == 1 ? scales[g * N + n] : scales[n * sw + g];
}

__global__ void awq_repack_kernel(const int32_t* __restrict__ qweight, const __half* __restrict__ scales,
                                  const int32_t* __restrict__ qzeros, int layout, int G, int64_t N, int64_t K, int zw,
                                  int sw, int32_t* __restrict__ wp, __half* __restrict__ sc, __half* __restrict__ zr) {
  const int64_t words = N * (K / 8);
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < words;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t n = idx / (K / 8), w = idx % (K / 8);
    uint32_t out = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) out |= static_cast<uint32_t>(awq_nibble(qweight, layout, n, 8 * w + i, N, K)) << (4 * kOrderDev[i]);
    wp[idx] = static_cast<int32_t>(out);
  }
  const int64_t ng = K / G;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < N * ng;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t n = idx / ng, g = idx % ng;
    sc[idx] = awq_scale(scales, layout, n, g, N, sw);
    zr[idx] = __int2half_rn(awq_zero(qzeros, layout, n, g, N, zw));
  }
}

// ops::DequantizeAwq: reference layouts -> W [K, N] fp16 (src/ops/awq/dequantize_gpu.cu:8-62)
__global__ void awq_dequantize_ref_layout_kernel(const int32_t* __restrict__ qweight, const __half* __restrict__ scales,
                                                 const int32_t* __restrict__ qzeros, int layout, int G, int64_t N,
                                                 int64_t K, int zw, int sw, __half* __restrict__ w_out) {
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < N * K;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t k = idx / N, n = idx % N;
    const __half q = __int2half_rn(awq_nibble(qweight, layout, n, k, N, K));
    const __half z = __int2half_rn(awq_zero(qzeros, layout, n, k / G, N, zw));
    w_out[idx] = __hmul(__hsub(q, z), awq_scale(scales, layout, n, k / G, N, sw));
  }
}

// native layout -> W^T [N, K] fp16 (K-major, what gemm_f16_tc consumes) for the prefill arm
__global__ void awq_dequantize_native_kernel(const int32_t* __restrict__ wp, const __half* __restrict__ sc,
                                             const __half* __restrict__ zr, int G, int64_t N, int64_t K,
                                             __half* __restrict__ w_out) {
  const int64_t words = N * (K / 8);
  const int64_t ng = K / G;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < words;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t n = idx / (K / 8), w = idx % (K / 8);
    const int64_t g = (8 * w) / G;
    const __half z = zr[n * ng + g], s = sc[n * ng + g];
    const __half2 zb = __half2half2(__hadd(__float2half(1024.f), z));
    const __half2 zt = __half2half2(__hneg(__hadd(__float2half(64.f), z)));
    *reinterpret_cast<uint4*>(w_out + n * K + 8 * w) = awq_dequant_word(static_cast<uint32_t>(wp[idx]), zb, zt, __half2half2(s));
  }
}

// ---------------------------------------------------------------------------------------------
// decode GEMM: y[m,n] = x[m,:] . deq(W)[n,:]  (swap-AB: weights on the wgmma M side)
// ---------------------------------------------------------------------------------------------
constexpr int kAwqThreads = 288;      // warps 0-3 wgmma + epilogue, warp 4 TMA, warps 5-8 dequantize
constexpr int kDeqWarps = 4;          // one thread per weight row, 64 channels (8 packed words) per K block
constexpr int kRowGridBlocks = 1024;   // grid-stride element-wise kernels
constexpr int kBKh = 64;              // fp16 elements of K per stage (one 128-byte swizzle atom)
constexpr int kPackedTile = kTileM * kBKh / 2;      // 4096 bytes of nibbles per weight tile per stage

struct AwqParams {
  int64_t n, m, k;
  int group;
  sk::Schedule sched;
  const __half* sc[2];     // [n, k/group] scales (index 1: GLU "up" matrix)
  const __half* zr[2];
  FloatEpilogue fl;
  FloatGluEpilogue glu;
  uint32_t* slots;         // partial-tile slots of the shared tiles [ctas][2][NB * 128 * BN]
  int32_t* counters;
};

template <int BN, int NB>
struct AwqSmem {
  static constexpr int kA = NB * kTileM * kSwizzleBytes;      // dequantized fp16 weight tiles (wgmma M side)
  static constexpr int kP = NB * kPackedTile;                 // packed nibbles staged by TMA
  static constexpr int kX = BN * kSwizzleBytes;               // activations (wgmma N side)
  static constexpr int kStage = kA + kP + kX;
  static constexpr int kAcc = acc_bytes(NB * BN);             // accumulators parked for the epilogue
  static constexpr int kStages = ((200 * 1024 - kAcc) / kStage) > 8 ? 8 : ((200 * 1024 - kAcc) / kStage);
  static constexpr size_t kBytes = kAcc + static_cast<size_t>(kStages) * kStage + 1024 + 512;
};

// epilogue of one output channel over kCols batch rows; loads first, then arithmetic + stores
template <int NB, int kCols>
__device__ __forceinline__ void awq_chunk_epilogue(const AwqParams& p, const uint32_t (&acc)[NB][kCols], int64_t nrow, int64_t m0) {
  if (nrow >= p.n) return;
  const int64_t rows = min(static_cast<int64_t>(kCols), p.m - m0);
  if (rows <= 0) return;
  if constexpr (NB == 2) {
    __half* h = static_cast<__half*>(p.glu.h);
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      if (j >= rows) break;
      const float g = round_to<__half>(apply_act(round_to<__half>(__uint_as_float(acc[0][j])), p.glu.act));
      h[(m0 + j) * p.glu.ldh + nrow] = __float2half_rn(g * round_to<__half>(__uint_as_float(acc[1][j])));
    }
  } else {
    const __half* bias = static_cast<const __half*>(p.fl.bias);
    const __half* residual = static_cast<const __half*>(p.fl.residual);
    __half* y = static_cast<__half*>(p.fl.y);
    const float b = bias ? __half2float(bias[nrow]) : 0.f;
    float res[kCols];
#pragma unroll
    for (int j = 0; j < kCols; ++j) res[j] = (residual && j < rows) ? __half2float(residual[(m0 + j) * p.fl.ldy + nrow]) : 0.f;
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      if (j >= rows) break;
      float v = round_to<__half>(__uint_as_float(acc[0][j]));
      if (bias) v = round_to<__half>(v + b);
      if (p.fl.act >= 0) v = round_to<__half>(apply_act(v, p.fl.act));
      if (residual) v = v + res[j];
      y[(m0 + j) * p.fl.ldy + nrow] = __float2half_rn(v);
    }
  }
}

template <int BN, int NB>
__global__ void __launch_bounds__(kAwqThreads, 1)
    gemm_awq_tc_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                       const __grid_constant__ CUtensorMap tm_w2, const AwqParams p) {
  using S = AwqSmem<BN, NB>;
  constexpr int kStages = S::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint32_t* accs = reinterpret_cast<uint32_t*>(smem);  // [NB * BN columns][kAccPitch]
  uint8_t* ring = smem + S::kAcc;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ring + kStages * S::kStage);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* ready_bar = empty_bar + kStages;           // dequantized A tile of the stage is in place

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int64_t u_begin, u_end;
  p.sched.range(blockIdx.x, u_begin, u_end);
  if (threadIdx.x == 0)
    for (int s = 0; s < kStages; ++s) mbar_init(ready_bar + s, kDeqWarps);
  ring_init<1>(full_bar, empty_bar, kStages);

  if (warp == kProducerWarp) {
    // ===== TMA producer: packed weight tile(s) + activation tile =====
    if (elect_one()) {
      sk::Cursor wc(p.sched, u_begin), xc = wc;      // unit of the next weight / activation copy
      auto weights = [&](int s, int) {
        uint8_t* st = ring + s * S::kStage + S::kA;
        tma_load_2d(st, &tm_w, full_bar + s, wc.kb * (kBKh / 2), wc.ta * kTileM, kEvictFirst);
        if (NB == 2) tma_load_2d(st + kPackedTile, &tm_w2, full_bar + s, wc.kb * (kBKh / 2), wc.ta * kTileM, kEvictFirst);
        wc.next(p.sched);
      };
      auto acts = [&](int s, int) {
        tma_load_2d(ring + s * S::kStage + S::kA + S::kP, &tm_x, full_bar + s, xc.kb * kBKh, 0, kEvictLast);
        xc.next(p.sched);
      };
      produce(full_bar, empty_bar, kStages, S::kP + S::kX, static_cast<int>(u_begin), static_cast<int>(u_end - u_begin), weights, acts);
    }
  } else if (warp > kProducerWarp) {
    // ===== dequantize warps: packed nibbles -> fp16 (q - z) * s into the swizzled wgmma A tile =====
    const int r = threadIdx.x - (kProducerWarp + 1) * 32;   // tile row owned by this thread
    const int64_t ng = p.k / p.group;
    // group scale / zero are fetched one group ahead (they change every group/64 K blocks), so the global-load
    // latency is off the per-block critical path
    int64_t cur_g = -1;
    int cur_tile = -1;
    __half zc[NB], sc_[NB], zn[NB], sn_[NB];
    auto fetch = [&](int64_t row, int64_t g, __half (&z)[NB], __half (&sc)[NB]) {
#pragma unroll
      for (int w = 0; w < NB; ++w) {
        const bool ok = row < p.n && g < ng;
        z[w] = ok ? p.zr[w][row * ng + g] : __float2half(0.f);
        sc[w] = ok ? p.sc[w][row * ng + g] : __float2half(0.f);
      }
    };
    sk::Cursor cur(p.sched, u_begin);
    for (int it = 0; it < u_end - u_begin; ++it, cur.next(p.sched)) {
      const int tile = cur.ta, kb = cur.kb;
      const int s = it % kStages;
      const uint32_t ph = (it / kStages) & 1;
      const int64_t row = static_cast<int64_t>(tile) * kTileM + r;
      const int64_t g = (static_cast<int64_t>(kb) * kBKh) / p.group;
      if (tile != cur_tile || g != cur_g) {
        if (tile == cur_tile && g == cur_g + 1) {
#pragma unroll
          for (int w = 0; w < NB; ++w) { zc[w] = zn[w]; sc_[w] = sn_[w]; }
        } else {
          fetch(row, g, zc, sc_);
        }
        fetch(row, g + 1, zn, sn_);                     // prefetch the next group of this row
        cur_tile = tile;
        cur_g = g;
      }
      mbar_wait(full_bar + s, ph);
      uint8_t* st = ring + s * S::kStage;
#pragma unroll
      for (int wh = 0; wh < 2 * NB; ++wh) {
        const int w = wh >> 1, half = wh & 1;                 // weight, 32-channel half of the 64-channel K block
        const __half2 zb = __half2half2(__hadd(__float2half(1024.f), zc[w]));
        const __half2 zt = __half2half2(__hneg(__hadd(__float2half(64.f), zc[w])));
        const __half2 s2 = __half2half2(sc_[w]);
        const uint4 wv = *reinterpret_cast<const uint4*>(st + S::kA + w * kPackedTile + r * (kBKh / 2) + half * 16);
        const uint32_t words[4] = {wv.x, wv.y, wv.z, wv.w};
        uint8_t* arow = st + w * kTileM * kSwizzleBytes + r * kSwizzleBytes;
#pragma unroll
        for (int c = 0; c < 4; ++c) {    // 16-byte chunk cc of the row lives at chunk (cc ^ (r & 7)) under SWIZZLE_128B
          const int cc = half * 4 + c;
          *reinterpret_cast<uint4*>(arow + ((cc ^ (r & 7)) << 4)) = awq_dequant_word(words[c], zb, zt, s2);
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to wgmma
      __syncwarp();
      if (lane == 0) mbar_arrive(ready_bar + s);
    }
  } else {
    // ===== consumer warpgroup: wgmma over a segment's K blocks, then its epilogue =====
    griddep_wait();                                     // bias / residual may come from the previous kernel
    constexpr int kC = BN < 32 ? BN : 32;               // columns per chunk
    const int rloc = threadIdx.x;                       // output channel of the tile owned by this thread
    int it = 0;
    auto mma = [&](int kb0, int kb1) {
      Acc<BN> acc[NB];
#pragma unroll 1
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % kStages;
        const uint32_t ph = (it / kStages) & 1;
        mbar_wait(full_bar + s, ph);                    // activations landed
        mbar_wait(ready_bar + s, ph);                   // weights dequantized
        const uint32_t sa = smem_u32(ring + s * S::kStage);
        wgmma_fence();
#pragma unroll
        for (int w = 0; w < NB; ++w) mma_block<1, BN>(acc[w], sa + w * kTileM * kSwizzleBytes, sa + S::kA + S::kP, kb == kb0);
        wgmma_commit();
        wgmma_wait();
        if (lane == 0) mbar_arrive(empty_bar + s);
      }
      epi_bar_sync();                                   // the previous segment's rows have been read out of accs
#pragma unroll
      for (int w = 0; w < NB; ++w) acc_store<BN>(acc[w], accs + w * BN * kAccPitch);
      epi_bar_sync();
    };
    struct NoInputs {};
    auto load = [](NoInputs&, int64_t, int64_t) {};
    auto finish = [&](const NoInputs&, const uint32_t (&r)[NB][kC], int64_t a0, int64_t m0) {
      awq_chunk_epilogue<NB, kC>(p, r, a0 + rloc, m0);
    };
    sk::consume<NB, BN, kC, false, NoInputs>(p.sched, blockIdx.x, u_begin, u_end, p.m, accs, p.slots, p.counters, mma, load, finish);
  }
}

CUtensorMap make_packed_map(const void* wp, int64_t n, int64_t k) {
  // wp as bytes [n, k/2]; box = 128 rows x 32 bytes, no swizzle
  CUtensorMap m;
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(k / 2), static_cast<cuuint64_t>(n)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(k / 2)};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(kBKh / 2), static_cast<cuuint32_t>(kTileM)};
  cuuint32_t estr[2] = {1, 1};
  const CUresult r = get_tensor_map_encoder()(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(wp), dims, strides, box,
                                              estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled (awq) failed with code " + std::to_string(r));
  return m;
}

template <int BN, int NB>
void launch_awq(const void* x, const AwqNative& w, const AwqNative* w2, int64_t m, AwqParams p, cudaStream_t st) {
  using S = AwqSmem<BN, NB>;
  auto kernel = gemm_awq_tc_kernel<BN, NB>;
  allow_dynamic_smem(kernel, S::kBytes);
  const CUtensorMap tmx = make_operand_map(x, m, w.k, 2, 1, BN);
  const CUtensorMap tmw = make_packed_map(w.wp, w.n, w.k);
  const CUtensorMap tmw2 = make_packed_map(w2 ? w2->wp : w.wp, w.n, w.k);
  p.n = w.n; p.m = m; p.k = w.k; p.group = w.group;
  p.sc[0] = static_cast<const __half*>(w.sc); p.zr[0] = static_cast<const __half*>(w.zr);
  p.sc[1] = static_cast<const __half*>(w2 ? w2->sc : w.sc); p.zr[1] = static_cast<const __half*>(w2 ? w2->zr : w.zr);
  SplitKWorkspace& wsp = SplitKWorkspace::get(st);
  p.sched = sk::stream_k(div_up(w.n, kTileM), 1, div_up(w.k, kBKh), wsp.sm_count);
  CT2_REQUIRE(sk::slots_fit(p.sched, NB * kTileM * BN, wsp), "awq: scratch too small");
  p.slots = reinterpret_cast<uint32_t*>(wsp.accum2);
  p.counters = wsp.counters;
  launch_pdl(kernel, dim3(static_cast<unsigned>(p.sched.ctas)), dim3(kAwqThreads), S::kBytes, st, tmx, tmw, tmw2, p);
  check_launch();
}

}  // namespace

// ---- host API ----
void awq_repack(const int32_t* qweight, const void* scales, const int32_t* qzeros, int layout, int group, int64_t n,
                int64_t k, int32_t* wp, void* sc, void* zr, cudaStream_t st) {
  CT2_REQUIRE(layout == 1 || layout == 2, "awq: layout must be 1 (AWQ_GEMM) or 2 (AWQ_GEMV)");
  CT2_REQUIRE(group > 0 && k % group == 0 && group % kBKh == 0 && n % 8 == 0 && k % 8 == 0, "awq: unsupported shape/group size");
  const int64_t ng = k / group;
  const int zw = layout == 2 ? static_cast<int>((group == 64 ? ((ng + 7) / 8 + 1) / 2 * 2 : (ng + 7) / 8)) : 0;
  const int sw = zw * 8;
  awq_repack_kernel<<<kRowGridBlocks, 256, 0, st>>>(qweight, static_cast<const __half*>(scales), qzeros, layout, group, n, k, zw, sw,
                                             wp, static_cast<__half*>(sc), static_cast<__half*>(zr));
  check_launch();
}

void awq_dequantize_ref_layout(const int32_t* qweight, const void* scales, const int32_t* qzeros, int layout, int group,
                               int64_t n, int64_t k, void* w_out, cudaStream_t st) {
  CT2_REQUIRE(layout == 1 || layout == 2, "awq: layout must be 1 (AWQ_GEMM) or 2 (AWQ_GEMV)");
  const int64_t ng = k / group;
  const int zw = layout == 2 ? static_cast<int>((group == 64 ? ((ng + 7) / 8 + 1) / 2 * 2 : (ng + 7) / 8)) : 0;
  awq_dequantize_ref_layout_kernel<<<kRowGridBlocks, 256, 0, st>>>(qweight, static_cast<const __half*>(scales), qzeros, layout, group,
                                                            n, k, zw, zw * 8, static_cast<__half*>(w_out));
  check_launch();
}

namespace {
__global__ void awq_group_major_kernel(const __half* __restrict__ sc, const __half* __restrict__ zr, int64_t n, int64_t ng,
                                       __half2* __restrict__ sz) {
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < n * ng;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t g = idx / n, row = idx % n;
    sz[idx] = __halves2half2(sc[row * ng + g], zr[row * ng + g]);
  }
}
}  // namespace

void awq_build_group_major(const AwqNative& w, void* sz_out, cudaStream_t st) {
  awq_group_major_kernel<<<kRowGridBlocks, 256, 0, st>>>(static_cast<const __half*>(w.sc), static_cast<const __half*>(w.zr), w.n,
                                                  w.k / w.group, static_cast<__half2*>(sz_out));
  check_launch();
}

void awq_dequantize_native(const AwqNative& w, void* w_out /* f16 [n,k] */, cudaStream_t st) {
  awq_dequantize_native_kernel<<<kRowGridBlocks, 256, 0, st>>>(static_cast<const int32_t*>(w.wp), static_cast<const __half*>(w.sc),
                                                        static_cast<const __half*>(w.zr), w.group, w.n, w.k,
                                                        static_cast<__half*>(w_out));
  check_launch();
}

// y[m,n] = act(x . deq(W)^T + bias) + residual  (m <= 64: fused dequant GEMM; else dequantize + f16 GEMM via `scratch`)
void dense_awq(const void* x, const AwqNative& w, const void* bias, const void* residual, int act, int64_t m, void* y,
               void* scratch_nk_f16, cudaStream_t st) {
  if (m == 0) return;
  if (m > 64) {
    CT2_REQUIRE(scratch_nk_f16 != nullptr, "awq: prefill needs an [n,k] fp16 scratch");
    awq_dequantize_native(w, scratch_nk_f16, st);
    gemm_f16_tc(x, scratch_nk_f16, bias, residual, act, m, w.n, w.k, y, CT2B200_F16, st);
    return;
  }
  if (dense_awq_gemv(x, w, bias, residual, act, m, y, st)) return;
  if (dense_awq_decode(x, w, bias, residual, act, m, y, st)) return;
  AwqParams p{};
  p.fl = FloatEpilogue{bias, residual, y, act, w.n};
  if (m <= 16) launch_awq<16, 1>(x, w, nullptr, m, p, st);
  else if (m <= 32) launch_awq<32, 1>(x, w, nullptr, m, p, st);
  else launch_awq<64, 1>(x, w, nullptr, m, p, st);
}

// h[m,n] = act(x . deq(Wgate)^T) * (x . deq(Wup)^T)
void dense_awq_glu(const void* x, const AwqNative& wg, const AwqNative& wu, int act, int64_t m, void* h,
                   void* scratch_nk_f16, void* scratch_mn_f16, cudaStream_t st) {
  if (m == 0) return;
  if (m > 64) {
    CT2_REQUIRE(scratch_nk_f16 && scratch_mn_f16, "awq: prefill needs scratch buffers");
    awq_dequantize_native(wg, scratch_nk_f16, st);
    gemm_f16_tc(x, scratch_nk_f16, nullptr, nullptr, act, m, wg.n, wg.k, scratch_mn_f16, CT2B200_F16, st);
    awq_dequantize_native(wu, scratch_nk_f16, st);
    gemm_f16_tc(x, scratch_nk_f16, nullptr, nullptr, -1, m, wu.n, wu.k, h, CT2B200_F16, st);
    launch_mul_inplace_f16(h, scratch_mn_f16, m * wg.n, st);
    return;
  }
  if (dense_awq_glu_gemv(x, wg, wu, act, m, h, st)) return;
  if (dense_awq_glu_decode(x, wg, wu, act, m, h, st)) return;
  AwqParams p{};
  p.glu = FloatGluEpilogue{h, act, wg.n};
  if (m <= 16) launch_awq<16, 2>(x, wg, &wu, m, p, st);
  else if (m <= 32) launch_awq<32, 2>(x, wg, &wu, m, p, st);
  else launch_awq<64, 2>(x, wg, &wu, m, p, st);
}

}  // namespace ct2b200
