// gemm_prefill.cu — compute-bound GEMM of the prompt pass (many activation rows) on wgmma, with the whole
// Dense epilogue fused: y[m, n] = epilogue(x[m, k] * W[n, k]^T).
//
// Replaces ops::Gemm (cuBLAS) + ops::Dequantize::dequantize_gemm_output + bias/activation + ops::Add / ops::Mul
// (reference src/layers/common.cc:353-401, 440; src/ops/gemm.cc:45-107; src/ops/dequantize_gpu.cu:30-144;
// FeedForwardNetwork gate/up, src/layers/transformer.cc:21-51) for m > 64.
//
// Shape of the problem: tensor-core bound.  One persistent CTA per SM walks 128 x 256 output tiles (GLU: 128 rows x
// 128 gate + 128 up columns), M fastest so that the CTAs running at the same time share one weight tile in L2.
//   warp 8      TMA producer: 3-stage ring of (A 128 x 128 B, B 256 x 128 B) operand slabs, SWIZZLE_128B; it runs ahead
//               into the next tile while the consumers finish the current one
//   warps 0-7   two consumer warpgroups; warpgroup h owns one half of the tile's output columns: per 32 bytes of K two m64
//               wgmma row halves x its 64-column pieces (128 accumulator registers per thread), each K block waited for
//               before the stage is handed back.  Then its epilogue: 32 accumulator columns at a time go through a
//               [column][row] shared-memory buffer of the warpgroup to one output row per thread, 16-byte loads / stores
//               of the residual and the result.  The epilogue of a tile does not overlap the MMAs of the next.
// Rounding points: DenseEpilogue / GluEpilogue / FloatEpilogue (common.cuh, gemm_common.cuh).
#include <algorithm>
#include <cstdlib>

#include "gemm_common.cuh"
#include "kernels.h"
#include "tc_common.cuh"

namespace ct2b200 {
namespace {

using namespace tc;

constexpr int kThreads = 288;          // two consumer warpgroups (wgmma + epilogue of one half of the columns each), TMA warp
constexpr int kTmaWarp = 8;
constexpr int kBN = 256;               // accumulator columns per tile (NB = 2: 128 gate + 128 up)
constexpr int kStages = 3;
constexpr int kStageA = kTileM * kSwizzleBytes;      // 16 KB
constexpr int kStageB = kBN * kSwizzleBytes;         // 32 KB
constexpr int kStage = kStageA + kStageB;
constexpr int kCtrl = 256;                           // barriers
constexpr int kScaleBytes = 2 * kBN * 4 * 2;         // [buf][256] weight scales + [buf][256] bias (fp32)
constexpr int kChunk = 32;                           // accumulator columns handed to the row-per-thread epilogue at a time
constexpr int kAccWg = acc_bytes(2 * kChunk);        // per warpgroup: one chunk of each of up to two weights
constexpr size_t kSmemBytes = static_cast<size_t>(kStages) * kStage + 2 * kAccWg + kCtrl + kScaleBytes + 1024;

// columns [C0, C0 + kChunk) of a warpgroup's accumulators -> dst[column][kAccPitch] (see acc_store)
template <int C0, int BNH>
__device__ __forceinline__ void store_chunk(const Acc<BNH>& c, uint32_t* dst) {
  const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < kChunk / 8; ++j) {
      uint32_t* q = dst + (j * 8 + (l & 3) * 2) * kAccPitch + h * 64 + w * 16 + (l >> 2);
      const uint32_t* d = c.d[h][C0 / 64] + 4 * ((C0 % 64) / 8 + j);
      q[0] = d[0];
      q[kAccPitch] = d[1];
      q[8] = d[2];
      q[kAccPitch + 8] = d[3];
    }
}

struct PreParams {
  int64_t m, n;          // output rows / channels (NB = 2: n = channels of ONE of the two weights)
  int kb_total;          // K blocks of 128 bytes
  int tiles_m, tiles_n;
  const float* a_scale;      // [m]
  const float* w_scale0;     // [n]
  const float* w_scale1;     // [n] (GLU up)
  const void* bias;          // [n] T or null
  const void* residual;      // [m, n] T or null
  void* y;
  int act;
  int64_t ldy;
};

__device__ __forceinline__ void epi_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void wg_sync(int half) { asm volatile("bar.sync %0, 128;" ::"r"(2 + half) : "memory"); }

// T = output dtype (2 or 4 bytes), KIND = 0 s8 / 1 f16 / 2 bf16, NB = 2: gate/up fusion, BN = accumulator columns per tile:
// 256, or 64 for Dense layers whose 128 x 256 tiles would occupy a handful of SMs (Transformer-base at 256 rows: 4 tiles; the
// shared-memory stage layout stays that of the wide tile, a narrow tile simply uses the first 64 rows of the B slot)
template <typename T, int KIND, int NB, int BN = kBN>
__global__ void __launch_bounds__(kThreads, 1)
    gemm_prefill_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                        const __grid_constant__ CUtensorMap tm_w2, const PreParams p) {
  constexpr int kElem = Elem<KIND>::bytes;
  constexpr int BK = kSwizzleBytes / kElem;
  static_assert(NB == 1 || BN == kBN, "narrow tiles are for the plain Dense");
  constexpr int kWRows = NB == 2 ? BN / 2 : BN;        // weight rows per TMA box
  constexpr int kOutCols = NB == 2 ? BN / 2 : BN;      // output columns per tile

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* accs = smem + kStages * kStage;                     // [warpgroup][2 * kChunk columns][kAccPitch]
  uint8_t* ctrl = accs + 2 * kAccWg;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ctrl);     // [kStages]
  uint64_t* empty_bar = full_bar + kStages;                    // [kStages]
  float* s_scale = reinterpret_cast<float*>(ctrl + kCtrl);     // [2][256]
  float* s_bias = s_scale + 2 * kBN;                           // [2][256]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.tiles_m * p.tiles_n;
  const int KB = p.kb_total;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar + s, 1);
      mbar_init(empty_bar + s, 8);                 // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  griddep_launch();

  if (warp == kTmaWarp) {
    // ===== TMA producer =====
    if (elect_one()) {
      griddep_wait();                              // the activations come from the previous kernel
      int it = 0;
#pragma unroll 1
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile % p.tiles_m) * kTileM;
        const int n0 = (tile / p.tiles_m) * kOutCols;
#pragma unroll 1
        for (int kb = 0; kb < KB; ++kb, ++it) {
          const int s = it % kStages;
          if (it >= kStages) mbar_wait(empty_bar + s, ((it / kStages) & 1) ^ 1);
          uint8_t* sa = smem + s * kStage;
          uint8_t* sb = sa + kStageA;
          mbar_expect_tx(full_bar + s, kStageA + BN * kSwizzleBytes);
          tma_load_2d(sa, &tm_x, full_bar + s, kb * BK, m0, kEvictLast);
          tma_load_2d(sb, &tm_w, full_bar + s, kb * BK, n0, kEvictFirst);
          if (NB == 2) tma_load_2d(sb + kWRows * kSwizzleBytes, &tm_w2, full_bar + s, kb * BK, n0, kEvictFirst);
        }
      }
    }
  } else {
    // ===== consumer warpgroups: wgmma over the K blocks of a tile, then its epilogue =====
    griddep_wait();
    const int q = warp & 3;
    const int half = warp >> 2;                    // which half of the output columns this warpgroup computes
    const int et = threadIdx.x;                    // 0..255
    uint32_t* my_acc = reinterpret_cast<uint32_t*>(accs + half * kAccWg);
    constexpr int kAccN = NB == 2 ? kOutCols / 2 : BN / 2;     // accumulator columns per weight and warpgroup
    int it = 0;
    const int rloc = q * 32 + lane;
    constexpr int kColsPerWarp = kOutCols / 2;     // 128 (NB = 1) or 64 (NB = 2)
    constexpr int kVec = 16 / sizeof(T);           // elements per 16-byte access
    const T* bias = static_cast<const T*>(p.bias);
    int seq = 0;
#pragma unroll 1
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++seq) {
      const int buf = seq & 1;
      const int m0 = (tile % p.tiles_m) * kTileM;
      const int n0 = (tile / p.tiles_m) * kOutCols;
      const int64_t row = static_cast<int64_t>(m0) + rloc;
      const bool row_ok = row < p.m;
      // per-tile column constants -> shared memory (weight scales, bias), one value per epilogue thread
      float* ws = s_scale + buf * kBN;
      float* bs = s_bias + buf * kBN;
      {
        float sv = 1.f, bv = 0.f;
        if constexpr (NB == 2) {
          const int c = et & (kOutCols - 1);
          const int64_t col = static_cast<int64_t>(n0) + c;
          if constexpr (KIND == 0) sv = col < p.n ? __ldg((et < kOutCols ? p.w_scale0 : p.w_scale1) + col) : 1.f;
        } else {
          const int64_t col = static_cast<int64_t>(n0) + et;
          const bool mine = et < kOutCols && col < p.n;
          if constexpr (KIND == 0) sv = mine ? __ldg(p.w_scale0 + col) : 1.f;
          if (bias) bv = mine ? to_f32(bias[col]) : 0.f;
        }
        ws[et] = sv;
        bs[et] = bv;
      }
      float sa = 1.f;
      if constexpr (KIND == 0) sa = row_ok ? p.a_scale[row] : 1.f;      // written by the previous kernel: not through the read-only path (build.py)
      Acc<kAccN> acc[NB];
#pragma unroll 1
      for (int kb = 0; kb < KB; ++kb, ++it) {
        const int s = it % kStages;
        mbar_wait(full_bar + s, (it / kStages) & 1);
        const uint32_t sa = smem_u32(smem + s * kStage);
        const uint32_t sb = sa + kStageA + half * kAccN * kSwizzleBytes;
        wgmma_fence();
#pragma unroll
        for (int w = 0; w < NB; ++w) mma_block<KIND, kAccN>(acc[w], sa, sb + w * kWRows * kSwizzleBytes, kb == 0);
        wgmma_commit();
        wgmma_wait();
        if (lane == 0) mbar_arrive(empty_bar + s);  // this warp's share of the stage has been read
      }
      epi_sync();                                  // column constants of this tile are in place
      T* yrow = static_cast<T*>(p.y) + row * p.ldy + n0;
      const T* rrow = p.residual ? static_cast<const T*>(p.residual) + row * p.ldy + n0 : nullptr;
#pragma unroll
      for (int cc = 0; cc < kColsPerWarp; cc += kChunk) {
        const int c0 = half * kColsPerWarp + cc;
        // this chunk of the fragments -> shared memory -> one row per thread
        wg_sync(half);
#pragma unroll
        for (int w = 0; w < NB; ++w) {
          if (cc == 0) store_chunk<0>(acc[w], my_acc + w * kChunk * kAccPitch);
          if (cc == 32) store_chunk<32 % kAccN>(acc[w], my_acc + w * kChunk * kAccPitch);
          if (cc == 64) store_chunk<64 % kAccN>(acc[w], my_acc + w * kChunk * kAccPitch);
          if (cc == 96) store_chunk<96 % kAccN>(acc[w], my_acc + w * kChunk * kAccPitch);
        }
        wg_sync(half);
        // The residual of the whole 32-column chunk is requested before the accumulators are read.  y may alias the residual
        // (in-place x += Dense(...)), so loads left between the stores below stay in program order: one L2 round trip per
        // 16-byte vector, 16 per thread and tile.
        Vec16<T> res[32 / kVec];
        if constexpr (NB == 1) {
          if (rrow && row_ok) {
#pragma unroll
            for (int v = 0; v < 32 / kVec; ++v)
              if (n0 + c0 + v * kVec < p.n) res[v] = ld16(rrow + c0 + v * kVec);
          }
        }
        uint32_t r0[32];
        acc_load<32>(my_acc, rloc, r0);
        if constexpr (NB == 2) {
          uint32_t r1[32];
          acc_load<32>(my_acc + kChunk * kAccPitch, rloc, r1);
          if (row_ok) {
#pragma unroll
            for (int v0 = 0; v0 < 32; v0 += kVec) {
              if (n0 + c0 + v0 >= p.n) break;
              Vec16<T> o;
#pragma unroll
              for (int i = 0; i < kVec; ++i) {
                const int c = c0 + v0 + i;
                float gate, up;
                if constexpr (KIND == 0) {
                  gate = __fdividef(static_cast<float>(static_cast<int32_t>(r0[v0 + i])), sa * ws[c]);
                  up = __fdividef(static_cast<float>(static_cast<int32_t>(r1[v0 + i])), sa * ws[kOutCols + c]);
                } else {
                  gate = __uint_as_float(r0[v0 + i]);
                  up = __uint_as_float(r1[v0 + i]);
                }
                gate = round_to<T>(act_call(round_to<T>(gate), p.act));
                o.v[i] = from_f32<T>(gate * round_to<T>(up));
              }
              st16(yrow + c0 + v0, o);
            }
          }
        } else {
          if (row_ok) {
#pragma unroll
            for (int v0 = 0; v0 < 32; v0 += kVec) {
              if (n0 + c0 + v0 >= p.n) break;
              Vec16<T> o;
#pragma unroll
              for (int i = 0; i < kVec; ++i) {
                const int c = c0 + v0 + i;
                float v;
                if constexpr (KIND == 0) v = __fdividef(static_cast<float>(static_cast<int32_t>(r0[v0 + i])), sa * ws[c]);
                else v = __uint_as_float(r0[v0 + i]);
                v = round_to<T>(round_to<T>(v) + bs[c]);
                if (p.act >= 0) v = round_to<T>(act_call(v, p.act));
                if (rrow) v = v + to_f32(res[v0 / kVec].v[i]);
                o.v[i] = from_f32<T>(v);
              }
              st16(yrow + c0 + v0, o);
            }
          }
        }
      }
    }
  }
}

template <typename T, int KIND, int NB, int BN>
void launch_prefill_bn(const void* x, const void* w, const void* w2, int64_t m, int64_t n, int64_t k, PreParams p, int sms,
                       cudaStream_t st) {
  constexpr int elem = Elem<KIND>::bytes;
  auto kernel = gemm_prefill_kernel<T, KIND, NB, BN>;
  allow_dynamic_smem(kernel, kSmemBytes);
  constexpr int out_cols = NB == 2 ? BN / 2 : BN;
  p.m = m;
  p.n = n;
  p.kb_total = div_up(k, kSwizzleBytes / elem);
  p.tiles_m = div_up(m, kTileM);
  p.tiles_n = div_up(n, out_cols);
  const CUtensorMap tmx = make_operand_map(x, m, k, elem, KIND, kTileM);
  const CUtensorMap tmw = make_operand_map(w, n, k, elem, KIND, out_cols);
  const CUtensorMap tmw2 = make_operand_map(w2 ? w2 : w, n, k, elem, KIND, out_cols);
  const int64_t tiles = static_cast<int64_t>(p.tiles_m) * p.tiles_n;
  const unsigned grid = static_cast<unsigned>(std::min<int64_t>(sms, tiles));
  launch_pdl(kernel, dim3(grid), dim3(kThreads), kSmemBytes, st, tmx, tmw, tmw2, p);
  check_launch();
}

template <typename T, int KIND, int NB>
void launch_prefill(const void* x, const void* w, const void* w2, int64_t m, int64_t n, int64_t k, const PreParams& p,
                    cudaStream_t st) {
  const int sms = sm_count_of_current_device();
  if constexpr (NB == 1) {
    // latency-bound regime: the wide tiles would run on fewer than a quarter of the SMs -> 64-column tiles (CT2B200_GEMM_PREFILL_BN pins)
    static const int force_bn = [] { const char* e = std::getenv("CT2B200_GEMM_PREFILL_BN"); return e ? std::atoi(e) : 0; }();
    const int64_t wide_tiles = static_cast<int64_t>(div_up(m, kTileM)) * div_up(n, kBN);
    if (force_bn == 64 || (force_bn == 0 && wide_tiles * 4 <= sms)) {
      launch_prefill_bn<T, KIND, NB, 64>(x, w, w2, m, n, k, p, sms, st);
      return;
    }
  }
  launch_prefill_bn<T, KIND, NB, kBN>(x, w, w2, m, n, k, p, sms, st);
}

bool prefill_kernel_enabled() {
  static const bool on = [] { const char* e = std::getenv("CT2B200_GEMM_PREFILL"); return !e || std::atoi(e) != 0; }();
  return on;
}

// 16-byte stores of y / loads of the residual need n (and the pointers) aligned to 16 bytes
bool aligned_for(const void* y, const void* residual, int64_t ldy, size_t elem) {
  return (ldy * elem) % 16 == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0 && (reinterpret_cast<uintptr_t>(residual) & 15) == 0;
}

}  // namespace

// false = shape not covered (m <= 64, raw int32 output, unaligned rows): the caller uses another kernel
bool gemm_s8_prefill(const int8_t* A, const int8_t* B, int64_t M, int64_t N, int64_t K, const DenseEpilogue& e, int dtype,
                     cudaStream_t st) {
  if (!prefill_kernel_enabled() || M <= 64 || e.a_scale == nullptr || K % 16 != 0 ||
      !aligned_for(e.y, e.residual, e.ldy, dtype_size(dtype)))
    return false;
  PreParams p{};
  p.a_scale = e.a_scale;
  p.w_scale0 = e.b_scale;
  p.bias = e.bias;
  p.residual = e.residual;
  p.y = e.y;
  p.act = e.act;
  p.ldy = e.ldy;
  CT2_DISPATCH_DTYPE(dtype, (launch_prefill<T, 0, 1>(A, B, nullptr, M, N, K, p, st)));
  return true;
}

bool gemm_s8_glu_prefill(const int8_t* A, const int8_t* Bgate, const int8_t* Bup, int64_t M, int64_t N, int64_t K,
                         const GluEpilogue& g, int dtype, cudaStream_t st) {
  if (!prefill_kernel_enabled() || M <= 64 || K % 16 != 0 || !aligned_for(g.h, nullptr, g.ldh, dtype_size(dtype))) return false;
  PreParams p{};
  p.a_scale = g.a_scale;
  p.w_scale0 = g.gate_scale;
  p.w_scale1 = g.up_scale;
  p.y = g.h;
  p.act = g.act;
  p.ldy = g.ldh;
  CT2_DISPATCH_DTYPE(dtype, (launch_prefill<T, 0, 2>(A, Bgate, Bup, M, N, K, p, st)));
  return true;
}

bool gemm_f16_prefill(const void* A, const void* B, const void* bias, const void* residual, int act, int64_t M, int64_t N,
                      int64_t K, void* C, int dtype, cudaStream_t st) {
  if (!prefill_kernel_enabled() || M <= 64 || K % 8 != 0 || !aligned_for(C, residual, N, 2)) return false;
  PreParams p{};
  p.bias = bias;
  p.residual = residual;
  p.y = C;
  p.act = act;
  p.ldy = N;
  if (dtype == CT2B200_F16) launch_prefill<__half, 1, 1>(A, B, nullptr, M, N, K, p, st);
  else if (dtype == CT2B200_BF16) launch_prefill<__nv_bfloat16, 2, 1>(A, B, nullptr, M, N, K, p, st);
  else return false;
  return true;
}

}  // namespace ct2b200
