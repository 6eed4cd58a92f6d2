// awq_gemv.cu — AWQ-INT4 Dense for ONE activation row on the CUDA cores: the latency path of the decode step (batch 1).
//
// Replaces ops::GemvAwq (src/ops/awq/gemv_gpu.cu:289-470: one warp per output channel, fp32 FMAs, a second launch for the
// split-K sum at m > 8) + bias / activation / Mul.  At m = 1, 2 the tensor cores have nothing to amortise: the work is
// streaming 0.5 byte per weight and turning it into fp16 once.  One warp owns 4 output channels (2 gate + 2 up in the fused
// SwiGLU form); per trip and channel a lane loads 16 bytes of packed nibbles (32 input channels, one quantization group), turns them into the exact integers q - z as fp16 with the
// lop3 magic-number trick of awq_common.cuh and multiplies them with the activation rows in packed half2 math; 16 products
// accumulate in half2, then the partial sum is scaled by the group's scale and folded into fp32 accumulators
// (sum_k s (q - z) x = s sum_k (q - z) x inside a group: one multiply per 16 channels instead of one per channel; the
// reference's gemv applies s per weight in fp32, gemv_gpu.cu:331-352 — same value up to fp16 summation rounding).
// ~1.5 instructions per weight (the tensor-core kernels of awq.cu / awq_decode.cu pay a shared- or tensor-memory round trip
// per tile and a pipeline hand-over per K block instead).  No shared memory, no barriers; the activations come through L1.
//
// Native layout (ct2b200_awq_repack): wp int32 [n, k/8] (word w of row c = channels 8w .. 8w+7 in nibbles {0,4,1,5,2,6,3,7}),
// sc / zr fp16 [n, k/group].  group = 128 (what AutoAWQ writes and the reference's kernels assume), k % 128 == 0, k <= 16384;
// other shapes and m > 1 go to the tensor-core kernels (awq_decode.cu, awq.cu).
#include "awq_common.cuh"
#include "gemm_decode_common.cuh"
#include "kernels.h"

namespace ct2b200 {
namespace {

constexpr int kWarps = 8;

struct GemvWeight {
  const uint32_t* wp;
  const __half* sc;
  const __half* zr;
};

struct GemvParams {
  int64_t n, k;
  int group;
  // plain Dense epilogue (NB == 1) / SwiGLU (NB == 2)
  const __half* bias;
  const __half* residual;
  __half* y;
  int act;
};

// One warp = R output channels (of each of the NB weights).  A "trip" is 1024 input channels: a lane owns 32 of them = one
// 16-byte load of nibbles per channel and 64 bytes of the activation row, which are converted once and reused by all NB * R
// channels — with one channel per warp the activation reads through L1 (8 KB per 2 KB of nibbles at k = 4096) cost as many
// load wavefronts as the HBM stream itself.  Two trips of all channels are requested before the first is
// used (128 bytes per lane in flight).  The group scales / zeros of a row (k / 128 of each) are fetched once with coalesced
// loads — lane g holds group g + 32 c — and handed to the lane that needs them by shuffle: trip t uses group 8 t + lane / 4.
constexpr int kMaxQuads = 4;           // quads of 4 trips: k <= 16384

// KS = warps per row group: with KS = 2 the pairs of trips alternate between two adjacent warps and the partial sums meet in
// shared memory.  Small matrices need it to have enough warps in flight: out-proj (4096 x 4096) is 1024 row groups = 7 warps
// per SM, and a warp only keeps 4 KB of the stream in flight.
template <int NB, int R, int KS>
__global__ void __launch_bounds__(kWarps * 32) awq_gemv_kernel(const __half* __restrict__ x, GemvWeight w0, GemvWeight w1,
                                                               GemvParams p) {
  constexpr int NS = NB * R;           // weight rows streamed by this warp
  __shared__ float s_part[kWarps][NS];
  griddep_launch();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ks = warp % KS;
  const int64_t ch0 = ((static_cast<int64_t>(blockIdx.x) * kWarps + warp) / KS) * R;
  const bool active = ch0 < p.n;       // warp-uniform; inactive warps still reach the barrier below
  const int64_t words = p.k / 8;
  const int ng = static_cast<int>(p.k / 128);
  const int trips = static_cast<int>((p.k + 1023) / 1024);
  const uint32_t* wrow[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    const GemvWeight& w = s / R == 0 ? w0 : w1;
    wrow[s] = w.wp + min(ch0 + s % R, p.n - 1) * words;
  }
  // the weights, scales and zeros never depend on the previous kernel: requested before the dependency wait
  __half2 sz_r[NS][kMaxQuads];         // {scale, zero} of group 32 c + lane
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    const GemvWeight& w = s / R == 0 ? w0 : w1;
    const int64_t ch = min(ch0 + s % R, p.n - 1);
#pragma unroll
    for (int c = 0; c < kMaxQuads; ++c) {
      const int g = c * 32 + lane;
      sz_r[s][c] = g < ng ? __halves2half2(w.sc[ch * ng + g], w.zr[ch * ng + g]) : __float2half2_rn(0.f);
    }
  }
  float acc[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) acc[s] = 0.f;
  uint4 q[NS][2];
  auto load_pair = [&](int t0) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int64_t k0 = static_cast<int64_t>(t0 + u) * 1024 + lane * 32;
#pragma unroll
      for (int s = 0; s < NS; ++s)
        q[s][u] = k0 < p.k ? __ldcs(reinterpret_cast<const uint4*>(wrow[s] + k0 / 8)) : make_uint4(0, 0, 0, 0);
    }
  };
  if (active) load_pair(2 * ks);
  griddep_wait();                                  // the activations come from the previous kernel

#pragma unroll
  for (int c = 0; c < kMaxQuads; ++c) {
    if (c * 4 >= trips) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int t0 = c * 4 + h * 2;
      if (t0 >= trips) break;
      if (!active || (KS > 1 && ((c * 2 + h) % KS) != ks)) continue;       // the other warp of the row group owns this pair
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int64_t k0 = static_cast<int64_t>(t0 + u) * 1024 + lane * 32;
        const bool live = k0 < p.k;
        uint4 xv[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) xv[j] = live ? *(reinterpret_cast<const uint4*>(x + k0) + j) : make_uint4(0, 0, 0, 0);
        const int src = (h * 2 + u) * 8 + (lane >> 2);
#pragma unroll
        for (int s = 0; s < NS; ++s) {
          const __half2 sz = __shfl_sync(0xffffffffu, sz_r[s][c], src);
          const __half zp = __high2half(sz);
          const __half2 zb = __half2half2(__hadd(__float2half(1024.f), zp));
          const __half2 zt = __half2half2(__hneg(__hadd(__float2half(64.f), zp)));
          const float sc_f = live ? __low2float(sz) : 0.f;
          const uint32_t wq[4] = {q[s][u].x, q[s][u].y, q[s][u].z, q[s][u].w};
#pragma unroll
          for (int half_trip = 0; half_trip < 2; ++half_trip) {      // 16 channels -> one half2 partial sum
            __half2 part = __float2half2_rn(0.f);
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
              const int j = half_trip * 2 + jj;
              const uint4 d = awq_unscaled_word(wq[j], zb, zt);
              const __half2* dv = reinterpret_cast<const __half2*>(&d);
              const __half2* xh = reinterpret_cast<const __half2*>(&xv[j]);
#pragma unroll
              for (int i = 0; i < 4; ++i) part = __hfma2(dv[i], xh[i], part);
            }
            const float2 f = __half22float2(part);
            acc[s] = fmaf(f.x + f.y, sc_f, acc[s]);
          }
        }
      }
      if (t0 + 2 * KS < trips) load_pair(t0 + 2 * KS);
    }
  }
#pragma unroll
  for (int s = 0; s < NS; ++s) acc[s] = warp_sum(acc[s]);
  if constexpr (KS > 1) {
    if (lane == 0 && ks != 0)
#pragma unroll
      for (int s = 0; s < NS; ++s) s_part[warp][s] = acc[s];
    __syncthreads();
    if (ks != 0) return;
#pragma unroll
    for (int o = 1; o < KS; ++o)
#pragma unroll
      for (int s = 0; s < NS; ++s) acc[s] += s_part[warp + o][s];
  }
  if (lane == 0 && active) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int64_t ch = ch0 + r;
      if (ch >= p.n) break;
      if constexpr (NB == 1) {
        FloatEpilogue e{p.bias, p.residual, p.y, p.act, p.n};
        float_epilogue_store<__half>(e, acc[r], 0, ch);
      } else {
        FloatGluEpilogue e{p.y, p.act, p.n};
        float_glu_epilogue_store<__half>(e, acc[r], acc[R + r], 0, ch);
      }
    }
  }
}

template <int NB>
void launch_gemv(const void* x, const AwqNative& a, const AwqNative* b, const GemvParams& p, cudaStream_t st) {
  constexpr int R = NB == 1 ? 4 : 2;
  const GemvWeight w0{static_cast<const uint32_t*>(a.wp), static_cast<const __half*>(a.sc), static_cast<const __half*>(a.zr)};
  const GemvWeight w1 = b ? GemvWeight{static_cast<const uint32_t*>(b->wp), static_cast<const __half*>(b->sc),
                                       static_cast<const __half*>(b->zr)} : w0;
  const int64_t groups = (a.n + R - 1) / R;        // row groups = warps at KS = 1
  const int force_ks = dec::env_int("CT2B200_AWQ_GEMV_KS", 0);
  const bool split = force_ks ? force_ks == 2 : (groups < 2 * static_cast<int64_t>(sm_count_of_current_device()) * kWarps && a.k >= 4096);
  const dim3 block(kWarps * 32);
  if (split) {
    const dim3 grid(static_cast<unsigned>((groups * 2 + kWarps - 1) / kWarps));
    launch_pdl(awq_gemv_kernel<NB, R, 2>, grid, block, 0, st, static_cast<const __half*>(x), w0, w1, p);
  } else {
    const dim3 grid(static_cast<unsigned>((groups + kWarps - 1) / kWarps));
    launch_pdl(awq_gemv_kernel<NB, R, 1>, grid, block, 0, st, static_cast<const __half*>(x), w0, w1, p);
  }
  check_launch();
}

bool covered(const AwqNative& w, int64_t m, const void* x) {
  return m == 1 && w.group == 128 && w.k % 128 == 0 && w.k <= 4096 * kMaxQuads &&
         (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w.wp) & 15) == 0;
}

// CT2B200_AWQ_GEMV: 1 = use this kernel for m == 1
bool enabled() { return dec::env_int("CT2B200_AWQ_GEMV", CT2B200_DEFAULT_AWQ_GEMV) != 0; }

}  // namespace

bool dense_awq_gemv(const void* x, const AwqNative& w, const void* bias, const void* residual, int act, int64_t m, void* y,
                    cudaStream_t st) {
  if (!enabled() || !covered(w, m, x)) return false;
  GemvParams p{w.n, w.k, w.group, static_cast<const __half*>(bias), static_cast<const __half*>(residual), static_cast<__half*>(y), act};
  launch_gemv<1>(x, w, nullptr, p, st);
  return true;
}

bool dense_awq_glu_gemv(const void* x, const AwqNative& wg, const AwqNative& wu, int act, int64_t m, void* h, cudaStream_t st) {
  if (!enabled() || !covered(wg, m, x) || !covered(wu, m, x) || wg.n != wu.n || wg.k != wu.k || wg.group != wu.group) return false;
  GemvParams p{wg.n, wg.k, wg.group, nullptr, nullptr, static_cast<__half*>(h), act};
  launch_gemv<2>(x, wg, &wu, p, st);
  return true;
}

}  // namespace ct2b200
