// awq_decode.cu — AWQ-INT4 weight-streaming GEMM of the decode step (m <= 64) on wgmma, A operand in REGISTERS.
//
// Replaces ops::GemmAwq / ops::GemvAwq (+ ops::Sum over split-K planes, + bias / activation / Mul) of the reference
// (src/ops/awq/gemm_gpu.cu, gemv_gpu.cu; dispatch src/layers/common.cc:402-438) by one kernel per Dense.
//
// Same plan as gemm_decode.cu (one tile per CTA, "swap AB": 128 output channels = the wgmma M side, activations = N side;
// DSMEM split-K cluster chosen so that tiles x CS fills the SMs in one wave; weights prefetched before griddepcontrol.wait),
// plus what 4-bit weights need:
//   * the only bytes that come from HBM are the packed nibbles.  A ring slot holds a SUPER-BLOCK of four K blocks (256 input
//     channels): per weight one TMA box of 128 rows x 128 bytes (SWIZZLE_128B, so that the rows a warp reads land in
//     different banks), the {scale, zero} pairs of its groups (512 B each, cp.async.bulk from the group-major array) and the
//     four activation atoms, so the consumer warps never touch global memory.  TMA works row by row: one wide box per
//     super-block needs a quarter of the row requests of one box per 64-channel block.
//   * the dequantized fp16 operand never goes back to shared memory: wgmma takes its A operand from registers.  The thread
//     that holds rows g, g + 8 and the channel pairs 2t, 2t + 1 (+ 8) of the m64k16 A fragment converts exactly those pairs
//     ((q - z) * s: exact subtraction, one fp16 rounding — the arithmetic of the reference's dequantize_s4_to_fp16x2 +
//     sub.f16x2 + fma.rn.f16x2): in the native word layout the pair (k 2t, k 2t + 1) of a word is one lop3 away.
//   * wgmma f16 with A from registers, B (activations) from 128B-swizzled smem, fp32 accumulators in registers;
//     epilogue = gemm_decode_common.cuh (float arm).
#include "awq_common.cuh"
#include "gemm_decode_common.cuh"
#include "kernels.h"

namespace ct2b200 {
namespace {

using namespace tc;
using namespace dec;

constexpr int kThreads = kTcThreads;   // warps 0-3 convert + wgmma + epilogue, warp 4 TMA
constexpr int kBKh = 64;               // fp16 channels per K block (one 128-byte swizzle atom of the activation operand)
constexpr int kSub = 4;                         // K blocks per ring slot
constexpr int kSlotK = kSub * kBKh;             // 256 input channels per slot
constexpr int kPacked = kTileM * kSlotK / 2;    // 16 KB of nibbles per weight per slot (128 rows x 128 B, SWIZZLE_128B)
constexpr int kPairBytes = 512;                 // the 128 {scale, zero} pairs of one group of a weight
constexpr int kPairs = kSub * kPairBytes;       // up to 4 groups per slot (group 64); 2 KB keeps what follows 1024-byte aligned
constexpr int kMaxP = 8;

struct AwqDecParams {
  DecParams d;                   // d.stages = depth of the packed / pairs / activation ring
  int group;
  int sb_total;                  // super-blocks (256 channels) along K
  const __half2* sz[2];          // {scale, zero} [k/group, n] (group-major): 512 contiguous bytes per tile and group
};

template <int BN, int NB>
struct AwqDecSmem {
  static constexpr int kAct = BN * kSwizzleBytes;                           // one activation atom (64 channels)
  static constexpr int kP = NB * (kPacked + kPairs) + kSub * kAct;          // one ring slot: nibbles | pairs | 4 activation atoms
  static constexpr int kCtrl = 1024;
  static constexpr int kAcc = acc_bytes(NB * BN);                           // accumulators parked for the row-per-thread epilogue
  static size_t bytes(int p_stages, int cs) {
    return kAcc + static_cast<size_t>(p_stages) * kP + kCtrl + red_bytes(cs, NB, BN) + 1024;
  }
};

// channels (2t, 2t + 1) of a native word: pair t is the bottom (t even) or top (t odd) nibble pair of w >> (t >= 2 ? 8 : 0);
// mask / mul / add select the arm of awq_dequant_word (bottom: h - (1024 + z); top: h / 16 - (64 + z)), then one rounding by s
__device__ __forceinline__ uint32_t awq_dequant_pair(uint32_t w, uint32_t shift, uint32_t mask, __half2 mul, __half2 add, __half2 s2) {
  constexpr uint32_t kLut = (0xf0 & 0xcc) | 0xaa, kMagic = 0x64006400;
  uint32_t h;
  asm volatile("lop3.b32 %0, %1, %2, %3, %4;" : "=r"(h) : "r"(w >> shift), "r"(mask), "n"(kMagic), "n"(kLut));
  const __half2 v = __hmul2(__hfma2(*reinterpret_cast<__half2*>(&h), mul, add), s2);
  return *reinterpret_cast<const uint32_t*>(&v);
}
// global -> shared bulk copy (bytes % 16 == 0, both addresses 16-byte aligned), completion on an mbarrier
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

template <int BN, int NB, int CS>
__global__ void __launch_bounds__(kThreads, 1)
    awq_decode_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                      const __grid_constant__ CUtensorMap tm_w2, const AwqDecParams ap) {
  using S = AwqDecSmem<BN, NB>;
  const DecParams& p = ap.d;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint32_t* accs = reinterpret_cast<uint32_t*>(smem);             // [NB * BN columns][kAccPitch]
  uint8_t* p_ring = smem + S::kAcc;                               // [p_stages][nibbles NB x 16 KB | pairs NB x 2 KB | x 4 x BN x 128 B]
  const int PD = p.stages;
  uint8_t* ctrl = p_ring + static_cast<size_t>(PD) * S::kP;
  uint64_t* p_full = reinterpret_cast<uint64_t*>(ctrl);           // [kMaxP] TMA landed
  uint64_t* p_free = p_full + kMaxP;                              // [kMaxP] the consumer warps are done with the slot
  uint32_t* red = reinterpret_cast<uint32_t*>(ctrl + S::kCtrl);   // split-K exchange buffer (CS > 1)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x / CS;
  const int crank = CS > 1 ? static_cast<int>(blockIdx.x % CS) : 0;
  const int sb_lo = crank * ap.sb_total / CS, sb_hi = (crank + 1) * ap.sb_total / CS;
  const int nsb = sb_hi - sb_lo;                                   // super-blocks of this CTA
  const int a0 = tile * p.tile_rows;
  const int ngs = max(1, kSlotK / ap.group);                       // distinct groups inside a super-block (group >= 64)

  ring_init<CS>(p_full, p_free, PD);

  if (warp == kProducerWarp) {
    // ===== TMA producer: packed nibbles, {scale, zero} pairs (both weights are constants: issued before the grid
    // dependency resolves) and the activation block =====
    if (elect_one()) {
      const int rows_here = static_cast<int>(min(static_cast<int64_t>(p.tile_rows), p.n - a0));
      const uint32_t pair_bytes = static_cast<uint32_t>(rows_here) * 4u;
      const uint32_t tx = static_cast<uint32_t>(NB * p.tile_rows * (kSlotK / 2)) + NB * ngs * pair_bytes + kSub * S::kAct;
      auto weights = [&](int s, int sb) {
        uint8_t* st = p_ring + static_cast<size_t>(s) * S::kP;
        const int64_t g0 = (static_cast<int64_t>(sb) * kSlotK) / ap.group;
        tma_load_2d(st, &tm_w, p_full + s, sb * (kSlotK / 2), a0, kEvictFirst);
        if (NB == 2) tma_load_2d(st + kPacked, &tm_w2, p_full + s, sb * (kSlotK / 2), a0, kEvictFirst);
        for (int g = 0; g < ngs; ++g) {
          bulk_load(st + NB * kPacked + g * kPairBytes, ap.sz[0] + (g0 + g) * p.n + a0, pair_bytes, p_full + s);
          if (NB == 2) bulk_load(st + NB * kPacked + kPairs + g * kPairBytes, ap.sz[1] + (g0 + g) * p.n + a0, pair_bytes, p_full + s);
        }
      };
      auto acts = [&](int s, int sb) {
        uint8_t* at = p_ring + static_cast<size_t>(s) * S::kP + NB * (kPacked + kPairs);
#pragma unroll
        for (int j = 0; j < kSub; ++j) tma_load_2d(at + j * S::kAct, &tm_x, p_full + s, (sb * kSub + j) * kBKh, 0, kEvictLast);
      };
      produce(p_full, p_free, PD, tx, sb_lo, nsb, weights, acts);
    }
    split_k_epilogue<__half, 1, BN, NB, CS, false>(p, accs, red, a0, crank);
  } else {
    // ===== consumer warpgroup: nibbles -> fp16 A fragments in registers -> wgmma =====
    const int q = warp & 3;
    const int t = lane & 3;                                      // channel pair of the A fragment held by this thread
    const uint32_t shift = (t & 2) ? 8u : 0u, mask = (t & 1) ? 0x00f000f0u : 0x000f000fu;
    const __half2 mul = __float2half2_rn((t & 1) ? 0.0625f : 1.f);
    Acc<BN> acc[NB];
#pragma unroll 1
    for (int sb = 0; sb < nsb; ++sb) {
      const int sp = sb % PD;
      mbar_wait(p_full + sp, (sb / PD) & 1);
      const uint8_t* pk = p_ring + static_cast<size_t>(sp) * S::kP;
      const uint32_t act0 = smem_u32(pk + NB * (kPacked + kPairs));
#pragma unroll 1
      for (int j = 0; j < kSub; ++j) {                           // K block j of the slot: 32 bytes of every packed row
        const int pair_slot = (j * kBKh) / ap.group < ngs ? (j * kBKh) / ap.group : ngs - 1;
        const uint64_t db = make_smem_desc(act0 + j * S::kAct);
#pragma unroll
        for (int w = 0; w < NB; ++w)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint32_t a[kBKh / 16][4];
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {                     // rows g, g + 8 of this warp's 16
              const int r = h * 64 + q * 16 + (lane >> 2) + rr * 8;
              const __half2 sz = *reinterpret_cast<const __half2*>(pk + NB * kPacked + w * kPairs + pair_slot * kPairBytes + r * 4);
              const __half zp = __high2half(sz);
              const __half2 add = __half2half2((t & 1) ? __hneg(__hadd(__float2half(64.f), zp)) : __hneg(__hadd(__float2half(1024.f), zp)));
              const __half2 s2 = __half2half2(__low2half(sz));
              // the 16-byte chunks 2j, 2j + 1 of the row's 128 bytes are stored at chunk ^ (r % 8) by the 128-byte swizzle
              const uint8_t* row = pk + w * kPacked + r * kSwizzleBytes;
              const uint4 w0 = *reinterpret_cast<const uint4*>(row + (((2 * j) ^ (r & 7)) << 4));
              const uint4 w1 = *reinterpret_cast<const uint4*>(row + (((2 * j + 1) ^ (r & 7)) << 4));
              const uint32_t words[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
              for (int k = 0; k < kBKh / 16; ++k) {              // word 2k = channels 16k .. 16k+7, word 2k+1 = 16k+8 .. 16k+15
                a[k][rr] = awq_dequant_pair(words[2 * k], shift, mask, mul, add, s2);
                a[k][2 + rr] = awq_dequant_pair(words[2 * k + 1], shift, mask, mul, add, s2);
              }
            }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBKh / 16; ++k)
              wgmma_rs_f16(acc[w].d[h][0], a[k], db + 2 * k, (sb == 0 && j == 0 && k == 0) ? 0u : 1u);
            wgmma_commit();
            wgmma_wait();                                        // the A registers are rewritten by the next conversion
          }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(p_free + sp);
    }
#pragma unroll
    for (int w = 0; w < NB; ++w) acc_store<BN>(acc[w], accs + w * BN * kAccPitch);
    epi_bar_sync();
    split_k_epilogue<__half, 1, BN, NB, CS, true>(p, accs, red, a0, crank);   // float arm: fp32 partials, no scales
  }
}

// ---- host side ----
CUtensorMap make_packed_map(const void* wp, int64_t n, int64_t k, int box_rows) {
  // wp as bytes [n, k/2]; box = box_rows x 128 bytes (a super-block of 256 channels), 128-byte swizzle
  CUtensorMap m;
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(k / 2), static_cast<cuuint64_t>(n)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(k / 2)};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(kSlotK / 2), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  const CUresult r = get_tensor_map_encoder()(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(wp), dims, strides, box,
                                              estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled (awq) failed with code " + std::to_string(r));
  return m;
}

template <int BN, int NB>
int p_stages_for(int cs, int nkb) {
  using S = AwqDecSmem<BN, NB>;
  const size_t cap = 220 * 1024;
  const size_t fixed = S::kAcc + S::kCtrl + red_bytes(cs, NB, BN) + 1024;
  if (fixed + 2 * S::kP > cap) return 0;
  int st = static_cast<int>((cap - fixed) / S::kP);
  st = std::min(st, kMaxP);
  return std::max(2, std::min(st, std::max(nkb, 2)));
}

template <int BN, int NB>
Plan plan_awq(int64_t n, int kb_total /* super-blocks */, int sm_count, int force_cs, int force_rows) {
  Plan best;
  double best_cost = 1e30;
  for (int cs = 1; cs <= 4; ++cs) {
    if (force_cs && cs != force_cs) continue;
    if (cs > 1 && kb_total < 2 * cs) continue;
    const int nkb = (kb_total + cs - 1) / cs;
    const int ps = p_stages_for<BN, NB>(cs, nkb);
    if (ps == 0) continue;
    const int maxc = dispatch_cs(cs, [&](auto c) {
      return max_clusters(awq_decode_kernel<BN, NB, decltype(c)::value>, cs, kThreads, AwqDecSmem<BN, NB>::bytes(ps, cs), sm_count);
    });
    // Tile height.  The conversion covers all 128 rows of a block whatever the tile height, so full-height tiles waste nothing;
    // a shorter tile that puts the stream on more SMs wins when 128-row tiles leave many idle.
    // cost = streamed rows x K blocks per CTA (+ the cluster exchange).
    const int full = static_cast<int>((n + 127) / 128);
    int cand[2] = {128, 128};
    if (!force_rows && full * 10 < maxc * 9) {
      const int r = static_cast<int>((((n + maxc - 1) / maxc) + 7) / 8 * 8);
      if (r >= 64 && r < 128) cand[1] = r;
    }
    for (int ci = 0; ci < 2; ++ci) {
      const int rows = force_rows ? force_rows : cand[ci];
      const int tiles = static_cast<int>((n + rows - 1) / rows);
      if (tiles > maxc) continue;
      const double cost = static_cast<double>(nkb) * (rows / 128.0) + (cs > 1 ? 1.0 : 0.0);
      if (cost < best_cost) {
        best_cost = cost;
        best.cs = cs;
        best.tile_rows = rows;
        best.tiles = tiles;
        best.stages = ps;
      }
    }
  }
  return best;
}

template <int BN, int NB>
bool run(const void* x, const AwqNative& w, const AwqNative* w2, int64_t m, AwqDecParams p, cudaStream_t st) {
  const int sb_total = static_cast<int>(w.k / kSlotK);
  const int sms = sm_count_of_current_device();
  const Plan plan = cached_plan(w.n, sb_total, false,
                                [&](int force_cs, int force_rows) { return plan_awq<BN, NB>(w.n, sb_total, sms, force_cs, force_rows); });
  if (plan.cs == 0) return false;
  p.d.n = w.n;
  p.d.m = m;
  p.d.kb_total = sb_total * kSub;
  p.sb_total = sb_total;
  p.d.tile_rows = plan.tile_rows;
  p.d.stages = plan.stages;
  p.group = w.group;
  p.sz[0] = static_cast<const __half2*>(w.sz);
  p.sz[1] = static_cast<const __half2*>(w2 ? w2->sz : w.sz);
  const CUtensorMap tmx = make_operand_map(x, m, w.k, 2, 1, BN);
  const CUtensorMap tmw = make_packed_map(w.wp, w.n, w.k, plan.tile_rows);
  const CUtensorMap tmw2 = make_packed_map(w2 ? w2->wp : w.wp, w.n, w.k, plan.tile_rows);
  dispatch_cs(plan.cs, [&](auto c) {
    auto kernel = awq_decode_kernel<BN, NB, decltype(c)::value>;
    allow_dynamic_smem(kernel, kMaxDynSmem);
    launch_clustered(kernel, dim3(static_cast<unsigned>(plan.tiles * plan.cs)), dim3(kThreads), AwqDecSmem<BN, NB>::bytes(plan.stages, plan.cs),
                     plan.cs, st, tmx, tmw, tmw2, p);
  });
  check_launch();
  return true;
}

template <int NB>
bool run_m(const void* x, const AwqNative& w, const AwqNative* w2, int64_t m, const AwqDecParams& p, cudaStream_t st) {
  if (m <= 16) return run<16, NB>(x, w, w2, m, p, st);
  if (m <= 32) return run<32, NB>(x, w, w2, m, p, st);
  return run<64, NB>(x, w, w2, m, p, st);
}

// CT2B200_AWQ_DECODE=0 selects the general stream-K kernel of awq.cu (CT2B200_AWQ_DECODE_GLU does the same for the
// fused gate/up launch only).
bool enabled() { return env_int("CT2B200_AWQ_DECODE", CT2B200_DEFAULT_AWQ_DECODE) != 0; }
bool glu_enabled() { return env_int("CT2B200_AWQ_DECODE_GLU", env_int("CT2B200_AWQ_DECODE", CT2B200_DEFAULT_AWQ_DECODE)) != 0; }

}  // namespace

// false = shape not covered (more tiles than one wave holds, group not a multiple of 64): caller uses gemm_awq_tc_kernel
bool dense_awq_decode(const void* x, const AwqNative& w, const void* bias, const void* residual, int act, int64_t m, void* y,
                      cudaStream_t st) {
  if (!enabled() || m < 1 || m > 64 || w.group % kBKh != 0 || w.k % kSlotK != 0 || w.sz == nullptr || w.n % 8 != 0) return false;
  AwqDecParams p{};
  p.d.bias = bias;
  p.d.residual = residual;
  p.d.y = y;
  p.d.act = act;
  p.d.ldy = w.n;
  return run_m<1>(x, w, nullptr, m, p, st);
}

bool dense_awq_glu_decode(const void* x, const AwqNative& wg, const AwqNative& wu, int act, int64_t m, void* h, cudaStream_t st) {
  if (!glu_enabled() || m < 1 || m > 64 || wg.group % kBKh != 0 || wg.k % kSlotK != 0 || wg.group != wu.group ||
      wg.sz == nullptr || wu.sz == nullptr || wg.n % 8 != 0)
    return false;
  AwqDecParams p{};
  p.d.y = h;
  p.d.act = act;
  p.d.ldy = wg.n;
  return run_m<2>(x, wg, &wu, m, p, st);
}

}  // namespace ct2b200
