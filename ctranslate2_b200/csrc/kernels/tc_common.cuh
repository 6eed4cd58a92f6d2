// tc_common.cuh — inline-PTX wrappers shared by the wgmma kernels (gemm_tc.cu, gemm_decode.cu, gemm_prefill.cu, awq.cu,
// awq_decode.cu): mbarrier, TMA (cp.async.bulk.tensor), the operand ring (barrier set-up and producer schedule), wgmma with
// its shared-memory descriptors, and the hand-over of the register accumulators to the row-per-thread epilogues.
// Bit layouts follow cute::GmmaDescriptor (CUTLASS, cute/arch/mma_sm90_desc.hpp).
#pragma once

#include <cuda.h>
#include <cudaTypedefs.h>

#include <string>

#include "../common.cuh"

namespace ct2b200 {
namespace tc {

constexpr int kTcThreads = 160;          // warps 0-3 = the consumer warpgroup (wgmma + epilogue), warp 4 = TMA producer
constexpr int kProducerWarp = 4;
constexpr int kTileM = 128;              // tile rows: two m64 wgmma instructions
constexpr int kSwizzleBytes = 128;       // bytes of K per smem row (= one 128B swizzle atom)
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

// operand kinds of the kernels: KIND = 0 s8 / 1 f16 / 2 bf16
template <int KIND> struct Elem { static constexpr int bytes = KIND == 0 ? 1 : 2; };

// Activation out of line: the epilogues are unrolled over the columns of a chunk, and inlining erff/tanhf/expf
// into every unrolled copy made the kernels 20-30 k SASS instructions (0.3-0.5 MB), i.e. instruction-fetch bound.
static __device__ __noinline__ float act_call(float x, int act) {
  if (act == CT2B200_ACT_SWISH) return __fdividef(x, 1.f + __expf(-x));     // the hot one (SwiGLU)
  return apply_act(x, act);
}

// ---- PTX wrappers ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// One lane of a CONVERGED warp, chosen by elect.sync.  The single-thread roles (TMA producer, MMA issuer) must be entered through
// this and not through `lane == 0`: cp.async.bulk.tensor executes on the uniform datapath, and inside a branch the compiler
// cannot prove single-threaded it wraps EVERY such instruction in an ELECT ... BRA.U.ANY loop over the active lanes.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "elect.sync _|p, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}
// ---- wgmma (sm_90a): D[64 x N] (+)= A[64 x K] * B[N x K]^T, both operands K-major in 128B-swizzled shared memory (or A in
// registers), accumulators in the registers of the four warps of a warpgroup ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// K-major, SWIZZLE_128B shared-memory matrix descriptor (cute::GmmaDescriptor): rows of 128 bytes,
// 8-row groups 1024 bytes apart (SBO), layout type 1 (B128) in bits [62,64).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);        // start address, bits [0,14)
  d |= static_cast<uint64_t>(1) << 16;                           // leading byte offset (unused for SW128 K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;                   // stride byte offset, bits [32,46)
  d |= static_cast<uint64_t>(1) << 62;                           // SWIZZLE_128B
  return d;
}

#define CT2_WG_R4(d, o) "+r"(d[o]), "+r"(d[o + 1]), "+r"(d[o + 2]), "+r"(d[o + 3])
#define CT2_WG_R8(d, o) CT2_WG_R4(d, o), CT2_WG_R4(d, o + 4)
#define CT2_WG_R16(d, o) CT2_WG_R8(d, o), CT2_WG_R8(d, o + 8)
#define CT2_WG_R32(d, o) CT2_WG_R16(d, o), CT2_WG_R16(d, o + 16)
#define CT2_WG_L8 "{%0,%1,%2,%3,%4,%5,%6,%7}"
#define CT2_WG_L16 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}"
#define CT2_WG_L32 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}"
// KIND = 0 s8 (K = 32 per instruction) / 1 f16 / 2 bf16 (K = 16); acc == 0 overwrites D.  NR = N / 2 registers per thread:
// d[4j], d[4j+1] = row 16 * warp + lane / 4, columns 8j + 2 * (lane % 4) + {0, 1};  d[4j+2], d[4j+3] = the same columns 8 rows below.
#define CT2_WGMMA_SS(N, NR, LIST, REGS, A, B, P)                                                                                 \
  template <int KIND>                                                                                                            \
  __device__ __forceinline__ void wgmma_ss(uint32_t (&d)[NR], uint64_t da, uint64_t db, uint32_t acc) {                          \
    if constexpr (KIND == 0)                                                                                                     \
      asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, " P ", 0;\nwgmma.mma_async.sync.aligned.m64n" #N "k32.s32.s8.s8 " LIST      \
                   ", " A ", " B ", p;\n}\n" : REGS(d, 0) : "l"(da), "l"(db), "r"(acc));                                         \
    else if constexpr (KIND == 1)                                                                                                \
      asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, " P ", 0;\nwgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 " LIST    \
                   ", " A ", " B ", p, 1, 1, 0, 0;\n}\n" : REGS(d, 0) : "l"(da), "l"(db), "r"(acc));                             \
    else                                                                                                                         \
      asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, " P ", 0;\nwgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 " LIST  \
                   ", " A ", " B ", p, 1, 1, 0, 0;\n}\n" : REGS(d, 0) : "l"(da), "l"(db), "r"(acc));                             \
  }
CT2_WGMMA_SS(16, 8, CT2_WG_L8, CT2_WG_R8, "%8", "%9", "%10")
CT2_WGMMA_SS(32, 16, CT2_WG_L16, CT2_WG_R16, "%16", "%17", "%18")
CT2_WGMMA_SS(64, 32, CT2_WG_L32, CT2_WG_R32, "%32", "%33", "%34")
// fp16 A fragment from registers (a[0..3] = the m16n8k16 A fragment of this warp's 16 rows), B from shared memory
#define CT2_WGMMA_RS(N, NR, LIST, REGS, A0, A1, A2, A3, B, P)                                                                    \
  __device__ __forceinline__ void wgmma_rs_f16(uint32_t (&d)[NR], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {           \
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, " P ", 0;\nwgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 " LIST      \
                 ", {" A0 "," A1 "," A2 "," A3 "}, " B ", p, 1, 1, 0;\n}\n"                                                      \
                 : REGS(d, 0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));                                  \
  }
CT2_WGMMA_RS(16, 8, CT2_WG_L8, CT2_WG_R8, "%8", "%9", "%10", "%11", "%12", "%13")
CT2_WGMMA_RS(32, 16, CT2_WG_L16, CT2_WG_R16, "%16", "%17", "%18", "%19", "%20", "%21")
CT2_WGMMA_RS(64, 32, CT2_WG_L32, CT2_WG_R32, "%32", "%33", "%34", "%35", "%36", "%37")

// Accumulators of one 128 x BN tile in the registers of one warpgroup: [64-row half][64-column piece][wgmma D fragment]
template <int BN> struct AccShape {
  static_assert(BN == 16 || BN == 32 || BN % 64 == 0, "tile widths: 16, 32 or a multiple of 64");
  static constexpr int kPiece = BN < 64 ? BN : 64;
  static constexpr int kPieces = BN / kPiece;
  static constexpr int kRegs = kPiece / 2;
};
template <int BN> struct Acc { uint32_t d[2][AccShape<BN>::kPieces][AccShape<BN>::kRegs]; };
constexpr int kHalfTileBytes = 64 * kSwizzleBytes;      // 64 rows of a swizzled operand tile

// one K block (128 bytes of K) of a 128 x BN tile: A tile at sa (128 rows), B tile at sb (BN rows); first == overwrite
template <int KIND, int BN>
__device__ __forceinline__ void mma_block(Acc<BN>& c, uint32_t sa, uint32_t sb, bool first) {
  using A = AccShape<BN>;
#pragma unroll
  for (int k = 0; k < kSwizzleBytes / 32; ++k)          // +32 bytes of K inside the swizzle atom = +2 on the address field
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int pc = 0; pc < A::kPieces; ++pc)
        wgmma_ss<KIND>(c.d[h][pc], make_smem_desc(sa + h * kHalfTileBytes) + 2 * k, make_smem_desc(sb + pc * kHalfTileBytes) + 2 * k,
                       (first && k == 0) ? 0u : 1u);
}

// The fused epilogues work one output row per thread.  The warpgroup parks its fragments in shared memory as
// [column][kAccPitch rows] (pitch 132 words: the fragment stores and the row-wise loads are both bank-conflict free).
constexpr int kAccPitch = kTileM + 4;
constexpr int acc_bytes(int cols) { return (cols * kAccPitch * 4 + 1023) / 1024 * 1024; }
template <int BN>
__device__ __forceinline__ void acc_store(const Acc<BN>& c, uint32_t* dst) {
  using A = AccShape<BN>;
  const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int pc = 0; pc < A::kPieces; ++pc)
#pragma unroll
      for (int j = 0; j < A::kPiece / 8; ++j) {
        uint32_t* q = dst + (pc * 64 + j * 8 + (l & 3) * 2) * kAccPitch + h * 64 + w * 16 + (l >> 2);
        q[0] = c.d[h][pc][4 * j];
        q[kAccPitch] = c.d[h][pc][4 * j + 1];
        q[8] = c.d[h][pc][4 * j + 2];
        q[kAccPitch + 8] = c.d[h][pc][4 * j + 3];
      }
}
// NC consecutive columns of row `rloc`
template <int NC>
__device__ __forceinline__ void acc_load(const uint32_t* src, int rloc, uint32_t (&r)[NC]) {
#pragma unroll
  for (int j = 0; j < NC; ++j) r[j] = src[j * kAccPitch + rloc];
}


__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

// mbarriers of the operand ring; then the next kernel may be scheduled, and phase 1 of the cluster barrier is signalled
// (this CTA is alive: peers may write its shared memory once they have waited for the phase)
template <int CS>
__device__ __forceinline__ void ring_init(uint64_t* full_bar, uint64_t* free_bar, int nstages) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < nstages; ++s) {
      mbar_init(full_bar + s, 1);
      mbar_init(free_bar + s, 4);                    // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  griddep_launch();
  if (CS > 1) cluster_arrive();
}

// Producer schedule of one elected lane over blocks [lo, lo + n): weights(slot, block) and acts(slot, block) issue the
// copies of one ring slot (tx_bytes in all).  The weights never depend on the previous kernel, so the first ring fill is
// issued BEFORE the dependency wait and overlaps the predecessor's tail.
template <typename W, typename A>
__device__ __forceinline__ void produce(uint64_t* full_bar, uint64_t* free_bar, int nstages, uint32_t tx_bytes, int lo, int n,
                                        const W& weights, const A& acts) {
  const int pre = min(nstages, n);
#pragma unroll 1
  for (int i = 0; i < pre; ++i) {
    mbar_expect_tx(full_bar + i, tx_bytes);
    weights(i, lo + i);
  }
  griddep_wait();
#pragma unroll 1
  for (int i = 0; i < pre; ++i) acts(i, lo + i);
#pragma unroll 1
  for (int it = pre; it < n; ++it) {
    const int s = it % nstages;
    mbar_wait(free_bar + s, ((it / nstages) & 1) ^ 1);
    mbar_expect_tx(full_bar + s, tx_bytes);
    weights(s, lo + it);
    acts(s, lo + it);
  }
}


// ---- host side ----
inline PFN_cuTensorMapEncodeTiled_v12000 get_tensor_map_encoder() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CT2_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres));
    if (qres != cudaDriverEntryPointSuccess || !ptr) throw std::runtime_error("cuTensorMapEncodeTiled is unavailable");
    fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr);
  }
  return fn;
}

// [rows, k] row-major matrix of `elem` bytes; box = box_rows x 128 bytes, 128B swizzle, zero OOB fill.
inline CUtensorMap make_operand_map(const void* base, int64_t rows, int64_t k, int elem, int kind, int box_rows) {
  CUtensorMap m;
  const CUtensorMapDataType dt = kind == 0 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                               : kind == 1 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(k), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(k) * elem};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(kSwizzleBytes / elem), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  const CUresult r = get_tensor_map_encoder()(&m, dt, 2, const_cast<void*>(base), dims, strides, box, estr,
                                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled failed with code " + std::to_string(r));
  return m;
}


}  // namespace tc
}  // namespace ct2b200
