// attention_tile.cuh — the 64-key tile step shared by the decode attention kernels (attention_decode.cu,
// attention_mma.cu): cp.async staging into XOR-swizzled shared memory, S = Q K^T, online softmax, O += P V for the
// 16 keys a warp owns.
//
// A naive version of this loop spends most of its instructions on integer address arithmetic and is issue bound.
// Hence everything that does not depend on the tile is
// hoisted: per-thread cp.async / ldmatrix offsets are computed once (the 8 rows a thread copies differ by a constant
// stride, so the copies use immediate offsets), masking and zero-fill only exist on the ragged last tile of a
// sequence, the accumulator rescale is skipped while the running maximum is unchanged, and the unused lower half of
// every MMA accumulator lives in four rotating dummy registers instead of being zeroed per instruction.
#pragma once

#include "mma_common.cuh"

namespace ct2b200 {
namespace attn {

using namespace mma;

constexpr int kTileKeys = 64;
constexpr int kTileThreads = 128;

// mma.m16n8k16 whose accumulator rows 8..15 are known to stay zero (A rows 8..15 are zero): only c0, c1 are live
template <typename T>
__device__ __forceinline__ void mma_top(float& c0, float& c1, float (&z)[2], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {
  const uint32_t zero = 0u;
  if constexpr (std::is_same<T, __half>::value) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c0), "+f"(c1), "+f"(z[0]), "+f"(z[1])
                 : "r"(a0), "r"(zero), "r"(a2), "r"(zero), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c0), "+f"(c1), "+f"(z[0]), "+f"(z[1])
                 : "r"(a0), "r"(zero), "r"(a2), "r"(zero), "r"(b0), "r"(b1));
  }
}

__device__ __forceinline__ void cp16_full(uint32_t smem_addr, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_addr), "l"(gmem));
}
__device__ __forceinline__ void cp16_zfill(uint32_t smem_addr, const void* gmem, bool valid) {
  const int bytes = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_addr), "l"(gmem), "r"(bytes));
}
__device__ __forceinline__ void ldsm4_u32(uint32_t (&r)[4], uint32_t s) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(s));
}
__device__ __forceinline__ void ldsm4_t_u32(uint32_t (&r)[4], uint32_t s) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(s));
}

// Tile-invariant per-thread state.  Two shared-memory tile layouts:
//   kTma = false (cp.async staging):  [64 keys][D] T, 16-byte chunk c of key r stored at chunk c ^ (r & 7);
//   kTma = true  (cp.async.bulk.tensor, SWIZZLE_128B boxes of 64 keys x 128 bytes):  [D*2/128 column halves][64 keys][128 B],
//                chunk c (0..7) of a 128-byte row stored at c ^ (r & 7) — the hardware swizzle; tile base 1024-aligned.
// Both are conflict-free for the 8-row ldmatrix reads.
template <typename T, int D, bool kTma = false>
struct TileCtx {
  static constexpr int CH = D / 8;                                   // 16-byte chunks per key
  static constexpr int kRowsPerPass = kTileThreads / CH;             // keys copied per cp.async pass of the CTA
  static constexpr int kPasses = kTileKeys / kRowsPerPass;
  static constexpr int kPassBytes = kRowsPerPass * D * static_cast<int>(sizeof(T));
  static constexpr int kTileBytes = kTileKeys * D * static_cast<int>(sizeof(T));
  static constexpr int kBoxBytes = kTileKeys * 128;                  // one TMA box: 64 keys x 128 bytes
  static constexpr int kBoxes = D * static_cast<int>(sizeof(T)) / 128;
  uint32_t cp_smem;        // byte offset of this thread's first chunk inside a tile
  uint32_t cp_gmem;        // byte offset of the same chunk relative to the tile's first key in the cache
  int cp_row;              // first key this thread copies (the others are cp_row + i * kRowsPerPass)
  uint32_t k_off[D / 16];  // ldmatrix offsets (bytes, relative to the warp's 16-key slab): QK^T, k-step kk
  uint32_t v_off[D / 16];  // ldmatrix.trans offsets: PV, n-tile pair j

  // byte offset of 16-byte chunk `c` of key `rr` (relative to the slab of 16 keys the row belongs to)
  static __device__ __forceinline__ uint32_t chunk_offset(int rr, int c) {
    if constexpr (kTma) return static_cast<uint32_t>((c >> 3) * kBoxBytes + rr * 128 + (((c & 7) ^ (rr & 7)) * 16));
    else return static_cast<uint32_t>(rr * D * sizeof(T) + ((c ^ (rr & 7)) * 16));
  }
  // byte offset of the warp's 16-key slab inside a tile
  static __device__ __forceinline__ uint32_t slab_offset(int warp) {
    return static_cast<uint32_t>(warp * 16 * (kTma ? 128 : D * static_cast<int>(sizeof(T))));
  }

  __device__ __forceinline__ void init(int tid) {
    const int lane = tid & 31;
    const int r = tid / CH, ch = tid % CH;
    cp_row = r;
    cp_smem = static_cast<uint32_t>(r * D * sizeof(T) + ((ch ^ (r & 7)) * 16));
    cp_gmem = static_cast<uint32_t>(r * D * sizeof(T) + ch * 16);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const int rr = (lane & 7) + (lane >> 4) * 8;
      k_off[kk] = chunk_offset(rr, kk * 2 + ((lane >> 3) & 1));
      const int rv = (lane & 7) + ((lane >> 3) & 1) * 8;
      v_off[kk] = chunk_offset(rv, kk * 2 + (lane >> 4));
    }
  }

  // copy one K and one V tile (64 keys starting at `k_tile` / `v_tile` in the cache) into the stage at shared
  // addresses sk / sv; `nvalid` < 64 only on the last, ragged tile of a sequence (rows beyond it are zero filled)
  __device__ __forceinline__ void load(uint32_t sk, uint32_t sv, const T* k_tile, const T* v_tile, int nvalid) const {
    const uint8_t* gk = reinterpret_cast<const uint8_t*>(k_tile) + cp_gmem;
    const uint8_t* gv = reinterpret_cast<const uint8_t*>(v_tile) + cp_gmem;
    const uint32_t dk = sk + cp_smem, dv = sv + cp_smem;
    if (nvalid >= kTileKeys) {
#pragma unroll
      for (int i = 0; i < kPasses; ++i) {
        cp16_full(dk + i * kPassBytes, gk + i * kPassBytes);
        cp16_full(dv + i * kPassBytes, gv + i * kPassBytes);
      }
    } else {
#pragma unroll
      for (int i = 0; i < kPasses; ++i) {
        const bool ok = cp_row + i * kRowsPerPass < nvalid;
        cp16_zfill(dk + i * kPassBytes, ok ? gk + i * kPassBytes : gk, ok);
        cp16_zfill(dv + i * kPassBytes, ok ? gv + i * kPassBytes : gv, ok);
      }
    }
  }
};

// Running softmax state of one warp for the query rows it holds (row g = lane / 4 < G is real)
template <int D>
struct WarpAcc {
  float o[D / 8][2];
  float m, l;
  __device__ __forceinline__ void reset() {
#pragma unroll
    for (int j = 0; j < D / 8; ++j) o[j][0] = o[j][1] = 0.f;
    m = -INFINITY;
    l = 0.f;
  }
};

// One tile for one warp: keys [warp*16, warp*16+16) of the staged tile.  qf = Q as A fragments (rows 0..G-1 real,
// pre-scaled by log2(e)/sqrt(d)); nvalid = valid keys of the tile (64 except on the ragged last tile).
template <typename T, int D, bool kTma>
__device__ __forceinline__ void tile_step(const TileCtx<T, D, kTma>& cx, uint32_t sk, uint32_t sv, int warp, int lane,
                                          const uint32_t (&qf)[D / 16][2], WarpAcc<D>& acc, int nvalid) {
  const int t4 = lane & 3;
  const uint32_t ks = sk + TileCtx<T, D, kTma>::slab_offset(warp);
  const uint32_t vs = sv + TileCtx<T, D, kTma>::slab_offset(warp);
  float z[4][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};      // accumulator rows 8..15: stay zero
  // scores of keys 2*t4 (+1) and 8 + 2*t4 (+1); two partial sums each (even / odd k-steps) halve the HMMA chains
  float s0[2] = {0.f, 0.f}, s1[2] = {0.f, 0.f}, s0b[2] = {0.f, 0.f}, s1b[2] = {0.f, 0.f};
#pragma unroll
  for (int kk = 0; kk < D / 16; kk += 2) {
    uint32_t bf[4], bg[4];
    ldsm4_u32(bf, ks + cx.k_off[kk]);
    ldsm4_u32(bg, ks + cx.k_off[kk + 1]);
    mma_top<T>(s0[0], s0[1], z[0], qf[kk][0], qf[kk][1], bf[0], bf[1]);
    mma_top<T>(s1[0], s1[1], z[1], qf[kk][0], qf[kk][1], bf[2], bf[3]);
    mma_top<T>(s0b[0], s0b[1], z[2], qf[kk + 1][0], qf[kk + 1][1], bg[0], bg[1]);
    mma_top<T>(s1b[0], s1b[1], z[3], qf[kk + 1][0], qf[kk + 1][1], bg[2], bg[3]);
  }
  s0[0] += s0b[0]; s0[1] += s0b[1]; s1[0] += s1b[0]; s1[1] += s1b[1];
  if (nvalid < kTileKeys) {                        // ragged last tile: mask the keys past the end
    const int kb = warp * 16 + 2 * t4;
    if (kb >= nvalid) s0[0] = -INFINITY;
    if (kb + 1 >= nvalid) s0[1] = -INFINITY;
    if (kb + 8 >= nvalid) s1[0] = -INFINITY;
    if (kb + 9 >= nvalid) s1[1] = -INFINITY;
  }
  float mx = fmaxf(fmaxf(s0[0], s0[1]), fmaxf(s1[0], s1[1]));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
  if (__any_sync(0xffffffffu, mx > acc.m)) {       // the running maximum moved for some row: rescale
    const float nm = fmaxf(acc.m, mx);
    const float corr = (nm == -INFINITY) ? 1.f : exp2f(acc.m - nm);
    acc.m = nm;
    acc.l *= corr;
#pragma unroll
    for (int j = 0; j < D / 8; ++j) { acc.o[j][0] *= corr; acc.o[j][1] *= corr; }
  }
  const float mref = acc.m == -INFINITY ? 0.f : acc.m;   // all keys masked: exp2(-inf - 0) = 0
  const float p00 = exp2f(s0[0] - mref), p01 = exp2f(s0[1] - mref), p10 = exp2f(s1[0] - mref), p11 = exp2f(s1[1] - mref);
  acc.l += (p00 + p01) + (p10 + p11);
  const uint32_t pa0 = pack2<T>(p00, p01), pa2 = pack2<T>(p10, p11);
#pragma unroll
  for (int j = 0; j < D / 16; ++j) {
    uint32_t bf[4];
    ldsm4_t_u32(bf, vs + cx.v_off[j]);
    mma_top<T>(acc.o[2 * j][0], acc.o[2 * j][1], z[j & 1], pa0, pa2, bf[0], bf[1]);
    mma_top<T>(acc.o[2 * j + 1][0], acc.o[2 * j + 1][1], z[2 + (j & 1)], pa0, pa2, bf[2], bf[3]);
  }
}

}  // namespace attn
}  // namespace ct2b200
