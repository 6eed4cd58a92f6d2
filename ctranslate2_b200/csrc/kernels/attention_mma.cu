// attention_mma.cu — causal prefill attention and encoder self-attention on tensor cores for fp16/bf16 activations.
// Flash-attention style: a CTA owns 64 query rows of one (batch, head); 4 warps x 16 rows; K/V tiles of 64
// keys are staged through shared memory with cp.async (double buffered) straight from the un-replicated GQA
// cache [slot, Hkv, max_len, D]; S = Q K^T and O += P V run on mma.sync.m16n8k16 with fp32 accumulation and
// an fp32 online softmax; P never leaves registers.  Replaces MatMul + SoftMax + MatMul over a materialised
// [B,H,T,S] score tensor (reference src/layers/attention.cc:178-287, 536-602).
// (Decode attention is HBM-bound and lives in attention.cu; wgmma needs M >= 64 rows per head-tile, which
// a 16-row warp tile does not give, so the warp-level MMA is the right instrument for this shape.)
#include <type_traits>

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

constexpr int kQTile = 64, kKTile = 64, kThreads = 128;

// kEncoder = false: causal prefill, K/V read from the cache [slot, Hkv, max_len, D] (`time` new rows after `offset`).
// kEncoder = true: encoder self-attention (TransformerEncoder, src/layers/transformer.cc:427-471), K/V read from the fused
// qkv rows [batch * time, 3d] themselves; non-causal, keys at or past lengths[b] masked (null = time).  Query tiles wholly
// past the length are not computed: their rows are written as zeros (any finite value would do; they are ignored).
template <typename T, int D, bool kEncoder>
__global__ void __launch_bounds__(kThreads)
    attention_prefill_mma_kernel(const T* __restrict__ qkv, const T* __restrict__ k_cache, const T* __restrict__ v_cache,
                                 const int32_t* __restrict__ lengths, int64_t time, int64_t offset, int H, int Hkv,
                                 int64_t max_len, float scale_log2, T* __restrict__ out) {
  constexpr int LD = D + 8;                   // padded smem pitch (elements): conflict-free ldmatrix
  constexpr int CH = D / 8;                   // 16-byte chunks per row
  extern __shared__ __align__(16) uint8_t smem_raw[];
  T* sQ = reinterpret_cast<T*>(smem_raw);     // [64][LD]
  T* sK = sQ + kQTile * LD;                   // [2][64][LD]
  T* sV = sK + 2 * kKTile * LD;               // [2][64][LD]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int64_t q0 = static_cast<int64_t>(blockIdx.x) * kQTile;
  const int h = blockIdx.y;
  const int64_t b = blockIdx.z;
  const int kvh = h / (H / Hkv);
  const int64_t row_w = static_cast<int64_t>(H + 2 * Hkv) * D;
  const T* qbase = qkv + (b * time + q0) * row_w + static_cast<int64_t>(h) * D;
  const T* kc;
  const T* vc;
  int64_t kv_w;                               // elements between consecutive keys
  int nkeys;
  if constexpr (kEncoder) {
    nkeys = lengths ? lengths[b] : static_cast<int>(time);
    if (q0 >= nkeys) {                        // every query row of the tile is past the length
      for (int c = tid; c < kQTile * CH; c += kThreads) {
        const int r = c / CH, ch = c % CH;
        if (q0 + r < time)
          *reinterpret_cast<uint4*>(out + ((b * time + q0 + r) * H + h) * D + ch * 8) = make_uint4(0u, 0u, 0u, 0u);
      }
      return;
    }
    kc = qkv + b * time * row_w + static_cast<int64_t>(H + kvh) * D;
    vc = kc + static_cast<int64_t>(Hkv) * D;
    kv_w = row_w;
  } else {
    // keys visible to this query tile: 0 .. offset + min(q0+63, time-1)
    const int64_t last_q = min(q0 + kQTile, time) - 1;
    nkeys = static_cast<int>(offset + last_q + 1);
    kc = k_cache + (b * Hkv + kvh) * max_len * D;
    vc = v_cache + (b * Hkv + kvh) * max_len * D;
    kv_w = D;
  }
  const int ntiles = (nkeys + kKTile - 1) / kKTile;

  auto load_kv = [&](int stage, int kt) {
    const int64_t k0 = static_cast<int64_t>(kt) * kKTile;
    for (int c = tid; c < kKTile * CH; c += kThreads) {
      const int r = c / CH, ch = c % CH;
      const bool ok = k0 + r < nkeys;
      const int64_t off = (ok ? k0 + r : 0) * kv_w + ch * 8;
      cp16(sK + (stage * kKTile + r) * LD + ch * 8, kc + off, ok);
      cp16(sV + (stage * kKTile + r) * LD + ch * 8, vc + off, ok);
    }
  };
  // Q tile + first K/V tile
  for (int c = tid; c < kQTile * CH; c += kThreads) {
    const int r = c / CH, ch = c % CH;
    const bool ok = q0 + r < time;
    cp16(sQ + r * LD + ch * 8, qbase + (ok ? r : 0) * row_w + ch * 8, ok);
  }
  load_kv(0, 0);
  asm volatile("cp.async.commit_group;\n" ::);

  float o[D / 8][4];
#pragma unroll
  for (int j = 0; j < D / 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  uint32_t qf[D / 16][4];
  const int64_t qpos0 = offset + q0 + warp * 16 + g;       // absolute position of row g (row g+8: +8)

  for (int kt = 0; kt < ntiles; ++kt) {
    const int stage = kt & 1;
    if (kt + 1 < ntiles) load_kv(stage ^ 1, kt + 1);
    asm volatile("cp.async.commit_group;\n" ::);
    asm volatile("cp.async.wait_group 1;\n" ::);
    __syncthreads();
    if (kt == 0) {
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk)      // A fragments of this warp's 16 query rows
        ldsm4(qf[kk], sQ + (warp * 16 + (lane & 15)) * LD + kk * 16 + (lane >> 4) * 8);
    }
    const T* ks = sK + stage * kKTile * LD;
    const T* vs = sV + stage * kKTile * LD;

    // ---- S = Q K^T (16 x 64 per warp) ----
    float s[kKTile / 8][4];
#pragma unroll
    for (int j = 0; j < kKTile / 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
      for (int j = 0; j < kKTile / 8; j += 2) {
        uint32_t bf[4];   // {b0,b1} of key tile j, {b0,b1} of key tile j+1
        ldsm4(bf, ks + (j * 8 + (lane & 7) + (lane >> 4) * 8) * LD + kk * 16 + ((lane >> 3) & 1) * 8);
        mma16816<T>(s[j], qf[kk], bf[0], bf[1]);
        mma16816<T>(s[j + 1], qf[kk], bf[2], bf[3]);
      }
    }
    // ---- scale, causal mask, online softmax (rows g and g+8) ----
    const int64_t kbase = static_cast<int64_t>(kt) * kKTile;
    float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
    for (int j = 0; j < kKTile / 8; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int64_t key = kbase + j * 8 + 2 * t + (r & 1);
        const int64_t qp = qpos0 + (r >= 2 ? 8 : 0);
        const bool visible = kEncoder ? key < nkeys : key <= qp;
        const float v = visible ? s[j][r] * scale_log2 : -INFINITY;
        s[j][r] = v;
        mx[r >> 1] = fmaxf(mx[r >> 1], v);
      }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float corr[2], rs[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      corr[r] = (mx[r] == -INFINITY) ? 1.f : exp2f(m_run[r] - mx[r]);
      m_run[r] = mx[r];
    }
#pragma unroll
    for (int j = 0; j < kKTile / 8; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float p = (s[j][r] == -INFINITY) ? 0.f : exp2f(s[j][r] - mx[r >> 1]);
        s[j][r] = p;
        rs[r >> 1] += p;
      }
#pragma unroll
    for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * corr[r] + rs[r];
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      o[j][0] *= corr[0]; o[j][1] *= corr[0];
      o[j][2] *= corr[1]; o[j][3] *= corr[1];
    }
    // ---- O += P V ----
#pragma unroll
    for (int kk = 0; kk < kKTile / 16; ++kk) {
      uint32_t pa[4];
      pa[0] = pack2<T>(s[2 * kk][0], s[2 * kk][1]);
      pa[1] = pack2<T>(s[2 * kk][2], s[2 * kk][3]);
      pa[2] = pack2<T>(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      pa[3] = pack2<T>(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int j = 0; j < D / 8; j += 2) {
        uint32_t bf[4];   // V^T fragments: {b0,b1} for dims j*8.., {b0,b1} for dims (j+1)*8..
        ldsm4_t(bf, vs + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + j * 8 + (lane >> 4) * 8);
        mma16816<T>(o[j], pa, bf[0], bf[1]);
        mma16816<T>(o[j + 1], pa, bf[2], bf[3]);
      }
    }
    __syncthreads();    // everyone is done with this stage before it is refilled
  }

  // ---- finalize: row sums across the quad, normalise, store ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int64_t qi = q0 + warp * 16 + g + r * 8;
    if (qi >= time) continue;
    const float inv = l_run[r] > 0.f ? 1.f / l_run[r] : 0.f;
    T* orow = out + ((b * time + qi) * H + h) * D;
#pragma unroll
    for (int j = 0; j < D / 8; ++j)
      *reinterpret_cast<uint32_t*>(orow + j * 8 + 2 * t) = pack2<T>(o[j][2 * r] * inv, o[j][2 * r + 1] * inv);
  }
}


// Combine of the split partials by the last CTA of a (batch, kv-head): two batched load phases instead of a
// per-split dependent chain.  `scratch` = shared floats, at least 2*G*64 + G.
template <typename T, int D, int G>
__device__ __forceinline__ void decode_combine(const float* part, int nsplit, T* out_row, float* scratch) {
  const size_t PS = static_cast<size_t>(D) + 2;
  float* sm = scratch;                 // [G][nsplit] max
  float* sl = scratch + G * 64;        // [G][nsplit] sum
  float* sw = scratch + 2 * G * 64;    // [G] final 1/l
  __syncthreads();
  for (int e = threadIdx.x; e < G * nsplit; e += blockDim.x) {
    const int h = e / nsplit, s = e % nsplit;
    sm[h * 64 + s] = __ldcg(part + (static_cast<int64_t>(h) * nsplit + s) * PS + D);
    sl[h * 64 + s] = __ldcg(part + (static_cast<int64_t>(h) * nsplit + s) * PS + D + 1);
  }
  __syncthreads();
  if (threadIdx.x < G) {
    const int h = threadIdx.x;
    float mm = -INFINITY;
    for (int s = 0; s < nsplit; ++s) mm = fmaxf(mm, sm[h * 64 + s]);
    float ll = 0.f;
    for (int s = 0; s < nsplit; ++s) {
      const float c = sm[h * 64 + s] == -INFINITY ? 0.f : exp2f(sm[h * 64 + s] - mm);
      sm[h * 64 + s] = c;              // weight of split s
      ll += sl[h * 64 + s] * c;
    }
    sw[h] = 1.f / ll;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < G * D; e += blockDim.x) {
    const int h = e / D, i = e % D;
    const float* ph = part + static_cast<int64_t>(h) * nsplit * PS + i;
    float a = 0.f;
#pragma unroll 8
    for (int s = 0; s < nsplit; ++s) a += __ldcg(ph + s * PS) * sm[h * 64 + s];
    out_row[h * D + i] = from_f32<T>(a * sw[h]);
  }
}

// ---------------------------------------------------------------------------------------------
// Decode attention on tensor cores (one new token per sequence).  Same split-KV scheme and partial/ticket
// protocol as attention_decode_kernel (attention.cu), but the inner loop is MMA based: the G query heads of a KV
// head are rows 0..G-1 of a 16-row A tile, a CTA streams 64-key K/V tiles of its slice through shared memory with
// cp.async (3 stages), warp w owns keys [16w, 16w+16) of every tile: S = Q K^T (16 mma), fp32 online softmax,
// O += P V (16 mma).  ~2 tensor instructions per key instead of ~60 SIMT instructions, so the kernel is bound by
// the 16-byte coalesced cache reads, not by issue slots.
// ---------------------------------------------------------------------------------------------
constexpr int kDecTile = 64, kDecStages = 3;

__host__ __device__ inline size_t dec_partial_stride(int D) { return static_cast<size_t>(D) + 2; }

template <typename T>
__device__ __forceinline__ float rope_at_mma(const T* x, const float* sin, const float* cos, int i, int D, bool interleave) {
  float other;
  if (interleave) other = (i & 1) ? to_f32(x[i - 1]) : -to_f32(x[i + 1]);
  else other = (i < D / 2) ? -to_f32(x[i + D / 2]) : to_f32(x[i - D / 2]);
  return to_f32(x[i]) * cos[i] + other * sin[i];
}

template <typename T, int D, int G>
__global__ void __launch_bounds__(kThreads, 2)
    attention_decode_mma_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                                const T* __restrict__ qkv, T* __restrict__ k_cache, T* __restrict__ v_cache,
                                const float* __restrict__ sin_t, const float* __restrict__ cos_t,
                                const int32_t* __restrict__ lens, int H, int Hkv, int64_t max_len, bool interleave,
                                float scale_log2, T* __restrict__ out, float* __restrict__ partials,
                                int32_t* __restrict__ tickets) {
  using namespace attn;
  using Ctx = TileCtx<T, D, true>;
  constexpr int NW = kThreads / 32;
  constexpr int kTileElems = kDecTile * D;
  extern __shared__ uint8_t smem_dyn[];
  // the TMA boxes (SWIZZLE_128B) need a 1024-byte aligned base
  uint8_t* smem_raw = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  T* sK = reinterpret_cast<T*>(smem_raw);                       // [stages][D/64 boxes][64 keys][128 B]
  T* sV = sK + kDecStages * kTileElems;
  float* s_q = reinterpret_cast<float*>(sV + kDecStages * kTileElems);   // [G][D]
  __shared__ float s_m[NW][G], s_l[NW][G];
  __shared__ bool s_last;
  __shared__ __align__(8) uint64_t full_bar[kDecStages];

  if (threadIdx.x == 0) {
    for (int st = 0; st < kDecStages; ++st) tc::mbar_init(full_bar + st, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  griddep_launch();
  griddep_wait();
  const int split = blockIdx.x, nsplit = gridDim.x, kvh = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int pos = lens[b];
  const int nkeys = pos + 1;
  const int64_t row_w = static_cast<int64_t>(H + 2 * Hkv) * D;
  const T* q_in = qkv + b * row_w + static_cast<int64_t>(kvh) * G * D;
  const T* k_in = qkv + b * row_w + static_cast<int64_t>(H) * D + static_cast<int64_t>(kvh) * D;
  const T* v_in = k_in + static_cast<int64_t>(Hkv) * D;
  T* kc = k_cache + (static_cast<int64_t>(b) * Hkv + kvh) * max_len * D;
  T* vc = v_cache + (static_cast<int64_t>(b) * Hkv + kvh) * max_len * D;
  const float* sn = sin_t + static_cast<int64_t>(pos) * D;
  const float* cs = cos_t + static_cast<int64_t>(pos) * D;

  int per = (nkeys + nsplit - 1) / nsplit;
  per = ((per + kDecTile - 1) / kDecTile) * kDecTile;           // slices are whole 64-key tiles
  const int s0 = split * per;
  const int s1 = min(nkeys, s0 + per);
  const int ntiles = s1 > s0 ? (s1 - s0 + kDecTile - 1) / kDecTile : 0;

  Ctx cx;
  cx.init(tid);
  const uint32_t sK_u32 = static_cast<uint32_t>(__cvta_generic_to_shared(sK));
  const uint32_t sV_u32 = static_cast<uint32_t>(__cvta_generic_to_shared(sV));
  // K/V tiles by TMA: D*2/128 boxes of 64 keys x 128 bytes each, one mbarrier per stage (issued by thread 0)
  const int row0 = static_cast<int>((static_cast<int64_t>(b) * Hkv + kvh) * max_len) + s0;
  auto load_tile = [&](int stage, int kt) {
    tc::mbar_expect_tx(full_bar + stage, 2 * Ctx::kTileBytes);
#pragma unroll
    for (int h = 0; h < Ctx::kBoxes; ++h) {
      tc::tma_load_2d(reinterpret_cast<uint8_t*>(sK) + stage * Ctx::kTileBytes + h * Ctx::kBoxBytes, &tm_k, full_bar + stage,
                      h * 64, row0 + kt * kDecTile, tc::kEvictFirst);
      tc::tma_load_2d(reinterpret_cast<uint8_t*>(sV) + stage * Ctx::kTileBytes + h * Ctx::kBoxBytes, &tm_v, full_bar + stage,
                      h * 64, row0 + kt * kDecTile, tc::kEvictFirst);
    }
  };
  // The first tiles are requested right away, so the loads fly while the queries are rotated — except the tile that
  // contains position `pos`: it is loaded after the new token's K/V have been appended below.
  const bool owner = pos >= s0 && pos < s1;                     // this slice holds position `pos`
  const int kt_pos = owner ? (pos - s0) / kDecTile : -1;
  __syncthreads();                                              // mbarrier inits (thread 0) before anyone may wait on them
  if (warp == 0 && tc::elect_one()) {                           // single-thread role: tc_common.cuh, elect_one
#pragma unroll
    for (int st = 0; st < kDecStages - 1; ++st)
      if (st < ntiles && st != kt_pos) load_tile(st, st);
  }

  for (int e = tid; e < G * D; e += kThreads) {
    const int h = e / D, i = e % D;
    s_q[e] = rope_at_mma(q_in + h * D, sn, cs, i, D, interleave) * scale_log2;
  }
  if (owner) {                                                  // the owner of position `pos` appends k_new / v_new
    for (int i = tid; i < D; i += kThreads) {
      kc[static_cast<int64_t>(pos) * D + i] = from_f32<T>(rope_at_mma(k_in, sn, cs, i, D, interleave));
      vc[static_cast<int64_t>(pos) * D + i] = v_in[i];
    }
    asm volatile("fence.proxy.async;" ::: "memory");            // generic-proxy stores before the TMA (async proxy) reads
  }
  __syncthreads();
  if (warp == 0 && kt_pos >= 0 && kt_pos < kDecStages - 1 && tc::elect_one()) load_tile(kt_pos, kt_pos);

  // Q as A fragments: rows 0..G-1 = heads, rows G..15 = 0
  uint32_t qf[D / 16][2];
#pragma unroll
  for (int kk = 0; kk < D / 16; ++kk) {
    const float* qr = s_q + (g < G ? g : 0) * D + kk * 16 + 2 * t;
    const bool real = g < G;
    qf[kk][0] = real ? pack2<T>(qr[0], qr[1]) : 0u;
    qf[kk][1] = real ? pack2<T>(qr[8], qr[9]) : 0u;
  }
  WarpAcc<D> acc;
  acc.reset();

  for (int kt = 0; kt < ntiles; ++kt) {
    const int stage = kt % kDecStages;
    // the stage refilled here was consumed in iteration kt - 1 (trailing __syncthreads)
    if (warp == 0 && kt + kDecStages - 1 < ntiles && tc::elect_one())
      load_tile((kt + kDecStages - 1) % kDecStages, kt + kDecStages - 1);
    tc::mbar_wait(full_bar + stage, (kt / kDecStages) & 1);
    tile_step<T, D, true>(cx, sK_u32 + stage * Ctx::kTileBytes, sV_u32 + stage * Ctx::kTileBytes, warp, lane, qf, acc,
                          s1 - (s0 + kt * kDecTile));
    __syncthreads();
  }

  // ---- merge the 4 warps (each holds m, l, O for rows g < G over its keys) ----
  float l_run = acc.l;
  l_run += __shfl_xor_sync(0xffffffffu, l_run, 1);
  l_run += __shfl_xor_sync(0xffffffffu, l_run, 2);
  if (g < G && t == 0) { s_m[warp][g] = acc.m; s_l[warp][g] = l_run; }
  float* s_o = reinterpret_cast<float*>(smem_raw);              // [NW][G][D] fp32, reuses the K/V staging area
  __syncthreads();                                              // all tiles consumed before the area is reused
  if (g < G) {
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      s_o[(warp * G + g) * D + j * 8 + 2 * t] = acc.o[j][0];
      s_o[(warp * G + g) * D + j * 8 + 2 * t + 1] = acc.o[j][1];
    }
  }
  __syncthreads();
  const size_t PS = dec_partial_stride(D);
  float* part = partials + ((static_cast<int64_t>(b) * H + static_cast<int64_t>(kvh) * G) * nsplit) * PS;
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
    if (nsplit == 1) {                                          // single slice: no partials, no ticket, no combine
      out[static_cast<int64_t>(b) * H * D + (static_cast<int64_t>(kvh) * G + h) * D + i] = from_f32<T>(a * (1.f / ll));
      continue;
    }
    float* ph = part + (static_cast<int64_t>(h) * nsplit + split) * PS;
    ph[i] = a;
    if (i == 0) { ph[D] = mm; ph[D + 1] = ll; }
  }
  if (nsplit == 1) return;
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(tickets + b * Hkv + kvh, 1) == nsplit - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  decode_combine<T, D, G>(part, nsplit, out + static_cast<int64_t>(b) * H * D + static_cast<int64_t>(kvh) * G * D, s_o);
  if (tid == 0) tickets[b * Hkv + kvh] = 0;
}

template <typename T, int D>
void launch_mma(const void* qkv, const void* kc, const void* vc, int64_t batch, int64_t time, int64_t offset, int H,
                int Hkv, int64_t max_len, float scale, void* out, cudaStream_t st) {
  constexpr size_t smem = static_cast<size_t>(kQTile + 4 * kKTile) * (D + 8) * sizeof(T);
  auto kernel = attention_prefill_mma_kernel<T, D, false>;
  allow_dynamic_smem(kernel, smem);
  dim3 grid(div_up(time, kQTile), H, static_cast<unsigned>(batch));
  kernel<<<grid, kThreads, smem, st>>>(static_cast<const T*>(qkv), static_cast<const T*>(kc), static_cast<const T*>(vc),
                                       nullptr, time, offset, H, Hkv, max_len, scale * 1.4426950408889634f,
                                       static_cast<T*>(out));
  check_launch();
}

template <typename T, int D>
void launch_encoder_mma(const void* qkv, const int32_t* lengths, int64_t batch, int S, int H, float scale, void* out,
                        cudaStream_t st) {
  constexpr size_t smem = static_cast<size_t>(kQTile + 4 * kKTile) * (D + 8) * sizeof(T);
  auto kernel = attention_prefill_mma_kernel<T, D, true>;
  allow_dynamic_smem(kernel, smem);
  dim3 grid(div_up(S, kQTile), H, static_cast<unsigned>(batch));
  kernel<<<grid, kThreads, smem, st>>>(static_cast<const T*>(qkv), nullptr, nullptr, lengths, S, 0, H, H, 0,
                                       scale * 1.4426950408889634f, static_cast<T*>(out));
  check_launch();
}


template <typename T, int D>
bool launch_decode_mma_g(const void* qkv, void* kc, void* vc, const float* sn, const float* cs, const int32_t* lens,
                         int64_t batch, int H, int Hkv, int64_t max_len, bool interleave, float scale, void* out,
                         float* partials, int32_t* tickets, int splits, cudaStream_t st) {
  const int G = H / Hkv;
  constexpr size_t smem = static_cast<size_t>(2 * kDecStages * kDecTile) * D * sizeof(T) + 8 * D * sizeof(float) + 1024;
  // the caches as 2-D tensors [rows = batch * Hkv * max_len, D]; box = 64 keys x 128 bytes, 128B swizzle
  const int kind = std::is_same<T, __half>::value ? 1 : 2;
  const CUtensorMap tmk = tc::make_operand_map(kc, batch * Hkv * max_len, D, 2, kind, kDecTile);
  const CUtensorMap tmv = tc::make_operand_map(vc, batch * Hkv * max_len, D, 2, kind, kDecTile);
  const float scale_log2 = scale * 1.4426950408889634f;
  dim3 grid(splits, Hkv, static_cast<unsigned>(batch));
#define CT2_DEC_MMA(GV)                                                                                           \
  {                                                                                                               \
    auto kernel = attention_decode_mma_kernel<T, D, GV>;                                                          \
    allow_dynamic_smem(kernel, smem);                                                                             \
    launch_pdl(kernel, grid, dim3(kThreads), smem, st, tmk, tmv, static_cast<const T*>(qkv), static_cast<T*>(kc), \
               static_cast<T*>(vc), sn, cs, lens, H, Hkv, max_len, interleave, scale_log2, static_cast<T*>(out),  \
               partials, tickets);                                                                                \
  }
  switch (G) {
    case 1: CT2_DEC_MMA(1); break;
    case 2: CT2_DEC_MMA(2); break;
    case 4: CT2_DEC_MMA(4); break;
    case 8: CT2_DEC_MMA(8); break;
    default: return false;
  }
#undef CT2_DEC_MMA
  check_launch();
  return true;
}

}  // namespace

// fp16 / bf16, head_dim 64 or 128, no per-row lengths.  Returns false when the shape is not covered (caller falls
// back to the generic kernel in attention.cu).
bool launch_attention_prefill_mma(const void* qkv, const void* kc, const void* vc, int64_t batch, int64_t time,
                                  int64_t offset, int H, int Hkv, int D, int64_t max_len, float scale, void* out,
                                  int dtype, cudaStream_t st) {
  if (dtype == CT2B200_F32 || (D != 128 && D != 64)) return false;
  if (batch * time == 0) return true;
  if (dtype == CT2B200_F16) {
    if (D == 128) launch_mma<__half, 128>(qkv, kc, vc, batch, time, offset, H, Hkv, max_len, scale, out, st);
    else launch_mma<__half, 64>(qkv, kc, vc, batch, time, offset, H, Hkv, max_len, scale, out, st);
  } else {
    if (D == 128) launch_mma<__nv_bfloat16, 128>(qkv, kc, vc, batch, time, offset, H, Hkv, max_len, scale, out, st);
    else launch_mma<__nv_bfloat16, 64>(qkv, kc, vc, batch, time, offset, H, Hkv, max_len, scale, out, st);
  }
  return true;
}

// tensor-core decode attention; false = shape not covered (fp32, head_dim other than 64/128)
bool launch_attention_decode_mma(const void* qkv, void* kc, void* vc, const float* sn, const float* cs,
                                 const int32_t* lens, int64_t batch, int H, int Hkv, int D, int64_t max_len,
                                 bool interleave, float scale, void* out, float* partials, int32_t* tickets, int splits,
                                 int dtype, cudaStream_t st) {
  const char* e = std::getenv("CT2B200_ATTN_DECODE");
  const bool off = e && std::string(e) == "simt";
  if (off || dtype == CT2B200_F32 || (D != 128 && D != 64) || splits > 16) return false;
  if (dtype == CT2B200_F16) {
    return D == 128 ? launch_decode_mma_g<__half, 128>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, splits, st)
                    : launch_decode_mma_g<__half, 64>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, splits, st);
  }
  return D == 128 ? launch_decode_mma_g<__nv_bfloat16, 128>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, splits, st)
                  : launch_decode_mma_g<__nv_bfloat16, 64>(qkv, kc, vc, sn, cs, lens, batch, H, Hkv, max_len, interleave, scale, out, partials, tickets, splits, st);
}

// tensor-core encoder self-attention; false = shape not covered (fp32, head_dim other than 64/128)
bool launch_attention_encoder_mma(const void* qkv, const int32_t* lengths, int64_t batch, int S, int H, int D, float scale,
                                  void* out, int dtype, cudaStream_t st) {
  if (dtype == CT2B200_F32 || (D != 128 && D != 64)) return false;
  if (batch * S == 0) return true;
  if (dtype == CT2B200_F16) {
    if (D == 128) launch_encoder_mma<__half, 128>(qkv, lengths, batch, S, H, scale, out, st);
    else launch_encoder_mma<__half, 64>(qkv, lengths, batch, S, H, scale, out, st);
  } else {
    if (D == 128) launch_encoder_mma<__nv_bfloat16, 128>(qkv, lengths, batch, S, H, scale, out, st);
    else launch_encoder_mma<__nv_bfloat16, 64>(qkv, lengths, batch, S, H, scale, out, st);
  }
  return true;
}

void launch_attention_prefill(const void* qkv, const void* kc, const void* vc, const int32_t* lengths, int64_t batch,
                              int64_t time, int64_t offset, int H, int Hkv, int D, int64_t max_len, float scale,
                              void* out, int dtype, cudaStream_t st) {
  static const bool force_simple = [] {
    const char* e = std::getenv("CT2B200_ATTN_PREFILL");
    return e && std::string(e) == "simple";
  }();
  if (!force_simple && lengths == nullptr &&
      launch_attention_prefill_mma(qkv, kc, vc, batch, time, offset, H, Hkv, D, max_len, scale, out, dtype, st))
    return;
  launch_attention_prefill_simple(qkv, kc, vc, lengths, batch, time, offset, H, Hkv, D, max_len, scale, out, dtype, st);
}

}  // namespace ct2b200
