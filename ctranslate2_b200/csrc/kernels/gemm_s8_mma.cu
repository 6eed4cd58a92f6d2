// gemm_s8_mma.cu — INT8 GEMM C[m,n] = A[m,k] · B[n,k]^T (int32 accumulate) with the fused Dense
// epilogue, on legacy warp-level tensor-core instructions (mma.sync.m16n8k32.s8) with a cp.async
// multi-stage pipeline.  This is the portable fallback / cross-check of the wgmma kernel in
// gemm_tc.cu (SURVEY §0 fact 10 asks for one); the engine prefers wgmma.
//
// Replaces: cublasGemmEx(CUDA_R_8I) src/cuda/primitives.cu:571-597 + dequantize_gemm_output_kernel
// src/ops/dequantize_gpu.cu:30-121 + ops::Add / ops::Mul (src/layers/common.cc:392-401, transformer.cc:31-37).
//
// Split-K: partial int32 tiles are reduced with red.global.add.s32 into a zeroed scratch buffer; the
// last CTA of a tile (atomic ticket) runs the epilogue and re-zeroes the scratch.  Integer addition is
// associative, so the result is bit-exact whatever the arrival order.
#include "../common.cuh"
#include "gemm_common.cuh"

namespace ct2b200 {

namespace {

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  const int bytes = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void mma_s8(int32_t (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// BM x BN CTA tile, BK bytes of K per stage, WARPS_M x WARPS_N warps, kGlu: two B matrices (gate, up).
template <typename T, int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES, bool kGlu>
__global__ void __launch_bounds__(WARPS_M* WARPS_N * 32)
    gemm_s8_mma_kernel(const int8_t* __restrict__ A, const int8_t* __restrict__ B, const int8_t* __restrict__ B2,
                       int64_t M, int64_t N, int64_t K, int splits, DenseEpilogue epi, GluEpilogue glu,
                       int32_t* __restrict__ ws, int32_t* __restrict__ counters) {
  constexpr int THREADS = WARPS_M * WARPS_N * 32;
  constexpr int LDS = BK + 16;                 // padded smem row pitch (bytes): conflict-free fragment loads
  constexpr int WM = BM / WARPS_M, WN = BN / WARPS_N;
  constexpr int MT = WM / 16, NT = WN / 8;
  constexpr int NB = kGlu ? 2 : 1;
  static_assert(WM % 16 == 0 && WN % 8 == 0 && BK % 32 == 0, "bad tile");

  extern __shared__ __align__(16) uint8_t smem[];
  uint8_t* sA = smem;                                   // [STAGES][BM][LDS]
  uint8_t* sB = smem + STAGES * BM * LDS;               // [STAGES][NB][BN][LDS]
  __shared__ bool s_last;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp / WARPS_N, wn = warp % WARPS_N;
  const int g = lane >> 2, t = lane & 3;
  const int64_t m0 = static_cast<int64_t>(blockIdx.y) * BM, n0 = static_cast<int64_t>(blockIdx.x) * BN;

  // K range of this split (in BK tiles)
  const int kt_total = static_cast<int>((K + BK - 1) / BK);
  const int kt_per = (kt_total + splits - 1) / splits;
  const int kt_begin = blockIdx.z * kt_per;
  const int kt_end = min(kt_total, kt_begin + kt_per);
  const int nkt = max(0, kt_end - kt_begin);

  auto load_stage = [&](int stage, int kt) {
    const int64_t kbase = static_cast<int64_t>(kt) * BK;
    constexpr int CH = BK / 16;
    for (int c = tid; c < BM * CH; c += THREADS) {
      const int r = c / CH, ch = c % CH;
      const int64_t row = m0 + r, kk = kbase + ch * 16;
      const bool ok = row < M && kk < K;
      cp_async16(sA + (stage * BM + r) * LDS + ch * 16, A + (ok ? row * K + kk : 0), ok);
    }
#pragma unroll
    for (int bsel = 0; bsel < NB; ++bsel) {
      const int8_t* Bp = bsel == 0 ? B : B2;
      for (int c = tid; c < BN * CH; c += THREADS) {
        const int r = c / CH, ch = c % CH;
        const int64_t row = n0 + r, kk = kbase + ch * 16;
        const bool ok = row < N && kk < K;
        cp_async16(sB + ((stage * NB + bsel) * BN + r) * LDS + ch * 16, Bp + (ok ? row * K + kk : 0), ok);
      }
    }
  };

  int32_t acc[NB][MT][NT][4];
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[b][i][j][r] = 0;

  // prologue
#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nkt) load_stage(s, kt_begin + s);
    cp_async_commit();
  }

  for (int it = 0; it < nkt; ++it) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    {  // prefetch tile it+STAGES-1 into the slot freed at iteration it-1
      const int nx = it + STAGES - 1;
      if (nx < nkt) load_stage(nx % STAGES, kt_begin + nx);
      cp_async_commit();
    }
    const int stage = it % STAGES;
    const uint8_t* a_s = sA + stage * BM * LDS;
#pragma unroll
    for (int kk = 0; kk < BK; kk += 32) {
      uint32_t af[MT][4];
#pragma unroll
      for (int i = 0; i < MT; ++i) {
        const uint8_t* p = a_s + (wm * WM + i * 16 + g) * LDS + kk + 4 * t;
        af[i][0] = *reinterpret_cast<const uint32_t*>(p);
        af[i][1] = *reinterpret_cast<const uint32_t*>(p + 8 * LDS);
        af[i][2] = *reinterpret_cast<const uint32_t*>(p + 16);
        af[i][3] = *reinterpret_cast<const uint32_t*>(p + 8 * LDS + 16);
      }
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const uint8_t* b_s = sB + (stage * NB + b) * BN * LDS;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          const uint8_t* p = b_s + (wn * WN + j * 8 + g) * LDS + kk + 4 * t;
          uint32_t bf[2] = {*reinterpret_cast<const uint32_t*>(p), *reinterpret_cast<const uint32_t*>(p + 16)};
#pragma unroll
          for (int i = 0; i < MT; ++i) mma_s8(acc[b][i][j], af[i], bf);
        }
      }
    }
  }
  cp_async_wait<0>();

  // ---- epilogue ----
  auto for_each_acc = [&](auto&& f) {
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int64_t row = m0 + wm * WM + i * 16 + g + (r >= 2 ? 8 : 0);
          const int64_t col = n0 + wn * WN + j * 8 + 2 * t + (r & 1);
          if (row < M && col < N) f(i, j, r, row, col);
        }
  };

  if (splits == 1) {
    for_each_acc([&](int i, int j, int r, int64_t row, int64_t col) {
      if constexpr (kGlu) glu_epilogue_store<T>(glu, acc[0][i][j][r], acc[NB - 1][i][j][r], row, col);
      else dense_epilogue_store<T>(epi, acc[0][i][j][r], row, col);
    });
    return;
  }

  const int64_t plane = M * N;
  for_each_acc([&](int i, int j, int r, int64_t row, int64_t col) {
    atomicAdd(ws + row * N + col, acc[0][i][j][r]);
    if constexpr (kGlu) atomicAdd(ws + plane + row * N + col, acc[NB - 1][i][j][r]);
  });
  __threadfence();
  __syncthreads();
  const int tile_id = blockIdx.y * gridDim.x + blockIdx.x;
  if (tid == 0) s_last = atomicAdd(counters + tile_id, 1) == splits - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int e = tid; e < BM * BN; e += THREADS) {
    const int64_t row = m0 + e / BN, col = n0 + e % BN;
    if (row >= M || col >= N) continue;
    const int32_t v = __ldcg(ws + row * N + col);
    ws[row * N + col] = 0;
    if constexpr (kGlu) {
      const int32_t v2 = __ldcg(ws + plane + row * N + col);
      ws[plane + row * N + col] = 0;
      glu_epilogue_store<T>(glu, v, v2, row, col);
    } else {
      dense_epilogue_store<T>(epi, v, row, col);
    }
  }
  if (tid == 0) counters[tile_id] = 0;
}

template <typename T, int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES, bool kGlu>
void launch_cfg(const int8_t* A, const int8_t* B, const int8_t* B2, int64_t M, int64_t N, int64_t K,
                const DenseEpilogue& epi, const GluEpilogue& glu, cudaStream_t st) {
  constexpr int NB = kGlu ? 2 : 1;
  constexpr int LDS = BK + 16;
  constexpr size_t smem = static_cast<size_t>(STAGES) * (BM + NB * BN) * LDS;
  auto kernel = gemm_s8_mma_kernel<T, BM, BN, BK, WARPS_M, WARPS_N, STAGES, kGlu>;
  allow_dynamic_smem(kernel, smem);
  const int tiles_m = div_up(M, BM), tiles_n = div_up(N, BN);
  const int kt_total = div_up(K, BK);
  SplitKWorkspace& w = SplitKWorkspace::get(st);
  int splits = choose_splits(tiles_m * tiles_n, kt_total, M * N * NB, w);
  dim3 grid(tiles_n, tiles_m, splits);
  kernel<<<grid, WARPS_M * WARPS_N * 32, smem, st>>>(A, B, B2, M, N, K, splits, epi, glu, w.accum, w.counters);
  check_launch();
}

template <typename T, bool kGlu>
void launch_shape(const int8_t* A, const int8_t* B, const int8_t* B2, int64_t M, int64_t N, int64_t K,
                  const DenseEpilogue& epi, const GluEpilogue& glu, cudaStream_t st) {
  if (M <= 16) launch_cfg<T, 16, 64, 128, 1, 8, 5, kGlu>(A, B, B2, M, N, K, epi, glu, st);
  else if (M <= 32) launch_cfg<T, 32, 64, 128, 1, 8, 5, kGlu>(A, B, B2, M, N, K, epi, glu, st);
  else if (M <= 64) launch_cfg<T, 64, 64, 64, 2, 4, 4, kGlu>(A, B, B2, M, N, K, epi, glu, st);
  else launch_cfg<T, 128, 128, 64, 2, 4, 4, kGlu>(A, B, B2, M, N, K, epi, glu, st);
}

}  // namespace

void gemm_s8_mma(const int8_t* A, const int8_t* B, int64_t M, int64_t N, int64_t K, const DenseEpilogue& epi,
                 int dtype, cudaStream_t st) {
  if (M == 0 || N == 0) return;
  CT2_REQUIRE(K % 16 == 0, "gemm_s8: k must be a multiple of 16");
  GluEpilogue glu{};
  CT2_DISPATCH_DTYPE(dtype, (launch_shape<T, false>(A, B, nullptr, M, N, K, epi, glu, st)));
}

void gemm_s8_glu_mma(const int8_t* A, const int8_t* Bgate, const int8_t* Bup, int64_t M, int64_t N, int64_t K,
                     const GluEpilogue& glu, int dtype, cudaStream_t st) {
  if (M == 0 || N == 0) return;
  CT2_REQUIRE(K % 16 == 0, "gemm_s8: k must be a multiple of 16");
  DenseEpilogue epi{};
  CT2_DISPATCH_DTYPE(dtype, (launch_shape<T, true>(A, Bgate, Bup, M, N, K, epi, glu, st)));
}

}  // namespace ct2b200
