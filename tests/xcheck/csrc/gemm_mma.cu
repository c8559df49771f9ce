// Legacy-tensor-core (mma.sync m16n8k16) bf16 GEMM with the same contract as gemm_tc() (csrc/gemm_wgmma.cu).
// TEST-ONLY: an independent on-device cross-check for the product's wgmma kernel (tests compare the two).  Built into
// tests/xcheck/libmuse_b200_xcheck.so, never into libmuse_b200.so.
#include "common.cuh"

namespace muse {
namespace {

constexpr int TM = 64, TN = 64, TK = 32;
constexpr int LDS = TK + 8;  // padded smem row (elements): 80 B stride -> conflict-free 32-bit fragment loads

enum Epi { EPI_BF16 = 0, EPI_F32 = 1, EPI_ATOMIC_F32 = 2, EPI_RESADD_F32 = 3 };

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// Loads a [TILE x TK] operand tile into smem as s[mn][k] from either major-ness, zero-filling OOB.
template <int TILE>
__device__ __forceinline__ void load_tile(bf16* s, const bf16* g, int mn0, int k0, int MN, int K, int ld, bool mn_major) {
  const bf16 zero = __float2bfloat16(0.f);
  for (int i = threadIdx.x; i < TILE * TK; i += blockDim.x) {
    int mn, k;
    if (!mn_major) { mn = i / TK; k = i % TK; } else { k = i / TILE; mn = i % TILE; }
    const int gmn = mn0 + mn, gk = k0 + k;
    bf16 v = zero;
    if (gmn < MN && gk < K) v = mn_major ? g[static_cast<size_t>(gk) * ld + gmn] : g[static_cast<size_t>(gmn) * ld + gk];
    s[mn * LDS + k] = v;
  }
}

template <int EPI>
__global__ void __launch_bounds__(128)
gemm_mma_kernel(const bf16* __restrict__ A, const bf16* __restrict__ B, void* C, const float* __restrict__ res, int M,
                int N, int K, int lda, int ldb, int ldc, int a_mn, int b_mn, int k_per_split) {
  __shared__ __align__(16) bf16 sA[TM * LDS];
  __shared__ __align__(16) bf16 sB[TN * LDS];
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  const int kbeg = blockIdx.z * k_per_split;
  const int kend = min(K, kbeg + k_per_split);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  const int g = lane >> 2, t = lane & 3;
  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

  for (int k0 = kbeg; k0 < kend; k0 += TK) {
    load_tile<TM>(sA, A, m0, k0, M, kend, lda, a_mn != 0);
    load_tile<TN>(sB, B, n0, k0, N, kend, ldb, b_mn != 0);
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TK; kk += 16) {
      uint32_t af[2][4], bfr[4][2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const bf16* base = sA + (wm + i * 16) * LDS + kk;
        af[i][0] = *reinterpret_cast<const uint32_t*>(base + (g)*LDS + 2 * t);
        af[i][1] = *reinterpret_cast<const uint32_t*>(base + (g + 8) * LDS + 2 * t);
        af[i][2] = *reinterpret_cast<const uint32_t*>(base + (g)*LDS + 2 * t + 8);
        af[i][3] = *reinterpret_cast<const uint32_t*>(base + (g + 8) * LDS + 2 * t + 8);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const bf16* base = sB + (wn + j * 8 + g) * LDS + kk;
        bfr[j][0] = *reinterpret_cast<const uint32_t*>(base + 2 * t);
        bfr[j][1] = *reinterpret_cast<const uint32_t*>(base + 2 * t + 8);
      }
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) mma16816(acc[i][j], af[i], bfr[j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int row = m0 + wm + i * 16 + g + (q >> 1) * 8;
        const int col = n0 + wn + j * 8 + 2 * t + (q & 1);
        if (row < M && col < N) {
          const size_t off = static_cast<size_t>(row) * ldc + col;
          const float v = acc[i][j][q];
          if (EPI == EPI_BF16) reinterpret_cast<bf16*>(C)[off] = __float2bfloat16_rn(v);
          else if (EPI == EPI_F32) reinterpret_cast<float*>(C)[off] = v;
          else if (EPI == EPI_ATOMIC_F32) atomicAdd(reinterpret_cast<float*>(C) + off, v);
          else reinterpret_cast<float*>(C)[off] = res[off] + bf16_round(v);
        }
      }
}

}  // namespace

int gemm_mma(const void* A, const void* B, void* C, const float* res, int M, int N, int K, int lda, int ldb, int ldc,
             int a_mn, int b_mn, int epi, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return MUSE_OK;
  int splits = 1;
  int k_per_split = K;
  if (epi == EPI_ATOMIC_F32) {
    const int tiles = ceil_div(M, TM) * ceil_div(N, TN);
    splits = 592 / tiles;
    if (splits < 1) splits = 1;
    k_per_split = ceil_div(ceil_div(K, splits), TK) * TK;
    splits = ceil_div(K, k_per_split);
  }
  dim3 grid(ceil_div(N, TN), ceil_div(M, TM), splits);
  const bf16* a = reinterpret_cast<const bf16*>(A);
  const bf16* b = reinterpret_cast<const bf16*>(B);
  switch (epi) {
    case EPI_BF16: gemm_mma_kernel<EPI_BF16><<<grid, 128, 0, stream>>>(a, b, C, res, M, N, K, lda, ldb, ldc, a_mn, b_mn, k_per_split); break;
    case EPI_F32: gemm_mma_kernel<EPI_F32><<<grid, 128, 0, stream>>>(a, b, C, res, M, N, K, lda, ldb, ldc, a_mn, b_mn, k_per_split); break;
    case EPI_ATOMIC_F32: gemm_mma_kernel<EPI_ATOMIC_F32><<<grid, 128, 0, stream>>>(a, b, C, res, M, N, K, lda, ldb, ldc, a_mn, b_mn, k_per_split); break;
    case EPI_RESADD_F32: gemm_mma_kernel<EPI_RESADD_F32><<<grid, 128, 0, stream>>>(a, b, C, res, M, N, K, lda, ldb, ldc, a_mn, b_mn, k_per_split); break;
    default: set_last_error("gemm_mma: unknown epilogue %d", epi); return MUSE_ERR_INVALID;
  }
  return check_launch("gemm_mma");
}

}  // namespace muse
