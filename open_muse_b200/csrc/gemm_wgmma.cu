// bf16 GEMM on the Hopper tensor cores: C[M,N] = A[M,K] * B[N,K]^T, fp32 accumulation in registers (wgmma).
//
// This is the kernel every nn.Linear of the reference's transformer maps to
// (muse/modeling_transformer.py:198-200,218 q/k/v/out; :789-798 wi_0/wi_1/wo; :980,984 mlm head)
// and, with transposed operand views, their dgrad / wgrad in backward.
//
// Structure: the persistent warp-specialised pipeline of tc_pipeline.cuh.  The producer thread loads 2-D TMA tiles of A
// and B; each consumer warpgroup converts its 64-row half of the accumulator in 128-byte column chunks into two
// double-buffered shared-memory staging buffers and stores them with TMA (bf16 / fp32 / +residual / split-K partial; the
// fp32 residual arrives by TMA into the same buffers ahead of use).  The stores are asynchronous, so they drain while the
// warpgroup's next tile runs its MMAs; the producer runs up to a ring's worth of k-blocks ahead, so it keeps loading the
// next tile meanwhile.  The atomic epilogue adds straight from the accumulator registers.
//
// FP8 (muse_gemm_fp8, inference): A and B e4m3, both K-major, with fp32 scales per row of A and per row of B (= column
// of C); the same pipeline with k32 e4m3 MMAs, and the bf16 epilogue stores bf16(acc * sa[m] * sb[n]).  muse_gemm_fp8_res
// stores res + bf16(acc * sa[m] * sb[n]) in fp32 instead, with the residual prefetch and TMA stores of EPI_RESADD_F32.
//
// Operand "major-ness": an operand is K-major when the reduction dim is contiguous in memory
// (activations X[T,K], weights W[N,K] in forward) and MN-major when the M/N dim is contiguous
// (W[N,K] used as the B operand of dgrad; dY[T,N] and X[T,K] as operands of wgrad, where the
// reduction runs over T). Both are fed straight from their row-major tensors through TMA; the
// smem (matrix) descriptors and the wgmma transpose flags tell the tensor core which layout it is looking at, so no
// transposes are materialised anywhere in the training step.
#include "common.cuh"
#include "tc_host.cuh"
#include "tc_pipeline.cuh"

namespace muse {

namespace {

using tc::BK;
using tc::BM;

// EPI_SPLITK_F32: deterministic split-K.  Every split stores its fp32 partial tile into a workspace and a second, fully
// parallel kernel sums the partials in split order and STORES the result, so the output needs no zero fill and is
// bit-identical from run to run (the atomic variant is order-dependent).
// EPI_FP8_BF16: e4m3 operands (muse_gemm_fp8 only), C bf16 = acc * sa[row] * sb[col].
// EPI_FP8_RESADD_F32: e4m3 operands (muse_gemm_fp8_res only), C fp32 = res + bf16(acc * sa[row] * sb[col]).
enum Epi {
  EPI_BF16 = 0, EPI_F32 = 1, EPI_ATOMIC_F32 = 2, EPI_RESADD_F32 = 3, EPI_SPLITK_F32 = 4, EPI_FP8_BF16 = 5,
  EPI_FP8_RESADD_F32 = 6
};


// Epilogue staging buffer: 64 rows x 128 B (a chunk of 64 bf16 or 32 fp32 columns of a warpgroup's half tile), laid out
// with the 128-byte swizzle of the output tensor map.  Two per consumer warpgroup, then one mbarrier per buffer for the
// residual loads of EPI_RESADD_F32.
constexpr int kEpiBuf = 64 * 128;

template <int BN, typename T = bf16>
using Ring = tc::Ring<BN, (BN == 256) ? 4 : 6, 4 * kEpiBuf + 4 * 8, T>;

struct GemmParams {
  void* C;  // EPI_ATOMIC_F32 only; the other epilogues store through the output tensor map
  int M, N, K;
  int ldc;
  int num_m, num_n, num_kb, kb_per_split, splits;
  const float* sa;  // FP8 epilogues: scales of the rows of A [M] and of B [N]
  const float* sb;
};

// tmC: the output, box {128 B of columns, 64 rows}: C [M, N] (pitch ldc), or for split-K partial tiles the workspace
// [splits * num_m * num_n * BM, BN] fp32.  tmR: the fp32 residual [M, N] (pitch ldc) of the residual epilogues, same box.
template <int BN, bool A_MN, bool B_MN, int EPI>
__global__ void __launch_bounds__(tc::kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR, const GemmParams p) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  constexpr bool kFp8 = EPI == EPI_FP8_BF16 || EPI == EPI_FP8_RESADD_F32;
  constexpr bool kRes = EPI == EPI_RESADD_F32 || EPI == EPI_FP8_RESADD_F32;
  using R = Ring<BN, std::conditional_t<kFp8, __nv_fp8_e4m3, bf16>>;
  constexpr int kBK = R::kBK;
  R ring(smem_raw);

  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
    if (EPI != EPI_ATOMIC_F32) ptx::prefetch_tmap(&tmC);
    if (kRes) {
      ptx::prefetch_tmap(&tmR);
      uint64_t* rbar = reinterpret_cast<uint64_t*>(ring.extra() + 4 * kEpiBuf);
      for (int i = 0; i < 4; ++i) ptx::mbar_init(&rbar[i], 1);
    }
    ring.init();  // ends with the barrier-init fence
  }
  __syncthreads();
  pdl_wait();  // everything above touches only shared memory / kernel parameters

  const int tiles_mn = p.num_m * p.num_n;
  const int total_tiles = tiles_mn * p.splits;

  if (wg == 0) {
    ptx::setmaxnreg_dec<tc::kProducerRegs>();
    if (threadIdx.x == 0) {
      // ------------------------------------------------------------ TMA producer
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n_idx = tile % p.num_n;
        const int m_idx = (tile / p.num_n) % p.num_m;
        const int split = tile / tiles_mn;
        const int kb0 = split * p.kb_per_split;
        const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);
        const int m0 = m_idx * BM, n0 = n_idx * BN;
        for (int kb = kb0; kb < kb1; ++kb) {
          const auto s = ring.produce();
          if (!A_MN) {
            ptx::tma_load_2d(s.a, &tmA, s.bar, kb * kBK, m0);
          } else {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)
              ptx::tma_load_2d(s.a + i * (BK * 128), &tmA, s.bar, m0 + i * 64, kb * BK);
          }
          if (!B_MN) {
            ptx::tma_load_2d(s.b, &tmB, s.bar, kb * kBK, n0);
          } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)
              ptx::tma_load_2d(s.b + i * (BK * 128), &tmB, s.bar, n0 + i * 64, kb * BK);
          }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<tc::kConsumerRegs>();
    // -------------------------------------------------------------- consumers: rows [64 * half, 64 * half + 64) of a tile
    const int half = wg - 1;
    const bool leader = (threadIdx.x & 127) == 0;  // issues the warpgroup's bulk copies
    const int fr = ptx::frag_row();                 // half-local row of d[4j], d[4j+1]; +8 for d[4j+2..3]
    const int lc = ptx::frag_col();                 // tile-local column of d[4j] within its 8-column group
    uint8_t* ebuf = ring.extra() + half * 2 * kEpiBuf;  // this warpgroup's two staging buffers
    uint64_t* rbar = reinterpret_cast<uint64_t*>(ring.extra() + 4 * kEpiBuf) + 2 * half;
    // A chunk is 128 B of each of the 64 rows; chunk q goes through buffer q & 1.  Every epilogue has an even number of
    // chunks per tile, so each tile starts on buffer 0 and the residual barriers on phase 0.
    constexpr bool kF32 = EPI != EPI_BF16 && EPI != EPI_FP8_BF16;
    constexpr int kCols = kF32 ? 32 : 64;
    constexpr int kChunks = BN / kCols;
    constexpr int kJ = kCols / 8;  // 8-column fragment groups per chunk
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int n_idx = tile % p.num_n;
      const int m_idx = (tile / p.num_n) % p.num_m;
      const int split = tile / tiles_mn;
      const int kb0 = split * p.kb_per_split;
      const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);
      // output coordinates of this warpgroup's half; the split-K partial of `tile` is workspace rows [BM tile, BM tile + BM)
      const bool partial = EPI == EPI_SPLITK_F32 && p.splits > 1;
      const int orow = (partial ? tile * BM : m_idx * BM) + half * 64;
      const int ocol = partial ? 0 : n_idx * BN;
      if (kRes && leader) {
        // the first two residual chunks load during the mainloop, once the previous tile's stores have read the buffers
        ptx::bulk_wait_read<0>();
        for (int b = 0; b < 2; ++b) {
          ptx::mbar_expect_tx(&rbar[b], kEpiBuf);
          ptx::tma_load_2d(ebuf + b * kEpiBuf, &tmR, &rbar[b], ocol + b * kCols, orow);
        }
      }
      if constexpr (kFp8) {
        // the e4m3 MMA keeps fewer accumulator bits than fp32: each k-block's partial sum is promoted into the fp32
        // registers of acc (DESIGN.md section 4 has the measurement with and without)
        float part[BN / 2];
        ring.consume_promoted(acc, part, kb0, kb1, half);
      } else {
        ring.template consume<A_MN, B_MN>(acc, kb0, kb1, half);
      }
      float sx[2] = {1.f, 1.f};  // FP8 epilogues: scales of the thread's rows fr and fr + 8 (0 past M)
      if constexpr (kFp8) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int grow = orow + fr + 8 * hr;
          sx[hr] = grow < p.M ? p.sa[grow] : 0.f;
        }
      }
      if constexpr (EPI == EPI_ATOMIC_F32) {
        // ---------------------------------------------------------- fp32 atomics straight from the accumulator registers
        const int lr = half * 64 + fr;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const float v0 = acc[4 * j + 2 * hr], v1 = acc[4 * j + 2 * hr + 1];
            const int grow = m_idx * BM + lr + 8 * hr, gcol = n_idx * BN + 8 * j + lc;
            if (grow >= p.M || gcol >= p.N) continue;
            float* dst = reinterpret_cast<float*>(p.C) + static_cast<size_t>(grow) * p.ldc + gcol;
            if (gcol + 1 < p.N) atomicAdd(reinterpret_cast<float2*>(dst), make_float2(v0, v1));
            else atomicAdd(dst, v0);
          }
        }
      } else {
        // ---------------------------------------------------------- chunks through shared memory, TMA stores
#pragma unroll
        for (int q = 0; q < kChunks; ++q) {
          uint8_t* buf = ebuf + (q & 1) * kEpiBuf;
          if (kRes) {
            ptx::mbar_wait(&rbar[q & 1], (q >> 1) & 1);  // residual chunk q has landed (so the store of q - 2 has read buf)
          } else {
            if (leader) ptx::bulk_wait_read<1>();  // the store of chunk q - 2 has read buf
            ptx::named_barrier_sync(1 + half, 128);
          }
#pragma unroll
          for (int jj = 0; jj < kJ; ++jj) {
            const int j = q * kJ + jj;
            float2 sw = make_float2(1.f, 1.f);  // FP8 epilogues: scales of columns lc, lc + 1 of this 8-column group
            if constexpr (kFp8) {
              const int gcol = ocol + q * kCols + 8 * jj + lc;  // N % 8 == 0: both columns are inside or both past N
              sw = gcol < p.N ? *reinterpret_cast<const float2*>(p.sb + gcol) : make_float2(0.f, 0.f);
            }
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              float v0 = acc[4 * j + 2 * hr], v1 = acc[4 * j + 2 * hr + 1];
              if constexpr (kFp8) {
                v0 = v0 * sx[hr] * sw.x;
                v1 = v1 * sx[hr] * sw.y;
              }
              const int r = fr + 8 * hr;
              // 16-byte unit u of row r sits at unit u ^ (r & 7): the 128-byte swizzle, so the 8 rows of a warp's store
              // fall into different banks
              if (!kF32) {
                *reinterpret_cast<uint32_t*>(buf + r * 128 + ((jj ^ (r & 7)) << 4) + 2 * lc) = pack_bf16(v0, v1);
              } else {
                float2* dst = reinterpret_cast<float2*>(buf + r * 128 + (((2 * jj + (lc >> 2)) ^ (r & 7)) << 4) + 4 * (lc & 3));
                if (kRes) {  // out = residual + bf16(acc)  (Linear output is bf16 under autocast)
                  const float2 rs = *dst;
                  *dst = make_float2(rs.x + bf16_round(v0), rs.y + bf16_round(v1));
                } else {
                  *dst = make_float2(v0, v1);
                }
              }
            }
          }
          ptx::fence_proxy_async();  // the chunk is visible to the TMA unit
          ptx::named_barrier_sync(1 + half, 128);
          if (leader) {
            ptx::tma_store_2d(&tmC, buf, ocol + q * kCols, orow);
            ptx::bulk_commit();
            if (kRes && q + 2 < kChunks) {
              ptx::bulk_wait_read<0>();
              ptx::mbar_expect_tx(&rbar[q & 1], kEpiBuf);
              ptx::tma_load_2d(buf, &tmR, &rbar[q & 1], ocol + (q + 2) * kCols, orow);
            }
          }
        }
      }
    }
    if (leader) ptx::bulk_wait<0>();  // shared memory must outlive the last stores
  }
}

// C[r][c..c+3] = sum over splits (ascending) of the partial tiles; one thread per float4 of the output
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ ws, float* __restrict__ C, int M, int N, int ldc, int num_n, int tiles_mn,
                     int bn, int splits) {
  pdl_enter();
  const int n4 = (N + 3) >> 2;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= static_cast<long long>(M) * n4) return;
  const int r = static_cast<int>(idx / n4), c = static_cast<int>(idx % n4) * 4;
  const int tile = (r / BM) * num_n + c / bn;
  const float* src = ws + static_cast<size_t>(tile) * (BM * bn) + static_cast<size_t>(r % BM) * bn + (c % bn);
  const size_t stride = static_cast<size_t>(tiles_mn) * (BM * bn);
  float4 a = *reinterpret_cast<const float4*>(src);
  for (int sp = 1; sp < splits; ++sp) {
    const float4 b = *reinterpret_cast<const float4*>(src + sp * stride);
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
  }
  float* dst = C + static_cast<size_t>(r) * ldc + c;
  if (c + 4 <= N) *reinterpret_cast<float4*>(dst) = a;
  else { const float f[4] = {a.x, a.y, a.z, a.w}; for (int k = 0; k < 4 && c + k < N; ++k) dst[k] = f[k]; }
}

// ------------------------------------------------------------------ host side
int g_reserved_sms = 0;  // SMs left free for concurrently running collective kernels (set_reserved_sms)
int num_sms() {
  const int n = sm_count() - g_reserved_sms;
  return n > 16 ? n : 16;
}

// A, B, the output and the residual (EPI_RESADD_F32; a copy of the output map otherwise)
struct GemmMaps {
  CUtensorMap a, b, c, r;
};

template <int BN, bool A_MN, bool B_MN, int EPI>
int launch(const GemmMaps& m, const GemmParams& p, cudaStream_t stream) {
  constexpr auto kern = gemm_wgmma_kernel<BN, A_MN, B_MN, EPI>;
  constexpr int kSmem = Ring<BN>::kSmemBytes;  // the same for both operand types
  if (int rc = set_max_dynamic_smem<kern>(kSmem)) return rc;
  const int total = p.num_m * p.num_n * p.splits;
  const int grid = total < num_sms() ? total : num_sms();
  pdl_launch(grid, tc::kThreads, kSmem, stream)(kern, m.a, m.b, m.c, m.r, p);
  return check_launch("gemm_wgmma");
}

template <int BN, bool A_MN, bool B_MN>
int launch_epi(int epi, const GemmMaps& m, const GemmParams& p, cudaStream_t s) {
  switch (epi) {
    case EPI_BF16: return launch<BN, A_MN, B_MN, EPI_BF16>(m, p, s);
    case EPI_F32: return launch<BN, A_MN, B_MN, EPI_F32>(m, p, s);
    case EPI_ATOMIC_F32: return launch<BN, A_MN, B_MN, EPI_ATOMIC_F32>(m, p, s);
    case EPI_RESADD_F32: return launch<BN, A_MN, B_MN, EPI_RESADD_F32>(m, p, s);
    case EPI_SPLITK_F32: return launch<BN, A_MN, B_MN, EPI_SPLITK_F32>(m, p, s);
  }
  set_last_error("gemm: unknown epilogue %d", epi);
  return MUSE_ERR_INVALID;
}

template <int BN>
int launch_major(int a_mn, int b_mn, int epi, const GemmMaps& m, const GemmParams& p, cudaStream_t s) {
  if (!a_mn && !b_mn) return launch_epi<BN, false, false>(epi, m, p, s);
  if (!a_mn && b_mn) return launch_epi<BN, false, true>(epi, m, p, s);
  if (a_mn && b_mn) return launch_epi<BN, true, true>(epi, m, p, s);
  return launch_epi<BN, true, false>(epi, m, p, s);
}

}  // namespace

// C[M,N] (ldc) = op(A) * op(B)^T with op selected by a_mn / b_mn:
//   a_mn == 0: A points at a row-major [M, K] matrix (pitch lda);  a_mn == 1: at a row-major [K, M] matrix.
//   b_mn == 0: B points at a row-major [N, K] matrix (pitch ldb);  b_mn == 1: at a row-major [K, N] matrix.
// Split plan shared by the launcher and the workspace query: how many K splits a weight-gradient GEMM (few output tiles,
// very long K = tokens) needs to fill the SMs.
static void split_plan(int M, int N, int K, int* num_m, int* num_n, int* num_kb, int* kb_per_split, int* splits, int* bn) {
  *bn = (N >= 256) ? 256 : 128;
  *num_m = ceil_div(M, BM);
  *num_n = ceil_div(N, *bn);
  *num_kb = ceil_div(K, BK);
  const int tiles = *num_m * *num_n;
  int want = num_sms() / tiles;
  if (want < 1) want = 1;
  if (want > *num_kb) want = *num_kb;
  *kb_per_split = ceil_div(*num_kb, want);
  *splits = ceil_div(*num_kb, *kb_per_split);
}

static int gemm_tc(const void* A, const void* B, void* C, const float* res, int M, int N, int K, int lda, int ldb,
                   int ldc, int a_mn, int b_mn, int epi, cudaStream_t stream, void* ws, long long ws_bytes) {
  if (M <= 0 || N <= 0 || K <= 0) return MUSE_OK;
  if (epi == EPI_BF16 ? (ldc % 8 != 0) : (ldc % 4 != 0)) {
    set_last_error("gemm: ldc=%d must be a multiple of %d", ldc, epi == EPI_BF16 ? 8 : 4);
    return MUSE_ERR_INVALID;
  }
  // The TMA-store epilogues do not clip a partial 16-byte unit at column N: they would overwrite the pad columns of that
  // unit (N = 2025 into ldc = 2048 zeroes columns 2025..).  Only the atomic epilogue, which stores per element, takes any N.
  if (epi != EPI_ATOMIC_F32 && N % (epi == EPI_BF16 ? 8 : 4) != 0) {
    set_last_error("gemm: N=%d must be a multiple of %d for this epilogue (its TMA stores write whole 16-byte units)", N,
                   epi == EPI_BF16 ? 8 : 4);
    return MUSE_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(C) & 15) != 0) {
    set_last_error("gemm: C must be 16B aligned");
    return MUSE_ERR_INVALID;
  }
  if (epi == EPI_RESADD_F32 && (res == nullptr || (reinterpret_cast<uintptr_t>(res) & 15) != 0)) {
    set_last_error("gemm: the residual epilogue needs a 16B-aligned residual");
    return MUSE_ERR_INVALID;
  }
  const int BN = (N >= 256) ? 256 : 128;
  constexpr CUtensorMapDataType kBf16 = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, kF32 = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  // K-major operands: boxes of BK columns x the tile's rows; MN-major: 64-column chunks x BK rows
  GemmMaps m;
  int rc;
  rc = a_mn ? make_tmap(&m.a, "gemm", kBf16, A, {M, K}, {2LL * lda}, {64, BK})
            : make_tmap(&m.a, "gemm", kBf16, A, {K, M}, {2LL * lda}, {BK, BM});
  if (rc) return rc;
  rc = b_mn ? make_tmap(&m.b, "gemm", kBf16, B, {N, K}, {2LL * ldb}, {64, BK})
            : make_tmap(&m.b, "gemm", kBf16, B, {K, N}, {2LL * ldb}, {BK, BN});
  if (rc) return rc;

  GemmParams p;
  p.C = C;
  p.M = M; p.N = N; p.K = K; p.ldc = ldc;
  p.num_m = ceil_div(M, BM);
  p.num_n = ceil_div(N, BN);
  p.num_kb = ceil_div(K, BK);
  p.splits = 1;
  p.kb_per_split = p.num_kb;
  p.sa = p.sb = nullptr;
  if (epi == EPI_ATOMIC_F32 || epi == EPI_SPLITK_F32) {
    int num_m, num_n, num_kb, bn;
    split_plan(M, N, K, &num_m, &num_n, &num_kb, &p.kb_per_split, &p.splits, &bn);
    if (epi == EPI_SPLITK_F32 && p.splits > 1) {
      const long long need = static_cast<long long>(p.splits) * p.num_m * p.num_n * BM * BN * 4;
      if (ws == nullptr || ws_bytes < need || (reinterpret_cast<uintptr_t>(ws) & 15) != 0) {
        set_last_error("gemm: deterministic split-K needs a 16B-aligned workspace of %lld bytes (got %lld)", need, ws_bytes);
        return MUSE_ERR_INVALID;
      }
    }
  }
  // The output map clips at M and N, so rows past M, pad columns (ldc > N) and the neighbours of a column slice of a
  // wider tensor are never written.  Boxes are 128 B of columns x the 64 rows of a consumer warpgroup.
  if (epi == EPI_SPLITK_F32 && p.splits > 1)
    rc = make_tmap(&m.c, "gemm", kF32, ws, {BN, 1LL * p.splits * p.num_m * p.num_n * BM}, {4LL * BN}, {32, 64});
  else if (epi == EPI_BF16)
    rc = make_tmap(&m.c, "gemm", kBf16, C, {N, M}, {2LL * ldc}, {64, 64});
  else
    rc = make_tmap(&m.c, "gemm", kF32, C, {N, M}, {4LL * ldc}, {32, 64});
  if (rc) return rc;
  m.r = m.c;
  if (epi == EPI_RESADD_F32 && (rc = make_tmap(&m.r, "gemm", kF32, res, {N, M}, {4LL * ldc}, {32, 64}))) return rc;
  rc = (BN == 256) ? launch_major<256>(a_mn, b_mn, epi, m, p, stream) : launch_major<128>(a_mn, b_mn, epi, m, p, stream);
  if (rc || epi != EPI_SPLITK_F32 || p.splits <= 1) return rc;
  const long long n_out4 = static_cast<long long>(M) * ((N + 3) / 4);
  pdl_launch(static_cast<unsigned>(ceil_div_ll(n_out4, 256)), 256, 0, stream)(splitk_reduce_kernel,
      reinterpret_cast<const float*>(ws), reinterpret_cast<float*>(C), M, N, ldc, p.num_n, p.num_m * p.num_n, BN, p.splits);
  return check_launch("gemm splitk reduce");
}

// C bf16 [M,N] (ldc) = (A e4m3 [M,K] (lda) * diag(sa)) (B e4m3 [N,K] (ldb) * diag(sb))^T; pitches in elements = bytes.
// res given: C fp32 [M,N] (ldc) = res (ldc) + bf16(that product).
static int gemm_fp8(const void* A, const float* sa, const void* B, const float* sb, const float* res, void* C, int M, int N,
                    int K, int lda, int ldb, int ldc, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return MUSE_OK;
  if (res != nullptr && (reinterpret_cast<uintptr_t>(res) & 15) != 0) {
    set_last_error("gemm_fp8: the residual must be 16B aligned");
    return MUSE_ERR_INVALID;
  }
  if (ldc % 8 != 0 || N % 8 != 0) {
    set_last_error("gemm_fp8: N=%d and ldc=%d must be multiples of 8 (the TMA stores write whole 16-byte units)", N, ldc);
    return MUSE_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(C) & 15) != 0 || sa == nullptr || sb == nullptr ||
      (reinterpret_cast<uintptr_t>(sb) & 7) != 0) {
    set_last_error("gemm_fp8: C must be 16B aligned and the scales given, sb 8B aligned");
    return MUSE_ERR_INVALID;
  }
  constexpr int BN = 128;
  constexpr int kBK = Ring<BN, __nv_fp8_e4m3>::kBK;
  GemmMaps m;
  int rc;
  if ((rc = make_tmap(&m.a, "gemm_fp8", CU_TENSOR_MAP_DATA_TYPE_UINT8, A, {K, M}, {1LL * lda}, {kBK, BM}))) return rc;
  if ((rc = make_tmap(&m.b, "gemm_fp8", CU_TENSOR_MAP_DATA_TYPE_UINT8, B, {K, N}, {1LL * ldb}, {kBK, BN}))) return rc;
  if (res == nullptr) {
    if ((rc = make_tmap(&m.c, "gemm_fp8", CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, C, {N, M}, {2LL * ldc}, {64, 64}))) return rc;
    m.r = m.c;
  } else {
    if ((rc = make_tmap(&m.c, "gemm_fp8", CU_TENSOR_MAP_DATA_TYPE_FLOAT32, C, {N, M}, {4LL * ldc}, {32, 64}))) return rc;
    if ((rc = make_tmap(&m.r, "gemm_fp8", CU_TENSOR_MAP_DATA_TYPE_FLOAT32, res, {N, M}, {4LL * ldc}, {32, 64}))) return rc;
  }
  GemmParams p;
  p.C = C;
  p.M = M; p.N = N; p.K = K; p.ldc = ldc;
  p.num_m = ceil_div(M, BM);
  p.num_n = ceil_div(N, BN);
  p.num_kb = ceil_div(K, kBK);
  p.splits = 1;
  p.kb_per_split = p.num_kb;
  p.sa = sa;
  p.sb = sb;
  return res == nullptr ? launch<BN, false, false, EPI_FP8_BF16>(m, p, stream)
                        : launch<BN, false, false, EPI_FP8_RESADD_F32>(m, p, stream);
}

}  // namespace muse

using namespace muse;

extern "C" {

// The persistent GEMM owns one CTA per SM with a static tile assignment, so a CTA that cannot start (its SM is held by an
// NCCL all-reduce CTA during data-parallel training) delays the whole kernel by its full duration.  Under DDP the host
// reserves as many SMs as NCCL has channels: the GEMM grid shrinks by that many CTAs and both kernels fit side by side.
int muse_reserve_sms(int n) {
  g_reserved_sms = n < 0 ? 0 : n;
  return MUSE_OK;
}

int muse_gemm_bf16(const void* A, const void* B, void* C, const float* res, int M, int N, int K, int lda, int ldb,
                   int ldc, int a_mn, int b_mn, int epilogue, void* stream) {
  if (epilogue == MUSE_EPI_RESADD_F32 && res == nullptr) { set_last_error("gemm: RESADD epilogue needs res"); return MUSE_ERR_INVALID; }
  if (epilogue == MUSE_EPI_SPLITK_F32) { set_last_error("gemm: the deterministic split-K epilogue goes through muse_gemm_bf16_splitk"); return MUSE_ERR_INVALID; }
  return gemm_tc(A, B, C, res, M, N, K, lda, ldb, ldc, a_mn, b_mn, epilogue, static_cast<cudaStream_t>(stream), nullptr, 0);
}

int muse_gemm_fp8(const void* A, const float* sa, const void* B, const float* sb, void* C, int M, int N, int K, int lda,
                  int ldb, int ldc, void* stream) {
  return gemm_fp8(A, sa, B, sb, nullptr, C, M, N, K, lda, ldb, ldc, static_cast<cudaStream_t>(stream));
}

int muse_gemm_fp8_res(const void* A, const float* sa, const void* B, const float* sb, const float* res, float* C, int M,
                      int N, int K, int lda, int ldb, int ldc, void* stream) {
  if (res == nullptr) { set_last_error("gemm_fp8_res: needs res"); return MUSE_ERR_INVALID; }
  return gemm_fp8(A, sa, B, sb, res, C, M, N, K, lda, ldb, ldc, static_cast<cudaStream_t>(stream));
}

long long muse_gemm_splitk_workspace_bytes(int M, int N, int K) {
  int num_m, num_n, num_kb, kbs, splits, bn;
  split_plan(M, N, K, &num_m, &num_n, &num_kb, &kbs, &splits, &bn);
  if (splits <= 1) return 0;
  return static_cast<long long>(splits) * num_m * num_n * BM * bn * 4;
}

int muse_gemm_bf16_splitk(const void* A, const void* B, float* C, int M, int N, int K, int lda, int ldb, int ldc,
                          int a_mn, int b_mn, void* ws, long long ws_bytes, void* stream) {
  return gemm_tc(A, B, C, nullptr, M, N, K, lda, ldb, ldc, a_mn, b_mn, MUSE_EPI_SPLITK_F32, static_cast<cudaStream_t>(stream),
                 ws, ws_bytes);
}

}  // extern "C"
