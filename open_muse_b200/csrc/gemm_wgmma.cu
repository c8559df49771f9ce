// bf16 GEMM on the Hopper tensor cores: C[M,N] = A[M,K] * B[N,K]^T, fp32 accumulation in registers (wgmma).
//
// This is the kernel every nn.Linear of the reference's transformer maps to
// (muse/modeling_transformer.py:198-200,218 q/k/v/out; :789-798 wi_0/wi_1/wo; :980,984 mlm head)
// and, with transposed operand views, their dgrad / wgrad in backward.
//
// Structure (persistent, warp-specialised, one CTA per SM, 384 threads):
//   warpgroup 0  : TMA producer  - one thread issues cp.async.bulk.tensor 2D tiles (128B swizzle) into a smem ring
//   warpgroups 1-2: consumers    - each issues wgmma m64 x BN x k16 on its 64-row half of the 128-row tile, then runs
//                                  the epilogue straight from its accumulator registers (bf16 / fp32 / atomic / +residual)
// The producer runs up to kStages k-blocks ahead, so it keeps loading the next tile while the consumers store this one.
//
// Operand "major-ness": an operand is K-major when the reduction dim is contiguous in memory
// (activations X[T,K], weights W[N,K] in forward) and MN-major when the M/N dim is contiguous
// (W[N,K] used as the B operand of dgrad; dY[T,N] and X[T,K] as operands of wgrad, where the
// reduction runs over T). Both are fed straight from their row-major tensors through TMA; the
// smem (matrix) descriptors and the wgmma transpose flags tell the tensor core which layout it is looking at, so no
// transposes are materialised anywhere in the training step.
#include "common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace muse {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle row

// EPI_SPLITK_F32: deterministic split-K.  Every split stores its fp32 partial tile into a workspace and a second, fully
// parallel kernel sums the partials in split order and STORES the result, so the output needs no zero fill and is
// bit-identical from run to run (the atomic variant is order-dependent).
enum Epi { EPI_BF16 = 0, EPI_F32 = 1, EPI_ATOMIC_F32 = 2, EPI_RESADD_F32 = 3, EPI_SPLITK_F32 = 4 };

template <int BN>
struct Cfg {
  static constexpr int kStages = (BN == 256) ? 4 : 6;
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarBytes = 256;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 + kBarBytes;
};

struct GemmParams {
  void* C;
  const float* res;
  int M, N, K;
  int ldc;
  int num_m, num_n, num_kb, kb_per_split, splits;
  float* ws;      // EPI_SPLITK_F32: [splits][num_m * num_n][BM * BN] fp32 partial tiles
};

template <int BN, bool A_MN, bool B_MN, int EPI>
__global__ void __launch_bounds__(384, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const GemmParams p) {
  pdl_trigger();
  using C_ = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C_::kStages * C_::kStageBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + C_::kStages;

  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
    for (int i = 0; i < C_::kStages; ++i) {
      ptx::mbar_init(&full_bar[i], 1);
      ptx::mbar_init(&empty_bar[i], 2);  // one arrive per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // everything above touches only shared memory / kernel parameters

  const int tiles_mn = p.num_m * p.num_n;
  const int total_tiles = tiles_mn * p.splits;

  if (wg == 0) {
    ptx::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      // ------------------------------------------------------------ TMA producer
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n_idx = tile % p.num_n;
        const int m_idx = (tile / p.num_n) % p.num_m;
        const int split = tile / tiles_mn;
        const int kb0 = split * p.kb_per_split;
        const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);
        const int m0 = m_idx * BM, n0 = n_idx * BN;
        for (int kb = kb0; kb < kb1; ++kb) {
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          ptx::mbar_expect_tx(&full_bar[stage], C_::kStageBytes);
          uint8_t* sa = smem + stage * C_::kStageBytes;
          uint8_t* sb = sa + C_::kABytes;
          if (!A_MN) {
            ptx::tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, m0);
          } else {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)
              ptx::tma_load_2d(sa + i * (BK * 128), &tmA, &full_bar[stage], m0 + i * 64, kb * BK);
          }
          if (!B_MN) {
            ptx::tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, n0);
          } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)
              ptx::tma_load_2d(sb + i * (BK * 128), &tmB, &full_bar[stage], n0 + i * 64, kb * BK);
          }
          if (++stage == C_::kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<232>();
    // -------------------------------------------------------------- consumers: rows [64 * half, 64 * half + 64) of a tile
    const int half = wg - 1;
    const int t = threadIdx.x & 127;
    const int lr = half * 64 + (t >> 5) * 16 + ((t & 31) >> 2);  // tile-local row of d[4j], d[4j+1]; +8 for d[4j+2..3]
    const int lc = 2 * (t & 3);                                  // tile-local column of d[4j] within its 8-column group
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int n_idx = tile % p.num_n;
      const int m_idx = (tile / p.num_n) % p.num_m;
      const int split = tile / tiles_mn;
      const int kb0 = split * p.kb_per_split;
      const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);
      for (int kb = kb0; kb < kb1; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = ptx::smem_u32(smem + stage * C_::kStageBytes) + half * 8192;
        const uint32_t b_addr = ptx::smem_u32(smem + stage * C_::kStageBytes + C_::kABytes);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          // K-major  : 8-row groups 1024 B apart (SBO); a 16-element K step is +32 B inside the row.
          // MN-major : 64-element MN chunks BK*128 B apart (LBO), 8-k-row groups 1024 B apart (SBO);
          //            a 16-row K step is +2048 B.  The 64 rows of this half are one such chunk for A.
          const uint64_t adesc = A_MN ? ptx::make_smem_desc_sw128(a_addr + k * 2048, BK * 128, 1024)
                                      : ptx::make_smem_desc_sw128(a_addr + k * 32, 16, 1024);
          const uint64_t bdesc = B_MN ? ptx::make_smem_desc_sw128(b_addr + k * 2048, BK * 128, 1024)
                                      : ptx::make_smem_desc_sw128(b_addr + k * 32, 16, 1024);
          ptx::Wgmma<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>::run(acc, adesc, bdesc, (kb > kb0 || k > 0) ? 1 : 0);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        if (t == 0) ptx::mbar_arrive(&empty_bar[stage]);  // smem slot free: this warpgroup's MMAs have read it
        if (++stage == C_::kStages) { stage = 0; phase ^= 1; }
      }
      // ------------------------------------------------------------ epilogue from the accumulator registers
      const bool partial = (EPI == EPI_SPLITK_F32) && p.splits > 1;
      float* ws_tile = nullptr;
      if (EPI == EPI_SPLITK_F32 && partial)
        ws_tile = p.ws + (static_cast<size_t>(split) * tiles_mn + tile % tiles_mn) * (BM * BN);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const float v0 = acc[4 * j + 2 * hr], v1 = acc[4 * j + 2 * hr + 1];
          const int r = lr + 8 * hr, c = 8 * j + lc;
          if (EPI == EPI_SPLITK_F32 && partial) {
            *reinterpret_cast<float2*>(ws_tile + static_cast<size_t>(r) * BN + c) = make_float2(v0, v1);
            continue;
          }
          const int grow = m_idx * BM + r, gcol = n_idx * BN + c;
          if (grow >= p.M || gcol >= p.N) continue;
          const size_t off = static_cast<size_t>(grow) * p.ldc + gcol;
          const bool pair = gcol + 1 < p.N;
          if (EPI == EPI_BF16) {
            bf16* dst = reinterpret_cast<bf16*>(p.C) + off;
            if (pair) *reinterpret_cast<uint32_t*>(dst) = pack_bf16(v0, v1);
            else dst[0] = __float2bfloat16_rn(v0);
          } else {
            float* dst = reinterpret_cast<float*>(p.C) + off;
            if (EPI == EPI_F32 || EPI == EPI_SPLITK_F32) {
              if (pair) *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
              else dst[0] = v0;
            } else if (EPI == EPI_ATOMIC_F32) {
              if (pair) atomicAdd(reinterpret_cast<float2*>(dst), make_float2(v0, v1));
              else atomicAdd(dst, v0);
            } else {  // EPI_RESADD_F32: out = residual + bf16(acc)  (Linear output is bf16 under autocast)
              const float* rs = p.res + off;
              if (pair) {
                const float2 q2 = *reinterpret_cast<const float2*>(rs);
                *reinterpret_cast<float2*>(dst) = make_float2(q2.x + bf16_round(v0), q2.y + bf16_round(v1));
              } else {
                dst[0] = rs[0] + bf16_round(v0);
              }
            }
          }
        }
      }
    }
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
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || ptr == nullptr) {
    set_last_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(e));
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(ptr);
  return fn;
}

// 2D bf16 tensor map: inner (contiguous) extent `inner`, outer extent `outer`, row pitch `ld` elements.
int make_tmap(CUtensorMap* map, const void* base, long long inner, long long outer, long long ld, int box_inner,
              int box_outer) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return MUSE_ERR_CUDA;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld * 2) % 16 != 0) {
    set_last_error("gemm: operand base must be 16B aligned and leading dim a multiple of 8 elements");
    return MUSE_ERR_INVALID;
  }
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(outer)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_inner), static_cast<cuuint32_t>(box_outer)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult %d (inner=%lld outer=%lld ld=%lld)", (int)r, inner,
                   outer, ld);
    return MUSE_ERR_CUDA;
  }
  return MUSE_OK;
}

}  // namespace

// 3-D bf16 tensor map {cols, rows, batches} over a [batches*rows, pitch] row-major buffer: box {64 cols, box_rows, 1},
// 128-byte swizzle.  Rows past `rows` inside a batch are out of bounds -> zero-filled by the TMA unit.
int make_tmap3(CUtensorMap* map, const void* base, long long cols, long long rows, long long batches,
               long long row_pitch_elems, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return MUSE_ERR_CUDA;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (row_pitch_elems * 2) % 16 != 0) {
    set_last_error("attention: operand base must be 16B aligned and the row stride a multiple of 8 elements");
    return MUSE_ERR_INVALID;
  }
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(batches)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(row_pitch_elems) * 2,
                           static_cast<cuuint64_t>(rows) * static_cast<cuuint64_t>(row_pitch_elems) * 2};
  cuuint32_t box[3] = {64, static_cast<cuuint32_t>(box_rows), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled(3D) failed with CUresult %d (cols=%lld rows=%lld batches=%lld pitch=%lld)",
                   (int)r, cols, rows, batches, row_pitch_elems);
    return MUSE_ERR_CUDA;
  }
  return MUSE_OK;
}

// Generic bf16 tensor map (rank <= 5), 128-byte swizzle, zero fill out of bounds.  dims[0] is the contiguous dimension;
// strides_bytes[i] is the byte stride of dims[i + 1].
int make_tmap_nd(CUtensorMap* map, const void* base, int rank, const unsigned long long* dims,
                 const unsigned long long* strides_bytes, const unsigned* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return MUSE_ERR_CUDA;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) { set_last_error("tensor map: base must be 16B aligned"); return MUSE_ERR_INVALID; }
  cuuint64_t d[5], st[4];
  cuuint32_t bx[5], estr[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; bx[i] = box[i]; estr[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) {
    st[i] = strides_bytes[i];
    if (st[i] % 16 != 0) { set_last_error("tensor map: stride %d (%llu B) must be a multiple of 16 B", i, strides_bytes[i]); return MUSE_ERR_INVALID; }
  }
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), d, st, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error("cuTensorMapEncodeTiled(rank %d) failed with CUresult %d", rank, (int)r); return MUSE_ERR_CUDA; }
  return MUSE_OK;
}

namespace {

int g_num_sms = 0;
int g_reserved_sms = 0;  // SMs left free for concurrently running collective kernels (set_reserved_sms)
int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  const int n = g_num_sms - g_reserved_sms;
  return n > 16 ? n : 16;
}

template <int BN, bool A_MN, bool B_MN, int EPI>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  auto kern = gemm_wgmma_kernel<BN, A_MN, B_MN, EPI>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::kSmemBytes);
    if (e != cudaSuccess) {
      set_last_error("cudaFuncSetAttribute(gemm smem=%d): %s", Cfg<BN>::kSmemBytes, cudaGetErrorString(e));
      return MUSE_ERR_CUDA;
    }
    attr_set = true;
  }
  const int total = p.num_m * p.num_n * p.splits;
  const int grid = total < num_sms() ? total : num_sms();
  pdl_launch(grid, 384, Cfg<BN>::kSmemBytes, stream)(kern, ta, tb, p);
  return check_launch("gemm_wgmma");
}

template <int BN, bool A_MN, bool B_MN>
int launch_epi(int epi, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t s) {
  switch (epi) {
    case EPI_BF16: return launch<BN, A_MN, B_MN, EPI_BF16>(ta, tb, p, s);
    case EPI_F32: return launch<BN, A_MN, B_MN, EPI_F32>(ta, tb, p, s);
    case EPI_ATOMIC_F32: return launch<BN, A_MN, B_MN, EPI_ATOMIC_F32>(ta, tb, p, s);
    case EPI_RESADD_F32: return launch<BN, A_MN, B_MN, EPI_RESADD_F32>(ta, tb, p, s);
    case EPI_SPLITK_F32: return launch<BN, A_MN, B_MN, EPI_SPLITK_F32>(ta, tb, p, s);
  }
  set_last_error("gemm: unknown epilogue %d", epi);
  return MUSE_ERR_INVALID;
}

template <int BN>
int launch_major(int a_mn, int b_mn, int epi, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                 cudaStream_t s) {
  if (!a_mn && !b_mn) return launch_epi<BN, false, false>(epi, ta, tb, p, s);
  if (!a_mn && b_mn) return launch_epi<BN, false, true>(epi, ta, tb, p, s);
  if (a_mn && b_mn) return launch_epi<BN, true, true>(epi, ta, tb, p, s);
  return launch_epi<BN, true, false>(epi, ta, tb, p, s);
}

}  // namespace

// The persistent GEMM owns one CTA per SM with a static tile assignment, so a CTA that cannot start (its SM is held by an
// NCCL all-reduce CTA during data-parallel training) delays the whole kernel by its full duration.  Under DDP the host
// reserves as many SMs as NCCL has channels: the GEMM grid shrinks by that many CTAs and both kernels fit side by side.
void set_reserved_sms(int n) { g_reserved_sms = n < 0 ? 0 : n; }

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

long long gemm_splitk_workspace_bytes(int M, int N, int K) {
  int num_m, num_n, num_kb, kbs, splits, bn;
  split_plan(M, N, K, &num_m, &num_n, &num_kb, &kbs, &splits, &bn);
  if (splits <= 1) return 0;
  return static_cast<long long>(splits) * num_m * num_n * BM * bn * 4;
}

int gemm_tc(const void* A, const void* B, void* C, const float* res, int M, int N, int K, int lda, int ldb,
                 int ldc, int a_mn, int b_mn, int epi, cudaStream_t stream, void* ws, long long ws_bytes) {
  if (M <= 0 || N <= 0 || K <= 0) return MUSE_OK;
  if (epi == EPI_BF16 ? (ldc % 8 != 0) : (ldc % 4 != 0)) {
    set_last_error("gemm: ldc=%d must be a multiple of %d", ldc, epi == EPI_BF16 ? 8 : 4);
    return MUSE_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(C) & 15) != 0) {
    set_last_error("gemm: C must be 16B aligned");
    return MUSE_ERR_INVALID;
  }
  const int BN = (N >= 256) ? 256 : 128;
  CUtensorMap ta, tb;
  int rc;
  rc = a_mn ? make_tmap(&ta, A, M, K, lda, 64, BK) : make_tmap(&ta, A, K, M, lda, BK, BM);
  if (rc) return rc;
  rc = b_mn ? make_tmap(&tb, B, N, K, ldb, 64, BK) : make_tmap(&tb, B, K, N, ldb, BK, BN);
  if (rc) return rc;

  GemmParams p;
  p.C = C;
  p.res = res;
  p.M = M; p.N = N; p.K = K; p.ldc = ldc;
  p.num_m = ceil_div(M, BM);
  p.num_n = ceil_div(N, BN);
  p.num_kb = ceil_div(K, BK);
  p.splits = 1;
  p.kb_per_split = p.num_kb;
  p.ws = reinterpret_cast<float*>(ws);
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
  rc = (BN == 256) ? launch_major<256>(a_mn, b_mn, epi, ta, tb, p, stream) : launch_major<128>(a_mn, b_mn, epi, ta, tb, p, stream);
  if (rc || epi != EPI_SPLITK_F32 || p.splits <= 1) return rc;
  const long long n_out4 = static_cast<long long>(M) * ((N + 3) / 4);
  pdl_launch(static_cast<unsigned>(ceil_div_ll(n_out4, 256)), 256, 0, stream)(splitk_reduce_kernel,
      p.ws, reinterpret_cast<float*>(C), M, N, ldc, p.num_n, p.num_m * p.num_n, BN, p.splits);
  return check_launch("gemm splitk reduce");
}

}  // namespace muse
