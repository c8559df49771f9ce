// wgmma / TMA attention for head_dim 64 and 48 (sm_90a): forward, dQ and dK/dV kernels.
// Replaces the reference's materialised attention (muse/modeling_transformer.py:221-241) and its autograd backward.
//
// One CTA = one (batch, head) x one 128-row tile of the "owned" sequence dimension.  Every warpgroup of the CTA issues
// wgmma on 64-row halves of the tile.  Score-like products (S, dP) land in an fp32 [128 x 64] shared-memory tile from
// which the softmax math reads whole rows (one row per thread, as written below); the accumulating products (O, dQ, dK,
// dV) stay in the wgmma accumulator registers for the whole loop and are stored once at the end.
//
//   forward  : owned = q rows.   S = Q K_j^T -> online softmax (fp32) -> P (bf16, smem) -> O += P V_j
//   dQ       : owned = q rows.   S, dP = dO V_j^T -> sweep 1: D = sum P*dP ; sweep 2: dS -> dQ += dS K_j
//   dK/dV    : owned = kv rows.  S^T = K Q_i^T, dP^T = V dO_i^T -> P^T, dS^T -> dV += P^T dO_i, dK += dS^T Q_i
// Operands are read straight from the strided [tokens, 3H] QKV projection through 3-D TMA tensor maps
// {64 head columns, S rows, B} (rows past the end of a sequence are zero-filled by the TMA unit), with the same
// 128-byte-swizzled tiles serving as K-major or MN-major MMA operands depending on the product.  The looped tiles sit in
// a TMA ring that is refilled while the current tile is being processed.
// The owned dimension is cut into ceil(S / 128) tiles of EQUAL height R = ceil(S / tiles) (S = 257 with the class token ->
// three tiles of 86 rows; S = 256 -> two of 128; the 77 text states of cross-attention -> one of 77): a tile starts at row
// i * R, its CTA still loads a 128-row box (rows past R belong to the next tile or are zero-filled past the sequence), the
// MMAs run on all 128 rows, but only rows < R are kept, and warps whose 32 rows all lie past R skip the softmax math.
// The looped dimension handles ragged tails by shrinking the MMA N/K to a multiple of 16.
#include "common.cuh"
#include "ptx.cuh"
#include "tc_host.cuh"
#include "wgmma.cuh"

namespace muse {

namespace {

// Head dimension HD is a template parameter: 64 (every text-to-image / U-ViT config, BASELINE configs) or 48 (configs/imagenet.yaml:
// hidden 768, 16 heads -- the configuration training/train_maskgit_imagenet.py is written for).  For HD = 48 the TMA boxes stay
// 64 columns wide (head h starts at column 48 h; the 16 trailing columns belong to the next head or are zero-filled past the
// tensor) and simply never enter a product: Q K^T / dO V^T run 3 instead of 4 k-steps, and the accumulate MMAs (P V, dS K,
// dS^T Q, P^T dO) have N = 48, reading the first 48 columns of their MN-major 128-byte rows.
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// exp2 on the SFU without the denormal/range fix-ups of exp2f (inputs here are <= 0 or bounded scores)
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// named barrier over the 256 math threads (barrier 0 stays __syncthreads for the whole CTA)
__device__ __forceinline__ void math_sync() { asm volatile("bar.sync 1, 256;\n" ::: "memory"); }

// Store 8 consecutive bf16 (one 16-byte chunk) of row r, columns [k0, k0+8) of a [128 x K] K-major SW128 operand
// made of 64-column atoms (16 KB each).
__device__ __forceinline__ void st_operand_chunk(uint8_t* base, int r, int k0, uint4 v) {
  const int atom = k0 >> 6, c8 = (k0 & 63) >> 3;
  *reinterpret_cast<uint4*>(base + atom * 16384 + r * 128 + ((c8 ^ (r & 7)) << 4)) = v;
}

struct TcParams {
  int Sq, Skv, nh;
  int tile_rows;  // R: owned rows per CTA (<= 128)
  float scale;
  // outputs / side inputs (plain global pointers; rows addressed as b*S + s)
  bf16* out0;  long long out0_rs;   // fwd: O ; dq: dQ ; dkdv: dK
  bf16* out1;  long long out1_rs;   // dkdv: dV
  float* lse;                        // [B, nh, Sq]
  float* dvec;                       // [B, nh, Sq]
};

// ------------------------------------------------------------------------------------------------ wgmma helpers
constexpr int SP = 68;  // row pitch (floats) of the fp32 score tiles: float4 row reads by 8 consecutive rows hit 32 banks
constexpr int SCORE_BYTES = 128 * SP * 4;

// d (+)= A[64 rows x 16*ksteps] * B, A a K-major tile, B K-major (TB = 0, N rows) or MN-major (TB = 1, N columns).
template <int N, int TB>
__device__ __forceinline__ void mma_tile(float (&d)[N / 2], uint32_t a, uint32_t b, int ksteps, int accumulate) {
  ptx::wgmma_fence();
  for (int ks = 0; ks < ksteps; ++ks)
    ptx::Wgmma<N, 0, TB>::run(d, ptx::desc_kmajor(a, ks), TB ? ptx::desc_mnmajor(b, ks) : ptx::desc_kmajor(b, ks),
                              (accumulate || ks > 0) ? 1 : 0);
  ptx::wgmma_commit();
  ptx::wgmma_wait<0>();
}

template <int N>
__device__ __forceinline__ void scores_n(uint32_t a, uint32_t b, int ksteps, float* dst, int row0) {
  float d[N / 2];
  mma_tile<N, 0>(d, a, b, ksteps, 0);
  const int r = row0 + ptx::frag_row(), c = ptx::frag_col();
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    *reinterpret_cast<float2*>(dst + r * SP + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(dst + (r + 8) * SP + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// rows [row0, row0 + 64) of A B^T (both K-major, N = n16 <= 64 rows of B) -> the fp32 score tile
__device__ __forceinline__ void scores_to_smem(uint32_t a, uint32_t b, int n16, int ksteps, float* dst, int row0) {
  switch (n16) {
    case 16: scores_n<16>(a, b, ksteps, dst, row0); break;
    case 32: scores_n<32>(a, b, ksteps, dst, row0); break;
    case 48: scores_n<48>(a, b, ksteps, dst, row0); break;
    default: scores_n<64>(a, b, ksteps, dst, row0); break;
  }
}

// bf16 store of an [64 x HD] accumulator fragment: rows row0 + (fragment row) of `base` (row stride rs), if < rows_ok
template <int HD>
__device__ __forceinline__ void store_acc(const float (&d)[HD / 2], bf16* base, long long rs, int row0, int rows_ok,
                                          const float* row_scale) {
  const int r = row0 + ptx::frag_row(), c = ptx::frag_col();
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int rr = r + 8 * hr;
    if (rr >= rows_ok) continue;
    const float sc = row_scale ? row_scale[rr] : 1.f;
    bf16* dst = base + rr * rs;
#pragma unroll
    for (int j = 0; j < HD / 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j + c) = pack_bf16(d[4 * j + 2 * hr] * sc, d[4 * j + 2 * hr + 1] * sc);
  }
}

// ------------------------------------------------------------------------------------------------ forward
// 128 threads = one warpgroup, which issues the MMAs of both 64-row halves (O of both halves in registers).
// smem: Q 16K | K 8K | V 8K | P 16K | S fp32 | per-row scale | barriers -> two co-resident CTAs per SM overlap each other's
// TMA / MMA / softmax phases.
constexpr int FWD_BN = 64;
constexpr int FWD_SMEM = 16384 /*Q*/ + 8192 /*K*/ + 8192 /*V*/ + 16384 /*P*/ + SCORE_BYTES + 512 + 64;

template <int HD>
__global__ void __launch_bounds__(128, 2)
attn_fwd_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, const TcParams p) {
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t smem_raw[];  // 128B-swizzled tiles need 1024 B alignment
  uint8_t* smem = smem_raw;
  if ((ptx::smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sQ = smem;
  uint8_t* sK = smem + 16384;
  uint8_t* sV = smem + 24576;
  uint8_t* sP = smem + 32768;
  float* sS = reinterpret_cast<float*>(smem + 49152);
  float* sRow = reinterpret_cast<float*>(smem + 49152 + SCORE_BYTES);  // per-row alpha, then 1 / l
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 49152 + SCORE_BYTES + 512);
  uint64_t* bar_kv = bars;      // Q (first use) + K tile landed
  uint64_t* bar_v = bars + 1;   // V tile landed

  const int tid = threadIdx.x, warp = tid >> 5;
  const int q0 = blockIdx.x * p.tile_rows, h = blockIdx.y, b = blockIdx.z;
  const int rows_here = min(p.tile_rows, p.Sq - q0);
  const bool warp_active = warp * 32 < rows_here;  // warps whose rows all belong to the next tile skip the softmax math
  if (tid == 0) {
    ptx::mbar_init(bar_kv, 1);
    ptx::mbar_init(bar_v, 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // everything above touches only shared memory / kernel parameters
  const int ntiles = ceil_div(p.Skv, FWD_BN);

  if (tid == 0) {
    ptx::mbar_expect_tx(bar_kv, 16384 + 8192);
    ptx::tma_load_3d(sQ, &tmQ, bar_kv, h * HD, q0, b);
    ptx::tma_load_3d(sK, &tmK, bar_kv, h * HD, 0, b);
    ptx::mbar_expect_tx(bar_v, 8192);
    ptx::tma_load_3d(sV, &tmV, bar_v, h * HD, 0, b);
  }
  const float sl2 = p.scale * kLog2e;
  float m = -INFINITY, l = 0.f;
  float o[2][HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) { o[0][i] = 0.f; o[1][i] = 0.f; }

  for (int j = 0; j < ntiles; ++j) {
    const uint32_t par = j & 1;
    const int nvalid = min(FWD_BN, p.Skv - j * FWD_BN);
    const int n16 = (nvalid + 15) & ~15;
    ptx::mbar_wait(bar_kv, par);
    scores_to_smem(ptx::smem_u32(sQ), ptx::smem_u32(sK), n16, HD / 16, sS, 0);
    scores_to_smem(ptx::smem_u32(sQ) + 8192, ptx::smem_u32(sK), n16, HD / 16, sS, 64);
    __syncthreads();  // S_j is in shared memory and K_j has been consumed
    if (tid == 0 && j + 1 < ntiles) {  // fetch K_{j+1} under the softmax math
      ptx::mbar_expect_tx(bar_kv, 8192);
      ptx::tma_load_3d(sK, &tmK, bar_kv, h * HD, (j + 1) * FWD_BN, b);
    }
    float alpha = 1.f;
    if (warp_active) {
    // the whole score row (<= 64 columns) fits in registers.  The instruction count per score element is what bounds
    // this loop, so the ragged-tail masking is kept out of the full-tile path and the softmax scale is folded into one
    // FFMA per element.
    float sc[64];
#pragma unroll
    for (int c = 0; c < 64; c += 4) {
      if (c < n16) {
        const float4 v = *reinterpret_cast<const float4*>(sS + tid * SP + c);
        sc[c] = v.x; sc[c + 1] = v.y; sc[c + 2] = v.z; sc[c + 3] = v.w;
      } else {
        sc[c] = sc[c + 1] = sc[c + 2] = sc[c + 3] = -INFINITY;
      }
    }
    if (nvalid < FWD_BN) {
#pragma unroll
      for (int i = 0; i < 64; ++i) sc[i] = (i < nvalid) ? sc[i] : -INFINITY;
    }
    float raw = -INFINITY;
#pragma unroll
    for (int i = 0; i < 64; ++i) raw = fmaxf(raw, sc[i]);
    // Lazy running maximum: the reference point m only moves when the tile's maximum exceeds it by more than 8 (log2
    // units), i.e. P entries stay below 2^8 -- harmless in bf16 / fp32 -- and the final 1 / l normalisation and the LSE
    // (m + log2 l) are exact for any reference point.  Most tiles then leave m alone and alpha is exactly 1.
    const float cand = raw * sl2;
    const float mx = (cand > m + 8.0f) ? cand : m;
    alpha = ex2(m - mx);  // 0 on the first tile (m = -inf), 1 when the reference point stays
    m = mx;
    float l4[4] = {0.f, 0.f, 0.f, 0.f};  // four independent chains instead of one 64-long dependent add chain
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      sc[i] = ex2(fmaf(sc[i], sl2, -m));
      l4[i & 3] += sc[i];
    }
    l = fmaf(l, alpha, (l4[0] + l4[1]) + (l4[2] + l4[3]));
#pragma unroll
    for (int i = 0; i < 64; i += 8) {
      if (i < n16) {
        uint4 u;
        u.x = pack_bf16(sc[i], sc[i + 1]); u.y = pack_bf16(sc[i + 2], sc[i + 3]);
        u.z = pack_bf16(sc[i + 4], sc[i + 5]); u.w = pack_bf16(sc[i + 6], sc[i + 7]);
        st_operand_chunk(sP, tid, i, u);
      }
    }
    }  // warp_active
    sRow[tid] = alpha;
    ptx::fence_proxy_async();
    __syncthreads();  // P_j is visible to the tensor core, every row's alpha to every thread
    if (j > 0) {  // rescale the running output
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const float a0 = sRow[hh * 64 + ptx::frag_row()], a1 = sRow[hh * 64 + ptx::frag_row() + 8];
#pragma unroll
        for (int i = 0; i < HD / 2; i += 4) {
          o[hh][i] *= a0; o[hh][i + 1] *= a0; o[hh][i + 2] *= a1; o[hh][i + 3] *= a1;
        }
      }
    }
    ptx::mbar_wait(bar_v, par);
    mma_tile<HD, 1>(o[0], ptx::smem_u32(sP), ptx::smem_u32(sV), n16 >> 4, j > 0);
    mma_tile<HD, 1>(o[1], ptx::smem_u32(sP) + 8192, ptx::smem_u32(sV), n16 >> 4, j > 0);
    __syncthreads();  // P_j and V_j have been consumed
    if (tid == 0 && j + 1 < ntiles) {
      ptx::mbar_expect_tx(bar_v, 8192);
      ptx::tma_load_3d(sV, &tmV, bar_v, h * HD, (j + 1) * FWD_BN, b);
    }
  }
  // epilogue: O / l -> bf16 rows, LSE
  const int row = q0 + tid;
  sRow[tid] = 1.f / l;
  if (tid < rows_here) p.lse[(static_cast<long long>(b) * p.nh + h) * p.Sq + row] = (m + log2f(l)) * kLn2;
  __syncthreads();
  bf16* obase = p.out0 + (static_cast<long long>(b) * p.Sq + q0) * p.out0_rs + h * HD;
  store_acc<HD>(o[0], obase, p.out0_rs, 0, rows_here, sRow);
  store_acc<HD>(o[1], obase, p.out0_rs, 64, rows_here, sRow);
}

// ------------------------------------------------------------------------------------------------ backward: dQ
// 256 threads = two warpgroups; warpgroup g issues the MMAs of rows [64 g, 64 g + 64) and keeps that half of dQ in
// registers.  In the softmax math, warps w and w+4 share rows 32*(w%4).. and split the 64 score columns in two halves.
// K/V tiles sit in a 3-stage TMA ring with prefetch distance 2.
// smem: Q 16K | dO 16K | 3 x {K_j 8K, V_j 8K} | dS 16K (the partial-D exchange buffer aliases it) | S, dP fp32
constexpr int BWD_BN = 64;
constexpr int DQ_SMEM = 16384 * 2 + 3 * 16384 + 16384 + 2 * SCORE_BYTES + 64;

template <int HD>
__global__ void __launch_bounds__(256, 1)
attn_bwd_dq_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO,
                      const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                      const TcParams p) {
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if ((ptx::smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sQ = smem;
  uint8_t* sdO = smem + 16384;
  uint8_t* sKV = smem + 32768;             // 3 stages x {K 8 KB, V 8 KB}
  uint8_t* sdS = smem + 32768 + 49152;
  float* sDp = reinterpret_cast<float*>(sdS);  // [2][128] partial D (only used between the two sweeps)
  float* sS = reinterpret_cast<float*>(sdS + 16384);
  float* sdP = sS + 128 * SP;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sdS + 16384 + 2 * SCORE_BYTES);
  uint64_t* bar_kv = bars;       // [3] TMA landed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = tid >> 7;                     // warpgroup: MMA rows [64 g, 64 g + 64)
  const int half = warp >> 2;                 // column half handled by this thread
  const int r = (warp & 3) * 32 + lane;       // row handled by this thread
  const int q0 = blockIdx.x * p.tile_rows, h = blockIdx.y, b = blockIdx.z;
  const int rows_here = min(p.tile_rows, p.Sq - q0);
  const bool warp_active = (warp & 3) * 32 < rows_here;  // other warps keep the barrier protocol but skip the math
  const bool row_ok = r < rows_here;
  if (tid == 0) {
    for (int i = 0; i < 3; ++i) ptx::mbar_init(&bar_kv[i], 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // everything above touches only shared memory / kernel parameters
  const int ntiles = ceil_div(p.Skv, BWD_BN);
  const int nsteps = 2 * ntiles;
  const int row = q0 + r;
  const long long stat_idx = (static_cast<long long>(b) * p.nh + h) * p.Sq + row;
  const float lse2 = row_ok ? p.lse[stat_idx] * kLog2e : 0.f;
  const float sl2 = p.scale * kLog2e;

  auto load_kv = [&](int step) {       // thread 0: TMA of the K/V tile of `step` into its ring stage
    uint8_t* sK = sKV + (step % 3) * 16384;
    const int jn = step % ntiles;
    ptx::tma_load_3d(sK, &tmK, &bar_kv[step % 3], h * HD, jn * BWD_BN, b);
    ptx::tma_load_3d(sK + 8192, &tmV, &bar_kv[step % 3], h * HD, jn * BWD_BN, b);
  };
  if (tid == 0) {
    ptx::mbar_expect_tx(&bar_kv[0], 16384 * 2 + 8192 * 2);
    ptx::tma_load_3d(sQ, &tmQ, &bar_kv[0], h * HD, q0, b);
    ptx::tma_load_3d(sdO, &tmdO, &bar_kv[0], h * HD, q0, b);
    load_kv(0);
    if (nsteps > 1) {
      ptx::mbar_expect_tx(&bar_kv[1], 8192 * 2);
      load_kv(1);
    }
  }
  float dq[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) dq[i] = 0.f;
  float dsum = 0.f;
  for (int st = 0; st < nsteps; ++st) {
    const int j = st % ntiles;
    const bool sweep2 = st >= ntiles;
    const int u = st - ntiles;  // index among the sweep-2 steps
    const int nvalid = min(BWD_BN, p.Skv - j * BWD_BN);
    const int n16 = (nvalid + 15) & ~15;
    if (tid == 0 && st + 2 < nsteps) {  // ring stage (st+2)%3 was last read in step st-1, which every thread has left
      ptx::mbar_expect_tx(&bar_kv[(st + 2) % 3], 8192 * 2);
      load_kv(st + 2);
    }
    ptx::mbar_wait(&bar_kv[st % 3], (st / 3) & 1);
    uint8_t* sK = sKV + (st % 3) * 16384;
    scores_to_smem(ptx::smem_u32(sQ) + g * 8192, ptx::smem_u32(sK), n16, HD / 16, sS, g * 64);
    scores_to_smem(ptx::smem_u32(sdO) + g * 8192, ptx::smem_u32(sK) + 8192, n16, HD / 16, sdP, g * 64);
    math_sync();  // S and dP of this step are in shared memory
    float s_reg[32], d_reg[32];
    if (warp_active) {
#pragma unroll
      for (int cc = 0; cc < 32; cc += 4) {
        const int c = half * 32 + cc;
        if (c < n16) {
          const float4 a4 = *reinterpret_cast<const float4*>(sS + r * SP + c);
          const float4 b4 = *reinterpret_cast<const float4*>(sdP + r * SP + c);
          s_reg[cc] = a4.x; s_reg[cc + 1] = a4.y; s_reg[cc + 2] = a4.z; s_reg[cc + 3] = a4.w;
          d_reg[cc] = b4.x; d_reg[cc + 1] = b4.y; d_reg[cc + 2] = b4.z; d_reg[cc + 3] = b4.w;
        }
      }
    }
    const float neg_d_scaled = -dsum * p.scale;
#pragma unroll
    for (int cc = 0; cc < 32; cc += 16) {
      const int c = half * 32 + cc;
      if (warp_active && c < n16) {
#pragma unroll
        for (int i8 = 0; i8 < 16; i8 += 8) {
          float pr[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) pr[i] = ex2(fmaf(s_reg[cc + i8 + i], sl2, -lse2));
          if (nvalid < BWD_BN) {  // ragged last tile only
#pragma unroll
            for (int i = 0; i < 8; ++i) pr[i] = (c + i8 + i < nvalid) ? pr[i] : 0.f;
          }
          if (!sweep2) {
#pragma unroll
            for (int i = 0; i < 8; ++i) dsum = fmaf(pr[i], d_reg[cc + i8 + i], dsum);
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) pr[i] *= fmaf(d_reg[cc + i8 + i], p.scale, neg_d_scaled);
            uint4 v;
            v.x = pack_bf16(pr[0], pr[1]); v.y = pack_bf16(pr[2], pr[3]);
            v.z = pack_bf16(pr[4], pr[5]); v.w = pack_bf16(pr[6], pr[7]);
            st_operand_chunk(sdS, r, c + i8, v);
          }
        }
      }
    }
    if (sweep2) {
      ptx::fence_proxy_async();
      math_sync();  // dS is visible to the tensor core
      mma_tile<HD, 1>(dq, ptx::smem_u32(sdS) + g * 8192, ptx::smem_u32(sK), n16 >> 4, u > 0);  // dQ += dS K_j
    }
    if (st == ntiles - 1) {  // D = sum over both column halves, identical in both threads of the row
      sDp[half * 128 + r] = dsum;
      math_sync();
      dsum = sDp[r] + sDp[128 + r];
      if (half == 0 && row_ok) p.dvec[stat_idx] = dsum;  // for the dK/dV kernels
    }
    math_sync();  // end of step: score tiles, dS and the ring stage are free again
  }
  store_acc<HD>(dq, p.out0 + (static_cast<long long>(b) * p.Sq + q0) * p.out0_rs + h * HD, p.out0_rs, g * 64, rows_here,
                nullptr);
}

// ------------------------------------------------------------------------------------------------ backward: dK, dV
// Same structure as the dQ kernel, looping over 64-row q tiles; dK and dV of the warpgroup's 64 kv rows in registers.
// smem: K_j 16K | V_j 16K | 3 x {Q_i 8K, dO_i 8K} | P^T 16K | dS^T 16K | lse/D 512 B | S^T, dP^T fp32
constexpr int DKDV_SMEM = 16384 * 2 + 3 * 16384 + 16384 * 2 + 512 + 2 * SCORE_BYTES + 64;

template <int HD>
__global__ void __launch_bounds__(256, 1)
attn_bwd_dkdv_tc_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                        const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO,
                        const TcParams p) {
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if ((ptx::smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sK = smem;
  uint8_t* sV = smem + 16384;
  uint8_t* sQO = smem + 32768;             // 3 stages x {Q_i 8 KB, dO_i 8 KB}
  uint8_t* sPT = smem + 32768 + 49152;
  uint8_t* sdST = sPT + 16384;
  float* sLD = reinterpret_cast<float*>(sdST + 16384);  // [lse 64 | D 64] of the current q tile
  float* sS = sLD + 128;
  float* sdP = sS + 128 * SP;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sdST + 16384 + 512 + 2 * SCORE_BYTES);
  uint64_t* bar_ld = bars;       // [3] TMA landed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = tid >> 7;
  const int half = warp >> 2;
  const int r = (warp & 3) * 32 + lane;
  const int kv0 = blockIdx.x * p.tile_rows, h = blockIdx.y, b = blockIdx.z;
  const int rows_here = min(p.tile_rows, p.Skv - kv0);
  const bool warp_active = (warp & 3) * 32 < rows_here;
  if (tid == 0) {
    for (int i = 0; i < 3; ++i) ptx::mbar_init(&bar_ld[i], 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // everything above touches only shared memory / kernel parameters
  const int ntiles = ceil_div(p.Sq, BWD_BN);
  const bool kv_ok = r < rows_here;  // rows past the tile's share belong to the next CTA (or lie past the sequence)
  const float sl2 = p.scale * kLog2e;
  const long long stat_base = (static_cast<long long>(b) * p.nh + h) * p.Sq;

  auto load_q = [&](int i) {
    uint8_t* sQ = sQO + (i % 3) * 16384;
    ptx::tma_load_3d(sQ, &tmQ, &bar_ld[i % 3], h * HD, i * BWD_BN, b);
    ptx::tma_load_3d(sQ + 8192, &tmdO, &bar_ld[i % 3], h * HD, i * BWD_BN, b);
  };
  if (tid == 0) {
    ptx::mbar_expect_tx(&bar_ld[0], 16384 * 2 + 8192 * 2);
    ptx::tma_load_3d(sK, &tmK, &bar_ld[0], h * HD, kv0, b);
    ptx::tma_load_3d(sV, &tmV, &bar_ld[0], h * HD, kv0, b);
    load_q(0);
    if (ntiles > 1) {
      ptx::mbar_expect_tx(&bar_ld[1], 8192 * 2);
      load_q(1);
    }
  }
  float dk[HD / 2], dv[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) { dk[i] = 0.f; dv[i] = 0.f; }
  for (int i = 0; i < ntiles; ++i) {
    const int q0 = i * BWD_BN;
    const int nvalid = min(BWD_BN, p.Sq - q0);
    const int n16 = (nvalid + 15) & ~15;
    float* sL = sLD;
    float* sD = sL + 64;
    if (tid < BWD_BN) {
      const int qr = q0 + tid;
      sL[tid] = (qr < p.Sq) ? p.lse[stat_base + qr] * kLog2e : 0.f;
      sD[tid] = (qr < p.Sq) ? p.dvec[stat_base + qr] * p.scale : 0.f;  // pre-scaled: dS = P (dP*scale - D*scale)
    }
    if (tid == 0 && i + 2 < ntiles) {  // ring stage (i+2)%3 was last read in step i-1, which every thread has left
      ptx::mbar_expect_tx(&bar_ld[(i + 2) % 3], 8192 * 2);
      load_q(i + 2);
    }
    ptx::mbar_wait(&bar_ld[i % 3], (i / 3) & 1);
    uint8_t* sQ = sQO + (i % 3) * 16384;
    scores_to_smem(ptx::smem_u32(sK) + g * 8192, ptx::smem_u32(sQ), n16, HD / 16, sS, g * 64);
    scores_to_smem(ptx::smem_u32(sV) + g * 8192, ptx::smem_u32(sQ) + 8192, n16, HD / 16, sdP, g * 64);
    math_sync();  // S^T, dP^T and this step's lse / D are visible to all threads
    float s_reg[32], d_reg[32];
    if (warp_active) {
#pragma unroll
      for (int cc = 0; cc < 32; cc += 4) {
        const int c = half * 32 + cc;
        if (c < n16) {
          const float4 a4 = *reinterpret_cast<const float4*>(sS + r * SP + c);
          const float4 b4 = *reinterpret_cast<const float4*>(sdP + r * SP + c);
          s_reg[cc] = a4.x; s_reg[cc + 1] = a4.y; s_reg[cc + 2] = a4.z; s_reg[cc + 3] = a4.w;
          d_reg[cc] = b4.x; d_reg[cc + 1] = b4.y; d_reg[cc + 2] = b4.z; d_reg[cc + 3] = b4.w;
        }
      }
    }
#pragma unroll
    for (int cc = 0; cc < 32; cc += 16) {
      const int c = half * 32 + cc;
      if (warp_active && c < n16) {
#pragma unroll
        for (int k8 = 0; k8 < 16; k8 += 8) {
          float pt[8], ds[8], lq[8], dq_[8];
#pragma unroll
          for (int k = 0; k < 8; k += 4) {  // per-column lse / D: 16-byte broadcast reads
            const float4 a = *reinterpret_cast<const float4*>(sL + c + k8 + k);
            const float4 e = *reinterpret_cast<const float4*>(sD + c + k8 + k);
            lq[k] = a.x; lq[k + 1] = a.y; lq[k + 2] = a.z; lq[k + 3] = a.w;
            dq_[k] = e.x; dq_[k + 1] = e.y; dq_[k + 2] = e.z; dq_[k + 3] = e.w;
          }
#pragma unroll
          for (int k = 0; k < 8; ++k) pt[k] = ex2(fmaf(s_reg[cc + k8 + k], sl2, -lq[k]));
          if (nvalid < BWD_BN || !kv_ok) {  // ragged q tile / kv rows past the end of the sequence
#pragma unroll
            for (int k = 0; k < 8; ++k) pt[k] = (kv_ok && c + k8 + k < nvalid) ? pt[k] : 0.f;
          }
#pragma unroll
          for (int k = 0; k < 8; ++k) ds[k] = pt[k] * fmaf(d_reg[cc + k8 + k], p.scale, -dq_[k]);
          uint4 x, y;
          x.x = pack_bf16(pt[0], pt[1]); x.y = pack_bf16(pt[2], pt[3]);
          x.z = pack_bf16(pt[4], pt[5]); x.w = pack_bf16(pt[6], pt[7]);
          y.x = pack_bf16(ds[0], ds[1]); y.y = pack_bf16(ds[2], ds[3]);
          y.z = pack_bf16(ds[4], ds[5]); y.w = pack_bf16(ds[6], ds[7]);
          st_operand_chunk(sPT, r, c + k8, x);
          st_operand_chunk(sdST, r, c + k8, y);
        }
      }
    }
    ptx::fence_proxy_async();
    math_sync();  // P^T / dS^T are visible to the tensor core
    mma_tile<HD, 1>(dv, ptx::smem_u32(sPT) + g * 8192, ptx::smem_u32(sQ) + 8192, n16 >> 4, i > 0);  // dV += P^T dO_i
    mma_tile<HD, 1>(dk, ptx::smem_u32(sdST) + g * 8192, ptx::smem_u32(sQ), n16 >> 4, i > 0);         // dK += dS^T Q_i
    math_sync();  // end of step: the score tiles, P^T / dS^T, lse / D and the ring stage are free again
  }
  const long long base = static_cast<long long>(b) * p.Skv + kv0;
  store_acc<HD>(dk, p.out0 + base * p.out0_rs + h * HD, p.out0_rs, g * 64, rows_here, nullptr);
  store_acc<HD>(dv, p.out1 + base * p.out1_rs + h * HD, p.out1_rs, g * 64, rows_here, nullptr);
}

// Raises kernel K's dynamic shared-memory limit and asks for all of L1 as shared memory, once per kernel.
template <auto K>
int set_smem(int bytes) {
  static bool carveout = false;
  if (!carveout) {
    cudaFuncSetAttribute(K, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    carveout = true;
  }
  return set_max_dynamic_smem<K>(bytes);
}

// Balanced tiling of an owned dimension of S rows: ceil(S / 128) tiles of R = ceil(S / tiles) rows each.
void balanced_tiles(int S, int* ntile, int* rows) {
  *ntile = ceil_div(S, 128);
  *rows = ceil_div(S, *ntile);
}

// 3-D map {cols, S rows, B} of a [B * S, rs] row-major operand, box {64 columns, box_rows rows, 1}: rows past S inside a
// batch are out of bounds and read as zeros.
int qkv_tmap(CUtensorMap* map, const void* base, int cols, int S, int B, int rs, int box_rows) {
  return make_tmap_bf16(map, "attention", base, {cols, S, B}, {2LL * rs, 2LL * rs * S}, {64, box_rows, 1});
}

template <int HD>
int attn_fwd_impl(const void* q, const void* k, const void* v, void* o, float* lse, int B, int nh, int Sq, int Skv, int q_rs,
                  int k_rs, int v_rs, int o_rs, float scale, cudaStream_t s) {
  int ntile, tile_rows;
  balanced_tiles(Sq, &ntile, &tile_rows);
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = qkv_tmap(&tq, q, nh * HD, Sq, B, q_rs, 128))) return rc;
  if ((rc = qkv_tmap(&tk, k, nh * HD, Skv, B, k_rs, FWD_BN))) return rc;
  if ((rc = qkv_tmap(&tv, v, nh * HD, Skv, B, v_rs, FWD_BN))) return rc;
  if ((rc = set_smem<attn_fwd_tc_kernel<HD>>(FWD_SMEM))) return rc;
  TcParams p{};
  p.Sq = Sq; p.Skv = Skv; p.nh = nh; p.scale = scale; p.tile_rows = tile_rows;
  p.out0 = reinterpret_cast<bf16*>(o); p.out0_rs = o_rs; p.lse = lse;
  pdl_launch(dim3(ntile, nh, B), 128, FWD_SMEM, s)(attn_fwd_tc_kernel<HD>, tq, tk, tv, p);
  return check_launch("attn_fwd_tc");
}

// dQ (and D, into dvec) over q row tiles, then dK / dV over kv row tiles
template <int HD>
int attn_bwd_impl(const void* q, const void* k, const void* v, const void* d_o, const float* lse, float* dvec, void* dq,
                  void* dk, void* dv, int B, int nh, int Sq, int Skv, int q_rs, int k_rs, int v_rs, int do_rs, int dq_rs,
                  int dk_rs, int dv_rs, float scale, cudaStream_t s) {
  int ntile, tile_rows;
  balanced_tiles(Sq, &ntile, &tile_rows);
  CUtensorMap tq, tdo, tk, tv;
  int rc;
  if ((rc = qkv_tmap(&tq, q, nh * HD, Sq, B, q_rs, 128))) return rc;
  if ((rc = qkv_tmap(&tdo, d_o, nh * HD, Sq, B, do_rs, 128))) return rc;
  if ((rc = qkv_tmap(&tk, k, nh * HD, Skv, B, k_rs, BWD_BN))) return rc;
  if ((rc = qkv_tmap(&tv, v, nh * HD, Skv, B, v_rs, BWD_BN))) return rc;
  if ((rc = set_smem<attn_bwd_dq_tc_kernel<HD>>(DQ_SMEM))) return rc;
  TcParams p{};
  p.Sq = Sq; p.Skv = Skv; p.nh = nh; p.scale = scale;
  p.out0 = reinterpret_cast<bf16*>(dq); p.out0_rs = dq_rs; p.lse = const_cast<float*>(lse); p.dvec = dvec;
  p.tile_rows = tile_rows;
  pdl_launch(dim3(ntile, nh, B), 256, DQ_SMEM, s)(attn_bwd_dq_tc_kernel<HD>, tq, tdo, tk, tv, p);
  if ((rc = check_launch("attn_bwd_dq_tc"))) return rc;

  balanced_tiles(Skv, &ntile, &tile_rows);
  if ((rc = qkv_tmap(&tk, k, nh * HD, Skv, B, k_rs, 128))) return rc;
  if ((rc = qkv_tmap(&tv, v, nh * HD, Skv, B, v_rs, 128))) return rc;
  if ((rc = qkv_tmap(&tq, q, nh * HD, Sq, B, q_rs, BWD_BN))) return rc;
  if ((rc = qkv_tmap(&tdo, d_o, nh * HD, Sq, B, do_rs, BWD_BN))) return rc;
  if ((rc = set_smem<attn_bwd_dkdv_tc_kernel<HD>>(DKDV_SMEM))) return rc;
  p.out0 = reinterpret_cast<bf16*>(dk); p.out0_rs = dk_rs; p.out1 = reinterpret_cast<bf16*>(dv); p.out1_rs = dv_rs;
  p.tile_rows = tile_rows;
  pdl_launch(dim3(ntile, nh, B), 256, DKDV_SMEM, s)(attn_bwd_dkdv_tc_kernel<HD>, tk, tv, tq, tdo, p);
  return check_launch("attn_bwd_dkdv_tc");
}

int check_args(const char* who, int hd, int a, int b, int c) {
  if (hd != 64 && hd != 48) { set_last_error("%s: head_dim %d unsupported (64 and 48 are built)", who, hd); return MUSE_ERR_UNSUPPORTED; }
  if (((a | b | c) & 7) != 0) { set_last_error("%s: row strides must be multiples of 8 elements", who); return MUSE_ERR_INVALID; }
  return MUSE_OK;
}

}  // namespace

// Entry points of the C ABI: Attention.attention of the reference (muse/modeling_transformer.py:221-241) and its autograd
// backward, head_dim 64 or 48, no mask, no dropout.
int attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int nh, int Sq, int Skv, int hd,
             int q_rs, int k_rs, int v_rs, int o_rs, float scale, cudaStream_t s) {
  if (B <= 0 || Sq <= 0 || Skv <= 0) return MUSE_OK;
  int rc = check_args("attn_fwd", hd, q_rs | o_rs, k_rs, v_rs);
  if (rc) return rc;
  return hd == 64 ? attn_fwd_impl<64>(q, k, v, o, lse, B, nh, Sq, Skv, q_rs, k_rs, v_rs, o_rs, scale, s)
                  : attn_fwd_impl<48>(q, k, v, o, lse, B, nh, Sq, Skv, q_rs, k_rs, v_rs, o_rs, scale, s);
}

int attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
             float* dvec, void* dq, void* dk, void* dv, int B, int nh, int Sq, int Skv, int hd, int q_rs, int k_rs,
             int v_rs, int o_rs, int do_rs, int dq_rs, int dk_rs, int dv_rs, float scale, cudaStream_t s) {
  if (B <= 0 || Sq <= 0 || Skv <= 0) return MUSE_OK;
  int rc = check_args("attn_bwd", hd, q_rs | o_rs | do_rs | dq_rs, k_rs | dk_rs, v_rs | dv_rs);
  if (rc) return rc;
  (void)o;  // D is recomputed from (P, dP) inside the dQ kernel; O is not needed by backward
  return hd == 64 ? attn_bwd_impl<64>(q, k, v, d_o, lse, dvec, dq, dk, dv, B, nh, Sq, Skv, q_rs, k_rs, v_rs, do_rs, dq_rs,
                                      dk_rs, dv_rs, scale, s)
                  : attn_bwd_impl<48>(q, k, v, d_o, lse, dvec, dq, dk, dv, B, nh, Sq, Skv, q_rs, k_rs, v_rs, do_rs, dq_rs,
                                      dk_rs, dv_rs, scale, s);
}

}  // namespace muse
