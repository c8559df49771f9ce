// Fused multi-head attention, forward and backward, head_dim = 64, no mask, no dropout.
// Replaces the reference's materialised path (muse/modeling_transformer.py:221-241):
//   transpose+contiguous x3 -> baddbmm(zeros, q, k^T, alpha=1/sqrt(hd)) -> softmax -> matmul(P, V)
//   -> transpose+contiguous,
// i.e. three [B*nh, S, S] tensors and five layout copies per layer, with a flash-style kernel that
// keeps scores on-chip (online softmax, fp32 statistics) and reads Q/K/V straight out of the fused
// [tokens, 3H] QKV projection (strided per head) and writes [tokens, H] context directly.
// Used for self-attention (kv_len = S = 257/256/1024) and cross-attention (kv_len = 77, :886-899).
//
// TEST-ONLY: the first-generation mma.sync.m16n8k16 implementation, kept as an independent on-device cross-check of the
// product's wgmma kernels (open_muse_b200/csrc/attention_tc.cu).  Built into tests/xcheck/libmuse_b200_xcheck.so,
// never into libmuse_b200.so.
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace muse {
namespace {

constexpr int D = 64;     // head dim
constexpr int BQ = 64;    // rows per CTA (4 warps x 16)
constexpr int BKV = 64;   // kv rows per inner step
constexpr int LDS = 72;   // padded smem row stride (elements) = 144 B: conflict-free ldmatrix
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const bf16* p) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const bf16* p) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}

// Cooperative load of a [64 x 64] bf16 tile (rows row0.., row pitch rs elements) into padded smem;
// rows >= nrows are zero-filled.  128 threads.
__device__ __forceinline__ void load_tile(bf16* s, const bf16* g, int row0, int nrows, long long rs) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = threadIdx.x + i * 128;  // 512 16-byte chunks
    const int r = idx >> 3, c = (idx & 7) * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row0 + r < nrows) v = *reinterpret_cast<const uint4*>(g + static_cast<long long>(row0 + r) * rs + c);
    *reinterpret_cast<uint4*>(s + r * LDS + c) = v;
  }
}

// Asynchronous variant (cp.async, 16 B per request, zero-fill for rows >= nrows): lets the next K/V (or Q/dO)
// chunk stream in while the tensor cores work on the current one.
__device__ __forceinline__ void load_tile_async(bf16* s, const bf16* g, int row0, int nrows, long long rs) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = threadIdx.x + i * 128;
    const int r = idx >> 3, c = (idx & 7) * 8;
    const bool ok = row0 + r < nrows;
    const bf16* src = g + static_cast<long long>(ok ? row0 + r : 0) * rs + c;
    const uint32_t dst = static_cast<uint32_t>(__cvta_generic_to_shared(s + r * LDS + c));
    const int bytes = ok ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
  }
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// A fragments (16 rows x 64 k) of this warp's rows from a smem tile: a[ks][0..3]
__device__ __forceinline__ void load_a_frags(uint32_t (&a)[4][4], const bf16* s, int warp_row0, int lane) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const bf16* p = s + (warp_row0 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + ks * 16 + (lane >> 4) * 8;
    ldsm_x4(a[ks], p);
  }
}

// C[16 x 64] = A(frags, 16 x 64k) * T^T where T is a smem tile [64 n][64 k] (row = n, contiguous k).
// Only the first nb_lim 8-column blocks are computed (ragged last chunk: S = 257 leaves a 1-column tail).
__device__ __forceinline__ void gemm_a_tT(float (&c)[8][4], const uint32_t (&a)[4][4], const bf16* t, int lane,
                                          int nb_lim) {
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    if (nb >= nb_lim) break;
#pragma unroll
    for (int kp = 0; kp < 2; ++kp) {  // pairs of k-steps
      uint32_t b[4];
      ldsm_x4(b, t + (nb * 8 + (lane & 7)) * LDS + kp * 32 + (lane >> 3) * 8);
      mma16816(c[nb], a[kp * 2], b[0], b[1]);
      mma16816(c[nb], a[kp * 2 + 1], b[2], b[3]);
    }
  }
}

// C[16 x 64] += A(frags, 16 x 64k) * T where T is a smem tile [64 k][64 n] (row = k, contiguous n).
// Only the first ks_lim 16-row k-steps are computed.
__device__ __forceinline__ void gemm_a_t(float (&c)[8][4], const uint32_t (&a)[4][4], const bf16* t, int lane,
                                         int ks_lim) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    if (ks >= ks_lim) break;
#pragma unroll
    for (int np = 0; np < 4; ++np) {  // pairs of n-blocks
      uint32_t b[4];
      ldsm_x4_t(b, t + (ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + np * 16 + (lane >> 4) * 8);
      mma16816(c[np * 2], a[ks], b[0], b[1]);
      mma16816(c[np * 2 + 1], a[ks], b[2], b[3]);
    }
  }
}

// fp32 C fragments [16 x 64] -> bf16 A fragments (16 x 64k)
__device__ __forceinline__ void c_to_a(uint32_t (&a)[4][4], const float (&c)[8][4]) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = pack_bf16(c[2 * ks][0], c[2 * ks][1]);
    a[ks][1] = pack_bf16(c[2 * ks][2], c[2 * ks][3]);
    a[ks][2] = pack_bf16(c[2 * ks + 1][0], c[2 * ks + 1][1]);
    a[ks][3] = pack_bf16(c[2 * ks + 1][2], c[2 * ks + 1][3]);
  }
}

struct AttnPtrs {
  const bf16* q; const bf16* k; const bf16* v;
  long long q_bs, k_bs, v_bs;  // batch strides (elements)
  int q_rs, k_rs, v_rs;        // row strides (elements)
};

// ------------------------------------------------------------------ forward
__global__ void __launch_bounds__(128)
attn_fwd_kernel(AttnPtrs P, bf16* __restrict__ O, long long o_bs, int o_rs, float* __restrict__ LSE, int Sq, int Skv,
                int nh, float scale, int blk0) {
  __shared__ __align__(16) bf16 sQ[BQ * LDS];
  __shared__ __align__(16) bf16 sK[2][BKV * LDS];
  __shared__ __align__(16) bf16 sV[2][BKV * LDS];
  const int q0 = (blockIdx.x + blk0) * BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const bf16* qg = P.q + b * P.q_bs + h * D;
  const bf16* kg = P.k + b * P.k_bs + h * D;
  const bf16* vg = P.v + b * P.v_bs + h * D;
  const bool warp_active = q0 + warp * 16 < Sq;  // ragged last q block: idle warps only help with the loads
  const int nchunks = ceil_div(Skv, BKV);

  load_tile_async(sQ, qg, q0, Sq, P.q_rs);
  load_tile_async(sK[0], kg, 0, Skv, P.k_rs);
  load_tile_async(sV[0], vg, 0, Skv, P.v_rs);
  cp_async_commit();

  const float sl2 = scale * kLog2e;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  uint32_t qf[4][4];

  for (int c = 0; c < nchunks; ++c) {
    const int kv0 = c * BKV;
    if (c + 1 < nchunks) {
      load_tile_async(sK[(c + 1) & 1], kg, kv0 + BKV, Skv, P.k_rs);
      load_tile_async(sV[(c + 1) & 1], vg, kv0 + BKV, Skv, P.v_rs);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (c == 0) load_a_frags(qf, sQ, warp * 16, lane);
    if (warp_active) {
      const bf16* tK = sK[c & 1];
      const bf16* tV = sV[c & 1];
      const int nvalid = min(BKV, Skv - kv0);
      const int nb_lim = (nvalid + 7) >> 3, ks_lim = (nvalid + 15) >> 4;
      float s[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
      gemm_a_tT(s, qf, tK, lane, nb_lim);
      float mx[2] = {m[0], m[1]};
#pragma unroll
      for (int nb = 0; nb < 8; ++nb)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int col = kv0 + nb * 8 + 2 * t + (j & 1);
          const float v = (col < Skv) ? s[nb][j] * sl2 : -INFINITY;
          s[nb][j] = v;
          mx[j >> 1] = fmaxf(mx[j >> 1], v);
        }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      }
      float corr[2], rs[2] = {0.f, 0.f};
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        corr[r] = exp2f(m[r] - mx[r]);  // m = -inf on the first chunk -> 0
        m[r] = mx[r];
      }
#pragma unroll
      for (int nb = 0; nb < 8; ++nb)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float p = exp2f(s[nb][j] - m[j >> 1]);
          s[nb][j] = p;
          rs[j >> 1] += p;
        }
#pragma unroll
      for (int r = 0; r < 2; ++r) l[r] = l[r] * corr[r] + rs[r];
#pragma unroll
      for (int nb = 0; nb < 8; ++nb)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[nb][j] *= corr[j >> 1];
      uint32_t pf[4][4];
      c_to_a(pf, s);
      gemm_a_t(o, pf, tV, lane, ks_lim);
    }
    __syncthreads();  // everyone is done with buffer c&1 before iteration c+1 prefetches into it
  }
  if (!warp_active) return;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
  const float inv[2] = {1.f / l[0], 1.f / l[1]};
  // stage the output tile through this warp's rows of sQ (already consumed into registers)
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    *reinterpret_cast<uint32_t*>(sQ + (warp * 16 + g) * LDS + nb * 8 + 2 * t) = pack_bf16(o[nb][0] * inv[0], o[nb][1] * inv[0]);
    *reinterpret_cast<uint32_t*>(sQ + (warp * 16 + g + 8) * LDS + nb * 8 + 2 * t) = pack_bf16(o[nb][2] * inv[1], o[nb][3] * inv[1]);
  }
  __syncwarp();
  bf16* og = O + b * o_bs + h * D;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = lane + i * 32;  // 16 rows x 8 chunks
    const int r = warp * 16 + (idx >> 3), c = (idx & 7) * 8;
    if (q0 + r < Sq)
      *reinterpret_cast<uint4*>(og + static_cast<long long>(q0 + r) * o_rs + c) = *reinterpret_cast<const uint4*>(sQ + r * LDS + c);
  }
  if (t == 0) {
    const int r0 = q0 + warp * 16 + g;
    float* lse = LSE + (static_cast<long long>(b) * nh + h) * Sq;
    if (r0 < Sq) lse[r0] = (m[0] + log2f(l[0])) * kLn2;
    if (r0 + 8 < Sq) lse[r0 + 8] = (m[1] + log2f(l[1])) * kLn2;
  }
}

// ------------------------------------------------------------------ backward: dK, dV (CTA owns 64 kv rows)
__global__ void __launch_bounds__(128)
attn_bwd_dkdv_kernel(AttnPtrs P, const bf16* __restrict__ dO, long long do_bs, int do_rs, const float* __restrict__ LSE,
                     const float* __restrict__ Dv, bf16* __restrict__ dK, long long dk_bs, int dk_rs,
                     bf16* __restrict__ dV, long long dv_bs, int dv_rs, int Sq, int Skv, int nh, float scale, int blk0) {
  __shared__ __align__(16) bf16 sA[2][BKV * LDS];  // K_j (buffer 1) then Q_i chunks (alternating)
  __shared__ __align__(16) bf16 sB[2][BKV * LDS];  // V_j (buffer 1) then dO_i chunks
  __shared__ float sL[2][BQ], sD[2][BQ];
  const int kv0 = (blockIdx.x + blk0) * BKV, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const bf16* qg = P.q + b * P.q_bs + h * D;
  const bf16* kg = P.k + b * P.k_bs + h * D;
  const bf16* vg = P.v + b * P.v_bs + h * D;
  const bf16* dog = dO + b * do_bs + h * D;
  const float* lse = LSE + (static_cast<long long>(b) * nh + h) * Sq;
  const float* dv_ = Dv + (static_cast<long long>(b) * nh + h) * Sq;
  const bool warp_active = kv0 + warp * 16 < Skv;
  const int nchunks = ceil_div(Sq, BQ);

  load_tile_async(sA[1], kg, kv0, Skv, P.k_rs);
  load_tile_async(sB[1], vg, kv0, Skv, P.v_rs);
  cp_async_commit();
  load_tile_async(sA[0], qg, 0, Sq, P.q_rs);
  load_tile_async(sB[0], dog, 0, Sq, do_rs);
  cp_async_commit();
  if (threadIdx.x < BQ) {
    sL[0][threadIdx.x] = (threadIdx.x < Sq) ? lse[threadIdx.x] * kLog2e : 0.f;
    sD[0][threadIdx.x] = (threadIdx.x < Sq) ? dv_[threadIdx.x] : 0.f;
  }
  cp_async_wait<1>();
  __syncthreads();
  uint32_t kf[4][4], vf[4][4];
  load_a_frags(kf, sA[1], warp * 16, lane);
  load_a_frags(vf, sB[1], warp * 16, lane);
  __syncthreads();  // K_j / V_j are in registers: buffer 1 may be overwritten by the prefetch of chunk 1

  const float sl2 = scale * kLog2e;
  float dk[8][4], dvv[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { dk[i][j] = 0.f; dvv[i][j] = 0.f; }
  const int kvr0 = kv0 + warp * 16 + g;  // this thread's kv rows: kvr0, kvr0 + 8

  for (int c = 0; c < nchunks; ++c) {
    const int q0 = c * BQ;
    if (c + 1 < nchunks) {
      load_tile_async(sA[(c + 1) & 1], qg, q0 + BQ, Sq, P.q_rs);
      load_tile_async(sB[(c + 1) & 1], dog, q0 + BQ, Sq, do_rs);
      cp_async_commit();
      if (threadIdx.x < BQ) {
        const int r = q0 + BQ + threadIdx.x;
        sL[(c + 1) & 1][threadIdx.x] = (r < Sq) ? lse[r] * kLog2e : 0.f;
        sD[(c + 1) & 1][threadIdx.x] = (r < Sq) ? dv_[r] : 0.f;
      }
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (warp_active) {
      const bf16* tQ = sA[c & 1];
      const bf16* tdO = sB[c & 1];
      const float* cL = sL[c & 1];
      const float* cD = sD[c & 1];
      const int nvalid = min(BQ, Sq - q0);
      const int nb_lim = (nvalid + 7) >> 3, ks_lim = (nvalid + 15) >> 4;
      // S^T = K_j Q_i^T  (rows: kv, cols: q)
      float st[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) st[i][j] = 0.f;
      gemm_a_tT(st, kf, tQ, lane, nb_lim);
#pragma unroll
      for (int nb = 0; nb < 8; ++nb)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int qc = nb * 8 + 2 * t + (j & 1);
          const int kr = kvr0 + (j >> 1) * 8;
          const bool ok = (q0 + qc < Sq) && (kr < Skv);
          st[nb][j] = ok ? exp2f(st[nb][j] * sl2 - cL[qc]) : 0.f;
        }
      uint32_t pf[4][4];
      c_to_a(pf, st);
      gemm_a_t(dvv, pf, tdO, lane, ks_lim);  // dV += P^T dO
      // dP^T = V_j dO_i^T
      float dp[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dp[i][j] = 0.f;
      gemm_a_tT(dp, vf, tdO, lane, nb_lim);
#pragma unroll
      for (int nb = 0; nb < 8; ++nb)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int qc = nb * 8 + 2 * t + (j & 1);
          dp[nb][j] = st[nb][j] * (dp[nb][j] - cD[qc]) * scale;
        }
      c_to_a(pf, dp);
      gemm_a_t(dk, pf, tQ, lane, ks_lim);  // dK += dS^T Q
    }
    __syncthreads();
  }
  if (!warp_active) return;
  // write dK, dV (bf16) through this warp's rows of smem for 16B stores (all chunk buffers are idle now)
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    *reinterpret_cast<uint32_t*>(sA[0] + (warp * 16 + g) * LDS + nb * 8 + 2 * t) = pack_bf16(dk[nb][0], dk[nb][1]);
    *reinterpret_cast<uint32_t*>(sA[0] + (warp * 16 + g + 8) * LDS + nb * 8 + 2 * t) = pack_bf16(dk[nb][2], dk[nb][3]);
    *reinterpret_cast<uint32_t*>(sB[0] + (warp * 16 + g) * LDS + nb * 8 + 2 * t) = pack_bf16(dvv[nb][0], dvv[nb][1]);
    *reinterpret_cast<uint32_t*>(sB[0] + (warp * 16 + g + 8) * LDS + nb * 8 + 2 * t) = pack_bf16(dvv[nb][2], dvv[nb][3]);
  }
  __syncwarp();
  bf16* dkg = dK + b * dk_bs + h * D;
  bf16* dvg = dV + b * dv_bs + h * D;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = lane + i * 32;
    const int r = warp * 16 + (idx >> 3), c = (idx & 7) * 8;
    if (kv0 + r < Skv) {
      *reinterpret_cast<uint4*>(dkg + static_cast<long long>(kv0 + r) * dk_rs + c) = *reinterpret_cast<const uint4*>(sA[0] + r * LDS + c);
      *reinterpret_cast<uint4*>(dvg + static_cast<long long>(kv0 + r) * dv_rs + c) = *reinterpret_cast<const uint4*>(sB[0] + r * LDS + c);
    }
  }
}

// ------------------------------------------------------------------ backward: dQ (CTA owns 64 q rows)
// Two sweeps over the kv chunks.  Sweep 1: D_i = sum_j P_ij * dP_ij from the SAME fp32 P and dP that sweep 2 uses, so
// sum_j dS_ij == 0 up to fp32 rounding (softmax backward as the reference's fp32 autograd computes it); the usual
// rowsum(dO * O) with the bf16-rounded O leaves a systematic P_ij * eps_i term that swamps the (tiny) true dQ/dK when
// attention is near-uniform (random init).  D is also written out for the dK/dV kernel.  Sweep 2: dS, dQ += dS K.
__global__ void __launch_bounds__(128)
attn_bwd_dq_kernel(AttnPtrs P, const bf16* __restrict__ dO, long long do_bs, int do_rs, const float* __restrict__ LSE,
                   float* __restrict__ Dv, bf16* __restrict__ dQ, long long dq_bs, int dq_rs, int Sq, int Skv,
                   int nh, float scale, int blk0) {
  __shared__ __align__(16) bf16 sA[2][BKV * LDS];  // Q_i (buffer 1) then K_j chunks
  __shared__ __align__(16) bf16 sB[2][BKV * LDS];  // dO_i (buffer 1) then V_j chunks
  const int q0 = (blockIdx.x + blk0) * BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const bf16* qg = P.q + b * P.q_bs + h * D;
  const bf16* kg = P.k + b * P.k_bs + h * D;
  const bf16* vg = P.v + b * P.v_bs + h * D;
  const bf16* dog = dO + b * do_bs + h * D;
  const float* lse = LSE + (static_cast<long long>(b) * nh + h) * Sq;
  float* dv_ = Dv + (static_cast<long long>(b) * nh + h) * Sq;
  const bool warp_active = q0 + warp * 16 < Sq;
  const int nchunks = ceil_div(Skv, BKV);
  const int nsteps = 2 * nchunks;

  load_tile_async(sA[1], qg, q0, Sq, P.q_rs);
  load_tile_async(sB[1], dog, q0, Sq, do_rs);
  cp_async_commit();
  load_tile_async(sA[0], kg, 0, Skv, P.k_rs);
  load_tile_async(sB[0], vg, 0, Skv, P.v_rs);
  cp_async_commit();
  cp_async_wait<1>();
  __syncthreads();
  uint32_t qf[4][4], dof[4][4];
  load_a_frags(qf, sA[1], warp * 16, lane);
  load_a_frags(dof, sB[1], warp * 16, lane);
  __syncthreads();
  const int r0 = q0 + warp * 16 + g;
  float l2[2], dd[2] = {0.f, 0.f};
  l2[0] = (r0 < Sq) ? lse[r0] * kLog2e : 0.f;
  l2[1] = (r0 + 8 < Sq) ? lse[r0 + 8] * kLog2e : 0.f;
  const float sl2 = scale * kLog2e;
  float dq[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) dq[i][j] = 0.f;

  for (int st = 0; st < nsteps; ++st) {
    const int c = st % nchunks;
    const int kv0 = c * BKV;
    if (st + 1 < nsteps) {
      const int nkv0 = ((st + 1) % nchunks) * BKV;
      load_tile_async(sA[(st + 1) & 1], kg, nkv0, Skv, P.k_rs);
      load_tile_async(sB[(st + 1) & 1], vg, nkv0, Skv, P.v_rs);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (warp_active) {
      const bf16* tK = sA[st & 1];
      const bf16* tV = sB[st & 1];
      const int nvalid = min(BKV, Skv - kv0);
      const int nb_lim = (nvalid + 7) >> 3, ks_lim = (nvalid + 15) >> 4;
      float s[8][4], dp[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) { s[i][j] = 0.f; dp[i][j] = 0.f; }
      gemm_a_tT(s, qf, tK, lane, nb_lim);     // S = Q K^T
      gemm_a_tT(dp, dof, tV, lane, nb_lim);   // dP = dO V^T
      if (st < nchunks) {
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int col = kv0 + nb * 8 + 2 * t + (j & 1);
            const int rr = r0 + (j >> 1) * 8;
            const bool ok = (col < Skv) && (rr < Sq);
            const float p = ok ? exp2f(s[nb][j] * sl2 - l2[j >> 1]) : 0.f;
            dd[j >> 1] += p * dp[nb][j];
          }
        if (st == nchunks - 1) {
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            dd[r] += __shfl_xor_sync(0xffffffffu, dd[r], 1);
            dd[r] += __shfl_xor_sync(0xffffffffu, dd[r], 2);
          }
          if (t == 0) {
            if (r0 < Sq) dv_[r0] = dd[0];
            if (r0 + 8 < Sq) dv_[r0 + 8] = dd[1];
          }
        }
      } else {
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int col = kv0 + nb * 8 + 2 * t + (j & 1);
            const int rr = r0 + (j >> 1) * 8;
            const bool ok = (col < Skv) && (rr < Sq);
            const float p = ok ? exp2f(s[nb][j] * sl2 - l2[j >> 1]) : 0.f;
            s[nb][j] = p * (dp[nb][j] - dd[j >> 1]) * scale;
          }
        uint32_t dsf[4][4];
        c_to_a(dsf, s);
        gemm_a_t(dq, dsf, tK, lane, ks_lim);  // dQ += dS K
      }
    }
    __syncthreads();
  }
  if (!warp_active) return;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    *reinterpret_cast<uint32_t*>(sA[0] + (warp * 16 + g) * LDS + nb * 8 + 2 * t) = pack_bf16(dq[nb][0], dq[nb][1]);
    *reinterpret_cast<uint32_t*>(sA[0] + (warp * 16 + g + 8) * LDS + nb * 8 + 2 * t) = pack_bf16(dq[nb][2], dq[nb][3]);
  }
  __syncwarp();
  bf16* dqg = dQ + b * dq_bs + h * D;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = lane + i * 32;
    const int r = warp * 16 + (idx >> 3), c = (idx & 7) * 8;
    if (q0 + r < Sq)
      *reinterpret_cast<uint4*>(dqg + static_cast<long long>(q0 + r) * dq_rs + c) = *reinterpret_cast<const uint4*>(sA[0] + r * LDS + c);
  }
}

int check_strides(const char* who, int hd, int a, int b, int c) {
  if (hd != D) { set_last_error("%s: head_dim=%d unsupported (only 64)", who, hd); return MUSE_ERR_UNSUPPORTED; }
  if ((a | b | c) % 8 != 0) { set_last_error("%s: row strides must be multiples of 8 elements", who); return MUSE_ERR_INVALID; }
  return MUSE_OK;
}

}  // namespace

// TEST-ONLY cross-check library (tests/xcheck): the mma.sync kernels above behind the product's attention contract.
int attn_fwd_legacy(const void* q, const void* k, const void* v, void* o, float* lse, int B, int nh, int Sq, int Skv, int hd,
             int q_rs, int k_rs, int v_rs, int o_rs, float scale, cudaStream_t s) {
  if (B <= 0 || Sq <= 0 || Skv <= 0) return MUSE_OK;
  int rc = check_strides("attn_fwd", hd, q_rs | o_rs, k_rs, v_rs);
  if (rc) return rc;
  const int done = 0;
  AttnPtrs P;
  P.q = reinterpret_cast<const bf16*>(q); P.k = reinterpret_cast<const bf16*>(k); P.v = reinterpret_cast<const bf16*>(v);
  P.q_rs = q_rs; P.k_rs = k_rs; P.v_rs = v_rs;
  P.q_bs = static_cast<long long>(Sq) * q_rs; P.k_bs = static_cast<long long>(Skv) * k_rs; P.v_bs = static_cast<long long>(Skv) * v_rs;
  const int blk0 = done / BQ;
  dim3 grid(ceil_div(Sq, BQ) - blk0, nh, B);
  attn_fwd_kernel<<<grid, 128, 0, s>>>(P, reinterpret_cast<bf16*>(o), static_cast<long long>(Sq) * o_rs, o_rs, lse, Sq, Skv, nh, scale, blk0);
  return check_launch("attn_fwd");
}

int attn_bwd_legacy(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
             float* dvec, void* dq, void* dk, void* dv, int B, int nh, int Sq, int Skv, int hd, int q_rs, int k_rs,
             int v_rs, int o_rs, int do_rs, int dq_rs, int dk_rs, int dv_rs, float scale, cudaStream_t s) {
  if (B <= 0 || Sq <= 0 || Skv <= 0) return MUSE_OK;
  int rc = check_strides("attn_bwd", hd, q_rs | o_rs | do_rs | dq_rs, k_rs | dk_rs, v_rs | dv_rs);
  if (rc) return rc;
  (void)o; (void)o_rs;  // D is recomputed from (P, dP) inside the dQ kernels; O is not needed by backward
  AttnPtrs P;
  P.q = reinterpret_cast<const bf16*>(q); P.k = reinterpret_cast<const bf16*>(k); P.v = reinterpret_cast<const bf16*>(v);
  P.q_rs = q_rs; P.k_rs = k_rs; P.v_rs = v_rs;
  P.q_bs = static_cast<long long>(Sq) * q_rs; P.k_bs = static_cast<long long>(Skv) * k_rs; P.v_bs = static_cast<long long>(Skv) * v_rs;
  const int done_q = 0, done_kv = 0;
  {
    const int blk0 = done_q / BQ;
    attn_bwd_dq_kernel<<<dim3(ceil_div(Sq, BQ) - blk0, nh, B), 128, 0, s>>>(
        P, reinterpret_cast<const bf16*>(d_o), static_cast<long long>(Sq) * do_rs, do_rs, lse, dvec,
        reinterpret_cast<bf16*>(dq), static_cast<long long>(Sq) * dq_rs, dq_rs, Sq, Skv, nh, scale, blk0);
    rc = check_launch("attn_bwd_dq");
    if (rc) return rc;
  }
  {
    const int blk0 = done_kv / BKV;
    attn_bwd_dkdv_kernel<<<dim3(ceil_div(Skv, BKV) - blk0, nh, B), 128, 0, s>>>(
        P, reinterpret_cast<const bf16*>(d_o), static_cast<long long>(Sq) * do_rs, do_rs, lse, dvec,
        reinterpret_cast<bf16*>(dk), static_cast<long long>(Skv) * dk_rs, dk_rs, reinterpret_cast<bf16*>(dv),
        static_cast<long long>(Skv) * dv_rs, dv_rs, Sq, Skv, nh, scale, blk0);
    rc = check_launch("attn_bwd_dkdv");
    if (rc) return rc;
  }
  return MUSE_OK;
}

}  // namespace muse
