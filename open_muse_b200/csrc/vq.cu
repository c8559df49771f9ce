// Vector-quantiser nearest-codebook search (MaskGitVQGAN tokenise) with a bit-exact contract.
// Reference: VectorQuantizer.compute_distances + argmin, muse/modeling_maskgit_vqgan.py:303-316,342-348:
//     d[r,c] = (||z_r||^2 + ||e_c||^2) - 2 <z_r, e_c>   ;   id[r] = argmin_c d[r,c]  (first minimum)
// Arithmetic is pinned so that this kernel and oracle/vq_oracle.c agree bit-for-bit on EVERY input:
//     norm  = fma chain over k = 0..D-1 in ascending order, starting from 0
//     dot   = fma chain over k = 0..D-1 in ascending order, starting from 0
//     d     = fmaf(-2, dot, fl(znorm + enorm))
//     argmin keeps the lowest index among equal distances.
// fp32 SIMT (no tensor cores: TF32/bf16 products would change token ids - SURVEY H1).
// 128 x 128 register-tiled SGEMM (8 x 8 micro-tile per thread); each accumulator is its own
// ascending-k fma chain, so tiling does not perturb the summation order.
#include "common.cuh"

namespace muse {
namespace {

constexpr int TR = 128;  // rows (tokens) per CTA
constexpr int TC = 128;  // codes per inner chunk
constexpr int TKK = 16;  // k per smem stage

__global__ void __launch_bounds__(256) sqnorm_kernel(const float* __restrict__ x, float* __restrict__ out, int n, int D) {
  pdl_enter();
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const float* r = x + static_cast<size_t>(i) * D;
  float acc = 0.f;
  for (int k = 0; k < D; ++k) acc = fmaf(r[k], r[k], acc);
  out[i] = acc;
}

__global__ void __launch_bounds__(256)
vq_argmin_kernel(const float* __restrict__ z, const float* __restrict__ cb, const float* __restrict__ enorm,
                 long long* __restrict__ ids, float* __restrict__ dmin_out, float* __restrict__ dist_out, int n,
                 int ncodes, int D) {
  pdl_enter();
  __shared__ __align__(16) float sZ[TKK][TR];
  __shared__ __align__(16) float sE[TKK][TC];
  __shared__ float sZn[TR];
  __shared__ float sBestV[TR][17];
  __shared__ int sBestI[TR][17];
  const int row0 = blockIdx.x * TR;
  const int tx = threadIdx.x & 15;   // code direction
  const int ty = threadIdx.x >> 4;   // row direction
  if (threadIdx.x < TR) {
    const int r = row0 + threadIdx.x;
    float acc = 0.f;
    if (r < n) {
      const float* zr = z + static_cast<size_t>(r) * D;
      for (int k = 0; k < D; ++k) acc = fmaf(zr[k], zr[k], acc);
    }
    sZn[threadIdx.x] = acc;
  }
  float bestv[8];
  int besti[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { bestv[i] = INFINITY; besti[i] = 0; }

  for (int c0 = 0; c0 < ncodes; c0 += TC) {
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < D; k0 += TKK) {
      __syncthreads();
#pragma unroll
      for (int it = 0; it < 2; ++it) {
        const int idx = threadIdx.x + it * 256;  // 128 rows x 4 float4
        const int r = idx >> 2, kq = (idx & 3) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        // k past D (D % 16 != 0, e.g. the Paella latent D = 4) loads zeros: fmaf(0, 0, acc) == acc, so every chain is
        // the same as if it stopped at D
        const bool kin = k0 + kq < D;
        if (row0 + r < n && kin) v = *reinterpret_cast<const float4*>(z + static_cast<size_t>(row0 + r) * D + k0 + kq);
        sZ[kq + 0][r] = v.x; sZ[kq + 1][r] = v.y; sZ[kq + 2][r] = v.z; sZ[kq + 3][r] = v.w;
        float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c0 + r < ncodes && kin) e = *reinterpret_cast<const float4*>(cb + static_cast<size_t>(c0 + r) * D + k0 + kq);
        sE[kq + 0][r] = e.x; sE[kq + 1][r] = e.y; sE[kq + 2][r] = e.z; sE[kq + 3][r] = e.w;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < TKK; ++kk) {
        float a[8], b[8];
        *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&sZ[kk][ty * 8]);
        *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&sZ[kk][ty * 8 + 4]);
        *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&sE[kk][tx * 8]);
        *reinterpret_cast<float4*>(&b[4]) = *reinterpret_cast<const float4*>(&sE[kk][tx * 8 + 4]);
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float zn = sZn[ty * 8 + i];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int code = c0 + tx * 8 + j;
        if (code < ncodes) {
          const float d = fmaf(-2.0f, acc[i][j], zn + enorm[code]);
          if (d < bestv[i]) { bestv[i] = d; besti[i] = code; }  // strict: lowest index wins ties
          if (dist_out != nullptr && row0 + ty * 8 + i < n)
            dist_out[static_cast<size_t>(row0 + ty * 8 + i) * ncodes + code] = d;
        }
      }
    }
  }
  // reduce across the 16 threads (tx) that share a row: (value, index) lexicographic min
#pragma unroll
  for (int i = 0; i < 8; ++i) { sBestV[ty * 8 + i][tx] = bestv[i]; sBestI[ty * 8 + i][tx] = besti[i]; }
  __syncthreads();
  if (threadIdx.x < TR) {
    const int r = row0 + threadIdx.x;
    if (r < n) {
      float bv = sBestV[threadIdx.x][0];
      int bi = sBestI[threadIdx.x][0];
      for (int q = 1; q < 16; ++q) {
        const float v = sBestV[threadIdx.x][q];
        const int ix = sBestI[threadIdx.x][q];
        if (v < bv || (v == bv && ix < bi)) { bv = v; bi = ix; }
      }
      ids[r] = bi;
      if (dmin_out) dmin_out[r] = bv;
    }
  }
}

// VectorQuantizer.get_soft_code (muse/modeling_maskgit_vqgan.py:327-340): soft = softmax(-d / temp) over the codebook,
// in place over the distance matrix written by vq_argmin_kernel; optional stochastic code = multinomial(soft, 1),
// realised as argmax_c soft[c] / q[c] with q ~ Exp(1) pre-drawn by the caller (the construction torch.multinomial
// itself uses for one sample). One warp per row.
__global__ void __launch_bounds__(256)
vq_soft_kernel(float* __restrict__ dist, const float* __restrict__ expo, long long* __restrict__ ids, float temp, int n,
               int ncodes) {
  pdl_enter();
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= n) return;
  const int lane = threadIdx.x & 31;
  float* row = dist + static_cast<size_t>(r) * ncodes;
  float m = -INFINITY;
  for (int c = lane; c < ncodes; c += 32) m = fmaxf(m, -row[c] / temp);
  m = warp_max(m);
  float sum = 0.f;
  for (int c = lane; c < ncodes; c += 32) sum += expf(-row[c] / temp - m);
  sum = warp_sum(sum);
  float bestv = -INFINITY;
  int besti = 0x7fffffff;
  const float* q = expo ? expo + static_cast<size_t>(r) * ncodes : nullptr;
  for (int c = lane; c < ncodes; c += 32) {
    const float p = expf(-row[c] / temp - m) / sum;
    row[c] = p;
    if (q) {
      const float v = p / q[c];
      if (v > bestv) { bestv = v; besti = c; }
    }
  }
  if (q) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bestv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
      if (ov > bestv || (ov == bestv && oi < besti)) { bestv = ov; besti = oi; }
    }
    if (lane == 0) ids[r] = besti;
  }
}

// z_q[b, c, p] = codebook[ids[b, p], c]  (get_codebook_entry + permute to NCHW, :318-324)
__global__ void __launch_bounds__(256)
vq_lookup_nchw_kernel(const long long* __restrict__ ids, const float* __restrict__ cb, float* __restrict__ out, int B,
                      int P, int D, int ncodes) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  const long long total = static_cast<long long>(B) * D * P;
  if (i >= total) return;
  const int p = static_cast<int>(i % P);
  const int c = static_cast<int>((i / P) % D);
  const int b = static_cast<int>(i / (static_cast<long long>(P) * D));
  long long id = ids[static_cast<long long>(b) * P + p];
  if (id < 0 || id >= ncodes) id = 0;
  out[i] = cb[id * D + c];
}

}  // namespace
}  // namespace muse

using namespace muse;

extern "C" {

int muse_vq_argmin(const float* z, const float* codebook, float* enorm_ws, long long* ids, float* dmin, int n, int ncodes,
                   int D, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0) return MUSE_OK;
  if (D % 4 != 0 || D <= 0) { set_last_error("vq_argmin: D=%d must be a positive multiple of 4", D); return MUSE_ERR_UNSUPPORTED; }
  pdl_launch(ceil_div(ncodes, 256), 256, 0, s)(sqnorm_kernel, codebook, enorm_ws, ncodes, D);
  int rc = check_launch("vq_sqnorm");
  if (rc) return rc;
  pdl_launch(ceil_div(n, TR), 256, 0, s)(vq_argmin_kernel, z, codebook, enorm_ws, ids, dmin, nullptr, n, ncodes, D);
  return check_launch("vq_argmin");
}

int muse_vq_soft_code(const float* z, const float* codebook, float* enorm_ws, float* soft, long long* ids, const float* expo,
                      float temp, int n, int ncodes, int D, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0) return MUSE_OK;
  if (D % 4 != 0 || D <= 0) { set_last_error("vq_soft_code: D=%d must be a positive multiple of 4", D); return MUSE_ERR_UNSUPPORTED; }
  if (!(temp > 0.f)) { set_last_error("vq_soft_code: temp must be > 0"); return MUSE_ERR_INVALID; }
  pdl_launch(ceil_div(ncodes, 256), 256, 0, s)(sqnorm_kernel, codebook, enorm_ws, ncodes, D);
  int rc = check_launch("vq_sqnorm");
  if (rc) return rc;
  pdl_launch(ceil_div(n, TR), 256, 0, s)(vq_argmin_kernel, z, codebook, enorm_ws, ids, nullptr, soft, n, ncodes, D);
  rc = check_launch("vq_argmin(dist)");
  if (rc) return rc;
  pdl_launch(ceil_div(n, 8), 256, 0, s)(vq_soft_kernel, soft, expo, ids, temp, n, ncodes);
  return check_launch("vq_soft");
}

int muse_vq_lookup_nchw(const long long* ids, const float* codebook, float* out, int B, int P, int D, int ncodes,
                        void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long total = static_cast<long long>(B) * D * P;
  if (total <= 0) return MUSE_OK;
  pdl_launch(static_cast<unsigned>(ceil_div_ll(total, 256)), 256, 0, s)(vq_lookup_nchw_kernel, ids, codebook, out, B, P, D, ncodes);
  return check_launch("vq_lookup_nchw");
}

}  // extern "C"
