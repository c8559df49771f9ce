// MaskGitVQGAN encoder / decoder building blocks in fp32, NHWC (muse/modeling_maskgit_vqgan.py):
//   * conv2d 'same' stride-1, k = 3 or 1 (Conv2dSame :33-45) as an implicit GEMM:
//       M = B*H*W output pixels, N = C_out, K = k*k*C_in  (weights pre-packed to [K, C_out])
//     with fused bias, fused residual add (ResnetBlock :82-85) and the nearest x2 upsample of
//     UpsamplingBlock (:146) folded into the input gather (index >> 1) so the 4x larger tensor is never written.
//   * GroupNorm(32, eps=1e-6) + SiLU (:61-79): deterministic statistics pass (per-block partials, fp64 final sum)
//     + one apply pass.
//   * avg_pool2d(2,2) (:112), NCHW <-> NHWC layout changes at the model boundary.
// fp32 SIMT on purpose: token ids must agree with the fp32 reference (SURVEY H1); each output is one ascending-K
// fma chain (taps row-major, then input channel), so results do not depend on tiling.
// This is the general-shape kernel (3-channel stem / head, odd geometries); the heavy layers run on the tensor cores
// with the same fp32-level accuracy in conv_tc.cu.
#include "common.cuh"

namespace muse {
namespace {

constexpr int KT = 8;  // k per smem stage

template <int TM, int TN, bool VEC>
__global__ void __launch_bounds__(256)
conv2d_nhwc_kernel(const float* __restrict__ x, const float* __restrict__ wk, const float* __restrict__ bias,
                   const float* __restrict__ res, float* __restrict__ y, int B, int H, int W, int Cin, int Cout,
                   int ksize, int mode) {
  pdl_enter();
  constexpr int BM = 16 * TM, BN = 16 * TN;
  __shared__ __align__(16) float sA[KT][BM];
  __shared__ __align__(16) float sB[KT][BN];
  // mode: enum muse_conv_mode of include/muse_b200.h.  MUSE_CONV_TRANSPOSE_S2 runs as four 2x2 parity convolutions on the
  // H/2 x W/2 input, parity blockIdx.z.
  const int md = mode & MUSE_CONV_GEOMETRY, gelu = mode & MUSE_CONV_GELU, shuf = mode & MUSE_CONV_PIXEL_SHUFFLE;
  const int s2 = (md == MUSE_CONV_STRIDE2 || md == MUSE_CONV_S2P1), tr = (md == MUSE_CONV_TRANSPOSE_S2);
  const int par = tr ? static_cast<int>(blockIdx.z) : 0;
  const int Hg = tr ? H / 2 : H, Wg = tr ? W / 2 : W;  // the grid the output rows m run over
  const long long M = static_cast<long long>(B) * Hg * Wg;
  const int kk_size = tr ? 2 : ksize;
  const int K = kk_size * kk_size * Cin;
  wk += static_cast<long long>(par) * K * Cout;
  const long long m0 = static_cast<long long>(blockIdx.x) * BM;
  const int n0 = blockIdx.y * BN;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int up = md == MUSE_CONV_UPSAMPLE2X;
  const int Hi = up ? H / 2 : (s2 ? 2 * H : Hg), Wi = up ? W / 2 : (s2 ? 2 * W : Wg);
  const int Hb = up ? H : Hi, Wb = up ? W : Wi;  // bounds of the (virtual) input grid the taps index
  const int offy = tr ? (par >> 1) - 1 : (md == MUSE_CONV_S2P1 ? -1 : (s2 ? 0 : -(ksize / 2)));
  const int offx = tr ? (par & 1) - 1 : offy;
  const int st = s2 ? 2 : 1;

  // A-loader role: BM rows x 8 k per stage. VEC: one float4 per (row, half); scalar: BM*8/256 elements.
  constexpr int A_PER_THREAD = BM * KT / 256;  // 4 for BM=128
  int a_row[A_PER_THREAD], a_k[A_PER_THREAD];
  int ab[A_PER_THREAD], ay[A_PER_THREAD], ax[A_PER_THREAD];
  bool a_ok[A_PER_THREAD];
  if (VEC) {
    const int r = threadIdx.x / 2;  // requires BM == 128
    a_row[0] = r; a_k[0] = (threadIdx.x & 1) * 4;
  } else {
#pragma unroll
    for (int i = 0; i < A_PER_THREAD; ++i) {
      const int idx = threadIdx.x + i * 256;
      a_row[i] = idx / KT; a_k[i] = idx % KT;
    }
  }
#pragma unroll
  for (int i = 0; i < (VEC ? 1 : A_PER_THREAD); ++i) {
    const long long m = m0 + a_row[i];
    a_ok[i] = m < M;
    const long long mm = a_ok[i] ? m : 0;
    ax[i] = static_cast<int>(mm % Wg);
    ay[i] = static_cast<int>((mm / Wg) % Hg);
    ab[i] = static_cast<int>(mm / (static_cast<long long>(Wg) * Hg));
  }

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += KT) {
    __syncthreads();
    if (VEC) {
      const int k = k0 + a_k[0];
      const int tap = k / Cin, ci = k % Cin;
      const int iy = ay[0] * st + tap / kk_size + offy, ix = ax[0] * st + tap % kk_size + offx;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (a_ok[0] && iy >= 0 && iy < Hb && ix >= 0 && ix < Wb) {
        const int sy = up ? (iy >> 1) : iy, sx = up ? (ix >> 1) : ix;
        v = *reinterpret_cast<const float4*>(x + ((static_cast<long long>(ab[0]) * Hi + sy) * Wi + sx) * Cin + ci);
      }
      sA[a_k[0] + 0][a_row[0]] = v.x; sA[a_k[0] + 1][a_row[0]] = v.y;
      sA[a_k[0] + 2][a_row[0]] = v.z; sA[a_k[0] + 3][a_row[0]] = v.w;
    } else {
#pragma unroll
      for (int i = 0; i < A_PER_THREAD; ++i) {
        const int k = k0 + a_k[i];
        float v = 0.f;
        if (k < K && a_ok[i]) {
          const int tap = k / Cin, ci = k % Cin;
          const int iy = ay[i] * st + tap / kk_size + offy, ix = ax[i] * st + tap % kk_size + offx;
          if (iy >= 0 && iy < Hb && ix >= 0 && ix < Wb) {
            const int sy = up ? (iy >> 1) : iy, sx = up ? (ix >> 1) : ix;
            v = x[((static_cast<long long>(ab[i]) * Hi + sy) * Wi + sx) * Cin + ci];
          }
        }
        sA[a_k[i]][a_row[i]] = v;
      }
    }
    // B tile: [KT][BN] from wk[k][n]
    for (int idx = threadIdx.x; idx < KT * BN; idx += 256) {
      const int kk = idx / BN, nn = idx % BN;
      const int k = k0 + kk, n = n0 + nn;
      sB[kk][nn] = (k < K && n < Cout) ? wk[static_cast<long long>(k) * Cout + n] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < KT; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = sA[kk][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = sB[kk][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const long long m = m0 + ty * TM + i;
    if (m >= M) continue;
    const long long gx = m % Wg, gy = (m / Wg) % Hg, gb = m / (static_cast<long long>(Wg) * Hg);
    const long long orow = tr ? (gb * H + 2 * gy + (par >> 1)) * W + 2 * gx + (par & 1) : m;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + tx * TN + j;
      if (n < Cout) {
        float v = acc[i][j];
        if (bias) v += bias[n];
        if (res) v += res[orow * Cout + n];
        if (gelu) v = 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
        long long off = orow * Cout + n;
        if (shuf) off = ((gb * 2 * H + 2 * gy + ((n >> 1) & 1)) * 2 * W + 2 * gx + (n & 1)) * (Cout / 4) + (n >> 2);
        y[off] = v;
      }
    }
  }
}

// ---------------------------------------------------------------- GroupNorm + SiLU (NHWC)
// pass 1: per-(image, pixel block, channel) partials {sum, M2}, M2 = sum of squared deviations from the block's own mean
//         (or the same per pixel tile from the epilogue of the tensor-core convolution that produced x)
// pass 2: merge the partials of each group in fp64 (Chan et al.) -> per-(image, channel) scale = rstd*gamma,
//         shift = beta - mean*scale (fp64, kept as two floats hi + lo)
// pass 3: y = silu(fma(x, scale, shift_hi) + shift_lo)
// A variance taken as E[x^2] - mean^2 from fp32 sums loses ~2^-24 (mean^2 + var) / var of itself: at |mean| = 100 std the
// GroupNorm output would be off by ~3e-4.  Deviations from a partial's own mean keep the error independent of the mean.
__global__ void __launch_bounds__(256)
gn_stats_kernel(const float* __restrict__ x, float* __restrict__ partials, int HW, int C, int rows_per_block) {
  pdl_enter();
  // deterministic: fixed thread->data mapping, fixed-order in-block merge, per-block partials (no atomics)
  extern __shared__ float s_part[];  // [rstep][C][2]: {mean of v - K, M2} of each row lane's rows
  const int b = blockIdx.y;
  const int c4 = C / 4;
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(HW, r0 + rows_per_block);
  const float* base = x + static_cast<long long>(b) * HW * C;
  const int q = threadIdx.x % c4;          // fixed channel quad per thread (256 % c4 == 0)
  const int lane_r = threadIdx.x / c4;
  const int rstep = blockDim.x / c4;
  // Welford per thread over its rows r0 + lane_r, r0 + lane_r + rstep, ... of v - K, K = the image's first pixel: the
  // stored sum is then of values ~ the spread, and its fp32 rounding no longer scales with the mean
  const float4 k4 = *reinterpret_cast<const float4*>(base + q * 4);
  const float K[4] = {k4.x, k4.y, k4.z, k4.w};
  float mu[4] = {0.f, 0.f, 0.f, 0.f}, m2[4] = {0.f, 0.f, 0.f, 0.f};
  int cnt = 0;
  for (int r = r0 + lane_r; r < r1; r += rstep) {
    const float4 v4 = *reinterpret_cast<const float4*>(base + static_cast<long long>(r) * C + q * 4);
    const float v[4] = {v4.x, v4.y, v4.z, v4.w};
    const float inv = __frcp_rn(static_cast<float>(++cnt));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float u = v[j] - K[j];
      const float d = u - mu[j];
      mu[j] = fmaf(d, inv, mu[j]);
      m2[j] = fmaf(d, u - mu[j], m2[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    s_part[(lane_r * C + q * 4 + j) * 2] = mu[j];
    s_part[(lane_r * C + q * 4 + j) * 2 + 1] = m2[j];
  }
  __syncthreads();
  float* out = partials + (static_cast<long long>(b) * gridDim.x + blockIdx.x) * C * 2;  // [image][block][C][2]
  const int rows = r1 - r0;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    // merge the row lanes in order; lane k holds rows k, k + rstep, ... of the block
    float n = 0.f, mean = 0.f, M2 = 0.f;
    for (int k = 0; k < rstep && k < rows; ++k) {
      const float nk = static_cast<float>((rows - k + rstep - 1) / rstep);
      const float mk = s_part[(k * C + c) * 2], m2k = s_part[(k * C + c) * 2 + 1];
      const float d = mk - mean, nn = n + nk;
      mean = fmaf(d, nk / nn, mean);
      M2 += m2k + d * d * (n * nk / nn);
      n = nn;
    }
    out[c * 2] = mean * n;
    out[c * 2 + 1] = M2;
  }
}

// one warp per (image, group): fp64 merge of the per-block partials {sum, M2} [image][block][C][2] in a fixed order
// (deterministic).  Block blk covers min(rows_per_block, HW - blk * rows_per_block) pixels.  shift_x (nullable): the
// sums are of x - K with K the image's first pixel x[b, 0, c] (the statistics pass); NULL: of x (conv epilogue tiles).
__global__ void __launch_bounds__(256)
gn_finalize_kernel(const float* __restrict__ partials, int nblocks, int rows_per_block, const float* __restrict__ shift_x,
                   const float* __restrict__ gamma,
                   const float* __restrict__ beta, float* __restrict__ scale_shift, float* __restrict__ shift_lo, int B,
                   int HW, int C, int groups, float eps) {
  pdl_enter();
  const int w = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (w >= B * groups) return;
  const int lane = threadIdx.x & 31;
  const int b = w / groups, g = w % groups;
  const int cpg = C / groups;
  const float* base = partials + static_cast<long long>(b) * nblocks * C * 2;
  const int items = nblocks * cpg;
  auto partial = [&](int i) {
    const int blk = i / cpg, k = i % cpg;
    return *reinterpret_cast<const float2*>(base + (static_cast<long long>(blk) * C + g * cpg + k) * 2);
  };
  auto warp_sum_d = [](double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  };
  auto rows_of = [&](int i) { return static_cast<double>(min(rows_per_block, HW - (i / cpg) * rows_per_block)); };
  auto shift = [&](int i) {
    return shift_x ? static_cast<double>(shift_x[static_cast<long long>(b) * HW * C + g * cpg + i % cpg]) : 0.0;
  };
  double sum = 0.0;
  for (int i = lane; i < items; i += 32) sum += static_cast<double>(partial(i).x) + rows_of(i) * shift(i);
  const double n = static_cast<double>(HW) * cpg;
  const double mean = warp_sum_d(sum) / n;
  // Chan et al.: M2 = sum_i M2_i + n_i (mean_i - mean)^2
  double m2 = 0.0;
  for (int i = lane; i < items; i += 32) {
    const float2 v = partial(i);
    const double ni = rows_of(i);
    const double d = static_cast<double>(v.x) / ni + shift(i) - mean;
    m2 += static_cast<double>(v.y) + ni * d * d;
  }
  const double var = warp_sum_d(m2) / n;
  const float rstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  // shift = beta - mean * scale in fp64 with the fp32 scale, carried as hi + lo: y = fma(x, scale, hi) + lo is
  // (x - mean) * scale + beta to fp32 rounding however large the mean (a one-float shift is off by ~2^-25 |mean| scale).
  for (int k = lane; k < cpg; k += 32) {
    const int c = g * cpg + k;
    const float sc = rstd * gamma[c];
    const double sh = static_cast<double>(beta[c]) - mean * static_cast<double>(sc);
    const float sh_hi = static_cast<float>(sh);
    scale_shift[(static_cast<long long>(b) * C + c) * 2] = sc;
    scale_shift[(static_cast<long long>(b) * C + c) * 2 + 1] = sh_hi;
    shift_lo[static_cast<long long>(b) * C + c] = static_cast<float>(sh - static_cast<double>(sh_hi));
  }
}

// Spatial modulation of the apply pass (MoVQ SpatialNorm, muse/modeling_movq.py:21-49): out = GN(x) * Ym + Bm with
// Ym[c] = by[c] + sum_d wy[c][d] zq[b, y / ry, x / rx, d] and Bm likewise from wb / bb, the 1x1 conv_y / conv_b of the
// nearest-upsampled latent computed per pixel from its latent pixel (never written out: at C = 512 Ym and Bm would be
// twice the bytes of x).  Integer ratios ry = H / Hz, rx = W / Wz; dq % 4 == 0, dq <= 16.
struct GnMod {
  const float* zq;                  // [B, Hz, Wz, dq] NHWC latent
  const float* wy; const float* wb;  // [C][dq]
  const float* by; const float* bb;  // [C]
  int W, Hz, Wz, ry, rx, dq;
};

// o[j] = fma(o[j], Ym[c0 + j], Bm[c0 + j]) for pixel p (flat over the batch), channels c0 .. c0 + N - 1
template <int N>
__device__ __forceinline__ void gn_modulate(const GnMod& m, long long p, int HW, int c0, float (&o)[N]) {
  const int b = static_cast<int>(p / HW), r = static_cast<int>(p - static_cast<long long>(b) * HW);
  const int zy = (r / m.W) / m.ry, zx = (r % m.W) / m.rx;
  const float* z = m.zq + ((static_cast<long long>(b) * m.Hz + zy) * m.Wz + zx) * m.dq;
  float ym[N], bm[N];
#pragma unroll
  for (int j = 0; j < N; ++j) { ym[j] = m.by[c0 + j]; bm[j] = m.bb[c0 + j]; }
  for (int k = 0; k < m.dq; k += 4) {
    const float4 z4 = *reinterpret_cast<const float4*>(z + k);
#pragma unroll
    for (int j = 0; j < N; ++j) {
      const float4 a = *reinterpret_cast<const float4*>(m.wy + (c0 + j) * m.dq + k);
      const float4 e = *reinterpret_cast<const float4*>(m.wb + (c0 + j) * m.dq + k);
      ym[j] = fmaf(a.w, z4.w, fmaf(a.z, z4.z, fmaf(a.y, z4.y, fmaf(a.x, z4.x, ym[j]))));
      bm[j] = fmaf(e.w, z4.w, fmaf(e.z, z4.z, fmaf(e.y, z4.y, fmaf(e.x, z4.x, bm[j]))));
    }
  }
#pragma unroll
  for (int j = 0; j < N; ++j) o[j] = fmaf(o[j], ym[j], bm[j]);
}

// SPLIT: instead of fp32 y, emit the bf16 hi/lo planes (y = hi + lo) the tensor-core convolution consumes (conv_tc.cu)
// MOD: the SpatialNorm modulation above, before the SiLU
template <bool SPLIT, bool MOD>
__global__ void __launch_bounds__(256)
gn_apply_silu_kernel(const float* __restrict__ x, const float* __restrict__ scale_shift, const float* __restrict__ shift_lo,
                     float* __restrict__ y, bf16* __restrict__ y_hi, bf16* __restrict__ y_lo, long long total4, int HW, int C,
                     int silu, GnMod mod) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= total4) return;
  const int c4 = C / 4;
  const int q = static_cast<int>(i % c4);
  const int b = static_cast<int>(i / (static_cast<long long>(c4) * HW));
  const float4 v = *reinterpret_cast<const float4*>(x + i * 4);
  const float4 s0 = *reinterpret_cast<const float4*>(scale_shift + (static_cast<long long>(b) * C + q * 4) * 2);
  const float4 s1 = *reinterpret_cast<const float4*>(scale_shift + (static_cast<long long>(b) * C + q * 4) * 2 + 4);
  const float4 l = *reinterpret_cast<const float4*>(shift_lo + static_cast<long long>(b) * C + q * 4);
  float o[4] = {fmaf(v.x, s0.x, s0.y) + l.x, fmaf(v.y, s0.z, s0.w) + l.y, fmaf(v.z, s1.x, s1.y) + l.z,
                fmaf(v.w, s1.z, s1.w) + l.w};
  if (MOD) gn_modulate<4>(mod, i / c4, HW, q * 4, o);
#pragma unroll
  for (int j = 0; j < 4; ++j) o[j] = silu ? o[j] / (1.f + expf(-o[j])) : o[j];
  if (SPLIT) {
    float h[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) h[j] = bf16_round(o[j]);
    uint2 uh, ul;
    uh.x = pack_bf16(h[0], h[1]); uh.y = pack_bf16(h[2], h[3]);
    ul.x = pack_bf16(o[0] - h[0], o[1] - h[1]); ul.y = pack_bf16(o[2] - h[2], o[3] - h[3]);
    *reinterpret_cast<uint2*>(y_hi + i * 4) = uh;
    if (y_lo) *reinterpret_cast<uint2*>(y_lo + i * 4) = ul;
  } else {
    *reinterpret_cast<float4*>(y + i * 4) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// 8 channels per thread variant of the SPLIT apply (two 16-byte loads in flight, 16-byte stores per plane)
template <bool MOD>
__global__ void __launch_bounds__(256)
gn_apply_silu_split8_kernel(const float* __restrict__ x, const float* __restrict__ scale_shift,
                            const float* __restrict__ shift_lo, bf16* __restrict__ y_hi, bf16* __restrict__ y_lo,
                            long long total8, int HW, int C, int silu, GnMod mod) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= total8) return;
  const int c8 = C / 8;
  const int q = static_cast<int>(i % c8);
  const int b = static_cast<int>(i / (static_cast<long long>(c8) * HW));
  float v[8], sl[8];
  load8(x + i * 8, v);
  load8(shift_lo + static_cast<long long>(b) * C + q * 8, sl);
  const float4* ssp = reinterpret_cast<const float4*>(scale_shift + (static_cast<long long>(b) * C + q * 8) * 2);
  float h[8], l[8];
  if (MOD) {
    float o[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 s2 = ssp[j];
      o[2 * j] = fmaf(v[2 * j], s2.x, s2.y) + sl[2 * j];
      o[2 * j + 1] = fmaf(v[2 * j + 1], s2.z, s2.w) + sl[2 * j + 1];
    }
    gn_modulate<8>(mod, i / c8, HW, q * 8, o);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float t = silu ? o[j] / (1.f + expf(-o[j])) : o[j];
      h[j] = bf16_round(t);
      l[j] = t - h[j];
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 s2 = ssp[j];  // {scale, shift} of channels 2j, 2j+1
      float o0 = fmaf(v[2 * j], s2.x, s2.y) + sl[2 * j], o1 = fmaf(v[2 * j + 1], s2.z, s2.w) + sl[2 * j + 1];
      if (silu) {
        o0 = o0 / (1.f + expf(-o0));
        o1 = o1 / (1.f + expf(-o1));
      }
      h[2 * j] = bf16_round(o0); h[2 * j + 1] = bf16_round(o1);
      l[2 * j] = o0 - h[2 * j]; l[2 * j + 1] = o1 - h[2 * j + 1];
    }
  }
  store8(y_hi + i * 8, h);
  if (y_lo) store8(y_lo + i * 8, l);  // single-pass bf16 tokenizer mode needs the hi plane only
}

// ---------------------------------------------------------------- pooling / layout
__global__ void __launch_bounds__(256)
avgpool2_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int Ho, int Wo, int C) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  const int c4 = C / 4;
  const long long total = static_cast<long long>(B) * Ho * Wo * c4;
  if (i >= total) return;
  const int q = static_cast<int>(i % c4);
  const int ox = static_cast<int>((i / c4) % Wo);
  const int oy = static_cast<int>((i / (static_cast<long long>(c4) * Wo)) % Ho);
  const int b = static_cast<int>(i / (static_cast<long long>(c4) * Wo * Ho));
  const int Wi = Wo * 2;
  const float* p = x + ((static_cast<long long>(b) * Ho * 2 + oy * 2) * Wi + ox * 2) * C + q * 4;
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 bb = *reinterpret_cast<const float4*>(p + C);
  const float4 c = *reinterpret_cast<const float4*>(p + static_cast<long long>(Wi) * C);
  const float4 d = *reinterpret_cast<const float4*>(p + static_cast<long long>(Wi) * C + C);
  // same association as ATen's avg_pool2d accumulation: ((a + b) + c) + d, then / 4
  *reinterpret_cast<float4*>(y + i * 4) = make_float4(((a.x + bb.x) + c.x + d.x) * 0.25f, ((a.y + bb.y) + c.y + d.y) * 0.25f,
                                                      ((a.z + bb.z) + c.z + d.z) * 0.25f, ((a.w + bb.w) + c.w + d.w) * 0.25f);
}

// out[b, p, c] = in[b, c, p] (to_nhwc) or the inverse; 32x32 smem transpose tiles
__global__ void __launch_bounds__(256)
transpose_cp_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols) {
  pdl_enter();
  __shared__ float t[32][33];
  const int b = blockIdx.z;
  const float* ip = in + static_cast<long long>(b) * rows * cols;
  float* op = out + static_cast<long long>(b) * rows * cols;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int j = ty; j < 32; j += 8) {
    const int r = r0 + j, c = c0 + tx;
    if (r < rows && c < cols) t[j][tx] = ip[static_cast<long long>(r) * cols + c];
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, r = r0 + tx;
    if (r < rows && c < cols) op[static_cast<long long>(c) * rows + r] = t[tx][j];
  }
}

}  // namespace

// Decoder output -> display bytes with the reference's recipe (muse/pipeline_muse.py:245-252, quirk Q10), same fp32 operation
// order so the bytes are identical: t = 2x - 1; t = clip(t, -1, 1); t = (t + 1) / 2; byte = (uint8)(255 * t)  (truncation).
// Input is the decoder's native NHWC tensor, output HWC uint8 per image: the NCHW round trip of the reference
// (decode -> permute(1, 2, 0) -> numpy) and the 4x larger fp32 device->host copy disappear.
__global__ void __launch_bounds__(256)
image_to_uint8_kernel(const float* __restrict__ x, unsigned char* __restrict__ y, long long n4) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n4) return;
  const float4 v = *reinterpret_cast<const float4*>(x + i * 4);
  const float f[4] = {v.x, v.y, v.z, v.w};
  uchar4 o;
  unsigned char* ob = reinterpret_cast<unsigned char*>(&o);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float t = __fsub_rn(__fmul_rn(2.0f, f[k]), 1.0f);
    t = fminf(fmaxf(t, -1.0f), 1.0f);
    t = __fdiv_rn(__fadd_rn(t, 1.0f), 2.0f);
    ob[k] = static_cast<unsigned char>(static_cast<int>(__fmul_rn(255.0f, t)));  // truncation toward zero, values in [0, 255]
  }
  *reinterpret_cast<uchar4*>(y + i * 4) = o;
}

// workspace: partials float [nblocks*B*C*2] with nblocks = ceil(HW / rows_per_block) (see muse_groupnorm_workspace_floats)
static int gn_rows_per_block(int C) { return (256 / (C / 4)) * 64; }

// argument checks shared by both GroupNorm entry points; run before any launch
static int gn_check(const char* what, const float* y, const void* y_hi, const void* y_lo, int C, int groups) {
  if ((y != nullptr) == (y_hi != nullptr) || (y_hi == nullptr && y_lo != nullptr)) {
    set_last_error("%s: give either y (fp32) or y_hi (+ y_lo unless the single-pass bf16 mode is used)", what);
    return MUSE_ERR_INVALID;
  }
  if (C % groups != 0 || C % 4 != 0 || C > 1024 || 256 % (C / 4) != 0) {
    set_last_error("%s: C=%d groups=%d unsupported (C must divide into groups, C/4 must divide 256)", what, C, groups);
    return MUSE_ERR_UNSUPPORTED;
  }
  return MUSE_OK;
}

// statistics pass (or the conv epilogue's tiles) + fp64 finalize: per-(image, channel) {scale, shift_hi} in
// scale_shift_ws, shift_lo after them
static int gn_scale_shift(const float* x, const float* gamma, const float* beta, float* partials_ws, float* scale_shift_ws, int B,
                   int HW, int C, int groups, float eps, int precomputed_tiles, cudaStream_t s) {
  // precomputed_tiles > 0: partials_ws already holds {sum, M2} per [image][tile][C] (HW / tiles pixels each), written by the
  // epilogue of the tensor-core convolution that produced x (conv_tc.cu), and the statistics pass over x is skipped.
  int nblocks = precomputed_tiles;
  int rows_per_block = precomputed_tiles > 0 ? HW / precomputed_tiles : gn_rows_per_block(C);
  int rc;
  if (precomputed_tiles > 0 && HW % precomputed_tiles != 0) {
    set_last_error("groupnorm: %d precomputed tiles do not split HW=%d evenly", precomputed_tiles, HW);
    return MUSE_ERR_INVALID;
  }
  if (precomputed_tiles <= 0) {
    nblocks = ceil_div(HW, rows_per_block);
    const int rstep = 256 / (C / 4);
    pdl_launch(dim3(nblocks, B), 256, rstep * C * 2 * sizeof(float), s)(gn_stats_kernel, x, partials_ws, HW, C, rows_per_block);
    rc = check_launch("gn_stats");
    if (rc) return rc;
  }
  float* shift_lo = scale_shift_ws + 2LL * B * C;
  pdl_launch(ceil_div(B * groups, 8), 256, 0, s)(gn_finalize_kernel, partials_ws, nblocks, rows_per_block,
                                                             precomputed_tiles > 0 ? nullptr : x, gamma, beta,
                                                             scale_shift_ws, shift_lo, B, HW, C, groups, eps);
  return check_launch("gn_finalize");
}

template <bool MOD>
static int gn_apply(const float* x, const float* scale_shift_ws, float* y, void* y_hi, void* y_lo, int B, int HW, int C,
             int apply_silu, const GnMod& mod, cudaStream_t s) {
  const float* shift_lo = scale_shift_ws + 2LL * B * C;
  const long long total4 = static_cast<long long>(B) * HW * (C / 4);
  const unsigned blocks = static_cast<unsigned>(ceil_div_ll(total4, 256));
  if (y != nullptr)
    pdl_launch(blocks, 256, 0, s)(gn_apply_silu_kernel<false, MOD>, x, scale_shift_ws, shift_lo, y, nullptr, nullptr, total4, HW,
                                  C, apply_silu, mod);
  else if (C % 8 == 0)
    pdl_launch(static_cast<unsigned>(ceil_div_ll(total4 / 2, 256)), 256, 0, s)(gn_apply_silu_split8_kernel<MOD>,
        x, scale_shift_ws, shift_lo, reinterpret_cast<bf16*>(y_hi), reinterpret_cast<bf16*>(y_lo), total4 / 2, HW, C, apply_silu,
        mod);
  else
    pdl_launch(blocks, 256, 0, s)(gn_apply_silu_kernel<true, MOD>, x, scale_shift_ws, shift_lo, nullptr, reinterpret_cast<bf16*>(y_hi),
                                  reinterpret_cast<bf16*>(y_lo), total4, HW, C, apply_silu, mod);
  return check_launch(MOD ? "spatial_gn_apply_silu" : "gn_apply_silu");
}

}  // namespace muse

using namespace muse;

extern "C" {

int muse_conv2d_nhwc(const float* x, const float* wk, const float* bias, const float* res, float* y, int B, int H, int W,
                     int Cin, int Cout, int ksize, int mode, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int md = mode & MUSE_CONV_GEOMETRY;
  if (md > MUSE_CONV_TRANSPOSE_S2 || (mode & ~(MUSE_CONV_GEOMETRY | MUSE_CONV_GELU | MUSE_CONV_PIXEL_SHUFFLE)) != 0) {
    set_last_error("conv2d: bad mode %d", mode);
    return MUSE_ERR_INVALID;
  }
  const bool k_ok = md == MUSE_CONV_STRIDE2 ? (ksize == 2 || ksize == 3)
                                            : (md >= MUSE_CONV_S2P1 ? ksize == 4 : (ksize == 1 || ksize == 3));
  if (!k_ok) { set_last_error("conv2d: kernel size %d unsupported in mode %d", ksize, md); return MUSE_ERR_UNSUPPORTED; }
  const bool upsampling = md == MUSE_CONV_UPSAMPLE2X || md == MUSE_CONV_TRANSPOSE_S2;
  if (upsampling && ((H | W) & 1)) { set_last_error("conv2d: upsampling modes need even output dims"); return MUSE_ERR_INVALID; }
  if ((mode & MUSE_CONV_GELU) && res) { set_last_error("conv2d: the GELU epilogue takes no residual"); return MUSE_ERR_INVALID; }
  if ((mode & MUSE_CONV_PIXEL_SHUFFLE) && (res || md != MUSE_CONV_SAME || Cout % 4 != 0)) {
    set_last_error("conv2d: the PixelShuffle store needs Cout %% 4 == 0, stride 1, no residual");
    return MUSE_ERR_INVALID;
  }
  const long long M = static_cast<long long>(B) * H * W / (md == MUSE_CONV_TRANSPOSE_S2 ? 4 : 1);
  if (M <= 0) return MUSE_OK;
  const bool vec = (Cin % 8 == 0);
  const unsigned gz = md == MUSE_CONV_TRANSPOSE_S2 ? 4 : 1;
  if (Cout > 16) {
    dim3 grid(static_cast<unsigned>(ceil_div_ll(M, 128)), ceil_div(Cout, 128), gz);
    if (vec) pdl_launch(grid, 256, 0, s)(conv2d_nhwc_kernel<8, 8, true>, x, wk, bias, res, y, B, H, W, Cin, Cout, ksize, mode);
    else pdl_launch(grid, 256, 0, s)(conv2d_nhwc_kernel<8, 8, false>, x, wk, bias, res, y, B, H, W, Cin, Cout, ksize, mode);
  } else {
    dim3 grid(static_cast<unsigned>(ceil_div_ll(M, 128)), 1, gz);
    if (vec) pdl_launch(grid, 256, 0, s)(conv2d_nhwc_kernel<8, 1, true>, x, wk, bias, res, y, B, H, W, Cin, Cout, ksize, mode);
    else pdl_launch(grid, 256, 0, s)(conv2d_nhwc_kernel<8, 1, false>, x, wk, bias, res, y, B, H, W, Cin, Cout, ksize, mode);
  }
  return check_launch("conv2d_nhwc");
}

long long muse_groupnorm_workspace_floats(int B, int HW, int C) {
  if (C % 4 != 0 || C > 1024 || 256 % (C / 4) != 0) return -1;
  return static_cast<long long>(ceil_div(HW, gn_rows_per_block(C))) * B * C * 2;
}

// y (fp32) or y_hi / y_lo (bf16 split planes) receive the result: exactly one of the two forms must be given.
int muse_groupnorm_silu_nhwc(const float* x, const float* gamma, const float* beta, float* y, void* y_hi, void* y_lo,
                             float* partials_ws, float* scale_shift_ws, int B, int HW, int C, int groups, float eps,
                             int precomputed_tiles, int apply_silu, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc = gn_check("groupnorm", y, y_hi, y_lo, C, groups);
  if (rc) return rc;
  if (B <= 0 || HW <= 0) return MUSE_OK;
  rc = gn_scale_shift(x, gamma, beta, partials_ws, scale_shift_ws, B, HW, C, groups, eps, precomputed_tiles, s);
  if (rc) return rc;
  return gn_apply<false>(x, scale_shift_ws, y, y_hi, y_lo, B, HW, C, apply_silu, GnMod{}, s);
}

int muse_spatial_groupnorm_silu_nhwc(const float* x, const float* gamma, const float* beta, const float* zq, const float* wy,
                                     const float* by, const float* wb, const float* bb, float* y, void* y_hi, void* y_lo,
                                     float* partials_ws, float* scale_shift_ws, int B, int H, int W, int C, int groups,
                                     float eps, int hz, int wz, int dq, int precomputed_tiles, int apply_silu, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc = gn_check("spatial groupnorm", y, y_hi, y_lo, C, groups);
  if (rc) return rc;
  if (dq <= 0 || dq % 4 != 0 || dq > 16) {
    set_last_error("spatial groupnorm: latent channels %d unsupported (a multiple of 4, at most 16)", dq);
    return MUSE_ERR_UNSUPPORTED;
  }
  if (hz <= 0 || wz <= 0 || H <= 0 || W <= 0 || H % hz != 0 || W % wz != 0) {
    set_last_error("spatial groupnorm: %dx%d is not an integer multiple of the %dx%d latent grid", H, W, hz, wz);
    return MUSE_ERR_UNSUPPORTED;
  }
  if (!zq || !wy || !by || !wb || !bb ||
      ((reinterpret_cast<uintptr_t>(zq) | reinterpret_cast<uintptr_t>(wy) | reinterpret_cast<uintptr_t>(wb)) & 15)) {
    set_last_error("spatial groupnorm: zq, wy, wb, by, bb are required; zq, wy and wb 16-byte aligned");
    return MUSE_ERR_INVALID;
  }
  if (B <= 0) return MUSE_OK;
  const int HW = H * W;
  rc = gn_scale_shift(x, gamma, beta, partials_ws, scale_shift_ws, B, HW, C, groups, eps, precomputed_tiles, s);
  if (rc) return rc;
  const GnMod mod{zq, wy, wb, by, bb, W, hz, wz, H / hz, W / wz, dq};
  return gn_apply<true>(x, scale_shift_ws, y, y_hi, y_lo, B, HW, C, apply_silu, mod, s);
}

int muse_image_to_uint8(const float* x, unsigned char* y, long long n, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0) return MUSE_OK;
  if (n % 4 != 0) { set_last_error("image_to_uint8: element count must be a multiple of 4"); return MUSE_ERR_INVALID; }
  pdl_launch(static_cast<unsigned>(ceil_div_ll(n / 4, 256)), 256, 0, s)(image_to_uint8_kernel, x, y, n / 4);
  return check_launch("image_to_uint8");
}

int muse_avgpool2_nhwc(const float* x, float* y, int B, int Ho, int Wo, int C, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (C % 4 != 0) { set_last_error("avgpool: C must be a multiple of 4"); return MUSE_ERR_UNSUPPORTED; }
  const long long total = static_cast<long long>(B) * Ho * Wo * (C / 4);
  if (total <= 0) return MUSE_OK;
  pdl_launch(static_cast<unsigned>(ceil_div_ll(total, 256)), 256, 0, s)(avgpool2_nhwc_kernel, x, y, B, Ho, Wo, C);
  return check_launch("avgpool2_nhwc");
}

// in: [B, rows, cols] -> out: [B, cols, rows]
int muse_transpose_batched(const float* in, float* out, int B, int rows, int cols, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (B <= 0 || rows <= 0 || cols <= 0) return MUSE_OK;
  pdl_launch(dim3(ceil_div(cols, 32), ceil_div(rows, 32), B), 256, 0, s)(transpose_cp_kernel, in, out, rows, cols);
  return check_launch("transpose_batched");
}

}  // extern "C"
