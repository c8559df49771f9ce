// Row normalisation (LayerNorm without bias / RMSNorm), forward and backward, HBM-bound.
// Reference: muse/modeling_transformer.py:124-137 (LayerNorm -> F.layer_norm, weight only),
// :79-100 (RMSNorm).  One warp owns one row (16-byte vector loads, shuffle reductions, no block barriers); every
// element is read from HBM once and written once.
// Fusions folded in (they are separate ATen launches in the reference):
//   * act=1  : exact GELU applied to the input first (mlm_dense -> gelu -> mlm_ln, :980-983)
//   * act=2  : GLU: the input is [rows, 2H] = [a | b] and the normalised value is bf16(gelu(a)) * b, i.e. the
//              FeedForward product (:789-792) feeding mid_mlp_layer_norm (:795-796) without materialising it;
//              backward recomputes it and emits d[a | b] directly (LN backward + GLU backward in one pass)
//   * residual: y = residual + norm(x) (normformer post-attention norm + residual add, :882-884)
//   * backward: dx = norm_bwd(dy) (+ dres), so the residual-stream gradient add is free.
//   * act=2 with dropout: FeedForward.dropout (:797) on the normalised output -- the forward draws the keep bits
//              (philox.cuh) and writes the dropped bf16 output and the bits, the backward scales dy by them as it reads it
#include <climits>
#include <cstdlib>

#include "philox.cuh"
#include "ptx.cuh"
#include "row_norm.cuh"

namespace muse {
namespace {

constexpr int ACT_NONE = 0, ACT_GELU = 1, ACT_GLU = 2;

// ---- warp-per-row kernels (H <= 1024, no GLU): the whole row lives in registers (row_norm.cuh), no block barriers
constexpr int kWarpsPerBlock = 4;

// F8: y is the e4m3 operand of muse_gemm_fp8 (TY = uint8_t) and row_scale [rows] its scales (row_store_e4m3).
template <typename TX, typename TY, int CH, bool F8>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
norm_fwd_warp_kernel(const TX* __restrict__ x, const float* __restrict__ w, const float* __restrict__ res,
                TY* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows, int H,
                float eps, int act, int rms, float* __restrict__ row_scale) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (row >= rows) return;
  const TX* xr = x + static_cast<size_t>(row) * H;
  float v[CH][8];
  const float inv_h = 1.0f / static_cast<float>(H);
  const float sum = row_load(v, H, lane, [&](int col, float (&vc)[8]) {
    load8(xr + col, vc);
    if (act) {
#pragma unroll
      for (int j = 0; j < 8; ++j) vc[j] = gelu_f(vc[j]);
    }
  });
  float mean, rstd;
  row_stats(v, sum, H, inv_h, lane, eps, rms, mean, rstd);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  TY* yr = y + static_cast<size_t>(row) * H;
  const float* rr = res ? res + static_cast<size_t>(row) * H : nullptr;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = row_col(c, lane);
    if (col < H) {
      float o[8], wv[8];
      if (w) load8(w + col, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[c][j] - mean) * rstd * (w ? wv[j] : 1.f);
      if (rr) {
        float r8[8];
        load8(rr + col, r8);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += r8[j];
      }
      if constexpr (F8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[c][j] = o[j];
      } else {
        store8(yr + col, o);
      }
    }
  }
  if constexpr (F8) row_store_e4m3(v, H, lane, reinterpret_cast<uint8_t*>(yr), row_scale + row);
}

// Weight gradients (dw[H] = sum over rows of dy * xhat) are reduced in a FIXED order so that the result is bit-identical
// from run to run: every warp owns a static set of rows (grid-stride) and keeps its partial in registers / a private
// shared-memory row, the CTA sums its warps in warp order, and
//   * dw_ws != nullptr: the CTA stores its partial row to dw_ws[blockIdx.x][H]; colsum_ordered_kernel then sums the CTA
//     rows in index order and STORES dw (no zero fill needed);
//   * dw_ws == nullptr: the CTA adds its partial to dw with atomics (accumulating, order-dependent; legacy callers).
constexpr int kBwdWarps = 8;

__device__ __forceinline__ void flush_cta_dw(const float* s_dw, int nwarps, int H, float* dw, float* dw_ws) {
  __syncthreads();
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    float acc = 0.f;
    for (int k = 0; k < nwarps; ++k) acc += s_dw[static_cast<size_t>(k) * H + i];
    if (dw_ws) dw_ws[static_cast<size_t>(blockIdx.x) * H + i] = acc;
    else atomicAdd(&dw[i], acc);
  }
}

// dw[i] = sum_g ws[g][i] in ascending g (32 x 32 threads: thread (ty, tx) sums rows ty, ty+32, ... of column tx).
__global__ void __launch_bounds__(1024) colsum_ordered_kernel(const float* __restrict__ ws, float* __restrict__ dw, int G, int H) {
  pdl_enter();
  __shared__ float s[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + tx;
  float acc = 0.f;
  if (col < H) {
#pragma unroll 8
    for (int g = ty; g < G; g += 32) acc += ws[static_cast<size_t>(g) * H + col];
  }
  s[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && col < H) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) t += s[k][tx];
    dw[col] = t;
  }
}

// L2 prefetch (a hint: no register, no scoreboard entry).  The persistent row-streaming backward kernels of the register
// path are bound by exposed load latency rather than by issue slots or DRAM bandwidth (the row-ring kernels further down
// take their place wherever they apply).  A warp walks its rows strictly one after the
// other, so the lines of the row it will touch NEXT are requested from HBM while the current row is processed and the demand
// loads become L2 hits.  prefetch_row: the lanes of a warp cover the 128-byte lines of one row of H elements.
// The GLU + LayerNorm backward prefetches two loop iterations ahead instead (see glu_norm_bwd_kernel).
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
template <typename T>
__device__ __forceinline__ void prefetch_row(const T* row, int H, int lane) {
  const int bytes = H * static_cast<int>(sizeof(T));
  for (int off = lane * 128; off < bytes; off += 32 * 128) prefetch_l2(reinterpret_cast<const char*>(row) + off);
}

template <typename TDY, typename TX, typename TDX, int CH>
__global__ void __launch_bounds__(kBwdWarps * 32)
norm_bwd_warp_kernel(const TDY* __restrict__ dy, const TX* __restrict__ x, const float* __restrict__ w,
                const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                const float* __restrict__ dres, TDX* __restrict__ dx, bf16* __restrict__ dx_copy, float* __restrict__ dw,
                float* __restrict__ dw_ws, int rows, int H, int act, int rms) {
  pdl_enter();
  extern __shared__ float s_dw[];  // [kBwdWarps][H] private rows
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  float dw_acc[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) dw_acc[c][j] = 0.f;
  const float inv_h = 1.0f / static_cast<float>(H);

  for (int row = blockIdx.x * kBwdWarps + warp; row < rows; row += gridDim.x * kBwdWarps) {
    const TX* xr = x + static_cast<size_t>(row) * H;
    const TDY* dyr = dy + static_cast<size_t>(row) * H;
    const float mean = rms ? 0.f : mean_in[row];
    const float rstd = rstd_in[row];
    float xh[CH][8], g[CH][8], rs[CH][8];
    float s1 = 0.f, s2 = 0.f;
    const float* drr = dres ? dres + static_cast<size_t>(row) * H : nullptr;
    const int next = row + gridDim.x * kBwdWarps;
    if (next < rows) {  // this warp's next row (see prefetch_row)
      prefetch_row(x + static_cast<size_t>(next) * H, H, lane);
      prefetch_row(dy + static_cast<size_t>(next) * H, H, lane);
      if (dres) prefetch_row(dres + static_cast<size_t>(next) * H, H, lane);
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float xv[8], dv[8], wv[8];
        load8(xr + col, xv);
        load8(dyr + col, dv);
        if (drr) load8(drr + col, rs[c]);  // residual-gradient row fetched with the first wave of loads, not after the reductions
        if (w) load8(w + col, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float a = act ? gelu_f(xv[j]) : xv[j];
          xh[c][j] = (a - mean) * rstd;
          dw_acc[c][j] += dv[j] * xh[c][j];
          g[c][j] = dv[j] * (w ? wv[j] : 1.f);
          row_bwd_acc(g[c][j], xh[c][j], s1, s2);
        }
      }
    }
    row_bwd_sums(inv_h, rms, s1, s2);
    TDX* dxr = dx + static_cast<size_t>(row) * H;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = row_dx(g[c][j], xh[c][j], s1, s2, rstd);
        if (act) {
          float xv[8];
          load8(xr + col, xv);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] *= gelu_grad_f(xv[j]);
        }
        if (drr) {
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += rs[c][j];
        }
        store8(dxr + col, o);
        // bf16 copy of the residual-stream gradient: the GEMM operand of the previous layer's wo dgrad / wgrad (saves the
        // separate fp32 -> bf16 cast pass over the same tensor)
        if (dx_copy) store8(dx_copy + static_cast<size_t>(row) * H + col, o);
      }
    }
  }
  if (dw) {
    float* my_dw = s_dw + static_cast<size_t>(warp) * H;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) store8(my_dw + col, dw_acc[c]);
    }
    flush_cta_dw(s_dw, kBwdWarps, H, dw, dw_ws);
  }
}


// ---- two chained norms in one pass (normformer layer, H <= 1024): the post-attention norm with its residual add
// (reference :882-884: x2 = x + post_attn_layer_norm(attention_output)) immediately followed by the FeedForward's
// pre_mlp_layer_norm (:787, always LayerNorm).  Separately these are two HBM round trips of the residual stream (x2 is
// written by the first and read back by the second); fused, the row stays in registers: 12 instead of 16 bytes per element
// forward, 18 instead of 22 backward.
// F8: h2 is the e4m3 operand of muse_gemm_fp8 (TH = uint8_t) and row_scale [rows] its scales; x2 and the statistics
// are the same as the bf16 form's.
template <int CH, bool F8, typename TH = bf16>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
norm2_fwd_warp_kernel(const bf16* __restrict__ a, const float* __restrict__ res, const float* __restrict__ w1,
                      const float* __restrict__ w2, float* __restrict__ x2, TH* __restrict__ h2,
                      float* __restrict__ mean1_out, float* __restrict__ rstd1_out, float* __restrict__ mean2_out,
                      float* __restrict__ rstd2_out, int rows, int H, float eps, int rms1, int rms2,
                      float* __restrict__ row_scale) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float inv_h = 1.0f / static_cast<float>(H);
  float v[CH][8];
  const float sum1 = row_load(v, H, lane, [&](int col, float (&vc)[8]) { load8(a + static_cast<size_t>(row) * H + col, vc); });
  float mean1, rstd1;
  row_stats(v, sum1, H, inv_h, lane, eps, rms1, mean1, rstd1);
  // x2 = res + norm1(a) * w1  (kept in v), second statistics over x2
  float sum2 = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = row_col(c, lane);
    if (col < H) {
      float wv[8], r8[8];
      load8(w1 + col, wv);
      load8(res + static_cast<size_t>(row) * H + col, r8);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[c][j] = r8[j] + (v[c][j] - mean1) * rstd1 * wv[j];
        sum2 += v[c][j];
      }
      store8(x2 + static_cast<size_t>(row) * H + col, v[c]);
    }
  }
  float mean2, rstd2;
  row_stats(v, sum2, H, inv_h, lane, eps, rms2, mean2, rstd2);
  if (lane == 0) {
    if (mean1_out) { mean1_out[row] = mean1; rstd1_out[row] = rstd1; mean2_out[row] = mean2; rstd2_out[row] = rstd2; }
  }
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = row_col(c, lane);
    if (col < H) {
      float wv[8], o[8];
      load8(w2 + col, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[c][j] - mean2) * rstd2 * wv[j];
      if constexpr (F8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[c][j] = o[j];
      } else {
        store8(h2 + static_cast<size_t>(row) * H + col, o);
      }
    }
  }
  if constexpr (F8) {
    // the row index passes through a shuffle so that the e4m3 row's addresses are formed here: held from the start of the
    // kernel, the two 64-bit addresses were spilled to the stack at 2 chunks (264 <= H <= 512)
    const int r = __shfl_sync(0xffffffffu, row, 0);
    row_store_e4m3(v, H, lane, h2 + static_cast<size_t>(r) * H, row_scale + r);
  }
}

// backward of the pair: dx2 = LN2_bwd(d_h2; x2) + dres ; d_a = LN1_bwd(dx2; a) ; dw2 += d_h2 * x2hat ; dw1 += dx2 * ahat
template <int CH>
__global__ void __launch_bounds__(kBwdWarps * 32)
norm2_bwd_warp_kernel(const bf16* __restrict__ d_h2, const float* __restrict__ x2, const float* __restrict__ w2,
                      const float* __restrict__ mean2_in, const float* __restrict__ rstd2_in, const float* __restrict__ dres,
                      const bf16* __restrict__ a, const float* __restrict__ w1, const float* __restrict__ mean1_in,
                      const float* __restrict__ rstd1_in, float* __restrict__ dx2, bf16* __restrict__ d_a,
                      float* __restrict__ dw2_ws, float* __restrict__ dw1_ws, int rows, int H, int rms1, int rms2) {
  pdl_enter();
  extern __shared__ float s_dw[];  // [2][kBwdWarps][H] private rows (dw2 then dw1)
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  float acc2[CH][8], acc1[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc2[c][j] = 0.f; acc1[c][j] = 0.f; }
  const float inv_h = 1.0f / static_cast<float>(H);
  for (int row = blockIdx.x * kBwdWarps + warp; row < rows; row += gridDim.x * kBwdWarps) {
    const size_t off = static_cast<size_t>(row) * H;
    const float mean2 = rms2 ? 0.f : mean2_in[row], rstd2 = rstd2_in[row];
    const float mean1 = rms1 ? 0.f : mean1_in[row], rstd1 = rstd1_in[row];
    float xh[CH][8], g[CH][8], rs[CH][8], av[CH][8];
    float s1 = 0.f, s2 = 0.f;
    const int next = row + gridDim.x * kBwdWarps;
    if (next < rows) {  // this warp's next row (see prefetch_row)
      const size_t noff = static_cast<size_t>(next) * H;
      prefetch_row(x2 + noff, H, lane);
      prefetch_row(d_h2 + noff, H, lane);
      prefetch_row(dres + noff, H, lane);
      prefetch_row(a + noff, H, lane);
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float xv[8], dv[8], wv[8];
        load8(x2 + off + col, xv);
        load8(d_h2 + off + col, dv);
        load8(dres + off + col, rs[c]);
        load8(a + off + col, av[c]);   // all four streams are requested before the first reduction
        load8(w2 + col, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[c][j] = (xv[j] - mean2) * rstd2;
          acc2[c][j] += dv[j] * xh[c][j];
          g[c][j] = dv[j] * wv[j];
          row_bwd_acc(g[c][j], xh[c][j], s1, s2);
        }
      }
    }
    row_bwd_sums(inv_h, rms2, s1, s2);
    float t1 = 0.f, t2 = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float wv[8];
        load8(w1 + col, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d2 = row_dx(g[c][j], xh[c][j], s1, s2, rstd2) + rs[c][j];  // dx2
          rs[c][j] = d2;
          const float ah = (av[c][j] - mean1) * rstd1;
          av[c][j] = ah;
          acc1[c][j] += d2 * ah;
          g[c][j] = d2 * wv[j];
          row_bwd_acc(g[c][j], ah, t1, t2);
        }
        store8(dx2 + off + col, rs[c]);
      }
    }
    row_bwd_sums(inv_h, rms1, t1, t2);
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = row_dx(g[c][j], av[c][j], t1, t2, rstd1);
        store8(d_a + off + col, o);
      }
    }
  }
  float* my2 = s_dw + static_cast<size_t>(warp) * H;
  float* my1 = s_dw + static_cast<size_t>(kBwdWarps + warp) * H;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = row_col(c, lane);
    if (col < H) { store8(my2 + col, acc2[c]); store8(my1 + col, acc1[c]); }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    float u2 = 0.f, u1 = 0.f;
    for (int k = 0; k < kBwdWarps; ++k) {
      u2 += s_dw[static_cast<size_t>(k) * H + i];
      u1 += s_dw[static_cast<size_t>(kBwdWarps + k) * H + i];
    }
    dw2_ws[static_cast<size_t>(blockIdx.x) * H + i] = u2;
    dw1_ws[static_cast<size_t>(blockIdx.x) * H + i] = u1;
  }
}

// ---- wide rows (H > 1024): warp-per-row STREAMING kernels.  Nothing row-sized lives in registers:
// pass 1 streams the row for the statistics, pass 2 streams it again (L1/L2 hits) to produce the output.  Few
// registers -> many resident warps -> enough bytes in flight to approach HBM bandwidth without any block barrier.
// (A CTA-per-row variant with barriers measured 2-3x below the HBM roofline: two resident rows per SM.)

// v = value to normalise; ga8 = gelu'(x) (GELU mode)
template <typename TX>
__device__ __forceinline__ void load_value(const TX* xr, int col, int act, float (&v)[8], float (&ga8)[8]) {
  load8(xr + col, v);
  if (act == ACT_GELU) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float gv;
      gelu_eval(v[j], gv, ga8[j]);
      v[j] = gv;
    }
  }
}

constexpr int kWideWarps = 8;

template <typename TX, typename TY>
__global__ void __launch_bounds__(kWideWarps * 32)
norm_fwd_wide_kernel(const TX* __restrict__ x, const float* __restrict__ w, const float* __restrict__ res,
                     TY* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows, int H,
                     float eps, int act, int rms) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kWideWarps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const TX* xr = x + static_cast<size_t>(row) * H;
  float ga8[8];
  // pass 1: shifted single-pass moments (shift = first element of the row kills the cancellation in E[v^2]-E[v]^2)
  float shift;
  {
    float v0[8];
    if (lane == 0) load_value(xr, 0, act, v0, ga8);
    shift = rms ? 0.f : __shfl_sync(0xffffffffu, v0[0], 0);
  }
  float s = 0.f, ss = 0.f;
  for (int col = lane * 8; col < H; col += 256) {
    float v[8];
    load_value(xr, col, act, v, ga8);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float d = v[j] - shift; s += d; ss += d * d; }
  }
  s = warp_sum(s);
  ss = warp_sum(ss);
  const float inv_h = 1.0f / static_cast<float>(H);
  const float dm = rms ? 0.f : s * inv_h;          // mean - shift
  const float mean = shift + dm;
  const float var = fmaxf(ss * inv_h - dm * dm, 0.f);
  const float rstd = rsqrtf(var + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  TY* yr = y + static_cast<size_t>(row) * H;
  const float* rr = res ? res + static_cast<size_t>(row) * H : nullptr;
  for (int col = lane * 8; col < H; col += 256) {
    float v[8], o[8], wv[8];
    load_value(xr, col, act, v, ga8);
    if (w) load8(w + col, wv);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = (v[j] - mean) * rstd * (w ? wv[j] : 1.f);
    if (rr) {
      float r8[8];
      load8(rr + col, r8);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] += r8[j];
    }
    store8(yr + col, o);
  }
}

// Four CTAs per SM, the residency bwd_grid sizes the grid for (and 64 registers, so no spill).
template <typename TDY, typename TX, typename TDX>
__global__ void __launch_bounds__(kWideWarps * 32, 4)
norm_bwd_wide_kernel(const TDY* __restrict__ dy, const TX* __restrict__ x, const float* __restrict__ w,
                     const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                     const float* __restrict__ dres, TDX* __restrict__ dx, float* __restrict__ dw,
                     float* __restrict__ dw_ws, int rows, int H, int act, int rms) {
  pdl_enter();
  extern __shared__ __align__(16) float s_dw[];  // [kWideWarps][H] private per-warp weight-gradient rows
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  float* my_dw = s_dw + static_cast<size_t>(warp) * H;
  if (dw) {
    for (int i = lane * 4; i < H; i += 128) *reinterpret_cast<float4*>(my_dw + i) = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncwarp();
  }
  const float inv_h = 1.0f / static_cast<float>(H);
  for (int row = blockIdx.x * kWideWarps + warp; row < rows; row += gridDim.x * kWideWarps) {
    const TX* xr = x + static_cast<size_t>(row) * H;
    const TDY* dyr = dy + static_cast<size_t>(row) * H;
    const float mean = rms ? 0.f : mean_in[row];
    const float rstd = rstd_in[row];
    float s1 = 0.f, s2 = 0.f;
    for (int col = lane * 8; col < H; col += 256) {
      float v[8], ga8[8], dv[8], wv[8], pr[8];
      load_value(xr, col, act, v, ga8);
      load8(dyr + col, dv);
      if (w) load8(w + col, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (v[j] - mean) * rstd;
        const float g = dv[j] * (w ? wv[j] : 1.f);
        s1 += g;
        s2 += g * xh;
        pr[j] = dv[j] * xh;
      }
      if (dw) {
        float e[8];
        load8(my_dw + col, e);
#pragma unroll
        for (int j = 0; j < 8; ++j) e[j] += pr[j];
        store8(my_dw + col, e);
      }
    }
    s1 = rms ? 0.f : warp_sum(s1) * inv_h;
    s2 = warp_sum(s2) * inv_h;
    TDX* dxr = dx + static_cast<size_t>(row) * H;
    const float* drr = dres ? dres + static_cast<size_t>(row) * H : nullptr;
    for (int col = lane * 8; col < H; col += 256) {
      float v[8], ga8[8], dv[8], wv[8], o[8];
      load_value(xr, col, act, v, ga8);
      load8(dyr + col, dv);
      if (w) load8(w + col, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (v[j] - mean) * rstd;
        const float g = dv[j] * (w ? wv[j] : 1.f);
        o[j] = rstd * (g - s1 - xh * s2);
      }
      if (act == ACT_GELU) {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] *= ga8[j];
      }
      if (drr) {
        float r8[8];
        load8(drr + col, r8);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += r8[j];
      }
      store8(dxr + col, o);
    }
  }
  if (dw) flush_cta_dw(s_dw, kWideWarps, H, dw, dw_ws);
}

// ---- GLU + LayerNorm/RMSNorm fused (act = 2), the FeedForward middle of every normformer layer ([T, 2I] -> [T, I]).
// These two passes are compute-heavy for an "elementwise" op (erf, exp, rcp per element), so the GELU is evaluated
// exactly ONCE per element: forward keeps v = bf16(bf16(gelu(a)) * b) packed as bf16 pairs in registers between the
// statistics and the normalise pass (v is bf16-exact, so packing loses nothing); backward keeps bf16(gelu(a)) and
// gelu'(a) packed and re-reads b / dy from L2 for the second pass.  Weight gradients accumulate in a PRIVATE
// per-warp shared-memory row (plain vector read-modify-write; shared-memory float atomics cost ~64 cycles per warp
// instruction and made the first version of this kernel 4x slower than its HBM roofline).
constexpr int kGluWarps = 8;

// 16-byte read-only load that bypasses L1 allocation (streamed once)
__device__ __forceinline__ uint4 ld_nc16(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ uint32_t bf16x2_mul(uint32_t a, uint32_t b) {  // bf16 * bf16 -> bf16 (rn), two lanes
  __nv_bfloat162 r = __hmul2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b));
  return *reinterpret_cast<uint32_t*>(&r);
}

// forward: v = bf16(bf16(gelu(a)) * b) is produced directly as packed bf16 pairs (cvt.rn.bf16x2 + HMUL2.BF16) and
// stays in registers between the statistics and the normalise pass.
// The row's 2 * CH 16-byte loads are all issued before any math (CH <= 8: 64 registers of loads in flight per lane, two CTAs
// per SM): with the loads interleaved chunk by chunk only ~24 KB per SM were in flight, which by Little's law capped the
// kernel at ~3.7 TB/s whatever the instruction count (same-box A/B: 219 -> 193 us at [65 792, 2 x 2048]).  The backward
// got nothing from the same treatment (362 -> 360 us) at three CTAs per SM; its loads go through a shared-memory row ring
// instead (glu_norm_bwd_ring_kernel).
// F8 (never with DROP; H <= 4096): y is the e4m3 operand of muse_gemm_fp8 (TY = uint8_t) and row_scale [rows] its
// scales.  The normalised row is kept as fp32 register chunks (128 values per lane at H = 4096) until its amax is known,
// then stored with row_store_e4m3.
template <int CH, bool DROP, bool F8 = false, typename TY = bf16>
__global__ void __launch_bounds__(kGluWarps * 32, (CH <= 8) ? 2 : 1)
glu_norm_fwd_kernel(const bf16* __restrict__ ab, const float* __restrict__ w, TY* __restrict__ y,
                    float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows, int H, float eps, int rms,
                    const philox::ElemDrop drop, float* __restrict__ row_scale) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kGluWarps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const bf16* xr = ab + static_cast<size_t>(row) * 2 * H;
  uint32_t vp[CH][4];
  float sum = 0.f;
  constexpr bool kPf = CH <= 8;
  constexpr int PF = kPf ? CH : 1;  // chunks whose loads are in flight together
  uint4 aq[PF], bq[PF];
  if (kPf) {
#pragma unroll
    for (int c = 0; c < PF; ++c) {
      const int col = (c * 32 + lane) * 8;
      if (col < H) {
        aq[c] = ld_nc16(xr + col);
        bq[c] = ld_nc16(xr + H + col);
      }
    }
  }
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = (c * 32 + lane) * 8;
    if (col < H) {
      const uint4 au = kPf ? aq[c % PF] : *reinterpret_cast<const uint4*>(xr + col);
      const uint4 bu = kPf ? bq[c % PF] : *reinterpret_cast<const uint4*>(xr + H + col);
      const uint32_t aw[4] = {au.x, au.y, au.z, au.w}, bw[4] = {bu.x, bu.y, bu.z, bu.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 a2 = unpack_bf16(aw[j]);
        float g0, g1, d0, d1;
        gelu_eval(a2.x, g0, d0);
        gelu_eval(a2.y, g1, d1);
        vp[c][j] = bf16x2_mul(pack_bf16(g0, g1), bw[j]);
        const float2 v2 = unpack_bf16(vp[c][j]);
        sum += v2.x + v2.y;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) vp[c][j] = 0u;
    }
  }
  const float inv_h = 1.0f / static_cast<float>(H);
  const float mean = rms ? 0.f : warp_sum(sum) * inv_h;
  float sq = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    if ((c * 32 + lane) * 8 < H) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 p = unpack_bf16(vp[c][j]);
        const float dx = p.x - mean, dy_ = p.y - mean;
        sq = fmaf(dx, dx, sq);
        sq = fmaf(dy_, dy_, sq);
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) * inv_h + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  TY* yr = y + static_cast<size_t>(row) * H;
  unsigned long long seed = 0;
  if constexpr (DROP) seed = *drop.seed;
  float fv[F8 ? CH : 1][8];  // F8: the normalised row, zeros past H
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = (c * 32 + lane) * 8;
    if constexpr (F8) {
      if (col < H) {
        float wv[8];
        if (w) load8(w + col, wv);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 p = unpack_bf16(vp[c][j]);
          fv[c][2 * j] = (p.x - mean) * (w ? rstd * wv[2 * j] : rstd);
          fv[c][2 * j + 1] = (p.y - mean) * (w ? rstd * wv[2 * j + 1] : rstd);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) fv[c][j] = 0.f;
      }
    } else if (col < H) {
      float wv[8];
      if (w) load8(w + col, wv);
      uint32_t kb = 0xFFu;
      if constexpr (DROP) kb = philox::elem_keep8(seed, drop.site, static_cast<uint32_t>(row), col / 8, drop.thresh);
      uint4 ou;
      uint32_t* op = reinterpret_cast<uint32_t*>(&ou);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 p = unpack_bf16(vp[c][j]);
        float r0 = w ? rstd * wv[2 * j] : rstd, r1 = w ? rstd * wv[2 * j + 1] : rstd;
        if constexpr (DROP) {  // the dropped output is the wo operand (and what the wo weight gradient reads)
          r0 *= philox::keep_z(kb, 2 * j, drop.scale);
          r1 *= philox::keep_z(kb, 2 * j + 1, drop.scale);
        }
        op[j] = pack_bf16((p.x - mean) * r0, (p.y - mean) * r1);
      }
      *reinterpret_cast<uint4*>(yr + col) = ou;
      if constexpr (DROP) drop.bits[static_cast<size_t>(row) * drop.row_bytes + col / 8] = static_cast<uint8_t>(kb);
    } else if (DROP && col / 8 < drop.row_bytes) {
      drop.bits[static_cast<size_t>(row) * drop.row_bytes + col / 8] = 0;  // pad bytes of the row's last word
    }
  }
  if constexpr (F8) row_store_e4m3(fv, H, lane, yr, row_scale + row);
}

// backward: two streaming passes over the row with the GELU recomputed in the second one (nothing row-sized in
// registers -> 3 CTAs/SM); weight gradients go to a private per-warp shared-memory row.
// HAVE_Y: the saved forward output y = bf16(xhat * w) is available, so the first pass gets its two row reductions from
// (dy, y) alone -- s1 = mean(dy * w), s2 = mean(dy * w * xhat) = mean(dy * y) -- without reading [a | b] or evaluating the
// GELU, and the weight-gradient accumulation moves into the second pass.
// DROP (never with HAVE_Y: the saved output is the dropped one): dy is the gradient of the dropped output and is scaled
// by the stored keep bits as it is read, in both passes.
template <bool HAVE_Y, bool DROP>
__global__ void __launch_bounds__(kGluWarps * 32, 3)
glu_norm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ ab, const float* __restrict__ w,
                    const float* __restrict__ mean_in, const float* __restrict__ rstd_in, bf16* __restrict__ dab,
                    float* __restrict__ dw, float* __restrict__ dw_ws, const bf16* __restrict__ yf, int rows, int H,
                    int rms, const philox::ElemDrop drop) {
  static_assert(!(HAVE_Y && DROP), "the dropout backward recomputes the GLU product");
  pdl_enter();
  extern __shared__ __align__(16) float s_dw[];  // [kGluWarps][H] private rows
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  float* my_dw = s_dw + static_cast<size_t>(warp) * H;
  if (dw) {
    for (int i = lane * 4; i < H; i += 128) *reinterpret_cast<float4*>(my_dw + i) = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncwarp();
  }
  const float inv_h = 1.0f / static_cast<float>(H);
  for (int row = blockIdx.x * kGluWarps + warp; row < rows; row += gridDim.x * kGluWarps) {
    const bf16* xr = ab + static_cast<size_t>(row) * 2 * H;
    const bf16* dyr = dy + static_cast<size_t>(row) * H;
    const float mean = rms ? 0.f : mean_in[row];
    const float rstd = rstd_in[row];
    float s1 = 0.f, s2 = 0.f;
    // Software pipeline of L2 prefetch hints, two loop iterations (2 x 256 columns) ahead of the demand loads: lanes 0-3
    // request the four 128-byte lines per stream of the iteration after next -- first the rest of this pass, then the first
    // columns of the next pass / of this warp's next row.  (Prefetching whole rows one row ahead measured SLOWER here, 375 ->
    // 392 us: 3 552 warps x 16 KB of requested-but-unused lines do not survive in L2; for the H <= 1024 kernels it wins.)
    const int next = row + gridDim.x * kGluWarps;
    if (HAVE_Y) {
      const bf16* yr = yf + static_cast<size_t>(row) * H;
      for (int col = lane * 8; col < H; col += 256) {
        if (lane < 4) {
          const int nb = col - lane * 8 + 512 + lane * 64;
          if (nb < H) { prefetch_l2(dyr + nb); prefetch_l2(yr + nb); }
          else if (nb - H < H) { prefetch_l2(xr + (nb - H)); prefetch_l2(xr + H + (nb - H)); }
        }
        float d[8], yv[8], wv[8];
        load8(dyr + col, d);
        load8(yr + col, yv);
        if (w) load8(w + col, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s1 += w ? d[j] * wv[j] : d[j];
          s2 = fmaf(d[j], yv[j], s2);
        }
      }
    }
    for (int col = lane * 8; !HAVE_Y && col < H; col += 256) {
      const uint4 au = *reinterpret_cast<const uint4*>(xr + col);
      const uint4 bu = *reinterpret_cast<const uint4*>(xr + H + col);
      const uint4 du = *reinterpret_cast<const uint4*>(dyr + col);
      const uint32_t aw[4] = {au.x, au.y, au.z, au.w}, bw[4] = {bu.x, bu.y, bu.z, bu.w}, dd[4] = {du.x, du.y, du.z, du.w};
      float wv[8], pr[8];
      if (w) load8(w + col, wv);
      uint32_t kb = 0xFFu;
      if constexpr (DROP) kb = drop.bits[static_cast<size_t>(row) * drop.row_bytes + col / 8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 a2 = unpack_bf16(aw[j]);
        float g0, g1, t0, t1;
        gelu_eval(a2.x, g0, t0);
        gelu_eval(a2.y, g1, t1);
        const float2 v2 = unpack_bf16(bf16x2_mul(pack_bf16(g0, g1), bw[j]));
        float2 d2 = unpack_bf16(dd[j]);
        if constexpr (DROP) {
          d2.x *= philox::keep_z(kb, 2 * j, drop.scale);
          d2.y *= philox::keep_z(kb, 2 * j + 1, drop.scale);
        }
        const float xh0 = (v2.x - mean) * rstd, xh1 = (v2.y - mean) * rstd;
        const float q0 = w ? d2.x * wv[2 * j] : d2.x, q1 = w ? d2.y * wv[2 * j + 1] : d2.y;
        s1 += q0 + q1;
        s2 = fmaf(q0, xh0, s2);
        s2 = fmaf(q1, xh1, s2);
        pr[2 * j] = d2.x * xh0;
        pr[2 * j + 1] = d2.y * xh1;
      }
      if (dw) {
        float4 e0 = *reinterpret_cast<float4*>(my_dw + col);
        float4 e1 = *reinterpret_cast<float4*>(my_dw + col + 4);
        e0.x += pr[0]; e0.y += pr[1]; e0.z += pr[2]; e0.w += pr[3];
        e1.x += pr[4]; e1.y += pr[5]; e1.z += pr[6]; e1.w += pr[7];
        *reinterpret_cast<float4*>(my_dw + col) = e0;
        *reinterpret_cast<float4*>(my_dw + col + 4) = e1;
      }
    }
    s1 = rms ? 0.f : warp_sum(s1) * inv_h;
    s2 = warp_sum(s2) * inv_h;
    bf16* dr = dab + static_cast<size_t>(row) * 2 * H;
    for (int col = lane * 8; col < H; col += 256) {
      if (HAVE_Y && lane < 4) {
        const int nb = col - lane * 8 + 512 + lane * 64;
        if (nb < H) { prefetch_l2(xr + nb); prefetch_l2(xr + H + nb); }
        else if (next < rows && nb - H < H) {
          prefetch_l2(dy + static_cast<size_t>(next) * H + (nb - H));
          prefetch_l2(yf + static_cast<size_t>(next) * H + (nb - H));
        }
      }
      const uint4 au = *reinterpret_cast<const uint4*>(xr + col);
      const uint4 bu = *reinterpret_cast<const uint4*>(xr + H + col);
      const uint4 du = *reinterpret_cast<const uint4*>(dyr + col);
      const uint32_t aw[4] = {au.x, au.y, au.z, au.w}, bw[4] = {bu.x, bu.y, bu.z, bu.w}, dd[4] = {du.x, du.y, du.z, du.w};
      float wv[8];
      if (w) load8(w + col, wv);
      uint32_t kb = 0xFFu;
      if constexpr (DROP) kb = drop.bits[static_cast<size_t>(row) * drop.row_bytes + col / 8];
      uint4 oa, ob;
      float pr2[8];
      uint32_t* pa = reinterpret_cast<uint32_t*>(&oa);
      uint32_t* pb = reinterpret_cast<uint32_t*>(&ob);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 a2 = unpack_bf16(aw[j]);
        float g0, g1, t0, t1;
        gelu_eval(a2.x, g0, t0);
        gelu_eval(a2.y, g1, t1);
        const uint32_t gp = pack_bf16(g0, g1);
        const float2 gr = unpack_bf16(gp);  // bf16(gelu(a))
        const float2 v2 = unpack_bf16(bf16x2_mul(gp, bw[j]));
        const float2 b2 = unpack_bf16(bw[j]);
        float2 d2 = unpack_bf16(dd[j]);
        if constexpr (DROP) {
          d2.x *= philox::keep_z(kb, 2 * j, drop.scale);
          d2.y *= philox::keep_z(kb, 2 * j + 1, drop.scale);
        }
        const float xh0 = (v2.x - mean) * rstd, xh1 = (v2.y - mean) * rstd;
        const float q0 = w ? d2.x * wv[2 * j] : d2.x, q1 = w ? d2.y * wv[2 * j + 1] : d2.y;
        const float o0 = rstd * (q0 - s1 - xh0 * s2), o1 = rstd * (q1 - s1 - xh1 * s2);
        pa[j] = pack_bf16(o0 * b2.x * t0, o1 * b2.y * t1);
        pb[j] = pack_bf16(o0 * gr.x, o1 * gr.y);
        pr2[2 * j] = d2.x * xh0;
        pr2[2 * j + 1] = d2.y * xh1;
      }
      if (HAVE_Y && dw) {
        float4 e0 = *reinterpret_cast<float4*>(my_dw + col);
        float4 e1 = *reinterpret_cast<float4*>(my_dw + col + 4);
        e0.x += pr2[0]; e0.y += pr2[1]; e0.z += pr2[2]; e0.w += pr2[3];
        e1.x += pr2[4]; e1.y += pr2[5]; e1.z += pr2[6]; e1.w += pr2[7];
        *reinterpret_cast<float4*>(my_dw + col) = e0;
        *reinterpret_cast<float4*>(my_dw + col + 4) = e1;
      }
      *reinterpret_cast<uint4*>(dr + col) = oa;
      *reinterpret_cast<uint4*>(dr + H + col) = ob;
    }
  }
  if (dw) flush_cta_dw(s_dw, kGluWarps, H, dw, dw_ws);
}

// ---- row-ring backward kernels of a transformer layer: norm_bwd with dres (H <= 1024), norm2_bwd (H <= 512) and the GLU
// backward with the saved y (H <= 2048).  Same rows, same per-row arithmetic and same weight-gradient order as the
// register-path kernels above, which stay for the other cases, for inputs that are not 16-byte aligned, and as the
// cross-check of these (MUSE_NORM_BWD_RING=0).
// The register-path kernels load through registers and are bound by exposed load latency: a warp keeps its current row
// (plus a prefetch hint) in flight.  Here one producer thread per CTA copies the CTA's input rows, in the order the warps
// consume them, into a ring of row stages with 1-D bulk copies (a full / empty mbarrier per stage), and refills a stage
// as soon as its warp releases it.  The bytes in flight are then set by the ring, not by registers, and every input row
// is read from HBM exactly once (both passes of the GLU backward read dy from the stage).
// Row mapping: the register path runs G = bwd_grid(rows) CTAs of 8 warps, CTA b warp w taking rows b*8 + w + k*8G.  A
// ring CTA has 8 consumer warps and walks the "virtual CTAs" b = blockIdx.x, blockIdx.x + gridDim.x, ... < G one after
// the other with exactly that mapping.  Each warp keeps its weight-gradient partial in registers (a lane owns fixed
// columns, as norm_bwd_warp_kernel's does) and virtual CTA b's warp-ordered sum goes to dw_ws[b] as before, so dx and dw
// are bit-identical to the register path.
constexpr int kRingWarps = 8;                        // one virtual CTA: kBwdWarps == kGluWarps
constexpr int kRingThreads = (kRingWarps + 1) * 32;  // + the producer warp
constexpr int kRingStages = kRingWarps;              // see ring_plan
constexpr int kRingBarBytes = 2 * kRingStages * 8;   // full[], empty[]

struct RowRing {
  uint64_t* full;
  uint64_t* empty;
  uint8_t* stages;
  int nstages, stage_bytes;
  __device__ __forceinline__ uint8_t* stage(int n) const { return stages + static_cast<size_t>(n % nstages) * stage_bytes; }
  __device__ __forceinline__ uint32_t parity(int n) const { return static_cast<uint32_t>(n / nstages) & 1u; }
};

// Dynamic shared memory: barriers | sum_floats floats (the CTA's weight-gradient sums) | nstages row stages.
__host__ __device__ __forceinline__ int ring_sum_bytes(int sum_floats) { return (sum_floats * 4 + 127) & ~127; }

__device__ __forceinline__ RowRing ring_setup(uint8_t* smem, int nstages, int stage_bytes, int sum_floats, float*& s_sum) {
  RowRing r{reinterpret_cast<uint64_t*>(smem), reinterpret_cast<uint64_t*>(smem) + kRingStages,
            smem + kRingBarBytes + ring_sum_bytes(sum_floats), nstages, stage_bytes};
  s_sum = reinterpret_cast<float*>(smem + kRingBarBytes);
  if (threadIdx.x == 0) {
    for (int i = 0; i < nstages; ++i) {
      ptx::mbar_init(&r.full[i], 1);
      ptx::mbar_init(&r.empty[i], 1);  // the consuming warp
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  return r;
}

// Calls row_fn(n, row) for the CTA's rows in ring order (n counts them): every row for the producer (warp < 0), warp
// `warp`'s rows for a consumer; end_vb(vb) after each virtual CTA.
template <typename RowFn, typename EndFn>
__device__ __forceinline__ void ring_walk(int rows, int G, int warp, RowFn&& row_fn, EndFn&& end_vb) {
  int n0 = 0;
  for (int vb = blockIdx.x; vb < G; vb += gridDim.x) {
    for (int base = vb * kRingWarps; base < rows; base += G * kRingWarps) {
      const int cnt = min(kRingWarps, rows - base);
      if (warp < 0) {
        for (int i = 0; i < cnt; ++i) row_fn(n0 + i, base + i);
      } else {
        if (warp < cnt) row_fn(n0 + warp, base + warp);
        // No consumer starts a round before every row of the previous one is released: with nstages >= kRingWarps the
        // stage of ring position n has then completed the fill of n - nstages, so the parity wait cannot alias.
        ptx::named_barrier_sync(1, kRingWarps * 32);
      }
      n0 += cnt;
    }
    end_vb(vb);
  }
}

// Producer side of one row: waits for the stage to be released, arms its full barrier for `bytes` and hands it to
// copy(stage, bar), which issues the bulk copies.
template <typename CopyFn>
__device__ __forceinline__ void ring_produce(const RowRing& r, int n, uint32_t bytes, CopyFn&& copy) {
  ptx::mbar_wait(&r.empty[n % r.nstages], r.parity(n) ^ 1u);
  uint64_t* bar = &r.full[n % r.nstages];
  ptx::mbar_expect_tx(bar, bytes);
  copy(r.stage(n), bar);
}
__device__ __forceinline__ void ring_release(const RowRing& r, int n, int lane) {
  __syncwarp();
  if (lane == 0) ptx::mbar_arrive(&r.empty[n % r.nstages]);
}

// Virtual CTA vb's weight gradient from the consumer warps' register partials (which are reset): summed in warp order
// starting from 0 (flush_cta_dw's order) in s_sum, then stored to dw_ws[vb] or added to dw.
template <int CH>
__device__ __forceinline__ void ring_flush_dw(float (&acc)[CH][8], float* s_sum, int H, int warp, int lane, float* dw,
                                              float* dw_ws, int vb) {
  for (int k = 0; k < kRingWarps; ++k) {
    if (warp == k) {
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const int col = row_col(c, lane);
        if (col < H) {
          float e[8];
          if (k == 0) {
#pragma unroll
            for (int j = 0; j < 8; ++j) e[j] = 0.f;
          } else {
            load8(s_sum + col, e);
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) { e[j] += acc[c][j]; acc[c][j] = 0.f; }
          store8(s_sum + col, e);
        }
      }
    }
    ptx::named_barrier_sync(1, kRingWarps * 32);
  }
  for (int i = threadIdx.x; i < H; i += kRingWarps * 32) {
    if (dw_ws) dw_ws[static_cast<size_t>(vb) * H + i] = s_sum[i];
    else atomicAdd(&dw[i], s_sum[i]);
  }
  ptx::named_barrier_sync(1, kRingWarps * 32);  // s_sum is free for the next virtual CTA
}

// norm_bwd_warp_kernel on the ring, with dres.  Stage: x | dy | dres.
template <typename TDY, typename TX, typename TDX, int CH>
__global__ void __launch_bounds__(kRingThreads, 1)
norm_bwd_ring_kernel(const TDY* __restrict__ dy, const TX* __restrict__ x, const float* __restrict__ w,
                     const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                     const float* __restrict__ dres, TDX* __restrict__ dx, bf16* __restrict__ dx_copy,
                     float* __restrict__ dw, float* __restrict__ dw_ws, int rows, int H, int act, int rms, int G,
                     int nstages) {
  pdl_enter();
  extern __shared__ __align__(128) uint8_t smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int xb = H * static_cast<int>(sizeof(TX)), db = H * static_cast<int>(sizeof(TDY)), rb = H * 4;
  float* s_sum;
  const RowRing ring = ring_setup(smem, nstages, xb + db + rb, dw ? H : 0, s_sum);
  if (warp == kRingWarps) {
    if (lane == 0)
      ring_walk(rows, G, -1, [&](int n, int row) {
        ring_produce(ring, n, xb + db + rb, [&](uint8_t* st, uint64_t* bar) {
          ptx::bulk_load_1d(st, x + static_cast<size_t>(row) * H, xb, bar);
          ptx::bulk_load_1d(st + xb, dy + static_cast<size_t>(row) * H, db, bar);
          ptx::bulk_load_1d(st + xb + db, dres + static_cast<size_t>(row) * H, rb, bar);
        });
      }, [](int) {});
    return;
  }
  float dw_acc[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) dw_acc[c][j] = 0.f;
  const float inv_h = 1.0f / static_cast<float>(H);
  ring_walk(rows, G, warp, [&](int n, int row) {
    const float mean = rms ? 0.f : mean_in[row];
    const float rstd = rstd_in[row];
    ptx::mbar_wait(&ring.full[n % ring.nstages], ring.parity(n));
    const uint8_t* st = ring.stage(n);
    const TX* xr = reinterpret_cast<const TX*>(st);
    const TDY* dyr = reinterpret_cast<const TDY*>(st + xb);
    const float* drr = reinterpret_cast<const float*>(st + xb + db);
    // the register path's statements, with the row read from the stage instead of global memory
    float xh[CH][8], g[CH][8], rs[CH][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float xv[8], dv[8], wv[8];
        load8(xr + col, xv);
        load8(dyr + col, dv);
        if (drr) load8(drr + col, rs[c]);
        if (w) load8(w + col, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float a = act ? gelu_f(xv[j]) : xv[j];
          xh[c][j] = (a - mean) * rstd;
          dw_acc[c][j] += dv[j] * xh[c][j];
          g[c][j] = dv[j] * (w ? wv[j] : 1.f);
          row_bwd_acc(g[c][j], xh[c][j], s1, s2);
        }
      }
    }
    row_bwd_sums(inv_h, rms, s1, s2);
    TDX* dxr = dx + static_cast<size_t>(row) * H;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = row_dx(g[c][j], xh[c][j], s1, s2, rstd);
        if (act) {
          float xv[8];
          load8(xr + col, xv);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] *= gelu_grad_f(xv[j]);
        }
        if (drr) {
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += rs[c][j];
        }
        store8(dxr + col, o);
        if (dx_copy) store8(dx_copy + static_cast<size_t>(row) * H + col, o);
      }
    }
    ring_release(ring, n, lane);
  }, [&](int vb) {
    if (dw) ring_flush_dw(dw_acc, s_sum, H, warp, lane, dw, dw_ws, vb);
  });
}

// norm2_bwd_warp_kernel on the ring, H <= 512.  Stage: x2 | dres | d_h2 | a.  (At H = 1024 the register path's four row
// arrays and two weight-gradient partials spill.)
template <int CH>
__global__ void __launch_bounds__(kRingThreads, 1)
norm2_bwd_ring_kernel(const bf16* __restrict__ d_h2, const float* __restrict__ x2, const float* __restrict__ w2,
                      const float* __restrict__ mean2_in, const float* __restrict__ rstd2_in, const float* __restrict__ dres,
                      const bf16* __restrict__ a, const float* __restrict__ w1, const float* __restrict__ mean1_in,
                      const float* __restrict__ rstd1_in, float* __restrict__ dx2, bf16* __restrict__ d_a,
                      float* __restrict__ dw2_ws, float* __restrict__ dw1_ws, int rows, int H, int rms1, int rms2, int G,
                      int nstages) {
  pdl_enter();
  extern __shared__ __align__(128) uint8_t smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int fb = H * 4, hb = H * 2;
  float* s_sum;
  const RowRing ring = ring_setup(smem, nstages, 2 * fb + 2 * hb, H, s_sum);
  if (warp == kRingWarps) {
    if (lane == 0)
      ring_walk(rows, G, -1, [&](int n, int row) {
        ring_produce(ring, n, 2 * fb + 2 * hb, [&](uint8_t* st, uint64_t* bar) {
          const size_t off = static_cast<size_t>(row) * H;
          ptx::bulk_load_1d(st, x2 + off, fb, bar);
          ptx::bulk_load_1d(st + fb, dres + off, fb, bar);
          ptx::bulk_load_1d(st + 2 * fb, d_h2 + off, hb, bar);
          ptx::bulk_load_1d(st + 2 * fb + hb, a + off, hb, bar);
        });
      }, [](int) {});
    return;
  }
  float acc2[CH][8], acc1[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc2[c][j] = 0.f; acc1[c][j] = 0.f; }
  const float inv_h = 1.0f / static_cast<float>(H);
  ring_walk(rows, G, warp, [&](int n, int row) {
    const size_t off = static_cast<size_t>(row) * H;
    const float mean2 = rms2 ? 0.f : mean2_in[row], rstd2 = rstd2_in[row];
    const float mean1 = rms1 ? 0.f : mean1_in[row], rstd1 = rstd1_in[row];
    ptx::mbar_wait(&ring.full[n % ring.nstages], ring.parity(n));
    const uint8_t* st = ring.stage(n);
    const float* xr = reinterpret_cast<const float*>(st);
    const float* rr = reinterpret_cast<const float*>(st + fb);
    const bf16* dr = reinterpret_cast<const bf16*>(st + 2 * fb);
    const bf16* ar = reinterpret_cast<const bf16*>(st + 2 * fb + hb);
    // the register path's statements, with the row read from the stage instead of global memory
    float xh[CH][8], g[CH][8], rs[CH][8], av[CH][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float xv[8], dv[8], wv[8];
        load8(xr + col, xv);
        load8(dr + col, dv);
        load8(rr + col, rs[c]);
        load8(ar + col, av[c]);
        load8(w2 + col, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[c][j] = (xv[j] - mean2) * rstd2;
          acc2[c][j] += dv[j] * xh[c][j];
          g[c][j] = dv[j] * wv[j];
          row_bwd_acc(g[c][j], xh[c][j], s1, s2);
        }
      }
    }
    row_bwd_sums(inv_h, rms2, s1, s2);
    float t1 = 0.f, t2 = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float wv[8];
        load8(w1 + col, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d2 = row_dx(g[c][j], xh[c][j], s1, s2, rstd2) + rs[c][j];  // dx2
          rs[c][j] = d2;
          const float ah = (av[c][j] - mean1) * rstd1;
          av[c][j] = ah;
          acc1[c][j] += d2 * ah;
          g[c][j] = d2 * wv[j];
          row_bwd_acc(g[c][j], ah, t1, t2);
        }
        store8(dx2 + off + col, rs[c]);
      }
    }
    row_bwd_sums(inv_h, rms1, t1, t2);
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = row_dx(g[c][j], av[c][j], t1, t2, rstd1);
        store8(d_a + off + col, o);
      }
    }
    ring_release(ring, n, lane);
  }, [&](int vb) {
    ring_flush_dw(acc2, s_sum, H, warp, lane, nullptr, dw2_ws, vb);
    ring_flush_dw(acc1, s_sum, H, warp, lane, nullptr, dw1_ws, vb);
  });
}

// glu_norm_bwd_kernel<HAVE_Y = true> on the ring, for H <= 2048: the saved forward output y gives the first pass its
// sums, so a row is dy | y | [a | b], 8 H bytes, and dy is read from the stage by both passes.  (The dropout and
// recompute variants evaluate the GELU in both passes and stay on the register path.)  Products that the register path
// rounds before adding them -- behind a `w ?` select, or stored for the shared-memory read-modify-write -- are rounded
// here too (__fmul_rn), where unrolling would otherwise let the compiler fuse them into the add.
template <int CH>
__global__ void __launch_bounds__(kRingThreads, 1)
glu_norm_bwd_ring_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ ab, const float* __restrict__ w,
                         const float* __restrict__ mean_in, const float* __restrict__ rstd_in, bf16* __restrict__ dab,
                         float* __restrict__ dw, float* __restrict__ dw_ws, const bf16* __restrict__ yf, int rows, int H,
                         int rms, int G, int nstages) {
  pdl_enter();
  extern __shared__ __align__(128) uint8_t smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int hb = H * 2;
  float* s_sum;
  const RowRing ring = ring_setup(smem, nstages, 4 * hb, dw ? H : 0, s_sum);
  if (warp == kRingWarps) {
    if (lane == 0)
      ring_walk(rows, G, -1, [&](int n, int row) {
        ring_produce(ring, n, 4 * hb, [&](uint8_t* st, uint64_t* bar) {
          ptx::bulk_load_1d(st, dy + static_cast<size_t>(row) * H, hb, bar);
          ptx::bulk_load_1d(st + hb, yf + static_cast<size_t>(row) * H, hb, bar);
          ptx::bulk_load_1d(st + 2 * hb, ab + static_cast<size_t>(row) * 2 * H, 2 * hb, bar);
        });
      }, [](int) {});
    return;
  }
  float acc[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[c][j] = 0.f;
  const float inv_h = 1.0f / static_cast<float>(H);
  ring_walk(rows, G, warp, [&](int n, int row) {
    const float mean = rms ? 0.f : mean_in[row];
    const float rstd = rstd_in[row];
    ptx::mbar_wait(&ring.full[n % ring.nstages], ring.parity(n));
    const uint8_t* st = ring.stage(n);
    const bf16* dyr = reinterpret_cast<const bf16*>(st);
    const bf16* yr = reinterpret_cast<const bf16*>(st + hb);
    const bf16* xr = reinterpret_cast<const bf16*>(st + 2 * hb);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float d[8], yv[8], wv[8];
        load8(dyr + col, d);
        load8(yr + col, yv);
        if (w) load8(w + col, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s1 += w ? d[j] * wv[j] : d[j];
          s2 = fmaf(d[j], yv[j], s2);
        }
      }
    }
    s1 = rms ? 0.f : warp_sum(s1) * inv_h;
    s2 = warp_sum(s2) * inv_h;
    bf16* dr = dab + static_cast<size_t>(row) * 2 * H;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        const uint4 au = *reinterpret_cast<const uint4*>(xr + col);
        const uint4 bu = *reinterpret_cast<const uint4*>(xr + H + col);
        const uint4 du = *reinterpret_cast<const uint4*>(dyr + col);
        const uint32_t aw[4] = {au.x, au.y, au.z, au.w}, bw[4] = {bu.x, bu.y, bu.z, bu.w}, dd[4] = {du.x, du.y, du.z, du.w};
        float wv[8];
        if (w) load8(w + col, wv);
        uint4 oa, ob;
        uint32_t* pa = reinterpret_cast<uint32_t*>(&oa);
        uint32_t* pb = reinterpret_cast<uint32_t*>(&ob);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 a2 = unpack_bf16(aw[j]);
          float g0, g1, t0, t1;
          gelu_eval(a2.x, g0, t0);
          gelu_eval(a2.y, g1, t1);
          const uint32_t gp = pack_bf16(g0, g1);
          const float2 gr = unpack_bf16(gp);  // bf16(gelu(a))
          const float2 v2 = unpack_bf16(bf16x2_mul(gp, bw[j]));
          const float2 b2 = unpack_bf16(bw[j]);
          const float2 d2 = unpack_bf16(dd[j]);
          const float xh0 = (v2.x - mean) * rstd, xh1 = (v2.y - mean) * rstd;
          const float q0 = w ? __fmul_rn(d2.x, wv[2 * j]) : d2.x, q1 = w ? __fmul_rn(d2.y, wv[2 * j + 1]) : d2.y;
          const float o0 = rstd * (q0 - s1 - xh0 * s2), o1 = rstd * (q1 - s1 - xh1 * s2);
          pa[j] = pack_bf16(o0 * b2.x * t0, o1 * b2.y * t1);
          pb[j] = pack_bf16(o0 * gr.x, o1 * gr.y);
          acc[c][2 * j] += __fmul_rn(d2.x, xh0);
          acc[c][2 * j + 1] += __fmul_rn(d2.y, xh1);
        }
        *reinterpret_cast<uint4*>(dr + col) = oa;
        *reinterpret_cast<uint4*>(dr + H + col) = ob;
      }
    }
    ring_release(ring, n, lane);
  }, [&](int vb) {
    if (dw) ring_flush_dw(acc, s_sum, H, warp, lane, dw, dw_ws, vb);
  });
}

template <typename TX, typename TY>
int fwd_dispatch(const void* x, const float* w, const float* res, void* y, float* mean, float* rstd, int rows, int H,
                 float eps, int act, int rms, cudaStream_t s) {
  const TX* xp = reinterpret_cast<const TX*>(x);
  TY* yp = reinterpret_cast<TY*>(y);
  if (H <= 1024) {
    with_row_chunks<1, 2, 4>(H, [&](auto ch) {
      pdl_launch(ceil_div(rows, kWarpsPerBlock), kWarpsPerBlock * 32, 0, s)(
          norm_fwd_warp_kernel<TX, TY, decltype(ch)::value, false>, xp, w, res, yp, mean, rstd, rows, H, eps, act, rms,
          nullptr);
    });
  } else {
    pdl_launch(ceil_div(rows, kWideWarps), kWideWarps * 32, 0, s)(norm_fwd_wide_kernel<TX, TY>, xp, w, res, yp, mean, rstd,
                                                                  rows, H, eps, act, rms);
  }
  return check_launch("norm_fwd");
}

int bwd_grid(int rows, int H, int act) {
  if (act == ACT_GLU) { const int g = ceil_div(rows, kGluWarps); return g > 132 * 3 ? 132 * 3 : g; }
  if (H <= 1024) { const int g = ceil_div(rows, kBwdWarps); return g > 132 * 4 ? 132 * 4 : g; }
  const int g = ceil_div(rows, kWideWarps);
  return g > 132 * 4 ? 132 * 4 : g;
}

int reduce_dw(const float* dw_ws, float* dw, int grid, int H, cudaStream_t s) {
  pdl_launch(ceil_div(H, 32), 1024, 0, s)(colsum_ordered_kernel, dw_ws, dw, grid, H);
  return check_launch("norm_bwd colsum");
}

// Launch shape of a row-ring kernel: one CTA per SM, walking the G virtual CTAs, with kRingStages stages.  Eight
// stages -- one per consumer warp, the fewest ring_walk allows -- measured fastest for the GLU backward on an H100
// 80GB HBM3 (700 W): 574 us at [65 792, 2 x 2048] against 589 us with 10 and 716 us with 13, which leave the L1 cache
// (the same 256 KB as shared memory) too little room for the weight vector; the H = 512 passes measured within 3 %
// of each other from 8 stages up.  MUSE_NORM_BWD_RING=0 selects the register-path kernels instead (the reference the
// tests compare against).  stages == 0: take the register path.
struct RingPlan {
  int stages = 0, grid = 0;
  size_t smem = 0;
};
constexpr int kSms = 132;

RingPlan ring_plan(int G, int stage_bytes, int sum_floats, std::initializer_list<const void*> inputs) {
  RingPlan p;
  for (const void* q : inputs)
    if (reinterpret_cast<uintptr_t>(q) % 16 != 0) return p;  // the bulk copies need 16-byte aligned rows
  const char* env = getenv("MUSE_NORM_BWD_RING");
  if (env && env[0] == '0' && env[1] == 0) return p;
  const size_t smem = static_cast<size_t>(kRingBarBytes + ring_sum_bytes(sum_floats)) +
                      static_cast<size_t>(kRingStages) * stage_bytes;
  if (smem > 227 * 1024) return p;
  p.stages = kRingStages;
  p.smem = smem;
  p.grid = G < kSms ? G : kSms;
  return p;
}

template <typename TDY, typename TX, typename TDX>
int bwd_dispatch(const void* dy, const void* x, const float* w, const float* mean, const float* rstd,
                 const float* dres, void* dx, void* dx_copy, float* dw, float* dw_ws, int rows, int H, int act, int rms,
                 cudaStream_t s) {
  const int grid = bwd_grid(rows, H, act);
  const TDY* dyp = reinterpret_cast<const TDY*>(dy);
  const TX* xp = reinterpret_cast<const TX*>(x);
  TDX* dxp = reinterpret_cast<TDX*>(dx);
  const int stage_bytes = H * static_cast<int>(sizeof(TX) + sizeof(TDY) + sizeof(float));
  // the attention pre-norm of every layer (+ dres); the single norms of the embedding and the head stay on the register path
  const RingPlan rp = (dres && H <= 1024) ? ring_plan(grid, stage_bytes, dw ? H : 0, {dy, x, dres}) : RingPlan{};
  if (rp.stages) {
    with_row_chunks<1, 2, 4>(H, [&](auto ch) {
      constexpr int CH = decltype(ch)::value;
      allow_dynamic_smem_once<norm_bwd_ring_kernel<TDY, TX, TDX, CH>>(227 * 1024);
      pdl_launch(rp.grid, kRingThreads, rp.smem, s)(norm_bwd_ring_kernel<TDY, TX, TDX, CH>, dyp, xp, w, mean, rstd, dres,
                                                    dxp, reinterpret_cast<bf16*>(dx_copy), dw, dw_ws, rows, H, act, rms,
                                                    grid, rp.stages);
    });
  } else if (H <= 1024) {
    const size_t smem = dw ? static_cast<size_t>(kBwdWarps) * H * sizeof(float) : 0;
    with_row_chunks<1, 2, 4>(H, [&](auto ch) {
      pdl_launch(grid, kBwdWarps * 32, smem, s)(norm_bwd_warp_kernel<TDY, TX, TDX, decltype(ch)::value>, dyp, xp, w, mean,
                                                rstd, dres, dxp, reinterpret_cast<bf16*>(dx_copy), dw, dw_ws, rows, H, act,
                                                rms);
    });
  } else {
    if (dx_copy) { set_last_error("norm_bwd: the bf16 copy of dx is only produced for H <= 1024"); return MUSE_ERR_UNSUPPORTED; }
    const size_t smem = dw ? static_cast<size_t>(kWideWarps) * H * sizeof(float) : 0;
    allow_dynamic_smem_once<norm_bwd_wide_kernel<TDY, TX, TDX>>(kWideWarps * 4096 * 4);
    pdl_launch(grid, kWideWarps * 32, smem, s)(norm_bwd_wide_kernel<TDY, TX, TDX>, dyp, xp, w, mean, rstd, dres, dxp, dw,
                                               dw_ws, rows, H, act, rms);
  }
  int rc = check_launch("norm_bwd");
  if (rc || !dw || !dw_ws) return rc;
  return reduce_dw(dw_ws, dw, grid, H, s);
}

int check_args(const char* who, int H, int act, const void* res_or_dres) {
  if (H % 8 != 0 || H > 4096 || H < 8) {
    set_last_error("%s: H=%d must be a multiple of 8 in [8, 4096]", who, H);
    return MUSE_ERR_UNSUPPORTED;
  }
  if (act < 0 || act > 2) { set_last_error("%s: bad act %d", who, act); return MUSE_ERR_INVALID; }
  if (act == ACT_GLU && res_or_dres) { set_last_error("%s: GLU mode does not take a residual", who); return MUSE_ERR_INVALID; }
  return MUSE_OK;
}

}  // namespace
}  // namespace muse

using namespace muse;

extern "C" {

// dtype codes: 0 = fp32, 1 = bf16.  act: 0 none, 1 GELU(x), 2 GLU (x is [rows, 2H]).
// bits (act 2, bf16 in and out): FeedForward.dropout fused into the GLU + mid norm pass, y is the dropped output and bits
// [rows, ceil(H / 32)] uint32 words are written (philox.cuh elementwise mapping, seed read from *seed).
int muse_norm_fwd(const void* x, int x_dt, const float* w, const float* res, void* y, int y_dt, float* mean, float* rstd,
                  unsigned int* bits, const unsigned long long* seed, int site, float p, int rows, int H, float eps,
                  int act, int rms, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0) return MUSE_OK;
  int rc = check_args("norm_fwd", H, act, res);
  if (rc) return rc;
  if (bits != nullptr && (act != ACT_GLU || x_dt != 1 || y_dt != 1 || seed == nullptr)) {
    set_last_error("norm_fwd: dropout needs act 2, bf16 x and y, and a seed");
    return MUSE_ERR_INVALID;
  }
  if (act == ACT_GLU && (x_dt == 0 || y_dt == 0)) {
    set_last_error("norm_fwd: GLU mode (act 2) takes bf16 x and y only");
    return MUSE_ERR_UNSUPPORTED;
  }
  if (act == ACT_GLU && x_dt == 1 && y_dt == 1) {
    const philox::ElemDrop drop = philox::elem_drop(bits, seed, site, p, H);
    with_row_chunks<1, 2, 4, 8, 16>(H, [&](auto ch) {
      constexpr int CH = decltype(ch)::value;
      pdl_launch(ceil_div(rows, kGluWarps), kGluWarps * 32, 0, s)(
          bits ? glu_norm_fwd_kernel<CH, true> : glu_norm_fwd_kernel<CH, false>, reinterpret_cast<const bf16*>(x), w,
          reinterpret_cast<bf16*>(y), mean, rstd, rows, H, eps, rms, drop, nullptr);
    });
    return check_launch("glu_norm_fwd");
  }
  return dtype_dispatch("norm_fwd", [&](auto x_t, auto y_t) {
    return fwd_dispatch<decltype(x_t), decltype(y_t)>(x, w, res, y, mean, rstd, rows, H, eps, act, rms, s);
  }, x_dt, y_dt);
}

// x2 = res + norm1(a) * w1 ; h2 = norm2(x2) * w2  (a bf16 [rows,H], res / x2 fp32, h2 bf16; H % 8 == 0, H <= 1024)
int muse_norm2_fwd(const void* a, const float* res, const float* w1, const float* w2, float* x2, void* h2, float* mean1,
                   float* rstd1, float* mean2, float* rstd2, int rows, int H, float eps, int rms1, int rms2, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0) return MUSE_OK;
  if (H % 8 != 0 || H > 1024 || H < 8) { set_last_error("norm2_fwd: H=%d must be a multiple of 8 in [8, 1024]", H); return MUSE_ERR_UNSUPPORTED; }
  with_row_chunks<1, 2, 4>(H, [&](auto ch) {
    pdl_launch(ceil_div(rows, kWarpsPerBlock), kWarpsPerBlock * 32, 0, s)(
        norm2_fwd_warp_kernel<decltype(ch)::value, false>, reinterpret_cast<const bf16*>(a), res, w1, w2, x2,
        reinterpret_cast<bf16*>(h2), mean1, rstd1, mean2, rstd2, rows, H, eps, rms1, rms2, nullptr);
  });
  return check_launch("norm2_fwd");
}

// e4m3 forms of muse_norm_fwd (act 0, H <= 1024; act 2, H <= 4096, no dropout) and muse_norm2_fwd: the operands of the
// FP8 GEMMs of MaskGitTransformer.  q e4m3 [rows, H], row_scale fp32 [rows]; statistics as the bf16 forms.
int muse_norm_fwd_e4m3(const void* x, int x_dt, const float* w, const float* res, void* q, float* row_scale, float* mean,
                       float* rstd, int rows, int H, float eps, int act, int rms, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0) return MUSE_OK;
  int rc = check_args("norm_fwd_e4m3", H, act, res);
  if (rc) return rc;
  if (q == nullptr || row_scale == nullptr) { set_last_error("norm_fwd_e4m3: needs q and row_scale"); return MUSE_ERR_INVALID; }
  uint8_t* qp = reinterpret_cast<uint8_t*>(q);
  if (act == ACT_GLU) {
    if (x_dt != 1) { set_last_error("norm_fwd_e4m3: GLU mode (act 2) takes bf16 x only"); return MUSE_ERR_UNSUPPORTED; }
    with_row_chunks<1, 2, 4, 8, 16>(H, [&](auto ch) {
      constexpr int CH = decltype(ch)::value;
      pdl_launch(ceil_div(rows, kGluWarps), kGluWarps * 32, 0, s)(
          glu_norm_fwd_kernel<CH, false, true, uint8_t>, reinterpret_cast<const bf16*>(x), w, qp, mean, rstd, rows, H, eps,
          rms, philox::ElemDrop{}, row_scale);
    });
    return check_launch("glu_norm_fwd_e4m3");
  }
  if (act != ACT_NONE || H > 1024) {
    set_last_error("norm_fwd_e4m3: act %d, H %d (act 0 with H <= 1024, or act 2)", act, H);
    return MUSE_ERR_UNSUPPORTED;
  }
  return dtype_dispatch("norm_fwd_e4m3", [&](auto x_t) {
    using TX = decltype(x_t);
    with_row_chunks<1, 2, 4>(H, [&](auto ch) {
      pdl_launch(ceil_div(rows, kWarpsPerBlock), kWarpsPerBlock * 32, 0, s)(
          norm_fwd_warp_kernel<TX, uint8_t, decltype(ch)::value, true>, reinterpret_cast<const TX*>(x), w, res, qp, mean,
          rstd, rows, H, eps, act, rms, row_scale);
    });
    return check_launch("norm_fwd_e4m3");
  }, x_dt);
}

int muse_norm2_fwd_e4m3(const void* a, const float* res, const float* w1, const float* w2, float* x2, void* q,
                        float* row_scale, float* mean1, float* rstd1, float* mean2, float* rstd2, int rows, int H, float eps,
                        int rms1, int rms2, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0) return MUSE_OK;
  if (H % 8 != 0 || H > 1024 || H < 8) { set_last_error("norm2_fwd_e4m3: H=%d must be a multiple of 8 in [8, 1024]", H); return MUSE_ERR_UNSUPPORTED; }
  if (q == nullptr || row_scale == nullptr) { set_last_error("norm2_fwd_e4m3: needs q and row_scale"); return MUSE_ERR_INVALID; }
  with_row_chunks<1, 2, 4>(H, [&](auto ch) {
    pdl_launch(ceil_div(rows, kWarpsPerBlock), kWarpsPerBlock * 32, 0, s)(
        norm2_fwd_warp_kernel<decltype(ch)::value, true, uint8_t>, reinterpret_cast<const bf16*>(a), res, w1, w2, x2,
        reinterpret_cast<uint8_t*>(q), mean1, rstd1, mean2, rstd2, rows, H, eps, rms1, rms2, row_scale);
  });
  return check_launch("norm2_fwd_e4m3");
}

// ws: 2 * norm_bwd_workspace_floats(rows, H, 0) floats (dw2 partial rows, then dw1 partial rows); dw2 / dw1 are STORED.
int muse_norm2_bwd(const void* d_h2, const float* x2, const float* w2, const float* mean2, const float* rstd2, const float* dres,
                   const void* a, const float* w1, const float* mean1, const float* rstd1, float* dx2, void* d_a, float* dw2,
                   float* dw1, float* ws, int rows, int H, int rms1, int rms2, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0) return MUSE_OK;
  if (H % 8 != 0 || H > 1024 || H < 8) { set_last_error("norm2_bwd: H=%d must be a multiple of 8 in [8, 1024]", H); return MUSE_ERR_UNSUPPORTED; }
  const int grid = bwd_grid(rows, H, 0);
  float* ws2 = ws;
  float* ws1 = ws + static_cast<size_t>(grid) * H;
  const RingPlan rp = H <= 512 ? ring_plan(grid, 12 * H, H, {d_h2, x2, dres, a}) : RingPlan{};
  if (rp.stages) {
    with_row_chunks<1, 2>(H, [&](auto ch) {
      constexpr int CH = decltype(ch)::value;
      allow_dynamic_smem_once<norm2_bwd_ring_kernel<CH>>(227 * 1024);
      pdl_launch(rp.grid, kRingThreads, rp.smem, s)(norm2_bwd_ring_kernel<CH>, reinterpret_cast<const bf16*>(d_h2), x2, w2,
                                                    mean2, rstd2, dres, reinterpret_cast<const bf16*>(a), w1, mean1, rstd1,
                                                    dx2, reinterpret_cast<bf16*>(d_a), ws2, ws1, rows, H, rms1, rms2, grid,
                                                    rp.stages);
    });
  } else {
    const size_t smem = static_cast<size_t>(2) * kBwdWarps * H * sizeof(float);
    with_row_chunks<1, 2, 4>(H, [&](auto ch) {
      constexpr int CH = decltype(ch)::value;
      allow_dynamic_smem_once<norm2_bwd_warp_kernel<CH>>(2 * kBwdWarps * 1024 * 4);
      pdl_launch(grid, kBwdWarps * 32, smem, s)(norm2_bwd_warp_kernel<CH>, reinterpret_cast<const bf16*>(d_h2), x2, w2,
                                                mean2, rstd2, dres, reinterpret_cast<const bf16*>(a), w1, mean1, rstd1, dx2,
                                                reinterpret_cast<bf16*>(d_a), ws2, ws1, rows, H, rms1, rms2);
    });
  }
  int rc = check_launch("norm2_bwd");
  if (rc) return rc;
  if ((rc = reduce_dw(ws2, dw2, grid, H, s))) return rc;
  return reduce_dw(ws1, dw1, grid, H, s);
}

// floats of workspace a deterministic (dw_ws != nullptr) backward needs: one partial row of H per CTA
long long muse_norm_bwd_workspace_floats(int rows, int H, int act) {
  if (rows <= 0) return 0;
  return static_cast<long long>(bwd_grid(rows, H, act)) * H;
}

int muse_norm_bwd(const void* dy, int dy_dt, const void* x, int x_dt, const float* w, const float* mean, const float* rstd,
                  const float* dres, const void* y_fwd, const unsigned int* bits, float p, void* dx, int dx_dt,
                  void* dx_copy, float* dw, float* dw_ws, int rows, int H, int act, int rms, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0) return MUSE_OK;
  int rc = check_args("norm_bwd", H, act, dres);
  if (rc) return rc;
  if (dx_copy && (dx_dt != 0 || act == ACT_GLU)) { set_last_error("norm_bwd: dx_copy needs an fp32 dx and no GLU"); return MUSE_ERR_INVALID; }
  // with bits, dy is the gradient of the dropped output: scaled by the bits as it is read, the GLU product recomputed
  if (bits != nullptr && (act != ACT_GLU || dy_dt != 1 || x_dt != 1 || dx_dt != 1 || y_fwd != nullptr)) {
    set_last_error("norm_bwd: dropout needs act 2, bf16 dy, x and dx, and no y_fwd");
    return MUSE_ERR_INVALID;
  }
  if (act == ACT_GLU && (dy_dt == 0 || x_dt == 0 || dx_dt == 0)) {
    set_last_error("norm_bwd: GLU mode (act 2) takes bf16 dy, x and dx only");
    return MUSE_ERR_UNSUPPORTED;
  }
  if (act == ACT_GLU && dy_dt == 1 && x_dt == 1 && dx_dt == 1) {
    const int grid = bwd_grid(rows, H, act);
    const size_t smem = dw ? static_cast<size_t>(kGluWarps) * H * sizeof(float) : 0;
    const philox::ElemDrop drop = philox::elem_drop(const_cast<unsigned int*>(bits), nullptr, 0, p, H);
    const RingPlan rp = (y_fwd && H <= 2048) ? ring_plan(grid, 8 * H, dw ? H : 0, {dy, x, y_fwd}) : RingPlan{};
    if (rp.stages) {
      with_row_chunks<1, 2, 4, 8>(H, [&](auto ch) {
        constexpr int CH = decltype(ch)::value;
        allow_dynamic_smem_once<glu_norm_bwd_ring_kernel<CH>>(227 * 1024);
        pdl_launch(rp.grid, kRingThreads, rp.smem, s)(glu_norm_bwd_ring_kernel<CH>, reinterpret_cast<const bf16*>(dy),
            reinterpret_cast<const bf16*>(x), w, mean, rstd, reinterpret_cast<bf16*>(dx), dw, dw_ws,
            reinterpret_cast<const bf16*>(y_fwd), rows, H, rms, grid, rp.stages);
      });
      rc = check_launch("glu_norm_bwd");
      if (rc || !dw || !dw_ws) return rc;
      return reduce_dw(dw_ws, dw, grid, H, s);
    }
    allow_dynamic_smem_once<glu_norm_bwd_kernel<false, false>, glu_norm_bwd_kernel<true, false>,
                            glu_norm_bwd_kernel<false, true>>(kGluWarps * 4096 * 4);
    if (y_fwd != nullptr)
      pdl_launch(grid, kGluWarps * 32, smem, s)(glu_norm_bwd_kernel<true, false>,
          reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(x), w, mean, rstd, reinterpret_cast<bf16*>(dx), dw,
          dw_ws, reinterpret_cast<const bf16*>(y_fwd), rows, H, rms, drop);
    else
      pdl_launch(grid, kGluWarps * 32, smem, s)(bits ? glu_norm_bwd_kernel<false, true> : glu_norm_bwd_kernel<false, false>,
          reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(x), w, mean, rstd, reinterpret_cast<bf16*>(dx), dw,
          dw_ws, nullptr, rows, H, rms, drop);
    rc = check_launch("glu_norm_bwd");
    if (rc || !dw || !dw_ws) return rc;
    return reduce_dw(dw_ws, dw, grid, H, s);
  }
  return dtype_dispatch("norm_bwd", [&](auto dy_t, auto x_t, auto dx_t) {
    return bwd_dispatch<decltype(dy_t), decltype(x_t), decltype(dx_t)>(dy, x, w, mean, rstd, dres, dx, dx_copy, dw, dw_ws,
                                                                       rows, H, act, rms, s);
  }, dy_dt, x_dt, dx_dt);
}

}  // extern "C"
