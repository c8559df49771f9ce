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
#include "common.cuh"

namespace muse {
namespace {

constexpr int ACT_NONE = 0, ACT_GELU = 1, ACT_GLU = 2;

// ---- warp-per-row kernels (H <= 1024, no GLU): the whole row lives in registers, no block barriers
constexpr int kWarpsPerBlock = 4;

template <typename TX, typename TY, int CH>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
norm_fwd_warp_kernel(const TX* __restrict__ x, const float* __restrict__ w, const float* __restrict__ res,
                TY* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows, int H,
                float eps, int act, int rms) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (row >= rows) return;
  const TX* xr = x + static_cast<size_t>(row) * H;
  float v[CH][8];
  float sum = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = (c * 32 + lane) * 8;
    if (col < H) {
      load8(xr + col, v[c]);
      if (act) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[c][j] = gelu_f(v[c][j]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[c][j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[c][j] = 0.f;
    }
  }
  const float inv_h = 1.0f / static_cast<float>(H);
  float mean = rms ? 0.f : warp_sum(sum) * inv_h;
  float sq = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = (c * 32 + lane) * 8;
    if (col < H) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[c][j] - mean;
        sq += d * d;
      }
    }
  }
  const float var = warp_sum(sq) * inv_h;
  const float rstd = rsqrtf(var + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  TY* yr = y + static_cast<size_t>(row) * H;
  const float* rr = res ? res + static_cast<size_t>(row) * H : nullptr;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = (c * 32 + lane) * 8;
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
      store8(yr + col, o);
    }
  }
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

// L2 prefetch (a hint: no register, no scoreboard entry).  The persistent row-streaming backward kernels are bound by
// exposed load latency rather than by issue slots or DRAM bandwidth.  A warp walks its rows strictly one after the
// other, so the lines of the row it will touch NEXT are requested from HBM while the current row is processed and the demand
// loads become L2 hits.  prefetch_row: the lanes of a warp cover the 128-byte lines of one row of H elements.
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
template <typename T>
__device__ __forceinline__ void prefetch_row(const T* row, int H, int lane) {
  const int bytes = H * static_cast<int>(sizeof(T));
  for (int off = lane * 128; off < bytes; off += 32 * 128) prefetch_l2(reinterpret_cast<const char*>(row) + off);
}
// Next-row prefetch for the LayerNorm backward, two iterations ahead for GLU + LayerNorm backward.  The kernels take the
// switch as an argument so that an A/B comparison needs one binary.
constexpr int kRowPrefetch = 1;

template <typename TDY, typename TX, typename TDX, int CH>
__global__ void __launch_bounds__(kBwdWarps * 32)
norm_bwd_warp_kernel(const TDY* __restrict__ dy, const TX* __restrict__ x, const float* __restrict__ w,
                const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                const float* __restrict__ dres, TDX* __restrict__ dx, bf16* __restrict__ dx_copy, float* __restrict__ dw,
                float* __restrict__ dw_ws, int rows, int H, int act, int rms, int pf) {
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
    if (pf && next < rows) {  // this warp's next row (see prefetch_row)
      prefetch_row(x + static_cast<size_t>(next) * H, H, lane);
      prefetch_row(dy + static_cast<size_t>(next) * H, H, lane);
      if (dres) prefetch_row(dres + static_cast<size_t>(next) * H, H, lane);
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = (c * 32 + lane) * 8;
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
          s1 += g[c][j];
          s2 += g[c][j] * xh[c][j];
        }
      }
    }
    s1 = rms ? 0.f : warp_sum(s1) * inv_h;
    s2 = warp_sum(s2) * inv_h;
    TDX* dxr = dx + static_cast<size_t>(row) * H;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = (c * 32 + lane) * 8;
      if (col < H) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (g[c][j] - s1 - xh[c][j] * s2);
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
      const int col = (c * 32 + lane) * 8;
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
template <int CH>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
norm2_fwd_warp_kernel(const bf16* __restrict__ a, const float* __restrict__ res, const float* __restrict__ w1,
                      const float* __restrict__ w2, float* __restrict__ x2, bf16* __restrict__ h2,
                      float* __restrict__ mean1_out, float* __restrict__ rstd1_out, float* __restrict__ mean2_out,
                      float* __restrict__ rstd2_out, int rows, int H, float eps, int rms1, int rms2) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float inv_h = 1.0f / static_cast<float>(H);
  float v[CH][8];
  float sum = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = (c * 32 + lane) * 8;
    if (col < H) {
      load8(a + static_cast<size_t>(row) * H + col, v[c]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[c][j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[c][j] = 0.f;
    }
  }
  const float mean1 = rms1 ? 0.f : warp_sum(sum) * inv_h;
  float sq = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c)
    if ((c * 32 + lane) * 8 < H) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = v[c][j] - mean1; sq += d * d; }
    }
  const float rstd1 = rsqrtf(warp_sum(sq) * inv_h + eps);
  // x2 = res + norm1(a) * w1  (kept in v), second statistics over x2
  float sum2 = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = (c * 32 + lane) * 8;
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
  const float mean2 = rms2 ? 0.f : warp_sum(sum2) * inv_h;
  float sq2 = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c)
    if ((c * 32 + lane) * 8 < H) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = v[c][j] - mean2; sq2 += d * d; }
    }
  const float rstd2 = rsqrtf(warp_sum(sq2) * inv_h + eps);
  if (lane == 0) {
    if (mean1_out) { mean1_out[row] = mean1; rstd1_out[row] = rstd1; mean2_out[row] = mean2; rstd2_out[row] = rstd2; }
  }
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = (c * 32 + lane) * 8;
    if (col < H) {
      float wv[8], o[8];
      load8(w2 + col, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[c][j] - mean2) * rstd2 * wv[j];
      store8(h2 + static_cast<size_t>(row) * H + col, o);
    }
  }
}

// backward of the pair: dx2 = LN2_bwd(d_h2; x2) + dres ; d_a = LN1_bwd(dx2; a) ; dw2 += d_h2 * x2hat ; dw1 += dx2 * ahat
template <int CH>
__global__ void __launch_bounds__(kBwdWarps * 32)
norm2_bwd_warp_kernel(const bf16* __restrict__ d_h2, const float* __restrict__ x2, const float* __restrict__ w2,
                      const float* __restrict__ mean2_in, const float* __restrict__ rstd2_in, const float* __restrict__ dres,
                      const bf16* __restrict__ a, const float* __restrict__ w1, const float* __restrict__ mean1_in,
                      const float* __restrict__ rstd1_in, float* __restrict__ dx2, bf16* __restrict__ d_a,
                      float* __restrict__ dw2_ws, float* __restrict__ dw1_ws, int rows, int H, int rms1, int rms2, int pf) {
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
    if (pf && next < rows) {  // this warp's next row (see prefetch_row)
      const size_t noff = static_cast<size_t>(next) * H;
      prefetch_row(x2 + noff, H, lane);
      prefetch_row(d_h2 + noff, H, lane);
      prefetch_row(dres + noff, H, lane);
      prefetch_row(a + noff, H, lane);
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = (c * 32 + lane) * 8;
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
          s1 += g[c][j];
          s2 += g[c][j] * xh[c][j];
        }
      }
    }
    s1 = rms2 ? 0.f : warp_sum(s1) * inv_h;
    s2 = warp_sum(s2) * inv_h;
    float t1 = 0.f, t2 = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = (c * 32 + lane) * 8;
      if (col < H) {
        float wv[8];
        load8(w1 + col, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d2 = rstd2 * (g[c][j] - s1 - xh[c][j] * s2) + rs[c][j];  // dx2
          rs[c][j] = d2;
          const float ah = (av[c][j] - mean1) * rstd1;
          av[c][j] = ah;
          acc1[c][j] += d2 * ah;
          g[c][j] = d2 * wv[j];
          t1 += g[c][j];
          t2 += g[c][j] * ah;
        }
        store8(dx2 + off + col, rs[c]);
      }
    }
    t1 = rms1 ? 0.f : warp_sum(t1) * inv_h;
    t2 = warp_sum(t2) * inv_h;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = (c * 32 + lane) * 8;
      if (col < H) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd1 * (g[c][j] - t1 - av[c][j] * t2);
        store8(d_a + off + col, o);
      }
    }
  }
  float* my2 = s_dw + static_cast<size_t>(warp) * H;
  float* my1 = s_dw + static_cast<size_t>(kBwdWarps + warp) * H;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = (c * 32 + lane) * 8;
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

// ---- wide rows (H > 1024) and GLU mode: warp-per-row STREAMING kernels.  Nothing row-sized lives in registers:
// pass 1 streams the row for the statistics, pass 2 streams it again (L1/L2 hits) to produce the output.  Few
// registers -> many resident warps -> enough bytes in flight to approach HBM bandwidth without any block barrier.
// (A CTA-per-row variant with barriers measured 2-3x below the HBM roofline: two resident rows per SM.)

// v = value to normalise; gv8 = bf16(gelu(a)) and ga8 = gelu'(a) (GLU / GELU modes), b8 = the linear GLU half
template <typename TX>
__device__ __forceinline__ void load_value(const TX* xr, int col, int H, int act, float (&v)[8], float (&gv8)[8],
                                           float (&ga8)[8], float (&b8)[8]) {
  if (act == ACT_GLU) {
    float a8[8];
    load8(xr + col, a8);
    load8(xr + H + col, b8);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float gv;
      gelu_eval(a8[j], gv, ga8[j]);
      gv8[j] = bf16_round(gv);
      v[j] = bf16_round(gv8[j] * b8[j]);
    }
  } else {
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
  const int xs = (act == ACT_GLU) ? 2 * H : H;
  const TX* xr = x + static_cast<size_t>(row) * xs;
  float gv8[8], ga8[8], b8[8];
  // pass 1: shifted single-pass moments (shift = first element of the row kills the cancellation in E[v^2]-E[v]^2)
  float shift;
  {
    float v0[8];
    if (lane == 0) load_value(xr, 0, H, act, v0, gv8, ga8, b8);
    shift = rms ? 0.f : __shfl_sync(0xffffffffu, v0[0], 0);
  }
  float s = 0.f, ss = 0.f;
  for (int col = lane * 8; col < H; col += 256) {
    float v[8];
    load_value(xr, col, H, act, v, gv8, ga8, b8);
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
    load_value(xr, col, H, act, v, gv8, ga8, b8);
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

template <typename TDY, typename TX, typename TDX>
__global__ void __launch_bounds__(kWideWarps * 32)
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
  const int xs = (act == ACT_GLU) ? 2 * H : H;
  const float inv_h = 1.0f / static_cast<float>(H);
  for (int row = blockIdx.x * kWideWarps + warp; row < rows; row += gridDim.x * kWideWarps) {
    const TX* xr = x + static_cast<size_t>(row) * xs;
    const TDY* dyr = dy + static_cast<size_t>(row) * H;
    const float mean = rms ? 0.f : mean_in[row];
    const float rstd = rstd_in[row];
    float s1 = 0.f, s2 = 0.f;
    for (int col = lane * 8; col < H; col += 256) {
      float v[8], gv8[8], ga8[8], b8[8], dv[8], wv[8], pr[8];
      load_value(xr, col, H, act, v, gv8, ga8, b8);
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
    TDX* dxr = dx + static_cast<size_t>(row) * xs;
    const float* drr = dres ? dres + static_cast<size_t>(row) * H : nullptr;
    for (int col = lane * 8; col < H; col += 256) {
      float v[8], gv8[8], ga8[8], b8[8], dv[8], wv[8], o[8];
      load_value(xr, col, H, act, v, gv8, ga8, b8);
      load8(dyr + col, dv);
      if (w) load8(w + col, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (v[j] - mean) * rstd;
        const float g = dv[j] * (w ? wv[j] : 1.f);
        o[j] = rstd * (g - s1 - xh * s2);
      }
      if (act == ACT_GLU) {
        float da[8], db[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { da[j] = o[j] * b8[j] * ga8[j]; db[j] = o[j] * gv8[j]; }
        store8(dxr + col, da);
        store8(dxr + H + col, db);
      } else {
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
// got nothing from the same treatment (362 -> 360 us): it is bound by instruction issue, and keeps three CTAs per SM.
template <int CH>
__global__ void __launch_bounds__(kGluWarps * 32, (CH <= 8) ? 2 : 1)
glu_norm_fwd_kernel(const bf16* __restrict__ ab, const float* __restrict__ w, bf16* __restrict__ y,
                    float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows, int H, float eps, int rms) {
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
  bf16* yr = y + static_cast<size_t>(row) * H;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = (c * 32 + lane) * 8;
    if (col < H) {
      float wv[8];
      if (w) load8(w + col, wv);
      uint4 ou;
      uint32_t* op = reinterpret_cast<uint32_t*>(&ou);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 p = unpack_bf16(vp[c][j]);
        const float r0 = w ? rstd * wv[2 * j] : rstd, r1 = w ? rstd * wv[2 * j + 1] : rstd;
        op[j] = pack_bf16((p.x - mean) * r0, (p.y - mean) * r1);
      }
      *reinterpret_cast<uint4*>(yr + col) = ou;
    }
  }
}

// backward: two streaming passes over the row with the GELU recomputed in the second one (nothing row-sized in
// registers -> 3 CTAs/SM); weight gradients go to a private per-warp shared-memory row.
// HAVE_Y: the saved forward output y = bf16(xhat * w) is available, so the first pass gets its two row reductions from
// (dy, y) alone -- s1 = mean(dy * w), s2 = mean(dy * w * xhat) = mean(dy * y) -- without reading [a | b] or evaluating the
// GELU, and the weight-gradient accumulation moves into the second pass.
template <bool HAVE_Y>
__global__ void __launch_bounds__(kGluWarps * 32, 3)
glu_norm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ ab, const float* __restrict__ w,
                    const float* __restrict__ mean_in, const float* __restrict__ rstd_in, bf16* __restrict__ dab,
                    float* __restrict__ dw, float* __restrict__ dw_ws, const bf16* __restrict__ yf, int rows, int H,
                    int rms, int pf) {
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
        if (pf && lane < 4) {
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
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 a2 = unpack_bf16(aw[j]);
        float g0, g1, t0, t1;
        gelu_eval(a2.x, g0, t0);
        gelu_eval(a2.y, g1, t1);
        const float2 v2 = unpack_bf16(bf16x2_mul(pack_bf16(g0, g1), bw[j]));
        const float2 d2 = unpack_bf16(dd[j]);
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
      if (pf && HAVE_Y && lane < 4) {
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
        const float2 d2 = unpack_bf16(dd[j]);
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

template <typename TX, typename TY>
int fwd_dispatch(const void* x, const float* w, const float* res, void* y, float* mean, float* rstd, int rows, int H,
                 float eps, int act, int rms, cudaStream_t s) {
  if (H <= 1024 && act != ACT_GLU) {
    const int grid = ceil_div(rows, kWarpsPerBlock);
    const int ch = ceil_div(H, 256);
#define MUSE_NF(CH)                                                                                                \
  pdl_launch(grid, kWarpsPerBlock * 32, 0, s)(norm_fwd_warp_kernel<TX, TY, CH>, reinterpret_cast<const TX*>(x), w, res,    \
                                                                         reinterpret_cast<TY*>(y), mean, rstd, rows, \
                                                                         H, eps, act, rms)
    if (ch <= 1) MUSE_NF(1);
    else if (ch <= 2) MUSE_NF(2);
    else MUSE_NF(4);
#undef MUSE_NF
    return check_launch("norm_fwd");
  }
  pdl_launch(ceil_div(rows, kWideWarps), kWideWarps * 32, 0, s)(norm_fwd_wide_kernel<TX, TY>,
      reinterpret_cast<const TX*>(x), w, res, reinterpret_cast<TY*>(y), mean, rstd, rows, H, eps, act, rms);
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

template <typename TDY, typename TX, typename TDX>
int bwd_dispatch(const void* dy, const void* x, const float* w, const float* mean, const float* rstd,
                 const float* dres, void* dx, void* dx_copy, float* dw, float* dw_ws, int rows, int H, int act, int rms,
                 cudaStream_t s) {
  const int grid = bwd_grid(rows, H, act);
  if (H <= 1024 && act != ACT_GLU) {
    const int ch = ceil_div(H, 256);
    const size_t smem = dw ? static_cast<size_t>(kBwdWarps) * H * sizeof(float) : 0;
#define MUSE_NB(CH)                                                                                          \
  pdl_launch(grid, kBwdWarps * 32, smem, s)(norm_bwd_warp_kernel<TDY, TX, TDX, CH>,                                  \
      reinterpret_cast<const TDY*>(dy), reinterpret_cast<const TX*>(x), w, mean, rstd, dres,                 \
      reinterpret_cast<TDX*>(dx), reinterpret_cast<bf16*>(dx_copy), dw, dw_ws, rows, H, act, rms, kRowPrefetch)
    if (ch <= 1) MUSE_NB(1);
    else if (ch <= 2) MUSE_NB(2);
    else MUSE_NB(4);
#undef MUSE_NB
  } else {
    if (dx_copy) { set_last_error("norm_bwd: the bf16 copy of dx is only produced for H <= 1024 without GLU"); return MUSE_ERR_UNSUPPORTED; }
    const size_t smem = dw ? static_cast<size_t>(kWideWarps) * H * sizeof(float) : 0;
    auto kern = norm_bwd_wide_kernel<TDY, TX, TDX>;
    static bool attr = false;
    if (!attr) {
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kWideWarps * 4096 * 4);
      attr = true;
    }
    pdl_launch(grid, kWideWarps * 32, smem, s)(kern, reinterpret_cast<const TDY*>(dy), reinterpret_cast<const TX*>(x), w, mean, rstd,
                                             dres, reinterpret_cast<TDX*>(dx), dw, dw_ws, rows, H, act, rms);
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

// dtype codes: 0 = fp32, 1 = bf16.  act: 0 none, 1 GELU(x), 2 GLU (x is [rows, 2H]).
int norm_fwd(const void* x, int x_dt, const float* w, const float* res, void* y, int y_dt, float* mean, float* rstd,
             int rows, int H, float eps, int act, int rms, cudaStream_t s) {
  if (rows <= 0) return MUSE_OK;
  int rc = check_args("norm_fwd", H, act, res);
  if (rc) return rc;
  if (act == ACT_GLU && x_dt == 1 && y_dt == 1 && H <= 4096) {
    const int grid = ceil_div(rows, kGluWarps);
    const int ch = ceil_div(H, 256);
#define MUSE_GF(CH) pdl_launch(grid, kGluWarps * 32, 0, s)(glu_norm_fwd_kernel<CH>, reinterpret_cast<const bf16*>(x), w, reinterpret_cast<bf16*>(y), mean, rstd, rows, H, eps, rms)
    if (ch <= 1) MUSE_GF(1); else if (ch <= 2) MUSE_GF(2); else if (ch <= 4) MUSE_GF(4); else if (ch <= 8) MUSE_GF(8); else MUSE_GF(16);
#undef MUSE_GF
    return check_launch("glu_norm_fwd");
  }
  if (x_dt == 0 && y_dt == 1) return fwd_dispatch<float, bf16>(x, w, res, y, mean, rstd, rows, H, eps, act, rms, s);
  if (x_dt == 1 && y_dt == 1) return fwd_dispatch<bf16, bf16>(x, w, res, y, mean, rstd, rows, H, eps, act, rms, s);
  if (x_dt == 1 && y_dt == 0) return fwd_dispatch<bf16, float>(x, w, res, y, mean, rstd, rows, H, eps, act, rms, s);
  if (x_dt == 0 && y_dt == 0) return fwd_dispatch<float, float>(x, w, res, y, mean, rstd, rows, H, eps, act, rms, s);
  set_last_error("norm_fwd: bad dtype codes %d %d", x_dt, y_dt);
  return MUSE_ERR_INVALID;
}

// x2 = res + norm1(a) * w1 ; h2 = norm2(x2) * w2  (a bf16 [rows,H], res / x2 fp32, h2 bf16; H % 8 == 0, H <= 1024)
int norm2_fwd(const void* a, const float* res, const float* w1, const float* w2, float* x2, void* h2, float* mean1,
              float* rstd1, float* mean2, float* rstd2, int rows, int H, float eps, int rms1, int rms2, cudaStream_t s) {
  if (rows <= 0) return MUSE_OK;
  if (H % 8 != 0 || H > 1024 || H < 8) { set_last_error("norm2_fwd: H=%d must be a multiple of 8 in [8, 1024]", H); return MUSE_ERR_UNSUPPORTED; }
  const int grid = ceil_div(rows, kWarpsPerBlock);
  const int ch = ceil_div(H, 256);
#define MUSE_N2F(CH) pdl_launch(grid, kWarpsPerBlock * 32, 0, s)(norm2_fwd_warp_kernel<CH>, reinterpret_cast<const bf16*>(a), res, w1, w2, x2, reinterpret_cast<bf16*>(h2), mean1, rstd1, mean2, rstd2, rows, H, eps, rms1, rms2)
  if (ch <= 1) MUSE_N2F(1); else if (ch <= 2) MUSE_N2F(2); else MUSE_N2F(4);
#undef MUSE_N2F
  return check_launch("norm2_fwd");
}

// ws: 2 * norm_bwd_workspace_floats(rows, H, 0) floats (dw2 partial rows, then dw1 partial rows); dw2 / dw1 are STORED.
int norm2_bwd(const void* d_h2, const float* x2, const float* w2, const float* mean2, const float* rstd2, const float* dres,
              const void* a, const float* w1, const float* mean1, const float* rstd1, float* dx2, void* d_a, float* dw2,
              float* dw1, float* ws, int rows, int H, int rms1, int rms2, cudaStream_t s) {
  if (rows <= 0) return MUSE_OK;
  if (H % 8 != 0 || H > 1024 || H < 8) { set_last_error("norm2_bwd: H=%d must be a multiple of 8 in [8, 1024]", H); return MUSE_ERR_UNSUPPORTED; }
  const int grid = bwd_grid(rows, H, 0);
  const int ch = ceil_div(H, 256);
  float* ws2 = ws;
  float* ws1 = ws + static_cast<size_t>(grid) * H;
  const size_t smem = static_cast<size_t>(2) * kBwdWarps * H * sizeof(float);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(norm2_bwd_warp_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * kBwdWarps * 1024 * 4);
    cudaFuncSetAttribute(norm2_bwd_warp_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * kBwdWarps * 1024 * 4);
    cudaFuncSetAttribute(norm2_bwd_warp_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * kBwdWarps * 1024 * 4);
    attr = true;
  }
#define MUSE_N2B(CH) pdl_launch(grid, kBwdWarps * 32, smem, s)(norm2_bwd_warp_kernel<CH>, reinterpret_cast<const bf16*>(d_h2), x2, w2, mean2, rstd2, dres, reinterpret_cast<const bf16*>(a), w1, mean1, rstd1, dx2, reinterpret_cast<bf16*>(d_a), ws2, ws1, rows, H, rms1, rms2, kRowPrefetch)
  if (ch <= 1) MUSE_N2B(1); else if (ch <= 2) MUSE_N2B(2); else MUSE_N2B(4);
#undef MUSE_N2B
  int rc = check_launch("norm2_bwd");
  if (rc) return rc;
  if ((rc = reduce_dw(ws2, dw2, grid, H, s))) return rc;
  return reduce_dw(ws1, dw1, grid, H, s);
}

// floats of workspace a deterministic (dw_ws != nullptr) backward needs: one partial row of H per CTA
long long norm_bwd_workspace_floats(int rows, int H, int act) {
  if (rows <= 0) return 0;
  return static_cast<long long>(bwd_grid(rows, H, act)) * H;
}

int norm_bwd(const void* dy, int dy_dt, const void* x, int x_dt, const float* w, const float* mean, const float* rstd,
             const float* dres, const void* y_fwd, void* dx, int dx_dt, void* dx_copy, float* dw, float* dw_ws, int rows,
             int H, int act, int rms, cudaStream_t s) {
  if (rows <= 0) return MUSE_OK;
  int rc = check_args("norm_bwd", H, act, dres);
  if (rc) return rc;
  if (dx_copy && (dx_dt != 0 || act == ACT_GLU)) { set_last_error("norm_bwd: dx_copy needs an fp32 dx and no GLU"); return MUSE_ERR_INVALID; }
  if (act == ACT_GLU && dy_dt == 1 && x_dt == 1 && dx_dt == 1 && H <= 4096) {
    const int grid = bwd_grid(rows, H, act);
    const size_t smem = dw ? static_cast<size_t>(kGluWarps) * H * sizeof(float) : 0;
    static bool attr = false;
    if (!attr) {
      cudaFuncSetAttribute(glu_norm_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGluWarps * 4096 * 4);
      cudaFuncSetAttribute(glu_norm_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGluWarps * 4096 * 4);
      attr = true;
    }
    if (y_fwd != nullptr)
      pdl_launch(grid, kGluWarps * 32, smem, s)(glu_norm_bwd_kernel<true>,
          reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(x), w, mean, rstd, reinterpret_cast<bf16*>(dx), dw,
          dw_ws, reinterpret_cast<const bf16*>(y_fwd), rows, H, rms, kRowPrefetch);
    else
      pdl_launch(grid, kGluWarps * 32, smem, s)(glu_norm_bwd_kernel<false>,
          reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(x), w, mean, rstd, reinterpret_cast<bf16*>(dx), dw,
          dw_ws, nullptr, rows, H, rms, 0);
    rc = check_launch("glu_norm_bwd");
    if (rc || !dw || !dw_ws) return rc;
    return reduce_dw(dw_ws, dw, grid, H, s);
  }
  const int key = dy_dt * 4 + x_dt * 2 + dx_dt;
  switch (key) {
    case 0: return bwd_dispatch<float, float, float>(dy, x, w, mean, rstd, dres, dx, dx_copy, dw, dw_ws, rows, H, act, rms, s);
    case 1: return bwd_dispatch<float, float, bf16>(dy, x, w, mean, rstd, dres, dx, dx_copy, dw, dw_ws, rows, H, act, rms, s);
    case 2: return bwd_dispatch<float, bf16, float>(dy, x, w, mean, rstd, dres, dx, dx_copy, dw, dw_ws, rows, H, act, rms, s);
    case 3: return bwd_dispatch<float, bf16, bf16>(dy, x, w, mean, rstd, dres, dx, dx_copy, dw, dw_ws, rows, H, act, rms, s);
    case 4: return bwd_dispatch<bf16, float, float>(dy, x, w, mean, rstd, dres, dx, dx_copy, dw, dw_ws, rows, H, act, rms, s);
    case 5: return bwd_dispatch<bf16, float, bf16>(dy, x, w, mean, rstd, dres, dx, dx_copy, dw, dw_ws, rows, H, act, rms, s);
    case 6: return bwd_dispatch<bf16, bf16, float>(dy, x, w, mean, rstd, dres, dx, dx_copy, dw, dw_ws, rows, H, act, rms, s);
    case 7: return bwd_dispatch<bf16, bf16, bf16>(dy, x, w, mean, rstd, dres, dx, dx_copy, dw, dw_ws, rows, H, act, rms, s);
  }
  set_last_error("norm_bwd: bad dtype codes");
  return MUSE_ERR_INVALID;
}

}  // namespace muse
