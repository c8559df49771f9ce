// Spatial half of the Paella ResBlock (muse/modeling_paella_vq.py:112-145), NHWC fp32, one warp per pixel on the
// row_norm.cuh core:
//
//     x1 = x + dw(LN1(x))          dw = ReplicationPad2d(1) + depthwise 3x3 with bias
//     n2 = LN2(x1)                 written as the operand of the c -> 4c Linear that follows
//
// Both LayerNorms are over channels without affine, eps 1e-6.  The host folds the ResBlock's gammas into the weights:
// (1 + g0), g1 and g2 into the depthwise weight and bias (exact in real arithmetic because replication padding gives every
// output all nine taps, so the constant shift g1 stays a constant), (1 + g3), g4 into the first Linear and g5 into the
// second.  The LN1 statistics of every pixel come from a pre-pass (resblock_stats_kernel), so each warp normalises its nine
// clamped neighbours on the fly and nothing but x is read.
#include "row_norm.cuh"

namespace muse {
namespace {

constexpr int kWarps = 8;

// stats[pix] = {mean, rstd} of LN1 over the C channels of x[pix]
template <int CH>
__global__ void __launch_bounds__(kWarps * 32)
resblock_stats_kernel(const float* __restrict__ x, float2* __restrict__ stats, long long pixels, int C, float eps) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const long long pix = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5);
  if (pix >= pixels) return;
  float v[CH][8];
  const float sum = row_load(v, C, lane, [&](int col, float (&vc)[8]) { load8(x + pix * C + col, vc); });
  float mean, rstd;
  row_stats(v, sum, C, 1.0f / static_cast<float>(C), lane, eps, 0, mean, rstd);
  if (lane == 0) stats[pix] = make_float2(mean, rstd);
}

// x1 = x + bias + sum_t wk[t] * LN1(x[clamp(pix + t)]); n2 = LN2(x1) as fp32 (SPLIT false) or bf16 planes hi (+ lo).
template <int CH, bool SPLIT>
__global__ void __launch_bounds__(kWarps * 32)
resblock_spatial_kernel(const float* __restrict__ x, const float2* __restrict__ stats, const float* __restrict__ wk,
                        const float* __restrict__ bias, float* __restrict__ x1, float* __restrict__ n2,
                        bf16* __restrict__ n2_hi, bf16* __restrict__ n2_lo, int B, int H, int W, int C, float eps) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const long long pix = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5);
  if (pix >= static_cast<long long>(B) * H * W) return;
  const int px = static_cast<int>(pix % W);
  const int py = static_cast<int>((pix / W) % H);
  const long long b = pix / (static_cast<long long>(W) * H);
  long long nb[9];
  float2 st[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) {  // ReplicationPad2d(1): the neighbour index is clamped into the image
    const int iy = min(max(py + t / 3 - 1, 0), H - 1), ix = min(max(px + t % 3 - 1, 0), W - 1);
    nb[t] = (b * H + iy) * W + ix;
    st[t] = stats[nb[t]];
  }
  float v[CH][8];
  const float sum = row_load(v, C, lane, [&](int col, float (&vc)[8]) {
    float bv[8], xv[8];
    load8(bias + col, bv);
#pragma unroll
    for (int j = 0; j < 8; ++j) vc[j] = bv[j];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      float kv[8];
      load8(x + nb[t] * C + col, xv);
      load8(wk + t * C + col, kv);
#pragma unroll
      for (int j = 0; j < 8; ++j) vc[j] = fmaf((xv[j] - st[t].x) * st[t].y, kv[j], vc[j]);
    }
    load8(x + pix * C + col, xv);
#pragma unroll
    for (int j = 0; j < 8; ++j) vc[j] += xv[j];
    store8(x1 + pix * C + col, vc);
  });
  float mean, rstd;
  row_stats(v, sum, C, 1.0f / static_cast<float>(C), lane, eps, 0, mean, rstd);
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = row_col(c, lane);
    if (col < C) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[c][j] - mean) * rstd;
      if (SPLIT) {
        float h[8], l[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          h[j] = bf16_round(o[j]);
          l[j] = o[j] - h[j];
        }
        store8(n2_hi + pix * C + col, h);
        if (n2_lo != nullptr) store8(n2_lo + pix * C + col, l);
      } else {
        store8(n2 + pix * C + col, o);
      }
    }
  }
}

}  // namespace
}  // namespace muse

using namespace muse;

extern "C" {

// x fp32 [B,H,W,C] -> stats_ws float2 [B*H*W] (LN1 mean, rstd), then x1 fp32 [B,H,W,C] and LN2(x1) as n2 fp32 or as
// the bf16 planes n2_hi (+ n2_lo, nullable: single-pass mode); exactly one of n2 / n2_hi is given.
// wk fp32 [9][C] (tap-major, gammas folded in), bias fp32 [C].  C % 8 == 0, C <= 1024.
int muse_paella_resblock_spatial(const float* x, const float* wk, const float* bias, float* stats_ws, float* x1, float* n2,
                                 void* n2_hi, void* n2_lo, int B, int H, int W, int C, float eps, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if ((n2 != nullptr) == (n2_hi != nullptr) || (n2_hi == nullptr && n2_lo != nullptr)) {
    set_last_error("paella_resblock_spatial: give either n2 (fp32) or n2_hi (+ n2_lo)");
    return MUSE_ERR_INVALID;
  }
  if (C % 8 != 0 || C < 8 || C > 1024) {
    set_last_error("paella_resblock_spatial: C=%d must be a multiple of 8 in [8, 1024]", C);
    return MUSE_ERR_UNSUPPORTED;
  }
  const long long pixels = static_cast<long long>(B) * H * W;
  if (pixels <= 0) return MUSE_OK;
  if (pixels > static_cast<long long>(INT_MAX) * kWarps) { set_last_error("paella_resblock_spatial: too many pixels"); return MUSE_ERR_UNSUPPORTED; }
  const unsigned grid = static_cast<unsigned>(ceil_div_ll(pixels, kWarps));
  float2* st = reinterpret_cast<float2*>(stats_ws);
  with_row_chunks<1, 2, 4>(C, [&](auto ch) {
    constexpr int CH = decltype(ch)::value;
    pdl_launch(grid, kWarps * 32, 0, s)(resblock_stats_kernel<CH>, x, st, pixels, C, eps);
  });
  if (int rc = check_launch("paella_resblock_stats")) return rc;
  with_row_chunks<1, 2, 4>(C, [&](auto ch) {
    constexpr int CH = decltype(ch)::value;
    pdl_launch(grid, kWarps * 32, 0, s)(n2_hi ? resblock_spatial_kernel<CH, true> : resblock_spatial_kernel<CH, false>, x, st,
                                        wk, bias, x1, n2, reinterpret_cast<bf16*>(n2_hi), reinterpret_cast<bf16*>(n2_lo), B, H,
                                        W, C, eps);
  });
  return check_launch("paella_resblock_spatial");
}

}  // extern "C"
