// Forward kernels specific to MaskGiTUViT_v2 (muse/modeling_transformer_v2.py); the GEMMs, attention, GLU and
// cross-entropy are the kernels of the v1 path.  All HBM-bound, token-major [rows = B*h*w, C] activations.
//   * add_norm_mod : prenorm-residual norm (unfused_rms_norm / unfused_layer_norm, :673-738): r' = a + r ; y = norm(r') * w,
//                    optionally followed by the adaLN modulation y * (1 + scale_b) + shift_b (AdaLNModulation :1025-1037)
//                    of the TransformerLayer / GLUFeedForward (:757-792, :926-951).  One pass instead of add, norm, modulate.
//   * dwconv3x3_norm: ResBlock head (:604-612): depthwise 3x3 conv (bf16-rounded like the autocast conv output) + Norm2D.
//   * grn           : GELU + GlobalResponseNorm (:741-751): Gx = ||g||_2 over (h, w) per (image, channel),
//                     Nx = Gx / (mean_c Gx + 1e-6), out = gamma * (g * Nx) + beta + g.
//                     With dropout: the ResBlock's nn.Dropout between GRN and channelwise[4] (:603-609) fused into the
//                     apply pass, which draws the keep bits (philox.cuh) and writes the dropped output and the bits.
//   * adaln_apply   : in-place fp32 x * (1 + scale_b) + shift_b at the end of a ResBlock.
//   * silu          : SiLU of the conditioning vectors / text states feeding the adaLN and kv mappers.
#include "philox.cuh"
#include "row_norm.cuh"

namespace muse {
namespace {

constexpr int kWarps = 4;

// a: [rows, H] (TA = bf16 | float), r: fp32 [rows, H] or null, w: fp32 [H] or null,
// ss: fp32, scale of sample b at ss[b * ss_stride + 0 .. H), shift at ss[b * ss_stride + H .. 2H); null -> no modulation
// r_out: fp32 [rows, H] or null ; y: TY [rows, H]
// F8: y is the e4m3 operand of muse_gemm_fp8 (TY = uint8_t) and row_scale [rows] its scales (row_store_e4m3).
template <typename TA, typename TY, int CH, bool F8>
__global__ void __launch_bounds__(kWarps * 32)
add_norm_mod_kernel(const TA* __restrict__ a, const float* __restrict__ r, const float* __restrict__ w,
                    const float* __restrict__ ss, long long ss_stride, int rows_per_sample, float* __restrict__ r_out,
                    TY* __restrict__ y, int rows, int H, float eps, int rms, float* __restrict__ row_scale) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const size_t base = static_cast<size_t>(row) * H;
  float v[CH][8];
  const float sum = row_load(v, H, lane, [&](int col, float (&vc)[8]) {
    load8(a + base + col, vc);
    if (r != nullptr) {
      float rv[8];
      load8(r + base + col, rv);
#pragma unroll
      for (int j = 0; j < 8; ++j) vc[j] += rv[j];
    }
    if (r_out != nullptr) store8(r_out + base + col, vc);
  });
  float mean, rstd;
  row_stats(v, sum, H, 1.0f / static_cast<float>(H), lane, eps, rms, mean, rstd);
  const float* sc = ss ? ss + static_cast<size_t>(row / rows_per_sample) * ss_stride : nullptr;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = row_col(c, lane);
    if (col < H) {
      float o[8], wv[8];
      if (w) load8(w + col, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j] = (v[c][j] - mean) * rstd;
        if (w) o[j] *= wv[j];
      }
      if (sc) {
        float s8[8], h8[8];
        load8(sc + col, s8);
        load8(sc + H + col, h8);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(o[j], 1.f + s8[j], h8[j]);
      }
      if constexpr (F8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[c][j] = o[j];
      } else {
        store8(y + base + col, o);
      }
    }
  }
  if constexpr (F8) row_store_e4m3(v, H, lane, y + base, row_scale + row);
}

// x fp32 [B, hh, ww, C]; wk fp32 [9][C] (tap-major); nw fp32 [C] or null; y bf16 [B, hh, ww, C].  One warp per pixel.
// F8: y is e4m3 (TY = uint8_t) with one scale per pixel in row_scale (row_store_e4m3).
template <int CH, bool F8, typename TY = bf16>
__global__ void __launch_bounds__(kWarps * 32)
dwconv3x3_norm_kernel(const float* __restrict__ x, const float* __restrict__ wk, const float* __restrict__ nw,
                      TY* __restrict__ y, bf16* __restrict__ conv_out, int B, int hh, int ww, int C, float eps, int rms,
                      float* __restrict__ row_scale) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const long long pix = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5);
  if (pix >= static_cast<long long>(B) * hh * ww) return;
  const int px = static_cast<int>(pix % ww);
  const int py = static_cast<int>((pix / ww) % hh);
  const long long b = pix / (static_cast<long long>(ww) * hh);
  float v[CH][8];
  const float sum = row_load(v, C, lane, [&](int col, float (&vc)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) vc[j] = 0.f;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int iy = py + t / 3 - 1, ix = px + t % 3 - 1;
      if (iy >= 0 && iy < hh && ix >= 0 && ix < ww) {
        float xv[8], kv[8];
        load8(x + ((b * hh + iy) * ww + ix) * C + col, xv);
        load8(wk + t * C + col, kv);
#pragma unroll
        for (int j = 0; j < 8; ++j) vc[j] = fmaf(xv[j], kv[j], vc[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) vc[j] = bf16_round(vc[j]);  // the conv output is a bf16 tensor under autocast
    if (conv_out != nullptr) store8(conv_out + pix * C + col, vc);  // saved for the backward pass
  });
  float mean, rstd;
  row_stats(v, sum, C, 1.0f / static_cast<float>(C), lane, eps, rms, mean, rstd);
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = row_col(c, lane);
    if (col < C) {
      float o[8], wv[8];
      if (nw) load8(nw + col, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[c][j] - mean) * rstd * (nw ? wv[j] : 1.f);
      if constexpr (F8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[c][j] = o[j];
      } else {
        store8(y + pix * C + col, o);
      }
    }
  }
  if constexpr (F8) row_store_e4m3(v, C, lane, y + pix * C, row_scale + pix);
}

// GRN pass 1: sumsq[b, c] = sum over the image's tokens of bf16(gelu(x))^2.  grid (C/256, B), 128 threads x 2 channels.
__global__ void __launch_bounds__(128)
grn_stats_kernel(const bf16* __restrict__ x, float* __restrict__ sumsq, int HW, int C) {
  pdl_enter();
  const int c = (blockIdx.x * 128 + threadIdx.x) * 2;
  if (c >= C) return;
  const int b = blockIdx.y;
  const bf16* p = x + static_cast<size_t>(b) * HW * C + c;
  float s0 = 0.f, s1 = 0.f;
  for (int t = 0; t < HW; ++t) {
    const float2 v = unpack_bf16(*reinterpret_cast<const uint32_t*>(p + static_cast<size_t>(t) * C));
    const float g0 = bf16_round(gelu_f(v.x)), g1 = bf16_round(gelu_f(v.y));
    s0 = fmaf(g0, g0, s0);
    s1 = fmaf(g1, g1, s1);
  }
  sumsq[static_cast<size_t>(b) * C + c] = s0;
  sumsq[static_cast<size_t>(b) * C + c + 1] = s1;
}

// GRN pass 2 (one CTA per image): nx[c] = sqrt(sumsq[c]) / (mean_c sqrt(sumsq) + 1e-6)
__global__ void __launch_bounds__(256)
grn_finalize_kernel(const float* __restrict__ stat, float* __restrict__ nx_out, int C) {
  pdl_enter();
  __shared__ float s_part[8];
  const float* p = stat + static_cast<size_t>(blockIdx.x) * C;
  float* o = nx_out + static_cast<size_t>(blockIdx.x) * C;
  float acc = 0.f;
  for (int c = threadIdx.x; c < C; c += 256) acc += sqrtf(p[c]);
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += s_part[i];
  const float denom = tot / static_cast<float>(C) + 1e-6f;
  for (int c = threadIdx.x; c < C; c += 256) o[c] = sqrtf(p[c]) / denom;
}

// GRN pass 3: out = gamma * (g * nx) + beta + g, g = bf16(gelu(x)); 8 channels per thread
// DROP: the thread's 8 channels of one token row are one Philox call of the elementwise mapping (row = token of the
// B*HW rows, columns = the C channels): the fp32 output is scaled by keep / (1 - p_eff) and rounded once, and the keep
// byte is stored (the last chunk of a row also zeroes the pad bytes of the row's last word).
template <bool DROP>
__global__ void __launch_bounds__(256)
grn_apply_kernel(const bf16* __restrict__ x, const float* __restrict__ nx, const float* __restrict__ gamma,
                 const float* __restrict__ beta, bf16* __restrict__ out, long long total8, int HW, int C,
                 const philox::ElemDrop drop) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= total8) return;
  const int c8 = C / 8;
  const int col = static_cast<int>(i % c8) * 8;
  const long long b = i / (static_cast<long long>(c8) * HW);
  float v[8], n8[8], g8[8], b8[8], o[8];
  load8(x + i * 8, v);
  load8(nx + b * C + col, n8);
  load8(gamma + col, g8);
  load8(beta + col, b8);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float g = bf16_round(gelu_f(v[j]));
    o[j] = fmaf(g8[j], g * n8[j], b8[j]) + g;
  }
  if constexpr (DROP) {
    const long long row = i / c8;
    const int k = col / 8;
    const uint32_t kb = philox::elem_keep8(*drop.seed, drop.site, static_cast<uint32_t>(row), k, drop.thresh);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] *= philox::keep_z(kb, j, drop.scale);
    uint8_t* br = drop.bits + row * drop.row_bytes;
    br[k] = static_cast<uint8_t>(kb);
    if (k == c8 - 1)
      for (int q = c8; q < drop.row_bytes; ++q) br[q] = 0;
  }
  store8(out + i * 8, o);
}

__global__ void __launch_bounds__(256)
adaln_apply_kernel(float* __restrict__ x, const float* __restrict__ ss, long long ss_stride, long long total4,
                   int rows_per_sample, int C) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= total4) return;
  const int c4 = C / 4;
  const int col = static_cast<int>(i % c4) * 4;
  const long long b = i / (static_cast<long long>(c4) * rows_per_sample);
  const float* sc = ss + b * ss_stride;
  float4 v = *reinterpret_cast<float4*>(x + i * 4);
  const float4 s = *reinterpret_cast<const float4*>(sc + col);
  const float4 h = *reinterpret_cast<const float4*>(sc + C + col);
  v.x = fmaf(v.x, 1.f + s.x, h.x); v.y = fmaf(v.y, 1.f + s.y, h.y);
  v.z = fmaf(v.z, 1.f + s.z, h.z); v.w = fmaf(v.w, 1.f + s.w, h.w);
  *reinterpret_cast<float4*>(x + i * 4) = v;
}

template <typename TX>
__global__ void __launch_bounds__(256) silu_kernel(const TX* __restrict__ x, bf16* __restrict__ y, long long n8) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n8) return;
  float v[8];
  load8(x + i * 8, v);
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = v[j] / (1.f + expf(-v[j]));
  store8(y + i * 8, v);
}

}  // namespace
}  // namespace muse

using namespace muse;

extern "C" {

int muse_add_norm_mod_fwd(const void* a, int a_dt, const float* r, const float* w, const float* ss, long long ss_stride,
                          int rows_per_sample, float* r_out, void* y, int y_dt, float* row_scale, int rows, int H,
                          float eps, int rms, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0) return MUSE_OK;
  if (H % 8 != 0 || H > 1024) { set_last_error("add_norm_mod: H=%d must be a multiple of 8 and <= 1024", H); return MUSE_ERR_UNSUPPORTED; }
  if (ss != nullptr && (rows_per_sample <= 0 || ss_stride % 4 != 0)) { set_last_error("add_norm_mod: bad modulation layout"); return MUSE_ERR_INVALID; }
  if (ss == nullptr) rows_per_sample = 1;
  auto run = [&](auto a_t, auto y_t, auto f8) {
    using TA = decltype(a_t);
    using TY = decltype(y_t);
    with_row_chunks<1, 2, 3, 4>(H, [&](auto ch) {
      pdl_launch(ceil_div(rows, kWarps), kWarps * 32, 0, s)(
          add_norm_mod_kernel<TA, TY, decltype(ch)::value, decltype(f8)::value>, reinterpret_cast<const TA*>(a), r, w, ss,
          ss_stride, rows_per_sample, r_out, reinterpret_cast<TY*>(y), rows, H, eps, rms, row_scale);
    });
    return check_launch("add_norm_mod");
  };
  if (y_dt == 2) {
    if (row_scale == nullptr) { set_last_error("add_norm_mod: the e4m3 output needs row_scale"); return MUSE_ERR_INVALID; }
    return dtype_dispatch("add_norm_mod", [&](auto a_t) { return run(a_t, uint8_t(), std::true_type()); }, a_dt);
  }
  return dtype_dispatch("add_norm_mod", [&](auto a_t, auto y_t) { return run(a_t, y_t, std::false_type()); }, a_dt, y_dt);
}

int muse_dwconv3x3_norm_fwd(const float* x, const float* wk, const float* nw, void* y, int y_dt, float* row_scale,
                            void* conv_out, int B, int hh, int ww, int C, float eps, int rms, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long pixels = static_cast<long long>(B) * hh * ww;
  if (y_dt != 1 && y_dt != 2) { set_last_error("dwconv3x3_norm: y dtype code %d (bf16 = 1 or e4m3 = 2)", y_dt); return MUSE_ERR_INVALID; }
  if (y_dt == 2 && row_scale == nullptr) { set_last_error("dwconv3x3_norm: the e4m3 output needs row_scale"); return MUSE_ERR_INVALID; }
  if (pixels <= 0) return MUSE_OK;
  if (C % 8 != 0 || C > 1024) { set_last_error("dwconv3x3_norm: C=%d must be a multiple of 8 and <= 1024", C); return MUSE_ERR_UNSUPPORTED; }
  const unsigned grid = static_cast<unsigned>(ceil_div_ll(pixels, kWarps));
  with_row_chunks<1, 2, 3, 4>(C, [&](auto ch) {
    constexpr int CH = decltype(ch)::value;
    if (y_dt == 2)
      pdl_launch(grid, kWarps * 32, 0, s)(dwconv3x3_norm_kernel<CH, true, uint8_t>, x, wk, nw, reinterpret_cast<uint8_t*>(y),
                                          reinterpret_cast<bf16*>(conv_out), B, hh, ww, C, eps, rms, row_scale);
    else
      pdl_launch(grid, kWarps * 32, 0, s)(dwconv3x3_norm_kernel<CH, false>, x, wk, nw, reinterpret_cast<bf16*>(y),
                                          reinterpret_cast<bf16*>(conv_out), B, hh, ww, C, eps, rms, row_scale);
  });
  return check_launch("dwconv3x3_norm");
}

// x bf16 [B, HW, C] -> out bf16 [B, HW, C]; sumsq_ws / nx_ws fp32 [B, C] (kept by the caller for the backward pass).
// bits != nullptr: the ResBlock's dropout (:607) fused into the apply pass, out is the dropped output and bits
// [B * HW, ceil(C / 32)] uint32 words are written (philox.cuh elementwise mapping, seed read from *seed).
int muse_grn_fwd(const void* x, const float* gamma, const float* beta, void* out, float* stat_ws, float* nx_ws,
                 unsigned int* bits, const unsigned long long* seed, int site, float p, int B, int HW, int C,
                 void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (bits != nullptr && seed == nullptr) { set_last_error("grn_fwd: dropout needs a seed"); return MUSE_ERR_INVALID; }
  if (B <= 0 || HW <= 0) return MUSE_OK;
  if (C % 8 != 0) { set_last_error("grn: C must be a multiple of 8"); return MUSE_ERR_UNSUPPORTED; }
  const bf16* xp = reinterpret_cast<const bf16*>(x);
  pdl_launch(dim3(ceil_div(C, 256), B), 128, 0, s)(grn_stats_kernel, xp, stat_ws, HW, C);
  int rc = check_launch("grn_stats");
  if (rc) return rc;
  pdl_launch(B, 256, 0, s)(grn_finalize_kernel, stat_ws, nx_ws, C);
  rc = check_launch("grn_finalize");
  if (rc) return rc;
  const long long total8 = static_cast<long long>(B) * HW * (C / 8);
  pdl_launch(static_cast<unsigned>(ceil_div_ll(total8, 256)), 256, 0, s)(bits ? grn_apply_kernel<true> : grn_apply_kernel<false>,
      xp, nx_ws, gamma, beta, reinterpret_cast<bf16*>(out), total8, HW, C, philox::elem_drop(bits, seed, site, p, C));
  return check_launch(bits ? "grn_apply_dropout" : "grn_apply");
}

int muse_adaln_apply(float* x, const float* ss, long long ss_stride, int B, int rows_per_sample, int C, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (C % 4 != 0 || ss_stride % 4 != 0) { set_last_error("adaln_apply: C and the modulation stride must be multiples of 4"); return MUSE_ERR_UNSUPPORTED; }
  const long long total4 = static_cast<long long>(B) * rows_per_sample * (C / 4);
  if (total4 <= 0) return MUSE_OK;
  pdl_launch(static_cast<unsigned>(ceil_div_ll(total4, 256)), 256, 0, s)(adaln_apply_kernel, x, ss, ss_stride, total4, rows_per_sample, C);
  return check_launch("adaln_apply");
}

int muse_silu_bf16(const void* x, int x_dt, void* y, long long n, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0) return MUSE_OK;
  if (n % 8 != 0) { set_last_error("silu: n must be a multiple of 8"); return MUSE_ERR_INVALID; }
  const long long n8 = n / 8;
  const unsigned grid = static_cast<unsigned>(ceil_div_ll(n8, 256));
  if (x_dt == 0) pdl_launch(grid, 256, 0, s)(silu_kernel<float>, reinterpret_cast<const float*>(x), reinterpret_cast<bf16*>(y), n8);
  else pdl_launch(grid, 256, 0, s)(silu_kernel<bf16>, reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(y), n8);
  return check_launch("silu");
}

}  // extern "C"
