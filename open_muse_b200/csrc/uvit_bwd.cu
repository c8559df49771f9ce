// Backward kernels of the MaskGiTUViT_v2-specific ops of uvit.cu (the GEMM dgrad/wgrad, attention, GLU, cross-entropy and
// embedding backward are shared with the v1 path).  All HBM-bound; parameter / per-sample reductions are folded in
// registers and shared memory before touching global atomics.
#include <limits.h>

#include "philox.cuh"
#include "row_norm.cuh"

namespace muse {
namespace {

constexpr int kWarps = 4;
constexpr int kRowsPerWarp = 8;

// Backward of add_norm_mod (uvit.cu):  x = a + r (saved as r_out),  n = norm(x) * w,  y = n * (1 + s_b) + t_b.
//   g  = norm_bwd(dy * (1 + s_b)) + dr_out         -> da (TA) and dr (fp32, optional): both equal g
//   dw += sum_rows dy (1 + s) xhat ;  ds_b += sum_{rows of b} dy * n ;  dt_b += sum_{rows of b} dy
// One warp walks kRowsPerWarp consecutive rows, keeps the three reductions in registers and flushes the per-sample ones
// whenever the sample index changes (rows of one sample are contiguous).  MOD = false: no modulation (ss, dss unused),
// no per-sample reductions.  Also step 1 of the depthwise conv + Norm2D backward (x = the saved bf16 conv output).
template <typename TDY, typename TX, typename TA, bool MOD, int CH>
__global__ void __launch_bounds__(kWarps * 32)
add_norm_mod_bwd_kernel(const TDY* __restrict__ dy, const float* __restrict__ dr_out, const TX* __restrict__ x,
                        const float* __restrict__ w, const float* __restrict__ ss, long long ss_stride, int rows_per_sample,
                        TA* __restrict__ da, float* __restrict__ dr, float* __restrict__ dw, float* __restrict__ dss,
                        int rows, int H, float eps, int rms) {
  pdl_enter();
  extern __shared__ float s_dw[];  // [H]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (dw) {
    for (int i = threadIdx.x; i < H; i += blockDim.x) s_dw[i] = 0.f;
    __syncthreads();
  }
  float dw_acc[CH][8], ds_acc[CH][8], dt_acc[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) dw_acc[c][j] = ds_acc[c][j] = dt_acc[c][j] = 0.f;
  const float inv_h = 1.0f / static_cast<float>(H);
  const int row0 = (blockIdx.x * kWarps + warp) * kRowsPerWarp;
  int cur_b = -1;
  auto flush = [&](int b) {
    if (!MOD || dss == nullptr || b < 0) return;
    float* d = dss + static_cast<size_t>(b) * ss_stride;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          atomicAdd(d + col + j, ds_acc[c][j]);
          atomicAdd(d + H + col + j, dt_acc[c][j]);
          ds_acc[c][j] = dt_acc[c][j] = 0.f;
        }
      }
    }
  };
  for (int k = 0; k < kRowsPerWarp; ++k) {
    const int row = row0 + k;
    if (row >= rows) break;
    const int b = (MOD && ss) ? row / rows_per_sample : 0;
    if (b != cur_b) { flush(cur_b); cur_b = b; }
    const float* sc = (MOD && ss) ? ss + static_cast<size_t>(b) * ss_stride : nullptr;
    const size_t base = static_cast<size_t>(row) * H;
    float xv[CH][8], gv[CH][8];
    const float sum = row_load(xv, H, lane, [&](int col, float (&vc)[8]) { load8(x + base + col, vc); });
    float mean, rstd;
    row_stats(xv, sum, H, inv_h, lane, eps, rms, mean, rstd);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float dv[8], wv[8], s8[8];
        load8(dy + base + col, dv);
        if (w) load8(w + col, wv);
        if (sc) load8(sc + col, s8);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = (xv[c][j] - mean) * rstd;
          const float wj = w ? wv[j] : 1.f;
          const float dn = sc ? dv[j] * (1.f + s8[j]) : dv[j];  // grad wrt n = xhat * w
          if (MOD) {
            ds_acc[c][j] = fmaf(dv[j], xh * wj, ds_acc[c][j]);
            dt_acc[c][j] += dv[j];
          }
          dw_acc[c][j] = fmaf(dn, xh, dw_acc[c][j]);
          gv[c][j] = dn * wj;  // grad wrt xhat
          xv[c][j] = xh;
          row_bwd_acc(gv[c][j], xh, s1, s2);
        }
      }
    }
    row_bwd_sums(inv_h, rms, s1, s2);
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = row_dx(gv[c][j], xv[c][j], s1, s2, rstd);
        if (dr_out) {
          float r8[8];
          load8(dr_out + base + col, r8);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += r8[j];
        }
        store8(da + base + col, o);
        if (dr) store8(dr + base + col, o);
      }
    }
  }
  flush(cur_b);
  if (dw) {
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = row_col(c, lane);
      if (col < H) {
#pragma unroll
        for (int j = 0; j < 8; ++j) atomicAdd(&s_dw[col + j], dw_acc[c][j]);
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < H; i += blockDim.x) atomicAdd(&dw[i], s_dw[i]);
  }
}

// ---- depthwise conv + Norm2D backward -----------------------------------------------------------------------------
// step 1 (add_norm_mod_bwd_kernel, warp per pixel): norm backward on the saved conv output c (bf16): d_c fp32,
// dnw += sum dy * xhat
// step 2: dx[p] = dres[p] + sum_t wk[t] * d_c[p - off(t)]   and   dwk[t] += sum_p d_c[p] * x[p + off(t)]
// thread = (pixel strip, 4 channels); each thread walks kStrip pixels of one image row keeping dwk[9][4] in registers.
constexpr int kStrip = 16;
__global__ void __launch_bounds__(256)
dwconv_bwd_kernel(const float* __restrict__ dc, const float* __restrict__ x, const float* __restrict__ wk,
                  const float* __restrict__ dres, float* __restrict__ dx, float* __restrict__ dwk, int B, int hh, int ww,
                  int C) {
  pdl_enter();
  const int c4 = C / 4;
  const long long strips_per_row = (ww + kStrip - 1) / kStrip;
  const long long total = static_cast<long long>(B) * hh * strips_per_row * c4;
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= total) return;
  const int q = static_cast<int>(i % c4);
  const long long sidx = i / c4;
  const int xs = static_cast<int>(sidx % strips_per_row) * kStrip;
  const int py = static_cast<int>((sidx / strips_per_row) % hh);
  const long long b = sidx / (strips_per_row * hh);
  const int col = q * 4;
  float4 wt[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wt[t] = *reinterpret_cast<const float4*>(wk + t * C + col);
  float4 acc[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int px = xs; px < min(ww, xs + kStrip); ++px) {
    const long long p = (b * hh + py) * ww + px;
    const float4 g = *reinterpret_cast<const float4*>(dc + p * C + col);
    float4 o = dres ? *reinterpret_cast<const float4*>(dres + p * C + col) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int dyo = t / 3 - 1, dxo = t % 3 - 1;
      const int fy = py + dyo, fx = px + dxo;  // forward tap position (for dwk): x[p + off]
      if (fy >= 0 && fy < hh && fx >= 0 && fx < ww) {
        const float4 xv = *reinterpret_cast<const float4*>(x + ((b * hh + fy) * ww + fx) * C + col);
        acc[t].x = fmaf(g.x, xv.x, acc[t].x); acc[t].y = fmaf(g.y, xv.y, acc[t].y);
        acc[t].z = fmaf(g.z, xv.z, acc[t].z); acc[t].w = fmaf(g.w, xv.w, acc[t].w);
      }
      const int by = py - dyo, bx = px - dxo;  // pixel whose forward tap t read this pixel: d_c[p - off]
      if (by >= 0 && by < hh && bx >= 0 && bx < ww) {
        const float4 gv = *reinterpret_cast<const float4*>(dc + ((b * hh + by) * ww + bx) * C + col);
        o.x = fmaf(wt[t].x, gv.x, o.x); o.y = fmaf(wt[t].y, gv.y, o.y);
        o.z = fmaf(wt[t].z, gv.z, o.z); o.w = fmaf(wt[t].w, gv.w, o.w);
      }
    }
    *reinterpret_cast<float4*>(dx + p * C + col) = o;
  }
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    float* d = dwk + t * C + col;
    atomicAdd(d + 0, acc[t].x); atomicAdd(d + 1, acc[t].y); atomicAdd(d + 2, acc[t].z); atomicAdd(d + 3, acc[t].w);
  }
}

// ---- GELU + GRN backward --------------------------------------------------------------------------------------------
// DROP (both passes that read dout): dout is the gradient of the dropped output (the ResBlock's dropout after GRN) and
// is scaled by the stored keep bits as it is read -- 2 bits of one byte per token here, one byte of 8 in pass C.
// pass A: per (image, channel) S1 = sum_hw dout * g ; dbeta += sum dout ; dgamma += nx * S1
template <bool DROP>
__global__ void __launch_bounds__(128)
grn_bwd_stats_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dout, const float* __restrict__ nx,
                     float* __restrict__ s1_out, float* __restrict__ dgamma, float* __restrict__ dbeta, int HW, int C,
                     const philox::ElemDrop drop) {
  pdl_enter();
  const int c = (blockIdx.x * 128 + threadIdx.x) * 2;
  if (c >= C) return;
  const int b = blockIdx.y;
  const size_t off = static_cast<size_t>(b) * HW * C + c;
  float a0 = 0.f, a1 = 0.f, d0 = 0.f, d1 = 0.f;
  for (int t = 0; t < HW; ++t) {
    const float2 v = unpack_bf16(*reinterpret_cast<const uint32_t*>(x + off + static_cast<size_t>(t) * C));
    float2 d = unpack_bf16(*reinterpret_cast<const uint32_t*>(dout + off + static_cast<size_t>(t) * C));
    if constexpr (DROP) {
      const uint32_t kb = drop.bits[(static_cast<size_t>(b) * HW + t) * drop.row_bytes + c / 8];
      d.x *= philox::keep_z(kb, c % 8, drop.scale);
      d.y *= philox::keep_z(kb, c % 8 + 1, drop.scale);
    }
    a0 = fmaf(d.x, bf16_round(gelu_f(v.x)), a0);
    a1 = fmaf(d.y, bf16_round(gelu_f(v.y)), a1);
    d0 += d.x;
    d1 += d.y;
  }
  s1_out[static_cast<size_t>(b) * C + c] = a0;
  s1_out[static_cast<size_t>(b) * C + c + 1] = a1;
  atomicAdd(dgamma + c, nx[static_cast<size_t>(b) * C + c] * a0);
  atomicAdd(dgamma + c + 1, nx[static_cast<size_t>(b) * C + c + 1] * a1);
  atomicAdd(dbeta + c, d0);
  atomicAdd(dbeta + c + 1, d1);
}

// pass B (one CTA per image): coef[c] = dGx[c] / Gx[c] with dGx = dnx / M - (sum_j dnx_j Gx_j) / (M^2 C), dnx = gamma * S1,
// Gx = sqrt(sumsq), M = mean_c Gx + 1e-6.  coef overwrites s1.
__global__ void __launch_bounds__(256)
grn_bwd_finalize_kernel(float* __restrict__ s1, const float* __restrict__ sumsq, const float* __restrict__ gamma, int C) {
  pdl_enter();
  __shared__ float s_a[8], s_b[8];
  float* s = s1 + static_cast<size_t>(blockIdx.x) * C;
  const float* q = sumsq + static_cast<size_t>(blockIdx.x) * C;
  float g_sum = 0.f, dot = 0.f;
  for (int c = threadIdx.x; c < C; c += 256) {
    const float gx = sqrtf(q[c]);
    g_sum += gx;
    dot = fmaf(gamma[c] * s[c], gx, dot);
  }
  g_sum = warp_sum(g_sum);
  dot = warp_sum(dot);
  if ((threadIdx.x & 31) == 0) { s_a[threadIdx.x >> 5] = g_sum; s_b[threadIdx.x >> 5] = dot; }
  __syncthreads();
  float ta = 0.f, tb = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { ta += s_a[i]; tb += s_b[i]; }
  const float M = ta / static_cast<float>(C) + 1e-6f;
  const float common = tb / (M * M * static_cast<float>(C));
  for (int c = threadIdx.x; c < C; c += 256) {
    const float gx = sqrtf(q[c]);
    const float dgx = gamma[c] * s[c] / M - common;
    s[c] = gx > 0.f ? dgx / gx : 0.f;
  }
}

// pass C: dg = dout * (gamma * nx + 1) + coef * g ; dx = dg * gelu'(x)
template <bool DROP>
__global__ void __launch_bounds__(256)
grn_bwd_apply_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dout, const float* __restrict__ nx,
                     const float* __restrict__ coef, const float* __restrict__ gamma, bf16* __restrict__ dx,
                     long long total8, int HW, int C, const philox::ElemDrop drop) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= total8) return;
  const int c8 = C / 8;
  const int col = static_cast<int>(i % c8) * 8;
  const long long b = i / (static_cast<long long>(c8) * HW);
  float v[8], d[8], n8[8], k8[8], g8[8], o[8];
  load8(x + i * 8, v);
  load8(dout + i * 8, d);
  if constexpr (DROP) {
    const uint32_t kb = drop.bits[(i / c8) * drop.row_bytes + col / 8];
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] *= philox::keep_z(kb, j, drop.scale);
  }
  load8(nx + b * C + col, n8);
  load8(coef + b * C + col, k8);
  load8(gamma + col, g8);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float gv, gg;
    gelu_eval(v[j], gv, gg);
    const float g = bf16_round(gv);
    o[j] = (d[j] * fmaf(g8[j], n8[j], 1.f) + k8[j] * g) * gg;
  }
  store8(dx + i * 8, o);
}

// y = x (1 + s_b) + t_b : dx = dy (1 + s_b) ; ds_b = sum_tokens dy * x ; dt_b = sum_tokens dy (one thread owns (b, channel))
__global__ void __launch_bounds__(128)
adaln_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ ss, long long ss_stride,
                 float* __restrict__ dx, float* __restrict__ dss, int rows_per_sample, int C) {
  pdl_enter();
  const int c = blockIdx.x * 128 + threadIdx.x;
  if (c >= C) return;
  const int b = blockIdx.y;
  const float s = 1.f + ss[static_cast<size_t>(b) * ss_stride + c];
  const size_t off = static_cast<size_t>(b) * rows_per_sample * C + c;
  float ds = 0.f, dt = 0.f;
  for (int t = 0; t < rows_per_sample; ++t) {
    const float g = dy[off + static_cast<size_t>(t) * C];
    ds = fmaf(g, x[off + static_cast<size_t>(t) * C], ds);
    dt += g;
    dx[off + static_cast<size_t>(t) * C] = g * s;
  }
  float* d = dss + static_cast<size_t>(b) * ss_stride;
  d[c] += ds;       // this (b, c) slot belongs to exactly one op and one thread
  d[C + c] += dt;
}

// dx (+)= dy * sigmoid(x) * (1 + x (1 - sigmoid(x)))
template <typename TX, typename TDX>
__global__ void __launch_bounds__(256)
silu_bwd_kernel(const bf16* __restrict__ dy, const TX* __restrict__ x, TDX* __restrict__ dx, long long n8, int accumulate) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n8) return;
  float d[8], v[8], o[8];
  load8(dy + i * 8, d);
  load8(x + i * 8, v);
  if (accumulate) load8(dx + i * 8, o);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float sg = 1.f / (1.f + expf(-v[j]));
    const float g = d[j] * sg * (1.f + v[j] * (1.f - sg));
    o[j] = accumulate ? o[j] + g : g;
  }
  store8(dx + i * 8, o);
}

// ss == nullptr selects the kernel without modulation
template <typename TDY, typename TX, typename TA>
int launch_anm_bwd(const void* dy, const float* dr_out, const void* x, const float* w, const float* ss, long long ss_stride,
                   int rows_per_sample, void* da, float* dr, float* dw, float* dss, int rows, int H, float eps, int rms,
                   cudaStream_t s) {
  const size_t smem = dw ? static_cast<size_t>(H) * sizeof(float) : 0;
  with_row_chunks<1, 2, 3, 4>(H, [&](auto ch) {
    constexpr int CH = decltype(ch)::value;
    pdl_launch(ceil_div(rows, kWarps * kRowsPerWarp), kWarps * 32, smem, s)(
        ss ? add_norm_mod_bwd_kernel<TDY, TX, TA, true, CH> : add_norm_mod_bwd_kernel<TDY, TX, TA, false, CH>,
        reinterpret_cast<const TDY*>(dy), dr_out, reinterpret_cast<const TX*>(x), w, ss, ss_stride, rows_per_sample,
        reinterpret_cast<TA*>(da), dr, dw, dss, rows, H, eps, rms);
  });
  return check_launch("add_norm_mod_bwd");
}

}  // namespace
}  // namespace muse

using namespace muse;

extern "C" {

// dy: grad wrt y (dtype code), dr_out: grad wrt the prenorm residual output (fp32, nullable), x: saved r_out;
// outputs da (dtype code) and dr (fp32, nullable) both = g; dw [H] and dss [B, ss_stride] accumulate (+=).
int muse_add_norm_mod_bwd(const void* dy, int dy_dt, const float* dr_out, const float* x, const float* w, const float* ss,
                          long long ss_stride, int rows_per_sample, void* da, int da_dt, float* dr, float* dw, float* dss,
                          int rows, int H, float eps, int rms, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0) return MUSE_OK;
  if (H % 8 != 0 || H > 1024) { set_last_error("add_norm_mod_bwd: H=%d must be a multiple of 8 and <= 1024", H); return MUSE_ERR_UNSUPPORTED; }
  return dtype_dispatch("add_norm_mod_bwd", [&](auto dy_t, auto da_t) {
    return launch_anm_bwd<decltype(dy_t), float, decltype(da_t)>(dy, dr_out, x, w, ss, ss_stride, rows_per_sample, da, dr,
                                                                  dw, dss, rows, H, eps, rms, s);
  }, dy_dt, da_dt);
}

// dy bf16 (grad wrt the normalised output), conv bf16 (saved conv output), x fp32 (block input), wk fp32 [9,C];
// dc_ws fp32 [pixels, C] scratch; dx fp32 = dres + conv-transpose(d_c); dwk [9,C] and dnw [C] accumulate.
int muse_dwconv3x3_norm_bwd(const void* dy, const void* conv, const float* x, const float* wk, const float* nw, const float* dres,
                            float* dc_ws, float* dx, float* dwk, float* dnw, int B, int hh, int ww, int C, float eps, int rms,
                            void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long pixels = static_cast<long long>(B) * hh * ww;
  if (pixels <= 0) return MUSE_OK;
  if (C % 8 != 0 || C > 1024) { set_last_error("dwconv3x3_norm_bwd: C=%d unsupported", C); return MUSE_ERR_UNSUPPORTED; }
  if (pixels > INT_MAX) { set_last_error("dwconv3x3_norm_bwd: %lld pixels, at most INT_MAX supported", pixels); return MUSE_ERR_UNSUPPORTED; }
  int rc = launch_anm_bwd<bf16, bf16, float>(dy, nullptr, conv, nw, nullptr, 0, 1, dc_ws, nullptr, dnw, nullptr,
                                             static_cast<int>(pixels), C, eps, rms, s);
  if (rc) return rc;
  const long long strips = static_cast<long long>(B) * hh * ((ww + kStrip - 1) / kStrip) * (C / 4);
  pdl_launch(static_cast<unsigned>(ceil_div_ll(strips, 256)), 256, 0, s)(dwconv_bwd_kernel, dc_ws, x, wk, dres, dx, dwk, B, hh, ww, C);
  return check_launch("dwconv_bwd");
}

// x bf16 (GEMM output before GELU), dout bf16, nx / sumsq fp32 [B,C] saved by the forward; s1_ws fp32 [B,C] scratch;
// dx bf16; dgamma / dbeta [C] accumulate.  bits != nullptr: those muse_grn_fwd wrote; dout (the gradient of the dropped
// output) is scaled by them as it is read.
int muse_grn_bwd(const void* x, const void* dout, const float* nx, const float* sumsq, const float* gamma, float* s1_ws,
                 void* dx, float* dgamma, float* dbeta, const unsigned int* bits, float p, int B, int HW, int C,
                 void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (B <= 0 || HW <= 0) return MUSE_OK;
  if (C % 8 != 0) { set_last_error("grn_bwd: C must be a multiple of 8"); return MUSE_ERR_UNSUPPORTED; }
  const bf16* xp = reinterpret_cast<const bf16*>(x);
  const bf16* dp = reinterpret_cast<const bf16*>(dout);
  const philox::ElemDrop drop = philox::elem_drop(const_cast<unsigned int*>(bits), nullptr, 0, p, C);
  pdl_launch(dim3(ceil_div(C, 256), B), 128, 0, s)(bits ? grn_bwd_stats_kernel<true> : grn_bwd_stats_kernel<false>, xp, dp,
                                                   nx, s1_ws, dgamma, dbeta, HW, C, drop);
  int rc = check_launch(bits ? "grn_bwd_stats_dropout" : "grn_bwd_stats");
  if (rc) return rc;
  pdl_launch(B, 256, 0, s)(grn_bwd_finalize_kernel, s1_ws, sumsq, gamma, C);
  rc = check_launch("grn_bwd_finalize");
  if (rc) return rc;
  const long long total8 = static_cast<long long>(B) * HW * (C / 8);
  pdl_launch(static_cast<unsigned>(ceil_div_ll(total8, 256)), 256, 0, s)(bits ? grn_bwd_apply_kernel<true> : grn_bwd_apply_kernel<false>,
      xp, dp, nx, s1_ws, gamma, reinterpret_cast<bf16*>(dx), total8, HW, C, drop);
  return check_launch(bits ? "grn_bwd_apply_dropout" : "grn_bwd_apply");
}

int muse_adaln_bwd(const float* dy, const float* x, const float* ss, long long ss_stride, float* dx, float* dss, int B,
                   int rows_per_sample, int C, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (B <= 0 || rows_per_sample <= 0) return MUSE_OK;
  pdl_launch(dim3(ceil_div(C, 128), B), 128, 0, s)(adaln_bwd_kernel, dy, x, ss, ss_stride, dx, dss, rows_per_sample, C);
  return check_launch("adaln_bwd");
}

int muse_silu_bwd(const void* dy, const void* x, int x_dt, void* dx, int dx_dt, long long n, int accumulate, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0) return MUSE_OK;
  if (n % 8 != 0) { set_last_error("silu_bwd: n must be a multiple of 8"); return MUSE_ERR_INVALID; }
  const long long n8 = n / 8;
  const unsigned grid = static_cast<unsigned>(ceil_div_ll(n8, 256));
  const bf16* dyp = reinterpret_cast<const bf16*>(dy);
  if (x_dt == 1 && dx_dt == 1) pdl_launch(grid, 256, 0, s)(silu_bwd_kernel<bf16, bf16>, dyp, reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(dx), n8, accumulate);
  else if (x_dt == 1 && dx_dt == 0) pdl_launch(grid, 256, 0, s)(silu_bwd_kernel<bf16, float>, dyp, reinterpret_cast<const bf16*>(x), reinterpret_cast<float*>(dx), n8, accumulate);
  else if (x_dt == 0 && dx_dt == 0) pdl_launch(grid, 256, 0, s)(silu_bwd_kernel<float, float>, dyp, reinterpret_cast<const float*>(x), reinterpret_cast<float*>(dx), n8, accumulate);
  else { set_last_error("silu_bwd: unsupported dtype combination"); return MUSE_ERR_INVALID; }
  return check_launch("silu_bwd");
}

}  // extern "C"
