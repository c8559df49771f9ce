// Warp-per-row LayerNorm / RMSNorm core of the H <= 1024 norm kernels (norm.cu, uvit.cu, uvit_bwd.cu).
// One warp owns one row and holds it in registers as float v[CH][8]: chunk c of lane `lane` is the 8 columns starting at
// row_col(c, lane), and chunks at or past H are zero.  Each helper fixes the order of its floating-point operations, so
// every kernel built on them produces the same bits for the same row.  The GLU and wide streaming kernels of norm.cu
// keep their own loops: they do not hold the row as floats (packed bf16 pairs, or no row at all).  row_store_e4m3 writes
// a finished row as the e4m3 operand of muse_gemm_fp8, which needs the row's absolute maximum before any element.
#pragma once
#include <cuda_fp8.h>

#include <type_traits>

#include "common.cuh"

namespace muse {

__device__ __forceinline__ int row_col(int c, int lane) { return (c * 32 + lane) * 8; }

// Fills the register row: load(col, v[c]) for every chunk inside the row, zeros past H.  Returns the lane's sum of
// the loaded values, accumulated chunk by chunk as they arrive.
template <int CH, typename Load>
__device__ __forceinline__ float row_load(float (&v)[CH][8], int H, int lane, Load&& load) {
  float sum = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = row_col(c, lane);
    if (col < H) {
      load(col, v[c]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[c][j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[c][j] = 0.f;
    }
  }
  return sum;
}

// Two-pass forward statistics of the register row from the lane sums `sum` of its values (row_load): mean (0 for
// RMSNorm), then rstd = 1 / sqrt(mean((v - mean)^2) + eps).  inv_h = 1 / H is computed once by the caller, outside any
// row loop.
template <int CH>
__device__ __forceinline__ void row_stats(const float (&v)[CH][8], float sum, int H, float inv_h, int lane, float eps,
                                          int rms, float& mean, float& rstd) {
  mean = rms ? 0.f : warp_sum(sum) * inv_h;
  float sq = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c)
    if (row_col(c, lane) < H) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[c][j] - mean;
        sq = fmaf(d, d, sq);
      }
    }
  rstd = rsqrtf(warp_sum(sq) * inv_h + eps);
}

// Backward, with g = dL/dxhat: each lane accumulates s1 += g and s2 += g * xhat over its elements (element by element,
// inside the kernel's own loop), row_bwd_sums turns the lane sums into s1 = mean(g) (0 for RMSNorm) and
// s2 = mean(g * xhat), and row_dx gives dL/dv = rstd * (g - s1 - xhat * s2).
__device__ __forceinline__ void row_bwd_acc(float g, float xh, float& s1, float& s2) {
  s1 += g;
  s2 = fmaf(g, xh, s2);
}
__device__ __forceinline__ void row_bwd_sums(float inv_h, int rms, float& s1, float& s2) {
  s1 = rms ? 0.f : warp_sum(s1) * inv_h;
  s2 = warp_sum(s2) * inv_h;
}
__device__ __forceinline__ float row_dx(float g, float xh, float s1, float s2, float rstd) {
  return rstd * (g - s1 - xh * s2);
}

// e4m3 form of a finished register row (chunks at or past H hold zeros): s = amax / 448, or 1 for an all-zero row;
// q[col] = e4m3_rn_satfinite(v / s) with a correctly rounded division, s to row_scale[0] (lane 0).  q: the row's bytes.
template <int CH>
__device__ __forceinline__ void row_store_e4m3(const float (&v)[CH][8], int H, int lane, uint8_t* q, float* row_scale) {
  float amax = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(v[c][j]));
  amax = warp_max(amax);
  const float s = amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f;
  if (lane == 0) *row_scale = s;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int col = row_col(c, lane);
    if (col < H) {
      uint32_t w[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float* x = &v[c][4 * h];
        const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(x[0], s), __fdiv_rn(x[1], s)), __NV_SATFINITE, __NV_E4M3);
        const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(x[2], s), __fdiv_rn(x[3], s)), __NV_SATFINITE, __NV_E4M3);
        w[h] = lo | (hi << 16);
      }
      *reinterpret_cast<uint2*>(q + col) = make_uint2(w[0], w[1]);
    }
  }
}

// ---- host side

// Calls f(std::integral_constant<int, CH>()) with the first CH of the list whose CH * 256 columns cover H, or the last one.
// Each call site lists the chunk counts its kernel is instantiated for.
template <int CH, int... More, typename F>
void with_row_chunks(int H, F&& f) {
  if constexpr (sizeof...(More) == 0) {
    f(std::integral_constant<int, CH>());
  } else {
    if (H <= CH * 256) f(std::integral_constant<int, CH>());
    else with_row_chunks<More...>(H, f);
  }
}

// Calls f(T0(), T1(), ...) with Ti = float for dtype code 0 and bf16 for code 1, one type per code, and returns its status.
template <typename... Ts, typename F>
int dtype_dispatch(const char* who, F&& f) {
  return f(Ts()...);
}
template <typename... Ts, typename F, typename... Codes>
int dtype_dispatch(const char* who, F&& f, int code, Codes... more) {
  if (code == 0) return dtype_dispatch<Ts..., float>(who, f, more...);
  if (code == 1) return dtype_dispatch<Ts..., bf16>(who, f, more...);
  set_last_error("%s: bad dtype code %d", who, code);
  return MUSE_ERR_INVALID;
}

// Raises the dynamic shared-memory limit of each listed kernel to `bytes`, the first time it is called for that list.
template <auto... Kernels>
void allow_dynamic_smem_once(int bytes) {
  static const bool done =
      ((cudaFuncSetAttribute(Kernels, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes), ...), true);
  (void)done;
}

}  // namespace muse
