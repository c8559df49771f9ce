// extern "C" boundary of libmuse_b200.so (declared in include/muse_b200.h).
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/muse_b200.h"
#include "common.cuh"

namespace muse {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// Programmatic dependent launch switch (common.cuh).  Process-wide; the initial value comes from MUSE_B200_PDL.
static int g_pdl = -1;
bool pdl_enabled() {
  if (g_pdl < 0) {
    const char* e = getenv("MUSE_B200_PDL");
    g_pdl = (e != nullptr) ? (atoi(e) != 0) : MUSE_B200_PDL_DEFAULT;
  }
  return g_pdl != 0;
}
void set_pdl(int on) { g_pdl = on ? 1 : 0; }

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
    return MUSE_ERR_CUDA;
  }
  return MUSE_OK;
}

// kernels (defined in the other translation units)
int gemm_tc(const void*, const void*, void*, const float*, int, int, int, int, int, int, int, int, int, cudaStream_t, void*, long long);
long long gemm_splitk_workspace_bytes(int, int, int);
void set_reserved_sms(int);
int pack_bf16(const void*, int, long long, cudaStream_t);
int adamw_ema_step(const void*, int, float*, long long*, const float*, float, float, float, float, float, int, float, float, int, int, int, float, float, cudaStream_t);
int cast_bf16(const float*, void*, long long, cudaStream_t);
int embed_fwd(const long long*, const float*, const float*, float*, int, int, int, int, cudaStream_t);
int embed_bwd(const long long*, const float*, float*, float*, int, int, int, int, cudaStream_t);
int embed_bwd_sorted(const long long*, const long long*, const float*, float*, float*, void*, int, int, int, int, cudaStream_t);
long long embed_bwd_sorted_workspace_bytes(int, int, int);
int norm_fwd(const void*, int, const float*, const float*, void*, int, float*, float*, int, int, float, int, int, cudaStream_t);
int norm_bwd(const void*, int, const void*, int, const float*, const float*, const float*, const float*, const void*, void*, int, void*, float*, float*, int, int, int, int, cudaStream_t);
long long norm_bwd_workspace_floats(int, int, int);
int norm2_fwd(const void*, const float*, const float*, const float*, float*, void*, float*, float*, float*, float*, int, int, float, int, int, cudaStream_t);
int norm2_bwd(const void*, const float*, const float*, const float*, const float*, const float*, const void*, const float*, const float*, const float*, float*, void*, float*, float*, float*, int, int, int, int, cudaStream_t);
int glu_fwd(const void*, void*, long long, int, cudaStream_t);
int glu_bwd(const void*, const void*, void*, long long, int, cudaStream_t);
int attn_fwd(const void*, const void*, const void*, void*, float*, int, int, int, int, int, int, int, int, int, float, cudaStream_t);
int attn_bwd(const void*, const void*, const void*, const void*, const void*, const float*, float*, void*, void*, void*, int, int, int, int, int, int, int, int, int, int, int, int, int, float, cudaStream_t);
int ce_fwd(const void*, const long long*, float*, float*, float*, int, int, int, float, cudaStream_t);
int ce_bwd(const void*, const long long*, const float*, const float*, const float*, const float*, void*, int, int, int, float, cudaStream_t);
int vq_argmin(const float*, const float*, float*, long long*, float*, int, int, int, cudaStream_t);
int vq_lookup_nchw(const long long*, const float*, float*, int, int, int, int, cudaStream_t);
int add_norm_mod_fwd(const void*, int, const float*, const float*, const float*, long long, int, float*, void*, int, int, int, float, int, cudaStream_t);
int dwconv3x3_norm_fwd(const float*, const float*, const float*, void*, void*, int, int, int, int, float, int, cudaStream_t);
int grn_fwd(const void*, const float*, const float*, void*, float*, float*, int, int, int, cudaStream_t);
int add_norm_mod_bwd(const void*, int, const float*, const float*, const float*, const float*, long long, int, void*, int, float*, float*, float*, int, int, float, int, cudaStream_t);
int dwconv3x3_norm_bwd(const void*, const void*, const float*, const float*, const float*, const float*, float*, float*, float*, float*, int, int, int, int, float, int, cudaStream_t);
int grn_bwd(const void*, const void*, const float*, const float*, const float*, float*, void*, float*, float*, int, int, int, cudaStream_t);
int adaln_bwd(const float*, const float*, const float*, long long, float*, float*, int, int, int, cudaStream_t);
int silu_bwd(const void*, const void*, int, void*, int, long long, int, cudaStream_t);
int adaln_apply(float*, const float*, long long, int, int, int, cudaStream_t);
int silu_bf16(const void*, int, void*, long long, cudaStream_t);
int vq_soft_code(const float*, const float*, float*, float*, long long*, const float*, float, int, int, int, cudaStream_t);
int sample_step(const void*, const void*, long long, long long, float, const long long*, const float*, const float*, long long*, long long*, float*, int, int, int, long long, int, float, cudaStream_t);
int conv2d_nhwc(const float*, const float*, const float*, const float*, float*, int, int, int, int, int, int, int, cudaStream_t);
int groupnorm_silu_nhwc(const float*, const float*, const float*, float*, void*, void*, float*, float*, int, int, int, int, float, int, int, cudaStream_t);
int split_s2d_bf16_nhwc(const float*, void*, void*, int, int, int, int, cudaStream_t);
int softmax_split_rows(const float*, void*, void*, float*, long long, int, float, cudaStream_t);
int conv2d_tc_tiles_per_image(int, int, int, int, int, int);
int conv2d_tc_supported(int, int, int, int, int);
int conv2d_tc(const void*, const void*, const void*, const void*, const float*, const float*, float*, float*, int, int, int, int, int, int, int, cudaStream_t);
int split_bf16_nhwc(const float*, void*, void*, int, int, int, int, int, cudaStream_t);
int im2col_split_nhwc(const float*, void*, void*, int, int, int, int, int, cudaStream_t);
long long gn_workspace_floats(int, int, int);
int avgpool2_nhwc(const float*, float*, int, int, int, int, cudaStream_t);
int image_to_uint8(const float*, unsigned char*, long long, cudaStream_t);
int transpose_batched(const float*, float*, int, int, int, cudaStream_t);

}  // namespace muse

using namespace muse;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int muse_abi_version(void) { return MUSE_B200_ABI_VERSION; }
const char* muse_last_error(void) { return g_err; }

int muse_set_device(int device) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) { set_last_error("cudaSetDevice(%d): %s", device, cudaGetErrorString(e)); return MUSE_ERR_CUDA; }
  return MUSE_OK;
}

int muse_device_info(int* sm_major, int* sm_minor, int* num_sms) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) { set_last_error("cudaGetDevice: %s", cudaGetErrorString(e)); return MUSE_ERR_CUDA; }
  cudaDeviceGetAttribute(sm_major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(sm_minor, cudaDevAttrComputeCapabilityMinor, dev);
  cudaDeviceGetAttribute(num_sms, cudaDevAttrMultiProcessorCount, dev);
  return MUSE_OK;
}

int muse_reserve_sms(int n) {
  set_reserved_sms(n);
  return MUSE_OK;
}

int muse_set_pdl(int enabled) {
  set_pdl(enabled);
  return MUSE_OK;
}
int muse_get_pdl(void) { return pdl_enabled() ? 1 : 0; }

int muse_gemm_bf16(const void* A, const void* B, void* C, const float* res, int M, int N, int K, int lda, int ldb,
                   int ldc, int a_mn, int b_mn, int epilogue, void* stream) {
  if (epilogue == MUSE_EPI_RESADD_F32 && res == nullptr) { set_last_error("gemm: RESADD epilogue needs res"); return MUSE_ERR_INVALID; }
  if (epilogue == MUSE_EPI_SPLITK_F32) { set_last_error("gemm: the deterministic split-K epilogue goes through muse_gemm_bf16_splitk"); return MUSE_ERR_INVALID; }
  return gemm_tc(A, B, C, res, M, N, K, lda, ldb, ldc, a_mn, b_mn, epilogue, ST(stream), nullptr, 0);
}

long long muse_gemm_splitk_workspace_bytes(int M, int N, int K) { return gemm_splitk_workspace_bytes(M, N, K); }
int muse_gemm_bf16_splitk(const void* A, const void* B, float* C, int M, int N, int K, int lda, int ldb, int ldc,
                          int a_mn, int b_mn, void* ws, long long ws_bytes, void* stream) {
  return gemm_tc(A, B, C, nullptr, M, N, K, lda, ldb, ldc, a_mn, b_mn, MUSE_EPI_SPLITK_F32, ST(stream), ws, ws_bytes);
}

int muse_pack_bf16(const void* table_dev, int n_entries, long long total_blocks, void* stream) {
  return pack_bf16(table_dev, n_entries, total_blocks, ST(stream));
}
int muse_cast_bf16(const float* src, void* dst, long long n, void* stream) { return cast_bf16(src, dst, n, ST(stream)); }
int muse_adamw_ema_step(const void* entries_host, int n_entries, float* scal_dev, long long* step_dev,
                        const float* lr_dev, float lr_host, float beta1, float beta2, float eps, float weight_decay,
                        int ema_enabled, float ema_decay, float ema_min_decay, int ema_update_after_step,
                        int ema_update_every, int ema_use_warmup, float ema_inv_gamma, float ema_power, void* stream) {
  return adamw_ema_step(entries_host, n_entries, scal_dev, step_dev, lr_dev, lr_host, beta1, beta2, eps,
                        weight_decay, ema_enabled, ema_decay, ema_min_decay, ema_update_after_step, ema_update_every,
                        ema_use_warmup, ema_inv_gamma, ema_power, ST(stream));
}

int muse_embed_fwd(const long long* ids, const float* word, const float* pos, float* out, int B, int S, int H, int vocab, void* stream) {
  return embed_fwd(ids, word, pos, out, B, S, H, vocab, ST(stream));
}
int muse_embed_bwd(const long long* ids, const float* dx, float* dword, float* dpos, int B, int S, int H, int vocab, void* stream) {
  return embed_bwd(ids, dx, dword, dpos, B, S, H, vocab, ST(stream));
}

long long muse_embed_bwd_sorted_workspace_bytes(int tokens, int H, int vocab) { return embed_bwd_sorted_workspace_bytes(tokens, H, vocab); }
int muse_embed_bwd_sorted(const long long* order, const long long* bounds, const float* dx, float* dword, float* dpos,
                          void* ws, int B, int S, int H, int vocab, void* stream) {
  return embed_bwd_sorted(order, bounds, dx, dword, dpos, ws, B, S, H, vocab, ST(stream));
}

int muse_norm_fwd(const void* x, int x_dtype, const float* w, const float* res, void* y, int y_dtype, float* mean,
                  float* rstd, int rows, int H, float eps, int act, int rms, void* stream) {
  return norm_fwd(x, x_dtype, w, res, y, y_dtype, mean, rstd, rows, H, eps, act, rms, ST(stream));
}
int muse_norm_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* w, const float* mean,
                  const float* rstd, const float* dres, const void* y_fwd, void* dx, int dx_dtype, void* dx_bf16_copy,
                  float* dw, float* dw_ws, int rows, int H, int act, int rms, void* stream) {
  return norm_bwd(dy, dy_dtype, x, x_dtype, w, mean, rstd, dres, y_fwd, dx, dx_dtype, dx_bf16_copy, dw, dw_ws, rows, H, act, rms,
                  ST(stream));
}
long long muse_norm_bwd_workspace_floats(int rows, int H, int act) { return norm_bwd_workspace_floats(rows, H, act); }
int muse_norm2_fwd(const void* a, const float* res, const float* w1, const float* w2, float* x2, void* h2, float* mean1,
                   float* rstd1, float* mean2, float* rstd2, int rows, int H, float eps, int rms1, int rms2, void* stream) {
  return norm2_fwd(a, res, w1, w2, x2, h2, mean1, rstd1, mean2, rstd2, rows, H, eps, rms1, rms2, ST(stream));
}
int muse_norm2_bwd(const void* d_h2, const float* x2, const float* w2, const float* mean2, const float* rstd2,
                   const float* dres, const void* a, const float* w1, const float* mean1, const float* rstd1, float* dx2,
                   void* d_a, float* dw2, float* dw1, float* ws, int rows, int H, int rms1, int rms2, void* stream) {
  return norm2_bwd(d_h2, x2, w2, mean2, rstd2, dres, a, w1, mean1, rstd1, dx2, d_a, dw2, dw1, ws, rows, H, rms1, rms2, ST(stream));
}

int muse_glu_fwd(const void* ab, void* out, long long rows, int I, void* stream) { return glu_fwd(ab, out, rows, I, ST(stream)); }
int muse_glu_bwd(const void* ab, const void* dout, void* dab, long long rows, int I, void* stream) {
  return glu_bwd(ab, dout, dab, rows, I, ST(stream));
}

int muse_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int nh, int Sq, int Skv,
                  int head_dim, int q_rs, int k_rs, int v_rs, int o_rs, float scale, void* stream) {
  return attn_fwd(q, k, v, o, lse, B, nh, Sq, Skv, head_dim, q_rs, k_rs, v_rs, o_rs, scale, ST(stream));
}
int muse_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                  float* dvec, void* dq, void* dk, void* dv, int B, int nh, int Sq, int Skv, int head_dim, int q_rs,
                  int k_rs, int v_rs, int o_rs, int do_rs, int dq_rs, int dk_rs, int dv_rs, float scale,
                  void* stream) {
  return attn_bwd(q, k, v, o, d_o, lse, dvec, dq, dk, dv, B, nh, Sq, Skv, head_dim, q_rs, k_rs, v_rs, o_rs, do_rs,
                  dq_rs, dk_rs, dv_rs, scale, ST(stream));
}

int muse_ce_fwd(const void* logits, const long long* labels, float* lse, float* row_loss, float* loss_out, int rows,
                int V, int ld, float label_smoothing, void* stream) {
  return ce_fwd(logits, labels, lse, row_loss, loss_out, rows, V, ld, label_smoothing, ST(stream));
}
int muse_ce_bwd(const void* logits, const long long* labels, const float* lse, const float* dloss,
                const float* loss_out, const float* row_scale, void* dlogits, int rows, int V, int ld,
                float label_smoothing, void* stream) {
  return ce_bwd(logits, labels, lse, dloss, loss_out, row_scale, dlogits, rows, V, ld, label_smoothing, ST(stream));
}

int muse_vq_argmin(const float* z, const float* codebook, float* enorm_ws, long long* ids, float* dmin, int n,
                   int ncodes, int D, void* stream) {
  return vq_argmin(z, codebook, enorm_ws, ids, dmin, n, ncodes, D, ST(stream));
}
int muse_add_norm_mod_fwd(const void* a, int a_dtype, const float* r, const float* w, const float* scale_shift,
                          long long ss_stride, int rows_per_sample, float* r_out, void* y, int y_dtype, int rows, int H,
                          float eps, int rms, void* stream) {
  return add_norm_mod_fwd(a, a_dtype, r, w, scale_shift, ss_stride, rows_per_sample, r_out, y, y_dtype, rows, H, eps, rms,
                          ST(stream));
}
int muse_dwconv3x3_norm_fwd(const float* x, const float* wk, const float* norm_w, void* y, void* conv_out, int B, int h,
                            int w, int C, float eps, int rms, void* stream) {
  return dwconv3x3_norm_fwd(x, wk, norm_w, y, conv_out, B, h, w, C, eps, rms, ST(stream));
}
int muse_grn_fwd(const void* x, const float* gamma, const float* beta, void* out, float* sumsq_ws, float* nx_ws, int B,
                 int HW, int C, void* stream) {
  return grn_fwd(x, gamma, beta, out, sumsq_ws, nx_ws, B, HW, C, ST(stream));
}
int muse_add_norm_mod_bwd(const void* dy, int dy_dtype, const float* dr_out, const float* x, const float* w,
                          const float* scale_shift, long long ss_stride, int rows_per_sample, void* da, int da_dtype,
                          float* dr, float* dw, float* dscale_shift, int rows, int H, float eps, int rms, void* stream) {
  return add_norm_mod_bwd(dy, dy_dtype, dr_out, x, w, scale_shift, ss_stride, rows_per_sample, da, da_dtype, dr, dw,
                          dscale_shift, rows, H, eps, rms, ST(stream));
}
int muse_dwconv3x3_norm_bwd(const void* dy, const void* conv, const float* x, const float* wk, const float* norm_w,
                            const float* dres, float* dc_ws, float* dx, float* dwk, float* dnorm_w, int B, int h, int w,
                            int C, float eps, int rms, void* stream) {
  return dwconv3x3_norm_bwd(dy, conv, x, wk, norm_w, dres, dc_ws, dx, dwk, dnorm_w, B, h, w, C, eps, rms, ST(stream));
}
int muse_grn_bwd(const void* x, const void* dout, const float* nx, const float* sumsq, const float* gamma, float* s1_ws,
                 void* dx, float* dgamma, float* dbeta, int B, int HW, int C, void* stream) {
  return grn_bwd(x, dout, nx, sumsq, gamma, s1_ws, dx, dgamma, dbeta, B, HW, C, ST(stream));
}
int muse_adaln_bwd(const float* dy, const float* x, const float* scale_shift, long long ss_stride, float* dx,
                   float* dscale_shift, int B, int rows_per_sample, int C, void* stream) {
  return adaln_bwd(dy, x, scale_shift, ss_stride, dx, dscale_shift, B, rows_per_sample, C, ST(stream));
}
int muse_silu_bwd(const void* dy, const void* x, int x_dtype, void* dx, int dx_dtype, long long n, int accumulate,
                  void* stream) {
  return silu_bwd(dy, x, x_dtype, dx, dx_dtype, n, accumulate, ST(stream));
}
int muse_adaln_apply(float* x, const float* scale_shift, long long ss_stride, int B, int rows_per_sample, int C,
                     void* stream) {
  return adaln_apply(x, scale_shift, ss_stride, B, rows_per_sample, C, ST(stream));
}
int muse_silu_bf16(const void* x, int x_dtype, void* y, long long n, void* stream) {
  return silu_bf16(x, x_dtype, y, n, ST(stream));
}
int muse_vq_soft_code(const float* z, const float* codebook, float* enorm_ws, float* soft, long long* ids,
                       const float* expo_noise, float temp, int n, int ncodes, int D, void* stream) {
  return vq_soft_code(z, codebook, enorm_ws, soft, ids, expo_noise, temp, n, ncodes, D, ST(stream));
}
int muse_vq_lookup_nchw(const long long* ids, const float* codebook, float* out, int B, int P, int D, int ncodes, void* stream) {
  return vq_lookup_nchw(ids, codebook, out, B, P, D, ncodes, ST(stream));
}

int muse_sample_step(const void* logits, const void* logits_unc, long long row_stride, long long batch_stride,
                     float guidance, const long long* input_ids, const float* q_exp, const float* u,
                     long long* sampled, long long* next_ids, float* conf_out, int B, int L, int K,
                     long long mask_id, int mask_len, float temperature, void* stream) {
  return sample_step(logits, logits_unc, row_stride, batch_stride, guidance, input_ids, q_exp, u, sampled, next_ids,
                     conf_out, B, L, K, mask_id, mask_len, temperature, ST(stream));
}
int muse_conv2d_nhwc(const float* x, const float* wk, const float* bias, const float* res, float* y, int B, int H,
                     int W, int Cin, int Cout, int ksize, int upsample2x, void* stream) {
  return conv2d_nhwc(x, wk, bias, res, y, B, H, W, Cin, Cout, ksize, upsample2x, ST(stream));
}
long long muse_groupnorm_workspace_floats(int B, int HW, int C) { return gn_workspace_floats(B, HW, C); }
int muse_groupnorm_silu_nhwc(const float* x, const float* gamma, const float* beta, float* y, void* y_hi, void* y_lo,
                             float* partials_ws, float* scale_shift_ws, int B, int HW, int C, int groups, float eps,
                             int precomputed_tiles, int apply_silu, void* stream) {
  return groupnorm_silu_nhwc(x, gamma, beta, y, y_hi, y_lo, partials_ws, scale_shift_ws, B, HW, C, groups, eps,
                             precomputed_tiles, apply_silu, ST(stream));
}
int muse_split_s2d_bf16_nhwc(const float* x, void* hi, void* lo, int B, int Ho, int Wo, int C, void* stream) {
  return split_s2d_bf16_nhwc(x, hi, lo, B, Ho, Wo, C, ST(stream));
}
int muse_softmax_split_rows(const float* x, void* hi, void* lo, float* out_f32, long long rows, int n, float scale,
                            void* stream) {
  return softmax_split_rows(x, hi, lo, out_f32, rows, n, scale, ST(stream));
}
int muse_conv2d_tc_tiles_per_image(int H, int W, int Cin, int Cout, int ksize, int upsample2x) {
  return conv2d_tc_tiles_per_image(H, W, Cin, Cout, ksize, upsample2x);
}
int muse_conv2d_tc_supported(int H, int W, int Cin, int Cout, int ksize) { return conv2d_tc_supported(H, W, Cin, Cout, ksize); }
int muse_conv2d_nhwc_tc(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, const float* bias,
                        const float* res, float* y, float* stats, int B, int H, int W, int Cin, int Cout, int ksize,
                        int mode, void* stream) {
  return conv2d_tc(x_hi, x_lo, w_hi, w_lo, bias, res, y, stats, B, H, W, Cin, Cout, ksize, mode, ST(stream));
}
int muse_split_bf16_nhwc(const float* x, void* hi, void* lo, int B, int H, int W, int C, int upsample2x, void* stream) {
  return split_bf16_nhwc(x, hi, lo, B, H, W, C, upsample2x, ST(stream));
}
int muse_im2col_split_nhwc(const float* x, void* hi, void* lo, int B, int H, int W, int Cin, int ksize, void* stream) {
  return im2col_split_nhwc(x, hi, lo, B, H, W, Cin, ksize, ST(stream));
}
int muse_avgpool2_nhwc(const float* x, float* y, int B, int Ho, int Wo, int C, void* stream) {
  return avgpool2_nhwc(x, y, B, Ho, Wo, C, ST(stream));
}
int muse_image_to_uint8(const float* x, unsigned char* y, long long n, void* stream) { return image_to_uint8(x, y, n, ST(stream)); }
int muse_transpose_batched(const float* in, float* out, int B, int rows, int cols, void* stream) {
  return transpose_batched(in, out, B, rows, cols, ST(stream));
}

}  // extern "C"
