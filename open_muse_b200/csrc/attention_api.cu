// Attention entry points of the C ABI: Attention.attention of the reference (muse/modeling_transformer.py:221-241) and its
// autograd backward, head_dim 64 or 48, no mask, no dropout.  Every shape runs on the wgmma / TMA kernels of
// attention_tc.cu (balanced row tiles cover ragged sequence lengths such as 257 = 256 + class token and the 77 text
// states of cross-attention); there is no second implementation in this library.
#include "common.cuh"

namespace muse {

int attn_fwd_tc(const void*, const void*, const void*, void*, float*, int, int, int, int, int, int, int, int, int, float,
                cudaStream_t, int*);
int attn_bwd_dq_tc(const void*, const void*, const void*, const void*, const float*, float*, void*, int, int, int, int,
                   int, int, int, int, int, int, float, cudaStream_t, int*);
int attn_bwd_dkdv_tc(const void*, const void*, const void*, const void*, const float*, const float*, void*, void*, int,
                     int, int, int, int, int, int, int, int, int, int, float, cudaStream_t, int*);

namespace {
int check_strides(const char* who, int hd, int a, int b, int c) {
  if (hd != 64 && hd != 48) { set_last_error("%s: head_dim %d unsupported (64 and 48 are built)", who, hd); return MUSE_ERR_UNSUPPORTED; }
  if (((a | b | c) & 7) != 0) { set_last_error("%s: row strides must be multiples of 8 elements", who); return MUSE_ERR_INVALID; }
  return MUSE_OK;
}
}  // namespace

int attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int nh, int Sq, int Skv, int hd,
             int q_rs, int k_rs, int v_rs, int o_rs, float scale, cudaStream_t s) {
  if (B <= 0 || Sq <= 0 || Skv <= 0) return MUSE_OK;
  int rc = check_strides("attn_fwd", hd, q_rs | o_rs, k_rs, v_rs);
  if (rc) return rc;
  int done = 0;
  return attn_fwd_tc(q, k, v, o, lse, B, nh, Sq, Skv, hd, q_rs, k_rs, v_rs, o_rs, scale, s, &done);
}

int attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
             float* dvec, void* dq, void* dk, void* dv, int B, int nh, int Sq, int Skv, int hd, int q_rs, int k_rs,
             int v_rs, int o_rs, int do_rs, int dq_rs, int dk_rs, int dv_rs, float scale, cudaStream_t s) {
  if (B <= 0 || Sq <= 0 || Skv <= 0) return MUSE_OK;
  int rc = check_strides("attn_bwd", hd, q_rs | o_rs | do_rs | dq_rs, k_rs | dk_rs, v_rs | dv_rs);
  if (rc) return rc;
  (void)o; (void)o_rs;  // D is recomputed from (P, dP) inside the dQ kernel; O is not needed by backward
  int done = 0;
  rc = attn_bwd_dq_tc(q, k, v, d_o, lse, dvec, dq, B, nh, Sq, Skv, hd, q_rs, k_rs, v_rs, do_rs, dq_rs, scale, s, &done);
  if (rc) return rc;
  return attn_bwd_dkdv_tc(q, k, v, d_o, lse, dvec, dk, dv, B, nh, Sq, Skv, hd, q_rs, k_rs, v_rs, do_rs, dk_rs, dv_rs, scale, s,
                          &done);
}

}  // namespace muse
