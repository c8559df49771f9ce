// Masked softmax cross-entropy over the vocabulary, forward and backward (HBM-bound).
// Reference: F.cross_entropy(logits.view(-1, V), labels.view(-1), ignore_index=-100,
// label_smoothing=ls) at muse/modeling_transformer.py:1276-1280.  Logits are the bf16 output of the
// to_logits GEMM (row pitch `ld` >= V, pad columns hold zeros and are ignored here).
//   forward : one warp per token row, single pass (online max / sum-exp), writes per-row LSE and
//             per-row loss; a single-block fixed-order reduction produces mean loss + valid count
//             (deterministic, unlike float atomics).
//   backward: dlogits = dloss/N_valid * (softmax - (1-ls) onehot - ls/V) for rows with a label, 0 otherwise.
#include "common.cuh"

namespace muse {
namespace {

constexpr long long kIgnore = -100;

__global__ void __launch_bounds__(128)
ce_fwd_kernel(const bf16* __restrict__ logits, const long long* __restrict__ labels, float* __restrict__ lse_out,
              float* __restrict__ row_loss, int rows, int V, int ld, float ls) {
  pdl_enter();
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const bf16* z = logits + static_cast<size_t>(row) * ld;
  float m = -INFINITY, s = 0.f, sz = 0.f;
  const int v8 = V & ~7;
  for (int c = lane * 8; c < v8; c += 256) {
    float v[8];
    load8(z + c, v);
    float cm = v[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) cm = fmaxf(cm, v[j]);
    const float nm = fmaxf(m, cm);
    float add = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) { add += __expf(v[j] - nm); sz += v[j]; }
    s = s * __expf(m - nm) + add;
    m = nm;
  }
  for (int c = v8 + lane; c < V; c += 32) {
    const float v = __bfloat162float(z[c]);
    const float nm = fmaxf(m, v);
    s = s * __expf(m - nm) + __expf(v - nm);
    m = nm;
    sz += v;
  }
  // merge lanes
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const float os = __shfl_xor_sync(0xffffffffu, s, o);
    const float nm = fmaxf(m, om);
    const float a = (m == -INFINITY) ? 0.f : s * __expf(m - nm);
    const float b = (om == -INFINITY) ? 0.f : os * __expf(om - nm);
    s = a + b;
    m = nm;
  }
  sz = warp_sum(sz);
  if (lane == 0) {
    const float lse = m + logf(s);
    lse_out[row] = lse;
    const long long y = labels[row];
    float loss = 0.f;
    if (y != kIgnore && y >= 0 && y < V) {
      const float zy = __bfloat162float(z[y]);
      loss = (1.f - ls) * (lse - zy) + ls * (lse - sz / static_cast<float>(V));
    }
    row_loss[row] = loss;
  }
}

// out[0] = mean loss over valid rows, out[1] = number of valid rows (as float)
__global__ void __launch_bounds__(1024)
ce_reduce_kernel(const float* __restrict__ row_loss, const long long* __restrict__ labels, float* __restrict__ out,
                 int rows, int V) {
  pdl_enter();
  __shared__ float s_sum[1024];
  __shared__ float s_cnt[1024];
  float a = 0.f, c = 0.f;
  for (int i = threadIdx.x; i < rows; i += 1024) {
    const long long y = labels[i];
    if (y != kIgnore && y >= 0 && y < V) { a += row_loss[i]; c += 1.f; }
  }
  s_sum[threadIdx.x] = a;
  s_cnt[threadIdx.x] = c;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      s_sum[threadIdx.x] += s_sum[threadIdx.x + o];
      s_cnt[threadIdx.x] += s_cnt[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[0] = s_sum[0] / s_cnt[0];
    out[1] = s_cnt[0];
  }
}

__global__ void __launch_bounds__(128)
ce_bwd_kernel(const bf16* __restrict__ logits, const long long* __restrict__ labels, const float* __restrict__ lse_in,
              const float* __restrict__ dloss, const float* __restrict__ loss_cnt, const float* __restrict__ row_scale,
              bf16* __restrict__ dlogits, int rows, int V, int ld, float ls) {
  pdl_enter();
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const bf16* z = logits + static_cast<size_t>(row) * ld;
  bf16* d = dlogits + static_cast<size_t>(row) * ld;
  const long long y = labels[row];
  const bool valid = (y != kIgnore && y >= 0 && y < V);
  if (!valid) {
    for (int c = lane * 8; c < ld; c += 256) *reinterpret_cast<uint4*>(d + c) = make_uint4(0, 0, 0, 0);
    return;
  }
  // mean over the valid rows, or (row_scale given) a caller-defined per-row weight w_r / sum w (loss_weight of
  // MaskGiTUViT_v2.forward, modeling_transformer_v2.py:305-317)
  const float scale = row_scale ? dloss[0] * row_scale[row] : dloss[0] / loss_cnt[1];
  const float lse = lse_in[row];
  const float smooth = ls / static_cast<float>(V);
  for (int c = lane * 8; c < ld; c += 256) {
    float v[8], o[8];
    load8(z + c, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = c + j;
      float g = __expf(v[j] - lse) - smooth;
      if (col == y) g -= (1.f - ls);
      o[j] = (col < V) ? g * scale : 0.f;
    }
    store8(d + c, o);
  }
}

}  // namespace
}  // namespace muse

using namespace muse;

extern "C" {

int muse_ce_fwd(const void* logits, const long long* labels, float* lse, float* row_loss, float* loss_out, int rows, int V,
                int ld, float ls, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0) return MUSE_OK;
  if (ld % 8 != 0 || ld < V) { set_last_error("ce_fwd: ld=%d must be a multiple of 8 and >= V=%d", ld, V); return MUSE_ERR_INVALID; }
  pdl_launch(ceil_div(rows, 4), 128, 0, s)(ce_fwd_kernel, reinterpret_cast<const bf16*>(logits), labels, lse, row_loss, rows, V, ld, ls);
  int rc = check_launch("ce_fwd");
  if (rc) return rc;
  pdl_launch(1, 1024, 0, s)(ce_reduce_kernel, row_loss, labels, loss_out, rows, V);
  return check_launch("ce_reduce");
}

int muse_ce_bwd(const void* logits, const long long* labels, const float* lse, const float* dloss, const float* loss_cnt,
                const float* row_scale, void* dlogits, int rows, int V, int ld, float ls, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0) return MUSE_OK;
  if (ld % 8 != 0 || ld < V) { set_last_error("ce_bwd: ld=%d must be a multiple of 8 and >= V=%d", ld, V); return MUSE_ERR_INVALID; }
  pdl_launch(ceil_div(rows, 4), 128, 0, s)(ce_bwd_kernel, reinterpret_cast<const bf16*>(logits), labels, lse, dloss, loss_cnt, row_scale, reinterpret_cast<bf16*>(dlogits), rows, V, ld, ls);
  return check_launch("ce_bwd");
}

}  // extern "C"
