// One generate2 decoding step (sample -> confidence -> per-row k-th smallest -> re-mask) as two kernels: a token-parallel
// pass over the [B, L, K] logits and noise (one warp per token: the whole GPU streams them once) and a per-row re-mask.
// Reference: muse/modeling_transformer.py:1424-1454 + muse/sampling.py:9-15,30-35, which is ~25 ATen launches
// per step (softmax, multinomial = exponential_ + div + argmax, where, gather, where, log, uniform_, log, log,
// mul, add, sort, gather, lt, where ...) over a [B, L, K] fp32 probability tensor.
//
// Randomness enters as PRE-DRAWN noise so the torch generator stream is the reference's own:
//   q_exp [B, L, K] ~ Exp(1)   torch.multinomial(p, 1) == argmax_c(p_c / q_c)   (ATen's n_sample == 1 recipe)
//   u     [B, L]    ~ U(0, 1)  gumbel = -log(-log(u))  (sampling.py:13-15, with the 1e-20 clamps of :9-10)
// Per token (one warp), then per row b (one CTA):
//   m = max_c x_c ; e_c = exp(x_c - m) ; sampled = first argmax_c e_c / q_c      (softmax normaliser cancels)
//   p_sel = e_sampled / sum_c e_c ; known tokens keep their id and get p_sel = FLT_MAX (:1430-1441)
//   conf = log(max(p_sel,1e-20)) + temperature * gumbel(u)
//   k = max(1, min(#unknown - 1, mask_len))  (:1443-1448);  cut = (k+1)-th smallest conf (sorted[k])
//   next_id = conf < cut ? mask_id : sampled                                       (sampling.py:32-35, :1454)
// "conf_i < sorted[k]"  <=>  #{j : conf_j <= conf_i} <= k, evaluated by counting (L <= 1024): no sort needed.
// Optional classifier-free guidance: x = unc + g * (cond - unc) (:1410-1414), fused into the logit read.
#include <float.h>

#include "common.cuh"

namespace muse {
namespace {

// Phase 1: one warp per token (grid over all B*L tokens, so the whole GPU streams the [B, L, K] logits and noise once).
constexpr int kTokWarps = 8;
__global__ void __launch_bounds__(kTokWarps * 32)
sample_tokens_kernel(const bf16* __restrict__ logits, const bf16* __restrict__ logits_unc, long long row_stride,
                     long long batch_stride, float guidance, const long long* __restrict__ input_ids,
                     const float* __restrict__ q_exp, const float* __restrict__ u, long long* __restrict__ sampled_out,
                     float* __restrict__ conf_out, int B, int L, int K, long long mask_id, float temperature) {
  pdl_enter();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long tok = static_cast<long long>(blockIdx.x) * kTokWarps + warp;
  if (tok >= static_cast<long long>(B) * L) return;
  const int b = static_cast<int>(tok / L), tkn = static_cast<int>(tok % L);
  const bf16* x = logits + b * batch_stride + tkn * row_stride;
  const bf16* xu = logits_unc ? logits_unc + b * batch_stride + tkn * row_stride : nullptr;
  const float* q = q_exp + tok * K;
  float m = -INFINITY, sum = 0.f, best = -1.f, e_best = 0.f;
  int besti = 0;
  // vector path (warp-uniform choice): 8 consecutive codes per lane and step -- one 16-byte logits load and two 16-byte noise
  // loads instead of 8 + 8 scalar ones (the scalar loop ran at 1.6 TB/s)
  const bool vec = (K & 7) == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(q)) & 15) == 0 &&
                   (xu == nullptr || (reinterpret_cast<uintptr_t>(xu) & 15) == 0);
  if (vec) {
    auto load8v = [&](int c0, float (&v)[8]) {
      load8(x + c0, v);
      if (xu) {
        float w[8];
        load8(xu + c0, w);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = w[i] + guidance * (v[i] - w[i]);
      }
    };
    for (int c0 = lane * 8; c0 < K; c0 += 256) {  // pass 1: row max
      float v[8];
      load8v(c0, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) m = fmaxf(m, v[i]);
    }
    m = warp_max(m);
    for (int c0 = lane * 8; c0 < K; c0 += 256) {  // pass 2: sum of exp, arg-max of exp / q (indices ascend: first wins ties)
      float v[8], qv[8];
      load8v(c0, v);
      load8(q + c0, qv);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float e = expf(v[i] - m);
        sum += e;
        const float sc = e / qv[i];
        if (sc > best) { best = sc; besti = c0 + i; e_best = e; }
      }
    }
  } else {
    for (int c = lane; c < K; c += 32) {  // pass 1: row max
      float v = __bfloat162float(x[c]);
      if (xu) { const float w = __bfloat162float(xu[c]); v = w + guidance * (v - w); }
      m = fmaxf(m, v);
    }
    m = warp_max(m);
    for (int c = lane; c < K; c += 32) {  // pass 2: sum of exp, arg-max of exp / q (lowest index on ties)
      float v = __bfloat162float(x[c]);
      if (xu) { const float w = __bfloat162float(xu[c]); v = w + guidance * (v - w); }
      const float e = expf(v - m);
      sum += e;
      const float sc = e / q[c];
      if (sc > best) { best = sc; besti = c; e_best = e; }
    }
  }
  sum = warp_sum(sum);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    const float oe = __shfl_xor_sync(0xffffffffu, e_best, o);
    if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; e_best = oe; }
  }
  if (lane == 0) {
    const long long cur = input_ids[tok];
    const bool unknown = (cur == mask_id);
    const long long sid = unknown ? static_cast<long long>(besti) : cur;
    const float p_sel = unknown ? e_best / sum : FLT_MAX;
    const float uu = u[tok];
    const float gum = -logf(fmaxf(-logf(fmaxf(uu, 1e-20f)), 1e-20f));
    conf_out[tok] = logf(fmaxf(p_sel, 1e-20f)) + temperature * gum;
    sampled_out[tok] = sid;
  }
}

// Phase 2: one CTA per batch row: k = clamp(#unknown - 1, 1, mask_len); re-mask the k lowest confidences by rank counting.
__global__ void __launch_bounds__(1024)
sample_remask_kernel(const long long* __restrict__ input_ids, const long long* __restrict__ sampled, const float* __restrict__ conf,
                     long long* __restrict__ next_ids, int L, long long mask_id, int mask_len) {
  pdl_enter();
  extern __shared__ float s_conf[];  // [L]
  __shared__ int s_unknown;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) s_unknown = 0;
  __syncthreads();
  int mine = 0;
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    s_conf[i] = conf[static_cast<long long>(b) * L + i];
    mine += (input_ids[static_cast<long long>(b) * L + i] == mask_id) ? 1 : 0;
  }
  mine = static_cast<int>(warp_sum(static_cast<float>(mine)) + 0.5f);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_unknown, mine);
  __syncthreads();
  int k = min(s_unknown - 1, mask_len);
  k = max(1, k);
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    const float ci = s_conf[i];
    int le = 0;
    for (int j = 0; j < L; ++j) le += (s_conf[j] <= ci) ? 1 : 0;
    next_ids[static_cast<long long>(b) * L + i] = (le <= k) ? mask_id : sampled[static_cast<long long>(b) * L + i];
  }
}

}  // namespace
}  // namespace muse

using namespace muse;

extern "C" {

int muse_sample_step(const void* logits, const void* logits_unc, long long row_stride, long long batch_stride,
                     float guidance, const long long* input_ids, const float* q_exp, const float* u,
                     long long* sampled, long long* next_ids, float* conf_out, int B, int L, int K, long long mask_id,
                     int mask_len, float temperature, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (B <= 0 || L <= 0) return MUSE_OK;
  if (L > 4096) { set_last_error("sample_step: L=%d too long (max 4096)", L); return MUSE_ERR_UNSUPPORTED; }
  if (conf_out == nullptr) { set_last_error("sample_step: conf_out (B*L floats) is required"); return MUSE_ERR_INVALID; }
  const long long tokens = static_cast<long long>(B) * L;
  pdl_launch(static_cast<unsigned>(ceil_div_ll(tokens, kTokWarps)), kTokWarps * 32, 0, s)(sample_tokens_kernel,
      reinterpret_cast<const bf16*>(logits), reinterpret_cast<const bf16*>(logits_unc), row_stride, batch_stride, guidance,
      input_ids, q_exp, u, sampled, conf_out, B, L, K, mask_id, temperature);
  int rc = check_launch("sample_tokens");
  if (rc) return rc;
  const int threads = L >= 1024 ? 1024 : ((L + 31) / 32) * 32;
  pdl_launch(B, threads, L * sizeof(float), s)(sample_remask_kernel, input_ids, sampled, conf_out, next_ids, L, mask_id, mask_len);
  return check_launch("sample_remask");
}

}  // extern "C"
