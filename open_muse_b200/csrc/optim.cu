// Step-adjacent host ops fused into ONE pass over the parameters (SURVEY.md 8f-4):
//   AdamW update (training/train_maskgit_imagenet.py:242-261,438: torch.optim.AdamW / apex FusedAdam, decoupled weight
//   decay) + EMA of the updated weights (muse/modeling_ema.py:108-126: s -= (1 - decay) * (s - p)) + the bf16 copy of the
//   updated weight into the packed GEMM operand cache (autocast's per-Linear weight cast).
// The reference runs these as a multi-tensor optimizer launch set, ~3 kernels PER PARAMETER for the EMA, and one cast per
// Linear per forward.  Here every parameter element is read once (p, g, m, v, ema) and written once (p, m, v, ema, bf16).
//
// Lion (training/optimizer.py::Lion, the scripts' `optimizer.name: lion`) runs through the same table, prepare kernel and
// chunk loop with one moment instead of two: the table's v slot is unused.
//
// Scalars that change every step (bias corrections, EMA decay, learning rate) live in a small device array filled by a
// one-thread pre-kernel from the device-resident step counter, so that the pair of launches is CUDA-graph capturable and
// replays advance the schedule correctly.
#include "common.cuh"

namespace muse {
namespace {

struct OptEntry {
  float* p;
  const float* g;
  float* m;
  float* v;
  float* ema;        // nullable
  bf16* packed;      // nullable: bf16 operand copy
  long long numel;   // multiple of 4
  long long first_block;
};

struct OptHyper {
  float beta1, beta2, eps, weight_decay;
  // EMA schedule (muse/modeling_ema.py:89-106)
  float ema_decay, ema_min_decay, ema_inv_gamma, ema_power;
  int ema_update_after_step, ema_update_every, ema_use_warmup, ema_enabled;
  // Lion only: 1 - beta1, 1 - beta2 and 1 - lr * weight_decay, each formed in double on the host and rounded once to fp32,
  // as the reference's Python scalars reach ATen (1.0f - beta computed in fp32 differs in the last bit for beta = 0.9)
  float one_minus_beta1, one_minus_beta2, wd_scale_host;
};

// scal: [0] step (after increment) [1] 1/bias_correction1 [2] 1/sqrt(bias_correction2) [3] lr [4] 1 - ema_decay_now (0: skip)
//       [5] ema_decay_now [6] Lion's 1 - lr * weight_decay
__global__ void opt_prepare_kernel(float* scal, long long* step, const float* lr_dev, float lr_host, OptHyper h) {
  pdl_enter();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const long long s = *step + 1;
  *step = s;
  const double bc1 = 1.0 - pow(static_cast<double>(h.beta1), static_cast<double>(s));
  const double bc2 = 1.0 - pow(static_cast<double>(h.beta2), static_cast<double>(s));
  scal[0] = static_cast<float>(s);
  scal[1] = static_cast<float>(1.0 / bc1);
  scal[2] = static_cast<float>(1.0 / sqrt(bc2));
  scal[3] = lr_dev ? *lr_dev : lr_host;
  // a device lr has no double to start from: 1 - lr * wd is formed in fp32 (one rounding per operation)
  scal[6] = lr_dev ? __fsub_rn(1.0f, __fmul_rn(*lr_dev, h.weight_decay)) : h.wd_scale_host;
  double decay = 0.0;
  bool update = false;
  if (h.ema_enabled) {
    update = ((s - 1) % h.ema_update_every) == 0;
    const long long st = max(0LL, s - h.ema_update_after_step - 1);
    if (st > 0) {
      const double value = h.ema_use_warmup ? 1.0 - pow(1.0 + static_cast<double>(st) / h.ema_inv_gamma, -static_cast<double>(h.ema_power))
                                            : (1.0 + st) / (10.0 + st);
      decay = fmax(fmin(value, static_cast<double>(h.ema_decay)), static_cast<double>(h.ema_min_decay));
    }
  }
  // the reference computes one_minus_decay = 1 - decay in Python doubles and multiplies fp32 tensors by it
  scal[4] = update ? static_cast<float>(1.0 - decay) : -1.0f;  // < 0: no EMA update this step
  scal[5] = static_cast<float>(decay);
}

// The parameter table travels in the kernel ARGUMENTS (like ATen's multi_tensor_apply), not in device memory: no
// host->device copy exists, so the step can be captured in a CUDA graph even when the gradient buffers move between the
// eager warm-up and the capture (the graph bakes the arguments of that launch).
constexpr int kOptChunk = 48;  // 48 x 64 B of entries + hyper-parameters stay under the 4 KB kernel-parameter limit
struct OptChunk {
  OptEntry e[kOptChunk];
  int n;
};

enum class OptAlgo { kAdamW, kLion };

// Lion's update of one element, in the reference's operation order (training/optimizer.py::Lion.step), one rounding per
// ATen op so that p and m equal torch's on the same GPU bit for bit:
//   p.mul_(1 - lr * wd)                      p * c_wd
//   update = m * beta1 + g * (1 - beta1)     three separate ops: two products and a sum, no contraction
//   p.add_(sign(update), alpha=-lr)          lr * sign is exact, so the fma rounds once, like ATen's a + alpha * b
//   m.mul_(beta2).add_(g, alpha=1 - beta2)   ATen's add functor (a + b * alpha) is contracted to one fma by nvcc
// sign(0) = 0 as torch.sign.
__device__ __forceinline__ void lion_update(float& p, float g, float& m, float c_wd, float lr, const OptHyper& h) {
  p = __fmul_rn(p, c_wd);
  const float u = __fadd_rn(__fmul_rn(m, h.beta1), __fmul_rn(g, h.one_minus_beta1));
  const float sg = static_cast<float>((0.0f < u) - (u < 0.0f));
  p = __fmaf_rn(-lr, sg, p);
  m = __fmaf_rn(g, h.one_minus_beta2, __fmul_rn(m, h.beta2));
}

template <OptAlgo kAlgo>
__global__ void __launch_bounds__(256)
opt_ema_pack_kernel(const __grid_constant__ OptChunk chunk, const float* __restrict__ scal, const OptHyper h) {
  pdl_enter();
  const long long blk = blockIdx.x;
  int lo = 0, hi = chunk.n - 1;
  while (lo < hi) {  // last entry with first_block <= blk
    const int mid = (lo + hi + 1) >> 1;
    if (chunk.e[mid].first_block <= blk) lo = mid; else hi = mid - 1;
  }
  const OptEntry& e = chunk.e[lo];
  const long long i = ((blk - e.first_block) * 256 + threadIdx.x) * 4;
  if (i >= e.numel) return;
  const float lr = scal[3], omd = scal[4];
  float4 p4 = *reinterpret_cast<const float4*>(e.p + i);
  const float4 g4 = *reinterpret_cast<const float4*>(e.g + i);
  float4 m4 = *reinterpret_cast<const float4*>(e.m + i);
  float p[4] = {p4.x, p4.y, p4.z, p4.w};
  const float g[4] = {g4.x, g4.y, g4.z, g4.w};
  float m[4] = {m4.x, m4.y, m4.z, m4.w};
  if constexpr (kAlgo == OptAlgo::kAdamW) {
    const float inv_bc1 = scal[1], inv_sqrt_bc2 = scal[2];
    float4 v4 = *reinterpret_cast<const float4*>(e.v + i);
    float v[4] = {v4.x, v4.y, v4.z, v4.w};
    const float step_size = lr * inv_bc1;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      p[k] -= lr * h.weight_decay * p[k];                       // decoupled weight decay
      m[k] = m[k] + (1.0f - h.beta1) * (g[k] - m[k]);            // lerp(m, g, 1 - beta1)
      v[k] = h.beta2 * v[k] + (1.0f - h.beta2) * g[k] * g[k];
      const float denom = sqrtf(v[k]) * inv_sqrt_bc2 + h.eps;
      p[k] -= step_size * m[k] / denom;
    }
    *reinterpret_cast<float4*>(e.v + i) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    const float c_wd = scal[6];
#pragma unroll
    for (int k = 0; k < 4; ++k) lion_update(p[k], g[k], m[k], c_wd, lr, h);
  }
  *reinterpret_cast<float4*>(e.p + i) = make_float4(p[0], p[1], p[2], p[3]);
  *reinterpret_cast<float4*>(e.m + i) = make_float4(m[0], m[1], m[2], m[3]);
  if (e.ema != nullptr && omd >= 0.f) {
    float4 s4 = *reinterpret_cast<const float4*>(e.ema + i);
    s4.x -= omd * (s4.x - p[0]); s4.y -= omd * (s4.y - p[1]); s4.z -= omd * (s4.z - p[2]); s4.w -= omd * (s4.w - p[3]);
    *reinterpret_cast<float4*>(e.ema + i) = s4;
  }
  if (e.packed != nullptr) {
    uint2 u;
    u.x = pack_bf16(p[0], p[1]);
    u.y = pack_bf16(p[2], p[3]);
    *reinterpret_cast<uint2*>(e.packed + i) = u;
  }
}

OptHyper make_hyper(float beta1, float beta2, int ema_enabled, float ema_decay, float ema_min_decay,
                    int ema_update_after_step, int ema_update_every, int ema_use_warmup, float ema_inv_gamma,
                    float ema_power) {
  OptHyper h = {};
  h.beta1 = beta1; h.beta2 = beta2;
  h.ema_enabled = ema_enabled; h.ema_decay = ema_decay; h.ema_min_decay = ema_min_decay;
  h.ema_update_after_step = ema_update_after_step; h.ema_update_every = ema_update_every < 1 ? 1 : ema_update_every;
  h.ema_use_warmup = ema_use_warmup; h.ema_inv_gamma = ema_inv_gamma; h.ema_power = ema_power;
  return h;
}

// the prepare launch, then one update launch per chunk of kOptChunk table entries
template <OptAlgo kAlgo>
int opt_step(const char* what, const void* entries_host, int n_entries, float* scal_dev, long long* step_dev,
             const float* lr_dev, float lr_host, const OptHyper& h, cudaStream_t s) {
  if (n_entries <= 0) return MUSE_OK;
  pdl_launch(1, 32, 0, s)(opt_prepare_kernel, scal_dev, step_dev, lr_dev, lr_host, h);
  int rc = check_launch(what);
  if (rc) return rc;
  const OptEntry* all = reinterpret_cast<const OptEntry*>(entries_host);
  for (int base = 0; base < n_entries; base += kOptChunk) {
    OptChunk chunk;
    chunk.n = n_entries - base < kOptChunk ? n_entries - base : kOptChunk;
    long long blocks = 0;
    for (int i = 0; i < chunk.n; ++i) {
      chunk.e[i] = all[base + i];
      if (chunk.e[i].numel % 4 != 0 || chunk.e[i].numel <= 0) {
        set_last_error("%s: numel must be a positive multiple of 4", what);
        return MUSE_ERR_INVALID;
      }
      chunk.e[i].first_block = blocks;
      blocks += (chunk.e[i].numel + 1023) / 1024;
    }
    pdl_launch(static_cast<unsigned>(blocks), 256, 0, s)(opt_ema_pack_kernel<kAlgo>, chunk, scal_dev, h);
    rc = check_launch(what);
    if (rc) return rc;
  }
  return MUSE_OK;
}

}  // namespace
}  // namespace muse

using namespace muse;

extern "C" {

// entries_host: HOST array of n_entries {p, g, m, v, ema, packed, numel, unused} (8 x int64 each; device pointers inside);
// scal_dev: 8 floats; step_dev: one int64 (number of optimizer steps taken so far); lr_dev: nullable device float
// (graph-capturable learning-rate schedule) else lr_host is used.
int muse_adamw_ema_step(const void* entries_host, int n_entries, float* scal_dev, long long* step_dev,
                        const float* lr_dev, float lr_host, float beta1, float beta2, float eps, float weight_decay,
                        int ema_enabled, float ema_decay, float ema_min_decay, int ema_update_after_step, int ema_update_every,
                        int ema_use_warmup, float ema_inv_gamma, float ema_power, void* stream) {
  OptHyper h = make_hyper(beta1, beta2, ema_enabled, ema_decay, ema_min_decay, ema_update_after_step, ema_update_every,
                          ema_use_warmup, ema_inv_gamma, ema_power);
  h.eps = eps; h.weight_decay = weight_decay;
  return opt_step<OptAlgo::kAdamW>("adamw_ema_step", entries_host, n_entries, scal_dev, step_dev, lr_dev, lr_host, h,
                                   static_cast<cudaStream_t>(stream));
}

// Same table (v unused), counters and EMA arguments as muse_adamw_ema_step.  one_minus_beta1 / one_minus_beta2 / wd_scale
// (= 1 - lr * weight_decay, used when lr_dev is null) are the host's double values rounded to fp32.
int muse_lion_ema_step(const void* entries_host, int n_entries, float* scal_dev, long long* step_dev,
                       const float* lr_dev, float lr_host, float wd_scale, float beta1, float beta2, float one_minus_beta1,
                       float one_minus_beta2, float weight_decay, int ema_enabled, float ema_decay, float ema_min_decay,
                       int ema_update_after_step, int ema_update_every, int ema_use_warmup, float ema_inv_gamma,
                       float ema_power, void* stream) {
  OptHyper h = make_hyper(beta1, beta2, ema_enabled, ema_decay, ema_min_decay, ema_update_after_step, ema_update_every,
                          ema_use_warmup, ema_inv_gamma, ema_power);
  h.weight_decay = weight_decay;
  h.one_minus_beta1 = one_minus_beta1; h.one_minus_beta2 = one_minus_beta2; h.wd_scale_host = wd_scale;
  return opt_step<OptAlgo::kLion>("lion_ema_step", entries_host, n_entries, scal_dev, step_dev, lr_dev, lr_host, h,
                                  static_cast<cudaStream_t>(stream));
}

}  // extern "C"
