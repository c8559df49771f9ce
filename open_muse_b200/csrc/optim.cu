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
// AdamW with 8-bit block-wise moments (Dettmers et al., "8-bit Optimizers via Block-wise Quantization", the scheme of
// bitsandbytes' AdamW8bit; the script's `optimizer.name: 8bit_adamw`) runs the same element update on moments decoded from
// uint8 codes, one fp32 absmax per 256-element block, and re-encodes them against 256-entry dynamic maps.  Tensors below
// the 8-bit threshold keep fp32 moments and go through the AdamW kernel in the same call, after the same prepare launch.
//
// Scalars that change every step (bias corrections, EMA decay, learning rate) live in a small device array filled by a
// one-thread pre-kernel from the device-resident step counter, so that the pair of launches is CUDA-graph capturable and
// replays advance the schedule correctly.
#include <vector>

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
// 48 entries per launch: 48 x 64 B (fp32 moments) or 48 x 80 B (8-bit moments: + two absmax pointers) of entries, plus the
// pointers and hyper-parameters, stay under the 4 KB kernel-parameter limit
constexpr int kOptChunk = 48;
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

// AdamW's update of four elements (torch.optim.AdamW order: decoupled decay first, then the bias-corrected Adam step),
// shared by the fp32-moment kernel and the 8-bit one.  It works on the caller's arrays in one unrolled loop, the form in
// which nvcc contracts it into the same fused multiply-adds in both kernels.
__device__ __forceinline__ void adamw_update4(float (&p)[4], const float (&g)[4], float (&m)[4], float (&v)[4], float lr,
                                              float inv_bc1, float inv_sqrt_bc2, const OptHyper& h) {
  const float step_size = lr * inv_bc1;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    p[k] -= lr * h.weight_decay * p[k];                       // decoupled weight decay
    m[k] = m[k] + (1.0f - h.beta1) * (g[k] - m[k]);            // lerp(m, g, 1 - beta1)
    v[k] = h.beta2 * v[k] + (1.0f - h.beta2) * g[k] * g[k];
    const float denom = sqrtf(v[k]) * inv_sqrt_bc2 + h.eps;
    p[k] -= step_size * m[k] / denom;
  }
}

// The tail every pass shares: the EMA of the four updated parameters at i (omd = 1 - decay; < 0: no EMA update this
// step) and their bf16 operand copy.  Either pointer may be null.
__device__ __forceinline__ void ema_and_pack(float* ema, bf16* packed, long long i, const float (&p)[4], float omd) {
  if (ema != nullptr && omd >= 0.f) {
    float4 s4 = *reinterpret_cast<const float4*>(ema + i);
    s4.x -= omd * (s4.x - p[0]); s4.y -= omd * (s4.y - p[1]); s4.z -= omd * (s4.z - p[2]); s4.w -= omd * (s4.w - p[3]);
    *reinterpret_cast<float4*>(ema + i) = s4;
  }
  if (packed != nullptr) {
    uint2 u;
    u.x = pack_bf16(p[0], p[1]);
    u.y = pack_bf16(p[2], p[3]);
    *reinterpret_cast<uint2*>(packed + i) = u;
  }
}

// index of the last entry of a chunk whose first_block <= blk
template <class Chunk>
__device__ __forceinline__ int find_entry(const Chunk& chunk, long long blk) {
  int lo = 0, hi = chunk.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (chunk.e[mid].first_block <= blk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

template <OptAlgo kAlgo>
__global__ void __launch_bounds__(256)
opt_ema_pack_kernel(const __grid_constant__ OptChunk chunk, const float* __restrict__ scal, const OptHyper h) {
  pdl_enter();
  const long long blk = blockIdx.x;
  const OptEntry& e = chunk.e[find_entry(chunk, blk)];
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
    adamw_update4(p, g, m, v, lr, inv_bc1, inv_sqrt_bc2, h);
    *reinterpret_cast<float4*>(e.v + i) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    const float c_wd = scal[6];
#pragma unroll
    for (int k = 0; k < 4; ++k) lion_update(p[k], g[k], m[k], c_wd, lr, h);
  }
  *reinterpret_cast<float4*>(e.p + i) = make_float4(p[0], p[1], p[2], p[3]);
  *reinterpret_cast<float4*>(e.m + i) = make_float4(m[0], m[1], m[2], m[3]);
  ema_and_pack(e.ema, e.packed, i, p, omd);
}

// ---------------------------------------------------------------------------------------------- 8-bit block-wise AdamW
// One table entry of the 8-bit pass: the moments are uint8 codes (state1: m against the signed map, state2: v against the
// unsigned map) with one fp32 absmax per 256-element block; blocks start at element 0 of the tensor, the last one may be
// partial.
struct Opt8Entry {
  float* p;
  const float* g;
  uint8_t* state1;
  uint8_t* state2;
  float* ema;        // nullable
  bf16* packed;      // nullable
  long long numel;   // multiple of 4
  long long first_block;
  float* absmax1;    // ceil(numel / 256)
  float* absmax2;
};

constexpr int kQBlock = 256;                       // elements per quantisation block: one warp, 8 per lane
constexpr int kOpt8WarpsPerCta = 8;
constexpr int kOpt8Passes = 2;                     // a CTA covers 2 x 8 blocks (4096 elements): one map staging per 4096
constexpr int kOpt8CtaElems = kQBlock * kOpt8WarpsPerCta * kOpt8Passes;
// The encoder's first guess: |x| falls in one of kBuckets buckets, its exponent and top 5 mantissa bits from 2^-24 up
// (bucket 0 also holds everything below, the last one 1.0).  Per bucket a byte table gives a code no larger than that of
// any x in it: #{k : M[k] < lowest x of the bucket}.  From there a forward neighbour compare reaches #{k : M[k] < x};
// it takes at most 2 steps for the signed map and 3 for the unsigned one (tests/test_adamw8bit_cpu.py).
constexpr int kBuckets = 769;
constexpr int kBucketBase = 103 << 5;              // (bits of 2^-24) >> 18
constexpr int kStartBytes = 784;                   // kBuckets rounded up to 16
// [Q1 | Q2 | M1 (255 used) | M2 (255 used)] as floats, then three byte tables: signed map for x >= 0, signed map for
// x < 0, unsigned map
constexpr int kMapFloats = 4 * 256 + 3 * kStartBytes / 4;

struct Opt8Chunk {
  Opt8Entry e[kOptChunk];
  int n;
};
// the 8-bit kernel's arguments (chunk, scalars and maps pointers, hyper-parameters) stay under the 4 KB limit
static_assert(sizeof(Opt8Chunk) + 2 * sizeof(void*) + sizeof(OptHyper) <= 4096, "8-bit table chunk over 4 KB");

// the code of x: #{k : M[k] < x} over the 255 increasing midpoints (= searchsorted(M, x, side="left")); ties go to the
// lower code.  The bucket table's start is a lower bound of the code, so the forward compare ends on it exactly.
__device__ __forceinline__ uint32_t quantize(const float* __restrict__ mid, const uint8_t* __restrict__ start_pos,
                                             const uint8_t* __restrict__ start_neg, float x) {
  const uint32_t u = __float_as_uint(x);
  const int b = min(max(static_cast<int>((u & 0x7fffffffu) >> 18) - kBucketBase, 0), kBuckets - 1);
  uint32_t k = (u >> 31 ? start_neg : start_pos)[b];
  while (k < 255 && mid[k] < x) ++k;
  return k;
}

__device__ __forceinline__ float warp_max(float x) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
  return x;
}

// One warp per 256-element block, 8 elements per lane in two float4 halves (lane * 4 and 128 + lane * 4), so the block's
// absmax is a warp reduction.  A lane past the end of a partial block loads nothing and contributes 0 to both maxima; a
// warp whose block starts past the end of the tensor has nothing to do.
__global__ void __launch_bounds__(256)
adamw8bit_kernel(const __grid_constant__ Opt8Chunk chunk, const float* __restrict__ scal,
                 const float* __restrict__ maps, const OptHyper h) {
  __shared__ __align__(16) float smap[kMapFloats];
  pdl_enter();
  for (int j = threadIdx.x; j < kMapFloats / 4; j += blockDim.x)
    reinterpret_cast<float4*>(smap)[j] = reinterpret_cast<const float4*>(maps)[j];
  __syncthreads();
  const float* Q1 = smap;
  const float* Q2 = smap + 256;
  const float* M1 = smap + 512;
  const float* M2 = smap + 768;
  const uint8_t* S1p = reinterpret_cast<const uint8_t*>(smap + 1024);
  const uint8_t* S1n = S1p + kStartBytes;
  const uint8_t* S2 = S1n + kStartBytes;  // v >= 0: one table (-0 starts at code 0 from either)
  const long long blk = blockIdx.x;
  const Opt8Entry& e = chunk.e[find_entry(chunk, blk)];
  const float lr = scal[3], omd = scal[4], inv_bc1 = scal[1], inv_sqrt_bc2 = scal[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int pass = 0; pass < kOpt8Passes; ++pass) {
    const long long qb = (blk - e.first_block) * (kOpt8WarpsPerCta * kOpt8Passes) + pass * kOpt8WarpsPerCta + warp;
    const long long base = qb * kQBlock;
    if (base >= e.numel) break;  // warp-uniform
    float p[2][4], m[2][4], v[2][4];
    bool ok[2];
    float amax1 = 0.f, amax2 = 0.f;
#pragma unroll
    for (int hlf = 0; hlf < 2; ++hlf) {
      const long long i = base + hlf * 128 + lane * 4;
      ok[hlf] = i < e.numel;
      if (!ok[hlf]) continue;
      const float4 p4 = *reinterpret_cast<const float4*>(e.p + i);
      const float4 g4 = *reinterpret_cast<const float4*>(e.g + i);
      const uchar4 c1 = *reinterpret_cast<const uchar4*>(e.state1 + i);
      const uchar4 c2 = *reinterpret_cast<const uchar4*>(e.state2 + i);
      const float a1 = e.absmax1[qb], a2 = e.absmax2[qb];
      const float g[4] = {g4.x, g4.y, g4.z, g4.w};
      const uint8_t k1[4] = {c1.x, c1.y, c1.z, c1.w}, k2[4] = {c2.x, c2.y, c2.z, c2.w};
      p[hlf][0] = p4.x; p[hlf][1] = p4.y; p[hlf][2] = p4.z; p[hlf][3] = p4.w;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        m[hlf][k] = __fmul_rn(Q1[k1[k]], a1);  // decode: one fp32 product each
        v[hlf][k] = __fmul_rn(Q2[k2[k]], a2);
      }
      adamw_update4(p[hlf], g, m[hlf], v[hlf], lr, inv_bc1, inv_sqrt_bc2, h);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        amax1 = fmaxf(amax1, fabsf(m[hlf][k]));
        amax2 = fmaxf(amax2, v[hlf][k]);
      }
      *reinterpret_cast<float4*>(e.p + i) = make_float4(p[hlf][0], p[hlf][1], p[hlf][2], p[hlf][3]);
      ema_and_pack(e.ema, e.packed, i, p[hlf], omd);
    }
    amax1 = warp_max(amax1);  // every lane of the warp takes part, past the end of the tensor or not
    amax2 = warp_max(amax2);
    if (lane == 0) {
      e.absmax1[qb] = amax1;
      e.absmax2[qb] = amax2;
    }
#pragma unroll
    for (int hlf = 0; hlf < 2; ++hlf) {
      if (!ok[hlf]) continue;
      const long long i = base + hlf * 128 + lane * 4;
      uint32_t w1 = 0, w2 = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float x1 = amax1 > 0.f ? __fdiv_rn(m[hlf][k], amax1) : 0.f;
        const float x2 = amax2 > 0.f ? __fdiv_rn(v[hlf][k], amax2) : 0.f;
        w1 |= quantize(M1, S1p, S1n, x1) << (8 * k);
        w2 |= quantize(M2, S2, S2, x2) << (8 * k);
      }
      *reinterpret_cast<uint32_t*>(e.state1 + i) = w1;
      *reinterpret_cast<uint32_t*>(e.state2 + i) = w2;
    }
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

int opt_prepare(const char* what, float* scal_dev, long long* step_dev, const float* lr_dev, float lr_host,
                const OptHyper& h, cudaStream_t s) {
  pdl_launch(1, 32, 0, s)(opt_prepare_kernel, scal_dev, step_dev, lr_dev, lr_host, h);
  return check_launch(what);
}

// one update launch per chunk of kOptChunk entries; a CTA covers cta_elems elements of one entry.  launch(chunk, blocks)
// enqueues the kernel.
template <class Chunk, class Entry, class Launch>
int opt_chunks(const char* what, const Entry* all, int n_entries, long long cta_elems, Launch launch) {
  for (int base = 0; base < n_entries; base += kOptChunk) {
    Chunk chunk;
    chunk.n = n_entries - base < kOptChunk ? n_entries - base : kOptChunk;
    long long blocks = 0;
    for (int i = 0; i < chunk.n; ++i) {
      chunk.e[i] = all[base + i];
      if (chunk.e[i].numel % 4 != 0 || chunk.e[i].numel <= 0) {
        set_last_error("%s: numel must be a positive multiple of 4", what);
        return MUSE_ERR_INVALID;
      }
      chunk.e[i].first_block = blocks;
      blocks += (chunk.e[i].numel + cta_elems - 1) / cta_elems;
    }
    launch(chunk, blocks);
    const int rc = check_launch(what);
    if (rc) return rc;
  }
  return MUSE_OK;
}

template <OptAlgo kAlgo>
int opt_launch(const char* what, const OptEntry* all, int n_entries, const float* scal_dev, const OptHyper& h,
               cudaStream_t s) {
  return opt_chunks<OptChunk>(what, all, n_entries, 1024, [&](const OptChunk& chunk, long long blocks) {
    pdl_launch(static_cast<unsigned>(blocks), 256, 0, s)(opt_ema_pack_kernel<kAlgo>, chunk, scal_dev, h);
  });
}

// the prepare launch, then one update launch per chunk of kOptChunk table entries
template <OptAlgo kAlgo>
int opt_step(const char* what, const void* entries_host, int n_entries, float* scal_dev, long long* step_dev,
             const float* lr_dev, float lr_host, const OptHyper& h, cudaStream_t s) {
  if (n_entries <= 0) return MUSE_OK;
  const int rc = opt_prepare(what, scal_dev, step_dev, lr_dev, lr_host, h, s);
  if (rc) return rc;
  return opt_launch<kAlgo>(what, reinterpret_cast<const OptEntry*>(entries_host), n_entries, scal_dev, h, s);
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

// AdamW with block-wise 8-bit moments.  entries_host: HOST array of n_entries {p, g, m, v, ema, packed, numel, unused,
// absmax1, absmax2} (10 x int64).  absmax1 == NULL: a 32-bit entry (m, v fp32), updated by muse_adamw_ema_step's kernel;
// else m / v are uint8 codes and absmax1 / absmax2 hold ceil(numel / 256) floats.  maps_dev: kMapFloats floats, laid out
// as above (built by open_muse_b200.optim).  Counters, scalars and EMA arguments as muse_adamw_ema_step: one prepare launch
// per call, whichever entries it holds.
int muse_adamw8bit_ema_step(const void* entries_host, int n_entries, const float* maps_dev, float* scal_dev,
                            long long* step_dev, const float* lr_dev, float lr_host, float beta1, float beta2, float eps,
                            float weight_decay, int ema_enabled, float ema_decay, float ema_min_decay,
                            int ema_update_after_step, int ema_update_every, int ema_use_warmup, float ema_inv_gamma,
                            float ema_power, void* stream) {
  const char* what = "adamw8bit_ema_step";
  if (n_entries <= 0) return MUSE_OK;
  if (maps_dev == nullptr) {
    set_last_error("%s: maps_dev is null", what);
    return MUSE_ERR_INVALID;
  }
  OptHyper h = make_hyper(beta1, beta2, ema_enabled, ema_decay, ema_min_decay, ema_update_after_step, ema_update_every,
                          ema_use_warmup, ema_inv_gamma, ema_power);
  h.eps = eps; h.weight_decay = weight_decay;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const Opt8Entry* rows = reinterpret_cast<const Opt8Entry*>(entries_host);
  std::vector<OptEntry> fp32;
  std::vector<Opt8Entry> q8;
  for (int i = 0; i < n_entries; ++i) {
    const Opt8Entry& r = rows[i];
    if (r.absmax1 == nullptr) {
      fp32.push_back(OptEntry{r.p, r.g, reinterpret_cast<float*>(r.state1), reinterpret_cast<float*>(r.state2), r.ema,
                              r.packed, r.numel, 0});
    } else if (r.absmax2 == nullptr) {
      set_last_error("%s: entry %d has absmax1 but no absmax2", what, i);
      return MUSE_ERR_INVALID;
    } else {
      q8.push_back(r);
    }
  }
  int rc = opt_prepare(what, scal_dev, step_dev, lr_dev, lr_host, h, s);
  if (rc) return rc;
  rc = opt_launch<OptAlgo::kAdamW>(what, fp32.data(), static_cast<int>(fp32.size()), scal_dev, h, s);
  if (rc) return rc;
  return opt_chunks<Opt8Chunk>(what, q8.data(), static_cast<int>(q8.size()), kOpt8CtaElems,
                               [&](const Opt8Chunk& chunk, long long blocks) {
    pdl_launch(static_cast<unsigned>(blocks), kOpt8WarpsPerCta * 32, 0, s)(adamw8bit_kernel, chunk, scal_dev, maps_dev, h);
  });
}

}  // extern "C"
