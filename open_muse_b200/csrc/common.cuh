// Shared device helpers for the non-GEMM kernels (bf16 pack/unpack, warp reductions, GELU).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#define MUSE_OK 0
#define MUSE_ERR_INVALID 1
#define MUSE_ERR_CUDA 2
#define MUSE_ERR_UNSUPPORTED 3

namespace muse {

typedef __nv_bfloat16 bf16;

// Error plumbing: kernels are launched asynchronously; launch-configuration errors are
// caught with cudaGetLastError() right after the launch and mapped to MUSE_ERR_CUDA.
void set_last_error(const char* fmt, ...);
int check_launch(const char* what);

// ---- Programmatic dependent launch (PDL) ---------------------------------------------------------------------------
// The hot paths are chains of 300 - 900 short kernels on one stream (a train step, a captured generate2 loop); a plain
// stream edge costs a full drain + launch between two kernels.  Every kernel of this library therefore (i) tells the
// hardware right away that its successor may be scheduled (griddepcontrol.launch_dependents: the successor's CTAs take
// the SM slots that free up while the tail of this grid drains, and run their prologue -- barrier init,
// tensor-map prefetch), and (ii) blocks in griddepcontrol.wait before its first global-memory access until the
// predecessor grid has COMPLETED and its writes are visible.  Correctness never depends on the trigger: with wait in
// front of every global access (reads AND writes, so there is no WAR hazard either) the order of memory effects is the
// stream order; completion is transitive because a grid cannot complete before its own wait returned.  Both
// instructions are no-ops in a grid launched without the attribute (ATen kernels in between are ordinary full edges).
// Host side: pdl_launch(grid, block, smem, stream)(kernel, args...) replaces kernel<<<...>>>(args...) and adds
// cudaLaunchAttributeProgrammaticStreamSerialization when muse_set_pdl(1) is in effect; stream capture records the edge
// as a programmatic dependency, so the captured step / decode graphs keep the overlap.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_enter() {
  pdl_trigger();
  pdl_wait();
}

bool pdl_enabled();  // capi.cu (muse_set_pdl / MUSE_B200_PDL)

struct PdlLaunch {
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr;
  template <typename... KArgs, typename... Args>
  void operator()(void (*kernel)(KArgs...), Args&&... args) {
    if (pdl_enabled()) {
      attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attr.val.programmaticStreamSerializationAllowed = 1;
      cfg.attrs = &attr;
      cfg.numAttrs = 1;
    }
    cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);  // errors surface through check_launch()
  }
};
inline PdlLaunch pdl_launch(dim3 grid, dim3 block, size_t smem, cudaStream_t stream) {
  PdlLaunch l{};
  l.cfg.gridDim = grid;
  l.cfg.blockDim = block;
  l.cfg.dynamicSmemBytes = smem;
  l.cfg.stream = stream;
  return l;
}

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
__device__ __forceinline__ float bf16_round(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

// Exact (erf-based) GELU, as F.gelu default (reference: muse/modeling_transformer.py:789,981), value and
// derivative from ONE exponential: erf through Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, i.e. fp32 ulp level for
// the CDF), whose exp(-z^2) with z = x/sqrt(2) is also the Gaussian pdf factor exp(-x^2/2) of the derivative.
// The elementwise GLU / GELU passes are otherwise limited by libdevice erff (~3 calls per element in backward).
__device__ __forceinline__ void gelu_eval(float x, float& val, float& grad) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));  // 1 MUFU, ~1 ulp
  const float e = __expf(-z * z);
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float erf_abs = fmaf(-p * t, e, 1.0f);
  const float cdf = 0.5f * (1.0f + copysignf(erf_abs, x));
  val = x * cdf;
  grad = fmaf(x * 0.39894228040143267794f, e, cdf);
}
__device__ __forceinline__ float gelu_f(float x) {
  float v, g;
  gelu_eval(x, v, g);
  return v;
}
__device__ __forceinline__ float gelu_grad_f(float x) {
  float v, g;
  gelu_eval(x, v, g);
  return g;
}

// 8 consecutive elements starting at p (16B for bf16, 32B for fp32) -> 8 floats.
__device__ __forceinline__ void load8(const bf16* p, float (&v)[8]) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  float4 a = *reinterpret_cast<const float4*>(p);
  float4 b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void store8(bf16* p, const float (&v)[8]) {
  uint4 u;
  u.x = pack_bf16(v[0], v[1]); u.y = pack_bf16(v[2], v[3]);
  u.z = pack_bf16(v[4], v[5]); u.w = pack_bf16(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ void store8(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

}  // namespace muse
