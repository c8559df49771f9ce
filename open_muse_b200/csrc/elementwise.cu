// HBM-bound elementwise / gather kernels of the transformer step:
//   * multi-tensor fp32 -> bf16 weight packing (one launch for all Linear weights of a model)
//   * token + position embedding gather (muse/modeling_transformer.py:942-957) and its backward
//   * the FFN activations, one templated pass: GLU gelu(a) * b (muse/modeling_transformer.py:789-792) and the ungated
//     tanh-GELU of FusedGeLUFeedForward (muse/modeling_transformer_v2.py:954-996), forward / backward; their e4m3 form (a
//     warp per row, which the row's scale needs) writes the wo operand of the FP8 GEMM
//   * per-row e4m3 quantization of the bf16 weight operands of the FP8 GEMM
//   * plain fp32 -> bf16 cast (gradient of the residual stream entering a dgrad GEMM)
//   * nn.Dropout of the embedding output and of the FFN hidden state (keep bits of philox.cuh) and its backward
#include "common.cuh"
#include "philox.cuh"
#include "row_norm.cuh"

namespace muse {
namespace {

// ---------------------------------------------------------------- multi-tensor pack
// table[i] = {src fp32 ptr, dst bf16 ptr, numel(multiple of 4), first 1024-element block index}
struct PackEntry {
  const float* src;
  bf16* dst;
  long long numel;
  long long first_block;
};

__global__ void __launch_bounds__(256) pack_bf16_kernel(const PackEntry* __restrict__ table, int n_entries) {
  pdl_enter();
  const long long blk = blockIdx.x;
  int lo = 0, hi = n_entries - 1;
  while (lo < hi) {  // last entry with first_block <= blk
    const int mid = (lo + hi + 1) >> 1;
    if (table[mid].first_block <= blk) lo = mid; else hi = mid - 1;
  }
  const PackEntry e = table[lo];
  const long long i = ((blk - e.first_block) * 256 + threadIdx.x) * 4;
  if (i < e.numel) {
    const float4 v = *reinterpret_cast<const float4*>(e.src + i);
    uint2 u;
    u.x = pack_bf16(v.x, v.y);
    u.y = pack_bf16(v.z, v.w);
    *reinterpret_cast<uint2*>(e.dst + i) = u;
  }
}

__global__ void __launch_bounds__(256) cast_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long n8) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i < n8) {
    float v[8];
    load8(src + i * 8, v);
    store8(dst + i * 8, v);
  }
}

// ---------------------------------------------------------------- embedding
__global__ void __launch_bounds__(128)
embed_fwd_kernel(const long long* __restrict__ ids, const float* __restrict__ word, const float* __restrict__ pos,
                 float* __restrict__ out, int tokens, int S, int H, int vocab) {
  pdl_enter();
  const int t = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (t >= tokens) return;
  const int lane = threadIdx.x & 31;
  long long id = ids[t];
  if (id < 0 || id >= vocab) id = 0;  // torch raises on OOB ids; host validates, device stays in-bounds
  const float* wr = word + id * H;
  const float* pr = pos ? pos + static_cast<size_t>(t % S) * H : nullptr;  // pos == null: plain gather (ConvEmbed of v2)
  float* o = out + static_cast<size_t>(t) * H;
  for (int c = lane * 4; c < H; c += 128) {
    const float4 a = *reinterpret_cast<const float4*>(wr + c);
    const float4 b = pr ? *reinterpret_cast<const float4*>(pr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(o + c) = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
}

// dword[ids[t]] += dx[t].  Roughly half of the tokens of a training batch are the mask token (id = vocab - 1 in every
// reference config, modeling_transformer.py:1128), so plain atomics serialise T/2 adds on one row.  Each warp therefore
// keeps the hot row's contribution of its 8 tokens in registers, the CTA folds its 8 warps in shared memory, and one
// atomic per column and CTA reaches global memory; all other ids (spread over ~1000 rows) use vector atomics directly.
constexpr int kEmbTokPerWarp = 8;
template <int CH>  // CH float4 chunks per lane: H = CH * 128
__global__ void __launch_bounds__(256)
embed_bwd_word_kernel(const long long* __restrict__ ids, const float* __restrict__ dx, float* __restrict__ dword,
                      int tokens, int H, int vocab, int hot_id) {
  pdl_enter();
  __shared__ float s_hot[CH * 128];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < CH * 128; i += 256) s_hot[i] = 0.f;
  __syncthreads();
  float4 acc[CH];
#pragma unroll
  for (int c = 0; c < CH; ++c) acc[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  bool any_hot = false;
  const int t0 = (blockIdx.x * 8 + warp) * kEmbTokPerWarp;
  for (int k = 0; k < kEmbTokPerWarp; ++k) {
    const int t = t0 + k;
    if (t >= tokens) break;
    const long long id = ids[t];
    if (id < 0 || id >= vocab) continue;
    const float* g = dx + static_cast<size_t>(t) * H;
    if (id == hot_id) {
      any_hot = true;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const float4 v = *reinterpret_cast<const float4*>(g + c * 128 + lane * 4);
        acc[c].x += v.x; acc[c].y += v.y; acc[c].z += v.z; acc[c].w += v.w;
      }
    } else {
      float* d = dword + id * H;
#pragma unroll
      for (int c = 0; c < CH; ++c)
        atomicAdd(reinterpret_cast<float4*>(d + c * 128 + lane * 4), *reinterpret_cast<const float4*>(g + c * 128 + lane * 4));
    }
  }
  if (any_hot) {
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      float* h = s_hot + c * 128 + lane * 4;
      atomicAdd(h + 0, acc[c].x); atomicAdd(h + 1, acc[c].y); atomicAdd(h + 2, acc[c].z); atomicAdd(h + 3, acc[c].w);
    }
  }
  __syncthreads();
  if (hot_id >= 0 && hot_id < vocab) {
    float* d = dword + static_cast<size_t>(hot_id) * H;
    for (int i = threadIdx.x; i < CH * 128; i += 256) {
      const float v = s_hot[i];
      if (v != 0.f) atomicAdd(d + i, v);
    }
  }
}

// generic H (any multiple of 4): one warp per token, vector atomics
__global__ void __launch_bounds__(128)
embed_bwd_word_generic_kernel(const long long* __restrict__ ids, const float* __restrict__ dx, float* __restrict__ dword,
                              int tokens, int H, int vocab) {
  pdl_enter();
  const int t = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (t >= tokens) return;
  const int lane = threadIdx.x & 31;
  long long id = ids[t];
  if (id < 0 || id >= vocab) return;
  const float* g = dx + static_cast<size_t>(t) * H;
  float* d = dword + id * H;
  for (int c = lane * 4; c < H; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(g + c);
    atomicAdd(reinterpret_cast<float4*>(d + c), v);
  }
}

// dpos[s] += sum_b dx[b, s]; block (s, column chunk of 128 floats), threads stride over batch
__global__ void __launch_bounds__(128)
embed_bwd_pos_kernel(const float* __restrict__ dx, float* __restrict__ dpos, int B, int S, int H) {
  pdl_enter();
  const int s = blockIdx.x;
  const int c = blockIdx.y * 128 + threadIdx.x;
  if (c >= H) return;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) acc += dx[(static_cast<size_t>(b) * S + s) * H + c];
  dpos[static_cast<size_t>(s) * H + c] = acc;  // fixed summation order, plain store: reproducible, no zero fill
}

// ---------------------------------------------------------------- reproducible word-embedding gradient
// dword[v] = sum of dx[t] over the tokens t with ids[t] == v, summed in ascending t whatever the launch order:
// the host passes the stable sort permutation of the ids (`order`) and the segment bounds (`bounds[v]` = first sorted
// position of id v); segments are cut into chunks of kSegChunk tokens, every chunk is summed by one CTA (four thread
// groups take a quarter each, rows in order, then the quarters are added in order), single-chunk segments are stored
// straight to dword[v], longer ones go through per-chunk partial rows that a second kernel adds in chunk order.
constexpr int kSegChunk = 256;

__global__ void __launch_bounds__(1024)
embed_seg_plan_kernel(const long long* __restrict__ bounds, int* __restrict__ chunk_off, int vocab) {
  pdl_enter();
  __shared__ int s_part[1024];
  const int per = ceil_div(vocab, 1024);
  const int v0 = threadIdx.x * per;
  int sum = 0;
  for (int v = v0; v < min(vocab, v0 + per); ++v)
    sum += static_cast<int>((bounds[v + 1] - bounds[v] + kSegChunk - 1) / kSegChunk);
  s_part[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int i = 0; i < 1024; ++i) { const int t = s_part[i]; s_part[i] = run; run += t; }
    chunk_off[vocab] = run;
  }
  __syncthreads();
  int run = s_part[threadIdx.x];
  for (int v = v0; v < min(vocab, v0 + per); ++v) {
    chunk_off[v] = run;
    run += static_cast<int>((bounds[v + 1] - bounds[v] + kSegChunk - 1) / kSegChunk);
  }
}

// ordered sum of `n` rows of H floats: row(i) gives the row pointer; 4 groups x ncol threads, result valid in group 0
template <typename RowFn>
__device__ __forceinline__ void ordered_rows_sum(RowFn row, int n, int H, float* s_q, float* out_row) {
  const int ncol = blockDim.x >> 2;
  const int grp = threadIdx.x / ncol, tx = threadIdx.x % ncol;
  const int per = (n + 3) >> 2;
  const int i0 = grp * per, i1 = min(n, i0 + per);
  for (int c = tx * 4; c < H; c += ncol * 4) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
    for (int i = i0; i < i1; ++i) {
      const float4 v = *reinterpret_cast<const float4*>(row(i) + c);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    *reinterpret_cast<float4*>(s_q + static_cast<size_t>(grp) * H + c) = acc;
  }
  __syncthreads();
  if (grp == 0) {
    for (int c = tx * 4; c < H; c += ncol * 4) {
      float4 a = *reinterpret_cast<const float4*>(s_q + c);
#pragma unroll
      for (int g = 1; g < 4; ++g) {
        const float4 b = *reinterpret_cast<const float4*>(s_q + static_cast<size_t>(g) * H + c);
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
      }
      *reinterpret_cast<float4*>(out_row + c) = a;
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(512) embed_seg_chunk_kernel(const long long* __restrict__ order, const long long* __restrict__ bounds,
                                       const int* __restrict__ chunk_off, const float* __restrict__ dx,
                                       float* __restrict__ dword, float* __restrict__ ws, int H, int vocab) {
  pdl_enter();
  extern __shared__ __align__(16) float s_q[];  // [4][H]
  const int g = blockIdx.x;
  if (g >= chunk_off[vocab]) return;
  int lo = 0, hi = vocab - 1;
  while (lo < hi) {  // last v with chunk_off[v] <= g (empty segments share their successor's offset and lose the tie)
    const int mid = (lo + hi + 1) >> 1;
    if (chunk_off[mid] <= g) lo = mid; else hi = mid - 1;
  }
  const int v = lo;
  const int j = g - chunk_off[v];
  const long long p0 = bounds[v] + static_cast<long long>(j) * kSegChunk;
  const int n = static_cast<int>(min(static_cast<long long>(kSegChunk), bounds[v + 1] - p0));
  const bool single = (chunk_off[v + 1] - chunk_off[v]) == 1;
  float* out = single ? dword + static_cast<size_t>(v) * H : ws + static_cast<size_t>(g) * H;
  ordered_rows_sum([&](int i) { return dx + static_cast<size_t>(order[p0 + i]) * H; }, n, H, s_q, out);
}

__global__ void __launch_bounds__(512) embed_seg_final_kernel(const int* __restrict__ chunk_off, const float* __restrict__ ws,
                                       float* __restrict__ dword, int H, int vocab) {
  pdl_enter();
  extern __shared__ __align__(16) float s_q[];
  const int v = blockIdx.x;
  const int c0 = chunk_off[v], nc = chunk_off[v + 1] - c0;
  if (nc == 1) return;  // stored by the chunk kernel
  float* out = dword + static_cast<size_t>(v) * H;
  if (nc == 0) {
    for (int c = threadIdx.x * 4; c < H; c += blockDim.x * 4) *reinterpret_cast<float4*>(out + c) = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  ordered_rows_sum([&](int i) { return ws + static_cast<size_t>(c0 + i) * H; }, nc, H, s_q, out);
}

// ---------------------------------------------------------------- FFN activation: GLU / tanh-GELU
// GATED (GLUFeedForward): ab [rows, 2*I] bf16 (a = cols [0,I), b = cols [I,2I)); out [rows, I] bf16 = bf16(gelu(a)) * b.
// Rounding points follow the reference under bf16 autocast: gelu(a) is rounded to bf16 before the product.
// !GATED (FusedGeLUFeedForward, muse/modeling_transformer_v2.py:954-996): ab is the pre-activation [rows, I] bf16 and
// out = gelu_tanh(pre); the reference's dropout module of that block is never applied, so there is no DROP variant.
// DROP: FeedForward.dropout (:797) fused -- the forward draws the chunk's keep byte (philox.cuh elementwise mapping), writes
// the dropped product and the byte (the last chunk of a row also zeroes the pad bytes of the row's last word); the
// backward scales dout by the stored byte as it reads it.

// F.gelu(x, approximate="tanh") and its derivative with torch's formula and constants (ATen GeluKernel), accurate tanhf
constexpr float kGeluTanhBeta = 0.7978845608028654f;  // sqrt(2 / pi)
constexpr float kGeluTanhKappa = 0.044715f;
__device__ __forceinline__ float gelu_tanh_f(float x) {
  const float inner = kGeluTanhBeta * (x + kGeluTanhKappa * (x * x * x));
  return 0.5f * x * (1.f + tanhf(inner));
}
__device__ __forceinline__ float gelu_tanh_grad_f(float x) {
  const float x_sq = x * x;
  const float t = tanhf(kGeluTanhBeta * (x + kGeluTanhKappa * (x_sq * x)));
  const float left = 0.5f * x, right = 1.f + t;
  return 0.5f * right + left * (1.f - t * t) * kGeluTanhBeta * (1.f + 3.f * kGeluTanhKappa * x_sq);
}

template <bool GATED, bool DROP>
__global__ void __launch_bounds__(256)
ffn_act_fwd_kernel(const bf16* __restrict__ ab, bf16* __restrict__ out, long long rows, int I, const philox::ElemDrop dr) {
  static_assert(GATED || !DROP, "the tanh-GELU pass has no dropout");
  pdl_enter();
  const int chunks = I / 8;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= rows * chunks) return;
  const long long r = idx / chunks;
  const int c = static_cast<int>(idx % chunks) * 8;
  float a[8], o[8];
  if constexpr (GATED) {
    float b[8];
    load8(ab + r * 2 * I + c, a);
    load8(ab + r * 2 * I + I + c, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = bf16_round(gelu_f(a[j])) * b[j];
  } else {
    load8(ab + r * I + c, a);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = gelu_tanh_f(a[j]);
  }
  if constexpr (DROP) {
    const uint32_t kb = philox::elem_keep8(*dr.seed, dr.site, static_cast<uint32_t>(r), c / 8, dr.thresh);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] *= philox::keep_z(kb, j, dr.scale);
    uint8_t* br = dr.bits + r * dr.row_bytes;
    br[c / 8] = static_cast<uint8_t>(kb);
    if (c / 8 == chunks - 1)
      for (int k = chunks; k < dr.row_bytes; ++k) br[k] = 0;
  }
  store8(out + r * I + c, o);
}

// GATED: dab = [d a | d b]; !GATED: dab = dpre [rows, I] = dout * gelu_tanh'(pre)
template <bool GATED, bool DROP>
__global__ void __launch_bounds__(256)
ffn_act_bwd_kernel(const bf16* __restrict__ ab, const bf16* __restrict__ dout, bf16* __restrict__ dab, long long rows, int I,
                   const philox::ElemDrop dr) {
  static_assert(GATED || !DROP, "the tanh-GELU pass has no dropout");
  pdl_enter();
  const int chunks = I / 8;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= rows * chunks) return;
  const long long r = idx / chunks;
  const int c = static_cast<int>(idx % chunks) * 8;
  if constexpr (GATED) {
    float a[8], b[8], d[8], da[8], db[8];
    load8(ab + r * 2 * I + c, a);
    load8(ab + r * 2 * I + I + c, b);
    load8(dout + r * I + c, d);
    if constexpr (DROP) {
      const uint32_t kb = dr.bits[r * dr.row_bytes + c / 8];
#pragma unroll
      for (int j = 0; j < 8; ++j) d[j] *= philox::keep_z(kb, j, dr.scale);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float gv, gg;
      gelu_eval(a[j], gv, gg);
      da[j] = d[j] * b[j] * gg;
      db[j] = d[j] * bf16_round(gv);
    }
    store8(dab + r * 2 * I + c, da);
    store8(dab + r * 2 * I + I + c, db);
  } else {
    float a[8], d[8];
    load8(ab + r * I + c, a);
    load8(dout + r * I + c, d);
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] *= gelu_tanh_grad_f(a[j]);
    store8(dab + r * I + c, d);
  }
}

// ---------------------------------------------------------------- dropout (elementwise sites)
// One thread per 8 columns of a row = one Philox call = one byte of the row's keep-bit words (little-endian: byte k of
// the row is bits 8 (k % 4) .. of word k / 4, i.e. columns 8 k .. 8 k + 7).  Threads past the last column zero the pad
// bytes of the row's last word.  y may alias x.
template <typename T>
__global__ void __launch_bounds__(256)
dropout_fwd_kernel(const T* x, T* y, uint8_t* __restrict__ bits, const unsigned long long* __restrict__ seed,
                   uint32_t site, uint32_t t, float scale, long long rows, int cols, int row_bytes) {
  pdl_enter();
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= rows * row_bytes) return;
  const long long r = idx / row_bytes;
  const int k = static_cast<int>(idx % row_bytes);
  if (8 * k >= cols) {
    bits[idx] = 0;
    return;
  }
  const uint32_t kb = philox::elem_keep8(*seed, site, static_cast<uint32_t>(r), static_cast<uint32_t>(k), t);
  float v[8];
  load8(x + r * cols + 8 * k, v);
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = ((kb >> j) & 1u) ? v[j] * scale : 0.f;
  store8(y + r * cols + 8 * k, v);
  bits[idx] = static_cast<uint8_t>(kb);
}

// dx = dy * keep * scale; dx may alias dy
template <typename T>
__global__ void __launch_bounds__(256)
dropout_bwd_kernel(const T* dy, T* dx, const uint8_t* __restrict__ bits, float scale, long long rows, int cols,
                   int row_bytes) {
  pdl_enter();
  const int chunks = cols / 8;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= rows * chunks) return;
  const long long r = idx / chunks;
  const int k = static_cast<int>(idx % chunks);
  const uint32_t kb = bits[r * row_bytes + k];
  float v[8];
  load8(dy + r * cols + 8 * k, v);
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = ((kb >> j) & 1u) ? v[j] * scale : 0.f;
  store8(dx + r * cols + 8 * k, v);
}

// e4m3 form of the FFN activation: one warp per row holds the fp32 value the bf16 form rounds (GATED: gelu(a) * b,
// else gelu_tanh(pre)) as a register row, then stores it with row_store_e4m3.  ab bf16 [rows, 2I] (GATED) or [rows, I],
// q [rows, I] bytes, row_scale fp32 [rows].
constexpr int kGluRowWarps = 4;
template <bool GATED, int CH>
__global__ void __launch_bounds__(kGluRowWarps * 32)
ffn_act_fwd_e4m3_kernel(const bf16* __restrict__ ab, uint8_t* __restrict__ q, float* __restrict__ row_scale, long long rows,
                        int I) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const long long r = static_cast<long long>(blockIdx.x) * kGluRowWarps + (threadIdx.x >> 5);
  if (r >= rows) return;
  float v[CH][8];
  row_load(v, I, lane, [&](int col, float (&vc)[8]) {
    if constexpr (GATED) {
      float b[8];
      load8(ab + r * 2 * I + col, vc);
      load8(ab + r * 2 * I + I + col, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) vc[j] = bf16_round(gelu_f(vc[j])) * b[j];
    } else {
      load8(ab + r * I + col, vc);
#pragma unroll
      for (int j = 0; j < 8; ++j) vc[j] = gelu_tanh_f(vc[j]);
    }
  });
  row_store_e4m3(v, I, lane, q + r * I, row_scale + r);
}

// Per-row e4m3 quantization, one warp per row, 8 elements (16 bytes in, 8 bytes out) per lane and access: the row's
// amax over |x| first, then q = e4m3_rn_satfinite(x / s) on a second read of the row (from L1 / L2).
__global__ void __launch_bounds__(256)
quantize_rows_e4m3_kernel(const bf16* __restrict__ x, int ldx, uint8_t* __restrict__ q, int ldq, float* __restrict__ scale,
                          int rows, int K) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const bf16* xr = x + static_cast<size_t>(r) * ldx;
  float amax = 0.f;
  for (int k = lane * 8; k < K; k += 256) {
    float v[8];
    load8(xr + k, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(v[j]));
  }
  amax = warp_max(amax);
  const float s = amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f;
  if (lane == 0) scale[r] = s;
  uint8_t* qr = q + static_cast<size_t>(r) * ldq;
  for (int k = lane * 8; k < K; k += 256) {
    float v[8];
    load8(xr + k, v);
    uint32_t w[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float* e = &v[4 * h];
      const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(e[0], s), __fdiv_rn(e[1], s)), __NV_SATFINITE, __NV_E4M3);
      const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(e[2], s), __fdiv_rn(e[3], s)), __NV_SATFINITE, __NV_E4M3);
      w[h] = lo | (hi << 16);
    }
    *reinterpret_cast<uint2*>(qr + k) = make_uint2(w[0], w[1]);
  }
}

// ---------------------------------------------------------------- FFN activation launchers (GLU and tanh-GELU entry points)
template <bool GATED>
int ffn_act_fwd(const char* name, const void* ab, void* out, int out_dt, float* row_scale, unsigned int* bits,
                const unsigned long long* seed, int site, float p, long long rows, int I, cudaStream_t s) {
  if (I % 8 != 0) { set_last_error("%s: I must be a multiple of 8", name); return MUSE_ERR_INVALID; }
  if (bits != nullptr && seed == nullptr) { set_last_error("%s: dropout needs a seed", name); return MUSE_ERR_INVALID; }
  if (out_dt != 1 && out_dt != 2) { set_last_error("%s: out dtype code %d (bf16 = 1 or e4m3 = 2)", name, out_dt); return MUSE_ERR_INVALID; }
  if (out_dt == 2) {
    if (row_scale == nullptr || bits != nullptr || I > 4096) {
      set_last_error("%s: the e4m3 output needs row_scale, takes no dropout and I <= 4096 (I = %d)", name, I);
      return MUSE_ERR_INVALID;
    }
    if (rows <= 0) return MUSE_OK;
    const unsigned grid = static_cast<unsigned>(ceil_div_ll(rows, kGluRowWarps));
    with_row_chunks<1, 2, 4, 8, 12, 16>(I, [&](auto ch) {
      pdl_launch(grid, kGluRowWarps * 32, 0, s)(ffn_act_fwd_e4m3_kernel<GATED, decltype(ch)::value>,
                                                reinterpret_cast<const bf16*>(ab), reinterpret_cast<uint8_t*>(out), row_scale,
                                                rows, I);
    });
    return check_launch(name);
  }
  const long long n = rows * (I / 8);
  if (n <= 0) return MUSE_OK;
  const philox::ElemDrop dr = philox::elem_drop(bits, seed, site, p, I);
  if constexpr (GATED)
    pdl_launch(static_cast<unsigned>(ceil_div_ll(n, 256)), 256, 0, s)(bits ? ffn_act_fwd_kernel<true, true> : ffn_act_fwd_kernel<true, false>,
        reinterpret_cast<const bf16*>(ab), reinterpret_cast<bf16*>(out), rows, I, dr);
  else
    pdl_launch(static_cast<unsigned>(ceil_div_ll(n, 256)), 256, 0, s)(ffn_act_fwd_kernel<false, false>,
        reinterpret_cast<const bf16*>(ab), reinterpret_cast<bf16*>(out), rows, I, dr);
  return check_launch(name);
}

template <bool GATED>
int ffn_act_bwd(const char* name, const void* ab, const void* dout, const unsigned int* bits, float p, void* dab,
                long long rows, int I, cudaStream_t s) {
  if (I % 8 != 0) { set_last_error("%s: I must be a multiple of 8", name); return MUSE_ERR_INVALID; }
  const long long n = rows * (I / 8);
  if (n <= 0) return MUSE_OK;
  const philox::ElemDrop dr = philox::elem_drop(const_cast<unsigned int*>(bits), nullptr, 0, p, I);
  if constexpr (GATED)
    pdl_launch(static_cast<unsigned>(ceil_div_ll(n, 256)), 256, 0, s)(bits ? ffn_act_bwd_kernel<true, true> : ffn_act_bwd_kernel<true, false>,
        reinterpret_cast<const bf16*>(ab), reinterpret_cast<const bf16*>(dout), reinterpret_cast<bf16*>(dab), rows, I, dr);
  else
    pdl_launch(static_cast<unsigned>(ceil_div_ll(n, 256)), 256, 0, s)(ffn_act_bwd_kernel<false, false>,
        reinterpret_cast<const bf16*>(ab), reinterpret_cast<const bf16*>(dout), reinterpret_cast<bf16*>(dab), rows, I, dr);
  return check_launch(name);
}

}  // namespace
}  // namespace muse

using namespace muse;

extern "C" {

int muse_dropout_fwd(const void* x, void* y, int dtype, unsigned int* bits, const unsigned long long* seed, int site,
                     float p, long long rows, int cols, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (cols % 8 != 0) { set_last_error("dropout_fwd: cols=%d must be a multiple of 8", cols); return MUSE_ERR_INVALID; }
  if (bits == nullptr || seed == nullptr) { set_last_error("dropout_fwd: bits and seed are required"); return MUSE_ERR_INVALID; }
  const int row_bytes = 4 * ceil_div(cols, 32);
  const long long n = rows * row_bytes;
  if (n <= 0) return MUSE_OK;
  const uint32_t t = philox::threshold(p);
  const float scale = philox::keep_scale(t);
  uint8_t* b = reinterpret_cast<uint8_t*>(bits);
  const unsigned grid = static_cast<unsigned>(ceil_div_ll(n, 256));
  if (dtype == 0)
    pdl_launch(grid, 256, 0, s)(dropout_fwd_kernel<float>, reinterpret_cast<const float*>(x), reinterpret_cast<float*>(y), b,
                                seed, static_cast<uint32_t>(site), t, scale, rows, cols, row_bytes);
  else
    pdl_launch(grid, 256, 0, s)(dropout_fwd_kernel<bf16>, reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(y), b,
                                seed, static_cast<uint32_t>(site), t, scale, rows, cols, row_bytes);
  return check_launch("dropout_fwd");
}

int muse_dropout_bwd(const void* dy, void* dx, int dtype, const unsigned int* bits, float p, long long rows, int cols,
                     void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (cols % 8 != 0) { set_last_error("dropout_bwd: cols=%d must be a multiple of 8", cols); return MUSE_ERR_INVALID; }
  const long long n = rows * (cols / 8);
  if (n <= 0) return MUSE_OK;
  const int row_bytes = 4 * ceil_div(cols, 32);
  const float scale = philox::keep_scale(philox::threshold(p));
  const uint8_t* b = reinterpret_cast<const uint8_t*>(bits);
  const unsigned grid = static_cast<unsigned>(ceil_div_ll(n, 256));
  if (dtype == 0)
    pdl_launch(grid, 256, 0, s)(dropout_bwd_kernel<float>, reinterpret_cast<const float*>(dy), reinterpret_cast<float*>(dx), b,
                                scale, rows, cols, row_bytes);
  else
    pdl_launch(grid, 256, 0, s)(dropout_bwd_kernel<bf16>, reinterpret_cast<const bf16*>(dy), reinterpret_cast<bf16*>(dx), b,
                                scale, rows, cols, row_bytes);
  return check_launch("dropout_bwd");
}

int muse_pack_bf16(const void* table_dev, int n_entries, long long total_blocks, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n_entries <= 0 || total_blocks <= 0) return MUSE_OK;
  pdl_launch(static_cast<unsigned>(total_blocks), 256, 0, s)(pack_bf16_kernel, reinterpret_cast<const PackEntry*>(table_dev), n_entries);
  return check_launch("pack_bf16");
}

int muse_cast_bf16(const float* src, void* dst, long long n, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0) return MUSE_OK;
  if (n % 8 != 0) { set_last_error("cast_bf16: n=%lld must be a multiple of 8", n); return MUSE_ERR_INVALID; }
  const long long n8 = n / 8;
  pdl_launch(static_cast<unsigned>(ceil_div_ll(n8, 256)), 256, 0, s)(cast_bf16_kernel, src, reinterpret_cast<bf16*>(dst), n8);
  return check_launch("cast_bf16");
}

int muse_embed_fwd(const long long* ids, const float* word, const float* pos, float* out, int B, int S, int H, int vocab,
                   void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (H % 4 != 0) { set_last_error("embed_fwd: H must be a multiple of 4"); return MUSE_ERR_INVALID; }
  const int tokens = B * S;
  if (tokens <= 0) return MUSE_OK;
  pdl_launch(ceil_div(tokens, 4), 128, 0, s)(embed_fwd_kernel, ids, word, pos, out, tokens, S, H, vocab);
  return check_launch("embed_fwd");
}

int muse_embed_bwd(const long long* ids, const float* dx, float* dword, float* dpos, int B, int S, int H, int vocab,
                   void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (H % 4 != 0) { set_last_error("embed_bwd: H must be a multiple of 4"); return MUSE_ERR_INVALID; }
  const int tokens = B * S;
  if (tokens <= 0) return MUSE_OK;
  const int hot = vocab - 1;  // the reference's mask_token_id
  const int grid = ceil_div(tokens, 8 * kEmbTokPerWarp);
  if (H == 512) pdl_launch(grid, 256, 0, s)(embed_bwd_word_kernel<4>, ids, dx, dword, tokens, H, vocab, hot);
  else if (H == 768) pdl_launch(grid, 256, 0, s)(embed_bwd_word_kernel<6>, ids, dx, dword, tokens, H, vocab, hot);
  else if (H == 1024) pdl_launch(grid, 256, 0, s)(embed_bwd_word_kernel<8>, ids, dx, dword, tokens, H, vocab, hot);
  else if (H == 128) pdl_launch(grid, 256, 0, s)(embed_bwd_word_kernel<1>, ids, dx, dword, tokens, H, vocab, hot);
  else pdl_launch(ceil_div(tokens, 4), 128, 0, s)(embed_bwd_word_generic_kernel, ids, dx, dword, tokens, H, vocab);
  int rc = check_launch("embed_bwd_word");
  if (rc) return rc;
  if (dpos == nullptr) return MUSE_OK;  // no position table (ConvEmbed of MaskGiTUViT_v2)
  pdl_launch(dim3(S, ceil_div(H, 128)), 128, 0, s)(embed_bwd_pos_kernel, dx, dpos, B, S, H);
  return check_launch("embed_bwd_pos");
}

// workspace: (tokens / kSegChunk + vocab) partial rows of H floats, then vocab + 1 ints of chunk offsets
long long muse_embed_bwd_sorted_workspace_bytes(int tokens, int H, int vocab) {
  return (static_cast<long long>(tokens) / kSegChunk + vocab) * H * 4 + (static_cast<long long>(vocab) + 1) * 4;
}

int muse_embed_bwd_sorted(const long long* order, const long long* bounds, const float* dx, float* dword, float* dpos,
                          void* ws, int B, int S, int H, int vocab, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (H % 4 != 0) { set_last_error("embed_bwd_sorted: H must be a multiple of 4"); return MUSE_ERR_INVALID; }
  const int tokens = B * S;
  if (tokens <= 0 || vocab <= 0) return MUSE_OK;
  const int max_chunks = tokens / kSegChunk + vocab;
  float* partial = reinterpret_cast<float*>(ws);
  int* chunk_off = reinterpret_cast<int*>(partial + static_cast<size_t>(max_chunks) * H);
  int ncol = H / 4;
  if (ncol > 128) ncol = 128;  // 4 groups x ncol threads <= 512 (the kernels' launch bound)
  const size_t smem = static_cast<size_t>(4) * H * sizeof(float);
  if (smem > 48 * 1024) { set_last_error("embed_bwd_sorted: H=%d too wide", H); return MUSE_ERR_UNSUPPORTED; }
  pdl_launch(1, 1024, 0, s)(embed_seg_plan_kernel, bounds, chunk_off, vocab);
  pdl_launch(max_chunks, 4 * ncol, smem, s)(embed_seg_chunk_kernel, order, bounds, chunk_off, dx, dword, partial, H, vocab);
  pdl_launch(vocab, 4 * ncol, smem, s)(embed_seg_final_kernel, chunk_off, partial, dword, H, vocab);
  int rc = check_launch("embed_bwd_sorted");
  if (rc) return rc;
  if (dpos == nullptr) return MUSE_OK;
  pdl_launch(dim3(S, ceil_div(H, 128)), 128, 0, s)(embed_bwd_pos_kernel, dx, dpos, B, S, H);
  return check_launch("embed_bwd_pos");
}

int muse_quantize_rows_e4m3(const void* x, int ldx, void* q, int ldq, float* scale, int rows, int K, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0 || K <= 0) return MUSE_OK;
  if (ldx < K || ldq < K) { set_last_error("quantize_rows_e4m3: pitches %d / %d below K = %d", ldx, ldq, K); return MUSE_ERR_INVALID; }
  if (K % 8 != 0 || ldx % 8 != 0 || ldq % 8 != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(q) & 7) != 0) {
    set_last_error("quantize_rows_e4m3: K, ldx and ldq must be multiples of 8, x 16-byte and q 8-byte aligned");
    return MUSE_ERR_INVALID;
  }
  pdl_launch(ceil_div(rows, 8), 256, 0, s)(quantize_rows_e4m3_kernel, reinterpret_cast<const bf16*>(x), ldx,
                                           reinterpret_cast<uint8_t*>(q), ldq, scale, rows, K);
  return check_launch("quantize_rows_e4m3");
}

// bits == nullptr: no dropout; else FeedForward.dropout fused into the pass, bits [rows, ceil(I / 32)] written.
int muse_glu_fwd(const void* ab, void* out, int out_dt, float* row_scale, unsigned int* bits, const unsigned long long* seed,
                 int site, float p, long long rows, int I, void* stream) {
  return ffn_act_fwd<true>("glu_fwd", ab, out, out_dt, row_scale, bits, seed, site, p, rows, I, static_cast<cudaStream_t>(stream));
}

// bits: those muse_glu_fwd wrote (nullptr: no dropout); dout is scaled by them as it is read.
int muse_glu_bwd(const void* ab, const void* dout, const unsigned int* bits, float p, void* dab, long long rows, int I,
                 void* stream) {
  return ffn_act_bwd<true>("glu_bwd", ab, dout, bits, p, dab, rows, I, static_cast<cudaStream_t>(stream));
}

int muse_gelu_tanh_fwd(const void* pre, void* out, int out_dt, float* row_scale, long long rows, int I, void* stream) {
  return ffn_act_fwd<false>("gelu_tanh_fwd", pre, out, out_dt, row_scale, nullptr, nullptr, 0, 0.f, rows, I,
                            static_cast<cudaStream_t>(stream));
}

int muse_gelu_tanh_bwd(const void* pre, const void* dout, void* dpre, long long rows, int I, void* stream) {
  return ffn_act_bwd<false>("gelu_tanh_bwd", pre, dout, nullptr, 0.f, dpre, rows, I, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
