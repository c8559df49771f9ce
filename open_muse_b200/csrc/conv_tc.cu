// MaskGitVQGAN convolutions on the Hopper tensor cores (wgmma) (muse/modeling_maskgit_vqgan.py:33-45 Conv2dSame, stride 1,
// k = 3 or 1) as an implicit GEMM with fp32-faithful accuracy:
//
//     y[m, co] = bias[co] + res[m, co] + sum_{tap, ci} x[pixel(m) + tap, ci] * w[co, tap, ci]
//
//   M = B*H*W output pixels (128 per tile), N = C_out (128 or 256 per tile), K = k*k*C_in.
//
// * No im2col buffer: activations stay NHWC and the A tile of one (tap, 64-channel chunk) is ONE 4-D TMA box
//   {64 ch, tile_w, tile_h, 1 image} fetched at pixel offset (kw - pad, kh - pad); coordinates outside the image are
//   zero-filled by the TMA unit, which is exactly the 'same' padding.  The box lands in shared memory as 128 rows x 128 B
//   (128-byte swizzle) = a K-major wgmma operand, rows ordered like the output pixels of the tile.
// * fp32 accuracy from bf16 tensor cores: every fp32 operand is carried as two bf16 planes  v = hi + lo
//   (hi = bf16(v), lo = bf16(v - hi), representation error 2^-18 |v|) and the product is accumulated as
//   hi*hi + lo*hi + hi*lo in the fp32 register accumulator (the dropped lo*lo term is ~2^-18 relative).  The token ids of the
//   quantiser downstream need this: a single bf16/TF32 pass perturbs z by ~1e-3 and flips near-tie codes (SURVEY H1).
//   The planes are produced by the preceding GroupNorm+SiLU kernel (same bytes as one fp32 tensor) or by
//   split_bf16_nhwc (which also folds the nearest x2 upsample of UpsamplingBlock :146 into its gather).
// * UpsamplingBlock (nearest x2 then 3x3 conv, :141-149) never materialises the upsampled tensor and skips its redundant
//   arithmetic: output pixel (2y+py, 2x+px) only sees a 2x2 window of the low-resolution input, so each of the four
//   parities (py, px) is a 2x2 convolution with pre-summed weights (K = 4*C_in instead of 9*C_in, 2.25x fewer FLOPs)
//   whose tile rows scatter to every other output pixel.
// * Same persistent warp-specialised pipeline as gemm_wgmma.cu: one TMA producer thread, two consumer warpgroups
//   (wgmma m64 x BN x k16 on their 64-pixel halves of the tile); the epilogue adds bias / residual to the accumulator
//   registers, writes fp32 NHWC rows and folds the per-channel GroupNorm statistics of the tile.
#include "common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace muse {

int make_tmap_nd(CUtensorMap* map, const void* base, int rank, const unsigned long long* dims,
                 const unsigned long long* strides_bytes, const unsigned* box);

namespace {

constexpr int BM = 128;
constexpr int BK = 64;

template <int BN>
struct Cfg {
  static constexpr int kStages = (BN == 256) ? 4 : (BN == 128 ? 6 : 8);
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;  // a multiple of 1024 for BN in {16, 128, 256}
  static constexpr int kBarBytes = 256;
  static constexpr int kStatBytes = 8 * BN * 2 * 4;  // per-consumer-warp {sum, sumsq} of every tile column
  static constexpr int kSmemBytes = kStages * kStageBytes + kStatBytes + 1024 + kBarBytes;
};

struct ConvParams {
  float* y;
  const float* bias;
  const float* res;
  float* stats;  // nullable: per [pixel tile][C_out] {sum, sumsq} of y, the GroupNorm statistics of the next layer
  int N;  // C_out
  int H, W, Cin, ksize;
  int tile_w, tile_h, tiles_x, tiles_per_img;
  int up, tile_w_log2;  // up: nearest x2 upsample folded in as four 2x2 parity convolutions on the H x W (input) grid
  int fwd2x2;           // taps are the 2x2 window at offsets (0..1, 0..1): the stride-2 3x3 conv after space-to-depth
  int wbatch;           // weights are per image: [B][C_out][K] (attention scores / values as 1x1 convolutions)
  int num_m, num_n, cchunks, num_kb;
  int passes;           // 3: bf16x3 (hi*hi + lo*hi + hi*lo, fp32-faithful); 1: hi*hi only (plain bf16 operands, fast mode)
};

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];\n" ::
          "r"(ptx::smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(ptx::smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n" ::
          "r"(ptx::smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(ptx::smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

template <int BN>
__global__ void __launch_bounds__(384, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
               const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl, const ConvParams p) {
  pdl_trigger();
  using C_ = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  float* stat_smem = reinterpret_cast<float*>(smem + C_::kStages * C_::kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C_::kStages * C_::kStageBytes + C_::kStatBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + C_::kStages;

  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmAh);
    ptx::prefetch_tmap(&tmAl);
    ptx::prefetch_tmap(&tmBh);
    ptx::prefetch_tmap(&tmBl);
    for (int i = 0; i < C_::kStages; ++i) {
      ptx::mbar_init(&full_bar[i], 1);
      ptx::mbar_init(&empty_bar[i], 2);  // one arrive per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // everything above touches only shared memory / kernel parameters
  const int tiles_mn = p.num_m * p.num_n;
  const int total_tiles = tiles_mn * (p.up ? 4 : 1);
  const int pad = p.ksize / 2;

  if (wg == 0) {
    ptx::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      // ------------------------------------------------------------ TMA producer
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int parity = tile / tiles_mn, tl = tile % tiles_mn;
        const int n_idx = tl % p.num_n;
        const int m_idx = tl / p.num_n;
        const int img = m_idx / p.tiles_per_img;
        const int t = m_idx % p.tiles_per_img;
        const int y0 = (t / p.tiles_x) * p.tile_h, x0 = (t % p.tiles_x) * p.tile_w;
        const int n0 = n_idx * BN;
        const int wrow0 = parity * p.N;  // up: the four parity weight matrices are stacked along the rows
        int pass = 0, cc = 0, tap = 0;  // kb = (tap * cchunks + cc) * passes + pass
        for (int kb = 0; kb < p.num_kb; ++kb) {
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          ptx::mbar_expect_tx(&full_bar[stage], C_::kStageBytes);
          uint8_t* sa = smem + stage * C_::kStageBytes;
          uint8_t* sb = sa + C_::kABytes;
          // passes: 0 = hi*hi, 1 = lo(A)*hi(B), 2 = hi(A)*lo(B)
          const int dy = p.up ? (tap >> 1) + (parity >> 1) - 1 : (p.fwd2x2 ? (tap >> 1) : tap / p.ksize - pad);
          const int dx = p.up ? (tap & 1) + (parity & 1) - 1 : (p.fwd2x2 ? (tap & 1) : tap % p.ksize - pad);
          const int wb = p.wbatch ? img : 0;
          tma_load_4d(sa, pass == 1 ? &tmAl : &tmAh, &full_bar[stage], cc * BK, x0 + dx, y0 + dy, img);
          tma_load_3d(sb, pass == 2 ? &tmBl : &tmBh, &full_bar[stage], tap * p.Cin + cc * BK, wrow0 + n0, wb);
          if (++stage == C_::kStages) { stage = 0; phase ^= 1; }
          if (++pass == p.passes) {
            pass = 0;
            if (++cc == p.cchunks) { cc = 0; ++tap; }
          }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<232>();
    // -------------------------------------------------------------- consumers: y = acc + bias (+ res), fp32 NHWC
    const int half = wg - 1;
    const int t = threadIdx.x & 127;
    const int cw = threadIdx.x / 32 - 4;                         // consumer warp 0..7
    const int lr = half * 64 + (t >> 5) * 16 + ((t & 31) >> 2);  // tile pixel of d[4j], d[4j+1]; +8 for d[4j+2..3]
    const int lc = 2 * (t & 3);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      for (int kb = 0; kb < p.num_kb; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = ptx::smem_u32(smem + stage * C_::kStageBytes) + half * 8192;
        const uint32_t b_addr = ptx::smem_u32(smem + stage * C_::kStageBytes + C_::kABytes);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          ptx::Wgmma<BN, 0, 0>::run(acc, ptx::make_smem_desc_sw128(a_addr + k * 32, 16, 1024),
                                    ptx::make_smem_desc_sw128(b_addr + k * 32, 16, 1024), (kb > 0 || k > 0) ? 1 : 0);
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        if (t == 0) ptx::mbar_arrive(&empty_bar[stage]);
        if (++stage == C_::kStages) { stage = 0; phase ^= 1; }
      }
      const int parity = tile / tiles_mn, tl = tile % tiles_mn;
      const int n_idx = tl % p.num_n;
      const int m_idx = tl / p.num_n;
      const int img = m_idx / p.tiles_per_img;
      const int tt = m_idx % p.tiles_per_img;
      const int y0 = (tt / p.tiles_x) * p.tile_h, x0 = (tt % p.tiles_x) * p.tile_w;
      const long long row_base0 = (static_cast<long long>(img) * p.H + y0) * p.W + x0;  // tile pixels are contiguous
      // output row (pixel index) of tile-local pixel tr; up: parity (py, px) scatters to every other pixel of the 2H x 2W grid
      auto out_row = [&](int tr) -> long long {
        if (!p.up) return row_base0 + tr;
        const int ty = tr >> p.tile_w_log2, tx = tr & (p.tile_w - 1);
        return (static_cast<long long>(img) * (2 * p.H) + 2 * (y0 + ty) + (parity >> 1)) * (2 * p.W) + 2 * (x0 + tx) + (parity & 1);
      };
      const size_t stat_row = p.up ? (static_cast<size_t>(img) * 4 + parity) * p.tiles_per_img + tt : static_cast<size_t>(m_idx);
      const int n0 = n_idx * BN;
      const long long orow[2] = {out_row(lr), out_row(lr + 8)};
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + 8 * j + lc;
        float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
        if (BN == 16) {  // narrow head (C_out <= 16, e.g. the 3-channel pixel output): element-wise, no statistics
#pragma unroll
          for (int hr = 0; hr < 2; ++hr)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              if (col + e < p.N) {
                const size_t off = static_cast<size_t>(orow[hr]) * p.N + col + e;
                float v = acc[4 * j + 2 * hr + e];
                if (p.bias != nullptr) v += p.bias[col + e];
                if (p.res != nullptr) v += p.res[off];
                p.y[off] = v;
              }
            }
        } else if (col < p.N) {  // N % 4 == 0
          float2 b2 = make_float2(0.f, 0.f);
          if (p.bias != nullptr) b2 = *reinterpret_cast<const float2*>(p.bias + col);
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const size_t off = static_cast<size_t>(orow[hr]) * p.N + col;
            float2 o = make_float2(acc[4 * j + 2 * hr] + b2.x, acc[4 * j + 2 * hr + 1] + b2.y);
            if (p.res != nullptr) {
              const float2 r2 = *reinterpret_cast<const float2*>(p.res + off);
              o.x += r2.x; o.y += r2.y;
            }
            *reinterpret_cast<float2*>(p.y + off) = o;
            s0 += o.x; s1 += o.y;
            q0 = fmaf(o.x, o.x, q0); q1 = fmaf(o.y, o.y, q1);
          }
        }
        if (BN != 16 && p.stats != nullptr) {  // fold the 8 row groups of the warp (lane >> 2); lanes 0-3 publish
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, o);
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
            q0 += __shfl_xor_sync(0xffffffffu, q0, o);
            q1 += __shfl_xor_sync(0xffffffffu, q1, o);
          }
          if ((t & 31) < 4)
            *reinterpret_cast<float4*>(stat_smem + (cw * BN + 8 * j + lc) * 2) = make_float4(s0, q0, s1, q1);
        }
      }
      if (BN != 16 && p.stats != nullptr) {
        asm volatile("bar.sync 1, 256;" ::: "memory");  // the eight consumer warps
        for (int col = threadIdx.x - 128; col < BN; col += 256) {
          if (n0 + col < p.N) {
            float2 a = make_float2(0.f, 0.f);
#pragma unroll
            for (int wq = 0; wq < 8; ++wq) {
              const float2 v = *reinterpret_cast<const float2*>(stat_smem + ((wq * BN) + col) * 2);
              a.x += v.x; a.y += v.y;
            }
            *reinterpret_cast<float2*>(p.stats + (stat_row * p.N + n0 + col) * 2) = a;
          }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
    }
  }
}

// v = hi + lo with hi = bf16(v), lo = bf16(v - hi); optional nearest x2 upsample folded into the gather.
__global__ void __launch_bounds__(256)
split_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ hi, bf16* __restrict__ lo, long long total8, int H, int W,
                  int C, int up) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= total8) return;
  long long src = i;
  if (up) {
    const int c8 = C / 8;
    const int q = static_cast<int>(i % c8);
    const long long pix = i / c8;
    const int ox = static_cast<int>(pix % W);
    const int oy = static_cast<int>((pix / W) % H);
    const long long b = pix / (static_cast<long long>(W) * H);
    src = ((b * (H / 2) + (oy >> 1)) * (W / 2) + (ox >> 1)) * c8 + q;
  }
  float v[8], h[8], l[8];
  load8(x + src * 8, v);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    h[j] = bf16_round(v[j]);
    l[j] = v[j] - h[j];
  }
  store8(hi + i * 8, h);
  if (lo) store8(lo + i * 8, l);
}

// Small-C_in stem (3 -> 128 at full resolution): im2col of the k*k*C_in <= 64 taps into 64-wide bf16 hi/lo rows, so the
// stem runs as a 1x1 tensor-core convolution with C_in = 64 (zero columns past k*k*C_in).  8 threads per pixel.
__global__ void __launch_bounds__(256)
im2col_split_kernel(const float* __restrict__ x, bf16* __restrict__ hi, bf16* __restrict__ lo, long long pixels, int H, int W,
                    int Cin, int ksize) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= pixels * 8) return;
  const long long pix = i >> 3;
  const int chunk = static_cast<int>(i & 7);
  const int ox = static_cast<int>(pix % W);
  const int oy = static_cast<int>((pix / W) % H);
  const long long b = pix / (static_cast<long long>(W) * H);
  const int pad = ksize / 2, K = ksize * ksize * Cin;
  float h[8], l[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int k = chunk * 8 + j;
    float v = 0.f;
    if (k < K) {
      const int tap = k / Cin, ci = k % Cin;
      const int iy = oy + tap / ksize - pad, ix = ox + tap % ksize - pad;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = x[((b * H + iy) * W + ix) * Cin + ci];
    }
    h[j] = bf16_round(v);
    l[j] = v - h[j];
  }
  store8(hi + i * 8, h);
  if (lo) store8(lo + i * 8, l);
}

// space-to-depth + hi/lo split: x fp32 [B,H,W,C] -> planes bf16 [B,H/2,W/2,4C], channel = (row parity * 2 + col parity) * C + c
__global__ void __launch_bounds__(256)
split_s2d_kernel(const float* __restrict__ x, bf16* __restrict__ hi, bf16* __restrict__ lo, long long total8, int Ho, int Wo,
                 int C) {
  pdl_enter();
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= total8) return;
  const int c8 = C / 8;
  const int q = static_cast<int>(i % c8);
  const int par = static_cast<int>((i / c8) % 4);
  const long long pix = i / (static_cast<long long>(c8) * 4);
  const int ox = static_cast<int>(pix % Wo);
  const int oy = static_cast<int>((pix / Wo) % Ho);
  const long long b = pix / (static_cast<long long>(Wo) * Ho);
  const long long src = ((b * (2 * Ho) + 2 * oy + (par >> 1)) * (2 * Wo) + 2 * ox + (par & 1)) * C + q * 8;
  float v[8], h[8], l[8];
  load8(x + src, v);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    h[j] = bf16_round(v[j]);
    l[j] = v[j] - h[j];
  }
  store8(hi + i * 8, h);
  if (lo) store8(lo + i * 8, l);
}

// softmax(scale * x) over rows of n fp32 values (one warp per row), emitted as bf16 hi/lo planes
__global__ void __launch_bounds__(256)
softmax_split_kernel(const float* __restrict__ x, bf16* __restrict__ hi, bf16* __restrict__ lo, float* __restrict__ out,
                     long long rows, int n, float scale) {
  pdl_enter();
  const long long row = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* xr = x + row * n;
  float m = -INFINITY;
  for (int c = lane; c < n; c += 32) m = fmaxf(m, xr[c] * scale);
  m = warp_max(m);
  float sum = 0.f;
  for (int c = lane; c < n; c += 32) sum += expf(xr[c] * scale - m);
  sum = warp_sum(sum);
  for (int c = lane; c < n; c += 32) {
    const float pv = expf(xr[c] * scale - m) / sum;
    if (out) { out[row * n + c] = pv; continue; }
    const float h = bf16_round(pv);
    hi[row * n + c] = __float2bfloat16_rn(h);
    lo[row * n + c] = __float2bfloat16_rn(pv - h);
  }
}

int g_sms = 0;
int sm_count() {
  if (g_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_sms <= 0) g_sms = 132;
  }
  return g_sms;
}

template <int BN>
int launch_conv(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh, const CUtensorMap& bl,
                const ConvParams& p, cudaStream_t s) {
  auto kern = conv_tc_kernel<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::kSmemBytes);
    if (e != cudaSuccess) { set_last_error("cudaFuncSetAttribute(conv_tc): %s", cudaGetErrorString(e)); return MUSE_ERR_CUDA; }
    attr_set = true;
  }
  const int total = p.num_m * p.num_n;
  const int grid = total < sm_count() ? total : sm_count();
  pdl_launch(grid, 384, Cfg<BN>::kSmemBytes, s)(kern, ah, al, bh, bl, p);
  return check_launch("conv_tc");
}

}  // namespace

// 1 if conv2d_tc handles the shape (otherwise the caller uses the fp32 SIMT kernel of conv.cu).
int conv2d_tc_supported(int H, int W, int Cin, int Cout, int ksize) {
  if (ksize != 1 && ksize != 3 && ksize != 2) return 0;  // 2: the 2x2 forward-offset window (mode 2 of conv2d_tc)
  if (Cin % 64 != 0 || Cout < 1 || (Cout > 16 && Cout % 4 != 0)) return 0;
  if (W >= 128) return W % 128 == 0;
  if (W < 8 || 128 % W != 0) return 0;
  return H % (128 / W) == 0;
}

// Pixel tiles per image of conv2d_tc for this shape (= the leading extent of its stats output), 0 if unsupported.
// H, W are the OUTPUT dims; with upsample2x the tiling runs on the H/2 x W/2 input grid, four parities each.
int conv2d_tc_tiles_per_image(int H, int W, int Cin, int Cout, int ksize, int upsample2x) {
  if (upsample2x) {
    if ((H | W) & 1 || ksize != 3 || Cout <= 16) return 0;
    H /= 2; W /= 2;
  }
  if (!conv2d_tc_supported(H, W, Cin, Cout, ksize)) return 0;
  return (upsample2x ? 4 : 1) * (H * W / 128);
}

// mode & 3 == 1 (upsample2x): x planes are the LOW-resolution input [B,H/2,W/2,Cin] and w planes the four stacked parity
//   matrices [4*Cout, 4*Cin] (ops.py packs them); y / res / stats are at the output resolution [B,H,W,Cout].
// mode & 3 == 2: ksize 2, taps at offsets (0,0),(0,1),(1,0),(1,1), zero beyond the right / bottom edge -- a stride-2 3x3
//   convolution with pad (0,1,0,1) (taming Downsample) after a space-to-depth of its input (w: [Cout, 4 * Cin]).
// mode & 4: per-image weights, w planes are [B][Cout][K].
// mode & 8: single-pass bf16 (fast tokenizer mode): only the hi planes are multiplied (x_lo / w_lo may be null): one tensor-core
//   product per fp32 product instead of three, bf16-operand accuracy (~4e-3 per layer instead of ~2e-5).
// x_hi/x_lo: bf16 [B,H,W,Cin]; w_hi/w_lo: bf16 [Cout, k*k*Cin] (tap-major, then input channel); y fp32 [B,H,W,Cout].
int conv2d_tc(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, const float* bias, const float* res,
              float* y, float* stats, int B, int H, int W, int Cin, int Cout, int ksize, int mode, cudaStream_t s) {
  if (B <= 0) return MUSE_OK;
  const int upsample2x = (mode & 3) == 1;
  const int fwd2x2 = (mode & 3) == 2;
  if (fwd2x2 != (ksize == 2)) { set_last_error("conv2d_tc: ksize 2 and mode 2 go together"); return MUSE_ERR_INVALID; }
  if (upsample2x) {
    if (conv2d_tc_tiles_per_image(H, W, Cin, Cout, ksize, 1) == 0) {
      set_last_error("conv2d_tc: unsupported upsample shape H=%d W=%d Cin=%d Cout=%d k=%d", H, W, Cin, Cout, ksize);
      return MUSE_ERR_UNSUPPORTED;
    }
    H /= 2; W /= 2;  // the tiling / TMA grid is the input grid
  }
  if (!conv2d_tc_supported(H, W, Cin, Cout, ksize)) {
    set_last_error("conv2d_tc: unsupported shape H=%d W=%d Cin=%d Cout=%d k=%d", H, W, Cin, Cout, ksize);
    return MUSE_ERR_UNSUPPORTED;
  }
  if ((reinterpret_cast<uintptr_t>(y) & 15) || (bias && (reinterpret_cast<uintptr_t>(bias) & 15)) ||
      (res && (reinterpret_cast<uintptr_t>(res) & 15))) {
    set_last_error("conv2d_tc: y / bias / res must be 16B aligned");
    return MUSE_ERR_INVALID;
  }
  ConvParams p;
  p.y = y; p.bias = bias; p.res = res; p.stats = (Cout > 16) ? stats : nullptr;
  p.N = Cout; p.H = H; p.W = W; p.Cin = Cin; p.ksize = ksize;
  const int tile_px = 128;
  p.tile_w = W >= tile_px ? tile_px : W;
  p.tile_h = tile_px / p.tile_w;
  p.tiles_x = W / p.tile_w;
  p.tiles_per_img = p.tiles_x * (H / p.tile_h);
  p.num_m = B * p.tiles_per_img;
  p.up = upsample2x ? 1 : 0;
  p.fwd2x2 = fwd2x2;
  p.wbatch = (mode & 4) ? 1 : 0;
  p.tile_w_log2 = 0;
  while ((1 << p.tile_w_log2) < p.tile_w) ++p.tile_w_log2;
  if (p.up && (1 << p.tile_w_log2) != p.tile_w) { set_last_error("conv2d_tc: upsample needs a power-of-two tile width"); return MUSE_ERR_UNSUPPORTED; }
  const int BN = Cout >= 256 ? 256 : (Cout > 16 ? 128 : 16);
  p.num_n = ceil_div(Cout, BN);
  p.cchunks = Cin / BK;
  const int taps = (p.up || p.fwd2x2) ? 4 : ksize * ksize;
  p.passes = (mode & 8) ? 1 : 3;
  p.num_kb = taps * p.cchunks * p.passes;
  if (p.passes == 1) { x_lo = x_hi; w_lo = w_hi; }  // the lo maps are never dereferenced; keep the encodes valid

  CUtensorMap ah, al, bh, bl;
  const unsigned long long adims[4] = {(unsigned long long)Cin, (unsigned long long)W, (unsigned long long)H, (unsigned long long)B};
  const unsigned long long astr[3] = {(unsigned long long)Cin * 2, (unsigned long long)W * Cin * 2, (unsigned long long)H * W * Cin * 2};
  const unsigned abox[4] = {64, (unsigned)p.tile_w, (unsigned)p.tile_h, 1};
  int rc;
  if ((rc = make_tmap_nd(&ah, x_hi, 4, adims, astr, abox))) return rc;
  if ((rc = make_tmap_nd(&al, x_lo, 4, adims, astr, abox))) return rc;
  const unsigned long long K = static_cast<unsigned long long>(taps) * Cin;
  const unsigned long long wrows = (unsigned long long)Cout * (p.up ? 4 : 1);
  const unsigned long long bdims[3] = {K, wrows, (unsigned long long)(p.wbatch ? B : 1)};
  const unsigned long long bstr[2] = {K * 2, K * 2 * wrows};
  const unsigned bbox[3] = {64, (unsigned)BN, 1};
  if ((rc = make_tmap_nd(&bh, w_hi, 3, bdims, bstr, bbox))) return rc;
  if ((rc = make_tmap_nd(&bl, w_lo, 3, bdims, bstr, bbox))) return rc;
  if (BN == 256) return launch_conv<256>(ah, al, bh, bl, p, s);
  if (BN == 128) return launch_conv<128>(ah, al, bh, bl, p, s);
  return launch_conv<16>(ah, al, bh, bl, p, s);
}

// x fp32 [B,H,W,Cin] with k*k*Cin <= 64 -> hi, lo bf16 [B,H,W,64]: row = the k*k*Cin taps of the pixel (tap-major), zero padded
int im2col_split_nhwc(const float* x, void* hi, void* lo, int B, int H, int W, int Cin, int ksize, cudaStream_t s) {
  if (ksize * ksize * Cin > 64 || (ksize != 1 && ksize != 3)) {
    set_last_error("im2col_split: k*k*Cin = %d must be <= 64", ksize * ksize * Cin);
    return MUSE_ERR_UNSUPPORTED;
  }
  const long long pixels = static_cast<long long>(B) * H * W;
  if (pixels <= 0) return MUSE_OK;
  pdl_launch(static_cast<unsigned>(ceil_div_ll(pixels * 8, 256)), 256, 0, s)(im2col_split_kernel,
      x, reinterpret_cast<bf16*>(hi), reinterpret_cast<bf16*>(lo), pixels, H, W, Cin, ksize);
  return check_launch("im2col_split");
}

// x fp32 [B,2Ho,2Wo,C] -> hi, lo bf16 [B,Ho,Wo,4C]
int split_s2d_bf16_nhwc(const float* x, void* hi, void* lo, int B, int Ho, int Wo, int C, cudaStream_t s) {
  if (C % 8 != 0) { set_last_error("split_s2d: C must be a multiple of 8"); return MUSE_ERR_UNSUPPORTED; }
  const long long total8 = static_cast<long long>(B) * Ho * Wo * 4 * (C / 8);
  if (total8 <= 0) return MUSE_OK;
  pdl_launch(static_cast<unsigned>(ceil_div_ll(total8, 256)), 256, 0, s)(split_s2d_kernel, x, reinterpret_cast<bf16*>(hi),
                                                                                   reinterpret_cast<bf16*>(lo), total8, Ho, Wo, C);
  return check_launch("split_s2d");
}

// out_f32 given: plain fp32 softmax (hi / lo unused); else the bf16 hi/lo planes
int softmax_split_rows(const float* x, void* hi, void* lo, float* out_f32, long long rows, int n, float scale, cudaStream_t s) {
  if (rows <= 0 || n <= 0) return MUSE_OK;
  if (out_f32 == x) { set_last_error("softmax: in-place output is not supported"); return MUSE_ERR_INVALID; }
  pdl_launch(static_cast<unsigned>(ceil_div_ll(rows, 8)), 256, 0, s)(softmax_split_kernel, x, reinterpret_cast<bf16*>(hi),
                                                                                   reinterpret_cast<bf16*>(lo), out_f32, rows, n, scale);
  return check_launch("softmax_split");
}

// x fp32 [B, H/(1+up), W/(1+up), C] -> hi, lo bf16 [B,H,W,C]
int split_bf16_nhwc(const float* x, void* hi, void* lo, int B, int H, int W, int C, int upsample2x, cudaStream_t s) {
  if (C % 8 != 0) { set_last_error("split_bf16: C must be a multiple of 8"); return MUSE_ERR_UNSUPPORTED; }
  if (upsample2x && ((H | W) & 1)) { set_last_error("split_bf16: upsample2x needs even output dims"); return MUSE_ERR_INVALID; }
  const long long total8 = static_cast<long long>(B) * H * W * (C / 8);
  if (total8 <= 0) return MUSE_OK;
  pdl_launch(static_cast<unsigned>(ceil_div_ll(total8, 256)), 256, 0, s)(split_bf16_kernel, x, reinterpret_cast<bf16*>(hi),
                                                                                    reinterpret_cast<bf16*>(lo), total8, H, W, C, upsample2x);
  return check_launch("split_bf16");
}

}  // namespace muse
