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
// * The persistent warp-specialised pipeline of tc_pipeline.cuh (wgmma m64 x BN x k16 on the two 64-pixel halves of the
//   tile); the epilogue adds bias / residual to the accumulator registers, writes fp32 NHWC rows and folds the
//   per-channel GroupNorm statistics of the tile: its sum, then the squared deviations from the tile mean (M2).
#include "common.cuh"
#include "tc_host.cuh"
#include "tc_pipeline.cuh"

namespace muse {

namespace {

using tc::BK;

// Stages of the ring: a multiple of 1024 B for BN in {16, 128, 256}.  Behind them, per consumer warp, {sum, M2} of
// every tile column over the warp's 16 pixels.
template <int BN>
using Ring = tc::Ring<BN, (BN == 256) ? 4 : (BN == 128 ? 6 : 8), 8 * BN * 2 * 4>;

struct ConvParams {
  float* y;
  const float* bias;
  const float* res;
  float* stats;  // nullable: per [pixel tile][C_out] {sum, M2} of y (M2 about the tile mean), the next GroupNorm's statistics
  int N;  // C_out
  int H, W, Cin, ksize;
  int tile_w, tile_h, tiles_x, tiles_per_img;
  int up, tile_w_log2;  // up: nearest x2 upsample folded in as four 2x2 parity convolutions on the H x W (input) grid
  int fwd2x2;           // taps are the 2x2 window at offsets (0..1, 0..1): the stride-2 3x3 conv after space-to-depth
  int wbatch;           // weights are per image: [B][C_out][K] (attention scores / values as 1x1 convolutions)
  int num_m, num_n, cchunks, num_kb;
  int passes;           // 3: bf16x3 (hi*hi + lo*hi + hi*lo, fp32-faithful); 1: hi*hi only (plain bf16 operands, fast mode)
  bf16* yh;             // non-null: y = GELU(acc + bias) is stored as these bf16 planes (yl: lo, nullable) instead of fp32 y
  bf16* yl;
  int shuffle;          // C_out <= 16: PixelShuffle(2) folded into the store, y is [B, 2H, 2W, C_out / 4]
};

// nn.GELU() (exact erf form) of the Paella ResBlock's channelwise MLP
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }

template <int BN>
__global__ void __launch_bounds__(tc::kThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
               const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl, const ConvParams p) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  Ring<BN> ring(smem_raw);
  float* stat_smem = reinterpret_cast<float*>(ring.extra());

  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmAh);
    ptx::prefetch_tmap(&tmAl);
    ptx::prefetch_tmap(&tmBh);
    ptx::prefetch_tmap(&tmBl);
    ring.init();
  }
  __syncthreads();
  pdl_wait();  // everything above touches only shared memory / kernel parameters
  const int tiles_mn = p.num_m * p.num_n;
  const int total_tiles = tiles_mn * (p.up ? 4 : 1);
  const int pad = p.ksize / 2;

  if (wg == 0) {
    ptx::setmaxnreg_dec<tc::kProducerRegs>();
    if (threadIdx.x == 0) {
      // ------------------------------------------------------------ TMA producer
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
          const auto s = ring.produce();
          // passes: 0 = hi*hi, 1 = lo(A)*hi(B), 2 = hi(A)*lo(B)
          const int dy = p.up ? (tap >> 1) + (parity >> 1) - 1 : (p.fwd2x2 ? (tap >> 1) : tap / p.ksize - pad);
          const int dx = p.up ? (tap & 1) + (parity & 1) - 1 : (p.fwd2x2 ? (tap & 1) : tap % p.ksize - pad);
          const int wb = p.wbatch ? img : 0;
          ptx::tma_load_4d(s.a, pass == 1 ? &tmAl : &tmAh, s.bar, cc * BK, x0 + dx, y0 + dy, img);
          ptx::tma_load_3d(s.b, pass == 2 ? &tmBl : &tmBh, s.bar, tap * p.Cin + cc * BK, wrow0 + n0, wb);
          if (++pass == p.passes) {
            pass = 0;
            if (++cc == p.cchunks) { cc = 0; ++tap; }
          }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<tc::kConsumerRegs>();
    // -------------------------------------------------------------- consumers: y = acc + bias (+ res), fp32 NHWC
    const int half = wg - 1;
    const int t = threadIdx.x & 127;
    const int cw = threadIdx.x / 32 - 4;          // consumer warp 0..7
    const int lr = half * 64 + ptx::frag_row();  // tile pixel of d[4j], d[4j+1]; +8 for d[4j+2..3]
    const int lc = ptx::frag_col();
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      ring.template consume<false, false>(acc, 0, p.num_kb, half);
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
        if (BN == 16) {  // narrow head (C_out <= 16, e.g. the 3-channel pixel output): element-wise, no statistics
#pragma unroll
          for (int hr = 0; hr < 2; ++hr)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              if (col + e < p.N) {
                size_t off = static_cast<size_t>(orow[hr]) * p.N + col + e;
                float v = acc[4 * j + 2 * hr + e];
                if (p.bias != nullptr) v += p.bias[col + e];
                if (p.res != nullptr) v += p.res[off];
                if (p.shuffle) {  // channel c*4 + dy*2 + dx of pixel (y, x) -> channel c of pixel (2y + dy, 2x + dx)
                  const long long px = orow[hr], xx = px % p.W, yy = (px / p.W) % p.H, b = px / (static_cast<long long>(p.W) * p.H);
                  const int ch = col + e;
                  off = static_cast<size_t>(((b * 2 * p.H + 2 * yy + ((ch >> 1) & 1)) * 2 * p.W + 2 * xx + (ch & 1)) * (p.N / 4) + (ch >> 2));
                }
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
            if (p.yh != nullptr) {  // GELU, stored as the operand planes of the next 1x1 convolution
              const float g0 = gelu_erf(o.x), g1 = gelu_erf(o.y);
              const float h0 = bf16_round(g0), h1 = bf16_round(g1);
              *reinterpret_cast<uint32_t*>(p.yh + off) = pack_bf16(h0, h1);
              if (p.yl != nullptr) *reinterpret_cast<uint32_t*>(p.yl + off) = pack_bf16(g0 - h0, g1 - h1);
              continue;
            }
            if (p.res != nullptr) {
              const float2 r2 = *reinterpret_cast<const float2*>(p.res + off);
              o.x += r2.x; o.y += r2.y;
            }
            *reinterpret_cast<float2*>(p.y + off) = o;
            acc[4 * j + 2 * hr] = o.x; acc[4 * j + 2 * hr + 1] = o.y;  // y, for the statistics (the next tile overwrites acc)
          }
        }
        if (BN != 16 && p.stats != nullptr) {
          // the warp's 16 pixels of columns col, col + 1: sum over the 8 row groups (lane >> 2; the xor tree leaves it in
          // every lane), then M2 about the warp's own mean.  Lanes 0-3 publish {sum, M2}.
          float s0 = acc[4 * j] + acc[4 * j + 2], s1 = acc[4 * j + 1] + acc[4 * j + 3];
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, o);
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
          }
          const float m0 = s0 * (1.f / 16), m1 = s1 * (1.f / 16);
          const float d00 = acc[4 * j] - m0, d01 = acc[4 * j + 2] - m0;
          const float d10 = acc[4 * j + 1] - m1, d11 = acc[4 * j + 3] - m1;
          float q0 = fmaf(d01, d01, d00 * d00), q1 = fmaf(d11, d11, d10 * d10);
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
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
            // the tile's {sum, M2} from the eight warps' {sum, M2} of 16 pixels each (Chan et al.), in warp order
            float sw[8], s = 0.f, m2 = 0.f;
#pragma unroll
            for (int wq = 0; wq < 8; ++wq) {
              const float2 v = *reinterpret_cast<const float2*>(stat_smem + ((wq * BN) + col) * 2);
              sw[wq] = v.x;
              s += v.x; m2 += v.y;
            }
            const float mean = s * (1.f / 128);
#pragma unroll
            for (int wq = 0; wq < 8; ++wq) {
              const float d = fmaf(sw[wq], 1.f / 16, -mean);
              m2 = fmaf(16.f * d, d, m2);
            }
            *reinterpret_cast<float2*>(p.stats + (stat_row * p.N + n0 + col) * 2) = make_float2(s, m2);
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
// ksize 2: nn.PixelUnshuffle(2) of the [B, 2H, 2W, C_in] input (Paella in_block), column c*4 + dy*2 + dx of output pixel
// (y, x) = x[2y + dy, 2x + dx, c].
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
    if (k < K && ksize == 2) {
      v = x[((b * 2 * H + 2 * oy + ((k >> 1) & 1)) * 2 * W + 2 * ox + (k & 1)) * Cin + (k >> 2)];
    } else if (k < K) {
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

template <int BN>
int launch_conv(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh, const CUtensorMap& bl,
                const ConvParams& p, cudaStream_t s) {
  constexpr auto kern = conv_tc_kernel<BN>;
  if (int rc = set_max_dynamic_smem<kern>(Ring<BN>::kSmemBytes)) return rc;
  const int total = p.num_m * p.num_n;
  const int grid = total < sm_count() ? total : sm_count();
  pdl_launch(grid, tc::kThreads, Ring<BN>::kSmemBytes, s)(kern, ah, al, bh, bl, p);
  return check_launch("conv_tc");
}

}  // namespace
}  // namespace muse

using namespace muse;

extern "C" {

// 1 if muse_conv2d_nhwc_tc handles the shape (otherwise the caller uses the fp32 SIMT kernel of conv.cu).
int muse_conv2d_tc_supported(int H, int W, int Cin, int Cout, int ksize) {
  if (ksize != 1 && ksize != 3 && ksize != 2) return 0;  // 2: the 2x2 forward-offset window of MUSE_CONV_TC_FWD2X2
  if (Cin % 64 != 0 || Cout < 1 || (Cout > 16 && Cout % 4 != 0)) return 0;
  if (W >= 128) return W % 128 == 0;
  if (W < 8 || 128 % W != 0) return 0;
  return H % (128 / W) == 0;
}

// Pixel tiles per image of muse_conv2d_nhwc_tc for this shape (= the leading extent of its stats output), 0 if unsupported.
// H, W are the OUTPUT dims; with upsample2x the tiling runs on the H/2 x W/2 input grid, four parities each.
int muse_conv2d_tc_tiles_per_image(int H, int W, int Cin, int Cout, int ksize, int upsample2x) {
  if (upsample2x) {
    if ((H | W) & 1 || ksize != 3 || Cout <= 16) return 0;
    H /= 2; W /= 2;
  }
  if (!muse_conv2d_tc_supported(H, W, Cin, Cout, ksize)) return 0;
  return (upsample2x ? 4 : 1) * (H * W / 128);
}

// mode: enum muse_conv_tc_mode of include/muse_b200.h.  MUSE_CONV_TC_UPSAMPLE2X: y / res / stats are at the output
// resolution [B,H,W,Cout], the x planes at the input resolution.  MUSE_CONV_TC_SINGLE_PASS: bf16-operand accuracy (~4e-3
// per layer instead of ~2e-5).
// x_hi/x_lo: bf16 [B,H,W,Cin]; w_hi/w_lo: bf16 [Cout, k*k*Cin] (tap-major, then input channel); y fp32 [B,H,W,Cout].
}  // extern "C"

namespace {
// muse_conv2d_nhwc_tc, and with yh != nullptr muse_conv2d_nhwc_tc_gelu_split
int conv_tc(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, const float* bias, const float* res,
            float* y, bf16* yh, bf16* yl, float* stats, int B, int H, int W, int Cin, int Cout, int ksize, int mode,
            cudaStream_t s) {
  if (B <= 0) return MUSE_OK;
  const int geometry = mode & MUSE_CONV_TC_GEOMETRY;
  const int shuffle = (mode & MUSE_CONV_TC_PIXEL_SHUFFLE) ? 1 : 0;
  if (shuffle && (Cout > 16 || Cout % 4 != 0 || res != nullptr || geometry != MUSE_CONV_TC_SAME)) {
    set_last_error("conv2d_tc: the PixelShuffle store needs C_out <= 16, C_out %% 4 == 0, no residual, stride 1");
    return MUSE_ERR_UNSUPPORTED;
  }
  if (yh != nullptr && (Cout <= 16 || res != nullptr || geometry != MUSE_CONV_TC_SAME || (mode & MUSE_CONV_TC_PER_IMAGE_WEIGHTS))) {
    set_last_error("conv2d_tc: the GELU split epilogue needs C_out > 16, no residual, a plain stride-1 convolution");
    return MUSE_ERR_UNSUPPORTED;
  }
  const int upsample2x = geometry == MUSE_CONV_TC_UPSAMPLE2X;
  const int fwd2x2 = geometry == MUSE_CONV_TC_FWD2X2;
  if (fwd2x2 != (ksize == 2)) { set_last_error("conv2d_tc: ksize 2 and MUSE_CONV_TC_FWD2X2 go together"); return MUSE_ERR_INVALID; }
  if (upsample2x) {
    if (muse_conv2d_tc_tiles_per_image(H, W, Cin, Cout, ksize, 1) == 0) {
      set_last_error("conv2d_tc: unsupported upsample shape H=%d W=%d Cin=%d Cout=%d k=%d", H, W, Cin, Cout, ksize);
      return MUSE_ERR_UNSUPPORTED;
    }
    H /= 2; W /= 2;  // the tiling / TMA grid is the input grid
  }
  if (!muse_conv2d_tc_supported(H, W, Cin, Cout, ksize)) {
    set_last_error("conv2d_tc: unsupported shape H=%d W=%d Cin=%d Cout=%d k=%d", H, W, Cin, Cout, ksize);
    return MUSE_ERR_UNSUPPORTED;
  }
  if ((reinterpret_cast<uintptr_t>(y) & 15) || (reinterpret_cast<uintptr_t>(yh) & 15) || (reinterpret_cast<uintptr_t>(yl) & 15) ||
      (bias && (reinterpret_cast<uintptr_t>(bias) & 15)) ||
      (res && (reinterpret_cast<uintptr_t>(res) & 15))) {
    set_last_error("conv2d_tc: y / bias / res must be 16B aligned");
    return MUSE_ERR_INVALID;
  }
  ConvParams p;
  p.y = y; p.bias = bias; p.res = res; p.stats = (Cout > 16 && yh == nullptr) ? stats : nullptr;
  const bool single_pass = (mode & MUSE_CONV_TC_SINGLE_PASS) != 0;
  p.yh = yh; p.yl = single_pass ? nullptr : yl; p.shuffle = shuffle;
  p.N = Cout; p.H = H; p.W = W; p.Cin = Cin; p.ksize = ksize;
  const int tile_px = 128;
  p.tile_w = W >= tile_px ? tile_px : W;
  p.tile_h = tile_px / p.tile_w;
  p.tiles_x = W / p.tile_w;
  p.tiles_per_img = p.tiles_x * (H / p.tile_h);
  p.num_m = B * p.tiles_per_img;
  p.up = upsample2x ? 1 : 0;
  p.fwd2x2 = fwd2x2;
  p.wbatch = (mode & MUSE_CONV_TC_PER_IMAGE_WEIGHTS) ? 1 : 0;
  p.tile_w_log2 = 0;
  while ((1 << p.tile_w_log2) < p.tile_w) ++p.tile_w_log2;
  if (p.up && (1 << p.tile_w_log2) != p.tile_w) { set_last_error("conv2d_tc: upsample needs a power-of-two tile width"); return MUSE_ERR_UNSUPPORTED; }
  const int BN = Cout >= 256 ? 256 : (Cout > 16 ? 128 : 16);
  p.num_n = ceil_div(Cout, BN);
  p.cchunks = Cin / BK;
  const int taps = (p.up || p.fwd2x2) ? 4 : ksize * ksize;
  p.passes = single_pass ? 1 : 3;
  p.num_kb = taps * p.cchunks * p.passes;
  if (p.passes == 1) { x_lo = x_hi; w_lo = w_hi; }  // the lo maps are never dereferenced; keep the encodes valid

  CUtensorMap ah, al, bh, bl;
  const long long px = 2LL * Cin;  // bytes per pixel
  const long long K = static_cast<long long>(taps) * Cin;
  const long long wrows = static_cast<long long>(Cout) * (p.up ? 4 : 1);
  int rc;
  if ((rc = make_tmap(&ah, "conv2d_tc", CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, x_hi, {Cin, W, H, B}, {px, px * W, px * W * H},
                           {64, p.tile_w, p.tile_h, 1})))
    return rc;
  if ((rc = make_tmap(&al, "conv2d_tc", CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, x_lo, {Cin, W, H, B}, {px, px * W, px * W * H},
                           {64, p.tile_w, p.tile_h, 1})))
    return rc;
  if ((rc = make_tmap(&bh, "conv2d_tc", CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, w_hi, {K, wrows, p.wbatch ? B : 1}, {2 * K, 2 * K * wrows}, {64, BN, 1})))
    return rc;
  if ((rc = make_tmap(&bl, "conv2d_tc", CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, w_lo, {K, wrows, p.wbatch ? B : 1}, {2 * K, 2 * K * wrows}, {64, BN, 1})))
    return rc;
  if (BN == 256) return launch_conv<256>(ah, al, bh, bl, p, s);
  if (BN == 128) return launch_conv<128>(ah, al, bh, bl, p, s);
  return launch_conv<16>(ah, al, bh, bl, p, s);
}
}  // namespace

extern "C" {

int muse_conv2d_nhwc_tc(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, const float* bias, const float* res,
                        float* y, float* stats, int B, int H, int W, int Cin, int Cout, int ksize, int mode, void* stream) {
  return conv_tc(x_hi, x_lo, w_hi, w_lo, bias, res, y, nullptr, nullptr, stats, B, H, W, Cin, Cout, ksize, mode,
                 static_cast<cudaStream_t>(stream));
}

// y = GELU(conv(x) + bias) written as bf16 planes y_hi [B,H,W,Cout] (+ y_lo unless MUSE_CONV_TC_SINGLE_PASS), the operands
// of the next tensor-core convolution: the c -> 4c Linear + GELU of the Paella ResBlock.  MUSE_CONV_TC_SAME only.
int muse_conv2d_nhwc_tc_gelu_split(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, const float* bias,
                                   void* y_hi, void* y_lo, int B, int H, int W, int Cin, int Cout, int ksize, int mode,
                                   void* stream) {
  if (y_hi == nullptr || ((mode & MUSE_CONV_TC_SINGLE_PASS) == 0 && y_lo == nullptr)) {
    set_last_error("conv2d_tc_gelu_split: y_hi (and y_lo unless single-pass) are required");
    return MUSE_ERR_INVALID;
  }
  return conv_tc(x_hi, x_lo, w_hi, w_lo, bias, nullptr, nullptr, reinterpret_cast<bf16*>(y_hi), reinterpret_cast<bf16*>(y_lo),
                 nullptr, B, H, W, Cin, Cout, ksize, mode, static_cast<cudaStream_t>(stream));
}

// x fp32 [B,H,W,Cin] with k*k*Cin <= 64 -> hi, lo bf16 [B,H,W,64]: row = the k*k*Cin taps of the pixel (tap-major), zero padded;
// ksize 2: x is [B,2H,2W,Cin] and the row is its PixelUnshuffle(2) (column c*4 + dy*2 + dx)
int muse_im2col_split_nhwc(const float* x, void* hi, void* lo, int B, int H, int W, int Cin, int ksize, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (ksize * ksize * Cin > 64 || (ksize != 1 && ksize != 2 && ksize != 3)) {
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
int muse_split_s2d_bf16_nhwc(const float* x, void* hi, void* lo, int B, int Ho, int Wo, int C, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (C % 8 != 0) { set_last_error("split_s2d: C must be a multiple of 8"); return MUSE_ERR_UNSUPPORTED; }
  const long long total8 = static_cast<long long>(B) * Ho * Wo * 4 * (C / 8);
  if (total8 <= 0) return MUSE_OK;
  pdl_launch(static_cast<unsigned>(ceil_div_ll(total8, 256)), 256, 0, s)(split_s2d_kernel, x, reinterpret_cast<bf16*>(hi),
                                                                                   reinterpret_cast<bf16*>(lo), total8, Ho, Wo, C);
  return check_launch("split_s2d");
}

// out_f32 given: plain fp32 softmax (hi / lo unused); else the bf16 hi/lo planes
int muse_softmax_split_rows(const float* x, void* hi, void* lo, float* out_f32, long long rows, int n, float scale, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows <= 0 || n <= 0) return MUSE_OK;
  if (out_f32 == x) { set_last_error("softmax: in-place output is not supported"); return MUSE_ERR_INVALID; }
  pdl_launch(static_cast<unsigned>(ceil_div_ll(rows, 8)), 256, 0, s)(softmax_split_kernel, x, reinterpret_cast<bf16*>(hi),
                                                                                   reinterpret_cast<bf16*>(lo), out_f32, rows, n, scale);
  return check_launch("softmax_split");
}

// x fp32 [B, H/(1+up), W/(1+up), C] -> hi, lo bf16 [B,H,W,C]
int muse_split_bf16_nhwc(const float* x, void* hi, void* lo, int B, int H, int W, int C, int upsample2x, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (C % 8 != 0) { set_last_error("split_bf16: C must be a multiple of 8"); return MUSE_ERR_UNSUPPORTED; }
  if (upsample2x && ((H | W) & 1)) { set_last_error("split_bf16: upsample2x needs even output dims"); return MUSE_ERR_INVALID; }
  const long long total8 = static_cast<long long>(B) * H * W * (C / 8);
  if (total8 <= 0) return MUSE_OK;
  pdl_launch(static_cast<unsigned>(ceil_div_ll(total8, 256)), 256, 0, s)(split_bf16_kernel, x, reinterpret_cast<bf16*>(hi),
                                                                                    reinterpret_cast<bf16*>(lo), total8, H, W, C, upsample2x);
  return check_launch("split_bf16");
}

}  // extern "C"
