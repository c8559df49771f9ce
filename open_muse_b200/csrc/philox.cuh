// Dropout keep masks: Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011) and the ONE
// mapping from (seed, site, coordinates) to keep bits.  Every dropout kernel (attention_tc.cu, elementwise.cu, norm.cu,
// uvit.cu) draws its bits through the functions below; the CPU restatement in tests/test_dropout_cpu.py is the only
// other copy.
//
//   key     = the 64-bit seed (lo, hi words), read by the kernels from device memory (drawn on the device per forward)
//   counter = (c0, c1, c2, site): the last word is the site id, unique within one forward (layer x site kind)
//
// Site ids.  MaskGitTransformer: 0 the embedding; layer i: 1 + 3 i self-attention, 2 + 3 i cross-attention, 3 + 3 i FFN.
// MaskGiTUViT_v2: unit j = down pairs 0 .. R-1, then layers R .. R+L-1, then up pairs R+L .. 2R+L-1 (R = num_res_blocks,
// L = num_hidden_layers) owns 3 j + kind; a ResBlock + AttentionBlock2D pair: 0 the ResBlock's dropout after GRN (an
// elementwise site over [B*h*w, 4C]), 1 attention, 2 crossattention; a layer: 0 attention, 1 crossattention, 2 FFN.
//   output  = four 32-bit words = eight 16-bit uniforms u, lane L = bits 16 (L & 1) .. of word L >> 1
//   keep    = u >= t, with t = round(p * 65536); kept values are scaled by 65536 / (65536 - t)
// With 16-bit uniforms the effective rate is p_eff = t / 65536 (|p_eff - p| <= 2^-17 = 7.6e-6) and the scale makes the
// expectation exactly the input for this generator.
//
// Attention site, element (q, k) of head (b, h), Skv columns: counter = (call, q, b * nh + h, site) with
//   call = (k / 64) * 8 + ((k % 64) / 32) * 4 + (k % 8) / 2  and lane 2 ((k / 8) % 4) + (k % 2):
// a wgmma accumulator fragment holds columns 8 g + c, 8 g + c + 1 (g = 0..7, c = 2 (lane % 4)) of its rows, so one call
// covers exactly the 8 columns {8 g + c, +1 : g = 4 G .. 4 G + 3} a thread owns in one 32-column half of a 64-column tile.
// Elementwise site, element (row, col): counter = (col / 8, row, 0, site), lane col % 8.
//
// Stored masks: uint32 words, rows padded to 32 bits, bit k % 32 of word k / 32 set = element k kept (pad bits are 0).
#pragma once
#include <stdint.h>

namespace muse {
namespace philox {

struct U4 {
  uint32_t x, y, z, w;
};

__host__ __device__ __forceinline__ uint32_t mulhilo(uint32_t a, uint32_t b, uint32_t& hi) {
#ifdef __CUDA_ARCH__
  hi = __umulhi(a, b);
  return a * b;
#else
  const uint64_t p = static_cast<uint64_t>(a) * b;
  hi = static_cast<uint32_t>(p >> 32);
  return static_cast<uint32_t>(p);
#endif
}

// Philox4x32 with 10 rounds (Random123's philox4x32_R(10, ...))
__host__ __device__ __forceinline__ U4 philox4x32_10(U4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    uint32_t hi0, hi1;
    const uint32_t lo0 = mulhilo(0xD2511F53u, c.x, hi0);
    const uint32_t lo1 = mulhilo(0xCD9E8D57u, c.z, hi1);
    c = U4{hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0};
  }
  return c;
}

// t = round(p * 65536): keep iff the 16-bit uniform is >= t
__host__ __device__ __forceinline__ uint32_t threshold(float p) {
  const float t = rintf(p * 65536.0f);
  return t <= 0.f ? 0u : (t >= 65536.f ? 65536u : static_cast<uint32_t>(t));
}
__host__ __device__ __forceinline__ float keep_scale(uint32_t t) { return t >= 65536u ? 0.f : 65536.0f / (65536u - t); }

// The 8 keep bits of one call (bit L = lane L kept)
__host__ __device__ __forceinline__ uint32_t keep8(U4 c, uint64_t seed, uint32_t t) {
  const U4 o = philox4x32_10(c, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  const uint32_t w[4] = {o.x, o.y, o.z, o.w};
  uint32_t bits = 0;
#pragma unroll
  for (int l = 0; l < 8; ++l) bits |= static_cast<uint32_t>(((w[l >> 1] >> (16 * (l & 1))) & 0xFFFFu) >= t) << l;
  return bits;
}

// Attention: the keep bits of call `call` of row q of head bh = b * nh + h (lane L of the call is bit L)
__host__ __device__ __forceinline__ uint32_t attn_keep8(uint64_t seed, uint32_t site, uint32_t bh, uint32_t q, uint32_t call,
                                                        uint32_t t) {
  return keep8(U4{call, q, bh, site}, seed, t);
}

// Elementwise: the keep bits of columns 8 chunk .. 8 chunk + 7 of `row` (bit j = column 8 chunk + j)
__host__ __device__ __forceinline__ uint32_t elem_keep8(uint64_t seed, uint32_t site, uint32_t row, uint32_t chunk,
                                                        uint32_t t) {
  return keep8(U4{chunk, row, 0u, site}, seed, t);
}

// Elementwise dropout fused into a pass over [rows, cols] (cols % 8 == 0): the pass handles 8 columns at a time, i.e.
// one Philox call and one byte of the row's keep-bit words (little-endian: byte k of a row = columns 8 k .. 8 k + 7).
// The forward draws and writes the bytes (and zeroes the pad bytes of the row's last word), the backward reads them.
struct ElemDrop {
  uint8_t* bits;                   // [rows][row_bytes]
  const unsigned long long* seed;  // forward only: device pointer to the 64-bit key
  uint32_t site, thresh;
  float scale;
  int row_bytes;                   // 4 * ceil(cols / 32)
};

inline ElemDrop elem_drop(void* bits, const unsigned long long* seed, int site, float p, int cols) {
  ElemDrop d;
  d.bits = static_cast<uint8_t*>(bits);
  d.seed = seed;
  d.site = static_cast<uint32_t>(site);
  d.thresh = threshold(p);
  d.scale = keep_scale(d.thresh);
  d.row_bytes = 4 * ((cols + 31) / 32);
  return d;
}

// the factor of element j (0..7) of a chunk with keep byte kb: scale if kept, else 0
__host__ __device__ __forceinline__ float keep_z(uint32_t kb, int j, float scale) { return ((kb >> j) & 1u) ? scale : 0.f; }

}  // namespace philox
}  // namespace muse
