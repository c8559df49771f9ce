// wgmma / TMA attention for head_dim 64, 48, 128 and 96 (sm_90a): forward, dQ and dK/dV kernels.
// Replaces the reference's materialised attention (muse/modeling_transformer.py:221-241) and its autograd backward.
//
// One CTA = one (batch, head) x one 64-row tile of the "owned" sequence dimension: a consumer warpgroup that issues the
// wgmma and does the softmax math, and a producer warp that streams the looped 64-row tiles through a ring of
// shared-memory stages with TMA (`full` / `empty` mbarriers per stage).  Score-like products (S, dP) stay in the wgmma
// accumulator registers; the softmax math runs on the fragment (row statistics with quad shuffles), and P / dS are
// packed to bf16 in registers and fed straight back as the register A operand of the accumulating products, whose
// accumulators (O, dQ, dK, dV) stay in registers for the whole loop and are stored once at the end.
//
//   forward  : owned = q rows.   S = Q K_j^T -> online softmax (fp32) -> P (bf16 regs) -> O += P V_j
//   dQ       : owned = q rows.   S, dP = dO V_j^T -> sweep 1: D = sum P*dP ; sweep 2: dS -> dQ += dS K_j
//   dK/dV    : owned = kv rows.  S^T = K Q_i^T, dP^T = V dO_i^T -> P^T, dS^T -> dV += P^T dO_i, dK += dS^T Q_i
// Operands are read straight from the strided [tokens, 3H] QKV projection through 3-D TMA tensor maps
// {64 head columns, S rows, B} (rows past the end of a sequence are zero-filled by the TMA unit; a head wider than 64
// columns is two such boxes, 8 KB apart in shared memory), with the same
// 128-byte-swizzled tiles serving as K-major or MN-major MMA operands depending on the product.
// The owned dimension is cut into ceil(S / 64) tiles of EQUAL height R = ceil(S / tiles) (S = 257 with the class token ->
// five tiles of 52 rows; S = 256 -> four of 64; the 77 text states of cross-attention -> two of 39): a tile starts at row
// i * R, its CTA loads a 64-row box (rows past R belong to the next tile or are zero-filled past the sequence), the MMAs
// run on all 64 rows, but only rows < R are kept.  The looped dimension's ragged tail is zero-filled by TMA and masked.
// Several CTAs share an SM, so one CTA's softmax math runs under another's MMAs and loads.
//
// Dropout on the probabilities (DROP = true instantiations; the DROP = false ones are the kernels without it): the forward
// draws the keep bits of its fragment with philox.cuh's attention mapping (four Philox calls per thread and 64 x 64 tile),
// stores them, and scales the bf16 P operand of O += P V by Z = keep / (1 - p) -- l and the LSE stay those of the
// undropped P.  The dQ kernel reads the bits of its rows and applies Z to dP (dP = Z (dO V^T); D = rowsum(P dP) as
// before); the dK/dV kernel, which walks S^T, has its producer warp stage each q tile's 64 x 64 bits (funnel-shifted to
// the CTA's first kv row) next to lse / D and applies Z to P^T (dV) and to dP^T (dS).
#include "common.cuh"
#include "philox.cuh"
#include "ptx.cuh"
#include "tc_host.cuh"
#include "wgmma.cuh"

namespace muse {

namespace {

// Head dimension HD is a template parameter: 64 (every text-to-image / U-ViT config, BASELINE configs) or 48 (configs/imagenet.yaml:
// hidden 768, 16 heads -- the configuration training/train_maskgit_imagenet.py is written for).  For HD = 48 the TMA boxes stay
// 64 columns wide (head h starts at column 48 h; the 16 trailing columns belong to the next head or are zero-filled past the
// tensor) and simply never enter a product: Q K^T / dO V^T run 3 instead of 4 k-steps, and the accumulate MMAs (P V, dS K,
// dS^T Q, P^T dO) have N = 48, reading the first 48 columns of their MN-major 128-byte rows.
// HD = 128 and 96 (hidden 1024 / 8 heads, 768 / 6 heads) go past one box: a Q / K / V / dO tile is two 64-column boxes,
// loaded at columns h HD and h HD + 64 and stored 8 KB apart.  The score products run 8 (HD 128) or 6 (HD 96) k-steps,
// the K-major descriptors moving to the second box from k-step 4 on; the accumulate MMAs have N = 128 / 96 and read the
// second box through the MN-major descriptor's 64-column chunk stride (LBO = 8 KB).  For HD = 96 the second box's last
// 32 columns belong to the next head (or are zero-filled past the tensor) and never enter a product, as for HD = 48.
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// exp2 on the SFU without the denormal/range fix-ups of exp2f (inputs here are <= 0 or bounded scores)
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

constexpr int kBM = 64;                 // owned rows per CTA (one consumer warpgroup)
constexpr int kBN = 64;                 // rows of a looped tile
constexpr int kConsumers = 128;         // threads of the consumer warpgroup; the producer warp follows
constexpr int kThreads = kConsumers + 32;
constexpr int kStages = 2;              // ring stages of looped tiles
constexpr int kTile = 64 * 64 * 2;      // one 64-row x 64-column bf16 TMA box, 8 KB
// one 64-row Q / K / V / dO tile of head width HD: ceil(HD / 64) boxes, kTile apart
template <int HD>
constexpr int kHdTile = (HD + 63) / 64 * kTile;

struct TcParams {
  int Sq, Skv, nh;
  int tile_rows;  // R: owned rows per CTA (<= 64)
  float scale;
  // outputs / side inputs (plain global pointers; rows addressed as b*S + s)
  bf16* out0;  long long out0_rs;   // fwd: O ; dq: dQ ; dkdv: dK
  bf16* out1;  long long out1_rs;   // dkdv: dV
  float* lse;                        // [B, nh, Sq]
  float* dvec;                       // [B, nh, Sq]
  // dropout on the probabilities (DROP instantiations only): keep bits [B, nh, Sq, bwords] (philox.cuh), written by the
  // forward from (seed, site), read by both backward kernels
  uint32_t* bits;
  const unsigned long long* seed;
  uint32_t site, thresh;
  int bwords;   // ceil(Skv / 32)
  float dscale; // 1 / (1 - p_eff)
};

// Barriers behind the tiles: own (the CTA's owned tiles, loaded once), full[kStages], empty[kStages].  Step st of the loop
// uses stage st % kStages in phase (st / kStages) & 1.  `empty` gets one arrival from the consumer warpgroup once the
// MMAs that read the stage have completed.
struct Bars {
  uint64_t* own;
  uint64_t* full;
  uint64_t* empty;
  __device__ explicit Bars(uint8_t* p)
      : own(reinterpret_cast<uint64_t*>(p)), full(own + 1), empty(own + 1 + kStages) {}
  __device__ void init() const {  // one thread, before the __syncthreads that publishes the barriers
    ptx::mbar_init(own, 1);
    for (int i = 0; i < kStages; ++i) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], 1);
    }
    ptx::fence_barrier_init();
  }
  // producer: the consumers have released the stage of step st (i.e. finished step st - kStages)
  __device__ void wait_empty(int st) const { ptx::mbar_wait(&empty[st % kStages], ((st / kStages) & 1) ^ 1); }
  __device__ void wait_full(int st) const { ptx::mbar_wait(&full[st % kStages], (st / kStages) & 1); }
  // consumer thread 0, once the MMAs of step st have completed
  __device__ void release(int st) const { ptx::mbar_arrive(&empty[st % kStages]); }
};
constexpr int kBarBytes = 64;

// ------------------------------------------------------------------------------------------------ wgmma helpers
// The MMAs always run the full 64-row looped tile: rows past the sequence are zero-filled by TMA and their score columns
// are masked, so a ragged tail costs MMA work but no code path.  (Shrinking the MMA to the tail puts wgmma on a
// data-dependent branch, and ptxas then serialises every wgmma of the kernel.)  Each step's MMAs are retired before
// the next step's are issued, for the same reason: ptxas serialises a pipeline stage across which the next step's
// fragments are defined.
// d = A B^T for the 64 rows of A and of B, both K-major with 16 KS columns (k-steps 4 .. 7 in the second box)
template <int KS>
__device__ __forceinline__ void issue_scores(float (&d)[32], uint32_t a, uint32_t b) {
  constexpr int KS0 = KS < 4 ? KS : 4;
#pragma unroll
  for (int ks = 0; ks < KS0; ++ks) ptx::Wgmma<64, 0, 0>::run(d, ptx::desc_kmajor(a, ks), ptx::desc_kmajor(b, ks), ks > 0);
#pragma unroll
  for (int ks = 0; ks < KS - KS0; ++ks)
    ptx::Wgmma<64, 0, 0>::run(d, ptx::desc_kmajor(a + kTile, ks), ptx::desc_kmajor(b + kTile, ks), 1);
}

// Loads the 64-row tile of head columns [col, col + HD) at row `row` of batch b: one TMA box per 64 columns.
template <int HD>
__device__ __forceinline__ void load_tile(uint8_t* dst, const CUtensorMap* m, uint64_t* bar, int col, int row, int b) {
#pragma unroll
  for (int x = 0; x < kHdTile<HD> / kTile; ++x) ptx::tma_load_3d(dst + x * kTile, m, bar, col + 64 * x, row, b);
}

// d += A B: A the bf16 register fragment of a 64 x 64 product (wgmma.cuh), B MN-major with HD columns (past 64 columns
// the descriptor's LBO steps to the second box)
template <int HD>
__device__ __forceinline__ void issue_acc(float (&d)[HD / 2], const uint32_t (&a)[16], uint32_t b) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) ptx::WgmmaRs<HD, 1>::run(d, a + 4 * ks, ptx::desc_mnmajor(b, ks), 1);
}

// reductions over the four threads that hold one fragment row
__device__ __forceinline__ float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
__device__ __forceinline__ float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// bf16 store of an [64 x HD] accumulator fragment to rows (fragment row) of `base` (row stride rs) that are < rows_ok,
// row r scaled by sc[0], row r + 8 by sc[1]
template <int HD>
__device__ __forceinline__ void store_acc(const float (&d)[HD / 2], bf16* base, long long rs, int rows_ok,
                                          const float (&sc)[2]) {
  const int r = ptx::frag_row(), c = ptx::frag_col();
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int rr = r + 8 * hr;
    if (rr >= rows_ok) continue;
    bf16* dst = base + rr * rs;
#pragma unroll
    for (int j = 0; j < HD / 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j + c) = pack_bf16(d[4 * j + 2 * hr] * sc[hr], d[4 * j + 2 * hr + 1] * sc[hr]);
  }
}

// column (within the 64-column tile) of fragment element i
__device__ __forceinline__ int frag_col_of(int i) { return 8 * (i >> 2) + ptx::frag_col() + (i & 1); }

// ------------------------------------------------------------------------------------------------ dropout helpers
// The keep bits a thread owns in one 32-column half G of a tile row are the 8 lanes of one Philox call (philox.cuh):
// lane 2 (g % 4) + e is column 8 g + c + e (g = 4 G .. 4 G + 3, e = 0, 1).  As a stored word they sit at bit
// 8 (g % 4) + c + e, so a word shifted right by c and a call's lanes are read the same way: lane l <-> bit 8 (l >> 1) + (l & 1).
__device__ __forceinline__ uint32_t lanes_to_word(uint32_t kb, int c) {
  return ((kb & 3u) | ((kb & 0xCu) << 6) | ((kb & 0x30u) << 12) | ((kb & 0xC0u) << 18)) << c;
}
// keep bit of accumulator element i, from the shifted words w[hr][G] of its rows
__device__ __forceinline__ bool kept(const uint32_t (&w)[2][2], int i) {
  return (w[(i >> 1) & 1][i >> 4] >> (8 * ((i >> 2) & 3) + (i & 1))) & 1u;
}

// ------------------------------------------------------------------------------------------------ forward
// smem: Q T | kStages x {K T, V T} | barriers, T = kHdTile<HD> (8 KB up to HD 64: three CTAs per SM; 16 KB past it,
// 80 KB per CTA: two)
template <int HD>
constexpr int fwd_smem() { return kHdTile<HD> + kStages * 2 * kHdTile<HD> + kBarBytes; }

template <int HD, bool DROP>
__global__ void __launch_bounds__(kThreads, HD > 64 ? 2 : 3)
attn_fwd_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, const TcParams p) {
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t smem[];  // 128B-swizzled tiles need 1024 B alignment
  if ((ptx::smem_u32(smem) & 1023u) != 0) __trap();
  constexpr int T = kHdTile<HD>;
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + T;
  const Bars bars(sKV + kStages * 2 * T);

  const int tid = threadIdx.x;
  const int q0 = blockIdx.x * p.tile_rows, h = blockIdx.y, b = blockIdx.z;
  const int rows_here = min(p.tile_rows, p.Sq - q0);
  if (tid == 0) bars.init();
  __syncthreads();
  pdl_wait();  // everything above touches only shared memory / kernel parameters
  const int ntiles = ceil_div(p.Skv, kBN);

  if (tid >= kConsumers) {  // producer warp: Q once, then K_j / V_j through the ring
    if (tid == kConsumers) {
      ptx::mbar_expect_tx(bars.own, T);
      load_tile<HD>(sQ, &tmQ, bars.own, h * HD, q0, b);
      for (int j = 0; j < ntiles; ++j) {
        bars.wait_empty(j);
        uint64_t* full = &bars.full[j % kStages];
        uint8_t* sK = sKV + (j % kStages) * 2 * T;
        ptx::mbar_expect_tx(full, 2 * T);
        load_tile<HD>(sK, &tmK, full, h * HD, j * kBN, b);
        load_tile<HD>(sK + T, &tmV, full, h * HD, j * kBN, b);
      }
    }
    return;
  }

  const float sl2 = p.scale * kLog2e;
  const uint32_t bh = static_cast<uint32_t>(b * p.nh + h);
  unsigned long long seed = 0;
  if constexpr (DROP) seed = *p.seed;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // per fragment row r, r + 8; l is this thread's partial sum
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  ptx::mbar_wait(bars.own, 0);
  for (int j = 0; j < ntiles; ++j) {
    const int nvalid = min(kBN, p.Skv - j * kBN);
    const uint32_t sK = ptx::smem_u32(sKV + (j % kStages) * 2 * T);
    float s[32];
    bars.wait_full(j);
    ptx::wgmma_fence();
    issue_scores<HD / 16>(s, ptx::smem_u32(sQ), sK);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_operand(s);
    if (nvalid < kBN) {  // ragged last tile only
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] = frag_col_of(i) < nvalid ? s[i] : -INFINITY;
    }
    float alpha[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float raw = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) raw = fmaxf(raw, fmaxf(s[4 * jj + 2 * hr], s[4 * jj + 2 * hr + 1]));
      // Lazy running maximum: the reference point m only moves when the tile's maximum exceeds it by more than 8 (log2
      // units), i.e. P entries stay below 2^8 -- harmless in bf16 / fp32 -- and the final 1 / l normalisation and the
      // LSE (m + log2 l) are exact for any reference point.  Most tiles then leave m alone and alpha is exactly 1.
      const float cand = quad_max(raw) * sl2;
      const float mx = (cand > m[hr] + 8.0f) ? cand : m[hr];
      alpha[hr] = ex2(m[hr] - mx);  // 0 on the first tile (m = -inf), 1 when the reference point stays
      m[hr] = mx;
    }
    uint32_t pa[16];
    float ls[2] = {0.f, 0.f};
    uint32_t kw[2][2];  // keep bits of rows r, r + 8 x column halves, as (unshifted) words
    if constexpr (DROP) {
      const int c = ptx::frag_col();
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const uint32_t q = q0 + ptx::frag_row() + 8 * hr;
#pragma unroll
        for (int G = 0; G < 2; ++G) {
          kw[hr][G] = lanes_to_word(philox::attn_keep8(seed, p.site, bh, q, 8 * j + 4 * G + c / 2, p.thresh), 0);
          // the quad's four threads hold the four column pairs of the word: OR them, thread 2 hr + G stores it
          uint32_t w = kw[hr][G] << c;
          w |= __shfl_xor_sync(0xffffffffu, w, 1);
          w |= __shfl_xor_sync(0xffffffffu, w, 2);
          const int word = 2 * j + G, nv = p.Skv - 32 * word;
          if ((tid & 3) == 2 * hr + G && ptx::frag_row() + 8 * hr < rows_here && word < p.bwords)
            p.bits[(static_cast<long long>(bh) * p.Sq + q) * p.bwords + word] = nv >= 32 ? w : w & ((1u << nv) - 1u);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {  // s[2 i], s[2 i + 1] lie in row r + 8 (i & 1)
      float p0 = ex2(fmaf(s[2 * i], sl2, -m[i & 1])), p1 = ex2(fmaf(s[2 * i + 1], sl2, -m[i & 1]));
      ls[i & 1] += p0 + p1;
      if constexpr (DROP) {  // l keeps the undropped sum; only the P V operand is dropped and rescaled
        p0 = kept(kw, 2 * i) ? p0 * p.dscale : 0.f;
        p1 = kept(kw, 2 * i + 1) ? p1 * p.dscale : 0.f;
      }
      pa[i] = pack_bf16(p0, p1);
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) l[hr] = fmaf(l[hr], alpha[hr], ls[hr]);
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    ptx::wgmma_fence();
    issue_acc<HD>(o, pa, sK + T);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_operand(o);
    if (tid == 0) bars.release(j);
  }
  // epilogue: O / l -> bf16 rows, LSE
  const int r = ptx::frag_row();
  float inv[2];
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const float lsum = quad_sum(l[hr]);
    inv[hr] = 1.f / lsum;
    if ((tid & 3) == 0 && r + 8 * hr < rows_here)
      p.lse[(static_cast<long long>(b) * p.nh + h) * p.Sq + q0 + r + 8 * hr] = (m[hr] + log2f(lsum)) * kLn2;
  }
  store_acc<HD>(o, p.out0 + (static_cast<long long>(b) * p.Sq + q0) * p.out0_rs + h * HD, p.out0_rs, rows_here, inv);
}

// ------------------------------------------------------------------------------------------------ backward: dQ
// The ring streams the K/V tiles twice: sweep 1 accumulates D = sum_j P dP per row, sweep 2 forms dS and dQ.
// smem: Q T | dO T | kStages x {K_j T, V_j T} | barriers (48 KB up to HD 64, three CTAs per SM; 96 KB past it, two)
template <int HD>
constexpr int dq_smem() { return 2 * kHdTile<HD> + kStages * 2 * kHdTile<HD> + kBarBytes; }

template <int HD, bool DROP>
__global__ void __launch_bounds__(kThreads, HD > 64 ? 2 : 3)
attn_bwd_dq_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO,
                      const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                      const TcParams p) {
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((ptx::smem_u32(smem) & 1023u) != 0) __trap();
  constexpr int T = kHdTile<HD>;
  uint8_t* sQ = smem;
  uint8_t* sdO = smem + T;
  uint8_t* sKV = smem + 2 * T;
  const Bars bars(sKV + kStages * 2 * T);

  const int tid = threadIdx.x;
  const int q0 = blockIdx.x * p.tile_rows, h = blockIdx.y, b = blockIdx.z;
  const int rows_here = min(p.tile_rows, p.Sq - q0);
  if (tid == 0) bars.init();
  __syncthreads();
  pdl_wait();  // everything above touches only shared memory / kernel parameters
  const int ntiles = ceil_div(p.Skv, kBN);
  const int nsteps = 2 * ntiles;

  if (tid >= kConsumers) {  // producer warp: Q, dO once, then K_j / V_j twice through the ring
    if (tid == kConsumers) {
      ptx::mbar_expect_tx(bars.own, 2 * T);
      load_tile<HD>(sQ, &tmQ, bars.own, h * HD, q0, b);
      load_tile<HD>(sdO, &tmdO, bars.own, h * HD, q0, b);
      for (int st = 0; st < nsteps; ++st) {
        bars.wait_empty(st);
        uint64_t* full = &bars.full[st % kStages];
        uint8_t* sK = sKV + (st % kStages) * 2 * T;
        const int j = st % ntiles;
        ptx::mbar_expect_tx(full, 2 * T);
        load_tile<HD>(sK, &tmK, full, h * HD, j * kBN, b);
        load_tile<HD>(sK + T, &tmV, full, h * HD, j * kBN, b);
      }
    }
    return;
  }

  const int r = ptx::frag_row(), c = ptx::frag_col();
  const long long stat_base = (static_cast<long long>(b) * p.nh + h) * p.Sq + q0;
  const float sl2 = p.scale * kLog2e;
  float lse2[2], dsum[2] = {0.f, 0.f};
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) lse2[hr] = (r + 8 * hr < rows_here) ? p.lse[stat_base + r + 8 * hr] * kLog2e : 0.f;
  float dq[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) dq[i] = 0.f;
  ptx::mbar_wait(bars.own, 0);
  for (int st = 0; st < nsteps; ++st) {
    const int j = st % ntiles;
    const int nvalid = min(kBN, p.Skv - j * kBN);
    const uint32_t sK = ptx::smem_u32(sKV + (st % kStages) * 2 * T);
    float s[32], dp[32];
    uint32_t kw[2][2];  // keep bits of rows r, r + 8 x column halves of tile j, shifted to this thread's column pairs
    if constexpr (DROP) {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr)
#pragma unroll
        for (int G = 0; G < 2; ++G) {
          const int word = 2 * j + G;
          kw[hr][G] = (r + 8 * hr < rows_here && word < p.bwords) ? p.bits[(stat_base + r + 8 * hr) * p.bwords + word] >> c : 0u;
        }
    }
    bars.wait_full(st);
    ptx::wgmma_fence();
    issue_scores<HD / 16>(s, ptx::smem_u32(sQ), sK);
    issue_scores<HD / 16>(dp, ptx::smem_u32(sdO), sK + T);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_operand(s);
    ptx::fence_operand(dp);
    if constexpr (DROP) {  // dP = Z (dO V^T)
#pragma unroll
      for (int i = 0; i < 32; ++i) dp[i] = kept(kw, i) ? dp[i] * p.dscale : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = ex2(fmaf(s[i], sl2, -lse2[(i >> 1) & 1]));  // P
    if (nvalid < kBN) {  // ragged last tile only
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] = frag_col_of(i) < nvalid ? s[i] : 0.f;
    }
    if (st < ntiles) {
#pragma unroll
      for (int i = 0; i < 32; ++i) dsum[(i >> 1) & 1] = fmaf(s[i], dp[i], dsum[(i >> 1) & 1]);
      if (st == ntiles - 1) {  // D of the row, for sweep 2 and for the dK/dV kernel
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          dsum[hr] = quad_sum(dsum[hr]);
          if ((tid & 3) == 0 && r + 8 * hr < rows_here) p.dvec[stat_base + r + 8 * hr] = dsum[hr];
        }
      }
    } else {
      const float nd[2] = {-dsum[0] * p.scale, -dsum[1] * p.scale};
      uint32_t da[16];
#pragma unroll
      for (int i = 0; i < 16; ++i)
        da[i] = pack_bf16(s[2 * i] * fmaf(dp[2 * i], p.scale, nd[i & 1]), s[2 * i + 1] * fmaf(dp[2 * i + 1], p.scale, nd[i & 1]));
      ptx::wgmma_fence();
      issue_acc<HD>(dq, da, sK);  // dQ += dS K_j
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::fence_operand(dq);
    }
    if (tid == 0) bars.release(st);
  }
  const float one[2] = {1.f, 1.f};
  store_acc<HD>(dq, p.out0 + (static_cast<long long>(b) * p.Sq + q0) * p.out0_rs + h * HD, p.out0_rs, rows_here, one);
}

// ------------------------------------------------------------------------------------------------ backward: dK, dV
// Same structure as the dQ kernel, looping over 64-row q tiles; dK and dV of the CTA's kv rows in registers.  The producer
// warp also stages each q tile's lse (x log2 e) and D (x scale) as 64-float vectors next to the ring, read per column.
// With dropout the producer also stages the q tile's keep bits: 64 q rows x 2 words (the CTA's 64 kv rows).
// smem: K T | V T | kStages x {Q_i T, dO_i T} | kStages x {lse 64, D 64} floats | [kStages x 128 bit words] | barriers
template <int HD, bool DROP>
constexpr int dkdv_smem() {
  return 2 * kHdTile<HD> + kStages * 2 * kHdTile<HD> + kStages * 2 * kBN * 4 + (DROP ? kStages * 2 * kBN * 4 : 0) + kBarBytes;
}

// Past HD 64 the dK and dV accumulators (HD / 2 floats each) and the two score fragments need up to 245 registers: the
// kernel keeps its single consumer warpgroup and runs one CTA per SM (two would cap it at 168 registers and spill).
template <int HD, bool DROP>
__global__ void __launch_bounds__(kThreads, HD > 64 ? 1 : 2)
attn_bwd_dkdv_tc_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                        const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO,
                        const TcParams p) {
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((ptx::smem_u32(smem) & 1023u) != 0) __trap();
  constexpr int T = kHdTile<HD>;
  uint8_t* sK = smem;
  uint8_t* sV = smem + T;
  uint8_t* sQO = smem + 2 * T;
  float* sLD = reinterpret_cast<float*>(sQO + kStages * 2 * T);
  uint32_t* sBits = reinterpret_cast<uint32_t*>(sLD + kStages * 2 * kBN);  // DROP only: [stage][q 64][2 words]
  const Bars bars(reinterpret_cast<uint8_t*>(sLD + kStages * 2 * kBN) + (DROP ? kStages * 2 * kBN * 4 : 0));

  const int tid = threadIdx.x;
  const int kv0 = blockIdx.x * p.tile_rows, h = blockIdx.y, b = blockIdx.z;
  const int rows_here = min(p.tile_rows, p.Skv - kv0);
  if (tid == 0) bars.init();
  __syncthreads();
  pdl_wait();  // everything above touches only shared memory / kernel parameters
  const int ntiles = ceil_div(p.Sq, kBN);
  const long long stat_base = (static_cast<long long>(b) * p.nh + h) * p.Sq;

  if (tid >= kConsumers) {  // producer warp: K, V once, then {Q_i, dO_i, lse_i, D_i} through the ring
    const int lane = tid & 31;
    if (lane == 0) {
      ptx::mbar_expect_tx(bars.own, 2 * T);
      load_tile<HD>(sK, &tmK, bars.own, h * HD, kv0, b);
      load_tile<HD>(sV, &tmV, bars.own, h * HD, kv0, b);
    }
    for (int i = 0; i < ntiles; ++i) {
      bars.wait_empty(i);
      float* ld = sLD + (i % kStages) * 2 * kBN;
      for (int k = lane; k < kBN; k += 32) {
        const int qr = i * kBN + k;
        ld[k] = (qr < p.Sq) ? p.lse[stat_base + qr] * kLog2e : 0.f;
        ld[kBN + k] = (qr < p.Sq) ? p.dvec[stat_base + qr] * p.scale : 0.f;  // pre-scaled: dS = P (dP*scale - D*scale)
        if constexpr (DROP) {  // bits kv0 .. kv0 + 63 of row qr: three stored words, funnel-shifted to kv0
          uint32_t w[3] = {0u, 0u, 0u};
          const int w0 = kv0 >> 5;
          if (qr < p.Sq) {
            const uint32_t* row = p.bits + (stat_base + qr) * p.bwords;
#pragma unroll
            for (int t = 0; t < 3; ++t) w[t] = (w0 + t < p.bwords) ? row[w0 + t] : 0u;
          }
          uint32_t* bt = sBits + (i % kStages) * 2 * kBN + 2 * k;
          bt[0] = __funnelshift_r(w[0], w[1], kv0 & 31);
          bt[1] = __funnelshift_r(w[1], w[2], kv0 & 31);
        }
      }
      __syncwarp();  // the vectors are written before lane 0's arrival publishes the stage
      if (lane == 0) {
        uint64_t* full = &bars.full[i % kStages];
        uint8_t* sQ = sQO + (i % kStages) * 2 * T;
        ptx::mbar_expect_tx(full, 2 * T);
        load_tile<HD>(sQ, &tmQ, full, h * HD, i * kBN, b);
        load_tile<HD>(sQ + T, &tmdO, full, h * HD, i * kBN, b);
      }
    }
    return;
  }

  const int r = ptx::frag_row(), c = ptx::frag_col();
  const bool kv_ok = r + 8 < rows_here;  // both fragment rows are kept (rows past R belong to the next CTA)
  const float sl2 = p.scale * kLog2e;
  float dk[HD / 2], dv[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) { dk[i] = 0.f; dv[i] = 0.f; }
  ptx::mbar_wait(bars.own, 0);
  for (int i = 0; i < ntiles; ++i) {
    const int nvalid = min(kBN, p.Sq - i * kBN);
    const uint32_t sQ = ptx::smem_u32(sQO + (i % kStages) * 2 * T);
    const float* sL = sLD + (i % kStages) * 2 * kBN;
    const float* sD = sL + kBN;
    float s[32], dp[32];
    bars.wait_full(i);
    ptx::wgmma_fence();
    issue_scores<HD / 16>(s, ptx::smem_u32(sK), sQ);
    issue_scores<HD / 16>(dp, ptx::smem_u32(sV), sQ + T);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_operand(s);
    ptx::fence_operand(dp);
    uint32_t pa[16], da[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {  // s[2 k], s[2 k + 1]: row r + 8 (k & 1), q columns col, col + 1
      const int col = 8 * (k >> 1) + c;
      const float2 lq = *reinterpret_cast<const float2*>(sL + col);
      const float2 dd = *reinterpret_cast<const float2*>(sD + col);
      float p0 = ex2(fmaf(s[2 * k], sl2, -lq.x)), p1 = ex2(fmaf(s[2 * k + 1], sl2, -lq.y));
      if (nvalid < kBN || !kv_ok) {  // ragged q tile / kv rows that are not kept
        const bool row_ok = r + 8 * (k & 1) < rows_here;
        p0 = (row_ok && col < nvalid) ? p0 : 0.f;
        p1 = (row_ok && col + 1 < nvalid) ? p1 : 0.f;
      }
      if constexpr (DROP) {  // dV += (P Z)^T dO_i ; dS = P (Z dP - D)
        const uint32_t* bt = sBits + (i % kStages) * 2 * kBN + (r >> 5);
        const int sh = (r & 31) + 8 * (k & 1);
        const bool z0 = (bt[2 * col] >> sh) & 1u, z1 = (bt[2 * col + 2] >> sh) & 1u;
        const float dp0 = z0 ? dp[2 * k] * p.dscale : 0.f, dp1 = z1 ? dp[2 * k + 1] * p.dscale : 0.f;
        pa[k] = pack_bf16(z0 ? p0 * p.dscale : 0.f, z1 ? p1 * p.dscale : 0.f);
        da[k] = pack_bf16(p0 * fmaf(dp0, p.scale, -dd.x), p1 * fmaf(dp1, p.scale, -dd.y));
      } else {
        pa[k] = pack_bf16(p0, p1);
        da[k] = pack_bf16(p0 * fmaf(dp[2 * k], p.scale, -dd.x), p1 * fmaf(dp[2 * k + 1], p.scale, -dd.y));
      }
    }
    ptx::wgmma_fence();
    issue_acc<HD>(dv, pa, sQ + T);  // dV += P^T dO_i
    issue_acc<HD>(dk, da, sQ);          // dK += dS^T Q_i
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_operand(dk);
    ptx::fence_operand(dv);
    if (tid == 0) bars.release(i);
  }
  const long long base = static_cast<long long>(b) * p.Skv + kv0;
  const float one[2] = {1.f, 1.f};
  store_acc<HD>(dk, p.out0 + base * p.out0_rs + h * HD, p.out0_rs, rows_here, one);
  store_acc<HD>(dv, p.out1 + base * p.out1_rs + h * HD, p.out1_rs, rows_here, one);
}

// Raises kernel K's dynamic shared-memory limit and asks for all of L1 as shared memory, once per kernel.
template <auto K>
int set_smem(int bytes) {
  static bool carveout = false;
  if (!carveout) {
    cudaFuncSetAttribute(K, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    carveout = true;
  }
  return set_max_dynamic_smem<K>(bytes);
}

// Balanced tiling of an owned dimension of S rows: ceil(S / 64) tiles of R = ceil(S / tiles) rows each.
void balanced_tiles(int S, int* ntile, int* rows) {
  *ntile = ceil_div(S, kBM);
  *rows = ceil_div(S, *ntile);
}

// 3-D map {cols, S rows, B} of a [B * S, rs] row-major operand, box {64 columns, 64 rows, 1}: rows past S inside a
// batch are out of bounds and read as zeros.
int qkv_tmap(CUtensorMap* map, const void* base, int cols, int S, int B, int rs) {
  return make_tmap(map, "attention", CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, {cols, S, B}, {2LL * rs, 2LL * rs * S}, {64, 64, 1});
}

// Dropout arguments of one attention call: bits == nullptr means no dropout (the DROP = false kernels)
struct Drop {
  uint32_t* bits;                  // [B, nh, Sq, ceil(Skv / 32)] keep bits (written by the forward, read by the backward)
  const unsigned long long* seed;  // forward only: device pointer to the 64-bit Philox key
  int site;
  float p;
};

void set_drop(TcParams& p, const Drop& d, int Skv) {
  p.bits = d.bits; p.seed = d.seed; p.site = static_cast<uint32_t>(d.site);
  p.thresh = philox::threshold(d.p);
  p.dscale = philox::keep_scale(p.thresh);
  p.bwords = ceil_div(Skv, 32);
}

template <int HD, bool DROP>
int attn_fwd_impl(const void* q, const void* k, const void* v, void* o, float* lse, int B, int nh, int Sq, int Skv, int q_rs,
                  int k_rs, int v_rs, int o_rs, float scale, const Drop& drop, cudaStream_t s) {
  int ntile, tile_rows;
  balanced_tiles(Sq, &ntile, &tile_rows);
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = qkv_tmap(&tq, q, nh * HD, Sq, B, q_rs))) return rc;
  if ((rc = qkv_tmap(&tk, k, nh * HD, Skv, B, k_rs))) return rc;
  if ((rc = qkv_tmap(&tv, v, nh * HD, Skv, B, v_rs))) return rc;
  if ((rc = set_smem<attn_fwd_tc_kernel<HD, DROP>>(fwd_smem<HD>()))) return rc;
  TcParams p{};
  p.Sq = Sq; p.Skv = Skv; p.nh = nh; p.scale = scale; p.tile_rows = tile_rows;
  p.out0 = reinterpret_cast<bf16*>(o); p.out0_rs = o_rs; p.lse = lse;
  if (DROP) set_drop(p, drop, Skv);
  pdl_launch(dim3(ntile, nh, B), kThreads, fwd_smem<HD>(), s)(attn_fwd_tc_kernel<HD, DROP>, tq, tk, tv, p);
  return check_launch("attn_fwd_tc");
}

// dQ (and D, into dvec) over q row tiles, then dK / dV over kv row tiles
template <int HD, bool DROP>
int attn_bwd_impl(const void* q, const void* k, const void* v, const void* d_o, const float* lse, float* dvec, void* dq,
                  void* dk, void* dv, int B, int nh, int Sq, int Skv, int q_rs, int k_rs, int v_rs, int do_rs, int dq_rs,
                  int dk_rs, int dv_rs, float scale, const Drop& drop, cudaStream_t s) {
  int ntile, tile_rows;
  balanced_tiles(Sq, &ntile, &tile_rows);
  CUtensorMap tq, tdo, tk, tv;
  int rc;
  if ((rc = qkv_tmap(&tq, q, nh * HD, Sq, B, q_rs))) return rc;
  if ((rc = qkv_tmap(&tdo, d_o, nh * HD, Sq, B, do_rs))) return rc;
  if ((rc = qkv_tmap(&tk, k, nh * HD, Skv, B, k_rs))) return rc;
  if ((rc = qkv_tmap(&tv, v, nh * HD, Skv, B, v_rs))) return rc;
  if ((rc = set_smem<attn_bwd_dq_tc_kernel<HD, DROP>>(dq_smem<HD>()))) return rc;
  TcParams p{};
  p.Sq = Sq; p.Skv = Skv; p.nh = nh; p.scale = scale;
  p.out0 = reinterpret_cast<bf16*>(dq); p.out0_rs = dq_rs; p.lse = const_cast<float*>(lse); p.dvec = dvec;
  p.tile_rows = tile_rows;
  if (DROP) set_drop(p, drop, Skv);
  pdl_launch(dim3(ntile, nh, B), kThreads, dq_smem<HD>(), s)(attn_bwd_dq_tc_kernel<HD, DROP>, tq, tdo, tk, tv, p);
  if ((rc = check_launch("attn_bwd_dq_tc"))) return rc;

  balanced_tiles(Skv, &ntile, &tile_rows);
  constexpr int smem = dkdv_smem<HD, DROP>();
  if ((rc = set_smem<attn_bwd_dkdv_tc_kernel<HD, DROP>>(smem))) return rc;
  p.out0 = reinterpret_cast<bf16*>(dk); p.out0_rs = dk_rs; p.out1 = reinterpret_cast<bf16*>(dv); p.out1_rs = dv_rs;
  p.tile_rows = tile_rows;
  pdl_launch(dim3(ntile, nh, B), kThreads, smem, s)(attn_bwd_dkdv_tc_kernel<HD, DROP>, tk, tv, tq, tdo, p);
  return check_launch("attn_bwd_dkdv_tc");
}

int check_args(const char* who, int hd, int a, int b, int c) {
  if (hd != 48 && hd != 64 && hd != 96 && hd != 128) {
    set_last_error("%s: head_dim %d unsupported (48, 64, 96 and 128 are built)", who, hd);
    return MUSE_ERR_UNSUPPORTED;
  }
  if (((a | b | c) & 7) != 0) { set_last_error("%s: row strides must be multiples of 8 elements", who); return MUSE_ERR_INVALID; }
  return MUSE_OK;
}

}  // namespace
}  // namespace muse

using namespace muse;

extern "C" {

// Entry points of the C ABI: Attention.attention of the reference (muse/modeling_transformer.py:221-241) and its autograd
// backward, head_dim 48, 64, 96 or 128, no mask; with bits, nn.Dropout(p) is applied to the probabilities (:236-237) with the keep
// bits of philox.cuh (the DROP = true kernels).
int muse_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, unsigned int* bits,
                  const unsigned long long* seed, int site, float p, int B, int nh, int Sq, int Skv, int hd, int q_rs,
                  int k_rs, int v_rs, int o_rs, float scale, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (bits != nullptr && seed == nullptr) { set_last_error("attn_fwd: dropout needs a seed"); return MUSE_ERR_INVALID; }
  if (B <= 0 || Sq <= 0 || Skv <= 0) return MUSE_OK;
  int rc = check_args("attn_fwd", hd, q_rs | o_rs, k_rs, v_rs);
  if (rc) return rc;
  const Drop d{bits, seed, site, p};
#define MUSE_ATTN_FWD(HD, DROP) attn_fwd_impl<HD, DROP>(q, k, v, o, lse, B, nh, Sq, Skv, q_rs, k_rs, v_rs, o_rs, scale, d, s)
#define MUSE_ATTN_FWD_HD(DROP)                                                                 \
  switch (hd) {                                                                                \
    case 48: return MUSE_ATTN_FWD(48, DROP);                                                   \
    case 64: return MUSE_ATTN_FWD(64, DROP);                                                   \
    case 96: return MUSE_ATTN_FWD(96, DROP);                                                   \
    default: return MUSE_ATTN_FWD(128, DROP);                                                  \
  }
  if (bits == nullptr) MUSE_ATTN_FWD_HD(false)
  MUSE_ATTN_FWD_HD(true)
#undef MUSE_ATTN_FWD_HD
#undef MUSE_ATTN_FWD
}

// D is recomputed from (P, dP) inside the dQ kernel, so the backward does not read O.
int muse_attn_bwd(const void* q, const void* k, const void* v, const void* d_o, const float* lse, const unsigned int* bits,
                  float p, float* dvec, void* dq, void* dk, void* dv, int B, int nh, int Sq, int Skv, int hd, int q_rs,
                  int k_rs, int v_rs, int do_rs, int dq_rs, int dk_rs, int dv_rs, float scale, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (B <= 0 || Sq <= 0 || Skv <= 0) return MUSE_OK;
  int rc = check_args("attn_bwd", hd, q_rs | do_rs | dq_rs, k_rs | dk_rs, v_rs | dv_rs);
  if (rc) return rc;
  const Drop d{const_cast<unsigned int*>(bits), nullptr, 0, p};
#define MUSE_ATTN_BWD(HD, DROP) \
  attn_bwd_impl<HD, DROP>(q, k, v, d_o, lse, dvec, dq, dk, dv, B, nh, Sq, Skv, q_rs, k_rs, v_rs, do_rs, dq_rs, dk_rs, dv_rs, scale, d, s)
#define MUSE_ATTN_BWD_HD(DROP)                                                                 \
  switch (hd) {                                                                                \
    case 48: return MUSE_ATTN_BWD(48, DROP);                                                   \
    case 64: return MUSE_ATTN_BWD(64, DROP);                                                   \
    case 96: return MUSE_ATTN_BWD(96, DROP);                                                   \
    default: return MUSE_ATTN_BWD(128, DROP);                                                  \
  }
  if (bits == nullptr) MUSE_ATTN_BWD_HD(false)
  MUSE_ATTN_BWD_HD(true)
#undef MUSE_ATTN_BWD_HD
#undef MUSE_ATTN_BWD
}

}  // extern "C"
