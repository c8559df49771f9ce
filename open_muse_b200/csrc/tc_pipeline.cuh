// The persistent, warp-specialised TMA -> wgmma pipeline of the GEMM (gemm_wgmma.cu) and the implicit-GEMM convolution
// (conv_tc.cu).  One CTA of kThreads threads per SM:
//   warpgroup 0   : gives its registers back; one thread (the producer) fills a ring of shared-memory stages with TMA
//                   loads, one k-block per stage: A [BM x BK] then B [BN x BK], both 128-byte swizzled;
//   warpgroups 1-2: take the registers; each accumulates wgmma m64 x BN x k16 (bf16) or k32 (e4m3) on its 64-row half of
//                   the BM-row tile in fp32 registers, then runs the caller's epilogue from them.
// The operand element type T only changes the instruction: a k-block is 128 bytes of every operand row (64 bf16 or 128
// e4m3 elements), one swizzle row, so the TMA boxes, stage bytes, descriptors and 32-byte k-step advance are shared.
// Each stage has a `full` barrier (the producer's arrival plus the stage's TMA bytes) and an `empty` barrier (one arrival
// per consumer warpgroup once its MMAs on the stage have completed).  The caller owns the tile walk, the TMA coordinates
// and the epilogue.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp8.h>

#include <type_traits>

#include "ptx.cuh"
#include "wgmma.cuh"

namespace muse {
namespace tc {

constexpr int BM = 128;        // tile rows: two consumer warpgroups x 64
constexpr int BK = 64;         // k-block of bf16 operands: 64 bf16 = 128 B = one swizzle row
constexpr int kThreads = 384;  // the producer warpgroup and two consumer warpgroups
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;  // 128 x 40 + 256 x 232 registers fit the SM's 64 K

// Shared memory: STAGES x {A, B} | EXTRA bytes of the caller | full[STAGES], empty[STAGES], behind 1024 B of slack that
// aligns the swizzled tiles.  Each thread keeps its own position (stage, phase) in the ring.
template <int BN, int STAGES, int EXTRA = 0, typename T = __nv_bfloat16>
struct Ring {
  static constexpr bool kFp8 = std::is_same_v<T, __nv_fp8_e4m3>;
  static constexpr int kBK = 128 / sizeof(T);  // k-block in elements
  static constexpr int kStages = STAGES;
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kStageBytes = kABytes + BN * BK * 2;
  static constexpr int kSmemBytes = kStages * kStageBytes + EXTRA + 1024 + 256;

  uint8_t* smem;
  uint64_t* full;
  uint64_t* empty;
  int stage = 0;
  uint32_t phase = 0;

  __device__ __forceinline__ explicit Ring(uint8_t* smem_raw)
      : smem(reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023))),
        full(reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes + EXTRA)),
        empty(full + kStages) {}

  __device__ __forceinline__ uint8_t* extra() const { return smem + kStages * kStageBytes; }

  // one thread, before the __syncthreads that publishes the barriers to the CTA
  __device__ __forceinline__ void init() const {
    for (int i = 0; i < kStages; ++i) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }

  __device__ __forceinline__ void advance() {
    if (++stage == kStages) { stage = 0; phase ^= 1; }
  }

  struct Slot {
    uint8_t* a;
    uint8_t* b;
    uint64_t* bar;
  };
  // Producer: waits until the consumers have released the next stage and arms its full barrier for kStageBytes.  The
  // caller then issues the TMA loads of the k-block into slot.a / slot.b, completing on slot.bar.
  __device__ __forceinline__ Slot produce() {
    ptx::mbar_wait(&empty[stage], phase ^ 1);
    ptx::mbar_expect_tx(&full[stage], kStageBytes);
    uint8_t* a = smem + stage * kStageBytes;
    const Slot s{a, a + kABytes, &full[stage]};
    advance();
    return s;
  }

  // Consumer warpgroup `half`: acc = (rows [64 half, 64 half + 64) of A) x B^T over the next kb1 - kb0 stages, which hold
  // k-blocks [kb0, kb1); the first k-step overwrites acc.  A_MN / B_MN: the operand's M/N dimension is the contiguous one.
  // bf16 operands; e4m3 ones go through consume_promoted.
  // One wgmma group stays in flight: k-block kb is issued before the group of kb - 1 is waited for and its stage released,
  // so the tensor pipe does not drain between k-blocks.  acc is complete on return.
  template <bool A_MN, bool B_MN>
  __device__ __forceinline__ void consume(float (&acc)[BN / 2], int kb0, int kb1, int half) {
    static_assert(!kFp8, "e4m3 operands: consume_promoted");
    const bool leader = (threadIdx.x & 127) == 0;
    int prev = -1;  // stage of the group still in flight
    for (int kb = kb0; kb < kb1; ++kb) {
      ptx::mbar_wait(&full[stage], phase);
      // 64 rows of A are 8 KB in both layouts: 64 K-major rows, or one 64-element MN chunk
      const uint32_t a = ptx::smem_u32(smem + stage * kStageBytes) + half * 8192;
      const uint32_t b = ptx::smem_u32(smem + stage * kStageBytes + kABytes);
      ptx::fence_operand(acc);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        ptx::Wgmma<BN, A_MN, B_MN>::run(acc, A_MN ? ptx::desc_mnmajor(a, k) : ptx::desc_kmajor(a, k),
                                        B_MN ? ptx::desc_mnmajor(b, k) : ptx::desc_kmajor(b, k), (kb > kb0 || k > 0) ? 1 : 0);
      ptx::wgmma_commit();
      ptx::wgmma_wait<1>();
      ptx::fence_operand(acc);
      if (leader && prev >= 0) ptx::mbar_arrive(&empty[prev]);  // the MMAs of k-block kb - 1 have read its stage
      prev = stage;
      advance();
    }
    ptx::wgmma_wait<0>();
    ptx::fence_operand(acc);
    if (leader && prev >= 0) ptx::mbar_arrive(&empty[prev]);
  }

  // e4m3 operands (both K-major), with promotion: each k-block's four MMAs accumulate into `part` (overwritten at the
  // block's first k-step), which is added to the fp32 registers of acc once the block's group has completed, so the
  // tensor core's own accumulator never sums more than one k-block (128 products).  The group is waited for before the
  // add: no MMA is in flight across k-blocks.
  __device__ __forceinline__ void consume_promoted(float (&acc)[BN / 2], float (&part)[BN / 2], int kb0, int kb1, int half) {
    static_assert(kFp8, "promotion is for e4m3 operands");
    const bool leader = (threadIdx.x & 127) == 0;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kb = kb0; kb < kb1; ++kb) {
      ptx::mbar_wait(&full[stage], phase);
      const uint32_t a = ptx::smem_u32(smem + stage * kStageBytes) + half * 8192;
      const uint32_t b = ptx::smem_u32(smem + stage * kStageBytes + kABytes);
      ptx::fence_operand(part);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        ptx::WgmmaF8<BN>::run(part, ptx::desc_kmajor(a, k), ptx::desc_kmajor(b, k), k > 0 ? 1 : 0);
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::fence_operand(part);
      if (leader) ptx::mbar_arrive(&empty[stage]);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
      advance();
    }
  }
};

}  // namespace tc
}  // namespace muse
