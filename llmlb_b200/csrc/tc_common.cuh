// PTX wrappers and the warpgroup main loop / epilogue shared by the wgmma GEMM kernels (1-CTA gemm_tc.cu, CTA-pair
// gemm_tc2.cu): mbarrier, TMA tensor loads / multicast / L2 prefetch, wgmma fences, smem matrix descriptors.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "tp_common.cuh"
#include "wgmma.cuh"

namespace llmlb {

// internal epilogue (not in the public header): fp32 partial product of K-split `ks` stored at
// out + ks * n_tokens * out_stride; the consumer adds the slots in a fixed order (deterministic)
constexpr int kEpiPartialF32 = 4;
// tensor parallel, protocol B (tp_common.cuh): the fp32 partial of token row t, K-split ks, goes
// straight into the slot of the rank that OWNS the row: part (rank * split_k + ks), row t % rpr
constexpr int kEpiPushRS = 5;
// the same for narrow steps (batched decode, T <= kTpLLTokens): every pushed 8-byte word carries two bf16 values of
// adjacent output features AND the collective's epoch, so the owner's reduce kernel spins on the data itself —
// no system fence per CTA, no ticket, no flag round at the end of the GEMM grid (tp_common.cuh, "LL" variant)
constexpr int kEpiPushRSLL = 6;
constexpr uint32_t kTpLLTokens = 128;
struct TpPushRS {
  TpCtx ctx;
  uint32_t coll;      // kEpiPushRS: collective index within the step (slot = coll & 1)
  uint32_t rpr;       // kEpiPushRS: token rows per owner rank = ceil(n_tokens / size)
  uint32_t wait_coll_plus1;   // any epilogue: the activation operand is y of collective (this - 1): the TMA
                              // producer waits for its all-gather flags before the first activation load (0 = none)
  // in-kernel K-split of the store epilogues (bf16 / SiLU*up / fp32): fp32 partial tiles parked in sk_ws,
  // one arrival counter per output tile in sk_cnt (zero between launches); nullptr = no K-split
  float* sk_ws;
  unsigned int* sk_cnt;
  // row window of W this launch covers (a projection may be issued as whole waves of CTA-pair tiles plus a K-split
  // tail launch for the rows of the ragged last wave): rows [row0, row0 + n_rows), n_rows == 0 = all rows
  uint32_t row0, n_rows;
};
constexpr size_t kSkWsBytes = size_t(kNumSMs) * 128 * 256 * 4;   // every CTA of a full grid parks one 128 x 256 fp32 tile
constexpr uint32_t kSkCounters = 256;
constexpr int kBM = 128;          // weight rows per tile: two consumer warpgroups of 64 (wgmma M)
constexpr int kBK = 64;           // bf16 per K slab = 128 B = one swizzle row
constexpr int kTcThreads = 384;    // warpgroup 0: TMA producer (warp 0); warpgroups 1, 2: wgmma + epilogue

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive on the barrier at the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  asm volatile(
      "{\n.reg .b32 ra;\nmapa.shared::cluster.u32 ra, %0, %1;\n"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n}\n" ::"r"(smem_u32(bar)), "r"(rank)
      : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, "
      "{%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// the same tile into every CTA of `mask` (same smem offset, each completing on its own barrier at `bar`'s offset)
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar,
                                                      int32_t c0, int32_t c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, "
      "{%3, %4}], [%2], %5;" ::"r"(smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}
// pull a tile into L2 only (no smem, no barrier): hides HBM latency behind the smem ring
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* tmap, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global [%0, {%1, %2}];" ::"l"(tmap), "r"(c0), "r"(c1)
               : "memory");
}
// wgmma ordering: fence before the first wgmma that reads / writes accumulator registers touched by ordinary code
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int R>
__device__ __forceinline__ void wgmma_hold(float (&d)[R]) {   // keeps the compiler from touching d across an async wgmma
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major, 128B-swizzled operand tile (what TMA writes with SWIZZLE_128B and a 64-element box row):
// rows of 128 B, 8-row groups 1024 B apart (SBO), LBO unused (=1), layout type 1 (SWIZZLE_128B).
// A k-step of 16 bf16 inside the swizzle row advances the start address by 32 B (+2 in the 16-byte field).
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= uint64_t((smem_addr >> 4) & 0x3FFF);
  d |= uint64_t(1) << 16;
  d |= uint64_t(1024 >> 4) << 32;
  d |= uint64_t(1) << 62;
  return d;
}

__device__ __forceinline__ void epi_bar() {  // the 8 consumer warps only
  asm volatile("bar.sync 1, 256;" ::: "memory");
}
// tile configuration of the GEMM kernels: a 128-row W slab (A) and a BN-token X tile (B) per stage
template <int BN>
struct TcCfg {
  static constexpr int kStageBytes = kBM * kBK * 2 + BN * kBK * 2;
  static constexpr int kStages = (BN >= 256) ? 4 : (BN >= 128 ? 6 : 8);
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 256 /*barriers*/;
};

// One consumer warpgroup's main loop over K blocks [kb0, kb1) of a tile: acc (64 weight rows x BN tokens, wgmma
// fragment) = sum over the blocks of W[64 rows of warpgroup wg] . X^T.  The previous block's wgmmas stay in flight
// while the next block is issued; a stage is released (one arrival per consumer warp, on this CTA's empty barrier
// and, for a CTA pair, on the peer's as well: its producer multicasts into our stage) once its wgmmas retired.
template <int BN, bool PAIR>
__device__ __forceinline__ void tc_mainloop(float (&acc)[BN / 2], uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                            uint32_t kb0, uint32_t kb1, uint32_t wg, uint32_t& stage, uint32_t& phase,
                                            long long& c_wait) {
  using Cfg = TcCfg<BN>;
  const uint32_t lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  auto release = [&](uint32_t s) {
    if (lane == 0) {
      mbar_arrive(empty_bar + s);
      if constexpr (PAIR) {
        uint32_t r;
        asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
        mbar_arrive_cluster(empty_bar + s, r ^ 1u);
      }
    }
  };
  uint32_t prev = 0;
  for (uint32_t kb = kb0; kb < kb1; ++kb) {
    { const long long c0 = clock64(); mbar_wait(full_bar + stage, phase); c_wait += clock64() - c0; }
    const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes) + wg * (64 * 128);
    const uint32_t sb = smem_u32(smem + stage * Cfg::kStageBytes) + kBM * kBK * 2;
    const uint64_t adesc = make_sw128_desc(sa), bdesc = make_sw128_desc(sb);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k) wgmma_ss<BN>(acc, adesc + uint64_t(k * 2), bdesc + uint64_t(k * 2), 1u);
    wgmma_commit();
    wgmma_hold(acc);
    if (kb > kb0) {
      wgmma_wait<1>();
      __syncwarp();
      release(prev);
    }
    prev = stage;
    if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_hold(acc);
  __syncwarp();
  if (kb1 > kb0) release(prev);
}

// Epilogue of one warp of a consumer warpgroup for the plain epilogues (bf16 / fp32 store, residual add, SiLU*up, fp32
// K-split partial, tensor-parallel push).  n0: the output feature of fragment row 0 of this warp (16 rows per warp);
// rows n0 + l / 4 + 8 i, token columns t0 + 8 c + 2 (l % 4) + j.  Pairs of adjacent rows (gate, up of SiLU*up) sit in
// lanes l and l ^ 4.  ep_ll: the collective's epoch (kEpiPushRSLL).
template <int BN, int EPI>
__device__ __forceinline__ void tc_epilogue(const float (&acc)[BN / 2], void* __restrict__ out, uint32_t n0, uint32_t t0,
                                            uint32_t n_tokens, uint32_t n_out, uint32_t out_stride, uint32_t ks,
                                            uint32_t split_k, const TpPushRS& tp, uint8_t* const* s_peer_slot,
                                            uint32_t ep_ll) {
  const uint32_t lane = threadIdx.x & 31;
  const bool odd = (lane >> 2) & 1;
#pragma unroll
  for (int c = 0; c < BN / 8; ++c) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t n = n0 + (lane >> 2) + 8 * i;
      const uint32_t t = t0 + 8 * c + 2 * (lane & 3);
      const float v0 = acc[4 * c + 2 * i], v1 = acc[4 * c + 2 * i + 1];
      if constexpr (EPI == LLMLB_EPI_SILU_MUL) {
        // the even row (gate) finishes token t, the odd row (up) token t + 1
        const float o0 = __shfl_xor_sync(0xffffffffu, v0, 4), o1 = __shfl_xor_sync(0xffffffffu, v1, 4);
        const float g = odd ? o1 : v0, u = odd ? v1 : o0;
        const uint32_t tt = t + (odd ? 1u : 0u);
        if ((n | 1) < n_out && tt < n_tokens) {
          const float s = __fdividef(g, 1.f + __expf(-g));  // IEEE division was ~half of the epilogue's instructions
          reinterpret_cast<__nv_bfloat16*>(out)[size_t(tt) * out_stride + (n >> 1)] = __float2bfloat16_rn(s * u);
        }
      } else if constexpr (EPI == kEpiPushRSLL) {
        // one 8-byte word {bf16 n, bf16 n+1, epoch} per token: the even row sends token t, the odd row token t + 1
        const float o0 = __shfl_xor_sync(0xffffffffu, v0, 4), o1 = __shfl_xor_sync(0xffffffffu, v1, 4);
        const float lo = odd ? o1 : v0, hi = odd ? v1 : o0;
        const uint32_t tt = t + (odd ? 1u : 0u);
        if ((n | 1) < n_out && tt < n_tokens) {
          const uint32_t owner = tt / tp.rpr, tl = tt - owner * tp.rpr;
          uint2 w;
          w.x = pack_bf16(lo, hi);
          w.y = ep_ll;
          st_peer_u2(reinterpret_cast<uint2*>(s_peer_slot[owner]) +
                         (size_t(tp.ctx.rank * split_k + ks) * tp.rpr + tl) * (out_stride / 2) + (n >> 1), w);
        }
      } else if (n < n_out) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const uint32_t tj = t + j;
          if (tj >= n_tokens) continue;
          const float v = j ? v1 : v0;
          const size_t idx = size_t(tj) * out_stride + n;
          if constexpr (EPI == LLMLB_EPI_STORE_BF16)
            reinterpret_cast<__nv_bfloat16*>(out)[idx] = __float2bfloat16_rn(v);
          else if constexpr (EPI == LLMLB_EPI_STORE_F32)
            reinterpret_cast<float*>(out)[idx] = v;
          else if constexpr (EPI == kEpiPartialF32)  // deterministic split-K: slot ks of the workspace
            reinterpret_cast<float*>(out)[size_t(ks) * n_tokens * out_stride + idx] = v;
          else if constexpr (EPI == kEpiPushRS) {    // reduce-scatter by address into the row owner's slot
            const uint32_t owner = tj / tp.rpr, tl = tj - owner * tp.rpr;
            st_peer_bf16(reinterpret_cast<__nv_bfloat16*>(s_peer_slot[owner]) +
                             (size_t(tp.ctx.rank * split_k + ks) * tp.rpr + tl) * out_stride + n, v);
          } else {
            if (split_k > 1) atomicAdd(reinterpret_cast<float*>(out) + idx, v);
            else reinterpret_cast<float*>(out)[idx] += v;
          }
        }
      }
    }
  }
}

}  // namespace llmlb
