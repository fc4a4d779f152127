// Prefill projections, CTA-pair variant: a thread-block cluster of 2 CTAs owns a 256-row slab of W x BN tokens.
// Each CTA computes ITS 128 weight rows against the whole token tile, but loads only HALF of the token tile and
// multicasts it into both CTAs' shared memory, so the activation operand crosses L2->SM once per pair instead of
// once per CTA (32 KiB instead of 48 KiB of L2 reads per K slab per pair member).
//
//   both CTAs : warp 0 lane 0 TMA producer — own 128 W rows into its own stage, own half of the tokens multicast
//               into the same stage of both CTAs (each CTA's full barrier expects the whole 48 KiB stage);
//               warpgroups 1, 2 consumers — wgmma on 64 weight rows each, fused epilogue from registers
//   barriers  : full[stage]   per CTA, count 1 (own expect_tx), bytes from both producers
//               empty[stage]  per CTA, count 16: the 8 consumer warps of BOTH CTAs (either producer writes the slot)
#include <cuda.h>

#include "../../include/llmlb_b200.h"
#include "common.cuh"
#include "tc_common.cuh"

namespace llmlb {

static __device__ TraceBuf d_trace_tc2;
void tc2_set_trace(const TraceBuf& tb) { cudaMemcpyToSymbol(d_trace_tc2, &tb, sizeof(tb)); }

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

template <int BN, int EPI>
__global__ void __launch_bounds__(kTcThreads, 1)
gemm_tc2_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                void* __restrict__ out, uint32_t n_tokens, uint32_t n_out, uint32_t K, uint32_t out_stride,
                uint32_t m_tiles /*256-row slabs*/, uint32_t t_tiles, uint32_t split_k, const TpPushRS tp) {
  const uint32_t m_tile0 = tp.row0 / 256;
  using Cfg = TcCfg<BN>;
  constexpr int kHalfN = BN / 2;                                   // tokens each CTA loads (and multicasts)
  const TraceBuf tb = d_trace_tc2;
  unsigned long long tr0 = 0, tr1 = 0;
  if (tb.data && threadIdx.x == 0) tr0 = gtime_ns();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the next kernel may set itself up on freed SMs
  __shared__ uint8_t* s_peer_slot[kTpMaxRanks];   // kEpiPushRS: slot base of every rank
  if constexpr (EPI == kEpiPushRS) {
    if (threadIdx.x < tp.ctx.size) s_peer_slot[threadIdx.x] = tp.ctx.base[threadIdx.x] + tp.ctx.slot_off[tp.coll & 1];
  }
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::kStages;

  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  const uint32_t pair = blockIdx.x >> 1, n_pairs = gridDim.x >> 1;
  const uint32_t k_blocks_total = (K + kBK - 1) / kBK;
  const uint32_t k_per_split = (k_blocks_total + split_k - 1) / split_k;
  const uint32_t n_tiles = m_tiles * t_tiles * split_k;

  if (warp == 0 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_w) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(full_bar + i, 1);
      mbar_init(empty_bar + i, 16);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  cluster_sync_all();  // peer barriers are initialised before anyone signals them
  // programmatic dependent launch: barrier init and the tensor-map fetch above overlapped the previous kernel's
  // tail; its outputs (our activations) are needed from here on
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (tb.data && threadIdx.x == 0) tr1 = gtime_ns();

  auto decode_tile = [&](uint32_t tile, uint32_t& mt, uint32_t& tt, uint32_t& ks) {
    tt = tile % t_tiles;
    uint32_t r = tile / t_tiles;
    ks = r % split_k;
    mt = r / split_k + m_tile0;
  };

  if (warp == 0) {
    if (lane == 0) {  // ---- TMA producer (both CTAs) ----
      if (tp.wait_coll_plus1) tp_wait_ag_single(tp.ctx, tp.wait_coll_plus1 - 1);
      uint32_t stage = 0, phase = 0;
      for (uint32_t tile = pair; tile < n_tiles; tile += n_pairs) {
        uint32_t mt, tt, ks;
        decode_tile(tile, mt, tt, ks);
        const uint32_t kb0 = ks * k_per_split;
        const uint32_t kb1 = min(k_blocks_total, kb0 + k_per_split);
        for (uint32_t kb = kb0; kb < kb1; ++kb) {
          mbar_wait(empty_bar + stage, phase ^ 1);   // both CTAs' consumers are done with this slot
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + kBM * kBK * 2;
          mbar_expect_tx(full_bar + stage, Cfg::kStageBytes);
          tma_load_2d(sa, &tmap_w, full_bar + stage, int32_t(kb * kBK), int32_t(mt * 256 + rank * kBM));
          tma_load_2d_multicast(sb + rank * (kHalfN * kBK * 2), &tmap_x, full_bar + stage, int32_t(kb * kBK),
                                int32_t(tt * BN + rank * kHalfN), uint16_t(3));
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {  // ---- consumers (both CTAs, own 128 weight rows) ----
    const uint32_t wg = (warp >> 2) - 1;
    const uint32_t wrow = wg * 64 + (warp & 3) * 16;
    uint32_t stage = 0, phase = 0;
    long long c_wait = 0;
    for (uint32_t tile = pair; tile < n_tiles; tile += n_pairs) {
      uint32_t mt, tt, ks;
      decode_tile(tile, mt, tt, ks);
      const uint32_t kb0 = ks * k_per_split;
      const uint32_t kb1 = min(k_blocks_total, kb0 + k_per_split);
      float acc[BN / 2];
      tc_mainloop<BN, true>(acc, smem, full_bar, empty_bar, kb0, kb1, wg, stage, phase, c_wait);
      tc_epilogue<BN, EPI>(acc, out, mt * 256 + rank * kBM + wrow, tt * BN, n_tokens, n_out, out_stride, ks, split_k, tp,
                           s_peer_slot, 0u);
    }
  }

  cluster_sync_all();  // nobody exits while the peer may still multicast into it or arrive on its barriers
  if (tb.data && threadIdx.x == 0)
    trace_emit(tb, (4ull << 60) | ((unsigned long long)EPI << 56) | ((unsigned long long)n_out << 32) | K, tr0, tr1, gtime_ns(), n_tokens);
  if constexpr (EPI == kEpiPushRS) {
    const uint32_t slot = tp.coll & 1;
    tp_signal_when_grid_done(tp.ctx, &tp_flags(tp.ctx, tp.ctx.rank)->done[slot], gridDim.x, tp_epoch(tp.ctx, tp.coll),
                             [&](TpFlags* f) { return &f->push_flag[slot][tp.ctx.rank]; });
  }
}

template <int BN, int EPI>
static int launch_tc2(const CUtensorMap& tw, const CUtensorMap& tx_half, void* out, uint32_t n_tokens, uint32_t n_out,
                      uint32_t k, uint32_t out_stride, uint32_t split_k, cudaStream_t st, const TpPushRS* tpp = nullptr) {
  using Cfg = TcCfg<BN>;
  auto kern = gemm_tc2_kernel<BN, EPI>;
  static bool configured = false;
  if (!configured) {
    LLMLB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    configured = true;
  }
  TpPushRS tp{};
  if (tpp) tp = *tpp;
  const uint32_t rows = tp.n_rows ? tp.n_rows : n_out;
  const uint32_t m_tiles = (rows + 255) / 256, t_tiles = (n_tokens + BN - 1) / BN;
  const uint32_t tiles = m_tiles * t_tiles * split_k;
  uint32_t pairs = tiles < (uint32_t)(kNumSMs / 2) ? tiles : (uint32_t)(kNumSMs / 2);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(pairs * 2);
  cfg.blockDim = dim3(kTcThreads);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (g_dbg_no_pdl & 16u) ? 1 : 2;
  LLMLB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, tw, tx_half, out, n_tokens, n_out, k, out_stride, m_tiles, t_tiles, split_k, tp));
  LLMLB_LAUNCH_CHECK();
  return LLMLB_OK;
}

// BN = 256 only (n_tokens > 128).  tx_half: activation tensor map with a 128-row box.
int gemm_tc2_launch(const CUtensorMap& tw, const CUtensorMap& tx_half, void* out, uint32_t n_tokens, uint32_t n_out,
                    uint32_t k, uint32_t epi, uint32_t out_stride, cudaStream_t st, uint32_t* n_parts,
                    const TpPushRS* tpp, uint32_t max_split) {
  uint32_t split_k = 1;
  if (epi == LLMLB_EPI_RESID_F32 || epi == (uint32_t)kEpiPartialF32 || epi == (uint32_t)kEpiPushRS) {
    uint32_t tiles = (((tpp && tpp->n_rows ? tpp->n_rows : n_out) + 255) / 256) * ((n_tokens + 255) / 256);
    uint32_t kblocks = (k + kBK - 1) / kBK;
    while (tiles * split_k * 2 <= (uint32_t)(kNumSMs / 2) && kblocks / (split_k * 2) >= 8 && split_k * 2 <= max_split) split_k *= 2;
  }
  if (n_parts) *n_parts = split_k;
  switch (epi) {
    case LLMLB_EPI_STORE_BF16: return launch_tc2<256, LLMLB_EPI_STORE_BF16>(tw, tx_half, out, n_tokens, n_out, k, out_stride, 1, st, tpp);
    case LLMLB_EPI_RESID_F32: return launch_tc2<256, LLMLB_EPI_RESID_F32>(tw, tx_half, out, n_tokens, n_out, k, out_stride, split_k, st);
    case LLMLB_EPI_SILU_MUL: return launch_tc2<256, LLMLB_EPI_SILU_MUL>(tw, tx_half, out, n_tokens, n_out, k, out_stride, 1, st, tpp);
    case LLMLB_EPI_STORE_F32: return launch_tc2<256, LLMLB_EPI_STORE_F32>(tw, tx_half, out, n_tokens, n_out, k, out_stride, 1, st, tpp);
    case kEpiPartialF32: return launch_tc2<256, kEpiPartialF32>(tw, tx_half, out, n_tokens, n_out, k, out_stride, split_k, st);
    case kEpiPushRS: return launch_tc2<256, kEpiPushRS>(tw, tx_half, out, n_tokens, n_out, k, out_stride, split_k, st, tpp);
  }
  set_error("gemm_tc2: unknown epilogue");
  return LLMLB_E_INVALID_ARG;
}

}  // namespace llmlb
