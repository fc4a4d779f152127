// Prefill attention on the Hopper tensor cores (SURVEY §8 a2.6): causal GQA flash attention over the paged KV
// cache with wgmma, accumulators in registers, operands staged by TMA.
//
// One CTA per (q tile of up to 128 rows, q head); two consumer warpgroups own 64 q rows each.  Per KV block of
// 128 tokens (two 64-token pages):
//
//   S[64 q, 128 kv]  = Q · K^T      wgmma m64n128k16 per warpgroup, 8 k-steps over head_dim 128; Q and K
//                                   K-major in 128B-swizzled shared memory (TMA boxes of 64 columns)
//   softmax          in registers on the S fragment: scale + causal mask, running max / sum per row (a row is
//                                   spread over the 4 lanes of a quad), P rounded to bf16
//   O[64 q, 128 d]  += P · V        wgmma m64n128k16 with A = P straight from registers (the S fragment of two
//                                   8-column groups is exactly the A fragment of one 16-wide k-step) and B = V
//                                   **MN-major**: a V page is [token][d] (d contiguous), which is the MN-major
//                                   128B-swizzle canonical layout: LBO = distance between the two 64-wide d
//                                   halves, SBO = 1024 B between 8-token groups — no transposed copy of V
//
// Warp roles (384 threads): warp 0 lane 0 TMA producer (Q once; K/V pages of block j+1 while block j computes,
// 2 stages), warpgroups 1 and 2 consumers.  K/V pages are addressed through ONE 5-D tensor map per pool
// [layer][page][kv head][64][128]; q rows through a 2-D map over the qkv activation.  Masked scores are exactly 0
// in P, and pages only ever hold finite values (the pool is zero-filled at creation), so stale tokens past the
// causal horizon contribute exactly nothing.
// Algorithmic work: 4 * n_rows * kv_len * 128 flop per (tile, head) (half of it above the diagonal
// is masked but still issued inside a 128-block).
#include <cuda.h>

#include "../../include/llmlb_b200.h"
#include "common.cuh"
#include "tc_common.cuh"

namespace llmlb {

constexpr int kAtRows = 128;        // q rows per CTA (two warpgroups of wgmma M = 64)
constexpr int kAtBlock = 128;       // kv tokens per block (N of S, K of PV)
constexpr int kAtThreads = 384;
constexpr int kAtStages = 2;
constexpr uint32_t kAtSlab = kAtRows * 64 * 2;          // 16 KiB: 128 rows x 64 bf16, one swizzle slab
constexpr uint32_t kAtQBytes = 2 * kAtSlab;             // Q: two 64-wide d slabs
constexpr uint32_t kAtKBytes = 2 * kAtSlab;             // K block: [d half][page a | page b][64 tok][64 d]
constexpr uint32_t kAtVBytes = 2 * kAtSlab;
constexpr uint32_t kAtSmem = kAtQBytes + kAtStages * (kAtKBytes + kAtVBytes) + 1024 /*align*/ + 256 /*barriers*/;

__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int32_t c0, int32_t c1,
                                            int32_t c2, int32_t c3, int32_t c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
// MN-major, 128B swizzle: LBO = bytes between 64-element atoms along MN, SBO = bytes between 8-row groups along K
__device__ __forceinline__ uint64_t make_sw128_mn_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= uint64_t((smem_addr >> 4) & 0x3FFF);
  d |= uint64_t((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= uint64_t((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= uint64_t(1) << 62;   // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

__global__ void __launch_bounds__(kAtThreads, 1)
prefill_attention_kernel_tc(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                            const __grid_constant__ CUtensorMap tmap_v, uint32_t layer,
                            const int32_t* __restrict__ block_tables, uint32_t bt_stride, const int4* __restrict__ tiles,
                            __nv_bfloat16* __restrict__ out, uint32_t n_heads, uint32_t n_kv, uint32_t pdl) {
  extern __shared__ uint8_t at_smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_dyn) + 1023) & ~uintptr_t(1023));
  uint8_t* sq = smem;
  uint8_t* skv = sq + kAtQBytes;                                   // [stage][K | V]
  uint64_t* bars = reinterpret_cast<uint64_t*>(skv + kAtStages * (kAtKBytes + kAtVBytes));
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;        // [2]
  uint64_t* kv_empty = bars + 3;       // [2]

  if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int4 tile = tiles[blockIdx.x];
  const uint32_t q_row0 = tile.x, n_rows = tile.y, pos0 = tile.z, bt_row = tile.w;
  const uint32_t head = blockIdx.y, kvh = head / (n_heads / n_kv);
  const uint32_t kv_len = pos0 + n_rows;                           // causal horizon of the tile
  const uint32_t n_blocks = (kv_len + kAtBlock - 1) / kAtBlock;
  const uint32_t n_pages = (kv_len + kPageTokens - 1) / kPageTokens;

  if (warp == 0 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_q) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_k) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_v) : "memory");
  }
  if (warp == 1 && lane == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < kAtStages; ++i) { mbar_init(kv_full + i, 1); mbar_init(kv_empty + i, 8); }   // 8 consumer warps
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // everything above overlapped the previous kernel's tail; qkv / the pages it wrote are needed from here on
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");

  if (warp == 0) {
    if (lane == 0) {   // ---- TMA producer ----
      const int32_t* bt = block_tables + size_t(bt_row) * bt_stride;
      mbar_expect_tx(q_full, kAtQBytes);
      tma_load_2d(sq, &tmap_q, q_full, int32_t(head * kHeadDim), int32_t(q_row0));
      tma_load_2d(sq + kAtSlab, &tmap_q, q_full, int32_t(head * kHeadDim + 64), int32_t(q_row0));
      for (uint32_t j = 0; j < n_blocks; ++j) {
        const uint32_t stage = j & 1, phase = (j >> 1) & 1;
        mbar_wait(kv_empty + stage, phase ^ 1);
        const int32_t pa = bt[2 * j];
        const int32_t pb = (2 * j + 1 < n_pages) ? bt[2 * j + 1] : pa;   // absent page: any valid page, fully masked
        uint8_t* sk = skv + stage * (kAtKBytes + kAtVBytes);
        uint8_t* sv = sk + kAtKBytes;
        mbar_expect_tx(kv_full + stage, kAtKBytes + kAtVBytes);
#pragma unroll
        for (int h = 0; h < 2; ++h) {   // d half; per half: page a then page b, 8 KiB each
          tma_load_5d(sk + h * kAtSlab, &tmap_k, kv_full + stage, h * 64, 0, int32_t(kvh), pa, int32_t(layer));
          tma_load_5d(sk + h * kAtSlab + kAtSlab / 2, &tmap_k, kv_full + stage, h * 64, 0, int32_t(kvh), pb, int32_t(layer));
          tma_load_5d(sv + h * kAtSlab, &tmap_v, kv_full + stage, h * 64, 0, int32_t(kvh), pa, int32_t(layer));
          tma_load_5d(sv + h * kAtSlab + kAtSlab / 2, &tmap_v, kv_full + stage, h * 64, 0, int32_t(kvh), pb, int32_t(layer));
        }
      }
    }
  } else if (warp >= 4) {   // ---- consumers: warpgroup wg owns q rows [64 wg, 64 wg + 64) ----
    const uint32_t wg = (warp >> 2) - 1;
    const uint32_t r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows r0 and r0 + 8
    const float scale = rsqrtf(float(kHeadDim)) * 1.4426950408889634f;
    const uint32_t q_pos[2] = {pos0 + r0, pos0 + r0 + 8};
    float o[64], s[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const uint32_t qa = smem_u32(sq) + wg * (64 * 128);
    mbar_wait(q_full, 0);
    for (uint32_t j = 0; j < n_blocks; ++j) {
      const uint32_t stage = j & 1;
      mbar_wait(kv_full + stage, (j >> 1) & 1);
      const uint32_t sk = smem_u32(skv + stage * (kAtKBytes + kAtVBytes));
      const uint32_t sv = sk + kAtKBytes;
      // S = Q K^T: k-step ks covers d [16 ks, 16 ks + 16): slab ks / 4, 32 bytes per step inside the swizzle row
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const uint64_t adesc = make_sw128_desc(qa + (ks >> 2) * kAtSlab) + uint64_t((ks & 3) * 2);
        const uint64_t bdesc = make_sw128_desc(sk + (ks >> 2) * kAtSlab) + uint64_t((ks & 3) * 2);
        wgmma_ss<128>(s, adesc, bdesc, ks > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_hold(s);
      // online softmax on the fragment: s[4c + 2i + jj] is row r0 + 8i, kv column j * 128 + 8c + 2 (lane % 4) + jj
      const uint32_t kv0 = j * kAtBlock + 2 * (lane & 3);
      float corr[2], mu[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float mx = -INFINITY;
#pragma unroll
        for (int c = 0; c < 16; ++c)
#pragma unroll
          for (int jj = 0; jj < 2; ++jj) {
            const float v = (kv0 + 8 * c + jj <= q_pos[i]) ? s[4 * c + 2 * i + jj] * scale : -INFINITY;
            s[4 * c + 2 * i + jj] = v;
            mx = fmaxf(mx, v);
          }
        const float m_new = fmaxf(m_run[i], quad_max(mx));
        mu[i] = (m_new == -INFINITY) ? 0.f : m_new;
        corr[i] = exp2f(m_run[i] - mu[i]);   // m_run = -inf -> 0
        m_run[i] = m_new;
      }
      float rsum[2] = {0.f, 0.f};
      uint32_t p[32];
#pragma unroll
      for (int c = 0; c < 16; ++c)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float e0 = exp2f(s[4 * c + 2 * i] - mu[i]), e1 = exp2f(s[4 * c + 2 * i + 1] - mu[i]);
          rsum[i] += e0 + e1;
          p[2 * c + i] = pack_bf16(e0, e1);
        }
#pragma unroll
      for (int i = 0; i < 2; ++i) l_run[i] = l_run[i] * corr[i] + rsum[i];
#pragma unroll
      for (int c = 0; c < 16; ++c)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          o[4 * c + 2 * i] *= corr[i];
          o[4 * c + 2 * i + 1] *= corr[i];
        }
      // O += P V: k-step ks covers kv tokens [16 ks, 16 ks + 16) = fragment column groups 2 ks, 2 ks + 1;
      // V rows advance 16 x 128 B per step
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const uint32_t a[4] = {p[4 * ks], p[4 * ks + 1], p[4 * ks + 2], p[4 * ks + 3]};
        wgmma_rs_n128_bmn(o, a, make_sw128_mn_desc(sv + ks * 2048, kAtSlab, 1024), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_hold(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(kv_empty + stage);   // K and V of this stage are free
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t row = r0 + 8 * i;
      const float inv = 1.f / quad_sum(l_run[i]);
      if (row < n_rows) {
        __nv_bfloat16* dst = out + size_t(q_row0 + row) * n_heads * kHeadDim + size_t(head) * kHeadDim + 2 * (lane & 3);
#pragma unroll
        for (int c = 0; c < 16; ++c)
          *reinterpret_cast<uint32_t*>(dst + 8 * c) = pack_bf16(o[4 * c + 2 * i] * inv, o[4 * c + 2 * i + 1] * inv);
      }
    }
  }
}

// ----------------------------------------------------------------- host side ----------------
int make_tmap_nd(CUtensorMap* m, const void* base, uint32_t rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box);

// q rows: 2-D over the qkv activation [n_tokens, width], box = 64 columns x 128 rows
int make_tmap_attn_q(CUtensorMap* m, const void* qkv, uint64_t n_tokens, uint64_t width) {
  const uint64_t dims[2] = {width, n_tokens}, strides[1] = {width * 2};
  const uint32_t box[2] = {64, (uint32_t)kAtRows};
  return make_tmap_nd(m, qkv, 2, dims, strides, box);
}
// K or V pool [n_layers][n_pages][n_kv][64 tokens][128]: 5-D, box = 64 columns x 64 tokens of one (layer, page, head)
int make_tmap_attn_kv(CUtensorMap* m, const void* pool, uint64_t n_layers, uint64_t n_pages, uint64_t n_kv) {
  const uint64_t dims[5] = {(uint64_t)kHeadDim, (uint64_t)kPageTokens, n_kv, n_pages, n_layers};
  const uint64_t page_bytes = uint64_t(kPageTokens) * kHeadDim * 2;
  const uint64_t strides[4] = {uint64_t(kHeadDim) * 2, page_bytes, page_bytes * n_kv, page_bytes * n_kv * n_pages};
  const uint32_t box[5] = {64, (uint32_t)kPageTokens, 1, 1, 1};
  return make_tmap_nd(m, pool, 5, dims, strides, box);
}

int prefill_attention_tc_launch(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, uint32_t layer,
                                const int32_t* block_tables, uint32_t bt_stride, const int32_t* tiles, uint32_t n_tiles,
                                void* out, uint32_t n_heads, uint32_t n_kv, bool pdl, cudaStream_t st) {
  if (n_tiles == 0) return LLMLB_OK;
  static bool configured = false;
  if (!configured) {
    LLMLB_CUDA_CHECK(cudaFuncSetAttribute(prefill_attention_kernel_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAtSmem));
    configured = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(n_tiles, n_heads);
  cfg.blockDim = dim3(kAtThreads);
  cfg.dynamicSmemBytes = kAtSmem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (pdl && !(g_dbg_no_pdl & 16u)) ? 1 : 0;
  LLMLB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, prefill_attention_kernel_tc, mq, mk, mv, layer, block_tables, bt_stride,
                                      (const int4*)tiles, (__nv_bfloat16*)out, n_heads, n_kv, pdl ? 1u : 0u));
  LLMLB_LAUNCH_CHECK();
  return LLMLB_OK;
}

}  // namespace llmlb

using namespace llmlb;

// a2.6 on wgmma.  tiles: int32[n_tiles][4] = {first q row, q rows in tile (<= 128), position of the
// first row, row into block_tables}.  k_pages / v_pages: ONE layer's pool [n_pages][n_kv][64][128].
extern "C" int llmlb_op_prefill_attention_tc(const void* qkv, uint32_t n_tokens, const void* k_pages, const void* v_pages,
                                             uint32_t n_pages, const int32_t* block_tables, uint32_t bt_stride,
                                             const int32_t* tiles, uint32_t n_tiles, void* out, uint32_t n_heads,
                                             uint32_t n_kv, void* stream) {
  if (!qkv || !k_pages || !v_pages || !block_tables || !tiles || !out || n_kv == 0 || n_heads % n_kv || n_tokens == 0 || n_pages == 0) {
    set_error("llmlb_op_prefill_attention_tc: bad argument");
    return LLMLB_E_INVALID_ARG;
  }
  CUtensorMap mq, mk, mv;
  int rc = make_tmap_attn_q(&mq, qkv, n_tokens, uint64_t(n_heads + 2 * n_kv) * kHeadDim);
  if (rc) return rc;
  rc = make_tmap_attn_kv(&mk, k_pages, 1, n_pages, n_kv);
  if (rc) return rc;
  rc = make_tmap_attn_kv(&mv, v_pages, 1, n_pages, n_kv);
  if (rc) return rc;
  return prefill_attention_tc_launch(mq, mk, mv, 0, block_tables, bt_stride, tiles, n_tiles, out, n_heads, n_kv, false,
                                     (cudaStream_t)stream);
}
