// kv_fork: copy the first rows of one KV page into other pages, in K and V, for every layer and KV head of this rank.
//
// A request with n choices prefills its prompt once.  The choices then share the prompt's full pages and each gets its
// own copy of the last, partial page: this kernel makes those copies in one launch.  Pool layout (engine.cu, alloc_all):
// [layer][page][kv_head][64][128] bf16, so the rows [0, rows) of one (layer, page, head) are rows * 256 contiguous bytes.
// One CTA per (K or V, head, layer) reads each 16-byte vector of the source once and writes it to every destination;
// rows rows..63 of the destinations and every other page are not touched.
#include "../../include/llmlb_b200.h"
#include "common.cuh"

namespace llmlb {

constexpr uint32_t kForkThreads = 256;
constexpr uint32_t kForkMaxDst = 1024;   // destination page ids staged in shared memory (4 KiB)

__global__ void __launch_bounds__(kForkThreads) kv_fork_kernel(__nv_bfloat16* __restrict__ k_pool, __nv_bfloat16* __restrict__ v_pool,
                                                              uint32_t n_pages, uint32_t n_kv, int32_t src_page,
                                                              const int32_t* __restrict__ dst_pages, uint32_t n_dst, uint32_t rows) {
  extern __shared__ int32_t s_dst[];
  for (uint32_t d = threadIdx.x; d < n_dst; d += blockDim.x) s_dst[d] = dst_pages[d];
  __syncthreads();
  const uint32_t head = blockIdx.x >> 1, layer = blockIdx.y;
  __nv_bfloat16* pool = (blockIdx.x & 1) ? v_pool : k_pool;
  const size_t page_elems = size_t(n_kv) * kPageTokens * kHeadDim;
  const size_t base = size_t(layer) * n_pages * page_elems + size_t(head) * kPageTokens * kHeadDim;
  const uint4* src = reinterpret_cast<const uint4*>(pool + base + size_t(src_page) * page_elems);
  const uint32_t n_vec = rows * (kHeadDim * 2 / 16);
  for (uint32_t i = threadIdx.x; i < n_vec; i += blockDim.x) {
    const uint4 v = src[i];
    for (uint32_t d = 0; d < n_dst; ++d) {
      const uint32_t p = uint32_t(s_dst[d]);
      if (p >= n_pages) continue;   // not a page of this pool: nothing is written
      reinterpret_cast<uint4*>(pool + base + size_t(p) * page_elems)[i] = v;
    }
  }
}

int kv_fork_launch(__nv_bfloat16* k_pool, __nv_bfloat16* v_pool, uint32_t n_layers, uint32_t n_pages, uint32_t n_kv,
                   int32_t src_page, const int32_t* dst_pages, uint32_t n_dst, uint32_t rows, cudaStream_t st) {
  dim3 grid(2 * n_kv, n_layers);
  kv_fork_kernel<<<grid, kForkThreads, n_dst * sizeof(int32_t), st>>>(k_pool, v_pool, n_pages, n_kv, src_page, dst_pages, n_dst, rows);
  LLMLB_LAUNCH_CHECK();
  return LLMLB_OK;
}

}  // namespace llmlb

using namespace llmlb;

extern "C" int llmlb_op_kv_fork(void* k_pool, void* v_pool, uint32_t n_layers, uint32_t n_pages, uint32_t n_kv, int32_t src_page,
                                const int32_t* dst_pages, uint32_t n_dst, uint32_t rows, void* stream) {
  auto bad = [](const char* m) { set_error(std::string("llmlb_op_kv_fork: ") + m); return LLMLB_E_INVALID_ARG; };
  if (!k_pool || !v_pool || !dst_pages) return bad("null argument");
  if (n_layers == 0 || n_layers > 65535) return bad("n_layers must be in [1, 65535]");
  if (n_kv == 0 || n_kv > 256) return bad("n_kv must be in [1, 256]");
  if (n_pages == 0 || uint64_t(n_layers) * n_pages * n_kv * kPageTokens * kHeadDim > (uint64_t(1) << 40))
    return bad("n_pages must be positive and the pool at most 2^40 elements");
  if (src_page < 0 || uint32_t(src_page) >= n_pages) return bad("src_page outside the pool");
  if (n_dst == 0 || n_dst > kForkMaxDst) return bad("n_dst must be in [1, 1024]");
  if (rows == 0 || rows > uint32_t(kPageTokens)) return bad("rows must be in [1, 64]");
  return kv_fork_launch(static_cast<__nv_bfloat16*>(k_pool), static_cast<__nv_bfloat16*>(v_pool), n_layers, n_pages, n_kv, src_page,
                        dst_pages, n_dst, rows, (cudaStream_t)stream);
}
