// Embedding gather (a2.1), RMSNorm (a2.2) and the synthetic-weight generator.
// All three are HBM-bound: 16-byte accesses, one row per CTA, no re-reads.
#include "../../include/llmlb_b200.h"
#include "common.cuh"

namespace llmlb {

// x[t, :] = float(E[ids[t], :]).  One CTA per token; 8 bf16 per thread per trip.
__global__ void __launch_bounds__(256) embed_kernel(const __nv_bfloat16* __restrict__ table,
                                                    const int32_t* __restrict__ ids,
                                                    float* __restrict__ x, uint32_t hidden,
                                                    uint32_t vocab) {
  const uint32_t t = blockIdx.x;
  int32_t id = ids[t];
  if (id < 0 || uint32_t(id) >= vocab) id = 0;  // out-of-range ids read row 0 (host validates)
  const uint4* src = reinterpret_cast<const uint4*>(table + size_t(id) * hidden);
  float4* dst = reinterpret_cast<float4*>(x + size_t(t) * hidden);
  for (uint32_t i = threadIdx.x; i < hidden / 8; i += blockDim.x) {
    uint4 v = __ldg(src + i);
    dst[2 * i] = make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y));
    dst[2 * i + 1] = make_float4(bf16_lo(v.z), bf16_hi(v.z), bf16_lo(v.w), bf16_hi(v.w));
  }
}

// y = x * rsqrt(mean(x^2) + eps) * g.  fp32 residual in, bf16 out; one CTA (256 thr) per token.
__global__ void __launch_bounds__(256) rmsnorm_kernel(const float* __restrict__ x,
                                                      const __nv_bfloat16* __restrict__ gain,
                                                      __nv_bfloat16* __restrict__ y,
                                                      uint32_t hidden, float eps) {
  __shared__ float red[8];
  const uint32_t t = blockIdx.x;
  const float4* src = reinterpret_cast<const float4*>(x + size_t(t) * hidden);
  float ss = 0.f;
  for (uint32_t i = threadIdx.x; i < hidden / 4; i += blockDim.x) {
    float4 v = src[i];
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[w];
  const float r = rsqrtf(tot / float(hidden) + eps);
  uint2* dst = reinterpret_cast<uint2*>(y + size_t(t) * hidden);
  const uint2* g2 = reinterpret_cast<const uint2*>(gain);
  for (uint32_t i = threadIdx.x; i < hidden / 4; i += blockDim.x) {
    float4 v = src[i];
    uint2 g = __ldg(g2 + i);
    uint2 o;
    o.x = pack_bf16(v.x * r * bf16_lo(g.x), v.y * r * bf16_hi(g.x));
    o.y = pack_bf16(v.z * r * bf16_lo(g.y), v.w * r * bf16_hi(g.y));
    dst[i] = o;
  }
}

// x[t,:] += sum_p parts[p][t,:] (p ascending: deterministic), then optionally y = RMSNorm(x)*g.
// This is where the K-split partial products of the O / down projections are folded into the
// residual stream — a fixed-order replacement for fp32 atomics (and the hook for TP partials).
__global__ void __launch_bounds__(256) rmsnorm_parts_kernel(float* __restrict__ x,
                                                            const float* parts /* predecessor output: no restrict (PDL) */,
                                                            uint32_t n_parts, size_t part_stride,
                                                            const __nv_bfloat16* __restrict__ gain,
                                                            __nv_bfloat16* __restrict__ y,
                                                            uint32_t hidden, float eps, uint32_t pdl) {
  __shared__ float red[8];
  // lets a PDL-launched successor (the next projection GEMM) start pulling its weights now; a
  // no-op for ordinary launches
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // pdl: this grid was itself scheduled while the projection that feeds it may still be running
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  const uint32_t t = blockIdx.x;
  float4* xr = reinterpret_cast<float4*>(x + size_t(t) * hidden);
  float ss = 0.f;
  for (uint32_t i = threadIdx.x; i < hidden / 4; i += blockDim.x) {
    float4 v = xr[i];
    for (uint32_t p = 0; p < n_parts; ++p) {
      const float4 a = reinterpret_cast<const float4*>(parts + p * part_stride + size_t(t) * hidden)[i];
      v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
    }
    xr[i] = v;
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  if (!gain) return;
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[w];
  const float r = rsqrtf(tot / float(hidden) + eps);
  uint2* dst = reinterpret_cast<uint2*>(y + size_t(t) * hidden);
  const uint2* g2 = reinterpret_cast<const uint2*>(gain);
  for (uint32_t i = threadIdx.x; i < hidden / 4; i += blockDim.x) {
    float4 v = xr[i];  // own writes, same thread
    uint2 g = __ldg(g2 + i);
    uint2 o;
    o.x = pack_bf16(v.x * r * bf16_lo(g.x), v.y * r * bf16_hi(g.x));
    o.y = pack_bf16(v.z * r * bf16_lo(g.y), v.w * r * bf16_hi(g.y));
    dst[i] = o;
  }
}

// The same fold + RMSNorm with a CLUSTER of 4 CTAs per token row: each CTA owns a quarter of the
// columns (one float4 per thread at hidden 4096), the four partial sums of squares are exchanged
// through distributed shared memory.  For narrow steps (batched decode: 16..256 rows) one CTA per
// row leaves most SMs idle and the kernel is pure latency (7.2 us at 64 rows in round 1).
__global__ void __launch_bounds__(256) rmsnorm_parts_cluster_kernel(float* __restrict__ x, const float* __restrict__ parts,
                                                                    uint32_t n_parts, size_t part_stride,
                                                                    const __nv_bfloat16* __restrict__ gain,
                                                                    __nv_bfloat16* __restrict__ y, uint32_t hidden, float eps) {
  __shared__ float red[8];
  __shared__ float s_ss[4];   // partial sums of squares of the 4 CTAs of the cluster (every CTA gets all four)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // A CTA may touch a peer's shared memory only once every CTA of the cluster is running: arrive now, wait before the
  // first remote store (after the fold loop, so the wait costs nothing there).  Fold-only launches touch no peer.
  if (gain) asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
  uint32_t cr;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(cr));
  const uint32_t t = blockIdx.x >> 2;
  const uint32_t q4 = hidden / 16;                    // float4 per CTA
  float4* xr = reinterpret_cast<float4*>(x + size_t(t) * hidden) + size_t(cr) * q4;
  float ss = 0.f;
  for (uint32_t i = threadIdx.x; i < q4; i += blockDim.x) {
    float4 v = xr[i];
    for (uint32_t p = 0; p < n_parts; ++p) {
      const float4 a = (reinterpret_cast<const float4*>(parts + p * part_stride + size_t(t) * hidden) + size_t(cr) * q4)[i];
      v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
    }
    xr[i] = v;
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  if (!gain) return;   // uniform over the cluster
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  asm volatile("barrier.cluster.wait.aligned;" ::: "memory");   // every peer CTA has started: its s_ss is live
  if (threadIdx.x < 4) {   // thread q stores this CTA's partial into CTA q's s_ss[cr]
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += red[w];
    const uint32_t local = (uint32_t)__cvta_generic_to_shared(&s_ss[cr]);
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(threadIdx.x));
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(remote), "f"(tot) : "memory");
  }
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  const float r = rsqrtf((s_ss[0] + s_ss[1] + s_ss[2] + s_ss[3]) / float(hidden) + eps);   // fixed order: same value in all 4 CTAs
  uint2* dst = reinterpret_cast<uint2*>(y + size_t(t) * hidden) + size_t(cr) * q4;
  const uint2* g2 = reinterpret_cast<const uint2*>(gain) + size_t(cr) * q4;
  for (uint32_t i = threadIdx.x; i < q4; i += blockDim.x) {
    const float4 v = xr[i];  // own writes, same thread
    const uint2 g = __ldg(g2 + i);
    uint2 o;
    o.x = pack_bf16(v.x * r * bf16_lo(g.x), v.y * r * bf16_hi(g.x));
    o.y = pack_bf16(v.z * r * bf16_lo(g.y), v.w * r * bf16_hi(g.y));
    dst[i] = o;
  }
}

int rmsnorm_parts_launch(float* x, const float* parts, uint32_t n_parts, size_t part_stride, const void* gain,
                         void* y, uint32_t n_tokens, uint32_t hidden, float eps, cudaStream_t st) {
  if (n_tokens == 0) return LLMLB_OK;
  if (n_tokens <= 256 && hidden % 16 == 0) {   // narrow step (batched decode, short chunks): 4 CTAs per row
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(n_tokens * 4);
    cfg.blockDim = dim3(256);
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 4;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    LLMLB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, rmsnorm_parts_cluster_kernel, x, parts, n_parts, part_stride, (const __nv_bfloat16*)gain,
                                        (__nv_bfloat16*)y, hidden, eps));
    LLMLB_LAUNCH_CHECK();
    return LLMLB_OK;
  }
  // plain launch: launching this small kernel itself as a programmatic dependent measured SLOWER
  // (64 streams: 13.56k -> 12.52k tok/s) — the projection behind it then starts, and holds SMs,
  // two kernels early
  rmsnorm_parts_kernel<<<n_tokens, 256, 0, st>>>(x, parts, n_parts, part_stride, (const __nv_bfloat16*)gain,
                                                 (__nv_bfloat16*)y, hidden, eps, 0u);
  LLMLB_LAUNCH_CHECK();
  return LLMLB_OK;
}

__global__ void __launch_bounds__(256) synth_kernel(__nv_bfloat16* __restrict__ out,
                                                    uint64_t rows, uint64_t cols, uint64_t row0,
                                                    uint64_t col0, uint64_t ld, uint64_t seed,
                                                    uint32_t tensor_id, float scale) {
  const uint64_t n = rows * cols;
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += uint64_t(gridDim.x) * blockDim.x) {
    uint64_t r = i / cols, c = i - r * cols;
    uint64_t gidx = (row0 + r) * ld + (col0 + c);
    out[i] = __float2bfloat16_rn(synth_value(seed, tensor_id, gidx, scale));
  }
}

}  // namespace llmlb

using namespace llmlb;

extern "C" int llmlb_op_embed(const void* table, const int32_t* ids, float* x, uint32_t n_tokens,
                              uint32_t hidden, uint32_t vocab, void* stream) {
  if (!table || !ids || !x || hidden % 8) {
    set_error("llmlb_op_embed: bad argument");
    return LLMLB_E_INVALID_ARG;
  }
  if (n_tokens == 0) return LLMLB_OK;
  embed_kernel<<<n_tokens, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)table, ids, x, hidden, vocab);
  LLMLB_LAUNCH_CHECK();
  return LLMLB_OK;
}

extern "C" int llmlb_op_rmsnorm(const float* x, const void* gain, void* y, uint32_t n_tokens,
                                uint32_t hidden, float eps, void* stream) {
  if (!x || !gain || !y || hidden % 4) {
    set_error("llmlb_op_rmsnorm: bad argument");
    return LLMLB_E_INVALID_ARG;
  }
  if (n_tokens == 0) return LLMLB_OK;
  rmsnorm_kernel<<<n_tokens, 256, 0, (cudaStream_t)stream>>>(
      x, (const __nv_bfloat16*)gain, (__nv_bfloat16*)y, hidden, eps);
  LLMLB_LAUNCH_CHECK();
  return LLMLB_OK;
}

// The residual fold + RMSNorm exactly as forward_tokens launches it between projections (kernel tests): n_tokens picks
// the 4-CTA cluster kernel or the one-CTA-per-row kernel, as in the engine.
extern "C" int llmlb_debug_rmsnorm_parts(float* x, const float* parts, uint32_t n_parts, uint64_t part_stride,
                                         const void* gain, void* y, uint32_t n_tokens, uint32_t hidden, float eps,
                                         void* stream) {
  if (!x || (n_parts > 0 && !parts) || (gain && !y) || hidden % 4 || n_parts > 16 ||
      part_stride < uint64_t(n_tokens) * hidden) {
    set_error("llmlb_debug_rmsnorm_parts: bad argument");
    return LLMLB_E_INVALID_ARG;
  }
  return rmsnorm_parts_launch(x, parts, n_parts, part_stride, gain, y, n_tokens, hidden, eps, (cudaStream_t)stream);
}

extern "C" int llmlb_op_synth_bf16(void* out, uint64_t rows, uint64_t cols, uint64_t row0,
                                   uint64_t col0, uint64_t ld, uint64_t seed, uint32_t tensor_id,
                                   float std, void* stream) {
  if (!out) {
    set_error("llmlb_op_synth_bf16: null output");
    return LLMLB_E_INVALID_ARG;
  }
  if (rows * cols == 0) return LLMLB_OK;
  uint64_t n = rows * cols;
  uint32_t grid = (uint32_t)((n + 255) / 256 < uint64_t(kNumSMs) * 16 ? (n + 255) / 256
                                                                        : uint64_t(kNumSMs) * 16);
  synth_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)out, rows, cols, row0,
                                                       col0, ld, seed, tensor_id,
                                                       std / kSynthSumStd);
  LLMLB_LAUNCH_CHECK();
  return LLMLB_OK;
}
