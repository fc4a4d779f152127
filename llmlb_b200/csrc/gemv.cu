// Decode projections (SURVEY §8 a2.3/8/9/10/11 at 1..4 tokens): an HBM-bound GEMV.
//
// out[t, n] = sum_k x[t, k] * W[n, k], W row-major bf16 [n_out, k] streamed exactly once.
// Layout of the work: a warp owns groups of 4 consecutive weight rows; each lane streams
// 16-byte pieces of those rows (fully coalesced 512 B per warp per row) with
// ld.global.nc.L1::no_allocate, the activation vector sits in shared memory as bf16, fp32
// accumulation, one xor-shuffle tree per row, epilogue on lane 0.  The first row group's
// loads are issued BEFORE the prologue so the RMSNorm (fused: a2.2) overlaps the HBM latency.
// Algorithmic bytes per launch: n_out*k*2 (weights) — x and out are noise.
#include "../../include/llmlb_b200.h"

#include "common.cuh"

namespace llmlb {

constexpr int kGemvThreads = 512;
constexpr int kGemvRows = 4;  // rows per warp trip


template <int B, int EPI>
__device__ __forceinline__ void gemv_epilogue(const float (&acc)[kGemvRows][B], void* out,
                                              uint32_t row0, uint32_t n_out,
                                              uint32_t out_stride) {
  if constexpr (EPI == LLMLB_EPI_SILU_MUL) {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
#pragma unroll
    for (int r = 0; r < kGemvRows; r += 2) {
      if (row0 + r + 1 < n_out) {
#pragma unroll
        for (int b = 0; b < B; ++b) {
          float g = acc[r][b], u = acc[r + 1][b];
          float s = g / (1.f + __expf(-g));
          o[size_t(b) * out_stride + ((row0 + r) >> 1)] = __float2bfloat16_rn(s * u);
        }
      }
    }
  } else {
#pragma unroll
    for (int r = 0; r < kGemvRows; ++r) {
      if (row0 + r < n_out) {
#pragma unroll
        for (int b = 0; b < B; ++b) {
          size_t idx = size_t(b) * out_stride + row0 + r;
          if constexpr (EPI == LLMLB_EPI_STORE_BF16)
            reinterpret_cast<__nv_bfloat16*>(out)[idx] = __float2bfloat16_rn(acc[r][b]);
          else if constexpr (EPI == LLMLB_EPI_RESID_F32)
            reinterpret_cast<float*>(out)[idx] += acc[r][b];
          else
            reinterpret_cast<float*>(out)[idx] = acc[r][b];
        }
      }
    }
  }
}

template <int B, int EPI, bool NORM>
__global__ void __launch_bounds__(kGemvThreads)
gemv_kernel(const __nv_bfloat16* __restrict__ W, const void* __restrict__ xin,
            const __nv_bfloat16* __restrict__ gain, float eps, void* __restrict__ out,
            uint32_t n_out, uint32_t K, uint32_t out_stride) {
  constexpr int U = 2;  // 16-byte loads in flight per row per lane (x2: register double buffer)
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(smem_raw);  // [B][K]
  __shared__ float red[B][kGemvThreads / 32];

  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t warps_total = gridDim.x * (kGemvThreads / 32);
  const uint32_t n_groups = (n_out + kGemvRows - 1) / kGemvRows;
  uint32_t group = blockIdx.x * (kGemvThreads / 32) + warp;

  // ---- prefetch the first row group (weights do not depend on the prologue) ----
  uint4 wf[kGemvRows][U];
  auto load_rows = [&](uint32_t g, uint32_t kk) {
#pragma unroll
    for (int r = 0; r < kGemvRows; ++r) {
      uint32_t row = min(g * kGemvRows + r, n_out - 1);
      const __nv_bfloat16* p = W + size_t(row) * K + kk;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (kk + u * 256 < K) wf[r][u] = ldg_stream(p + u * 256);
        else wf[r][u] = make_uint4(0, 0, 0, 0);
      }
    }
  };
  if (group < n_groups) load_rows(group, lane * 8);

  // ---- prologue: stage x in shared memory as bf16 (optionally RMS-normalised) ----
  if constexpr (NORM) {
    const float* xf = reinterpret_cast<const float*>(xin);
    float ss[B];
#pragma unroll
    for (int b = 0; b < B; ++b) ss[b] = 0.f;
    for (uint32_t i = threadIdx.x; i < K / 4; i += kGemvThreads) {
#pragma unroll
      for (int b = 0; b < B; ++b) {
        float4 v = reinterpret_cast<const float4*>(xf + size_t(b) * K)[i];
        ss[b] += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      }
    }
#pragma unroll
    for (int b = 0; b < B; ++b) {
      float s = warp_sum(ss[b]);
      if (lane == 0) red[b][warp] = s;
    }
    __syncthreads();
    float rs[B];
#pragma unroll
    for (int b = 0; b < B; ++b) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < kGemvThreads / 32; ++w) tot += red[b][w];
      rs[b] = rsqrtf(tot / float(K) + eps);
    }
    for (uint32_t i = threadIdx.x; i < K / 4; i += kGemvThreads) {
      uint2 g = __ldg(reinterpret_cast<const uint2*>(gain) + i);
#pragma unroll
      for (int b = 0; b < B; ++b) {
        float4 v = reinterpret_cast<const float4*>(xf + size_t(b) * K)[i];
        uint2 o;
        o.x = pack_bf16(v.x * rs[b] * bf16_lo(g.x), v.y * rs[b] * bf16_hi(g.x));
        o.y = pack_bf16(v.z * rs[b] * bf16_lo(g.y), v.w * rs[b] * bf16_hi(g.y));
        reinterpret_cast<uint2*>(xs + size_t(b) * K)[i] = o;
      }
    }
  } else {
    const uint4* xb = reinterpret_cast<const uint4*>(xin);
    for (uint32_t i = threadIdx.x; i < B * K / 8; i += kGemvThreads)
      reinterpret_cast<uint4*>(xs)[i] = xb[i];
  }
  __syncthreads();

  // ---- main loop over row groups ----
  for (; group < n_groups; group += warps_total) {
    float acc[kGemvRows][B];
#pragma unroll
    for (int r = 0; r < kGemvRows; ++r)
#pragma unroll
      for (int b = 0; b < B; ++b) acc[r][b] = 0.f;

    for (uint32_t kk = lane * 8; kk < K; kk += 256 * U) {
      // weights of this trip are already in wf (prefetched); copy and fetch the next trip
      uint4 wc[kGemvRows][U];
#pragma unroll
      for (int r = 0; r < kGemvRows; ++r)
#pragma unroll
        for (int u = 0; u < U; ++u) wc[r][u] = wf[r][u];
      {
        uint32_t nk = kk + 256 * U;
        uint32_t ng = group;
        if (nk >= K) { nk = lane * 8; ng = group + warps_total; }
        if (ng < n_groups) load_rows(ng, nk);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (kk + u * 256 < K) {
#pragma unroll
          for (int b = 0; b < B; ++b) {
            uint4 xv = *reinterpret_cast<const uint4*>(xs + size_t(b) * K + kk + u * 256);
            float x0 = bf16_lo(xv.x), x1 = bf16_hi(xv.x), x2 = bf16_lo(xv.y), x3 = bf16_hi(xv.y);
            float x4 = bf16_lo(xv.z), x5 = bf16_hi(xv.z), x6 = bf16_lo(xv.w), x7 = bf16_hi(xv.w);
#pragma unroll
            for (int r = 0; r < kGemvRows; ++r) {
              uint4 w = wc[r][u];
              float a = acc[r][b];
              a = fmaf(bf16_lo(w.x), x0, a); a = fmaf(bf16_hi(w.x), x1, a);
              a = fmaf(bf16_lo(w.y), x2, a); a = fmaf(bf16_hi(w.y), x3, a);
              a = fmaf(bf16_lo(w.z), x4, a); a = fmaf(bf16_hi(w.z), x5, a);
              a = fmaf(bf16_lo(w.w), x6, a); a = fmaf(bf16_hi(w.w), x7, a);
              acc[r][b] = a;
            }
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < kGemvRows; ++r)
#pragma unroll
      for (int b = 0; b < B; ++b) acc[r][b] = warp_sum(acc[r][b]);
    if (lane == 0) gemv_epilogue<B, EPI>(acc, out, group * kGemvRows, n_out, out_stride);
  }
}

template <int B, int EPI, bool NORM>
int launch_gemv(const void* w, const void* x, const void* gain, float eps, void* out,
                uint32_t n_out, uint32_t k, uint32_t out_stride, cudaStream_t st) {
  auto kern = gemv_kernel<B, EPI, NORM>;
  size_t smem = size_t(B) * k * 2;
  static size_t configured = 0;  // per instantiation (process-wide: one GPU per process)
  static int blocks_per_sm = 0;
  if (smem > configured) {
    LLMLB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)smem));
    configured = smem;
    blocks_per_sm = 0;
  }
  if (blocks_per_sm == 0) {
    LLMLB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kern,
                                                                  kGemvThreads, smem));
    if (blocks_per_sm < 1) blocks_per_sm = 1;
    if (blocks_per_sm > 2) blocks_per_sm = 2;
  }
  int n_sm = kNumSMs;
  uint32_t n_groups = (n_out + kGemvRows - 1) / kGemvRows;
  uint32_t need = (n_groups + kGemvThreads / 32 - 1) / (kGemvThreads / 32);
  uint32_t grid = (uint32_t)(n_sm * blocks_per_sm);
  if (grid > need) grid = need;
  kern<<<grid, kGemvThreads, smem, st>>>((const __nv_bfloat16*)w, x, (const __nv_bfloat16*)gain,
                                         eps, out, n_out, k, out_stride);
  LLMLB_LAUNCH_CHECK();
  return LLMLB_OK;
}

template <int B, int EPI>
int dispatch_norm(bool norm, const void* w, const void* x, const void* gain, float eps, void* out,
                  uint32_t n_out, uint32_t k, uint32_t out_stride, cudaStream_t st) {
  if (norm) return launch_gemv<B, EPI, true>(w, x, gain, eps, out, n_out, k, out_stride, st);
  return launch_gemv<B, EPI, false>(w, x, gain, eps, out, n_out, k, out_stride, st);
}

template <int B>
int dispatch_epi(uint32_t epi, bool norm, const void* w, const void* x, const void* gain,
                 float eps, void* out, uint32_t n_out, uint32_t k, uint32_t out_stride,
                 cudaStream_t st) {
  switch (epi) {
    case LLMLB_EPI_STORE_BF16:
      return dispatch_norm<B, LLMLB_EPI_STORE_BF16>(norm, w, x, gain, eps, out, n_out, k,
                                                    out_stride, st);
    case LLMLB_EPI_RESID_F32:
      return dispatch_norm<B, LLMLB_EPI_RESID_F32>(norm, w, x, gain, eps, out, n_out, k,
                                                   out_stride, st);
    case LLMLB_EPI_SILU_MUL:
      return dispatch_norm<B, LLMLB_EPI_SILU_MUL>(norm, w, x, gain, eps, out, n_out, k,
                                                  out_stride, st);
    case LLMLB_EPI_STORE_F32:
      return dispatch_norm<B, LLMLB_EPI_STORE_F32>(norm, w, x, gain, eps, out, n_out, k,
                                                   out_stride, st);
  }
  set_error("llmlb_op_gemv: unknown epilogue");
  return LLMLB_E_INVALID_ARG;
}

int gemv_ks_try(const void* w, const void* x, const void* gain, float eps, void* out,
                uint32_t n_tokens, uint32_t n_out, uint32_t k, uint32_t epi, uint32_t out_stride,
                cudaStream_t st, const void* pf_ptr = nullptr, uint32_t pf_bytes = 0);

// Decode projection (engine-internal): the K-split kernel when the shape fits, else the public op
int gemv_decode(const void* w, const void* x, const void* gain, float eps, void* out, uint32_t n_tokens,
                uint32_t n_out, uint32_t k, uint32_t epi, uint32_t out_stride, cudaStream_t st) {
  int rc = gemv_ks_try(w, x, gain, eps, out, n_tokens, n_out, k, epi, out_stride, st);
  if (rc != LLMLB_E_UNSUPPORTED) return rc;
  return llmlb_op_gemv(w, x, gain, eps, out, n_tokens, n_out, k, epi, out_stride, st);
}

}  // namespace llmlb

using namespace llmlb;

extern "C" int llmlb_op_gemv(const void* w, const void* x, const void* gain, float eps, void* out,
                             uint32_t n_tokens, uint32_t n_out, uint32_t k, uint32_t epilogue,
                             uint32_t out_stride, void* stream) {
  if (!w || !x || !out || n_out == 0 || k == 0 || k % 8 != 0) {
    set_error("llmlb_op_gemv: bad argument (k must be a multiple of 8)");
    return LLMLB_E_INVALID_ARG;
  }
  if (epilogue == LLMLB_EPI_SILU_MUL && (n_out & 1)) {
    set_error("llmlb_op_gemv: SILU_MUL needs interleaved gate/up rows (even n_out)");
    return LLMLB_E_INVALID_ARG;
  }
  if (size_t(k) * 2 > 200 * 1024) {
    set_error("llmlb_op_gemv: k too large for the shared-memory activation stage");
    return LLMLB_E_INVALID_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  bool norm = gain != nullptr;
  if (n_tokens > 1 && n_tokens <= 4 && size_t(n_tokens) * k * 2 > 200 * 1024) {
    // very wide K (e.g. an un-sharded 70B down projection): one token per pass — the weights are
    // streamed once per token on this rare path
    const size_t x_step = size_t(k) * (norm ? 4 : 2);
    const size_t o_elems = epilogue == LLMLB_EPI_SILU_MUL ? out_stride : out_stride;
    const size_t o_step = o_elems * ((epilogue == LLMLB_EPI_STORE_BF16 || epilogue == LLMLB_EPI_SILU_MUL) ? 2 : 4);
    for (uint32_t t = 0; t < n_tokens; ++t) {
      int rc = llmlb_op_gemv(w, (const uint8_t*)x + t * x_step, gain, eps, (uint8_t*)out + t * o_step, 1, n_out, k,
                             epilogue, out_stride, stream);
      if (rc != LLMLB_OK) return rc;
    }
    return LLMLB_OK;
  }
  if (n_tokens >= 1 && n_tokens <= 4 && epilogue <= LLMLB_EPI_STORE_F32) {
    // K-split kernel (gemv_ks.cu) for every shape it takes; the row-owner kernel below is the
    // fallback for odd K.  (A bulk-copy shared-memory ring variant measured slower in round 1 and is not
    // part of the library.)
    int rc = gemv_ks_try(w, x, gain, eps, out, n_tokens, n_out, k, epilogue, out_stride, st);
    if (rc != LLMLB_E_UNSUPPORTED) return rc;
  }
  switch (n_tokens) {
    case 0: return LLMLB_OK;
    case 1: return dispatch_epi<1>(epilogue, norm, w, x, gain, eps, out, n_out, k, out_stride, st);
    case 2: return dispatch_epi<2>(epilogue, norm, w, x, gain, eps, out, n_out, k, out_stride, st);
    case 3: return dispatch_epi<3>(epilogue, norm, w, x, gain, eps, out, n_out, k, out_stride, st);
    case 4: return dispatch_epi<4>(epilogue, norm, w, x, gain, eps, out, n_out, k, out_stride, st);
  }
  set_error("llmlb_op_gemv: n_tokens must be 1..4 (use llmlb_op_gemm beyond)");
  return LLMLB_E_INVALID_ARG;
}
