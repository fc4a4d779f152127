// Token sampling (SURVEY §8 a2.12): arg-max, or temperature / top-k / top-p with a counter RNG.
//
// One CTA (1024 threads) per row of fp32 logits [vocab].  Definition (mirrored by
// oracle/sampling_ref.py):
//   T <= 0 (or NaN): arg-max, lowest index on ties
//   e_i = exp((logit_i - max logit) / T)                      (the max maps to exactly 1: no finite
//                                                               T > 0 overflows into inf - inf)
//   top-k : keep e_i >= (k-th largest e)                      (ties at the threshold all kept)
//   top-p : for top_p < 1, of those keep e_i >= v where v is the value at which the descending
//           cumulative mass first reaches top_p * (kept mass) (ties kept; top_p <= 0 keeps the
//           maximum(s))
//   draw  : u = U[0,1) from (seed, step); the first index in VOCAB order whose running kept
//           mass exceeds u * (kept mass)
// Thresholds are found by an 8-bit radix select over the (monotone) bit pattern of e_i: each
// pass histograms count and mass per bin in shared memory and a single warp suffix-scans the
// 256 bins with shuffles to pick the bin where the cumulative crosses the target.
// The per-bin masses are accumulated in 2^-40 FIXED POINT with integer atomics: integer addition is
// associative, so the threshold — and with it the sampled token — does not depend on the order in
// which threads reach the atomics.  Tensor-parallel ranks sample the same all-gathered logits
// independently and must agree bit for bit (their schedulers replay each other's finishes).
// The draw sums e in fp32 in a fixed order (no atomics), and always resolves to a kept token
// with e > 0 inside the warp span that holds the target (see the search below).
#include "../../include/llmlb_b200.h"
#include "common.cuh"

namespace llmlb {

constexpr int kSampThreads = 1024;
typedef unsigned long long u64q;   // probability mass in units of 2^-40 (e <= 1, vocab < 2^17: sums stay below 2^58)
__device__ __forceinline__ u64q mass_q(float e) { return (u64q)__float2ull_rd(e * 1099511627776.f); }

// e = exp((logit - lmax) / T).  The max maps to exp(0) = 1 and everything below it to a finite or
// -inf exponent, even when 1/T overflows to inf (T below ~3e-39): (0 * inf) is never formed.
__device__ __forceinline__ float scaled_exp(float logit, float lmax, float inv_t) {
  const float d = logit - lmax;
  return __expf(d < 0.f ? d * inv_t : 0.f);
}

__device__ __forceinline__ float block_reduce_max(float v, float* red) {
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[threadIdx.x & 31];
  r = warp_max(r);
  __syncthreads();
  return r;
}
__device__ __forceinline__ float block_reduce_sum(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[threadIdx.x & 31];
  r = warp_sum(r);
  __syncthreads();
  return r;
}

// Radix select on keys e_i (as uint bits) restricted to e_i >= floor_key.
// mode 0: largest key v such that count(e >= v) >= target_count
// mode 1: largest key v such that mass(e >= v)  >= target_mass
__device__ uint32_t radix_select(const float* __restrict__ logits, uint32_t vocab, float inv_t,
                                 float lmax, uint32_t floor_key, int mode, uint32_t target_count,
                                 u64q target_mass, int* s_cnt, u64q* s_mass, uint32_t* s_sel,
                                 u64q* s_above) {
  uint32_t prefix = 0, prefix_mask = 0;
  uint32_t cnt_above = 0;
  u64q mass_above = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += kSampThreads) {
      s_cnt[i] = 0;
      s_mass[i] = 0;
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < vocab; i += kSampThreads) {
      float e = scaled_exp(logits[i], lmax, inv_t);
      uint32_t key = __float_as_uint(e);
      if (key >= floor_key && (key & prefix_mask) == prefix) {
        uint32_t b = (key >> shift) & 255u;
        atomicAdd(&s_cnt[b], 1);
        if (mode == 1) atomicAdd(&s_mass[b], mass_q(e));
      }
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      // suffix scan from bin 255 down: lane l owns bins [255-8l-7, 255-8l]
      const int lane = threadIdx.x;
      int c_loc[8];
      u64q m_loc[8];
      int c_sum = 0;
      u64q m_sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int b = 255 - (lane * 8 + j);
        c_loc[j] = s_cnt[b];
        m_loc[j] = s_mass[b];
        c_sum += c_loc[j];
        m_sum += m_loc[j];
      }
      int c_inc = c_sum;
      u64q m_inc = m_sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int c2 = __shfl_up_sync(0xffffffffu, c_inc, o);
        u64q m2 = __shfl_up_sync(0xffffffffu, m_inc, o);
        if (lane >= o) { c_inc += c2; m_inc += m2; }
      }
      int c_run = c_inc - c_sum + int(cnt_above);   // mass/count strictly above this lane's bins
      u64q m_run = m_inc - m_sum + mass_above;
      int found_bin = -1;
      int c_at = 0;
      u64q m_at = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        bool hit = (mode == 0) ? (uint32_t(c_run + c_loc[j]) >= target_count)
                               : (m_run + m_loc[j] >= target_mass);
        if (found_bin < 0 && hit && c_loc[j] > 0) {
          found_bin = 255 - (lane * 8 + j);
          c_at = c_run;
          m_at = m_run;
        }
        c_run += c_loc[j];
        m_run += m_loc[j];
      }
      // first lane (highest bins) that found a crossing wins
      uint32_t ballot = __ballot_sync(0xffffffffu, found_bin >= 0);
      if (ballot == 0) {
        // target beyond the total: take the lowest non-empty bin
        uint32_t nz = 0;
        int low = -1;
#pragma unroll
        for (int j = 7; j >= 0; --j)
          if (c_loc[j] > 0 && low < 0) low = 255 - (lane * 8 + j);
        nz = __ballot_sync(0xffffffffu, low >= 0);
        int src = nz ? (31 - __clz(nz)) : 0;
        int lb = __shfl_sync(0xffffffffu, low, src);
        if (lane == 0) {
          s_sel[0] = uint32_t(lb < 0 ? 0 : lb);
          s_sel[1] = cnt_above;
          s_above[0] = mass_above;
          s_sel[2] = 1;  // exhausted
        }
      } else {
        int src = __ffs(ballot) - 1;
        int fb = __shfl_sync(0xffffffffu, found_bin, src);
        int ca = __shfl_sync(0xffffffffu, c_at, src);
        u64q ma = __shfl_sync(0xffffffffu, m_at, src);
        if (lane == 0) {
          s_sel[0] = uint32_t(fb);
          s_sel[1] = uint32_t(ca);
          s_above[0] = ma;
          s_sel[2] = 0;
        }
      }
    }
    __syncthreads();
    prefix |= s_sel[0] << shift;
    prefix_mask |= 255u << shift;
    cnt_above = s_sel[1];
    mass_above = s_above[0];
    __syncthreads();
  }
  return prefix;
}

__global__ void __launch_bounds__(kSampThreads)
sample_kernel(const float* __restrict__ logits_all, uint32_t vocab,
              const float* __restrict__ temperature, const float* __restrict__ top_p,
              const int32_t* __restrict__ top_k, const uint64_t* __restrict__ seed,
              const uint64_t* __restrict__ step, int32_t* __restrict__ out_ids) {
  __shared__ float red[32];
  __shared__ int red_i[32];
  __shared__ int s_cnt[256];
  __shared__ u64q s_mass[256];
  __shared__ uint32_t s_sel[4];
  __shared__ u64q s_above[2];
  __shared__ u64q red_q[32];
  __shared__ float s_warp_tot[32];
  __shared__ int s_result;

  const uint32_t row = blockIdx.x;
  const float* logits = logits_all + size_t(row) * vocab;
  const float T = temperature ? temperature[row] : 0.f;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  if (!(T > 0.f)) {  // greedy: max value, lowest index on ties
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (uint32_t i = threadIdx.x; i < vocab; i += kSampThreads) {
      float v = logits[i];
      if (v > best) { best = v; bi = int(i); }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float ov = __shfl_xor_sync(0xffffffffu, best, o);
      int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) { red[warp] = best; red_i[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
      best = red[lane];
      bi = red_i[lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        float ov = __shfl_xor_sync(0xffffffffu, best, o);
        int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
      }
      if (lane == 0) out_ids[row] = (bi == 0x7fffffff) ? 0 : bi;
    }
    return;
  }

  const float inv_t = 1.f / T;
  float lmax = -INFINITY;
  for (uint32_t i = threadIdx.x; i < vocab; i += kSampThreads) lmax = fmaxf(lmax, logits[i]);
  lmax = block_reduce_max(lmax, red);

  uint32_t floor_key = 0;
  const int32_t k = top_k ? top_k[row] : 0;
  if (k > 0 && uint32_t(k) < vocab)
    floor_key = radix_select(logits, vocab, inv_t, lmax, 0u, 0, uint32_t(k), 0ull, s_cnt, s_mass,
                             s_sel, s_above);
  const float p = top_p ? top_p[row] : 1.f;
  if (p < 1.f) {   // top_p <= 0: a target mass of 0 selects the largest key, the maximum(s)
    u64q mass = 0;   // kept mass, same fixed point as the bins (integer sums: order-free)
    for (uint32_t i = threadIdx.x; i < vocab; i += kSampThreads) {
      float e = scaled_exp(logits[i], lmax, inv_t);
      if (__float_as_uint(e) >= floor_key) mass += mass_q(e);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mass += __shfl_xor_sync(0xffffffffu, mass, o);
    if (lane == 0) red_q[warp] = mass;
    __syncthreads();
    mass = 0;
    for (int w = 0; w < 32; ++w) mass += red_q[w];
    __syncthreads();
    const u64q target_q = (u64q)__double2ull_rd(double(p) * double(mass));
    floor_key = radix_select(logits, vocab, inv_t, lmax, floor_key, 1, 0u, target_q, s_cnt, s_mass,
                             s_sel, s_above);
  }

  // draw in vocab order: warp w owns a contiguous span, lanes interleaved (coalesced)
  const uint32_t span = ((vocab + 1023) / 1024) * 32;  // elements per warp
  const uint32_t w0 = warp * span;
  float wsum = 0.f;
  for (uint32_t i = w0 + lane; i < min(vocab, w0 + span); i += 32) {
    float e = scaled_exp(logits[i], lmax, inv_t);
    if (__float_as_uint(e) >= floor_key) wsum += e;
  }
  wsum = warp_sum(wsum);
  if (lane == 0) s_warp_tot[warp] = wsum;
  if (threadIdx.x == 0) s_result = -1;
  __syncthreads();
  float total = 0.f;
  float before = 0.f;  // mass in warps ahead of mine
  for (int w = 0; w < 32; ++w) {
    float t = s_warp_tot[w];
    if (w < int(warp)) before += t;
    total += t;
  }
  uint64_t h = mix64(mix64(seed ? seed[row] : 0ull) + (step ? step[row] : 0ull));
  const float u = float(uint32_t(h >> 40)) * (1.0f / 16777216.0f);
  const float target = u * total;
  // The warp intervals [before, before + wsum) tile [0, total) exactly: every thread forms `before`
  // and `total` by the same fp32 chain over s_warp_tot, and target = fl(u * total) < total for
  // u <= 1 - 2^-24.  So exactly one warp holds the target whenever total is finite.
  if (target >= before && target < before + wsum) {
    // The search below adds the same e in a different fp32 order (row scans, carried across rows)
    // than the lane sums and butterfly that formed wsum; the two totals differ by a few ulps.  A
    // target in between crosses no lane: it then belongs to this span's last kept token with e > 0
    // (one exists, since wsum > 0), whose CDF end is within that rounding of the target.
    float run = before;
    int found = -1, last = -1;
    for (uint32_t base = w0; base < min(vocab, w0 + span); base += 32) {
      uint32_t i = base + lane;
      float e = 0.f;
      if (i < vocab) {
        float ee = scaled_exp(logits[i], lmax, inv_t);
        if (__float_as_uint(ee) >= floor_key) e = ee;
      }
      float inc = e;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        float t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= uint32_t(o)) inc += t;
      }
      uint32_t hit = __ballot_sync(0xffffffffu, e > 0.f && run + inc > target);
      if (hit) {
        found = int(base + (__ffs(hit) - 1));
        break;
      }
      uint32_t pos = __ballot_sync(0xffffffffu, e > 0.f);
      if (pos) last = int(base + (31 - __clz(pos)));
      run += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) s_result = found >= 0 ? found : last;
  }
  __syncthreads();
  // s_result < 0 only when no warp holds the target: NaN or infinite logits (total not finite)
  if (threadIdx.x == 0) out_ids[row] = s_result < 0 ? 0 : s_result;
}

}  // namespace llmlb

using namespace llmlb;

extern "C" int llmlb_op_sample(const float* logits, uint32_t n_rows, uint32_t vocab,
                               const float* temperature, const float* top_p, const int32_t* top_k,
                               const uint64_t* seed, const uint64_t* step, int32_t* out_ids,
                               void* stream) {
  if (!logits || !out_ids || vocab == 0) {
    set_error("llmlb_op_sample: bad argument");
    return LLMLB_E_INVALID_ARG;
  }
  if (n_rows == 0) return LLMLB_OK;
  sample_kernel<<<n_rows, kSampThreads, 0, (cudaStream_t)stream>>>(
      logits, vocab, temperature, top_p, top_k, seed, step, out_ids);
  LLMLB_LAUNCH_CHECK();
  return LLMLB_OK;
}
