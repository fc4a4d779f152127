// Token log-probabilities (OpenAI logprobs / top_logprobs), computed on the device right after sample_kernel from the
// row it sampled.  Definition (include/llmlb_b200.h at llmlb_token_logprobs; mirrored by tests/logprob_oracle.py):
//   z    = the logits row sample_kernel reads: after penalties and logit bias, before temperature, top-k and top-p
//   m    = max z,  s = sum_j expf(z_j - m)   (accurate expf; the fp32 terms are summed in fp64, rounded once to fp32)
//   lp_j = (z_j - m) - logf(s)               (fp32; a -inf entry gives -inf)
//   top-n: the n = min(top_n, vocab) largest z, ordered by descending z with ties by ascending token id.
// The sampled token's value comes from the same expression, so it equals its list entry bit for bit.
//
// One CTA per row.  The n-th largest element is found by a radix select over a 64-bit key that orders elements
// exactly as the list does: (order-preserving bits of z) << 32 | ~id.  Keys are distinct, so exactly n elements have
// a key >= the selected one; they are collected in any order and sorted by one warp.  Nothing depends on the order in
// which threads run: tensor-parallel ranks compute identical records from the same all-gathered logits.
// A plain launch: no programmatic dependency, no wait on another CTA, legal inside stream capture.
#include "../../include/llmlb_b200.h"
#include "common.cuh"

namespace llmlb {

constexpr int kLpThreads = 1024;
static_assert(sizeof(llmlb_token_logprobs) == 168, "logprob record layout");

// z -> uint32 whose unsigned order is z's order; -0 maps to +0 (equal values are ties, broken by id)
__device__ __forceinline__ uint32_t lp_order_key(float z) {
  const uint32_t u = z == 0.f ? 0u : __float_as_uint(z);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ uint64_t lp_key(float z, uint32_t id) { return (uint64_t(lp_order_key(z)) << 32) | (~id); }

// One pass over the row: f(i, z[i], in_row) for i = threadIdx.x + k * kLpThreads, in increasing i per thread.  The loads
// of kLpUnroll iterations are issued before any is used (one CTA streams a whole row: without that the pass waits on one
// load per thread at a time), and every thread runs the same number of iterations, so f may use warp collectives.
constexpr int kLpUnroll = 8;
// The select only looks at z >= m - d for the smallest d of these that leaves at least n elements (counted in the sum
// pass): a language model's row has few such elements, so the select passes skip nearly every warp.
constexpr int kLpFloors = 6;
__device__ __forceinline__ float lp_floor_gap(int f) { return 0.25f * float(1 << (2 * f)); }   // 1/4, 1, 4, 16, 64, 256
template <typename F>
__device__ __forceinline__ void lp_row_pass(const float* __restrict__ z, uint32_t vocab, F&& f) {
  for (uint32_t base = 0; base < vocab; base += kLpThreads * kLpUnroll) {
    float v[kLpUnroll];
#pragma unroll
    for (int u = 0; u < kLpUnroll; ++u) {
      const uint32_t i = base + u * kLpThreads + threadIdx.x;
      v[u] = i < vocab ? z[i] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < kLpUnroll; ++u) {
      const uint32_t i = base + u * kLpThreads + threadIdx.x;
      f(i, v[u], i < vocab);
    }
  }
}

// rows with top_n[slot] < 0 are skipped (their records are not written)
__global__ void __launch_bounds__(kLpThreads)
logprob_kernel(const float* __restrict__ logits_all, uint32_t vocab, const int32_t* __restrict__ tokens,
               const int32_t* __restrict__ top_n, const int32_t* __restrict__ row_slot,
               llmlb_token_logprobs* __restrict__ out) {
  __shared__ float s_redf[32];
  __shared__ double s_redd[32];
  __shared__ uint32_t s_hist[256];
  __shared__ uint64_t s_prefix;
  __shared__ uint32_t s_need, s_done, s_n_found;
  __shared__ uint64_t s_win_key[LLMLB_MAX_TOP_LOGPROBS];
  __shared__ uint32_t s_cnt[32][kLpFloors];

  const uint32_t row = blockIdx.x;
  const int32_t n_req = top_n[row_slot ? row_slot[row] : row];
  if (n_req < 0) return;
  const uint32_t n = min(uint32_t(n_req), min(vocab, uint32_t(LLMLB_MAX_TOP_LOGPROBS)));
  const float* z = logits_all + size_t(row) * vocab;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  // m = max z
  float m = -INFINITY;
  lp_row_pass(z, vocab, [&](uint32_t, float v, bool in) { if (in) m = fmaxf(m, v); });
  m = warp_max(m);
  if (lane == 0) s_redf[warp] = m;
  __syncthreads();
  m = warp_max(s_redf[lane]);

  // s = sum expf(z - m): fp32 terms, fp64 sums (fixed order: strided per thread, butterfly, warps 0..31); and the
  // number of elements above each candidate floor
  double acc = 0.0;
  uint32_t cnt[kLpFloors] = {};
  lp_row_pass(z, vocab, [&](uint32_t, float v, bool in) {
    if (!in) return;
    acc += double(expf(__fsub_rn(v, m)));
#pragma unroll
    for (int f = 0; f < kLpFloors; ++f) cnt[f] += v >= __fsub_rn(m, lp_floor_gap(f));
  });
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    acc += __shfl_xor_sync(0xffffffffu, acc, o);
#pragma unroll
    for (int f = 0; f < kLpFloors; ++f) cnt[f] += __shfl_xor_sync(0xffffffffu, cnt[f], o);
  }
  if (lane == 0) {
    s_redd[warp] = acc;
#pragma unroll
    for (int f = 0; f < kLpFloors; ++f) s_cnt[warp][f] = cnt[f];
  }
  __syncthreads();
  double tot = 0.0;
  for (int w = 0; w < 32; ++w) tot += s_redd[w];
  const float ls = logf(__double2float_rn(tot));
  bool use_floor = false;   // no floor: every element takes part
  float floor_v = -INFINITY;
  for (int f = kLpFloors - 1; f >= 0; --f) {
    uint32_t c = 0;
    for (int w = 0; w < 32; ++w) c += s_cnt[w][f];
    if (c >= n) { use_floor = true; floor_v = __fsub_rn(m, lp_floor_gap(f)); }
  }
  auto cand = [&](float v) { return !use_floor || v >= floor_v; };

  // threshold: the n-th largest key (all keys >= thr are the list); n == 0 skips the select, n == vocab takes all
  uint64_t thr = 0;
  if (n > 0 && n < vocab) {
    if (threadIdx.x == 0) { s_prefix = 0; s_need = n; s_done = 0; }
    for (int shift = 56; shift >= 0; shift -= 8) {
      for (uint32_t i = threadIdx.x; i < 256; i += kLpThreads) s_hist[i] = 0;
      __syncthreads();
      const uint64_t prefix = s_prefix;
      const uint64_t pmask = shift == 56 ? 0ull : (~0ull << (shift + 8));
      // After the first pass few elements still match the prefix: a warp without one skips at the cost of a ballot.  The
      // first pass puts most of a row into a few bins: the lanes that share the first active lane's bin add once.
      lp_row_pass(z, vocab, [&](uint32_t i, float v, bool in) {
        uint32_t bin = 256u;   // outside the row or the prefix
        if (in && cand(v)) {
          const uint64_t k = lp_key(v, i);
          if ((k & pmask) == prefix) bin = uint32_t(k >> shift) & 255u;
        }
        const uint32_t act = __ballot_sync(0xffffffffu, bin < 256u);
        if (act) {
          const int first = __ffs(act) - 1;
          const uint32_t lead = __shfl_sync(0xffffffffu, bin, first);
          const uint32_t same = __ballot_sync(0xffffffffu, bin == lead);
          if (lane == uint32_t(first)) atomicAdd(&s_hist[lead], uint32_t(__popc(same)));
          else if (bin < 256u && bin != lead) atomicAdd(&s_hist[bin], 1u);
        }
      });
      __syncthreads();
      if (warp == 0) {   // from the top bin down: the bin where the running count reaches s_need
        uint32_t c[8], sum = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) { c[j] = s_hist[255 - (lane * 8 + j)]; sum += c[j]; }
        uint32_t inc = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= uint32_t(o)) inc += t;
        }
        const uint32_t need = s_need;
        uint32_t above = inc - sum;   // count in higher bins
        int bin = -1;
        uint32_t above_at = 0, cnt_at = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (bin < 0 && above + c[j] >= need) { bin = 255 - (lane * 8 + j); above_at = above; cnt_at = c[j]; }
          above += c[j];
        }
        const uint32_t hit = __ballot_sync(0xffffffffu, bin >= 0);
        const int src = __ffs(hit) - 1;   // need <= elements under the prefix: some lane hits
        bin = __shfl_sync(0xffffffffu, bin, src);
        above_at = __shfl_sync(0xffffffffu, above_at, src);
        cnt_at = __shfl_sync(0xffffffffu, cnt_at, src);
        if (lane == 0) {
          s_prefix = prefix | (uint64_t(bin) << shift);
          s_need = need - above_at;
          s_done = cnt_at == need - above_at;   // the whole bin is in the list: keys >= prefix are exactly n
        }
      }
      __syncthreads();
      if (s_done) break;
    }
    thr = s_prefix;
  }

  // gather the list (any order), then one warp sorts it by key, descending
  if (threadIdx.x == 0) s_n_found = 0;
  __syncthreads();
  if (n > 0) {
    lp_row_pass(z, vocab, [&](uint32_t i, float v, bool in) {
      if (in && cand(v) && lp_key(v, i) >= thr) s_win_key[atomicAdd(&s_n_found, 1u)] = lp_key(v, i);
    });
  }
  __syncthreads();
  llmlb_token_logprobs* rec = out + row;
  if (warp == 0) {
    if (lane < n) {
      const uint64_t k = s_win_key[lane];
      uint32_t rank = 0;
      for (uint32_t j = 0; j < n; ++j) rank += s_win_key[j] > k;
      const uint32_t id = ~uint32_t(k);
      rec->top_ids[rank] = int32_t(id);
      rec->top_logprobs[rank] = __fsub_rn(__fsub_rn(z[id], m), ls);
    } else if (lane < LLMLB_MAX_TOP_LOGPROBS) {   // unused entries: a fixed filler, so equal rows give equal records
      rec->top_ids[lane] = -1;
      rec->top_logprobs[lane] = 0.f;
    }
    if (lane == 0) {
      const int32_t t = tokens[row];
      rec->n_top = n;
      rec->logprob = (t >= 0 && uint32_t(t) < vocab) ? __fsub_rn(__fsub_rn(z[t], m), ls) : __int_as_float(0x7fc00000);
    }
  }
}

int logprob_launch(const float* logits, uint32_t n_rows, uint32_t vocab, const int32_t* tokens, const int32_t* top_n,
                   const int32_t* row_slot, llmlb_token_logprobs* out, cudaStream_t st) {
  if (n_rows == 0) return LLMLB_OK;
  logprob_kernel<<<n_rows, kLpThreads, 0, st>>>(logits, vocab, tokens, top_n, row_slot, out);
  LLMLB_LAUNCH_CHECK();
  return LLMLB_OK;
}

}  // namespace llmlb

using namespace llmlb;

extern "C" int llmlb_op_logprobs(const float* logits, uint32_t n_rows, uint32_t vocab, const int32_t* tokens,
                                 const int32_t* top_n, llmlb_token_logprobs* out_records, void* stream) {
  if (!logits || !tokens || !top_n || !out_records || vocab == 0) {
    set_error("llmlb_op_logprobs: bad argument");
    return LLMLB_E_INVALID_ARG;
  }
  return logprob_launch(logits, n_rows, vocab, tokens, top_n, nullptr, out_records, (cudaStream_t)stream);
}
