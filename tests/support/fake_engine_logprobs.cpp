// TEST INFRASTRUCTURE — NOT PRODUCT.  The scripted engine of fake_engine_penalties.cpp (included below, unchanged) plus
// llmlb_request_submit_logprobs and llmlb_request_poll_logprobs, so that the HTTP shim's handling of OpenAI logprobs can be
// tested without a GPU (tests/test_logprobs_server_cpu.py).  The entry points make the product's argument checks; the
// scripted record of token t is  logprob = -(1 + t % 7) / 4  with alternatives t, t + 7, t + 14, ... (mod vocab) at
// logprob, logprob - 1, logprob - 2, ... — exact in binary, so the test can restate every value.  A server linked to
// fake_engine_penalties.cpp alone stands for an engine library that predates the entry points.
#include <limits>

#include "fake_engine_penalties.cpp"

namespace {
std::mutex g_lp_mu;
std::map<std::pair<const llmlb_engine*, uint64_t>, uint32_t> g_lp;   // (engine, request) -> top_logprobs (ids are never reused)
}  // namespace

extern "C" {
int llmlb_request_submit_logprobs(llmlb_engine* e, const int32_t* ids, uint32_t n, const llmlb_sampling* s, const llmlb_penalties* pen,
                                  uint32_t top_logprobs, uint64_t* req_id) {
  if (top_logprobs > LLMLB_MAX_TOP_LOGPROBS) return fail(LLMLB_E_INVALID_ARG, "top_logprobs must be in [0, 20]");
  const int rc = pen ? llmlb_request_submit_penalized(e, ids, n, s, pen, req_id) : llmlb_request_submit(e, ids, n, s, req_id);
  if (rc == LLMLB_OK) {
    std::lock_guard<std::mutex> lk(g_lp_mu);
    g_lp[{e, *req_id}] = top_logprobs;
  }
  return rc;
}

int llmlb_request_poll_logprobs(llmlb_engine* e, uint64_t req_id, llmlb_token_event* out, llmlb_token_logprobs* lp, uint32_t cap,
                                uint32_t* n_out, int timeout_ms) {
  const int rc = llmlb_request_poll(e, req_id, out, cap, n_out, timeout_ms);
  if (rc != LLMLB_OK || !lp) return rc;
  int top = -1;
  {
    std::lock_guard<std::mutex> lk(g_lp_mu);
    auto it = g_lp.find({e, req_id});
    if (it != g_lp.end()) top = int(it->second);
  }
  const int32_t vocab = int32_t(e->cfg.model.vocab);
  for (uint32_t i = 0; i < *n_out; ++i) {
    llmlb_token_logprobs r{};
    r.logprob = std::numeric_limits<float>::quiet_NaN();
    const int32_t t = out[i].token_id;
    if (top >= 0 && t >= 0) {
      r.logprob = -float(1 + t % 7) / 4.f;
      r.n_top = uint32_t(std::min(top, int(vocab)));
      for (uint32_t j = 0; j < r.n_top; ++j) { r.top_ids[j] = int32_t((t + 7 * int64_t(j)) % vocab); r.top_logprobs[j] = r.logprob - float(j); }
    }
    lp[i] = r;
  }
  return rc;
}
}  // extern "C"
