// TEST INFRASTRUCTURE — NOT PRODUCT.  The scripted engine of fake_engine_logprobs.cpp (included below, unchanged) plus
// llmlb_request_submit_prompt_logprobs and llmlb_request_poll_prompt_logprobs, so that the HTTP shim's handling of OpenAI
// completions' echo with logprobs can be tested without a GPU (tests/test_prompt_logprobs_server_cpu.py).  Prompt record i
// reports t = prompt[i + 1] with the scripted record of fake_engine_logprobs.cpp:  logprob = -(1 + t % 7) / 4,
// alternatives t, t + 7, t + 14, ... (mod vocab) at logprob, logprob - 1, ... — exact in binary.  The first poll returns
// them all, later polls none.  A server linked to fake_engine_logprobs.cpp alone stands for an engine library that predates
// the entry points.
#include <algorithm>

#include "fake_engine_logprobs.cpp"

namespace {
std::mutex g_plp_mu;
std::map<std::pair<const llmlb_engine*, uint64_t>, std::deque<llmlb_token_logprobs>> g_plp;   // undelivered prompt records
}  // namespace

extern "C" {
int llmlb_request_submit_prompt_logprobs(llmlb_engine* e, const int32_t* ids, uint32_t n, const llmlb_sampling* s,
                                         const llmlb_penalties* pen, uint32_t top_logprobs, uint64_t* req_id) {
  if (top_logprobs > LLMLB_MAX_TOP_LOGPROBS) return fail(LLMLB_E_INVALID_ARG, "top_logprobs must be in [0, 20]");
  const int rc = llmlb_request_submit_logprobs(e, ids, n, s, pen, top_logprobs, req_id);
  if (rc != LLMLB_OK) return rc;
  const int32_t vocab = int32_t(e->cfg.model.vocab);
  std::deque<llmlb_token_logprobs> recs;
  for (uint32_t i = 0; i + 1 < n; ++i) {
    const int32_t t = ids[i + 1];
    llmlb_token_logprobs r{};
    r.logprob = -float(1 + t % 7) / 4.f;
    r.n_top = std::min(top_logprobs, uint32_t(vocab));
    for (uint32_t j = 0; j < r.n_top; ++j) { r.top_ids[j] = int32_t((t + 7 * int64_t(j)) % vocab); r.top_logprobs[j] = r.logprob - float(j); }
    recs.push_back(r);
  }
  std::lock_guard<std::mutex> lk(g_plp_mu);
  g_plp[{e, *req_id}] = std::move(recs);
  return rc;
}

int llmlb_request_poll_prompt_logprobs(llmlb_engine* e, uint64_t req_id, llmlb_token_logprobs* out, uint32_t cap, uint32_t* n_out) {
  if (!e || !out || !n_out || cap == 0) return fail(LLMLB_E_INVALID_ARG, "llmlb_request_poll_prompt_logprobs: bad argument");
  *n_out = 0;
  {
    std::lock_guard<std::mutex> lk(e->mu);
    if (!e->reqs.count(req_id)) return fail(LLMLB_E_NOT_FOUND, "unknown request id");
  }
  std::lock_guard<std::mutex> lk(g_plp_mu);
  auto it = g_plp.find({e, req_id});
  if (it == g_plp.end()) return LLMLB_OK;
  while (*n_out < cap && !it->second.empty()) { out[(*n_out)++] = it->second.front(); it->second.pop_front(); }
  return LLMLB_OK;
}
}  // extern "C"
