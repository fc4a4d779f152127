// TEST INFRASTRUCTURE — NOT PRODUCT.  The scripted engine of fake_engine_prompt_logprobs.cpp (included below, unchanged) plus
// llmlb_request_cached_tokens and llmlb_engine_prefix_cache_stats, so that the HTTP shim's usage reporting of the prefix
// cache can be tested without a GPU (tests/test_prefix_cache_server_cpu.py).  With llmlb_engine_config.prefix_cache set, a
// request of n prompt tokens reports 64 * floor((n - 1) / 64) cached tokens, the most the engine can match; otherwise 0.
// A server linked to fake_engine_prompt_logprobs.cpp alone stands for an engine library without the prefix cache.
#include "fake_engine_prompt_logprobs.cpp"

extern "C" {
int llmlb_request_cached_tokens(llmlb_engine* e, uint64_t req_id, uint32_t* n) {
  if (!e || !n) return fail(LLMLB_E_INVALID_ARG, "llmlb_request_cached_tokens: null argument");
  std::lock_guard<std::mutex> lk(e->mu);
  auto it = e->reqs.find(req_id);
  if (it == e->reqs.end()) return fail(LLMLB_E_NOT_FOUND, "unknown request id");
  const uint32_t np = uint32_t(it->second->prompt.size());
  *n = e->cfg.prefix_cache ? 64 * ((np - 1) / 64) : 0;
  return LLMLB_OK;
}

int llmlb_engine_prefix_cache_stats(const llmlb_engine* e, llmlb_prefix_cache_stats* out) {
  if (!e || !out) return fail(LLMLB_E_INVALID_ARG, "llmlb_engine_prefix_cache_stats: null argument");
  memset(out, 0, sizeof(*out));
  return LLMLB_OK;
}
}  // extern "C"
