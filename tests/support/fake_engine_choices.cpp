// TEST INFRASTRUCTURE — NOT PRODUCT.  The scripted engine of fake_engine_prefix_cache.cpp (included below, unchanged) plus
// llmlb_request_submit_choices, so that the HTTP shim's handling of OpenAI's n can be tested without a GPU
// (tests/test_choices_server_cpu.py).  Choice i is the request the matching single submit makes with seed + i: with a
// temperature the choices draw different scripted tokens, greedy ones the same.  n outside [1, max_seqs] is refused with
// the engine's message.  A server linked to fake_engine_prefix_cache.cpp alone stands for an engine library without it.
#include "fake_engine_prefix_cache.cpp"

extern "C" {
int llmlb_request_submit_choices(llmlb_engine* e, const int32_t* ids, uint32_t n_prompt, const llmlb_sampling* s,
                                 const llmlb_penalties* pen, int32_t top_logprobs, uint32_t prompt_logprobs, uint32_t n,
                                 uint64_t* req_ids) {
  if (!e || !s || !req_ids) return fail(LLMLB_E_INVALID_ARG, "llmlb_request_submit_choices: bad argument");
  if (n == 0 || n > e->cfg.max_seqs)
    return fail(LLMLB_E_INVALID_ARG, "llmlb_request_submit_choices: n must be in [1, max_seqs = " + std::to_string(e->cfg.max_seqs) +
                                         "], got " + std::to_string(n));
  for (uint32_t i = 0; i < n; ++i) {
    llmlb_sampling si = *s;
    si.seed = s->seed + i;
    const int rc = prompt_logprobs ? llmlb_request_submit_prompt_logprobs(e, ids, n_prompt, &si, pen, uint32_t(top_logprobs), &req_ids[i])
                 : top_logprobs >= 0 ? llmlb_request_submit_logprobs(e, ids, n_prompt, &si, pen, uint32_t(top_logprobs), &req_ids[i])
                 : pen ? llmlb_request_submit_penalized(e, ids, n_prompt, &si, pen, &req_ids[i])
                       : llmlb_request_submit(e, ids, n_prompt, &si, &req_ids[i]);
    if (rc != LLMLB_OK) {
      for (uint32_t j = 0; j < i; ++j) { llmlb_request_cancel(e, req_ids[j]); llmlb_request_release(e, req_ids[j]); }
      return rc;
    }
  }
  return LLMLB_OK;
}
}  // extern "C"
