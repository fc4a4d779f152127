// TEST INFRASTRUCTURE — NOT PRODUCT.  The scripted engine of fake_engine.cpp (included below, unchanged) plus
// llmlb_request_submit_penalized, so that the HTTP shim's handling of frequency_penalty / presence_penalty / logit_bias can
// be tested without a GPU (tests/test_penalties_server_cpu.py).  The entry point makes the product's argument checks; the
// scripted effect is that a bias of +100 forces its token — every token event of the request carries that id, as greedy
// decoding would produce (poll rewrites the scripted ids, so stop ids still see the scripted source).  A server linked to
// fake_engine.cpp alone stands for an engine library that predates the entry point.
#include <cmath>
#include <map>
#include <mutex>
#include <set>

// the scripted source's own poll / release, wrapped below.  Its anonymous-namespace types live in this file's unit now,
// which is what the warning would point out.
#pragma GCC diagnostic ignored "-Wsubobject-linkage"
#define llmlb_request_poll scripted_request_poll
#define llmlb_request_release scripted_request_release
#include "fake_engine.cpp"
#undef llmlb_request_poll
#undef llmlb_request_release

namespace {
std::mutex g_forced_mu;
std::map<std::pair<const llmlb_engine*, uint64_t>, int32_t> g_forced;   // (engine, request) -> forced token id
}  // namespace

extern "C" {
int llmlb_request_submit_penalized(llmlb_engine* e, const int32_t* ids, uint32_t n, const llmlb_sampling* s, const llmlb_penalties* pen,
                                   uint64_t* req_id) {
  int32_t forced = -1;
  if (pen) {
    auto in = [](float v, float lim) { return std::isfinite(v) && v >= -lim && v <= lim; };
    if (!in(pen->frequency_penalty, 2.f)) return fail(LLMLB_E_INVALID_ARG, "frequency_penalty must be finite and in [-2, 2]");
    if (!in(pen->presence_penalty, 2.f)) return fail(LLMLB_E_INVALID_ARG, "presence_penalty must be finite and in [-2, 2]");
    if (pen->n_bias > LLMLB_MAX_LOGIT_BIAS) return fail(LLMLB_E_INVALID_ARG, "logit_bias has more than 1024 entries");
    if (pen->n_bias && (!pen->bias_ids || !pen->bias_values)) return fail(LLMLB_E_INVALID_ARG, "logit_bias: NULL ids or values");
    if (!e) return fail(LLMLB_E_INVALID_ARG, "bad argument");
    std::set<int32_t> seen;
    for (uint32_t i = 0; i < pen->n_bias; ++i) {
      const int32_t id = pen->bias_ids[i];
      if (id < 0 || uint32_t(id) >= e->cfg.model.vocab) return fail(LLMLB_E_INVALID_ARG, "logit_bias: token id outside the vocabulary");
      if (!seen.insert(id).second) return fail(LLMLB_E_INVALID_ARG, "logit_bias: duplicate token id");
      if (!in(pen->bias_values[i], 100.f)) return fail(LLMLB_E_INVALID_ARG, "logit_bias: value must be finite and in [-100, 100]");
      if (pen->bias_values[i] == 100.f && forced < 0) forced = id;
    }
  }
  const int rc = llmlb_request_submit(e, ids, n, s, req_id);
  if (rc == LLMLB_OK && forced >= 0) {
    std::lock_guard<std::mutex> lk(g_forced_mu);
    g_forced[{e, *req_id}] = forced;
  }
  return rc;
}

int llmlb_request_poll(llmlb_engine* e, uint64_t req_id, llmlb_token_event* out, uint32_t cap, uint32_t* n_out, int timeout_ms) {
  const int rc = scripted_request_poll(e, req_id, out, cap, n_out, timeout_ms);
  if (rc != LLMLB_OK) return rc;
  std::lock_guard<std::mutex> lk(g_forced_mu);
  auto it = g_forced.find({e, req_id});
  if (it != g_forced.end())
    for (uint32_t i = 0; i < *n_out; ++i)
      if (out[i].token_id >= 0) out[i].token_id = it->second;
  return rc;
}

int llmlb_request_release(llmlb_engine* e, uint64_t req_id) {
  {
    std::lock_guard<std::mutex> lk(g_forced_mu);
    g_forced.erase({e, req_id});
  }
  return scripted_request_release(e, req_id);
}
}  // extern "C"
