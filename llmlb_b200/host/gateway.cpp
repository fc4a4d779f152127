// Implementation of gateway.hpp plus an extern "C" surface (host_abi) for ctypes-driven tests.
#include "gateway.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace llmlb_host {

// ---------------------------------------------------------------- ModelTpsState --------------
void ModelTpsState::update_tps(uint64_t output_tokens, uint64_t duration_ms) {
  if (duration_ms == 0) return;
  const double current = double(output_tokens) / (double(duration_ms) / 1000.0);
  constexpr double kAlpha = 0.2;
  tps_ema = has_ema ? kAlpha * current + (1.0 - kAlpha) * tps_ema : current;
  has_ema = true;
  request_count += 1;
  total_output_tokens += output_tokens;
  total_duration_ms += duration_ms;
}

// ---------------------------------------------------------------- LoadManager ----------------
static bool id_eq(const std::string& a, const std::string& b) {
  if (a == b) return true;
  if (a.size() != b.size()) return false;
  for (size_t i = 0; i < a.size(); ++i) {
    char x = a[i], y = b[i];
    if (x >= 'A' && x <= 'Z') x = char(x - 'A' + 'a');
    if (y >= 'A' && y <= 'Z') y = char(y - 'A' + 'a');
    if (x != y) return false;
  }
  return true;
}

void LoadManager::add_mapping(const std::string& canonical, const std::string& alias) {
  std::lock_guard<std::mutex> lk(mu_);
  for (auto& m : mappings_)
    if (m.canonical == canonical) { m.aliases.push_back(alias); return; }
  mappings_.push_back({canonical, {alias}});
}

const ModelMapping* LoadManager::find_mapping(const std::string& model_id) const {
  for (auto& m : mappings_) {
    if (id_eq(m.canonical, model_id)) return &m;
    for (auto& a : m.aliases) if (id_eq(a, model_id)) return &m;
  }
  return nullptr;
}

static void push_unique(std::vector<std::string>& v, const std::string& s) {
  if (std::find(v.begin(), v.end(), s) == v.end()) v.push_back(s);
}

std::vector<std::string> LoadManager::model_lookup_keys(const std::string& model_id) const {
  std::vector<std::string> keys{model_id};
  if (const ModelMapping* m = find_mapping(model_id)) {
    push_unique(keys, m->canonical);
    for (auto& a : m->aliases) push_unique(keys, a);
  }
  return keys;
}

Endpoint* LoadManager::find(const std::string& id) {
  for (auto& e : endpoints_) if (e.id == id) return &e;
  return nullptr;
}
const Endpoint* LoadManager::find(const std::string& id) const {
  for (auto& e : endpoints_) if (e.id == id) return &e;
  return nullptr;
}

void LoadManager::add_endpoint(const std::string& id, bool online, bool initializing) {
  std::lock_guard<std::mutex> lk(mu_);
  if (find(id)) return;
  Endpoint e; e.id = id; e.online = online; e.initializing = initializing;
  endpoints_.push_back(e);
}
bool LoadManager::add_model(const std::string& eid, const std::string& model_id, const std::string& canonical) {
  std::lock_guard<std::mutex> lk(mu_);
  Endpoint* e = find(eid);
  if (!e) return false;
  e->models.push_back({model_id, canonical});
  return true;
}
bool LoadManager::set_status(const std::string& eid, bool online) {
  std::lock_guard<std::mutex> lk(mu_);
  Endpoint* e = find(eid);
  if (!e) return false;
  e->online = online;
  if (!online) {  // health/endpoint_checker.rs:313-317 clear_tps_for_endpoint
    for (auto it = tps_.begin(); it != tps_.end();) it = (std::get<0>(it->first) == eid) ? tps_.erase(it) : std::next(it);
  }
  return true;
}
bool LoadManager::set_initializing(const std::string& eid, bool v) {
  std::lock_guard<std::mutex> lk(mu_);
  Endpoint* e = find(eid);
  if (!e) return false;
  e->initializing = v;
  return true;
}

std::vector<std::string> LoadManager::find_by_model(const std::string& model_id) const {
  std::lock_guard<std::mutex> lk(mu_);
  const auto keys = model_lookup_keys(model_id);
  std::vector<std::string> out;
  for (auto& ep : endpoints_) {
    if (!ep.online) continue;
    bool hit = false;
    for (auto& m : ep.models) {
      auto ek = model_lookup_keys(m.model_id);
      if (!m.canonical_name.empty()) for (auto& k : model_lookup_keys(m.canonical_name)) push_unique(ek, k);
      for (auto& k : keys) if (std::find(ek.begin(), ek.end(), k) != ek.end()) hit = true;
    }
    if (hit) out.push_back(ep.id);
  }
  return out;
}

void LoadManager::update_tps(const std::string& eid, const std::string& model_id, TpsApiKind kind,
                             uint64_t output_tokens, uint64_t duration_ms) {
  std::lock_guard<std::mutex> lk(mu_);
  tps_[std::make_tuple(eid, model_id, int(kind))].update_tps(output_tokens, duration_ms);
}
bool LoadManager::get_tps(const std::string& eid, const std::string& model_id, TpsApiKind kind, ModelTpsState* out) const {
  std::lock_guard<std::mutex> lk(mu_);
  auto it = tps_.find(std::make_tuple(eid, model_id, int(kind)));
  if (it == tps_.end()) return false;
  *out = it->second;
  return true;
}

double LoadManager::score(const Endpoint& ep, const std::string* model, int kind) const {
  if (model) {
    if (kind < 0) return 0.0;
    double best = 0.0;
    for (auto& kv : tps_)
      if (std::get<0>(kv.first) == ep.id && std::get<1>(kv.first) == *model && std::get<2>(kv.first) == kind && kv.second.has_ema)
        best = std::max(best, kv.second.tps_ema);
    return best;
  }
  uint64_t tok = 0, dur = 0;
  for (auto& kv : tps_)
    if (std::get<0>(kv.first) == ep.id && (kind < 0 || std::get<2>(kv.first) == kind)) {
      tok += kv.second.total_output_tokens;
      dur += kv.second.total_duration_ms;
    }
  return dur > 0 ? double(tok) / (double(dur) / 1000.0) : 0.0;
}

SelectError LoadManager::select(const std::string* model, int kind, std::string* out_id) {
  std::vector<std::string> ids;
  if (model) ids = find_by_model(*model);
  std::lock_guard<std::mutex> lk(mu_);
  std::vector<const Endpoint*> eps;
  if (model) { for (auto& id : ids) eps.push_back(find(id)); }
  else { for (auto& e : endpoints_) if (e.online) eps.push_back(&e); }
  if (eps.empty()) return model ? kNoCapableEndpoints : kNoEndpointsAvailable;
  std::vector<const Endpoint*> cands;
  for (auto* e : eps) if (!e->initializing) cands.push_back(e);
  if (cands.empty()) return kNoEndpointsAvailable;
  const uint64_t cursor = round_robin_.fetch_add(1);
  const size_t n = cands.size(), start = size_t(cursor % n);
  struct Item { const Endpoint* e; double s; size_t rank; };
  std::vector<Item> items;
  for (size_t i = 0; i < n; ++i) items.push_back({cands[i], score(*cands[i], model, kind), (i + n - start) % n});
  std::stable_sort(items.begin(), items.end(), [](const Item& a, const Item& b) {
    if (a.s != b.s) return a.s > b.s;
    return a.rank < b.rank;
  });
  *out_id = items[0].e->id;
  return kSelectOk;
}

bool LoadManager::begin_request(const std::string& eid) {
  std::lock_guard<std::mutex> lk(mu_);
  Endpoint* e = find(eid);
  if (!e) return false;
  e->active_requests += 1;
  e->total_requests += 1;
  return true;
}
bool LoadManager::finish_request(const std::string& eid, bool success, uint64_t duration_ms, uint64_t output_tokens) {
  std::lock_guard<std::mutex> lk(mu_);
  Endpoint* e = find(eid);
  if (!e) return false;
  if (e->active_requests) e->active_requests -= 1;
  (success ? e->success : e->errors) += 1;
  e->latency_ms_sum += duration_ms;
  e->output_tokens += output_tokens;
  return true;
}
bool LoadManager::begin_request_lease(const std::string& eid, RequestLease* out) {
  if (!begin_request(eid)) return false;   // EndpointNotFound (balancer/mod.rs:2274-2276)
  *out = RequestLease(this, eid);
  return true;
}
bool LoadManager::finish_request_outcome(const std::string& eid, RequestOutcome outcome, uint64_t duration_ms,
                                         const TokenUsage* usage) {
  std::lock_guard<std::mutex> lk(mu_);
  Endpoint* e = find(eid);
  if (!e) return false;
  if (outcome == RequestOutcome::Queued) return true;   // mod.rs:2300-2301: nothing moves
  if (e->active_requests) e->active_requests -= 1;
  (outcome == RequestOutcome::Success ? e->success : e->errors) += 1;
  e->latency_ms_sum += duration_ms;
  if (usage) {   // mod.rs:2376-2396
    if (usage->has_in) e->input_tokens += usage->in;
    if (usage->has_out) e->output_tokens += usage->out;
    if (usage->has_total) e->total_tokens += usage->total;
    else if (usage->has_in || usage->has_out) e->total_tokens += uint64_t(usage->has_in ? usage->in : 0) + (usage->has_out ? usage->out : 0);
  }
  return true;
}
bool LoadManager::endpoint_stats(const std::string& eid, Endpoint* out) const {
  std::lock_guard<std::mutex> lk(mu_);
  const Endpoint* e = find(eid);
  if (!e) return false;
  *out = *e;
  return true;
}
double LoadManager::average_latency_ms(const std::string& eid) const {
  std::lock_guard<std::mutex> lk(mu_);
  const Endpoint* e = find(eid);
  const uint64_t completed = e ? e->success + e->errors : 0;
  return completed ? double(e->latency_ms_sum) / double(completed) : -1.0;
}

RequestLease::RequestLease(LoadManager* lm, std::string endpoint_id)
    : lm_(lm), endpoint_id_(std::move(endpoint_id)), started_(std::chrono::steady_clock::now()) {}
RequestLease::RequestLease(RequestLease&& o) noexcept : lm_(o.lm_), endpoint_id_(std::move(o.endpoint_id_)), started_(o.started_) { o.lm_ = nullptr; }
RequestLease& RequestLease::operator=(RequestLease&& o) noexcept {
  if (this != &o) {
    if (lm_) lm_->finish_request_outcome(endpoint_id_, RequestOutcome::Error, elapsed_ms(), nullptr);   // the lease being overwritten leaks
    lm_ = o.lm_; endpoint_id_ = std::move(o.endpoint_id_); started_ = o.started_;
    o.lm_ = nullptr;
  }
  return *this;
}
RequestLease::~RequestLease() {   // lease.rs:71-100: dropped without complete => Error, elapsed time
  if (lm_) lm_->finish_request_outcome(endpoint_id_, RequestOutcome::Error, elapsed_ms(), nullptr);
  lm_ = nullptr;
}
uint64_t RequestLease::elapsed_ms() const {
  return uint64_t(std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::steady_clock::now() - started_).count());
}
bool RequestLease::complete(RequestOutcome outcome, uint64_t duration_ms) { return complete_with_tokens(outcome, duration_ms, nullptr); }
bool RequestLease::complete_with_tokens(RequestOutcome outcome, uint64_t duration_ms, const TokenUsage* usage) {
  LoadManager* lm = lm_;
  lm_ = nullptr;                       // take(): a second complete, or the destructor, is a no-op
  if (!lm) return true;
  return lm->finish_request_outcome(endpoint_id_, outcome, duration_ms, usage);
}

uint32_t LoadManager::active_requests(const std::string& eid) const {
  std::lock_guard<std::mutex> lk(mu_);
  const Endpoint* e = find(eid);
  return e ? e->active_requests : 0;
}

// ---------------------------------------------------------------- usage / accumulator --------
TokenUsage extract_or_estimate_tokens(const Json& body, const std::string* request_text, const std::string* response_text,
                                      TokenCountFn count, void* ctx) {
  TokenUsage u;
  if (extract_usage_from_response(body, &u)) return u;     // the usage field wins (token/mod.rs:241-244)
  u = TokenUsage{};
  auto est = [&](const std::string* t, bool* has, uint32_t* v) {
    if (!t || !count) return;
    const int64_t n = count(*t, ctx);
    if (n >= 0) { *has = true; *v = uint32_t(n); }
  };
  est(request_text, &u.has_in, &u.in);
  est(response_text, &u.has_out, &u.out);
  if (u.has_in || u.has_out) { u.has_total = true; u.total = (u.has_in ? u.in : 0) + (u.has_out ? u.out : 0); }
  return u;
}

bool extract_usage_from_response(const Json& body, TokenUsage* u) {
  const Json* usage = body.get("usage");
  if (!usage) {
    const Json* r = body.get("response");
    usage = r ? r->get("usage") : nullptr;
  }
  if (!usage) return false;
  *u = TokenUsage();
  auto pick = [&](const char* a, const char* b, bool* has, uint32_t* v) {
    const Json* j = usage->get(a);
    if (!j && b) j = usage->get(b);
    uint64_t x;
    if (j && j->as_u64(&x)) { *has = true; *v = uint32_t(x); }
  };
  pick("prompt_tokens", "input_tokens", &u->has_in, &u->in);
  pick("completion_tokens", "output_tokens", &u->has_out, &u->out);
  pick("total_tokens", nullptr, &u->has_total, &u->total);
  return true;
}

static std::string trim(const std::string& s) {
  size_t a = 0, b = s.size();
  auto ws = [](unsigned char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\f' || c == '\v'; };
  while (a < b && ws(s[a])) ++a;
  while (b > a && ws(s[b - 1])) --b;
  return s.substr(a, b - a);
}

void StreamingTokenAccumulator::process_chunk(const std::string& raw) {
  const std::string chunk = trim(raw);
  if (chunk.empty() || chunk[0] == ':') return;
  std::string data;
  if (chunk.compare(0, 6, "data: ") == 0) data = chunk.substr(6);
  else if (chunk.compare(0, 5, "data:") == 0) data = trim(chunk.substr(5));
  else return;
  if (data == "[DONE]") { done_ = true; return; }
  Json js;
  if (!Json::parse(data, &js)) return;
  TokenUsage u;
  if (extract_usage_from_response(js, &u)) { usage_ = u; has_usage_ = true; }
  if (const Json* choices = js.get("choices")) {
    if (choices->is_array())
      for (auto& c : choices->items()) {
        const Json* d = c.get("delta");
        const Json* content = d ? d->get("content") : nullptr;
        if (content && content->is_string()) content_ += content->str();
      }
  }
  if (const Json* t = js.get("type")) {
    if (t->is_string()) {
      if (t->str() == "response.output_text.delta") {
        const Json* d = js.get("delta");
        if (d && d->is_string()) content_ += d->str();
      } else if (t->str() == "response.output_text.done" && content_.empty()) {
        const Json* x = js.get("text");
        if (x && x->is_string()) content_ += x->str();
      }
    }
  }
}

void StreamingTokenAccumulator::feed(const char* data, size_t n) {
  line_buf_.append(data, n);
  size_t pos;
  while ((pos = line_buf_.find('\n')) != std::string::npos) {
    process_chunk(line_buf_.substr(0, pos));
    line_buf_.erase(0, pos + 1);
  }
}

TokenUsage StreamingTokenAccumulator::finalize(uint32_t (*estimate)(const std::string&)) const {
  if (has_usage_) return usage_;
  TokenUsage u;
  if (content_.empty()) { u.has_out = true; u.out = 0; }
  else if (estimate) { u.has_out = true; u.out = estimate(content_); }
  if (has_input_) { u.has_in = true; u.in = input_; }
  if (u.has_in && u.has_out) { u.has_total = true; u.total = u.in + u.out; }
  else if (u.has_in) { u.has_total = true; u.total = u.in; }
  else if (u.has_out) { u.has_total = true; u.total = u.out; }
  return u;
}

// ---------------------------------------------------------------- names / errors / auth ------
bool parse_quantized_model_name(const std::string& model, ParsedModelName* out) {
  out->raw = model;
  size_t pos = model.find(':');
  if (pos == std::string::npos) { out->base = model; out->has_quant = false; out->quantization.clear(); return true; }
  if (model.find(':', pos + 1) != std::string::npos || pos == 0 || pos == model.size() - 1) return false;
  out->base = model.substr(0, pos);
  out->quantization = model.substr(pos + 1);
  out->has_quant = true;
  return true;
}

std::string openai_error_body(const std::string& message, const std::string& type, int status) {
  Json err = Json::object();
  err.set("message", message); err.set("type", type); err.set("code", status);
  Json root = Json::object(); root.set("error", err);
  return root.dump();
}
std::string model_unavailable_body(const std::string& message, const std::string& code) {
  Json err = Json::object();
  err.set("message", message); err.set("type", "service_unavailable"); err.set("code", code);
  Json root = Json::object(); root.set("error", err);
  return root.dump();
}

// ---- error conventions -------------------------------------------------------------------------
ClientError classify_upstream_request_error(UpstreamFailure kind, uint32_t timeout_secs, const std::string* ollama_loading_model) {
  ClientError e;
  if (kind == UpstreamFailure::Timeout) {
    e.status = 504;
    if (ollama_loading_model) {
      e.type = "model_loading";
      e.message = "Ollama model '" + *ollama_loading_model + "' is still loading. Retry after the initial load finishes or increase endpoint inference timeout above " +
                  std::to_string(timeout_secs) + " seconds.";
    } else {
      e.type = "timeout";
      e.message = "Upstream endpoint request timed out after " + std::to_string(timeout_secs) + " seconds";
    }
    return e;
  }
  e.status = 502;
  if (kind == UpstreamFailure::Connect) { e.type = "connection_error"; e.message = "Failed to connect to upstream endpoint"; }
  else { e.type = "endpoint_request_error"; e.message = "Failed to proxy request to upstream endpoint"; }
  return e;
}
ClientError queue_capacity_exceeded(uint64_t queue_timeout_secs) {
  ClientError e;
  e.status = 429; e.type = "rate_limit_exceeded"; e.message = "Request queue is full";
  e.retry_after = (long long)(queue_timeout_secs < 1 ? 1 : queue_timeout_secs);
  return e;
}
ClientError queue_wait_timeout() {
  ClientError e;
  e.status = 504; e.type = "timeout"; e.message = "Queue wait timeout";
  return e;
}

namespace {
struct LbRow { const char* name; int status; const char* type; const char* external; bool expose_detail; };
// common/error.rs:124-204 (external_message, error_type, status_code) and api/error.rs:162-195 (which text reaches the client)
const LbRow kLbRows[] = {
    {"common_validation", 400, "invalid_request_error", "Request error", true},
    {"common_other", 400, "invalid_request_error", "Request error", false},
    {"endpoint_not_found", 404, "not_found_error", "Endpoint not found", false},
    {"not_found", 404, "not_found_error", "Not found", true},
    {"no_endpoints_available", 503, "service_unavailable", "No available endpoints", false},
    {"no_capable_endpoints", 404, "not_found_error", "No capable endpoints", false},
    {"database", 500, "server_error", "Database error", false},
    {"http", 502, "service_unavailable", "Backend service unavailable", false},
    {"timeout", 504, "server_error", "Request timeout", false},
    {"service_unavailable", 503, "service_unavailable", "Service temporarily unavailable", false},
    {"internal", 500, "server_error", "Internal server error", false},
    {"endpoint_offline", 503, "service_unavailable", "Endpoint offline", false},
    {"invalid_model_name", 400, "invalid_request_error", "Invalid model name", true},
    {"insufficient_storage", 507, "server_error", "Insufficient storage", true},
    {"password_hash", 401, "authentication_error", "Authentication error", false},
    {"jwt", 401, "authentication_error", "Authentication error", false},
    {"authentication", 401, "authentication_error", "Authentication failed", true},
    {"authorization", 403, "permission_error", "Access denied", true},
    {"conflict", 409, "invalid_request_error", "Resource conflict", true},
};
static_assert(sizeof(kLbRows) / sizeof(kLbRows[0]) == size_t(LbErrorKind::kCount), "one row per LbError variant");
const LbRow& lb_row(LbErrorKind k) { return kLbRows[size_t(k) < size_t(LbErrorKind::kCount) ? size_t(k) : size_t(LbErrorKind::Internal)]; }
}  // namespace
int lb_error_status(LbErrorKind k) { return lb_row(k).status; }
const char* lb_error_type(LbErrorKind k) { return lb_row(k).type; }
const char* lb_error_external_message(LbErrorKind k) { return lb_row(k).external; }
const char* lb_error_name(LbErrorKind k) { return lb_row(k).name; }
std::string lb_error_openai_body(LbErrorKind k) {
  Json err = Json::object();
  err.set("message", std::string(lb_row(k).external)); err.set("type", std::string(lb_row(k).type)); err.set("code", std::to_string(lb_row(k).status));
  Json root = Json::object(); root.set("error", err);
  return root.dump();
}
std::string app_error_body(LbErrorKind k, const std::string& detail) {
  bool expose = lb_row(k).expose_detail;
  if (k == LbErrorKind::CommonOther)   // only the GPU-requirement text of a non-validation CommonError is passed through
    expose = detail.find("GPU is required") != std::string::npos || detail.find("GPU hardware is required") != std::string::npos;
  Json root = Json::object();
  root.set("error", expose ? detail : std::string(lb_row(k).external));
  return root.dump();
}

int extract_api_key(const char* x_api_key, const char* authorization, std::string* key, std::string* err) {
  if (x_api_key) { *key = x_api_key; return 0; }
  if (authorization) {
    if (strncmp(authorization, "Bearer ", 7) == 0) { *key = authorization + 7; return 0; }
    *err = "Invalid Authorization header format. Expected 'Bearer <token>'";
    return 1;
  }
  *err = "Missing X-API-Key header or Authorization header";
  return 2;
}

// FIPS 180-4 SHA-256 (api keys are stored as SHA-256 hex, auth/middleware.rs:254-289)
std::string sha256_hex(const std::string& data) {
  static const uint32_t K[64] = {
      0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
      0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
      0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
      0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
      0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
      0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
      0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
  uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  std::string m = data;
  const uint64_t bits = uint64_t(data.size()) * 8;
  m.push_back(char(0x80));
  while (m.size() % 64 != 56) m.push_back(0);
  for (int i = 7; i >= 0; --i) m.push_back(char((bits >> (8 * i)) & 0xFF));
  auto rotr = [](uint32_t x, int n) { return (x >> n) | (x << (32 - n)); };
  for (size_t off = 0; off < m.size(); off += 64) {
    uint32_t w[64];
    for (int i = 0; i < 16; ++i)
      w[i] = (uint32_t(uint8_t(m[off + 4 * i])) << 24) | (uint32_t(uint8_t(m[off + 4 * i + 1])) << 16) |
             (uint32_t(uint8_t(m[off + 4 * i + 2])) << 8) | uint32_t(uint8_t(m[off + 4 * i + 3]));
    for (int i = 16; i < 64; ++i) {
      uint32_t s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
      uint32_t s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
      w[i] = w[i - 16] + s0 + w[i - 7] + s1;
    }
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
    for (int i = 0; i < 64; ++i) {
      uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25), ch = (e & f) ^ (~e & g);
      uint32_t t1 = hh + S1 + ch + K[i] + w[i];
      uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22), mj = (a & b) ^ (a & c) ^ (b & c);
      uint32_t t2 = S0 + mj;
      hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
  }
  char buf[65];
  for (int i = 0; i < 8; ++i) snprintf(buf + 8 * i, 9, "%08x", h[i]);
  return std::string(buf, 64);
}

// ---------------------------------------------------------------- wire format ----------------
std::string sse_event(const Json& j) { return "data: " + j.dump() + "\n\n"; }

Json chat_chunk(const std::string& id, const std::string& model, int64_t created,
                const std::string* role, const std::string* content, const char* finish_reason, const Json* logprobs,
                uint32_t index) {
  Json delta = Json::object();
  if (role) delta.set("role", *role);
  if (content) delta.set("content", *content);
  Json choice = Json::object();
  choice.set("index", index); choice.set("delta", delta);
  if (logprobs) choice.set("logprobs", *logprobs);
  choice.set("finish_reason", finish_reason ? Json(finish_reason) : Json());
  Json root = Json::object();
  root.set("id", id); root.set("object", "chat.completion.chunk"); root.set("created", created);
  root.set("model", model);
  Json choices = Json::array(); choices.push(choice);
  root.set("choices", choices);
  return root;
}
static Json cached_details(uint32_t n) {
  Json d = Json::object();
  d.set("cached_tokens", n);
  return d;
}
static Json chat_usage(uint32_t p, uint32_t c, const uint32_t* cached) {
  Json u = Json::object();
  u.set("prompt_tokens", p); u.set("completion_tokens", c); u.set("total_tokens", p + c);
  if (cached) u.set("prompt_tokens_details", cached_details(*cached));
  return u;
}
Json chat_usage_chunk(const std::string& id, const std::string& model, int64_t created, uint32_t p, uint32_t c, const uint32_t* cached) {
  Json root = Json::object();
  root.set("id", id); root.set("object", "chat.completion.chunk"); root.set("created", created);
  root.set("model", model); root.set("choices", Json::array()); root.set("usage", chat_usage(p, c, cached));
  return root;
}
Json chat_completion_body(const std::string& id, const std::string& model, int64_t created,
                          const std::string& content, const char* finish_reason, uint32_t p, uint32_t c, const Json* logprobs,
                          const uint32_t* cached) {
  return chat_completion_body(id, model, created, std::vector<ChoiceOut>{{content, finish_reason, logprobs}}, p, c, cached);
}
Json chat_completion_body(const std::string& id, const std::string& model, int64_t created, const std::vector<ChoiceOut>& outs,
                          uint32_t p, uint32_t c, const uint32_t* cached) {
  Json choices = Json::array();
  for (size_t i = 0; i < outs.size(); ++i) {
    Json msg = Json::object(); msg.set("role", "assistant"); msg.set("content", outs[i].text);
    Json choice = Json::object();
    choice.set("index", uint32_t(i)); choice.set("message", msg);
    if (outs[i].logprobs) choice.set("logprobs", *outs[i].logprobs);
    choice.set("finish_reason", outs[i].finish_reason ? Json(outs[i].finish_reason) : Json());
    choices.push(choice);
  }
  Json root = Json::object();
  root.set("id", id); root.set("object", "chat.completion"); root.set("created", created); root.set("model", model);
  root.set("choices", choices); root.set("usage", chat_usage(p, c, cached));
  return root;
}
Json completion_body(const std::string& id, const std::string& model, int64_t created,
                     const std::string& text, const char* finish_reason, uint32_t p, uint32_t c, const Json* logprobs,
                     const uint32_t* cached) {
  return completion_body(id, model, created, std::vector<ChoiceOut>{{text, finish_reason, logprobs}}, p, c, cached);
}
Json completion_body(const std::string& id, const std::string& model, int64_t created, const std::vector<ChoiceOut>& outs,
                     uint32_t p, uint32_t c, const uint32_t* cached) {
  Json choices = Json::array();
  for (size_t i = 0; i < outs.size(); ++i) {
    Json choice = Json::object();
    choice.set("index", uint32_t(i)); choice.set("text", outs[i].text);
    if (outs[i].logprobs) choice.set("logprobs", *outs[i].logprobs);
    choice.set("finish_reason", outs[i].finish_reason ? Json(outs[i].finish_reason) : Json());
    choices.push(choice);
  }
  Json root = Json::object();
  root.set("id", id); root.set("object", "text_completion"); root.set("created", created); root.set("model", model);
  root.set("choices", choices); root.set("usage", chat_usage(p, c, cached));
  return root;
}
Json completion_chunk(const std::string& id, const std::string& model, int64_t created, const std::string* text, const char* finish_reason,
                      const Json* logprobs, uint32_t index) {
  Json choice = Json::object();
  choice.set("index", index); choice.set("text", text ? *text : std::string()); choice.set("logprobs", logprobs ? *logprobs : Json());
  choice.set("finish_reason", finish_reason ? Json(finish_reason) : Json());
  Json choices = Json::array(); choices.push(choice);
  Json root = Json::object();
  root.set("id", id); root.set("object", "text_completion"); root.set("created", created); root.set("model", model);
  root.set("choices", choices);
  return root;
}
Json completion_usage_chunk(const std::string& id, const std::string& model, int64_t created, uint32_t p, uint32_t c,
                            const uint32_t* cached) {
  Json root = Json::object();
  root.set("id", id); root.set("object", "text_completion"); root.set("created", created);
  root.set("model", model); root.set("choices", Json::array()); root.set("usage", chat_usage(p, c, cached));
  return root;
}
// OpenAI writes a log-probability it cannot represent (-inf) as -9999.0
static Json logprob_value(float v) { return Json(std::isfinite(v) ? double(v) : -9999.0); }
static Json logprob_bytes(const std::string& b) {
  Json a = Json::array();
  for (unsigned char c : b) a.push(Json(int(c)));
  return a;
}
static Json chat_logprob_token(const LogprobToken& t) {
  Json j = Json::object();
  j.set("token", t.token); j.set("logprob", logprob_value(t.logprob)); j.set("bytes", logprob_bytes(t.bytes));
  return j;
}
Json chat_logprobs(const std::vector<LogprobEntry>& entries) {
  Json content = Json::array();
  for (const auto& e : entries) {
    Json j = chat_logprob_token(e.tok);
    Json top = Json::array();
    for (const auto& t : e.top) top.push(chat_logprob_token(t));
    j.set("top_logprobs", top);
    content.push(j);
  }
  Json root = Json::object();
  root.set("content", content); root.set("refusal", Json());
  return root;
}
Json completion_logprobs(const std::vector<LogprobEntry>& entries) {
  Json tokens = Json::array(), lps = Json::array(), tops = Json::array(), offs = Json::array();
  for (const auto& e : entries) {
    tokens.push(e.tok.token);
    if (!e.scored) {
      lps.push(Json());
      tops.push(Json());
    } else {
      lps.push(logprob_value(e.tok.logprob));
      Json top = Json::object();   // two alternatives with the same text: the more probable one is kept
      for (const auto& t : e.top) if (!top.get(t.token)) top.set(t.token, logprob_value(t.logprob));
      tops.push(top);
    }
    offs.push(Json(e.text_offset));
  }
  Json root = Json::object();
  root.set("tokens", tokens); root.set("token_logprobs", lps); root.set("top_logprobs", tops); root.set("text_offset", offs);
  return root;
}

static Json resp_usage(uint32_t i, uint32_t o, const uint32_t* cached) {
  Json u = Json::object();
  u.set("input_tokens", i); u.set("output_tokens", o); u.set("total_tokens", i + o);
  if (cached) u.set("input_tokens_details", cached_details(*cached));
  return u;
}
Json responses_body(const std::string& id, const std::string& model, int64_t created,
                    const std::string& text, uint32_t in, uint32_t out, const char* status, const uint32_t* cached) {
  Json part = Json::object(); part.set("type", "output_text"); part.set("text", text);
  Json content = Json::array(); content.push(part);
  Json item = Json::object(); item.set("type", "message"); item.set("role", "assistant"); item.set("content", content);
  Json output = Json::array(); output.push(item);
  Json root = Json::object();
  root.set("id", id); root.set("object", "response"); root.set("created_at", created); root.set("model", model);
  root.set("status", status); root.set("output", output); root.set("usage", resp_usage(in, out, cached));
  return root;
}
Json responses_event_created(const std::string& id, const std::string& model) {
  Json r = Json::object(); r.set("id", id); r.set("object", "response"); r.set("model", model);
  Json e = Json::object(); e.set("type", "response.created"); e.set("response", r);
  return e;
}
Json responses_event_item_added() {
  Json it = Json::object(); it.set("type", "message"); it.set("role", "assistant");
  Json e = Json::object(); e.set("type", "response.output_item.added"); e.set("item", it);
  return e;
}
Json responses_event_part_added() {
  Json p = Json::object(); p.set("type", "text"); p.set("text", "");
  Json e = Json::object(); e.set("type", "response.content_part.added"); e.set("part", p);
  return e;
}
Json responses_event_delta(const std::string& d) {
  Json e = Json::object(); e.set("type", "response.output_text.delta"); e.set("delta", d);
  return e;
}
Json responses_event_text_done(const std::string& t) {
  Json e = Json::object(); e.set("type", "response.output_text.done"); e.set("text", t);
  return e;
}
Json responses_event_done(const std::string& id, uint32_t in, uint32_t out, const uint32_t* cached) {
  Json r = Json::object(); r.set("id", id); r.set("object", "response"); r.set("status", "completed");
  r.set("usage", resp_usage(in, out, cached));
  Json e = Json::object(); e.set("type", "response.done"); e.set("response", r);
  return e;
}

std::vector<int32_t> byte_tokenize(const std::string& text, uint32_t vocab) {
  std::vector<int32_t> ids;
  for (unsigned char c : text) ids.push_back(int32_t((3u + c) % vocab));
  if (ids.empty()) ids.push_back(1);
  return ids;
}
std::string byte_detokenize(int32_t id) {
  if (id >= 3 && id < 259) {
    unsigned char c = (unsigned char)(id - 3);
    if (c < 0x80 && (c >= 0x20 || c == '\n' || c == '\t')) return std::string(1, char(c));
  }
  return "<|" + std::to_string(id) + "|>";
}

}  // namespace llmlb_host

// ---- 60-minute request history --------------------------------------------------------------------
namespace llmlb_host {
void RequestHistory::record(RequestOutcome outcome, int64_t ts) {
  const int64_t minute = align_to_minute(ts);
  std::lock_guard<std::mutex> lk(mu_);
  if (points_.empty() || points_.back().minute != minute) {
    RequestHistoryPoint p;
    p.minute = minute;
    points_.push_back(p);
  }
  RequestHistoryPoint& last = points_.back();
  if (outcome == RequestOutcome::Success) { if (last.success != UINT64_MAX) ++last.success; }
  else if (outcome == RequestOutcome::Error) { if (last.error != UINT64_MAX) ++last.error; }
  const int64_t cutoff = minute - 60 * (kWindowMinutes - 1);
  size_t drop = 0;
  while (drop < points_.size() && points_[drop].minute < cutoff) ++drop;
  if (drop) points_.erase(points_.begin(), points_.begin() + drop);
}

std::vector<RequestHistoryPoint> RequestHistory::window(int64_t now) const {
  now = align_to_minute(now);
  std::vector<RequestHistoryPoint> out;
  out.reserve(size_t(kWindowMinutes));
  std::lock_guard<std::mutex> lk(mu_);
  for (int64_t m = now - 60 * (kWindowMinutes - 1); m <= now; m += 60) {
    RequestHistoryPoint p;
    p.minute = m;
    for (const auto& q : points_)
      if (q.minute == m) { p = q; break; }
    out.push_back(p);
  }
  return out;
}
}  // namespace llmlb_host

// ---- stop strings -------------------------------------------------------------------------------
namespace llmlb_host {
StopMatcher::StopMatcher(std::vector<std::string> stops) {
  for (auto& st : stops)
    if (!st.empty()) stops_.push_back(std::move(st));
}

std::string StopMatcher::feed(const std::string& piece) {
  if (hit_) return "";
  if (stops_.empty()) return piece;
  held_ += piece;
  // earliest complete stop string (leftmost; the longer one when two start at the same place)
  size_t best = std::string::npos, best_len = 0;
  for (const auto& st : stops_) {
    const size_t p = held_.find(st);
    if (p != std::string::npos && (p < best || (p == best && st.size() > best_len))) { best = p; best_len = st.size(); }
  }
  if (best != std::string::npos) {
    hit_ = true;
    matched_ = held_.substr(best, best_len);
    std::string out = held_.substr(0, best);
    held_.clear();
    return out;
  }
  // longest suffix of the held text that is a proper prefix of some stop string stays held
  size_t keep = 0;
  for (const auto& st : stops_) {
    const size_t max_k = std::min(held_.size(), st.size() - 1);
    for (size_t k = max_k; k > keep; --k)
      if (held_.compare(held_.size() - k, k, st, 0, k) == 0) { keep = k; break; }
  }
  std::string out = held_.substr(0, held_.size() - keep);
  held_.erase(0, held_.size() - keep);
  return out;
}

std::string StopMatcher::flush() {
  std::string out;
  if (!hit_) out.swap(held_);
  held_.clear();
  return out;
}
}  // namespace llmlb_host

// ---- outbound payload preparation --------------------------------------------------------------
namespace llmlb_host {
namespace {
bool id_eq_ci(const std::string& a, const std::string& b) {
  if (a.size() != b.size()) return false;
  for (size_t i = 0; i < a.size(); ++i)
    if (tolower((unsigned char)a[i]) != tolower((unsigned char)b[i])) return false;
  return true;
}
}  // namespace

std::string resolve_engine_name(const std::string& model, const std::string& endpoint_type, const std::vector<EngineMapping>& mappings) {
  for (const auto& m : mappings) {
    bool knows = id_eq_ci(m.canonical, model);
    for (const auto& a : m.aliases) knows |= id_eq_ci(a.name, model);
    if (!knows) continue;
    for (const auto& a : m.aliases)
      if (a.engine == endpoint_type) return a.name;
    return "";
  }
  return "";
}

std::string resolve_runtime_model_name_for_endpoint(const std::string& requested, const std::string& selected,
                                                    const std::string& endpoint_type, const std::vector<EndpointModel>& endpoint_models,
                                                    const std::vector<EngineMapping>& mappings) {
  for (const auto& em : endpoint_models)
    if (em.model_id == requested) return requested;
  for (const auto& em : endpoint_models) {
    if (em.model_id == selected) return em.model_id;
    if (!em.canonical_name.empty() && (em.canonical_name == selected || em.canonical_name == requested)) return em.model_id;
  }
  const std::string alias = resolve_engine_name(selected, endpoint_type, mappings);
  return alias.empty() ? selected : alias;
}

Json rewrite_payload_model_for_endpoint(const Json& payload, const std::string& selected, const std::string& endpoint_type,
                                        const std::vector<EndpointModel>& endpoint_models, const std::vector<EngineMapping>& mappings) {
  const Json* m = payload.get("model");
  if (!m || !m->is_string()) return payload;
  const std::string runtime = resolve_runtime_model_name_for_endpoint(m->str(), selected, endpoint_type, endpoint_models, mappings);
  if (runtime == m->str()) return payload;
  Json out = payload;
  out.set("model", runtime);
  return out;
}

Json prepare_upstream_payload(const Json& payload, const std::string& upstream_model, bool stream) {
  Json out = payload;
  if (!out.is_object()) return out;
  out.set("model", upstream_model);
  if (stream) {
    const Json* opts = out.get("stream_options");
    if (!opts) {
      Json o = Json::object();
      o.set("include_usage", Json(true));
      out.set("stream_options", o);
    } else if (opts->is_object() && !opts->get("include_usage")) {
      Json o = *opts;
      o.set("include_usage", Json(true));
      out.set("stream_options", o);
    }
  }
  return out;
}
}  // namespace llmlb_host

// =============================================================================================
// extern "C" surface for ctypes tests (tests/test_host_gateway.py)
// =============================================================================================
using namespace llmlb_host;

static size_t copy_out(const std::string& s, char* out, size_t cap) {
  if (out && cap) {
    size_t n = std::min(cap - 1, s.size());
    memcpy(out, s.data(), n);
    out[n] = 0;
  }
  return s.size();
}

#include "../../include/llmlb_gateway.h"   // the exported signatures are checked against the public header at compile time
extern "C" {
void* llmlb_lm_create() { return new LoadManager(); }
void llmlb_lm_destroy(void* p) { delete static_cast<LoadManager*>(p); }
void llmlb_lm_add_mapping(void* p, const char* canonical, const char* alias) { static_cast<LoadManager*>(p)->add_mapping(canonical, alias); }
void llmlb_lm_add_endpoint(void* p, const char* id, int online, int initializing) { static_cast<LoadManager*>(p)->add_endpoint(id, online != 0, initializing != 0); }
int llmlb_lm_add_model(void* p, const char* eid, const char* model, const char* canonical) { return static_cast<LoadManager*>(p)->add_model(eid, model, canonical ? canonical : "") ? 0 : -1; }
int llmlb_lm_set_status(void* p, const char* eid, int online) { return static_cast<LoadManager*>(p)->set_status(eid, online != 0) ? 0 : -1; }
int llmlb_lm_set_initializing(void* p, const char* eid, int v) { return static_cast<LoadManager*>(p)->set_initializing(eid, v != 0) ? 0 : -1; }
void llmlb_lm_update_tps(void* p, const char* eid, const char* model, int kind, uint64_t tokens, uint64_t ms) { static_cast<LoadManager*>(p)->update_tps(eid, model, TpsApiKind(kind), tokens, ms); }
int llmlb_lm_get_tps(void* p, const char* eid, const char* model, int kind, double* ema, uint64_t* count, uint64_t* tokens, uint64_t* ms) {
  ModelTpsState s;
  if (!static_cast<LoadManager*>(p)->get_tps(eid, model, TpsApiKind(kind), &s)) return 0;
  *ema = s.has_ema ? s.tps_ema : -1.0; *count = s.request_count; *tokens = s.total_output_tokens; *ms = s.total_duration_ms;
  return 1;
}
int llmlb_lm_select(void* p, const char* model, int kind, char* out, size_t cap) {
  std::string id, m = model ? model : "";
  SelectError e = static_cast<LoadManager*>(p)->select(model ? &m : nullptr, kind, &id);
  if (e == kSelectOk) copy_out(id, out, cap);
  return int(e);
}
size_t llmlb_lm_lookup_keys(void* p, const char* model, char* out, size_t cap) {
  std::string joined;
  for (auto& k : static_cast<LoadManager*>(p)->model_lookup_keys(model)) { if (!joined.empty()) joined += "\n"; joined += k; }
  return copy_out(joined, out, cap);
}
int llmlb_lm_begin_request(void* p, const char* eid) { return static_cast<LoadManager*>(p)->begin_request(eid) ? 0 : -1; }
int llmlb_lm_finish_request(void* p, const char* eid, int success, uint64_t ms, uint64_t tokens) { return static_cast<LoadManager*>(p)->finish_request(eid, success != 0, ms, tokens) ? 0 : -1; }
uint32_t llmlb_lm_active(void* p, const char* eid) { return static_cast<LoadManager*>(p)->active_requests(eid); }
// leases: begin -> handle; complete (usage fields < 0 = absent) or drop (leak: the destructor finishes it as Error)
void* llmlb_lm_lease_begin(void* p, const char* eid) {
  RequestLease* l = new RequestLease();
  if (!static_cast<LoadManager*>(p)->begin_request_lease(eid, l)) { delete l; return nullptr; }
  return l;
}
int llmlb_lm_lease_complete(void* lease, int outcome, uint64_t ms, int with_usage, int64_t in, int64_t out, int64_t total) {
  RequestLease* l = static_cast<RequestLease*>(lease);
  TokenUsage u;
  if (in >= 0) { u.has_in = true; u.in = uint32_t(in); }
  if (out >= 0) { u.has_out = true; u.out = uint32_t(out); }
  if (total >= 0) { u.has_total = true; u.total = uint32_t(total); }
  return l->complete_with_tokens(RequestOutcome(outcome), ms, with_usage ? &u : nullptr) ? 0 : -1;
}
void llmlb_lm_lease_drop(void* lease) { delete static_cast<RequestLease*>(lease); }
// out[8]: active, total_assigned, success, errors, latency_ms_sum, input_tokens, output_tokens, total_tokens
int llmlb_lm_stats(void* p, const char* eid, uint64_t* out8) {
  Endpoint e;
  if (!static_cast<LoadManager*>(p)->endpoint_stats(eid, &e)) return -1;
  const uint64_t v[8] = {e.active_requests, e.total_requests, e.success, e.errors, e.latency_ms_sum, e.input_tokens, e.output_tokens, e.total_tokens};
  for (int i = 0; i < 8; ++i) out8[i] = v[i];
  return 0;
}
double llmlb_lm_average_latency(void* p, const char* eid) { return static_cast<LoadManager*>(p)->average_latency_ms(eid); }
// extract_or_estimate_tokens with a whitespace-word counter standing in for the tokenizer (tests);
// returns has-bits (1 in, 2 out, 4 total), values in out3
static int64_t count_words(const std::string& t, void*) { int64_t n = 0; bool in = false; for (char c : t) { const bool w = c != ' ' && c != '\n' && c != '\t'; if (w && !in) ++n; in = w; } return n; }
int llmlb_extract_or_estimate(const char* body_json, const char* req_text, const char* resp_text, int with_counter, uint32_t* out3) {
  Json body;
  if (!Json::parse(body_json ? body_json : "null", &body)) body = Json();
  std::string rq = req_text ? req_text : "", rs = resp_text ? resp_text : "";
  TokenUsage u = extract_or_estimate_tokens(body, req_text ? &rq : nullptr, resp_text ? &rs : nullptr, with_counter ? count_words : nullptr, nullptr);
  out3[0] = u.in; out3[1] = u.out; out3[2] = u.total;
  return (u.has_in ? 1 : 0) | (u.has_out ? 2 : 0) | (u.has_total ? 4 : 0);
}

static void usage_out(const TokenUsage& u, int64_t out[3]) {
  out[0] = u.has_in ? int64_t(u.in) : -1; out[1] = u.has_out ? int64_t(u.out) : -1; out[2] = u.has_total ? int64_t(u.total) : -1;
}
int llmlb_extract_usage(const char* json, int64_t out[3]) {
  Json j; TokenUsage u;
  if (!Json::parse(json, &j) || !extract_usage_from_response(j, &u)) return 0;
  usage_out(u, out);
  return 1;
}
void* llmlb_acc_create(const char* model) { return new StreamingTokenAccumulator(model); }
void llmlb_acc_destroy(void* a) { delete static_cast<StreamingTokenAccumulator*>(a); }
void llmlb_acc_set_input_tokens(void* a, uint32_t n) { static_cast<StreamingTokenAccumulator*>(a)->set_input_tokens(n); }
void llmlb_acc_process_chunk(void* a, const char* chunk) { static_cast<StreamingTokenAccumulator*>(a)->process_chunk(chunk); }
void llmlb_acc_feed(void* a, const char* data, size_t n) { static_cast<StreamingTokenAccumulator*>(a)->feed(data, n); }
size_t llmlb_acc_content(void* a, char* out, size_t cap) { return copy_out(static_cast<StreamingTokenAccumulator*>(a)->accumulated_content(), out, cap); }
int llmlb_acc_done(void* a) { return static_cast<StreamingTokenAccumulator*>(a)->is_done() ? 1 : 0; }
void llmlb_acc_finalize(void* a, int64_t out[3]) { usage_out(static_cast<StreamingTokenAccumulator*>(a)->finalize(), out); }

int llmlb_parse_model_name(const char* model, char* base, char* quant, size_t cap) {
  ParsedModelName p;
  if (!parse_quantized_model_name(model, &p)) return -1;
  copy_out(p.base, base, cap); copy_out(p.quantization, quant, cap);
  return p.has_quant ? 1 : 0;
}
size_t llmlb_error_body(const char* message, const char* type, int status, char* out, size_t cap) { return copy_out(openai_error_body(message, type, status), out, cap); }
size_t llmlb_gate_rejection_body(char* out, size_t cap) { return copy_out(InferenceGate::rejection_body(), out, cap); }
// error conventions: JSON {"status","type","message","retry_after"(-1 = none),"body"} of the classified failure
static std::string client_error_json(const ClientError& e) {
  Json j = Json::object();
  j.set("status", e.status); j.set("type", e.type); j.set("message", e.message); j.set("retry_after", int64_t(e.retry_after)); j.set("body", e.body());
  return j.dump();
}
size_t llmlb_classify_upstream_error(int kind, uint32_t timeout_secs, const char* ollama_loading_model, char* out, size_t cap) {
  std::string m = ollama_loading_model ? ollama_loading_model : "";
  return copy_out(client_error_json(classify_upstream_request_error(UpstreamFailure(kind < 0 || kind > 2 ? 2 : kind), timeout_secs, ollama_loading_model ? &m : nullptr)), out, cap);
}
size_t llmlb_queue_error(int which, uint64_t queue_timeout_secs, char* out, size_t cap) {   // 0 capacity exceeded, 1 wait timeout
  return copy_out(client_error_json(which == 0 ? queue_capacity_exceeded(queue_timeout_secs) : queue_wait_timeout()), out, cap);
}
int llmlb_lb_error_count(void) { return int(LbErrorKind::kCount); }
// JSON {"name","status","type","external","openai_body","app_body"} of LbError variant `kind` carrying `detail`
size_t llmlb_lb_error(int kind, const char* detail, char* out, size_t cap) {
  if (kind < 0 || kind >= int(LbErrorKind::kCount)) return 0;
  const LbErrorKind k = LbErrorKind(kind);
  Json j = Json::object();
  j.set("name", std::string(lb_error_name(k))); j.set("status", lb_error_status(k)); j.set("type", std::string(lb_error_type(k)));
  j.set("external", std::string(lb_error_external_message(k))); j.set("openai_body", lb_error_openai_body(k)); j.set("app_body", app_error_body(k, detail ? detail : ""));
  return copy_out(j.dump(), out, cap);
}
int llmlb_extract_api_key(const char* x_api_key, const char* authorization, char* out, size_t cap) {
  std::string key, err;
  int rc = extract_api_key(x_api_key, authorization, &key, &err);
  copy_out(rc == 0 ? key : err, out, cap);
  return rc;
}
void llmlb_sha256_hex(const char* data, size_t n, char out[65]) { std::string h = sha256_hex(std::string(data, n)); memcpy(out, h.c_str(), 65); }
void* llmlb_gate_create() { return new InferenceGate(); }
void llmlb_gate_destroy(void* g) { delete static_cast<InferenceGate*>(g); }
int llmlb_gate_try_begin(void* g) { return static_cast<InferenceGate*>(g)->try_begin() ? 0 : 503; }
void llmlb_gate_end(void* g) { static_cast<InferenceGate*>(g)->end(); }
void llmlb_gate_set_rejecting(void* g, int v) { static_cast<InferenceGate*>(g)->set_rejecting(v != 0); }
uint32_t llmlb_gate_in_flight(void* g) { return static_cast<InferenceGate*>(g)->in_flight(); }

// framing: kind 0 chat SSE stream, 1 chat body, 2 responses SSE stream, 3 responses body, 4 completion body
size_t llmlb_frame(int kind, const char* id, const char* model, int64_t created, const char* const* pieces,
                   uint32_t n_pieces, uint32_t prompt_tokens, const char* finish_reason, char* out, size_t cap) {
  std::string text, s;
  for (uint32_t i = 0; i < n_pieces; ++i) text += pieces[i];
  const std::string role = "assistant";
  switch (kind) {
    case 0:
      s += sse_event(chat_chunk(id, model, created, &role, nullptr, nullptr));
      for (uint32_t i = 0; i < n_pieces; ++i) { std::string p = pieces[i]; s += sse_event(chat_chunk(id, model, created, nullptr, &p, nullptr)); }
      s += sse_event(chat_chunk(id, model, created, nullptr, nullptr, finish_reason));
      s += sse_event(chat_usage_chunk(id, model, created, prompt_tokens, n_pieces));
      s += sse_done();
      break;
    case 1: s = chat_completion_body(id, model, created, text, finish_reason, prompt_tokens, n_pieces).dump(); break;
    case 2:
      s += sse_event(responses_event_created(id, model));
      s += sse_event(responses_event_item_added());
      s += sse_event(responses_event_part_added());
      for (uint32_t i = 0; i < n_pieces; ++i) s += sse_event(responses_event_delta(pieces[i]));
      s += sse_event(responses_event_text_done(text));
      s += sse_event(responses_event_done(id, prompt_tokens, n_pieces));
      s += sse_done();
      break;
    case 3: s = responses_body(id, model, created, text, prompt_tokens, n_pieces, "completed").dump(); break;
    case 4: s = completion_body(id, model, created, text, finish_reason, prompt_tokens, n_pieces).dump(); break;
    default: return 0;
  }
  return copy_out(s, out, cap);
}
// one step of a stream, for hosts that frame while token events arrive (llmlb_frame above is the same thing all at once)
size_t llmlb_sse_event(int api, int what, const char* id, const char* model, int64_t created, const char* text,
                       uint32_t prompt_tokens, uint32_t completion_tokens, char* out, size_t cap) {
  if (!id || !model || api < 0 || api > 2 || what < 0 || what > 4) return 0;
  if (what == 4) return copy_out(sse_done(), out, cap);
  const std::string t = text ? text : "", role = "assistant";
  std::string s;
  if (api == 0) {
    switch (what) {
      case 0: s = sse_event(chat_chunk(id, model, created, &role, nullptr, nullptr)); break;
      case 1: s = sse_event(chat_chunk(id, model, created, nullptr, &t, nullptr)); break;
      case 2: s = sse_event(chat_chunk(id, model, created, nullptr, nullptr, t.c_str())); break;
      case 3: s = sse_event(chat_usage_chunk(id, model, created, prompt_tokens, completion_tokens)); break;
    }
  } else if (api == 1) {
    switch (what) {
      case 0: break;                                           // a text_completion stream has no role chunk
      case 1: s = sse_event(completion_chunk(id, model, created, &t, nullptr)); break;
      case 2: s = sse_event(completion_chunk(id, model, created, nullptr, t.c_str())); break;
      case 3: s = sse_event(completion_usage_chunk(id, model, created, prompt_tokens, completion_tokens)); break;
    }
  } else {
    switch (what) {
      case 0: s = sse_event(responses_event_created(id, model)) + sse_event(responses_event_item_added()) + sse_event(responses_event_part_added()); break;
      case 1: s = sse_event(responses_event_delta(t)); break;
      case 2: s = sse_event(responses_event_text_done(t)); break;
      case 3: s = sse_event(responses_event_done(id, prompt_tokens, completion_tokens)); break;
    }
  }
  return copy_out(s, out, cap);
}
size_t llmlb_json_roundtrip(const char* text, char* out, size_t cap) {
  Json j;
  if (!Json::parse(text, &j)) return 0;
  return copy_out(j.dump(), out, cap);
}
// spec: {"payload":{...},"selected":"..","endpoint_type":"..","endpoint_models":[[id,canonical|null],..],
//        "mappings":[{"canonical","aliases":[..],"engines":{alias:engine}}]} -> rewritten payload JSON
size_t llmlb_rewrite_payload(const char* spec_json, char* out, size_t cap) {
  Json spec;
  if (!Json::parse(spec_json, &spec)) return 0;
  std::vector<EndpointModel> ems;
  if (const Json* a = spec.get("endpoint_models"))
    for (const Json& e : a->items()) {
      EndpointModel em;
      if (e.items().size() >= 1 && e.items()[0].is_string()) em.model_id = e.items()[0].str();
      if (e.items().size() >= 2 && e.items()[1].is_string()) em.canonical_name = e.items()[1].str();
      ems.push_back(em);
    }
  std::vector<EngineMapping> maps;
  if (const Json* a = spec.get("mappings"))
    for (const Json& m : a->items()) {
      EngineMapping em;
      if (const Json* c = m.get("canonical")) em.canonical = c->str();
      const Json* eng = m.get("engines");
      if (const Json* al = m.get("aliases"))
        for (const Json& x : al->items()) {
          EngineAlias ea;
          ea.name = x.str();
          if (eng) if (const Json* e = eng->get(ea.name)) ea.engine = e->str();
          em.aliases.push_back(ea);
        }
      maps.push_back(em);
    }
  const Json* payload = spec.get("payload");
  const Json* sel = spec.get("selected");
  const Json* et = spec.get("endpoint_type");
  if (!payload || !sel || !et) return 0;
  return copy_out(rewrite_payload_model_for_endpoint(*payload, sel->str(), et->str(), ems, maps).dump(), out, cap);
}
size_t llmlb_prepare_upstream_payload(const char* payload_json, const char* upstream_model, int stream, char* out, size_t cap) {
  Json p;
  if (!Json::parse(payload_json, &p)) return 0;
  return copy_out(prepare_upstream_payload(p, upstream_model, stream != 0).dump(), out, cap);
}
void* llmlb_history_create() { return new RequestHistory(); }
void llmlb_history_destroy(void* h) { delete static_cast<RequestHistory*>(h); }
int64_t llmlb_history_align(int64_t ts) { return RequestHistory::align_to_minute(ts); }
void llmlb_history_record(void* h, int outcome, int64_t ts) { static_cast<RequestHistory*>(h)->record(RequestOutcome(outcome), ts); }
// out: triples (minute, success, error); window = 1: the zero-filled 60-minute view ending at `now`
uint32_t llmlb_history_get(void* h, int window, int64_t now, int64_t* out, uint32_t cap_points) {
  const auto pts = window ? static_cast<RequestHistory*>(h)->window(now) : static_cast<RequestHistory*>(h)->points();
  for (uint32_t i = 0; i < pts.size() && i < cap_points; ++i) { out[3 * i] = pts[i].minute; out[3 * i + 1] = int64_t(pts[i].success); out[3 * i + 2] = int64_t(pts[i].error); }
  return uint32_t(pts.size());
}
// ops: 'u' value = update(value), 'r' = reset; returns for_sort() (inf when never measured) and *has
double llmlb_latency_play(const char* ops, const double* values, uint32_t n, int* has) {
  InferenceLatency l;
  for (uint32_t i = 0; i < n; ++i) { if (ops[i] == 'u') l.update(values[i]); else l.reset(); }
  if (has) *has = l.has ? 1 : 0;
  return l.for_sort();
}
// stops_json: ["...", ...]
void* llmlb_stop_create(const char* stops_json) {
  Json j;
  std::vector<std::string> stops;
  if (Json::parse(stops_json, &j) && j.is_array())
    for (const Json& x : j.items()) if (x.is_string()) stops.push_back(x.str());
  return new StopMatcher(stops);
}
void llmlb_stop_destroy(void* m) { delete static_cast<StopMatcher*>(m); }
size_t llmlb_stop_feed(void* m, const char* piece, size_t n, char* out, size_t cap) { return copy_out(static_cast<StopMatcher*>(m)->feed(std::string(piece, n)), out, cap); }
size_t llmlb_stop_flush(void* m, char* out, size_t cap) { return copy_out(static_cast<StopMatcher*>(m)->flush(), out, cap); }
int llmlb_stop_hit(void* m, char* matched, size_t cap) {
  auto* sm = static_cast<StopMatcher*>(m);
  if (sm->hit() && matched) copy_out(sm->matched(), matched, cap);
  return sm->hit() ? 1 : 0;
}
}  // extern "C"
