// Gateway-side hot path above the C ABI (SURVEY.md §8 a1 rows), in C++ because the reference is
// compiled (Rust) code and no cargo exists in this image.  Names and semantics mirror the
// reference so the tests read like its own:
//   ModelTpsState::update_tps            llmlb/src/balancer/types.rs:102-118
//   LoadManager::{update_tps, select_endpoint_by_tps_ready_for_model, begin_request, finish_request}
//                                        llmlb/src/balancer/mod.rs:1770,1873-1985,2273-2425,2949
//   EndpointRegistry::find_by_model      llmlb/src/registry/endpoints.rs:16-73,209-231
//   StreamingTokenAccumulator, extract_usage_from_response   llmlb/src/token/mod.rs:41-206
//   process_sse_lines                    llmlb/src/api/proxy.rs:104-116
//   parse_quantized_model_name           llmlb/src/api/model_name.rs:19-40
//   openai_error_response_with_type      llmlb/src/api/openai_util.rs:242-257
//   InferenceGate                        llmlb/src/inference_gate.rs:17-230
//   RequestHistory (60-minute window)    llmlb/src/balancer/mod.rs:2643-2658,2973-3060
//   extract_api_key                      llmlb/src/auth/middleware.rs:292-321
//   rewrite_payload_model_for_endpoint, resolve_runtime_model_name_for_endpoint  llmlb/src/api/model_name.rs:43-108
//   resolve_engine_name                  llmlb/src/models/mapping.rs:302-323
//   stream_options.include_usage injection  llmlb/src/api/openai.rs:977-992
#pragma once
#include <atomic>
#include <chrono>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "json.hpp"

namespace llmlb_host {

enum class TpsApiKind { ChatCompletions = 0, Completions = 1, Responses = 2 };

struct ModelTpsState {
  bool has_ema = false;
  double tps_ema = 0.0;
  uint64_t request_count = 0, total_output_tokens = 0, total_duration_ms = 0;
  void update_tps(uint64_t output_tokens, uint64_t duration_ms);
};

struct ModelMapping { std::string canonical; std::vector<std::string> aliases; };
struct EndpointModel { std::string model_id; std::string canonical_name; };  // "" = none
struct Endpoint {
  std::string id;
  bool online = true;
  bool initializing = false;
  std::vector<EndpointModel> models;
  // LoadManager state (balancer/types.rs:157-173)
  uint32_t active_requests = 0;
  uint64_t total_requests = 0, success = 0, errors = 0, latency_ms_sum = 0, output_tokens = 0;
  uint64_t input_tokens = 0, total_tokens = 0;   // finish_request_with_tokens (balancer/mod.rs:2346-2425)
};

enum SelectError { kSelectOk = 0, kNoCapableEndpoints = 1, kNoEndpointsAvailable = 2 };
enum class RequestOutcome { Success = 0, Error = 1, Queued = 2 };
struct TokenUsage { bool has_in = false, has_out = false, has_total = false; uint32_t in = 0, out = 0, total = 0; };
class LoadManager;

// RAII request lease (llmlb/src/balancer/lease.rs:16-100): a request that is neither completed
// explicitly nor survives to its normal end (early return, exception, client gone) still gives
// its active slot back — the destructor finishes it as Error with the elapsed time.
class RequestLease {
 public:
  RequestLease() = default;
  RequestLease(LoadManager* lm, std::string endpoint_id);
  RequestLease(RequestLease&& o) noexcept;
  RequestLease& operator=(RequestLease&& o) noexcept;
  RequestLease(const RequestLease&) = delete;
  RequestLease& operator=(const RequestLease&) = delete;
  ~RequestLease();
  const std::string& endpoint_id() const { return endpoint_id_; }
  uint64_t elapsed_ms() const;
  bool armed() const { return lm_ != nullptr; }
  // both return true when there is nothing to do (already completed / never armed), like the
  // reference's Ok(()) for a lease without a load manager (lease.rs:47-49)
  bool complete(RequestOutcome outcome, uint64_t duration_ms);
  bool complete_with_tokens(RequestOutcome outcome, uint64_t duration_ms, const TokenUsage* usage);
 private:
  LoadManager* lm_ = nullptr;
  std::string endpoint_id_;
  std::chrono::steady_clock::time_point started_{};
};

class LoadManager {
 public:
  void add_mapping(const std::string& canonical, const std::string& alias);
  std::vector<std::string> model_lookup_keys(const std::string& model_id) const;
  void add_endpoint(const std::string& id, bool online, bool initializing);
  bool add_model(const std::string& endpoint_id, const std::string& model_id, const std::string& canonical);
  bool set_status(const std::string& endpoint_id, bool online);       // offline clears its TPS
  bool set_initializing(const std::string& endpoint_id, bool v);
  std::vector<std::string> find_by_model(const std::string& model_id) const;
  void update_tps(const std::string& endpoint_id, const std::string& model_id, TpsApiKind kind,
                  uint64_t output_tokens, uint64_t duration_ms);
  bool get_tps(const std::string& endpoint_id, const std::string& model_id, TpsApiKind kind,
               ModelTpsState* out) const;
  // model == nullptr: aggregate routing (select_endpoint_by_tps_direct); kind < 0: none
  SelectError select(const std::string* model, int kind, std::string* out_id);
  bool begin_request(const std::string& endpoint_id);
  bool finish_request(const std::string& endpoint_id, bool success, uint64_t duration_ms,
                      uint64_t output_tokens);
  // balancer/mod.rs:2273-2425.  Queued leaves every counter alone; usage == nullptr = finish_request
  bool begin_request_lease(const std::string& endpoint_id, RequestLease* out);
  bool finish_request_outcome(const std::string& endpoint_id, RequestOutcome outcome, uint64_t duration_ms,
                              const TokenUsage* usage);
  bool endpoint_stats(const std::string& endpoint_id, Endpoint* out) const;   // copy of the counters
  // mean latency over completed requests, < 0 when none completed (balancer/types.rs:188-195)
  double average_latency_ms(const std::string& endpoint_id) const;
  uint32_t active_requests(const std::string& endpoint_id) const;

 private:
  double score(const Endpoint& ep, const std::string* model, int kind) const;
  const ModelMapping* find_mapping(const std::string& model_id) const;
  Endpoint* find(const std::string& id);
  const Endpoint* find(const std::string& id) const;
  mutable std::mutex mu_;
  std::vector<Endpoint> endpoints_;  // registration order
  std::vector<ModelMapping> mappings_;
  std::map<std::tuple<std::string, std::string, int>, ModelTpsState> tps_;
  std::atomic<uint64_t> round_robin_{0};
};

// Inference latency EMA, alpha 0.2 (types/endpoint.rs:419-440): first sample or first after a reset
// replaces the value; reset (endpoint offline) = +inf so the endpoint sorts last.
struct InferenceLatency {
  bool has = false;
  double ms = 0.0;
  void update(double new_ms) {
    const bool finite = has && ms == ms && ms != __builtin_inf() && ms != -__builtin_inf();
    ms = finite ? 0.2 * new_ms + (1.0 - 0.2) * ms : new_ms;
    has = true;
  }
  void reset() { has = true; ms = __builtin_inf(); }
  double for_sort() const { return has ? ms : __builtin_inf(); }
};

// 60-minute request history (balancer/mod.rs:2643-2658, 2973-3060): per-minute success / error
// counts, newest minute incremented in place, points older than the window dropped on insert;
// window(now) = exactly 60 points, oldest first, zero-filled.  Timestamps are unix seconds.
struct RequestHistoryPoint { int64_t minute = 0; uint64_t success = 0, error = 0; };
class RequestHistory {
 public:
  static constexpr int64_t kWindowMinutes = 60;
  static int64_t align_to_minute(int64_t ts) { return ts - ((ts % 60) + 60) % 60; }
  void record(RequestOutcome outcome, int64_t ts);
  std::vector<RequestHistoryPoint> window(int64_t now) const;
  std::vector<RequestHistoryPoint> points() const { std::lock_guard<std::mutex> lk(mu_); return points_; }
 private:
  mutable std::mutex mu_;
  std::vector<RequestHistoryPoint> points_;
};

bool extract_usage_from_response(const Json& body, TokenUsage* usage);
// token/mod.rs:235-259: usage when the body carries one, else an estimate of the request / response
// texts.  The reference estimates with tiktoken's cl100k_base ranks (token/mod.rs:217-223), a
// third-party table; an in-process endpoint has the MODEL's tokenizer instead, so `count` is
// that tokenizer's encode-with-specials length (nullptr or a negative return = cannot estimate).
typedef int64_t (*TokenCountFn)(const std::string& text, void* ctx);
TokenUsage extract_or_estimate_tokens(const Json& body, const std::string* request_text, const std::string* response_text,
                                      TokenCountFn count, void* ctx);

class StreamingTokenAccumulator {
 public:
  explicit StreamingTokenAccumulator(const std::string& model) : model_(model) {}
  void set_input_tokens(uint32_t n) { has_input_ = true; input_ = n; }
  void process_chunk(const std::string& chunk);
  // process_sse_lines with carry-over between network chunks
  void feed(const char* data, size_t n);
  const std::string& accumulated_content() const { return content_; }
  bool is_done() const { return done_; }
  // estimate: tokens for the accumulated text when the stream carried no usage (the reference
  // uses tiktoken there; hosts of this engine always get usage so the hook is rarely used)
  TokenUsage finalize(uint32_t (*estimate)(const std::string&) = nullptr) const;

 private:
  std::string model_, content_, line_buf_;
  bool has_input_ = false, has_usage_ = false, done_ = false;
  uint32_t input_ = 0;
  TokenUsage usage_;
};

struct ParsedModelName { std::string raw, base, quantization; bool has_quant = false; };
bool parse_quantized_model_name(const std::string& model, ParsedModelName* out);

std::string openai_error_body(const std::string& message, const std::string& type, int status);
std::string model_unavailable_body(const std::string& message, const std::string& code);

// ---- error conventions (SURVEY row a1.16) ----
// What a client sees for a failed request: status, OpenAI error type, message, optional Retry-After seconds (-1 = no header).
struct ClientError { int status = 502; std::string type, message; long long retry_after = -1; std::string body() const { return openai_error_body(message, type, status); } };
// reqwest failure classes of the upstream call (is_timeout / is_connect / anything else): api/openai_util.rs:86-134.  For the in-process
// engine: Timeout = the request deadline (types/endpoint.rs:389), Other = the engine failed the request.
enum class UpstreamFailure { Timeout = 0, Connect = 1, Other = 2 };
ClientError classify_upstream_request_error(UpstreamFailure kind, uint32_t timeout_secs, const std::string* ollama_loading_model = nullptr);
ClientError queue_capacity_exceeded(uint64_t queue_timeout_secs);   // api/openai.rs:841-861: 429 rate_limit_exceeded, Retry-After max(1, secs)
ClientError queue_wait_timeout();                                   // api/openai.rs:863-882: 504 timeout
// LbError (common/error.rs:41-214): one row per variant; order = the reference's declaration order, Common split in two
enum class LbErrorKind { CommonValidation = 0, CommonOther, EndpointNotFound, NotFound, NoEndpointsAvailable, NoCapableEndpoints, Database, Http, Timeout,
                         ServiceUnavailable, Internal, EndpointOffline, InvalidModelName, InsufficientStorage, PasswordHash, Jwt, Authentication,
                         Authorization, Conflict, kCount };
int lb_error_status(LbErrorKind k);
const char* lb_error_type(LbErrorKind k);
const char* lb_error_external_message(LbErrorKind k);
const char* lb_error_name(LbErrorKind k);                             // snake_case name used by the tests / oracle
std::string lb_error_openai_body(LbErrorKind k);                      // to_openai_error: {"error":{"message","type","code":"<status>"}}
std::string app_error_body(LbErrorKind k, const std::string& detail); // api/error.rs:154-203: {"error": detail or the generic message}

// 0 ok; 1 invalid Authorization format; 2 missing  (messages as auth/middleware.rs:292-321)
int extract_api_key(const char* x_api_key, const char* authorization, std::string* key, std::string* err);
std::string sha256_hex(const std::string& data);

class InferenceGate {  // inference_gate.rs: reject-when-draining + in-flight count
 public:
  bool try_begin() { if (rejecting_.load()) return false; in_flight_.fetch_add(1); return true; }
  void end() { in_flight_.fetch_sub(1); }
  void set_rejecting(bool v) { rejecting_.store(v); }
  uint32_t in_flight() const { return in_flight_.load(); }
  static std::string rejection_body() { return openai_error_body("Server is updating. Please retry.", "service_unavailable", 503); }
 private:
  std::atomic<bool> rejecting_{false};
  std::atomic<uint32_t> in_flight_{0};
};

// ---- outbound payload preparation (model_name.rs:43-108, openai.rs:977-992, mapping.rs:302-323) ----
struct EngineAlias { std::string name, engine; };             // engine: "ollama", "lm_studio", "xllm", "vllm", ...
struct EngineMapping { std::string canonical; std::vector<EngineAlias> aliases; };
// first alias of the mapping that knows `model` (canonical or alias, case-insensitively) for that engine; "" if none
std::string resolve_engine_name(const std::string& model, const std::string& endpoint_type, const std::vector<EngineMapping>& mappings);
std::string resolve_runtime_model_name_for_endpoint(const std::string& requested, const std::string& selected,
                                                    const std::string& endpoint_type, const std::vector<EndpointModel>& endpoint_models,
                                                    const std::vector<EngineMapping>& mappings);
Json rewrite_payload_model_for_endpoint(const Json& payload, const std::string& selected, const std::string& endpoint_type,
                                        const std::vector<EndpointModel>& endpoint_models, const std::vector<EngineMapping>& mappings);
// model := upstream name; streaming requests get stream_options.include_usage = true unless the client set it
Json prepare_upstream_payload(const Json& payload, const std::string& upstream_model, bool stream);

// ---- `stop` strings (OpenAI `stop`, Anthropic `stop_sequences`) on the detokenised stream ----------
// feed() takes the next piece of generated text and returns what may be shown to the client now:
// text that could still turn out to be the beginning of a stop string is held back; once a stop
// string is complete the output ends right before it (the stop string itself is never emitted),
// hit() becomes true and everything after is dropped.  flush() releases held-back text when
// generation ends without a match.
class StopMatcher {
 public:
  explicit StopMatcher(std::vector<std::string> stops);
  std::string feed(const std::string& piece);
  std::string flush();
  bool hit() const { return hit_; }
  const std::string& matched() const { return matched_; }
  bool empty() const { return stops_.empty(); }
 private:
  std::vector<std::string> stops_;
  std::string held_, matched_;
  bool hit_ = false;
};

// ---- wire format writers (shapes pinned by the reference's fixtures, SURVEY.md §8b) ----
std::string sse_event(const Json& j);                       // "data: {...}\n\n"
inline std::string sse_done() { return "data: [DONE]\n\n"; }
// logprobs (optional): the choice's "logprobs" value (chat_logprobs / completion_logprobs); without it the shapes are the
// ones above, byte for byte.  cached_tokens (optional, a prefix-cache engine): usage gains
// "prompt_tokens_details":{"cached_tokens":N} ("input_tokens_details" on responses); without it usage is unchanged
// index: the choice a chunk carries (OpenAI's n; 0 = the only one)
Json chat_chunk(const std::string& id, const std::string& model, int64_t created,
                const std::string* role, const std::string* content, const char* finish_reason,
                const Json* logprobs = nullptr, uint32_t index = 0);
Json chat_usage_chunk(const std::string& id, const std::string& model, int64_t created,
                      uint32_t prompt_tokens, uint32_t completion_tokens, const uint32_t* cached_tokens = nullptr);
Json chat_completion_body(const std::string& id, const std::string& model, int64_t created,
                          const std::string& content, const char* finish_reason,
                          uint32_t prompt_tokens, uint32_t completion_tokens, const Json* logprobs = nullptr,
                          const uint32_t* cached_tokens = nullptr);
// One choice of a body with several (OpenAI's n): its text, finish reason and logprobs value (optional).  The one-choice
// bodies above are these with a single choice, byte for byte.
struct ChoiceOut {
  std::string text;
  const char* finish_reason = nullptr;
  const Json* logprobs = nullptr;
};
Json chat_completion_body(const std::string& id, const std::string& model, int64_t created, const std::vector<ChoiceOut>& choices,
                          uint32_t prompt_tokens, uint32_t completion_tokens, const uint32_t* cached_tokens = nullptr);
// legacy /v1/completions stream: {"object":"text_completion","choices":[{"index":0,"text":...,"finish_reason":...}]}
Json completion_chunk(const std::string& id, const std::string& model, int64_t created, const std::string* text, const char* finish_reason,
                      const Json* logprobs = nullptr, uint32_t index = 0);
Json completion_usage_chunk(const std::string& id, const std::string& model, int64_t created, uint32_t prompt_tokens, uint32_t completion_tokens,
                            const uint32_t* cached_tokens = nullptr);
Json completion_body(const std::string& id, const std::string& model, int64_t created,
                     const std::string& text, const char* finish_reason, uint32_t prompt_tokens,
                     uint32_t completion_tokens, const Json* logprobs = nullptr, const uint32_t* cached_tokens = nullptr);
Json completion_body(const std::string& id, const std::string& model, int64_t created, const std::vector<ChoiceOut>& choices,
                     uint32_t prompt_tokens, uint32_t completion_tokens, const uint32_t* cached_tokens = nullptr);

// ---- OpenAI logprobs ----
// One listed token (or one of its alternatives): text through from_utf8_lossy, raw bytes, log-probability.
struct LogprobToken {
  std::string token, bytes;
  float logprob = 0.f;
};
struct LogprobEntry {
  LogprobToken tok;
  std::vector<LogprobToken> top;   // most probable first
  uint32_t text_offset = 0;        // code points of completion text released before the token was fed
  bool scored = true;              // false: an echoed prompt's first token, which has no record (logprob and top are null)
};
// chat: {"content":[{"token","logprob","bytes","top_logprobs":[{"token","logprob","bytes"}]}],"refusal":null}
Json chat_logprobs(const std::vector<LogprobEntry>& entries);
// completions: {"tokens":[...],"token_logprobs":[...],"top_logprobs":[{token: logprob}],"text_offset":[...]}
Json completion_logprobs(const std::vector<LogprobEntry>& entries);
Json responses_body(const std::string& id, const std::string& model, int64_t created,
                    const std::string& text, uint32_t input_tokens, uint32_t output_tokens,
                    const char* status, const uint32_t* cached_tokens = nullptr);
Json responses_event_created(const std::string& id, const std::string& model);
Json responses_event_item_added();
Json responses_event_part_added();
Json responses_event_delta(const std::string& delta);
Json responses_event_text_done(const std::string& text);
Json responses_event_done(const std::string& id, uint32_t input_tokens, uint32_t output_tokens, const uint32_t* cached_tokens = nullptr);

// Byte-level placeholder tokenizer (no tokenizer assets exist on the box): ids 0..255 are raw
// bytes shifted by 3 reserved ids; anything else renders as "<|id|>".
std::vector<int32_t> byte_tokenize(const std::string& text, uint32_t vocab);
std::string byte_detokenize(int32_t id);

}  // namespace llmlb_host
