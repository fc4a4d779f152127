// llmlb_b200_server — the endpoint contract llmlb already consumes (SURVEY.md §8b), served
// straight from the in-process engine through the C ABI.  An unmodified llmlb registers it with
// POST /api/endpoints {"name","base_url"} (llmlb/src/api/endpoints.rs:505): detection sees
// /api/system with "xllm_version" (detection/xllm.rs:27-66), health pulls /api/health
// (health/endpoint_checker.rs:515-557), sync reads /v1/models (sync/parser.rs:78-110).
//
// Plain blocking HTTP/1.1 (thread per connection, keep-alive, chunked SSE).  With
// `--tokenizer tokenizer.json` prompts go through the native Llama-3 BPE tokenizer + chat template
// (tokenizer.hpp) and SSE deltas through its UTF-8-safe streaming detokenizer; without it (no
// tokenizer assets exist on the build box) the byte-level placeholder of gateway.hpp is used.
// A request may always carry "prompt_token_ids" instead of text.
#include <arpa/inet.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <signal.h>
#include <strings.h>
#include <sys/socket.h>
#include <sys/time.h>
#include <unistd.h>

#include <algorithm>
#include <cerrno>
#include <chrono>
#include <climits>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include "../../include/llmlb_b200.h"
#include "anthropic.hpp"
#include "checkpoint.hpp"
#include "download.hpp"
#include "gateway.hpp"
#include "tokenizer.hpp"

using namespace llmlb_host;

struct Server {
  llmlb_engine* eng = nullptr;
  std::string model_id, api_key;
  uint32_t vocab = 0, max_ctx = 0;
  LoadManager lm;
  InferenceGate gate;
  std::atomic<uint64_t> seq{0};
  std::unique_ptr<BpeTokenizer> tok;   // null: byte-level placeholder
  std::vector<int32_t> stop_ids;       // <|eot_id|>, <|end_of_text|>, <|eom_id|> when a tokenizer is loaded
  uint32_t queue_timeout_ms = 60000, request_timeout_ms = 120000;
  // a client that stops reading must not pin a server thread, an engine slot and its KV pages for ever: a blocked send gives
  // up after send_timeout_ms (the request is then cancelled like any hang-up); an idle keep-alive connection is closed after
  // idle_timeout_ms without a request (reqwest's pool re-connects transparently)
  uint32_t send_timeout_ms = 30000, idle_timeout_ms = 300000;
  std::atomic<uint32_t> connections{0};
  uint32_t max_connections = 1024;
  std::unique_ptr<DownloadManager> downloads;   // POST /api/models/download, GET /api/download/progress (xllm/download.rs:97,147)
};
static Server G;

struct Request {
  std::string method, path, body;
  std::map<std::string, std::string> headers;  // lower-cased names
};

static bool send_all(int fd, const std::string& s);

// kReqClosed: the peer went away (or sent nothing more); the other failures are answered before the connection is
// dropped, the way hyper/axum in front of the reference's handlers do: 400 for a request line that does not parse,
// 431 for a header block over 1 MiB, 413 over the 20 MiB body limit (DefaultBodyLimit, api/mod.rs:58,536).
enum ReqStatus { kReqOk, kReqClosed, kReqBad = 400, kReqTooLarge = 413, kReqHeadersTooLarge = 431 };

static ReqStatus read_request(int fd, std::string& buf, Request* rq) {
  size_t hdr_end;
  while ((hdr_end = buf.find("\r\n\r\n")) == std::string::npos) {
    if (buf.size() > (1u << 20)) return kReqHeadersTooLarge;
    char tmp[8192];
    ssize_t n = recv(fd, tmp, sizeof tmp, 0);
    if (n <= 0) return kReqClosed;
    buf.append(tmp, size_t(n));
  }
  std::string head = buf.substr(0, hdr_end);
  size_t line_end = head.find("\r\n");
  std::string first = head.substr(0, line_end);
  size_t a = first.find(' '), b = first.rfind(' ');
  if (a == std::string::npos || b == a || a == 0 || first.compare(b + 1, 5, "HTTP/") != 0) return kReqBad;
  rq->method = first.substr(0, a);
  rq->path = first.substr(a + 1, b - a - 1);
  rq->headers.clear();
  size_t pos = line_end == std::string::npos ? head.size() : line_end + 2;
  while (pos < head.size()) {
    size_t e = head.find("\r\n", pos);
    if (e == std::string::npos) e = head.size();
    std::string line = head.substr(pos, e - pos);
    size_t c = line.find(':');
    if (c != std::string::npos) {
      std::string k = line.substr(0, c), v = line.substr(c + 1);
      for (auto& ch : k) if (ch >= 'A' && ch <= 'Z') ch = char(ch - 'A' + 'a');
      while (!v.empty() && (v[0] == ' ' || v[0] == '\t')) v.erase(0, 1);
      while (!v.empty() && (v.back() == ' ' || v.back() == '\t')) v.pop_back();
      rq->headers[k] = v;
    }
    pos = e + 2;
  }
  size_t need = 0;
  auto it = rq->headers.find("content-length");
  if (it != rq->headers.end()) {
    const std::string& v = it->second;
    if (v.empty() || v.size() > 18 || v.find_first_not_of("0123456789") != std::string::npos) return kReqBad;
    need = size_t(strtoull(v.c_str(), nullptr, 10));
  } else if (rq->headers.count("transfer-encoding")) {
    return kReqBad;                           // the gateway's client (reqwest .json(), openai.rs:995-1005) always sends a length
  }
  if (need > (20u << 20)) return kReqTooLarge;
  size_t have = buf.size() - (hdr_end + 4);
  if (have < need) {                          // curl and friends wait up to a second for this before sending a large body
    auto ex = rq->headers.find("expect");
    if (ex != rq->headers.end() && strncasecmp(ex->second.c_str(), "100-continue", 12) == 0 &&
        !send_all(fd, "HTTP/1.1 100 Continue\r\n\r\n")) return kReqClosed;
  }
  while (have < need) {
    char tmp[65536];
    ssize_t n = recv(fd, tmp, sizeof tmp, 0);
    if (n <= 0) return kReqClosed;
    buf.append(tmp, size_t(n));
    have += size_t(n);
  }
  rq->body = buf.substr(hdr_end + 4, need);
  buf.erase(0, hdr_end + 4 + need);
  return kReqOk;
}

// the peer closed its end (orderly shutdown or reset) and nothing is left to read: a non-blocking one-byte peek
static bool peer_closed(int fd) {
  char c;
  const ssize_t n = recv(fd, &c, 1, MSG_PEEK | MSG_DONTWAIT);
  if (n == 0) return true;
  return n < 0 && errno != EAGAIN && errno != EWOULDBLOCK && errno != EINTR;
}

static bool send_all(int fd, const std::string& s) {
  size_t off = 0;
  while (off < s.size()) {
    ssize_t n = send(fd, s.data() + off, s.size() - off, MSG_NOSIGNAL);
    if (n <= 0) return false;
    off += size_t(n);
  }
  return true;
}
static const char* reason(int st) {
  switch (st) { case 200: return "OK"; case 400: return "Bad Request"; case 401: return "Unauthorized";
    case 404: return "Not Found"; case 405: return "Method Not Allowed"; case 413: return "Payload Too Large";
    case 431: return "Request Header Fields Too Large"; case 429: return "Too Many Requests"; case 502: return "Bad Gateway";
    case 503: return "Service Unavailable"; case 504: return "Gateway Timeout"; default: return "Error"; }
}
static bool send_json(int fd, int status, const std::string& body, const char* extra = "") {
  std::string h = "HTTP/1.1 " + std::to_string(status) + " " + reason(status) +
                  "\r\nContent-Type: application/json\r\nContent-Length: " + std::to_string(body.size()) + "\r\n" + extra + "\r\n";
  return send_all(fd, h + body);
}
static bool send_chunk(int fd, const std::string& data) {
  char hdr[32];
  snprintf(hdr, sizeof hdr, "%zx\r\n", data.size());
  return send_all(fd, std::string(hdr) + data + "\r\n");
}
static int map_error(int rc) {  // LbError -> status (api/error.rs:31-110)
  switch (rc) { case LLMLB_E_INVALID_ARG: return 400; case LLMLB_E_MODEL_NOT_FOUND: return 404;
    case LLMLB_E_QUEUE_FULL: return 503; case LLMLB_E_TIMEOUT: return 504; default: return 502; }
}

static std::string percent_decode(const std::string& s) {
  auto hex = [](char c) { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1; };
  std::string out;
  for (size_t i = 0; i < s.size(); ++i) {
    if (s[i] == '%' && i + 2 < s.size() && hex(s[i + 1]) >= 0 && hex(s[i + 2]) >= 0) { out.push_back(char(hex(s[i + 1]) * 16 + hex(s[i + 2]))); i += 2; }
    else out.push_back(s[i]);
  }
  return out;
}

static std::string content_text(const Json& c) {  // string or [{type:text,text}] parts
  if (c.is_string()) return c.str();
  std::string s;
  if (c.is_array())
    for (auto& p : c.items()) { const Json* t = p.get("text"); if (t && t->is_string()) s += t->str(); }
  return s;
}

// Anthropic error types by status (anthropic.rs:1594-1611 anthropic_error_from_lb_error)
static std::string anthropic_error_body(int status, const std::string& message) {
  AnthropicError e;
  e.status = status;
  e.type = status == 400 ? "invalid_request_error" : status == 401 ? "authentication_error" : status == 403 ? "permission_error"
         : status == 404 ? "not_found_error" : "api_error";
  e.message = message;
  return e.body();
}

// kind: 0 chat, 1 responses, 2 completions.  anthropic: the request came in through /v1/messages
// (already translated to the chat form in `pre`); errors, the body and the SSE events leave in
// Anthropic shape — the chat chunks produced below are run through AnthropicStreamTransformer,
// the same transformation the reference applies to an upstream's OpenAI stream.
static void handle_generate(int fd, const Request& rq, int kind, const Json* pre = nullptr, bool anthropic = false) {
  auto send_err = [&](int status, const std::string& message, const char* type, const char* extra = "") {
    send_json(fd, status, anthropic ? anthropic_error_body(status, message) : openai_error_body(message, type, status), extra);
  };
  if (!G.gate.try_begin()) {
    if (anthropic) send_err(503, "Server is updating. Please retry.", "service_unavailable", "Retry-After: 30\r\n");
    else send_json(fd, 503, InferenceGate::rejection_body(), "Retry-After: 30\r\n");
    return;
  }
  struct GateGuard { ~GateGuard() { G.gate.end(); } } guard;
  Json req;
  if (pre) req = *pre;
  else if (!Json::parse(rq.body, &req) || !req.is_object()) { send_err(400, "invalid JSON body", "invalid_request_error"); return; }
  const Json* jm = req.get("model");
  if (!jm || !jm->is_string() || jm->str().empty()) { send_err(400, "model is required", "invalid_request_error"); return; }
  ParsedModelName pm;
  if (!parse_quantized_model_name(jm->str(), &pm)) { send_err(400, "Invalid model name (quantization format): " + jm->str(), "invalid_request_error"); return; }
  std::string ep;
  const TpsApiKind api = kind == 0 ? TpsApiKind::ChatCompletions : kind == 1 ? TpsApiKind::Responses : TpsApiKind::Completions;
  if (G.lm.select(&pm.base, int(api), &ep) != kSelectOk) {
    send_err(404, "The model '" + jm->str() + "' does not exist", "invalid_request_error");
    return;
  }
  if (const Json* n = req.get("n"))                         // one choice per request: more would be answered with one, silently
    if (n->is_number() && n->as_int() != 1) { send_err(400, "n must be 1: this endpoint returns one choice per request", "invalid_request_error"); return; }
  // prompt
  std::vector<int32_t> ids;
  if (const Json* raw = req.get("prompt_token_ids")) {
    if (raw->is_array()) for (auto& v : raw->items()) ids.push_back(int32_t(v.as_int()));
  } else if (kind == 0) {
    const Json* msgs = req.get("messages");
    if (!msgs || !msgs->is_array() || msgs->items().empty()) { send_err(400, "messages is required", "invalid_request_error"); return; }
    for (auto& m : msgs->items()) if (!m.is_object()) { send_err(400, "messages must be an array of objects", "invalid_request_error"); return; }
    std::string text;
    std::vector<ChatMessage> chat;
    for (auto& m : msgs->items()) {
      const Json* role = m.get("role"); const Json* c = m.get("content");
      // image parts are rejected by the gateway before the boundary (openai.rs:617); mirror it
      if (c && c->is_array()) for (auto& p : c->items()) { const Json* t = p.get("type"); if (t && t->is_string() && t->str() == "image_url") { send_err(400, "image inputs are not supported", "invalid_request_error"); return; } }
      chat.push_back(ChatMessage{role && role->is_string() ? role->str() : "user", c ? content_text(*c) : ""});
      text += chat.back().role + ": " + chat.back().content + "\n";
    }
    text += "assistant: ";
    ids = G.tok ? G.tok->encode_chat(chat) : byte_tokenize(text, G.vocab);
  } else if (kind == 1) {
    const Json* in = req.get("input");
    std::string text;
    std::vector<ChatMessage> chat;
    if (!in || !(in->is_string() || (in->is_array() && !in->items().empty()))) { send_err(400, "input is required (a string or an array of input items)", "invalid_request_error"); return; }
    if (in->is_string()) { text = in->str(); chat.push_back(ChatMessage{"user", text}); }
    else for (auto& m : in->items()) {
      const Json* role = m.get("role"); const Json* c = m.get("content");
      if (c) { text += content_text(*c) + "\n"; chat.push_back(ChatMessage{role && role->is_string() ? role->str() : "user", content_text(*c)}); }
    }
    ids = G.tok ? G.tok->encode_chat(chat) : byte_tokenize(text, G.vocab);
  } else {
    // OpenAI's four prompt forms: "text" | ["text"] | [id, ...] | [[id, ...]].  Several prompts in one request (one choice
    // per prompt) are not served by this shim: refused, not answered for the first one only; anything else is a 400 instead of
    // the completion of an empty prompt that a silent "" would produce.
    const Json* p = req.get("prompt");
    auto all_ints = [](const Json& a) { for (auto& v : a.items()) if (!v.is_number() || v.as_double() != double(v.as_int())) return false; return !a.items().empty(); };
    const Json* one = p;
    if (p && p->is_array() && p->items().size() == 1 && (p->items()[0].is_string() || p->items()[0].is_array())) one = &p->items()[0];
    if (one && one->is_string()) {
      ids = G.tok ? G.tok->encode(one->str(), /*add_bos=*/true, /*parse_special=*/false) : byte_tokenize(one->str(), G.vocab);
    } else if (one && one->is_array() && all_ints(*one)) {
      for (auto& v : one->items()) ids.push_back(int32_t(std::max<int64_t>(-1, std::min<int64_t>(v.as_int(), INT32_MAX))));
    } else if (p && p->is_array() && p->items().size() > 1 && (p->items()[0].is_string() || p->items()[0].is_array())) {
      send_err(400, "several prompts in one request are not supported: send one request per prompt", "invalid_request_error");
      return;
    } else {
      send_err(400, "prompt must be a string, an array with one string, or an array of token ids", "invalid_request_error");
      return;
    }
  }
  for (int32_t t : ids)
    if (t < 0 || uint32_t(t) >= G.vocab) { send_err(400, "prompt token id outside the model vocabulary", "invalid_request_error"); return; }
  llmlb_sampling s{};
  const Json* mt = req.get(kind == 1 ? "max_output_tokens" : "max_tokens");
  if (!mt && kind == 0) mt = req.get("max_completion_tokens");
  if (mt && !mt->is_null() && (!mt->is_number() || mt->as_int() < 1 || mt->as_double() != double(mt->as_int()))) {
    send_err(400, std::string(kind == 1 ? "max_output_tokens" : "max_tokens") + " must be a positive integer", "invalid_request_error");
    return;
  }
  s.max_tokens = mt && mt->is_number() ? uint32_t(std::min<int64_t>(mt->as_int(), INT32_MAX)) : 128;
  const Json* t = req.get("temperature");
  s.temperature = t && t->is_number() ? float(t->as_double()) : 1.0f;
  const Json* tp = req.get("top_p");
  s.top_p = tp && tp->is_number() ? float(tp->as_double()) : 1.0f;
  const Json* tk = req.get("top_k");
  s.top_k = tk && tk->is_number() ? uint32_t(tk->as_int()) : 0;
  const Json* sd = req.get("seed");
  s.seed = sd && sd->is_number() ? uint64_t(sd->as_int()) : G.seq.load();
  const Json* ie = req.get("ignore_eos");
  s.ignore_eos = ie && ie->as_bool() ? 1 : 0;
  if (!G.stop_ids.empty()) { s.stop_ids = G.stop_ids.data(); s.n_stop_ids = uint32_t(G.stop_ids.size()); }
  std::vector<std::string> stop_strings;   // OpenAI `stop`: a string or up to a few strings, matched on the text
  if (const Json* sp = req.get("stop")) {
    if (sp->is_string()) stop_strings.push_back(sp->str());
    else if (sp->is_array()) for (auto& x : sp->items()) if (x.is_string()) stop_strings.push_back(x.str());
  }
  StopMatcher stopper(stop_strings);
  const bool stream = req.get("stream") && req.get("stream")->as_bool();
  bool include_usage = kind == 1;
  if (const Json* so = req.get("stream_options")) if (const Json* iu = so->get("include_usage")) include_usage = iu->as_bool();
  if (ids.size() + s.max_tokens > G.max_ctx) s.max_tokens = ids.size() < G.max_ctx ? uint32_t(G.max_ctx - ids.size()) : 0;

  const auto t0 = std::chrono::steady_clock::now();
  uint64_t rid = 0;
  int rc = s.max_tokens ? llmlb_request_submit(G.eng, ids.data(), uint32_t(ids.size()), &s, &rid) : LLMLB_E_INVALID_ARG;
  if (rc == LLMLB_E_QUEUE_FULL) {   // openai.rs:841-861: 429 rate_limit_exceeded + Retry-After = queue timeout
    const ClientError qe = queue_capacity_exceeded(G.queue_timeout_ms / 1000);
    const std::string ra = "Retry-After: " + std::to_string(qe.retry_after) + "\r\n";
    send_err(qe.status, qe.message, qe.type.c_str(), ra.c_str());
    return;
  }
  if (rc != LLMLB_OK) {
    int st = map_error(rc);
    send_err(st, s.max_tokens ? llmlb_last_error() : "prompt exceeds the context length", st == 400 ? "invalid_request_error" : "endpoint_request_error");
    return;
  }
  // every exit path below gives the endpoint's active slot back: a path that forgets to complete
  // the lease finishes it as Error when the lease goes out of scope (balancer/lease.rs:71-100)
  RequestLease lease;
  if (!G.lm.begin_request_lease(ep, &lease)) { llmlb_request_cancel(G.eng, rid); llmlb_request_release(G.eng, rid); send_err(502, "endpoint disappeared", "endpoint_request_error"); return; }
  const uint64_t n = G.seq.fetch_add(1);
  const std::string id = std::string(kind == 0 ? "chatcmpl-" : kind == 1 ? "resp_" : "cmpl-") + std::to_string(n);
  const int64_t created = int64_t(std::chrono::duration_cast<std::chrono::seconds>(std::chrono::system_clock::now().time_since_epoch()).count());
  const std::string role = "assistant";
  bool ok = true, client_gone = false;
  AnthropicStreamTransformer to_anthropic(jm->str(), int64_t(ids.size()), "msg_" + std::to_string(n));
  // every SSE chunk leaves through here: verbatim, or re-framed as Anthropic events
  auto send_sse = [&](const std::string& openai_sse) -> bool {
    if (!anthropic) return send_chunk(fd, openai_sse);
    to_anthropic.feed(openai_sse);
    const std::string out = to_anthropic.take_output();
    return out.empty() ? true : send_chunk(fd, out);
  };
  if (stream) {
    ok = send_all(fd, "HTTP/1.1 200 OK\r\nContent-Type: text/event-stream\r\nCache-Control: no-cache\r\nTransfer-Encoding: chunked\r\n\r\n");
    if (kind == 0) ok = ok && send_sse(sse_event(chat_chunk(id, jm->str(), created, &role, nullptr, nullptr)));
    if (kind == 1) ok = ok && send_chunk(fd, sse_event(responses_event_created(id, jm->str())) + sse_event(responses_event_item_added()) + sse_event(responses_event_part_added()));
  }
  std::string text;
  BpeTokenizer::Stream detok;
  uint32_t prompt_tokens = uint32_t(ids.size()), completion_tokens = 0, finish = LLMLB_FINISH_NONE;
  while (finish == LLMLB_FINISH_NONE) {
    llmlb_token_event ev[64];
    uint32_t got = 0;
    rc = llmlb_request_poll(G.eng, rid, ev, 64, &got, 100);
    if (rc != LLMLB_OK && rc != LLMLB_E_TIMEOUT) { finish = LLMLB_FINISH_ERROR; break; }
    // a client that went away stops the generation, streamed or not — the reference's handler future is dropped with the
    // connection and its upstream request with it; a buffered response would otherwise run to its last token for nobody
    if (!client_gone && peer_closed(fd)) { ok = false; client_gone = true; llmlb_request_cancel(G.eng, rid); }
    std::string out;
    for (uint32_t i = 0; i < got; ++i) {
      if (ev[i].token_id >= 0) {
        // with a tokenizer a delta only carries complete UTF-8 (a character split over tokens waits)
        const std::string raw_piece = G.tok ? G.tok->decode_next(&detok, ev[i].token_id, /*skip_special=*/true)
                                            : byte_detokenize(ev[i].token_id);
        // a stop string may span tokens: text that could still become one is held back
        const std::string piece = stopper.feed(raw_piece);
        text += piece;
        if (stream && !piece.empty()) out += kind == 1 ? sse_event(responses_event_delta(piece))
                                     : kind == 2 ? sse_event(completion_chunk(id, jm->str(), created, &piece, nullptr))
                                     : sse_event(chat_chunk(id, jm->str(), created, nullptr, &piece, nullptr));
      }
      prompt_tokens = ev[i].prompt_tokens; completion_tokens = ev[i].completion_tokens;
      if (ev[i].finish_reason) finish = ev[i].finish_reason;
      if (stopper.hit()) {   // the text ends before the stop string: stop generating, report "stop"
        llmlb_request_cancel(G.eng, rid);
        finish = LLMLB_FINISH_STOP;
        break;
      }
    }
    if (stream && !out.empty() && ok && !send_sse(out)) { ok = false; client_gone = true; llmlb_request_cancel(G.eng, rid); }
  }
  if (!stopper.hit()) {  // text held back as a possible stop prefix, and a character cut by the end of generation
    std::string rest = stopper.feed(G.tok ? BpeTokenizer::flush(&detok) : std::string());
    if (!stopper.hit()) rest += stopper.flush();
    if (!rest.empty()) {
      text += rest;
      if (stream && ok) send_sse(kind == 1 ? sse_event(responses_event_delta(rest))
                                 : kind == 2 ? sse_event(completion_chunk(id, jm->str(), created, &rest, nullptr))
                                 : sse_event(chat_chunk(id, jm->str(), created, nullptr, &rest, nullptr)));
    }
  }
  llmlb_request_release(G.eng, rid);
  const uint64_t ms = uint64_t(std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::steady_clock::now() - t0).count());
  // streaming drop still counts as success when tokens flowed (openai.rs:2556-2648)
  const bool success = finish == LLMLB_FINISH_STOP || finish == LLMLB_FINISH_LENGTH || (client_gone && completion_tokens > 0);
  {
    TokenUsage tu; tu.has_in = tu.has_out = tu.has_total = true; tu.in = prompt_tokens; tu.out = completion_tokens; tu.total = prompt_tokens + completion_tokens;
    lease.complete_with_tokens(success ? RequestOutcome::Success : RequestOutcome::Error, ms, &tu);
  }
  if (success && completion_tokens) G.lm.update_tps(ep, pm.base, api, completion_tokens, std::max<uint64_t>(1, ms));   // `.as_millis().max(1)`: openai.rs:1241-1245, proxy.rs:157
  const char* fr = finish == LLMLB_FINISH_STOP ? "stop" : "length";
  // failures map like the gateway maps an upstream's (openai.rs:862-882, openai_util.rs:86-134)
  const bool failed = finish != LLMLB_FINISH_STOP && finish != LLMLB_FINISH_LENGTH && !(client_gone && completion_tokens > 0);
  ClientError fe = classify_upstream_request_error(UpstreamFailure::Other, 0);                 // the engine failed the request
  if (finish == LLMLB_FINISH_QUEUE_TIMEOUT) fe = queue_wait_timeout();
  else if (finish == LLMLB_FINISH_DEADLINE) fe = classify_upstream_request_error(UpstreamFailure::Timeout, (G.request_timeout_ms + 999) / 1000);
  const int fail_status = fe.status;
  const std::string fail_msg = fe.message, fail_type = fe.type;
  if (failed && !stream) { send_err(fail_status, fail_msg, fail_type.c_str()); return; }
  if (stream) {
    if (!ok) return;
    if (failed) {   // headers are gone: say so in-band and end the stream WITHOUT a finish chunk or [DONE]
      if (anthropic) {   // Anthropic's streaming error event: `event: error` + {"type":"error","error":{"type","message"}}
        send_chunk(fd, "event: error\ndata: " + anthropic_error_body(fail_status, fail_msg) + "\n\n");
        send_all(fd, "0\r\n\r\n");
        return;
      }
      Json err = Json::object(); err.set("message", fail_msg); err.set("type", fail_type); err.set("code", fail_status);
      Json root = Json::object(); root.set("error", err);
      send_chunk(fd, sse_event(root));
      send_all(fd, "0\r\n\r\n");
      return;
    }
    std::string tail;
    if (kind == 0) {
      tail += sse_event(chat_chunk(id, jm->str(), created, nullptr, nullptr, fr));
      if (include_usage) tail += sse_event(chat_usage_chunk(id, jm->str(), created, prompt_tokens, completion_tokens));
    } else if (kind == 1) {
      tail += sse_event(responses_event_text_done(text)) + sse_event(responses_event_done(id, prompt_tokens, completion_tokens));
    } else {   // legacy completions: text_completion chunks, a finish chunk, optional usage
      tail += sse_event(completion_chunk(id, jm->str(), created, nullptr, fr));
      if (include_usage) tail += sse_event(completion_usage_chunk(id, jm->str(), created, prompt_tokens, completion_tokens));
    }
    tail += sse_done();
    if (anthropic) {  // usage always travels to the transformer (message_delta carries output_tokens)
      if (!include_usage) to_anthropic.feed(sse_event(chat_usage_chunk(id, jm->str(), created, prompt_tokens, completion_tokens)));
      to_anthropic.feed(tail);
      to_anthropic.finish();
      send_chunk(fd, to_anthropic.take_output());
    } else {
      send_chunk(fd, tail);
    }
    send_all(fd, "0\r\n\r\n");
  } else if (anthropic) {
    const Json chat = chat_completion_body(id, jm->str(), created, text, fr, prompt_tokens, completion_tokens);
    send_json(fd, 200, openai_to_anthropic_message_response(chat, jm->str(), prompt_tokens, completion_tokens, "msg_" + std::to_string(n)).dump());
  } else {
    Json body = kind == 0 ? chat_completion_body(id, jm->str(), created, text, fr, prompt_tokens, completion_tokens)
              : kind == 1 ? responses_body(id, jm->str(), created, text, prompt_tokens, completion_tokens, "completed")
                          : completion_body(id, jm->str(), created, text, fr, prompt_tokens, completion_tokens);
    send_json(fd, 200, body.dump());
  }
}

// POST /v1/messages (llmlb/src/api/anthropic.rs:83-135 handle_messages): version header, request
// translation, then the chat path with Anthropic framing.  "anthropic:" cloud models are the
// gateway's business, not this endpoint's.
static void handle_messages(int fd, const Request& rq) {
  AnthropicError err;
  auto ver = rq.headers.find("anthropic-version");
  if (!anthropic_required_header(ver != rq.headers.end() ? ver->second.c_str() : nullptr, "anthropic-version", &err)) { send_json(fd, err.status, err.body()); return; }
  Json payload, openai;
  if (!Json::parse(rq.body, &payload) || !payload.is_object()) { send_json(fd, 400, anthropic_error_body(400, "invalid JSON body")); return; }
  if (!anthropic_request_to_openai(payload, &openai, nullptr, nullptr, &err)) { send_json(fd, err.status, err.body()); return; }
  handle_generate(fd, rq, 0, &openai, true);
}

static void handle(int fd, const Request& rq) {
  const std::string path = rq.path.substr(0, rq.path.find('?'));
  if (!G.api_key.empty()) {  // endpoint registered with an api_key => every call carries Bearer (proxy.rs:390-392)
    std::string key, err;
    auto xa = rq.headers.find("x-api-key"); auto au = rq.headers.find("authorization");
    int rc = extract_api_key(xa != rq.headers.end() ? xa->second.c_str() : nullptr, au != rq.headers.end() ? au->second.c_str() : nullptr, &key, &err);
    if (rc != 0 || key != G.api_key) {
      if (path == "/v1/messages") send_json(fd, 401, anthropic_error_body(401, "Invalid or missing x-api-key"));   // auth/middleware.rs:551-557
      else send_json(fd, 401, openai_error_body(rc ? err : "Invalid API key", "invalid_request_error", 401));
      return;
    }
  }
  if (rq.method == "GET" && path == "/v1/models") {
    Json m = Json::object(); m.set("id", G.model_id); m.set("object", "model"); m.set("created", 0); m.set("owned_by", "llmlb_b200");
    Json data = Json::array(); data.push(m);
    Json root = Json::object(); root.set("object", "list"); root.set("data", data);
    send_json(fd, 200, root.dump());
  } else if (rq.method == "GET" && path == "/api/system") {
    Json root = Json::object(); root.set("xllm_version", "llmlb_b200-0.1"); root.set("engine", "llmlb_b200"); root.set("device", "NVIDIA H100");
    send_json(fd, 200, root.dump());
  } else if (rq.method == "GET" && path == "/api/health") {
    llmlb_health h; llmlb_engine_health(G.eng, &h);
    Json gpu = Json::object(); gpu.set("device_count", h.device_count); gpu.set("total_memory_bytes", h.total_memory_bytes);
    gpu.set("used_memory_bytes", h.used_memory_bytes); gpu.set("capability_score", 100);
    Json load = Json::object(); load.set("active_requests", h.active_requests); load.set("queued_requests", h.queued_requests);
    load.set("in_flight_http", G.gate.in_flight());
    Json kv = Json::object(); kv.set("free_pages", h.free_kv_pages); kv.set("total_pages", h.total_kv_pages);
    Json root = Json::object(); root.set("status", "ok"); root.set("gpu", gpu); root.set("load", load); root.set("kv", kv);
    send_json(fd, 200, root.dump());
  } else if (rq.method == "GET" && path.compare(0, 12, "/api/models/") == 0 && path.size() > 17 && path.compare(path.size() - 5, 5, "/info") == 0) {
    // the gateway escapes ' ', '/' and ':' in the id (metadata/xllm.rs:54-63: "meta-llama/Llama-3-8B" arrives as meta-llama%2FLlama-3-8B)
    const std::string name = percent_decode(path.substr(12, path.size() - 17));
    if (name != G.model_id) { send_json(fd, 404, openai_error_body("model not found", "invalid_request_error", 404)); return; }
    llmlb_model_info mi; llmlb_engine_model_info(G.eng, &mi);
    Json root = Json::object(); root.set("model", G.model_id); root.set("context_length", mi.context_length);
    root.set("vocab_size", mi.vocab); root.set("num_layers", mi.n_layers); root.set("hidden_size", mi.hidden);
    send_json(fd, 200, root.dump());
  } else if (rq.method == "POST" && path == "/v1/chat/completions") handle_generate(fd, rq, 0);
  else if (rq.method == "POST" && path == "/v1/responses") handle_generate(fd, rq, 1);
  else if (rq.method == "POST" && path == "/v1/completions") handle_generate(fd, rq, 2);
  else if (rq.method == "POST" && path == "/v1/messages") handle_messages(fd, rq);
  else if (rq.method == "POST" && path == "/api/models/download") {        // llmlb/src/xllm/download.rs:97-139 is the client of this route
    Json body, resp;
    if (!Json::parse(rq.body, &body)) { send_json(fd, 400, "{\"error\":\"invalid JSON body\"}"); return; }
    const int st = G.downloads->start(body, &resp);
    send_json(fd, st, resp.dump());
  } else if (rq.method == "GET" && path == "/api/download/progress") {       // download.rs:147-190
    std::string task_id;
    const size_t q = rq.path.find("task_id=");
    if (q != std::string::npos) { task_id = rq.path.substr(q + 8); task_id = task_id.substr(0, task_id.find('&')); }
    Json resp;
    const int st = G.downloads->progress(task_id, &resp);
    send_json(fd, st, resp.dump());
  }
  else if (rq.method == "POST" && path == "/admin/drain") { G.gate.set_rejecting(rq.body.find("true") != std::string::npos); send_json(fd, 200, "{\"ok\":true}"); }
  else send_json(fd, 404, openai_error_body("not found", "invalid_request_error", 404));
}

static void serve_conn(int fd) {
  int one = 1;
  setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof one);
  auto tv = [](uint32_t ms) { timeval t; t.tv_sec = ms / 1000; t.tv_usec = (ms % 1000) * 1000; return t; };
  if (G.send_timeout_ms) { const timeval t = tv(G.send_timeout_ms); setsockopt(fd, SOL_SOCKET, SO_SNDTIMEO, &t, sizeof t); }
  if (G.idle_timeout_ms) { const timeval t = tv(G.idle_timeout_ms); setsockopt(fd, SOL_SOCKET, SO_RCVTIMEO, &t, sizeof t); }
  std::string buf;
  Request rq;
  for (;;) {
    const ReqStatus st = read_request(fd, buf, &rq);
    if (st != kReqOk) {
      if (st != kReqClosed)
        send_json(fd, int(st), openai_error_body(st == kReqTooLarge ? "request body exceeds the 20 MiB limit" : st == kReqBad ? "malformed HTTP request" : "request headers too large",
                                                 "invalid_request_error", int(st)), "Connection: close\r\n");
      break;
    }
    handle(fd, rq);
    auto c = rq.headers.find("connection");
    if (c != rq.headers.end() && strcasecmp(c->second.c_str(), "close") == 0) break;
  }
  close(fd);
}

// ---- checkpoint planning (no GPU involved; `--dry-run` stops after it) ----
// geometry of a sharded checkpoint: every file contributes what it knows; the layer count is the
// maximum (safetensors shards only see their own layers), everything else must agree
static bool merge_geometry(CkptGeometry* g, const CkptGeometry& f, std::string* err) {
  auto take = [&](uint32_t* dst, uint32_t v, const char* what) {
    if (!v) return true;
    if (*dst && *dst != v) { *err = std::string("the weight files disagree about ") + what; return false; }
    *dst = v;
    return true;
  };
  g->n_layers = std::max(g->n_layers, f.n_layers);
  if (f.known || f.hidden) { g->rope_theta = f.rope_theta; g->rms_eps = f.rms_eps; }
  return take(&g->hidden, f.hidden, "hidden") && take(&g->n_heads, f.n_heads, "n_heads") && take(&g->n_kv_heads, f.n_kv_heads, "n_kv_heads") &&
         take(&g->head_dim, f.head_dim, "head_dim") && take(&g->ffn, f.ffn, "ffn") && take(&g->vocab, f.vocab, "vocab");
}

struct WeightPlan {
  struct Load { size_t ckpt, index; std::string as; };   // tensor `index` of file `ckpt`, loaded under engine name `as`
  std::vector<Load> loads;
  bool lm_head_tied = false;
};

// buffers that ship inside checkpoints but are not model weights
static bool is_ignorable_tensor(const std::string& n) {
  auto ends = [&](const char* suf) { const size_t l = strlen(suf); return n.size() >= l && n.compare(n.size() - l, l, suf) == 0; };
  return ends("rotary_emb.inv_freq") || ends("rope_freqs.weight") || ends(".attn.bias") || ends(".masked_bias");
}

static bool plan_weights(const llmlb_model_config& m, const std::vector<std::unique_ptr<Checkpoint>>& ckpts, WeightPlan* plan, std::string* err) {
  std::map<std::string, std::pair<uint64_t, uint64_t>> want;   // name -> full (rows, cols)
  const uint64_t H = m.hidden, q = uint64_t(m.n_heads) * m.head_dim, kv = uint64_t(m.n_kv_heads) * m.head_dim, F = m.ffn, V = m.vocab;
  want["model.embed_tokens.weight"] = {V, H}; want["model.norm.weight"] = {1, H}; want["lm_head.weight"] = {V, H};
  for (uint32_t l = 0; l < m.n_layers; ++l) {
    const std::string p = "model.layers." + std::to_string(l) + ".";
    want[p + "self_attn.q_proj.weight"] = {q, H}; want[p + "self_attn.k_proj.weight"] = {kv, H}; want[p + "self_attn.v_proj.weight"] = {kv, H};
    want[p + "self_attn.o_proj.weight"] = {H, q}; want[p + "mlp.gate_proj.weight"] = {F, H}; want[p + "mlp.up_proj.weight"] = {F, H};
    want[p + "mlp.down_proj.weight"] = {H, F}; want[p + "input_layernorm.weight"] = {1, H}; want[p + "post_attention_layernorm.weight"] = {1, H};
  }
  std::map<std::string, WeightPlan::Load> found;
  for (size_t ci = 0; ci < ckpts.size(); ++ci) {
    const auto& ts = ckpts[ci]->tensors();
    for (size_t i = 0; i < ts.size(); ++i) {
      const CkptTensor& t = ts[i];
      auto w = want.find(t.name);
      if (w == want.end()) {
        if (is_ignorable_tensor(t.name)) continue;
        *err = "unexpected tensor " + t.name + " (not part of a Llama decoder of this geometry)";
        return false;
      }
      if (t.rows != w->second.first || t.cols != w->second.second) {
        *err = t.name + " is " + std::to_string(t.rows) + "x" + std::to_string(t.cols) + ", the model needs " + std::to_string(w->second.first) + "x" + std::to_string(w->second.second);
        return false;
      }
      if (found.count(t.name)) { *err = t.name + " appears in more than one file"; return false; }
      found[t.name] = WeightPlan::Load{ci, i, t.name};
    }
  }
  // a tied output head (no lm_head.weight in the files): serve it from the embedding
  if (!found.count("lm_head.weight") && found.count("model.embed_tokens.weight")) {
    WeightPlan::Load ld = found["model.embed_tokens.weight"];
    ld.as = "lm_head.weight";
    found["lm_head.weight"] = ld;
    plan->lm_head_tied = true;
  }
  std::string missing;
  size_t n_missing = 0;
  for (const auto& w : want)
    if (!found.count(w.first)) { if (n_missing++ < 4) missing += (missing.empty() ? "" : ", ") + w.first; }
  if (n_missing) { *err = std::to_string(n_missing) + " weights of the model are in none of the files: " + missing + (n_missing > 4 ? ", ..." : ""); return false; }
  for (const auto& f : found) plan->loads.push_back(f.second);
  return true;
}

int main(int argc, char** argv) {
  signal(SIGPIPE, SIG_IGN);
  int port = 8011; std::string geometry = "8b", tokenizer_path, mirror_root, models_dir;
  std::vector<std::string> weight_files;   // --weights x.gguf | shard.safetensors (repeatable)
  uint32_t max_seqs = 64, max_ctx = 2048, vocab_override = 0;
  // queue limits of the gateway (llmlb/src/config.rs:80-99: LLMLB_QUEUE_MAX 100, LLMLB_QUEUE_TIMEOUT_SECS 60)
  // and its per-request inference timeout (types/endpoint.rs:389: 120 s)
  uint32_t queue_max = 100, queue_timeout_ms = 60000, request_timeout_ms = 120000;
  bool dry_run = false;
  G.model_id = "llama-3-8b";
  for (int i = 1; i < argc; ++i) if (std::string(argv[i]) == "--dry-run") { dry_run = true; for (int j = i; j + 1 < argc; ++j) argv[j] = argv[j + 1]; --argc; --i; }
  for (int i = 1; i + 1 < argc; i += 2) {
    std::string k = argv[i], v = argv[i + 1];
    if (k == "--port") port = atoi(v.c_str()); else if (k == "--model") geometry = v;
    else if (k == "--model-id") G.model_id = v; else if (k == "--max-seqs") max_seqs = uint32_t(atoi(v.c_str()));
    else if (k == "--max-ctx") max_ctx = uint32_t(atoi(v.c_str())); else if (k == "--api-key") G.api_key = v;
    else if (k == "--tokenizer") tokenizer_path = v;
    else if (k == "--weights") weight_files.push_back(v);
    else if (k == "--vocab") vocab_override = uint32_t(atoi(v.c_str()));
    else if (k == "--queue-max") queue_max = uint32_t(atoi(v.c_str()));
    else if (k == "--queue-timeout-ms") queue_timeout_ms = uint32_t(atoi(v.c_str()));
    else if (k == "--request-timeout-ms") request_timeout_ms = uint32_t(atoi(v.c_str()));
    else if (k == "--send-timeout-ms") G.send_timeout_ms = uint32_t(atoi(v.c_str()));
    else if (k == "--idle-timeout-ms") G.idle_timeout_ms = uint32_t(atoi(v.c_str()));
    else if (k == "--max-connections") G.max_connections = uint32_t(atoi(v.c_str()));
    else if (k == "--mirror-root") mirror_root = v;      // local mirror of the model hub (the box has no network)
    else if (k == "--models-dir") models_dir = v;        // where downloaded files land
  }
  llmlb_engine_config cfg; memset(&cfg, 0, sizeof cfg);
  cfg.abi_version = LLMLB_ABI_VERSION;
  if (geometry == "tiny") cfg.model = {512, 2, 8, 2, 128, 1024, 2048, 500000.f, 1e-5f};
  else cfg.model = {4096, 32, 32, 8, 128, 14336, 128256, 500000.f, 1e-5f};
  // real checkpoints: geometry merged over ALL files (--model auto; a sharded safetensors checkpoint
  // spreads the layers over its shards), every tensor validated BEFORE the engine exists, and
  // start-up fails unless every weight of the model was found (no silently synthetic layers)
  std::vector<std::unique_ptr<Checkpoint>> ckpts;
  for (const auto& wf : weight_files) {
    std::string err;
    ckpts.emplace_back(new Checkpoint());
    if (!ckpts.back()->open(wf, &err)) { fprintf(stderr, "weights %s: %s\n", wf.c_str(), err.c_str()); return 2; }
  }
  if (geometry == "auto") {
    if (ckpts.empty()) { fprintf(stderr, "--model auto needs --weights with a file that describes the model\n"); return 2; }
    CkptGeometry g{};
    std::string err;
    for (const auto& c : ckpts) if (!merge_geometry(&g, c->geometry(), &err)) { fprintf(stderr, "weights: %s\n", err.c_str()); return 2; }
    if (!(g.hidden && g.n_layers && g.n_heads && g.n_kv_heads && g.ffn && g.vocab)) { fprintf(stderr, "--model auto: the weight files do not describe the whole model (hidden %u, layers %u, heads %u/%u, ffn %u, vocab %u)\n", g.hidden, g.n_layers, g.n_heads, g.n_kv_heads, g.ffn, g.vocab); return 2; }
    cfg.model = {g.hidden, g.n_layers, g.n_heads, g.n_kv_heads, g.head_dim ? g.head_dim : 128, g.ffn, g.vocab, g.rope_theta, g.rms_eps};
  }
  if (vocab_override) cfg.model.vocab = vocab_override;   // synthetic weights: any vocabulary size works
  WeightPlan plan;
  if (!ckpts.empty()) {
    std::string err;
    if (!plan_weights(cfg.model, ckpts, &plan, &err)) { fprintf(stderr, "weights: %s\n", err.c_str()); return 2; }
  }
  strncpy(cfg.model_id, G.model_id.c_str(), sizeof cfg.model_id - 1);
  cfg.tp_size = 1; cfg.max_seqs = max_seqs; cfg.max_ctx = max_ctx; cfg.kv_block_tokens = 64; cfg.use_cuda_graphs = 1;
  cfg.queue_max = queue_max; cfg.queue_timeout_ms = queue_timeout_ms; cfg.request_timeout_ms = request_timeout_ms;
  G.vocab = cfg.model.vocab; G.max_ctx = max_ctx; G.queue_timeout_ms = queue_timeout_ms; G.request_timeout_ms = request_timeout_ms;
  // tokenizer: --tokenizer file, else the one a .gguf carries
  std::string tok_json, tok_src = tokenizer_path;
  if (!tokenizer_path.empty()) {
    std::ifstream f(tokenizer_path, std::ios::binary);
    std::stringstream ss; ss << f.rdbuf();
    if (!f) { fprintf(stderr, "tokenizer %s: cannot read\n", tokenizer_path.c_str()); return 2; }
    tok_json = ss.str();
  } else {
    for (size_t ci = 0; ci < ckpts.size() && tok_json.empty(); ++ci) { tok_json = ckpts[ci]->tokenizer_json(); tok_src = "embedded in " + weight_files[ci]; }
  }
  if (!tok_json.empty()) {
    std::string err;
    G.tok.reset(new BpeTokenizer());
    if (!G.tok->load_json(tok_json, &err)) { fprintf(stderr, "tokenizer %s: %s\n", tok_src.c_str(), err.c_str()); return 2; }
    if (G.tok->vocab_size() > G.vocab) { fprintf(stderr, "tokenizer has %u entries, the model only %u\n", G.tok->vocab_size(), G.vocab); return 2; }
    for (const char* name : {"<|eot_id|>", "<|end_of_text|>", "<|eom_id|>"}) { const int32_t id = G.tok->special_id(name); if (id >= 0) G.stop_ids.push_back(id); }
    fprintf(stderr, "tokenizer: %u entries, %zu stop ids\n", G.tok->vocab_size(), G.stop_ids.size());
  }
  if (dry_run) {   // everything that does not need the GPU has been checked: report and leave
    const llmlb_model_config& m = cfg.model;
    printf("{\"dry_run\":true,\"model\":{\"hidden\":%u,\"n_layers\":%u,\"n_heads\":%u,\"n_kv_heads\":%u,\"head_dim\":%u,\"ffn\":%u,\"vocab\":%u},"
           "\"tensors_to_load\":%zu,\"lm_head_tied\":%s,\"tokenizer_entries\":%u,\"stop_ids\":%zu}\n",
           m.hidden, m.n_layers, m.n_heads, m.n_kv_heads, m.head_dim, m.ffn, m.vocab, plan.loads.size(), plan.lm_head_tied ? "true" : "false",
           G.tok ? G.tok->vocab_size() : 0u, G.stop_ids.size());
    return 0;
  }
  if (llmlb_engine_create(&cfg, &G.eng) != LLMLB_OK) { fprintf(stderr, "engine: %s\n", llmlb_last_error()); return 2; }
  {
    std::vector<uint16_t> bits;
    for (const WeightPlan::Load& ld : plan.loads) {
      const CkptTensor& t = ckpts[ld.ckpt]->tensors()[ld.index];
      std::string err;
      if (!ckpts[ld.ckpt]->read_bf16(ld.index, &bits, &err)) { fprintf(stderr, "weights: %s\n", err.c_str()); return 2; }
      if (llmlb_engine_load_tensor(G.eng, ld.as.c_str(), bits.data(), t.rows, t.cols) != LLMLB_OK) { fprintf(stderr, "weights: %s: %s\n", ld.as.c_str(), llmlb_last_error()); return 2; }
    }
    if (!plan.loads.empty()) fprintf(stderr, "weights: %zu tensors loaded from %zu file(s)%s\n", plan.loads.size(), ckpts.size(), plan.lm_head_tied ? " (lm_head tied to the embedding)" : "");
  }
  ckpts.clear();
  G.downloads.reset(new DownloadManager(mirror_root, models_dir));   // unconfigured: the routes answer 503
  G.lm.add_endpoint("local", true, false);
  G.lm.add_model("local", G.model_id, "");
  int ls = socket(AF_INET, SOCK_STREAM, 0), one = 1;
  setsockopt(ls, SOL_SOCKET, SO_REUSEADDR, &one, sizeof one);
  sockaddr_in addr{}; addr.sin_family = AF_INET; addr.sin_port = htons(uint16_t(port)); addr.sin_addr.s_addr = htonl(INADDR_LOOPBACK);
  if (bind(ls, (sockaddr*)&addr, sizeof addr) != 0 || listen(ls, 256) != 0) { perror("bind/listen"); return 3; }
  fprintf(stderr, "llmlb_b200_server listening on 127.0.0.1:%d model=%s\n", port, G.model_id.c_str());
  fflush(stderr);
  for (;;) {
    int fd = accept(ls, nullptr, nullptr);
    if (fd < 0) continue;
    // one thread per connection: bounded, so that a flood of connections costs file descriptors for an instant, not threads
    if (G.connections.load() >= G.max_connections) {
      send_json(fd, 503, openai_error_body("too many connections", "service_unavailable", 503), "Connection: close\r\nRetry-After: 1\r\n");
      close(fd);
      continue;
    }
    G.connections.fetch_add(1);
    std::thread([fd] { serve_conn(fd); G.connections.fetch_sub(1); }).detach();
  }
}
