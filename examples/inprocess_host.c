/* inprocess_host.c — the gateway's hot path with the engine IN the process: no HTTP between router and model.
 *
 * This is, in plain C over the three public headers, what the Rust FFI crate's in-process endpoint does
 * (ffi/llmlb-b200-sys/, INTEGRATION.md §2) — the steps of `proxy_openai_post` (llmlb/src/api/openai.rs:761-1338)
 * and `forward_streaming_response_with_tps_tracking` (llmlb/src/api/proxy.rs:120-270) with the single
 * `request_builder.send().await` (openai.rs:995-1005) replaced by submit / poll on the engine:
 *
 *   drain gate (inference_gate.rs:200-230)           llmlb_gate_try_begin
 *   endpoint pick by TPS EMA (balancer/mod.rs:2949)   llmlb_lm_select
 *   lease (balancer/lease.rs)                         llmlb_lm_lease_begin
 *   >>> the boundary <<<                              llmlb_request_submit / llmlb_request_poll
 *   SSE to the client                                 llmlb_tok_stream_next (ids -> UTF-8) + llmlb_sse_event
 *   the relay's side channel (token/mod.rs:72-171)    llmlb_acc_feed over the very bytes sent to the client
 *   end of stream: usage, lease, TPS (proxy.rs:147-203, 290-368)
 *                                                     llmlb_acc_finalize, llmlb_lm_lease_complete, llmlb_lm_update_tps
 *
 * Build (real engine; needs an H100):
 *   gcc -std=c99 -O2 -Iinclude examples/inprocess_host.c -Lllmlb_b200 -lllmlb_b200 -lllmlb_host -Wl,-rpath,$PWD/llmlb_b200 -o inprocess_host
 * The CPU suite builds it against tests/support/fake_engine.cpp (same ABI, scripted tokens): tests/test_inprocess_host_cpu.py.
 *
 * stdout: the client-visible SSE of every request, each preceded by a line "### request <i>".
 * stderr: one JSON object per request {"request","tokens","ms","usage":[in,out,total],"content_bytes"} and a final
 *         {"tps_ema","request_count","total_output_tokens","total_duration_ms","stats":[8]} — the router's state.     */
#define _POSIX_C_SOURCE 200809L
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "llmlb_b200.h"
#include "llmlb_gateway.h"
#include "llmlb_host.h"

static double now_ms(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec * 1e3 + ts.tv_nsec / 1e6;
}

static void die(const char* what) {
  fprintf(stderr, "inprocess_host: %s: %s\n", what, llmlb_last_error());
  exit(1);
}

typedef struct {
  const char* model_id;
  const char* tokenizer_path; /* NULL: tokens are rendered as "<id> " */
  int api;                    /* 0 chat completions, 2 responses (TpsApiKind numbering) */
  int requests, prompt_len, max_tokens;
  uint32_t vocab;
} Options;

/* Emit one piece of the stream: to the client (stdout) and through the accumulator, byte for byte the same. */
static void emit(void* acc, const char* bytes, size_t n) {
  fwrite(bytes, 1, n, stdout);
  llmlb_acc_feed(acc, bytes, n);
}

static void emit_event(void* acc, int api, int what, const char* id, const char* model, const char* text, uint32_t pt, uint32_t ct) {
  static char buf[1 << 16];
  size_t n = llmlb_sse_event(api, what, id, model, 1704067200, text, pt, ct, buf, sizeof buf);
  if (n >= sizeof buf) n = sizeof buf - 1;
  emit(acc, buf, n);
}

static int serve_one(llmlb_engine* eng, void* lm, void* gate, void* tok, const Options* o, int index) {
  char endpoint[128], id[64], piece[1024];
  /* a1.1: refuse while draining */
  if (llmlb_gate_try_begin(gate) != 0) return 503;
  /* a1.6: the router picks the endpoint that serves this model with the best TPS EMA */
  if (llmlb_lm_select(lm, o->model_id, o->api, endpoint, sizeof endpoint) != 0) { llmlb_gate_end(gate); return 503; }
  /* a1.9: lease — dropped without completion it would count as an error */
  void* lease = llmlb_lm_lease_begin(lm, endpoint);
  if (!lease) { llmlb_gate_end(gate); return 502; }

  /* the request: synthetic ids (BASELINE-style prompts), or chat-templated text when a tokenizer is loaded */
  int32_t* ids = malloc(sizeof(int32_t) * (size_t)(o->prompt_len + 64));
  int64_t n_ids = 0;
  if (tok) {
    const char* msgs = "[{\"role\":\"user\",\"content\":\"Say hello in three languages.\"}]";
    n_ids = llmlb_tok_chat_ids(tok, msgs, strlen(msgs), ids, (uint64_t)(o->prompt_len + 64));
  }
  if (n_ids <= 0) {
    uint64_t s = 0x9E3779B97F4A7C15ull * (uint64_t)(index + 1);
    for (n_ids = 0; n_ids < o->prompt_len; ++n_ids) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; ids[n_ids] = (int32_t)(s % o->vocab); }
  }
  llmlb_sampling sp;
  memset(&sp, 0, sizeof sp);
  sp.max_tokens = (uint32_t)o->max_tokens;
  sp.temperature = 0.f;
  sp.ignore_eos = 1;

  void* acc = llmlb_acc_create(o->model_id);
  void* detok = tok ? llmlb_tok_stream_create() : NULL;
  snprintf(id, sizeof id, "%s-%d", o->api == 2 ? "resp" : "chatcmpl", index);
  printf("### request %d\n", index);

  const double t0 = now_ms();
  uint64_t rid = 0;
  int rc = llmlb_request_submit(eng, ids, (uint32_t)n_ids, &sp, &rid);    /* <<< THE BOUNDARY (never blocks) */
  free(ids);
  if (rc != LLMLB_OK) {
    fprintf(stderr, "inprocess_host: submit: %s\n", llmlb_last_error());
    llmlb_lm_lease_complete(lease, 1, (uint64_t)(now_ms() - t0), 0, -1, -1, -1);
    llmlb_lm_lease_drop(lease); llmlb_acc_destroy(acc); llmlb_gate_end(gate);
    return rc == LLMLB_E_QUEUE_FULL ? 429 : 400;
  }
  const int sse_api = o->api == 2 ? 2 : 0;
  emit_event(acc, sse_api, 0, id, o->model_id, NULL, 0, 0);
  static char whole[1 << 20];
  size_t whole_n = 0;
  uint32_t prompt_tokens = 0, completion_tokens = 0, finish = 0;
  while (!finish) {
    llmlb_token_event ev[64];
    uint32_t n = 0;
    rc = llmlb_request_poll(eng, rid, ev, 64, &n, 50);
    if (rc != LLMLB_OK && rc != LLMLB_E_TIMEOUT) die("poll");
    for (uint32_t i = 0; i < n; ++i) {
      if (ev[i].token_id >= 0) {
        int64_t pn;
        if (tok) pn = llmlb_tok_stream_next(tok, detok, ev[i].token_id, 1, piece, sizeof piece);   /* only complete UTF-8 comes out */
        else pn = snprintf(piece, sizeof piece, "<%d> ", ev[i].token_id);
        if (pn > 0 && (size_t)pn < sizeof piece) {
          piece[pn] = 0;
          emit_event(acc, sse_api, 1, id, o->model_id, piece, 0, 0);
          if (whole_n + (size_t)pn < sizeof whole) { memcpy(whole + whole_n, piece, (size_t)pn); whole_n += (size_t)pn; }
        }
      }
      prompt_tokens = ev[i].prompt_tokens;
      completion_tokens = ev[i].completion_tokens;
      if (ev[i].finish_reason) finish = ev[i].finish_reason;
    }
  }
  if (detok) {
    int64_t pn = llmlb_tok_stream_flush(detok, piece, sizeof piece);
    if (pn > 0 && (size_t)pn < sizeof piece) {
      piece[pn] = 0;
      emit_event(acc, sse_api, 1, id, o->model_id, piece, 0, 0);
      if (whole_n + (size_t)pn < sizeof whole) { memcpy(whole + whole_n, piece, (size_t)pn); whole_n += (size_t)pn; }
    }
    llmlb_tok_stream_destroy(detok);
  }
  whole[whole_n] = 0;
  const int ok = finish == LLMLB_FINISH_STOP || finish == LLMLB_FINISH_LENGTH;
  if (ok) {
    emit_event(acc, sse_api, 2, id, o->model_id, sse_api == 2 ? whole : (finish == LLMLB_FINISH_STOP ? "stop" : "length"), 0, 0);
    emit_event(acc, sse_api, 3, id, o->model_id, NULL, prompt_tokens, completion_tokens);
    emit_event(acc, sse_api, 4, id, o->model_id, NULL, 0, 0);
  }
  llmlb_request_release(eng, rid);
  uint64_t ms = (uint64_t)(now_ms() - t0);                 /* request start -> last byte ... */
  if (ms < 1) ms = 1;                                      /* ... clamped like `elapsed().as_millis().max(1)`, proxy.rs:154-160 */

  /* end of stream: what the relay learned from the bytes it forwarded */
  int64_t u[3];
  llmlb_acc_finalize(acc, u);
  llmlb_lm_lease_complete(lease, ok ? 0 : 1, ms, ok, u[0], u[1], u[2]);
  llmlb_lm_lease_drop(lease);
  if (ok && u[1] > 0) llmlb_lm_update_tps(lm, endpoint, o->model_id, o->api, (uint64_t)u[1], ms);
  static char content[1 << 20];
  const size_t content_n = llmlb_acc_content(acc, content, sizeof content);
  fprintf(stderr, "{\"request\": %d, \"endpoint\": \"%s\", \"tokens\": %u, \"ms\": %llu, \"usage\": [%lld, %lld, %lld], \"content_bytes\": %zu, \"sent_bytes\": %zu, \"done\": %d, \"finish\": %u}\n",
          index, endpoint, completion_tokens, (unsigned long long)ms, (long long)u[0], (long long)u[1], (long long)u[2], content_n, whole_n,
          llmlb_acc_done(acc), finish);
  llmlb_acc_destroy(acc);
  llmlb_gate_end(gate);
  return ok ? 200 : 502;
}

int main(int argc, char** argv) {
  Options o = {"llama-tiny", NULL, 0, 3, 24, 16, 3072};
  uint32_t hidden = 512, layers = 2, heads = 8, kv_heads = 2, ffn = 1024;
  for (int i = 1; i + 1 < argc; i += 2) {
    const char* k = argv[i];
    const char* v = argv[i + 1];
    if (!strcmp(k, "--model-id")) o.model_id = v;
    else if (!strcmp(k, "--tokenizer")) o.tokenizer_path = v;
    else if (!strcmp(k, "--api")) o.api = !strcmp(v, "responses") ? 2 : 0;
    else if (!strcmp(k, "--requests")) o.requests = atoi(v);
    else if (!strcmp(k, "--prompt-len")) o.prompt_len = atoi(v);
    else if (!strcmp(k, "--max-tokens")) o.max_tokens = atoi(v);
    else if (!strcmp(k, "--vocab")) o.vocab = (uint32_t)atoi(v);
    else if (!strcmp(k, "--hidden")) hidden = (uint32_t)atoi(v);
    else if (!strcmp(k, "--layers")) layers = (uint32_t)atoi(v);
    else if (!strcmp(k, "--heads")) heads = (uint32_t)atoi(v);
    else if (!strcmp(k, "--kv-heads")) kv_heads = (uint32_t)atoi(v);
    else if (!strcmp(k, "--ffn")) ffn = (uint32_t)atoi(v);
    else { fprintf(stderr, "unknown option %s\n", k); return 2; }
  }

  void* tok = NULL;
  if (o.tokenizer_path) {
    FILE* f = fopen(o.tokenizer_path, "rb");
    if (!f) { perror(o.tokenizer_path); return 2; }
    fseek(f, 0, SEEK_END);
    long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    char* text = malloc((size_t)n + 1);
    if (fread(text, 1, (size_t)n, f) != (size_t)n) { perror("read"); return 2; }
    fclose(f);
    char err[256] = "";
    tok = llmlb_tok_create(text, (uint64_t)n, err, sizeof err);
    free(text);
    if (!tok) { fprintf(stderr, "tokenizer: %s\n", err); return 2; }
    o.vocab = llmlb_tok_vocab_size(tok) > o.vocab ? llmlb_tok_vocab_size(tok) : o.vocab;
  }

  llmlb_engine_config cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.abi_version = LLMLB_ABI_VERSION;
  cfg.model.hidden = hidden; cfg.model.n_layers = layers; cfg.model.n_heads = heads; cfg.model.n_kv_heads = kv_heads;
  cfg.model.head_dim = 128; cfg.model.ffn = ffn; cfg.model.vocab = o.vocab;
  cfg.model.rope_theta = 500000.f; cfg.model.rms_eps = 1e-5f;
  snprintf(cfg.model_id, sizeof cfg.model_id, "%s", o.model_id);
  cfg.device = 0; cfg.tp_rank = 0; cfg.tp_size = 1;
  cfg.max_seqs = 8; cfg.max_ctx = 1024; cfg.kv_block_tokens = 64;
  cfg.synthetic_seed = 0; cfg.use_cuda_graphs = 1;
  llmlb_engine* eng = NULL;
  if (llmlb_engine_create(&cfg, &eng) != LLMLB_OK) die("engine_create");      /* no GPU, no engine: there is no CPU path */

  /* bootstrap (bootstrap.rs:85-91): the local engine registered as one endpoint serving its model id */
  void* lm = llmlb_lm_create();
  void* gate = llmlb_gate_create();
  llmlb_model_info info;
  if (llmlb_engine_model_info(eng, &info) != LLMLB_OK) die("model_info");
  llmlb_lm_add_endpoint(lm, "in-process", 1, 0);
  llmlb_lm_add_model(lm, "in-process", info.id, NULL);

  int bad = 0;
  for (int i = 0; i < o.requests; ++i) bad += serve_one(eng, lm, gate, tok, &o, i) != 200;

  double ema = -1.0;
  uint64_t cnt = 0, toks = 0, ms = 0, st[8] = {0};
  llmlb_lm_get_tps(lm, "in-process", o.model_id, o.api, &ema, &cnt, &toks, &ms);
  llmlb_lm_stats(lm, "in-process", st);
  fprintf(stderr, "{\"tps_ema\": %.17g, \"request_count\": %llu, \"total_output_tokens\": %llu, \"total_duration_ms\": %llu, \"in_flight\": %u, "
                  "\"stats\": [%llu, %llu, %llu, %llu, %llu, %llu, %llu, %llu]}\n",
          ema, (unsigned long long)cnt, (unsigned long long)toks, (unsigned long long)ms, llmlb_gate_in_flight(gate),
          (unsigned long long)st[0], (unsigned long long)st[1], (unsigned long long)st[2], (unsigned long long)st[3], (unsigned long long)st[4],
          (unsigned long long)st[5], (unsigned long long)st[6], (unsigned long long)st[7]);
  llmlb_gate_destroy(gate);
  llmlb_lm_destroy(lm);
  llmlb_engine_destroy(eng);
  if (tok) llmlb_tok_destroy(tok);
  return bad ? 1 : 0;
}
