/* llmlb_gateway.h — C ABI of libllmlb_host.so, part 2: the gateway rows of the hot path (SURVEY.md §8 a1.x),
 * the checkpoint readers and the model-download contract (§8 f.4).  No GPU, no CUDA.
 *
 * The reference does all of this in Rust inside the gateway process; these are the same functions behind plain
 * pointers and sizes, each group citing what it stands for.  A Rust / Go / Python host binds them the way
 * INTEGRATION.md §2 binds the engine; the CPU suite (tests/test_host_gateway.py, test_host_checkpoint.py,
 * test_host_download.py) drives exactly this surface through ctypes against the reference's own test vectors.
 * Part 1 (tokenizer, Anthropic translation) is llmlb_host.h; the engine is llmlb_b200.h.
 *
 * Conventions: NUL-terminated strings in; "out, cap" receives a NUL-terminated copy truncated to cap-1 and the
 * function returns the FULL length (call again with a larger buffer when it is >= cap); handles are opaque,
 * one owner at a time (LoadManager, InferenceGate and DownloadManager lock internally); enums travel as int.   */
#ifndef LLMLB_GATEWAY_H
#define LLMLB_GATEWAY_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* TpsApiKind (llmlb/src/common/protocol.rs:135-160): 0 chat_completions, 1 completions, 2 responses.
 * RequestOutcome (balancer/types.rs): 0 success, 1 error, 2 queued.                                             */

/* ---- a1.6 / a1.7 / a1.8 / a1.9 / a1.14: LoadManager ------------------------------------------------------------
 * registry lookup through alias keys   llmlb/src/registry/endpoints.rs:16-73,209-231
 * update_tps + EMA (alpha 0.2)         llmlb/src/balancer/mod.rs:1770, balancer/types.rs:102-118
 * TPS-priority selection, round-robin ties   balancer/mod.rs:1873-1985,2949
 * begin/finish_request(_with_tokens)   balancer/mod.rs:2273-2425;  RequestLease (drop = Error)  balancer/lease.rs:16-100 */
void* llmlb_lm_create(void);
void llmlb_lm_destroy(void* lm);
void llmlb_lm_add_mapping(void* lm, const char* canonical, const char* alias);            /* models/mapping.rs:43 table rows */
void llmlb_lm_add_endpoint(void* lm, const char* endpoint_id, int online, int initializing);
int llmlb_lm_add_model(void* lm, const char* endpoint_id, const char* model, const char* canonical /* NULL = none */);   /* 0 / -1 unknown endpoint */
int llmlb_lm_set_status(void* lm, const char* endpoint_id, int online);                   /* offline clears the TPS state (health/endpoint_checker.rs) */
int llmlb_lm_set_initializing(void* lm, const char* endpoint_id, int initializing);
void llmlb_lm_update_tps(void* lm, const char* endpoint_id, const char* model, int api_kind, uint64_t output_tokens, uint64_t duration_ms);
/* 1 when a state exists; *ema = -1.0 while no sample has been taken */
int llmlb_lm_get_tps(void* lm, const char* endpoint_id, const char* model, int api_kind, double* ema, uint64_t* request_count,
                     uint64_t* total_output_tokens, uint64_t* total_duration_ms);
/* 0 = selected (id in out), 1 = NoCapableEndpoints, 2 = NoEndpointsAvailable; model NULL = any */
int llmlb_lm_select(void* lm, const char* model, int api_kind, char* out, size_t cap);
size_t llmlb_lm_lookup_keys(void* lm, const char* model, char* out, size_t cap);          /* '\n'-joined, in lookup order */
int llmlb_lm_begin_request(void* lm, const char* endpoint_id);
int llmlb_lm_finish_request(void* lm, const char* endpoint_id, int success, uint64_t duration_ms, uint64_t output_tokens);
uint32_t llmlb_lm_active(void* lm, const char* endpoint_id);
void* llmlb_lm_lease_begin(void* lm, const char* endpoint_id);                            /* NULL: unknown endpoint */
/* usage fields < 0 = absent; with_usage 0 = complete() without tokens.  0 / -1 (already completed) */
int llmlb_lm_lease_complete(void* lease, int outcome, uint64_t duration_ms, int with_usage, int64_t input_tokens, int64_t output_tokens,
                            int64_t total_tokens);
void llmlb_lm_lease_drop(void* lease);                                                    /* a lease never completed finishes as Error here */
/* out8: active, total_assigned, success, errors, latency_ms_sum, input_tokens, output_tokens, total_tokens */
int llmlb_lm_stats(void* lm, const char* endpoint_id, uint64_t* out8);
double llmlb_lm_average_latency(void* lm, const char* endpoint_id);
/* 60-minute request history (balancer/mod.rs:2643-2658,2973-3060) */
void* llmlb_history_create(void);
void llmlb_history_destroy(void* h);
int64_t llmlb_history_align(int64_t unix_seconds);
void llmlb_history_record(void* h, int outcome, int64_t unix_seconds);
/* out: (minute, success, error) triples; window 1 = the zero-filled 60 minutes ending at now. Returns the point count */
uint32_t llmlb_history_get(void* h, int window, int64_t now, int64_t* out, uint32_t cap_points);
/* inference-latency EMA (api/openai.rs:52-72, types/endpoint.rs): ops[i] 'u' = update(values[i]), 'r' = reset;
 * returns the sort key (infinity while unmeasured) */
double llmlb_latency_play(const char* ops, const double* values, uint32_t n, int* has_value);

/* ---- a1.12 / a1.13: SSE relay accounting and usage extraction (llmlb/src/token/mod.rs:41-259, api/proxy.rs:104-116) */
void* llmlb_acc_create(const char* model);
void llmlb_acc_destroy(void* acc);
void llmlb_acc_set_input_tokens(void* acc, uint32_t n);
void llmlb_acc_process_chunk(void* acc, const char* one_data_payload);                    /* StreamingTokenAccumulator::process_chunk */
void llmlb_acc_feed(void* acc, const char* bytes, size_t n);                              /* process_sse_lines over raw network chunks */
size_t llmlb_acc_content(void* acc, char* out, size_t cap);
int llmlb_acc_done(void* acc);
void llmlb_acc_finalize(void* acc, int64_t out3[3]);                                      /* input, output, total; -1 = absent */
int llmlb_extract_usage(const char* body_json, int64_t out3[3]);                          /* extract_usage_from_response; 1 = found */
/* extract_or_estimate_tokens (token/mod.rs:225-259); returns has-bits 1 in | 2 out | 4 total */
int llmlb_extract_or_estimate(const char* body_json, const char* request_text, const char* response_text, int with_counter, uint32_t* out3);

/* ---- a1.1 / a1.2: drain gate (llmlb/src/inference_gate.rs:17-230) and API key (auth/middleware.rs:254-321) ---- */
void* llmlb_gate_create(void);
void llmlb_gate_destroy(void* gate);
int llmlb_gate_try_begin(void* gate);                                                     /* 0, or 503 while draining */
void llmlb_gate_end(void* gate);
void llmlb_gate_set_rejecting(void* gate, int rejecting);
uint32_t llmlb_gate_in_flight(void* gate);
size_t llmlb_gate_rejection_body(char* out, size_t cap);
int llmlb_extract_api_key(const char* x_api_key, const char* authorization, char* out, size_t cap);   /* 0 = key in out; else 401 + message */
void llmlb_sha256_hex(const char* data, size_t n, char out[65]);

/* ---- a1.3 / a1.5 / a1.10: model names and the upstream payload ------------------------------------------------
 * parse_quantized_model_name  api/model_name.rs:19-40;  rewrite_payload_model_for_endpoint  api/model_name.rs:43-108;
 * resolve_engine_name  models/mapping.rs:302-323;  stream_options.include_usage  api/openai.rs:977-992 */
int llmlb_parse_model_name(const char* model, char* base, char* quant, size_t cap);       /* 1 with suffix, 0 without, -1 invalid */
size_t llmlb_rewrite_payload(const char* spec_json, char* out, size_t cap);
size_t llmlb_prepare_upstream_payload(const char* payload_json, const char* upstream_model, int stream, char* out, size_t cap);

/* ---- a1.16: error conventions --------------------------------------------------------------------------------
 * openai_error_response_with_type  api/openai_util.rs:242-257;  classify_upstream_request_error  :86-134 (kind 0 timeout,
 * 1 connect, 2 other);  queue errors  api/openai.rs:841-882, openai_util.rs:264-292 (which 0 capacity, 1 wait timeout);
 * LbError table  common/error.rs:41-214 + AppError::into_response  api/error.rs:154-203.
 * The classify / queue / lb functions return JSON describing status, type, message, Retry-After and the body. */
size_t llmlb_error_body(const char* message, const char* type, int status, char* out, size_t cap);
size_t llmlb_classify_upstream_error(int kind, uint32_t timeout_secs, const char* ollama_loading_model /* NULL */, char* out, size_t cap);
size_t llmlb_queue_error(int which, uint64_t queue_timeout_secs, char* out, size_t cap);
int llmlb_lb_error_count(void);
size_t llmlb_lb_error(int kind, const char* detail, char* out, size_t cap);

/* ---- wire framing the host produces from token events (§8b rows; goldens api/openai.rs:2477-2481,
 * tests/integration/responses_streaming_test.rs:64-136, responses_api_test.rs:58-82) ---------------------------
 * kind 0 chat SSE stream, 1 chat body, 2 responses SSE stream, 3 responses body, 4 completion body */
size_t llmlb_frame(int kind, const char* id, const char* model, int64_t created, const char* const* pieces, uint32_t n_pieces,
                   uint32_t prompt_tokens, const char* finish_reason, char* out, size_t cap);
/* the same stream one step at a time, for a host that frames while token events arrive.
 * api 0 chat.completion.chunk, 1 text_completion (legacy /v1/completions), 2 Responses events.
 * what 0 opening (chat: role chunk; Responses: created + output_item.added + content_part.added; completions: nothing),
 *      1 text delta, 2 finish (chat / completions: text = finish_reason; Responses: output_text.done, text = whole text),
 *      3 usage (chat / completions: the include_usage chunk; Responses: response.done), 4 "data: [DONE]".            */
size_t llmlb_sse_event(int api, int what, const char* id, const char* model, int64_t created, const char* text,
                       uint32_t prompt_tokens, uint32_t completion_tokens, char* out, size_t cap);
size_t llmlb_json_roundtrip(const char* text, char* out, size_t cap);                     /* 0 = not JSON */
/* `stop` strings over streamed text: text that may still become a stop is held back */
void* llmlb_stop_create(const char* stops_json);
void llmlb_stop_destroy(void* m);
size_t llmlb_stop_feed(void* m, const char* piece, size_t n, char* out, size_t cap);
size_t llmlb_stop_flush(void* m, char* out, size_t cap);
int llmlb_stop_hit(void* m, char* matched, size_t cap);

/* ---- f.4: checkpoints (safetensors, GGUF incl. Q4_0..Q6_K dequantised on load; format reference
 * poc/nemotron-safetensors-cpp/main.cpp:101-113) -> row-major bf16 under Hugging Face names, what
 * llmlb_engine_load_tensor takes.  Files are untrusted input: sizes and offsets are checked, never trusted. */
void* llmlb_ckpt_open(const char* path, char* err, uint32_t err_cap);
void llmlb_ckpt_close(void* ckpt);
uint32_t llmlb_ckpt_count(void* ckpt);
int llmlb_ckpt_is_gguf(void* ckpt);
/* u7: hidden, n_layers, n_heads, n_kv_heads, head_dim, ffn, vocab; f2: rope_theta, rms_eps.  1 = geometry complete */
int llmlb_ckpt_geometry(void* ckpt, uint32_t* u7, float* f2);
/* RoPE frequency scaling the file states (GGUF rope_freqs.weight / linear metadata, llama3 or linear in a config.json
 * beside a safetensors file): per-frequency divisors, up to cap of them written to out.  Returns how many there are
 * (head_dim/2), 0 = no scaling. */
uint32_t llmlb_ckpt_rope_freq_factors(void* ckpt, float* out, uint32_t cap);
int64_t llmlb_ckpt_tensor_info(void* ckpt, uint32_t index, char* name, uint32_t name_cap, uint64_t* rows, uint64_t* cols);   /* element count, -1 bad index */
int llmlb_ckpt_tensor_bf16(void* ckpt, uint32_t index, uint16_t* out, uint64_t cap_elems);
int64_t llmlb_ckpt_tokenizer_json(void* ckpt, char* out, uint64_t cap);                   /* GGUF tokenizer.ggml.* as tokenizer.json text */

/* ---- f.4: model download contract, endpoint side (the reference is its client: llmlb/src/xllm/download.rs:31-190) -- */
void* llmlb_dl_create(const char* mirror_root, const char* models_dir, size_t chunk_bytes, unsigned throttle_us);
void llmlb_dl_destroy(void* dl);
int llmlb_dl_start(void* dl, const char* request_json, char* out, size_t cap);            /* HTTP status; body in out */
int llmlb_dl_progress(void* dl, const char* task_id, char* out, size_t cap);
int llmlb_dl_cancel(void* dl, const char* task_id, char* out, size_t cap);
size_t llmlb_dl_choose_best(const char* names_json, char* out, size_t cap);               /* "xLLM will choose the best quantization", download.rs:37-38 */
size_t llmlb_dl_quantization_of(const char* filename, char* out, size_t cap);
int llmlb_dl_safe_path(const char* relative_path);

#ifdef __cplusplus
}
#endif
#endif /* LLMLB_GATEWAY_H */
