//! `llmlb/src/api/inprocess.rs` (NEW file in the gateway): an endpoint that lives in the gateway
//! process.  It answers the same question `forward_to_endpoint` (llmlb/src/api/proxy.rs:372-431)
//! and the inline builder (llmlb/src/api/openai.rs:995-1005) answer today — "give me the upstream's
//! response for this payload" — from `libllmlb_b200.so` instead of over HTTP, and hands back the very
//! shape the callers already consume: status + headers + a byte stream of OpenAI JSON / SSE.
//! That keeps `forward_streaming_response_with_tps_tracking` (proxy.rs:120-270), the
//! `StreamingTokenAccumulator`, `record_endpoint_request_stats` and the request history untouched.
//!
//! Source only: there is no Rust toolchain in the build image of llmlb_b200; see README.md beside
//! this file for the four edits that wire it in.
use std::sync::Arc;
use std::time::{Duration, Instant};

use bytes::Bytes;
use futures::Stream;
use llmlb_b200_sys::{llmlb_token_event, Engine, EngineError, RequestGuard, Sampling, LLMLB_FINISH_DEADLINE,
                     LLMLB_FINISH_LENGTH, LLMLB_FINISH_QUEUE_TIMEOUT, LLMLB_FINISH_STOP};
use serde_json::{json, Value};

/// Text <-> token ids.  The gateway may bind `libllmlb_host.so` (`include/llmlb_host.h`:
/// llmlb_tok_chat_ids / llmlb_tok_stream_next) or bring its own tokenizer crate.
pub trait Tokenizer: Send + Sync {
    fn chat_ids(&self, messages: &Value) -> Result<Vec<i32>, String>;
    fn encode(&self, text: &str) -> Vec<i32>;
    /// streaming detokeniser state; returns only complete UTF-8
    fn new_stream(&self) -> Box<dyn DetokStream>;
    fn stop_ids(&self) -> Vec<i32>;
}
pub trait DetokStream: Send {
    fn next(&mut self, id: i32) -> String;
    fn flush(&mut self) -> String;
}

pub struct InProcessEndpoint {
    pub engine: Arc<Engine>,
    pub tokenizer: Arc<dyn Tokenizer>,
    pub model_id: String,
}

/// What the HTTP path gets from reqwest, reduced to what the callers read.
pub struct LocalResponse {
    pub status: u16,
    pub content_type: &'static str,
    pub body: LocalBody,
}
pub enum LocalBody {
    Json(Value),
    Sse(std::pin::Pin<Box<dyn Stream<Item = Result<Bytes, std::io::Error>> + Send>>),
}

/// `frequency_penalty`, `presence_penalty` (null or absent: 0) and `logit_bias` ({"token id": value}) as OpenAI sends them;
/// a bias key that is not a decimal token id is kept as -1, which the engine refuses with a 400 naming the field.
fn sampling_from(payload: &Value, max_key: &str, stop_ids: Vec<i32>) -> Sampling {
    let logit_bias = payload
        .get("logit_bias")
        .and_then(Value::as_object)
        .map(|m| m.iter().map(|(k, v)| (k.parse::<i32>().unwrap_or(-1), v.as_f64().unwrap_or(f64::NAN) as f32)).collect())
        .unwrap_or_default();
    Sampling {
        max_tokens: payload.get(max_key).and_then(Value::as_u64).unwrap_or(128).max(1) as u32,
        temperature: payload.get("temperature").and_then(Value::as_f64).unwrap_or(1.0) as f32,
        top_k: payload.get("top_k").and_then(Value::as_u64).unwrap_or(0) as u32,
        top_p: payload.get("top_p").and_then(Value::as_f64).unwrap_or(1.0) as f32,
        seed: payload.get("seed").and_then(Value::as_u64).unwrap_or(0),
        stop_ids,
        ignore_eos: false,
        frequency_penalty: payload.get("frequency_penalty").and_then(Value::as_f64).unwrap_or(0.0) as f32,
        presence_penalty: payload.get("presence_penalty").and_then(Value::as_f64).unwrap_or(0.0) as f32,
        logit_bias,
    }
}

fn error_response(e: &EngineError) -> LocalResponse {
    // the shapes of openai_error_response_with_type / queue_error_response (api/openai_util.rs:242-290)
    let (kind, msg) = match e.status() {
        429 => ("rate_limit_exceeded", "Request queue is full".to_string()),
        504 => ("timeout", e.message.clone()),
        400 => ("invalid_request_error", e.message.clone()),
        _ => ("endpoint_request_error", e.message.clone()),
    };
    LocalResponse {
        status: e.status(),
        content_type: "application/json",
        body: LocalBody::Json(json!({"error": {"message": msg, "type": kind, "code": e.status()}})),
    }
}

impl InProcessEndpoint {
    /// `/v1/chat/completions` for a payload already rewritten by `proxy_openai_post`
    /// (model id of the endpoint, `stream_options.include_usage` injected: openai.rs:977-992).
    pub async fn chat_completions(self: Arc<Self>, payload: Value) -> LocalResponse {
        let stream = payload.get("stream").and_then(Value::as_bool).unwrap_or(false);
        let ids = match payload.get("messages").map(|m| self.tokenizer.chat_ids(m)) {
            Some(Ok(ids)) => ids,
            _ => {
                return LocalResponse { status: 400, content_type: "application/json",
                                       body: LocalBody::Json(json!({"error": {"message": "messages is required", "type": "invalid_request_error", "code": 400}})) }
            }
        };
        let sampling = sampling_from(&payload, "max_tokens", self.tokenizer.stop_ids());
        let this = self.clone();
        let model = self.model_id.clone();
        let started = Instant::now();
        if !stream {
            // blocking section is short-polled so that a dropped future cancels the request (RequestGuard)
            let mut guard = match RequestGuard::submit(&this.engine, &ids, &sampling) {
                Ok(g) => g,
                Err(e) => return error_response(&e),
            };
            let mut detok = this.tokenizer.new_stream();
            let (mut text, mut last) = (String::new(), llmlb_token_event::default());
            let mut buf = [llmlb_token_event::default(); 64];
            while !guard.is_finished() {
                match guard.next(&mut buf, Duration::ZERO) {
                    Ok(0) => tokio::time::sleep(Duration::from_micros(200)).await,
                    Ok(n) => {
                        for ev in &buf[..n] {
                            if ev.token_id >= 0 { text.push_str(&detok.next(ev.token_id)); }
                            last = *ev;
                        }
                    }
                    Err(e) => return error_response(&e),
                }
            }
            text.push_str(&detok.flush());
            return match last.finish_reason {
                LLMLB_FINISH_STOP | LLMLB_FINISH_LENGTH => LocalResponse {
                    status: 200,
                    content_type: "application/json",
                    body: LocalBody::Json(json!({
                        "id": format!("chatcmpl-{}", guard.id), "object": "chat.completion", "model": model,
                        "choices": [{"index": 0, "message": {"role": "assistant", "content": text},
                                     "finish_reason": if last.finish_reason == LLMLB_FINISH_STOP { "stop" } else { "length" }}],
                        "usage": {"prompt_tokens": last.prompt_tokens, "completion_tokens": last.completion_tokens,
                                  "total_tokens": last.prompt_tokens + last.completion_tokens}})),
                },
                LLMLB_FINISH_QUEUE_TIMEOUT => error_response(&EngineError { code: llmlb_b200_sys::LLMLB_E_TIMEOUT, message: "Queue wait timeout".into() }),
                LLMLB_FINISH_DEADLINE => error_response(&EngineError { code: llmlb_b200_sys::LLMLB_E_TIMEOUT,
                    message: format!("Upstream endpoint request timed out after {} seconds", started.elapsed().as_secs()) }),
                _ => error_response(&EngineError { code: llmlb_b200_sys::LLMLB_E_INTERNAL, message: "Failed to proxy request to upstream endpoint".into() }),
            };
        }
        // streaming: the same chunks an upstream would send; the relay + accumulator downstream do the accounting
        let body = async_stream::stream! {
            let mut guard = match RequestGuard::submit(&this.engine, &ids, &sampling) {
                Ok(g) => g,
                Err(e) => { yield Err(std::io::Error::new(std::io::ErrorKind::Other, e.to_string())); return; }
            };
            let id = format!("chatcmpl-{}", guard.id);
            let chunk = |delta: Value, finish: Value| Bytes::from(format!("data: {}\n\n", json!({
                "id": id, "object": "chat.completion.chunk", "model": model,
                "choices": [{"index": 0, "delta": delta, "finish_reason": finish}]})));
            yield Ok(chunk(json!({"role": "assistant"}), Value::Null));
            let mut detok = this.tokenizer.new_stream();
            let mut buf = [llmlb_token_event::default(); 64];
            let mut last = llmlb_token_event::default();
            while !guard.is_finished() {
                match guard.next(&mut buf, Duration::ZERO) {
                    Ok(0) => tokio::time::sleep(Duration::from_micros(200)).await,
                    Ok(n) => for ev in &buf[..n] {
                        if ev.token_id >= 0 {
                            let piece = detok.next(ev.token_id);
                            if !piece.is_empty() { yield Ok(chunk(json!({"content": piece}), Value::Null)); }
                        }
                        last = *ev;
                    },
                    Err(e) => { yield Err(std::io::Error::new(std::io::ErrorKind::Other, e.to_string())); return; }
                }
            }
            let rest = detok.flush();
            if !rest.is_empty() { yield Ok(chunk(json!({"content": rest}), Value::Null)); }
            if last.finish_reason == LLMLB_FINISH_STOP || last.finish_reason == LLMLB_FINISH_LENGTH {
                yield Ok(chunk(json!({}), json!(if last.finish_reason == LLMLB_FINISH_STOP { "stop" } else { "length" })));
                yield Ok(Bytes::from(format!("data: {}\n\n", json!({"id": id, "object": "chat.completion.chunk", "model": model, "choices": [],
                    "usage": {"prompt_tokens": last.prompt_tokens, "completion_tokens": last.completion_tokens,
                              "total_tokens": last.prompt_tokens + last.completion_tokens}}))));
                yield Ok(Bytes::from_static(b"data: [DONE]\n\n"));
            }
            // failure mid-stream: the stream ends without [DONE]; the relay counts it as an upstream error
        };
        LocalResponse { status: 200, content_type: "text/event-stream", body: LocalBody::Sse(Box::pin(body)) }
    }

    /// `GET /api/health` numbers for health/endpoint_checker.rs:515-557 without the HTTP round trip.
    pub fn health_json(&self) -> Value {
        match self.engine.health() {
            Ok(h) => json!({"gpu": {"device_count": h.device_count, "total_memory_bytes": h.total_memory_bytes,
                                   "used_memory_bytes": h.used_memory_bytes, "capability_score": 100},
                            "load": {"active_requests": h.active_requests}}),
            Err(_) => json!({}),
        }
    }
}
