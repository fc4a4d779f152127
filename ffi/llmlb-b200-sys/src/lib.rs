//! Bindings for `include/llmlb_b200.h` — the C ABI that replaces the gateway's HTTP hop
//! (`llmlb/src/api/openai.rs:995-1005`, `llmlb/src/api/proxy.rs:372-401`) with an in-process call.
//!
//! Layout is checked against the header by `tools/check_rust_layout.py` (gcc `offsetof` probe);
//! keep field order, types and names in sync with the header.
#![allow(non_camel_case_types)]

use std::ffi::{c_char, c_int, CStr};
use std::time::Duration;

pub const LLMLB_ABI_VERSION: u32 = 1;
pub const LLMLB_IPC_HANDLE_BYTES: usize = 64;
pub const LLMLB_MAX_TOP_LOGPROBS: usize = 20;

pub const LLMLB_OK: c_int = 0;
pub const LLMLB_E_INVALID_ARG: c_int = -1;
pub const LLMLB_E_MODEL_NOT_FOUND: c_int = -2;
pub const LLMLB_E_QUEUE_FULL: c_int = -3;
pub const LLMLB_E_TIMEOUT: c_int = -4;
pub const LLMLB_E_DEVICE: c_int = -5;
pub const LLMLB_E_INTERNAL: c_int = -6;
pub const LLMLB_E_NOT_FOUND: c_int = -7;
pub const LLMLB_E_UNSUPPORTED: c_int = -8;

pub const LLMLB_FINISH_NONE: u32 = 0;
pub const LLMLB_FINISH_STOP: u32 = 1;
pub const LLMLB_FINISH_LENGTH: u32 = 2;
pub const LLMLB_FINISH_CANCELLED: u32 = 3;
pub const LLMLB_FINISH_ERROR: u32 = 4;
pub const LLMLB_FINISH_QUEUE_TIMEOUT: u32 = 5;
pub const LLMLB_FINISH_DEADLINE: u32 = 6;

#[repr(C)]
pub struct llmlb_engine {
    _private: [u8; 0],
}

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct llmlb_model_config {
    pub hidden: u32,
    pub n_layers: u32,
    pub n_heads: u32,
    pub n_kv_heads: u32,
    pub head_dim: u32,
    pub ffn: u32,
    pub vocab: u32,
    pub rope_theta: f32,
    pub rms_eps: f32,
}

#[repr(C)]
#[derive(Clone, Copy)]
pub struct llmlb_engine_config {
    pub abi_version: u32,
    pub model: llmlb_model_config,
    pub model_id: [c_char; 128],
    pub device: i32,
    pub tp_rank: u32,
    pub tp_size: u32,
    pub max_seqs: u32,
    pub max_ctx: u32,
    pub kv_block_tokens: u32,
    pub kv_pages: u32,
    pub max_step_tokens: u32,
    pub synthetic_seed: u64,
    pub use_cuda_graphs: u32,
    pub gemm_impl: u32,
    pub lookahead: u32,
    pub queue_max: u32,
    pub queue_timeout_ms: u32,
    pub request_timeout_ms: u32,
    pub attn_impl: u32,
    pub tp_proto: u32,
    /// automatic prefix caching: 0 = off (the header documents the policy)
    pub prefix_cache: u32,
    pub reserved: [u32; 2],
}

#[repr(C)]
#[derive(Clone, Copy)]
pub struct llmlb_model_info {
    pub id: [c_char; 128],
    pub context_length: u32,
    pub vocab: u32,
    pub n_layers: u32,
    pub hidden: u32,
    pub param_bytes: u64,
}

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct llmlb_health {
    pub device_count: u32,
    pub total_memory_bytes: u64,
    pub used_memory_bytes: u64,
    pub active_requests: u32,
    pub queued_requests: u32,
    pub free_kv_pages: u32,
    pub total_kv_pages: u32,
    pub steps_prefill: u64,
    pub steps_decode: u64,
    pub tokens_prefill: u64,
    pub tokens_decode: u64,
    pub gpu_ms_prefill: f64,
    pub gpu_ms_decode: f64,
    pub kernel_launches: u64,
    pub preemptions: u64,
}

/// Prefix-cache counters (`llmlb_engine_prefix_cache_stats`); all 0 with the cache off.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct llmlb_prefix_cache_stats {
    pub cached_pages: u32,
    pub evictable_pages: u32,
    pub lookups: u64,
    pub hit_tokens: u64,
    pub published_pages: u64,
    pub evicted_pages: u64,
}

#[repr(C)]
#[derive(Clone, Copy)]
pub struct llmlb_sampling {
    pub max_tokens: u32,
    pub temperature: f32,
    pub top_k: u32,
    pub top_p: f32,
    pub seed: u64,
    pub stop_ids: *const i32,
    pub n_stop_ids: u32,
    pub ignore_eos: u32,
}

/// OpenAI's frequency_penalty, presence_penalty and logit_bias (`llmlb_request_submit_penalized`).
#[repr(C)]
#[derive(Clone, Copy)]
pub struct llmlb_penalties {
    pub frequency_penalty: f32,
    pub presence_penalty: f32,
    pub bias_ids: *const i32,
    pub bias_values: *const f32,
    pub n_bias: u32,
}

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct llmlb_token_event {
    pub token_id: i32,
    pub index: u32,
    pub finish_reason: u32,
    pub prompt_tokens: u32,
    pub completion_tokens: u32,
    pub t_ms: f64,
}

/// Logprobs of one token event (`llmlb_request_poll_logprobs`): log_softmax of the row the sampler read.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct llmlb_token_logprobs {
    pub logprob: f32,
    pub n_top: u32,
    pub top_ids: [i32; 20],
    pub top_logprobs: [f32; 20],
}

extern "C" {
    pub fn llmlb_abi_version() -> u32;
    pub fn llmlb_last_error() -> *const c_char;
    pub fn llmlb_engine_create(cfg: *const llmlb_engine_config, out: *mut *mut llmlb_engine) -> c_int;
    pub fn llmlb_engine_destroy(e: *mut llmlb_engine);
    pub fn llmlb_engine_model_info(e: *const llmlb_engine, out: *mut llmlb_model_info) -> c_int;
    pub fn llmlb_engine_health(e: *const llmlb_engine, out: *mut llmlb_health) -> c_int;
    pub fn llmlb_engine_prefix_cache_stats(e: *const llmlb_engine, out: *mut llmlb_prefix_cache_stats) -> c_int;
    pub fn llmlb_engine_load_tensor(e: *mut llmlb_engine, name: *const c_char, host_bf16: *const u8, rows: u64, cols: u64) -> c_int;
    pub fn llmlb_engine_set_rope_freq_factors(e: *mut llmlb_engine, factors: *const f32, n: u32) -> c_int;
    pub fn llmlb_engine_tp_export(e: *mut llmlb_engine, handle: *mut u8) -> c_int;
    pub fn llmlb_engine_tp_import(e: *mut llmlb_engine, handles: *const u8, n: u32) -> c_int;
    pub fn llmlb_engine_tp_plan_channel(e: *mut llmlb_engine, shm_name: *const c_char) -> c_int;
    pub fn llmlb_engine_pause(e: *mut llmlb_engine, paused: u32) -> c_int;
    pub fn llmlb_request_submit(e: *mut llmlb_engine, prompt_ids: *const i32, n_prompt: u32, s: *const llmlb_sampling, req_id: *mut u64) -> c_int;
    pub fn llmlb_request_submit_penalized(e: *mut llmlb_engine, prompt_ids: *const i32, n_prompt: u32, s: *const llmlb_sampling, pen: *const llmlb_penalties, req_id: *mut u64) -> c_int;
    pub fn llmlb_request_submit_logprobs(e: *mut llmlb_engine, prompt_ids: *const i32, n_prompt: u32, s: *const llmlb_sampling, pen: *const llmlb_penalties, top_logprobs: u32, req_id: *mut u64) -> c_int;
    pub fn llmlb_request_poll(e: *mut llmlb_engine, req_id: u64, out: *mut llmlb_token_event, cap: u32, n_out: *mut u32, timeout_ms: c_int) -> c_int;
    pub fn llmlb_request_poll_logprobs(e: *mut llmlb_engine, req_id: u64, out: *mut llmlb_token_event, lp: *mut llmlb_token_logprobs, cap: u32, n_out: *mut u32, timeout_ms: c_int) -> c_int;
    pub fn llmlb_request_submit_prompt_logprobs(e: *mut llmlb_engine, prompt_ids: *const i32, n_prompt: u32, s: *const llmlb_sampling, pen: *const llmlb_penalties, top_logprobs: u32, req_id: *mut u64) -> c_int;
    pub fn llmlb_request_poll_prompt_logprobs(e: *mut llmlb_engine, req_id: u64, out: *mut llmlb_token_logprobs, cap: u32, n_out: *mut u32) -> c_int;
    pub fn llmlb_request_cached_tokens(e: *mut llmlb_engine, req_id: u64, n: *mut u32) -> c_int;
    pub fn llmlb_request_submit_choices(e: *mut llmlb_engine, prompt_ids: *const i32, n_prompt: u32, s: *const llmlb_sampling, pen: *const llmlb_penalties, top_logprobs: i32, prompt_logprobs: u32, n: u32, req_ids: *mut u64) -> c_int;
    pub fn llmlb_request_cancel(e: *mut llmlb_engine, req_id: u64) -> c_int;
    pub fn llmlb_request_release(e: *mut llmlb_engine, req_id: u64) -> c_int;
}

/// The gateway's error type for this boundary; `status()` is the mapping of `llmlb/src/api/error.rs:31-110`
/// the header documents (E_INVALID_ARG→400, E_MODEL_NOT_FOUND→404, E_QUEUE_FULL→429, E_TIMEOUT→504, else 502).
#[derive(Debug, Clone)]
pub struct EngineError {
    pub code: c_int,
    pub message: String,
}

impl EngineError {
    fn last(code: c_int) -> Self {
        let message = unsafe {
            let p = llmlb_last_error();
            if p.is_null() { String::new() } else { CStr::from_ptr(p).to_string_lossy().into_owned() }
        };
        Self { code, message }
    }
    pub fn status(&self) -> u16 {
        match self.code {
            LLMLB_E_INVALID_ARG => 400,
            LLMLB_E_MODEL_NOT_FOUND => 404,
            LLMLB_E_QUEUE_FULL => 429,
            LLMLB_E_TIMEOUT => 504,
            _ => 502,
        }
    }
}

impl std::fmt::Display for EngineError {
    fn fmt(&self, f: &mut std::fmt::Formatter<'_>) -> std::fmt::Result {
        write!(f, "llmlb_b200 error {}: {}", self.code, self.message)
    }
}
impl std::error::Error for EngineError {}

fn check(rc: c_int) -> Result<(), EngineError> {
    if rc == LLMLB_OK { Ok(()) } else { Err(EngineError::last(rc)) }
}

/// Owner of an `llmlb_engine*`.  Every method is a thin call into the C ABI; all of them are
/// thread-safe on the C side and `submit` / `poll(Duration::ZERO)` / `cancel` never block on the GPU,
/// so they may be called from tokio workers without `spawn_blocking` (`llmlb/src/main.rs:64,131`).
pub struct Engine {
    raw: *mut llmlb_engine,
}

// the C library serialises internally (one scheduler thread, mutex-protected queues)
unsafe impl Send for Engine {}
unsafe impl Sync for Engine {}

#[derive(Clone, Debug)]
pub struct Sampling {
    pub max_tokens: u32,
    pub temperature: f32,
    pub top_k: u32,
    pub top_p: f32,
    pub seed: u64,
    pub stop_ids: Vec<i32>,
    pub ignore_eos: bool,
    /// OpenAI penalties, applied on the device before sampling; both 0 and no bias: not penalised
    pub frequency_penalty: f32,
    pub presence_penalty: f32,
    pub logit_bias: Vec<(i32, f32)>,
}

impl Default for Sampling {
    fn default() -> Self {
        Self { max_tokens: 128, temperature: 1.0, top_k: 0, top_p: 1.0, seed: 0, stop_ids: Vec::new(), ignore_eos: false,
               frequency_penalty: 0.0, presence_penalty: 0.0, logit_bias: Vec::new() }
    }
}

impl Engine {
    pub fn new(mut cfg: llmlb_engine_config) -> Result<Self, EngineError> {
        cfg.abi_version = LLMLB_ABI_VERSION;
        let mut raw: *mut llmlb_engine = std::ptr::null_mut();
        check(unsafe { llmlb_engine_create(&cfg, &mut raw) })?;
        Ok(Self { raw })
    }

    /// Llama-3-8B geometry with the gateway's own queue limits (`llmlb/src/config.rs:80-99`) and
    /// per-request timeout (`llmlb/src/types/endpoint.rs:389`).
    pub fn llama3_8b_config(model_id: &str, device: i32) -> llmlb_engine_config {
        let mut id = [0 as c_char; 128];
        for (dst, src) in id.iter_mut().zip(model_id.bytes().take(127)) {
            *dst = src as c_char;
        }
        llmlb_engine_config {
            abi_version: LLMLB_ABI_VERSION,
            model: llmlb_model_config { hidden: 4096, n_layers: 32, n_heads: 32, n_kv_heads: 8, head_dim: 128, ffn: 14336, vocab: 128256, rope_theta: 500000.0, rms_eps: 1e-5 },
            model_id: id,
            device,
            tp_rank: 0,
            tp_size: 1,
            max_seqs: 64,
            max_ctx: 8192,
            kv_block_tokens: 64,
            kv_pages: 0,
            max_step_tokens: 0,
            synthetic_seed: 0,
            use_cuda_graphs: 1,
            gemm_impl: 0,
            lookahead: 0,
            queue_max: 100,
            queue_timeout_ms: 60_000,
            request_timeout_ms: 120_000,
            attn_impl: 0,
            tp_proto: 0,
            prefix_cache: 0,
            reserved: [0; 2],
        }
    }

    /// RoPE frequency scaling (llama3 / linear): 64 per-frequency divisors, before the first request.
    pub fn set_rope_freq_factors(&self, factors: &[f32]) -> Result<(), EngineError> {
        check(unsafe { llmlb_engine_set_rope_freq_factors(self.raw, factors.as_ptr(), factors.len() as u32) })
    }

    pub fn submit(&self, prompt_ids: &[i32], s: &Sampling) -> Result<u64, EngineError> {
        let raw_s = llmlb_sampling {
            max_tokens: s.max_tokens,
            temperature: s.temperature,
            top_k: s.top_k,
            top_p: s.top_p,
            seed: s.seed,
            stop_ids: if s.stop_ids.is_empty() { std::ptr::null() } else { s.stop_ids.as_ptr() },
            n_stop_ids: s.stop_ids.len() as u32,
            ignore_eos: s.ignore_eos as u32,
        };
        let mut id = 0u64;
        if s.frequency_penalty == 0.0 && s.presence_penalty == 0.0 && s.logit_bias.is_empty() {
            check(unsafe { llmlb_request_submit(self.raw, prompt_ids.as_ptr(), prompt_ids.len() as u32, &raw_s, &mut id) })?;
            return Ok(id);
        }
        let ids: Vec<i32> = s.logit_bias.iter().map(|b| b.0).collect();
        let vals: Vec<f32> = s.logit_bias.iter().map(|b| b.1).collect();
        let pen = llmlb_penalties {
            frequency_penalty: s.frequency_penalty,
            presence_penalty: s.presence_penalty,
            bias_ids: if ids.is_empty() { std::ptr::null() } else { ids.as_ptr() },
            bias_values: if vals.is_empty() { std::ptr::null() } else { vals.as_ptr() },
            n_bias: ids.len() as u32,
        };
        check(unsafe { llmlb_request_submit_penalized(self.raw, prompt_ids.as_ptr(), prompt_ids.len() as u32, &raw_s, &pen, &mut id) })?;
        Ok(id)
    }

    /// OpenAI's `n`: `n` choices of one prompt, prefilled once; returns their ids, choice `i` sampling with `seed + i`.
    /// `top_logprobs`: `None` = no logprobs, `Some(0..=20)` alternatives per token (read with `llmlb_request_poll_logprobs`);
    /// `prompt_logprobs` (with `top_logprobs`): the prompt's records too, delivered to every choice.
    pub fn submit_choices(&self, prompt_ids: &[i32], s: &Sampling, n: u32, top_logprobs: Option<u32>, prompt_logprobs: bool)
        -> Result<Vec<u64>, EngineError> {
        let raw_s = llmlb_sampling {
            max_tokens: s.max_tokens,
            temperature: s.temperature,
            top_k: s.top_k,
            top_p: s.top_p,
            seed: s.seed,
            stop_ids: if s.stop_ids.is_empty() { std::ptr::null() } else { s.stop_ids.as_ptr() },
            n_stop_ids: s.stop_ids.len() as u32,
            ignore_eos: s.ignore_eos as u32,
        };
        let ids: Vec<i32> = s.logit_bias.iter().map(|b| b.0).collect();
        let vals: Vec<f32> = s.logit_bias.iter().map(|b| b.1).collect();
        let pen = llmlb_penalties {
            frequency_penalty: s.frequency_penalty,
            presence_penalty: s.presence_penalty,
            bias_ids: if ids.is_empty() { std::ptr::null() } else { ids.as_ptr() },
            bias_values: if vals.is_empty() { std::ptr::null() } else { vals.as_ptr() },
            n_bias: ids.len() as u32,
        };
        let neutral = s.frequency_penalty == 0.0 && s.presence_penalty == 0.0 && s.logit_bias.is_empty();
        let mut out = vec![0u64; n.max(1) as usize];
        check(unsafe {
            llmlb_request_submit_choices(self.raw, prompt_ids.as_ptr(), prompt_ids.len() as u32, &raw_s,
                                         if neutral { std::ptr::null() } else { &pen }, top_logprobs.map_or(-1, |t| t as i32),
                                         prompt_logprobs as u32, n, out.as_mut_ptr())
        })?;
        out.truncate(n as usize);
        Ok(out)
    }

    /// Drains up to `buf.len()` events; `timeout` zero returns at once.  `Ok(0)` on timeout.
    pub fn poll(&self, req_id: u64, buf: &mut [llmlb_token_event], timeout: Duration) -> Result<usize, EngineError> {
        let mut n = 0u32;
        let rc = unsafe { llmlb_request_poll(self.raw, req_id, buf.as_mut_ptr(), buf.len() as u32, &mut n, timeout.as_millis() as c_int) };
        if rc == LLMLB_E_TIMEOUT {
            return Ok(0);
        }
        check(rc)?;
        Ok(n as usize)
    }

    pub fn cancel(&self, req_id: u64) -> Result<(), EngineError> {
        check(unsafe { llmlb_request_cancel(self.raw, req_id) })
    }

    pub fn release(&self, req_id: u64) -> Result<(), EngineError> {
        check(unsafe { llmlb_request_release(self.raw, req_id) })
    }

    pub fn health(&self) -> Result<llmlb_health, EngineError> {
        let mut h = llmlb_health::default();
        check(unsafe { llmlb_engine_health(self.raw, &mut h) })?;
        Ok(h)
    }

    /// Prefix-cache counters (all 0 with `prefix_cache` off).
    pub fn prefix_cache_stats(&self) -> Result<llmlb_prefix_cache_stats, EngineError> {
        let mut st = llmlb_prefix_cache_stats::default();
        check(unsafe { llmlb_engine_prefix_cache_stats(self.raw, &mut st) })?;
        Ok(st)
    }

    /// OpenAI's `usage.prompt_tokens_details.cached_tokens` of a request.
    pub fn cached_tokens(&self, req_id: u64) -> Result<u32, EngineError> {
        let mut n = 0u32;
        check(unsafe { llmlb_request_cached_tokens(self.raw, req_id, &mut n) })?;
        Ok(n)
    }

    pub fn model_info(&self) -> Result<llmlb_model_info, EngineError> {
        let mut m: llmlb_model_info = unsafe { std::mem::zeroed() };
        check(unsafe { llmlb_engine_model_info(self.raw, &mut m) })?;
        Ok(m)
    }
}

impl Drop for Engine {
    fn drop(&mut self) {
        unsafe { llmlb_engine_destroy(self.raw) }
    }
}

/// A request whose engine-side state is cancelled and released when the guard is dropped — the
/// boundary-side twin of `RequestLease` (`llmlb/src/balancer/lease.rs:71-100`): a handler that
/// returns early (client disconnect, drain abort `inference_gate.rs:73-76`) leaks nothing.
pub struct RequestGuard<'a> {
    engine: &'a Engine,
    pub id: u64,
    finished: bool,
}

impl<'a> RequestGuard<'a> {
    pub fn submit(engine: &'a Engine, prompt_ids: &[i32], s: &Sampling) -> Result<Self, EngineError> {
        Ok(Self { engine, id: engine.submit(prompt_ids, s)?, finished: false })
    }
    /// Next batch of events; marks the request finished when the last one carries a finish reason.
    pub fn next(&mut self, buf: &mut [llmlb_token_event], timeout: Duration) -> Result<usize, EngineError> {
        let n = self.engine.poll(self.id, buf, timeout)?;
        if n > 0 && buf[n - 1].finish_reason != LLMLB_FINISH_NONE {
            self.finished = true;
        }
        Ok(n)
    }
    pub fn is_finished(&self) -> bool {
        self.finished
    }
}

impl Drop for RequestGuard<'_> {
    fn drop(&mut self) {
        if !self.finished {
            let _ = self.engine.cancel(self.id);
        }
        let _ = self.engine.release(self.id);
    }
}
