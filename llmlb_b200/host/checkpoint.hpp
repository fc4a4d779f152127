// Native checkpoint readers for the HTTP shim (SURVEY.md §8f.4): safetensors and GGUF files are
// memory-mapped, every tensor is delivered as row-major bf16 under its Hugging Face Llama name —
// exactly what llmlb_engine_load_tensor (include/llmlb_b200.h) takes.  GGUF blocks (Q8_0, Q4_0,
// Q4_1, Q5_0, Q5_1, Q4_K, Q5_K, Q6_K, F16, F32, BF16) are dequantised on load; llama.cpp tensor
// names are mapped and the converter's Q/K rotary row permutation is undone.  The C++ mirrors
// llmlb_b200/gguf.py + weights.py (which are pinned to llama.cpp's `gguf` package) and is compared
// with them bit for bit in tests/test_host_checkpoint.py.
#pragma once
#include <cstdint>
#include <functional>
#include <map>
#include <string>
#include <vector>

namespace llmlb_host {

struct CkptTensor {
  std::string name;                 // Hugging Face name ("model.layers.3.mlp.up_proj.weight")
  uint64_t rows = 0, cols = 0;
  // source description
  std::string src_name;             // name inside the file
  uint32_t dtype = 0;               // safetensors: 0 F32, 1 F16, 30 BF16 (ggml numbering); GGUF: ggml type id
  uint64_t offset = 0, nbytes = 0;  // absolute file offset
  uint32_t unpermute_heads = 0;     // GGUF Q/K: number of heads to un-permute, 0 = none
};

struct CkptGeometry {               // the fields of llmlb_model_config, when the file knows them
  bool known = false;
  uint32_t hidden = 0, n_layers = 0, n_heads = 0, n_kv_heads = 0, head_dim = 0, ffn = 0, vocab = 0;
  float rope_theta = 10000.f, rms_eps = 1e-5f;
  // RoPE frequency scaling as fixed per-frequency divisors (inv_freq[j] = theta^(-2j/hd) / f[j]).
  // rope_known: the file states theta, eps and the scaling (GGUF metadata, or a config.json beside a
  // safetensors file); a safetensors file without one has no say.  rope_scaling: "none", "llama3",
  // "linear" or "rope_freqs" (a GGUF per-frequency tensor); rope_freq_factors: head_dim/2 values, empty = none.
  bool rope_known = false;
  std::string rope_scaling = "none";
  std::vector<float> rope_freq_factors;
};

// The divisors of a llama3 or linear `rope_scaling` (rope_type / type, factor, ...; transformers'
// _compute_llama3_parameters / _compute_linear_scaling_rope_parameters), computed in fp64.  "default" or
// "none" give no factors.  Any other type (dynamic, yarn, longrope: tables that depend on the sequence
// length or scale attention) is refused: false + *err.
bool rope_scaling_factors(const std::string& type, double factor, double low_freq_factor, double high_freq_factor,
                          double original_ctx, double theta, uint32_t head_dim, std::vector<float>* out, std::string* err);

class Checkpoint {
 public:
  ~Checkpoint();
  // Opens a .safetensors or .gguf file (by magic, not by extension).  false + *err on failure.
  bool open(const std::string& path, std::string* err);
  const std::vector<CkptTensor>& tensors() const { return tensors_; }
  const CkptGeometry& geometry() const { return geo_; }
  bool is_gguf() const { return gguf_; }
  // bf16 bit patterns of tensor i, row-major [rows, cols] (converted / dequantised / un-permuted)
  bool read_bf16(size_t i, std::vector<uint16_t>* out, std::string* err) const;
  // GGUF only: tokenizer.json text rebuilt from tokenizer.ggml.* ("" when the file carries none)
  std::string tokenizer_json() const;
  // A tied output head: GGUF files without output.weight serve lm_head from the embedding
  bool tied_lm_head() const { return tied_lm_head_; }

 private:
  bool open_safetensors(std::string* err);
  bool read_config_json(int64_t max_layer, std::string* err);   // safetensors: config.json beside the file, if any
  bool open_gguf(std::string* err);
  std::string path_;
  const uint8_t* data_ = nullptr;
  size_t size_ = 0;
  bool gguf_ = false, tied_lm_head_ = false;
  std::vector<CkptTensor> tensors_;
  CkptGeometry geo_;
  // GGUF tokenizer metadata
  std::string tok_model_, tok_pre_;
  std::vector<std::string> tok_tokens_, tok_merges_;
  std::vector<int32_t> tok_types_;
  int64_t tok_bos_ = -1;
};

// float32 -> bf16 bits, round to nearest even (NaN kept quiet)
uint16_t f32_to_bf16_bits(float x);
// dequantise `n` elements of ggml type `type` from `src` into `dst` (float32); false if unsupported
bool ggml_dequantize(uint32_t type, const uint8_t* src, size_t nbytes, float* dst, size_t n);

}  // namespace llmlb_host
