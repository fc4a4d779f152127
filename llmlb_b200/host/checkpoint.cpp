// See checkpoint.hpp.  Block layouts are ggml's (ggml-common.h): Q4_0 {f16 d; u8 qs[16]},
// Q4_1 {f16 d, m; qs[16]}, Q5_0 {f16 d; u8 qh[4]; qs[16]}, Q5_1 {f16 d, m; qh[4]; qs[16]},
// Q8_0 {f16 d; i8 qs[32]}, Q4_K {f16 d, dmin; u8 scales[12]; qs[128]},
// Q5_K {f16 d, dmin; scales[12]; qh[32]; qs[128]}, Q6_K {u8 ql[128]; qh[64]; i8 scales[16]; f16 d}.
#include "checkpoint.hpp"

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cmath>
#include <cstring>
#include <fstream>
#include <sstream>

#include "json.hpp"

namespace llmlb_host {

namespace {

constexpr uint32_t kF32 = 0, kF16 = 1, kQ4_0 = 2, kQ4_1 = 3, kQ5_0 = 6, kQ5_1 = 7, kQ8_0 = 8, kQ4_K = 12, kQ5_K = 13,
                   kQ6_K = 14, kBF16 = 30;

bool block_shape(uint32_t type, uint32_t* per, uint32_t* bytes) {
  switch (type) {
    case kF32: *per = 1; *bytes = 4; return true;
    case kF16: case kBF16: *per = 1; *bytes = 2; return true;
    case kQ4_0: *per = 32; *bytes = 18; return true;
    case kQ4_1: *per = 32; *bytes = 20; return true;
    case kQ5_0: *per = 32; *bytes = 22; return true;
    case kQ5_1: *per = 32; *bytes = 24; return true;
    case kQ8_0: *per = 32; *bytes = 34; return true;
    case kQ4_K: *per = 256; *bytes = 144; return true;
    case kQ5_K: *per = 256; *bytes = 176; return true;
    case kQ6_K: *per = 256; *bytes = 210; return true;
  }
  return false;
}

float f16_to_f32(uint16_t h) {
  const uint32_t sign = uint32_t(h & 0x8000u) << 16;
  uint32_t exp = (h >> 10) & 0x1Fu, man = h & 0x3FFu, bits;
  if (exp == 0) {
    if (man == 0) bits = sign;
    else {  // subnormal: renormalise
      int shift = 0;
      while (!(man & 0x400u)) { man <<= 1; ++shift; }
      man &= 0x3FFu;
      bits = sign | ((113u - uint32_t(shift)) << 23) | (man << 13);
    }
  } else if (exp == 31) bits = sign | 0x7F800000u | (man << 13);
  else bits = sign | ((exp + 112u) << 23) | (man << 13);
  float f;
  memcpy(&f, &bits, 4);
  return f;
}
inline float rd_f16(const uint8_t* p) { uint16_t h; memcpy(&h, p, 2); return f16_to_f32(h); }

// 12-byte scale field of Q4_K / Q5_K: sub-block j -> (6-bit scale, 6-bit minimum)
inline void k_scale_min(const uint8_t* q, int j, uint8_t* sc, uint8_t* mn) {
  if (j < 4) { *sc = q[j] & 63; *mn = q[j + 4] & 63; }
  else { *sc = uint8_t((q[j + 4] & 0x0F) | ((q[j - 4] >> 6) << 4)); *mn = uint8_t((q[j + 4] >> 4) | ((q[j] >> 6) << 4)); }
}

void deq_block(uint32_t type, const uint8_t* b, float* y) {
  switch (type) {
    case kQ8_0: {
      const float d = rd_f16(b);
      for (int i = 0; i < 32; ++i) y[i] = d * float(int8_t(b[2 + i]));
      break;
    }
    case kQ4_0: {
      const float d = rd_f16(b);
      for (int i = 0; i < 16; ++i) {
        y[i] = d * float(int8_t(int(b[2 + i] & 15) - 8));
        y[i + 16] = d * float(int8_t(int(b[2 + i] >> 4) - 8));
      }
      break;
    }
    case kQ4_1: {
      const float d = rd_f16(b), m = rd_f16(b + 2);
      for (int i = 0; i < 16; ++i) {
        y[i] = d * float(b[4 + i] & 15) + m;
        y[i + 16] = d * float(b[4 + i] >> 4) + m;
      }
      break;
    }
    case kQ5_0: {
      const float d = rd_f16(b);
      uint32_t qh;
      memcpy(&qh, b + 2, 4);
      for (int i = 0; i < 16; ++i) {
        const int lo = (b[6 + i] & 15) | int(((qh >> i) & 1u) << 4);
        const int hi = (b[6 + i] >> 4) | int(((qh >> (i + 16)) & 1u) << 4);
        y[i] = d * float(lo - 16);
        y[i + 16] = d * float(hi - 16);
      }
      break;
    }
    case kQ5_1: {
      const float d = rd_f16(b), m = rd_f16(b + 2);
      uint32_t qh;
      memcpy(&qh, b + 4, 4);
      for (int i = 0; i < 16; ++i) {
        const int lo = (b[8 + i] & 15) | int(((qh >> i) & 1u) << 4);
        const int hi = (b[8 + i] >> 4) | int(((qh >> (i + 16)) & 1u) << 4);
        y[i] = d * float(lo) + m;
        y[i + 16] = d * float(hi) + m;
      }
      break;
    }
    case kQ4_K: {
      const float d = rd_f16(b), dmin = rd_f16(b + 2);
      const uint8_t* sc12 = b + 4;
      const uint8_t* qs = b + 16;
      for (int g = 0; g < 4; ++g) {   // 64 elements per group: low nibbles sub-block 2g, high nibbles 2g+1
        uint8_t s0, m0, s1, m1;
        k_scale_min(sc12, 2 * g, &s0, &m0);
        k_scale_min(sc12, 2 * g + 1, &s1, &m1);
        const float d0 = d * float(s0), n0 = dmin * float(m0), d1 = d * float(s1), n1 = dmin * float(m1);
        for (int l = 0; l < 32; ++l) {
          y[g * 64 + l] = d0 * float(qs[g * 32 + l] & 15) - n0;
          y[g * 64 + 32 + l] = d1 * float(qs[g * 32 + l] >> 4) - n1;
        }
      }
      break;
    }
    case kQ5_K: {
      const float d = rd_f16(b), dmin = rd_f16(b + 2);
      const uint8_t* sc12 = b + 4;
      const uint8_t* qh = b + 16;
      const uint8_t* qs = b + 48;
      for (int g = 0; g < 4; ++g) {
        uint8_t s0, m0, s1, m1;
        k_scale_min(sc12, 2 * g, &s0, &m0);
        k_scale_min(sc12, 2 * g + 1, &s1, &m1);
        const float d0 = d * float(s0), n0 = dmin * float(m0), d1 = d * float(s1), n1 = dmin * float(m1);
        for (int l = 0; l < 32; ++l) {
          const int lo = (qs[g * 32 + l] & 15) | (((qh[l] >> (2 * g)) & 1) << 4);
          const int hi = (qs[g * 32 + l] >> 4) | (((qh[l] >> (2 * g + 1)) & 1) << 4);
          y[g * 64 + l] = d0 * float(lo) - n0;
          y[g * 64 + 32 + l] = d1 * float(hi) - n1;
        }
      }
      break;
    }
    case kQ6_K: {
      const uint8_t* ql = b;
      const uint8_t* qh = b + 128;
      const int8_t* sc = reinterpret_cast<const int8_t*>(b + 192);
      const float d = rd_f16(b + 208);
      for (int half = 0; half < 2; ++half) {
        for (int l = 0; l < 32; ++l) {
          const int is = l / 16;
          const int q1 = int((ql[l] & 15) | (((qh[l] >> 0) & 3) << 4)) - 32;
          const int q2 = int((ql[l + 32] & 15) | (((qh[l] >> 2) & 3) << 4)) - 32;
          const int q3 = int((ql[l] >> 4) | (((qh[l] >> 4) & 3) << 4)) - 32;
          const int q4 = int((ql[l + 32] >> 4) | (((qh[l] >> 6) & 3) << 4)) - 32;
          y[l] = (d * float(sc[is])) * float(q1);
          y[l + 32] = (d * float(sc[is + 2])) * float(q2);
          y[l + 64] = (d * float(sc[is + 4])) * float(q3);
          y[l + 96] = (d * float(sc[is + 6])) * float(q4);
        }
        y += 128; ql += 64; qh += 32; sc += 8;
      }
      break;
    }
  }
}

struct Cur {   // bounds-checked little-endian reader over the mapped file
  const uint8_t* p; const uint8_t* end; bool ok = true;
  template <typename T> T take() { T v{}; if (size_t(end - p) < sizeof(T)) { ok = false; p = end; return v; } memcpy(&v, p, sizeof(T)); p += sizeof(T); return v; }
  std::string str() { const uint64_t n = take<uint64_t>(); if (!ok || uint64_t(end - p) < n) { ok = false; return ""; } std::string s(reinterpret_cast<const char*>(p), size_t(n)); p += n; return s; }
  void skip(uint64_t n) { if (uint64_t(end - p) < n) { ok = false; p = end; } else p += n; }
};
// arithmetic on numbers that come out of a file: products that wrap and doubles outside the target range are
// errors, not values (found by tools/fuzz: a zero `general.alignment`, zero-sized dims, 2^63-element shapes)
inline bool mul_ok(uint64_t a, uint64_t b, uint64_t* out) { return !__builtin_mul_overflow(a, b, out); }
inline uint32_t u32_of(double v) { return (v >= 0.0 && v <= 4294967295.0) ? uint32_t(v) : 0u; }
inline int64_t i64_of(double v, int64_t dflt) { return (v >= -9.0e18 && v <= 9.0e18) ? int64_t(v) : dflt; }
constexpr int64_t kMaxLayers = 4096;

size_t scalar_size(uint32_t t) {
  switch (t) { case 0: case 1: case 7: return 1; case 2: case 3: return 2; case 4: case 5: case 6: return 4; case 10: case 11: case 12: return 8; }
  return 0;
}

const char* kLayerMap[][2] = {{"attn_norm", "input_layernorm"}, {"attn_q", "self_attn.q_proj"}, {"attn_k", "self_attn.k_proj"},
                              {"attn_v", "self_attn.v_proj"}, {"attn_output", "self_attn.o_proj"}, {"ffn_norm", "post_attention_layernorm"},
                              {"ffn_gate", "mlp.gate_proj"}, {"ffn_up", "mlp.up_proj"}, {"ffn_down", "mlp.down_proj"}};

std::string hf_name(const std::string& g) {
  if (g == "token_embd.weight") return "model.embed_tokens.weight";
  if (g == "output_norm.weight") return "model.norm.weight";
  if (g == "output.weight") return "lm_head.weight";
  if (g.compare(0, 4, "blk.") != 0) return "";
  const size_t d1 = g.find('.', 4);
  if (d1 == std::string::npos || d1 == 4) return "";
  for (size_t i = 4; i < d1; ++i) if (g[i] < '0' || g[i] > '9') return "";
  const size_t d2 = g.find('.', d1 + 1);
  if (d2 == std::string::npos || g.substr(d2) != ".weight") return "";
  const std::string mid = g.substr(d1 + 1, d2 - d1 - 1);
  for (auto& m : kLayerMap)
    if (mid == m[0]) return "model.layers." + g.substr(4, d1 - 4) + "." + m[1] + ".weight";
  return "";
}

}  // namespace

uint16_t f32_to_bf16_bits(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  if ((u & 0x7FFFFFFFu) > 0x7F800000u) return uint16_t((u >> 16) | 0x40u);
  return uint16_t((u + 0x7FFFu + ((u >> 16) & 1u)) >> 16);
}

bool ggml_dequantize(uint32_t type, const uint8_t* src, size_t nbytes, float* dst, size_t n) {
  uint32_t per = 0, bsz = 0;
  if (!block_shape(type, &per, &bsz) || n % per || nbytes != n / per * bsz) return false;
  if (type == kF32) { memcpy(dst, src, n * 4); return true; }
  if (type == kF16) { for (size_t i = 0; i < n; ++i) dst[i] = rd_f16(src + 2 * i); return true; }
  if (type == kBF16) { for (size_t i = 0; i < n; ++i) { uint16_t h; memcpy(&h, src + 2 * i, 2); uint32_t u = uint32_t(h) << 16; memcpy(dst + i, &u, 4); } return true; }
  for (size_t blk = 0; blk < n / per; ++blk) deq_block(type, src + blk * bsz, dst + blk * per);
  return true;
}

bool rope_scaling_factors(const std::string& type, double factor, double low, double high, double old_ctx, double theta,
                          uint32_t head_dim, std::vector<float>* out, std::string* err) {
  out->clear();
  if (type.empty() || type == "default" || type == "none") return true;
  const uint32_t n = head_dim / 2;
  if (type != "llama3" && type != "linear") {
    if (err) *err = "unsupported RoPE scaling type '" + type + "': only llama3 and linear are served (dynamic, yarn and longrope "
                    "depend on the sequence length or scale attention)";
    return false;
  }
  if (!(factor > 0.0) || !std::isfinite(factor)) { if (err) *err = "RoPE scaling: factor must be finite and > 0"; return false; }
  if (type == "linear") { out->assign(n, float(factor)); return true; }
  if (!(low > 0.0) || !(high > low) || !std::isfinite(high) || !(old_ctx > 0.0) || !std::isfinite(old_ctx) || !(theta > 1.0)) {
    if (err) *err = "RoPE scaling llama3: needs low_freq_factor > 0, high_freq_factor > low_freq_factor, original_max_position_embeddings > 0";
    return false;
  }
  const double pi = 3.14159265358979323846;
  for (uint32_t j = 0; j < n; ++j) {
    const double inv = 1.0 / std::pow(theta, double(2 * j) / double(head_dim));
    const double wavelen = 2 * pi / inv;
    double f;
    if (wavelen < old_ctx / high) f = 1.0;                 // high frequencies: unchanged
    else if (wavelen > old_ctx / low) f = factor;          // low frequencies: divided by `factor`
    else {                                                 // medium: interpolated
      const double smooth = (old_ctx / wavelen - low) / (high - low);
      f = 1.0 / ((1 - smooth) / factor + smooth);
    }
    out->push_back(float(f));
  }
  return true;
}

Checkpoint::~Checkpoint() { if (data_) munmap(const_cast<uint8_t*>(data_), size_); }

bool Checkpoint::open(const std::string& path, std::string* err) {
  const int fd = ::open(path.c_str(), O_RDONLY);
  struct stat sb;
  if (fd < 0 || fstat(fd, &sb) != 0 || sb.st_size < 16) { if (fd >= 0) close(fd); if (err) *err = "cannot read " + path; return false; }
  size_ = size_t(sb.st_size);
  void* p = mmap(nullptr, size_, PROT_READ, MAP_PRIVATE, fd, 0);
  close(fd);
  if (p == MAP_FAILED) { if (err) *err = "mmap failed for " + path; return false; }
  data_ = static_cast<const uint8_t*>(p);
  path_ = path;
  gguf_ = memcmp(data_, "GGUF", 4) == 0;
  return gguf_ ? open_gguf(err) : open_safetensors(err);
}

bool Checkpoint::open_safetensors(std::string* err) {
  uint64_t hlen;
  memcpy(&hlen, data_, 8);
  if (hlen > size_ - 8) { if (err) *err = "safetensors: header length past the end of the file"; return false; }
  Json hdr;
  if (!Json::parse(std::string(reinterpret_cast<const char*>(data_ + 8), size_t(hlen)), &hdr) || !hdr.is_object()) { if (err) *err = "safetensors: header is not JSON"; return false; }
  const uint64_t base = 8 + hlen;
  int64_t max_layer = -1;
  for (const auto& kv : hdr.members()) {
    if (kv.first == "__metadata__") continue;
    const Json* dt = kv.second.get("dtype");
    const Json* sh = kv.second.get("shape");
    const Json* off = kv.second.get("data_offsets");
    if (!dt || !dt->is_string() || !sh || !sh->is_array() || !off || !off->is_array() || off->items().size() != 2) { if (err) *err = "safetensors: malformed entry " + kv.first; return false; }
    CkptTensor t;
    t.name = t.src_name = kv.first;
    if (dt->str() == "F32") t.dtype = kF32; else if (dt->str() == "F16") t.dtype = kF16; else if (dt->str() == "BF16") t.dtype = kBF16;
    else continue;  // integer buffers etc. are not model weights
    uint64_t a = 0, b = 0;
    if (!off->items()[0].as_u64(&a) || !off->items()[1].as_u64(&b) || b < a || b > size_ - base) { if (err) *err = "safetensors: offsets of " + kv.first; return false; }
    t.offset = base + a;
    t.nbytes = b - a;
    std::vector<uint64_t> dims;
    for (const Json& d : sh->items()) { uint64_t v = 0; if (!d.as_u64(&v)) { if (err) *err = "safetensors: shape of " + kv.first; return false; } dims.push_back(v); }
    if (dims.size() == 2) { t.rows = dims[0]; t.cols = dims[1]; } else if (dims.size() == 1) { t.rows = 1; t.cols = dims[0]; } else continue;
    uint64_t n_el = 0, n_by = 0;
    if (!mul_ok(t.rows, t.cols, &n_el) || !mul_ok(n_el, t.dtype == kF32 ? 4 : 2, &n_by) || n_by != t.nbytes) { if (err) *err = "safetensors: size of " + kv.first; return false; }
    // geometry from shapes (head_dim is 128 for every model the engine accepts)
    if (t.name == "model.embed_tokens.weight") { geo_.vocab = uint32_t(t.rows); geo_.hidden = uint32_t(t.cols); }
    if (t.name.compare(0, 13, "model.layers.") == 0) {
      const size_t d = t.name.find('.', 13);
      if (d != std::string::npos && d - 13 <= 6) {
        const int64_t layer = atoll(t.name.substr(13, d - 13).c_str());
        if (layer < 0 || layer >= kMaxLayers) { if (err) *err = "safetensors: layer index of " + kv.first; return false; }
        max_layer = std::max<int64_t>(max_layer, layer);
      }
      if (t.name.find("self_attn.q_proj.weight") != std::string::npos) geo_.n_heads = uint32_t(t.rows / 128);
      if (t.name.find("self_attn.k_proj.weight") != std::string::npos) geo_.n_kv_heads = uint32_t(t.rows / 128);
      if (t.name.find("mlp.gate_proj.weight") != std::string::npos) geo_.ffn = uint32_t(t.rows);
    }
    tensors_.push_back(t);
  }
  geo_.n_layers = uint32_t(max_layer + 1);
  geo_.head_dim = 128;
  geo_.rope_theta = 500000.f;   // not stored in the tensor file (config.json): Llama-3 values, overridable by the caller
  geo_.rms_eps = 1e-5f;
  geo_.known = geo_.hidden && geo_.n_layers && geo_.n_heads && geo_.n_kv_heads && geo_.ffn && geo_.vocab;
  return read_config_json(max_layer, err);
}

// The Hugging Face config.json beside a safetensors file: RoPE theta and scaling, RMSNorm eps, and the
// geometry, which must agree with the tensor shapes this file holds.  Without one nothing changes.
bool Checkpoint::read_config_json(int64_t max_layer, std::string* err) {
  const size_t slash = path_.rfind('/');
  const std::string cpath = (slash == std::string::npos ? std::string() : path_.substr(0, slash + 1)) + "config.json";
  std::ifstream f(cpath, std::ios::binary);
  if (!f) return true;
  std::stringstream ss;
  ss << f.rdbuf();
  auto fail = [&](const std::string& m) { if (err) *err = cpath + ": " + m; return false; };
  Json cfg;
  if (!Json::parse(ss.str(), &cfg) || !cfg.is_object()) return fail("not a JSON object");
  auto num = [](const Json* o, const char* k, double dflt) { const Json* v = o ? o->get(k) : nullptr; return v && v->is_number() ? v->as_double() : dflt; };
  auto str = [](const Json* o, const char* k) { const Json* v = o ? o->get(k) : nullptr; return v && v->is_string() ? v->str() : std::string(); };
  // geometry: every field the tensors of this file show must match
  const double heads = num(&cfg, "num_attention_heads", 0), hidden = num(&cfg, "hidden_size", 0);
  const double head_dim = num(&cfg, "head_dim", heads > 0 ? hidden / heads : 0);
  if (heads > 0 && head_dim != 128) return fail("head_dim " + std::to_string(int64_t(head_dim)) + ": the engine serves head_dim 128 only");
  struct { const char* key; double dflt; uint32_t seen; } checks[] = {
      {"hidden_size", 0, geo_.hidden}, {"num_attention_heads", 0, geo_.n_heads}, {"num_key_value_heads", heads, geo_.n_kv_heads},
      {"intermediate_size", 0, geo_.ffn}, {"vocab_size", 0, geo_.vocab}};
  for (const auto& c : checks) {
    const double v = num(&cfg, c.key, c.dflt);
    if (c.seen && v > 0 && v != double(c.seen))
      return fail(std::string(c.key) + " is " + std::to_string(int64_t(v)) + " but the tensor shapes say " + std::to_string(c.seen));
  }
  const double n_layers = num(&cfg, "num_hidden_layers", 0);
  if (n_layers > 0) {
    if (n_layers > double(kMaxLayers)) return fail("num_hidden_layers out of range");
    if (max_layer >= int64_t(n_layers))
      return fail("num_hidden_layers is " + std::to_string(int64_t(n_layers)) + " but the file holds layer " + std::to_string(max_layer));
    geo_.n_layers = uint32_t(n_layers);
  }
  // RoPE: transformers 5 writes rope_parameters {rope_type, rope_theta, ...}; earlier versions rope_theta and
  // rope_scaling {rope_type (or type), ...} (null = none).  Defaults are transformers' LlamaConfig ones.
  const Json* rp = cfg.get("rope_parameters");
  if (rp && !rp->is_object()) rp = nullptr;
  const Json* rs = rp ? rp : cfg.get("rope_scaling");
  if (rs && !rs->is_null() && !rs->is_object()) return fail("rope_scaling is not an object");
  if (rs && rs->is_null()) rs = nullptr;
  const double theta = num(&cfg, "rope_theta", num(rp, "rope_theta", 10000.0));
  if (!(theta > 1.0) || !std::isfinite(theta)) return fail("rope_theta must be finite and > 1");
  const double eps = num(&cfg, "rms_norm_eps", 1e-6);
  if (!(eps > 0.0) || !std::isfinite(eps)) return fail("rms_norm_eps must be finite and > 0");
  std::string type = str(rs, "rope_type");
  if (type.empty()) type = str(rs, "type");
  std::string e;
  if (!rope_scaling_factors(type, num(rs, "factor", 0), num(rs, "low_freq_factor", 0), num(rs, "high_freq_factor", 0),
                            num(rs, "original_max_position_embeddings", 0), theta, 128, &geo_.rope_freq_factors, &e))
    return fail(e);
  geo_.rope_theta = float(theta);
  geo_.rms_eps = float(eps);
  geo_.rope_scaling = geo_.rope_freq_factors.empty() ? "none" : type;
  geo_.rope_known = true;
  return true;
}

bool Checkpoint::open_gguf(std::string* err) {
  Cur c{data_ + 4, data_ + size_};
  const uint32_t version = c.take<uint32_t>();
  if (version != 2 && version != 3) { if (err) *err = "gguf: unsupported version " + std::to_string(version); return false; }
  const uint64_t n_tensors = c.take<uint64_t>(), n_kv = c.take<uint64_t>();
  std::map<std::string, double> num;
  std::map<std::string, std::string> str;
  uint64_t alignment = 32;
  for (uint64_t i = 0; i < n_kv && c.ok; ++i) {
    const std::string key = c.str();
    const uint32_t type = c.take<uint32_t>();
    auto scalar = [&](uint32_t t) -> double {
      switch (t) {
        case 0: return c.take<uint8_t>(); case 1: return c.take<int8_t>(); case 2: return c.take<uint16_t>(); case 3: return c.take<int16_t>();
        case 4: return c.take<uint32_t>(); case 5: return c.take<int32_t>(); case 6: return c.take<float>(); case 7: return c.take<uint8_t>();
        case 10: return double(c.take<uint64_t>()); case 11: return double(c.take<int64_t>()); case 12: return c.take<double>();
      }
      c.ok = false;
      return 0;
    };
    if (type == 8) str[key] = c.str();
    else if (type == 9) {
      const uint32_t et = c.take<uint32_t>();
      const uint64_t count = c.take<uint64_t>();
      const bool tokens = key == "tokenizer.ggml.tokens", merges = key == "tokenizer.ggml.merges", types = key == "tokenizer.ggml.token_type";
      if (et == 8) {
        for (uint64_t k = 0; k < count && c.ok; ++k) { std::string s = c.str(); if (tokens) tok_tokens_.push_back(std::move(s)); else if (merges) tok_merges_.push_back(std::move(s)); }
      } else if (scalar_size(et)) {
        uint64_t nb = 0;
        if (types) for (uint64_t k = 0; k < count && c.ok; ++k) tok_types_.push_back(int32_t(i64_of(scalar(et), 0) & 0xFF));
        else if (mul_ok(count, scalar_size(et), &nb)) c.skip(nb);
        else c.ok = false;
      } else { c.ok = false; }
    } else num[key] = scalar(type);
  }
  if (!c.ok) { if (err) *err = "gguf: truncated or malformed metadata"; return false; }
  if (num.count("general.alignment")) {
    const double a = num["general.alignment"];
    if (!(a >= 1.0 && a <= 1048576.0)) { if (err) *err = "gguf: general.alignment out of range"; return false; }
    alignment = uint64_t(a);
  }
  const std::string arch = str.count("general.architecture") ? str["general.architecture"] : "llama";
  auto g = [&](const char* k, double dflt) { auto it = num.find(arch + "." + k); return it == num.end() ? dflt : it->second; };
  struct Info { std::string name; std::vector<uint64_t> dims; uint32_t type; uint64_t off; };
  std::vector<Info> infos;
  for (uint64_t i = 0; i < n_tensors && c.ok; ++i) {
    Info in;
    in.name = c.str();
    const uint32_t nd = c.take<uint32_t>();
    if (nd > 4) { c.ok = false; break; }
    for (uint32_t d = 0; d < nd; ++d) in.dims.push_back(c.take<uint64_t>());   // innermost first
    in.type = c.take<uint32_t>();
    in.off = c.take<uint64_t>();
    infos.push_back(in);
  }
  if (!c.ok) { if (err) *err = "gguf: truncated tensor table"; return false; }
  const uint64_t base = (uint64_t(c.p - data_) + alignment - 1) / alignment * alignment;
  const uint32_t n_head = u32_of(g("attention.head_count", 1)), n_kv_head = u32_of(g("attention.head_count_kv", n_head));
  bool has_output = false;
  const Info* rope_freqs = nullptr;   // llama.cpp's per-frequency RoPE divisors (Llama 3.1+ llama3 scaling)
  for (const Info& in : infos) {
    has_output |= in.name == "output.weight";
    if (in.name == "rope_freqs.weight") rope_freqs = &in;
  }
  for (const Info& in : infos) {
    uint32_t per = 0, bsz = 0;
    if (!block_shape(in.type, &per, &bsz)) { if (err) *err = "gguf: tensor " + in.name + " has unsupported ggml type " + std::to_string(in.type); return false; }
    uint64_t n = 1;
    bool dims_ok = true;
    for (uint64_t d : in.dims) dims_ok = dims_ok && d != 0 && mul_ok(n, d, &n);
    if (!dims_ok) { if (err) *err = "gguf: shape of " + in.name; return false; }
    if (!in.dims.empty() && in.dims[0] % per) { if (err) *err = "gguf: row length of " + in.name; return false; }
    CkptTensor t;
    t.src_name = in.name;
    t.name = hf_name(in.name);
    t.dtype = in.type;
    if (!mul_ok(n / per, bsz, &t.nbytes) || base > size_ || in.off > size_ - base || t.nbytes > size_ - base - in.off) {
      if (err) *err = "gguf: data of " + in.name + " past the end of the file";
      return false;
    }
    t.offset = base + in.off;
    if (in.name == "token_embd.weight" && in.dims.size() == 2) geo_.vocab = uint32_t(in.dims[1]);
    if (t.name.empty()) continue;
    if (in.dims.size() == 2) { t.rows = in.dims[1]; t.cols = in.dims[0]; } else if (in.dims.size() == 1) { t.rows = 1; t.cols = in.dims[0]; } else continue;
    const std::string& s = in.name;
    if (s.size() > 13 && s.compare(s.size() - 13, 13, "attn_q.weight") == 0) t.unpermute_heads = n_head;
    if (s.size() > 13 && s.compare(s.size() - 13, 13, "attn_k.weight") == 0) t.unpermute_heads = n_kv_head;
    tensors_.push_back(t);
    if (t.name == "model.embed_tokens.weight" && !has_output) {   // tied head
      CkptTensor h = t;
      h.name = "lm_head.weight";
      tensors_.push_back(h);
      tied_lm_head_ = true;
    }
  }
  geo_.hidden = u32_of(g("embedding_length", 0));
  geo_.n_layers = u32_of(g("block_count", 0));
  if (geo_.n_layers > kMaxLayers) { if (err) *err = "gguf: block_count out of range"; return false; }
  geo_.n_heads = n_head;
  geo_.n_kv_heads = n_kv_head;
  // head width: metadata when present, else the q projection's own shape (rows / heads) — a model
  // whose head_dim is not hidden / heads (e.g. hidden 512, 8 heads of 128) must not be guessed wrong
  uint32_t hd_from_q = 0;
  for (const CkptTensor& t : tensors_)
    if (n_head && t.name.size() > 23 && t.name.compare(t.name.size() - 23, 23, "self_attn.q_proj.weight") == 0 && t.cols == geo_.hidden) { hd_from_q = uint32_t(t.rows / n_head); break; }
  geo_.head_dim = u32_of(g("attention.key_length", hd_from_q ? hd_from_q : (geo_.n_heads ? geo_.hidden / geo_.n_heads : 0)));
  geo_.ffn = u32_of(g("feed_forward_length", 0));
  if (!geo_.vocab) geo_.vocab = u32_of(g("vocab_size", double(tok_tokens_.size())));
  geo_.rope_theta = float(g("rope.freq_base", 10000.0));
  geo_.rms_eps = float(g("attention.layer_norm_rms_epsilon", 1e-5));
  geo_.known = geo_.hidden && geo_.n_layers && geo_.n_heads && geo_.ffn && geo_.vocab;
  // RoPE scaling: the rope_freqs tensor (bit for bit) and/or {arch}.rope.scaling.type = linear with its factor
  geo_.rope_known = true;
  if (rope_freqs) {
    const uint64_t want = geo_.head_dim / 2;
    if (rope_freqs->type != kF32 || rope_freqs->dims.size() != 1 || rope_freqs->dims[0] != want || want == 0) {
      if (err) *err = "gguf: rope_freqs.weight must be " + std::to_string(want) + " F32 values (head_dim / 2)";
      return false;
    }
    geo_.rope_freq_factors.resize(size_t(want));
    memcpy(geo_.rope_freq_factors.data(), data_ + base + rope_freqs->off, size_t(want) * 4);   // bounds checked in the loop above
    for (float v : geo_.rope_freq_factors)
      if (!(v > 0.f) || !std::isfinite(v)) { if (err) *err = "gguf: rope_freqs.weight holds a factor that is not finite and > 0"; return false; }
    geo_.rope_scaling = "rope_freqs";
  }
  const auto st = str.find(arch + ".rope.scaling.type");
  const std::string stype = st == str.end() ? std::string() : st->second;
  if (!stype.empty() && stype != "none") {
    std::vector<float> lin;
    std::string e;
    if (stype != "linear") e = "unsupported RoPE scaling type '" + stype + "': only linear and rope_freqs.weight are served";
    else rope_scaling_factors(stype, g("rope.scaling.factor", 0), 0, 0, 0, 0, geo_.head_dim, &lin, &e);
    if (!e.empty() || lin.empty()) { if (err) *err = "gguf: " + (e.empty() ? std::string("bad RoPE scaling") : e); return false; }
    if (geo_.rope_freq_factors.empty()) geo_.rope_freq_factors = lin;
    else for (size_t j = 0; j < lin.size(); ++j) geo_.rope_freq_factors[j] *= lin[j];   // llama.cpp applies both
    geo_.rope_scaling = "linear";
  }
  tok_model_ = str.count("tokenizer.ggml.model") ? str["tokenizer.ggml.model"] : "";
  tok_pre_ = str.count("tokenizer.ggml.pre") ? str["tokenizer.ggml.pre"] : "llama-bpe";
  tok_bos_ = num.count("tokenizer.ggml.bos_token_id") ? i64_of(num["tokenizer.ggml.bos_token_id"], -1) : -1;
  return true;
}

bool Checkpoint::read_bf16(size_t i, std::vector<uint16_t>* out, std::string* err) const {
  if (i >= tensors_.size()) { if (err) *err = "tensor index"; return false; }
  const CkptTensor& t = tensors_[i];
  const size_t n = size_t(t.rows * t.cols);          // open() checked the product and that [offset, offset + nbytes) is inside the file
  const uint8_t* src = data_ + t.offset;
  out->resize(n);
  if (n == 0) return true;
  if (t.dtype == kBF16 && !t.unpermute_heads) { memcpy(out->data(), src, n * 2); return true; }
  std::vector<float> f(n);
  if (!ggml_dequantize(t.dtype, src, size_t(t.nbytes), f.data(), n)) { if (err) *err = "cannot dequantise " + t.src_name; return false; }
  if (t.unpermute_heads) {
    // rows [head][pair][half] (llama.cpp's rotary layout) -> [head][half][pair] (Hugging Face / this engine)
    const size_t heads = t.unpermute_heads, hd = size_t(t.rows) / heads, half = hd / 2, cols = size_t(t.cols);
    for (size_t h = 0; h < heads; ++h)
      for (size_t p = 0; p < half; ++p)
        for (size_t s = 0; s < 2; ++s) {
          const float* srow = f.data() + (h * hd + p * 2 + s) * cols;
          uint16_t* drow = out->data() + (h * hd + s * half + p) * cols;
          for (size_t k = 0; k < cols; ++k) drow[k] = f32_to_bf16_bits(srow[k]);
        }
    return true;
  }
  for (size_t k = 0; k < n; ++k) (*out)[k] = f32_to_bf16_bits(f[k]);
  return true;
}

std::string Checkpoint::tokenizer_json() const {
  if (!gguf_ || tok_model_ != "gpt2" || tok_tokens_.empty()) return "";
  if (tok_pre_ != "llama-bpe" && tok_pre_ != "llama3" && tok_pre_ != "llama-v3") return "";
  Json vocab = Json::object(), added = Json::array(), merges = Json::array();
  for (size_t i = 0; i < tok_tokens_.size(); ++i) {
    const int32_t ty = i < tok_types_.size() ? tok_types_[i] : 1;
    if (ty == 3 || ty == 4) {
      Json a = Json::object();
      a.set("id", Json(int64_t(i)));
      a.set("content", tok_tokens_[i]);
      a.set("single_word", Json(false)); a.set("lstrip", Json(false)); a.set("rstrip", Json(false)); a.set("normalized", Json(false));
      a.set("special", Json(ty == 3));
      added.push(a);
    } else {
      vocab.append(tok_tokens_[i], Json(int64_t(i)));
    }
  }
  for (const std::string& m : tok_merges_) merges.push(Json(m));
  Json split = Json::object();
  Json pat = Json::object();
  pat.set("Regex", "(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\\r\\n\\p{L}\\p{N}]?\\p{L}+|\\p{N}{1,3}| ?[^\\s\\p{L}\\p{N}]+[\\r\\n]*|\\s*[\\r\\n]+|\\s+(?!\\S)|\\s+");
  split.set("type", "Split"); split.set("pattern", pat); split.set("behavior", "Isolated"); split.set("invert", Json(false));
  Json bl = Json::object();
  bl.set("type", "ByteLevel"); bl.set("add_prefix_space", Json(false)); bl.set("trim_offsets", Json(true)); bl.set("use_regex", Json(false));
  Json pts = Json::array();
  pts.push(split); pts.push(bl);
  Json pre = Json::object();
  pre.set("type", "Sequence"); pre.set("pretokenizers", pts);
  Json model = Json::object();
  model.set("type", "BPE"); model.set("byte_fallback", Json(false)); model.set("ignore_merges", Json(true));
  model.set("vocab", vocab); model.set("merges", merges);
  Json dec = Json::object();
  dec.set("type", "ByteLevel");
  Json root = Json::object();
  root.set("version", "1.0"); root.set("added_tokens", added); root.set("normalizer", Json());
  root.set("pre_tokenizer", pre); root.set("decoder", dec); root.set("model", model);
  if (tok_bos_ >= 0 && size_t(tok_bos_) < tok_tokens_.size()) {
    Json st = Json::object(); st.set("id", tok_tokens_[size_t(tok_bos_)]); st.set("type_id", Json(int64_t(0)));
    Json s0 = Json::object(); s0.set("SpecialToken", st);
    Json sq = Json::object(); sq.set("id", "A"); sq.set("type_id", Json(int64_t(0)));
    Json s1 = Json::object(); s1.set("Sequence", sq);
    Json single = Json::array(); single.push(s0); single.push(s1);
    Json pp = Json::object(); pp.set("type", "TemplateProcessing"); pp.set("single", single);
    root.set("post_processor", pp);
  }
  return root.dump();
}

}  // namespace llmlb_host

// =============================================================================================
// extern "C" surface for ctypes tests (tests/test_host_checkpoint.py)
// =============================================================================================
using llmlb_host::Checkpoint;

#include "../../include/llmlb_gateway.h"   // the exported signatures are checked against the public header at compile time
extern "C" {
void* llmlb_ckpt_open(const char* path, char* err, uint32_t err_cap) {
  auto* c = new Checkpoint();
  std::string e;
  if (!c->open(path, &e)) { if (err && err_cap) snprintf(err, err_cap, "%s", e.c_str()); delete c; return nullptr; }
  return c;
}
void llmlb_ckpt_close(void* c) { delete static_cast<Checkpoint*>(c); }
uint32_t llmlb_ckpt_count(void* c) { return uint32_t(static_cast<Checkpoint*>(c)->tensors().size()); }
int llmlb_ckpt_is_gguf(void* c) { return static_cast<Checkpoint*>(c)->is_gguf() ? 1 : 0; }
// geometry: hidden, n_layers, n_heads, n_kv_heads, head_dim, ffn, vocab as u32[7]; theta, eps as float[2]; returns known
int llmlb_ckpt_geometry(void* c, uint32_t* u7, float* f2) {
  const auto& g = static_cast<Checkpoint*>(c)->geometry();
  const uint32_t v[7] = {g.hidden, g.n_layers, g.n_heads, g.n_kv_heads, g.head_dim, g.ffn, g.vocab};
  memcpy(u7, v, sizeof v);
  f2[0] = g.rope_theta; f2[1] = g.rms_eps;
  return g.known ? 1 : 0;
}
uint32_t llmlb_ckpt_rope_freq_factors(void* c, float* out, uint32_t cap) {
  const auto& f = static_cast<Checkpoint*>(c)->geometry().rope_freq_factors;
  for (size_t j = 0; j < f.size() && j < cap && out; ++j) out[j] = f[j];
  return uint32_t(f.size());
}
int64_t llmlb_ckpt_tensor_info(void* c, uint32_t i, char* name, uint32_t name_cap, uint64_t* rows, uint64_t* cols) {
  const auto& ts = static_cast<Checkpoint*>(c)->tensors();
  if (i >= ts.size()) return -1;
  snprintf(name, name_cap, "%s", ts[i].name.c_str());
  *rows = ts[i].rows; *cols = ts[i].cols;
  return int64_t(ts[i].rows * ts[i].cols);
}
int llmlb_ckpt_tensor_bf16(void* c, uint32_t i, uint16_t* out, uint64_t cap_elems) {
  std::vector<uint16_t> v;
  std::string e;
  if (!static_cast<Checkpoint*>(c)->read_bf16(i, &v, &e) || v.size() > cap_elems) return -1;
  memcpy(out, v.data(), v.size() * 2);
  return 0;
}
int64_t llmlb_ckpt_tokenizer_json(void* c, char* out, uint64_t cap) {
  const std::string s = static_cast<Checkpoint*>(c)->tokenizer_json();
  const uint64_t n = s.size() < cap ? s.size() : cap;
  if (out && n) memcpy(out, s.data(), n);
  return int64_t(s.size());
}
}  // extern "C"
