// Llama-3 tokenizer in native code (SURVEY.md §8f.2): byte-level BPE loaded from a Hugging Face
// `tokenizer.json`, the Llama-3 pre-tokenizer pattern, special-token splitting, an incremental
// UTF-8-safe detokenizer for SSE deltas and the Llama-3 chat template.  Host side of the C ABI:
// the engine takes and returns token ids (include/llmlb_b200.h), this turns the gateway's JSON
// text into ids and ids back into text without Python on the token path.
//
// The reference itself only COUNTS tokens (tiktoken estimate when a stream carries no usage,
// llmlb/src/token/mod.rs:217-223); tokenisation proper happens inside the external engines it
// proxies to.  Parity is therefore pinned to the `tokenizers` library (0.22) on a tokenizer.json
// with the exact Llama-3 pipeline: tests/golden/make_tokenizer_golden.py.
#pragma once
#include <cstdint>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

namespace llmlb_host {

struct ChatMessage { std::string role, content; };

class BpeTokenizer {
 public:
  // Parses tokenizer.json (model.type == "BPE", byte-level).  False + *err on anything it cannot
  // represent (other model types, normalizers, byte_fallback).
  bool load_json(const std::string& text, std::string* err);

  // parse_special: occurrences of special/added tokens in `text` become their ids (the chat
  // template path); otherwise they are tokenised as plain text.  add_bos: prepend the
  // post-processor's begin-of-text token.
  std::vector<int32_t> encode(const std::string& text, bool add_bos, bool parse_special) const;
  // Raw bytes of the ids (may end inside a UTF-8 sequence).  skip_special drops special tokens.
  std::string decode(const std::vector<int32_t>& ids, bool skip_special) const;

  // Streaming detokenizer: feed ids one at a time, get only complete UTF-8 back; bytes of an
  // unfinished sequence are held in `pending` (flush() returns them, replacing an incomplete
  // tail by U+FFFD like `String::from_utf8_lossy`).
  struct Stream { std::string pending; };
  std::string decode_next(Stream* s, int32_t id, bool skip_special) const;
  static std::string flush(Stream* s);

  // Raw byte-level bytes of one token (a special token: its content; "" for an id outside the vocabulary), and those
  // bytes as text the way decode_next releases it (every ill-formed or cut UTF-8 subpart becomes one U+FFFD): the
  // `bytes` and `token` of an OpenAI logprobs entry.
  std::string token_bytes(int32_t id) const;
  static std::string lossy_text(const std::string& bytes);

  // <|begin_of_text|><|start_header_id|>{role}<|end_header_id|>\n\n{content|trim}<|eot_id|>...
  // followed by the assistant header when add_generation_prompt.
  std::string apply_chat_template(const std::vector<ChatMessage>& messages, bool add_generation_prompt) const;
  std::vector<int32_t> encode_chat(const std::vector<ChatMessage>& messages) const;

  int32_t token_to_id(const std::string& token) const;   // -1 if absent (vocab strings are byte-level text)
  int32_t special_id(const std::string& content) const;  // -1 if absent
  uint32_t vocab_size() const { return uint32_t(id_to_token_.size()); }
  int32_t bos_id() const { return bos_id_; }
  bool is_special(int32_t id) const { return id >= 0 && size_t(id) < special_flag_.size() && special_flag_[id]; }

  // The Llama-3 Split pattern, exposed for tests: byte ranges [begin, end) of the pieces.
  static std::vector<std::pair<uint32_t, uint32_t>> pretokenize(const std::string& utf8);

 private:
  void bpe_word(const std::string& piece, std::vector<int32_t>* out) const;
  void encode_plain(const std::string& text, std::vector<int32_t>* out) const;

  std::unordered_map<std::string, int32_t> vocab_;            // byte-level text -> id
  std::vector<std::string> id_to_token_;                       // id -> byte-level text ("" = hole)
  std::vector<std::string> id_to_bytes_;                       // id -> raw bytes (specials: their content)
  std::vector<uint8_t> special_flag_;
  std::unordered_map<uint64_t, std::pair<int32_t, int32_t>> merges_;  // (left id, right id) -> (rank, merged id)
  std::vector<std::pair<std::string, int32_t>> added_;         // added tokens, longest first
  bool ignore_merges_ = false;
  int32_t bos_id_ = -1;
};

}  // namespace llmlb_host
