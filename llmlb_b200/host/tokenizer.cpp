// Llama-3 byte-level BPE tokenizer, see tokenizer.hpp.  Behaviour is pinned to the `tokenizers`
// library (tests/golden/make_tokenizer_golden.py): same pre-tokenizer pattern semantics (ordered
// alternatives, greedy quantifiers, backtracking), same merge order (lowest rank first, leftmost
// on ties), ignore_merges, leftmost-longest special-token matching, ByteLevel decode.
#include "tokenizer.hpp"

#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstring>
#include <queue>

#include "json.hpp"

namespace llmlb_host {

namespace {

#include "unicode_tables.inc"

template <size_t N>
bool in_ranges(const uint32_t (&tab)[N][2], uint32_t cp) {
  size_t lo = 0, hi = N;
  while (lo < hi) {
    size_t mid = (lo + hi) / 2;
    if (cp < tab[mid][0]) hi = mid;
    else if (cp > tab[mid][1]) lo = mid + 1;
    else return true;
  }
  return false;
}
inline bool is_letter(uint32_t cp) {
  if (cp < 0x80) return (cp >= 'a' && cp <= 'z') || (cp >= 'A' && cp <= 'Z');
  return in_ranges(kUnicodeLetterRanges, cp);
}
inline bool is_number(uint32_t cp) {
  if (cp < 0x80) return cp >= '0' && cp <= '9';
  return in_ranges(kUnicodeNumberRanges, cp);
}
// \s of the pattern engine in Unicode mode: the White_Space property
inline bool is_space(uint32_t cp) {
  return (cp >= 0x09 && cp <= 0x0D) || cp == 0x20 || cp == 0x85 || cp == 0xA0 || cp == 0x1680 ||
         (cp >= 0x2000 && cp <= 0x200A) || cp == 0x2028 || cp == 0x2029 || cp == 0x202F ||
         cp == 0x205F || cp == 0x3000;
}
inline bool is_newline(uint32_t cp) { return cp == '\r' || cp == '\n'; }
inline bool is_other(uint32_t cp) { return !is_space(cp) && !is_letter(cp) && !is_number(cp); }

// UTF-8 -> code points with byte offsets; an invalid byte becomes its own U+FFFD "other" symbol
void decode_utf8(const std::string& s, std::vector<uint32_t>* cps, std::vector<uint32_t>* offs) {
  const size_t n = s.size();
  size_t i = 0;
  while (i < n) {
    const uint8_t c = uint8_t(s[i]);
    uint32_t cp = 0xFFFD;
    size_t len = 1;
    if (c < 0x80) cp = c;
    else if ((c >> 5) == 0x6 && i + 1 < n && (uint8_t(s[i + 1]) >> 6) == 0x2) {
      cp = ((c & 0x1Fu) << 6) | (uint8_t(s[i + 1]) & 0x3Fu);
      len = 2;
      if (cp < 0x80) { cp = 0xFFFD; len = 1; }
    } else if ((c >> 4) == 0xE && i + 2 < n && (uint8_t(s[i + 1]) >> 6) == 0x2 && (uint8_t(s[i + 2]) >> 6) == 0x2) {
      cp = ((c & 0x0Fu) << 12) | ((uint8_t(s[i + 1]) & 0x3Fu) << 6) | (uint8_t(s[i + 2]) & 0x3Fu);
      len = 3;
      if (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF)) { cp = 0xFFFD; len = 1; }
    } else if ((c >> 3) == 0x1E && i + 3 < n && (uint8_t(s[i + 1]) >> 6) == 0x2 && (uint8_t(s[i + 2]) >> 6) == 0x2 &&
               (uint8_t(s[i + 3]) >> 6) == 0x2) {
      cp = ((c & 0x07u) << 18) | ((uint8_t(s[i + 1]) & 0x3Fu) << 12) | ((uint8_t(s[i + 2]) & 0x3Fu) << 6) |
           (uint8_t(s[i + 3]) & 0x3Fu);
      len = 4;
      if (cp < 0x10000 || cp > 0x10FFFF) { cp = 0xFFFD; len = 1; }
    }
    cps->push_back(cp);
    offs->push_back(uint32_t(i));
    i += len;
  }
  offs->push_back(uint32_t(n));
}

void append_utf8(std::string* out, uint32_t cp) {
  if (cp < 0x80) out->push_back(char(cp));
  else if (cp < 0x800) { out->push_back(char(0xC0 | (cp >> 6))); out->push_back(char(0x80 | (cp & 0x3F))); }
  else if (cp < 0x10000) {
    out->push_back(char(0xE0 | (cp >> 12))); out->push_back(char(0x80 | ((cp >> 6) & 0x3F))); out->push_back(char(0x80 | (cp & 0x3F)));
  } else {
    out->push_back(char(0xF0 | (cp >> 18))); out->push_back(char(0x80 | ((cp >> 12) & 0x3F)));
    out->push_back(char(0x80 | ((cp >> 6) & 0x3F))); out->push_back(char(0x80 | (cp & 0x3F)));
  }
}

// GPT-2 byte <-> printable code point table used by the ByteLevel pre-tokenizer / decoder
struct ByteLevelMap {
  uint32_t byte_to_cp[256];
  std::string byte_to_str[256];
  std::unordered_map<uint32_t, uint8_t> cp_to_byte;
  ByteLevelMap() {
    bool direct[256] = {false};
    for (int b = 33; b <= 126; ++b) direct[b] = true;
    for (int b = 161; b <= 172; ++b) direct[b] = true;
    for (int b = 174; b <= 255; ++b) direct[b] = true;
    uint32_t next = 256;
    for (int b = 0; b < 256; ++b) {
      byte_to_cp[b] = direct[b] ? uint32_t(b) : next++;
      append_utf8(&byte_to_str[b], byte_to_cp[b]);
      cp_to_byte[byte_to_cp[b]] = uint8_t(b);
    }
  }
};
const ByteLevelMap& byte_level() {
  static const ByteLevelMap m;
  return m;
}

inline uint64_t pair_key(int32_t a, int32_t b) { return (uint64_t(uint32_t(a)) << 32) | uint32_t(b); }

const Json* find_template_processing(const Json& j) {
  if (j.is_object()) {
    const Json* t = j.get("type");
    if (t && t->is_string() && t->str() == "TemplateProcessing") return &j;
    if (const Json* p = j.get("processors"))
      if (p->is_array())
        for (size_t i = 0; i < p->items().size(); ++i)
          if (const Json* r = find_template_processing(p->items()[i])) return r;
  }
  return nullptr;
}

// Well-formed UTF-8 per Unicode Table 3-7.  Returns the length (1..4) of the well-formed sequence at s[i], or 0 when it is
// ill-formed; then *bad_len is the length of the MAXIMAL SUBPART (the longest prefix of a well-formed sequence, at least
// the one offending byte) that String::from_utf8_lossy / Python's errors="replace" substitute by ONE U+FFFD, and
// *truncated says the subpart runs to the end of the string and further bytes could still complete it.
static size_t utf8_wellformed(const std::string& s, size_t i, size_t* bad_len, bool* truncated) {
  const size_t n = s.size();
  const uint8_t b0 = uint8_t(s[i]);
  *bad_len = 1; *truncated = false;
  if (b0 < 0x80) return 1;
  size_t need;
  uint8_t lo = 0x80, hi = 0xBF;
  if (b0 >= 0xC2 && b0 <= 0xDF) need = 2;
  else if (b0 == 0xE0) { need = 3; lo = 0xA0; }
  else if ((b0 >= 0xE1 && b0 <= 0xEC) || b0 == 0xEE || b0 == 0xEF) need = 3;
  else if (b0 == 0xED) { need = 3; hi = 0x9F; }
  else if (b0 == 0xF0) { need = 4; lo = 0x90; }
  else if (b0 >= 0xF1 && b0 <= 0xF3) need = 4;
  else if (b0 == 0xF4) { need = 4; hi = 0x8F; }
  else return 0;                                   // 80..BF, C0, C1, F5..FF: never start a sequence
  size_t have = 1;
  while (have < need) {
    if (i + have >= n) { *bad_len = have; *truncated = true; return 0; }
    const uint8_t c = uint8_t(s[i + have]);
    const bool ok = have == 1 ? (c >= lo && c <= hi) : (c >= 0x80 && c <= 0xBF);
    if (!ok) { *bad_len = have; return 0; }
    ++have;
  }
  return need;
}

// true when [pos, size) is the beginning of a well-formed sequence that more bytes could still complete
bool incomplete_tail(const std::string& s, size_t pos) {
  size_t bad = 0;
  bool truncated = false;
  return utf8_wellformed(s, pos, &bad, &truncated) == 0 && truncated && pos + bad == s.size();
}

// String::from_utf8_lossy: well-formed sequences are copied, every maximal ill-formed subpart becomes one U+FFFD.
// (Round 2: the first version replaced byte by byte and let a lone 0xEF lead through raw — found with the scripted token
// source of tests/test_server_fake_engine_cpu.py, which emits byte-level tokens in random order.)
std::string utf8_lossy(const std::string& s) {
  std::string out;
  out.reserve(s.size());
  for (size_t i = 0; i < s.size();) {
    size_t bad = 0;
    bool truncated = false;
    const size_t len = utf8_wellformed(s, i, &bad, &truncated);
    if (len) { out.append(s, i, len); i += len; }
    else { out += "\xEF\xBF\xBD"; i += bad; }
  }
  return out;
}

std::string trim_ws(const std::string& s) {  // Jinja `trim`: strips ASCII/Unicode whitespace at both ends (ASCII is what chat content carries)
  size_t a = 0, b = s.size();
  while (a < b && (s[a] == ' ' || s[a] == '\n' || s[a] == '\t' || s[a] == '\r' || s[a] == '\f' || s[a] == '\v')) ++a;
  while (b > a && (s[b - 1] == ' ' || s[b - 1] == '\n' || s[b - 1] == '\t' || s[b - 1] == '\r' || s[b - 1] == '\f' || s[b - 1] == '\v')) --b;
  return s.substr(a, b - a);
}

}  // namespace

// (?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+
std::vector<std::pair<uint32_t, uint32_t>> BpeTokenizer::pretokenize(const std::string& utf8) {
  std::vector<uint32_t> cp, off;
  decode_utf8(utf8, &cp, &off);
  const size_t n = cp.size();
  std::vector<std::pair<uint32_t, uint32_t>> out;
  auto lower = [](uint32_t c) -> uint32_t {
    if (c >= 'A' && c <= 'Z') return c + 32;
    if (c == 0x17F) return 's';   // LATIN SMALL LETTER LONG S folds to s
    if (c == 0x212A) return 'k';  // KELVIN SIGN folds to k
    return c;
  };
  size_t i = 0;
  while (i < n) {
    size_t end = 0;
    const uint32_t c = cp[i];
    // 1. contractions
    if (c == '\'' && i + 1 < n) {
      const uint32_t a = lower(cp[i + 1]);
      const uint32_t b = i + 2 < n ? lower(cp[i + 2]) : 0;
      if (a == 's' || a == 't') end = i + 2;
      else if ((a == 'r' && b == 'e') || (a == 'v' && b == 'e')) end = i + 3;
      else if (a == 'm') end = i + 2;
      else if (a == 'l' && b == 'l') end = i + 3;
      else if (a == 'd') end = i + 2;
    }
    // 2. optional single non-letter/number/newline char + letters
    if (!end) {
      if (is_letter(c)) {
        size_t k = i;
        while (k < n && is_letter(cp[k])) ++k;
        end = k;
      } else if (!is_newline(c) && !is_number(c) && i + 1 < n && is_letter(cp[i + 1])) {
        size_t k = i + 1;
        while (k < n && is_letter(cp[k])) ++k;
        end = k;
      }
    }
    // 3. one to three numbers
    if (!end && is_number(c)) {
      size_t k = i;
      while (k < n && k < i + 3 && is_number(cp[k])) ++k;
      end = k;
    }
    // 4. optional space + punctuation run + trailing newlines
    if (!end) {
      size_t j = i;
      if (c == ' ' && i + 1 < n && is_other(cp[i + 1])) j = i + 1;
      if (is_other(cp[j])) {
        size_t k = j;
        while (k < n && is_other(cp[k])) ++k;
        while (k < n && is_newline(cp[k])) ++k;
        end = k;
      }
    }
    if (!end && is_space(c)) {
      size_t e = i;
      while (e < n && is_space(cp[e])) ++e;
      // 5. whitespace ending in newline(s): through the last newline of the run
      size_t last_nl = SIZE_MAX;
      for (size_t k = i; k < e; ++k)
        if (is_newline(cp[k])) last_nl = k;
      if (last_nl != SIZE_MAX) end = last_nl + 1;
      // 6. whitespace not followed by non-whitespace (leaves one space for the next word)
      else if (e == n) end = e;
      else if (e - i >= 2) end = e - 1;
      // 7. any whitespace
      else end = e;
    }
    if (!end) end = i + 1;  // unreachable for valid input: every class above is covered
    out.emplace_back(off[i], off[end]);
    i = end;
  }
  return out;
}

// ids index dense tables: a file that claims an id of 10^15 must be refused, not allocated for (the largest public
// vocabularies are ~260 k entries)
static constexpr uint64_t kMaxTokenId = 1u << 24;

bool BpeTokenizer::load_json(const std::string& text, std::string* err) {
  Json root;
  if (!Json::parse(text, &root)) { if (err) *err = "tokenizer.json: not valid JSON"; return false; }
  const Json* model = root.get("model");
  const Json* type = model ? model->get("type") : nullptr;
  if (!model || (type && type->is_string() && type->str() != "BPE")) { if (err) *err = "tokenizer.json: model.type must be BPE"; return false; }
  if (const Json* nz = root.get("normalizer"))
    if (!nz->is_null()) { if (err) *err = "tokenizer.json: normalizers are not supported (Llama-3 has none)"; return false; }
  if (const Json* bf = model->get("byte_fallback"))
    if (bf->as_bool()) { if (err) *err = "tokenizer.json: byte_fallback models are not byte-level BPE"; return false; }
  const Json* vocab = model->get("vocab");
  const Json* merges = model->get("merges");
  if (!vocab || !vocab->is_object() || !merges || !merges->is_array()) { if (err) *err = "tokenizer.json: model.vocab / model.merges missing"; return false; }
  ignore_merges_ = false;
  if (const Json* im = model->get("ignore_merges")) ignore_merges_ = im->as_bool();

  vocab_.clear(); id_to_token_.clear(); id_to_bytes_.clear(); special_flag_.clear(); merges_.clear(); added_.clear();
  size_t max_id = 0;
  for (const auto& kv : vocab->members()) {
    uint64_t id = 0;
    if (!kv.second.as_u64(&id) || id > kMaxTokenId) { if (err) *err = "tokenizer.json: vocab id is not an integer in [0, 2^24]"; return false; }
    vocab_[kv.first] = int32_t(id);
    max_id = std::max(max_id, size_t(id));
  }
  const Json* added = root.get("added_tokens");
  if (added && added->is_array())
    for (size_t i = 0; i < added->items().size(); ++i) {
      uint64_t id = 0;
      const Json* jid = added->items()[i].get("id");
      if (jid && jid->as_u64(&id)) {
        if (id > kMaxTokenId) { if (err) *err = "tokenizer.json: added token id out of range"; return false; }
        max_id = std::max(max_id, size_t(id));
      }
    }
  id_to_token_.assign(max_id + 1, std::string());
  id_to_bytes_.assign(max_id + 1, std::string());
  special_flag_.assign(max_id + 1, 0);
  const ByteLevelMap& bl = byte_level();
  for (const auto& kv : vocab_) {
    id_to_token_[kv.second] = kv.first;
    std::vector<uint32_t> cps, offs;
    decode_utf8(kv.first, &cps, &offs);
    std::string raw;
    for (uint32_t c : cps) {
      auto it = bl.cp_to_byte.find(c);
      if (it != bl.cp_to_byte.end()) raw.push_back(char(it->second));
      else append_utf8(&raw, c);  // not byte-level text (should not occur in a ByteLevel vocab)
    }
    id_to_bytes_[kv.second] = raw;
  }
  if (added && added->is_array()) {
    for (size_t i = 0; i < added->items().size(); ++i) {
      const Json& a = added->items()[i];
      const Json* jid = a.get("id");
      const Json* content = a.get("content");
      uint64_t id = 0;
      if (!jid || !jid->as_u64(&id) || !content || !content->is_string()) continue;
      const Json* sp = a.get("special");
      id_to_token_[id] = content->str();
      id_to_bytes_[id] = content->str();
      special_flag_[id] = (sp && sp->as_bool()) ? 1 : 0;
      added_.emplace_back(content->str(), int32_t(id));
    }
    std::stable_sort(added_.begin(), added_.end(), [](const std::pair<std::string, int32_t>& x, const std::pair<std::string, int32_t>& y) {
      return x.first.size() > y.first.size();
    });
  }
  for (size_t r = 0; r < merges->items().size(); ++r) {
    const Json& m = merges->items()[r];
    std::string a, b;
    if (m.is_string()) {  // "left right"
      const std::string& s = m.str();
      const size_t sp = s.find(' ');
      if (sp == std::string::npos) continue;
      a = s.substr(0, sp);
      b = s.substr(sp + 1);
    } else if (m.is_array() && m.items().size() == 2 && m.items()[0].is_string() && m.items()[1].is_string()) {
      a = m.items()[0].str();
      b = m.items()[1].str();
    } else continue;
    auto ia = vocab_.find(a), ib = vocab_.find(b), iab = vocab_.find(a + b);
    if (ia == vocab_.end() || ib == vocab_.end() || iab == vocab_.end()) continue;
    const uint64_t key = pair_key(ia->second, ib->second);
    if (!merges_.count(key)) merges_[key] = std::make_pair(int32_t(r), iab->second);
  }
  bos_id_ = -1;
  if (const Json* pp = root.get("post_processor")) {
    if (const Json* tp = find_template_processing(*pp)) {
      const Json* single = tp->get("single");
      if (single && single->is_array())
        for (size_t i = 0; i < single->items().size(); ++i) {
          const Json* st = single->items()[i].get("SpecialToken");
          if (single->items()[i].get("Sequence")) break;
          if (st && st->get("id") && st->get("id")->is_string()) { bos_id_ = special_id(st->get("id")->str()); break; }
        }
    }
  }
  if (bos_id_ < 0) bos_id_ = special_id("<|begin_of_text|>");
  return true;
}

int32_t BpeTokenizer::token_to_id(const std::string& token) const {
  auto it = vocab_.find(token);
  return it == vocab_.end() ? -1 : it->second;
}
int32_t BpeTokenizer::special_id(const std::string& content) const {
  for (const auto& a : added_)
    if (a.first == content) return a.second;
  return -1;
}

void BpeTokenizer::bpe_word(const std::string& piece, std::vector<int32_t>* out) const {
  const ByteLevelMap& bl = byte_level();
  if (ignore_merges_) {
    std::string mapped;
    for (unsigned char b : piece) mapped += bl.byte_to_str[b];
    auto it = vocab_.find(mapped);
    if (it != vocab_.end()) { out->push_back(it->second); return; }
  }
  std::vector<int32_t> sym;
  sym.reserve(piece.size());
  for (unsigned char b : piece) {
    auto it = vocab_.find(bl.byte_to_str[b]);
    if (it != vocab_.end()) sym.push_back(it->second);  // a byte-level vocab holds all 256; otherwise dropped like an unk-less model
  }
  if (sym.size() <= 48) {
    // short pieces (almost all of them): rescan for the lowest-rank pair, leftmost first
    while (sym.size() > 1) {
      int32_t best_rank = INT_MAX, best_id = -1;
      size_t best_pos = 0;
      for (size_t k = 0; k + 1 < sym.size(); ++k) {
        auto it = merges_.find(pair_key(sym[k], sym[k + 1]));
        if (it != merges_.end() && it->second.first < best_rank) {
          best_rank = it->second.first;
          best_id = it->second.second;
          best_pos = k;
        }
      }
      if (best_id < 0) break;
      sym[best_pos] = best_id;
      sym.erase(sym.begin() + best_pos + 1);
    }
  } else {
    // long pieces (a pre-token is an unbounded run of letters or of punctuation: 80 000 characters took 11-18 s with the
    // rescan, quadratic) — the same merge order from a heap of candidate pairs keyed (rank, position) over a linked list of
    // live symbols: O(n log n).  An entry is stale when either symbol died or changed since it was pushed.
    const uint32_t n = uint32_t(sym.size());
    struct Cand { int32_t rank; uint32_t pos; int32_t left, right, merged; };
    auto later = [](const Cand& a, const Cand& b) { return a.rank != b.rank ? a.rank > b.rank : a.pos > b.pos; };
    std::priority_queue<Cand, std::vector<Cand>, decltype(later)> heap(later);
    std::vector<uint32_t> next(n), prev(n);
    std::vector<uint8_t> alive(n, 1);
    for (uint32_t i = 0; i < n; ++i) { next[i] = i + 1; prev[i] = i ? i - 1 : n; }          // n = "none"
    auto push = [&](uint32_t pos) {
      const uint32_t r = next[pos];
      if (r >= n) return;
      auto it = merges_.find(pair_key(sym[pos], sym[r]));
      if (it != merges_.end()) heap.push(Cand{it->second.first, pos, sym[pos], sym[r], it->second.second});
    };
    for (uint32_t i = 0; i + 1 < n; ++i) push(i);
    while (!heap.empty()) {
      const Cand c = heap.top();
      heap.pop();
      if (!alive[c.pos]) continue;
      const uint32_t r = next[c.pos];
      if (r >= n || sym[c.pos] != c.left || sym[r] != c.right) continue;
      sym[c.pos] = c.merged;
      alive[r] = 0;
      next[c.pos] = next[r];
      if (next[r] < n) prev[next[r]] = c.pos;
      if (prev[c.pos] < n) push(prev[c.pos]);
      push(c.pos);
    }
    size_t w = 0;
    for (uint32_t i = 0; i < n; ++i) if (alive[i]) sym[w++] = sym[i];
    sym.resize(w);
  }
  out->insert(out->end(), sym.begin(), sym.end());
}

void BpeTokenizer::encode_plain(const std::string& text, std::vector<int32_t>* out) const {
  for (const auto& pr : pretokenize(text)) bpe_word(text.substr(pr.first, pr.second - pr.first), out);
}

std::vector<int32_t> BpeTokenizer::encode(const std::string& text, bool add_bos, bool parse_special) const {
  std::vector<int32_t> out;
  if (add_bos && bos_id_ >= 0) out.push_back(bos_id_);
  if (!parse_special || added_.empty()) {
    encode_plain(text, &out);
    return out;
  }
  // leftmost-longest match over the added tokens (added_ is sorted longest first); only positions
  // whose byte can start one are examined (Llama-3 has 256 of them, all beginning with '<')
  bool first_byte[256] = {false};
  for (const auto& a : added_)
    if (!a.first.empty()) first_byte[uint8_t(a.first[0])] = true;
  size_t start = 0, i = 0;
  const size_t n = text.size();
  while (i < n) {
    int32_t hit = -1;
    size_t hit_len = 0;
    if (!first_byte[uint8_t(text[i])]) { ++i; continue; }
    for (const auto& a : added_) {
      if (a.first.size() <= n - i && text.compare(i, a.first.size(), a.first) == 0) { hit = a.second; hit_len = a.first.size(); break; }
    }
    if (hit >= 0 && hit_len > 0) {
      if (i > start) encode_plain(text.substr(start, i - start), &out);
      out.push_back(hit);
      i += hit_len;
      start = i;
    } else {
      ++i;
    }
  }
  if (start < n) encode_plain(text.substr(start), &out);
  return out;
}

std::string BpeTokenizer::decode(const std::vector<int32_t>& ids, bool skip_special) const {
  std::string out;
  for (int32_t id : ids) {
    if (id < 0 || size_t(id) >= id_to_bytes_.size()) continue;
    if (skip_special && special_flag_[id]) continue;
    out += id_to_bytes_[id];
  }
  return out;
}

std::string BpeTokenizer::decode_next(Stream* s, int32_t id, bool skip_special) const {
  if (id >= 0 && size_t(id) < id_to_bytes_.size() && !(skip_special && special_flag_[id])) s->pending += id_to_bytes_[id];
  const std::string& p = s->pending;
  // hold back at most the last 3 bytes when they start a sequence that is not complete yet
  size_t cut = p.size();
  for (size_t back = 1; back <= 3 && back <= p.size(); ++back) {
    const size_t pos = p.size() - back;
    const uint8_t c = uint8_t(p[pos]);
    if ((c >> 6) == 0x2) continue;      // continuation byte: keep looking for its lead
    if (c >= 0xC0 && incomplete_tail(p, pos)) cut = pos;
    break;
  }
  std::string ready = utf8_lossy(p.substr(0, cut));
  s->pending = p.substr(cut);
  return ready;
}

std::string BpeTokenizer::token_bytes(int32_t id) const {
  return id >= 0 && size_t(id) < id_to_bytes_.size() ? id_to_bytes_[id] : std::string();
}

std::string BpeTokenizer::lossy_text(const std::string& bytes) { return utf8_lossy(bytes); }

std::string BpeTokenizer::flush(Stream* s) {
  std::string out = s->pending.empty() ? std::string() : std::string("\xEF\xBF\xBD");
  s->pending.clear();
  return out;
}

std::string BpeTokenizer::apply_chat_template(const std::vector<ChatMessage>& messages, bool add_generation_prompt) const {
  std::string out = "<|begin_of_text|>";
  for (const auto& m : messages) {
    out += "<|start_header_id|>" + m.role + "<|end_header_id|>\n\n" + trim_ws(m.content) + "<|eot_id|>";
  }
  if (add_generation_prompt) out += "<|start_header_id|>assistant<|end_header_id|>\n\n";
  return out;
}

// Role and content are tokenised as PLAIN text (a client cannot smuggle control tokens through
// message content); only the template's own markers become special ids.
std::vector<int32_t> BpeTokenizer::encode_chat(const std::vector<ChatMessage>& messages) const {
  std::vector<int32_t> out;
  auto sp = [&](const char* name) { const int32_t id = special_id(name); if (id >= 0) out.push_back(id); };
  sp("<|begin_of_text|>");
  for (const auto& m : messages) {
    sp("<|start_header_id|>");
    encode_plain(m.role, &out);
    sp("<|end_header_id|>");
    encode_plain("\n\n" + trim_ws(m.content), &out);
    sp("<|eot_id|>");
  }
  sp("<|start_header_id|>");
  encode_plain("assistant", &out);
  sp("<|end_header_id|>");
  encode_plain("\n\n", &out);
  return out;
}

}  // namespace llmlb_host

// =============================================================================================
// extern "C" surface for ctypes tests (tests/test_host_tokenizer.py) and non-C++ hosts
// =============================================================================================
using llmlb_host::BpeTokenizer;
using llmlb_host::ChatMessage;
using llmlb_host::Json;

static int64_t copy_out(const std::string& s, char* out, uint64_t cap) {
  const uint64_t n = s.size() < cap ? s.size() : cap;
  if (out && n) memcpy(out, s.data(), n);
  return int64_t(s.size());
}
static bool parse_messages(const char* json, uint64_t len, std::vector<ChatMessage>* out) {
  Json j;
  if (!Json::parse(std::string(json, len), &j) || !j.is_array()) return false;
  for (const Json& m : j.items()) {
    const Json* r = m.get("role");
    const Json* c = m.get("content");
    if (!r || !r->is_string() || !c || !c->is_string()) return false;
    out->push_back(ChatMessage{r->str(), c->str()});
  }
  return true;
}

#include "../../include/llmlb_host.h"   // the exported signatures are checked against the public header at compile time
extern "C" {
void* llmlb_tok_create(const char* json, uint64_t len, char* err, uint32_t err_cap) {
  auto* t = new BpeTokenizer();
  std::string e;
  if (!t->load_json(std::string(json, len), &e)) {
    if (err && err_cap) { snprintf(err, err_cap, "%s", e.c_str()); }
    delete t;
    return nullptr;
  }
  return t;
}
void llmlb_tok_destroy(void* t) { delete static_cast<BpeTokenizer*>(t); }
uint32_t llmlb_tok_vocab_size(void* t) { return static_cast<BpeTokenizer*>(t)->vocab_size(); }
int32_t llmlb_tok_bos_id(void* t) { return static_cast<BpeTokenizer*>(t)->bos_id(); }
int32_t llmlb_tok_special_id(void* t, const char* content) { return static_cast<BpeTokenizer*>(t)->special_id(content); }
// returns the number of ids (which may exceed cap: call again with a larger buffer)
int64_t llmlb_tok_encode(void* t, const char* text, uint64_t len, int add_bos, int parse_special, int32_t* out, uint64_t cap) {
  const std::vector<int32_t> ids = static_cast<BpeTokenizer*>(t)->encode(std::string(text, len), add_bos != 0, parse_special != 0);
  for (uint64_t i = 0; i < ids.size() && i < cap; ++i) out[i] = ids[i];
  return int64_t(ids.size());
}
int64_t llmlb_tok_decode(void* t, const int32_t* ids, uint64_t n, int skip_special, char* out, uint64_t cap) {
  return copy_out(static_cast<BpeTokenizer*>(t)->decode(std::vector<int32_t>(ids, ids + n), skip_special != 0), out, cap);
}
int64_t llmlb_tok_pretokenize(const char* text, uint64_t len, uint32_t* out_pairs, uint64_t cap_pairs) {
  const auto pieces = BpeTokenizer::pretokenize(std::string(text, len));
  for (uint64_t i = 0; i < pieces.size() && i < cap_pairs; ++i) { out_pairs[2 * i] = pieces[i].first; out_pairs[2 * i + 1] = pieces[i].second; }
  return int64_t(pieces.size());
}
void* llmlb_tok_stream_create() { return new BpeTokenizer::Stream(); }
void llmlb_tok_stream_destroy(void* s) { delete static_cast<BpeTokenizer::Stream*>(s); }
int64_t llmlb_tok_stream_next(void* t, void* s, int32_t id, int skip_special, char* out, uint64_t cap) {
  return copy_out(static_cast<BpeTokenizer*>(t)->decode_next(static_cast<BpeTokenizer::Stream*>(s), id, skip_special != 0), out, cap);
}
int64_t llmlb_tok_stream_flush(void* s, char* out, uint64_t cap) {
  return copy_out(BpeTokenizer::flush(static_cast<BpeTokenizer::Stream*>(s)), out, cap);
}
// messages_json: [{"role": "...", "content": "..."}, ...]; -1 on malformed input
int64_t llmlb_tok_chat_ids(void* t, const char* messages_json, uint64_t len, int32_t* out, uint64_t cap) {
  std::vector<ChatMessage> msgs;
  if (!parse_messages(messages_json, len, &msgs)) return -1;
  const std::vector<int32_t> ids = static_cast<BpeTokenizer*>(t)->encode_chat(msgs);
  for (uint64_t i = 0; i < ids.size() && i < cap; ++i) out[i] = ids[i];
  return int64_t(ids.size());
}
int64_t llmlb_tok_chat_text(void* t, const char* messages_json, uint64_t len, int add_generation_prompt, char* out, uint64_t cap) {
  std::vector<ChatMessage> msgs;
  if (!parse_messages(messages_json, len, &msgs)) return -1;
  return copy_out(static_cast<BpeTokenizer*>(t)->apply_chat_template(msgs, add_generation_prompt != 0), out, cap);
}
}  // extern "C"
