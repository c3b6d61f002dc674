// Byte-level BPE tokenizer that reads a local HF `tokenizer.json` of the Llama-3 family (SURVEY.md §8f-2: "real weights /
// tokenizer").  The reference never tokenizes: its backend pod does (vLLM loading the checkpoint's tokenizer.json through HF
// `tokenizers`, chat template included; internal/modelcontroller/engine_vllm.go:34-41 hands it the model directory).  This is
// that step restated on the host side of the C ABI:
//   added / special tokens   split out of the raw text first, leftmost-longest (tokenizers AddedVocabulary, normalized=false)
//   pre-tokenizer            Sequence[Split(<the GPT-4 / Llama-3 pattern>, Isolated), ByteLevel(use_regex=false)]; the pattern
//                            is matched by a hand-written scanner (alternation order and backtracking of the regex restated
//                            per alternative) over code-point classes generated from the tokenizers regex engine itself
//                            (unicode_ranges.h, scripts/gen_unicode_ranges.py)
//   model                    BPE over GPT-2 byte-level symbols: repeatedly merge the adjacent pair of lowest rank, leftmost
//                            first (tokenizers models/bpe/word.rs merge order); ignore_merges = whole pre-token in the vocab
//   decoder                  ByteLevel
//   chat template            Llama-3 instruct (header / eot framing), tokenised per segment
// Any other pipeline in the file is refused at load time rather than approximated.  Parity: tests/test_tokenizer.py compares ids
// with the `tokenizers` wheel on a tokenizer.json of this pipeline (ASCII, accents, CJK, emoji, whitespace runs, digits,
// contractions, random code points) and the chat template with transformers' apply_chat_template.
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200engine.h"
#include "errors.h"
#include "hostutil.h"
#include "tokenizer.h"
#include "unicode_ranges.h"

namespace b200 {
namespace {

const char kLlama3Pattern[] =
    "(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\\r\\n\\p{L}\\p{N}]?\\p{L}+|\\p{N}{1,3}| ?[^\\s\\p{L}\\p{N}]+[\\r\\n]*|\\s*[\\r\\n]+|\\s+(?!\\S)|\\s+";

template <size_t N>
bool in_ranges(const CpRange (&r)[N], uint32_t cp) {
  size_t lo = 0, hi = N;
  while (lo < hi) {
    const size_t mid = (lo + hi) / 2;
    if (cp < r[mid].lo) hi = mid;
    else if (cp > r[mid].hi) lo = mid + 1;
    else return true;
  }
  return false;
}
inline bool is_letter(uint32_t c) { return c < 0x80 ? ((c | 0x20) >= 'a' && (c | 0x20) <= 'z') : in_ranges(kUnicodeLetter, c); }
inline bool is_number(uint32_t c) { return c < 0x80 ? (c >= '0' && c <= '9') : in_ranges(kUnicodeNumber, c); }
inline bool is_space(uint32_t c) { return c < 0x80 ? (c == ' ' || (c >= 9 && c <= 13)) : in_ranges(kUnicodeSpace, c); }
inline bool is_newline(uint32_t c) { return c == '\r' || c == '\n'; }

// UTF-8 -> code points with the byte offset of each (invalid bytes become U+FFFD, one per byte, as from_utf8_lossy does)
void decode_utf8(const char* s, size_t n, std::vector<uint32_t>* cps, std::vector<uint32_t>* offs) {
  size_t i = 0;
  while (i < n) {
    const unsigned char c = static_cast<unsigned char>(s[i]);
    uint32_t cp = 0xFFFD;
    size_t len = 1;
    if (c < 0x80) cp = c;
    else if ((c & 0xE0) == 0xC0 && i + 1 < n && (s[i + 1] & 0xC0) == 0x80) { cp = ((c & 0x1F) << 6) | (s[i + 1] & 0x3F); len = 2; if (cp < 0x80) { cp = 0xFFFD; len = 1; } }
    else if ((c & 0xF0) == 0xE0 && i + 2 < n && (s[i + 1] & 0xC0) == 0x80 && (s[i + 2] & 0xC0) == 0x80) {
      cp = ((c & 0x0F) << 12) | ((s[i + 1] & 0x3F) << 6) | (s[i + 2] & 0x3F); len = 3;
      if (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF)) { cp = 0xFFFD; len = 1; }
    } else if ((c & 0xF8) == 0xF0 && i + 3 < n && (s[i + 1] & 0xC0) == 0x80 && (s[i + 2] & 0xC0) == 0x80 && (s[i + 3] & 0xC0) == 0x80) {
      cp = ((c & 0x07) << 18) | ((s[i + 1] & 0x3F) << 12) | ((s[i + 2] & 0x3F) << 6) | (s[i + 3] & 0x3F); len = 4;
      if (cp < 0x10000 || cp > 0x10FFFF) { cp = 0xFFFD; len = 1; }
    }
    cps->push_back(cp);
    offs->push_back(static_cast<uint32_t>(i));
    i += len;
  }
  offs->push_back(static_cast<uint32_t>(n));
}

void append_utf8(std::string* out, uint32_t cp) {
  if (cp < 0x80) out->push_back(static_cast<char>(cp));
  else if (cp < 0x800) { out->push_back(static_cast<char>(0xC0 | (cp >> 6))); out->push_back(static_cast<char>(0x80 | (cp & 0x3F))); }
  else if (cp < 0x10000) {
    out->push_back(static_cast<char>(0xE0 | (cp >> 12))); out->push_back(static_cast<char>(0x80 | ((cp >> 6) & 0x3F)));
    out->push_back(static_cast<char>(0x80 | (cp & 0x3F)));
  } else {
    out->push_back(static_cast<char>(0xF0 | (cp >> 18))); out->push_back(static_cast<char>(0x80 | ((cp >> 12) & 0x3F)));
    out->push_back(static_cast<char>(0x80 | ((cp >> 6) & 0x3F))); out->push_back(static_cast<char>(0x80 | (cp & 0x3F)));
  }
}

// length (in code points) of the pre-token that starts at i: the first alternative of the pattern that matches there
size_t next_piece(const std::vector<uint32_t>& c, size_t i) {
  const size_t n = c.size();
  auto at = [&](size_t k) { return k < n ? c[k] : 0xFFFFFFFFu; };
  auto lower = [](uint32_t x) { return (x >= 'A' && x <= 'Z') ? x + 32 : (x == 0x17F ? static_cast<uint32_t>('s') : x); };   // (?i): U+017F folds to s
  const uint32_t c0 = c[i];
  // 1. (?i:'s|'t|'re|'ve|'m|'ll|'d)
  if (c0 == '\'' && i + 1 < n) {
    const uint32_t a = lower(at(i + 1)), b = i + 2 < n ? lower(at(i + 2)) : 0;
    if (a == 's' || a == 't' || a == 'm' || a == 'd') return 2;
    if ((a == 'r' && b == 'e') || (a == 'v' && b == 'e') || (a == 'l' && b == 'l')) return 3;
  }
  // 2. [^\r\n\p{L}\p{N}]?\p{L}+
  {
    size_t j = i;
    if (!is_newline(c0) && !is_letter(c0) && !is_number(c0) && i + 1 < n && is_letter(c[i + 1])) j = i + 1;
    if (is_letter(at(j)) && j < n) {
      while (j < n && is_letter(c[j])) ++j;
      return j - i;
    }
  }
  // 3. \p{N}{1,3}
  if (is_number(c0)) {
    size_t j = i + 1;
    while (j < n && j < i + 3 && is_number(c[j])) ++j;
    return j - i;
  }
  // 4.  ?[^\s\p{L}\p{N}]+[\r\n]*
  {
    auto other = [&](uint32_t x) { return !is_space(x) && !is_letter(x) && !is_number(x); };
    size_t j = i;
    if (c0 == ' ' && i + 1 < n && other(c[i + 1])) j = i + 1;
    if (j < n && other(c[j])) {
      while (j < n && other(c[j])) ++j;
      while (j < n && is_newline(c[j])) ++j;
      return j - i;
    }
  }
  if (is_space(c0)) {
    size_t j = i;
    while (j < n && is_space(c[j])) ++j;      // the whitespace run [i, j)
    // 5. \s*[\r\n]+ : the longest prefix of the run that ends in a newline
    for (size_t k = j; k > i; --k)
      if (is_newline(c[k - 1])) return k - i;
    // 6. \s+(?!\S) : the run if the text ends there, else all but its last character (which must leave at least one)
    if (j == n) return j - i;
    if (j - i >= 2) return j - i - 1;
    // 7. \s+
    return j - i;
  }
  return 1;   // unreachable for valid input: every code point is a letter, a number, whitespace or "other"
}

struct PairHash {
  size_t operator()(uint64_t k) const { return static_cast<size_t>(k * 0x9E3779B97F4A7C15ull >> 17); }
};

}  // namespace
}  // namespace b200

struct b200_tokenizer {
  std::vector<std::string> id_to_token;                          // byte-level form (added tokens: their content)
  std::vector<uint8_t> is_added, is_special;
  std::unordered_map<std::string, int> vocab;                    // byte-level token string -> id
  std::unordered_map<uint64_t, std::pair<int, int>, b200::PairHash> merges;   // (left id, right id) -> (rank, merged id)
  std::vector<std::pair<std::string, int>> added;                // content -> id, longest first
  bool ignore_merges = false;
  uint32_t byte_to_cp[256];
  std::unordered_map<uint32_t, uint8_t> cp_to_byte;
  int byte_symbol[256];                                          // id of the one-byte symbol
  int bos = -1, start_header = -1, end_header = -1, eot = -1;
  // the TemplateProcessing post-processor (HF tokenizers processors/template.rs): per template, its pieces in order, each
  // sequence A (0), sequence B (1) or a special token's ids (-1).  has_template false: none, so encodings are concatenated
  // without special tokens.
  struct TplPiece {
    int seq;
    std::vector<int32_t> ids;
  };
  bool has_template = false;
  std::vector<TplPiece> tpl_single, tpl_pair;

  void bpe(const char* s, size_t n, std::vector<int32_t>* out) const;
  void encode_plain(const char* s, size_t n, std::vector<int32_t>* out) const;
  void encode(const char* s, size_t n, bool allow_special, std::vector<int32_t>* out) const;
};

void b200_tokenizer::bpe(const char* s, size_t n, std::vector<int32_t>* out) const {
  if (n == 0) return;
  std::string bl;
  bl.reserve(2 * n);
  for (size_t i = 0; i < n; ++i) b200::append_utf8(&bl, byte_to_cp[static_cast<unsigned char>(s[i])]);
  if (ignore_merges) {
    auto it = vocab.find(bl);
    if (it != vocab.end()) {
      out->push_back(it->second);
      return;
    }
  }
  // Symbols as a doubly linked list over the byte positions; candidate merges in a min-heap ordered by (rank, position of the
  // left symbol) — lowest rank first, leftmost among equals: the order tokenizers' merge queue pops (models/bpe/word.rs).  An
  // entry is stale when either symbol has since been merged away or changed; O(n log n) for a pre-token of n bytes (a single
  // "word" of a megabyte must not cost a quadratic scan).
  std::vector<int> sym(n), prev(n), next(n);
  for (size_t i = 0; i < n; ++i) {
    sym[i] = byte_symbol[static_cast<unsigned char>(s[i])];
    prev[i] = static_cast<int>(i) - 1;
    next[i] = i + 1 < n ? static_cast<int>(i) + 1 : -1;
  }
  struct Cand {
    int rank, pos, left, right, merged;
  };
  auto worse = [](const Cand& x, const Cand& y) { return x.rank != y.rank ? x.rank > y.rank : x.pos > y.pos; };
  std::vector<Cand> heap;
  auto push = [&](int pos) {
    const int nx = next[static_cast<size_t>(pos)];
    if (nx < 0) return;
    auto it = merges.find((static_cast<uint64_t>(static_cast<uint32_t>(sym[static_cast<size_t>(pos)])) << 32) | static_cast<uint32_t>(sym[static_cast<size_t>(nx)]));
    if (it == merges.end()) return;
    heap.push_back(Cand{it->second.first, pos, sym[static_cast<size_t>(pos)], sym[static_cast<size_t>(nx)], it->second.second});
    std::push_heap(heap.begin(), heap.end(), worse);
  };
  for (size_t i = 0; i + 1 < n; ++i) push(static_cast<int>(i));
  while (!heap.empty()) {
    std::pop_heap(heap.begin(), heap.end(), worse);
    const Cand c = heap.back();
    heap.pop_back();
    const size_t p = static_cast<size_t>(c.pos);
    if (sym[p] != c.left) continue;                       // the left symbol was merged away (-1) or has grown
    const int nx = next[p];
    if (nx < 0 || sym[static_cast<size_t>(nx)] != c.right) continue;
    sym[p] = c.merged;
    sym[static_cast<size_t>(nx)] = -1;
    next[p] = next[static_cast<size_t>(nx)];
    if (next[p] >= 0) prev[static_cast<size_t>(next[p])] = c.pos;
    if (prev[p] >= 0) push(prev[p]);
    push(c.pos);
  }
  for (int i = 0; i >= 0; i = next[static_cast<size_t>(i)]) out->push_back(sym[static_cast<size_t>(i)]);
}

void b200_tokenizer::encode_plain(const char* s, size_t n, std::vector<int32_t>* out) const {
  std::vector<uint32_t> cps, offs;
  b200::decode_utf8(s, n, &cps, &offs);
  size_t i = 0;
  while (i < cps.size()) {
    const size_t len = b200::next_piece(cps, i);
    bpe(s + offs[i], offs[i + len] - offs[i], out);
    i += len;
  }
}

void b200_tokenizer::encode(const char* s, size_t n, bool allow_special, std::vector<int32_t>* out) const {
  if (!allow_special || added.empty()) return encode_plain(s, n, out);
  size_t seg = 0, i = 0;
  while (i < n) {
    int hit = -1;
    size_t hit_len = 0;
    for (const auto& a : added) {   // sorted longest first: the first match at i is the longest
      if (a.first.size() <= n - i && a.first[0] == s[i] && memcmp(a.first.data(), s + i, a.first.size()) == 0) {
        hit = a.second;
        hit_len = a.first.size();
        break;
      }
    }
    if (hit < 0) {
      ++i;
      continue;
    }
    if (i > seg) encode_plain(s + seg, i - seg, out);
    out->push_back(hit);
    i += hit_len;
    seg = i;
  }
  if (n > seg) encode_plain(s + seg, n - seg, out);
}

namespace b200 {

void tokenizer_token_bytes(const b200_tokenizer* t, int32_t id, bool skip_special, std::string* out) {
  if (!t || id < 0 || static_cast<size_t>(id) >= t->id_to_token.size()) return;
  const size_t i = static_cast<size_t>(id);
  if (t->is_added[i]) {
    if (!(skip_special && t->is_special[i])) *out += t->id_to_token[i];
    return;
  }
  std::vector<uint32_t> cps, offs;
  const std::string& tok = t->id_to_token[i];
  decode_utf8(tok.data(), tok.size(), &cps, &offs);
  for (uint32_t cp : cps) {
    auto it = t->cp_to_byte.find(cp);
    if (it != t->cp_to_byte.end()) out->push_back(static_cast<char>(it->second));
  }
}
int32_t tokenizer_bos(const b200_tokenizer* t) { return t ? t->bos : -1; }

void tokenizer_encode_pair(const b200_tokenizer* t, const std::string& a, const std::string& b, bool join, bool special,
                           std::vector<int32_t>* out) {
  // HF tokenizer(text, text_pair) encodes each text on its own (added tokens in the text become their ids), then applies
  // the post-processor; tokenizer(text) the same with the single template
  std::vector<int32_t> enc[2];
  if (join) {
    const std::string ab = a + b;
    t->encode(ab.data(), ab.size(), true, &enc[0]);
  } else {
    t->encode(a.data(), a.size(), true, &enc[0]);
    t->encode(b.data(), b.size(), true, &enc[1]);
  }
  const auto& tpl = join ? t->tpl_single : t->tpl_pair;
  if (!special || !t->has_template) {
    for (auto& e : enc) out->insert(out->end(), e.begin(), e.end());
    return;
  }
  for (const auto& p : tpl) {
    const std::vector<int32_t>& src = p.seq < 0 ? p.ids : enc[p.seq];
    out->insert(out->end(), src.begin(), src.end());
  }
}
int32_t tokenizer_eot(const b200_tokenizer* t) { return t ? t->eot : -1; }

namespace {
// [0, n) -> valid UTF-8; every maximal invalid subpart (a byte that cannot start a sequence, or a lead byte with the valid
// continuation bytes that follow it when fewer than it announces) becomes ONE U+FFFD — the substitution Rust's
// String::from_utf8_lossy (hence HF tokenizers' decode) and Python's errors="replace" perform
std::string sanitize_utf8(const char* s, size_t n) {
  std::string out;
  out.reserve(n);
  auto u = [&](size_t k) { return static_cast<unsigned char>(s[k]); };
  auto cont = [&](size_t k) { return k < n && (u(k) & 0xC0) == 0x80; };
  size_t i = 0;
  while (i < n) {
    const unsigned char c = u(i);
    size_t need = 0;
    unsigned lo = 0x80, hi = 0xBF;
    if (c < 0x80) { out.push_back(static_cast<char>(c)); ++i; continue; }
    if (c >= 0xC2 && c <= 0xDF) need = 1;
    else if (c >= 0xE0 && c <= 0xEF) { need = 2; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F; }
    else if (c >= 0xF0 && c <= 0xF4) { need = 3; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F; }
    size_t got = 0;
    if (need >= 1 && i + 1 < n && u(i + 1) >= lo && u(i + 1) <= hi) {
      got = 1;
      while (got < need && cont(i + 1 + got)) ++got;
    }
    if (need > 0 && got == need) {
      out.append(s + i, need + 1);
      i += need + 1;
    } else {
      append_utf8(&out, 0xFFFD);
      i += 1 + got;
    }
  }
  return out;
}
// number of trailing bytes that are the beginning of a multi-byte sequence whose remaining bytes have not arrived yet
size_t incomplete_tail(const std::string& b) {
  const size_t n = b.size();
  for (size_t back = 1; back <= 3 && back <= n; ++back) {
    const unsigned char c = static_cast<unsigned char>(b[n - back]);
    if ((c & 0xC0) == 0x80) continue;                 // continuation byte: keep looking for its lead
    size_t need = (c & 0xE0) == 0xC0 ? 2 : (c & 0xF0) == 0xE0 ? 3 : (c & 0xF8) == 0xF0 ? 4 : 1;
    return need > back ? back : 0;                    // lead byte with fewer continuation bytes than it announces
  }
  return 0;
}
}  // namespace

std::string tokenizer_token_text(const b200_tokenizer* t, int32_t id) {
  std::string b;
  tokenizer_token_bytes(t, id, false, &b);
  return sanitize_utf8(b.data(), b.size());
}

std::string DetokStream::push(int32_t id) {
  tokenizer_token_bytes(tok, id, skip_special, &pending);
  const size_t hold = incomplete_tail(pending);
  std::string out = sanitize_utf8(pending.data(), pending.size() - hold);
  pending.erase(0, pending.size() - hold);
  return out;
}
std::string DetokStream::flush() {
  std::string out = sanitize_utf8(pending.data(), pending.size());
  pending.clear();
  return out;
}

}  // namespace b200

struct b200_detok_stream {
  b200::DetokStream s;
};

extern "C" {

b200_detok_stream* b200_tokenizer_stream_new(const b200_tokenizer* t, int32_t skip_special) {
  if (!t) return nullptr;
  auto* d = new b200_detok_stream();
  d->s.tok = t;
  d->s.skip_special = skip_special != 0;
  return d;
}
void b200_tokenizer_stream_free(b200_detok_stream* d) { delete d; }
/* id >= 0: feed one token; id < 0: flush what is held.  Returns the length of the newly complete text (copied to buf, NUL-terminated). */
int64_t b200_tokenizer_stream_push(b200_detok_stream* d, int32_t id, char* buf, size_t cap) {
  if (!d) return -1;
  const std::string out = id >= 0 ? d->s.push(id) : d->s.flush();
  if (buf && cap) {
    const size_t k = std::min(out.size(), cap - 1);
    memcpy(buf, out.data(), k);
    buf[k] = 0;
  }
  return static_cast<int64_t>(out.size());
}

int b200_tokenizer_load(const char* path, b200_tokenizer** out) {
  using namespace b200;
  if (!path || !out) { set_error("b200_tokenizer_load: bad arguments"); return B200_ERR_INVALID; }
  std::string text;
  {
    FILE* f = fopen(path, "rb");
    if (!f) { set_error("cannot open %s", path); return B200_ERR_INVALID; }
    char buf[1 << 16];
    size_t k;
    while ((k = fread(buf, 1, sizeof(buf), f)) > 0) text.append(buf, k);
    fclose(f);
  }
  JVal root;
  std::string err;
  if (!JParser(text.data(), text.size()).parse(&root, &err)) { set_error("%s: %s", path, err.c_str()); return B200_ERR_INVALID; }
  auto refuse = [&](const char* why) { set_error("%s: unsupported tokenizer (%s); only the Llama-3 byte-level BPE pipeline is implemented", path, why); return B200_ERR_INVALID; };
  const JVal* model = root.get("model");
  if (!model || !model->get("type") || model->get("type")->str != "BPE") return refuse("model.type is not BPE");
  if (const JVal* n = root.get("normalizer"); n && !n->is_null()) return refuse("a normalizer is configured");
  if (const JVal* b = model->get("byte_fallback"); b && b->type == JVal::Bool && b->b) return refuse("byte_fallback");
  for (const char* k : {"continuing_subword_prefix", "end_of_word_suffix"})
    if (const JVal* v = model->get(k); v && v->type == JVal::Str && !v->str.empty()) return refuse(k);
  // pre-tokenizer: Sequence[Split(pattern, Isolated), ByteLevel(use_regex = false)]
  {
    const JVal* pt = root.get("pre_tokenizer");
    const JVal* seq = pt ? pt->get("pretokenizers") : nullptr;
    if (!pt || !pt->get("type") || pt->get("type")->str != "Sequence" || !seq || seq->type != JVal::Arr || seq->arr.size() != 2)
      return refuse("pre_tokenizer is not Sequence[Split, ByteLevel]");
    const JVal& sp = seq->arr[0];
    const JVal& bl = seq->arr[1];
    const JVal* pat = sp.get("pattern") ? sp.get("pattern")->get("Regex") : nullptr;
    if (!sp.get("type") || sp.get("type")->str != "Split" || !pat || pat->str != kLlama3Pattern) return refuse("Split pattern is not the Llama-3 pattern");
    if (!sp.get("behavior") || sp.get("behavior")->str != "Isolated" || (sp.get("invert") && sp.get("invert")->b)) return refuse("Split behavior");
    if (!bl.get("type") || bl.get("type")->str != "ByteLevel" || (bl.get("use_regex") && bl.get("use_regex")->b) ||
        (bl.get("add_prefix_space") && bl.get("add_prefix_space")->b))
      return refuse("ByteLevel options");
  }
  if (const JVal* d = root.get("decoder"); !d || !d->get("type") || d->get("type")->str != "ByteLevel") return refuse("decoder is not ByteLevel");
  const JVal* vocab = model->get("vocab");
  const JVal* merges = model->get("merges");
  if (!vocab || vocab->type != JVal::Obj || !merges || merges->type != JVal::Arr) return refuse("vocab / merges missing");

  auto* t = new b200_tokenizer();
  // GPT-2 bytes_to_unicode: printable bytes map to themselves, the rest to U+0100...
  {
    int extra = 0;
    for (int b = 0; b < 256; ++b) {
      const bool printable = (b >= '!' && b <= '~') || (b >= 0xA1 && b <= 0xAC) || (b >= 0xAE && b <= 0xFF);
      t->byte_to_cp[b] = printable ? static_cast<uint32_t>(b) : 256u + static_cast<uint32_t>(extra++);
      t->cp_to_byte[t->byte_to_cp[b]] = static_cast<uint8_t>(b);
    }
  }
  int max_id = -1;
  for (const auto& kv : vocab->obj) {
    if (kv.second.type != JVal::Num || kv.second.num < 0 || kv.second.num > 1e8) { delete t; return refuse("vocab id"); }
    max_id = std::max(max_id, static_cast<int>(kv.second.num));
  }
  const JVal* added = root.get("added_tokens");
  if (added && added->type == JVal::Arr)
    for (const auto& a : added->arr)
      if (a.get("id") && a.get("id")->type == JVal::Num) max_id = std::max(max_id, static_cast<int>(a.get("id")->num));
  t->id_to_token.assign(static_cast<size_t>(max_id) + 1, std::string());
  t->is_added.assign(static_cast<size_t>(max_id) + 1, 0);
  t->is_special.assign(static_cast<size_t>(max_id) + 1, 0);
  t->vocab.reserve(vocab->obj.size() * 2);
  for (const auto& kv : vocab->obj) {
    const int id = static_cast<int>(kv.second.num);
    t->vocab.emplace(kv.first, id);
    t->id_to_token[static_cast<size_t>(id)] = kv.first;
  }
  for (int b = 0; b < 256; ++b) {
    std::string sym;
    append_utf8(&sym, t->byte_to_cp[b]);
    auto it = t->vocab.find(sym);
    if (it == t->vocab.end()) { delete t; return refuse("the byte-level alphabet is not in the vocab"); }
    t->byte_symbol[b] = it->second;
  }
  t->merges.reserve(merges->arr.size() * 2);
  int rank = 0;
  for (const auto& m : merges->arr) {
    std::string l, r;
    if (m.type == JVal::Arr && m.arr.size() == 2 && m.arr[0].type == JVal::Str && m.arr[1].type == JVal::Str) {
      l = m.arr[0].str;
      r = m.arr[1].str;
    } else if (m.type == JVal::Str) {   // older files: "left right"
      const size_t sp = m.str.find(' ');
      if (sp == std::string::npos) { delete t; return refuse("merge entry"); }
      l = m.str.substr(0, sp);
      r = m.str.substr(sp + 1);
    } else { delete t; return refuse("merge entry"); }
    auto il = t->vocab.find(l), ir = t->vocab.find(r), im = t->vocab.find(l + r);
    if (il == t->vocab.end() || ir == t->vocab.end() || im == t->vocab.end()) { delete t; return refuse("a merge names a token that is not in the vocab"); }
    t->merges.emplace((static_cast<uint64_t>(static_cast<uint32_t>(il->second)) << 32) | static_cast<uint32_t>(ir->second),
                      std::make_pair(rank, im->second));
    ++rank;
  }
  if (const JVal* im = model->get("ignore_merges"); im && im->type == JVal::Bool) t->ignore_merges = im->b;
  if (added && added->type == JVal::Arr) {
    for (const auto& a : added->arr) {
      const JVal* id = a.get("id");
      const JVal* content = a.get("content");
      if (!id || !content || content->type != JVal::Str || content->str.empty()) continue;
      if ((a.get("normalized") && a.get("normalized")->b) || (a.get("lstrip") && a.get("lstrip")->b) || (a.get("rstrip") && a.get("rstrip")->b) ||
          (a.get("single_word") && a.get("single_word")->b)) { delete t; return refuse("added token options (normalized / strip / single_word)"); }
      const size_t i = static_cast<size_t>(id->num);
      t->id_to_token[i] = content->str;
      t->is_added[i] = 1;
      t->is_special[i] = a.get("special") && a.get("special")->b;
      t->added.emplace_back(content->str, static_cast<int>(i));
    }
    std::stable_sort(t->added.begin(), t->added.end(), [](const auto& x, const auto& y) { return x.first.size() > y.first.size(); });
  }
  auto find_added = [&](const char* s) {
    for (const auto& a : t->added)
      if (a.first == s) return a.second;
    return -1;
  };
  // post_processor: a TemplateProcessing, alone or inside a Sequence (Llama-3: Sequence[ByteLevel, TemplateProcessing]);
  // any other processor adds no token ids to a byte-level BPE encoding and is ignored, as is the absence of one
  {
    const JVal* pp = root.get("post_processor");
    const JVal* tp = nullptr;
    if (pp && pp->type == JVal::Obj && pp->get("type") && pp->get("type")->str == "TemplateProcessing") tp = pp;
    else if (pp && pp->type == JVal::Obj && pp->get("type") && pp->get("type")->str == "Sequence" && pp->get("processors") &&
             pp->get("processors")->type == JVal::Arr)
      for (const auto& q : pp->get("processors")->arr)
        if (q.type == JVal::Obj && q.get("type") && q.get("type")->str == "TemplateProcessing") tp = &q;
    if (tp) {
      const JVal* specials = tp->get("special_tokens");
      auto parse = [&](const char* key, std::vector<b200_tokenizer::TplPiece>* out) {
        const JVal* arr = tp->get(key);
        if (!arr || arr->type != JVal::Arr) return false;
        for (const auto& piece : arr->arr) {
          if (const JVal* sq = piece.get("Sequence")) {
            const JVal* id = sq->get("id");
            if (!id || id->type != JVal::Str || (id->str != "A" && id->str != "B")) return false;
            out->push_back({id->str == "A" ? 0 : 1, {}});
          } else if (const JVal* sp = piece.get("SpecialToken")) {
            const JVal* id = sp->get("id");
            const JVal* st = id && id->type == JVal::Str && specials ? specials->get(id->str.c_str()) : nullptr;
            const JVal* ids = st ? st->get("ids") : nullptr;
            if (!ids || ids->type != JVal::Arr) return false;
            b200_tokenizer::TplPiece p{-1, {}};
            for (const auto& v : ids->arr) {
              if (v.type != JVal::Num || v.num < 0 || v.num >= static_cast<double>(t->id_to_token.size())) return false;
              p.ids.push_back(static_cast<int32_t>(v.num));
            }
            out->push_back(std::move(p));
          } else {
            return false;
          }
        }
        return true;
      };
      if (!parse("single", &t->tpl_single) || !parse("pair", &t->tpl_pair)) { delete t; return refuse("post_processor TemplateProcessing"); }
      t->has_template = true;
    }
  }
  t->bos = find_added("<|begin_of_text|>");
  t->start_header = find_added("<|start_header_id|>");
  t->end_header = find_added("<|end_header_id|>");
  t->eot = find_added("<|eot_id|>");
  *out = t;
  return 0;
}

void b200_tokenizer_destroy(b200_tokenizer* t) { delete t; }

int32_t b200_tokenizer_vocab_size(const b200_tokenizer* t) { return t ? static_cast<int32_t>(t->id_to_token.size()) : 0; }

int32_t b200_tokenizer_token_id(const b200_tokenizer* t, const char* content) {
  if (!t || !content) return -1;
  for (const auto& a : t->added)
    if (a.first == content) return a.second;
  auto it = t->vocab.find(content);
  return it == t->vocab.end() ? -1 : it->second;
}

int64_t b200_tokenizer_encode(const b200_tokenizer* t, const char* text, size_t len, int32_t allow_special, int32_t* ids, size_t cap) {
  if (!t || (!text && len)) return -1;
  std::vector<int32_t> out;
  t->encode(text, len, allow_special != 0, &out);
  for (size_t i = 0; i < out.size() && i < cap; ++i) ids[i] = out[i];
  return static_cast<int64_t>(out.size());
}

int64_t b200_tokenizer_encode_pair(const b200_tokenizer* t, const char* a, size_t alen, const char* b, size_t blen,
                                   int32_t join, int32_t add_special_tokens, int32_t* ids, size_t cap) {
  if (!t || (!a && alen) || (!b && blen)) return -1;
  std::vector<int32_t> out;
  b200::tokenizer_encode_pair(t, std::string(a ? a : "", alen), std::string(b ? b : "", blen), join != 0,
                              add_special_tokens != 0, &out);
  for (size_t i = 0; i < out.size() && i < cap; ++i) ids[i] = out[i];
  return static_cast<int64_t>(out.size());
}

int64_t b200_tokenizer_decode(const b200_tokenizer* t, const int32_t* ids, size_t n, int32_t skip_special, char* buf, size_t cap) {
  if (!t || (!ids && n)) return -1;
  std::string out;
  for (size_t i = 0; i < n; ++i) {
    if (ids[i] < 0 || static_cast<size_t>(ids[i]) >= t->id_to_token.size()) continue;
    const size_t id = static_cast<size_t>(ids[i]);
    if (t->is_added[id]) {
      if (!(skip_special && t->is_special[id])) out += t->id_to_token[id];
      continue;
    }
    std::vector<uint32_t> cps, offs;
    const std::string& tok = t->id_to_token[id];
    b200::decode_utf8(tok.data(), tok.size(), &cps, &offs);
    for (uint32_t cp : cps) {
      auto it = t->cp_to_byte.find(cp);
      if (it != t->cp_to_byte.end()) out.push_back(static_cast<char>(it->second));
    }
  }
  if (buf && cap) {
    const size_t k = std::min(out.size(), cap - 1);
    memcpy(buf, out.data(), k);
    buf[k] = 0;
  }
  return static_cast<int64_t>(out.size());
}

// Llama-3 instruct framing (the checkpoint's chat_template): <|begin_of_text|> then per message
// <|start_header_id|>role<|end_header_id|>\n\n + trimmed content + <|eot_id|>, and the assistant header when a reply is wanted.
int64_t b200_tokenizer_chat_llama3(const b200_tokenizer* t, const char* const* roles, const char* const* contents, int32_t n,
                                   int32_t add_generation_prompt, int32_t* ids, size_t cap) {
  if (!t || n < 0 || (n && (!roles || !contents))) return -1;
  if (t->bos < 0 || t->start_header < 0 || t->end_header < 0 || t->eot < 0) {
    b200::set_error("the tokenizer has no Llama-3 header / eot tokens");
    return -1;
  }
  std::vector<int32_t> out;
  auto trim = [](const char* s) {
    std::string x = s ? s : "";
    // jinja `trim` == Python str.strip(): ASCII whitespace and the Unicode spaces of kUnicodeSpace
    std::vector<uint32_t> cps, offs;
    b200::decode_utf8(x.data(), x.size(), &cps, &offs);
    size_t a = 0, b = cps.size();
    auto sp = [](uint32_t c) { return b200::is_space(c) || (c >= 0x1C && c <= 0x1F); };
    while (a < b && sp(cps[a])) ++a;
    while (b > a && sp(cps[b - 1])) --b;
    return x.substr(offs[a], offs[b] - offs[a]);
  };
  out.push_back(t->bos);
  for (int i = 0; i < n; ++i) {
    out.push_back(t->start_header);
    t->encode(roles[i], strlen(roles[i]), false, &out);
    out.push_back(t->end_header);
    const std::string body = "\n\n" + trim(contents[i]);
    t->encode(body.data(), body.size(), true, &out);
    out.push_back(t->eot);
  }
  if (add_generation_prompt) {
    out.push_back(t->start_header);
    t->encode("assistant", 9, false, &out);
    out.push_back(t->end_header);
    t->encode("\n\n", 2, false, &out);
  }
  for (size_t i = 0; i < out.size() && i < cap; ++i) ids[i] = out[i];
  return static_cast<int64_t>(out.size());
}

}  // extern "C"
