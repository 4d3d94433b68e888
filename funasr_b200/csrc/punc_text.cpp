// Host text side of CT-Transformer punctuation (no CUDA in this file): funasr_b200/punc.py:CTTransformerB200.inference restated in C++,
// the way vad_detector.cpp restates vad.py.  punc.py stays the readable specification; tests/test_offline_punc_host.py pins this walk
// to it and to the reference's goldens.  The one change of shape: the reference punctuates one text at a time, one window per forward;
// here every text advances one window per step, and all the windows of a step are scored as one padded batch.  The per-text state
// (carried tail, text so far, punctuation ids) evolves exactly as it does alone, since a window's scores depend on that window only.
#include "punc_text.h"

#include <ctype.h>
#include <algorithm>

namespace fa_punc {

namespace {

// length of the UTF-8 sequence that starts with byte c (a stray continuation byte counts as one)
int seq_len(unsigned char c) { return c < 0xC0 ? 1 : c < 0xE0 ? 2 : c < 0xF0 ? 3 : 4; }

uint32_t code_point(const std::string& s, size_t i, int len) {
  if (len == 1) return (unsigned char)s[i];
  uint32_t v = (unsigned char)s[i] & (0xFF >> (len + 1));
  for (int k = 1; k < len; ++k) v = (v << 6) | ((unsigned char)s[i + k] & 0x3F);
  return v;
}

// str.isspace() of CPython: the separators str.split() uses
bool py_space(uint32_t c) {
  return (c >= 0x09 && c <= 0x0D) || (c >= 0x1C && c <= 0x20) || c == 0x85 || c == 0xA0 || c == 0x1680 || (c >= 0x2000 && c <= 0x200A) ||
         c == 0x2028 || c == 0x2029 || c == 0x202F || c == 0x205F || c == 0x3000;
}

bool latin(const std::string& w) { return !w.empty() && (unsigned char)w[0] < 0x80; }

// the last code point of s and its byte offset
std::string last_char(const std::string& s, size_t* at) {
  size_t i = s.size();
  while (i > 0 && ((unsigned char)s[i - 1] & 0xC0) == 0x80) --i;
  if (i > 0) --i;
  if (i < s.size() && ((unsigned char)s[i] & 0xC0) == 0x80) i = s.size() - 1;   // no lead byte: the last byte alone
  *at = i;
  return s.substr(i);
}

}  // namespace

bool Vocab::init(const std::vector<std::string>& tokens, const std::vector<std::string>& punc_list, int32_t sentence_end, int32_t split,
                 std::string& err) {
  token_id.clear();
  for (size_t i = 0; i < tokens.size(); ++i)
    if (!token_id.emplace(tokens[i], (int32_t)i).second) { err = "token \"" + tokens[i] + "\" is duplicated"; return false; }   // abs_tokenizer.py:72-75
  auto it = token_id.find("<unk>");
  if (it == token_id.end()) { err = "the token list has no <unk> entry"; return false; }
  unk = it->second;
  punc = punc_list;
  if (sentence_end < 0 || sentence_end >= (int32_t)punc.size()) { err = "sentence_end_id outside the punctuation list"; return false; }
  if (split < 2) { err = "split_size must be at least 2"; return false; }
  sentence_end_id = sentence_end;
  split_size = split;
  return true;
}

std::vector<std::string> split_words(const std::string& s) {
  std::vector<std::string> words;
  std::string cur;
  size_t i = 0;
  while (i < s.size()) {
    const int len = std::min<int>(seq_len((unsigned char)s[i]), (int)(s.size() - i));
    const uint32_t c = code_point(s, i, len);
    if (py_space(c)) {
      if (!cur.empty()) { words.push_back(cur); cur.clear(); }
    } else if (c < 0x80) {
      cur += (char)c;
    } else {
      if (!cur.empty()) { words.push_back(cur); cur.clear(); }
      words.push_back(s.substr(i, len));
    }
    i += len;
  }
  if (!cur.empty()) words.push_back(cur);
  return words;
}

Text admit(const Vocab& v, const char* text) {
  Text x;
  x.words = split_words(text ? text : "");
  x.ids.reserve(x.words.size());
  for (const std::string& w : x.words) {                    // tokens2ids: exact lookup, unknown -> <unk>
    auto it = v.token_id.find(w);
    x.ids.push_back(it != v.token_id.end() ? it->second : v.unk);
  }
  const int64_t nw = (int64_t)x.words.size();
  x.n_windows = (nw + v.split_size - 1) / v.split_size;    // an empty or whitespace-only text: no window, "" and no ids
  return x;
}

int64_t window_len(const Vocab& v, const Text& x) {
  return (int64_t)x.cache_ids.size() + std::min<int64_t>(v.split_size, (int64_t)x.words.size() - x.next * v.split_size);
}

bool check_window(const Vocab& v, const Text& x, int32_t index, int64_t max_window, std::string& err) {
  const int64_t len = window_len(v, x);
  if (max_window <= 0 || len <= max_window) return true;
  err = "text " + std::to_string(index) + ": window " + std::to_string(x.next) + " holds " + std::to_string(len) +
        " words (an unfinished sentence carried over), more than the attention kernel takes (" + std::to_string(max_window) + ")";
  return false;
}

void compose(const Vocab& v, const std::vector<Text*>& rows, Step& s) {
  const int64_t split = v.split_size;
  int64_t t_max = 0;
  for (const Text* x : rows) t_max = std::max(t_max, window_len(v, *x));
  const int32_t B = (int32_t)rows.size();
  s.batch = B;
  s.t_max = (int32_t)t_max;
  s.ids.assign((size_t)B * t_max, 0);
  s.lens.assign((size_t)B, 0);
  s.pout.assign((size_t)B * t_max, 0);
  for (int32_t b = 0; b < B; ++b) {
    const Text& x = *rows[b];
    int32_t* row = s.ids.data() + (size_t)b * t_max;
    std::copy(x.cache_ids.begin(), x.cache_ids.end(), row);
    const int64_t w0 = x.next * split, w1 = std::min<int64_t>(w0 + split, (int64_t)x.ids.size());
    std::copy(x.ids.begin() + w0, x.ids.begin() + w1, row + x.cache_ids.size());
    s.lens[b] = (int32_t)(x.cache_ids.size() + (w1 - w0));
  }
}

bool apply(const Vocab& v, Text& x, const Step& s, int32_t b, std::string& err) {
  const std::vector<std::string>& pl = v.punc;
  auto is = [&](int32_t p, const char* str) { return pl[p] == str; };
  const int64_t split = v.split_size;
  const int64_t L = s.lens[b], w0 = x.next * split, w1 = std::min<int64_t>(w0 + split, (int64_t)x.ids.size());
  std::vector<int32_t> p(s.pout.begin() + (size_t)b * s.t_max, s.pout.begin() + (size_t)b * s.t_max + L);
  for (int32_t q : p)
    if (q < 0 || q >= (int32_t)pl.size()) { err = "scorer returned punctuation id " + std::to_string(q) + " outside the list"; return false; }
  std::vector<std::string> ms(x.cache_words);
  ms.insert(ms.end(), x.words.begin() + w0, x.words.begin() + w1);
  std::vector<int32_t> mi(x.cache_ids);
  mi.insert(mi.end(), x.ids.begin() + w0, x.ids.begin() + w1);
  const bool last = x.next == x.n_windows - 1;
  if (!last) {                                             // carry the unfinished tail over (model.py:350-374)
    int64_t end = -1, comma = -1;
    for (int64_t i = L - 2; i > 1; --i) {
      if (is(p[i], "。") || is(p[i], "？")) { end = i; break; }
      if (comma < 0 && is(p[i], "，")) comma = i;
    }
    if (end < 0 && L > 200 && comma >= 0) {               // cache_pop_trigger_limit: cut a long sentence at its last comma
      end = comma;
      p[end] = v.sentence_end_id;
    }
    x.cache_words.assign(ms.begin() + (end + 1), ms.end());
    x.cache_ids.assign(mi.begin() + (end + 1), mi.end());
    ms.resize((size_t)(end + 1));
    p.resize((size_t)(end + 1));
  } else {
    x.cache_words.clear();
    x.cache_ids.clear();
  }
  std::string piece;                                       // model.py:382-409
  for (size_t i = 0; i < ms.size(); ++i) {
    std::string& w = ms[i];
    const bool lat = latin(w);
    if ((i == 0 || is(p[i - 1], "。") || is(p[i - 1], "？")) && lat) {   // str.capitalize() of an ASCII word
      w[0] = (char)toupper((unsigned char)w[0]);
      for (size_t k = 1; k < w.size(); ++k) w[k] = (char)tolower((unsigned char)w[k]);
    }
    if (i == 0 && lat) w = " " + w;
    if (i > 0 && lat && latin(ms[i - 1])) w = " " + w;
    piece += w;
    if (pl[p[i]] != "_") {
      std::string r = pl[p[i]];
      if (lat) r = r == "，" ? "," : r == "。" ? "." : r == "？" ? "?" : r;
      piece += r;
    }
  }
  x.text += piece;
  if (last) {                                              // forced sentence end (model.py:413-449)
    size_t at = 0;
    const std::string c = last_char(x.text, &at);
    bool force = true;
    if (c == "，" || c == "、") x.text = x.text.substr(0, at) + "。";
    else if (c == ",") x.text = x.text.substr(0, at) + ".";
    else if (c != "。" && c != "？" && c.size() != 1) x.text += "。";
    else if (c != "." && c != "?" && c.size() == 1) x.text += ".";
    else force = false;
    if (force && !p.empty()) p.back() = v.sentence_end_id;
  }
  x.punc.insert(x.punc.end(), p.begin(), p.end());
  ++x.next;
  return true;
}

bool walk(const Vocab& v, const char* const* texts, int32_t n, int64_t max_window, const Scorer& score, Result& out, std::string& err) {
  std::vector<Text> st;
  st.reserve((size_t)n);
  for (int32_t t = 0; t < n; ++t) st.push_back(admit(v, texts[t]));
  std::vector<Text*> rows;
  Step s;
  out.steps = 0;
  for (;;) {
    rows.clear();
    for (int32_t t = 0; t < n; ++t) {
      if (!st[t].active()) continue;
      if (!check_window(v, st[t], t, max_window, err)) return false;
      rows.push_back(&st[t]);
    }
    if (rows.empty()) break;
    compose(v, rows, s);
    if (!score(s.ids.data(), s.lens.data(), s.batch, s.t_max, s.pout.data(), err)) return false;
    ++out.steps;
    for (int32_t b = 0; b < s.batch; ++b)
      if (!apply(v, *rows[b], s, b, err)) return false;
  }
  out.text.resize((size_t)n);
  out.ids.resize((size_t)n);
  for (int32_t t = 0; t < n; ++t) {
    out.text[t].swap(st[t].text);
    out.ids[t].swap(st[t].punc);
  }
  return true;
}

}  // namespace fa_punc
