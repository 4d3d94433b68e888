// FunOffline* — the OfflineStream entry points of FunASR's C++ runtime (runtime/onnxruntime/include/funasrruntime.h:100-116) with
// their exact C++ signatures, over this library's handle API (offline_asr.cu / offline_long.cu: fa_offline_*).  Host-only C++: file / buffer decoding
// (raw s16le PCM, RIFF WAV PCM16 / float32), the hotword encoder of ContextualParaformer (Embedding + 1-layer LSTM, O(#hotwords):
// the reference runs it on the CPU too — model_eb.onnx, runtime/onnxruntime/src/paraformer.cpp CompileHotwordEmbedding) and the
// ids -> text join.  Everything per audio frame runs in fa_offline_infer_audio on the GPU — or, with a VAD model ("vad-dir"), in
// fa_offline_infer_vad_audio.  FsmnVad* are the runtime's VAD entry points over fa_vad_infer_audio.
//
// Sample rates: audio at any rate (sampling_rate for "pcm", the header's for a WAV file or "wav" buffer) is resampled to 16 kHz on
// the device with FA_RESAMPLE_RUNTIME, the runtime's LinearResample.  One known difference: the runtime sends "wav" BUFFERS through
// ffmpeg (swresample) when it is built with it; the shim uses LinearResample for them as for everything else.
//
// SeACo (paraformer-zh): CompileHotwordEmbedding parses the hotword string as for ContextualParaformer and takes the rows from the
// handle's GPU hotword encoder (fa_offline_hotword_embed); FunOfflineInferBuffer passes them on, with or without "vad-dir".
//
// Timestamps: with a BiCifParaformer model file FunASRGetStamp returns the runtime's "[[b,e],[b,e],...]" (integer ms, absolute with
// "vad-dir"; funasrruntime.cpp:297-310), one pair per stamp of fa_offline_result_stamps.  The values are the library's one timestamp
// definition, the one the reference's Python BiCifParaformer produces (timestamp_tools.py:ts_prediction_lfr6_standard): the shim does
// not restate the runtime's own TimestampOnnx (util.cpp:838-965), which cuts tokens at 30 frames instead of 12, re-integrates in fp32
// with a tail fix-up and re-parses seconds strings to ms.  With "punc-dir" FunASRGetStampSents is the runtime's TimestampSentence over
// the punctuated text and those stamps; without it, it stays empty.
//
// Punctuation: with model_path["punc-dir"] FunOfflineInfer / FunOfflineInferBuffer punctuate each result text after the join, with or
// without "vad-dir" (funasrruntime.cpp:311-314), through fa_punc_infer; CTTransformer* are the runtime's offline punctuation entry
// points over the same handle.
#include "../../include/funasrruntime_b200.h"
#include "../../include/funasr_b200.h"

#include <math.h>
#include <stdio.h>
#include <string.h>
#include <fstream>
#include <sstream>

namespace {

thread_local std::string g_shim_err;

struct OfflineStream {
  void* h = nullptr;
  void* vad = nullptr;                 // fa_vad_init handle when model_path["vad-dir"] is given
  void* punc = nullptr;                // fa_punc_init handle when model_path["punc-dir"] is given
  int batch_size_s = 300;
  std::vector<std::string> vocab;
  std::unordered_map<std::string, int> token_id;
  int batch = 1;
};

struct VadStream {
  void* v = nullptr;
};

struct VadShimResult {
  std::vector<std::vector<int>> segments;
  float snippet_time = 0.f;
};

// the C++ runtime's VAD reads a fixed max_end_silence_time from its config (fsmn-vad.cpp) and has no dynamic schedule
FaVadRunOptions runtime_vad_options() {
  FaVadRunOptions o;
  o.dynamic_silence = 0; o.max_end_silence_time = 0; o.speech_noise_thres = NAN;
  return o;
}

int parse_device(std::map<std::string, std::string>& model_path) {
  auto gi = model_path.find("gpu-id");
  return gi != model_path.end() ? atoi(gi->second.c_str()) : 0;
}

struct ShimResult {
  std::vector<std::string> msgs;
  std::string stamp, stamp_sents;
  float snippet_time = 0.f;
};

// TimestampSentence of the C++ runtime (runtime/onnxruntime/src/util.cpp:569-637): the punctuated text split as
// TimestampSplitChiEngCharacters does (EncodeConverter's UTF-8 -> UTF-16 units: 3- and 2-byte sequences only, any other byte one 0
// unit that adds nothing; CJK, digits and the unit punctuation ranges are one character each, spaces split Latin words), the stamps of
// "[[b,e],...]" dealt out to the non-punctuation characters, one JSON object per punctuation mark (the bytewise TimestampIsPunctuation)
// and one for a tail without it.  tests/stampsent_ref.py restates the same function in Python, pinned to the compiled runtime.
bool unit_punc(uint32_t u) {
  if (u == 0x26 || u == 0x27 || u == 0x2D) return false;
  return (u >= 0x21 && u <= 0x2F) || (u >= 0x3A && u <= 0x40) || (u >= 0x5B && u <= 0x60) || (u >= 0x7B && u <= 0x7E) ||
         (u >= 0x2000 && u <= 0x206F) || (u >= 0x3000 && u <= 0x303F);
}

std::string unit_utf8(uint32_t u) {
  std::string s;
  if (u < 0x80) s += (char)u;
  else if (u < 0x800) { s += (char)(0xC0 | (u >> 6)); s += (char)(0x80 | (u & 0x3F)); }
  else { s += (char)(0xE0 | (u >> 12)); s += (char)(0x80 | ((u >> 6) & 0x3F)); s += (char)(0x80 | (u & 0x3F)); }
  return s;
}

std::vector<std::string> split_chi_eng(const std::string& text) {
  std::vector<std::string> chars;
  std::string eng;
  const unsigned char* b = reinterpret_cast<const unsigned char*>(text.data());
  const size_t n = text.size();
  auto flush = [&] { if (!eng.empty()) { chars.push_back(eng); eng.clear(); } };
  for (size_t i = 0; i < n;) {
    uint32_t u = 0;
    size_t step = 1;
    if ((b[i] & 0xF0) == 0xE0 && n - i >= 3) {
      if ((b[i + 1] & 0xC0) == 0x80 && (b[i + 2] & 0xC0) == 0x80) {
        u = ((b[i] & 0x0Fu) << 12) | ((b[i + 1] & 0x3Fu) << 6) | (b[i + 2] & 0x3Fu);
        if (u >= 0x800) step = 3; else u = 0;
      }
    } else if ((b[i] & 0xE0) == 0xC0 && n - i >= 2) {
      if ((b[i + 1] & 0xC0) == 0x80) {
        u = ((b[i] & 0x1Fu) << 6) | (b[i + 1] & 0x3Fu);
        if (u >= 0x80) step = 2; else u = 0;
      }
    } else if (b[i] < 0x80) {
      u = b[i];
    }
    i += step;
    if ((u >= 0x4E00 && u <= 0x9FFF) || (u >= 0x3400 && u <= 0x4DFF) || (u >= 0x30 && u <= 0x39) || unit_punc(u)) {
      flush();
      chars.push_back(unit_utf8(u));
    } else if (u == 0x20) {
      flush();
    } else if (u != 0) {
      eng += unit_utf8(u);
    }
  }
  flush();
  return chars;
}

bool is_punctuation(const std::string& s) {
  static const std::string punc = "，。？、,?";
  for (char c : s) if (punc.find(c) == std::string::npos) return false;
  return true;
}

std::string render_pairs(const std::vector<std::pair<int, int>>& v) {
  std::string s = "[";
  for (size_t i = 0; i < v.size(); ++i) s += (i ? ",[" : "[") + std::to_string(v[i].first) + "," + std::to_string(v[i].second) + "]";
  return s + "]";
}

std::string timestamp_sentence(const std::string& text, const void* r, int32_t index) {
  int32_t n_ts = 0;
  const int32_t* p = fa_offline_result_stamps(r, index, &n_ts);   // the pairs FunASRGetStamp renders, without the round trip
  const std::vector<std::string> chars = split_chi_eng(text);
  int idx_ts = 0, start = -1, end = -1;
  std::string text_seg, out;
  std::vector<std::pair<int, int>> seg;
  for (size_t i = 0; i < chars.size(); ++i) {
    if (is_punctuation(chars[i])) {
      if (!seg.empty()) { start = seg.front().first; end = seg.back().second; }
      out += "{\"text_seg\":\"" + text_seg + "\",\"punc\":\"" + chars[i] + "\",\"start\":" + std::to_string(start) + ",\"end\":" +
             std::to_string(end) + ",\"ts_list\":" + render_pairs(seg) + "}";
      if (i != chars.size() - 1) out += ",";
      text_seg.clear(); start = 0; end = 0; seg.clear();
    } else if (idx_ts < n_ts) {
      text_seg = text_seg.empty() ? chars[i] : text_seg + " " + chars[i];
      seg.emplace_back(p[2 * idx_ts], p[2 * idx_ts + 1]);
      ++idx_ts;
    }
  }
  if (!seg.empty())
    out += "{\"text_seg\":\"" + text_seg + "\",\"punc\":\"\",\"start\":" + std::to_string(seg.front().first) + ",\"end\":" +
           std::to_string(seg.back().second) + ",\"ts_list\":" + render_pairs(seg) + "}";
  return "[" + out + "]";
}

struct PuncShimResult {
  std::string msg;
};

// every text of `msgs` replaced by its punctuated form, in one fa_punc_infer call
bool punctuate(void* punc, std::vector<std::string>& msgs) {
  if (msgs.empty()) return true;
  std::vector<const char*> texts;
  for (const std::string& m : msgs) texts.push_back(m.c_str());
  void* r = fa_punc_infer(punc, texts.data(), (int32_t)texts.size());
  if (!r) { g_shim_err = fa_offline_last_error(); return false; }
  for (size_t i = 0; i < msgs.size(); ++i) msgs[i] = fa_punc_result_text(r, (int32_t)i);
  fa_punc_free_result(r);
  return true;
}

// "[[b,e],[b,e],...]" of entry `index` of a handle result; "" without stamps, as the runtime leaves it
std::string render_stamps(const void* r, int32_t index) {
  int32_t n = 0;
  const int32_t* p = fa_offline_result_stamps(r, index, &n);
  std::string s;
  for (int32_t i = 0; i < n; ++i) s += (i ? ",[" : "[[") + std::to_string(p[2 * i]) + "," + std::to_string(p[2 * i + 1]) + "]";
  return n ? s + "]" : s;
}

bool is_ascii_word(const std::string& s) {
  if (s.empty()) return false;
  for (unsigned char c : s) if (c >= 0x80) return false;
  return true;
}

// tokens -> text: word pieces ending in "@@" are glued to the next token, consecutive ASCII words are separated by one space,
// CJK tokens are concatenated.  A plain join in the spirit of the runtime's Vocab::Vector2StringV2 (runtime/onnxruntime/src/vocab.cpp:
// 164-278) for Paraformer's char / word vocabulary — NOT a restatement of it: that function also drops <s> / </s> / <unk>, keeps
// runs of single letters unspaced, repairs "xx@@" before a CJK token and has an en-bpe mode.  Text post-processing is CPU string
// work outside the accelerated path (DESIGN.md §7); the ids this shim returns are the parity-checked output.
std::string join_tokens(const OfflineStream& s, const int32_t* ids, int n) {
  std::string out;
  bool prev_ascii = false, glue = false;
  for (int i = 0; i < n; ++i) {
    std::string tok = (ids[i] >= 0 && ids[i] < (int)s.vocab.size()) ? s.vocab[ids[i]] : std::to_string(ids[i]);
    if (s.vocab.empty()) tok = std::to_string(ids[i]);
    bool next_glue = false;
    if (tok.size() > 2 && tok.compare(tok.size() - 2, 2, "@@") == 0) { tok.resize(tok.size() - 2); next_glue = true; }
    const bool ascii = is_ascii_word(tok);
    if (!out.empty() && !glue && ascii && prev_ascii) out += ' ';
    out += tok;
    prev_ascii = ascii;
    glue = next_glue;
  }
  return out;
}

// UTF-8 aware split of one hotword into vocabulary units: ASCII runs are one (lower-cased) unit, every other code point is one unit
std::vector<std::string> split_units(const std::string& w) {
  std::vector<std::string> u;
  size_t i = 0;
  while (i < w.size()) {
    const unsigned char c = (unsigned char)w[i];
    if (c < 0x80) {
      std::string a;
      while (i < w.size() && (unsigned char)w[i] < 0x80) { a += (char)tolower(w[i]); ++i; }
      u.push_back(a);
    } else {
      const int len = c >= 0xF0 ? 4 : (c >= 0xE0 ? 3 : 2);
      u.push_back(w.substr(i, len));
      i += len;
    }
  }
  return u;
}

// The hotword token lists of one hotword string (generate_hotwords_list for ContextualParaformer and SeacoParaformer alike): each
// whitespace-separated hotword split into vocabulary units (split_units, tokens.txt; decimal ids without it), a hotword with a unit
// outside the vocabulary dropped, then the <s> entry {1}
std::vector<std::vector<int>> hotword_lists(const OfflineStream& s, const std::string& hotwords, int vocab) {
  std::vector<std::vector<int>> lists;
  std::stringstream ss(hotwords);
  std::string w;
  while (ss >> w) {
    std::vector<int> ids;
    bool ok = true;
    for (const std::string& u : split_units(w)) {
      int id = -1;
      auto it = s.token_id.find(u);
      if (it != s.token_id.end()) id = it->second;
      else if (s.vocab.empty()) id = atoi(u.c_str());                   // no vocabulary file: decimal token ids
      if (id < 0 || id >= vocab) { ok = false; break; }
      ids.push_back(id);
    }
    if (ok && !ids.empty()) lists.push_back(ids);                      // hotwords with out-of-vocabulary units are dropped
  }
  lists.push_back({1});                                                // <s>
  return lists;
}

inline float sigm(float x) { return 1.0f / (1.0f + expf(-x)); }

// SenseVoice: the runtime's lid_map (sensevoice-small.h:110-118); an unknown svs_lang is "auto" (sensevoice-small.cpp:458-465)
const std::map<std::string, int32_t> kSvLidMap = {{"auto", 0}, {"zh", 3}, {"en", 4}, {"yue", 7}, {"ja", 11}, {"ko", 12}, {"nospeech", 13}};

// SenseVoiceSmall::CTCSearch (sensevoice-small.cpp:305-355) after its arg-max and collapse, over the handle's ids.  The runtime reads
// tokens[3] whenever it has at least 3 tokens, one past the end with exactly 3; here that fourth tag is empty.
std::string sv_ctc_text(const int32_t* ids, int n, const std::vector<std::string>& vocab) {
  auto piece = [&](int32_t id) { return id >= 0 && id < (int32_t)vocab.size() ? vocab[id] : std::to_string(id); };
  std::string lang, emo, event, itn, text;
  if (n >= 3) { lang = piece(ids[0]); emo = piece(ids[1]); event = piece(ids[2]); }
  if (n >= 4) itn = piece(ids[3]);
  for (int i = 4; i < n; ++i) {
    const std::string w = piece(ids[i]);
    text += w.find("\xe2\x96\x81") != std::string::npos ? " " + w.substr(3) : w;      // U+2581, three bytes
  }
  if (itn == "<|withitn|>") text += lang == "<|zh|>" ? "\xe3\x80\x82" : ".";              // U+3002
  return lang + emo + event + " " + text;
}

FaLongAudioOptions runtime_long_audio_options(const OfflineStream& s) {
  FaLongAudioOptions o;
  o.batch_size_s = s.batch_size_s; o.batch_size_threshold_s = 60; o.merge_vad = 0; o.merge_length_s = 15; o.vad = runtime_vad_options();
  return o;
}

// a SenseVoice handle: the query from svs_lang / svs_itn, each segment's CTCSearch text concatenated in time order without a separator
// (funasrruntime.cpp:287-296 for a language other than en-bpe); punctuation, ITN and stamps do not apply (offline-stream.cpp:147-150)
FUNASR_RESULT infer_sv(OfflineStream* s, const void* const* bufs, const int64_t* lens, const FaAudioFormat& fmt, const std::string& svs_lang,
                       bool svs_itn) {
  auto it = kSvLidMap.find(svs_lang);
  const int32_t lid = it != kSvLidMap.end() ? it->second : 0, itn = svs_itn ? 14 : 15;
  const FaLongAudioOptions o = runtime_long_audio_options(*s);
  void* r = s->vad ? fa_offline_infer_vad_audio(s->h, s->vad, nullptr, bufs, lens, 1, &fmt, nullptr, 0, &lid, &itn, &o, 0)
                   : fa_offline_infer_audio(s->h, bufs, lens, 1, &fmt, nullptr, 0, &lid, &itn);
  if (!r) { g_shim_err = fa_offline_last_error(); return nullptr; }
  int32_t k = 0, nseg = 0;
  const int32_t* ids = fa_offline_result_ids(r, 0, &k);
  std::string text;
  if (s->vad) {
    const int32_t* seg = fa_offline_result_segments(r, 0, &nseg);
    for (int32_t i = 0, pos = 0; i < nseg; ++i) {
      text += sv_ctc_text(ids + pos, seg[3 * i + 2], s->vocab);
      pos += seg[3 * i + 2];
    }
  } else {
    text = sv_ctc_text(ids, k, s->vocab);
  }
  ShimResult* out = new ShimResult();
  out->msgs.push_back(text);
  out->snippet_time = fa_offline_result_audio_seconds(r);
  fa_offline_free_result(r);
  return out;
}

// RIFF WAVE: returns the PCM payload and its format (1 = s16le, 0 = float32); mono or the first channel layout is required
bool parse_wav(const std::string& bytes, const char** data, size_t* n_bytes, int* fmt, int* rate) {
  if (bytes.size() < 44 || memcmp(bytes.data(), "RIFF", 4) != 0 || memcmp(bytes.data() + 8, "WAVE", 4) != 0) return false;
  size_t pos = 12;
  int channels = 1, bits = 16, tag = 1;
  *rate = 16000;
  while (pos + 8 <= bytes.size()) {
    uint32_t sz;
    memcpy(&sz, bytes.data() + pos + 4, 4);
    if (memcmp(bytes.data() + pos, "fmt ", 4) == 0 && pos + 8 + 16 <= bytes.size()) {
      uint16_t t, ch, b;
      uint32_t r;
      memcpy(&t, bytes.data() + pos + 8, 2); memcpy(&ch, bytes.data() + pos + 10, 2); memcpy(&r, bytes.data() + pos + 12, 4);
      memcpy(&b, bytes.data() + pos + 22, 2);
      tag = t; channels = ch; bits = b; *rate = (int)r;
    } else if (memcmp(bytes.data() + pos, "data", 4) == 0) {
      if (channels != 1) return false;
      *data = bytes.data() + pos + 8;
      *n_bytes = sz <= bytes.size() - pos - 8 ? sz : bytes.size() - pos - 8;
      if (tag == 1 && bits == 16) { *fmt = 1; return true; }
      if (tag == 3 && bits == 32) { *fmt = 0; return true; }
      return false;
    }
    pos += 8 + sz + (sz & 1);
  }
  return false;
}

// The runtime's Audio loaders scale s16 by 1/32768 and resample at the caller's rate with LinearResample (WavResample): the
// handle's FA_RESAMPLE_RUNTIME.  Scaling by a power of two commutes exactly with the filter's products and sums, so decoding to
// [-1, 1) before the filter gives the runtime's samples.
FaAudioFormat runtime_format(int fmt, int rate) { return FaAudioFormat{fmt, 1, rate, FA_RESAMPLE_RUNTIME}; }

FUNASR_RESULT infer_pcm(OfflineStream* s, const char* data, size_t n_bytes, const FaAudioFormat& fmt, const std::vector<std::vector<float>>& hw_emb,
                        const std::string& svs_lang, bool svs_itn) {
  const int64_t n = (int64_t)(n_bytes / (fmt.sample_format == 1 ? 2 : 4));
  const void* bufs[1] = {data};
  const int64_t lens[1] = {n};
  if (fa_offline_is_sensevoice(s->h)) return infer_sv(s, bufs, lens, fmt, svs_lang, svs_itn);
  std::vector<float> hw;
  int n_hw = 0;
  if (fa_offline_is_contextual(s->h) || fa_offline_is_seaco(s->h)) {   // SeACo without rows: the plain decoder distribution
    for (const auto& row : hw_emb) if (row.size() == 512) { hw.insert(hw.end(), row.begin(), row.end()); ++n_hw; }
    if (n_hw == 0 && fa_offline_is_contextual(s->h)) { g_shim_err = "contextual model: hw_emb must hold [n, 512] rows from CompileHotwordEmbedding"; return nullptr; }
  }
  if (s->vad) {                        // segment texts concatenated in time order (funasrruntime.cpp:287-296)
    const FaLongAudioOptions o = runtime_long_audio_options(*s);
    void* r = fa_offline_infer_vad_audio(s->h, s->vad, nullptr, bufs, lens, 1, &fmt, n_hw ? hw.data() : nullptr, n_hw, nullptr, nullptr, &o, 0);
    if (!r) { g_shim_err = fa_offline_last_error(); return nullptr; }
    int32_t k = 0, nseg = 0;
    const int32_t* ids = fa_offline_result_ids(r, 0, &k);
    const int32_t* seg = fa_offline_result_segments(r, 0, &nseg);
    std::string text;
    for (int32_t i = 0, pos = 0; i < nseg && ids; ++i) {
      text += join_tokens(*s, ids + pos, seg[3 * i + 2]);
      pos += seg[3 * i + 2];
    }
    ShimResult* out = new ShimResult();
    out->msgs.push_back(text);
    out->stamp = render_stamps(r, 0);
    out->snippet_time = fa_offline_result_audio_seconds(r);
    if (s->punc && !punctuate(s->punc, out->msgs)) { fa_offline_free_result(r); delete out; return nullptr; }
    if (s->punc && !out->stamp.empty()) out->stamp_sents = timestamp_sentence(out->msgs[0], r, 0);   // funasrruntime.cpp:327-329
    fa_offline_free_result(r);
    return out;
  }
  void* r = fa_offline_infer_audio(s->h, bufs, lens, 1, &fmt, n_hw ? hw.data() : nullptr, n_hw, nullptr, nullptr);
  if (!r) { g_shim_err = fa_offline_last_error(); return nullptr; }
  ShimResult* out = new ShimResult();
  const int cnt = fa_offline_result_count(r);
  for (int i = 0; i < cnt; ++i) {
    int32_t k = 0;
    const int32_t* ids = fa_offline_result_ids(r, i, &k);
    out->msgs.push_back(join_tokens(*s, ids, k));
    if (i == 0) out->stamp = render_stamps(r, 0);
  }
  out->snippet_time = fa_offline_result_audio_seconds(r);
  if (s->punc && !punctuate(s->punc, out->msgs)) { fa_offline_free_result(r); delete out; return nullptr; }
  if (s->punc && !out->stamp.empty() && !out->msgs.empty()) out->stamp_sents = timestamp_sentence(out->msgs[0], r, 0);
  fa_offline_free_result(r);
  return out;
}

}  // namespace

const char* FunB200LastError() { return g_shim_err.c_str(); }

extern "C" int64_t fa_sv_ctc_text_host(const int32_t* ids, int32_t n, const char* const* tokens, int32_t n_tokens, char* out, int64_t cap) {
  if ((!ids && n > 0) || n < 0 || (!tokens && n_tokens > 0) || n_tokens < 0 || (!out && cap > 0)) return -1;
  std::vector<std::string> vocab;
  for (int32_t i = 0; i < n_tokens; ++i) {
    if (!tokens[i]) return -1;
    vocab.push_back(tokens[i]);
  }
  const std::string s = sv_ctc_text(ids, n, vocab);
  if (cap > 0) {
    const size_t k = std::min<size_t>(s.size(), (size_t)(cap - 1));
    memcpy(out, s.data(), k);
    out[k] = '\0';
  }
  return (int64_t)s.size();
}

FUNASR_HANDLE FunOfflineInit(std::map<std::string, std::string>& model_path, int thread_num, bool use_gpu, int batch_size) {
  (void)thread_num; (void)use_gpu;
  g_shim_err.clear();
  auto it = model_path.find("model-dir");
  if (it == model_path.end()) { g_shim_err = "model_path[\"model-dir\"] is missing"; return nullptr; }
  const std::string dir = it->second;
  int mode = FA_GEMM_F16X3, device = 0;
  auto gm = model_path.find("gemm-mode");
  if (gm != model_path.end()) {
    if (gm->second == "fp32") mode = FA_GEMM_F32_SIMT;
    else if (gm->second == "fp16") mode = FA_GEMM_F16X1;
    else if (gm->second == "fp16x6") mode = FA_GEMM_F16X6;
    else if (gm->second != "fp16x3") { g_shim_err = "unknown gemm-mode " + gm->second; return nullptr; }
  }
  device = parse_device(model_path);
  OfflineStream* s = new OfflineStream();
  s->batch = batch_size > 0 ? batch_size : 1;
  auto bs = model_path.find("batch-size-s");
  if (bs != model_path.end()) s->batch_size_s = atoi(bs->second.c_str());
  if (s->batch_size_s <= 0) { g_shim_err = "batch-size-s must be a positive number of seconds"; delete s; return nullptr; }
  s->h = fa_offline_init((dir + "/model.fab2").c_str(), device, mode);
  if (!s->h) { g_shim_err = fa_offline_last_error(); delete s; return nullptr; }
  auto vd = model_path.find("vad-dir");
  if (vd != model_path.end()) {
    s->vad = fa_vad_init((vd->second + "/vad.fab2").c_str(), device);
    if (!s->vad) { g_shim_err = fa_offline_last_error(); fa_offline_uninit(s->h); delete s; return nullptr; }
  }
  auto pd = model_path.find("punc-dir");
  if (pd != model_path.end()) {
    s->punc = fa_punc_init((pd->second + "/punc.fab2").c_str(), device);
    if (!s->punc) { g_shim_err = fa_offline_last_error(); fa_vad_uninit(s->vad); fa_offline_uninit(s->h); delete s; return nullptr; }
  }
  std::ifstream tf(dir + "/tokens.txt");
  std::string line;
  while (tf && std::getline(tf, line)) {
    if (!line.empty() && line.back() == '\r') line.pop_back();
    s->token_id[line] = (int)s->vocab.size();
    s->vocab.push_back(line);
  }
  return s;
}

void FunOfflineReset(FUNASR_HANDLE, FUNASR_DEC_HANDLE) {}

void FunOfflineUninit(FUNASR_HANDLE handle) {
  OfflineStream* s = static_cast<OfflineStream*>(handle);
  if (!s) return;
  fa_offline_uninit(s->h);
  fa_vad_uninit(s->vad);
  fa_punc_uninit(s->punc);
  delete s;
}

FUNASR_RESULT FunOfflineInferBuffer(FUNASR_HANDLE handle, const char* sz_buf, int n_len, FUNASR_MODE, QM_CALLBACK fn_callback,
                                    const std::vector<std::vector<float>>& hw_emb, int sampling_rate, std::string wav_format, bool,
                                    FUNASR_DEC_HANDLE, std::string svs_lang, bool svs_itn) {
  g_shim_err.clear();
  OfflineStream* s = static_cast<OfflineStream*>(handle);
  if (!s || !sz_buf || n_len <= 0) { g_shim_err = "bad argument"; return nullptr; }
  const char* data = sz_buf;
  size_t nb = (size_t)n_len;
  int fmt = 1, rate = sampling_rate;
  std::string holder;
  if (wav_format == "wav") {
    holder.assign(sz_buf, (size_t)n_len);
    if (!parse_wav(holder, &data, &nb, &fmt, &rate)) { g_shim_err = "unsupported WAV (need mono PCM16 or float32)"; return nullptr; }
  } else if (wav_format != "pcm") { g_shim_err = "wav_format must be \"pcm\" (s16le) or \"wav\""; return nullptr; }
  FUNASR_RESULT r = infer_pcm(s, data, nb, runtime_format(fmt, rate), hw_emb, svs_lang, svs_itn);
  if (fn_callback) fn_callback(1, 1);
  return r;
}

FUNASR_RESULT FunOfflineInfer(FUNASR_HANDLE handle, const char* sz_filename, FUNASR_MODE mode, QM_CALLBACK fn_callback,
                              const std::vector<std::vector<float>>& hw_emb, int sampling_rate, bool itn, FUNASR_DEC_HANDLE dec_handle) {
  g_shim_err.clear();
  if (!sz_filename) { g_shim_err = "bad argument"; return nullptr; }
  std::ifstream f(sz_filename, std::ios::binary);
  if (!f) { g_shim_err = std::string("cannot open ") + sz_filename; return nullptr; }
  std::stringstream ss;
  ss << f.rdbuf();
  const std::string bytes = ss.str();
  const std::string name = sz_filename;
  const bool wav = name.size() > 4 && (name.compare(name.size() - 4, 4, ".wav") == 0 || name.compare(name.size() - 4, 4, ".WAV") == 0);
  return FunOfflineInferBuffer(handle, bytes.data(), (int)bytes.size(), mode, fn_callback, hw_emb, sampling_rate, wav ? "wav" : "pcm", itn, dec_handle);
}

// bias_embed -> 1-layer LSTM (gate order i, f, g, o) -> the hidden state after each hotword's last token
// (contextual_paraformer/model.py:350-372); the hotword list is followed by the <s> entry (model.py:606-607)
const std::vector<std::vector<float>> CompileHotwordEmbedding(FUNASR_HANDLE handle, std::string& hotwords, ASR_TYPE) {
  g_shim_err.clear();
  std::vector<std::vector<float>> out;
  OfflineStream* s = static_cast<OfflineStream*>(handle);
  if (s && fa_offline_is_sensevoice(s->h)) return {std::vector<float>(512, 0.f)};    // one zero row (sensevoice-small.cpp:423-429)
  if (s && fa_offline_is_seaco(s->h)) {                                 // the same hotword list, rows from the handle's GPU encoder
    const std::vector<std::vector<int>> lists = hotword_lists(*s, hotwords, (int)fa_offline_host_tensor(s->h, "__config__", nullptr)[5]);
    std::vector<int32_t> ids, lens;
    for (const auto& l : lists) { ids.insert(ids.end(), l.begin(), l.end()); lens.push_back((int32_t)l.size()); }
    std::vector<float> rows(lens.size() * 512);
    if (fa_offline_hotword_embed(s->h, ids.data(), lens.data(), (int32_t)lens.size(), rows.data()) != 0) { g_shim_err = fa_offline_last_error(); return out; }
    for (size_t i = 0; i < lens.size(); ++i) out.emplace_back(rows.begin() + i * 512, rows.begin() + (i + 1) * 512);
    return out;
  }
  // a model without a hotword branch (Paraformer, BiCif): one zero row of encoder_size (paraformer.cpp:557-564), so a server that
  // decodes only when the embedding is non-empty still decodes; infer_pcm passes no rows to such a model
  if (s && !fa_offline_is_contextual(s->h)) return {std::vector<float>(512, 0.f)};
  if (!s) return out;
  int64_t n_emb = 0, n_ih = 0, n_hh = 0, n_bi = 0, n_bh = 0;
  const float* emb = fa_offline_host_tensor(s->h, "bias_embed.weight", &n_emb);
  const float* w_ih = fa_offline_host_tensor(s->h, "bias_encoder.weight_ih_l0", &n_ih);
  const float* w_hh = fa_offline_host_tensor(s->h, "bias_encoder.weight_hh_l0", &n_hh);
  const float* b_ih = fa_offline_host_tensor(s->h, "bias_encoder.bias_ih_l0", &n_bi);
  const float* b_hh = fa_offline_host_tensor(s->h, "bias_encoder.bias_hh_l0", &n_bh);
  const int D = 512;
  if (!emb || !w_ih || !w_hh || !b_ih || !b_hh || n_ih != 4 * D * D || n_hh != 4 * D * D) { g_shim_err = "model file has no hotword encoder"; return out; }
  const std::vector<std::vector<int>> lists = hotword_lists(*s, hotwords, (int)(n_emb / D));
  std::vector<float> h(D), c(D), gates(4 * D);
  for (const auto& ids : lists) {
    std::fill(h.begin(), h.end(), 0.f);
    std::fill(c.begin(), c.end(), 0.f);
    for (int id : ids) {
      const float* x = emb + (size_t)id * D;
      for (int g = 0; g < 4 * D; ++g) {
        const float* wi = w_ih + (size_t)g * D;
        const float* wh = w_hh + (size_t)g * D;
        float a = b_ih[g] + b_hh[g];
        float acc1 = 0.f, acc2 = 0.f;
        for (int k = 0; k < D; ++k) { acc1 += wi[k] * x[k]; acc2 += wh[k] * h[k]; }
        gates[g] = a + acc1 + acc2;
      }
      for (int k = 0; k < D; ++k) {
        const float ig = sigm(gates[k]), fg = sigm(gates[D + k]), gg = tanhf(gates[2 * D + k]), og = sigm(gates[3 * D + k]);
        c[k] = fg * c[k] + ig * gg;
      }
      for (int k = 0; k < D; ++k) h[k] = sigm(gates[3 * D + k]) * tanhf(c[k]);
    }
    out.push_back(h);
  }
  return out;
}

const char* FunASRGetResult(FUNASR_RESULT result, int n_index) {
  ShimResult* r = static_cast<ShimResult*>(result);
  if (!r || n_index < 0 || n_index >= (int)r->msgs.size()) return nullptr;
  return r->msgs[n_index].c_str();
}
const char* FunASRGetStamp(FUNASR_RESULT result) { return result ? static_cast<ShimResult*>(result)->stamp.c_str() : nullptr; }
const char* FunASRGetStampSents(FUNASR_RESULT result) { return result ? static_cast<ShimResult*>(result)->stamp_sents.c_str() : nullptr; }
const int FunASRGetRetNumber(FUNASR_RESULT result) { return result ? (int)static_cast<ShimResult*>(result)->msgs.size() : 0; }
void FunASRFreeResult(FUNASR_RESULT result) { delete static_cast<ShimResult*>(result); }
const float FunASRGetRetSnippetTime(FUNASR_RESULT result) { return result ? static_cast<ShimResult*>(result)->snippet_time : 0.f; }

FUNASR_HANDLE FsmnVadInit(std::map<std::string, std::string>& model_path, int thread_num) {
  (void)thread_num;
  g_shim_err.clear();
  auto it = model_path.find("model-dir");
  if (it == model_path.end()) { g_shim_err = "model_path[\"model-dir\"] is missing"; return nullptr; }
  VadStream* s = new VadStream();
  s->v = fa_vad_init((it->second + "/vad.fab2").c_str(), parse_device(model_path));
  if (!s->v) { g_shim_err = fa_offline_last_error(); delete s; return nullptr; }
  return s;
}

FUNASR_RESULT FsmnVadInferBuffer(FUNASR_HANDLE handle, const char* sz_buf, int n_len, QM_CALLBACK fn_callback, bool input_finished, int sampling_rate,
                                 std::string wav_format) {
  g_shim_err.clear();
  VadStream* s = static_cast<VadStream*>(handle);
  if (!s || !sz_buf || n_len <= 0) { g_shim_err = "bad argument"; return nullptr; }
  if (!input_finished) { g_shim_err = "only offline VAD is provided: input_finished must be true"; return nullptr; }
  const char* data = sz_buf;
  size_t nb = (size_t)n_len;
  int fmt = 1, rate = sampling_rate;
  std::string holder;
  if (wav_format == "wav") {
    holder.assign(sz_buf, (size_t)n_len);
    if (!parse_wav(holder, &data, &nb, &fmt, &rate)) { g_shim_err = "unsupported WAV (need mono PCM16 or float32)"; return nullptr; }
  } else if (wav_format != "pcm" && wav_format != "PCM") { g_shim_err = "wav_format must be \"pcm\" (s16le) or \"wav\""; return nullptr; }
  const FaVadRunOptions o = runtime_vad_options();
  const FaAudioFormat f = runtime_format(fmt, rate);
  void* r = fa_vad_infer_audio(s->v, data, (int64_t)(nb / (fmt == 1 ? 2 : 4)), &f, &o);
  if (!r) { g_shim_err = fa_offline_last_error(); return nullptr; }
  VadShimResult* out = new VadShimResult();
  int64_t n = 0;
  const int32_t* seg = fa_vad_result_segments(r, &n);
  for (int64_t i = 0; i < n; ++i) out->segments.push_back({seg[2 * i], seg[2 * i + 1]});
  out->snippet_time = fa_vad_result_audio_seconds(r);
  fa_vad_free_result(r);
  if (fn_callback) fn_callback(1, 1);
  return out;
}

FUNASR_RESULT FsmnVadInfer(FUNASR_HANDLE handle, const char* sz_filename, QM_CALLBACK fn_callback, int sampling_rate) {
  g_shim_err.clear();
  if (!sz_filename) { g_shim_err = "bad argument"; return nullptr; }
  std::ifstream f(sz_filename, std::ios::binary);
  if (!f) { g_shim_err = std::string("cannot open ") + sz_filename; return nullptr; }
  std::stringstream ss;
  ss << f.rdbuf();
  const std::string bytes = ss.str();
  const std::string name = sz_filename;
  const bool wav = name.size() > 4 && (name.compare(name.size() - 4, 4, ".wav") == 0 || name.compare(name.size() - 4, 4, ".WAV") == 0);
  return FsmnVadInferBuffer(handle, bytes.data(), (int)bytes.size(), fn_callback, true, sampling_rate, wav ? "wav" : "pcm");
}

std::vector<std::vector<int>>* FsmnVadGetResult(FUNASR_RESULT result, int n_index) {
  VadShimResult* r = static_cast<VadShimResult*>(result);
  return r && n_index == 0 ? &r->segments : nullptr;
}
void FsmnVadFreeResult(FUNASR_RESULT result) { delete static_cast<VadShimResult*>(result); }
void FsmnVadUninit(FUNASR_HANDLE handle) {
  VadStream* s = static_cast<VadStream*>(handle);
  if (!s) return;
  fa_vad_uninit(s->v);
  delete s;
}
const float FsmnVadGetRetSnippetTime(FUNASR_RESULT result) { return result ? static_cast<VadShimResult*>(result)->snippet_time : 0.f; }

FUNASR_HANDLE CTTransformerInit(std::map<std::string, std::string>& model_path, int thread_num, PUNC_TYPE type) {
  (void)thread_num;
  g_shim_err.clear();
  if (type != PUNC_OFFLINE) { g_shim_err = "only offline punctuation is provided: type must be PUNC_OFFLINE"; return nullptr; }
  auto it = model_path.find("model-dir");
  if (it == model_path.end()) { g_shim_err = "model_path[\"model-dir\"] is missing"; return nullptr; }
  void* p = fa_punc_init((it->second + "/punc.fab2").c_str(), parse_device(model_path));
  if (!p) g_shim_err = fa_offline_last_error();
  return p;
}

FUNASR_RESULT CTTransformerInfer(FUNASR_HANDLE handle, const char* sz_sentence, FUNASR_MODE, QM_CALLBACK fn_callback, PUNC_TYPE type, FUNASR_RESULT) {
  g_shim_err.clear();
  if (!handle || !sz_sentence) { g_shim_err = "bad argument"; return nullptr; }
  if (type != PUNC_OFFLINE) { g_shim_err = "only offline punctuation is provided: type must be PUNC_OFFLINE"; return nullptr; }
  std::vector<std::string> msgs{sz_sentence};
  if (!punctuate(handle, msgs)) return nullptr;
  if (fn_callback) fn_callback(1, 1);
  PuncShimResult* r = new PuncShimResult();
  r->msg.swap(msgs[0]);
  return r;
}

const char* CTTransformerGetResult(FUNASR_RESULT result, int) { return result ? static_cast<PuncShimResult*>(result)->msg.c_str() : nullptr; }
void CTTransformerFreeResult(FUNASR_RESULT result) { delete static_cast<PuncShimResult*>(result); }
void CTTransformerUninit(FUNASR_HANDLE handle) { fa_punc_uninit(handle); }

FUNASR_DEC_HANDLE FunASRWfstDecoderInit(FUNASR_HANDLE, int, float, float, float) { return nullptr; }
void FunASRWfstDecoderUninit(FUNASR_DEC_HANDLE) {}
void FunWfstDecoderLoadHwsRes(FUNASR_DEC_HANDLE, int, std::unordered_map<std::string, int>&) {}
void FunWfstDecoderUnloadHwsRes(FUNASR_DEC_HANDLE) {}
