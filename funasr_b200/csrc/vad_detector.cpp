// Host-side end-point detector of the FSMN-VAD (no CUDA in this file): per-frame silence posteriors + frame energies of one whole
// recording -> [start_ms, end_ms] segments, as FsmnVADStreaming.inference produces them chunk by chunk
// (funasr/models/fsmn_vad_streaming/model.py: GetFrameState :761-823, WindowDetector :218-320, DetectOneFrame :1158-1302, the On*
// callbacks :641-736, the per-chunk dynamic end-silence schedule :1003-1067; frame delivery of WavFrontendOnline,
// frontends/wav_frontend.py:345-447, :591-603).  The reference walks over the frames one at a time in Python; funasr_b200/vad.py
// restates that walk step by step (and stays the readable specification, pinned to the reference's golden segments); this file is
// the same state machine in C++ — 23 ms of Python per 130 s recording (5 600x real time, an eighth of what one GPU transcribes)
// becomes ~0.1 ms.  Arithmetic follows the Python floats: IEEE doubles, libm log / exp (what CPython's math module calls).
#include "../../include/funasr_b200.h"

#include <math.h>
#include <stdint.h>
#include <algorithm>
#include <vector>

namespace {

enum Machine { kStartNotDetected = 1, kInSpeech = 2, kEndDetected = 3 };
enum Frame { kSil = 0, kSpeech = 1 };
enum Change { kSp2Sp = 0, kSp2Sil = 1, kSil2Sil = 2, kSil2Sp = 3 };

struct Segment { int64_t start_ms, end_ms; bool has_start, has_end; };

// sliding count of speech frames with hysteresis (WindowDetector)
struct Window {
  int n, to_speech, to_sil, pos = 0, total = 0, pre = kSil;
  std::vector<int> buf;
  explicit Window(const FaVadOptions& o)
      : n(o.window_size_ms / o.frame_in_ms), to_speech(o.sil_to_speech_time_thres / o.frame_in_ms), to_sil(o.speech_to_sil_time_thres / o.frame_in_ms),
        buf((size_t)std::max(n, 1), 0) {}
  void reset() { pos = 0; total = 0; pre = kSil; std::fill(buf.begin(), buf.end(), 0); }
  int step(int state) {
    total += state - buf[pos];
    buf[pos] = state;
    pos = (pos + 1) % n;
    if (pre == kSil && total >= to_speech) { pre = kSpeech; return kSil2Sp; }
    if (pre == kSpeech && total <= to_sil) { pre = kSil; return kSp2Sil; }
    return pre == kSil ? kSil2Sil : kSp2Sp;
  }
};

struct Detector {
  const FaVadOptions& o;
  Window win;
  const double* sil;
  const double* db;
  int64_t frm_cnt = 0, buf_start = 0, last_speech = 0, last_silence = -1, silence_run = 0, start_frame = -1, end_frame = -1, ends_seen = 0;
  int state = kStartNotDetected;
  double noise_db = -100.0, speech_noise_thres;
  int64_t end_sil_thresh_ms;                 // max_end_sil_frame_cnt_thresh (milliseconds despite its name in the reference)
  int64_t latency;
  std::vector<Segment> out;
  size_t out_offset = 0;
  bool bad_input = false;

  Detector(const FaVadOptions& opt, const double* s, const double* d, double thres)
      : o(opt), win(opt), sil(s), db(d), speech_noise_thres(thres), end_sil_thresh_ms(opt.max_end_silence_time - opt.speech_to_sil_time_thres),
        latency(win.n + (opt.do_extend ? opt.lookback_time_start_point / opt.frame_in_ms : 0)) {}

  int frame_state(int64_t t) {
    const double cur = db[t];
    const double snr = cur - noise_db;
    if (cur < o.decibel_thres) return kSil;
    const double p_sil = sil[t];
    if (!(p_sil > 0.0) || !(1.0 - p_sil > 0.0)) { bad_input = true; return kSil; }   // math.log would raise in the reference
    const double noise_prob = log(p_sil) * o.speech_2_noise_ratio;
    const double speech_prob = log(1.0 - p_sil);
    if (exp(speech_prob) >= exp(noise_prob) + speech_noise_thres) return (snr >= o.snr_thres && cur >= o.decibel_thres) ? kSpeech : kSil;
    if (noise_db < -99.9) noise_db = cur;
    else noise_db = (cur + noise_db * (double)(o.noise_frame_num_used_for_snr - 1)) / (double)o.noise_frame_num_used_for_snr;
    return kSil;
  }

  void pop_till(int64_t f) { if (buf_start < f) buf_start = f; }
  void pop_to_output(int64_t start, int64_t count, bool first_is_start, bool last_is_end) {
    const int64_t ms = o.frame_in_ms;
    pop_till(start);
    if (out.empty() || first_is_start) out.push_back({start * ms, start * ms, false, false});
    Segment& s = out.back();
    buf_start += count;
    s.end_ms = (start + count) * ms;
    if (first_is_start) s.has_start = true;
    if (last_is_end) s.has_end = true;
  }
  void on_silence(int64_t f) { last_silence = f; if (state == kStartNotDetected) pop_till(f); }
  void on_voice(int64_t f) { last_speech = f; pop_to_output(f, 1, false, false); }
  void on_voice_start(int64_t f, bool fake) {
    if (start_frame == -1) start_frame = f;
    if (!fake && state == kStartNotDetected) pop_to_output(start_frame, 1, true, false);
  }
  void on_voice_end(int64_t f, bool fake) {
    for (int64_t t = last_speech + 1; t < f; ++t) on_voice(t);
    if (end_frame == -1) end_frame = f;
    if (!fake) pop_to_output(end_frame, 1, false, true);
    ++ends_seen;
  }
  void reset_detection() {
    silence_run = 0; last_speech = 0; last_silence = -1; start_frame = -1; end_frame = -1; state = kStartNotDetected;
    win.reset();
  }
  bool too_long(int64_t cur) const { return (double)(cur - start_frame + 1) > (double)o.max_single_segment_time / (double)o.frame_in_ms; }
  void end_or_continue(int64_t cur, bool is_final) {
    if (too_long(cur)) { on_voice_end(cur, false); state = kEndDetected; }
    else if (!is_final) on_voice(cur);
    else { on_voice_end(cur, false); state = kEndDetected; }
  }

  void detect(int fs, int64_t cur, bool is_final) {
    const int64_t ms = o.frame_in_ms;
    if (fs == kSpeech && !(1.0 > o.fe_prior_thres)) fs = kSil;
    const int change = win.step(fs);
    if (change == kSil2Sp) {
      silence_run = 0;
      if (state == kStartNotDetected) {
        const int64_t start = std::max(buf_start, cur - latency);
        on_voice_start(start, false);
        state = kInSpeech;
        for (int64_t t = start + 1; t <= cur; ++t) on_voice(t);
      } else if (state == kInSpeech) {
        for (int64_t t = last_speech + 1; t < cur; ++t) on_voice(t);
        end_or_continue(cur, is_final);
      }
    } else if (change == kSp2Sil || change == kSp2Sp) {
      silence_run = 0;
      if (state == kInSpeech) end_or_continue(cur, is_final);
    } else {                                                   // kSil2Sil
      ++silence_run;
      if (state == kStartNotDetected) {
        if ((o.detect_mode == 0 && silence_run * ms > o.max_start_silence_time) || (is_final && ends_seen == 0)) {
          for (int64_t t = last_silence + 1; t < cur; ++t) on_silence(t);
          on_voice_start(0, true);
          on_voice_end(0, true);
          state = kEndDetected;
        } else if (cur >= latency) {
          on_silence(cur - latency);
        }
      } else if (state == kInSpeech) {
        if (silence_run * ms >= end_sil_thresh_ms) {
          int64_t lookback = end_sil_thresh_ms / ms;
          if (o.do_extend) lookback = std::max<int64_t>(0, lookback - o.lookahead_time_end_point / ms - 1);
          on_voice_end(cur - lookback, false);
          state = kEndDetected;
        } else if (too_long(cur)) {
          on_voice_end(cur, false);
          state = kEndDetected;
        } else if (o.do_extend && !is_final) {
          if (silence_run <= o.lookahead_time_end_point / ms) on_voice(cur);
        } else if (is_final) {
          on_voice_end(cur, false);
          state = kEndDetected;
        }
      }
    }
    if (state == kEndDetected && o.detect_mode == 1) reset_detection();
  }

  // one forward() of the reference over the frames [first, first + n) of one chunk
  void process_block(int64_t n, bool is_final) {
    if (n <= 0) return;
    const int64_t first = frm_cnt;
    frm_cnt += n;
    if (state == kEndDetected) return;
    for (int64_t k = 0; k < n; ++k) detect(frame_state(first + k), first + k, is_final && k == n - 1);
  }
  // segments completed since the last call (offline mode): appended to dst
  bool take_new(bool is_final, std::vector<Segment>* dst) {
    bool any = false;
    for (size_t i = out_offset; i < out.size(); ++i) {
      if (!is_final && (!out[i].has_start || !out[i].has_end)) continue;
      dst->push_back(out[i]);
      ++out_offset;
      any = true;
    }
    return any;
  }
};

// frames the reference's chunked frontend hands to the detector per waveform chunk (see funasr_b200/vad.py: chunk_frame_counts)
std::vector<int64_t> chunk_frame_counts(int64_t n_samples, int64_t chunk_ms, int64_t fs, int64_t lfr_m, int64_t frame_len, int64_t shift) {
  const int64_t stride = chunk_ms * fs / 1000;
  const int64_t n_chunks = n_samples / stride + 1;
  const int64_t half = (lfr_m - 1) / 2;
  std::vector<int64_t> out;
  int64_t leftover = 0, cached = -1;                    // cached < 0: no frame seen yet
  for (int64_t i = 0; i < n_chunks; ++i) {
    const bool final = i == n_chunks - 1;
    const int64_t fresh = std::min(stride, std::max<int64_t>(0, n_samples - i * stride));
    const int64_t total = leftover + fresh;
    int64_t f = total >= frame_len ? (total - frame_len) / shift + 1 : 0;
    if (f < 1) f = 0;
    leftover = total - f * shift;
    int64_t emitted = 0;
    if (f > 0) {
      if (cached < 0) cached = half;
      const int64_t t = cached + f;
      if (t >= lfr_m) {
        emitted = final ? t - half : t - (lfr_m - 1);
        cached = final ? t - std::min(t - 1, emitted) : t - emitted;
      } else {
        cached = t;
      }
    } else if (final && cached > 0) {
      emitted = std::max<int64_t>(cached - half, 0);
    }
    out.push_back(emitted);
  }
  return out;
}

}  // namespace

extern "C" int64_t fa_vad_detect_segments(const double* sil_prob, const double* decibel, int64_t frames, int64_t n_samples, const FaVadOptions* opts,
                                          int32_t chunk_ms, int32_t dynamic_silence, const double* schedule, int32_t n_schedule,
                                          double speech_noise_thres, int32_t* segments, int64_t max_segments) {
  if (!opts || frames < 0 || n_samples < 0 || (frames > 0 && (!sil_prob || !decibel)) || chunk_ms <= 0 || max_segments < 0 ||
      (max_segments > 0 && !segments) || (dynamic_silence && (n_schedule <= 0 || !schedule)))
    return FA_ERR_ARG;
  const FaVadOptions& o = *opts;
  if (o.frame_in_ms <= 0 || o.sample_rate <= 0 || o.window_size_ms < o.frame_in_ms || o.noise_frame_num_used_for_snr <= 0) return FA_ERR_ARG;
  Detector det(o, sil_prob, decibel, speech_noise_thres == speech_noise_thres ? speech_noise_thres : o.speech_noise_thres);   // NaN: the options' value
  const std::vector<int64_t> counts = chunk_frame_counts(n_samples, chunk_ms, o.sample_rate, 5, (int64_t)o.frame_length_ms * o.sample_rate / 1000,
                                                         (int64_t)o.frame_in_ms * o.sample_rate / 1000);
  std::vector<Segment> found;
  int64_t accumulated_ms = 0, pos = 0;
  bool in_speech = false;
  for (size_t i = 0; i < counts.size(); ++i) {
    const bool final = i + 1 == counts.size();
    if (dynamic_silence) {
      if (det.state == kInSpeech || in_speech) { accumulated_ms += chunk_ms; in_speech = true; }
      for (int32_t k = 0; k < n_schedule; ++k) {
        const double limit = schedule[2 * k];
        if (limit < 0 || (double)accumulated_ms <= limit) {
          det.end_sil_thresh_ms = std::max<int64_t>((int64_t)schedule[2 * k + 1] - o.speech_to_sil_time_thres, 0);
          det.speech_noise_thres = 0.5;
          break;
        }
      }
    }
    if (counts[i] <= 0) continue;
    const int64_t n = std::max<int64_t>(0, std::min(counts[i], frames - pos));   // the slice sil_prob[pos : pos + count] of the restatement
    det.process_block(n, final);
    if (det.bad_input) return FA_ERR_ARG;
    pos += counts[i];
    if (det.take_new(final, &found) && dynamic_silence) { accumulated_ms = 0; in_speech = false; }
  }
  for (size_t i = 0; i < found.size() && (int64_t)i < max_segments; ++i) {
    segments[2 * i] = (int32_t)found[i].start_ms;
    segments[2 * i + 1] = (int32_t)found[i].end_ms;
  }
  return (int64_t)found.size();
}

// What inference_with_vad does with the segments before decoding (funasr_b200/long_audio.py: pack_segments, vad.py: merge_vad stay the
// specification; tests hold the two identical).
extern "C" int64_t fa_pack_segments(const int32_t* segments, int64_t n, int32_t batch_size_s, int32_t batch_size_threshold_s, int32_t* order,
                                    int32_t* packs) {
  if (n < 0 || n > 0x7fffffff || (n > 0 && (!segments || !order || !packs))) return FA_ERR_ARG;
  if (n == 0) return 0;
  auto len = [&](int64_t i) { return (int64_t)segments[2 * i + 1] - (int64_t)segments[2 * i]; };
  std::vector<int32_t> idx((size_t)n);
  for (int64_t i = 0; i < n; ++i) idx[(size_t)i] = (int32_t)i;
  std::stable_sort(idx.begin(), idx.end(), [&](int32_t a, int32_t b) { return len(a) < len(b); });   // ties keep time order
  for (int64_t i = 0; i < n; ++i) order[i] = idx[(size_t)i];
  int64_t batch_size = std::max<int64_t>((int64_t)batch_size_s * 1000, 1);
  const int64_t threshold_ms = (int64_t)batch_size_threshold_s * 1000;
  batch_size = std::max(batch_size, len(idx[0]));
  int64_t n_packs = 0, beg = 0, end = 1, max_len = 0;
  for (int64_t j = 0; j < n; ++j) {
    const int64_t length = len(idx[(size_t)j]);
    const int64_t potential = std::max(max_len, length) * (j + 1 - beg);
    if (j < n - 1 && length < threshold_ms && potential < batch_size) {
      max_len = std::max(max_len, length);
      ++end;
      continue;
    }
    packs[2 * n_packs] = (int32_t)beg;
    packs[2 * n_packs + 1] = (int32_t)end;
    ++n_packs;
    beg = end;
    ++end;
    max_len = length;
  }
  return n_packs;
}

extern "C" int64_t fa_merge_vad(const int32_t* segments, int64_t n, int32_t max_length_ms, int32_t min_length_ms, int32_t* out) {
  if (n < 0 || (n > 0 && (!segments || !out))) return FA_ERR_ARG;
  if (n <= 1) {                                              // returned as given
    for (int64_t i = 0; i < 2 * n; ++i) out[i] = segments[i];
    return n;
  }
  std::vector<int32_t> steps(segments, segments + 2 * n);
  std::sort(steps.begin(), steps.end());
  steps.erase(std::unique(steps.begin(), steps.end()), steps.end());
  int64_t cnt = 0;
  int64_t bg = 0;
  for (size_t i = 0; i + 1 < steps.size(); ++i) {
    const int64_t time = steps[i];
    if ((int64_t)steps[i + 1] - bg < max_length_ms) continue;
    if (time - bg > min_length_ms) { out[2 * cnt] = (int32_t)bg; out[2 * cnt + 1] = (int32_t)time; ++cnt; }
    bg = time;
  }
  out[2 * cnt] = (int32_t)bg;
  out[2 * cnt + 1] = steps.back();
  return cnt + 1;
}
