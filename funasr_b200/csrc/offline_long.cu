// Long audio through the handle API: the call's recordings uploaded together and scored by one batched FSMN-VAD pass (vad_run_batch),
// then per recording its segments merged and packed by duration on the host (fa_merge_vad / fa_pack_segments), each pack gathered on the device and decoded by the recogniser
// (decode_pack); fa_offline_infer_vad_spk then diarizes every recording with the CAM++ handle (diarize).
#include "handle.h"

using namespace fa_handle;

namespace {

// padded 16 kHz samples one long-audio call uploads and scores at once: an hour of audio (230 MB of fp32 rows)
const int64_t kVadGroupSamples = 3600LL * 16000;

// one recording of fa_offline_infer_vad: inference_with_vad (auto_model.py:852-1035, funasr_b200/long_audio.py:LongAudioPipeline.generate)
// (lang, tn): the recording's SenseVoice query, the same for all its segments
// on the device recording rec [n] with its VAD result vr
bool long_audio_one(Model& m, const VadResult& vr, int rec_index, const float* rec, int64_t n, const float* hw_embed, int32_t n_hotwords,
                    int32_t lang, int32_t tn, const FaLongAudioOptions& o, std::vector<int32_t>& ids, std::vector<int32_t>& segs_out,
                    std::vector<int32_t>& stamps) {
  cudaStream_t st = m.file.st;
  std::vector<int32_t> segs = vr.seg;
  if (o.merge_vad) {
    segs.resize(2 * vr.seg.size() + 2);
    const int64_t k = fa_merge_vad(vr.seg.data(), (int64_t)vr.seg.size() / 2, o.merge_length_s * 1000, 0, segs.data());
    if (k < 0) { set_err("fa_merge_vad failed"); return false; }
    segs.resize((size_t)(2 * k));
  }
  const int64_t ns = (int64_t)segs.size() / 2;
  if (ns == 0) return true;                                  // no speech: no segment, no id
  std::vector<int32_t> order((size_t)ns), packs((size_t)(2 * ns));
  const int64_t np = fa_pack_segments(segs.data(), ns, o.batch_size_s, o.batch_size_threshold_s, order.data(), packs.data());
  if (np < 0) { set_err("fa_pack_segments failed"); return false; }
  std::vector<std::vector<int32_t>> seg_ids((size_t)ns), seg_stamps((size_t)ns);
  bool emptied = false;
  for (int64_t p = 0; p < np && !emptied; ++p) {
    const int beg = packs[2 * p], end = packs[2 * p + 1], B = end - beg;
    std::vector<int64_t> starts(B);
    std::vector<int32_t> lens(B);
    int64_t lmax = 0;
    for (int j = 0; j < B; ++j) {                            // slice_padding_audio_samples (utils/vad_utils.py:44-51)
      const int s = order[beg + j];
      const int64_t b0 = (int64_t)segs[2 * s] * 16, b1 = std::min<int64_t>((int64_t)segs[2 * s + 1] * 16, n), len = b1 - b0;
      if (len < 400) {
        set_err("recording " + std::to_string(rec_index) + ": VAD segment " + std::to_string(s) + " [" + std::to_string(segs[2 * s]) + ", " +
                std::to_string(segs[2 * s + 1]) + "] ms has " + std::to_string(len > 0 ? len : 0) + " samples; the recogniser needs >= 400 (25 ms)");
        return false;
      }
      starts[j] = b0; lens[j] = (int32_t)len;
      lmax = len > lmax ? len : lmax;
    }
    const int64_t stride = (lmax + 3) / 4 * 4;
    int64_t* starts_d;
    int32_t* lens_d;
    float* wav;
    if (!carve(m.pack, "segments", [&](fa::Arena& a) {
          starts_d = a.take<int64_t>(B); lens_d = a.take<int32_t>(B); wav = a.take<float>((size_t)B * stride);
        }))
      return false;
    if (!gather(rec, n, starts.data(), lens.data(), B, stride, starts_d, lens_d, wav, st)) return false;
    const std::vector<int32_t> lang_v(B, lang), tn_v(B, tn);
    const std::unique_ptr<Result> pr = decode_pack(m, wav, stride, lens, hw_embed, n_hotwords, lang_v.data(), tn_v.data());
    if (!pr) return false;
    int tmax = 0;
    for (int32_t t : pr->token_num) tmax = t > tmax ? t : tmax;
    // no token in the whole pack: the recording's result is empty (:990-999).  SenseVoiceSmall.inference returns a result for every
    // utterance, empty or not, so its packs never empty a recording.
    if (tmax < 1 && !m.sv) emptied = true;
    else
      for (int j = 0; j < B; ++j) {
        seg_ids[order[beg + j]].swap(pr->ids[j]);
        if (pr->ts) seg_stamps[order[beg + j]].swap(pr->stamps[j]);
      }
  }
  for (int64_t s = 0; s < ns; ++s) {
    const int32_t k = emptied ? 0 : (int32_t)seg_ids[s].size();
    segs_out.insert(segs_out.end(), {segs[2 * s], segs[2 * s + 1], k});
    if (emptied) continue;
    ids.insert(ids.end(), seg_ids[s].begin(), seg_ids[s].end());
    for (int32_t t : seg_stamps[s]) stamps.push_back(t + segs[2 * s]);       // absolute ms (auto_model.py:1008-1022)
  }
  return true;
}

// fa_offline_infer_vad* / fa_offline_infer_vad_audio: every recording decoded on its own; lang / tn one query per recording (NULL = the defaults)
// spk: diarize every recording that decoded at least one token (LongAudioPipeline.generate), preset_spk_num <= 0: no preset count
// fmt: the recordings' layout (the 16 kHz entries pass their pcm_format's)
void* infer_vad(void* asr, void* vad, const void* const* bufs, const int64_t* n_samples, int32_t batch, const FaAudioFormat* fmt, const float* hw_embed,
                int32_t n_hotwords, const int32_t* lang, const int32_t* tn, const FaLongAudioOptions* opts, Spk* spk = nullptr,
                int32_t preset_spk_num = 0) {
  Model* mp = static_cast<Model*>(asr);
  Vad* vp = static_cast<Vad*>(vad);
  if (!mp || !vp || !bufs || !n_samples || batch <= 0) return fail("bad argument");
  Audio au;
  if (!plan_audio(fmt, mp->resample, au)) return nullptr;
  if (mp->file.device != vp->file.device) return fail("the recogniser and the VAD live on different devices");
  if (spk && spk->file.device != mp->file.device) return fail("the recogniser and the speaker model live on different devices");
  if (!check_hotword_rows(*mp, hw_embed, n_hotwords)) return nullptr;
  if (mp->sv && !check_queries(*mp, lang, tn, batch, "recording")) return nullptr;
  FaLongAudioOptions o;
  if (opts) o = *opts;
  else { o.batch_size_s = 300; o.batch_size_threshold_s = 60; o.merge_vad = 0; o.merge_length_s = 15; o.vad = default_vad_run(); }
  std::vector<int64_t> n16(batch);
  for (int i = 0; i < batch; ++i) {
    if ((!bufs[i] && n_samples[i] > 0) || n_samples[i] < 0 || n_samples[i] > 0x7fffffffLL) return fail("bad recording " + std::to_string(i));
    n16[i] = au.len16(n_samples[i]);
    if (n16[i] > 0x7fffffffLL) return fail("bad recording " + std::to_string(i));
  }
  // recogniser -> VAD -> speaker (handle.h)
  std::lock_guard<std::mutex> asr_lock(mp->mu);
  std::lock_guard<std::mutex> vad_lock(vp->mu);
  std::unique_lock<std::mutex> spk_lock;
  if (spk) spk_lock = std::unique_lock<std::mutex>(spk->mu);
  cudaSetDevice(mp->file.device);
  std::unique_ptr<Result> r(new Result());
  r->ids.resize(batch);
  r->segs.resize(batch);
  r->token_num.assign(batch, 0);
  r->ts = mp->ts;
  r->stamps.resize(batch);
  r->spk.resize(batch);
  if (!no_throw("fa_offline_infer_vad: ", [&] {
        // recordings in arrival order, uploaded together in groups of at most kVadGroupSamples padded samples (a longer recording is
        // a group of its own) and scored by one batched VAD pass; then each recording's segments are packed and decoded on their own
        for (int g0 = 0, g1; g0 < batch; g0 = g1) {
          int64_t stride = (n16[g0] + 3) / 4 * 4;
          for (g1 = g0 + 1; g1 < batch; ++g1) {
            const int64_t w = std::max(stride, (n16[g1] + 3) / 4 * 4);
            if ((g1 - g0 + 1) * w > kVadGroupSamples) break;
            stride = w;
          }
          float* recs = nullptr;
          std::vector<VadResult> vr;
          if (!upload(&bufs[g0], &n_samples[g0], g1 - g0, stride, au, mp->resample, mp->upload, mp->file.st, &recs) ||
              !vad_run_batch(*vp, recs, stride, &n16[g0], g1 - g0, mp->file.st, o.vad, vr))
            return false;
          for (int i = g0; i < g1; ++i) {
            const float* rec = recs + (int64_t)(i - g0) * stride;
            if (!long_audio_one(*mp, vr[i - g0], i, rec, n16[i], hw_embed, n_hotwords, lang ? lang[i] : kSvAuto, tn ? tn[i] : kSvWoItn, o,
                                r->ids[i], r->segs[i], r->stamps[i]))
              return false;
            r->token_num[i] = (int32_t)r->ids[i].size();
            // the recogniser's stream is idle here (its results are on the host); the speaker work runs on the speaker handle's stream
            if (spk && !r->ids[i].empty() &&
                !diarize(*spk, rec, n16[i], r->segs[i], preset_spk_num, r->spk[i], "recording " + std::to_string(i) + ": "))
              return false;
          }
        }
        return true;
      }))
    return nullptr;
  r->audio_seconds = (float)au.seconds(n_samples, batch);
  return r.release();
}

const Result* as_result(const void* r) { return static_cast<const Result*>(r); }

}  // namespace

extern "C" void* fa_offline_infer_vad(void* asr, void* vad, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                                      const float* hw_embed, int32_t n_hotwords, const FaLongAudioOptions* opts) {
  g_err.clear();
  FaAudioFormat f;
  if (!pcm16k_format(pcm_format, f)) return fail("bad argument");
  return infer_vad(asr, vad, bufs, n_samples, batch, &f, hw_embed, n_hotwords, nullptr, nullptr, opts);
}

extern "C" void* fa_offline_infer_vad_sv(void* asr, void* vad, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                                         const int32_t* language_ids, const int32_t* textnorm_ids, const FaLongAudioOptions* opts) {
  g_err.clear();
  if (asr && !static_cast<Model*>(asr)->sv) return fail("fa_offline_infer_vad_sv: not a SenseVoice model file");
  FaAudioFormat f;
  if (!pcm16k_format(pcm_format, f)) return fail("bad argument");
  return infer_vad(asr, vad, bufs, n_samples, batch, &f, nullptr, 0, language_ids, textnorm_ids, opts);
}

extern "C" void* fa_offline_infer_vad_spk(void* asr, void* vad, void* spk, const void* const* bufs, const int64_t* n_samples, int32_t batch,
                                          int32_t pcm_format, const float* hw_embed, int32_t n_hotwords, const int32_t* language_ids,
                                          const int32_t* textnorm_ids, const FaLongAudioOptions* opts, int32_t preset_spk_num) {
  g_err.clear();
  if (!spk) return fail("fa_offline_infer_vad_spk: spk is NULL");
  if (asr && !static_cast<Model*>(asr)->sv && (language_ids || textnorm_ids)) return fail("fa_offline_infer_vad_spk: language / text-norm ids need a SenseVoice model file");
  FaAudioFormat f;
  if (!pcm16k_format(pcm_format, f)) return fail("bad argument");
  return infer_vad(asr, vad, bufs, n_samples, batch, &f, hw_embed, n_hotwords, language_ids, textnorm_ids, opts, static_cast<Spk*>(spk),
                   preset_spk_num);
}

extern "C" void* fa_offline_infer_vad_audio(void* asr, void* vad, void* spk, const void* const* bufs, const int64_t* n_samples, int32_t batch,
                                            const FaAudioFormat* fmt, const float* hw_embed, int32_t n_hotwords, const int32_t* language_ids,
                                            const int32_t* textnorm_ids, const FaLongAudioOptions* opts, int32_t preset_spk_num) {
  g_err.clear();
  if (asr && !static_cast<Model*>(asr)->sv && (language_ids || textnorm_ids))
    return fail("fa_offline_infer_vad_audio: language / text-norm ids need a SenseVoice model file");
  return infer_vad(asr, vad, bufs, n_samples, batch, fmt, hw_embed, n_hotwords, language_ids, textnorm_ids, opts, static_cast<Spk*>(spk),
                   preset_spk_num);
}

extern "C" const int32_t* fa_offline_result_spk(const void* result, int32_t index, int32_t* n) {
  return result_row(result ? &as_result(result)->spk : nullptr, index, n, 1, false);
}

extern "C" const int32_t* fa_offline_result_segments(const void* result, int32_t index, int32_t* n_segments) {
  return result_row(result ? &as_result(result)->segs : nullptr, index, n_segments, 3, false);
}
