// Long audio through the handle API: the entries check their arguments and post the call to the recogniser's request pool
// (offline_pool.cu), which runs the VAD, packs each recording's segments as the reference does and decodes them; for fa_offline_infer_vad_spk
// it then diarizes the recordings with the CAM++ handle, one speaker stage per group of the pass (diarize).
#include "handle.h"

using namespace fa_handle;

namespace {

// fa_offline_infer_vad* / fa_offline_infer_vad_audio: every recording decoded as if on its own; lang / tn one query per recording (NULL = the defaults)
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
  Ticket t;
  t.au = au;
  if (opts) t.opts = *opts;
  else { t.opts.batch_size_s = 300; t.opts.batch_size_threshold_s = 60; t.opts.merge_vad = 0; t.opts.merge_length_s = 15; t.opts.vad = default_vad_run(); }
  t.n16.resize(batch);
  for (int i = 0; i < batch; ++i) {
    if ((!bufs[i] && n_samples[i] > 0) || n_samples[i] < 0 || n_samples[i] > 0x7fffffffLL) return fail("bad recording " + std::to_string(i));
    t.n16[i] = au.len16(n_samples[i]);
    if (t.n16[i] > 0x7fffffffLL) return fail("bad recording " + std::to_string(i));
  }
  t.bufs = bufs; t.n_samples = n_samples; t.batch = batch;
  t.hw_embed = hw_embed; t.n_hotwords = n_hotwords; t.lang = lang; t.tn = tn;
  t.long_audio = true; t.vad = vp; t.spk = spk; t.preset_spk_num = preset_spk_num;
  return pool_call(*mp, t);
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
