// Handle-style FSMN-VAD: fa_vad_init (model file -> handle), fa_vad_infer (one recording -> [start_ms, end_ms] segments), and vad_run,
// which long audio (offline_long.cu) runs on a recording already on the device.
#include "handle.h"
#include <math.h>
#include <string.h>

using namespace fa_handle;

namespace {

// __vad_config__ of funasr_b200/pack.py:write_vad_model_file: float64 values stored as the bytes of an fp32 tensor (the detector
// compares in double precision: 0.6 and 1e-4 must arrive unrounded)
enum { kVadCfgInts = 14, kVadCfgDoubles = 5, kVadCfgLorder = 19, kVadCfgNSil = 20, kVadCfgSil = 21, kVadCfgLen = 25 };

bool build_vad(Vad& v, Builder& b) {
  const Tensor* cfg = b.get("__vad_config__");
  if (!cfg) return false;
  if (cfg->host.size() != 2 * kVadCfgLen) return b.refuse("bad __vad_config__");
  double c[kVadCfgLen];
  memcpy(c, cfg->host.data(), sizeof(c));
  int32_t* oi = &v.opts.sample_rate;                 // the 14 int32 fields, in declaration order
  for (int k = 0; k < kVadCfgInts; ++k) oi[k] = (int32_t)c[k];
  v.opts.speech_2_noise_ratio = c[14]; v.opts.snr_thres = c[15]; v.opts.decibel_thres = c[16]; v.opts.speech_noise_thres = c[17];
  v.opts.fe_prior_thres = c[18];
  const int lorder = (int)c[kVadCfgLorder], n_sil = (int)c[kVadCfgNSil];
  if (lorder != 20 || n_sil < 1 || n_sil > 4 || v.opts.frame_in_ms <= 0 || v.opts.window_size_ms < v.opts.frame_in_ms)
    return b.refuse("unsupported VAD config");
  b.fbank_tables();
  const Tensor* cmvn = b.opt("frontend.cmvn");
  if (cmvn && cmvn->numel() != 2 * 400) return b.refuse("frontend.cmvn must be [2, 400]");
  v.cmvn = cmvn ? cmvn->dev : nullptr;
  // weights [out, in] -> [out, in rounded up to 16] with zero columns (VadEngine._lin): the fp32 GEMMs read K = the padded width
  auto lin = [&](const std::string& p, bool bias) -> FaLinear {
    FaLinear L{};
    const Tensor* w = b.get(p + ".weight");
    if (!w || w->shape.size() != 2) { if (w) b.refuse("bad weight " + p); return L; }
    const int out_f = (int)w->shape[0], in_f = (int)w->shape[1], kp = (in_f + 15) / 16 * 16;
    const Tensor* bt = bias ? b.get(p + ".bias") : nullptr;
    if (bt && bt->numel() != out_f) b.refuse("bad bias " + p);
    if (!b.ok) return L;
    L.b = bt ? bt->dev : nullptr;
    L.out_f = out_f; L.in_f = kp; L.in_pad = kp;
    if (!b.f) return L;
    void* wp = b.f->alloc((size_t)out_f * kp * 4);
    if (!wp) { b.refuse("cudaMalloc weights"); return L; }
    if (cudaMemset(wp, 0, (size_t)out_f * kp * 4) != cudaSuccess ||
        cudaMemcpy2D(wp, (size_t)kp * 4, w->dev, (size_t)in_f * 4, (size_t)in_f * 4, out_f, cudaMemcpyDeviceToDevice) != cudaSuccess)
      b.refuse("weight copy failed");
    L.w = static_cast<const float*>(wp);
    return L;
  };
  int n_layers = 0;
  while (b.opt("encoder.fsmn." + std::to_string(n_layers) + ".linear.linear.weight")) ++n_layers;
  v.layers.resize(n_layers > 0 ? n_layers : 1);
  v.enc.in1 = lin("encoder.in_linear1.linear", true);
  v.enc.in2 = lin("encoder.in_linear2.linear", true);
  for (int i = 0; i < n_layers && b.ok; ++i) {
    const std::string p = "encoder.fsmn." + std::to_string(i) + ".";
    if (b.opt(p + "fsmn_block.conv_right.weight")) return b.refuse("FSMN-VAD with a right-context memory (rorder > 0) is not supported");
    v.layers[i].lin = lin(p + "linear.linear", false);
    const Tensor* cw = b.get(p + "fsmn_block.conv_left.weight");   // [proj, 1, lorder, 1] = [proj, lorder] contiguous
    if (!cw) return false;
    if (cw->shape.size() != 4 || cw->shape[1] != 1 || cw->shape[2] != lorder || cw->shape[3] != 1) return b.refuse("bad " + p + "fsmn_block.conv_left.weight");
    v.layers[i].conv_w = cw->dev;
    v.layers[i].affine = lin(p + "affine.linear", true);
  }
  v.enc.layers = v.layers.data(); v.enc.n_layers = n_layers; v.enc.lorder = lorder;
  v.enc.out1 = lin("encoder.out_linear1.linear", true);
  v.enc.out2 = lin("encoder.out_linear2.linear", true);
  for (int k = 0; k < n_sil; ++k) v.enc.sil_ids[k] = (int32_t)c[kVadCfgSil + k];
  v.enc.n_sil = n_sil;
  if (!b.ok) return false;
  if (v.enc.in1.in_f != 400) return b.refuse("the VAD frontend is 80 mel x LFR 5: in_linear1 must take 400 inputs");
  for (int k = 0; k < n_sil; ++k)
    if (v.enc.sil_ids[k] < 0 || v.enc.sil_ids[k] >= v.enc.out2.out_f) return b.refuse("sil_pdf_ids outside the output");
  return true;
}

const double kSilenceSchedule[] = {10000, 2000, 20000, 1000, 30000, 800, 40000, 600, 50000, 400, 60000, 200, -1, 100};   // vad.py

}  // namespace

namespace fa_handle {

bool vad_run_batch(Vad& v, const float* wav, int64_t stride, const int64_t* n, int B, cudaStream_t st, const FaVadRunOptions& ro,
                   std::vector<VadResult>& out) {
  out.assign(B, VadResult());
  std::vector<int32_t> io(2 * (size_t)B);                    // sample counts, then frame counts
  int32_t t_max = 0;
  for (int i = 0; i < B; ++i) {
    const int64_t T = n[i] >= 400 ? (n[i] - 400) / 160 + 1 : 0;
    out[i].audio_seconds = (float)((double)n[i] / 16000.0);
    out[i].frames.assign((size_t)(2 * T), 0.f);
    io[i] = (int32_t)n[i];
    io[B + i] = (int32_t)T;
    t_max = std::max(t_max, (int32_t)T);
  }
  if (t_max == 0) return true;                               // every recording shorter than one frame: nothing to score
  const size_t rows = (size_t)B * t_max;
  const size_t ws_bytes = fa_fsmn_vad_batch_workspace_bytes(&v.enc, B, t_max);
  int32_t *io_d, *flens;
  float *feats, *frames;
  void* ws;
  if (!carve(v.vad_run, "VAD", [&](fa::Arena& a) {
        io_d = a.take<int32_t>(io.size()); flens = a.take<int32_t>(B);
        feats = a.take<float>(rows * 400); frames = a.take<float>(rows * 2); ws = a.take<char>(ws_bytes);
      }))
    return false;
  cudaMemcpyAsync(io_d, io.data(), io.size() * 4, cudaMemcpyHostToDevice, st);
  int rc = fa_fbank_lfr_cmvn_tables(wav, io_d, B, stride, v.cmvn, v.file.fbank_tables, 5, 1, feats, t_max, flens, t_max, st);
  if (rc == FA_OK) rc = fa_fsmn_vad_forward_batch(&v.enc, feats, 400, io.data() + B, B, t_max, frames, ws, ws_bytes, st);
  if (rc == FA_OK) rc = fa_frame_decibels_batch(wav, stride, io_d + B, B, t_max, frames + rows, st);
  if (rc != FA_OK) { set_err(std::string("VAD: ") + fa_status_string(rc)); return false; }
  std::vector<float> frames_h(rows * 2);
  cudaMemcpyAsync(frames_h.data(), frames, rows * 8, cudaMemcpyDeviceToHost, st);     // the one copy back: two floats per frame
  if (!sync_stream(st)) return false;
  for (int i = 0; i < B; ++i) {
    const int64_t T = io[B + i];
    VadResult& r = out[i];
    if (T == 0) continue;
    std::copy(frames_h.begin() + (size_t)i * t_max, frames_h.begin() + (size_t)i * t_max + T, r.frames.begin());
    std::copy(frames_h.begin() + rows + (size_t)i * t_max, frames_h.begin() + rows + (size_t)i * t_max + T, r.frames.begin() + T);
    std::vector<double> sil(r.frames.begin(), r.frames.begin() + T), db(r.frames.begin() + T, r.frames.end());
    FaVadOptions o = v.opts;
    if (!ro.dynamic_silence && ro.max_end_silence_time > 0) o.max_end_silence_time = ro.max_end_silence_time;
    std::vector<int32_t> seg(128);
    for (;;) {
      const int64_t cap = (int64_t)seg.size() / 2;
      const int64_t k = fa_vad_detect_segments(sil.data(), db.data(), T, n[i], &o, 60000, ro.dynamic_silence ? 1 : 0, kSilenceSchedule,
                                               (int32_t)(sizeof(kSilenceSchedule) / sizeof(double) / 2), ro.speech_noise_thres, seg.data(), cap);
      if (k < 0) { set_err("fa_vad_detect_segments failed: posteriors must lie inside (0, 1)"); return false; }
      if (k <= cap) { seg.resize((size_t)(2 * k)); break; }
      seg.resize((size_t)(2 * k));
    }
    r.seg.swap(seg);
  }
  return true;
}

bool vad_run(Vad& v, const float* wav, int64_t n, cudaStream_t st, const FaVadRunOptions& ro, VadResult& out) {
  std::vector<VadResult> r;
  if (!vad_run_batch(v, wav, n, &n, 1, st, ro, r)) return false;
  out = std::move(r[0]);
  return true;
}

FaVadRunOptions default_vad_run() {
  FaVadRunOptions r;
  r.dynamic_silence = 1; r.max_end_silence_time = 0; r.speech_noise_thres = NAN;
  return r;
}

}  // namespace fa_handle

extern "C" void* fa_vad_init(const char* model_file, int32_t device) {
  g_err.clear();
  return open_handle(model_file, device, FA_GEMM_F32_SIMT, build_vad);
}

extern "C" void fa_vad_uninit(void* vad) { delete static_cast<Vad*>(vad); }

namespace {

// fa_vad_infer / fa_vad_infer_audio: one host recording -> 16 kHz on the device -> vad_run
void* vad_infer(void* vad, const void* buf, int64_t n_samples, const FaAudioFormat* fmt, const FaVadRunOptions* opts) {
  Vad* v = static_cast<Vad*>(vad);
  if (!v || (!buf && n_samples > 0) || n_samples < 0 || n_samples > 0x7fffffffLL) return fail("bad argument");
  Audio au;
  if (!plan_audio(fmt, v->resample, au)) return nullptr;
  const int64_t n16 = au.len16(n_samples);
  if (n16 > 0x7fffffffLL) return fail("bad argument");
  std::lock_guard<std::mutex> dev(v->mu);
  cudaSetDevice(v->file.device);
  std::unique_ptr<VadResult> r(new VadResult());
  float* wav = nullptr;
  if (!no_throw("fa_vad_infer: ", [&] {
        return upload(&buf, &n_samples, 1, (n16 + 3) / 4 * 4, au, v->resample, v->upload, v->file.st, &wav) &&
               vad_run(*v, wav, n16, v->file.st, opts ? *opts : default_vad_run(), *r);
      }))
    return nullptr;
  r->audio_seconds = (float)au.seconds(&n_samples, 1);
  return r.release();
}

}  // namespace

extern "C" void* fa_vad_infer(void* vad, const void* buf, int64_t n_samples, int32_t pcm_format, const FaVadRunOptions* opts) {
  g_err.clear();
  FaAudioFormat f;
  if (!pcm16k_format(pcm_format, f)) return fail("bad argument");
  return vad_infer(vad, buf, n_samples, &f, opts);
}

extern "C" void* fa_vad_infer_audio(void* vad, const void* buf, int64_t n_samples, const FaAudioFormat* fmt, const FaVadRunOptions* opts) {
  g_err.clear();
  return vad_infer(vad, buf, n_samples, fmt, opts);
}

extern "C" const int32_t* fa_vad_result_segments(const void* result, int64_t* n_segments) {
  const VadResult* r = static_cast<const VadResult*>(result);
  if (n_segments) *n_segments = r ? (int64_t)r->seg.size() / 2 : 0;
  return r && !r->seg.empty() ? r->seg.data() : nullptr;
}

extern "C" const float* fa_vad_result_frames(const void* result, int64_t* frames) {
  const VadResult* r = static_cast<const VadResult*>(result);
  if (frames) *frames = r ? (int64_t)r->frames.size() / 2 : 0;
  return r && !r->frames.empty() ? r->frames.data() : nullptr;
}

extern "C" float fa_vad_result_audio_seconds(const void* result) { return result ? static_cast<const VadResult*>(result)->audio_seconds : 0.f; }

extern "C" void fa_vad_free_result(void* result) { delete static_cast<VadResult*>(result); }
