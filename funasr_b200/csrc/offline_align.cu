// Handle-style MonotonicAligner (fa-zh; funasr/models/monotonic_aligner/model.py:182-267): [start_ms, end_ms] for each token of a
// transcript the caller already has.  The SAN-M encoder and CifPredictorV3's upsampled timestamp head on the device, the stamps of
// ts_prediction_lfr6_standard on the host (fa_ts_stamps_host); MonotonicAlignerB200.inference (modules.py) is the same chain in Python.
//
//   fa_align_init      model file (funasr_b200/pack.py:write_aligner_model_file) -> handle
//   fa_align_infer     batch of host PCM in any FaAudioFormat + one transcript (token ids) per utterance -> result
//   results            the recogniser's Result: fa_offline_result_{count, audio_seconds, ids, stamps}, fa_offline_free_result
#include "handle.h"

using namespace fa_handle;

namespace {

// __aligner_config__ of funasr_b200/pack.py:aligner_model_tensors
enum { kAlEnc = 0, kAlDModel, kAlHeads, kAlFeat, kAlEps, kAlThreshold, kAlEos, kAlCfgLen };

struct Aligner {
  std::mutex mu;                                     // device lock
  Loaded file;
  int mode = FA_GEMM_F32_SIMT;
  int enc_layers = 0, d_model = 0, heads = 0, feat_dim = 0, eos_id = -1;
  std::vector<FaEncLayer> enc_l;
  FaEncoder enc{};
  FaTimestampHead head{};
  const float* cmvn = nullptr;
  // device memory, each DevBuf carved by the function it is named after
  ResampleCache resample;
  DevBuf upload;                                     // align's batch
  DevBuf align;                                      // features, encoder output, the head's weights and fires
  DevBuf ws;                                         // the GEMM workspace of the encoder and the head
};

bool build_aligner(Aligner& m, Builder& b) {
  m.mode = b.mode;
  b.what = "MonotonicAligner model: ";
  if (b.opt("__config__")) return b.refuse("the file carries both __config__ (Paraformer) and __aligner_config__");
  if (b.opt("__sv_config__")) return b.refuse("the file carries both __sv_config__ (SenseVoice) and __aligner_config__");
  const Tensor* cfg = b.get("__aligner_config__");
  if (!cfg) return false;
  if (cfg->host.size() != kAlCfgLen) return b.refuse("bad __aligner_config__");
  const float* c = cfg->host.data();
  m.enc_layers = (int)c[kAlEnc]; m.d_model = (int)c[kAlDModel]; m.heads = (int)c[kAlHeads]; m.feat_dim = (int)c[kAlFeat];
  m.eos_id = (int)c[kAlEos];
  if (m.enc_layers < 1) return b.refuse("no encoder layer");
  const int hd = m.heads > 0 && m.d_model % m.heads == 0 ? m.d_model / m.heads : 0;
  if (!((m.d_model == 320 && hd == 80) || (m.d_model == 512 && hd == 128)))
    return b.refuse("d_model " + std::to_string(m.d_model) + " with " + std::to_string(m.heads) +
                    " heads (the attention runs d_model 320 as heads of 80 or d_model 512 as heads of 128)");
  if (m.feat_dim != 560) return b.refuse("feat_dim " + std::to_string(m.feat_dim) + " (the frontend is 80 mel x LFR 7 = 560)");
  const Tensor* cmvn = b.opt("frontend.cmvn");
  if (cmvn && cmvn->shape != std::vector<int64_t>{2, 560}) return b.refuse("frontend.cmvn must be [2, 560]");
  b.ln_eps = c[kAlEps];
  b.fbank_tables();
  m.cmvn = cmvn ? cmvn->dev : nullptr;
  bind_stack(b, false, m.enc_layers, m.feat_dim, m.d_model, m.heads, m.enc_l, m.enc);
  if (!b.ok) return false;
  b.what = "MonotonicAligner timestamp head: ";
  bind_ts_head(b, m.d_model, m.head);
  m.head.threshold = c[kAlThreshold];
  return b.ok;
}

// MonotonicAligner.inference over a padded batch already on the device (wav [B, stride], lens_h >= 400 samples each): one host-to-device
// copy of the sample and token counts, Fbank + LFR + CMVN, the encoder, the timestamp head, one copy of the encoder lengths and the
// head's weights and fires back, one synchronisation, then each utterance's stamps on the host.  n_tok[i]: the stamped tokens of
// utterance i (its transcript without a trailing eos_id).
bool align(Aligner& m, const float* wav, int64_t stride, const std::vector<int32_t>& lens_h, const int32_t* n_ids,
           const std::vector<int32_t>& n_tok, Result& r) {
  const int B = (int)lens_h.size(), D = m.d_model, F = m.feat_dim, U = m.head.up_times;
  cudaStream_t st = m.file.st;
  int T = 0;
  // sample counts [B], then token_num [B] = n_ids + 1: the transcript and its </s> (model.py:226-228)
  std::vector<int32_t> io((size_t)2 * B);
  for (int i = 0; i < B; ++i) {
    T = std::max(T, num_lfr_frames(lens_h[i]));
    io[i] = lens_h[i];
    io[B + i] = n_ids[i] + 1;
  }
  const int64_t TU = (int64_t)T * U;
  int32_t *io_d, *flens;
  float *feats, *enc, *us_alphas, *us_peaks;
  if (!carve(m.align, "aligner", [&](fa::Arena& a) {
        io_d = a.take<int32_t>(io.size()); flens = a.take<int32_t>(B);
        feats = a.take<float>((size_t)B * T * F); enc = a.take<float>((size_t)B * T * D);
        us_alphas = a.take<float>((size_t)B * TU); us_peaks = a.take<float>((size_t)B * TU);
      }))
    return false;
  const size_t ws = std::max(fa_sanm_encoder_workspace_bytes(B, T, m.mode), fa_timestamp_head_workspace_bytes(B, T, D, U, m.mode));
  if (!m.ws.reserve(ws)) { set_err("device allocation failed (workspace)"); return false; }
  cudaMemcpyAsync(io_d, io.data(), io.size() * 4, cudaMemcpyHostToDevice, st);
  int rc = fa_fbank_lfr_cmvn_tables(wav, io_d, B, stride, m.cmvn, m.file.fbank_tables, 7, 6, feats, T, flens, T, st);
  if (rc != FA_OK) { set_err(std::string("fa_fbank_lfr_cmvn_tables: ") + fa_status_string(rc)); return false; }
  rc = fa_sanm_encoder_forward(&m.enc, feats, flens, B, T, enc, m.mode, m.ws.p, m.ws.cap, st);
  if (rc != FA_OK) { set_err(std::string("fa_sanm_encoder_forward: ") + fa_status_string(rc)); return false; }
  // CifPredictorV3.get_upsample_timestamp (bicif_paraformer/cif_predictor.py:300-352)
  rc = fa_timestamp_head_forward(&m.head, enc, flens, io_d + B, B, T, us_alphas, us_peaks, m.mode, m.ws.p, m.ws.cap, st);
  if (rc != FA_OK) { set_err(std::string("timestamp head: ") + fa_status_string(rc)); return false; }
  std::vector<int32_t> enc_lens(B);
  std::vector<float> ua((size_t)B * TU), up((size_t)B * TU);
  cudaMemcpyAsync(enc_lens.data(), flens, (size_t)B * 4, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(ua.data(), us_alphas, ua.size() * 4, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(up.data(), us_peaks, up.size() * 4, cudaMemcpyDeviceToHost, st);
  if (!sync_stream(st)) return false;
  r.stamps.resize(B);
  for (int i = 0; i < B; ++i) {                              // model.py:243-247: each utterance's first 3 * enc_len frames
    const int64_t n = (int64_t)U * enc_lens[i];
    std::vector<int32_t>& sp = r.stamps[i];
    sp.resize((size_t)(2 * (n > 0 ? n : 1)));                // at most n - 1 spans
    const int64_t k = fa_ts_stamps_host(ua.data() + (size_t)i * TU, up.data() + (size_t)i * TU, n, n_tok[i], U, 0.0, sp.data(), n);
    if (k < 0) { set_err("fa_ts_stamps_host failed"); return false; }
    sp.resize((size_t)(2 * k));
  }
  return true;
}

// fa_align_infer's checks, all before any launch
bool check_transcripts(const Aligner& m, const int32_t* const* ids, const int32_t* n_ids, int B, std::vector<int32_t>& n_tok) {
  n_tok.assign(B, 0);
  for (int i = 0; i < B; ++i) {
    if (n_ids[i] < 0 || n_ids[i] > 0x7ffffffe) { set_err("utterance " + std::to_string(i) + ": bad transcript length " + std::to_string(n_ids[i])); return false; }
    if (n_ids[i] > 0 && (!ids || !ids[i])) { set_err("utterance " + std::to_string(i) + ": ids NULL with " + std::to_string(n_ids[i]) + " tokens"); return false; }
    // ts_prediction_lfr6_standard drops a trailing "</s>" before it counts the tokens
    n_tok[i] = n_ids[i] - (n_ids[i] > 0 && m.eos_id >= 0 && ids[i][n_ids[i] - 1] == m.eos_id ? 1 : 0);
  }
  return true;
}

}  // namespace

extern "C" void* fa_align_init(const char* model_file, int32_t device, int32_t gemm_mode) {
  g_err.clear();
  if (!model_file) return fail("model_file is NULL");
  if (!valid_gemm_mode(gemm_mode)) return fail("bad gemm_mode");
  return open_handle(model_file, device, gemm_mode, build_aligner);
}

extern "C" void fa_align_uninit(void* aligner) { delete static_cast<Aligner*>(aligner); }

extern "C" void* fa_align_infer(void* aligner, const void* const* bufs, const int64_t* n_frames, int32_t batch, const FaAudioFormat* fmt,
                                const int32_t* const* ids, const int32_t* n_ids) {
  g_err.clear();
  Aligner* mp = static_cast<Aligner*>(aligner);
  if (!mp || !bufs || !n_frames || !fmt || !n_ids || batch < 1) return fail("fa_align_infer: bad argument");
  Aligner& m = *mp;
  std::vector<int32_t> n_tok;
  if (!check_transcripts(m, ids, n_ids, batch, n_tok)) return nullptr;
  Audio au;
  if (!plan_audio(fmt, m.resample, au)) return nullptr;
  int64_t nmax = 0;
  std::vector<int32_t> lens_h(batch);
  for (int i = 0; i < batch; ++i) {
    const int64_t n16 = bufs[i] && n_frames[i] >= 0 && n_frames[i] <= 0x7fffffffLL ? au.len16(n_frames[i]) : 0;
    if (n16 < 400 || n16 > 0x7fffffffLL) return fail("utterance " + std::to_string(i) + ": needs >= 400 samples (25 ms)" + au.at16k());
    lens_h[i] = (int32_t)n16;
    nmax = std::max(nmax, n16);
  }
  std::lock_guard<std::mutex> dev(m.mu);
  cudaSetDevice(m.file.device);
  const int64_t stride = (nmax + 3) / 4 * 4;
  std::unique_ptr<Result> r(new Result());
  r->ts = true;
  r->token_num.assign(n_tok.begin(), n_tok.end());
  r->ids.resize(batch);
  for (int i = 0; i < batch; ++i)
    if (n_tok[i] > 0) r->ids[i].assign(ids[i], ids[i] + n_tok[i]);
  float* wav = nullptr;
  if (!no_throw("fa_align_infer: ", [&] {
        return upload(bufs, n_frames, batch, stride, au, m.resample, m.upload, m.file.st, &wav) &&
               align(m, wav, stride, lens_h, n_ids, n_tok, *r);
      }))
    return nullptr;
  r->audio_seconds = (float)au.seconds(n_frames, batch);
  return r.release();
}
