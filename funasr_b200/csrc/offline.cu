// Handle-style offline recogniser over the kernels of this library — the C-ABI counterpart of FunASR's C++ runtime
// surface (runtime/onnxruntime/include/funasrruntime.h:100-116: FunOfflineInit / FunOfflineInferBuffer / FunASRGetResult /
// FunASRFreeResult / FunOfflineUninit; its Paraformer::Forward is the same op chain with ONNX Runtime in the middle,
// runtime/onnxruntime/src/paraformer.cpp).  No Python, no torch: weights come from one flat file written by
// funasr_b200/pack.py (tensors under FunASR's own state_dict names), device memory from cudaMalloc.
//
//   fa_offline_init         model file -> handle (weights to HBM, fp16 planes for the tensor-core GEMMs)
//   fa_offline_infer        batch of host PCM buffers (f32 in [-1,1] or s16le) -> result (greedy token ids per utterance)
//   fa_offline_result_*     accessors;  fa_offline_free_result / fa_offline_uninit
//                           a BiCifParaformer file (its upsampled CIF timestamp head) adds per-token [start_ms, end_ms] stamps
//   fa_vad_init / fa_vad_infer       FSMN-VAD model file -> handle; one recording -> [start_ms, end_ms] segments
//   fa_offline_infer_vad    long recordings: VAD -> segments packed by duration -> each pack gathered on the device and decoded
//   fa_punc_init / fa_punc_infer     CT-Transformer model file -> handle; many texts -> punctuated texts, every text one window per
//                           lockstep step (the text walk: punc_text.cpp)
//   a SenseVoiceSmall file (__sv_config__) makes the same handle run SenseVoiceEngine's chain: per-utterance query rows
//                           (fa_sv_query_rows), the SAN-M and tp stacks, the CTC head; fa_offline_infer_sv / fa_offline_infer_vad_sv
//   a SeacoParaformer file (__seaco_config__): fa_offline_hotword_embed runs its hotword encoder (hotword.cu), the decode takes those
//                           rows through _seaco_decode_with_ASF (seaco_bias)
// The tokenizer (ids -> text) stays with the caller, like every other entry point of this ABI.
#include "common.cuh"
#include "punc_text.h"
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <exception>
#include <map>
#include <memory>
#include <string>
#include <vector>

namespace {

thread_local std::string g_err;
void set_err(const std::string& s) { g_err = s; }
std::nullptr_t fail(const std::string& s) { set_err(s); return nullptr; }

// f() with every C++ exception turned into an error message: none may cross the C ABI (a malformed file can ask for an absurd
// allocation)
template <typename F>
bool no_throw(const char* what, F f) {
  try {
    return f();
  } catch (const std::exception& e) {
    set_err(std::string(what) + e.what());
    return false;
  }
}

// the stream's work finished, or "CUDA error: ..." set
bool sync_stream(cudaStream_t st) {
  if (cudaStreamSynchronize(st) == cudaSuccess) return true;
  set_err(std::string("CUDA error: ") + cudaGetErrorString(cudaGetLastError()));
  return false;
}

struct Tensor {
  float* dev = nullptr;              // weights
  std::vector<float> host;           // the payload of the "__" configuration tensors, which stay on the host
  std::vector<int64_t> shape;
  int64_t numel() const { int64_t n = 1; for (auto d : shape) n *= d; return n; }
};

struct DevBuf {                      // grow-only device allocation
  void* p = nullptr;
  size_t cap = 0;
  bool reserve(size_t n) {
    if (n <= cap) return true;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    const size_t want = n + n / 8 + 4096;
    if (cudaMalloc(&p, want) != cudaSuccess) { cudaGetLastError(); return false; }
    cap = want;
    return true;
  }
  ~DevBuf() { if (p) cudaFree(p); }
};

bool read_exact(FILE* f, void* dst, size_t n) { return fread(dst, 1, n, f) == n; }

// File layout (funasr_b200/pack.py): "FAB2MDL1", u32 n_tensors, then per tensor:
//   u32 name_len, name, u32 ndim, i64 dims[ndim], u64 nbytes, zero padding to a 16-byte file offset, fp32 data
// The payload of a "__" configuration tensor is read into Tensor::host.  to_device = false skips the weights (names and shapes
// only): what can be checked before any device is touched.
bool load_file(std::map<std::string, Tensor>& tensors, const char* path, bool to_device = true) {
  FILE* f = fopen(path, "rb");
  if (!f) { set_err(std::string("cannot open ") + path); return false; }
  char magic[8];
  uint32_t n = 0;
  long fsize = 0;
  if (fseek(f, 0, SEEK_END) == 0) fsize = ftell(f);
  rewind(f);
  bool ok = fsize > 0 && read_exact(f, magic, 8) && memcmp(magic, "FAB2MDL1", 8) == 0 && read_exact(f, &n, 4);
  std::vector<float> host;
  for (uint32_t i = 0; ok && i < n; ++i) {
    uint32_t nl = 0, nd = 0;
    uint64_t nbytes = 0;
    ok = read_exact(f, &nl, 4) && nl < 4096;
    std::string name(ok ? nl : 0, '\0');
    ok = ok && read_exact(f, &name[0], nl) && read_exact(f, &nd, 4) && nd <= 8;
    Tensor tt;
    tt.shape.resize(nd);
    ok = ok && (nd == 0 || read_exact(f, tt.shape.data(), 8 * nd)) && read_exact(f, &nbytes, 8);
    if (!ok) break;
    const long pos = ftell(f);
    const long pad = (16 - pos % 16) % 16;
    ok = fseek(f, pad, SEEK_CUR) == 0 && nbytes == (uint64_t)tt.numel() * 4 &&
         pos + pad <= fsize && nbytes <= (uint64_t)(fsize - (pos + pad));   // the payload lies inside the file: a corrupt size cannot drive an allocation
    if (!ok) break;
    if (name.compare(0, 2, "__") == 0) {
      tt.host.resize(nbytes / 4);
      ok = read_exact(f, tt.host.data(), nbytes);
    } else if (!to_device) {
      ok = fseek(f, (long)nbytes, SEEK_CUR) == 0;
    } else {
      host.resize(nbytes / 4);
      ok = read_exact(f, host.data(), nbytes);
      if (!ok) break;
      if (cudaMalloc(&tt.dev, nbytes ? nbytes : 4) != cudaSuccess) { ok = false; set_err("cudaMalloc failed for " + name); break; }
      cudaMemcpy(tt.dev, host.data(), nbytes, cudaMemcpyHostToDevice);
    }
    if (!ok) break;
    tensors[name] = tt;
  }
  fclose(f);
  if (!ok && g_err.empty()) set_err(std::string("malformed model file ") + path);
  return ok;
}

// One model file loaded onto one device: its tensors, what the handle allocates beside them (weight planes, padded weights, the
// fbank tables), and the handle's stream
struct Loaded {
  int device = 0;
  std::map<std::string, Tensor> t;
  std::vector<void*> owned;
  cudaStream_t st = nullptr;
  float* fbank_tables = nullptr;
  bool open(const char* path, int dev) {
    if (cudaSetDevice(dev) != cudaSuccess) { cudaGetLastError(); set_err("no such CUDA device (this library has no CPU path)"); return false; }
    device = dev;
    if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) { set_err("cudaStreamCreate failed"); return false; }
    return load_file(t, path);
  }
  ~Loaded() {
    for (auto& kv : t) if (kv.second.dev) cudaFree(kv.second.dev);
    for (void* p : owned) cudaFree(p);
    if (st) cudaStreamDestroy(st);
  }
};

struct Model {
  Loaded file;
  int mode = 3;
  int enc_layers = 0, dec_layers = 0, d_model = 512, heads = 4, kernel = 11, vocab = 0, feat_dim = 560;
  float ln_eps = 1e-12f, cif_threshold = 1.f, tail_threshold = 0.45f;
  std::vector<FaEncLayer> enc_l;
  std::vector<FaDecLayer> dec_l;
  FaEncoder enc{};
  FaPredictor pred{};
  FaDecoder dec{};
  const float* cmvn = nullptr;
  DevBuf wav, pcm16, lens, feats, flens, encb, acoustic, tok, alphas, peaks, ws, ids, best, fids, flens_out, hw, hw_lens;
  DevBuf rec, gmeta;                                 // fa_offline_infer_vad: the device-resident recording, per-pack gather offsets
  bool contextual = false;                           // ContextualParaformer: decoder with a hotword bias branch
  bool ts = false;                                   // BiCifParaformer: CifPredictorV3's upsampled timestamp head
  FaTimestampHead head{};
  DevBuf us_alphas, us_peaks;
  std::map<std::string, std::vector<float>> host_cache;   // fa_offline_host_tensor
  bool sv = false;                                   // SenseVoiceSmall (__sv_config__): query rows, the SAN-M and tp stacks, the CTC head
  int tp_layers = 0, n_embed = 0, blank = 0;
  std::vector<FaEncLayer> tp_l;
  FaEncoder tp{};
  FaLinear ctc{};
  const float* embed = nullptr;
  DevBuf enc2, am;
  bool seaco = false;                                // SeacoParaformer (__seaco_config__): hotword encoder, SeACo decoder, NO_BIAS merge
  int no_bias = 0, nfilter = 0;
  std::vector<FaDecLayer> seaco_l;
  FaDecoder seaco_dec{};
  FaLinear hw_out{};
  std::vector<FaLinear> hw_ih, hw_hh;
  FaHotwordEncoder hw_enc{};
  DevBuf hw_rows, hidden, cif_att, dec_att, dha_ids, dha_best, sids, sbest, probs, hw_sel, sel_lens;
};

struct Result {
  std::vector<std::vector<int32_t>> ids;
  std::vector<int32_t> token_num;
  std::vector<std::vector<int32_t>> segs;            // fa_offline_infer_vad: {start_ms, end_ms, n_tokens} per segment, per recording
  bool ts = false;                                   // the model has the timestamp head: stamps[i] = {start_ms, end_ms} pairs
  std::vector<std::vector<int32_t>> stamps;
  std::vector<std::vector<int32_t>> spk;             // fa_offline_infer_vad_spk: one speaker per segment of a diarized recording
  float audio_seconds = 0.f;
};

__global__ void pcm16_to_f32_kernel(const int16_t* __restrict__ src, float* __restrict__ dst, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (float)src[i] * (1.0f / 32768.0f);     // exact; the frontend multiplies by 32768 again (wav_frontend.py:169)
}

// B host recordings bufs[i] of n[i] samples (f32, or s16le staged in pcm16) into rows of `stride` floats of dst
bool upload(const void* const* bufs, const int64_t* n, int B, int64_t stride, int32_t pcm_format, DevBuf& dst, DevBuf& pcm16,
            cudaStream_t st) {
  const int64_t tot = (int64_t)B * stride;
  if (!dst.reserve((size_t)(tot > 0 ? tot : 4) * 4)) { set_err("device allocation failed (waveforms)"); return false; }
  if (tot == 0) return true;
  float* wav = static_cast<float*>(dst.p);
  if (pcm_format == 1) {
    if (!pcm16.reserve((size_t)tot * 2)) { set_err("device allocation failed (pcm)"); return false; }
    int16_t* p16 = static_cast<int16_t*>(pcm16.p);
    for (int i = 0; i < B; ++i) cudaMemcpyAsync(p16 + (int64_t)i * stride, bufs[i], (size_t)n[i] * 2, cudaMemcpyHostToDevice, st);
    pcm16_to_f32_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(p16, wav, tot);
  } else {
    for (int i = 0; i < B; ++i) cudaMemcpyAsync(wav + (int64_t)i * stride, bufs[i], (size_t)n[i] * 4, cudaMemcpyHostToDevice, st);
  }
  return true;
}

// One model kind's description, run twice: over the file's index (f == nullptr: names and shapes only, nothing touches a device),
// then over the loaded file.  A file the index pass accepts is refused later only for a device failure.
struct Builder {
  const std::map<std::string, Tensor>& t;
  Loaded* f;                                         // nullptr: the index pass
  int mode = FA_GEMM_F32_SIMT;
  float ln_eps = 0.f;
  std::string what;                                  // prefix of every message: the model kind or the part being bound
  bool ok = true;                                    // the first refusal is the one reported
  bool refuse(const std::string& s) {
    if (ok) set_err(what + s);
    ok = false;
    return false;
  }
  const Tensor* opt(const std::string& k) const {
    auto it = t.find(k);
    return it == t.end() ? nullptr : &it->second;
  }
  const Tensor* get(const std::string& k) {
    const Tensor* x = opt(k);
    if (!x) refuse("missing tensor " + k);
    return x;
  }
  const Tensor* shaped(const std::string& k, std::initializer_list<int64_t> dims) {
    const Tensor* x = get(k);
    if (x && !std::equal(dims.begin(), dims.end(), x->shape.begin(), x->shape.end())) refuse("bad shape of " + k);
    return x;
  }
  const float* ptr(const std::string& k) { const Tensor* x = get(k); return x ? x->dev : nullptr; }   // nullptr on the index
  FaNorm norm(const std::string& p) {
    FaNorm nm{};
    const Tensor* w = get(p + ".weight");
    nm.g = w ? w->dev : nullptr; nm.b = ptr(p + ".bias"); nm.n = w ? (int32_t)w->numel() : 0; nm.eps = ln_eps;
    return nm;
  }
  FaLinear lin(const std::string& p, bool bias = true, const char* weight_key = nullptr, const char* bias_key = nullptr) {
    FaLinear L{};
    const Tensor* w = get(weight_key ? std::string(weight_key) : p + ".weight");
    // [out, in] or a k = 1 Conv1d weight [out, in, 1] (bias_output, contextual_paraformer/decoder.py:287)
    if (!w || !(w->shape.size() == 2 || (w->shape.size() == 3 && w->shape[2] == 1))) { if (w) refuse("bad weight " + p); return L; }
    L.w = w->dev; L.b = bias ? ptr(bias_key ? std::string(bias_key) : p + ".bias") : nullptr;
    L.out_f = (int32_t)w->shape[0]; L.in_f = (int32_t)w->shape[1]; L.in_pad = (L.in_f + 63) / 64 * 64;
    if (mode != FA_GEMM_F32_SIMT && f) {
      void* planes = nullptr;
      if (cudaMalloc(&planes, (size_t)3 * L.out_f * L.in_pad * 2) != cudaSuccess) { refuse("cudaMalloc planes"); return L; }
      f->owned.push_back(planes);
      if (fa_split_planes(L.w, L.in_f, L.out_f, L.in_f, L.in_pad, planes, f->st) != FA_OK) refuse("fa_split_planes failed");
      L.w_planes = planes;
    }
    return L;
  }
  // the frontend's fbank tables (fa_fbank_make_tables) from frontend.mel_banks and frontend.window
  void fbank_tables() {
    const Tensor* mel = get("frontend.mel_banks");
    const Tensor* win = get("frontend.window");
    if (!mel || !win || !f) return;
    void* tb = nullptr;
    if (cudaMalloc(&tb, fa_fbank_tables_bytes()) != cudaSuccess) { refuse("cudaMalloc fbank tables"); return; }
    f->owned.push_back(tb);
    f->fbank_tables = static_cast<float*>(tb);
    if (fa_fbank_make_tables(mel->dev, win->dev, f->fbank_tables, f->st) != FA_OK) refuse("fa_fbank_make_tables failed");
  }
};

// fa_offline_init / fa_vad_init / fa_punc_init: build() over the file's index into a throwaway handle (every refusal before any device
// work, naming the piece), then over the loaded file into the handle returned
template <typename H>
H* open_handle(const char* path, int device, int mode, bool (*build)(H&, Builder&)) {
  if (!path) return fail("model_file is NULL");
  std::unique_ptr<H> h;
  const bool ok = no_throw("model file rejected: ", [&] {
    std::map<std::string, Tensor> index;
    H probe;
    Builder on_index{index, nullptr, mode};
    if (!load_file(index, path, false) || !build(probe, on_index)) return false;
    h.reset(new H());
    Builder on_device{h->file.t, &h->file, mode};
    return h->file.open(path, device) && build(*h, on_device) && sync_stream(h->file.st);
  });
  return ok ? h.release() : nullptr;
}

// SANMEncoder keeps its first layer (input width -> d_model) apart as encoders0.0 (sanm/encoder.py:188-461); SenseVoice's
// tp_encoders are one plain list
std::string enc_layer_prefix(bool tp, int i) {
  if (tp) return "encoder.tp_encoders." + std::to_string(i);
  return i == 0 ? "encoder.encoders0.0" : "encoder.encoders." + std::to_string(i - 1);
}

// A SAN-M stack of n layers over `in` input features into e and L, in the shapes fa_sanm_encoder_forward takes: QKV [3D, in], FSMN
// [D, 1, K] with layer 0's K in every layer, FFN [F, D] / [D, F] with F <= 2048 (enc_carve's bound).  The main stack takes the
// position encoding and ends in encoder.after_norm; SenseVoice's tp stack (D in, possibly empty) in encoder.tp_norm.
void bind_stack(Builder& b, bool tp, int n, int in, int D, int heads, std::vector<FaEncLayer>& L, FaEncoder& e) {
  auto norm = [&](const std::string& p, int64_t w) {
    b.shaped(p + ".weight", {w}); b.shaped(p + ".bias", {w});
    return b.norm(p);
  };
  auto lin = [&](const std::string& p, int64_t out, int64_t k) {
    b.shaped(p + ".weight", {out, k}); b.shaped(p + ".bias", {out});
    return b.lin(p);
  };
  const Tensor* k0 = n > 0 ? b.get(enc_layer_prefix(tp, 0) + ".self_attn.fsmn_block.weight") : nullptr;
  const int64_t K = k0 && k0->shape.size() == 3 ? k0->shape[2] : 0;
  L.assign(n > 0 ? n : 1, FaEncLayer{});
  for (int i = 0; i < n; ++i) {
    const std::string p = enc_layer_prefix(tp, i);
    const int64_t x = i == 0 ? in : D;
    const Tensor* w1 = b.get(p + ".feed_forward.w_1.weight");
    const int64_t F = w1 && w1->shape.size() == 2 ? w1->shape[0] : 0;
    if (w1 && (F < 1 || F > 2048)) b.refuse("bad shape of " + p + ".feed_forward.w_1.weight (at most 2048 units)");
    L[i].norm1 = norm(p + ".norm1", x); L[i].norm2 = norm(p + ".norm2", D);
    L[i].qkv = lin(p + ".self_attn.linear_q_k_v", 3 * D, x); L[i].out = lin(p + ".self_attn.linear_out", D, D);
    b.shaped(p + ".self_attn.fsmn_block.weight", {D, 1, K});
    L[i].fsmn_w = b.ptr(p + ".self_attn.fsmn_block.weight");
    L[i].w1 = lin(p + ".feed_forward.w_1", F, D); L[i].w2 = lin(p + ".feed_forward.w_2", D, F);
  }
  e = FaEncoder{};
  e.layers = L.data(); e.n_layers = n; e.heads = heads; e.fsmn_k = (int)K;
  if (n > 0) e.after_norm = norm(tp ? "encoder.tp_norm" : "encoder.after_norm", D);
  if (!tp) {
    b.shaped("encoder.pe_inv_timescales", {in / 2});
    e.pe_inv_timescales = b.ptr("encoder.pe_inv_timescales");
  }
}

// A Paraformer file (ParaformerEngine, engine.py): plain, contextual (a hotword bias decoder) or BiCif (a timestamp head)
bool build_paraformer(Model& m, Builder& b) {
  m.mode = b.mode;
  // BiCifParaformer's timestamp head, recognised by predictor.upsample_cnn.weight: the tensors its launches read, in the shapes
  // pack.py:timestamp_head_tensors writes, and __ts_config__.  Bound first: its refusals come before the rest of the file's.
  m.ts = b.opt("predictor.upsample_cnn.weight") != nullptr;
  if (m.ts) {
    const Tensor* tc = b.opt("__ts_config__");
    if (!tc || tc->host.size() < 3)
      return b.refuse("BiCif timestamp head without __ts_config__ (a file packed before the handle read the head): re-pack it with "
                      "funasr_b200.pack.write_model_file");
    const float* c = tc->host.data();
    if (c[0] != 3.f) return b.refuse("BiCif timestamp head: upsample_times " + std::to_string(c[0]) + " in __ts_config__, only 3 is supported");
    b.what = "BiCif timestamp head: ";
    b.shaped("predictor.upsample_cnn.gemm_weight", {3 * 512, 512}); b.shaped("predictor.upsample_cnn.gemm_bias", {3 * 512});
    b.shaped("predictor.blstm.ih_gemm_weight", {8 * 512, 512});     b.shaped("predictor.blstm.ih_gemm_bias", {8 * 512});
    b.shaped("predictor.blstm.weight_hh_l0", {4 * 512, 512});       b.shaped("predictor.blstm.weight_hh_l0_reverse", {4 * 512, 512});
    b.shaped("predictor.cif_output2.weight", {1, 2 * 512});         b.shaped("predictor.cif_output2.bias", {1});
    FaTimestampHead& h = m.head;
    h.up_times = 3; h.smooth2 = c[1]; h.noise2 = c[2];
    h.upsample = b.lin("predictor.upsample_cnn", true, "predictor.upsample_cnn.gemm_weight", "predictor.upsample_cnn.gemm_bias");
    h.blstm_ih = b.lin("predictor.blstm.ih", true, "predictor.blstm.ih_gemm_weight", "predictor.blstm.ih_gemm_bias");
    h.w_hh_fwd = b.ptr("predictor.blstm.weight_hh_l0"); h.w_hh_bwd = b.ptr("predictor.blstm.weight_hh_l0_reverse");
    h.out2_w = b.ptr("predictor.cif_output2.weight"); h.out2_b = b.ptr("predictor.cif_output2.bias");
    b.what.clear();
  }
  const Tensor* cfg = b.opt("__config__");
  if (!cfg || cfg->host.size() < 10) return b.refuse("missing __config__");
  const float* c = cfg->host.data();
  m.enc_layers = (int)c[0]; m.dec_layers = (int)c[1]; m.d_model = (int)c[2]; m.heads = (int)c[3]; m.kernel = (int)c[4];
  m.vocab = (int)c[5]; m.feat_dim = (int)c[6]; m.ln_eps = c[7]; m.cif_threshold = c[8]; m.tail_threshold = c[9];
  if (m.enc_layers < 1 || m.dec_layers < 1 || m.d_model != 512 || m.heads * 128 != m.d_model) return b.refuse("unsupported config");
  b.ln_eps = m.ln_eps;
  b.fbank_tables();
  const Tensor* cmvn = b.opt("frontend.cmvn");
  m.cmvn = cmvn ? cmvn->dev : nullptr;
  // encoder (engine.py:_enc_stack; SANMEncoder encoder.py:188-461)
  bind_stack(b, false, m.enc_layers, m.feat_dim, m.d_model, m.heads, m.enc_l, m.enc);
  // predictor (CifPredictorV2 cif_predictor.py:209-314); conv weight already repacked to [512, 3*512] by pack.py
  m.pred.conv = b.lin("predictor.cif_conv1d", true, "predictor.cif_conv1d.gemm_weight");
  m.pred.out_w = b.ptr("predictor.cif_output.weight"); m.pred.out_b = b.ptr("predictor.cif_output.bias");
  m.pred.threshold = m.cif_threshold; m.pred.tail_threshold = m.tail_threshold; m.pred.smooth_factor = 1.f; m.pred.noise_threshold = 0.f;
  if (m.ts) {                   // BiCifParaformer: CifPredictorV3's sequential fp32 `cif` (bicif_paraformer/cif_predictor.py:37-84)
    m.pred.cif_variant = 1;
    m.head.threshold = m.cif_threshold;
  }
  // decoder (ParaformerSANMDecoder decoder.py:234-449)
  auto dec_layer = [&](FaDecLayer& L, const std::string& p, bool full) {
    L.norm1 = b.norm(p + ".norm1");
    L.ffn_w1 = b.lin(p + ".feed_forward.w_1"); L.ffn_norm = b.norm(p + ".feed_forward.norm"); L.ffn_w2 = b.lin(p + ".feed_forward.w_2", false);
    if (full) {
      L.norm2 = b.norm(p + ".norm2"); L.norm3 = b.norm(p + ".norm3");
      L.fsmn_w = b.ptr(p + ".self_attn.fsmn_block.weight");
      L.q = b.lin(p + ".src_attn.linear_q"); L.kv = b.lin(p + ".src_attn.linear_k_v"); L.out = b.lin(p + ".src_attn.linear_out");
    }
  };
  // ContextualParaformerDecoder (contextual_paraformer/decoder.py:133-352): the last attention layer is `last_decoder`, plus the
  // hotword branch bias_decoder (norm3 + cross attention) and bias_output (Conv1d 1024 -> 512, k = 1)
  m.contextual = b.opt("decoder.bias_decoder.norm3.weight") != nullptr;
  if (m.contextual && b.opt("__seaco_config__"))
    return b.refuse("SeACo model: the file carries both a contextual decoder.bias_decoder and __seaco_config__");
  const int n_plain = m.contextual ? m.dec_layers - 1 : m.dec_layers;
  m.dec_l.resize(n_plain > 0 ? n_plain : 1);
  for (int i = 0; i < n_plain; ++i) dec_layer(m.dec_l[i], "decoder.decoders." + std::to_string(i), true);
  m.dec.layers = m.dec_l.data(); m.dec.n_layers = n_plain; m.dec.heads = m.heads; m.dec.vocab = m.vocab;
  // the decoder's FSMN tap count is its own: encoder and decoder kernel_size are independent constructor arguments in the reference
  // (sanm/encoder.py:188, paraformer/decoder.py:234 — decoder default 21)
  const Tensor* dk = b.get(n_plain > 0 ? "decoder.decoders.0.self_attn.fsmn_block.weight" : "decoder.last_decoder.self_attn.fsmn_block.weight");
  m.dec.fsmn_k = dk && dk->shape.size() == 3 ? (int)dk->shape[2] : m.kernel;
  dec_layer(m.dec.last, "decoder.decoders3.0", false);
  m.dec.after_norm = b.norm("decoder.after_norm"); m.dec.output = b.lin("decoder.output_layer");
  m.dec.has_bias = 0;
  if (m.contextual) {
    dec_layer(m.dec.bias_last, "decoder.last_decoder", true);
    m.dec.bias_norm3 = b.norm("decoder.bias_decoder.norm3");
    m.dec.bias_q = b.lin("decoder.bias_decoder.src_attn.linear_q"); m.dec.bias_kv = b.lin("decoder.bias_decoder.src_attn.linear_k_v");
    m.dec.bias_out = b.lin("decoder.bias_decoder.src_attn.linear_out");
    m.dec.bias_output = b.lin("decoder.bias_output", false);
    m.dec.clas_scale = 1.0f;
  }
  const Tensor* sc = b.opt("__seaco_config__");
  m.seaco = sc != nullptr;
  if (m.seaco && b.ok) {
    b.what = "SeACo model: ";
    if (sc->host.size() != 3) return b.refuse("bad __seaco_config__");
    m.no_bias = (int)sc->host[0]; m.nfilter = (int)sc->host[1];
    const int layers = (int)sc->host[2], D = m.d_model;
    if (m.no_bias < 0 || m.no_bias >= m.vocab)
      return b.refuse("no_bias " + std::to_string(m.no_bias) + " outside the vocabulary [0, " + std::to_string(m.vocab) + ")");
    if (m.nfilter < 0) return b.refuse("nfilter " + std::to_string(m.nfilter) + " < 0");
    if (layers < 1 || layers > FA_HOTWORD_MAX_LAYERS) return b.refuse("bias_encoder with " + std::to_string(layers) + " layers");
    // the hotword encoder (seaco_paraformer/model.py:384-420): decoder.embed, then the bias_encoder LSTM; the GEMM bias b_ih + b_hh
    // comes folded from pack.py
    const Tensor* emb = b.shaped("decoder.embed.0.weight", {m.vocab, D});
    m.hw_ih.assign(layers, FaLinear{}); m.hw_hh.assign(layers, FaLinear{});
    for (int k = 0; k < layers; ++k) {
      const std::string s = std::to_string(k);
      b.shaped("bias_encoder.weight_ih_l" + s, {4 * D, D}); b.shaped("bias_encoder.weight_hh_l" + s, {4 * D, D});
      b.shaped("bias_encoder.bias_ih_l" + s, {4 * D}); b.shaped("bias_encoder.bias_hh_l" + s, {4 * D});
      b.shaped("bias_encoder.gemm_bias_l" + s, {4 * D});
      if (!b.ok) return false;
      m.hw_ih[k] = b.lin("bias_encoder.ih_l" + s, true, ("bias_encoder.weight_ih_l" + s).c_str(), ("bias_encoder.gemm_bias_l" + s).c_str());
      m.hw_hh[k] = b.lin("bias_encoder.hh_l" + s, false, ("bias_encoder.weight_hh_l" + s).c_str());
    }
    if (b.opt("bias_encoder.weight_ih_l" + std::to_string(layers))) return b.refuse("more bias_encoder layers than __seaco_config__ says");
    m.hw_enc = FaHotwordEncoder{emb ? emb->dev : nullptr, m.vocab, layers, m.hw_ih.data(), m.hw_hh.data()};
    // the SeACo decoder (model.py:100-110): ParaformerSANMDecoder without input / output layer; forward_asf6 reads layers 0..5
    int n_s = 0;
    while (b.opt("seaco_decoder.decoders." + std::to_string(n_s) + ".norm1.weight")) ++n_s;
    if (n_s < 6) return b.refuse(n_s == 0 ? std::string("missing tensor seaco_decoder.decoders.0.norm1.weight")
                                           : "seaco_decoder with " + std::to_string(n_s) + " attention layers (the attention-score filter reads 6)");
    const Tensor* sk = b.get("seaco_decoder.decoders.0.self_attn.fsmn_block.weight");
    const int64_t K = sk && sk->shape.size() == 3 ? sk->shape[2] : 0;
    m.seaco_l.assign(n_s, FaDecLayer{});
    for (int i = 0; i < n_s && b.ok; ++i) {
      const std::string p = "seaco_decoder.decoders." + std::to_string(i);
      const Tensor* w1 = b.get(p + ".feed_forward.w_1.weight");
      const int64_t F = w1 && w1->shape.size() == 2 ? w1->shape[0] : 0;
      if (w1 && (F < 1 || F > 2048)) return b.refuse("bad shape of " + p + ".feed_forward.w_1.weight (at most 2048 units)");
      b.shaped(p + ".feed_forward.w_1.weight", {F, D}); b.shaped(p + ".feed_forward.w_2.weight", {D, F});
      b.shaped(p + ".self_attn.fsmn_block.weight", {D, 1, K});
      b.shaped(p + ".src_attn.linear_q.weight", {D, D}); b.shaped(p + ".src_attn.linear_k_v.weight", {2 * D, D});
      b.shaped(p + ".src_attn.linear_out.weight", {D, D});
      dec_layer(m.seaco_l[i], p, true);
    }
    m.seaco_dec = FaDecoder{};
    m.seaco_dec.layers = m.seaco_l.data(); m.seaco_dec.n_layers = n_s; m.seaco_dec.heads = m.heads; m.seaco_dec.fsmn_k = (int)K;
    dec_layer(m.seaco_dec.last, "seaco_decoder.decoders3.0", false);
    m.seaco_dec.after_norm = b.norm("seaco_decoder.after_norm");
    b.shaped("hotword_output_layer.weight", {m.vocab, D}); b.shaped("hotword_output_layer.bias", {m.vocab});
    m.hw_out = b.lin("hotword_output_layer");
    b.what.clear();
  }
  return b.ok;
}

int num_lfr_frames(int64_t n) {       // wav_frontend.py:73 after kaldi.py snip_edges framing
  const int64_t mfr = n >= 400 ? 1 + (n - 400) / 160 : 0;
  return (int)((mfr + 5) / 6);
}

// SeACo's hotword biasing after the decoder (_seaco_decode_with_ASF, seaco_paraformer/model.py:271-382, as ParaformerEngine.seaco_decode
// runs it): the host hotword rows hw_host [n_hw, 512] on the device; with more rows than nfilter, the attention-score filter on
// utterance 0 (one host round trip: its probabilities out, fa_seaco_asf_select_host, the picked host rows back in); the SeACo decoder
// over the acoustic embeddings and over the decoder's hidden states; hotword_output_layer's arg-max over their sum; the NO_BIAS merge
// into m.sids.  m.ids / m.best / m.hidden hold the decoder's outputs, the workspace is sized for the stack and the arg-max.
bool seaco_bias(Model& m, int B, int n_max, int n_cap, const float* hw_host, int n_hw) {
  cudaStream_t st = m.file.st;
  const int D = m.d_model, V = m.vocab, n_s = m.seaco_dec.n_layers;
  const int64_t rows = (int64_t)B * n_max;
  if (!(m.hw_rows.reserve((size_t)n_hw * D * 4) && m.cif_att.reserve((size_t)rows * D * 4) && m.dec_att.reserve((size_t)rows * D * 4) &&
        m.dha_ids.reserve((size_t)rows * 4) && m.dha_best.reserve((size_t)rows * 4) && m.sids.reserve((size_t)rows * 4) &&
        m.sbest.reserve((size_t)rows * 4) && m.sel_lens.reserve((size_t)B * 4))) {
    set_err("device allocation failed (SeACo)");
    return false;
  }
  const float* hidden = static_cast<const float*>(m.hidden.p);
  const int32_t* tok = static_cast<const int32_t*>(m.tok.p);
  float* mem = static_cast<float*>(m.hw_rows.p);
  int32_t* mem_lens = static_cast<int32_t*>(m.sel_lens.p);
  cudaMemcpyAsync(mem, hw_host, (size_t)n_hw * D * 4, cudaMemcpyHostToDevice, st);
  int n_sel = n_hw;
  std::vector<float> picked_rows;
  int rc = FA_OK;
  if (m.nfilter > 0 && m.nfilter < n_hw) {                   // ASF (model.py:320-343): forward_asf6 on utterance 0
    const int H = m.seaco_dec.heads;
    const int32_t one = n_hw;
    if (!m.probs.reserve((size_t)H * n_max * n_hw * 4)) { set_err("device allocation failed (SeACo filter)"); return false; }
    cudaMemcpyAsync(mem_lens, &one, 4, cudaMemcpyHostToDevice, st);
    rc = fa_sanm_decoder_stack_forward(&m.seaco_dec, mem, mem_lens, 1, 1, n_hw, hidden, n_max, tok, n_max, 6, 0, nullptr,
                                       static_cast<float*>(m.probs.p), m.mode, m.ws.p, m.ws.cap, st);
    if (rc != FA_OK) { set_err(std::string("SeACo filter: ") + fa_status_string(rc)); return false; }
    std::vector<float> probs((size_t)H * n_max * n_hw);
    cudaMemcpyAsync(probs.data(), m.probs.p, probs.size() * 4, cudaMemcpyDeviceToHost, st);
    if (!sync_stream(st)) return false;
    std::vector<int32_t> picked((size_t)n_hw);
    n_sel = fa_seaco_asf_select_host(probs.data(), H, n_max, n_hw, m.nfilter, picked.data());
    if (n_sel < 1) { set_err("fa_seaco_asf_select_host failed"); return false; }
    picked_rows.resize((size_t)n_sel * D);
    for (int j = 0; j < n_sel; ++j) std::copy(hw_host + (size_t)picked[j] * D, hw_host + (size_t)(picked[j] + 1) * D, picked_rows.begin() + (size_t)j * D);
    cudaMemcpyAsync(mem, picked_rows.data(), picked_rows.size() * 4, cudaMemcpyHostToDevice, st);
  }
  const std::vector<int32_t> lens_h(B, n_sel);
  cudaMemcpyAsync(mem_lens, lens_h.data(), (size_t)B * 4, cudaMemcpyHostToDevice, st);
  float* cif_att = static_cast<float*>(m.cif_att.p);
  float* dec_att = static_cast<float*>(m.dec_att.p);
  rc = fa_sanm_decoder_stack_forward(&m.seaco_dec, mem, mem_lens, 1, B, n_sel, static_cast<const float*>(m.acoustic.p), n_cap, tok, n_max, n_s, 1,
                                     cif_att, nullptr, m.mode, m.ws.p, m.ws.cap, st);
  if (rc == FA_OK)
    rc = fa_sanm_decoder_stack_forward(&m.seaco_dec, mem, mem_lens, 1, B, n_sel, hidden, n_max, tok, n_max, n_s, 1, dec_att, nullptr, m.mode,
                                       m.ws.p, m.ws.cap, st);
  if (rc == FA_OK)
    rc = fa_linear_argmax(&m.hw_out, cif_att, dec_att, rows, static_cast<int32_t*>(m.dha_ids.p), static_cast<float*>(m.dha_best.p), nullptr,
                          m.mode, m.ws.p, m.ws.cap, st);
  if (rc == FA_OK)
    rc = fa_seaco_merge(static_cast<int32_t*>(m.ids.p), static_cast<float*>(m.best.p), static_cast<int32_t*>(m.dha_ids.p),
                        static_cast<float*>(m.dha_best.p), rows, m.no_bias, static_cast<int32_t*>(m.sids.p), static_cast<float*>(m.sbest.p),
                        nullptr, nullptr, nullptr, V, st);
  if (rc != FA_OK) { set_err(std::string("SeACo decoder: ") + fa_status_string(rc)); return false; }
  return sync_stream(st);                                    // lens_h and picked_rows are host vectors of this frame
}

// The recogniser over a padded batch already on the device: wav [B, stride] fp32 (m.wav or any buffer the call does not reuse),
// lens_h [B] samples (>= 400 each).  Everything after the host-to-device copy of fa_offline_infer_hw; fa_offline_infer_vad feeds it the
// gathered VAD segments of one pack.
std::unique_ptr<Result> decode_batch(Model& m, const float* wav, int64_t stride, const std::vector<int32_t>& lens_h, const float* hw_embed,
                                     int32_t n_hotwords) {
  const int B = (int)lens_h.size(), D = m.d_model;
  cudaStream_t st = m.file.st;
  int t_max = 0;
  double seconds = 0.0;
  for (int i = 0; i < B; ++i) {
    const int t = num_lfr_frames(lens_h[i]);
    t_max = t > t_max ? t : t_max;
    seconds += (double)lens_h[i] / 16000.0;
  }
  const int T = t_max;
  if (!m.lens.reserve((size_t)B * 4)) return fail("device allocation failed (lengths)");
  cudaMemcpyAsync(m.lens.p, lens_h.data(), (size_t)B * 4, cudaMemcpyHostToDevice, st);
  const int n_cap = T + 1;
  if (!(m.feats.reserve((size_t)B * T * m.feat_dim * 4) && m.flens.reserve((size_t)B * 4) && m.encb.reserve((size_t)B * T * D * 4) &&
        m.acoustic.reserve((size_t)B * n_cap * D * 4) && m.tok.reserve((size_t)B * 4) && m.alphas.reserve((size_t)B * n_cap * 4) &&
        m.peaks.reserve((size_t)B * n_cap * 4)))
    return fail("device allocation failed (activations)");
  size_t ws = fa_sanm_encoder_workspace_bytes(B, T, m.mode);
  const size_t ws2 = fa_cif_predictor_workspace_bytes(B, T, m.mode);
  ws = ws2 > ws ? ws2 : ws;
  if (!m.ws.reserve(ws)) return fail("device allocation failed (workspace)");
  int rc = fa_fbank_lfr_cmvn_tables(wav, static_cast<int32_t*>(m.lens.p), B, stride, m.cmvn, m.file.fbank_tables, 7, 6, static_cast<float*>(m.feats.p),
                                    T, static_cast<int32_t*>(m.flens.p), T, st);
  if (rc != FA_OK) return fail(std::string("fa_fbank_lfr_cmvn_tables: ") + fa_status_string(rc));
  rc = fa_sanm_encoder_forward(&m.enc, static_cast<float*>(m.feats.p), static_cast<int32_t*>(m.flens.p), B, T, static_cast<float*>(m.encb.p),
                               m.mode, m.ws.p, m.ws.cap, st);
  if (rc != FA_OK) return fail(std::string("fa_sanm_encoder_forward: ") + fa_status_string(rc));
  rc = fa_cif_predictor_forward(&m.pred, static_cast<float*>(m.encb.p), static_cast<int32_t*>(m.flens.p), B, T, static_cast<float*>(m.acoustic.p),
                                n_cap, static_cast<int32_t*>(m.tok.p), static_cast<float*>(m.alphas.p), static_cast<float*>(m.peaks.p), m.mode,
                                m.ws.p, m.ws.cap, st);
  if (rc != FA_OK) return fail(std::string("fa_cif_predictor_forward: ") + fa_status_string(rc));
  std::unique_ptr<Result> r(new Result());
  r->audio_seconds = (float)seconds;
  r->token_num.resize(B);
  r->ts = m.ts;
  if (m.ts) r->stamps.resize(B);
  cudaMemcpyAsync(r->token_num.data(), m.tok.p, (size_t)B * 4, cudaMemcpyDeviceToHost, st);
  if (!sync_stream(st)) return nullptr;
  int n_max = 0;                                             // the path's one host sync (cif_predictor.py:311)
  for (int i = 0; i < B; ++i) n_max = r->token_num[i] > n_max ? r->token_num[i] : n_max;
  r->ids.resize(B);
  if (n_max < 1) return r;                                   // paraformer/model.py:615-616
  const int nh = m.contextual ? n_hotwords : 0;
  // the timestamp head over the [B, 3T] upsampled frames shares the workspace with the decoder
  const int U = m.head.up_times, TU = T * U;
  const int64_t rows_up = (int64_t)B * TU;
  const int n_sw = m.seaco && hw_embed ? n_hotwords : 0;     // SeACo hotword rows (none: the plain decoder distribution)
  size_t ws_dec = fa_paraformer_decoder_workspace_bytes_hw(B, T, n_max, m.vocab, m.mode, nh);
  if (m.ts) ws_dec = std::max(ws_dec, fa_timestamp_head_workspace_bytes(B, T, D, U, m.mode));
  if (n_sw > 0)
    ws_dec = std::max({ws_dec, fa_sanm_decoder_stack_workspace_bytes(B, n_sw, n_max, m.mode), fa_linear_argmax_workspace_bytes((int64_t)B * n_max, m.vocab, m.mode)});
  if (!(m.ids.reserve((size_t)B * n_max * 4) && m.best.reserve((size_t)B * n_max * 4) && m.fids.reserve((size_t)B * n_max * 4) &&
        m.flens_out.reserve((size_t)B * 4) && m.ws.reserve(ws_dec)))
    return fail("device allocation failed (decoder)");
  if (m.ts && !(m.us_alphas.reserve((size_t)rows_up * 4) && m.us_peaks.reserve((size_t)rows_up * 4)))
    return fail("device allocation failed (timestamp head)");
  if (m.contextual) {                                        // hotword memory [n_hw, 512] (contextual_paraformer/model.py:350-372) + per-utterance counts
    if (!(m.hw.reserve((size_t)nh * D * 4) && m.hw_lens.reserve((size_t)B * 4))) return fail("device allocation failed (hotwords)");
    std::vector<int32_t> hl(B, nh);
    cudaMemcpyAsync(m.hw.p, hw_embed, (size_t)nh * D * 4, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(m.hw_lens.p, hl.data(), (size_t)B * 4, cudaMemcpyHostToDevice, st);
    cudaStreamSynchronize(st);                               // hl is a stack vector
    m.dec.has_bias = 1; m.dec.n_hotwords = nh;
    m.dec.hw_embed = static_cast<const float*>(m.hw.p); m.dec.hw_lens = static_cast<const int32_t*>(m.hw_lens.p);
  }
  const int32_t* final_ids = static_cast<int32_t*>(m.ids.p);
  if (m.seaco) {                                             // return_hidden: the decoder_hidden the SeACo decoder attends from
    if (!m.hidden.reserve((size_t)B * n_max * D * 4)) return fail("device allocation failed (SeACo)");
    rc = fa_paraformer_decoder_forward_hidden(&m.dec, static_cast<float*>(m.encb.p), static_cast<int32_t*>(m.flens.p), B, T,
                                              static_cast<float*>(m.acoustic.p), n_cap, static_cast<int32_t*>(m.tok.p), n_max,
                                              static_cast<int32_t*>(m.ids.p), static_cast<float*>(m.best.p), nullptr, 1,
                                              static_cast<float*>(m.hidden.p), m.mode, m.ws.p, m.ws.cap, st);
    if (rc == FA_OK && n_sw > 0) {
      if (!seaco_bias(m, B, n_max, n_cap, hw_embed, n_sw)) return nullptr;
      final_ids = static_cast<int32_t*>(m.sids.p);
    }
  } else {
    rc = fa_paraformer_decoder_forward(&m.dec, static_cast<float*>(m.encb.p), static_cast<int32_t*>(m.flens.p), B, T, static_cast<float*>(m.acoustic.p),
                                       n_cap, static_cast<int32_t*>(m.tok.p), n_max, static_cast<int32_t*>(m.ids.p), static_cast<float*>(m.best.p),
                                       nullptr, 1, m.mode, m.ws.p, m.ws.cap, st);
  }
  if (rc == FA_OK)
    rc = fa_greedy_filter(final_ids, static_cast<int32_t*>(m.tok.p), B, n_max, 1, 2, 0, static_cast<int32_t*>(m.fids.p),
                          static_cast<int32_t*>(m.flens_out.p), st);
  if (rc != FA_OK) return fail(std::string("decoder: ") + fa_status_string(rc));
  if (m.ts) {                   // CifPredictorV3.get_upsample_timestamp (bicif_paraformer/cif_predictor.py:300-352), engine.upsample_timestamp
    rc = fa_timestamp_head_forward(&m.head, static_cast<float*>(m.encb.p), static_cast<int32_t*>(m.flens.p), static_cast<int32_t*>(m.tok.p), B, T,
                                   static_cast<float*>(m.us_alphas.p), static_cast<float*>(m.us_peaks.p), m.mode, m.ws.p, m.ws.cap, st);
    if (rc != FA_OK) return fail(std::string("timestamp head: ") + fa_status_string(rc));
  }
  std::vector<int32_t> fids((size_t)B * n_max), fl(B), enc_lens(m.ts ? B : 0);
  std::vector<float> us_alphas(m.ts ? rows_up : 0), us_peaks(m.ts ? rows_up : 0);
  cudaMemcpyAsync(fids.data(), m.fids.p, fids.size() * 4, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(fl.data(), m.flens_out.p, (size_t)B * 4, cudaMemcpyDeviceToHost, st);
  if (m.ts) {                                                // on the same synchronisation as the ids
    cudaMemcpyAsync(enc_lens.data(), m.flens.p, (size_t)B * 4, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(us_alphas.data(), m.us_alphas.p, (size_t)rows_up * 4, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(us_peaks.data(), m.us_peaks.p, (size_t)rows_up * 4, cudaMemcpyDeviceToHost, st);
  }
  if (!sync_stream(st)) return nullptr;
  for (int i = 0; i < B; ++i) r->ids[i].assign(fids.begin() + (size_t)i * n_max, fids.begin() + (size_t)i * n_max + fl[i]);
  if (m.ts) {                                                // bicif_paraformer/model.py:402-407: each utterance's first 3 * enc_len frames
    for (int i = 0; i < B; ++i) {
      const int64_t n = (int64_t)U * enc_lens[i];
      std::vector<int32_t>& sp = r->stamps[i];
      sp.resize((size_t)(2 * (n > 0 ? n : 1)));              // at most n - 1 spans
      const int64_t k = fa_ts_stamps_host(us_alphas.data() + (size_t)i * TU, us_peaks.data() + (size_t)i * TU, n, (int64_t)r->ids[i].size(), U, 0.0,
                                          sp.data(), n);
      sp.resize(k > 0 ? (size_t)(2 * k) : 0);
    }
  }
  return r;
}

// ------------------------------------------------------------------------------------------------ SenseVoiceSmall
// __sv_config__ of funasr_b200/pack.py:write_sensevoice_model_file
enum { kSvEnc = 0, kSvTp, kSvDModel, kSvHeads, kSvKernel, kSvVocab, kSvFeat, kSvEps, kSvBlank, kSvCfgLen };
const int32_t kSvAuto = 0, kSvWoItn = 15;             // SenseVoiceSmall.inference's defaults: language "auto", text norm "woitn"

// SenseVoiceEngine of engine.py: the same weights, the same planes per gemm_mode
bool build_sv(Model& m, Builder& b) {
  m.mode = b.mode;
  b.what = "SenseVoice model: ";
  if (b.opt("__config__")) return b.refuse("the file carries both __config__ (Paraformer) and __sv_config__");
  const Tensor* cfg = b.get("__sv_config__");
  if (!cfg) return false;
  if (cfg->host.size() != kSvCfgLen) return b.refuse("bad __sv_config__");
  const float* c = cfg->host.data();
  m.enc_layers = (int)c[kSvEnc]; m.tp_layers = (int)c[kSvTp]; m.d_model = (int)c[kSvDModel]; m.heads = (int)c[kSvHeads];
  m.kernel = (int)c[kSvKernel]; m.vocab = (int)c[kSvVocab]; m.feat_dim = (int)c[kSvFeat]; m.ln_eps = c[kSvEps]; m.blank = (int)c[kSvBlank];
  if (m.enc_layers < 1 || m.tp_layers < 0) return b.refuse("no encoder layer");
  if (m.d_model != 512 || m.heads != 4)
    return b.refuse("d_model " + std::to_string(m.d_model) + " with " + std::to_string(m.heads) +
                    " heads (the tensor-core attention runs d_model 512 as 4 heads of 128)");
  if (m.vocab < 1 || m.vocab > 61440)
    return b.refuse("vocabulary of " + std::to_string(m.vocab) + " tokens (the CTC arg-max takes at most 61440)");
  if (m.feat_dim != 560) return b.refuse("feat_dim " + std::to_string(m.feat_dim) + " (the frontend is 80 mel x LFR 7 = 560)");
  if (m.blank < 0 || m.blank >= m.vocab) return b.refuse("blank_id outside the vocabulary");
  b.ln_eps = m.ln_eps;
  b.fbank_tables();
  const Tensor* cmvn = b.opt("frontend.cmvn");
  if (cmvn && cmvn->numel() != 2 * m.feat_dim) return b.refuse("frontend.cmvn must be [2, 560]");
  m.cmvn = cmvn ? cmvn->dev : nullptr;
  bind_stack(b, false, m.enc_layers, m.feat_dim, m.d_model, m.heads, m.enc_l, m.enc);
  bind_stack(b, true, m.tp_layers, m.d_model, m.d_model, m.heads, m.tp_l, m.tp);
  const Tensor* ctc = b.get("ctc.ctc_lo.weight");
  if (ctc && ctc->shape != std::vector<int64_t>{m.vocab, m.d_model}) return b.refuse("bad shape of ctc.ctc_lo.weight (want [vocab, 512])");
  m.ctc = b.lin("ctc.ctc_lo");
  const Tensor* emb = b.get("embed.weight");
  if (!emb) return false;
  if (emb->shape.size() != 2 || emb->shape[0] < 3 || emb->shape[1] != m.feat_dim) return b.refuse("bad shape of embed.weight (want [>= 3, 560])");
  m.embed = emb->dev;
  m.n_embed = (int)emb->shape[0];
  m.sv = true;
  return b.ok;
}

// every query id inside the embedding table; `what` names the unit ("utterance", "recording")
bool check_queries(const Model& m, const int32_t* lang, const int32_t* tn, int n, const char* what) {
  for (int i = 0; i < n; ++i) {
    const int32_t l = lang ? lang[i] : kSvAuto, t = tn ? tn[i] : kSvWoItn;
    if (l < 0 || l >= m.n_embed || t < 0 || t >= m.n_embed) {
      set_err(std::string(what) + " " + std::to_string(i) + ": " + (l < 0 || l >= m.n_embed ? "language id " + std::to_string(l) : "textnorm id " + std::to_string(t)) +
              " outside the embedding table [0, " + std::to_string(m.n_embed) + ")");
      return false;
    }
  }
  return true;
}

// SenseVoiceEngine.forward_wav over a padded batch already on the device (wav [B, stride], lens_h >= 400 samples each), utterance i
// queried with (lang[i], tn[i]) (NULL: the defaults; validated by check_queries).  The CTC head materialises the logits [B, T, vocab].
std::unique_ptr<Result> decode_sv(Model& m, const float* wav, int64_t stride, const std::vector<int32_t>& lens_h, const int32_t* lang,
                                  const int32_t* tn) {
  const int B = (int)lens_h.size(), D = m.d_model, F = m.feat_dim;
  cudaStream_t st = m.file.st;
  int t_feat = 0;
  double seconds = 0.0;
  // one host-to-device copy: sample counts [B], encoder lengths [B] (frames + the 4 query rows), query ids [B][2]
  std::vector<int32_t> io((size_t)4 * B);
  for (int i = 0; i < B; ++i) {
    const int t = num_lfr_frames(lens_h[i]);
    t_feat = t > t_feat ? t : t_feat;
    seconds += (double)lens_h[i] / 16000.0;
    io[i] = lens_h[i];
    io[B + i] = t + 4;
    io[2 * B + 2 * i] = lang ? lang[i] : kSvAuto;
    io[2 * B + 2 * i + 1] = tn ? tn[i] : kSvWoItn;
  }
  const int T = t_feat + 4;
  const size_t rows = (size_t)B * T;
  const size_t ws = std::max(fa_sanm_encoder_workspace_bytes(B, T, m.mode), fa_ctc_greedy_workspace_bytes(B, T, m.vocab, m.mode));
  if (!(m.lens.reserve(io.size() * 4) && m.feats.reserve(rows * F * 4) && m.flens.reserve((size_t)B * 4) && m.encb.reserve(rows * D * 4) &&
        m.enc2.reserve(rows * D * 4) && m.am.reserve(rows * 4) && m.ids.reserve(rows * 4) && m.flens_out.reserve((size_t)B * 4) && m.ws.reserve(ws)))
    return fail("device allocation failed (SenseVoice)");
  int32_t* io_d = static_cast<int32_t*>(m.lens.p);
  float* x = static_cast<float*>(m.feats.p);
  float* enc = static_cast<float*>(m.encb.p);
  cudaMemcpyAsync(io_d, io.data(), io.size() * 4, cudaMemcpyHostToDevice, st);
  int rc = fa_fbank_lfr_cmvn_tables(wav, io_d, B, stride, m.cmvn, m.file.fbank_tables, 7, 6, x + 4 * F, T, static_cast<int32_t*>(m.flens.p), t_feat, st);
  if (rc == FA_OK) rc = fa_sv_query_rows(m.embed, m.n_embed, F, io_d + 2 * B, B, x, T, st);
  if (rc == FA_OK) rc = fa_sanm_encoder_forward(&m.enc, x, io_d + B, B, T, enc, m.mode, m.ws.p, m.ws.cap, st);
  if (rc == FA_OK && m.tp_layers > 0) {
    rc = fa_sanm_encoder_forward(&m.tp, enc, io_d + B, B, T, static_cast<float*>(m.enc2.p), m.mode, m.ws.p, m.ws.cap, st);
    enc = static_cast<float*>(m.enc2.p);
  }
  if (rc == FA_OK)
    rc = fa_ctc_greedy_forward(&m.ctc, enc, io_d + B, B, T, m.blank, static_cast<int32_t*>(m.am.p), static_cast<int32_t*>(m.ids.p),
                               static_cast<int32_t*>(m.flens_out.p), nullptr, m.mode, m.ws.p, m.ws.cap, st);
  if (rc != FA_OK) return fail(std::string("SenseVoice: ") + fa_status_string(rc));
  std::unique_ptr<Result> r(new Result());
  r->audio_seconds = (float)seconds;
  r->token_num.resize(B);
  r->ids.resize(B);
  std::vector<int32_t> ids(rows);
  cudaMemcpyAsync(ids.data(), m.ids.p, rows * 4, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(r->token_num.data(), m.flens_out.p, (size_t)B * 4, cudaMemcpyDeviceToHost, st);
  if (!sync_stream(st)) return nullptr;
  for (int i = 0; i < B; ++i) r->ids[i].assign(ids.begin() + (size_t)i * T, ids.begin() + (size_t)i * T + r->token_num[i]);
  return r;
}

// one padded batch on the device decoded by the handle's model kind: the hotword memory reaches a contextual Paraformer, the queries
// (per row, NULL = the defaults) a SenseVoice model
std::unique_ptr<Result> decode_pack(Model& m, const float* wav, int64_t stride, const std::vector<int32_t>& lens_h, const float* hw_embed,
                                    int32_t n_hotwords, const int32_t* lang, const int32_t* tn) {
  return m.sv ? decode_sv(m, wav, stride, lens_h, lang, tn) : decode_batch(m, wav, stride, lens_h, hw_embed, n_hotwords);
}

// fa_offline_infer_hw / fa_offline_infer_sv: host buffers -> one padded batch -> decode_pack
void* infer_batch(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format, const float* hw_embed,
                  int32_t n_hotwords, const int32_t* lang, const int32_t* tn) {
  Model* mp = static_cast<Model*>(handle);
  if (!mp || !bufs || !n_samples || batch <= 0 || (pcm_format != 0 && pcm_format != 1)) return fail("bad argument");
  Model& m = *mp;
  if (m.contextual && (!hw_embed || n_hotwords < 1)) return fail("this model has a hotword bias decoder: pass hotword embeddings (at least the <s> entry)");
  if (m.seaco && (n_hotwords < 0 || (n_hotwords > 0 && !hw_embed))) return fail("bad hotword rows: hw_embed must hold n_hotwords rows of 512");
  if (m.sv && !check_queries(m, lang, tn, batch, "utterance")) return nullptr;
  cudaSetDevice(m.file.device);
  int64_t nmax = 0;
  std::vector<int32_t> lens_h(batch);
  for (int i = 0; i < batch; ++i) {
    if (!bufs[i] || n_samples[i] < 400 || n_samples[i] > 0x7fffffffLL) return fail("every buffer needs >= 400 samples (25 ms)");
    lens_h[i] = (int32_t)n_samples[i];
    nmax = n_samples[i] > nmax ? n_samples[i] : nmax;
  }
  const int64_t stride = (nmax + 3) / 4 * 4;
  if (!upload(bufs, n_samples, batch, stride, pcm_format, m.wav, m.pcm16, m.file.st)) return nullptr;
  return decode_pack(m, static_cast<const float*>(m.wav.p), stride, lens_h, hw_embed, n_hotwords, lang, tn).release();
}

// the model kind is the file's: SenseVoiceSmall by __sv_config__, Paraformer otherwise
bool build_offline(Model& m, Builder& b) { return b.opt("__sv_config__") ? build_sv(m, b) : build_paraformer(m, b); }

}  // namespace

extern "C" const char* fa_offline_last_error(void) { return g_err.c_str(); }
extern "C" void* fa_offline_infer_hw(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                                     const float* hw_embed, int32_t n_hotwords);

extern "C" void* fa_offline_init(const char* model_file, int32_t device, int32_t gemm_mode) {
  g_err.clear();
  if (!model_file) return fail("model_file is NULL");
  if (gemm_mode != FA_GEMM_F32_SIMT && gemm_mode != FA_GEMM_F16X1 && gemm_mode != FA_GEMM_F16X3 && gemm_mode != FA_GEMM_F16X6) return fail("bad gemm_mode");
  return open_handle(model_file, device, gemm_mode, build_offline);
}

extern "C" int32_t fa_offline_is_sensevoice(const void* handle) { return handle && static_cast<const Model*>(handle)->sv ? 1 : 0; }

extern "C" void* fa_offline_infer_sv(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                                     const int32_t* language_ids, const int32_t* textnorm_ids) {
  g_err.clear();
  if (handle && !static_cast<Model*>(handle)->sv) return fail("fa_offline_infer_sv: not a SenseVoice model file");
  return infer_batch(handle, bufs, n_samples, batch, pcm_format, nullptr, 0, language_ids, textnorm_ids);
}

extern "C" void fa_offline_uninit(void* handle) { delete static_cast<Model*>(handle); }

extern "C" int32_t fa_offline_is_contextual(const void* handle) { return handle && static_cast<const Model*>(handle)->contextual ? 1 : 0; }

extern "C" int32_t fa_offline_has_timestamps(const void* handle) { return handle && static_cast<const Model*>(handle)->ts ? 1 : 0; }

extern "C" int32_t fa_offline_is_seaco(const void* handle) { return handle && static_cast<const Model*>(handle)->seaco ? 1 : 0; }

extern "C" int fa_offline_hotword_embed(void* handle, const int32_t* ids, const int32_t* lens, int32_t n, float* rows_host) {
  g_err.clear();
  Model* m = static_cast<Model*>(handle);
  if (!m || !ids || !lens || n < 1 || !rows_host) { set_err("fa_offline_hotword_embed: bad argument"); return FA_ERR_ARG; }
  if (!m->seaco) { set_err("fa_offline_hotword_embed: not a SeACo model file (ContextualParaformer rows come from its own encoder)"); return FA_ERR_ARG; }
  int64_t n_tok = 0;
  for (int32_t i = 0; i < n; ++i) {                 // every id named before any launch
    if (lens[i] < 1) { set_err("hotword " + std::to_string(i) + " has no token"); return FA_ERR_ARG; }
    for (int32_t k = 0; k < lens[i]; ++k)
      if (ids[n_tok + k] < 0 || ids[n_tok + k] >= m->vocab) {
        set_err("hotword " + std::to_string(i) + ": token id " + std::to_string(ids[n_tok + k]) + " outside the vocabulary [0, " +
                std::to_string(m->vocab) + ")");
        return FA_ERR_ARG;
      }
    n_tok += lens[i];
  }
  cudaSetDevice(m->file.device);
  cudaStream_t st = m->file.st;
  const size_t ws = fa_hotword_encoder_workspace_bytes(n, n_tok, m->mode);
  if (ws == 0 || !m->ws.reserve(ws) || !m->hw_rows.reserve((size_t)n * m->d_model * 4)) {
    set_err("device allocation failed (hotword encoder)");
    return FA_ERR_CUDA;
  }
  const int rc = fa_hotword_encoder_forward(&m->hw_enc, ids, lens, n, static_cast<float*>(m->hw_rows.p), m->mode, m->ws.p, m->ws.cap, st);
  if (rc != FA_OK) { set_err(std::string("fa_hotword_encoder_forward: ") + fa_status_string(rc)); return rc; }
  cudaMemcpyAsync(rows_host, m->hw_rows.p, (size_t)n * m->d_model * 4, cudaMemcpyDeviceToHost, st);
  return sync_stream(st) ? FA_OK : FA_ERR_CUDA;
}

extern "C" const float* fa_offline_host_tensor(void* handle, const char* name, int64_t* numel) {
  Model* m = static_cast<Model*>(handle);
  if (numel) *numel = 0;
  if (!m || !name) return nullptr;
  auto it = m->file.t.find(name);
  if (it == m->file.t.end()) return nullptr;
  const Tensor& t = it->second;
  if (!t.dev) {                                 // a "__" configuration tensor: its payload is on the host already
    if (numel) *numel = (int64_t)t.host.size();
    return t.host.data();
  }
  auto& hc = m->host_cache[name];
  if (hc.empty() && t.numel() > 0) {
    hc.resize((size_t)t.numel());
    cudaSetDevice(m->file.device);
    if (cudaMemcpy(hc.data(), t.dev, hc.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess) { hc.clear(); return nullptr; }
  }
  if (numel) *numel = (int64_t)hc.size();
  return hc.data();
}

extern "C" void* fa_offline_infer(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format) {
  return fa_offline_infer_hw(handle, bufs, n_samples, batch, pcm_format, nullptr, 0);
}

extern "C" void* fa_offline_infer_hw(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                                     const float* hw_embed, int32_t n_hotwords) {
  g_err.clear();
  return infer_batch(handle, bufs, n_samples, batch, pcm_format, hw_embed, n_hotwords, nullptr, nullptr);
}

extern "C" int32_t fa_offline_result_count(const void* result) { return result ? (int32_t)static_cast<const Result*>(result)->ids.size() : 0; }

extern "C" const int32_t* fa_offline_result_ids(const void* result, int32_t index, int32_t* n_ids) {
  const Result* r = static_cast<const Result*>(result);
  if (!r || index < 0 || index >= (int32_t)r->ids.size()) { if (n_ids) *n_ids = 0; return nullptr; }
  if (n_ids) *n_ids = (int32_t)r->ids[index].size();
  return r->ids[index].data();
}

extern "C" float fa_offline_result_audio_seconds(const void* result) { return result ? static_cast<const Result*>(result)->audio_seconds : 0.f; }

extern "C" const int32_t* fa_offline_result_stamps(const void* result, int32_t index, int32_t* n_stamps) {
  const Result* r = static_cast<const Result*>(result);
  if (!r || !r->ts || index < 0 || index >= (int32_t)r->stamps.size() || r->stamps[index].empty()) { if (n_stamps) *n_stamps = 0; return nullptr; }
  if (n_stamps) *n_stamps = (int32_t)(r->stamps[index].size() / 2);
  return r->stamps[index].data();
}

extern "C" void fa_offline_free_result(void* result) { delete static_cast<Result*>(result); }

// ------------------------------------------------------------------------------------------------ FSMN-VAD handle + long audio
namespace {

// __vad_config__ of funasr_b200/pack.py:write_vad_model_file: float64 values stored as the bytes of an fp32 tensor (the detector
// compares in double precision: 0.6 and 1e-4 must arrive unrounded)
enum { kVadCfgInts = 14, kVadCfgDoubles = 5, kVadCfgLorder = 19, kVadCfgNSil = 20, kVadCfgSil = 21, kVadCfgLen = 25 };

struct Vad {
  Loaded file;
  std::vector<FaVadLayer> layers;
  FaVadEncoder enc{};
  FaVadOptions opts{};
  const float* cmvn = nullptr;
  DevBuf wav, pcm16, lens, feats, flens, frames, ws;
};

struct VadResult {
  std::vector<int32_t> seg;                          // {start_ms, end_ms} pairs
  std::vector<float> frames;                         // [2][frames]: silence posterior, frame energy
  float audio_seconds = 0.f;
};

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
    void* wp = nullptr;
    if (cudaMalloc(&wp, (size_t)out_f * kp * 4) != cudaSuccess) { b.refuse("cudaMalloc weights"); return L; }
    b.f->owned.push_back(wp);
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

// VAD of one device-resident recording wav [n] fp32 on stream st (the VAD's own, or the recogniser's in fa_offline_infer_vad)
bool vad_run(Vad& v, const float* wav, int64_t n, cudaStream_t st, const FaVadRunOptions& ro, VadResult& out) {
  out.audio_seconds = (float)((double)n / 16000.0);
  const int64_t T = n >= 400 ? (n - 400) / 160 + 1 : 0;
  out.seg.clear();
  out.frames.assign((size_t)(2 * T), 0.f);
  if (T == 0) return true;                                   // shorter than one frame: nothing to score
  const int32_t n32 = (int32_t)n;
  const size_t ws = fa_fsmn_vad_workspace_bytes(&v.enc, (int32_t)T);
  if (!(v.lens.reserve(4) && v.feats.reserve((size_t)T * 400 * 4) && v.flens.reserve(4) && v.frames.reserve((size_t)T * 8) && v.ws.reserve(ws))) {
    set_err("device allocation failed (VAD)"); return false;
  }
  float* frames = static_cast<float*>(v.frames.p);
  cudaMemcpyAsync(v.lens.p, &n32, 4, cudaMemcpyHostToDevice, st);
  int rc = fa_fbank_lfr_cmvn_tables(wav, static_cast<int32_t*>(v.lens.p), 1, n, v.cmvn, v.file.fbank_tables, 5, 1, static_cast<float*>(v.feats.p), T,
                                    static_cast<int32_t*>(v.flens.p), (int32_t)T, st);
  if (rc == FA_OK) rc = fa_fsmn_vad_forward(&v.enc, static_cast<float*>(v.feats.p), 400, (int32_t)T, frames, nullptr, v.ws.p, v.ws.cap, st);
  if (rc == FA_OK) rc = fa_frame_decibels(wav, n, (int32_t)T, frames + T, st);
  if (rc != FA_OK) { set_err(std::string("VAD: ") + fa_status_string(rc)); return false; }
  cudaMemcpyAsync(out.frames.data(), frames, (size_t)T * 8, cudaMemcpyDeviceToHost, st);     // the one copy back: two floats per frame
  if (!sync_stream(st)) return false;
  std::vector<double> sil(out.frames.begin(), out.frames.begin() + T), db(out.frames.begin() + T, out.frames.end());
  FaVadOptions o = v.opts;
  if (!ro.dynamic_silence && ro.max_end_silence_time > 0) o.max_end_silence_time = ro.max_end_silence_time;
  std::vector<int32_t> seg(128);
  for (;;) {
    const int64_t cap = (int64_t)seg.size() / 2;
    const int64_t k = fa_vad_detect_segments(sil.data(), db.data(), T, n, &o, 60000, ro.dynamic_silence ? 1 : 0, kSilenceSchedule,
                                             (int32_t)(sizeof(kSilenceSchedule) / sizeof(double) / 2), ro.speech_noise_thres, seg.data(), cap);
    if (k < 0) { set_err("fa_vad_detect_segments failed: posteriors must lie inside (0, 1)"); return false; }
    if (k <= cap) { seg.resize((size_t)(2 * k)); break; }
    seg.resize((size_t)(2 * k));
  }
  out.seg.swap(seg);
  return true;
}

FaVadRunOptions default_vad_run() {
  FaVadRunOptions r;
  r.dynamic_silence = 1; r.max_end_silence_time = 0; r.speech_noise_thres = NAN;
  return r;
}

// one recording (host) -> fp32 on the device in `dst`, its row rounded up to 4 samples
bool upload_one(const void* buf, int64_t n, int32_t pcm_format, DevBuf& dst, DevBuf& pcm16, cudaStream_t st) {
  return upload(&buf, &n, 1, (n + 3) / 4 * 4, pcm_format, dst, pcm16, st);
}

// four consecutive output columns per thread: scalar reads (a segment starts anywhere), one 16-byte store
__global__ void __launch_bounds__(256)
gather_segments_kernel(const float* __restrict__ rec, int64_t n_rec, const int64_t* __restrict__ starts, const int32_t* __restrict__ lens,
                       int64_t stride, float* __restrict__ out) {
  const int r = blockIdx.y;
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (c >= stride) return;
  const int64_t s = starts[r];
  const int32_t len = lens[r];
  float v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int64_t j = c + k, src = s + j;
    v[k] = (j < len && src >= 0 && src < n_rec) ? rec[src] : 0.f;
  }
  *reinterpret_cast<float4*>(out + (int64_t)r * stride + c) = make_float4(v[0], v[1], v[2], v[3]);
}

}  // namespace

extern "C" int fa_gather_segments(const float* rec, int64_t n_rec, const int64_t* starts, const int32_t* lens, int32_t rows, int64_t stride,
                                  float* out, fa_stream_t stream) {
  if (rows < 0 || rows > 65535 || n_rec < 0 || (rows > 0 && (!rec || !starts || !lens || !out || stride <= 0))) return FA_ERR_ARG;
  if (rows == 0) return FA_OK;
  if (stride % 4 || reinterpret_cast<uintptr_t>(out) % 16) return FA_ERR_UNSUPPORTED;
  const int64_t blocks = (stride / 4 + 255) / 256;
  if (blocks > 0x7fffffffLL) return FA_ERR_ARG;
  gather_segments_kernel<<<dim3((unsigned)blocks, (unsigned)rows), 256, 0, (cudaStream_t)stream>>>(rec, n_rec, starts, lens, stride, out);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" void* fa_vad_init(const char* model_file, int32_t device) {
  g_err.clear();
  return open_handle(model_file, device, FA_GEMM_F32_SIMT, build_vad);
}

extern "C" void fa_vad_uninit(void* vad) { delete static_cast<Vad*>(vad); }

extern "C" void* fa_vad_infer(void* vad, const void* buf, int64_t n_samples, int32_t pcm_format, const FaVadRunOptions* opts) {
  g_err.clear();
  Vad* v = static_cast<Vad*>(vad);
  if (!v || (!buf && n_samples > 0) || n_samples < 0 || n_samples > 0x7fffffffLL || (pcm_format != 0 && pcm_format != 1)) return fail("bad argument");
  cudaSetDevice(v->file.device);
  std::unique_ptr<VadResult> r(new VadResult());
  if (!no_throw("fa_vad_infer: ", [&] {
        return upload_one(buf, n_samples, pcm_format, v->wav, v->pcm16, v->file.st) &&
               vad_run(*v, static_cast<const float*>(v->wav.p), n_samples, v->file.st, opts ? *opts : default_vad_run(), *r);
      }))
    return nullptr;
  return r.release();
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

// ------------------------------------------------------------------------------------------------ CAM++ speaker handle + diarization
namespace {

// __spk_config__ of funasr_b200/pack.py:write_campplus_model_file: CAMPPlusB200's one supported shape
enum { kSpkFeat = 0, kSpkEmb, kSpkGrowth, kSpkBnSize, kSpkInit, kSpkCfgLen };
const float kSpkConfig[kSpkCfgLen] = {80, 192, 32, 4, 128};
const int kCamLayers[3] = {12, 24, 16}, kCamDilation[3] = {1, 2, 2};
const char* const kFcmConvs[12] = {"conv1", "layer1.0.conv1", "layer1.0.conv2", "layer1.0.shortcut.0", "layer1.1.conv1", "layer1.1.conv2",
                                   "layer2.0.conv1", "layer2.0.conv2", "layer2.0.shortcut.0", "layer2.1.conv1", "layer2.1.conv2", "conv2"};
const char* const kFcmBns[12] = {"bn1", "layer1.0.bn1", "layer1.0.bn2", "layer1.0.shortcut.1", "layer1.1.bn1", "layer1.1.bn2",
                                 "layer2.0.bn1", "layer2.0.bn2", "layer2.0.shortcut.1", "layer2.1.bn1", "layer2.1.bn2", "bn2"};
const int kFcmStride[12] = {1, 2, 1, 2, 1, 1, 2, 1, 2, 1, 1, 2};
const int kSpkEmbDim = 192, kSpkMaxFrames = 18800, kChunkLen = 24000, kChunkShift = 12000;
const size_t kSpkWorkspaceCap = (size_t)1 << 30;    // CampplusEngine.WORKSPACE_CAP: larger batches run in slices
const int kSpectralMaxChunks = 2048, kMaxSpks = 15;
const double kSpkPval = 0.022, kMergeThr = 0.78;

// every tensor of the reference CAMPPlus state_dict but num_batches_tracked (campplus.py:campplus_specs), in its order
template <typename F>
void campplus_spec(F f) {
  auto bn = [&](const std::string& p, int64_t n, bool affine) {
    if (affine) { f(p + ".weight", std::vector<int64_t>{n}); f(p + ".bias", std::vector<int64_t>{n}); }
    f(p + ".running_mean", std::vector<int64_t>{n}); f(p + ".running_var", std::vector<int64_t>{n});
  };
  for (int i = 0; i < 12; ++i) {
    const std::string conv = kFcmConvs[i];
    const int64_t cin = i == 0 ? 1 : 32, k = conv.size() > 10 && conv.compare(conv.size() - 10, 10, "shortcut.0") == 0 ? 1 : 3;
    f("head." + conv + ".weight", std::vector<int64_t>{32, cin, k, k});
    bn("head." + std::string(kFcmBns[i]), 32, true);
  }
  f("xvector.tdnn.linear.weight", std::vector<int64_t>{128, 320, 5});
  bn("xvector.tdnn.nonlinear.batchnorm", 128, true);
  int64_t c = 128;
  for (int i = 0; i < 3; ++i) {
    for (int l = 0; l < kCamLayers[i]; ++l) {
      const std::string p = "xvector.block" + std::to_string(i + 1) + ".tdnnd" + std::to_string(l + 1) + ".";
      bn(p + "nonlinear1.batchnorm", c + l * 32, true);
      f(p + "linear1.weight", std::vector<int64_t>{128, c + l * 32, 1});
      bn(p + "nonlinear2.batchnorm", 128, true);
      f(p + "cam_layer.linear_local.weight", std::vector<int64_t>{32, 128, 3});
      f(p + "cam_layer.linear1.weight", std::vector<int64_t>{64, 128, 1}); f(p + "cam_layer.linear1.bias", std::vector<int64_t>{64});
      f(p + "cam_layer.linear2.weight", std::vector<int64_t>{32, 64, 1}); f(p + "cam_layer.linear2.bias", std::vector<int64_t>{32});
    }
    c += kCamLayers[i] * 32;
    bn("xvector.transit" + std::to_string(i + 1) + ".nonlinear.batchnorm", c, true);
    f("xvector.transit" + std::to_string(i + 1) + ".linear.weight", std::vector<int64_t>{c / 2, c, 1});
    c /= 2;
  }
  bn("xvector.out_nonlinear.batchnorm", c, true);
  f("xvector.dense.linear.weight", std::vector<int64_t>{192, 2 * c, 1});
  bn("xvector.dense.nonlinear.batchnorm", 192, false);
}

struct Spk {
  Loaded file;
  int mode = FA_GEMM_F32_SIMT;
  FaCampplus model{};
  std::vector<FaCamLayer> layers;
  DevBuf wav, pcm16, lens, feats, flens, emb, ws, gmeta, lap, tri, tws, z;
};

// The BatchNorm folding of CampplusEngine (campplus.py: _bn, _folded, conv2d) on the host in float64 — the same IEEE multiplies,
// divisions and square roots, then one rounding to fp32 — so the folded weights are bit-identical to the Python engine's.
struct CamFolder {
  Builder& b;
  Loaded& f;
  int mode;
  std::vector<float> host(const std::string& k) {
    const Tensor* t = b.get(k);
    std::vector<float> h(t ? (size_t)t->numel() : 0);
    if (t && !h.empty() && cudaMemcpy(h.data(), t->dev, h.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess) b.refuse("copy of " + k + " failed");
    return h;
  }
  const float* up(const std::vector<double>& v) {
    std::vector<float> h(v.begin(), v.end());
    void* p = nullptr;
    if (cudaMalloc(&p, (h.size() ? h.size() : 1) * 4) != cudaSuccess) { b.refuse("cudaMalloc failed"); return nullptr; }
    f.owned.push_back(p);
    if (cudaMemcpy(p, h.data(), h.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) b.refuse("weight upload failed");
    return static_cast<const float*>(p);
  }
  // eval BatchNorm as y = x s + t
  void bn(const std::string& p, bool affine, std::vector<double>& s, std::vector<double>& t) {
    const std::vector<float> var = host(p + ".running_var"), mean = host(p + ".running_mean");
    const std::vector<float> g = affine ? host(p + ".weight") : std::vector<float>(), beta = affine ? host(p + ".bias") : std::vector<float>();
    s.resize(var.size()); t.resize(var.size());
    for (size_t i = 0; i < var.size(); ++i) {
      s[i] = 1.0 / std::sqrt((double)var[i] + 1e-5);
      if (affine) {
        s[i] = s[i] * (double)g[i];
        t[i] = (double)beta[i] - (double)mean[i] * s[i];
      } else {
        t[i] = -(double)mean[i] * s[i];
      }
    }
  }
  // weights [out, in] (float64) -> FaLinear with the tensor-core planes of the handle's mode
  FaLinear lin(const std::vector<double>& w, int out_f, int in_f, const std::vector<double>* bias) {
    FaLinear L{};
    L.w = up(w); L.b = bias ? up(*bias) : nullptr;
    L.out_f = out_f; L.in_f = in_f; L.in_pad = (in_f + 63) / 64 * 64;
    if (mode != FA_GEMM_F32_SIMT && b.ok) {
      void* planes = nullptr;
      if (cudaMalloc(&planes, (size_t)3 * out_f * L.in_pad * 2) != cudaSuccess) { b.refuse("cudaMalloc planes"); return L; }
      f.owned.push_back(planes);
      if (fa_split_planes(L.w, in_f, out_f, in_f, L.in_pad, planes, f.st) != FA_OK) b.refuse("fa_split_planes failed");
      L.w_planes = planes;
    }
    return L;
  }
  // conv (as [out, in]) followed by BN -> one Linear with bias
  FaLinear folded(const std::vector<float>& w, int out_f, int in_f, const std::string& bn_p, bool affine) {
    std::vector<double> s, t, wd((size_t)out_f * in_f);
    bn(bn_p, affine, s, t);
    for (int o = 0; o < out_f; ++o)
      for (int i = 0; i < in_f; ++i) wd[(size_t)o * in_f + i] = (double)w[(size_t)o * in_f + i] * s[o];
    return lin(wd, out_f, in_f, &t);
  }
  const float* plain(const std::string& k) {
    const std::vector<float> h = host(k);
    return up(std::vector<double>(h.begin(), h.end()));
  }
};

bool build_spk(Spk& h, Builder& b) {
  b.what = "CAM++ model: ";
  h.mode = b.mode;
  for (const char* other : {"__config__", "__sv_config__", "__seaco_config__", "__punc_config__", "__vad_config__"})
    if (b.opt(other)) return b.refuse(std::string("the file carries ") + other + " beside __spk_config__");
  const Tensor* cfg = b.get("__spk_config__");
  if (!cfg) return false;
  if (cfg->host.size() != kSpkCfgLen || !std::equal(cfg->host.begin(), cfg->host.end(), kSpkConfig))
    return b.refuse("bad __spk_config__ (the kernels are built for feat 80, embedding 192, growth 32, bn_size 4, init 128)");
  b.shaped("frontend.mel_banks", {80, 257});
  b.shaped("frontend.window", {400});
  campplus_spec([&](const std::string& k, const std::vector<int64_t>& dims) {
    const Tensor* x = b.get(k);
    if (x && x->shape != dims) b.refuse("bad shape of " + k);
  });
  if (!b.ok || !b.f) return b.ok;
  b.fbank_tables();
  CamFolder F{b, *b.f, b.mode};
  FaCampplus& m = h.model;
  for (int i = 0; i < 12; ++i) {                     // [kf * k + kt][ci][o] = w[o][ci][kf][kt] s[o]
    const std::vector<float> w = F.host("head." + std::string(kFcmConvs[i]) + ".weight");
    std::vector<double> s, t;
    F.bn("head." + std::string(kFcmBns[i]), true, s, t);
    const int cin = i == 0 ? 1 : 32, k = w.size() == (size_t)32 * cin ? 1 : 3;
    std::vector<double> wf((size_t)k * k * cin * 32);
    for (int o = 0; o < 32; ++o)
      for (int ci = 0; ci < cin; ++ci)
        for (int kk = 0; kk < k * k; ++kk) wf[((size_t)kk * cin + ci) * 32 + o] = (double)w[((size_t)o * cin + ci) * k * k + kk] * s[o];
    m.fcm[i] = FaCamConv2d{F.up(wf), F.up(t), cin, 32, k, kFcmStride[i]};
  }
  {                                                  // [o][k * 320 + c] = w[o][c][k]
    const std::vector<float> w = F.host("xvector.tdnn.linear.weight");
    std::vector<float> wp((size_t)128 * 1600);
    for (int o = 0; o < 128; ++o)
      for (int c = 0; c < 320; ++c)
        for (int k = 0; k < 5; ++k) wp[(size_t)o * 1600 + k * 320 + c] = w[((size_t)o * 320 + c) * 5 + k];
    m.tdnn = F.folded(wp, 128, 1600, "xvector.tdnn.nonlinear.batchnorm", true);
  }
  h.layers.assign(kCamLayers[0] + kCamLayers[1] + kCamLayers[2], FaCamLayer{});
  int li = 0, c = 128;
  for (int i = 0; i < 3; ++i) {
    m.n_layers[i] = kCamLayers[i]; m.dilation[i] = kCamDilation[i];
    for (int l = 0; l < kCamLayers[i]; ++l, ++li) {
      const std::string p = "xvector.block" + std::to_string(i + 1) + ".tdnnd" + std::to_string(l + 1) + ".";
      FaCamLayer& L = h.layers[li];
      std::vector<double> s, t;
      F.bn(p + "nonlinear1.batchnorm", true, s, t);
      L.bn1_scale = F.up(s); L.bn1_shift = F.up(t);
      L.linear1 = F.folded(F.host(p + "linear1.weight"), 128, c + l * 32, p + "nonlinear2.batchnorm", true);
      const std::vector<float> lw = F.host(p + "cam_layer.linear_local.weight");     // [k][c][o] = w[o][c][k]
      std::vector<double> lp((size_t)3 * 128 * 32);
      for (int o = 0; o < 32; ++o)
        for (int ci = 0; ci < 128; ++ci)
          for (int k = 0; k < 3; ++k) lp[((size_t)k * 128 + ci) * 32 + o] = lw[((size_t)o * 128 + ci) * 3 + k];
      L.local_w = F.up(lp);
      L.w1 = F.plain(p + "cam_layer.linear1.weight"); L.b1 = F.plain(p + "cam_layer.linear1.bias");
      L.w2 = F.plain(p + "cam_layer.linear2.weight"); L.b2 = F.plain(p + "cam_layer.linear2.bias");
    }
    c += kCamLayers[i] * 32;
    const std::string p = "xvector.transit" + std::to_string(i + 1) + ".";
    std::vector<double> s, t;
    F.bn(p + "nonlinear.batchnorm", true, s, t);
    m.transit[i].scale = F.up(s); m.transit[i].shift = F.up(t);
    const std::vector<float> w = F.host(p + "linear.weight");
    m.transit[i].linear = F.lin(std::vector<double>(w.begin(), w.end()), c / 2, c, nullptr);
    c /= 2;
  }
  m.layers = h.layers.data();
  std::vector<double> s, t;
  F.bn("xvector.out_nonlinear.batchnorm", true, s, t);
  m.out_scale = F.up(s); m.out_shift = F.up(t);
  m.dense = F.folded(F.host("xvector.dense.linear.weight"), kSpkEmbDim, 2 * c, "xvector.dense.nonlinear.batchnorm", false);
  return b.ok;
}

int fbank_frames(int64_t n) { return n >= 400 ? (int)(1 + (n - 400) / 160) : 0; }

// embeddings of a padded batch on the device (wav [B, stride], lens_d [B] on the device) -> emb [B, 192] on the device:
// fa_campplus_features with t_max frames, then fa_campplus_forward in slices of CampplusEngine.embed_feats' workspace cap
bool spk_embed_rows(Spk& s, const float* wav, int64_t stride, const int32_t* lens_d, int B, int t_max, float* emb) {
  cudaStream_t st = s.file.st;
  const size_t per = fa_campplus_workspace_bytes(&s.model, 1, t_max, s.mode);
  if (per == 0) { set_err("CAM++ takes 2 ... 18800 feature frames per input (got " + std::to_string(t_max) + ")"); return false; }
  const int step = (int)std::max<size_t>(1, std::min<size_t>((size_t)B, kSpkWorkspaceCap / per));
  if (!(s.feats.reserve((size_t)B * t_max * 80 * 4) && s.flens.reserve((size_t)B * 4) &&
        s.ws.reserve(fa_campplus_workspace_bytes(&s.model, step, t_max, s.mode)))) {
    set_err("device allocation failed (CAM++)"); return false;
  }
  float* feats = static_cast<float*>(s.feats.p);
  int rc = fa_campplus_features(wav, lens_d, B, stride, s.file.fbank_tables, feats, static_cast<int32_t*>(s.flens.p), t_max, st);
  for (int b0 = 0; b0 < B && rc == FA_OK; b0 += step) {
    const int nb = std::min(step, B - b0);
    rc = fa_campplus_forward(&s.model, feats + (size_t)b0 * t_max * 80, nb, t_max, emb + (size_t)b0 * kSpkEmbDim, s.mode, s.ws.p, s.ws.cap, st);
  }
  if (rc != FA_OK) { set_err(std::string("CAM++: ") + fa_status_string(rc)); return false; }
  return true;
}

// ClusterBackend over n embeddings emb_d [n, 192] on the device (emb_h: the same on the host) -> labels [n] (before correct_labels).
// preset <= 0: no preset count.  Fewer than 20 -> one speaker; fewer than 2048 -> the spectral path (the Laplacian and its
// tridiagonalisation on the device, the 16 smallest eigenvalues on the host, the eigengap count unless preset, k-means on the
// back-transformed vectors); otherwise k-means on the normalised rows with a preset count; merge_by_cos when no count was preset.
bool spk_cluster(Spk& s, int n, int preset, const float* emb_h, std::vector<int32_t>& labels, const std::string& what) {
  labels.assign((size_t)n, 0);
  if (n < 20) return true;
  if (preset > n) { set_err(what + "preset_spk_num " + std::to_string(preset) + " exceeds the " + std::to_string(n) + " speaker chunks"); return false; }
  std::vector<double> x;
  int k = preset, dim = 0;
  if (n < kSpectralMaxChunks) {
    cudaStream_t st = s.file.st;
    const size_t lws = fa_spk_laplacian_workspace_bytes(n, kSpkEmbDim), tws = fa_spk_tridiagonalize_workspace_bytes(n);
    const int m = std::max(std::min(kMaxSpks + 1, n), k);
    if (!(s.lap.reserve((size_t)n * n * 8) && s.tws.reserve(std::max(lws, tws)) && s.tri.reserve((size_t)3 * n * 8) && s.z.reserve((size_t)m * n * 8))) {
      set_err("device allocation failed (speaker clustering)"); return false;
    }
    double* lap = static_cast<double*>(s.lap.p);
    double* d = static_cast<double*>(s.tri.p);
    int rc = fa_spk_laplacian(static_cast<const float*>(s.emb.p), n, kSpkEmbDim, kSpkPval, lap, s.tws.p, s.tws.cap, st);
    if (rc == FA_OK) rc = fa_spk_tridiagonalize(lap, n, d, d + n, d + 2 * n, s.tws.p, s.tws.cap, st);
    if (rc != FA_OK) { set_err(what + "speaker clustering: " + fa_status_string(rc)); return false; }
    std::vector<double> de((size_t)2 * n), w((size_t)m);
    cudaMemcpyAsync(de.data(), d, (size_t)2 * n * 8, cudaMemcpyDeviceToHost, st);
    if (!sync_stream(st)) return false;
    if (k <= 0) {                                    // the largest gap among the 16 smallest eigenvalues (spec_embs)
      fa_sym_tridiag_smallest_host(de.data(), de.data() + n, n, m, 0, w.data(), nullptr);
      const int ne = std::min(kMaxSpks + 1, n);
      double gmax = -INFINITY;
      for (int i = 0; i + 1 < ne; ++i)
        if (w[i + 1] - w[i] > gmax) { gmax = w[i + 1] - w[i]; k = i + 1; }
    }
    std::vector<double> z((size_t)k * n);
    fa_sym_tridiag_smallest_host(de.data(), de.data() + n, n, std::max(m, k), k, w.data(), z.data());
    double* zd = static_cast<double*>(s.z.p);
    cudaMemcpyAsync(zd, z.data(), z.size() * 8, cudaMemcpyHostToDevice, st);
    rc = fa_spk_back_transform(lap, d + 2 * n, n, zd, k, st);
    if (rc != FA_OK) { set_err(what + "speaker clustering: " + fa_status_string(rc)); return false; }
    cudaMemcpyAsync(z.data(), zd, z.size() * 8, cudaMemcpyDeviceToHost, st);
    if (!sync_stream(st)) return false;
    x.resize((size_t)n * k);
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < k; ++j) x[(size_t)i * k + j] = z[(size_t)j * n + i];
    dim = k;
  } else if (preset > 0) {                           // _normalize_rows in fp32
    x.resize((size_t)n * kSpkEmbDim);
    for (int i = 0; i < n; ++i) {
      const float* r = emb_h + (size_t)i * kSpkEmbDim;
      float ss = 0.f;
      for (int c = 0; c < kSpkEmbDim; ++c) ss += r[c] * r[c];
      float nrm = std::sqrt(ss);
      if (nrm == 0.f) nrm = 1.f;
      for (int c = 0; c < kSpkEmbDim; ++c) x[(size_t)i * kSpkEmbDim + c] = (double)(r[c] / nrm);
    }
    dim = kSpkEmbDim;
  } else {
    set_err(what + std::to_string(n) + " speaker chunks without preset_spk_num: the reference clusters 2048 or more chunks with UMAP + "
            "HDBSCAN, which this backend does not provide; pass preset_spk_num or diarize fewer than 2048 chunks");
    return false;
  }
  if (fa_spk_kmeans_host(x.data(), n, dim, k, 0, 10, 300, labels.data()) != FA_OK) { set_err(what + "k-means failed"); return false; }
  if (preset <= 0 && fa_spk_merge_by_cos_host(labels.data(), emb_h, n, kSpkEmbDim, kMergeThr) != FA_OK) {
    set_err(what + "merge_by_cos failed"); return false;
  }
  return true;
}

// LongAudioPipeline.generate's diarization of one device-resident recording rec [n] (vad_segment mode): sv_chunk windows over every VAD
// segment (segs: {start_ms, end_ms, n_tokens} triples), gathered with zero tails and embedded in slices, clustered, post-processed
// and distributed over the segments -> spk [segments].  Runs on the speaker handle's stream; rec must be complete.
bool diarize(Spk& s, const float* rec, int64_t n, const std::vector<int32_t>& segs, int preset, std::vector<int32_t>& spk, const std::string& what) {
  cudaStream_t st = s.file.st;
  const int64_t ns = (int64_t)segs.size() / 3;
  std::vector<int64_t> starts;
  std::vector<double> times;
  for (int64_t g = 0; g < ns; ++g) {                 // long_audio.speaker_chunks / diarization.chunk_bounds
    const int64_t b0 = (int64_t)segs[3 * g] * 16, b1 = std::min<int64_t>((int64_t)segs[3 * g + 1] * 16, n), len = std::max<int64_t>(b1 - b0, 0);
    int64_t last_ed = 0;
    for (int64_t a = 0; a < len; a += kChunkShift) {
      const int64_t ed = std::min<int64_t>(a + kChunkLen, len);
      if (ed <= last_ed) break;
      last_ed = ed;
      const int64_t c0 = std::max<int64_t>(0, ed - kChunkLen);
      starts.push_back(b0 + c0);
      times.push_back((double)c0 / 16000 + (double)segs[3 * g] / 1000.0);
      times.push_back((double)ed / 16000 + (double)segs[3 * g] / 1000.0);
      starts.push_back(ed - c0);                     // interleaved: first sample, sample count
    }
  }
  const int nc = (int)(starts.size() / 2);
  spk.assign((size_t)ns, 0);
  if (nc == 0) return true;
  const int t_max = fbank_frames(kChunkLen);
  const size_t per = fa_campplus_workspace_bytes(&s.model, 1, t_max, s.mode);
  const int step = (int)std::max<size_t>(1, std::min<size_t>({(size_t)nc, kSpkWorkspaceCap / (per ? per : 1), (size_t)65535}));
  if (!(s.emb.reserve((size_t)nc * kSpkEmbDim * 4) && s.wav.reserve((size_t)step * kChunkLen * 4) && s.gmeta.reserve((size_t)step * 16) &&
        s.lens.reserve((size_t)step * 4))) {
    set_err("device allocation failed (speaker chunks)"); return false;
  }
  float* emb = static_cast<float*>(s.emb.p);
  float* wav = static_cast<float*>(s.wav.p);
  int64_t* starts_d = static_cast<int64_t*>(s.gmeta.p);
  int32_t* lens_d = reinterpret_cast<int32_t*>(starts_d + step);
  int32_t* full_d = static_cast<int32_t*>(s.lens.p);
  const std::vector<int32_t> full((size_t)step, kChunkLen);    // every window counts as 1.5 s of samples, its zero tail included
  cudaMemcpyAsync(full_d, full.data(), (size_t)step * 4, cudaMemcpyHostToDevice, st);
  std::vector<int64_t> sb((size_t)step);
  std::vector<int32_t> lb((size_t)step);
  for (int c0 = 0; c0 < nc; c0 += step) {
    const int nb = std::min(step, nc - c0);
    if (!sync_stream(st)) return false;               // sb / lb are reused: the previous slice's copies are done
    for (int r = 0; r < nb; ++r) { sb[r] = starts[2 * (c0 + r)]; lb[r] = (int32_t)starts[2 * (c0 + r) + 1]; }
    cudaMemcpyAsync(starts_d, sb.data(), (size_t)nb * 8, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(lens_d, lb.data(), (size_t)nb * 4, cudaMemcpyHostToDevice, st);
    const int rc = fa_gather_segments(rec, n, starts_d, lens_d, nb, kChunkLen, wav, st);
    if (rc != FA_OK) { set_err(std::string("fa_gather_segments: ") + fa_status_string(rc)); return false; }
    if (!spk_embed_rows(s, wav, kChunkLen, full_d, nb, t_max, emb + (size_t)c0 * kSpkEmbDim)) return false;
  }
  std::vector<float> emb_h((size_t)nc * kSpkEmbDim);
  cudaMemcpyAsync(emb_h.data(), emb, emb_h.size() * 4, cudaMemcpyDeviceToHost, st);
  if (!sync_stream(st)) return false;
  std::vector<int32_t> labels;
  if (!spk_cluster(s, nc, preset, emb_h.data(), labels, what)) return false;
  std::vector<double> turns((size_t)3 * nc);
  const int64_t nt = fa_spk_postprocess_host(times.data(), labels.data(), nc, turns.data());
  std::vector<int32_t> sent((size_t)2 * ns);
  for (int64_t g = 0; g < ns; ++g) { sent[2 * g] = segs[3 * g]; sent[2 * g + 1] = segs[3 * g + 1]; }
  if (nt < 0 || fa_spk_distribute_host(sent.data(), ns, turns.data(), nt, spk.data()) != FA_OK) { set_err(what + "speaker post-processing failed"); return false; }
  return true;
}

}  // namespace

extern "C" void* fa_spk_init(const char* model_file, int32_t device, int32_t gemm_mode) {
  g_err.clear();
  if (gemm_mode != FA_GEMM_F32_SIMT && gemm_mode != FA_GEMM_F16X1 && gemm_mode != FA_GEMM_F16X3 && gemm_mode != FA_GEMM_F16X6) return fail("bad gemm_mode");
  return open_handle(model_file, device, gemm_mode, build_spk);
}

extern "C" void fa_spk_uninit(void* spk) { delete static_cast<Spk*>(spk); }

extern "C" int fa_spk_embed(void* spk, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format, float* emb_host) {
  g_err.clear();
  Spk* s = static_cast<Spk*>(spk);
  if (!s || !bufs || !n_samples || batch <= 0 || (pcm_format != 0 && pcm_format != 1) || !emb_host) { set_err("fa_spk_embed: bad argument"); return FA_ERR_ARG; }
  int64_t nmax = 0;
  int longest = 0;
  for (int32_t i = 0; i < batch; ++i) {              // every input checked before any launch
    if (!bufs[i] || n_samples[i] < 400 || n_samples[i] > 0x7fffffffLL) {
      set_err("input " + std::to_string(i) + " has " + std::to_string(n_samples[i]) + " samples; CAM++ needs at least 400 (one 25 ms frame)");
      return FA_ERR_ARG;
    }
    if (n_samples[i] > nmax) { nmax = n_samples[i]; longest = i; }
  }
  const int t_max = fbank_frames(nmax);
  if (t_max > kSpkMaxFrames) {
    set_err("input " + std::to_string(longest) + " has " + std::to_string(t_max) + " feature frames; CAM++ takes at most " +
            std::to_string(kSpkMaxFrames) + " (MAX_FEAT_FRAMES)");
    return FA_ERR_UNSUPPORTED;
  }
  cudaSetDevice(s->file.device);
  cudaStream_t st = s->file.st;
  const int64_t stride = (nmax + 3) / 4 * 4;
  std::vector<int32_t> lens_h(batch);
  for (int32_t i = 0; i < batch; ++i) lens_h[i] = (int32_t)n_samples[i];
  const bool ok = no_throw("fa_spk_embed: ", [&] {
    if (!(s->lens.reserve((size_t)batch * 4) && s->emb.reserve((size_t)batch * kSpkEmbDim * 4))) { set_err("device allocation failed (CAM++)"); return false; }
    if (!upload(bufs, n_samples, batch, stride, pcm_format, s->wav, s->pcm16, st)) return false;
    cudaMemcpyAsync(s->lens.p, lens_h.data(), (size_t)batch * 4, cudaMemcpyHostToDevice, st);
    if (!spk_embed_rows(*s, static_cast<const float*>(s->wav.p), stride, static_cast<const int32_t*>(s->lens.p), batch, t_max, static_cast<float*>(s->emb.p)))
      return false;
    cudaMemcpyAsync(emb_host, s->emb.p, (size_t)batch * kSpkEmbDim * 4, cudaMemcpyDeviceToHost, st);
    return sync_stream(st);
  });
  return ok ? FA_OK : FA_ERR_CUDA;
}

extern "C" int fa_spk_cluster(void* spk, const float* emb_host, int32_t n, int32_t preset_spk_num, int32_t* labels) {
  g_err.clear();
  Spk* s = static_cast<Spk*>(spk);
  if (!s || !emb_host || n < 1 || !labels) { set_err("fa_spk_cluster: bad argument"); return FA_ERR_ARG; }
  if (n >= kSpectralMaxChunks && preset_spk_num <= 0) {
    set_err(std::to_string(n) + " speaker chunks without preset_spk_num: the reference clusters 2048 or more chunks with UMAP + HDBSCAN, which "
            "this backend does not provide; pass preset_spk_num or diarize fewer than 2048 chunks");
    return FA_ERR_UNSUPPORTED;
  }
  cudaSetDevice(s->file.device);
  std::vector<int32_t> lab;
  const bool ok = no_throw("fa_spk_cluster: ", [&] {
    if (!s->emb.reserve((size_t)n * kSpkEmbDim * 4)) { set_err("device allocation failed (speaker clustering)"); return false; }
    cudaMemcpyAsync(s->emb.p, emb_host, (size_t)n * kSpkEmbDim * 4, cudaMemcpyHostToDevice, s->file.st);
    return spk_cluster(*s, n, preset_spk_num, emb_host, lab, "");
  });
  if (!ok) return FA_ERR_CUDA;
  std::copy(lab.begin(), lab.end(), labels);
  return FA_OK;
}

namespace {

// one recording of fa_offline_infer_vad: inference_with_vad (auto_model.py:852-1035, funasr_b200/long_audio.py:LongAudioPipeline.generate)
// (lang, tn): the recording's SenseVoice query, the same for all its segments
bool long_audio_one(Model& m, Vad& v, int rec_index, const void* buf, int64_t n, int32_t pcm_format, const float* hw_embed, int32_t n_hotwords,
                    int32_t lang, int32_t tn, const FaLongAudioOptions& o, std::vector<int32_t>& ids, std::vector<int32_t>& segs_out,
                    std::vector<int32_t>& stamps) {
  cudaStream_t st = m.file.st;
  if (!upload_one(buf, n, pcm_format, m.rec, m.pcm16, st)) return false;
  const float* rec = static_cast<const float*>(m.rec.p);
  VadResult vr;
  if (!vad_run(v, rec, n, st, o.vad, vr)) return false;
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
    if (!(m.gmeta.reserve((size_t)B * 12) && m.wav.reserve((size_t)B * stride * 4))) { set_err("device allocation failed (segments)"); return false; }
    int64_t* starts_d = static_cast<int64_t*>(m.gmeta.p);
    int32_t* lens_d = reinterpret_cast<int32_t*>(starts_d + B);
    cudaMemcpyAsync(starts_d, starts.data(), (size_t)B * 8, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(lens_d, lens.data(), (size_t)B * 4, cudaMemcpyHostToDevice, st);
    float* wav = static_cast<float*>(m.wav.p);
    const int rc = fa_gather_segments(rec, n, starts_d, lens_d, B, stride, wav, st);
    if (rc != FA_OK) { set_err(std::string("fa_gather_segments: ") + fa_status_string(rc)); return false; }
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

// fa_offline_infer_vad / fa_offline_infer_vad_sv: every recording on its own; lang / tn one query per recording (NULL = the defaults)
// spk: diarize every recording that decoded at least one token (LongAudioPipeline.generate), preset_spk_num <= 0: no preset count
void* infer_vad(void* asr, void* vad, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format, const float* hw_embed,
                int32_t n_hotwords, const int32_t* lang, const int32_t* tn, const FaLongAudioOptions* opts, Spk* spk = nullptr,
                int32_t preset_spk_num = 0) {
  Model* mp = static_cast<Model*>(asr);
  Vad* vp = static_cast<Vad*>(vad);
  if (!mp || !vp || !bufs || !n_samples || batch <= 0 || (pcm_format != 0 && pcm_format != 1)) return fail("bad argument");
  if (mp->file.device != vp->file.device) return fail("the recogniser and the VAD live on different devices");
  if (spk && spk->file.device != mp->file.device) return fail("the recogniser and the speaker model live on different devices");
  if (mp->contextual && (!hw_embed || n_hotwords < 1)) return fail("this model has a hotword bias decoder: pass hotword embeddings (at least the <s> entry)");
  if (mp->seaco && (n_hotwords < 0 || (n_hotwords > 0 && !hw_embed))) return fail("bad hotword rows: hw_embed must hold n_hotwords rows of 512");
  if (mp->sv && !check_queries(*mp, lang, tn, batch, "recording")) return nullptr;
  FaLongAudioOptions o;
  if (opts) o = *opts;
  else { o.batch_size_s = 300; o.batch_size_threshold_s = 60; o.merge_vad = 0; o.merge_length_s = 15; o.vad = default_vad_run(); }
  for (int i = 0; i < batch; ++i)
    if ((!bufs[i] && n_samples[i] > 0) || n_samples[i] < 0 || n_samples[i] > 0x7fffffffLL) return fail("bad recording " + std::to_string(i));
  cudaSetDevice(mp->file.device);
  std::unique_ptr<Result> r(new Result());
  r->ids.resize(batch);
  r->segs.resize(batch);
  r->token_num.assign(batch, 0);
  r->ts = mp->ts;
  r->stamps.resize(batch);
  r->spk.resize(batch);
  double seconds = 0.0;
  if (!no_throw("fa_offline_infer_vad: ", [&] {
        for (int i = 0; i < batch; ++i) {
          seconds += (double)n_samples[i] / 16000.0;
          if (!long_audio_one(*mp, *vp, i, bufs[i], n_samples[i], pcm_format, hw_embed, n_hotwords, lang ? lang[i] : kSvAuto,
                              tn ? tn[i] : kSvWoItn, o, r->ids[i], r->segs[i], r->stamps[i]))
            return false;
          r->token_num[i] = (int32_t)r->ids[i].size();
          // the recogniser's stream is idle here (its results are on the host); the speaker work runs on the speaker handle's stream
          if (spk && !r->ids[i].empty() &&
              !diarize(*spk, static_cast<const float*>(mp->rec.p), n_samples[i], r->segs[i], preset_spk_num, r->spk[i],
                       "recording " + std::to_string(i) + ": "))
            return false;
        }
        return true;
      }))
    return nullptr;
  r->audio_seconds = (float)seconds;
  return r.release();
}

}  // namespace

extern "C" void* fa_offline_infer_vad(void* asr, void* vad, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                                      const float* hw_embed, int32_t n_hotwords, const FaLongAudioOptions* opts) {
  g_err.clear();
  return infer_vad(asr, vad, bufs, n_samples, batch, pcm_format, hw_embed, n_hotwords, nullptr, nullptr, opts);
}

extern "C" void* fa_offline_infer_vad_sv(void* asr, void* vad, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                                         const int32_t* language_ids, const int32_t* textnorm_ids, const FaLongAudioOptions* opts) {
  g_err.clear();
  if (asr && !static_cast<Model*>(asr)->sv) return fail("fa_offline_infer_vad_sv: not a SenseVoice model file");
  return infer_vad(asr, vad, bufs, n_samples, batch, pcm_format, nullptr, 0, language_ids, textnorm_ids, opts);
}

extern "C" void* fa_offline_infer_vad_spk(void* asr, void* vad, void* spk, const void* const* bufs, const int64_t* n_samples, int32_t batch,
                                          int32_t pcm_format, const float* hw_embed, int32_t n_hotwords, const int32_t* language_ids,
                                          const int32_t* textnorm_ids, const FaLongAudioOptions* opts, int32_t preset_spk_num) {
  g_err.clear();
  if (!spk) return fail("fa_offline_infer_vad_spk: spk is NULL");
  if (asr && !static_cast<Model*>(asr)->sv && (language_ids || textnorm_ids)) return fail("fa_offline_infer_vad_spk: language / text-norm ids need a SenseVoice model file");
  return infer_vad(asr, vad, bufs, n_samples, batch, pcm_format, hw_embed, n_hotwords, language_ids, textnorm_ids, opts, static_cast<Spk*>(spk),
                   preset_spk_num);
}

extern "C" const int32_t* fa_offline_result_spk(const void* result, int32_t index, int32_t* n) {
  const Result* r = static_cast<const Result*>(result);
  if (!r || index < 0 || index >= (int32_t)r->spk.size() || r->spk[index].empty()) { if (n) *n = 0; return nullptr; }
  if (n) *n = (int32_t)r->spk[index].size();
  return r->spk[index].data();
}

extern "C" const int32_t* fa_offline_result_segments(const void* result, int32_t index, int32_t* n_segments) {
  const Result* r = static_cast<const Result*>(result);
  if (!r || index < 0 || index >= (int32_t)r->segs.size() || r->segs[index].empty()) { if (n_segments) *n_segments = 0; return nullptr; }
  if (n_segments) *n_segments = (int32_t)(r->segs[index].size() / 3);
  return r->segs[index].data();
}

// ------------------------------------------------------------------------------------------------ CT-Transformer punctuation handle
namespace {

// __punc_config__ of funasr_b200/pack.py:write_punc_model_file
enum { kPuncLayers = 0, kPuncDModel, kPuncHeads, kPuncKernel, kPuncSentenceEnd, kPuncSplit, kPuncCfgLen };

struct Punc {
  Loaded file;
  fa_punc::Vocab vocab;
  int layers = 0, d_model = 0, heads = 0, d_in = 0, n_embed = 0;
  int64_t max_window = 0;                            // 0: no bound (128-wide heads run the tiled attention kernel)
  std::vector<FaEncLayer> enc_l;
  FaEncoder enc{};
  FaLinear out{};
  const float* embed = nullptr;
  DevBuf io, x, h, pids, best, ws;                   // grow-only, sized by each step's t_max
  std::vector<int32_t> host_io;                      // ids [batch, t_max] then lens [batch]: one host-to-device copy per step
};

// a newline-joined UTF-8 list stored as the bytes of an fp32 tensor
std::vector<std::string> blob_lines(const Tensor& t) {
  std::string s(reinterpret_cast<const char*>(t.host.data()), t.host.size() * 4);
  while (!s.empty() && s.back() == '\0') s.pop_back();
  std::vector<std::string> out;
  for (size_t a = 0;;) {
    const size_t b = s.find('\n', a);
    out.push_back(s.substr(a, b == std::string::npos ? std::string::npos : b - a));
    if (b == std::string::npos) break;
    a = b + 1;
  }
  return out;
}

bool build_punc(Punc& p, Builder& b) {
  b.what = "punctuation model: ";
  b.ln_eps = 1e-12f;                                 // SANMEncoder's LayerNorm; the fp32 path whatever the recogniser's gemm-mode (PuncEngine)
  const Tensor* cfg = b.get("__punc_config__");
  const Tensor* pl = b.get("__punc_list__");
  const Tensor* tl = cfg && pl ? b.get("__punc_tokens__") : nullptr;
  if (!tl) return false;
  if (cfg->host.size() != kPuncCfgLen) return b.refuse("bad __punc_config__");
  const float* c = cfg->host.data();
  p.layers = (int)c[kPuncLayers]; p.d_model = (int)c[kPuncDModel]; p.heads = (int)c[kPuncHeads];
  const int D = p.d_model, K = (int)c[kPuncKernel];
  if (p.layers < 1) return b.refuse("no encoder layer");
  if (K != 11 && K != 21 && K != 31) return b.refuse("FSMN kernel " + std::to_string(K) + " (the fp32 FSMN kernel takes 11, 21 or 31)");
  if (D > 512 || D < 64 || D % 16) return b.refuse("d_model " + std::to_string(D) + " (the encoder takes a multiple of 16 up to 512)");
  const int hd = p.heads > 0 && D % p.heads == 0 ? D / p.heads : 0;
  if (hd < 32 || hd > 128 || hd % 32)
    return b.refuse(std::to_string(p.heads) + " heads of d_model " + std::to_string(D) + " (the head dim must be a multiple of 32 up to 128)");
  std::string err;
  if (!p.vocab.init(blob_lines(*tl), blob_lines(*pl), (int32_t)c[kPuncSentenceEnd], (int32_t)c[kPuncSplit], err)) return b.refuse(err);
  const Tensor* emb = b.get("embed.weight");
  if (!emb) return false;
  if (emb->shape.size() != 2 || emb->shape[1] > 560 || emb->shape[1] % 16 || emb->shape[0] < 1) return b.refuse("bad shape of embed.weight");
  p.n_embed = (int)emb->shape[0]; p.d_in = (int)emb->shape[1];
  p.embed = emb->dev;
  b.shaped(enc_layer_prefix(false, 0) + ".self_attn.fsmn_block.weight", {D, 1, K});     // bind_stack holds every layer to layer 0's taps
  bind_stack(b, false, p.layers, p.d_in, D, p.heads, p.enc_l, p.enc);
  if (b.opt(enc_layer_prefix(false, p.layers) + ".norm1.weight")) return b.refuse("more encoder layers than __punc_config__ says");
  const int64_t n_punc = (int64_t)p.vocab.punc.size();
  b.shaped("decoder.weight", {n_punc, D}); b.shaped("decoder.bias", {n_punc});
  p.out = b.lin("decoder");
  p.max_window = hd == 128 ? 0 : 160 * 1024 / 16;     // fa_attention_f32_ex's warp-per-query kernel: 4 * tk floats of shared memory
  return b.ok;
}

// one lockstep step on the GPU: punc_forward (model.py:112-125) + arg-max over a padded batch of windows
bool punc_step(Punc& p, const int32_t* ids, const int32_t* lens, int32_t B, int32_t T, int32_t* punc_out, std::string& err) {
  cudaStream_t st = p.file.st;
  const int64_t M = (int64_t)B * T;
  const int n_punc = p.out.out_f;
  const size_t ws = std::max(fa_sanm_encoder_workspace_bytes(B, T, FA_GEMM_F32_SIMT), fa_linear_argmax_workspace_bytes(M, n_punc, FA_GEMM_F32_SIMT));
  if (!(p.io.reserve((size_t)(M + B) * 4) && p.x.reserve((size_t)M * p.d_in * 4) && p.h.reserve((size_t)M * p.d_model * 4) &&
        p.pids.reserve((size_t)M * 4) && p.best.reserve((size_t)M * 4) && p.ws.reserve(ws))) {
    err = "device allocation failed (punctuation)";
    return false;
  }
  p.host_io.assign(ids, ids + M);
  p.host_io.insert(p.host_io.end(), lens, lens + B);
  int32_t* ids_d = static_cast<int32_t*>(p.io.p);
  cudaMemcpyAsync(ids_d, p.host_io.data(), (size_t)(M + B) * 4, cudaMemcpyHostToDevice, st);
  float* x = static_cast<float*>(p.x.p);
  float* h = static_cast<float*>(p.h.p);
  int rc = fa_embedding(ids_d, p.embed, p.d_in, p.n_embed, M, x, st);
  if (rc == FA_OK) rc = fa_sanm_encoder_forward(&p.enc, x, ids_d + M, B, T, h, FA_GEMM_F32_SIMT, p.ws.p, p.ws.cap, st);
  if (rc == FA_OK)
    rc = fa_linear_argmax(&p.out, h, nullptr, M, static_cast<int32_t*>(p.pids.p), static_cast<float*>(p.best.p), nullptr, FA_GEMM_F32_SIMT, p.ws.p,
                          p.ws.cap, st);
  if (rc != FA_OK) { err = std::string("punctuation forward: ") + fa_status_string(rc); return false; }
  cudaMemcpyAsync(punc_out, p.pids.p, (size_t)M * 4, cudaMemcpyDeviceToHost, st);
  if (!sync_stream(st)) { err = g_err; return false; }
  return true;
}

}  // namespace

extern "C" void* fa_punc_init(const char* model_file, int32_t device) {
  g_err.clear();
  return open_handle(model_file, device, FA_GEMM_F32_SIMT, build_punc);
}

extern "C" void fa_punc_uninit(void* punc) { delete static_cast<Punc*>(punc); }

extern "C" void* fa_punc_infer(void* punc, const char* const* texts, int32_t n) {
  g_err.clear();
  Punc* p = static_cast<Punc*>(punc);
  if (!p || (!texts && n > 0) || n < 0) return fail("bad argument");
  for (int32_t i = 0; i < n; ++i)
    if (!texts[i]) return fail("text " + std::to_string(i) + " is NULL");
  cudaSetDevice(p->file.device);
  std::unique_ptr<fa_punc::Result> r(new fa_punc::Result());
  std::string err;
  const fa_punc::Scorer score = [p](const int32_t* ids, const int32_t* lens, int32_t B, int32_t T, int32_t* out, std::string& e) {
    return punc_step(*p, ids, lens, B, T, out, e);
  };
  if (!no_throw("fa_punc_infer: ", [&] { return fa_punc::walk(p->vocab, texts, n, p->max_window, score, *r, err) || (set_err(err), false); }))
    return nullptr;
  return r.release();
}

extern "C" void* fa_punc_walk_host(const char* const* texts, int32_t n, const char* const* tokens, int32_t n_tokens, const char* const* punc_list,
                                   int32_t n_punc, int32_t sentence_end_id, int32_t split_size, int64_t max_window, fa_punc_score_fn score_fn,
                                   void* ctx) {
  g_err.clear();
  if ((!texts && n > 0) || n < 0 || !tokens || n_tokens < 1 || !punc_list || n_punc < 1 || !score_fn) return fail("bad argument");
  for (int32_t i = 0; i < n; ++i)
    if (!texts[i]) return fail("text " + std::to_string(i) + " is NULL");
  std::unique_ptr<fa_punc::Result> r(new fa_punc::Result());
  std::string err;
  const bool ok = no_throw("fa_punc_walk_host: ", [&] {
    for (int32_t i = 0; i < n_tokens; ++i) if (!tokens[i]) { err = "token " + std::to_string(i) + " is NULL"; set_err(err); return false; }
    for (int32_t i = 0; i < n_punc; ++i) if (!punc_list[i]) { err = "punctuation " + std::to_string(i) + " is NULL"; set_err(err); return false; }
    std::vector<std::string> tok(tokens, tokens + n_tokens), pl(punc_list, punc_list + n_punc);
    fa_punc::Vocab v;
    const fa_punc::Scorer score = [&](const int32_t* ids, const int32_t* lens, int32_t B, int32_t T, int32_t* out, std::string& e) {
      const int32_t rc = score_fn(ctx, ids, lens, B, T, out);
      if (rc != 0) e = "scorer failed (" + std::to_string(rc) + ")";
      return rc == 0;
    };
    return (v.init(tok, pl, sentence_end_id, split_size, err) && fa_punc::walk(v, texts, n, max_window, score, *r, err)) || (set_err(err), false);
  });
  return ok ? r.release() : nullptr;
}

extern "C" const char* fa_punc_result_text(const void* result, int32_t index) {
  const fa_punc::Result* r = static_cast<const fa_punc::Result*>(result);
  return r && index >= 0 && index < (int32_t)r->text.size() ? r->text[index].c_str() : nullptr;
}

extern "C" const int32_t* fa_punc_result_ids(const void* result, int32_t index, int32_t* n) {
  const fa_punc::Result* r = static_cast<const fa_punc::Result*>(result);
  if (!r || index < 0 || index >= (int32_t)r->ids.size() || r->ids[index].empty()) { if (n) *n = 0; return nullptr; }
  if (n) *n = (int32_t)r->ids[index].size();
  return r->ids[index].data();
}

extern "C" int64_t fa_punc_result_steps(const void* result) { return result ? static_cast<const fa_punc::Result*>(result)->steps : 0; }

extern "C" void fa_punc_free_result(void* result) { delete static_cast<fa_punc::Result*>(result); }
