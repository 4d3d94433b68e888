// Handle-style offline recogniser over the kernels of this library — the C-ABI counterpart of FunASR's C++ runtime
// surface (runtime/onnxruntime/include/funasrruntime.h:100-116: FunOfflineInit / FunOfflineInferBuffer / FunASRGetResult /
// FunASRFreeResult / FunOfflineUninit; its Paraformer::Forward is the same op chain with ONNX Runtime in the middle,
// runtime/onnxruntime/src/paraformer.cpp).  No Python, no torch: weights come from one flat file written by
// funasr_b200/pack.py (tensors under FunASR's own state_dict names), device memory from cudaMalloc.
//
//   fa_offline_init         model file -> handle (weights to HBM, fp16 planes for the tensor-core GEMMs)
//   fa_offline_infer        batch of host PCM buffers (f32 in [-1,1] or s16le) -> result (greedy token ids per utterance)
//   fa_offline_result_*     accessors;  fa_offline_free_result / fa_offline_uninit
// The tokenizer (ids -> text) stays with the caller, like every other entry point of this ABI.
#include "common.cuh"
#include <stdio.h>
#include <string.h>
#include <exception>
#include <map>
#include <string>
#include <vector>

namespace {

thread_local std::string g_err;
void set_err(const std::string& s) { g_err = s; }

struct Tensor {
  float* dev = nullptr;
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

struct Model {
  int device = 0, mode = 3;
  int enc_layers = 0, dec_layers = 0, d_model = 512, heads = 4, kernel = 11, vocab = 0, feat_dim = 560;
  float ln_eps = 1e-12f, cif_threshold = 1.f, tail_threshold = 0.45f;
  std::map<std::string, Tensor> t;
  std::vector<void*> owned;                    // weight planes etc.
  std::vector<FaEncLayer> enc_l;
  std::vector<FaDecLayer> dec_l;
  FaEncoder enc{};
  FaPredictor pred{};
  FaDecoder dec{};
  const float *mel = nullptr, *window = nullptr, *cmvn = nullptr;
  float* fbank_tables = nullptr;                     // fa_fbank_make_tables output (owned)
  cudaStream_t st = nullptr;
  DevBuf wav, pcm16, lens, feats, flens, encb, acoustic, tok, alphas, peaks, ws, ids, best, fids, flens_out, hw, hw_lens;
  bool contextual = false;                           // ContextualParaformer: decoder with a hotword bias branch
  std::map<std::string, std::vector<float>> host_cache;   // fa_offline_host_tensor
  ~Model() {
    for (auto& kv : t) if (kv.second.dev) cudaFree(kv.second.dev);
    for (void* p : owned) cudaFree(p);
    if (st) cudaStreamDestroy(st);
  }
};

struct Result {
  std::vector<std::vector<int32_t>> ids;
  std::vector<int32_t> token_num;
  float audio_seconds = 0.f;
};

__global__ void pcm16_to_f32_kernel(const int16_t* __restrict__ src, float* __restrict__ dst, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (float)src[i] * (1.0f / 32768.0f);     // exact; the frontend multiplies by 32768 again (wav_frontend.py:169)
}

bool read_exact(FILE* f, void* dst, size_t n) { return fread(dst, 1, n, f) == n; }

// File layout (funasr_b200/pack.py): "FAB2MDL1", u32 n_tensors, then per tensor:
//   u32 name_len, name, u32 ndim, i64 dims[ndim], u64 nbytes, zero padding to a 16-byte file offset, fp32 data
bool load_file(Model& m, const char* path) {
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
    host.resize(nbytes / 4);
    ok = read_exact(f, host.data(), nbytes);
    if (!ok) break;
    if (cudaMalloc(&tt.dev, nbytes ? nbytes : 4) != cudaSuccess) { ok = false; set_err("cudaMalloc failed for " + name); break; }
    cudaMemcpy(tt.dev, host.data(), nbytes, cudaMemcpyHostToDevice);
    m.t[name] = tt;
  }
  fclose(f);
  if (!ok && g_err.empty()) set_err(std::string("malformed model file ") + path);
  return ok;
}

struct Builder {
  Model& m;
  bool ok = true;
  const Tensor* get(const std::string& k) {
    auto it = m.t.find(k);
    if (it == m.t.end()) { if (ok) set_err("missing tensor " + k); ok = false; return nullptr; }
    return &it->second;
  }
  const float* ptr(const std::string& k) { const Tensor* t = get(k); return t ? t->dev : nullptr; }
  FaNorm norm(const std::string& p) {
    FaNorm nm{};
    const Tensor* w = get(p + ".weight");
    nm.g = w ? w->dev : nullptr; nm.b = ptr(p + ".bias"); nm.n = w ? (int32_t)w->numel() : 0; nm.eps = m.ln_eps;
    return nm;
  }
  FaLinear lin(const std::string& p, bool bias = true, const char* weight_key = nullptr) {
    FaLinear L{};
    const Tensor* w = get(weight_key ? std::string(weight_key) : p + ".weight");
    // [out, in] or a k = 1 Conv1d weight [out, in, 1] (bias_output, contextual_paraformer/decoder.py:287)
    if (!w || !(w->shape.size() == 2 || (w->shape.size() == 3 && w->shape[2] == 1))) { if (ok) set_err("bad weight " + p); ok = false; return L; }
    L.w = w->dev; L.b = bias ? ptr(p + ".bias") : nullptr;
    L.out_f = (int32_t)w->shape[0]; L.in_f = (int32_t)w->shape[1]; L.in_pad = (L.in_f + 63) / 64 * 64;
    if (m.mode != FA_GEMM_F32_SIMT) {
      void* planes = nullptr;
      if (cudaMalloc(&planes, (size_t)3 * L.out_f * L.in_pad * 2) != cudaSuccess) { ok = false; set_err("cudaMalloc planes"); return L; }
      m.owned.push_back(planes);
      if (fa_split_planes(L.w, L.in_f, L.out_f, L.in_f, L.in_pad, planes, m.st) != FA_OK) { ok = false; set_err("fa_split_planes failed"); }
      L.w_planes = planes;
    }
    return L;
  }
};

bool build(Model& m) {
  Builder b{m};
  const Tensor* cfg = b.get("__config__");
  if (!cfg || cfg->numel() < 10) { set_err("missing __config__"); return false; }
  float c[10];
  cudaMemcpy(c, cfg->dev, sizeof(c), cudaMemcpyDeviceToHost);
  m.enc_layers = (int)c[0]; m.dec_layers = (int)c[1]; m.d_model = (int)c[2]; m.heads = (int)c[3]; m.kernel = (int)c[4];
  m.vocab = (int)c[5]; m.feat_dim = (int)c[6]; m.ln_eps = c[7]; m.cif_threshold = c[8]; m.tail_threshold = c[9];
  if (m.enc_layers < 1 || m.dec_layers < 1 || m.d_model != 512 || m.heads * 128 != m.d_model) { set_err("unsupported config"); return false; }
  // the FSMN tap count is read from each stack's own weight [512, 1, K]: encoder and decoder kernel_size are independent
  // constructor arguments in the reference (sanm/encoder.py:188, paraformer/decoder.py:234 — decoder default 21)
  auto fsmn_taps = [&](const char* key) -> int {
    const Tensor* t = b.get(key);
    return (t && t->shape.size() == 3) ? (int)t->shape[2] : m.kernel;
  };
  m.mel = b.ptr("frontend.mel_banks"); m.window = b.ptr("frontend.window");
  if (m.mel && m.window) {
    void* tb = nullptr;
    if (cudaMalloc(&tb, fa_fbank_tables_bytes()) != cudaSuccess) { set_err("cudaMalloc fbank tables"); return false; }
    m.owned.push_back(tb);
    m.fbank_tables = static_cast<float*>(tb);
    if (fa_fbank_make_tables(m.mel, m.window, m.fbank_tables, m.st) != FA_OK) { set_err("fa_fbank_make_tables failed"); return false; }
  }
  m.cmvn = m.t.count("frontend.cmvn") ? m.t["frontend.cmvn"].dev : nullptr;
  // encoder (engine.py:_enc_stack; SANMEncoder encoder.py:188-461)
  m.enc_l.resize(m.enc_layers);
  for (int i = 0; i < m.enc_layers; ++i) {
    const std::string p = i == 0 ? "encoder.encoders0.0" : "encoder.encoders." + std::to_string(i - 1);
    FaEncLayer& L = m.enc_l[i];
    L.norm1 = b.norm(p + ".norm1"); L.norm2 = b.norm(p + ".norm2");
    L.qkv = b.lin(p + ".self_attn.linear_q_k_v"); L.out = b.lin(p + ".self_attn.linear_out");
    L.fsmn_w = b.ptr(p + ".self_attn.fsmn_block.weight");
    L.w1 = b.lin(p + ".feed_forward.w_1"); L.w2 = b.lin(p + ".feed_forward.w_2");
  }
  m.enc.layers = m.enc_l.data(); m.enc.n_layers = m.enc_layers; m.enc.heads = m.heads; m.enc.fsmn_k = fsmn_taps("encoder.encoders0.0.self_attn.fsmn_block.weight");
  m.enc.after_norm = b.norm("encoder.after_norm"); m.enc.pe_inv_timescales = b.ptr("encoder.pe_inv_timescales");
  // predictor (CifPredictorV2 cif_predictor.py:209-314); conv weight already repacked to [512, 3*512] by pack.py
  m.pred.conv = b.lin("predictor.cif_conv1d", true, "predictor.cif_conv1d.gemm_weight");
  m.pred.out_w = b.ptr("predictor.cif_output.weight"); m.pred.out_b = b.ptr("predictor.cif_output.bias");
  m.pred.threshold = m.cif_threshold; m.pred.tail_threshold = m.tail_threshold; m.pred.smooth_factor = 1.f; m.pred.noise_threshold = 0.f;
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
  m.contextual = m.t.count("decoder.bias_decoder.norm3.weight") > 0;
  const int n_plain = m.contextual ? m.dec_layers - 1 : m.dec_layers;
  m.dec_l.resize(n_plain > 0 ? n_plain : 1);
  for (int i = 0; i < n_plain; ++i) dec_layer(m.dec_l[i], "decoder.decoders." + std::to_string(i), true);
  m.dec.layers = m.dec_l.data(); m.dec.n_layers = n_plain; m.dec.heads = m.heads; m.dec.vocab = m.vocab;
  m.dec.fsmn_k = fsmn_taps(n_plain > 0 ? "decoder.decoders.0.self_attn.fsmn_block.weight" : "decoder.last_decoder.self_attn.fsmn_block.weight");
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
  if (!b.ok) return false;
  return cudaStreamSynchronize(m.st) == cudaSuccess;
}

int num_lfr_frames(int64_t n) {       // wav_frontend.py:73 after kaldi.py snip_edges framing
  const int64_t mfr = n >= 400 ? 1 + (n - 400) / 160 : 0;
  return (int)((mfr + 5) / 6);
}

}  // namespace

extern "C" const char* fa_offline_last_error(void) { return g_err.c_str(); }
extern "C" void* fa_offline_infer_hw(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                                     const float* hw_embed, int32_t n_hotwords);

extern "C" void* fa_offline_init(const char* model_file, int32_t device, int32_t gemm_mode) {
  g_err.clear();
  if (!model_file) { set_err("model_file is NULL"); return nullptr; }
  if (gemm_mode != FA_GEMM_F32_SIMT && gemm_mode != FA_GEMM_F16X1 && gemm_mode != FA_GEMM_F16X3 && gemm_mode != FA_GEMM_F16X6) {
    set_err("bad gemm_mode"); return nullptr;
  }
  if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); set_err("no such CUDA device (this library has no CPU path)"); return nullptr; }
  Model* m = new Model();
  m->device = device; m->mode = gemm_mode;
  if (cudaStreamCreateWithFlags(&m->st, cudaStreamNonBlocking) != cudaSuccess) { set_err("cudaStreamCreate failed"); delete m; return nullptr; }
  bool ok = false;
  try {                                   // a malformed file can ask for an absurd allocation: no C++ exception may cross the C ABI
    ok = load_file(*m, model_file) && build(*m);
  } catch (const std::exception& e) {
    set_err(std::string("model file rejected: ") + e.what());
  }
  if (!ok) { delete m; return nullptr; }
  return m;
}

extern "C" void fa_offline_uninit(void* handle) { delete static_cast<Model*>(handle); }

extern "C" int32_t fa_offline_is_contextual(const void* handle) { return handle && static_cast<const Model*>(handle)->contextual ? 1 : 0; }

extern "C" const float* fa_offline_host_tensor(void* handle, const char* name, int64_t* numel) {
  Model* m = static_cast<Model*>(handle);
  if (numel) *numel = 0;
  if (!m || !name) return nullptr;
  auto it = m->t.find(name);
  if (it == m->t.end()) return nullptr;
  auto& hc = m->host_cache[name];
  if (hc.empty() && it->second.numel() > 0) {
    hc.resize((size_t)it->second.numel());
    cudaSetDevice(m->device);
    if (cudaMemcpy(hc.data(), it->second.dev, hc.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess) { hc.clear(); return nullptr; }
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
  Model* mp = static_cast<Model*>(handle);
  if (!mp || !bufs || !n_samples || batch <= 0 || (pcm_format != 0 && pcm_format != 1)) { set_err("bad argument"); return nullptr; }
  Model& m = *mp;
  if (m.contextual && (!hw_embed || n_hotwords < 1)) { set_err("this model has a hotword bias decoder: pass hotword embeddings (at least the <s> entry)"); return nullptr; }
  cudaSetDevice(m.device);
  int64_t nmax = 0;
  double seconds = 0.0;
  std::vector<int32_t> lens_h(batch);
  int t_max = 0;
  for (int i = 0; i < batch; ++i) {
    if (!bufs[i] || n_samples[i] < 400 || n_samples[i] > 0x7fffffffLL) { set_err("every buffer needs >= 400 samples (25 ms)"); return nullptr; }
    lens_h[i] = (int32_t)n_samples[i];
    nmax = n_samples[i] > nmax ? n_samples[i] : nmax;
    seconds += (double)n_samples[i] / 16000.0;
    const int t = num_lfr_frames(n_samples[i]);
    t_max = t > t_max ? t : t_max;
  }
  const int B = batch, D = m.d_model, T = t_max;
  const int64_t stride = (nmax + 3) / 4 * 4;
#define FA_OFF(x, msg) do { if (!(x)) { set_err(msg); return nullptr; } } while (0)
  FA_OFF(m.wav.reserve((size_t)B * stride * 4) && m.lens.reserve((size_t)B * 4), "device allocation failed (waveforms)");
  float* wav = static_cast<float*>(m.wav.p);
  if (pcm_format == 1) {
    FA_OFF(m.pcm16.reserve((size_t)B * stride * 2), "device allocation failed (pcm)");
    int16_t* p16 = static_cast<int16_t*>(m.pcm16.p);
    for (int i = 0; i < B; ++i) cudaMemcpyAsync(p16 + (int64_t)i * stride, bufs[i], (size_t)n_samples[i] * 2, cudaMemcpyHostToDevice, m.st);
    const int64_t tot = (int64_t)B * stride;
    pcm16_to_f32_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, m.st>>>(p16, wav, tot);
  } else {
    for (int i = 0; i < B; ++i) cudaMemcpyAsync(wav + (int64_t)i * stride, bufs[i], (size_t)n_samples[i] * 4, cudaMemcpyHostToDevice, m.st);
  }
  cudaMemcpyAsync(m.lens.p, lens_h.data(), (size_t)B * 4, cudaMemcpyHostToDevice, m.st);
  const int n_cap = T + 1;
  FA_OFF(m.feats.reserve((size_t)B * T * m.feat_dim * 4) && m.flens.reserve((size_t)B * 4) && m.encb.reserve((size_t)B * T * D * 4) &&
             m.acoustic.reserve((size_t)B * n_cap * D * 4) && m.tok.reserve((size_t)B * 4) && m.alphas.reserve((size_t)B * n_cap * 4) &&
             m.peaks.reserve((size_t)B * n_cap * 4),
         "device allocation failed (activations)");
  size_t ws = fa_sanm_encoder_workspace_bytes(B, T, m.mode);
  const size_t ws2 = fa_cif_predictor_workspace_bytes(B, T, m.mode);
  ws = ws2 > ws ? ws2 : ws;
  FA_OFF(m.ws.reserve(ws), "device allocation failed (workspace)");
  int rc = fa_fbank_lfr_cmvn_tables(wav, static_cast<int32_t*>(m.lens.p), B, stride, m.cmvn, m.fbank_tables, 7, 6, static_cast<float*>(m.feats.p),
                                    T, static_cast<int32_t*>(m.flens.p), T, m.st);
  FA_OFF(rc == FA_OK, std::string("fa_fbank_lfr_cmvn_tables: ") + fa_status_string(rc));
  rc = fa_sanm_encoder_forward(&m.enc, static_cast<float*>(m.feats.p), static_cast<int32_t*>(m.flens.p), B, T, static_cast<float*>(m.encb.p),
                               m.mode, m.ws.p, m.ws.cap, m.st);
  FA_OFF(rc == FA_OK, std::string("fa_sanm_encoder_forward: ") + fa_status_string(rc));
  rc = fa_cif_predictor_forward(&m.pred, static_cast<float*>(m.encb.p), static_cast<int32_t*>(m.flens.p), B, T, static_cast<float*>(m.acoustic.p),
                                n_cap, static_cast<int32_t*>(m.tok.p), static_cast<float*>(m.alphas.p), static_cast<float*>(m.peaks.p), m.mode,
                                m.ws.p, m.ws.cap, m.st);
  FA_OFF(rc == FA_OK, std::string("fa_cif_predictor_forward: ") + fa_status_string(rc));
  Result* r = new Result();
  r->audio_seconds = (float)seconds;
  r->token_num.resize(B);
  cudaMemcpyAsync(r->token_num.data(), m.tok.p, (size_t)B * 4, cudaMemcpyDeviceToHost, m.st);
  if (cudaStreamSynchronize(m.st) != cudaSuccess) { set_err(std::string("CUDA error: ") + cudaGetErrorString(cudaGetLastError())); delete r; return nullptr; }
  int n_max = 0;                                             // the path's one host sync (cif_predictor.py:311)
  for (int i = 0; i < B; ++i) n_max = r->token_num[i] > n_max ? r->token_num[i] : n_max;
  r->ids.resize(B);
  if (n_max < 1) return r;                                   // paraformer/model.py:615-616
  const int nh = m.contextual ? n_hotwords : 0;
  if (!(m.ids.reserve((size_t)B * n_max * 4) && m.best.reserve((size_t)B * n_max * 4) && m.fids.reserve((size_t)B * n_max * 4) &&
        m.flens_out.reserve((size_t)B * 4) && m.ws.reserve(fa_paraformer_decoder_workspace_bytes_hw(B, T, n_max, m.vocab, m.mode, nh)))) {
    set_err("device allocation failed (decoder)"); delete r; return nullptr;
  }
  if (m.contextual) {                                        // hotword memory [n_hw, 512] (contextual_paraformer/model.py:350-372) + per-utterance counts
    if (!(m.hw.reserve((size_t)nh * D * 4) && m.hw_lens.reserve((size_t)B * 4))) { set_err("device allocation failed (hotwords)"); delete r; return nullptr; }
    std::vector<int32_t> hl(B, nh);
    cudaMemcpyAsync(m.hw.p, hw_embed, (size_t)nh * D * 4, cudaMemcpyHostToDevice, m.st);
    cudaMemcpyAsync(m.hw_lens.p, hl.data(), (size_t)B * 4, cudaMemcpyHostToDevice, m.st);
    cudaStreamSynchronize(m.st);                             // hl is a stack vector
    m.dec.has_bias = 1; m.dec.n_hotwords = nh;
    m.dec.hw_embed = static_cast<const float*>(m.hw.p); m.dec.hw_lens = static_cast<const int32_t*>(m.hw_lens.p);
  }
  rc = fa_paraformer_decoder_forward(&m.dec, static_cast<float*>(m.encb.p), static_cast<int32_t*>(m.flens.p), B, T, static_cast<float*>(m.acoustic.p),
                                     n_cap, static_cast<int32_t*>(m.tok.p), n_max, static_cast<int32_t*>(m.ids.p), static_cast<float*>(m.best.p),
                                     nullptr, 1, m.mode, m.ws.p, m.ws.cap, m.st);
  if (rc == FA_OK)
    rc = fa_greedy_filter(static_cast<int32_t*>(m.ids.p), static_cast<int32_t*>(m.tok.p), B, n_max, 1, 2, 0, static_cast<int32_t*>(m.fids.p),
                          static_cast<int32_t*>(m.flens_out.p), m.st);
  if (rc != FA_OK) { set_err(std::string("decoder: ") + fa_status_string(rc)); delete r; return nullptr; }
  std::vector<int32_t> fids((size_t)B * n_max), fl(B);
  cudaMemcpyAsync(fids.data(), m.fids.p, fids.size() * 4, cudaMemcpyDeviceToHost, m.st);
  cudaMemcpyAsync(fl.data(), m.flens_out.p, (size_t)B * 4, cudaMemcpyDeviceToHost, m.st);
  if (cudaStreamSynchronize(m.st) != cudaSuccess) { set_err(std::string("CUDA error: ") + cudaGetErrorString(cudaGetLastError())); delete r; return nullptr; }
  for (int i = 0; i < B; ++i) r->ids[i].assign(fids.begin() + (size_t)i * n_max, fids.begin() + (size_t)i * n_max + fl[i]);
#undef FA_OFF
  return r;
}

extern "C" int32_t fa_offline_result_count(const void* result) { return result ? (int32_t)static_cast<const Result*>(result)->ids.size() : 0; }

extern "C" const int32_t* fa_offline_result_ids(const void* result, int32_t index, int32_t* n_ids) {
  const Result* r = static_cast<const Result*>(result);
  if (!r || index < 0 || index >= (int32_t)r->ids.size()) { if (n_ids) *n_ids = 0; return nullptr; }
  if (n_ids) *n_ids = (int32_t)r->ids[index].size();
  return r->ids[index].data();
}

extern "C" float fa_offline_result_audio_seconds(const void* result) { return result ? static_cast<const Result*>(result)->audio_seconds : 0.f; }

extern "C" void fa_offline_free_result(void* result) { delete static_cast<Result*>(result); }
