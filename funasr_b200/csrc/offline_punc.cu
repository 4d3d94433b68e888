// Handle-style CT-Transformer punctuation: fa_punc_init (model file -> handle), fa_punc_infer (many texts -> punctuated texts, every
// text one window per lockstep step), fa_punc_walk_host (the same walk over any scorer).  The text walk is punc_text.cpp.
#include "handle.h"
#include "punc_text.h"

using namespace fa_handle;

namespace {

// __punc_config__ of funasr_b200/pack.py:write_punc_model_file
enum { kPuncLayers = 0, kPuncDModel, kPuncHeads, kPuncKernel, kPuncSentenceEnd, kPuncSplit, kPuncCfgLen };

struct Punc {
  std::mutex mu;                                     // device lock
  Loaded file;
  fa_punc::Vocab vocab;
  int layers = 0, d_model = 0, heads = 0, d_in = 0, n_embed = 0;
  int64_t max_window = 0;                            // 0: no bound (128-wide heads run the tiled attention kernel)
  std::vector<FaEncLayer> enc_l;
  FaEncoder enc{};
  FaLinear out{};
  const float* embed = nullptr;
  DevBuf punc_step;                                  // grown to the largest step's t_max
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
  const size_t ws_bytes = std::max(fa_sanm_encoder_workspace_bytes(B, T, FA_GEMM_F32_SIMT), fa_linear_argmax_workspace_bytes(M, n_punc, FA_GEMM_F32_SIMT));
  int32_t *ids_d, *pids;
  float *x, *h, *best;
  void* ws;
  if (!carve(p.punc_step, "punctuation", [&](fa::Arena& a) {
        ids_d = a.take<int32_t>(M + B); x = a.take<float>((size_t)M * p.d_in); h = a.take<float>((size_t)M * p.d_model);
        pids = a.take<int32_t>(M); best = a.take<float>(M); ws = a.take<char>(ws_bytes);
      })) {
    err = g_err;
    return false;
  }
  p.host_io.assign(ids, ids + M);
  p.host_io.insert(p.host_io.end(), lens, lens + B);
  cudaMemcpyAsync(ids_d, p.host_io.data(), (size_t)(M + B) * 4, cudaMemcpyHostToDevice, st);
  int rc = fa_embedding(ids_d, p.embed, p.d_in, p.n_embed, M, x, st);
  if (rc == FA_OK) rc = fa_sanm_encoder_forward(&p.enc, x, ids_d + M, B, T, h, FA_GEMM_F32_SIMT, ws, ws_bytes, st);
  if (rc == FA_OK) rc = fa_linear_argmax(&p.out, h, nullptr, M, pids, best, nullptr, FA_GEMM_F32_SIMT, ws, ws_bytes, st);
  if (rc != FA_OK) { err = std::string("punctuation forward: ") + fa_status_string(rc); return false; }
  cudaMemcpyAsync(punc_out, pids, (size_t)M * 4, cudaMemcpyDeviceToHost, st);
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
  std::lock_guard<std::mutex> dev(p->mu);
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
  return result_row(result ? &static_cast<const fa_punc::Result*>(result)->ids : nullptr, index, n, 1, false);
}

extern "C" int64_t fa_punc_result_steps(const void* result) { return result ? static_cast<const fa_punc::Result*>(result)->steps : 0; }

extern "C" void fa_punc_free_result(void* result) { delete static_cast<fa_punc::Result*>(result); }
