// Handle-style CT-Transformer punctuation: fa_punc_init (model file -> handle), fa_punc_infer (many texts -> punctuated texts, every
// text one window per lockstep step), fa_punc_walk_host (the same walk over any scorer).  The text walk is punc_text.cpp.
//
// Concurrent fa_punc_infer calls on one handle share steps.  A window's punctuation depends on that window only (punc_text.cpp), and
// a step is one window per text, so the texts of many calls can advance in one lockstep walk, and a call can join it at any step
// boundary.  A call checks its arguments and splits its texts into words on its own thread, then posts a ticket holding their walk
// state to the handle's request pool (request_pool.h).  Each round of the pool's leader is one step: it admits the queued tickets in
// arrival order (while the step's carve stays within kStepBytes; the first on an idle pool always), composes one padded step from
// every active text of every admitted call, scores it under the device lock and applies the results; the calls that ended leave the
// pool.  Admitted calls stay held across steps, so the walk state lives in the tickets, not on a leader's stack.  A window over
// max_window fails only its own call, before that step's scorer runs, with the message it gets alone; a scorer or device failure fails
// every call that had a window in that step.
#include "handle.h"
#include "punc_text.h"

using namespace fa_handle;

namespace {

// __punc_config__ of funasr_b200/pack.py:write_punc_model_file
enum { kPuncLayers = 0, kPuncDModel, kPuncHeads, kPuncKernel, kPuncSentenceEnd, kPuncSplit, kPuncCfgLen };

// a further call joins a step only while the step's device buffers (punc_step's carve) stay within this
const size_t kStepBytes = size_t(1) << 30;

// One fa_punc_infer call in the pool: its texts' walk state, stepped by whichever thread leads
struct PuncTicket : PoolTicket {
  std::vector<fa_punc::Text> texts;
  int64_t steps = 0;                                 // the steps it had a window in
  std::unique_ptr<fa_punc::Result> res;              // written by the leader, read by the owner once done
};

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
  fa_punc_score_fn host_score = nullptr;             // fa_punc_init_host: steps call host_score(host_ctx, ...) in place of the network
  void* host_ctx = nullptr;
  DevBuf punc_step;                                  // grown to the largest step's t_max
  std::vector<int32_t> host_io;                      // ids [batch, t_max] then lens [batch]: one host-to-device copy per step
  RequestPool<PuncTicket> pool;                      // held: the admitted calls with windows left, in admission order
  fa_punc::Step step;                                // the leader's step
  std::atomic<int64_t> pool_steps{0};                // steps scored since init
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

// punc_step's device buffers for B windows of T words, taken from a
struct StepBufs {
  int32_t *ids_d, *pids;
  float *x, *h, *best;
  void* ws;
  size_t ws_bytes;
};
void take_step(const Punc& p, fa::Arena& a, int32_t B, int32_t T, StepBufs& s) {
  const int64_t M = (int64_t)B * T;
  s.ws_bytes = std::max(fa_sanm_encoder_workspace_bytes(B, T, FA_GEMM_F32_SIMT), fa_linear_argmax_workspace_bytes(M, p.out.out_f, FA_GEMM_F32_SIMT));
  s.ids_d = a.take<int32_t>(M + B); s.x = a.take<float>((size_t)M * p.d_in); s.h = a.take<float>((size_t)M * p.d_model);
  s.pids = a.take<int32_t>(M); s.best = a.take<float>(M); s.ws = a.take<char>(s.ws_bytes);
}

// the bytes punc_step carves for B windows of T words (0 on a host handle)
size_t step_bytes(const Punc& p, int64_t B, int64_t T) {
  if (p.host_score) return 0;
  if (B * T > INT32_MAX) return SIZE_MAX;
  fa::Arena m = fa::Arena::measuring();
  StepBufs s;
  take_step(p, m, (int32_t)B, (int32_t)T, s);
  return m.bytes();
}

// one lockstep step on the GPU: punc_forward (model.py:112-125) + arg-max over a padded batch of windows
bool punc_step(Punc& p, const int32_t* ids, const int32_t* lens, int32_t B, int32_t T, int32_t* punc_out, std::string& err) {
  cudaStream_t st = p.file.st;
  const int64_t M = (int64_t)B * T;
  StepBufs s;
  if (!carve(p.punc_step, "punctuation", [&](fa::Arena& a) { take_step(p, a, B, T, s); })) {
    err = g_err;
    return false;
  }
  p.host_io.assign(ids, ids + M);
  p.host_io.insert(p.host_io.end(), lens, lens + B);
  cudaMemcpyAsync(s.ids_d, p.host_io.data(), (size_t)(M + B) * 4, cudaMemcpyHostToDevice, st);
  int rc = fa_embedding(s.ids_d, p.embed, p.d_in, p.n_embed, M, s.x, st);
  if (rc == FA_OK) rc = fa_sanm_encoder_forward(&p.enc, s.x, s.ids_d + M, B, T, s.h, FA_GEMM_F32_SIMT, s.ws, s.ws_bytes, st);
  if (rc == FA_OK) rc = fa_linear_argmax(&p.out, s.h, nullptr, M, s.pids, s.best, nullptr, FA_GEMM_F32_SIMT, s.ws, s.ws_bytes, st);
  if (rc != FA_OK) { err = std::string("punctuation forward: ") + fa_status_string(rc); return false; }
  cudaMemcpyAsync(punc_out, s.pids, (size_t)M * 4, cudaMemcpyDeviceToHost, st);
  if (!sync_stream(st)) { err = g_err; return false; }
  return true;
}

bool score_step(Punc& p, fa_punc::Step& s, std::string& err) {
  if (!p.host_score) return punc_step(p, s.ids.data(), s.lens.data(), s.batch, s.t_max, s.pout.data(), err);
  const int32_t rc = p.host_score(p.host_ctx, s.ids.data(), s.lens.data(), s.batch, s.t_max, s.pout.data());
  if (rc != 0) err = "scorer failed (" + std::to_string(rc) + ")";
  return rc == 0;
}

// t's result: every text's punctuated text and ids, and the steps it had a window in
void finish(PuncTicket& t) {
  t.res.reset(new fa_punc::Result());
  const size_t n = t.texts.size();
  t.res->text.resize(n);
  t.res->ids.resize(n);
  for (size_t i = 0; i < n; ++i) {
    t.res->text[i].swap(t.texts[i].text);
    t.res->ids[i].swap(t.texts[i].punc);
  }
  t.res->steps = t.steps;
  t.texts.clear();
}

// A step's admission: queued tickets join the walk in arrival order while the next step's carve stays within kStepBytes; the first
// ticket of an idle walk always joins, and a ticket that does not fit holds back those behind it
void admit_queued(const Punc& p, std::deque<PuncTicket*>& queue, std::vector<PuncTicket*>& held) {
  int64_t B = 0, T = 0;
  auto extent = [&](const PuncTicket& t, int64_t& b, int64_t& tm) {
    for (const fa_punc::Text& x : t.texts)
      if (x.active()) { ++b; tm = std::max(tm, fa_punc::window_len(p.vocab, x)); }
  };
  for (const PuncTicket* t : held) extent(*t, B, T);
  while (!queue.empty()) {
    PuncTicket* t = queue.front();
    int64_t b = B, tm = T;
    extent(*t, b, tm);
    if (!held.empty() && step_bytes(p, b, tm) > kStepBytes) break;
    held.push_back(t);
    queue.pop_front();
    B = b; T = tm;
  }
}

bool has_ended(const PuncTicket& t) {
  return !t.err.empty() || std::none_of(t.texts.begin(), t.texts.end(), [](const fa_punc::Text& x) { return x.active(); });
}

// One step over every held call's active texts; the calls that ended, with a result or a message, move from held to `ended`
void run_step(Punc& p, std::vector<PuncTicket*>& held, std::vector<PuncTicket*>& ended) {
  std::vector<fa_punc::Text*> rows;
  std::vector<PuncTicket*> owner;                    // per row
  for (PuncTicket* t : held) {                       // a window over max_window fails its call before the scorer runs, as alone
    const size_t r0 = rows.size();
    for (size_t i = 0; i < t->texts.size() && t->err.empty(); ++i) {
      fa_punc::Text& x = t->texts[i];
      if (!x.active()) continue;
      if (!fa_punc::check_window(p.vocab, x, (int32_t)i, p.max_window, t->err)) break;
      rows.push_back(&x);
    }
    if (!t->err.empty()) rows.resize(r0);
    owner.resize(rows.size(), t);
  }
  if (!rows.empty()) {
    fa_punc::compose(p.vocab, rows, p.step);
    std::string err;
    bool ok;
    if (!p.host_score) cudaSetDevice(p.file.device);
    {
      std::lock_guard<std::mutex> dev(p.mu);
      ok = score_step(p, p.step, err);
    }
    if (ok) ++p.pool_steps;
    for (size_t b = 0; b < rows.size(); ++b) {
      PuncTicket* t = owner[b];
      if (!ok) { t->err = err; continue; }         // a failed step fails every call that had a window in it
      if (b == 0 || owner[b - 1] != t) ++t->steps;
      if (t->err.empty()) fa_punc::apply(p.vocab, *rows[b], p.step, (int32_t)b, t->err);
    }
  }
  for (PuncTicket* t : held) {
    if (!has_ended(*t)) continue;
    ended.push_back(t);
    if (t->err.empty()) finish(*t);
    t->texts.clear();
  }
  held.erase(std::remove_if(held.begin(), held.end(), [](const PuncTicket* t) { return has_ended(*t); }), held.end());
}

// fa_punc_init_host / fa_punc_walk_host: the caller's vocabulary, checked
bool host_vocab(const char* const* tokens, int32_t n_tokens, const char* const* punc_list, int32_t n_punc, int32_t sentence_end_id,
                int32_t split_size, fa_punc::Vocab& v) {
  std::string err;
  for (int32_t i = 0; i < n_tokens; ++i) if (!tokens[i]) { set_err("token " + std::to_string(i) + " is NULL"); return false; }
  for (int32_t i = 0; i < n_punc; ++i) if (!punc_list[i]) { set_err("punctuation " + std::to_string(i) + " is NULL"); return false; }
  std::vector<std::string> tok(tokens, tokens + n_tokens), pl(punc_list, punc_list + n_punc);
  return v.init(tok, pl, sentence_end_id, split_size, err) || (set_err(err), false);
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
  PuncTicket t;
  bool any = false;
  if (!no_throw("fa_punc_infer: ", [&] {
        t.texts.reserve((size_t)n);
        for (int32_t i = 0; i < n; ++i) {
          t.texts.push_back(fa_punc::admit(p->vocab, texts[i]));
          any = any || t.texts.back().active();
        }
        if (!any) finish(t);                                  // no window: "" and no ids, without the pool
        return true;
      }))
    return nullptr;
  if (!any) return t.res.release();
  p->pool.call(t, [&](std::deque<PuncTicket*>& queue, std::vector<PuncTicket*>& held) { admit_queued(*p, queue, held); },
               [&](std::vector<PuncTicket*>& held, std::vector<PuncTicket*>& ended) { run_step(*p, held, ended); }, "fa_punc_infer: ");
  if (!t.err.empty()) return fail(t.err);
  g_err.clear();
  return t.res.release();
}

extern "C" void* fa_punc_init_host(const char* const* tokens, int32_t n_tokens, const char* const* punc_list, int32_t n_punc,
                                   int32_t sentence_end_id, int32_t split_size, int64_t max_window, fa_punc_score_fn score_fn, void* ctx) {
  g_err.clear();
  if (!tokens || n_tokens < 1 || !punc_list || n_punc < 1 || !score_fn) return fail("bad argument");
  std::unique_ptr<Punc> p;
  const bool ok = no_throw("fa_punc_init_host: ", [&] {
    p.reset(new Punc());
    p->host_score = score_fn;
    p->host_ctx = ctx;
    p->max_window = max_window;
    return host_vocab(tokens, n_tokens, punc_list, n_punc, sentence_end_id, split_size, p->vocab);
  });
  return ok ? p.release() : nullptr;
}

extern "C" int fa_punc_pool_stats(const void* punc, int64_t* calls, int64_t* steps) {
  const Punc* p = static_cast<const Punc*>(punc);
  if (!p || !calls || !steps) return FA_ERR_ARG;
  *calls = p->pool.calls.load();
  *steps = p->pool_steps.load();
  return FA_OK;
}

extern "C" void* fa_punc_walk_host(const char* const* texts, int32_t n, const char* const* tokens, int32_t n_tokens, const char* const* punc_list,
                                   int32_t n_punc, int32_t sentence_end_id, int32_t split_size, int64_t max_window, fa_punc_score_fn score_fn,
                                   void* ctx) {
  g_err.clear();
  if ((!texts && n > 0) || n < 0 || !tokens || n_tokens < 1 || !punc_list || n_punc < 1 || !score_fn) return fail("bad argument");
  for (int32_t i = 0; i < n; ++i)
    if (!texts[i]) return fail("text " + std::to_string(i) + " is NULL");
  std::unique_ptr<fa_punc::Result> r(new fa_punc::Result());
  const bool ok = no_throw("fa_punc_walk_host: ", [&] {
    fa_punc::Vocab v;
    std::string err;
    const fa_punc::Scorer score = [&](const int32_t* ids, const int32_t* lens, int32_t B, int32_t T, int32_t* out, std::string& e) {
      const int32_t rc = score_fn(ctx, ids, lens, B, T, out);
      if (rc != 0) e = "scorer failed (" + std::to_string(rc) + ")";
      return rc == 0;
    };
    return host_vocab(tokens, n_tokens, punc_list, n_punc, sentence_end_id, split_size, v) &&
           (fa_punc::walk(v, texts, n, max_window, score, *r, err) || (set_err(err), false));
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
