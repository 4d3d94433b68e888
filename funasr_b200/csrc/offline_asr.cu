// Handle-style offline recogniser over the kernels of this library — the C-ABI counterpart of FunASR's C++ runtime surface
// (runtime/onnxruntime/include/funasrruntime.h:100-116: FunOfflineInit / FunOfflineInferBuffer / FunASRGetResult / FunASRFreeResult /
// FunOfflineUninit; its Paraformer::Forward is the same op chain with ONNX Runtime in the middle, runtime/onnxruntime/src/paraformer.cpp).
// No Python, no torch: weights come from one flat file written by funasr_b200/pack.py (tensors under FunASR's own state_dict names),
// device memory from cudaMalloc.
//
//   fa_offline_init         model file -> handle (weights to HBM, fp16 planes for the tensor-core GEMMs)
//   fa_offline_infer        batch of host PCM buffers (f32 in [-1,1] or s16le) -> result (greedy token ids per utterance)
//   fa_offline_result_*     accessors;  fa_offline_free_result / fa_offline_uninit
//                           a BiCifParaformer file (its upsampled CIF timestamp head) adds per-token [start_ms, end_ms] stamps
//   a SenseVoiceSmall file (__sv_config__) makes the same handle run SenseVoiceEngine's chain: per-utterance query rows
//                           (fa_sv_query_rows), the SAN-M and tp stacks, the CTC head; fa_offline_infer_sv
//   a SeacoParaformer file (__seaco_config__): fa_offline_hotword_embed runs its hotword encoder (hotword.cu), the decode takes those
//                           rows through _seaco_decode_with_ASF (seaco_bias)
// Long audio (VAD segments decoded in packs) is offline_long.cu.  The tokenizer (ids -> text) stays with the caller, like every other
// entry point of this ABI.
#include "handle.h"
#include "kernels.h"

using namespace fa_handle;

namespace {

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
    b.what = "BiCif timestamp head: ";
    bind_ts_head(b, 512, m.head);
    if (!b.ok) return false;
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
  m.dec.has_bias = m.contextual ? 1 : 0;                    // its hotword memories come with each pack (decode_batch)
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

// SeACo's hotword biasing after the decoder (_seaco_decode_with_ASF, seaco_paraformer/model.py:271-382, as ParaformerEngine.seaco_decode
// runs it) for every reference pack of a GPU pack.  The reference gives each of its batches one hotword memory: the batch's rows, or
// with more rows than nfilter the ones the attention-score filter (ASF) picks on the batch's utterance 0 over the batch's n_max query
// rows.  SeacoPlan lays out the pack's memories from the host token counts; seaco_bias runs them.
struct SeacoPlan {
  std::vector<int> probe;                            // the reference packs the ASF runs on, and their n_max
  std::vector<int32_t> probe_nmax;
  std::vector<int> probe_set;                        // the distinct sets they filter, and per probe its index there
  std::vector<int32_t> probe_group;
  int probe_nmax_all = 0, probe_rows = 0;            // the probe's query rows and memory length
  int groups = 0, rows_ub = 0;                       // the final memories and an upper bound of their length
  bool any = false;                                  // some reference pack has hotword rows
};

SeacoPlan seaco_plan(const Model& m, const PackHotwords& hw, const std::vector<int32_t>& tok_h) {
  SeacoPlan p;
  std::vector<char> plain_used(hw.n.size(), 0);
  for (const PackHotwords::Ref& r : hw.refs) {
    if (r.set < 0) continue;
    p.any = true;
    int nmax = 0;
    for (int i = r.first; i < r.first + r.count; ++i) nmax = std::max(nmax, tok_h[i]);
    const int n = hw.n[r.set];
    if (m.nfilter > 0 && m.nfilter < n && nmax > 0) {          // a batch without a token is never decoded (paraformer/model.py:615)
      const int k = (int)(std::find(p.probe_set.begin(), p.probe_set.end(), r.set) - p.probe_set.begin());
      if (k == (int)p.probe_set.size()) p.probe_set.push_back(r.set);
      p.probe.push_back((int)(&r - hw.refs.data()));
      p.probe_nmax.push_back(nmax);
      p.probe_group.push_back(k);
      p.probe_nmax_all = std::max(p.probe_nmax_all, nmax);
      p.probe_rows = std::max(p.probe_rows, n);
      ++p.groups;
      p.rows_ub = std::max(p.rows_ub, m.nfilter + 1);          // fa_seaco_asf_select_host keeps nfilter rows and <s>
    } else if (!plain_used[r.set]) {
      plain_used[r.set] = 1;
      ++p.groups;
      p.rows_ub = std::max(p.rows_ub, n);
    }
  }
  return p;
}

// The plan's memories over the GPU pack [B, n_max]: the ASF probes in one batched forward (the first row of each filtered reference pack,
// gathered, each against its own set), one host round trip, each pack's [heads, n_max_ref, n] block cut out for fa_seaco_asf_select_host,
// one upload of every memory; then the SeACo decoder over the acoustic embeddings and over the decoder's hidden states, each row against
// its reference pack's memory; hotword_output_layer's arg-max over their sum; the NO_BIAS merge of the decoder's ids / best into *sids.
// Rows of a reference pack without rows keep the decoder's ids (model.py:381-382).  The workspace is sized for every stage by the caller.
bool seaco_bias(Model& m, const SeacoPlan& plan, const PackHotwords& hw, const std::vector<int32_t>& tok_h, int B, int n_max, int n_cap,
                const float* acoustic, const float* hidden, const int32_t* tok, const int32_t* ids, const float* best, int32_t** sids) {
  cudaStream_t st = m.file.st;
  const int D = m.d_model, V = m.vocab, n_s = m.seaco_dec.n_layers, H = m.seaco_dec.heads;
  const int64_t rows = (int64_t)B * n_max;
  const int R = (int)plan.probe.size(), Gp = (int)plan.probe_set.size(), NP = plan.probe_rows, QP = plan.probe_nmax_all;
  const int G = plan.groups, NU = plan.rows_ub;
  float *mem, *cif_att, *dec_att, *dha_best, *sbest, *probs = nullptr, *mem_p = nullptr, *hx = nullptr;
  int32_t *dha_ids, *tok_p = nullptr, *rows_f;
  if (!carve(m.seaco_bias, "SeACo", [&](fa::Arena& a) {
        mem = a.take<float>((size_t)G * NU * D);
        cif_att = a.take<float>((size_t)rows * D); dec_att = a.take<float>((size_t)rows * D);
        dha_ids = a.take<int32_t>(rows); dha_best = a.take<float>(rows);
        *sids = a.take<int32_t>(rows); sbest = a.take<float>(rows);
        rows_f = a.take<int32_t>((size_t)2 * B);
        if (R > 0) {
          mem_p = a.take<float>((size_t)Gp * NP * D); hx = a.take<float>((size_t)R * n_max * D); tok_p = a.take<int32_t>(R);
          probs = a.take<float>((size_t)R * H * QP * NP);
        }
      }))
    return false;
  // each reference pack's memory: the picked rows of a filtered one, its set's rows (one copy per set) otherwise
  std::vector<std::vector<float>> picked(hw.refs.size());
  int rc = FA_OK;
  std::vector<float> host_p;
  std::vector<int32_t> lens_p(Gp), tok_ph(R), seq(R);
  if (R > 0) {
    host_p.assign((size_t)Gp * NP * D, 0.f);              // rows past a set's length are zeros: their projections are the bias
    for (int g = 0; g < Gp; ++g) {
      const int s = plan.probe_set[g];
      lens_p[g] = hw.n[s];
      std::copy(hw.rows[s], hw.rows[s] + (size_t)hw.n[s] * D, host_p.begin() + (size_t)g * NP * D);
    }
    for (int k = 0; k < R; ++k) {
      const int first = hw.refs[plan.probe[k]].first;
      tok_ph[k] = tok_h[first];
      seq[k] = k;
      cudaMemcpyAsync(hx + (size_t)k * n_max * D, hidden + (size_t)first * n_max * D, (size_t)n_max * D * 4, cudaMemcpyDeviceToDevice, st);
    }
    cudaMemcpyAsync(mem_p, host_p.data(), host_p.size() * 4, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(tok_p, tok_ph.data(), (size_t)R * 4, cudaMemcpyHostToDevice, st);
    rc = fa_sanm_decoder_stack_forward_grouped(&m.seaco_dec, mem_p, lens_p.data(), plan.probe_group.data(), Gp, R, NP, hx, n_max, tok_p, QP, 6, 0,
                                               nullptr, probs, seq.data(), R, m.mode, m.ws.p, m.ws.cap, st);
    if (rc != FA_OK) { set_err(std::string("SeACo filter: ") + fa_status_string(rc)); return false; }
    std::vector<float> probs_h((size_t)R * H * QP * NP);
    cudaMemcpyAsync(probs_h.data(), probs, probs_h.size() * 4, cudaMemcpyDeviceToHost, st);
    if (!sync_stream(st)) return false;
    for (int k = 0; k < R; ++k) {                          // the reference pack's own [heads, n_max_ref, n] block
      const int s = plan.probe_set[plan.probe_group[k]], n = hw.n[s], q = plan.probe_nmax[k];
      std::vector<float> blk((size_t)H * q * n);
      for (int h = 0; h < H; ++h)
        for (int i = 0; i < q; ++i)
          std::copy_n(probs_h.begin() + (((size_t)k * H + h) * QP + i) * NP, n, blk.begin() + ((size_t)h * q + i) * n);
      std::vector<int32_t> pick((size_t)n);
      const int n_sel = fa_seaco_asf_select_host(blk.data(), H, q, n, m.nfilter, pick.data());
      if (n_sel < 1) { set_err("fa_seaco_asf_select_host failed"); return false; }
      std::vector<float>& out = picked[plan.probe[k]];
      out.resize((size_t)n_sel * D);
      for (int j = 0; j < n_sel; ++j) std::copy_n(hw.rows[s] + (size_t)pick[j] * D, D, out.begin() + (size_t)j * D);
    }
  }
  // the final memories, one upload; every row's memory (a row without rows reads memory 0 and keeps the decoder's ids)
  std::vector<int32_t> lens_f, group_row(B, 0), set_group(hw.n.size(), -1);
  int nf = 1;
  for (size_t k = 0; k < hw.refs.size(); ++k) {
    const PackHotwords::Ref& r = hw.refs[k];
    if (r.set >= 0) nf = std::max(nf, picked[k].empty() ? hw.n[r.set] : (int)(picked[k].size() / D));
  }
  std::vector<float> host_f;
  host_f.reserve((size_t)G * nf * D);
  for (size_t k = 0; k < hw.refs.size(); ++k) {
    const PackHotwords::Ref& r = hw.refs[k];
    if (r.set < 0) continue;
    int g = set_group[r.set];
    if (!picked[k].empty() || g < 0) {
      g = (int)lens_f.size();
      const float* src = picked[k].empty() ? hw.rows[r.set] : picked[k].data();
      const int n = picked[k].empty() ? hw.n[r.set] : (int)(picked[k].size() / D);
      if (picked[k].empty()) set_group[r.set] = g;
      lens_f.push_back(n);
      host_f.insert(host_f.end(), src, src + (size_t)n * D);
      host_f.resize((size_t)(g + 1) * nf * D, 0.f);
    }
    std::fill(group_row.begin() + r.first, group_row.begin() + r.first + r.count, g);
  }
  // every row's [key count | memory], uploaded beside the memories: the two stacks below then copy nothing between their launches
  std::vector<int32_t> rows_h((size_t)2 * B);
  for (int b = 0; b < B; ++b) { rows_h[b] = lens_f[group_row[b]]; rows_h[B + b] = group_row[b]; }
  cudaMemcpyAsync(mem, host_f.data(), host_f.size() * 4, cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(rows_f, rows_h.data(), rows_h.size() * 4, cudaMemcpyHostToDevice, st);
  const int Gf = (int)lens_f.size();
  rc = fa::sanm_stack_grouped_dev(&m.seaco_dec, mem, rows_f, Gf, B, nf, acoustic, n_cap, tok, n_max, n_s, cif_att, m.mode, m.ws.p, m.ws.cap, st);
  if (rc == FA_OK)
    rc = fa::sanm_stack_grouped_dev(&m.seaco_dec, mem, rows_f, Gf, B, nf, hidden, n_max, tok, n_max, n_s, dec_att, m.mode, m.ws.p, m.ws.cap, st);
  if (rc == FA_OK) rc = fa_linear_argmax(&m.hw_out, cif_att, dec_att, rows, dha_ids, dha_best, nullptr, m.mode, m.ws.p, m.ws.cap, st);
  if (rc == FA_OK) rc = fa_seaco_merge(ids, best, dha_ids, dha_best, rows, m.no_bias, *sids, sbest, nullptr, nullptr, nullptr, V, st);
  if (rc != FA_OK) { set_err(std::string("SeACo decoder: ") + fa_status_string(rc)); return false; }
  for (const PackHotwords::Ref& r : hw.refs)
    if (r.set < 0)
      cudaMemcpyAsync(*sids + (size_t)r.first * n_max, ids + (size_t)r.first * n_max, (size_t)r.count * n_max * 4, cudaMemcpyDeviceToDevice, st);
  return sync_stream(st);                                    // the host vectors above are this frame's
}

// the workspace of seaco_bias's stages
size_t seaco_ws_bytes(const Model& m, const SeacoPlan& p, int B, int n_max) {
  const int R = (int)p.probe.size();
  size_t ws = std::max(fa_sanm_decoder_stack_grouped_workspace_bytes(B, p.groups, p.rows_ub, n_max, 0, m.mode),
                       fa_linear_argmax_workspace_bytes((int64_t)B * n_max, m.vocab, m.mode));
  if (R > 0)
    ws = std::max(ws, fa_sanm_decoder_stack_grouped_workspace_bytes(R, (int)p.probe_set.size(), p.probe_rows, p.probe_nmax_all, R, m.mode));
  return ws;
}

// The recogniser over a padded batch already on the device: wav [B, stride] fp32, lens_h [B] samples (>= 400 each), ext_h [B] each
// row's padded length in frames (decode_pack).  Everything after the pool gathered the pack's rows.
std::unique_ptr<Result> decode_batch(Model& m, const float* wav, int64_t stride, const std::vector<int32_t>& lens_h, const std::vector<int32_t>& ext_h,
                                     const PackHotwords* hwp) {
  const int B = (int)lens_h.size(), D = m.d_model;
  cudaStream_t st = m.file.st;
  int t_max = 0;
  double seconds = 0.0;
  std::vector<int32_t> fl_h(B);                              // encoder lengths, the host copy the _ext entries check ext_h against
  for (int i = 0; i < B; ++i) {
    const int t = num_lfr_frames(lens_h[i]);
    fl_h[i] = t;
    t_max = t > t_max ? t : t_max;
    seconds += (double)lens_h[i] / 16000.0;
  }
  const int T = t_max;
  const int n_cap = T + 1;
  int32_t *lens, *flens, *tok;
  float *feats, *encb, *acoustic, *alphas, *peaks;
  if (!carve(m.encode, "activations", [&](fa::Arena& a) {
        lens = a.take<int32_t>(B); flens = a.take<int32_t>(B); tok = a.take<int32_t>(B);
        feats = a.take<float>((size_t)B * T * m.feat_dim); encb = a.take<float>((size_t)B * T * D);
        acoustic = a.take<float>((size_t)B * n_cap * D);
        alphas = a.take<float>((size_t)B * n_cap); peaks = a.take<float>((size_t)B * n_cap);
      }))
    return nullptr;
  cudaMemcpyAsync(lens, lens_h.data(), (size_t)B * 4, cudaMemcpyHostToDevice, st);
  size_t ws = fa_sanm_encoder_workspace_bytes(B, T, m.mode);
  const size_t ws2 = fa_cif_predictor_ext_workspace_bytes(B, T, m.mode);
  ws = ws2 > ws ? ws2 : ws;
  if (!m.ws.reserve(ws)) return fail("device allocation failed (workspace)");
  int rc = fa_fbank_lfr_cmvn_tables(wav, lens, B, stride, m.cmvn, m.file.fbank_tables, 7, 6, feats, T, flens, T, st);
  if (rc != FA_OK) return fail(std::string("fa_fbank_lfr_cmvn_tables: ") + fa_status_string(rc));
  rc = fa_sanm_encoder_forward(&m.enc, feats, flens, B, T, encb, m.mode, m.ws.p, m.ws.cap, st);
  if (rc != FA_OK) return fail(std::string("fa_sanm_encoder_forward: ") + fa_status_string(rc));
  rc = fa_cif_predictor_forward_ext(&m.pred, encb, flens, B, T, acoustic, n_cap, tok, alphas, peaks, m.mode, m.ws.p, m.ws.cap, st, fl_h.data(),
                                    ext_h.data());
  if (rc != FA_OK) return fail(std::string("fa_cif_predictor_forward: ") + fa_status_string(rc));
  std::unique_ptr<Result> r(new Result());
  r->audio_seconds = (float)seconds;
  r->token_num.resize(B);
  r->ts = m.ts;
  if (m.ts) r->stamps.resize(B);
  cudaMemcpyAsync(r->token_num.data(), tok, (size_t)B * 4, cudaMemcpyDeviceToHost, st);
  if (!sync_stream(st)) return nullptr;
  int n_max = 0;                                             // the path's one host sync (cif_predictor.py:311)
  for (int i = 0; i < B; ++i) n_max = r->token_num[i] > n_max ? r->token_num[i] : n_max;
  r->ids.resize(B);
  if (n_max < 1) return r;                                   // paraformer/model.py:615-616
  // the timestamp head over the [B, 3T] upsampled frames shares the workspace with the decoder
  const int U = m.head.up_times, TU = T * U;
  const int64_t rows_up = (int64_t)B * TU;
  // contextual: the pack's distinct hotword sets as memories [G, nh_max, 512], zero rows past a set's length (contextual_paraformer/
  // model.py:350-372); every row's memory is its reference pack's
  std::vector<float> hw_h;
  std::vector<int32_t> hw_lens_h, hw_row_h(B, 0);
  int nh_max = 0;
  if (m.contextual && hwp) {
    for (int32_t n : hwp->n) nh_max = std::max(nh_max, n);
    hw_lens_h = hwp->n;
    hw_h.assign(hwp->n.size() * (size_t)nh_max * D, 0.f);
    for (size_t g = 0; g < hwp->n.size(); ++g) std::copy_n(hwp->rows[g], (size_t)hwp->n[g] * D, hw_h.begin() + g * nh_max * D);
    for (const PackHotwords::Ref& r : hwp->refs) std::fill(hw_row_h.begin() + r.first, hw_row_h.begin() + r.first + r.count, r.set);
  }
  const int G = (int)hw_lens_h.size();
  const SeacoPlan sp = m.seaco && hwp ? seaco_plan(m, *hwp, r->token_num) : SeacoPlan();
  size_t ws_dec = G > 0 ? fa_paraformer_decoder_grouped_workspace_bytes(B, T, n_max, m.vocab, m.mode, G, nh_max)
                        : fa_paraformer_decoder_workspace_bytes_hw(B, T, n_max, m.vocab, m.mode, 0);
  if (m.ts) ws_dec = std::max(ws_dec, fa_timestamp_head_ext_workspace_bytes(B, T, D, U, m.mode));
  if (sp.any) ws_dec = std::max(ws_dec, seaco_ws_bytes(m, sp, B, n_max));
  int32_t *ids, *fids, *flens_out;
  float *best, *us_alphas = nullptr, *us_peaks = nullptr, *hw = nullptr, *hidden = nullptr;
  if (!carve(m.decode, "decoder", [&](fa::Arena& a) {
        ids = a.take<int32_t>((size_t)B * n_max); best = a.take<float>((size_t)B * n_max); fids = a.take<int32_t>((size_t)B * n_max);
        flens_out = a.take<int32_t>(B);
        if (m.ts) { us_alphas = a.take<float>(rows_up); us_peaks = a.take<float>(rows_up); }
        if (G > 0) hw = a.take<float>(hw_h.size());
        if (m.seaco) hidden = a.take<float>((size_t)B * n_max * D);
      }))
    return nullptr;
  if (!m.ws.reserve(ws_dec)) return fail("device allocation failed (decoder)");
  if (G > 0) cudaMemcpyAsync(hw, hw_h.data(), hw_h.size() * 4, cudaMemcpyHostToDevice, st);
  const int32_t* final_ids = ids;
  if (m.seaco) {                                             // return_hidden: the decoder_hidden the SeACo decoder attends from
    rc = fa_paraformer_decoder_forward_hidden(&m.dec, encb, flens, B, T, acoustic, n_cap, tok, n_max, ids, best, nullptr, 1, hidden, m.mode,
                                              m.ws.p, m.ws.cap, st);
    if (rc == FA_OK && sp.any) {
      int32_t* sids = nullptr;
      if (!seaco_bias(m, sp, *hwp, r->token_num, B, n_max, n_cap, acoustic, hidden, tok, ids, best, &sids)) return nullptr;
      final_ids = sids;
    }
  } else if (G > 0) {
    rc = fa_paraformer_decoder_forward_grouped(&m.dec, encb, flens, B, T, acoustic, n_cap, tok, n_max, ids, best, nullptr, 1, nullptr, hw,
                                               hw_lens_h.data(), hw_row_h.data(), G, nh_max, m.mode, m.ws.p, m.ws.cap, st);
  } else {
    rc = fa_paraformer_decoder_forward(&m.dec, encb, flens, B, T, acoustic, n_cap, tok, n_max, ids, best, nullptr, 1, m.mode, m.ws.p, m.ws.cap, st);
  }
  if (rc == FA_OK) rc = fa_greedy_filter(final_ids, tok, B, n_max, 1, 2, 0, fids, flens_out, st);
  if (rc != FA_OK) return fail(std::string("decoder: ") + fa_status_string(rc));
  if (m.ts) {                   // CifPredictorV3.get_upsample_timestamp (bicif_paraformer/cif_predictor.py:300-352), engine.upsample_timestamp
    rc = fa_timestamp_head_forward_ext(&m.head, encb, flens, tok, B, T, us_alphas, us_peaks, m.mode, m.ws.p, m.ws.cap, st, fl_h.data(), ext_h.data());
    if (rc != FA_OK) return fail(std::string("timestamp head: ") + fa_status_string(rc));
  }
  std::vector<int32_t> fids_h((size_t)B * n_max), fl(B), enc_lens(m.ts ? B : 0);
  std::vector<float> us_alphas_h(m.ts ? rows_up : 0), us_peaks_h(m.ts ? rows_up : 0);
  cudaMemcpyAsync(fids_h.data(), fids, fids_h.size() * 4, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(fl.data(), flens_out, (size_t)B * 4, cudaMemcpyDeviceToHost, st);
  if (m.ts) {                                                // on the same synchronisation as the ids
    cudaMemcpyAsync(enc_lens.data(), flens, (size_t)B * 4, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(us_alphas_h.data(), us_alphas, (size_t)rows_up * 4, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(us_peaks_h.data(), us_peaks, (size_t)rows_up * 4, cudaMemcpyDeviceToHost, st);
  }
  if (!sync_stream(st)) return nullptr;
  for (int i = 0; i < B; ++i) r->ids[i].assign(fids_h.begin() + (size_t)i * n_max, fids_h.begin() + (size_t)i * n_max + fl[i]);
  if (m.ts) {                                                // bicif_paraformer/model.py:402-407: each utterance's first 3 * enc_len frames
    for (int i = 0; i < B; ++i) {
      const int64_t n = (int64_t)U * enc_lens[i];
      std::vector<int32_t>& sp = r->stamps[i];
      sp.resize((size_t)(2 * (n > 0 ? n : 1)));              // at most n - 1 spans
      const int64_t k = fa_ts_stamps_host(us_alphas_h.data() + (size_t)i * TU, us_peaks_h.data() + (size_t)i * TU, n, (int64_t)r->ids[i].size(), U,
                                          0.0, sp.data(), n);
      sp.resize(k > 0 ? (size_t)(2 * k) : 0);
    }
  }
  return r;
}

// ------------------------------------------------------------------------------------------------ SenseVoiceSmall
// __sv_config__ of funasr_b200/pack.py:write_sensevoice_model_file
enum { kSvEnc = 0, kSvTp, kSvDModel, kSvHeads, kSvKernel, kSvVocab, kSvFeat, kSvEps, kSvBlank, kSvCfgLen };

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
  int32_t *io_d, *flens, *am, *ids, *flens_out;
  float *x, *enc, *enc2;
  if (!carve(m.decode_sv, "SenseVoice", [&](fa::Arena& a) {
        io_d = a.take<int32_t>(io.size()); flens = a.take<int32_t>(B);
        x = a.take<float>(rows * F); enc = a.take<float>(rows * D); enc2 = a.take<float>(rows * D);
        am = a.take<int32_t>(rows); ids = a.take<int32_t>(rows); flens_out = a.take<int32_t>(B);
      }))
    return nullptr;
  if (!m.ws.reserve(ws)) return fail("device allocation failed (SenseVoice)");
  cudaMemcpyAsync(io_d, io.data(), io.size() * 4, cudaMemcpyHostToDevice, st);
  int rc = fa_fbank_lfr_cmvn_tables(wav, io_d, B, stride, m.cmvn, m.file.fbank_tables, 7, 6, x + 4 * F, T, flens, t_feat, st);
  if (rc == FA_OK) rc = fa_sv_query_rows(m.embed, m.n_embed, F, io_d + 2 * B, B, x, T, st);
  if (rc == FA_OK) rc = fa_sanm_encoder_forward(&m.enc, x, io_d + B, B, T, enc, m.mode, m.ws.p, m.ws.cap, st);
  if (rc == FA_OK && m.tp_layers > 0) {
    rc = fa_sanm_encoder_forward(&m.tp, enc, io_d + B, B, T, enc2, m.mode, m.ws.p, m.ws.cap, st);
    enc = enc2;
  }
  if (rc == FA_OK) rc = fa_ctc_greedy_forward(&m.ctc, enc, io_d + B, B, T, m.blank, am, ids, flens_out, nullptr, m.mode, m.ws.p, m.ws.cap, st);
  if (rc != FA_OK) return fail(std::string("SenseVoice: ") + fa_status_string(rc));
  std::unique_ptr<Result> r(new Result());
  r->audio_seconds = (float)seconds;
  r->token_num.resize(B);
  r->ids.resize(B);
  std::vector<int32_t> ids_h(rows);
  cudaMemcpyAsync(ids_h.data(), ids, rows * 4, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(r->token_num.data(), flens_out, (size_t)B * 4, cudaMemcpyDeviceToHost, st);
  if (!sync_stream(st)) return nullptr;
  for (int i = 0; i < B; ++i) r->ids[i].assign(ids_h.begin() + (size_t)i * T, ids_h.begin() + (size_t)i * T + r->token_num[i]);
  return r;
}

// fa_offline_infer_hw / fa_offline_infer_sv / fa_offline_infer_audio: the call checked on its own thread, then decoded through the
// request pool as one reference pack (the whole batch, as the reference decodes it)
void* infer_batch(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, const FaAudioFormat* fmt, const float* hw_embed,
                  int32_t n_hotwords, const int32_t* lang, const int32_t* tn) {
  Model* mp = static_cast<Model*>(handle);
  if (!mp || !bufs || !n_samples || batch <= 0) return fail("bad argument");
  Model& m = *mp;
  Ticket t;
  if (!plan_audio(fmt, m.resample, t.au)) return nullptr;
  if (!check_hotword_rows(m, hw_embed, n_hotwords)) return nullptr;
  if (m.sv && !check_queries(m, lang, tn, batch, "utterance")) return nullptr;
  t.n16.resize(batch);
  for (int i = 0; i < batch; ++i) {
    const int64_t n16 = bufs[i] && n_samples[i] >= 0 && n_samples[i] <= 0x7fffffffLL ? t.au.len16(n_samples[i]) : 0;
    if (n16 < 400 || n16 > 0x7fffffffLL) return fail("every buffer needs >= 400 samples (25 ms)" + t.au.at16k());
    t.n16[i] = n16;
  }
  t.bufs = bufs; t.n_samples = n_samples; t.batch = batch;
  t.hw_embed = hw_embed; t.n_hotwords = n_hotwords; t.lang = lang; t.tn = tn;
  return pool_call(m, t);
}

// the model kind is the file's: SenseVoiceSmall by __sv_config__, Paraformer otherwise; a MonotonicAligner file is fa_align_init's
bool build_offline(Model& m, Builder& b) {
  if (b.opt("__aligner_config__")) return b.refuse("a MonotonicAligner file (__aligner_config__): open it with fa_align_init");
  return b.opt("__sv_config__") ? build_sv(m, b) : build_paraformer(m, b);
}

const Result* as_result(const void* r) { return static_cast<const Result*>(r); }

}  // namespace

namespace fa_handle {

bool check_hotword_rows(const Model& m, const float* hw_embed, int32_t n_hotwords) {
  if (m.contextual && (!hw_embed || n_hotwords < 1)) {
    set_err("this model has a hotword bias decoder: pass hotword embeddings (at least the <s> entry)");
    return false;
  }
  if (m.seaco && (n_hotwords < 0 || (n_hotwords > 0 && !hw_embed))) {
    set_err("bad hotword rows: hw_embed must hold n_hotwords rows of 512");
    return false;
  }
  return true;
}

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

std::unique_ptr<Result> decode_pack(Model& m, const float* wav, int64_t stride, const std::vector<int32_t>& lens_h, const std::vector<int32_t>& ext_h,
                                    const PackHotwords* hw, const int32_t* lang, const int32_t* tn) {
  // SenseVoice has no CIF predictor: its rows read nothing past their own length
  return m.sv ? decode_sv(m, wav, stride, lens_h, lang, tn) : decode_batch(m, wav, stride, lens_h, ext_h, hw);
}

}  // namespace fa_handle

extern "C" void* fa_offline_init(const char* model_file, int32_t device, int32_t gemm_mode) {
  g_err.clear();
  if (!model_file) return fail("model_file is NULL");
  if (!valid_gemm_mode(gemm_mode)) return fail("bad gemm_mode");
  return open_handle(model_file, device, gemm_mode, build_offline);
}

extern "C" int32_t fa_offline_is_sensevoice(const void* handle) { return handle && static_cast<const Model*>(handle)->sv ? 1 : 0; }

extern "C" void* fa_offline_infer_sv(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                                     const int32_t* language_ids, const int32_t* textnorm_ids) {
  g_err.clear();
  if (handle && !static_cast<Model*>(handle)->sv) return fail("fa_offline_infer_sv: not a SenseVoice model file");
  FaAudioFormat f;
  if (!pcm16k_format(pcm_format, f)) return fail("bad argument");
  return infer_batch(handle, bufs, n_samples, batch, &f, nullptr, 0, language_ids, textnorm_ids);
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
  std::lock_guard<std::mutex> dev(m->mu);
  cudaSetDevice(m->file.device);
  cudaStream_t st = m->file.st;
  const size_t ws = fa_hotword_encoder_workspace_bytes(n, n_tok, m->mode);
  float* rows = nullptr;
  if (ws == 0 || !m->ws.reserve(ws)) { set_err("device allocation failed (hotword encoder)"); return FA_ERR_CUDA; }
  if (!carve(m->hotword_embed, "hotword encoder", [&](fa::Arena& a) { rows = a.take<float>((size_t)n * m->d_model); })) return FA_ERR_CUDA;
  const int rc = fa_hotword_encoder_forward(&m->hw_enc, ids, lens, n, rows, m->mode, m->ws.p, m->ws.cap, st);
  if (rc != FA_OK) { set_err(std::string("fa_hotword_encoder_forward: ") + fa_status_string(rc)); return rc; }
  cudaMemcpyAsync(rows_host, rows, (size_t)n * m->d_model * 4, cudaMemcpyDeviceToHost, st);
  return sync_stream(st) ? FA_OK : FA_ERR_CUDA;
}

extern "C" const float* fa_offline_host_tensor(void* handle, const char* name, int64_t* numel) {
  Model* m = static_cast<Model*>(handle);
  if (numel) *numel = 0;
  if (!m || !name) return nullptr;
  auto it = m->file.t.find(name);
  if (it == m->file.t.end()) return nullptr;
  const Tensor& t = it->second;
  std::lock_guard<std::mutex> lock(m->host_cache_mu);
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

extern "C" void* fa_offline_infer_hw(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                                     const float* hw_embed, int32_t n_hotwords) {
  g_err.clear();
  FaAudioFormat f;
  if (!pcm16k_format(pcm_format, f)) return fail("bad argument");
  return infer_batch(handle, bufs, n_samples, batch, &f, hw_embed, n_hotwords, nullptr, nullptr);
}

extern "C" void* fa_offline_infer_audio(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, const FaAudioFormat* fmt,
                                        const float* hw_embed, int32_t n_hotwords, const int32_t* language_ids, const int32_t* textnorm_ids) {
  g_err.clear();
  if (handle && !static_cast<Model*>(handle)->sv && (language_ids || textnorm_ids))
    return fail("fa_offline_infer_audio: language / text-norm ids need a SenseVoice model file");
  return infer_batch(handle, bufs, n_samples, batch, fmt, hw_embed, n_hotwords, language_ids, textnorm_ids);
}

extern "C" void* fa_offline_infer(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format) {
  return fa_offline_infer_hw(handle, bufs, n_samples, batch, pcm_format, nullptr, 0);
}

extern "C" int32_t fa_offline_result_count(const void* result) { return result ? (int32_t)as_result(result)->ids.size() : 0; }

// an empty row is still a row: its (possibly NULL) data with *n_ids = 0
extern "C" const int32_t* fa_offline_result_ids(const void* result, int32_t index, int32_t* n_ids) {
  return result_row(result ? &as_result(result)->ids : nullptr, index, n_ids, 1, true);
}

extern "C" float fa_offline_result_audio_seconds(const void* result) { return result ? as_result(result)->audio_seconds : 0.f; }

extern "C" const int32_t* fa_offline_result_stamps(const void* result, int32_t index, int32_t* n_stamps) {
  return result_row(result && as_result(result)->ts ? &as_result(result)->stamps : nullptr, index, n_stamps, 2, false);
}

extern "C" void fa_offline_free_result(void* result) { delete static_cast<Result*>(result); }
