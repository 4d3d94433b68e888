// Handle-style CAM++ speaker model: fa_spk_init (model file -> handle, the BatchNorms folded on the host), fa_spk_embed (host PCM ->
// 192-dim embeddings), fa_spk_cluster (ClusterBackend over host embeddings), and diarize, which the recogniser's request pool
// (offline_pool.cu) runs once over a group's diarized recordings already on the device.
//
// Speaker-only calls share passes through the handle's own request pool (request_pool.h): a call checks its arguments on its own
// thread and posts a ticket; each round of the pool's leader is one pass over the queued calls (arrival order, up to an hour of padded
// audio and kPoolClusterRows clustering rows), and every call of a pass ends with it.  Each call gets exactly what it gets alone: an
// embedding row carries its call's padded length (fa_campplus_forward_ext), and each clustering call is one set of spk_cluster.
#include "handle.h"
#include <math.h>

using namespace fa_handle;

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
const int64_t kPoolSamples = 3600LL * 16000;        // padded 16 kHz samples of the embedding calls one pass takes (230 MB of fp32 rows)
// clustering rows one pass takes: spectral sets are under 2048 rows each, so at most 2047 * 8192 doubles (134 MB) of Laplacians
const int64_t kPoolClusterRows = 8192;
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

// The BatchNorm folding of CampplusEngine (campplus.py: _bn, _folded, conv2d) on the host in float64 — the same IEEE multiplies,
// divisions and square roots, then one rounding to fp32 — so the folded weights are bit-identical to the Python engine's.  Runs on the
// loaded file only (b.f).
struct CamFolder {
  Builder& b;
  std::vector<float> host(const std::string& k) {
    const Tensor* t = b.get(k);
    std::vector<float> h(t ? (size_t)t->numel() : 0);
    if (t && !h.empty() && cudaMemcpy(h.data(), t->dev, h.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess) b.refuse("copy of " + k + " failed");
    return h;
  }
  const float* up(const std::vector<double>& v) {
    std::vector<float> h(v.begin(), v.end());
    void* p = b.f->alloc((h.size() ? h.size() : 1) * 4);
    if (!p) { b.refuse("cudaMalloc failed"); return nullptr; }
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
    if (b.mode != FA_GEMM_F32_SIMT && b.ok) b.split_planes(L);
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
  CamFolder F{b};
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
// fa_campplus_features with t_max frames, then fa_campplus_forward in slices of CampplusEngine.embed_feats' workspace cap, or
// fa_campplus_forward_ext with each row's padded length ext_h [B] (host, <= t_max)
bool spk_embed_rows(Spk& s, const float* wav, int64_t stride, const int32_t* lens_d, int B, int t_max, float* emb,
                    const int32_t* ext_h = nullptr) {
  cudaStream_t st = s.file.st;
  const size_t per = fa_campplus_workspace_bytes(&s.model, 1, t_max, s.mode);
  if (per == 0) { set_err("CAM++ takes 2 ... 18800 feature frames per input (got " + std::to_string(t_max) + ")"); return false; }
  const int step = (int)std::max<size_t>(1, std::min<size_t>((size_t)B, kSpkWorkspaceCap / per));
  const size_t ws_bytes = ext_h ? fa_campplus_ext_workspace_bytes(&s.model, step, t_max, s.mode)
                                : fa_campplus_workspace_bytes(&s.model, step, t_max, s.mode);
  float* feats;
  int32_t* flens;
  void* ws;
  if (!carve(s.spk_embed_rows, "CAM++", [&](fa::Arena& a) {
        feats = a.take<float>((size_t)B * t_max * 80); flens = a.take<int32_t>(B); ws = a.take<char>(ws_bytes);
      }))
    return false;
  int rc = fa_campplus_features(wav, lens_d, B, stride, s.file.fbank_tables, feats, flens, t_max, st);
  for (int b0 = 0; b0 < B && rc == FA_OK; b0 += step) {
    const int nb = std::min(step, B - b0);
    const float* f = feats + (size_t)b0 * t_max * 80;
    float* e = emb + (size_t)b0 * kSpkEmbDim;
    rc = ext_h ? fa_campplus_forward_ext(&s.model, f, nb, t_max, e, s.mode, ws, ws_bytes, st, ext_h + b0)
               : fa_campplus_forward(&s.model, f, nb, t_max, e, s.mode, ws, ws_bytes, st);
  }
  if (rc != FA_OK) { set_err(std::string("CAM++: ") + fa_status_string(rc)); return false; }
  return true;
}

// ClusterBackend's refusals for n chunks, in its order (empty: none): fewer than 20 chunks are one speaker whatever the preset; from 20
// up a preset above the chunk count, and 2048 or more chunks without one (the reference's UMAP + HDBSCAN path), are refused
std::string cluster_refusal(int n, int preset, const std::string& what) {
  if (n < 20) return std::string();
  if (preset > n) return what + "preset_spk_num " + std::to_string(preset) + " exceeds the " + std::to_string(n) + " speaker chunks";
  if (n >= kSpectralMaxChunks && preset <= 0)
    return what + std::to_string(n) + " speaker chunks without preset_spk_num: the reference clusters 2048 or more chunks with UMAP + "
           "HDBSCAN, which this backend does not provide; pass preset_spk_num or diarize fewer than 2048 chunks";
  return std::string();
}

// One embedding set of spk_cluster: n rows from row `first` of the embeddings, its preset count (<= 0: none) -> labels (before
// correct_labels), or its own refusal in err
struct ClusterSet {
  int first = 0, n = 0, preset = 0;
  std::string what;                                  // prefix of its messages
  std::vector<int32_t> labels;
  std::string err;
};

// ClusterBackend over every set of the embeddings emb_d [rows, 192] on the device (emb_h: the same on the host).  Fewer than 20 rows ->
// one speaker; fewer than 2048 -> the spectral path, every such set together (one fa_spk_laplacian_batch and fa_spk_tridiagonalize_batch,
// one copy of d / e to the host, the 16 smallest eigenvalues and the eigengap count unless preset per set on the host, one upload of
// the eigenvectors, one fa_spk_back_transform_batch and one copy back), then k-means on the back-transformed vectors; otherwise k-means
// on the normalised rows with a preset count; merge_by_cos when no count was preset.  false: a device failure.
bool spk_cluster(Spk& s, const float* emb_d, const float* emb_h, std::vector<ClusterSet>& sets) {
  cudaStream_t st = s.file.st;
  std::vector<int> spectral;
  for (size_t i = 0; i < sets.size(); ++i) {
    ClusterSet& c = sets[i];
    c.labels.assign((size_t)c.n, 0);
    c.err = cluster_refusal(c.n, c.preset, c.what);
    if (c.n >= 20 && c.err.empty() && c.n < kSpectralMaxChunks) spectral.push_back((int)i);
  }
  std::vector<std::vector<double>> x(sets.size());
  std::vector<int> dims(sets.size(), 0), ks(sets.size(), 0);
  if (!spectral.empty()) {
    const int S = (int)spectral.size();
    std::vector<int32_t> n((size_t)S), k((size_t)S);
    std::vector<int64_t> vo((size_t)S + 1, 0), zo((size_t)S + 1, 0);
    bool contiguous = true;
    for (int i = 0; i < S; ++i) {
      const ClusterSet& c = sets[spectral[i]];
      n[i] = c.n;
      k[i] = std::max(std::min(kMaxSpks + 1, c.n), c.preset);          // the vectors the set may ask for: max(m, preset)
      vo[i + 1] = vo[i] + c.n;
      zo[i + 1] = zo[i] + (int64_t)k[i] * c.n;
      contiguous = contiguous && c.first == sets[spectral[0]].first + vo[i];
    }
    const int64_t rows = vo[S];
    // Every set has at most 2047 rows, so sum n^2 <= 2047 sum n: a long-audio group (an hour of padded audio, under 4 800 chunks)
    // needs at most 79 MB of Laplacians and no further split.
    const size_t ws_bytes = std::max(fa_spk_laplacian_batch_workspace_bytes(n.data(), S, kSpkEmbDim), fa_spk_tridiagonalize_batch_workspace_bytes(n.data(), S));
    int64_t squares = 0;
    for (int32_t v : n) squares += (int64_t)v * v;
    double *lap, *de, *tau, *zd;
    float* packed = nullptr;
    void* ws;
    if (!carve(s.spk_cluster, "speaker clustering", [&](fa::Arena& a) {
          lap = a.take<double>((size_t)squares); de = a.take<double>((size_t)2 * rows); tau = a.take<double>((size_t)rows);
          zd = a.take<double>((size_t)zo[S]); ws = a.take<char>(ws_bytes);
          if (!contiguous) packed = a.take<float>((size_t)rows * kSpkEmbDim);
        }))
      return false;
    const float* emb = emb_d + (size_t)sets[spectral[0]].first * kSpkEmbDim;
    if (!contiguous) {                               // the spectral sets' rows gathered in set order
      for (int i = 0; i < S; ++i)
        cudaMemcpyAsync(packed + vo[i] * kSpkEmbDim, emb_d + (size_t)sets[spectral[i]].first * kSpkEmbDim, (size_t)n[i] * kSpkEmbDim * 4,
                        cudaMemcpyDeviceToDevice, st);
      emb = packed;
    }
    int rc = fa_spk_laplacian_batch(emb, n.data(), S, kSpkEmbDim, kSpkPval, lap, ws, ws_bytes, st);
    if (rc == FA_OK) rc = fa_spk_tridiagonalize_batch(lap, n.data(), S, de, de + rows, tau, ws, ws_bytes, st);
    if (rc != FA_OK) { set_err(std::string("speaker clustering: ") + fa_status_string(rc)); return false; }
    std::vector<double> de_h((size_t)2 * rows), z((size_t)zo[S]);
    cudaMemcpyAsync(de_h.data(), de, de_h.size() * 8, cudaMemcpyDeviceToHost, st);
    if (!sync_stream(st)) return false;
    for (int i = 0; i < S; ++i) {
      const ClusterSet& c = sets[spectral[i]];
      const double *d = de_h.data() + vo[i], *e = de_h.data() + rows + vo[i];
      const int m = std::max(std::min(kMaxSpks + 1, c.n), c.preset);
      std::vector<double> w((size_t)m);
      int kk = c.preset;
      if (kk <= 0) {                                 // the largest gap among the 16 smallest eigenvalues (spec_embs)
        fa_sym_tridiag_smallest_host(d, e, c.n, m, 0, w.data(), nullptr);
        const int ne = std::min(kMaxSpks + 1, c.n);
        double gmax = -INFINITY;
        for (int j = 0; j + 1 < ne; ++j)
          if (w[j + 1] - w[j] > gmax) { gmax = w[j + 1] - w[j]; kk = j + 1; }
      }
      k[i] = kk;
      ks[spectral[i]] = kk;
      fa_sym_tridiag_smallest_host(d, e, c.n, std::max(m, kk), kk, w.data(), z.data() + zo[i]);
    }
    // the sets' vectors packed at their own k: z [sum k n]
    std::vector<int64_t> zk((size_t)S + 1, 0);
    for (int i = 0; i < S; ++i) zk[i + 1] = zk[i] + (int64_t)k[i] * n[i];
    for (int i = 1; i < S; ++i) std::copy(z.begin() + zo[i], z.begin() + zo[i] + (int64_t)k[i] * n[i], z.begin() + zk[i]);
    cudaMemcpyAsync(zd, z.data(), (size_t)zk[S] * 8, cudaMemcpyHostToDevice, st);
    rc = fa_spk_back_transform_batch(lap, tau, n.data(), k.data(), S, zd, st);
    if (rc != FA_OK) { set_err(std::string("speaker clustering: ") + fa_status_string(rc)); return false; }
    cudaMemcpyAsync(z.data(), zd, (size_t)zk[S] * 8, cudaMemcpyDeviceToHost, st);
    if (!sync_stream(st)) return false;
    for (int i = 0; i < S; ++i) {
      const int si = spectral[i], nn = n[i], kk = k[i];
      const double* zi = z.data() + zk[i];
      x[si].resize((size_t)nn * kk);
      for (int r = 0; r < nn; ++r)
        for (int j = 0; j < kk; ++j) x[si][(size_t)r * kk + j] = zi[(size_t)j * nn + r];
      dims[si] = kk;
    }
  }
  for (size_t i = 0; i < sets.size(); ++i) {
    ClusterSet& c = sets[i];
    if (c.n < 20 || !c.err.empty()) continue;
    const float* eh = emb_h + (size_t)c.first * kSpkEmbDim;
    if (c.n >= kSpectralMaxChunks) {                 // _normalize_rows in fp32, with the preset count
      x[i].resize((size_t)c.n * kSpkEmbDim);
      for (int r = 0; r < c.n; ++r) {
        const float* row = eh + (size_t)r * kSpkEmbDim;
        float ss = 0.f;
        for (int j = 0; j < kSpkEmbDim; ++j) ss += row[j] * row[j];
        float nrm = std::sqrt(ss);
        if (nrm == 0.f) nrm = 1.f;
        for (int j = 0; j < kSpkEmbDim; ++j) x[i][(size_t)r * kSpkEmbDim + j] = (double)(row[j] / nrm);
      }
      dims[i] = kSpkEmbDim;
      ks[i] = c.preset;
    }
    if (fa_spk_kmeans_host(x[i].data(), c.n, dims[i], ks[i], 0, 10, 300, c.labels.data()) != FA_OK) { c.err = c.what + "k-means failed"; continue; }
    if (c.preset <= 0 && fa_spk_merge_by_cos_host(c.labels.data(), eh, c.n, kSpkEmbDim, kMergeThr) != FA_OK) c.err = c.what + "merge_by_cos failed";
  }
  return true;
}

}  // namespace

namespace fa_handle {

// sv_chunk windows over every VAD segment of every job (vad_segment mode); each job's refusal decided from its chunk count before any
// embedding; the chunks of the jobs that cluster gathered with zero tails and embedded together in slices, one copy of the embeddings
// to the host; clustered together (spk_cluster); post-processed and distributed over each job's segments
bool diarize(Spk& s, const float* recs, int64_t n_recs, std::vector<SpkJob>& jobs) {
  cudaStream_t st = s.file.st;
  const int J = (int)jobs.size();
  std::vector<std::vector<int64_t>> starts((size_t)J);             // per job, interleaved: first sample in recs, sample count
  std::vector<std::vector<double>> times((size_t)J);
  for (int q = 0; q < J; ++q) {
    SpkJob& jb = jobs[q];
    const std::vector<int32_t>& segs = *jb.segs;
    const int64_t ns = (int64_t)segs.size() / 3;
    for (int64_t g = 0; g < ns; ++g) {               // long_audio.speaker_chunks / diarization.chunk_bounds
      const int64_t b0 = (int64_t)segs[3 * g] * 16, b1 = std::min<int64_t>((int64_t)segs[3 * g + 1] * 16, jb.n), len = std::max<int64_t>(b1 - b0, 0);
      int64_t last_ed = 0;
      for (int64_t a = 0; a < len; a += kChunkShift) {
        const int64_t ed = std::min<int64_t>(a + kChunkLen, len);
        if (ed <= last_ed) break;
        last_ed = ed;
        const int64_t c0 = std::max<int64_t>(0, ed - kChunkLen);
        starts[q].push_back(jb.off + b0 + c0);
        starts[q].push_back(ed - c0);
        times[q].push_back((double)c0 / 16000 + (double)segs[3 * g] / 1000.0);
        times[q].push_back((double)ed / 16000 + (double)segs[3 * g] / 1000.0);
      }
    }
    jb.spk->assign((size_t)ns, 0);
    jb.err.clear();
  }
  // the sets to cluster: every job of 20 chunks or more that is not refused, the spectral ones (fewer than 2048) first, so their rows
  // are contiguous; fewer than 20 chunks are one speaker and need no embedding
  std::vector<ClusterSet> sets;
  std::vector<int> set_of((size_t)J, -1);
  int rows = 0;
  for (int pass = 0; pass < 2; ++pass)
    for (int q = 0; q < J; ++q) {
      const int nc = (int)(starts[q].size() / 2);
      if (pass == 0) jobs[q].err = cluster_refusal(nc, jobs[q].preset, jobs[q].what);
      if (nc < 20 || !jobs[q].err.empty() || (nc < kSpectralMaxChunks) != (pass == 0)) continue;
      ClusterSet c;
      c.first = rows; c.n = nc; c.preset = jobs[q].preset; c.what = jobs[q].what;
      set_of[q] = (int)sets.size();
      sets.push_back(std::move(c));
      rows += nc;
    }
  if (rows > 0) {
    std::vector<int64_t> win((size_t)2 * rows);      // the sets' windows in row order
    for (int q = 0; q < J; ++q)
      if (set_of[q] >= 0) std::copy(starts[q].begin(), starts[q].end(), win.begin() + 2 * (int64_t)sets[set_of[q]].first);
    const int t_max = fbank_frames(kChunkLen);
    const size_t per = fa_campplus_workspace_bytes(&s.model, 1, t_max, s.mode);
    const int step = (int)std::max<size_t>(1, std::min<size_t>({(size_t)rows, kSpkWorkspaceCap / (per ? per : 1), (size_t)65535}));
    float *emb, *wav;
    int64_t* starts_d;
    int32_t *lens_d, *full_d;
    if (!carve(s.diarize, "speaker chunks", [&](fa::Arena& a) {
          emb = a.take<float>((size_t)rows * kSpkEmbDim); wav = a.take<float>((size_t)step * kChunkLen);
          starts_d = a.take<int64_t>(step); lens_d = a.take<int32_t>(step); full_d = a.take<int32_t>(step);
        }))
      return false;
    const std::vector<int32_t> full((size_t)step, kChunkLen);  // every window counts as 1.5 s of samples, its zero tail included
    cudaMemcpyAsync(full_d, full.data(), (size_t)step * 4, cudaMemcpyHostToDevice, st);
    std::vector<int64_t> sb((size_t)step);
    std::vector<int32_t> lb((size_t)step);
    for (int c0 = 0; c0 < rows; c0 += step) {
      const int nb = std::min(step, rows - c0);
      if (!sync_stream(st)) return false;             // sb / lb are reused: the previous slice's copies are done
      for (int r = 0; r < nb; ++r) { sb[r] = win[2 * (c0 + r)]; lb[r] = (int32_t)win[2 * (c0 + r) + 1]; }
      if (!gather(recs, n_recs, sb.data(), lb.data(), nb, kChunkLen, starts_d, lens_d, wav, st)) return false;
      if (!spk_embed_rows(s, wav, kChunkLen, full_d, nb, t_max, emb + (size_t)c0 * kSpkEmbDim)) return false;
    }
    std::vector<float> emb_h((size_t)rows * kSpkEmbDim);
    cudaMemcpyAsync(emb_h.data(), emb, emb_h.size() * 4, cudaMemcpyDeviceToHost, st);
    if (!sync_stream(st)) return false;
    if (!spk_cluster(s, emb, emb_h.data(), sets)) return false;
  }
  for (int q = 0; q < J; ++q) {
    SpkJob& jb = jobs[q];
    const int nc = (int)(starts[q].size() / 2);
    if (nc == 0 || !jb.err.empty()) continue;
    std::vector<int32_t> labels((size_t)nc, 0);      // fewer than 20 chunks: one speaker
    if (set_of[q] >= 0) {
      ClusterSet& c = sets[set_of[q]];
      if (!c.err.empty()) { jb.err = c.err; continue; }
      labels.swap(c.labels);
    }
    const std::vector<int32_t>& segs = *jb.segs;
    const int64_t ns = (int64_t)segs.size() / 3;
    std::vector<double> turns((size_t)3 * nc);
    const int64_t nt = fa_spk_postprocess_host(times[q].data(), labels.data(), nc, turns.data());
    std::vector<int32_t> sent((size_t)2 * ns);
    for (int64_t g = 0; g < ns; ++g) { sent[2 * g] = segs[3 * g]; sent[2 * g + 1] = segs[3 * g + 1]; }
    if (nt < 0 || fa_spk_distribute_host(sent.data(), ns, turns.data(), nt, jb.spk->data()) != FA_OK) jb.err = jb.what + "speaker post-processing failed";
  }
  return true;
}

}  // namespace fa_handle

extern "C" void* fa_spk_init(const char* model_file, int32_t device, int32_t gemm_mode) {
  g_err.clear();
  if (!valid_gemm_mode(gemm_mode)) return fail("bad gemm_mode");
  return open_handle(model_file, device, gemm_mode, build_spk);
}

extern "C" void fa_spk_uninit(void* spk) { delete static_cast<Spk*>(spk); }

namespace fa_handle {

// One fa_spk_embed* or fa_spk_cluster call, its arguments checked, waiting in the speaker handle's pool
struct SpkTicket : PoolTicket {
  bool cluster = false;
  // fa_spk_embed*: batch rows of the caller's audio, their 16 kHz lengths, and the call's extent (fbank_frames of its longest row)
  const void* const* bufs = nullptr;
  const int64_t* n_samples = nullptr;
  int batch = 0;
  Audio au;
  std::vector<int32_t> lens;
  int t_max = 0;
  int64_t stride = 0;                                // the call's padded row: its longest row rounded up to 4 samples
  float* emb_host = nullptr;
  // fa_spk_cluster: n host embeddings, the preset count (<= 0: none) -> labels
  const float* emb_in = nullptr;
  int n = 0, preset = 0;
  int32_t* labels = nullptr;
};

}  // namespace fa_handle

namespace {

int64_t ticket_samples(const SpkTicket& t) { return t.cluster ? 0 : (int64_t)t.batch * t.stride; }

// A pass's admission: the head of the queue and the calls behind it in arrival order, until an hour of padded audio or
// kPoolClusterRows clustering rows
void admit(std::deque<SpkTicket*>& queue, std::vector<SpkTicket*>& pass) {
  int64_t samples = 0, rows = 0;
  while (!queue.empty()) {
    SpkTicket* c = queue.front();
    const int64_t sm = samples + ticket_samples(*c), r = rows + (c->cluster ? c->n : 0);
    if (!pass.empty() && (sm > kPoolSamples || r > kPoolClusterRows)) break;
    samples = sm;
    rows = r;
    pass.push_back(c);
    queue.pop_front();
  }
}

// The embedding calls of a pass.  Calls in order of extent (arrival order within one), so each call's rows are contiguous; packs of
// consecutive calls, a call of a larger extent joining while the pack stays within the workspace cap at that extent.  Per pack, in
// turn: its calls uploaded in their own formats at the pack's row pitch, its longest row's (a pack of one call: that call's upload, as
// before pooling; several: each written straight into the pack's buffer), so a pack holds its calls' own padded audio plus less than
// one fbank frame per row, or, mixing extents, less than the workspace cap's share; fa_campplus_features at its extent and
// fa_campplus_forward_ext with every row's own.  One copy of every embedding to the host.
bool embed_pass(Spk& s, std::vector<SpkTicket*> ts) {
  cudaStream_t st = s.file.st;
  std::stable_sort(ts.begin(), ts.end(), [](const SpkTicket* a, const SpkTicket* b) { return a->t_max < b->t_max; });
  const size_t nt = ts.size();
  std::vector<int> first(nt + 1, 0);
  for (size_t i = 0; i < nt; ++i) first[i + 1] = first[i] + ts[i]->batch;
  const int R = first[nt];
  std::vector<int32_t> lens((size_t)R), ext((size_t)R);
  for (size_t i = 0; i < nt; ++i) {
    std::copy(ts[i]->lens.begin(), ts[i]->lens.end(), lens.begin() + first[i]);
    std::fill(ext.begin() + first[i], ext.begin() + first[i + 1], ts[i]->t_max);
  }
  int32_t* lens_d;
  float* emb;
  if (!carve(s.embed, "CAM++", [&](fa::Arena& a) { lens_d = a.take<int32_t>(R); emb = a.take<float>((size_t)R * kSpkEmbDim); })) return false;
  cudaMemcpyAsync(lens_d, lens.data(), (size_t)R * 4, cudaMemcpyHostToDevice, st);
  for (size_t i = 0; i < nt;) {
    size_t j = i + 1;
    int64_t rows = ts[i]->batch, stride = ts[i]->stride;
    while (j < nt && (ts[j]->t_max == ts[j - 1]->t_max ||
                      (size_t)(rows + ts[j]->batch) * fa_campplus_workspace_bytes(&s.model, 1, ts[j]->t_max, s.mode) <= kSpkWorkspaceCap)) {
      stride = std::max(stride, ts[j]->stride);
      rows += ts[j++]->batch;
    }
    float* recs = nullptr;
    if (j > i + 1 && !carve(s.pool_recs, "recordings", [&](fa::Arena& a) { recs = a.take<float>((size_t)rows * stride); })) return false;
    for (size_t k = i; k < j; ++k) {
      const SpkTicket& t = *ts[k];
      float* into = recs ? recs + (int64_t)(first[k] - first[i]) * stride : nullptr;
      float* wav;
      if (!upload(t.bufs, t.n_samples, t.batch, stride, t.au, s.resample, s.upload, st, &wav, into)) return false;
      if (!recs) recs = wav;
    }
    // a pack of one extent (a lone call's) is fa_campplus_forward, bit for bit and with the kernels it always ran
    const int r0 = first[i];
    const bool one_extent = ts[i]->t_max == ts[j - 1]->t_max;
    if (!spk_embed_rows(s, recs, stride, lens_d + r0, (int)rows, ts[j - 1]->t_max, emb + (size_t)r0 * kSpkEmbDim,
                        one_extent ? nullptr : ext.data() + r0))
      return false;
    i = j;
  }
  std::vector<float> host(nt > 1 ? (size_t)R * kSpkEmbDim : 0);
  float* dst = nt == 1 ? ts[0]->emb_host : host.data();
  cudaMemcpyAsync(dst, emb, (size_t)R * kSpkEmbDim * 4, cudaMemcpyDeviceToHost, st);
  if (!sync_stream(st)) return false;
  if (nt > 1)
    for (size_t i = 0; i < nt; ++i)
      std::copy(host.begin() + (size_t)first[i] * kSpkEmbDim, host.begin() + (size_t)first[i + 1] * kSpkEmbDim, ts[i]->emb_host);
  return true;
}

// The clustering calls of a pass: their embeddings in one buffer (a lone call's straight from its host array, as before pooling), one
// spk_cluster over all their sets; a set's refusal fails only its own call, with the message it gets alone
bool cluster_pass(Spk& s, const std::vector<SpkTicket*>& ts) {
  std::vector<ClusterSet> sets(ts.size());
  int64_t rows = 0;
  for (size_t i = 0; i < ts.size(); ++i) {
    sets[i].first = (int)rows;
    sets[i].n = ts[i]->n;
    sets[i].preset = ts[i]->preset;
    rows += ts[i]->n;
  }
  std::vector<float> staged;
  const float* emb_h = ts[0]->emb_in;
  if (ts.size() > 1) {
    staged.resize((size_t)rows * kSpkEmbDim);
    for (size_t i = 0; i < ts.size(); ++i)
      std::copy(ts[i]->emb_in, ts[i]->emb_in + (size_t)ts[i]->n * kSpkEmbDim, staged.begin() + (size_t)sets[i].first * kSpkEmbDim);
    emb_h = staged.data();
  }
  float* emb;
  if (!carve(s.cluster_input, "speaker clustering", [&](fa::Arena& a) { emb = a.take<float>((size_t)rows * kSpkEmbDim); })) return false;
  cudaMemcpyAsync(emb, emb_h, (size_t)rows * kSpkEmbDim * 4, cudaMemcpyHostToDevice, s.file.st);
  if (!spk_cluster(s, emb, emb_h, sets)) return false;
  for (size_t i = 0; i < ts.size(); ++i) {
    if (!sets[i].err.empty()) ts[i]->err = sets[i].err;
    else std::copy(sets[i].labels.begin(), sets[i].labels.end(), ts[i]->labels);
  }
  return true;
}

// One pass under the speaker lock: the embedding calls, then the clustering calls.  A device failure fails every call of the pass.
void run_pass(Spk& s, const std::vector<SpkTicket*>& pass) {
  std::vector<SpkTicket*> emb, clu;
  for (SpkTicket* t : pass) (t->cluster ? clu : emb).push_back(t);
  {
    std::lock_guard<std::mutex> dev(s.mu);
    cudaSetDevice(s.file.device);
    const bool ok = no_throw("fa_spk_embed: ", [&] { return emb.empty() || embed_pass(s, emb); }) &&
                    no_throw("fa_spk_cluster: ", [&] { return clu.empty() || cluster_pass(s, clu); });
    if (!ok)
      for (SpkTicket* t : pass) t->err = g_err;
  }
  ++s.pool_passes;
}

// t's call through the pool -> its status, with its own message set as this thread's error
int pool_call(Spk& s, SpkTicket& t) {
  s.pool.call(t, admit, [&](std::vector<SpkTicket*>& pass, std::vector<SpkTicket*>& ended) {
    run_pass(s, pass);
    ended.swap(pass);
  }, "fa_spk: ");
  if (!t.err.empty()) { set_err(t.err); return FA_ERR_CUDA; }
  g_err.clear();
  return FA_OK;
}

// fa_spk_embed / fa_spk_embed_audio: every input checked at 16 kHz on the calling thread, then the call's rows through the pool, padded
// to its longest input
int spk_embed(void* spk, const void* const* bufs, const int64_t* n_samples, int32_t batch, const FaAudioFormat* fmt, float* emb_host) {
  Spk* s = static_cast<Spk*>(spk);
  if (!s || !bufs || !n_samples || batch <= 0 || !emb_host) { set_err("fa_spk_embed: bad argument"); return FA_ERR_ARG; }
  SpkTicket t;
  if (!plan_audio(fmt, s->resample, t.au)) return FA_ERR_ARG;
  int64_t nmax = 0;
  int longest = 0;
  const bool ok = no_throw("fa_spk_embed: ", [&] {
    t.lens.resize(batch);
    for (int32_t i = 0; i < batch; ++i) {            // every input checked before any launch
      const int64_t n16 = n_samples[i] >= 0 && n_samples[i] <= 0x7fffffffLL ? t.au.len16(n_samples[i]) : n_samples[i];
      if (!bufs[i] || n16 < 400 || n16 > 0x7fffffffLL) {
        set_err("input " + std::to_string(i) + " has " + std::to_string(n16) + " samples" + t.au.at16k() + "; CAM++ needs at least 400 (one 25 ms frame)");
        return false;
      }
      t.lens[i] = (int32_t)n16;
      if (n16 > nmax) { nmax = n16; longest = i; }
    }
    return true;
  });
  if (!ok) return FA_ERR_ARG;
  t.t_max = fbank_frames(nmax);
  if (t.t_max > kSpkMaxFrames) {
    set_err("input " + std::to_string(longest) + " has " + std::to_string(t.t_max) + " feature frames; CAM++ takes at most " +
            std::to_string(kSpkMaxFrames) + " (MAX_FEAT_FRAMES)");
    return FA_ERR_UNSUPPORTED;
  }
  t.bufs = bufs;
  t.n_samples = n_samples;
  t.batch = batch;
  t.stride = (nmax + 3) / 4 * 4;
  t.emb_host = emb_host;
  return pool_call(*s, t);
}

}  // namespace

extern "C" int fa_spk_embed(void* spk, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format, float* emb_host) {
  g_err.clear();
  FaAudioFormat f;
  if (!pcm16k_format(pcm_format, f)) { set_err("fa_spk_embed: bad argument"); return FA_ERR_ARG; }
  return spk_embed(spk, bufs, n_samples, batch, &f, emb_host);
}

extern "C" int fa_spk_embed_audio(void* spk, const void* const* bufs, const int64_t* n_samples, int32_t batch, const FaAudioFormat* fmt, float* emb_host) {
  g_err.clear();
  return spk_embed(spk, bufs, n_samples, batch, fmt, emb_host);
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
  SpkTicket t;
  t.cluster = true;
  t.emb_in = emb_host;
  t.n = n;
  t.preset = preset_spk_num;
  t.labels = labels;
  return pool_call(*s, t);
}

extern "C" int fa_spk_pool_stats(const void* spk, int64_t* calls, int64_t* passes) {
  const Spk* s = static_cast<const Spk*>(spk);
  if (!s || !calls || !passes) return FA_ERR_ARG;
  *calls = s->pool.calls.load();
  *passes = s->pool_passes.load();
  return FA_OK;
}
