// Model-level C-ABI entry points: the kernel sequences of SANMEncoder.forward, CifPredictorV2.forward and
// ParaformerSANMDecoder.forward (+ greedy arg-max), stream-ordered over a caller-provided workspace.
#include "common.cuh"
#include "kernels.h"
#include <string.h>
#include <math.h>
#include <algorithm>
#include <map>
#include <vector>
#include <mutex>
#include <utility>

namespace fa {

std::atomic<unsigned long long> g_launch_count{0};

// Side stream for the encoder's FSMN memory branch: it depends only on the QKV GEMM (like the attention kernel) and is HBM
// bound with a tiny footprint, so it runs concurrently with the latency-bound attention kernel and joins before the
// out-projection.  One lazily created (stream, fork event, join event) per device.
// The (side stream, fork event, join event) triple belongs to ONE caller stream on one device: two host threads that run
// encoders on different streams (two fa_offline handles, one worker thread per model) get different triples, so one thread's
// fork record can never be consumed by the other's side stream.  Calls that share a caller stream are ordered by that stream.
struct SideStream { cudaStream_t st = nullptr; cudaEvent_t fork = nullptr, join = nullptr; };
static SideStream* side_stream(cudaStream_t caller) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, SideStream*> pool;
  std::lock_guard<std::mutex> lock(mu);
  SideStream*& slot = pool[std::make_pair(dev, caller)];
  if (!slot) {
    SideStream* s = new SideStream();
    if (cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&s->fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&s->join, cudaEventDisableTiming) != cudaSuccess) {
      delete s;
      return nullptr;
    }
    slot = s;
  }
  return slot;
}

// ------------------------------------------------------------------------------------------------ encoder
// Sized for the largest supported stack (d_model 512, input 560, FFN 2048).  The fp32 path keeps every activation in fp32; the
// tensor-core path passes LayerNorm, attention and FFN w_1 outputs as fp16 planes and writes only the V columns of qkv in fp32.
struct EncBufs {
  float *u, *qkv, *mem, *ctx, *xa, *xb, *h;
  plane_t *ctx_planes, *h_planes, *u_planes;
  AttnPlanes att;                                                   // sized for width 512, whatever the model's width
};
static EncBufs enc_carve(Arena& a, int batch, int t_max, int mode) {
  const int64_t M = (int64_t)batch * t_max;
  const bool tc = mode != FA_GEMM_F32_SIMT;
  const size_t gpl = gemm_planes(mode);
  EncBufs b;
  b.u = tc ? nullptr : a.take<float>(M * 560ull);
  b.qkv = a.take<float>(M * 1536ull);
  b.mem = a.take<float>(M * 512ull);
  b.ctx = tc ? nullptr : a.take<float>(M * 512ull);
  b.xa = a.take<float>(M * 512ull);
  b.xb = a.take<float>(M * 512ull);
  b.h = tc ? nullptr : a.take<float>(M * 2048ull);
  b.ctx_planes = tc ? a.take<plane_t>(gpl * M * 512) : nullptr;
  b.h_planes = tc ? a.take<plane_t>(gpl * M * 2048) : nullptr;
  b.u_planes = tc ? a.take<plane_t>(gpl * M * 576) : nullptr;      // LN output: the QKV GEMM's K pad of a 560 input
  if (tc) b.att = attn_carve(a, batch, t_max, batch, t_max, 512, mode);
  return b;
}

}  // namespace fa

using namespace fa;

extern "C" size_t fa_sanm_encoder_workspace_bytes(int32_t batch, int32_t t_max, int32_t gemm_mode) {
  Arena m = Arena::measuring();
  enc_carve(m, batch, t_max, gemm_mode);
  return m.bytes();
}

extern "C" int fa_sanm_encoder_forward(const FaEncoder* enc, const float* feats, const int32_t* lens, int32_t batch,
                                       int32_t t_max, float* out, int32_t gemm_mode, void* workspace, size_t ws_bytes,
                                       fa_stream_t stream) {
  if (!enc || !enc->layers || !feats || !lens || !out || batch <= 0 || t_max <= 0 || enc->n_layers < 1) return FA_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t M = (int64_t)batch * t_max;
  const int D = enc->after_norm.n;
  const int din = enc->layers[0].norm1.n;
  const bool embed = enc->pe_inv_timescales != nullptr;   // false: plain stack over an existing [B,T,512] stream
  const int hd = enc->heads > 0 ? D / enc->heads : 0;
  // the tensor-core kernels are built for two shapes: Paraformer / SenseVoice (d = 512, 4 x 128) and the fa-zh aligner (d = 320,
  // 4 x 80); the fp32 path also runs the small SAN-M stacks around the hot path (CT-Transformer punctuation: d = 256, 8 x 32)
  if (D < 64 || D > 512 || (D & 15) || enc->heads < 1 || enc->heads * hd != D || hd < 32 || hd > 128 || ((hd & 31) && hd != 80) ||
      din > 560 || (din & 15) || (!embed && din != D))
    return FA_ERR_UNSUPPORTED;
  if (gemm_mode != FA_GEMM_F32_SIMT && !((D == 512 && hd == 128) || (D == 320 && hd == 80))) return FA_ERR_UNSUPPORTED;
  const bool tc = gemm_mode != FA_GEMM_F32_SIMT;
  // every layer's shape is checked before the first launch: a malformed layer enqueues nothing
  for (int l = 0; l < enc->n_layers; ++l) {
    const FaEncLayer& L = enc->layers[l];
    const int in = L.norm1.n;
    if (L.qkv.in_f != in || L.qkv.out_f != 3 * D || L.w1.in_f != D || L.w2.out_f != D || L.w2.in_f != L.w1.out_f) return FA_ERR_ARG;
    if (L.w1.out_f > 2048) return FA_ERR_UNSUPPORTED;      // enc_carve sizes the FFN hidden slice for linear_units <= 2048
    if (l > 0 && in != D) return FA_ERR_UNSUPPORTED;
    if (tc && (L.w1.out_f != L.w2.in_pad || L.w1.in_pad != D)) return FA_ERR_UNSUPPORTED;
  }
  const int npl = gemm_planes(gemm_mode);
  Arena a(workspace, ws_bytes);
  const EncBufs b = enc_carve(a, batch, t_max, gemm_mode);
  if (!a.ok()) return FA_ERR_WORKSPACE;
  float *u = b.u, *qkv = b.qkv, *mem = b.mem, *ctx = b.ctx, *xa = b.xa, *xb = b.xb, *h = b.h;
  plane_t *ctx_planes = b.ctx_planes, *h_planes = b.h_planes, *u_planes = b.u_planes;
  const AttnShape shape{batch, enc->heads, hd, t_max, t_max, 0};

  const float* x = embed ? nullptr : feats;  // residual stream (with PE input: undefined before layer 0, in_size != size)
  for (int l = 0; l < enc->n_layers; ++l) {
    const FaEncLayer& L = enc->layers[l];
    const int in = L.norm1.n;
    // x = x*sqrt(D) + PE is folded into the first LayerNorm (encoder.py:409,428)
    // tensor-core path: LayerNorm writes the fp16 planes the QKV GEMM consumes (no fp32 round trip, no split pass)
    const bool first = embed && l == 0;
    // a first layer with in_size == size keeps its residual (encoder.py:120-126): the embedded rows x*sqrt(d) + PE are then needed
    // beside their LayerNorm (CT-Transformer: 256 -> 256; Paraformer / SenseVoice: 560 -> 512, no residual)
    float* emb = (first && in == D) ? xa : nullptr;
    FA_RETURN_IF_ERR(layernorm_launch(first ? feats : x, M, L.norm1, tc ? nullptr : u, first ? enc->pe_inv_timescales : nullptr,
                                      first ? sqrtf((float)D) : 1.f, t_max, st, u_planes, npl, L.qkv.in_pad, emb));
    if (emb) x = emb;
    if (tc) {
      // QKV GEMM epilogue emits the attention operands directly: q (x d_k^-0.5) / k as fp16 planes, v transposed per head
      // as fp16 planes plus fp32 v (the only fp32 columns written) for the FSMN branch
      const AttnSinks sk = attn_sinks(b.att, 0, D, 2 * D, D, t_max, attn_qscale(hd));
      FA_RETURN_IF_ERR(gemm_tc_planes_launch(u_planes, M, L.qkv, GemmEpi().to(qkv, 3 * D).sinks(&sk), gemm_mode, st));
    } else {
      FA_RETURN_IF_ERR(gemm_rows(u, in, M, L.qkv, GemmEpi().to(qkv, 3 * D), gemm_mode, nullptr, st));
    }
    SideStream* side = tc ? side_stream(st) : nullptr;
    // x2 = (residual if in_size == size) + (linear_out(ctx) + fsmn_memory)     encoder.py:120-137, attention.py:327
    float* x2 = (x == xa) ? xb : xa;
    const float* res = (in == D && x != nullptr) ? x : nullptr;
    float* x3 = (x2 == xa) ? xb : xa;
    // tensor-core path: the FSMN kernel (HBM bound, on the side stream beside the latency-bound attention kernel) also adds the
    // layer's residual, so the out-projection epilogue reads ONE fp32 stream instead of two (it was bound by those reads:
    // 198 MB in 69 us, tensor pipe 43 %).  fp32 path: the reference's own association ((att + mem) + residual) is kept.
    const float* fsmn_res = tc ? res : nullptr;
    if (side) {                                     // FSMN memory branch runs beside the attention kernel (both need only QKV)
      FA_CUDA_OK(cudaEventRecord(side->fork, st));
      FA_CUDA_OK(cudaStreamWaitEvent(side->st, side->fork, 0));
      FA_RETURN_IF_ERR(fsmn_launch(qkv + 2 * D, 3 * D, lens, batch, t_max, D, L.fsmn_w, enc->fsmn_k, fsmn_res, D, mem, D, side->st));
      FA_CUDA_OK(cudaEventRecord(side->join, side->st));
    } else {
      FA_RETURN_IF_ERR(fsmn_launch(qkv + 2 * D, 3 * D, lens, batch, t_max, D, L.fsmn_w, enc->fsmn_k, fsmn_res, D, mem, D, st));
    }
    if (!tc) {
      FA_RETURN_IF_ERR(attention_rows(qkv, 3 * D, qkv + D, 3 * D, qkv + 2 * D, 3 * D, shape, lens, AttnOut().to(ctx, D), gemm_mode, nullptr, st));
      FA_RETURN_IF_ERR(gemm_rows(ctx, D, M, L.out, GemmEpi().add(mem, D, res, D).to(x2, D), gemm_mode, nullptr, st));
      FA_RETURN_IF_ERR(layernorm_launch(x2, M, L.norm2, u, nullptr, 1.f, t_max, st));
      FA_RETURN_IF_ERR(gemm_rows(u, D, M, L.w1, GemmEpi().relu().to(h, L.w1.out_f), gemm_mode, nullptr, st));
      FA_RETURN_IF_ERR(gemm_rows(h, L.w1.out_f, M, L.w2, GemmEpi().add(x2, D).to(x3, D), gemm_mode, nullptr, st));
    } else {
      // tensor-core path: attention emits the context as fp16 planes (A operand of linear_out); FFN w_1 emits its
      // ReLU output as planes for w_2 — neither intermediate makes an fp32 round trip through HBM
      FA_RETURN_IF_ERR(attention_planes(b.att, shape, lens, AttnOut().to(ctx_planes, D, npl), st));
      if (side) FA_CUDA_OK(cudaStreamWaitEvent(st, side->join, 0));          // join: linear_out adds the FSMN memory
      FA_RETURN_IF_ERR(gemm_tc_planes_launch(ctx_planes, M, L.out, GemmEpi().add(mem, D).to(x2, D), gemm_mode, st));   // mem already holds residual + memory
      FA_RETURN_IF_ERR(layernorm_launch(x2, M, L.norm2, nullptr, nullptr, 1.f, t_max, st, u_planes, npl, D));
      FA_RETURN_IF_ERR(gemm_tc_planes_launch(u_planes, M, L.w1, GemmEpi().relu().to(h_planes, L.w1.out_f), gemm_mode, st));
      FA_RETURN_IF_ERR(gemm_tc_planes_launch(h_planes, M, L.w2, GemmEpi().add(x2, D).to(x3, D), gemm_mode, st));
    }
    x = x3;
  }
  return layernorm_launch(x, M, enc->after_norm, out, nullptr, 1.f, t_max, st);
}

// ---------------------------------------------------------------------------------------------- predictor
// fp32: the im2col rows [M, 3D] and the conv output c [M, D].  Tensor cores: no im2col copy — the GEMM's A operand is the
// overlapping view of the zero-padded encoder planes pp (cif.cu), and its output c has the padded rows [batch * (t_max + 2), D].
struct CifBufs { float *xc, *c, *alpha_rows; plane_t* pp; int32_t* ext; };
static CifBufs cif_carve(Arena& a, int batch, int t_max, int mode, bool ext) {
  const int D = 512;
  const int64_t M = (int64_t)batch * t_max, Mp = (int64_t)batch * (t_max + 2);
  const bool tc = mode != FA_GEMM_F32_SIMT;
  CifBufs b;
  b.xc = tc ? nullptr : a.take<float>(M * 3ull * D);
  b.c = a.take<float>((tc ? Mp : M) * (size_t)D);
  b.alpha_rows = a.take<float>(M);
  b.pp = tc ? a.take<plane_t>((size_t)gemm_planes(mode) * (Mp + 2) * D) : nullptr;
  b.ext = ext ? a.take<int32_t>(batch) : nullptr;                 // last: the carve above is unchanged without it
  return b;
}

extern "C" size_t fa_cif_predictor_workspace_bytes(int32_t batch, int32_t t_max, int32_t gemm_mode) {
  Arena m = Arena::measuring();
  cif_carve(m, batch, t_max, gemm_mode, false);
  return m.bytes();
}

extern "C" size_t fa_cif_predictor_ext_workspace_bytes(int32_t batch, int32_t t_max, int32_t gemm_mode) {
  Arena m = Arena::measuring();
  cif_carve(m, batch, t_max, gemm_mode, true);
  return m.bytes();
}

// ext_h: each row's padded length (host, NULL: t_max for every row), copied into the workspace
static int cif_predictor(const FaPredictor* pred, const float* enc, const int32_t* lens, int32_t batch, int32_t t_max, float* acoustic,
                         int32_t n_cap, int32_t* token_num, float* alphas, float* peaks, int32_t gemm_mode, void* workspace, size_t ws_bytes,
                         cudaStream_t st, const int32_t* ext_h) {
  const int D = 512;
  if (pred->conv.out_f != D || pred->conv.in_f != 3 * D) return FA_ERR_UNSUPPORTED;
  const bool tc = gemm_mode != FA_GEMM_F32_SIMT;
  if (tc && !pred->conv.w_planes) return FA_ERR_ARG;
  if (tc && pred->conv.in_pad != 3 * D) return FA_ERR_UNSUPPORTED;    // the conv view reads K = 3 D unpadded
  const int64_t M = (int64_t)batch * t_max;
  Arena a(workspace, ws_bytes);
  const CifBufs b = cif_carve(a, batch, t_max, gemm_mode, ext_h != nullptr);
  if (!a.ok()) return FA_ERR_WORKSPACE;
  if (ext_h) FA_CUDA_OK(cudaMemcpyAsync(b.ext, ext_h, (size_t)batch * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (tc) {
    const int npl = gemm_planes(gemm_mode);
    const int64_t Mp = (int64_t)batch * (t_max + 2), rows_alloc = Mp + 2;
    FA_RETURN_IF_ERR(cif_pad_planes_launch(enc, batch, t_max, b.ext, D, npl, rows_alloc, b.pp, st));
    FA_RETURN_IF_ERR(gemm_tc_planes_launch(b.pp, Mp, pred->conv, GemmEpi().relu().to(b.c, D), gemm_mode, st, D, rows_alloc));
    FA_RETURN_IF_ERR(cif_alpha_launch(b.c, D, pred->out_w, pred->out_b, lens, t_max, M, pred->smooth_factor,
                                      pred->noise_threshold, b.alpha_rows, st, t_max + 2));
  } else {
    FA_RETURN_IF_ERR(cif_im2col_launch(enc, M, t_max, b.ext, D, b.xc, st));
    FA_RETURN_IF_ERR(gemm_rows(b.xc, 3 * D, M, pred->conv, GemmEpi().relu().to(b.c, D), gemm_mode, nullptr, st));
    FA_RETURN_IF_ERR(cif_alpha_launch(b.c, D, pred->out_w, pred->out_b, lens, t_max, M, pred->smooth_factor,
                                      pred->noise_threshold, b.alpha_rows, st));
  }
  FA_CUDA_OK(cudaMemsetAsync(acoustic, 0, (size_t)batch * n_cap * D * sizeof(float), st));
  if (pred->cif_variant == 1)     // CifPredictorV3 (BiCifParaformer): sequential fp32 `cif`
    return cif_fire_loop_launch(enc, b.alpha_rows, lens, b.ext, batch, t_max, D, pred->tail_threshold, pred->threshold, acoustic, n_cap,
                                token_num, alphas, peaks, st);
  if (pred->cif_variant != 0) return FA_ERR_ARG;
  return cif_fire_launch(enc, b.alpha_rows, lens, b.ext, batch, t_max, D, pred->tail_threshold, acoustic, n_cap, token_num, alphas,
                         peaks, st);
}

extern "C" int fa_cif_predictor_forward(const FaPredictor* pred, const float* enc, const int32_t* lens, int32_t batch,
                                        int32_t t_max, float* acoustic, int32_t n_cap, int32_t* token_num,
                                        float* alphas, float* peaks, int32_t gemm_mode, void* workspace, size_t ws_bytes,
                                        fa_stream_t stream) {
  if (!pred || !enc || !lens || !acoustic || !token_num || !alphas || !peaks || batch <= 0 || t_max <= 0 || n_cap <= 0)
    return FA_ERR_ARG;
  return cif_predictor(pred, enc, lens, batch, t_max, acoustic, n_cap, token_num, alphas, peaks, gemm_mode, workspace, ws_bytes,
                       (cudaStream_t)stream, nullptr);
}

// every row's padded length ext_h[b] inside [lens_h[b], t_max] (host arrays)
static bool ext_rows_ok(const int32_t* lens_h, const int32_t* ext_h, int32_t batch, int32_t t_max) {
  if (!lens_h || !ext_h) return false;
  for (int32_t b = 0; b < batch; ++b)
    if (lens_h[b] < 0 || ext_h[b] < lens_h[b] || ext_h[b] > t_max || ext_h[b] < 1) return false;
  return true;
}

extern "C" int fa_cif_predictor_forward_ext(const FaPredictor* pred, const float* enc, const int32_t* lens, int32_t batch,
                                            int32_t t_max, float* acoustic, int32_t n_cap, int32_t* token_num,
                                            float* alphas, float* peaks, int32_t gemm_mode, void* workspace, size_t ws_bytes,
                                            fa_stream_t stream, const int32_t* lens_h, const int32_t* ext_h) {
  if (!pred || !enc || !lens || !acoustic || !token_num || !alphas || !peaks || batch <= 0 || t_max <= 0 || n_cap <= 0 ||
      !ext_rows_ok(lens_h, ext_h, batch, t_max))
    return FA_ERR_ARG;
  return cif_predictor(pred, enc, lens, batch, t_max, acoustic, n_cap, token_num, alphas, peaks, gemm_mode, workspace, ws_bytes,
                       (cudaStream_t)stream, ext_h);
}

// CifPredictorV3.get_upsample_timestamp after the BLSTM (bicif_paraformer/cif_predictor.py:331-352)
extern "C" int fa_cif_upsample_alphas(const float* feat, int32_t dz, const float* w, const float* b, const int32_t* lens_up,
                                      const int32_t* token_num, int32_t batch, int32_t t_up, float smooth2, float noise2,
                                      float threshold, float* us_alphas, float* us_peaks, fa_stream_t stream) {
  if (!feat || !w || !b || !lens_up || !token_num || !us_alphas || !us_peaks || batch <= 0 || t_up <= 0 || dz <= 0 || (dz & 3))
    return FA_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  FA_RETURN_IF_ERR(cif_alpha_launch(feat, dz, w, b, lens_up, t_up, (int64_t)batch * t_up, smooth2, noise2, us_alphas, st));
  return cif_upsample_scan_launch(us_alphas, token_num, nullptr, batch, t_up, (float)((double)threshold - 1e-4), us_peaks, st);
}

// The timestamp head over B * U * t_max upsampled rows: the upsampled rows, both directions' input projections, the BLSTM output,
// the recurrence's scratch for one launch, the GEMM scratch for the larger (upsampled) GEMM — both have K = D — and lens x U
// (last: the other takes are whole multiples of 256 bytes, so the carve adds no padding); with per-row extents, ext and ext x U after it
static const int kBlstmMaxBatch = 256;          // fa_blstm_forward_tc holds at most 256 sequences per launch
struct TsHeadBufs { float *up, *xproj, *feat; void* lstm; size_t lstm_bytes; Arena gemm{nullptr, 0}; int32_t *lens_up, *ext, *ext_up; };
static TsHeadBufs ts_head_carve(Arena& a, int batch, int t_max, int d, int up_times, int mode, bool ext) {
  const int64_t rows = (int64_t)batch * t_max * up_times;
  TsHeadBufs b;
  b.up = a.take<float>((size_t)rows * d);
  b.xproj = a.take<float>((size_t)rows * 8 * d);
  b.feat = a.take<float>((size_t)rows * 2 * d);
  b.lstm_bytes = fa_blstm_tc_scratch_bytes(batch < kBlstmMaxBatch ? batch : kBlstmMaxBatch);
  b.lstm = a.take<char>(b.lstm_bytes);
  if (mode != FA_GEMM_F32_SIMT) b.gemm = a.sub(gemm_tc_scratch_bytes(rows, d, mode));
  b.lens_up = a.take<int32_t>(batch);
  b.ext = ext ? a.take<int32_t>(batch) : nullptr;
  b.ext_up = ext ? a.take<int32_t>(batch) : nullptr;
  return b;
}

__global__ void scale_lens_kernel(const int32_t* __restrict__ lens, int32_t k, int32_t n, int32_t* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = lens[i] * k;
}

extern "C" size_t fa_timestamp_head_workspace_bytes(int32_t batch, int32_t t_max, int32_t d_model, int32_t up_times, int32_t gemm_mode) {
  if (batch <= 0 || t_max <= 0 || d_model <= 0 || up_times <= 0) return 0;
  Arena m = Arena::measuring();
  ts_head_carve(m, batch, t_max, d_model, up_times, gemm_mode, false);
  return m.bytes();
}

extern "C" size_t fa_timestamp_head_ext_workspace_bytes(int32_t batch, int32_t t_max, int32_t d_model, int32_t up_times, int32_t gemm_mode) {
  if (batch <= 0 || t_max <= 0 || d_model <= 0 || up_times <= 0) return 0;
  Arena m = Arena::measuring();
  ts_head_carve(m, batch, t_max, d_model, up_times, gemm_mode, true);
  return m.bytes();
}

static int timestamp_head(const FaTimestampHead* head, const float* enc, const int32_t* lens, const int32_t* token_num, int32_t batch,
                          int32_t t_max, float* us_alphas, float* us_peaks, int32_t gemm_mode, void* workspace, size_t ws_bytes,
                          fa_stream_t stream, const int32_t* ext_h) {
  if (!head->w_hh_fwd || !head->w_hh_bwd || !head->out2_w || !head->out2_b) return FA_ERR_ARG;
  if (gemm_mode != FA_GEMM_F32_SIMT && gemm_mode != FA_GEMM_F16X1 && gemm_mode != FA_GEMM_F16X3 && gemm_mode != FA_GEMM_F16X6) return FA_ERR_ARG;
  const FaLinear &up_lin = head->upsample, &ih_lin = head->blstm_ih;
  const int D = up_lin.in_f, U = head->up_times;
  if (D != 512 && D != 320) return FA_ERR_UNSUPPORTED;        // the shapes the recurrence is built for
  if (up_lin.out_f != U * D || ih_lin.out_f != 8 * D || ih_lin.in_f != D) return FA_ERR_ARG;
  if (gemm_mode != FA_GEMM_F32_SIMT && (!up_lin.w_planes || !ih_lin.w_planes)) return FA_ERR_ARG;
  Arena a(workspace, ws_bytes);
  TsHeadBufs b = ts_head_carve(a, batch, t_max, D, U, gemm_mode, ext_h != nullptr);
  if (!a.ok()) return FA_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int TU = t_max * U;
  std::vector<int32_t> run_h;                 // per BLSTM launch: its longest sequence, in upsampled steps
  if (ext_h) {
    FA_CUDA_OK(cudaMemcpyAsync(b.ext, ext_h, (size_t)batch * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    scale_lens_kernel<<<(batch + 255) / 256, 256, 0, st>>>(b.ext, U, batch, b.ext_up);
    FA_CHECK_LAUNCH();
    for (int b0 = 0; b0 < batch; b0 += kBlstmMaxBatch)
      run_h.push_back(U * *std::max_element(ext_h + b0, ext_h + std::min(batch, b0 + kBlstmMaxBatch)));
  }
  FA_RETURN_IF_ERR(gemm_rows(enc, D, (int64_t)batch * t_max, up_lin, GemmEpi().to(b.up, (int64_t)U * D), gemm_mode, &b.gemm, st));
  FA_RETURN_IF_ERR(gemm_rows(b.up, D, (int64_t)batch * TU, ih_lin, GemmEpi().to(b.xproj, 8 * D), gemm_mode, &b.gemm, st));
  for (int b0 = 0; b0 < batch; b0 += kBlstmMaxBatch) {       // sequences are independent: larger batches run as consecutive launches
    const int bn = batch - b0 < kBlstmMaxBatch ? batch - b0 : kBlstmMaxBatch;
    FA_RETURN_IF_ERR(blstm_tc_launch(b.xproj + (int64_t)b0 * TU * 8 * D, head->w_hh_fwd, head->w_hh_bwd, bn, ext_h ? run_h[b0 / kBlstmMaxBatch] : TU,
                                     TU, ext_h ? b.ext_up + b0 : nullptr, D, b.feat + (int64_t)b0 * TU * 2 * D, b.lstm, b.lstm_bytes, st));
  }
  scale_lens_kernel<<<(batch + 255) / 256, 256, 0, st>>>(lens, U, batch, b.lens_up);
  FA_CHECK_LAUNCH();
  FA_RETURN_IF_ERR(cif_alpha_launch(b.feat, 2 * D, head->out2_w, head->out2_b, b.lens_up, TU, (int64_t)batch * TU, head->smooth2, head->noise2,
                                    us_alphas, st));
  return cif_upsample_scan_launch(us_alphas, token_num, b.ext_up, batch, TU, (float)((double)head->threshold - 1e-4), us_peaks, st);
}

extern "C" int fa_timestamp_head_forward(const FaTimestampHead* head, const float* enc, const int32_t* lens, const int32_t* token_num,
                                         int32_t batch, int32_t t_max, float* us_alphas, float* us_peaks, int32_t gemm_mode, void* workspace,
                                         size_t ws_bytes, fa_stream_t stream) {
  if (!head || !enc || !lens || !token_num || !us_alphas || !us_peaks || batch <= 0 || t_max <= 0 || head->up_times <= 0) return FA_ERR_ARG;
  return timestamp_head(head, enc, lens, token_num, batch, t_max, us_alphas, us_peaks, gemm_mode, workspace, ws_bytes, stream, nullptr);
}

extern "C" int fa_timestamp_head_forward_ext(const FaTimestampHead* head, const float* enc, const int32_t* lens, const int32_t* token_num,
                                             int32_t batch, int32_t t_max, float* us_alphas, float* us_peaks, int32_t gemm_mode, void* workspace,
                                             size_t ws_bytes, fa_stream_t stream, const int32_t* lens_h, const int32_t* ext_h) {
  if (!head || !enc || !lens || !token_num || !us_alphas || !us_peaks || batch <= 0 || t_max <= 0 || head->up_times <= 0 ||
      !ext_rows_ok(lens_h, ext_h, batch, t_max))
    return FA_ERR_ARG;
  return timestamp_head(head, enc, lens, token_num, batch, t_max, us_alphas, us_peaks, gemm_mode, workspace, ws_bytes, stream, ext_h);
}

// ------------------------------------------------------------------------------------------------ decoder
// Workspace of every decoder-stack entry point (d_model 512, 4 heads of 128, FFN <= 2048).  The memory has Mk = batch * t_max rows
// (an upper bound when it is shared).  contextual: the bias decoder over n_hotwords rows of hotword memory.  probs: the stack's ASF
// probe (attn_probs), which its query cannot see, so the stack always carves for it.  On the tensor-core path every layer passes
// its operands as fp16 planes; fp32 q / k|v / context rows and GEMM scratch serve only the calls that take fp32 operands.
// The grouped entries: mem_entries memories of t_max rows (0: batch of them), hw_groups hotword memories of n_hotwords rows each, and
// n_ints ints after the rest (the rows' key counts, memory indices and probed rows, copied from the host), so the other entries'
// carves are unchanged.
struct DecBuf {
  float *ya, *yb, *t1, *hq, *f, *qd, *ctx, *kv, *lg, *cat, *kvh;
  plane_t *ctx_planes, *mem_planes, *t1_planes, *hq_planes;
  AttnPlanes att;                     // per-utterance K / V: the stack's query cannot see mem_shared
  Arena scratch{nullptr, 0}, hw_scratch{nullptr, 0};
  int32_t* ints = nullptr;
};
static void dec_carve(Arena& a, DecBuf& b, int batch, int t_max, int n_max, int vocab, int mode, int n_hotwords, bool probs, int hw_groups = 1,
                      int mem_entries = 0, int n_ints = 0) {
  const bool grouped = mem_entries > 0;
  const int64_t Mq = (int64_t)batch * n_max, Mk = (int64_t)(grouped ? mem_entries : batch) * t_max;
  const bool tc = mode != FA_GEMM_F32_SIMT;
  const bool contextual = n_hotwords > 0;
  const size_t gpl = gemm_planes(mode);
  b.ya = a.take<float>(Mq * 512ull); b.yb = a.take<float>(Mq * 512ull); b.t1 = a.take<float>(Mq * 512ull);
  b.hq = a.take<float>(Mq * 2048ull); b.f = a.take<float>(Mq * 512ull);
  b.qd = (!tc || contextual || probs) ? a.take<float>(Mq * 512ull) : nullptr;
  b.ctx = (!tc || contextual) ? a.take<float>(Mq * 512ull) : nullptr;
  b.kv = (!tc || probs) ? a.take<float>(Mk * 1024ull) : nullptr;
  b.lg = a.take<float>(Mq * (size_t)vocab);                          // logits, used when the caller passes none
  b.cat = contextual ? a.take<float>(Mq * 1024ull) : nullptr;         // [x_src_attn ; cx]
  b.kvh = contextual ? a.take<float>((size_t)hw_groups * n_hotwords * 1024) : nullptr;   // k | v rows of the hotword memories
  b.ctx_planes = tc ? a.take<plane_t>(gpl * Mq * 512) : nullptr;
  b.mem_planes = tc ? a.take<plane_t>(gpl * Mk * 512) : nullptr;      // split once, reused by every layer's k|v GEMM
  b.t1_planes = tc ? a.take<plane_t>(gpl * Mq * 512) : nullptr;       // LN outputs
  b.hq_planes = tc ? a.take<plane_t>(gpl * Mq * 2048) : nullptr;      // FFN hidden
  if (tc) b.att = attn_carve(a, batch, n_max, grouped ? mem_entries : batch, t_max, 512, mode);
  if (tc && (contextual || probs)) {
    // contextual: bias_q, bias_out (K 512) and bias_output (K 1024) over Mq rows; probs: q of n_max rows, k|v of t_max rows (K 512),
    // grouped: q of every row, k|v of every memory
    const size_t sc = contextual ? gemm_tc_scratch_bytes(Mq, 1024, mode) : 0;
    const size_t sp = !probs ? 0 : grouped ? gemm_tc_scratch_bytes(std::max(Mq, Mk), 512, mode) : gemm_tc_scratch_bytes(n_max > t_max ? n_max : t_max, 512, mode);
    b.scratch = a.sub(sc > sp ? sc : sp);
  }
  if (tc && contextual) {
    // the hotword k|v GEMM (hw_groups x n_hotwords rows, K 512), then the attention over the hotword memories
    const size_t sg = gemm_tc_scratch_bytes((int64_t)hw_groups * n_hotwords, 512, mode);
    const size_t sa = attention_tc_scratch_bytes(batch, 4, n_max, hw_groups, n_hotwords, mode);
    b.hw_scratch = a.sub(sg > sa ? sg : sa);
  }
  if (n_ints > 0) b.ints = a.take<int32_t>(n_ints);
}

extern "C" size_t fa_paraformer_decoder_workspace_bytes_hw(int32_t batch, int32_t t_max, int32_t n_max, int32_t vocab,
                                                           int32_t gemm_mode, int32_t n_hotwords) {
  Arena m = Arena::measuring();
  DecBuf b;
  dec_carve(m, b, batch, t_max, n_max, vocab, gemm_mode, n_hotwords, false);
  return m.bytes();
}

// The FFN shapes dec_ffn runs, checked by every decoder entry for each layer it will run before its first launch
static int dec_ffn_check(const FaDecLayer& L, int mode) {
  if (L.ffn_w1.in_f != 512 || L.ffn_w2.out_f != 512 || L.ffn_w2.in_f != L.ffn_w1.out_f || L.ffn_norm.n != L.ffn_w1.out_f) return FA_ERR_ARG;
  if (L.ffn_w1.out_f > 2048) return FA_ERR_UNSUPPORTED;    // dec_carve sizes hq / hq_planes for linear_units <= 2048
  if (mode != FA_GEMM_F32_SIMT && (L.ffn_w1.in_pad != 512 || L.ffn_w2.in_pad != L.ffn_w1.out_f)) return FA_ERR_UNSUPPORTED;
  return FA_OK;
}

static int dec_ffn(const FaDecLayer& L, const float* y, int64_t Mq, float* t1, float* hq, float* f, int mode,
                   Arena* scratch, cudaStream_t st, plane_t* t1_planes, plane_t* hq_planes) {
  // f = w_2( LN_2048( relu( w_1( LN1(y) ) ) ) )   decoder.py:97-100, sanm/positionwise_feed_forward.py:33
  if (mode != FA_GEMM_F32_SIMT) {
    const int npl = gemm_planes(mode);
    FA_RETURN_IF_ERR(layernorm_launch(y, Mq, L.norm1, nullptr, nullptr, 1.f, 1, st, t1_planes, npl, 512));
    FA_RETURN_IF_ERR(gemm_tc_planes_launch(t1_planes, Mq, L.ffn_w1, GemmEpi().relu().to(hq, L.ffn_w1.out_f), mode, st));
    FA_RETURN_IF_ERR(layernorm_launch(hq, Mq, L.ffn_norm, nullptr, nullptr, 1.f, 1, st, hq_planes, npl, L.ffn_w1.out_f));
    return gemm_tc_planes_launch(hq_planes, Mq, L.ffn_w2, GemmEpi().to(f, 512), mode, st);
  }
  FA_RETURN_IF_ERR(layernorm_launch(y, Mq, L.norm1, t1, nullptr, 1.f, 1, st));
  FA_RETURN_IF_ERR(gemm_rows(t1, 512, Mq, L.ffn_w1, GemmEpi().relu().to(hq, L.ffn_w1.out_f), mode, scratch, st));
  FA_RETURN_IF_ERR(layernorm_launch(hq, Mq, L.ffn_norm, hq, nullptr, 1.f, 1, st));
  return gemm_rows(hq, L.ffn_w1.out_f, Mq, L.ffn_w2, GemmEpi().to(f, 512), mode, scratch, st);
}

// Cross-attention probabilities of the probed utterances (DecoderLayerSANM.get_attn_mat, decoder.py:123-146 ->
// MultiHeadedAttentionCrossAtt.forward_attention with ret_attn, sanm/attention.py:760-794): probs[p, h, n, t] =
// softmax_t( (q[b, n, h] * d_k^-0.5) . k[g, t, h] ) for utterance b = rows[p] (NULL: utterance 0) over memory g = kv_index[b] (NULL:
// memory 0), with keys t >= key_lens[b] masked to -inf before and to 0 after the softmax.  SeACo's attention-score filtering sums this
// matrix over heads and tokens on the host exactly like the reference (seaco_paraformer/model.py:325-328), so the matrix itself is the
// output.  One warp per (probe, head, query); tiny (N x n_hotwords).
__global__ void __launch_bounds__(128)
attn_probs_kernel(const float* __restrict__ q, int64_t ldq, const float* __restrict__ k, int64_t ldk, int heads, int n_q, int t_k,
                  const int32_t* __restrict__ key_lens, const int32_t* __restrict__ rows, const int32_t* __restrict__ kv_index, int n_probe,
                  float qscale, float* __restrict__ probs) {
  extern __shared__ float s_sc[];                       // [4 warps][t_k]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + warp;                // (p * heads + h) * n_q + n
  if (row >= n_probe * heads * n_q) return;
  const int n = row % n_q, h = (row / n_q) % heads, p = row / (n_q * heads);
  const int b = rows ? rows[p] : 0;
  const int klen = min(key_lens[b], t_k);
  float* sc = s_sc + warp * t_k;
  const float* qr = q + ((int64_t)b * n_q + n) * ldq + h * 128;
  k += (int64_t)(kv_index ? kv_index[b] : 0) * t_k * ldk;
  float qv[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) qv[j] = __fmul_rn(qr[lane + 32 * j], qscale);
  float mx = -INFINITY;
  for (int t = 0; t < t_k; ++t) {
    const float* kr = k + (int64_t)t * ldk + h * 128;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc = fmaf(qv[j], kr[lane + 32 * j], acc);
    acc = warp_sum(acc);
    const float sv = t < klen ? acc : -INFINITY;
    if (lane == 0) sc[t] = sv;
    mx = fmaxf(mx, sv);
  }
  __syncwarp();
  float sum = 0.f;
  for (int t = lane; t < t_k; t += 32) { const float e = t < klen ? expf(sc[t] - mx) : 0.f; sc[t] = e; sum += e; }
  sum = warp_sum(sum);
  __syncwarp();
  for (int t = lane; t < t_k; t += 32) probs[(int64_t)row * t_k + t] = t < klen ? sc[t] / sum : 0.f;
}

// attn_probs_kernel's dynamic shared memory: one row of t_k scores per warp; above 48 KB it needs the opt-in
static size_t attn_probs_smem(int t_k) { return (size_t)4 * t_k * sizeof(float); }
static const size_t kAttnProbsMaxSmem = 96 * 1024;

// One run of a SAN-M decoder stack over a cross-attention memory.  memory [mem_batch * t_mem, 512] with mem_batch = batch, or 1
// when mem_shared (the SeACo / contextual hotword memory: every utterance attends over the same rows — one k/v projection, one
// copy), or mem_entries when utterance b attends over memory kv_index[b] (device).  tgt [batch, n_max, 512] lives in b.ya on entry.
// The ASF probe reads utterances probe_rows[0 .. n_probe) (device; NULL: utterance 0).
struct DecRun {
  int batch, n_max, t_mem, heads, fsmn_k, mode, mem_shared;
  const float* memory; const int32_t* mem_lens; const int32_t* tok_lens;
  cudaStream_t st;
  DecBuf* b; Arena* scratch;
  int mem_entries = 0;
  const int32_t* kv_index = nullptr;
  const int32_t* probe_rows = nullptr;
  int n_probe = 1;
  int64_t Mq() const { return (int64_t)batch * n_max; }
  int64_t Mk() const { return (int64_t)(kv_index ? mem_entries : mem_shared ? 1 : batch) * t_mem; }
};

// One attention decoder layer (DecoderLayerSANM.forward, paraformer/decoder.py:78-121).  *x_self_out receives `residual +
// fsmn(...)` (x_self_attn); if src_out != nullptr the cross-attention output is written there WITHOUT the residual (x_src_attn,
// leading dim ld_src) and *y_next is not produced — the ContextualDecoderLayer contract (contextual_paraformer/decoder.py:60-100).
// attn_probs != nullptr: stop at the cross-attention and write the probed utterances' probability matrices [n_probe, heads, n_max,
// t_mem] instead (get_attn_mat, decoder.py:123-146).
static int dec_attention_layer(const DecRun& r, const FaDecLayer& L, float* yin, float** x_self_out, float* src_out, int64_t ld_src,
                               float** y_next, float* attn_probs) {
  DecBuf& b = *r.b;
  const int D = 512;
  const int64_t Mq = r.Mq(), Mk = r.Mk();
  const bool tc = r.mode != FA_GEMM_F32_SIMT;
  const int npl = gemm_planes(r.mode);
  AttnShape shape{r.batch, r.heads, 128, r.n_max, r.t_mem, r.mem_shared};
  shape.kv_batch = r.mem_entries; shape.kv_index = r.kv_index;
  cudaStream_t st = r.st;
  FA_RETURN_IF_ERR(dec_ffn(L, yin, Mq, b.t1, b.hq, b.f, r.mode, r.scratch, st, b.t1_planes, b.hq_planes));
  // x = residual + fsmn(LN2(f), tgt_mask)     decoder.py:103-107
  FA_RETURN_IF_ERR(layernorm_launch(b.f, Mq, L.norm2, b.t1, nullptr, 1.f, 1, st));
  float* x2 = (yin == b.ya) ? b.yb : b.ya;
  FA_RETURN_IF_ERR(fsmn_launch(b.t1, D, r.tok_lens, r.batch, r.n_max, D, L.fsmn_w, r.fsmn_k, yin, D, x2, D, st));
  *x_self_out = x2;
  if (attn_probs) {
    // q / k in fp32 through the mode's GEMM; only utterance 0's rows are needed (seaco_paraformer/model.py:325: hotword_scores[0]),
    // or with a probe list every utterance's rows over every memory
    const int64_t mq = r.probe_rows ? Mq : r.n_max, mk = r.kv_index ? Mk : r.t_mem;
    FA_RETURN_IF_ERR(layernorm_launch(x2, mq, L.norm3, b.t1, nullptr, 1.f, 1, st));
    FA_RETURN_IF_ERR(gemm_rows(b.t1, D, mq, L.q, GemmEpi().to(b.qd, D), r.mode, r.scratch, st));
    FA_RETURN_IF_ERR(gemm_rows(r.memory, D, mk, L.kv, GemmEpi().to(b.kv, 2 * D), r.mode, r.scratch, st));
    const int rows = r.n_probe * r.heads * r.n_max;
    const size_t smem = attn_probs_smem(r.t_mem);              // <= kAttnProbsMaxSmem: checked by the entry point
    if (smem > 48 * 1024) FA_CUDA_OK(cudaFuncSetAttribute(attn_probs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attn_probs_kernel<<<(rows + 3) / 4, 128, smem, st>>>(b.qd, D, b.kv, 2 * D, r.heads, r.n_max, r.t_mem, r.mem_lens, r.probe_rows, r.kv_index,
                                                         r.n_probe, attn_qscale(shape.head_dim), attn_probs);
    FA_CHECK_LAUNCH();
    return FA_OK;
  }
  // x = residual + src_attn(LN3(x), memory)    decoder.py:109-118, attention.py:796-813
  if (tc) {
    FA_RETURN_IF_ERR(layernorm_launch(x2, Mq, L.norm3, nullptr, nullptr, 1.f, 1, st, b.t1_planes, npl, D));
    const AttnSinks sq = attn_sinks(b.att, 0, -1, -1, D, r.n_max, attn_qscale(shape.head_dim));   // q -> scaled fp16 planes only (no fp32 round trip)
    FA_RETURN_IF_ERR(gemm_tc_planes_launch(b.t1_planes, Mq, L.q, GemmEpi().sinks(&sq), r.mode, st));
  } else {
    FA_RETURN_IF_ERR(layernorm_launch(x2, Mq, L.norm3, b.t1, nullptr, 1.f, 1, st));
    FA_RETURN_IF_ERR(gemm_rows(b.t1, D, Mq, L.q, GemmEpi().to(b.qd, D), r.mode, r.scratch, st));
  }
  float* y2 = (x2 == b.ya) ? b.yb : b.ya;
  float* dst = src_out ? src_out : y2;
  const int64_t ldd = src_out ? ld_src : D;
  const float* res = src_out ? nullptr : x2;
  if (!tc) {
    FA_RETURN_IF_ERR(gemm_rows(r.memory, D, Mk, L.kv, GemmEpi().to(b.kv, 2 * D), r.mode, r.scratch, st));
    FA_RETURN_IF_ERR(attention_rows(b.qd, D, b.kv, 2 * D, b.kv + D, 2 * D, shape, r.mem_lens, AttnOut().to(b.ctx, D), r.mode, nullptr, st));
    FA_RETURN_IF_ERR(gemm_rows(b.ctx, D, Mq, L.out, GemmEpi().add(res, D).to(dst, ldd), r.mode, r.scratch, st));
  } else {
    const AttnSinks skv = attn_sinks(b.att, -1, 0, D, D, r.t_mem, 1.f);   // k -> planes, v -> transposed planes; nothing in fp32
    FA_RETURN_IF_ERR(gemm_tc_planes_launch(b.mem_planes, Mk, L.kv, GemmEpi().sinks(&skv), r.mode, st));
    FA_RETURN_IF_ERR(attention_planes(b.att, shape, r.mem_lens, AttnOut().to(b.ctx_planes, D, npl), st));
    FA_RETURN_IF_ERR(gemm_tc_planes_launch(b.ctx_planes, Mq, L.out, GemmEpi().add(res, D).to(dst, ldd), r.mode, st));
  }
  if (y_next) *y_next = y2;
  return FA_OK;
}

// decoders3 (FFN only, no residual: decoder.py:97-102,121) + after_norm -> hidden fp32 (optional) and/or planes for output_layer
static int dec_finish(const DecRun& r, const FaDecoder* dec, float* y, float* hidden_out) {
  DecBuf& b = *r.b;
  const bool tc = r.mode != FA_GEMM_F32_SIMT;
  FA_RETURN_IF_ERR(dec_ffn(dec->last, y, r.Mq(), b.t1, b.hq, b.f, r.mode, r.scratch, r.st, b.t1_planes, b.hq_planes));
  if (tc) return layernorm_launch(b.f, r.Mq(), dec->after_norm, hidden_out, nullptr, 1.f, 1, r.st, b.t1_planes, gemm_planes(r.mode), 512);
  return layernorm_launch(b.f, r.Mq(), dec->after_norm, hidden_out ? hidden_out : b.t1, nullptr, 1.f, 1, r.st);
}

// The contextual decoder's hotword memories: groups x nh_max rows of 512 (device); per utterance its key count and its memory (device;
// index NULL: memory 0).  rows_h (host, grouped entry only): [lens | index] per utterance, copied into the workspace.
struct HwMem {
  const float* embed; const int32_t* lens; const int32_t* index; int groups, nh_max;
  const int32_t* rows_h = nullptr;
};

static int decoder_forward_impl(const FaDecoder* dec, const float* enc, const int32_t* enc_lens, int32_t batch, int32_t t_max,
                                const float* acoustic, int64_t ld_acoustic_rows, const int32_t* tok_lens, int32_t n_max,
                                int32_t* argmax_ids, float* argmax_logp, float* logits, int32_t log_softmax, float* hidden_out,
                                int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream, const HwMem* grouped = nullptr) {
  if (!dec || !enc || !enc_lens || !acoustic || !tok_lens || !argmax_ids || !argmax_logp || batch <= 0 || t_max <= 0 ||
      n_max <= 0 || ld_acoustic_rows < n_max)
    return FA_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int D = 512;
  if (dec->after_norm.n != D || dec->heads * 128 != D) return FA_ERR_UNSUPPORTED;
  const int64_t Mq = (int64_t)batch * n_max, Mk = (int64_t)batch * t_max;
  const int V = dec->vocab;
  const bool tc = gemm_mode != FA_GEMM_F32_SIMT;
  const bool contextual = dec->has_bias != 0;
  HwMem hw = grouped ? *grouped : HwMem{dec->hw_embed, dec->hw_lens, nullptr, 1, dec->n_hotwords};
  if (contextual && (!hw.embed || (!grouped && !hw.lens) || hw.nh_max <= 0 || dec->clas_scale != 1.0f)) return FA_ERR_UNSUPPORTED;
  for (int l = 0; l < dec->n_layers; ++l) FA_RETURN_IF_ERR(dec_ffn_check(dec->layers[l], gemm_mode));   // nothing enqueued on a refusal
  if (contextual) FA_RETURN_IF_ERR(dec_ffn_check(dec->bias_last, gemm_mode));
  FA_RETURN_IF_ERR(dec_ffn_check(dec->last, gemm_mode));
  Arena a(workspace, ws_bytes);
  DecBuf b;
  dec_carve(a, b, batch, t_max, n_max, V, gemm_mode, contextual ? hw.nh_max : 0, false, hw.groups, 0, grouped ? 2 * batch : 0);
  if (!a.ok()) return FA_ERR_WORKSPACE;
  if (grouped) {
    FA_CUDA_OK(cudaMemcpyAsync(b.ints, hw.rows_h, (size_t)2 * batch * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    hw.lens = b.ints; hw.index = b.ints + batch;
  }
  const int npl = gemm_planes(gemm_mode);
  float* lg = logits ? logits : b.lg;
  if (tc) FA_RETURN_IF_ERR(split_rows_launch(enc, D, Mk, D, D, npl, b.mem_planes, st));   // memory is layer-invariant

  // tgt = acoustic[:, :n_max]  (decoder.py:424)
  FA_CUDA_OK(cudaMemcpy2DAsync(b.ya, (size_t)n_max * D * 4, acoustic, (size_t)ld_acoustic_rows * D * 4, (size_t)n_max * D * 4,
                               batch, cudaMemcpyDeviceToDevice, st));
  fa::count_launch();
  DecRun r{batch, n_max, t_max, dec->heads, dec->fsmn_k, gemm_mode, 0, enc, enc_lens, tok_lens, st, &b, &b.scratch};
  float* y = b.ya;
  for (int l = 0; l < dec->n_layers; ++l) {
    float* xs = nullptr;
    FA_RETURN_IF_ERR(dec_attention_layer(r, dec->layers[l], y, &xs, nullptr, 0, &y, nullptr));
  }
  if (contextual) {
    // ContextualParaformerDecoder.forward decoder.py:325-340
    float* x_self = nullptr;
    FA_RETURN_IF_ERR(dec_attention_layer(r, dec->bias_last, y, &x_self, b.cat, 2 * D, nullptr, nullptr));      // cat[:, :512] = x_src_attn
    // bias decoder: cross attention of LN3(x_self_attn) over the hotword memory (identical for every utterance)
    FA_RETURN_IF_ERR(layernorm_launch(x_self, Mq, dec->bias_norm3, b.t1, nullptr, 1.f, 1, st));
    FA_RETURN_IF_ERR(gemm_rows(b.t1, D, Mq, dec->bias_q, GemmEpi().to(b.qd, D), gemm_mode, &b.scratch, st));
    // the hotword k | v rows [groups, nh_max, 1024]: one copy per memory (no per-utterance replication, so the hotword count is
    // independent of t_max), each utterance attending over its own; one memory is the kv_shared case
    float* kvh = b.kvh;
    FA_RETURN_IF_ERR(gemm_rows(hw.embed, D, (int64_t)hw.groups * hw.nh_max, dec->bias_kv, GemmEpi().to(kvh, 2 * D), gemm_mode, &b.hw_scratch, st));
    AttnShape hs{batch, dec->heads, 128, n_max, hw.nh_max, 1};
    hs.kv_batch = hw.groups; hs.kv_index = hw.index;
    FA_RETURN_IF_ERR(attention_rows(b.qd, D, kvh, 2 * D, kvh + D, 2 * D, hs, hw.lens, AttnOut().to(b.ctx, D), gemm_mode, &b.hw_scratch, st));
    FA_RETURN_IF_ERR(gemm_rows(b.ctx, D, Mq, dec->bias_out, GemmEpi().to(b.cat + D, 2 * D), gemm_mode, &b.scratch, st));   // cat[:, 512:] = cx
    float* y2 = (x_self == b.ya) ? b.yb : b.ya;
    FA_RETURN_IF_ERR(gemm_rows(b.cat, 2 * D, Mq, dec->bias_output, GemmEpi().add(x_self, D).to(y2, D), gemm_mode, &b.scratch, st));
    y = y2;
  }
  // decoders3, after_norm (-> hidden), output_layer
  FA_RETURN_IF_ERR(dec_finish(r, dec, y, hidden_out));
  if (tc) {
    FA_RETURN_IF_ERR(gemm_tc_planes_launch(b.t1_planes, Mq, dec->output, GemmEpi().to(lg, V), gemm_mode, st));
  } else {
    FA_RETURN_IF_ERR(gemm_rows(hidden_out ? hidden_out : b.t1, D, Mq, dec->output, GemmEpi().to(lg, V), gemm_mode, nullptr, st));
  }
  return argmax_lse_launch(lg, Mq, V, V, argmax_ids, argmax_logp, (logits && log_softmax) ? 1 : 0, st);
}

extern "C" int fa_paraformer_decoder_forward(const FaDecoder* dec, const float* enc, const int32_t* enc_lens,
                                             int32_t batch, int32_t t_max, const float* acoustic,
                                             int64_t ld_acoustic_rows, const int32_t* tok_lens, int32_t n_max,
                                             int32_t* argmax_ids, float* argmax_logp, float* logits, int32_t log_softmax,
                                             int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream) {
  return decoder_forward_impl(dec, enc, enc_lens, batch, t_max, acoustic, ld_acoustic_rows, tok_lens, n_max, argmax_ids, argmax_logp,
                              logits, log_softmax, nullptr, gemm_mode, workspace, ws_bytes, stream);
}

// return_hidden + return_both (decoder.py:441-449): additionally writes the after_norm output [B, n_max, 512]
extern "C" int fa_paraformer_decoder_forward_hidden(const FaDecoder* dec, const float* enc, const int32_t* enc_lens,
                                                    int32_t batch, int32_t t_max, const float* acoustic,
                                                    int64_t ld_acoustic_rows, const int32_t* tok_lens, int32_t n_max,
                                                    int32_t* argmax_ids, float* argmax_logp, float* logits, int32_t log_softmax,
                                                    float* hidden, int32_t gemm_mode, void* workspace, size_t ws_bytes,
                                                    fa_stream_t stream) {
  if (!hidden) return FA_ERR_ARG;
  return decoder_forward_impl(dec, enc, enc_lens, batch, t_max, acoustic, ld_acoustic_rows, tok_lens, n_max, argmax_ids, argmax_logp,
                              logits, log_softmax, hidden, gemm_mode, workspace, ws_bytes, stream);
}

// rows_h [2 * batch] = [key count | memory] per utterance from lens_h [groups] and group_h [batch] (host), every group's length in
// [1, nh_max] and every utterance's group in [0, groups); false: a refusal
static bool hw_rows_host(const int32_t* lens_h, const int32_t* group_h, int32_t groups, int32_t nh_max, int32_t batch, std::vector<int32_t>& rows_h) {
  if (!lens_h || !group_h || groups < 1 || nh_max < 1 || batch < 1) return false;
  for (int32_t g = 0; g < groups; ++g)
    if (lens_h[g] < 1 || lens_h[g] > nh_max) return false;
  rows_h.resize((size_t)2 * batch);
  for (int32_t b = 0; b < batch; ++b) {
    if (group_h[b] < 0 || group_h[b] >= groups) return false;
    rows_h[b] = lens_h[group_h[b]];
    rows_h[batch + b] = group_h[b];
  }
  return true;
}

extern "C" size_t fa_paraformer_decoder_grouped_workspace_bytes(int32_t batch, int32_t t_max, int32_t n_max, int32_t vocab, int32_t gemm_mode,
                                                                int32_t n_groups, int32_t nh_max) {
  if (batch < 1 || n_groups < 1 || nh_max < 1) return 0;
  Arena m = Arena::measuring();
  DecBuf b;
  dec_carve(m, b, batch, t_max, n_max, vocab, gemm_mode, nh_max, false, n_groups, 0, 2 * batch);
  return m.bytes();
}

extern "C" int fa_paraformer_decoder_forward_grouped(const FaDecoder* dec, const float* enc, const int32_t* enc_lens, int32_t batch, int32_t t_max,
                                                     const float* acoustic, int64_t ld_acoustic_rows, const int32_t* tok_lens, int32_t n_max,
                                                     int32_t* argmax_ids, float* argmax_logp, float* logits, int32_t log_softmax, float* hidden,
                                                     const float* hw_embed, const int32_t* hw_lens_h, const int32_t* row_group_h, int32_t n_groups,
                                                     int32_t nh_max, int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream) {
  std::vector<int32_t> rows_h;
  if (!dec || !dec->has_bias || !hw_embed || !hw_rows_host(hw_lens_h, row_group_h, n_groups, nh_max, batch, rows_h)) return FA_ERR_ARG;
  HwMem hw{hw_embed, nullptr, nullptr, n_groups, nh_max, rows_h.data()};
  return decoder_forward_impl(dec, enc, enc_lens, batch, t_max, acoustic, ld_acoustic_rows, tok_lens, n_max, argmax_ids, argmax_logp,
                              logits, log_softmax, hidden, gemm_mode, workspace, ws_bytes, stream, &hw);
}

// A SAN-M decoder stack WITHOUT input / output layer over an arbitrary memory — the SeACo decoder of SeacoParaformer
// (seaco_paraformer/model.py:100-110: ParaformerSANMDecoder(use_output_layer=False, wo_input_layer=True), FFN 1024, FSMN k = 21,
// 6 attention layers) attending over the hotword embeddings.  mem_shared != 0: memory is [t_mem, 512], the same for every
// utterance (model.py:306-308 repeats `selected` over the batch).  n_run = attention layers to run (<= dec->n_layers);
//   finish != 0      -> decoders3 + after_norm, hidden [B, n_max, 512] (ParaformerSANMDecoder.forward, decoder.py:397-449)
//   attn_probs != 0  -> instead, layer n_run - 1 stops at its cross-attention and writes utterance 0's probability matrix
//                       [heads, n_max, t_mem] (forward_asf6 / get_attn_mat, decoder.py:485-513,123-146); hidden is not written.
extern "C" size_t fa_sanm_decoder_stack_workspace_bytes(int32_t batch, int32_t t_mem, int32_t n_max, int32_t gemm_mode) {
  Arena m = Arena::measuring();
  DecBuf b;
  dec_carve(m, b, batch, t_mem, n_max, 0, gemm_mode, 0, true);
  return m.bytes();
}

// The grouped stack's memories: groups of t_mem rows; ints_h (host) = [key count | memory] per utterance, then the probed utterances,
// copied into the workspace; or ints_d, the same already on the device (no copy)
struct StackGroups { int groups, n_probe; const int32_t* ints_h; const int32_t* ints_d = nullptr; };

static int stack_forward(const FaDecoder* dec, const float* memory, const int32_t* mem_lens, int32_t mem_shared, int32_t batch, int32_t t_mem,
                         const float* x, int64_t ld_x_rows, const int32_t* tok_lens, int32_t n_max, int32_t n_run, int32_t finish, float* hidden,
                         float* attn_probs, int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream, const StackGroups* grouped) {
  if (!dec || !memory || (!grouped && !mem_lens) || !x || !tok_lens || batch <= 0 || t_mem <= 0 || n_max <= 0 || ld_x_rows < n_max || n_run < 0 ||
      n_run > dec->n_layers || (!hidden && !attn_probs) || (attn_probs && n_run < 1))
    return FA_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int D = 512;
  if (dec->after_norm.n != D || dec->heads * 128 != D) return FA_ERR_UNSUPPORTED;
  for (int l = 0; l < n_run; ++l) FA_RETURN_IF_ERR(dec_ffn_check(dec->layers[l], gemm_mode));   // nothing enqueued on a refusal
  if (!attn_probs && finish) FA_RETURN_IF_ERR(dec_ffn_check(dec->last, gemm_mode));
  if (attn_probs && attn_probs_smem(t_mem) > kAttnProbsMaxSmem) return FA_ERR_UNSUPPORTED;
  const int n_ints = grouped ? 2 * batch + grouped->n_probe : 0;
  Arena a(workspace, ws_bytes);
  DecBuf b;
  dec_carve(a, b, batch, t_mem, n_max, 0, gemm_mode, 0, true, 1, grouped ? grouped->groups : 0, n_ints);
  if (!a.ok()) return FA_ERR_WORKSPACE;
  const bool tc = gemm_mode != FA_GEMM_F32_SIMT;
  DecRun r{batch, n_max, t_mem, dec->heads, dec->fsmn_k, gemm_mode, mem_shared ? 1 : 0, memory, mem_lens, tok_lens, st, &b, &b.scratch};
  if (grouped) {
    const int32_t* ints = grouped->ints_d;
    if (!ints) {
      FA_CUDA_OK(cudaMemcpyAsync(b.ints, grouped->ints_h, (size_t)n_ints * sizeof(int32_t), cudaMemcpyHostToDevice, st));
      ints = b.ints;
    }
    r.mem_lens = ints; r.kv_index = ints + batch; r.mem_entries = grouped->groups;
    r.probe_rows = ints + 2 * batch; r.n_probe = grouped->n_probe;
  }
  if (tc) FA_RETURN_IF_ERR(split_rows_launch(memory, D, r.Mk(), D, D, gemm_planes(gemm_mode), b.mem_planes, st));
  FA_CUDA_OK(cudaMemcpy2DAsync(b.ya, (size_t)n_max * D * 4, x, (size_t)ld_x_rows * D * 4, (size_t)n_max * D * 4, batch,
                               cudaMemcpyDeviceToDevice, st));
  fa::count_launch();
  float* y = b.ya;
  for (int l = 0; l < n_run; ++l) {
    float* xs = nullptr;
    const bool last_probs = attn_probs && l == n_run - 1;
    FA_RETURN_IF_ERR(dec_attention_layer(r, dec->layers[l], y, &xs, nullptr, 0, last_probs ? nullptr : &y, last_probs ? attn_probs : nullptr));
  }
  if (attn_probs) return FA_OK;
  if (finish) return dec_finish(r, dec, y, hidden);
  FA_CUDA_OK(cudaMemcpyAsync(hidden, y, (size_t)r.Mq() * D * 4, cudaMemcpyDeviceToDevice, st));
  fa::count_launch();
  return FA_OK;
}

extern "C" int fa_sanm_decoder_stack_forward(const FaDecoder* dec, const float* memory, const int32_t* mem_lens, int32_t mem_shared,
                                             int32_t batch, int32_t t_mem, const float* x, int64_t ld_x_rows,
                                             const int32_t* tok_lens, int32_t n_max, int32_t n_run, int32_t finish, float* hidden,
                                             float* attn_probs, int32_t gemm_mode, void* workspace, size_t ws_bytes,
                                             fa_stream_t stream) {
  return stack_forward(dec, memory, mem_lens, mem_shared, batch, t_mem, x, ld_x_rows, tok_lens, n_max, n_run, finish, hidden, attn_probs,
                       gemm_mode, workspace, ws_bytes, stream, nullptr);
}

namespace fa {
// fa_sanm_decoder_stack_forward_grouped without a probe, its per-utterance [key count | memory] already on the device (rows_d [2 * batch],
// checked by the caller): a caller that uploads them with its memories saves a host-to-device copy between two stacks
int sanm_stack_grouped_dev(const FaDecoder* dec, const float* memory, const int32_t* rows_d, int32_t n_groups, int32_t batch, int32_t t_mem,
                           const float* x, int64_t ld_x_rows, const int32_t* tok_lens, int32_t n_max, int32_t n_run, float* hidden, int32_t gemm_mode,
                           void* workspace, size_t ws_bytes, cudaStream_t st) {
  if (!rows_d || n_groups < 1 || !hidden) return FA_ERR_ARG;
  StackGroups g{n_groups, 0, nullptr};
  g.ints_d = rows_d;
  return stack_forward(dec, memory, nullptr, 0, batch, t_mem, x, ld_x_rows, tok_lens, n_max, n_run, 1, hidden, nullptr, gemm_mode, workspace,
                       ws_bytes, (fa_stream_t)st, &g);
}
}  // namespace fa

extern "C" size_t fa_sanm_decoder_stack_grouped_workspace_bytes(int32_t batch, int32_t n_groups, int32_t t_mem, int32_t n_max, int32_t n_probe,
                                                                int32_t gemm_mode) {
  if (batch < 1 || n_groups < 1 || t_mem < 1 || n_probe < 0) return 0;
  Arena m = Arena::measuring();
  DecBuf b;
  dec_carve(m, b, batch, t_mem, n_max, 0, gemm_mode, 0, true, 1, n_groups, 2 * batch + n_probe);
  return m.bytes();
}

extern "C" int fa_sanm_decoder_stack_forward_grouped(const FaDecoder* dec, const float* memory, const int32_t* mem_lens_h, const int32_t* row_group_h,
                                                     int32_t n_groups, int32_t batch, int32_t t_mem, const float* x, int64_t ld_x_rows,
                                                     const int32_t* tok_lens, int32_t n_max, int32_t n_run, int32_t finish, float* hidden,
                                                     float* attn_probs, const int32_t* probe_rows_h, int32_t n_probe, int32_t gemm_mode,
                                                     void* workspace, size_t ws_bytes, fa_stream_t stream) {
  std::vector<int32_t> ints;
  if (!hw_rows_host(mem_lens_h, row_group_h, n_groups, t_mem, batch, ints)) return FA_ERR_ARG;
  if (attn_probs && (!probe_rows_h || n_probe < 1)) return FA_ERR_ARG;
  if (!attn_probs) n_probe = 0;
  for (int32_t p = 0; p < n_probe; ++p) {
    if (probe_rows_h[p] < 0 || probe_rows_h[p] >= batch) return FA_ERR_ARG;
    ints.push_back(probe_rows_h[p]);
  }
  const StackGroups g{n_groups, n_probe, ints.data()};
  return stack_forward(dec, memory, nullptr, 0, batch, t_mem, x, ld_x_rows, tok_lens, n_max, n_run, finish, hidden, attn_probs, gemm_mode,
                       workspace, ws_bytes, stream, &g);
}

// SeACo merge (seaco_paraformer/model.py:357-378 with seaco_weight = 1): per token row, if argmax(dha_pred) == NO_BIAS keep the
// decoder's distribution, else take the hotword decoder's -> merged arg-max id and its log-probability; optionally the full
// merged log-prob rows (both inputs must then be log-softmax rows).
__global__ void seaco_merge_kernel(const int32_t* __restrict__ dec_ids, const float* __restrict__ dec_best, const int32_t* __restrict__ dha_ids,
                                   const float* __restrict__ dha_best, int64_t rows, int no_bias, int32_t* __restrict__ out_ids,
                                   float* __restrict__ out_best, const float* __restrict__ dec_logp, const float* __restrict__ dha_logp,
                                   float* __restrict__ merged, int vocab) {
  const int64_t row = blockIdx.x;
  const bool keep_dec = dha_ids[row] == no_bias;
  if (threadIdx.x == 0) {
    out_ids[row] = keep_dec ? dec_ids[row] : dha_ids[row];
    out_best[row] = keep_dec ? dec_best[row] : dha_best[row];
  }
  if (merged) {
    const float* src = (keep_dec ? dec_logp : dha_logp) + row * vocab;
    // dec * mask + dha * (1 - mask) with mask in {0, 1}: x * 1 + y * 0 — the reference's arithmetic keeps x bit for bit (finite y)
    for (int c = threadIdx.x; c < vocab; c += blockDim.x) merged[row * vocab + c] = src[c];
  }
}

extern "C" int fa_seaco_merge(const int32_t* dec_ids, const float* dec_best, const int32_t* dha_ids, const float* dha_best, int64_t rows,
                              int32_t no_bias, int32_t* out_ids, float* out_best, const float* dec_logp, const float* dha_logp,
                              float* merged, int32_t vocab, fa_stream_t stream) {
  if (!dec_ids || !dec_best || !dha_ids || !dha_best || !out_ids || !out_best || rows < 0) return FA_ERR_ARG;
  if (merged && (!dec_logp || !dha_logp || vocab <= 0)) return FA_ERR_ARG;
  if (rows == 0) return FA_OK;
  seaco_merge_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(dec_ids, dec_best, dha_ids, dha_best, rows, no_bias, out_ids, out_best,
                                                                      dec_logp, dha_logp, merged, vocab);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

// hotword_output_layer + log-softmax arg-max over hidden rows (seaco_paraformer/model.py:352-355): logits = (a + b) W^T + bias for
// the two attended streams a = cif_attended, b = dec_attended (model.py:351: merged = cif_attended + dec_attended).
// a + b (carved whether or not b is given), logits (whether or not the caller takes them), GEMM scratch for K <= 512
struct LinArgmaxBufs { float *sum, *lg; Arena scratch{nullptr, 0}; };
static LinArgmaxBufs lin_argmax_carve(Arena& a, int64_t rows, int vocab, int mode) {
  LinArgmaxBufs b;
  b.sum = a.take<float>((size_t)rows * 512);
  b.lg = a.take<float>((size_t)rows * vocab);
  if (mode != FA_GEMM_F32_SIMT) b.scratch = a.sub(gemm_tc_scratch_bytes(rows, 512, mode));
  return b;
}

extern "C" size_t fa_linear_argmax_workspace_bytes(int64_t rows, int32_t vocab, int32_t gemm_mode) {
  Arena m = Arena::measuring();
  lin_argmax_carve(m, rows, vocab, gemm_mode);
  return m.bytes();
}

__global__ void add_rows_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ o, int64_t n4) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 x = reinterpret_cast<const float4*>(a)[i], y = reinterpret_cast<const float4*>(b)[i];
  reinterpret_cast<float4*>(o)[i] = make_float4(__fadd_rn(x.x, y.x), __fadd_rn(x.y, y.y), __fadd_rn(x.z, y.z), __fadd_rn(x.w, y.w));
}

extern "C" int fa_linear_argmax(const FaLinear* lin, const float* a, const float* b_or_null, int64_t rows, int32_t* ids, float* best_logp,
                                float* logp, int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream) {
  if (!lin || !a || !ids || !best_logp || rows <= 0 || lin->in_f <= 0 || lin->in_f > 512 || (lin->in_f & 3)) return FA_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int V = lin->out_f, K = lin->in_f;
  Arena ar(workspace, ws_bytes);
  LinArgmaxBufs w = lin_argmax_carve(ar, rows, V, gemm_mode);
  if (!ar.ok()) return FA_ERR_WORKSPACE;
  const float* x = a;
  if (b_or_null) {
    const int64_t n4 = rows * (K / 4);
    add_rows_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, st>>>(a, b_or_null, w.sum, n4);
    FA_CHECK_LAUNCH();
    x = w.sum;
  }
  float* lg = logp ? logp : w.lg;
  FA_RETURN_IF_ERR(gemm_rows(x, K, rows, *lin, GemmEpi().to(lg, V), gemm_mode, &w.scratch, st));
  return argmax_lse_launch(lg, rows, V, V, ids, best_logp, logp ? 1 : 0, st);
}

// ------------------------------------------------------------------------------------------ CTC greedy head
// internal logits rows are pitched to a multiple of 4 floats (25055 -> 25056) so the GEMM epilogue and the arg-max sweep use
// 16-byte accesses (carved whether or not the caller takes the log-probs), best log-probs, GEMM scratch for K <= 512
struct CtcBufs { float *lg, *best; Arena scratch{nullptr, 0}; };
static CtcBufs ctc_carve(Arena& a, int64_t M, int vocab, int mode) {
  CtcBufs b;
  b.lg = a.take<float>(M * (size_t)((vocab + 3) & ~3));
  b.best = a.take<float>(M);
  if (mode != FA_GEMM_F32_SIMT) b.scratch = a.sub(gemm_tc_scratch_bytes(M, 512, mode));
  return b;
}

extern "C" size_t fa_ctc_greedy_workspace_bytes(int32_t batch, int32_t t_max, int32_t vocab, int32_t gemm_mode) {
  Arena m = Arena::measuring();
  ctc_carve(m, (int64_t)batch * t_max, vocab, gemm_mode);
  return m.bytes();
}

extern "C" int fa_ctc_greedy_forward(const FaLinear* ctc_lo, const float* enc, const int32_t* lens, int32_t batch,
                                     int32_t t_max, int32_t blank, int32_t* argmax_ids, int32_t* out_ids, int32_t* out_lens,
                                     float* logp, int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream) {
  if (!ctc_lo || !enc || !lens || !argmax_ids || !out_ids || !out_lens || batch <= 0 || t_max <= 0) return FA_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t M = (int64_t)batch * t_max;
  const int V = ctc_lo->out_f;
  Arena a(workspace, ws_bytes);
  CtcBufs w = ctc_carve(a, M, V, gemm_mode);
  if (!a.ok()) return FA_ERR_WORKSPACE;
  // a caller-provided log-prob tensor keeps the dense [M, V] layout
  const int64_t ldv = logp ? V : ((V + 3) & ~3);
  float* lg = logp ? logp : w.lg;
  FA_RETURN_IF_ERR(gemm_rows(enc, ctc_lo->in_f, M, *ctc_lo, GemmEpi().to(lg, ldv), gemm_mode, &w.scratch, st));
  FA_RETURN_IF_ERR(argmax_lse_launch(lg, M, V, ldv, argmax_ids, w.best, logp ? 1 : 0, st));
  return ctc_filter_launch(argmax_ids, lens, batch, t_max, blank, out_ids, out_lens, st);
}

// ------------------------------------------------------------------------------------------ op-level + info
extern "C" size_t fa_linear_workspace_bytes(int64_t rows, int32_t in_f, int32_t gemm_mode) {
  if (rows < 0 || in_f <= 0) return 0;
  return gemm_tc_scratch_bytes(rows, in_f, gemm_mode);
}

extern "C" int fa_linear(const float* x, int64_t ldx, int64_t rows, const FaLinear* lin, int32_t relu, const float* res1,
                         int64_t ld_res1, const float* res2, int64_t ld_res2, float* y, int64_t ldy, int32_t gemm_mode,
                         void* workspace, size_t ws_bytes, fa_stream_t stream) {
  if (!lin || !x || !y) return FA_ERR_ARG;
  Arena scratch(workspace, ws_bytes);
  return gemm_rows(x, ldx, rows, *lin, GemmEpi().relu(relu).add(res1, ld_res1, res2, ld_res2).to(y, ldy), gemm_mode, &scratch,
                   (cudaStream_t)stream);
}

extern "C" int fa_split_rows(const float* x, int64_t ldx, int64_t rows, int32_t cols, int32_t cols_pad, int32_t nplanes, void* planes,
                             fa_stream_t stream) {
  if (!x || !planes || nplanes < 1 || nplanes > 3) return FA_ERR_ARG;
  return split_rows_launch(x, ldx, rows, cols, cols_pad, nplanes, reinterpret_cast<plane_t*>(planes), (cudaStream_t)stream);
}

extern "C" int fa_linear_planes(const void* a_planes, int64_t rows, const FaLinear* lin, int32_t relu, const float* res1,
                                int64_t ld_res1, const float* res2, int64_t ld_res2, float* y, int64_t ldy, int32_t gemm_mode,
                                fa_stream_t stream) {
  if (!a_planes || !lin || !y || gemm_mode == FA_GEMM_F32_SIMT) return FA_ERR_ARG;
  return gemm_tc_planes_launch(reinterpret_cast<const plane_t*>(a_planes), rows, *lin,
                               GemmEpi().relu(relu).add(res1, ld_res1, res2, ld_res2).to(y, ldy), gemm_mode, (cudaStream_t)stream);
}

extern "C" int fa_linear_attn_sinks(const void* a_planes, int64_t rows, const FaLinear* lin, int32_t q0, int32_t k0, int32_t v0,
                                    int32_t width, int32_t t_rows, int32_t t_pad, float qscale, void* q_planes, void* k_planes,
                                    void* vt_planes, float* v_f32, int64_t ld_v_f32, int32_t gemm_mode, fa_stream_t stream) {
  if (!a_planes || !lin || rows < 0) return FA_ERR_ARG;
  if (gemm_mode != FA_GEMM_F16X1 && gemm_mode != FA_GEMM_F16X3 && gemm_mode != FA_GEMM_F16X6) return FA_ERR_ARG;
  const int N = lin->out_f;
  if (width <= 0 || width % 32 != 0 || t_rows <= 0 || rows % t_rows != 0) return FA_ERR_ARG;
  const int32_t start[3] = {q0, k0, v0};
  void* const dst[3] = {q_planes, k_planes, vt_planes};
  int n_on = 0;
  for (int i = 0; i < 3; ++i) {
    if (start[i] < 0) continue;                                   // disabled
    // the epilogue routes whole 16-column chunks, stores 8 bytes at a time, and writes nothing outside the range it was given
    if (start[i] % 16 != 0 || start[i] + width > N || !dst[i] || (reinterpret_cast<uintptr_t>(dst[i]) & 7)) return FA_ERR_ARG;
    for (int j = 0; j < i; ++j)
      if (start[j] >= 0 && start[i] < start[j] + width && start[j] < start[i] + width) return FA_ERR_ARG;   // overlapping sinks
    ++n_on;
  }
  if (n_on == 0) return FA_ERR_ARG;
  if (v0 >= 0 && t_pad < t_rows) return FA_ERR_ARG;
  if (v_f32 && (v0 < 0 || ld_v_f32 < N)) return FA_ERR_ARG;       // fp32 V rows are the GEMM's output rows: columns [v0, v0 + width)
  const AttnPlanes pl{static_cast<plane_t*>(q_planes), static_cast<plane_t*>(k_planes), static_cast<plane_t*>(vt_planes),
                      attn_planes(gemm_mode), t_pad};   // t_pad is read only by a v sink
  const AttnSinks sk = attn_sinks(pl, q0, k0, v0, width, t_rows, qscale);
  return gemm_tc_planes_launch(reinterpret_cast<const plane_t*>(a_planes), rows, *lin, GemmEpi().to(v_f32, ld_v_f32).sinks(&sk), gemm_mode,
                               (cudaStream_t)stream);
}

extern "C" int fa_linear_planes_to_planes(const void* a_planes, int64_t rows, const FaLinear* lin, int32_t relu, void* out_planes,
                                          int64_t ld_out, int32_t gemm_mode, fa_stream_t stream) {
  if (!a_planes || !lin || !out_planes || gemm_mode == FA_GEMM_F32_SIMT) return FA_ERR_ARG;
  return gemm_tc_planes_launch(reinterpret_cast<const plane_t*>(a_planes), rows, *lin,
                               GemmEpi().relu(relu).to(reinterpret_cast<plane_t*>(out_planes), ld_out), gemm_mode, (cudaStream_t)stream);
}

// The GEMM over an overlapping ("conv view") A operand, as the CIF conv and the CAM++ TDNN launch it: row r of plane p is the
// in_pad elements at (p * a_plane_rows + r) * a_ld.  a_plane_rows >= rows + ceil((in_pad - a_ld) / a_ld) keeps every valid row's
// span inside its own plane, which is also what the tensor map's row count (gemm_tc_planes_launch) relies on.
extern "C" int fa_linear_planes_view(const void* a_planes, int64_t rows, int64_t a_ld, int64_t a_plane_rows, const FaLinear* lin,
                                     int32_t relu, float* y, int64_t ldy, int32_t gemm_mode, fa_stream_t stream) {
  if (!a_planes || !lin || !y || rows < 0 || a_ld <= 0) return FA_ERR_ARG;
  if (gemm_mode != FA_GEMM_F16X1 && gemm_mode != FA_GEMM_F16X3 && gemm_mode != FA_GEMM_F16X6) return FA_ERR_ARG;
  if (a_ld % 8 != 0) return FA_ERR_UNSUPPORTED;
  const int64_t kp = lin->in_pad;
  const int64_t extra = a_ld < kp ? (kp - a_ld + a_ld - 1) / a_ld : 0;
  if (a_plane_rows < rows + extra) return FA_ERR_ARG;
  return gemm_tc_planes_launch(reinterpret_cast<const plane_t*>(a_planes), rows, *lin, GemmEpi().relu(relu).to(y, ldy), gemm_mode,
                               (cudaStream_t)stream, a_ld, a_plane_rows);
}

// rows of an embedding table: out[i, :] = table[ids[i], :] (torch.nn.Embedding forward, e.g. CTTransformer.embed ct_transformer/model.py:120)
__global__ void embedding_kernel(const int32_t* __restrict__ ids, const float* __restrict__ table, int dim, int vocab, int64_t n, float* __restrict__ out) {
  const int64_t i = blockIdx.x;
  const int id = min(max(ids[i], 0), vocab - 1);
  for (int c = threadIdx.x; c < dim; c += blockDim.x) out[i * dim + c] = table[(int64_t)id * dim + c];
}
extern "C" int fa_embedding(const int32_t* ids, const float* table, int32_t dim, int32_t vocab, int64_t n, float* out, fa_stream_t stream) {
  if (!ids || !table || !out || dim <= 0 || vocab <= 0 || n < 0) return FA_ERR_ARG;
  if (n == 0) return FA_OK;
  embedding_kernel<<<(unsigned)n, 128, 0, (cudaStream_t)stream>>>(ids, table, dim, vocab, n, out);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" const char* fa_version(void) { return "funasr_b200 0.1.0 (sm_90a)"; }
extern "C" uint64_t fa_launch_count(void) { return (uint64_t)fa::g_launch_count.load(); }
extern "C" const char* fa_status_string(int status) {
  switch (status) {
    case FA_OK: return "ok";
    case FA_ERR_ARG: return "bad argument";
    case FA_ERR_CUDA: return "CUDA error";
    case FA_ERR_WORKSPACE: return "workspace too small";
    case FA_ERR_UNSUPPORTED: return "unsupported shape";
    default: return "unknown";
  }
}
