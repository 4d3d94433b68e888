// SeacoParaformer's hotword encoder (funasr/models/seaco_paraformer/model.py:384-420, `_hotword_representation`): decoder.embed over
// the hotword token ids, the n-layer LSTM `bias_encoder` (512 -> 512, batch_first) over the packed batch, and each hotword's top-layer
// output at its last token.  The one part of a SeACo request that grows with the hotword list (hundreds to thousands per call).
//
// The batch runs in PackedSequence order: hotwords sorted by length, longest first, so that step t works on the row prefix of the
// n_t hotwords longer than t, and the tokens of step t sit at rows [off_t, off_t + n_t) of every [tokens, *] buffer.  Per layer:
//   * one GEMM of this library over all tokens: xproj = x W_ih^T + (b_ih + b_hh)            (the bias folded by the model file)
//   * per step t >= 1 one GEMM gates = h_{t-1} W_hh^T + xproj_t over the n_t active rows (the residual epilogue adds xproj)
//   * per step one fused cell launch: sigmoid / tanh, c and h, h into the layer's output rows (the next layer's input); on the last
//     layer each hotword that ends at t scatters its h to the caller's row order.
// No host synchronisation between steps: every launch is stream ordered and the step shapes are known on the host up front.
#include "common.cuh"
#include "kernels.h"
#include <algorithm>
#include <vector>

namespace fa {

constexpr int HW_D = 512;           // inner_dim (SeacoParaformerB200 refuses other widths)
constexpr int HW_G = 4 * HW_D;      // gate rows i, f, g, o

__device__ __forceinline__ float hw_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// One LSTM step over the n_t active hotwords: thread = (hotword j, 4 consecutive units).  gates [n_t][2048] (i, f, g, o blocks), c [n][512]
// (read unless first), h_out [n_t][512]; rows != nullptr: hotwords j >= n_next end here and write h to rows[order[j]].
__global__ void __launch_bounds__(256)
hotword_cell_kernel(const float* __restrict__ gates, float* __restrict__ c, float* __restrict__ h_out, int n_t, int n_next, int first,
                    const int32_t* __restrict__ order, float* __restrict__ rows) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n_t * (HW_D / 4)) return;
  const int j = (int)(idx / (HW_D / 4)), u = (int)(idx % (HW_D / 4)) * 4;
  const float* g = gates + (int64_t)j * HW_G + u;
  const float4 i4 = *reinterpret_cast<const float4*>(g), f4 = *reinterpret_cast<const float4*>(g + HW_D);
  const float4 g4 = *reinterpret_cast<const float4*>(g + 2 * HW_D), o4 = *reinterpret_cast<const float4*>(g + 3 * HW_D);
  float* cp = c + (int64_t)j * HW_D + u;
  const float4 c0 = first ? make_float4(0.f, 0.f, 0.f, 0.f) : *reinterpret_cast<const float4*>(cp);
  const float iv[4] = {i4.x, i4.y, i4.z, i4.w}, fv[4] = {f4.x, f4.y, f4.z, f4.w}, gv[4] = {g4.x, g4.y, g4.z, g4.w};
  const float ov[4] = {o4.x, o4.y, o4.z, o4.w}, cv[4] = {c0.x, c0.y, c0.z, c0.w};
  float cn[4], hn[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    cn[k] = hw_sigmoid(fv[k]) * cv[k] + hw_sigmoid(iv[k]) * tanhf(gv[k]);
    hn[k] = hw_sigmoid(ov[k]) * tanhf(cn[k]);
  }
  *reinterpret_cast<float4*>(cp) = make_float4(cn[0], cn[1], cn[2], cn[3]);
  const float4 h4 = make_float4(hn[0], hn[1], hn[2], hn[3]);
  *reinterpret_cast<float4*>(h_out + (int64_t)j * HW_D + u) = h4;
  if (rows && j >= n_next) *reinterpret_cast<float4*>(rows + (int64_t)order[j] * HW_D + u) = h4;
}

// The forward's workspace: the packed ids and the row order, two [tokens, 512] layer buffers (embeddings / layer outputs, ping-pong),
// the input projections [tokens, 2048], one step's gates [n_hw, 2048], the cell state [n_hw, 512], and GEMM scratch for the largest
// A operand (all tokens, K = 512)
struct HwBufs { int32_t* io; float *xa, *xb, *xproj, *gates, *c; Arena gemm{nullptr, 0}; };
static HwBufs hw_carve(Arena& a, int64_t n_hw, int64_t n_tok, int mode) {
  HwBufs b;
  b.io = a.take<int32_t>((size_t)(n_tok + n_hw));
  b.xa = a.take<float>((size_t)n_tok * HW_D);
  b.xb = a.take<float>((size_t)n_tok * HW_D);
  b.xproj = a.take<float>((size_t)n_tok * HW_G);
  b.gates = a.take<float>((size_t)n_hw * HW_G);
  b.c = a.take<float>((size_t)n_hw * HW_D);
  if (mode != FA_GEMM_F32_SIMT) b.gemm = a.sub(gemm_tc_scratch_bytes(n_tok, HW_D, mode));
  return b;
}

static bool hw_mode_ok(int mode) {
  return mode == FA_GEMM_F32_SIMT || mode == FA_GEMM_F16X1 || mode == FA_GEMM_F16X3 || mode == FA_GEMM_F16X6;
}

static bool hw_lin_ok(const FaLinear& L, bool bias, int mode) {
  return L.w && L.out_f == HW_G && L.in_f == HW_D && L.in_pad == HW_D && (bias == (L.b != nullptr)) &&
         (mode == FA_GEMM_F32_SIMT || L.w_planes);
}

}  // namespace fa

extern "C" size_t fa_hotword_encoder_workspace_bytes(int32_t n_hw, int64_t n_tokens, int32_t gemm_mode) {
  if (n_hw <= 0 || n_tokens < n_hw || !fa::hw_mode_ok(gemm_mode)) return 0;
  fa::Arena m = fa::Arena::measuring();
  fa::hw_carve(m, n_hw, n_tokens, gemm_mode);
  return m.bytes();
}

extern "C" int fa_hotword_encoder_forward(const FaHotwordEncoder* enc, const int32_t* ids, const int32_t* lens, int32_t n_hw, float* rows,
                                          int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream) {
  using namespace fa;
  if (!enc || !ids || !lens || !rows || n_hw <= 0 || !enc->embed || !enc->ih || !enc->hh || !hw_mode_ok(gemm_mode)) return FA_ERR_ARG;
  if (enc->n_layers < 1 || enc->n_layers > FA_HOTWORD_MAX_LAYERS || enc->vocab < 1) return FA_ERR_ARG;
  for (int l = 0; l < enc->n_layers; ++l)
    if (!hw_lin_ok(enc->ih[l], true, gemm_mode) || !hw_lin_ok(enc->hh[l], false, gemm_mode)) return FA_ERR_ARG;
  // host-side validation and the packed order, before anything is enqueued
  int64_t n_tok = 0;
  int t_max = 0;
  for (int32_t i = 0; i < n_hw; ++i) {
    if (lens[i] < 1) return FA_ERR_ARG;
    n_tok += lens[i];
    t_max = lens[i] > t_max ? lens[i] : t_max;
  }
  if (n_tok > 0x7fffffffLL / HW_G) return FA_ERR_UNSUPPORTED;
  for (int64_t k = 0; k < n_tok; ++k)
    if (ids[k] < 0 || ids[k] >= enc->vocab) return FA_ERR_ARG;
  Arena a(workspace, ws_bytes);
  HwBufs b = hw_carve(a, n_hw, n_tok, gemm_mode);
  if (!a.ok()) return FA_ERR_WORKSPACE;
  std::vector<int64_t> start(n_hw);                               // each hotword's first id in `ids`
  for (int32_t i = 0, s = 0; i < n_hw; s += lens[i], ++i) start[i] = s;
  std::vector<int32_t> order(n_hw);
  for (int32_t i = 0; i < n_hw; ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](int32_t x, int32_t y) { return lens[x] > lens[y]; });
  std::vector<int32_t> cnt(t_max + 1, 0);                         // cnt[t]: hotwords longer than t (a prefix of `order`)
  std::vector<int64_t> off(t_max + 1, 0);                         // first packed row of step t
  for (int32_t i = 0; i < n_hw; ++i) cnt[lens[i] - 1] += 1;
  for (int t = t_max - 1; t > 0; --t) cnt[t - 1] += cnt[t];
  for (int t = 0; t < t_max; ++t) off[t + 1] = off[t] + cnt[t];
  std::vector<int32_t> io((size_t)(n_tok + n_hw));
  for (int t = 0; t < t_max; ++t)
    for (int32_t j = 0; j < cnt[t]; ++j) io[off[t] + j] = ids[start[order[j]] + t];
  std::copy(order.begin(), order.end(), io.begin() + n_tok);
  cudaStream_t st = (cudaStream_t)stream;
  FA_CUDA_OK(cudaMemcpyAsync(b.io, io.data(), io.size() * 4, cudaMemcpyHostToDevice, st));   // pageable: staged before the return
  const int32_t* order_d = b.io + n_tok;
  FA_RETURN_IF_ERR(fa_embedding(b.io, enc->embed, HW_D, enc->vocab, n_tok, b.xa, stream));
  const float* x = b.xa;
  float* y = b.xb;
  for (int l = 0; l < enc->n_layers; ++l) {
    const bool last = l == enc->n_layers - 1;
    FA_RETURN_IF_ERR(gemm_rows(x, HW_D, n_tok, enc->ih[l], GemmEpi().to(b.xproj, HW_G), gemm_mode, &b.gemm, st));
    for (int t = 0; t < t_max; ++t) {
      const int n_t = cnt[t], n_next = cnt[t + 1];
      const float* g = b.xproj;                                   // t = 0: h_{-1} = 0, the gates are the input projections
      if (t > 0) {
        FA_RETURN_IF_ERR(gemm_rows(y + off[t - 1] * HW_D, HW_D, n_t, enc->hh[l], GemmEpi().add(b.xproj + off[t] * HW_G, HW_G).to(b.gates, HW_G),
                                   gemm_mode, &b.gemm, st));
        g = b.gates;
      }
      const int64_t threads = (int64_t)n_t * (HW_D / 4);
      hotword_cell_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(g, b.c, y + off[t] * HW_D, n_t, n_next, t == 0 ? 1 : 0, order_d,
                                                                             last ? rows : nullptr);
      FA_CHECK_LAUNCH();
    }
    x = y;
    y = (y == b.xb) ? b.xa : b.xb;
  }
  return FA_OK;
}
