// FSMN-VAD on the GPU: what FsmnVADStreaming feeds its end-point detector with, for the WHOLE waveform in one pass
// (funasr/models/fsmn_vad_streaming): the FSMN encoder (encoder.py:355-377: in_linear1 -> in_linear2 -> ReLU -> 4 x [linear (no
// bias) -> causal depthwise memory -> affine -> ReLU] -> out_linear1 -> out_linear2 -> softmax) reduced to the silence posterior
// the detector reads (sum of the `sil_pdf_ids` columns, model.py:789-792), and the frame energies of ComputeDecibel
// (model.py:458-529).  The reference evaluates the encoder on 60 s chunks with a per-layer cache of the last lorder-1 frames
// (encoder.py:146-151); the memory is causal, so one pass over all frames computes the same values.
// The layers are tiny (400-140-250-128-...-248): fp32 SIMT GEMMs (gemm_f32.cu; K padded to a multiple of 16 by the weight
// packer) and HBM-bound row kernels — a few hundred microseconds per minute of audio.  The sequential decision logic over the
// posteriors stays on the host (funasr_b200/vad.py), as in the reference.
#include "common.cuh"
#include "kernels.h"
#include <math.h>
#include <algorithm>
#include <vector>

namespace fa {

// one warp per row: softmax over n logits -> sum of the silence columns (+ the full row when scores != nullptr)
__global__ void __launch_bounds__(256)
vad_softmax_sil_kernel(const float* __restrict__ logits, int64_t ld, int rows, int n, const int32_t* __restrict__ sil_ids, int n_sil,
                       float* __restrict__ sil_prob, float* __restrict__ scores) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* x = logits + (int64_t)row * ld;
  float mx = -INFINITY;
  for (int c = lane; c < n; c += 32) mx = fmaxf(mx, x[c]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = lane; c < n; c += 32) sum += expf(x[c] - mx);
  sum = warp_sum(sum);
  if (scores) for (int c = lane; c < n; c += 32) scores[(int64_t)row * n + c] = expf(x[c] - mx) / sum;
  if (lane == 0) {
    float p = 0.f;
    for (int k = 0; k < n_sil; ++k) p += expf(x[sil_ids[k]] - mx) / sum;
    sil_prob[row] = p;
  }
}

// 10 log10(sum x^2 + 1e-6) over the 400-sample frame starting at 160 t (ComputeDecibel model.py:516-525); one warp per frame.
// Row b of a ragged batch: wav + b * stride, frames[b] frames, db + b * t_max (frames == nullptr: one row of t_max frames).
__global__ void __launch_bounds__(256)
frame_decibel_kernel(const float* __restrict__ wav, int64_t stride, const int32_t* __restrict__ frames, int t_max, float* __restrict__ db) {
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, b = blockIdx.y;
  if (t >= (frames ? min(frames[b], t_max) : t_max)) return;
  const float* x = wav + (int64_t)b * stride + (int64_t)t * 160;
  float s = 0.f;
  for (int j = lane; j < 400; j += 32) s = fmaf(x[j], x[j], s);
  s = warp_sum(s);
  if (lane == 0) db[(int64_t)b * t_max + t] = 10.f * log10f(s + 0.000001f);
}

static inline int pad16(int k) { return (k + 15) / 16 * 16; }

// Activations at their padded widths, then the metadata.  The order matters: the forward zeroes a1 .. meta as one range.
struct VadBufs {
  float *a1, *h0, *h1, *q, *qm, *o1, *lg;
  int32_t* meta;   // [0..4) = silence ids, [8..8 + batch) = each row's frames; at least 16 entries
};
static VadBufs vad_carve(Arena& a, const FaVadEncoder* enc, int batch, int t) {
  const int Ap = pad16(enc->in1.out_f), Lp = pad16(enc->in2.out_f), Op = pad16(enc->out1.out_f), Vp = pad16(enc->out2.out_f);
  const size_t rows = (size_t)batch * t;
  VadBufs b;
  b.a1 = a.take<float>(rows * Ap);
  b.h0 = a.take<float>(rows * Lp);
  b.h1 = a.take<float>(rows * Lp);
  b.q = a.take<float>(rows * 128);
  b.qm = a.take<float>(rows * 128);
  b.o1 = a.take<float>(rows * Op);
  b.lg = a.take<float>(rows * Vp);
  b.meta = a.take<int32_t>((size_t)std::max(16, 8 + batch));
  return b;
}

// The FSMN-VAD forward over `batch` rows of t_max frames (feats [batch * t_max, ld_feats], row b's frames[b] <= t_max valid; host
// array).  Every GEMM, the softmax and the row kernels compute each frame on its own, and the memory block is causal and masked at
// each row's length, so a row's valid frames are those of the row run alone.
static int vad_forward(const FaVadEncoder* enc, const float* feats, int64_t ld_feats, const int32_t* frames, int batch, int t_max,
                       float* sil_prob, float* scores, void* workspace, size_t ws_bytes, cudaStream_t st) {
  if (!enc || !feats || !sil_prob || !frames || batch <= 0 || t_max <= 0 || !enc->layers || enc->n_layers < 0 || enc->n_sil < 1 ||
      enc->n_sil > 4 || (int64_t)batch * t_max > 0x7fffffffLL)
    return FA_ERR_ARG;
  for (int b = 0; b < batch; ++b)
    if (frames[b] < 0 || frames[b] > t_max) return FA_ERR_ARG;
  const int A = enc->in1.out_f, L = enc->in2.out_f, O = enc->out1.out_f, V = enc->out2.out_f;
  const int Ap = pad16(A), Lp = pad16(L), Op = pad16(O), Vp = pad16(V);
  // every GEMM reads K = the previous layer's PADDED width (zero columns in the activations, zero columns in the packed weights)
  if (enc->in1.in_f % 16 || enc->in2.in_f != Ap || enc->out1.in_f != Lp || enc->out2.in_f != Op) return FA_ERR_UNSUPPORTED;
  Arena a(workspace, ws_bytes);
  const VadBufs b = vad_carve(a, enc, batch, t_max);
  if (!a.ok()) return FA_ERR_WORKSPACE;
  const int rows = batch * t_max;
  float *a1 = b.a1, *h0 = b.h0, *h1 = b.h1, *q = b.q, *qm = b.qm, *o1 = b.o1, *lg = b.lg;
  int32_t* meta = b.meta;
  FA_CUDA_OK(cudaMemsetAsync(a1, 0, (size_t)((char*)meta - (char*)a1), st));      // padded columns must read as zero
  std::vector<int32_t> host_meta((size_t)std::max(16, 8 + batch), 0);
  for (int k = 0; k < enc->n_sil; ++k) host_meta[k] = enc->sil_ids[k];
  for (int r = 0; r < batch; ++r) host_meta[8 + r] = frames[r];
  FA_CUDA_OK(cudaMemcpyAsync(meta, host_meta.data(), host_meta.size() * 4, cudaMemcpyHostToDevice, st));
  FA_RETURN_IF_ERR(gemm_f32_launch(feats, ld_feats, rows, enc->in1.w, A, enc->in1.in_f, enc->in1.b, GemmEpi().to(a1, Ap), st));
  FA_RETURN_IF_ERR(gemm_f32_launch(a1, Ap, rows, enc->in2.w, L, Ap, enc->in2.b, GemmEpi().relu().to(h0, Lp), st));
  float* h = h0;
  for (int l = 0; l < enc->n_layers; ++l) {
    const FaVadLayer& Y = enc->layers[l];
    if (Y.lin.out_f != 128 || Y.lin.in_f != Lp || Y.affine.in_f != 128 || Y.affine.out_f != L || !Y.conv_w) return FA_ERR_UNSUPPORTED;
    FA_RETURN_IF_ERR(gemm_f32_launch(h, Lp, rows, Y.lin.w, 128, Lp, nullptr, GemmEpi().to(q, 128), st));
    FA_RETURN_IF_ERR(fsmn_launch(q, 128, meta + 8, batch, t_max, 128, Y.conv_w, enc->lorder, nullptr, 0, qm, 128, st, 1));
    float* hn = (h == h0) ? h1 : h0;
    FA_RETURN_IF_ERR(gemm_f32_launch(qm, 128, rows, Y.affine.w, L, 128, Y.affine.b, GemmEpi().relu().to(hn, Lp), st));
    h = hn;
  }
  FA_RETURN_IF_ERR(gemm_f32_launch(h, Lp, rows, enc->out1.w, O, Lp, enc->out1.b, GemmEpi().to(o1, Op), st));
  FA_RETURN_IF_ERR(gemm_f32_launch(o1, Op, rows, enc->out2.w, V, Op, enc->out2.b, GemmEpi().to(lg, Vp), st));
  vad_softmax_sil_kernel<<<(rows + 7) / 8, 256, 0, st>>>(lg, Vp, rows, V, meta, enc->n_sil, sil_prob, scores);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

}  // namespace fa

using namespace fa;

extern "C" size_t fa_fsmn_vad_workspace_bytes(const FaVadEncoder* enc, int32_t t) {
  return fa_fsmn_vad_batch_workspace_bytes(enc, 1, t);
}

extern "C" size_t fa_fsmn_vad_batch_workspace_bytes(const FaVadEncoder* enc, int32_t batch, int32_t t_max) {
  if (!enc || batch <= 0 || t_max <= 0) return 0;
  Arena m = Arena::measuring();
  vad_carve(m, enc, batch, t_max);
  return m.bytes();
}

extern "C" int fa_fsmn_vad_forward(const FaVadEncoder* enc, const float* feats, int64_t ld_feats, int32_t t, float* sil_prob,
                                   float* scores, void* workspace, size_t ws_bytes, fa_stream_t stream) {
  return vad_forward(enc, feats, ld_feats, &t, 1, t, sil_prob, scores, workspace, ws_bytes, (cudaStream_t)stream);
}

extern "C" int fa_fsmn_vad_forward_batch(const FaVadEncoder* enc, const float* feats, int64_t ld_feats, const int32_t* frames, int32_t batch,
                                         int32_t t_max, float* sil_prob, void* workspace, size_t ws_bytes, fa_stream_t stream) {
  return vad_forward(enc, feats, ld_feats, frames, batch, t_max, sil_prob, nullptr, workspace, ws_bytes, (cudaStream_t)stream);
}

extern "C" int fa_frame_decibels(const float* wav, int64_t n_samples, int32_t frames, float* decibel, fa_stream_t stream) {
  if (!wav || !decibel || frames < 0 || (frames > 0 && (int64_t)(frames - 1) * 160 + 400 > n_samples)) return FA_ERR_ARG;
  if (frames == 0) return FA_OK;
  frame_decibel_kernel<<<(frames + 7) / 8, 256, 0, (cudaStream_t)stream>>>(wav, 0, nullptr, frames, decibel);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" int fa_frame_decibels_batch(const float* wav, int64_t stride, const int32_t* frames, int32_t batch, int32_t t_max, float* decibel,
                                       fa_stream_t stream) {
  if (!wav || !frames || !decibel || batch < 0 || batch > 65535 || t_max < 0 || stride < 0) return FA_ERR_ARG;
  if (batch == 0 || t_max == 0) return FA_OK;
  frame_decibel_kernel<<<dim3((unsigned)((t_max + 7) / 8), (unsigned)batch), 256, 0, (cudaStream_t)stream>>>(wav, stride, frames, t_max, decibel);
  FA_CHECK_LAUNCH();
  return FA_OK;
}
