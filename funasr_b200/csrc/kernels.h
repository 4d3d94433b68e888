// Internal launch helpers shared between translation units (not part of the C ABI).
#pragma once
#include "common.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

namespace fa { typedef __half plane_t; }   // 16-bit operand plane element (tc_common.cuh)

namespace fa {

// y (fp32) and/or planes (fp16 [nplanes][rows][cols_pad], the A operand of a following tensor-core GEMM)
int layernorm_launch(const float* x, int64_t rows, const FaNorm& nm, float* y, const float* pe_inv, float xscale,
                     int rows_per_batch, cudaStream_t st, plane_t* planes = nullptr, int nplanes = 0, int cols_pad = 0,
                     float* emb_out = nullptr);   // emb_out: with pe_inv, also write the embedded (pre-norm) rows there
// Column-range sinks of a GEMM epilogue feeding the tensor-core attention (gemm_tc.cu): columns [q0, q0+width) -> q planes
// (scaled), [k0, k0+width) -> k planes, [v0, v0+width) -> transposed v planes (+ fp32 into the GEMM's C when C != null).
// A range is disabled by placing it outside [0, N) (e.g. -1000000).
struct AttnSinks {
  int enabled = 0;
  int q0 = -1000000, k0 = -1000000, v0 = -1000000;
  int width = 512;             // heads * 128
  int npl = 2;                 // planes written
  int t_rows = 1, t_pad = 64;  // rows per utterance (v rows = keys), padded key pitch of the transposed planes
  float qscale = 1.f;
  plane_t* q_planes = nullptr;   // [npl][M][width]
  plane_t* k_planes = nullptr;   // [npl][M][width]
  plane_t* vt_planes = nullptr;  // [npl][B*width][t_pad]
};
// What a GEMM's epilogue does with act(A W^T + b), the bias being the FaLinear's: fp32 rows y = that (+ r1) (+ r2), and / or fp16
// planes [nplanes][M][ldp] (the A operand of a following tensor-core GEMM), and / or the attention sinks.  A call names what it sets.
struct GemmEpi {
  int relu_on = 0;
  const float* r1 = nullptr; int64_t ld1 = 0;
  const float* r2 = nullptr; int64_t ld2 = 0;
  float* y = nullptr; int64_t ldy = 0;
  plane_t* planes = nullptr; int64_t ldp = 0;
  const AttnSinks* att = nullptr;
  GemmEpi& relu(int on = 1) { relu_on = on; return *this; }
  GemmEpi& add(const float* r, int64_t ld, const float* r_2 = nullptr, int64_t ld_2 = 0) { r1 = r; ld1 = ld; r2 = r_2; ld2 = ld_2; return *this; }
  GemmEpi& to(float* out, int64_t ld) { y = out; ldy = ld; return *this; }
  GemmEpi& to(plane_t* out, int64_t ld) { planes = out; ldp = ld; return *this; }
  GemmEpi& sinks(const AttnSinks* s) { att = s; return *this; }
};
// fp32 SIMT GEMM (gemm_f32.cu), K a multiple of 16; fp32 rows only (FA_ERR_ARG for planes or sinks)
int gemm_f32_launch(const float* A, int64_t lda, int64_t M, const float* W, int N, int K, const float* bias, const GemmEpi& epi, cudaStream_t st);
// wgmma fp16-split GEMM (gemm_tc.cu)
size_t gemm_tc_scratch_bytes(int64_t max_rows, int max_k, int mode);
// A GEMM over fp32 rows x [rows, lin.in_f] in any mode: the SIMT GEMM, or the split into fp16 planes carved from scratch
// (gemm_tc_scratch_bytes) and the tensor-core GEMM
int gemm_rows(const float* x, int64_t ldx, int64_t rows, const FaLinear& lin, const GemmEpi& epi, int mode, Arena* scratch, cudaStream_t st);
// The query scale d_k^-0.5 of scaled dot-product attention, rounded like the reference's float(d_k ** -0.5)
inline float attn_qscale(int head_dim) { return (float)(1.0 / sqrt((double)head_dim)); }
// The tensor-core attention's operand planes (attention_tc.cu owns this layout): q [npl][B*tq][width] (scaled by d_k^-0.5),
// k [npl][kv_batch*tk][width] and v transposed per head, vt [npl][kv_batch*width][t_pad], keys padded to t_pad = round_up(tk, 64)
struct AttnPlanes { plane_t *q = nullptr, *k = nullptr, *vt = nullptr; int npl = 0, t_pad = 0; };
// The planes for up to (batch, tq) queries over (kv_batch, tk) keys of the given width, attn_planes(mode) planes each
AttnPlanes attn_carve(Arena& a, int batch, int tq, int kv_batch, int tk, int width, int mode);
// The sinks of a GEMM epilogue that writes p: columns [q0, q0+width) -> q (x qscale), [k0, +width) -> k, [v0, +width) -> vt, with
// t_rows GEMM rows per utterance; a negative start leaves its range off
AttnSinks attn_sinks(const AttnPlanes& p, int q0, int k0, int v0, int width, int t_rows, float qscale);
// batch utterances of tq queries over tk keys, heads x head_dim wide.  K / V hold kv_entries() entries of tk keys and utterance b
// attends over entry kv_index[b] (device, kv_batch entries); without an index, entry 0 when kv_shared (ONE entry that all attend
// over: hotword memory), else entry b
struct AttnShape {
  int batch, heads, head_dim, tq, tk, kv_shared;
  int kv_batch = 0;
  const int32_t* kv_index = nullptr;
  int kv_entries() const { return kv_index ? kv_batch : kv_shared ? 1 : batch; }
};
// What an attention call writes: fp32 context rows [B*tq][ldc] and / or fp16 planes [nplanes][B*tq][ldp] (the out-projection's A)
struct AttnOut {
  float* ctx = nullptr; int64_t ldc = 0;
  plane_t* planes = nullptr; int64_t ldp = 0; int nplanes = 0;
  AttnOut& to(float* out, int64_t ld) { ctx = out; ldc = ld; return *this; }
  AttnOut& to(plane_t* out, int64_t ld, int n) { planes = out; ldp = ld; nplanes = n; return *this; }
};
// wgmma attention over operand planes already in place (attention_tc.cu); head_dim 128 or 80
int attention_planes(const AttnPlanes& p, const AttnShape& s, const int32_t* key_lens, const AttnOut& out, cudaStream_t st);
// Attention over fp32 rows in any mode: the fp32 kernels (fp32 context only), or the split into planes carved from scratch
// (attention_tc_scratch_bytes; head_dim 128) and attention_planes
int attention_rows(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, const AttnShape& s,
                   const int32_t* key_lens, const AttnOut& out, int mode, Arena* scratch, cudaStream_t st);
size_t attention_tc_scratch_bytes(int batch, int heads, int tq, int kv_batch, int tk, int mode);
int gemm_tc_planes_launch(const plane_t* a_planes, int64_t M, const FaLinear& lin, const GemmEpi& epi, int mode, cudaStream_t st,
                          int64_t a_ld = 0, int64_t a_plane_rows = 0);
// a_ld / a_plane_rows (0 = dense: K_pad / M): row pitch of the A planes and rows between planes when A is an overlapping view
int split_rows_launch(const float* x, int64_t ldx, int64_t rows, int cols, int cols_pad, int nplanes, plane_t* planes,
                      cudaStream_t st);
int fsmn_launch(const float* v, int64_t ldv, const int32_t* lens, int batch, int t_max, int channels, const float* w,
                int ksize, const float* res, int64_t ldr, float* out, int64_t ldo, cudaStream_t st, int causal = 0);
// ext / ext_up: each row's padded length on the device (NULL: t_max / t3 for every row), cif.cu
int cif_im2col_launch(const float* enc, int64_t rows, int t_max, const int32_t* ext, int d, float* xc, cudaStream_t st);
int cif_fire_loop_launch(const float* enc, const float* alpha_rows, const int32_t* lens, const int32_t* ext, int batch, int t_max, int d,
                         float tail, float threshold, float* acoustic, int n_cap, int32_t* token_num, float* alphas, float* peaks,
                         cudaStream_t st);
int cif_upsample_scan_launch(float* alphas2, const int32_t* token_num, const int32_t* ext_up, int batch, int t3, float thr, float* us_peaks,
                             cudaStream_t st);
int cif_alpha_launch(const float* c, int d, const float* w, const float* b0, const int32_t* lens, int t_max,
                     int64_t rows, float smooth, float noise, float* alpha_rows, cudaStream_t st, int c_rows_per_batch = 0);
int cif_pad_planes_launch(const float* enc, int batch, int t_max, const int32_t* ext, int d, int nplanes, int64_t rows_alloc, plane_t* planes,
                          cudaStream_t st);
int cif_fire_launch(const float* enc, const float* alpha_rows, const int32_t* lens, const int32_t* ext, int batch, int t_max, int d,
                    float tail, float* acoustic, int n_cap, int32_t* token_num, float* alphas, float* peaks,
                    cudaStream_t st);
// the persistent BLSTM (lstm.cu): T lockstep steps over sequences of t_ld steps, ext their own lengths on the device (NULL: T each)
int blstm_tc_launch(const float* xproj, const float* w_hh_f, const float* w_hh_b, int batch, int T, int t_ld, const int32_t* ext, int hidden,
                    float* out, void* scratch, size_t scratch_bytes, cudaStream_t st);
int ctc_filter_launch(const int32_t* ids, const int32_t* lens, int batch, int t_max, int blank, int32_t* out_ids,
                      int32_t* out_lens, cudaStream_t st);
// torchaudio kaldi.fbank defaults (no x32768, no LFR, no CMVN) through the table-driven kernel (fbank.cu): the CAM++ frontend
int fbank_unscaled_launch(const float* wav, const int32_t* wav_lens, int batch, int64_t wav_stride, const float* tables, float* feats,
                          int32_t* feat_lens, int t_max, cudaStream_t st);
int argmax_lse_launch(float* logits, int64_t rows, int vocab, int64_t ld, int32_t* ids, float* best_logp,
                      int write_log_softmax, cudaStream_t st);
// fa_sanm_decoder_stack_forward_grouped (finish, no probe) with its per-utterance [key count | memory] rows_d [2 * batch] already on the
// device (model.cu); its workspace is fa_sanm_decoder_stack_grouped_workspace_bytes(batch, n_groups, t_mem, n_max, 0, mode)
int sanm_stack_grouped_dev(const FaDecoder* dec, const float* memory, const int32_t* rows_d, int32_t n_groups, int32_t batch, int32_t t_mem,
                           const float* x, int64_t ld_x_rows, const int32_t* tok_lens, int32_t n_max, int32_t n_run, float* hidden, int32_t gemm_mode,
                           void* workspace, size_t ws_bytes, cudaStream_t st);

}  // namespace fa
