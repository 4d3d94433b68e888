/*
 * funasr_b200 — C ABI of the H100-native (sm_90a) backend for FunASR's offline Paraformer hot path.
 *
 * Every entry point takes plain device pointers, sizes and a CUDA stream (as void*); no torch / C++
 * types cross the boundary.  All functions are stream-ordered, re-entrant, hold no global state, never
 * synchronise the device, and return FA_OK (0) or a negative FaStatus.  The caller owns every buffer
 * (inputs, outputs, workspace); weights are borrowed pointers.  An entry point that takes a workspace has a *_workspace_bytes
 * (or *_scratch_bytes) query: it returns exactly the bytes the forward carves for the path its arguments select, and a workspace
 * of that size is enough.  A smaller one returns FA_ERR_WORKSPACE before any work is enqueued.
 *
 * Each entry point names the reference interface it replaces (paths relative to the FunASR tree,
 * commit 3c58cb5 / funasr 1.4.3).  The tensor-level operator boundary mirrors the reference's own
 * export signature  export_forward(speech[B,T,560], speech_lengths[B]) -> (logits[B,N,V], token_num[B])
 * (funasr/models/paraformer/export_meta.py) extended upward by the frontend and downward by greedy ids.
 *
 * Layout conventions: row-major, innermost dimension contiguous; a "row" is one (utterance, frame) or
 * (utterance, token) pair; nn.Linear weights keep their [out_features, in_features] layout.
 */
#ifndef FUNASR_B200_H_
#define FUNASR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* fa_stream_t; /* cudaStream_t */

typedef enum {
  FA_OK = 0,
  FA_ERR_ARG = -1,         /* null pointer / bad size */
  FA_ERR_CUDA = -2,        /* a CUDA runtime call or launch failed */
  FA_ERR_WORKSPACE = -3,   /* workspace too small */
  FA_ERR_UNSUPPORTED = -4  /* shape outside what the kernels are built for */
} FaStatus;

/* GEMM arithmetic modes (FaLinear contractions). fp32 accumulate everywhere. */
typedef enum {
  FA_GEMM_F32_SIMT = 0, /* fp32 FFMA tiles: the parity reference path */
  FA_GEMM_F16X1 = 1,   /* wgmma f16, one fp16 pass (fast mode) */
  FA_GEMM_F16X3 = 3,   /* wgmma, fp16 planes x = hi + lo: hi*hi + hi*lo + lo*hi (~2^-22 relative per product for operands above
                        * ~2^-3 in magnitude; ~2^-21 / 2^-20 for weights at 1/sqrt(512) / 1/sqrt(2048), whose mid plane is subnormal) */
  FA_GEMM_F16X6 = 6    /* wgmma, three fp16 planes, six products (~fp32 for operands above ~2^-3; no better than x3 below) */
} FaGemmMode;

/* nn.Linear: y = x W^T + b.  w_planes (optional) holds the fp16 planes made by fa_split_planes for the
 * tensor-core path: [3][out_f][in_pad] fp16 (hi, mid, lo), in_pad = in_f rounded up to 64. */
typedef struct {
  const float* w;        /* [out_f, in_f] */
  const float* b;        /* [out_f] or NULL */
  const void* w_planes;  /* or NULL */
  int32_t out_f, in_f, in_pad, _pad;
} FaLinear;

typedef struct {
  const float* g; /* weight [n] */
  const float* b; /* bias   [n] */
  int32_t n;
  float eps;
} FaNorm;

/* EncoderLayerSANM (funasr/models/sanm/encoder.py:44-148) */
typedef struct {
  FaNorm norm1;          /* over in_size (560 for encoders0, 512 otherwise) */
  FaLinear qkv;          /* self_attn.linear_q_k_v  [1536, in_size] */
  const float* fsmn_w;   /* self_attn.fsmn_block.weight [512, 11] (depthwise) */
  FaLinear out;          /* self_attn.linear_out    [512, 512] */
  FaNorm norm2;
  FaLinear w1;           /* feed_forward.w_1 [2048, 512] */
  FaLinear w2;           /* feed_forward.w_2 [512, 2048] */
} FaEncLayer;

/* SANMEncoder (funasr/models/sanm/encoder.py:188-461), input_layer == "pe" */
typedef struct {
  const FaEncLayer* layers;  /* host array, n_layers entries; [0] is encoders0.0 */
  int32_t n_layers;
  int32_t heads;
  int32_t fsmn_k;            /* 11 */
  int32_t _pad;
  FaNorm after_norm;
  const float* pe_inv_timescales; /* [in_size/2] device, transformer/embedding.py:409-414 */
} FaEncoder;

/* CifPredictorV2 (funasr/models/paraformer/cif_predictor.py:209-314) */
typedef struct {
  FaLinear conv;      /* cif_conv1d as a GEMM: weight repacked to [512, 3*512], W[n, k*512+c] = w[n,c,k] */
  const float* out_w; /* cif_output.weight [512] */
  const float* out_b; /* cif_output.bias   [1]   */
  float threshold;      /* 1.0 */
  float tail_threshold; /* 0.45 */
  float smooth_factor;  /* 1.0 */
  float noise_threshold;/* 0.0 */
  int32_t cif_variant;  /* 0: CifPredictorV2 `cif_v1` (fp64 prefix sums, paraformer/cif_predictor.py:818-908);
                         * 1: CifPredictorV3 `cif` (sequential fp32, bicif_paraformer/cif_predictor.py:37-84) */
  int32_t _pad;
} FaPredictor;

/* DecoderLayerSANM (funasr/models/paraformer/decoder.py:26-121) */
typedef struct {
  FaNorm norm1;
  FaLinear ffn_w1;       /* feed_forward.w_1 [2048, 512] */
  FaNorm ffn_norm;       /* feed_forward.norm over 2048 */
  FaLinear ffn_w2;       /* feed_forward.w_2 [512, 2048], no bias */
  FaNorm norm2;
  const float* fsmn_w;   /* self_attn.fsmn_block.weight [512, 11]; NULL for decoders3 */
  FaNorm norm3;
  FaLinear q;            /* src_attn.linear_q   [512, 512] */
  FaLinear kv;           /* src_attn.linear_k_v [1024, 512] */
  FaLinear out;          /* src_attn.linear_out [512, 512] */
} FaDecLayer;

/* ParaformerSANMDecoder (funasr/models/paraformer/decoder.py:234-449) */
typedef struct {
  const FaDecLayer* layers; /* host array, n_layers entries (decoders) */
  int32_t n_layers;
  int32_t heads;
  int32_t fsmn_k;
  int32_t vocab;
  FaDecLayer last;          /* decoders3.0: norm1 + ffn only */
  FaNorm after_norm;
  FaLinear output;          /* output_layer [vocab, 512] */
  /* ContextualParaformerDecoder (funasr/models/contextual_paraformer/decoder.py:133-352); has_bias == 0 for the plain
   * Paraformer decoder.  With has_bias: `layers` are decoders.{0..att_layer_num-2}, `bias_last` is last_decoder, and
   * x = x_self_attn + bias_output([x_src_attn ; clas_scale * bias_decoder(x_self_attn, hotword memory)]) (:330-340). */
  int32_t has_bias;
  int32_t n_hotwords;       /* rows of hw_embed, <= t_max */
  FaDecLayer bias_last;     /* last_decoder (ContextualDecoderLayer :22-100) */
  FaNorm bias_norm3;        /* bias_decoder.norm3 */
  FaLinear bias_q, bias_kv, bias_out; /* bias_decoder.src_attn.linear_q / linear_k_v / linear_out */
  FaLinear bias_output;     /* bias_output Conv1d(1024->512, k=1, no bias) as a [512, 1024] linear */
  const float* hw_embed;    /* [n_hotwords, 512] hotword memory (LSTM last hidden states, model.py:350-372) */
  const int32_t* hw_lens;   /* [batch] device, every entry == n_hotwords */
  float clas_scale;         /* 1.0 */
  int32_t _pad2;
} FaDecoder;

/* ---------------------------------------------------------------------------------------------
 * Library info
 * ------------------------------------------------------------------------------------------- */
const char* fa_version(void);
/* Monotone count of kernel launches issued by this library in this process (bench "gpu_launches"). */
uint64_t fa_launch_count(void);
const char* fa_status_string(int status);

/* ---------------------------------------------------------------------------------------------
 * Frontend — replaces WavFrontend.forward (funasr/frontends/wav_frontend.py:149-196), i.e.
 * torchaudio.compliance.kaldi.fbank (dither=0, hamming, 25 ms / 10 ms, 80 mel, snip_edges) + apply_lfr
 * (:63-86) + apply_cmvn (:46-60), fused.  wav is float32 in [-1,1] (x32768 applied inside,
 * :169).  Rows t >= feat_lens[b] of feats are zero-filled (pad_sequence(..., 0.0), :195).
 * ------------------------------------------------------------------------------------------- */
/* fa_fbank_make_tables derives, once per configuration, the sparse support of the 80 mel filters, the FFT twiddles, the window
 * and the mel tap schedule into `tables` (fa_fbank_tables_bytes() bytes of device memory) from
 *   mel_banks [80,257] (kaldi.py get_mel_banks + zero column), window [400] (hamming).
 * fa_fbank_lfr_cmvn_tables then computes, from those tables,
 *   wav [B, wav_stride], wav_lens[B] (samples, >= 400), cmvn [2, 80 * lfr_m] or NULL -> feats, feat_lens [B],
 * writing utterance b at feats + b * feats_batch_stride_rows * 80 * lfr_m (t_max rows each): a stride above t_max leaves room
 * for prepended frames, e.g. SenseVoiceSmall's 4 query frames (funasr/models/sense_voice/model.py:971-995).  lfr_m / lfr_n select
 * the low-frame-rate stacking: 7 / 6 (Paraformer, SenseVoice: feats [B, t_max, 560]) or 5 / 1 (the FSMN-VAD frontend,
 * fsmn_vad_streaming/template.yaml:54-62: feats [B, t_max, 400], one row per 10 ms frame).  An utterance with more than t_max rows
 * keeps its first t_max (the values an untruncated call gives them) and feat_lens[b] still reports its full row count. */
size_t fa_fbank_tables_bytes(void);
int fa_fbank_make_tables(const float* mel_banks, const float* window, float* tables, fa_stream_t stream);
int fa_fbank_lfr_cmvn_tables(const float* wav, const int32_t* wav_lens, int32_t batch, int64_t wav_stride, const float* cmvn,
                             const float* tables, int32_t lfr_m, int32_t lfr_n, float* feats, int64_t feats_batch_stride_rows,
                             int32_t* feat_lens, int32_t t_max, fa_stream_t stream);
/* One utterance shorter than a 25 ms frame (2 <= n_samples < 400): WavFrontend.forward passes frame_length = min(25 ms, len / fs)
 * (funasr/frontends/wav_frontend.py:174), so kaldi.fbank uses the whole utterance as ONE window of n_samples (hamming, `window`),
 * zero-padded to padded_fft = the next power of two, with mel_banks [80, padded_fft / 2 + 1] built for that FFT size; the single
 * log-mel frame is repeated lfr_m times and CMVN'd into feats_row [80 * lfr_m].  (The batched kernel above gives such rows
 * feat_lens = 0.) */
int fa_fbank_short(const float* wav, int32_t n_samples, const float* window, const float* mel_banks, int32_t padded_fft,
                   const float* cmvn, int32_t lfr_m, float* feats_row, fa_stream_t stream);
/* dst[b, r, :] = rows[r, :] for r < n_rows (dst rows of `cols` floats, utterances dst_batch_stride_rows apart):
 * the query-frame prepend `torch.cat((input_query, speech), dim=1)` of sense_voice/model.py:985-995. */
int fa_broadcast_rows(const float* rows, int32_t n_rows, int32_t cols, float* dst, int64_t dst_batch_stride_rows,
                      int32_t batch, fa_stream_t stream);
/* The same prepend with a query per utterance: dst[b, 0..3, :] = embed[ids[2b]], embed[1], embed[2], embed[ids[2b + 1]] (language,
 * event, emotion, text norm; sense_voice/model.py:971-995).  embed [n_embed, cols] and ids [batch, 2] (language id, textnorm id) are
 * device memory; ids are clamped to [0, n_embed) (validate them first).  Only the 4 query rows of every utterance are written. */
int fa_sv_query_rows(const float* embed, int32_t n_embed, int32_t cols, const int32_t* ids, int32_t batch, float* dst,
                     int64_t dst_batch_stride_rows, fa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Operator-level entry points (each is used by the model-level calls below and exposed for parity tests)
 * ------------------------------------------------------------------------------------------- */
/* LayerNorm over the last dim (funasr/models/transformer/layer_norm.py:13-39).  If pe_inv != NULL the
 * input row (b,t) is first mapped x*xscale + PE(t+1) (SANMEncoder.forward encoder.py:409,428 with
 * SinusoidalPositionEncoder embedding.py:396-432); rows_per_batch gives t = row % rows_per_batch. */
int fa_layernorm(const float* x, int64_t rows, const FaNorm* norm, float* y,
                 const float* pe_inv, float xscale, int32_t rows_per_batch, fa_stream_t stream);
/* The same LayerNorm with the fused outputs of the tensor-core path: planes != NULL receives the normalised rows as fp16 planes
 * [nplanes][rows][cols_pad] (hi, mid, lo; nplanes 1..3, n <= cols_pad <= 2048, cols_pad % 4 == 0) with columns [n, cols_pad) zero
 * in every plane: the A operand of the next GEMM (cols_pad = its in_pad).  y (fp32, may equal x) may be NULL when planes is set.
 * emb_out != NULL (needs pe_inv) also receives the embedded rows x * xscale + PE before the norm.  x, y, emb_out 16-byte aligned,
 * planes 8-byte aligned (FA_ERR_UNSUPPORTED otherwise). */
int fa_layernorm_planes(const float* x, int64_t rows, const FaNorm* norm, float* y, void* planes, int32_t nplanes, int32_t cols_pad,
                        const float* pe_inv, float xscale, int32_t rows_per_batch, float* emb_out, fa_stream_t stream);

/* y[rows, out_f] = act(x[rows, in_f(ldx)] W^T + b) (+ res1) (+ res2); replaces torch.nn.Linear calls
 * (attention.py:256,306; positionwise_feed_forward.py:34).  relu != 0 applies ReLU before residuals. */
int fa_linear(const float* x, int64_t ldx, int64_t rows, const FaLinear* lin, int32_t relu,
              const float* res1, int64_t ld_res1, const float* res2, int64_t ld_res2,
              float* y, int64_t ldy, int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream);
/* fa_linear's workspace: the fp16 planes of x for rows x in_f (in_pad = in_f rounded up to 64); 0 for FA_GEMM_F32_SIMT. */
size_t fa_linear_workspace_bytes(int64_t rows, int32_t in_f, int32_t gemm_mode);

/* The tensor-core GEMM alone, A operand already split into fp16 planes [npl][rows][lin->in_pad] (npl = 1 / 2 / 3 for
 * F16X1 / X3 / X6) by fa_split_rows: what the model-level calls launch between fused producers and consumers. */
int fa_split_rows(const float* x, int64_t ldx, int64_t rows, int32_t cols, int32_t cols_pad, int32_t nplanes, void* planes,
                  fa_stream_t stream);
int fa_linear_planes(const void* a_planes, int64_t rows, const FaLinear* lin, int32_t relu, const float* res1, int64_t ld_res1,
                     const float* res2, int64_t ld_res2, float* y, int64_t ldy, int32_t gemm_mode, fa_stream_t stream);
/* Same GEMM with the plane-emitting epilogue: out_planes [npl][rows][ld_out] fp16 (hi, lo, ...) of act(A W^T + b) — the launch the
 * encoder makes for FFN w_1, whose ReLU output feeds w_2 without an fp32 round trip (bench.py times exactly this launch). */
int fa_linear_planes_to_planes(const void* a_planes, int64_t rows, const FaLinear* lin, int32_t relu, void* out_planes,
                               int64_t ld_out, int32_t gemm_mode, fa_stream_t stream);
/* fa_linear_planes and fa_linear_planes_to_planes refuse, before any launch: bias / residual bases not 16-byte aligned, y not
 * 16-byte aligned with ldy % 4 == 0, residual pitches or ld_out not multiples of 4, out_planes not 8-byte aligned
 * (FA_ERR_UNSUPPORTED); ldy, ld_res1, ld_res2 or ld_out below out_f (FA_ERR_ARG). */
/* The same GEMM (fp32 output, no residual) over an overlapping "conv view" of the A planes, as the CIF conv (a_ld = 512,
 * in_pad = 1536: three consecutive frames per row) and the CAM++ TDNN (a_ld = 640, in_pad = 1600: kernel 5, stride 2) run it:
 * row r of plane p is the lin->in_pad elements starting at element (p * a_plane_rows + r) * a_ld of a_planes.  a_ld % 8 != 0 ->
 * FA_ERR_UNSUPPORTED; a_plane_rows < rows + ceil((in_pad - a_ld) / a_ld) when a_ld < in_pad (a valid row would reach into the next
 * plane), or < rows otherwise -> FA_ERR_ARG. */
int fa_linear_planes_view(const void* a_planes, int64_t rows, int64_t a_ld, int64_t a_plane_rows, const FaLinear* lin, int32_t relu,
                          float* y, int64_t ldy, int32_t gemm_mode, fa_stream_t stream);
/* Same GEMM with the attention-operand epilogue the QKV / q / kv projections use (no ReLU): output columns [q0, q0 + width) go to
 * q_planes [qpl][rows][width] as fp16 planes of fl(y * qscale), [k0, k0 + width) to k_planes [qpl][rows][width], and [v0, v0 + width)
 * to vt_planes [qpl][rows / t_rows * width][t_pad], V transposed per utterance of t_rows rows (row b * t_rows + t, column c ->
 * vt row b * width + c, column t; columns [t_rows, t_pad) are not written); qpl = 1 for FA_GEMM_F16X1, else 2.  A negative start
 * disables that sink; the enabled ranges must start at a multiple of 16, lie inside [0, out_f) and not overlap.  v_f32 != NULL
 * (leading dim ld_v_f32 >= out_f) also receives the fp32 V columns at their own column positions (the FSMN input); nothing else is
 * written there.  FA_ERR_ARG for rows % t_rows != 0, t_pad < t_rows with the V sink, or a bad sink range. */
int fa_linear_attn_sinks(const void* a_planes, int64_t rows, const FaLinear* lin, int32_t q0, int32_t k0, int32_t v0, int32_t width,
                         int32_t t_rows, int32_t t_pad, float qscale, void* q_planes, void* k_planes, void* vt_planes, float* v_f32,
                         int64_t ld_v_f32, int32_t gemm_mode, fa_stream_t stream);

/* FSMN memory block: out = m * (v*m + dwconv_k(v*m)) (+ res); m[t] = t < lens[b]
 * (MultiHeadedAttentionSANM.forward_fsmn attention.py:216-239; decoder variant :583-631).  out must not overlap v or res (the staged
 * kernel reads whole tiles ahead of its stores). */
int fa_fsmn(const float* v, int64_t ldv, const int32_t* lens, int32_t batch, int32_t t_max, int32_t channels,
            const float* w, int32_t ksize, const float* res, int64_t ld_res, float* out, int64_t ld_out,
            fa_stream_t stream);
/* The same memory block through the TMA-staged, warp-specialised kernel (persistent CTAs, cp.async.bulk.tensor ring of
 * [64 + k - 1] x 128-channel boxes, results bit-identical to fa_fsmn).  FA_ERR_UNSUPPORTED unless ksize is 11 or 21, channels is a
 * multiple of 128 and v / res are 16-byte aligned with pitches that are multiples of 4 floats.  fa_fsmn and the model-level calls
 * take this route when the shape allows it and t_max >= 64. */
int fa_fsmn_tma(const float* v, int64_t ldv, const int32_t* lens, int32_t batch, int32_t t_max, int32_t channels,
                const float* w, int32_t ksize, const float* res, int64_t ld_res, float* out, int64_t ld_out,
                fa_stream_t stream);
/* The SIMT strip kernel for every shape (ksize 11 / 21 / 31, any channel count or alignment): the A/B partner of fa_fsmn_tma. */
int fa_fsmn_simt(const float* v, int64_t ldv, const int32_t* lens, int32_t batch, int32_t t_max, int32_t channels,
                 const float* w, int32_t ksize, const float* res, int64_t ld_res, float* out, int64_t ld_out,
                 fa_stream_t stream);

/* Multi-head scaled-dot attention with key-padding mask: masked_fill(-inf) -> softmax -> masked_fill(0)
 * -> @V, heads merged (attention.py:288-304 self, :760-794 cross).  head_dim is 128.
 *   q [B, tq, ldq], k/v [B, tk, ldk/ldv] (head h at column h*128), ctx [B, tq, ld_ctx]. */
int fa_attention(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv,
                 const int32_t* key_lens, int32_t batch, int32_t heads, int32_t tq, int32_t tk,
                 float* ctx, int64_t ld_ctx, fa_stream_t stream);

/* Same contract on the tensor cores (wgmma; fp16 operand planes, fp32 accumulation in registers):
 * gemm_mode FA_GEMM_F16X1 (one plane) or FA_GEMM_F16X3/X6 (hi+lo planes, three MMA terms).  workspace holds the
 * operand planes (size from fa_attention_tc_workspace_bytes, exactly what the call carves). */
size_t fa_attention_tc_workspace_bytes(int32_t batch, int32_t heads, int32_t tq, int32_t tk, int32_t gemm_mode);
int fa_attention_tc(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv,
                    const int32_t* key_lens, int32_t batch, int32_t heads, int32_t tq, int32_t tk,
                    float* ctx, int64_t ld_ctx, int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream);
/* The tensor-core attention on operand planes already in place, as the models call it after fa_linear_attn_sinks:
 * q_planes [npl][B * tq][H * 128] (already scaled by d_k^-0.5), k_planes [npl][kb * tk][H * 128], vt_planes [npl][kb * H * 128][tkp]
 * with tkp = tk rounded up to 64 (columns >= tk are never read), npl = 1 for FA_GEMM_F16X1, else 2; kb = 1 when kv_shared != 0
 * (every utterance attends over the same keys and values, the hotword memory), else B.  Writes ctx [B * tq][ld_ctx] fp32 and / or
 * ctx_planes [out_nplanes][B * tq][ld_planes] fp16 (the split of the same fp32 values, the A operand of the out-projection):
 * out_nplanes 1 for FA_GEMM_F16X1, 2 or 3 otherwise (FA_ERR_UNSUPPORTED for the other pairings, FA_ERR_ARG outside 1..3). */
int fa_attention_tc_planes(const void* q_planes, const void* k_planes, const void* vt_planes, const int32_t* key_lens, int32_t batch,
                           int32_t heads, int32_t tq, int32_t tk, float* ctx, int64_t ld_ctx, void* ctx_planes, int64_t ld_planes,
                           int32_t out_nplanes, int32_t gemm_mode, int32_t kv_shared, fa_stream_t stream);
/* fa_attention_tc_planes with an explicit head_dim: 128 (the call above) or 80 (the fa-zh aligner, 4 x 80); every 128 of that
 * contract reads head_dim.  Any other head_dim returns FA_ERR_UNSUPPORTED. */
int fa_attention_tc_planes_ex(const void* q_planes, const void* k_planes, const void* vt_planes, const int32_t* key_lens, int32_t batch,
                              int32_t heads, int32_t head_dim, int32_t tq, int32_t tk, float* ctx, int64_t ld_ctx, void* ctx_planes,
                              int64_t ld_planes, int32_t out_nplanes, int32_t gemm_mode, int32_t kv_shared, fa_stream_t stream);
/* fp32 attention with the fp32 path's kernel choice: head_dim 128 -> the tiled kernel of fa_attention, any other multiple of 32 up
 * to 128, or 80 -> the warp-per-query kernel (CT-Transformer's 8 x 32 heads, the aligner's 4 x 80; FA_ERR_UNSUPPORTED when 4 * tk
 * floats exceed its 160 KB of shared memory).  kv_shared != 0: k / v hold one batch entry [tk, ld] that every utterance attends over. */
int fa_attention_f32_ex(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv,
                        const int32_t* key_lens, int32_t batch, int32_t heads, int32_t head_dim, int32_t tq, int32_t tk,
                        float* ctx, int64_t ld_ctx, int32_t kv_shared, fa_stream_t stream);
/* Attention with a K / V entry per utterance: k / v hold kv_batch entries [kv_batch, tk, ld] and utterance b attends over entry
 * kv_index_h[b] (host, each in [0, kv_batch), read before the call returns) with key_lens[b] (device) keys, through the same kernels as the calls above in any
 * gemm_mode (fp32: the fp32 kernels' choice by head_dim; tensor cores: head_dim 128).  Every index 0 with one entry is kv_shared, index
 * b with kv_batch = B the per-utterance case; a row gives exactly what the kv_shared call on its own entry gives, whatever the other
 * entries hold (rows of an entry past its keys must be finite: the last 64-key chunk reads them and multiplies them by 0).  The
 * workspace holds the index and, on the tensor cores, the operand planes; its query is exactly what the call carves.  Refusals
 * (NULL arguments, an index outside [0, kv_batch)) come before any device work. */
size_t fa_attention_grouped_workspace_bytes(int32_t batch, int32_t heads, int32_t tq, int32_t kv_batch, int32_t tk, int32_t gemm_mode);
int fa_attention_grouped(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, const int32_t* key_lens,
                         const int32_t* kv_index_h, int32_t kv_batch, int32_t batch, int32_t heads, int32_t head_dim, int32_t tq, int32_t tk,
                         float* ctx, int64_t ld_ctx, int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Model-level entry points
 * ------------------------------------------------------------------------------------------- */
/* SANMEncoder.forward (encoder.py:392-461): feats [B,T,560], lens[B] -> enc [B,T,512].
 * If enc->pe_inv_timescales == NULL the struct describes a plain stack of 512->512 SAN-M layers applied to an
 * existing [B,T,512] stream (no x*sqrt(d)+PE, every layer has its residual): SenseVoiceEncoderSmall's `tp_encoders`
 * + `tp_norm` (sense_voice/model.py:650-655).
 * Workspace: sized for d_model <= 512, input <= 560 and FFN <= 2048; exactly what the forward carves for gemm_mode. */
size_t fa_sanm_encoder_workspace_bytes(int32_t batch, int32_t t_max, int32_t gemm_mode);
int fa_sanm_encoder_forward(const FaEncoder* enc, const float* feats, const int32_t* lens, int32_t batch,
                            int32_t t_max, float* out, int32_t gemm_mode, void* workspace, size_t ws_bytes,
                            fa_stream_t stream);

/* CifPredictorV2.forward, inference branch (cif_predictor.py:253-314 + tail_process_fn :414-446 + cif_v1
 * :853-908).  enc [B,T,512], lens[B] ->
 *   acoustic [B, n_cap, 512] (rows >= fires zero-filled; n_cap >= 1, tokens beyond n_cap are dropped),
 *   token_num [B] int32 (= floor(sum alpha'), the reference's pre_token_length),
 *   alphas [B, T+1], peaks [B, T+1] (cif_peak / "fires").
 * The tensor-core modes need conv.in_pad == 1536 (FA_ERR_UNSUPPORTED otherwise).  The workspace query returns exactly what the
 * forward carves for gemm_mode. */
size_t fa_cif_predictor_workspace_bytes(int32_t batch, int32_t t_max, int32_t gemm_mode);
int fa_cif_predictor_forward(const FaPredictor* pred, const float* enc, const int32_t* lens, int32_t batch,
                             int32_t t_max, float* acoustic, int32_t n_cap, int32_t* token_num, float* alphas,
                             float* peaks, int32_t gemm_mode, void* workspace, size_t ws_bytes,
                             fa_stream_t stream);
/* The same with a padded length per row.  The reference's predictor reads past a row's end: the k = 3 conv at t = len - 1 reads
 * frame len, and tail_process_fn adds 0.45 * hidden[len] and sums the weights over the whole padded row.  So a row's result depends
 * on how far its batch was padded.  Row b here behaves exactly as in a batch padded to ext_h[b] frames: encoder frames at or past
 * ext_h[b] read zero, and token_num sums its ext_h[b] + 1 weights.  lens_h / ext_h [B] are HOST copies of the lengths and the
 * extents, lens_h[b] <= ext_h[b] <= t_max and ext_h[b] >= 1 (FA_ERR_ARG otherwise, before any device work).  Outputs past
 * ext_h[b] + 1 in alphas / peaks are not the reference's (it has none).  ext_h[b] == t_max for every row is
 * fa_cif_predictor_forward bit for bit.  Workspace: fa_cif_predictor_ext_workspace_bytes. */
size_t fa_cif_predictor_ext_workspace_bytes(int32_t batch, int32_t t_max, int32_t gemm_mode);
int fa_cif_predictor_forward_ext(const FaPredictor* pred, const float* enc, const int32_t* lens, int32_t batch,
                                 int32_t t_max, float* acoustic, int32_t n_cap, int32_t* token_num, float* alphas,
                                 float* peaks, int32_t gemm_mode, void* workspace, size_t ws_bytes,
                                 fa_stream_t stream, const int32_t* lens_h, const int32_t* ext_h);

/* out[r] = x[r, :n].sum() in fp32 with the summation order of torch's CPU kernel (ATen SumKernel.cpp: 8 SIMD lanes x 4 ILP
 * accumulators, 4-level cascade): the CIF predictor's integer token count is floor(alphas.sum(-1)) (cif_predictor.py:443-444),
 * so the order decides an integer outcome.  x [rows, ld] fp32 on the device, out [rows]. */
int fa_row_sum_f32(const float* x, int64_t ld, int32_t rows, int32_t n, float* out, fa_stream_t stream);

/* Timestamp head of CifPredictorV3.get_upsample_timestamp (bicif_paraformer/cif_predictor.py:331-352), after the
 * ConvTranspose1d upsampling (a fa_linear with the [3*512, 512] repacked weight) and the BLSTM:
 *   alphas2 = relu(sigmoid(feat . w + b) * smooth2 - noise2) * mask;  alphas2 *= token_num / sum(alphas2);
 *   us_peaks = cif_wo_hidden(alphas2, threshold - 1e-4).
 * feat [B, t_up, dz] (dz = 1024), lens_up[B] = 3 * encoder lengths, token_num[B]; us_alphas / us_peaks [B, t_up]. */
int fa_cif_upsample_alphas(const float* feat, int32_t dz, const float* w, const float* b, const int32_t* lens_up,
                           const int32_t* token_num, int32_t batch, int32_t t_up, float smooth2, float noise2,
                           float threshold, float* us_alphas, float* us_peaks, fa_stream_t stream);

/* CifPredictorV3's upsampled timestamp head (upsample_type "cnn_blstm", bicif_paraformer/cif_predictor.py:121-352) in the layout
 * funasr_b200/pack.py:timestamp_head_tensors writes; D = d_model (512 or 320), U = up_times. */
typedef struct {
  FaLinear upsample;        /* upsample_cnn (ConvTranspose1d, stride == kernel == U) as a GEMM: [U*D, D], bias repeated U times */
  FaLinear blstm_ih;        /* both BLSTM input projections [W_ih_fwd; W_ih_bwd]: [8D, D], bias b_ih + b_hh */
  const float* w_hh_fwd;    /* blstm.weight_hh_l0 [4D, D] */
  const float* w_hh_bwd;    /* blstm.weight_hh_l0_reverse [4D, D] */
  const float* out2_w;      /* cif_output2.weight [2D] */
  const float* out2_b;      /* cif_output2.bias [1] */
  int32_t up_times;         /* U */
  float smooth2, noise2;    /* smooth_factor2, noise_threshold2 */
  float threshold;          /* the CIF threshold */
} FaTimestampHead;
/* CifPredictorV3.get_upsample_timestamp (:300-352): enc [B, t_max, D], lens[B] encoder lengths, token_num[B] ->
 * us_alphas / us_peaks [B, U * t_max].  The upsample GEMM, the input-projection GEMM, fa_blstm_forward_tc over at most 256
 * sequences per launch, lens x U, then fa_cif_upsample_alphas.  D other than 512 / 320 -> FA_ERR_UNSUPPORTED; GEMM shapes other
 * than the struct's comments say -> FA_ERR_ARG.  The workspace query returns exactly what the forward carves. */
size_t fa_timestamp_head_workspace_bytes(int32_t batch, int32_t t_max, int32_t d_model, int32_t up_times, int32_t gemm_mode);
int fa_timestamp_head_forward(const FaTimestampHead* head, const float* enc, const int32_t* lens, const int32_t* token_num,
                              int32_t batch, int32_t t_max, float* us_alphas, float* us_peaks, int32_t gemm_mode, void* workspace,
                              size_t ws_bytes, fa_stream_t stream);
/* The same with a padded length per row, as fa_cif_predictor_forward_ext (lens_h / ext_h host arrays, the same refusals).  The
 * reference's BLSTM runs without packing, so its backward direction starts at the batch's padded end, and alphas2 is summed over the
 * padded row.  Row b behaves exactly as in a batch padded to ext_h[b] frames: its BLSTM runs fa_blstm_forward_tc_ext with U * ext_h[b]
 * steps, and the sum covers U * ext_h[b] weights.  Outputs past U * ext_h[b] are not the reference's.  ext_h[b] == t_max for every
 * row is fa_timestamp_head_forward bit for bit.  Workspace: fa_timestamp_head_ext_workspace_bytes. */
size_t fa_timestamp_head_ext_workspace_bytes(int32_t batch, int32_t t_max, int32_t d_model, int32_t up_times, int32_t gemm_mode);
int fa_timestamp_head_forward_ext(const FaTimestampHead* head, const float* enc, const int32_t* lens, const int32_t* token_num,
                                  int32_t batch, int32_t t_max, float* us_alphas, float* us_peaks, int32_t gemm_mode, void* workspace,
                                  size_t ws_bytes, fa_stream_t stream, const int32_t* lens_h, const int32_t* ext_h);

/* One-layer bidirectional LSTM recurrence (torch.nn.LSTM(H, H, 1, batch_first=True, bidirectional=True), the `blstm` of
 * CifPredictorV3, bicif_paraformer/cif_predictor.py:187-190) as a persistent weight-stationary kernel: the per-step
 * [B,H] x [H,4H] product on warp-level bf16 MMAs with the 3-product operand split (fp32 accumulate), h exchanged between
 * CTAs as bf16 hi / lo planes.  The caller supplies the input projections of ALL steps (one fa_linear):
 * xproj [B*T, 8H] = x [W_ih_fwd; W_ih_bwd]^T + (b_ih + b_hh), gate order i,f,g,o per direction.  w_hh_* [4H, H].
 * out [B, T, 2H] (forward | reverse).  batch <= 256, hidden H == 512 or 320 (else FA_ERR_UNSUPPORTED).
 * scratch >= fa_blstm_tc_scratch_bytes(batch) bytes of device memory (zeroed by the call). */
size_t fa_blstm_tc_scratch_bytes(int32_t batch);
int fa_blstm_forward_tc(const float* xproj, const float* w_hh_fwd, const float* w_hh_bwd, int32_t batch, int32_t t_len,
                        int32_t hidden, float* out, void* scratch, size_t scratch_bytes, fa_stream_t stream);
/* The same over sequences of their own lengths ext_h[b] (HOST array, 1 <= ext_h[b] <= t_len, FA_ERR_ARG otherwise before any device
 * work): sequence b equals fa_blstm_forward_tc run on its first ext_h[b] steps alone.  Its backward direction starts at step
 * ext_h[b] - 1 from a zero state.  Rows t >= ext_h[b] of out are not written.  The launch runs max(ext_h) steps.
 * scratch >= fa_blstm_tc_ext_scratch_bytes(batch). */
size_t fa_blstm_tc_ext_scratch_bytes(int32_t batch);
int fa_blstm_forward_tc_ext(const float* xproj, const float* w_hh_fwd, const float* w_hh_bwd, int32_t batch, int32_t t_len,
                            int32_t hidden, float* out, void* scratch, size_t scratch_bytes, fa_stream_t stream, const int32_t* ext_h);

/* ParaformerSANMDecoder.forward (decoder.py:397-449) + greedy argmax (paraformer/model.py:642-644).
 *   enc [B,T,512], enc_lens[B]; acoustic [B, ld_acoustic_rows, 512] of which the first n_max rows are used;
 *   tok_lens[B].  Outputs: argmax_ids [B, n_max] int32, argmax_logp [B, n_max] (log-softmax value of the
 *   arg-max, :643), and — if logits != NULL — the full pre-softmax logits [B, n_max, vocab].
 *   If log_softmax != 0 the logits buffer is converted in place to log_softmax (model.py:345). */
/* Workspace size, exactly what the forward carves: n_hotwords is the number of entries in the hotword memory of a contextual
 * decoder (FaDecoder.has_bias), 0 for a plain one.  The logits slice is always counted (the query cannot see whether the caller
 * passes logits). */
size_t fa_paraformer_decoder_workspace_bytes_hw(int32_t batch, int32_t t_max, int32_t n_max, int32_t vocab,
                                                int32_t gemm_mode, int32_t n_hotwords);
int fa_paraformer_decoder_forward(const FaDecoder* dec, const float* enc, const int32_t* enc_lens, int32_t batch,
                                  int32_t t_max, const float* acoustic, int64_t ld_acoustic_rows,
                                  const int32_t* tok_lens, int32_t n_max, int32_t* argmax_ids, float* argmax_logp,
                                  float* logits, int32_t log_softmax, int32_t gemm_mode, void* workspace,
                                  size_t ws_bytes, fa_stream_t stream);

/* The same with return_hidden + return_both (decoder.py:441-449): additionally writes the after_norm output `hidden`
 * [B, n_max, 512] — the `decoder_hidden` SeacoParaformer feeds to its hotword decoder (seaco_paraformer/model.py:290-297). */
int fa_paraformer_decoder_forward_hidden(const FaDecoder* dec, const float* enc, const int32_t* enc_lens, int32_t batch,
                                         int32_t t_max, const float* acoustic, int64_t ld_acoustic_rows,
                                         const int32_t* tok_lens, int32_t n_max, int32_t* argmax_ids, float* argmax_logp,
                                         float* logits, int32_t log_softmax, float* hidden, int32_t gemm_mode,
                                         void* workspace, size_t ws_bytes, fa_stream_t stream);

/* A contextual decoder (dec->has_bias) over G hotword memories instead of dec->hw_embed / hw_lens / n_hotwords: hw_embed [G, nh_max,
 * 512] (device; rows past a memory's length must be finite, zeros are fine), hw_lens_h [G] (host, each in [1, nh_max]) and
 * row_group_h [B] (host, each in [0, G)): utterance b's bias branch attends over memory row_group_h[b], exactly as
 * fa_paraformer_decoder_forward(_hidden) gives it with that memory alone.  One bias k|v GEMM runs over all G * nh_max rows.  hidden
 * may be NULL.  Refusals come before any device work; the workspace query is exactly what the call carves. */
size_t fa_paraformer_decoder_grouped_workspace_bytes(int32_t batch, int32_t t_max, int32_t n_max, int32_t vocab, int32_t gemm_mode,
                                                     int32_t n_groups, int32_t nh_max);
int fa_paraformer_decoder_forward_grouped(const FaDecoder* dec, const float* enc, const int32_t* enc_lens, int32_t batch, int32_t t_max,
                                          const float* acoustic, int64_t ld_acoustic_rows, const int32_t* tok_lens, int32_t n_max,
                                          int32_t* argmax_ids, float* argmax_logp, float* logits, int32_t log_softmax, float* hidden,
                                          const float* hw_embed, const int32_t* hw_lens_h, const int32_t* row_group_h, int32_t n_groups,
                                          int32_t nh_max, int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream);

/* A SAN-M decoder stack WITHOUT input / output layer over an arbitrary memory: the SeACo decoder of SeacoParaformer
 * (seaco_paraformer/model.py:100-110: ParaformerSANMDecoder(use_output_layer=False, wo_input_layer=True), FFN 1024, FSMN k=21,
 * 6 attention layers) attending over the hotword embeddings.  Uses dec->layers / n_layers / heads / fsmn_k / last / after_norm.
 *   memory [t_mem, 512] when mem_shared != 0 (the same hotword memory for every utterance, model.py:306-308), else
 *   [B, t_mem, 512]; mem_lens[B]; x [B, ld_x_rows, 512] of which n_max rows are used; tok_lens[B].
 *   n_run attention layers are run (<= dec->n_layers), then
 *     finish != 0     : decoders3 + after_norm -> hidden [B, n_max, 512]  (ParaformerSANMDecoder.forward, decoder.py:397-449)
 *     attn_probs != 0 : layer n_run-1 stops at its cross-attention and writes utterance 0's probability matrix
 *                       [heads, n_max, t_mem] (forward_asf6 / get_attn_mat, decoder.py:485-513, :123-146); hidden untouched.
 * The workspace query returns exactly what the forward carves; it counts the attn_probs path and a per-utterance memory, which
 * cover every call. */
size_t fa_sanm_decoder_stack_workspace_bytes(int32_t batch, int32_t t_mem, int32_t n_max, int32_t gemm_mode);
int fa_sanm_decoder_stack_forward(const FaDecoder* dec, const float* memory, const int32_t* mem_lens, int32_t mem_shared,
                                  int32_t batch, int32_t t_mem, const float* x, int64_t ld_x_rows, const int32_t* tok_lens,
                                  int32_t n_max, int32_t n_run, int32_t finish, float* hidden, float* attn_probs,
                                  int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream);
/* The same stack over G memories: memory [G, t_mem, 512] (device; rows past a memory's length must be finite), mem_lens_h [G] (host,
 * each in [1, t_mem]) and row_group_h [B] (host, each in [0, G)): utterance b attends over memory row_group_h[b], exactly as the call
 * above gives it with that memory shared.  attn_probs != 0 writes the matrices of the utterances probe_rows_h[0 .. n_probe) (host,
 * each in [0, B)), each against its own memory: [n_probe, heads, n_max, t_mem], the keys past a memory's length 0.  Refusals come
 * before any device work; the workspace query (n_probe 0 without attn_probs) is exactly what the call carves. */
size_t fa_sanm_decoder_stack_grouped_workspace_bytes(int32_t batch, int32_t n_groups, int32_t t_mem, int32_t n_max, int32_t n_probe,
                                                     int32_t gemm_mode);
int fa_sanm_decoder_stack_forward_grouped(const FaDecoder* dec, const float* memory, const int32_t* mem_lens_h, const int32_t* row_group_h,
                                          int32_t n_groups, int32_t batch, int32_t t_mem, const float* x, int64_t ld_x_rows,
                                          const int32_t* tok_lens, int32_t n_max, int32_t n_run, int32_t finish, float* hidden,
                                          float* attn_probs, const int32_t* probe_rows_h, int32_t n_probe, int32_t gemm_mode,
                                          void* workspace, size_t ws_bytes, fa_stream_t stream);

/* ids / best_logp [rows] = arg-max and its log-softmax value of (a (+ b)) W^T + bias — SeACo's hotword_output_layer over
 * cif_attended + dec_attended (seaco_paraformer/model.py:351-355); logp != NULL receives the full log-softmax rows [rows, out_f].
 * The workspace query returns exactly what the forward carves, counting the a + b rows and the logits whether or not b and logp
 * are given. */
size_t fa_linear_argmax_workspace_bytes(int64_t rows, int32_t vocab, int32_t gemm_mode);
int fa_linear_argmax(const FaLinear* lin, const float* a, const float* b_or_null, int64_t rows, int32_t* ids, float* best_logp,
                     float* logp, int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream);

/* SeACo merge with seaco_weight = 1 (seaco_paraformer/model.py:357-378): per token row, the decoder's arg-max where the hotword
 * decoder's arg-max is NO_BIAS, else the hotword decoder's.  merged != NULL additionally receives the merged log-prob rows
 * (dec_logp / dha_logp: full log-softmax rows [rows, vocab]). */
int fa_seaco_merge(const int32_t* dec_ids, const float* dec_best, const int32_t* dha_ids, const float* dha_best, int64_t rows,
                   int32_t no_bias, int32_t* out_ids, float* out_best, const float* dec_logp, const float* dha_logp,
                   float* merged, int32_t vocab, fa_stream_t stream);

/* SeACo's hotword encoder (_hotword_representation, seaco_paraformer/model.py:384-420): decoder.embed, then the n_layers LSTM
 * `bias_encoder` (512 -> 512, gate order i, f, g, o) over the packed batch, then each hotword's top-layer output at its last token.
 * ih[k] = weight_ih_l{k} [2048, 512] with bias b_ih + b_hh [2048] (the input projection of all tokens is one GEMM), hh[k] =
 * weight_hh_l{k} [2048, 512] without bias; in the tensor-core modes both carry their weight planes. */
#define FA_HOTWORD_MAX_LAYERS 8
typedef struct {
  const float* embed;       /* [vocab, 512] */
  int32_t vocab;
  int32_t n_layers;         /* 1 .. FA_HOTWORD_MAX_LAYERS */
  const FaLinear* ih;       /* [n_layers] */
  const FaLinear* hh;       /* [n_layers] */
} FaHotwordEncoder;
/* ids: HOST int32, the hotwords' token ids concatenated (sum of lens entries); lens: HOST [n_hw], each >= 1.  rows: device [n_hw, 512],
 * row i = hotword i's output.  Hotwords run longest first so that step t works on a row prefix: per layer one GEMM over all tokens, then
 * per step one [n_t, 512] x [512, 2048] GEMM and one fused cell launch; no host synchronisation between steps.  Every id is checked
 * against [0, vocab) on the host before anything is enqueued (FA_ERR_ARG, as for n_hw < 1, a length < 1 or a NULL pointer).  The
 * workspace query takes n_hw and the token count (the sum of lens) and returns exactly what the forward carves. */
/* Host only: SeACo's attention-score filter (seaco_paraformer/model.py:320-343) over utterance 0's cross-attention probabilities
 * probs [heads, n_rows, n_hw] (fa_sanm_decoder_stack_forward's attn_probs): picked = torch.topk(probs.sum(0).sum(0),
 * k = min(nfilter, n_hw - 1)).indices followed by n_hw - 1 (the <s> entry), with torch's CPU summation order (a cascade per column, not
 * a left fold) and torch.topk's order among equal scores: the selected rows feed the next attention in that order.  picked holds
 * k + 1 entries; returns k + 1, or FA_ERR_ARG (n_hw < 2, nfilter < 1, a NULL pointer). */
int32_t fa_seaco_asf_select_host(const float* probs, int32_t heads, int32_t n_rows, int32_t n_hw, int32_t nfilter, int32_t* picked);
size_t fa_hotword_encoder_workspace_bytes(int32_t n_hw, int64_t n_tokens, int32_t gemm_mode);
int fa_hotword_encoder_forward(const FaHotwordEncoder* enc, const int32_t* ids, const int32_t* lens, int32_t n_hw, float* rows,
                               int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * FSMN-VAD (funasr/models/fsmn_vad_streaming): the encoder FSMN.forward (encoder.py:355-377) over the LFR-5/1 features of a whole
 * waveform, reduced to the silence posterior per 10 ms frame that the end-point detector reads (model.py:789-792), and the frame
 * energies of ComputeDecibel (model.py:458-529).  The detector itself is sequential threshold logic and stays on the host
 * (funasr_b200/vad.py), as in the reference.
 *   Weights are fp32 [out, in_padded] with the input dimension zero-padded to a multiple of 16 (FaLinear.in_f = padded width):
 *   in1 400->140, in2 140(144)->250 + ReLU, per layer lin 250(256)->128 (no bias), conv_w [128, lorder] (causal depthwise taps,
 *   tap lorder-1 = the current frame), affine 128->250 + ReLU, out1 250(256)->140, out2 140(144)->248.
 *   feats [t, ld_feats] -> sil_prob [t]; scores != NULL additionally receives the full softmax [t, out2.out_f].
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  FaLinear lin;
  const float* conv_w;
  FaLinear affine;
} FaVadLayer;
typedef struct {
  FaLinear in1, in2;
  const FaVadLayer* layers;
  int32_t n_layers, lorder;
  FaLinear out1, out2;
  int32_t sil_ids[4];
  int32_t n_sil, _pad;
} FaVadEncoder;
size_t fa_fsmn_vad_workspace_bytes(const FaVadEncoder* enc, int32_t t);
int fa_fsmn_vad_forward(const FaVadEncoder* enc, const float* feats, int64_t ld_feats, int32_t t, float* sil_prob, float* scores,
                        void* workspace, size_t ws_bytes, fa_stream_t stream);
/* Host-side end-point detector (no GPU work): the per-frame silence posteriors and frame energies of ONE whole recording ->
 * [start_ms, end_ms] segments, as FsmnVADStreaming.inference produces them over its 60 s chunks (fsmn_vad_streaming/model.py:
 * GetFrameState :761-823, WindowDetector :218-320, DetectOneFrame :1158-1302, dynamic end-silence schedule :1003-1067).  The fields
 * are VADXOptions' (model.py:71-174).  schedule: n_schedule pairs {accumulated-speech limit in ms (< 0 = no limit), end silence in ms},
 * used when dynamic_silence != 0 (the reference's default when no max_end_silence_time is given); speech_noise_thres: NaN = the
 * options' value.  Returns the number of segments found (segments receives the first max_segments {start, end} pairs), or a negative
 * status (FA_ERR_ARG also for posteriors outside (0, 1), where the reference's math.log raises). */
typedef struct {
  int32_t sample_rate, detect_mode, max_end_silence_time, max_start_silence_time, window_size_ms, sil_to_speech_time_thres,
      speech_to_sil_time_thres, do_extend, lookback_time_start_point, lookahead_time_end_point, max_single_segment_time,
      noise_frame_num_used_for_snr, frame_in_ms, frame_length_ms;
  double speech_2_noise_ratio, snr_thres, decibel_thres, speech_noise_thres, fe_prior_thres;
} FaVadOptions;
int64_t fa_vad_detect_segments(const double* sil_prob, const double* decibel, int64_t frames, int64_t n_samples, const FaVadOptions* opts,
                               int32_t chunk_ms, int32_t dynamic_silence, const double* schedule, int32_t n_schedule,
                               double speech_noise_thres, int32_t* segments, int64_t max_segments);
/* Host only: the integrate-and-fire trace of one utterance's weights, funasr/utils/timestamp_tools.py:14-34 (cif_wo_hidden: fp32 running
 * sum, reduced by `threshold` after every frame that reaches it; trace[t] = the value before the reduction) — the re-integration step of
 * ts_prediction_lfr6_standard (:67-72). */
int fa_cif_wo_hidden_host(const float* alphas, int64_t n, float threshold, float* trace);
/* Host only: the [start_ms, end_ms] stamps of one utterance from its upsampled CIF weights / fires (us_alphas, us_peaks [n_frames]) and
 * its token count, as funasr/utils/timestamp_tools.py:37-123 (ts_prediction_lfr6_standard, force_time_shift -1.5) computes the stamps
 * (funasr_b200/timestamps.py:_stamps_only is the specification): the weights are rescaled and re-integrated (fa_cif_wo_hidden_host) when
 * the fire count is not n_tokens + 1; one stamp per span between consecutive fires, so the count is not always n_tokens (spans past the
 * token list are stamps too); every value in double arithmetic, + vad_offset_ms, truncated to integer ms.  upsample_rate: 3 for the
 * BiCif head, 1 for plain CIF fires.  The <sil> / </s> rules of the Python routine read token strings: the caller passes n_tokens
 * without a trailing </s>, and no token is spelled <sil>.  out receives the first max_out {start_ms, end_ms} pairs; returns the stamp
 * count (0 when nothing fires or n_tokens == 0), or FA_ERR_ARG. */
int64_t fa_ts_stamps_host(const float* us_alphas, const float* us_peaks, int64_t n_frames, int64_t n_tokens, int32_t upsample_rate,
                          double vad_offset_ms, int32_t* out, int64_t max_out);
/* decibel[f] = 10 log10(sum_{j<400} wav[160 f + j]^2 + 1e-6), f < frames (ComputeDecibel, model.py:516-525). */
int fa_frame_decibels(const float* wav, int64_t n_samples, int32_t frames, float* decibel, fa_stream_t stream);
/* The same two stages over a ragged batch of recordings, for long audio over many recordings at once.
 * fa_fsmn_vad_forward_batch: feats [batch * t_max, ld_feats] (row b's frames at rows b * t_max ..), frames [batch] HOST (row b's frame
 * count, <= t_max) -> sil_prob [batch, t_max]; workspace of fa_fsmn_vad_batch_workspace_bytes(enc, batch, t_max).  Row b's valid
 * values equal fa_fsmn_vad_forward on that row alone, bit for bit (every stage computes a frame on its own and the memory is causal and
 * masked at the row's length); values past frames[b] are unspecified.
 * fa_frame_decibels_batch: wav [batch, stride], frames [batch] DEVICE (each row needs (frames - 1) * 160 + 400 samples) ->
 * decibel [batch, t_max], frames past frames[b] unwritten; row b equals fa_frame_decibels on that row alone. */
size_t fa_fsmn_vad_batch_workspace_bytes(const FaVadEncoder* enc, int32_t batch, int32_t t_max);
int fa_fsmn_vad_forward_batch(const FaVadEncoder* enc, const float* feats, int64_t ld_feats, const int32_t* frames, int32_t batch, int32_t t_max,
                              float* sil_prob, void* workspace, size_t ws_bytes, fa_stream_t stream);
int fa_frame_decibels_batch(const float* wav, int64_t stride, const int32_t* frames, int32_t batch, int32_t t_max, float* decibel,
                            fa_stream_t stream);

/* Greedy post-filter (paraformer/model.py:655-666): keep argmax_ids[b, k] for k < tok_lens[b] that are not
 * in {blank=0, sos=1, eos=2}; out_ids [B, n_max] (padded with -1), out_lens [B]. */
int fa_greedy_filter(const int32_t* argmax_ids, const int32_t* tok_lens, int32_t batch, int32_t n_max,
                     int32_t sos, int32_t eos, int32_t blank, int32_t* out_ids, int32_t* out_lens,
                     fa_stream_t stream);

/* CTC greedy head of SenseVoiceSmall (sense_voice/model.py:1003-1025, ctc/ctc.py:192-203): logits = enc W^T + b,
 * log_softmax, arg-max per frame, torch.unique_consecutive, drop blank.
 *   enc [B,T,512], lens[B] -> out_ids [B,T] (padded with -1), out_lens [B]; if logp != NULL it receives the
 *   full log_softmax [B,T,vocab] (parity checks); argmax_ids [B,T] is scratch/diagnostic output.  The workspace query returns
 *   exactly what the forward carves, counting the logits whether or not logp is given. */
size_t fa_ctc_greedy_workspace_bytes(int32_t batch, int32_t t_max, int32_t vocab, int32_t gemm_mode);
int fa_ctc_greedy_forward(const FaLinear* ctc_lo, const float* enc, const int32_t* lens, int32_t batch, int32_t t_max,
                          int32_t blank, int32_t* argmax_ids, int32_t* out_ids, int32_t* out_lens, float* logp,
                          int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream);

/* Polyphase sinc resampler (torchaudio.functional.resample semantics, used by FunASR's loader when the input rate differs from
 * the model's: funasr/utils/load_utils.py:176-178).  orig / nnew are the rates divided by their gcd, table [nnew, 2*width + orig]
 * is torchaudio's _get_sinc_resample_kernel (funasr_b200/resample.py builds it).  x [B, x_stride] with lens[B] valid samples ->
 * y [B, y_stride], first y_cap columns written (zero beyond each row's length), out_lens[b] = min(ceil(nnew*lens[b]/orig), y_cap). */
int fa_resample(const float* x, const int32_t* lens, int32_t batch, int64_t x_stride, const float* table, int32_t orig,
                int32_t nnew, int32_t width, float* y, int64_t y_stride, int32_t y_cap, int32_t* out_lens, fa_stream_t stream);

/* out[i, :] = table[ids[i], :]  (torch.nn.Embedding forward; CTTransformer.embed, ct_transformer/model.py:120).  ids are clamped to the table. */
int fa_embedding(const int32_t* ids, const float* table, int32_t dim, int32_t vocab, int64_t n, float* out, fa_stream_t stream);

/* Sample decode of the audio loader on the device (funasr/utils/load_utils.py:48-179; torchaudio.load(normalize=True) scaling): interleaved
 * PCM frames (device memory) -> mono fp32 [frames] in [-1, 1), channels averaged.  sample_format: 0 = f32, 1 = s16le, 2 = s24le packed,
 * 3 = s32le, 4 = u8.  The container (RIFF WAV header) is parsed on the host (funasr_b200/audio.py). */
int fa_pcm_decode(const void* pcm, int32_t sample_format, int32_t channels, int64_t frames, float* out, fa_stream_t stream);

/* ---- Audio at any sample rate and PCM layout: the input descriptor of fa_offline_infer_audio, fa_offline_infer_vad_audio,
 * fa_vad_infer_audio and fa_spk_embed_audio.  Two resamplers to 16 kHz, each pinned to its own reference:
 *   FA_RESAMPLE_LOADER   torchaudio's sinc resampler (hann window, 6 zeros, rolloff 0.99) as FunASR's Python loader and
 *                        inference(fs=) apply it: the table of fa_loader_resample_table_host and fa_resample's arithmetic.
 *   FA_RESAMPLE_RUNTIME  the C++ runtime's kaldi LinearResample (cutoff 0.99 * 0.5 * min rate, 6 zeros, flushed) as its WavResample
 *                        applies it: the tables of fa_runtime_resample_table_host, sums in tap order without contraction.
 * At 16 000 Hz neither resamples (both references skip it).  Both give ceil(16000 n / rate) samples for n frames. */
#define FA_RESAMPLE_LOADER 0
#define FA_RESAMPLE_RUNTIME 1
typedef struct FaAudioFormat {
  int32_t sample_format;  /* fa_pcm_decode's codes: 0 f32, 1 s16le, 2 s24le packed, 3 s32le, 4 u8 */
  int32_t channels;       /* 1..64, interleaved; averaged to mono like the loader */
  int32_t sample_rate;    /* Hz of the caller's buffers, 1 000..192 000 */
  int32_t resampler;      /* FA_RESAMPLE_LOADER or FA_RESAMPLE_RUNTIME */
} FaAudioFormat;
/* Host only.  Rates outside 1 000..192 000 Hz -> FA_ERR_ARG; a table above 32 MiB (for example 16 001 Hz in loader mode, 1 GB) ->
 * FA_ERR_UNSUPPORTED.  Otherwise the number of floats of the weight table, written when weights is not NULL and cap holds it.
 * fa_loader_resample_table_host: resample.sinc_resample_table(rate, new_rate) bit for bit: *orig / *nnew the rates over their gcd,
 *   *width, table [nnew, 2 * width + orig].
 * fa_runtime_resample_table_host: LinearResample(rate, new_rate, 0.99 * 0.5 * min rate, 6)'s weights: *in_unit / *out_unit the
 *   rates over their gcd, per output phase p < out_unit the first input index first[p] (may be negative) and n_taps[p] weights in
 *   row p of weights [out_unit, *max_taps] (zero padded).  first / n_taps are written with the weights.
 * fa_runtime_resample_out_len_host: LinearResample's flushed output count for n input frames (64-bit tick arithmetic). */
int64_t fa_loader_resample_table_host(int32_t rate, int32_t new_rate, int32_t* orig, int32_t* nnew, int32_t* width, float* table, int64_t cap);
int64_t fa_runtime_resample_table_host(int32_t rate, int32_t new_rate, int32_t* in_unit, int32_t* out_unit, int32_t* max_taps,
                                       int32_t* first, int32_t* n_taps, float* weights, int64_t cap);
int64_t fa_runtime_resample_out_len_host(int32_t rate, int32_t new_rate, int64_t n);
/* One uploaded resampling table (device pointers).  mode: FA_RESAMPLE_LOADER (in_unit / out_unit = orig / nnew, width, taps =
 * 2 * width + orig, weights [out_unit, taps]; first / n_taps NULL, or [out_unit] each row's span of nonzero taps, which is all a sum
 * over finite samples needs: most of a row lies outside the window, where the table is exactly zero), FA_RESAMPLE_RUNTIME (in_unit /
 * out_unit, taps = the longest row, weights [out_unit, taps], first / n_taps [out_unit]); or -1: decode only (16 kHz input), every
 * other field ignored. */
typedef struct FaIngestTable {
  int32_t mode;
  int32_t in_unit, out_unit, width, taps;
  int32_t _pad;
  const float* weights;
  const int32_t* first;
  const int32_t* n_taps;
} FaIngestTable;
/* The handle's ingest, one launch: ragged interleaved PCM rows in device memory -> y [batch, stride] mono fp32 at 16 kHz.  rows
 * [batch][3] int64 on the device: byte offset of the row in raw (a multiple of the sample size), frames n, output length (<= stride).
 * Each output decodes the frames it needs straight from the bytes (fa_pcm_decode's operations and channel mean) and applies the
 * table: loader mode bit for bit fa_pcm_decode then fa_resample (with spans: for finite samples, which every integer format is); runtime mode out[t] = sum over taps j of w[p][j] * x[first[p] +
 * u * in_unit + j] (u = t / out_unit, p = t % out_unit), indices outside [0, n) skipped, each product and add rounded on its own.
 * Zero past each row's output length. */
int fa_ingest_pcm(const void* raw, const int64_t* rows, int32_t batch, int32_t sample_format, int32_t channels, const FaIngestTable* table,
                  float* y, int64_t stride, fa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * CAM++ speaker embedding (funasr/models/campplus/model.py CAMPPlus, feat 80, embedding 192, growth 32, bn 128, init 128,
 * batchnorm-relu).  Eval-mode BatchNorm that follows a conv is folded into that conv's weights and bias by the caller; BatchNorm
 * that precedes ReLU + conv is passed as a per-channel affine (scale = g / sqrt(var + eps), shift = b - mean * scale).
 * ------------------------------------------------------------------------------------------- */
/* FCM conv (Conv2d 3x3 or 1x1 over (freq, time), stride (stride_f, 1), padding ksize / 2) with its BN folded:
 * w [ksize * ksize][c_in][32] (tap-major kf * ksize + kt, output channels contiguous), b [32]. */
typedef struct {
  const float* w;
  const float* b;
  int32_t c_in, c_out, ksize, stride_f;
} FaCamConv2d;
/* One CAMDenseTDNNLayer (components.py): nonlinear1 as an affine [c_in]; linear1 c_in -> 128 with nonlinear2's BN folded (ReLU
 * applied); CAMLayer: local_w [3][128][32] (tap, input channel, output channel), linear1 w1 [64][128] + b1, linear2 w2 [32][64] + b2. */
typedef struct {
  const float* bn1_scale;
  const float* bn1_shift;
  FaLinear linear1;
  const float* local_w;
  const float* w1;
  const float* b1;
  const float* w2;
  const float* b2;
} FaCamLayer;
typedef struct {
  const float* scale;   /* nonlinear BN as an affine [in_f] */
  const float* shift;
  FaLinear linear;      /* in_f -> in_f / 2, no bias */
} FaCamTransit;
/* fcm: head.conv1, layer1.0.{conv1, conv2, shortcut}, layer1.1.{conv1, conv2}, layer2.0.{conv1, conv2, shortcut},
 * layer2.1.{conv1, conv2}, head.conv2.  tdnn: Conv1d(320, 128, 5, stride 2, pad 2) as [128][5 * 320] (w[o][k * 320 + c]) with its BN
 * folded.  layers: n_layers[0] + n_layers[1] + n_layers[2] CAM layers in order.  out_*: out_nonlinear BN as an affine [512].
 * dense: 1024 -> 192 with the affine-free BN folded. */
typedef struct {
  FaCamConv2d fcm[12];
  FaLinear tdnn;
  const FaCamLayer* layers;
  int32_t n_layers[3];
  int32_t dilation[3];
  FaCamTransit transit[3];
  const float* out_scale;
  const float* out_shift;
  FaLinear dense;
} FaCampplus;
/* Features (campplus/utils.py extract_feature): torchaudio kaldi.fbank(wav, num_mel_bins=80) with its defaults (no x32768 scaling,
 * window from `tables`: fa_fbank_make_tables with the povey window), then each utterance's mean over its own frames is subtracted.
 * wav [B, wav_stride] (lens >= 400 samples) -> feats [B, t_max, 80] (rows >= feat_lens[b] zero, pad_list(..., 0)), feat_lens [B].
 * feat_lens[b] is the utterance's full frame count even when it exceeds t_max; such an utterance keeps its first t_max frames, and
 * the mean subtracted from them is the mean over those t_max frames.  Nothing outside feats [B, t_max, 80] is written. */
int fa_campplus_features(const float* wav, const int32_t* wav_lens, int32_t batch, int64_t wav_stride, const float* tables,
                         float* feats, int32_t* feat_lens, int32_t t_max, fa_stream_t stream);
/* CAMPPlus.forward: feats [B, t, 80] (every frame used, no mask) -> emb [B, 192].  Stream-ordered, no host synchronisation.
 * 2 <= t <= 18 800 (at most 94 CAM segments of 100 TDNN frames, ~188 s): t < 2 -> FA_ERR_ARG, t > 18 800 -> FA_ERR_UNSUPPORTED,
 * both before anything is enqueued, and the workspace query returns 0 for either.  At t == 2 the single TDNN frame's unbiased
 * std is 0 / 0, so emb is NaN, as in the reference. */
size_t fa_campplus_workspace_bytes(const FaCampplus* model, int32_t batch, int32_t t, int32_t gemm_mode);
int fa_campplus_forward(const FaCampplus* model, const float* feats, int32_t batch, int32_t t, float* emb, int32_t gemm_mode,
                        void* workspace, size_t ws_bytes, fa_stream_t stream);
/* fa_campplus_forward with a padded length per row: row b's embedding equals fa_campplus_forward on feats[b, :ext_h[b]] alone
 * (a batch padded to ext_h[b] frames), bit for bit.  Frames at or past ext_h[b] are never read.  ext_h [B] is a HOST array,
 * 2 <= ext_h[b] <= t (FA_ERR_ARG otherwise), t <= 18 800 (FA_ERR_UNSUPPORTED), both before anything is enqueued; it may be reused
 * once the call returns.  ext_h[b] == t for every row is fa_campplus_forward bit for bit.  Workspace:
 * fa_campplus_ext_workspace_bytes (0 where fa_campplus_workspace_bytes is 0, at least that much otherwise). */
size_t fa_campplus_ext_workspace_bytes(const FaCampplus* model, int32_t batch, int32_t t, int32_t gemm_mode);
int fa_campplus_forward_ext(const FaCampplus* model, const float* feats, int32_t batch, int32_t t, float* emb, int32_t gemm_mode,
                            void* workspace, size_t ws_bytes, fa_stream_t stream, const int32_t* ext_h);
/* Layer entry points of the forward (exposed for parity tests).  conv2d: x [B][f_in][t][c_in] channels last -> y [B][f_out][t][32],
 * y = act(conv(x) + b (+ res)), res in y's layout or NULL. */
int fa_campplus_conv2d(const FaCamConv2d* conv, const float* x, int32_t batch, int32_t f_in, int32_t t, const float* res, float* y,
                       int32_t relu, fa_stream_t stream);
/* CAMLayer: h [B * t, 128] -> out[(b t + i) * ld_out + o] (32 columns); gates [B][ceil(t / 100)][32] receives the context gates. */
int fa_campplus_cam(const float* h, int32_t batch, int32_t t, int32_t dilation, const float* local_w, const float* w1, const float* b1,
                    const float* w2, const float* b2, float* gates, float* out, int64_t ld_out, fa_stream_t stream);
/* out_nonlinear + StatsPool: x [B * t, channels] -> stats [B, 2 * channels] = mean || unbiased std over t of relu(x * scale + shift). */
int fa_campplus_stats_pool(const float* x, int32_t batch, int32_t t, int32_t channels, const float* scale, const float* shift,
                           float* stats, fa_stream_t stream);

/* Split fp32 [rows, cols] into three fp16 planes [3][rows][cols_pad] (hi, mid, lo; zero padded columns):
 * weight repack for the tensor-core GEMM path (called once per weight after load_pretrained_model). */
int fa_split_planes(const float* src, int64_t ld_src, int64_t rows, int32_t cols, int32_t cols_pad,
                  void* planes, fa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Handle-style offline recogniser (no Python, no torch) — the counterpart of FunASR's C++ runtime surface
 * runtime/onnxruntime/include/funasrruntime.h:100-116:
 *   fa_offline_init          <-> FunOfflineInit(model_path, thread_num, use_gpu, batch_size)            :100
 *   fa_offline_infer         <-> FunOfflineInferBuffer(handle, sz_buf, n_len, ...) ("pcm" = s16le)       :103-106
 *   fa_offline_result_ids    <-> FunASRGetResult(result, n_index)   (token ids; the tokenizer stays with the caller) :69
 *   fa_offline_result_audio_seconds <-> FunASRGetRetSnippetTime                                         :77
 *   fa_offline_free_result / fa_offline_uninit <-> FunASRFreeResult :75 / FunOfflineUninit              :116
 * model_file: flat tensor file written by funasr_b200/pack.py from a FunASR state_dict (same tensor names as model.pt) plus
 * am.mvn and the kaldi mel/window tables.  pcm_format: 0 = float32 in [-1,1], 1 = int16 little endian (converted on the
 * device, halves the H2D bytes).  bufs are HOST pointers, n_samples[i] >= 400.  Returns NULL on error
 * (fa_offline_last_error() says why); there is no CPU fallback.  fa_offline_init refuses a BiCif timestamp head (recognised by
 * predictor.upsample_cnn.weight) without __ts_config__, with a missing or misshapen tensor or with upsample_times != 3 before it
 * touches a device, naming the piece.
 * ------------------------------------------------------------------------------------------- */
void* fa_offline_init(const char* model_file, int32_t device, int32_t gemm_mode);
void* fa_offline_infer(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format);
/* Same with a hotword memory for a ContextualParaformer model file (FunOfflineInferBuffer's `hw_emb`, funasrruntime.h:104): hw_embed
 * is HOST memory [n_hotwords, 512], the rows CompileHotwordEmbedding produces (last entry = the <s> hotword).  Required when
 * fa_offline_is_contextual(handle), ignored otherwise. */
void* fa_offline_infer_hw(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                          const float* hw_embed, int32_t n_hotwords);
int32_t fa_offline_is_contextual(const void* handle);
/* 1 when the model file carries BiCifParaformer's upsampled CIF timestamp head (predictor.upsample_cnn.*, predictor.blstm.*,
 * predictor.cif_output2.* and __ts_config__, written by funasr_b200/pack.py): its token branch then runs CifPredictorV3's sequential
 * fp32 `cif`, and every result carries per-token stamps (fa_offline_result_stamps).  0 otherwise, or for NULL. */
int32_t fa_offline_has_timestamps(const void* handle);
/* SeacoParaformer (paraformer-zh; seaco_paraformer/model.py:50-581), recognised by __seaco_config__ [no_bias, nfilter, lstm layers]
 * (funasr_b200/pack.py:write_seaco_model_file).  Before it touches a device fa_offline_init refuses, naming the piece: a file that is
 * also contextual, decoder.embed.0.weight other than [vocab, 512], a bias_encoder weight other than [2048, 512] or bias other than
 * [2048], fewer than 6 SeACo decoder layers or a misshapen one, hotword_output_layer other than [vocab, 512], no_bias outside
 * [0, vocab), nfilter < 0.  fa_offline_is_seaco: 1 for such a handle, 0 otherwise or for NULL.
 * fa_offline_hotword_embed: the hotword rows of a SeACo handle, the `hw_emb` of FunOfflineInferBuffer: ids (HOST, the hotwords' token
 * ids concatenated) and lens [n] (HOST) -> rows_host [n, 512] (HOST), each hotword's top-layer bias_encoder output at its last token
 * (fa_hotword_encoder_forward in the handle's gemm_mode).  The caller appends the <s> entry ({1}) as generate_hotwords_list does.  An
 * id outside the vocabulary fails before any launch, naming the hotword; any other handle kind is refused.  FA_OK or a negative status
 * (fa_offline_last_error()).
 * fa_offline_infer_hw / fa_offline_infer_vad on a SeACo handle take these rows (hw_embed [n_hotwords, 512], last row the <s> entry).
 * No rows (n_hotwords 0): the plain decoder distribution (model.py:381-382).  Otherwise _seaco_decode_with_ASF: with more rows than
 * nfilter, the SeACo decoder's attention on utterance 0 (of each VAD pack for long audio) keeps the nfilter rows it attends to most
 * plus the <s> row (fa_seaco_asf_select_host); the SeACo decoder over the acoustic embeddings and over the decoder's hidden states,
 * hotword_output_layer's arg-max of their sum, and the NO_BIAS merge.  Stamps as for BiCif when the file has the timestamp head. */
int32_t fa_offline_is_seaco(const void* handle);
int fa_offline_hotword_embed(void* handle, const int32_t* ids, const int32_t* lens, int32_t n, float* rows_host);
/* Host copy of a tensor of the model file by its FunASR state_dict name (e.g. "bias_embed.weight" for the hotword encoder that
 * runs on the host); owned by the handle.  NULL if absent. */
const float* fa_offline_host_tensor(void* handle, const char* name, int64_t* numel);
int32_t fa_offline_result_count(const void* result);
const int32_t* fa_offline_result_ids(const void* result, int32_t index, int32_t* n_ids);
float fa_offline_result_audio_seconds(const void* result);
/* n_stamps {start_ms, end_ms} pairs of entry `index` (owned by the result): the stamps the reference's BiCifParaformer.inference
 * gives (bicif_paraformer/model.py:402-407), computed by fa_ts_stamps_host from the head's upsampled weights.  One stamp per span
 * between fires, which is one per token id in the usual case; the count is returned on its own.  Stamps are per token id: the
 * <sil>-entry and </s> rules of the Python routine read token strings, which the handle does not have; ids 0 / 1 / 2 (blank, <s>,
 * </s>) are already removed by the greedy filter.  For fa_offline_infer_vad results the stamps are absolute: each segment's are
 * shifted by its start ms and concatenated in time order (auto_model.py:1008-1022).  NULL with 0 for a model without the head, for
 * an entry without stamps and for NULL / out-of-range arguments. */
const int32_t* fa_offline_result_stamps(const void* result, int32_t index, int32_t* n_stamps);
/* SenseVoiceSmall (sense_voice/model.py:918-1034).  fa_offline_init recognises its model file (funasr_b200/pack.py:
 * write_sensevoice_model_file) by __sv_config__ and refuses, before it touches a device and naming the piece: a file with both
 * __config__ and __sv_config__, a missing tensor, d_model != 512 or heads != 4 (the tensor-core attention shapes), a vocabulary above
 * 61440 (the CTC arg-max).  fa_offline_is_sensevoice: 1 for such a handle, 0 otherwise or for NULL.
 * fa_offline_infer_sv: like fa_offline_infer, utterance i queried with the embedding rows language_ids[i], 1, 2, textnorm_ids[i]
 * (SenseVoiceSmall.lid_dict / textnorm_dict ids; NULL = 0 "auto" / 15 "woitn", the Python model's defaults).  An id outside the
 * embedding table fails the call before any launch, naming the utterance.  Each result is the CTC-collapsed ids including the four tag
 * tokens (SenseVoiceSmall.inference's token_int); no stamps.  The CTC head materialises the logits: vocab x 4 bytes per frame (25055
 * tokens: about 3.2 GB at 64 utterances of 30 s).  fa_offline_infer / fa_offline_infer_hw on a SenseVoice handle use the defaults and
 * ignore hotwords; fa_offline_infer_sv on any other handle fails. */
int32_t fa_offline_is_sensevoice(const void* handle);
void* fa_offline_infer_sv(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                          const int32_t* language_ids, const int32_t* textnorm_ids);
/* Host only: the result text of SenseVoice's CTCSearch in FunASR's C++ runtime (runtime/onnxruntime/src/sensevoice-small.cpp:305-355)
 * over ids [n] and the token list tokens [n_tokens] (an id outside it, or any id when n_tokens is 0, reads as its decimal number):
 * the first three tags concatenated, " ", then the pieces from the fifth id on, a piece containing U+2581 adding " " and the piece
 * without its first 3 bytes; U+3002 after the language tag <|zh|> and "." otherwise when the fourth tag is <|withitn|>.  With exactly 3 ids the
 * fourth tag reads as empty (the runtime reads one past its token vector there).  Writes at most cap - 1 bytes and a NUL to out when
 * cap > 0; returns the text's length in bytes, or -1 for a bad argument. */
int64_t fa_sv_ctc_text_host(const int32_t* ids, int32_t n, const char* const* tokens, int32_t n_tokens, char* out, int64_t cap);
void fa_offline_free_result(void* result);
void fa_offline_uninit(void* handle);
const char* fa_offline_last_error(void);
/* Threads.  Every handle (recogniser, VAD, speaker, punctuation, aligner) may be shared by any number of threads.  A call checks its
 * arguments on the calling thread; a malformed call fails there, with its own fa_offline_last_error, before it touches the device.
 * The recogniser's decoding calls (fa_offline_infer*, fa_offline_infer_vad*) then join the handle's request pool: the thread that
 * finds no pass running leads one, draining the queued calls that may share GPU packs (in arrival order, up to an hour of padded
 * audio), decoding them together and waking their threads; the others wait.  The library creates no thread.  Each call still gets
 * exactly what it gets alone: every row carries the padded length of the batch the reference decodes it in (the call's whole batch;
 * a long recording's own packs), and the CIF predictor and timestamp head give it what that batch gives it
 * (fa_cif_predictor_forward_ext).  Calls with hotword rows (contextual and SeACo models) share packs too: the reference gives every
 * utterance of a batch that batch's hotword memory (for SeACo with more rows than nfilter, the rows the filter picks on the batch's
 * utterance 0), so each reference pack keeps its own memory and each row attends over its own (fa_attention_grouped); identical rows
 * (the same count and bytes) are one memory per pack, and a pack holds at most 4096 memory rows (memories x the longest).  Diarized
 * calls (fa_offline_infer_vad_spk, fa_offline_infer_vad_audio with a speaker handle) share packs too, and each group of a pass runs
 * one speaker stage over all of its diarized recordings (each still clustered on its own); a refusal of that stage fails only its own
 * call.  Long-audio calls share passes only with the same VAD handle and FaLongAudioOptions, diarized calls only with the same
 * speaker handle (preset_spk_num may differ).
 * A device failure during a pass fails every call of that pass with its message.  Punctuation calls (fa_punc_infer) on one handle
 * share lockstep steps: the thread that finds no step running leads, each step admitting the queued calls in arrival order and scoring
 * one window of every active text of every admitted call, and each text gets exactly what it gets alone (fa_punc_infer below).
 * Speaker-only calls (fa_spk_embed*, fa_spk_cluster) on one handle share passes: the leader drains the queued calls in arrival order
 * (up to an hour of padded audio and 8 192 clustering rows), embeds every row at its own call's padded length
 * (fa_campplus_forward_ext) in packs sorted by that length, and clusters every clustering call's set in one batched spectral pass; each
 * call gets exactly what it gets alone.  The aligner's and the VAD-only (fa_vad_infer*) calls hold the handle's lock for their device
 * work and run one after another.  A call that uses several handles (fa_offline_infer_vad*) locks them in the order recogniser, VAD,
 * speaker, so recognisers that share a VAD handle cannot deadlock; the speaker pool's leader holds only the speaker lock, and the
 * punctuation and aligner locks are never held with another.
 * fa_offline_last_error is per thread.  Uninit a handle only after every call on it has returned. */
/* Calls the recogniser handle's pool has decoded since init, and the GPU packs it decoded them in (packs < calls: calls were pooled).
 * 0, or FA_ERR_ARG for a NULL argument. */
int fa_offline_pool_stats(const void* handle, int64_t* calls, int64_t* packs);

/* ---------------------------------------------------------------------------------------------
 * Handle-style FSMN-VAD and long-audio recognition (no Python, no torch) — FunASR's `vad_model` path: FsmnVADStreaming.inference
 * (fsmn_vad_streaming/model.py) and AutoModel.inference_with_vad (auto/auto_model.py:852-1035), one recording at a time.
 * ------------------------------------------------------------------------------------------- */
/* Run options of the VAD: what FsmnVADStreaming.inference accepts.  dynamic_silence != 0: the per-chunk dynamic end-silence schedule
 * (the default when no max_end_silence_time is given, model.py:1003-1067); 0: a fixed end silence of max_end_silence_time ms, or of
 * the model file's value when max_end_silence_time <= 0 (the C++ runtime's fixed threshold).  speech_noise_thres: NaN = the model's. */
typedef struct {
  int32_t dynamic_silence;
  int32_t max_end_silence_time;
  double speech_noise_thres;
} FaVadRunOptions;
/* fa_vad_init: model file written by funasr_b200/pack.py:write_vad_model_file (FSMN weights under the reference's state_dict names,
 * the frontend tables, CMVN [2, 400] and the VADXOptions; input dimensions are zero-padded to a multiple of 16 here).
 * fa_vad_infer: ONE host recording (pcm_format 0 = float32 in [-1, 1], 1 = s16le; 16 kHz) -> segments [start_ms, end_ms].  On the
 * device: Fbank + LFR 5/1 + CMVN, the FSMN and the frame energies; then one copy of two floats per frame to the host and the end-point
 * walk of fa_vad_detect_segments.  opts NULL = dynamic schedule, the model's threshold.  A recording shorter than one 25 ms frame gives
 * no segment.  NULL on error (fa_offline_last_error()). */
void* fa_vad_init(const char* model_file, int32_t device);
void fa_vad_uninit(void* vad);
void* fa_vad_infer(void* vad, const void* buf, int64_t n_samples, int32_t pcm_format, const FaVadRunOptions* opts);
/* n_segments {start_ms, end_ms} pairs, owned by the result. */
const int32_t* fa_vad_result_segments(const void* result, int64_t* n_segments);
/* The per-frame values the walk read: [2][frames] (silence posterior, then frame energy in dB), owned by the result. */
const float* fa_vad_result_frames(const void* result, int64_t* frames);
float fa_vad_result_audio_seconds(const void* result);
void fa_vad_free_result(void* result);

/* Long-audio options: auto_model.py's batch_size_s / batch_size_threshold_s (seconds) and merge_vad / merge_length_s
 * (utils/vad_utils.py:57-91), plus the VAD run options.  NULL = 300, 60, no merge, 15, dynamic schedule. */
typedef struct {
  int32_t batch_size_s;
  int32_t batch_size_threshold_s;
  int32_t merge_vad;
  int32_t merge_length_s;
  FaVadRunOptions vad;
} FaLongAudioOptions;
/* Every recording on its own, as inference_with_vad treats it (the recordings are uploaded together and scored by one batched VAD
 * pass, which gives each the values it gets alone): VAD, optional merge, segments sorted by duration and packed
 * (fa_pack_segments), each pack gathered from the device-resident recording into one zero-padded batch (fa_gather_segments) and
 * decoded like fa_offline_infer_hw (the same hotword memory for every segment), results restored to time order.  Result entry i
 * holds recording i: fa_offline_result_ids = the ids of its segments concatenated in time order, fa_offline_result_segments = its
 * segments, fa_offline_result_stamps = its absolute stamps (BiCif).  A pack whose segments all yield no token empties the recording's
 * ids and stamps (auto_model.py:990-999; its segments are kept with
 * 0 tokens); a recording without speech has no segment.  A segment shorter than 400 samples fails the call with a message naming it.
 * asr and vad must live on the same device.  NULL on error (fa_offline_last_error()). */
void* fa_offline_infer_vad(void* asr, void* vad, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                           const float* hw_embed, int32_t n_hotwords, const FaLongAudioOptions* opts);
/* The same for a SenseVoice handle with one query per recording (language_ids[i], textnorm_ids[i]; NULL = the defaults), applied to
 * all of that recording's segments; an id outside the embedding table fails the call naming the recording.  SenseVoiceSmall.inference
 * returns a result for every segment, so a pack never empties a recording.  fa_offline_infer_vad on a SenseVoice handle uses the
 * defaults; fa_offline_infer_vad_sv on any other handle fails. */
void* fa_offline_infer_vad_sv(void* asr, void* vad, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format,
                              const int32_t* language_ids, const int32_t* textnorm_ids, const FaLongAudioOptions* opts);
/* n_segments {start_ms, end_ms, n_tokens} triples of recording `index` (time order); NULL with 0 for results of fa_offline_infer. */
const int32_t* fa_offline_result_segments(const void* result, int32_t index, int32_t* n_segments);
/* out [rows, stride] = rec[starts[r] .. starts[r] + lens[r]) then zeros (rec [n_rec] fp32; starts int64 / lens int32 [rows] device;
 * stride % 4 == 0, 16-byte aligned out; 0 <= lens[r] <= stride; samples at or beyond n_rec read as zero): the batch of VAD segments
 * that slice_padding_audio_samples (utils/vad_utils.py:28-54) + pad_sequence form. */
int fa_gather_segments(const float* rec, int64_t n_rec, const int64_t* starts, const int32_t* lens, int32_t rows, int64_t stride,
                       float* out, fa_stream_t stream);
/* Host only: the packing of auto_model.py:916-989 (funasr_b200/long_audio.py:pack_segments).  segments [n][2] ms -> order [n]
 * (indices sorted by duration, ties in time order) and packs [n][2] ([begin, end) ranges into order).  Returns the pack count, or
 * FA_ERR_ARG. */
int64_t fa_pack_segments(const int32_t* segments, int64_t n, int32_t batch_size_s, int32_t batch_size_threshold_s, int32_t* order,
                         int32_t* packs);
/* Host only: merge_vad (utils/vad_utils.py:57-91, funasr_b200/vad.py:merge_vad).  segments [n][2] -> out [<= 2n][2]; returns the
 * count, or FA_ERR_ARG. */
int64_t fa_merge_vad(const int32_t* segments, int64_t n, int32_t max_length_ms, int32_t min_length_ms, int32_t* out);

/* ---- Speaker diarization (CAMPPlus, campplus/model.py; ClusterBackend and the post-processing of campplus/cluster_backend.py and
 * utils.py; funasr_b200/diarization.py and long_audio.py are the specification)
 * fa_spk_init: model file written by funasr_b200/pack.py:write_campplus_model_file (the CAMPPlus state_dict under its own names,
 * unfolded, the povey-window fbank tables and __spk_config__ [80, 192, 32, 4, 128]).  Refused before any device is touched, naming the
 * piece: a missing or misshapen tensor, another __spk_config__, a file that also carries another model kind's config.  The BatchNorms
 * are folded on the host in float64 exactly as CampplusEngine folds them, so embeddings are bit-identical to it in every gemm_mode.
 * fa_spk_embed: batch HOST recordings (pcm_format 0 = float32, 1 = s16le; 16 kHz; ragged) -> emb_host [batch, 192]: CAMPPlus.inference
 * (features zero-padded to the longest input, the padded frames taking part in every mean; fa_campplus_features, fa_campplus_forward
 * in slices of 1 GiB of workspace, or fa_campplus_forward_ext at each call's padded length where pooled calls share a pack).  An input under 400 samples (FA_ERR_ARG) or with
 * more than 18 800 feature frames (FA_ERR_UNSUPPORTED) fails the call on its own thread before it joins the pool, naming the input.
 * Concurrent calls on one handle share passes (Threads above), and a lone call launches what one call launched before pooling.  FA_OK
 * or a negative status (fa_offline_last_error()).
 * fa_spk_cluster: ClusterBackend()(emb_host [n, 192], oracle_num = preset_spk_num > 0 ? preset_spk_num : None) -> labels [n] (before
 * correct_labels): fewer than 20 rows one speaker; fewer than 2048 the spectral path (fa_spk_laplacian, fa_spk_tridiagonalize,
 * fa_sym_tridiag_smallest_host, fa_spk_back_transform, the eigengap count unless preset, k-means); 2048 or more k-means on the
 * normalised rows with a preset count, and without one FA_ERR_UNSUPPORTED (the reference's UMAP + HDBSCAN path is not provided, refused
 * on the calling thread); merge_by_cos at 0.78 when no count is preset.  Concurrent calls on one handle are clustered together (the
 * _batch entries below), each set with exactly its own result; a refusal of one set (preset_spk_num above n) fails only its call. */
void* fa_spk_init(const char* model_file, int32_t device, int32_t gemm_mode);
void fa_spk_uninit(void* spk);
int fa_spk_embed(void* spk, const void* const* bufs, const int64_t* n_samples, int32_t batch, int32_t pcm_format, float* emb_host);
int fa_spk_cluster(void* spk, const float* emb_host, int32_t n, int32_t preset_spk_num, int32_t* labels);
/* Calls the speaker handle's pool has served since init (fa_spk_embed*, fa_spk_cluster) and the passes it ran them in (passes < calls:
 * calls were pooled).  0, or FA_ERR_ARG for a NULL argument. */
int fa_spk_pool_stats(const void* spk, int64_t* calls, int64_t* passes);
/* fa_offline_infer_vad (language_ids / textnorm_ids: fa_offline_infer_vad_sv's, NULL except on SenseVoice) followed, for every
 * recording that decoded at least one token, by LongAudioPipeline.generate's diarization in vad_segment mode: sv_chunk's 1.5 s windows
 * every 0.75 s over each VAD segment (the last pulled back), gathered from the device-resident recording with zero tails
 * (fa_gather_segments) and embedded in slices, clustered as fa_spk_cluster (preset_spk_num <= 0: none), post-processed (postprocess,
 * distribute_spk) -> one speaker per segment: fa_offline_result_spk.  The recordings of a pass's group are diarized together: their
 * chunks embedded in shared slices with one host copy, the spectral recordings clustered through the _batch entries below, each with
 * exactly its own result.  Refusals are decided from the chunk counts before any embedding, in ClusterBackend's order (fewer than 20
 * chunks: one speaker; then preset_spk_num above the chunk count, or 2048 or more chunks without one), named "recording i: "; a call
 * with several recordings fails with the first in recording order.  spk must live on the recogniser's device.  NULL on error. */
void* fa_offline_infer_vad_spk(void* asr, void* vad, void* spk, const void* const* bufs, const int64_t* n_samples, int32_t batch,
                               int32_t pcm_format, const float* hw_embed, int32_t n_hotwords, const int32_t* language_ids,
                               const int32_t* textnorm_ids, const FaLongAudioOptions* opts, int32_t preset_spk_num);
/* n speakers of recording `index`, one per segment in fa_offline_result_segments' order (labels in order of first appearance); NULL
 * with 0 for a recording that was not diarized and for results of the other entry points. */
const int32_t* fa_offline_result_spk(const void* result, int32_t index, int32_t* n);

/* ---- The handle entries for audio at any sample rate and PCM layout (FaAudioFormat).  Each is its 16 kHz counterpart with the
 * input turned into 16 kHz mono fp32 rows on the device first (fa_ingest_pcm, one launch per upload; 16 kHz mono f32 / s16 take the
 * old path and launch exactly what the old entries launch).  n_samples[i] counts frames (samples per channel).  Before any launch:
 * the descriptor is checked (NULL, sample_format, channels 1..64, rate 1 000..192 000, resampler, a table above 32 MiB), every 16 kHz
 * length is computed (ceil(16000 n / rate)) and the old entries' checks apply to it (400 samples, CAM++'s 18 800 frames).
 * audio_seconds counts the caller's frames at the caller's rate; segments and stamps are in ms of the same timeline.  An old entry
 * is the new one with {pcm_format, 1, 16000, either resampler}.
 *   fa_offline_infer_audio      fa_offline_infer_hw / fa_offline_infer_sv (language_ids / textnorm_ids: SenseVoice only, NULL = the defaults)
 *   fa_offline_infer_vad_audio  fa_offline_infer_vad / _sv / _spk (spk NULL: no diarization)
 *   fa_vad_infer_audio          fa_vad_infer
 *   fa_spk_embed_audio          fa_spk_embed */
void* fa_offline_infer_audio(void* handle, const void* const* bufs, const int64_t* n_samples, int32_t batch, const FaAudioFormat* fmt,
                             const float* hw_embed, int32_t n_hotwords, const int32_t* language_ids, const int32_t* textnorm_ids);
void* fa_offline_infer_vad_audio(void* asr, void* vad, void* spk, const void* const* bufs, const int64_t* n_samples, int32_t batch,
                                 const FaAudioFormat* fmt, const float* hw_embed, int32_t n_hotwords, const int32_t* language_ids,
                                 const int32_t* textnorm_ids, const FaLongAudioOptions* opts, int32_t preset_spk_num);
void* fa_vad_infer_audio(void* vad, const void* buf, int64_t n_samples, const FaAudioFormat* fmt, const FaVadRunOptions* opts);
int fa_spk_embed_audio(void* spk, const void* const* bufs, const int64_t* n_samples, int32_t batch, const FaAudioFormat* fmt, float* emb_host);
/* ---- Forced alignment: MonotonicAligner (fa-zh; monotonic_aligner/model.py:182-267, funasr_b200/modules.py MonotonicAlignerB200 is
 * the specification) -- [start_ms, end_ms] for each token of a transcript the caller already has.
 * fa_align_init: model file written by funasr_b200/pack.py:write_aligner_model_file (encoder.*, the repacked timestamp head,
 * __ts_config__, the frontend tables and CMVN, __aligner_config__).  Refused before any device is touched, naming the piece: no
 * __aligner_config__, a file that also carries __config__ or __sv_config__, (d_model, head dim) other than (320, 80) or (512, 128),
 * feat_dim != 560, CMVN other than [2, 560], upsample_times != 3, a missing or misshapen encoder or head tensor.  fa_offline_init
 * refuses an aligner file.
 * fa_align_infer: batch HOST recordings bufs[i] of n_frames[i] frames in fmt's layout (resampled to 16 kHz on the device as for
 * fa_offline_infer_audio) and transcripts ids[i] [n_ids[i]] -> a result for the recogniser's accessors:
 *   fa_offline_result_stamps(r, i)  utterance i's {start_ms, end_ms} pairs: ts_prediction_lfr6_standard over the timestamp head's
 *                                   first 3 * enc_len upsampled frames, run with token_num = n_ids[i] + 1 (the transcript and its </s>)
 *                                   and stamping n_ids[i] tokens, n_ids[i] - 1 when the last id is the file's eos_id (the routine drops
 *                                   a trailing "</s>").  An empty transcript gives no stamp; one with more tokens than the audio
 *                                   fires for gives fewer stamps than tokens (the count is returned on its own).
 *   fa_offline_result_ids(r, i)     the tokens those stamps belong to: the transcript without a trailing eos_id.
 *   fa_offline_result_count / fa_offline_result_audio_seconds / fa_offline_free_result as for recogniser results.
 * Stamps are per token id: the caller applies sentence_postprocess's merges of English sub-word pieces (nothing to merge for CJK
 * characters), and a token spelled "<sil>", whose stamp the Python routine drops by name, keeps its stamp here.
 * Before any launch, with the handle usable afterwards: NULL handle, bufs, n_frames, fmt or n_ids, batch < 1, n_ids[i] < 0, ids (or
 * ids[i]) NULL with n_ids[i] > 0, an utterance under 400 samples at 16 kHz (named by index), and every refusal of the audio
 * descriptor.  NULL on error (fa_offline_last_error()). */
void* fa_align_init(const char* model_file, int32_t device, int32_t gemm_mode);
void* fa_align_infer(void* aligner, const void* const* bufs, const int64_t* n_frames, int32_t batch, const FaAudioFormat* fmt,
                     const int32_t* const* ids, const int32_t* n_ids);
void fa_align_uninit(void* aligner);
/* p-pruning's effective pval for n rows (SpectralCluster.p_pruning): 6 / n when n * pval < 6, else pval (float64). */
double fa_spk_effective_pval(int32_t n, double pval);
/* SpectralCluster.sim_mat -> p_pruning -> 0.5 (P + P^T) -> laplacian over device embeddings emb [n, dim] fp32 (1 <= n <= 2047,
 * dim <= 1024): rows L2-normalised (a zero norm counts as 1), cosine similarity in fp32, per row the int((1 - pval') n) smallest
 * entries zeroed (pval' = fa_spk_effective_pval(n, pval); one CTA sorts each row's keys; equal values are taken in column order, the
 * one place where numpy's unstable argsort may pick others), symmetrised, zero diagonal, D - M -> lap [n, n] float64 (device).
 * Workspace: fa_spk_laplacian_workspace_bytes (0 for an unsupported shape). */
size_t fa_spk_laplacian_workspace_bytes(int32_t n, int32_t dim);
int fa_spk_laplacian(const float* emb, int32_t n, int32_t dim, double pval, double* lap, void* workspace, size_t ws_bytes, fa_stream_t stream);
/* Householder tridiagonalisation (LAPACK dsytd2, lower, unblocked) of the symmetric lap [n, n] float64 in place (n <= 2047):
 * T = Q^T lap Q with diagonal d [n] and off-diagonal e [n - 1]; Q = H(0) ... H(n - 2), H(j) = I - tau[j] v v^T, v = (1, lap[j][j+2:])
 * kept in row j (and column j) of lap.  Three launches per column, no grid-wide synchronisation; deterministic.  Device arrays. */
size_t fa_spk_tridiagonalize_workspace_bytes(int32_t n);
int fa_spk_tridiagonalize(double* lap, int32_t n, double* d, double* e, double* tau, void* workspace, size_t ws_bytes, fa_stream_t stream);
/* z [k, n] (device, one tridiagonal eigenvector per row) := Q z with fa_spk_tridiagonalize's reflectors (lap, tau): the eigenvectors
 * of the Laplacian.  One CTA per vector. */
int fa_spk_back_transform(const double* lap, const double* tau, int32_t n, double* z, int32_t k, fa_stream_t stream);
/* The three above over a ragged batch of count independent problems of n[s] rows (host arrays; the entry derives the offsets):
 * embeddings emb [sum n, dim], matrices lap [sum n^2], d / e / tau [sum n] each and z [sum k[s] n[s]] concatenated in set order (set
 * s's e holds n[s] - 1 entries of its n[s]).  Each set gets exactly what the single entry gives it (its own effective pval and pruned
 * entries; its own symv partials summed in the same order), and the single entries are the count = 1 case with the same workspace.
 * One launch sequence serves up to 64 sets, a larger batch one sequence per 64: the Laplacian is one row normalisation over all rows
 * and, per sequence, one cosine-tile, one pruning and one Laplacian launch; the tridiagonalisation runs column j of every set with
 * j < n[s] - 1 in one launch each of its three kernels, 3 (max n - 1) + 1 launches; the back-transform is one CTA per (vector, set).
 * Before any launch: a NULL array, count < 1, any n[s] < 1, k[s] < 1 or k[s] > n[s], dim < 1, a bad pval (FA_ERR_ARG), any
 * n[s] > 2047 or dim > 1024 (FA_ERR_UNSUPPORTED), a short workspace (FA_ERR_WORKSPACE).  The workspace queries return 0 for those
 * shapes. */
size_t fa_spk_laplacian_batch_workspace_bytes(const int32_t* n, int32_t count, int32_t dim);
int fa_spk_laplacian_batch(const float* emb, const int32_t* n, int32_t count, int32_t dim, double pval, double* lap, void* workspace,
                           size_t ws_bytes, fa_stream_t stream);
size_t fa_spk_tridiagonalize_batch_workspace_bytes(const int32_t* n, int32_t count);
int fa_spk_tridiagonalize_batch(double* lap, const int32_t* n, int32_t count, double* d, double* e, double* tau, void* workspace,
                                size_t ws_bytes, fa_stream_t stream);
int fa_spk_back_transform_batch(const double* lap, const double* tau, const int32_t* n, const int32_t* k, int32_t count, double* z,
                                fa_stream_t stream);
/* Host only.  The m smallest eigenvalues w [m] of the symmetric tridiagonal (d [n], e [n - 1]) by bisection with Sturm counts, and the
 * eigenvectors of the first k (k <= m) as rows of z [k, n] by inverse iteration, Gram-Schmidt within clusters of close eigenvalues. */
int fa_sym_tridiag_smallest_host(const double* d, const double* e, int32_t n, int32_t m, int32_t k, double* w, double* z);
/* Host only: k-means++ seeding, Lloyd iterations (at most max_iter), the best inertia of n_init starts, float64, from this library's
 * generator seeded by seed: x [n, dim] -> labels [n]. */
int fa_spk_kmeans_host(const double* x, int64_t n, int32_t dim, int32_t k, uint64_t seed, int32_t n_init, int32_t max_iter, int32_t* labels);
/* Host only: ClusterBackend.merge_by_cos over emb [n, dim] fp32 with threshold thr; labels [n] in place. */
int fa_spk_merge_by_cos_host(int32_t* labels, const float* emb, int64_t n, int32_t dim, double thr);
/* Host only: postprocess (correct_labels, merge_seque, overlap midpoint, smooth with Python's round(x, 2)) of chunks [n][2] seconds
 * and labels [n] -> turns [<= n][3] (start_s, end_s, speaker); returns the turn count or FA_ERR_ARG. */
int64_t fa_spk_postprocess_host(const double* chunks, const int32_t* labels, int64_t n, double* turns);
/* Host only: distribute_spk: sentences [ns][2] {start_ms, end_ms} -> spk [ns], the speaker of the turns [nt][3] overlapping most. */
int fa_spk_distribute_host(const int32_t* sentences, int64_t ns, const double* turns, int64_t nt, int32_t* spk);

/* ---- CT-Transformer punctuation (CTTransformer.inference, ct_transformer/model.py:309-473; funasr_b200/punc.py is the specification)
 * fa_punc_init: model file written by funasr_b200/pack.py:write_punc_model_file (the reference's state_dict names, __punc_config__ and
 * both lists).  Refused before any device is touched, naming the piece: d_model > 512 (the encoder workspace bound), a head dim that
 * is not a multiple of 32 up to 128, a missing tensor or list, a token list without <unk>.  The network always runs the fp32 path.
 * fa_punc_infer: n UTF-8 texts -> their punctuated texts and per-word punctuation ids (punc_array, after the forced sentence end).
 * The texts advance in lockstep: step s scores window s (split_size words plus the unfinished tail carried over) of every text that
 * still has one as ONE padded batch -- fa_embedding, fa_sanm_encoder_forward, fa_linear_argmax -- with one host-to-device copy of the
 * ids and lengths and one copy of the punctuation ids back; the carry runs on the host.  Each text's result equals punctuating it
 * alone.  An empty or whitespace-only text gives "" and no ids.  A window with more words than the fp32 attention kernel takes keys
 * (4 * t floats of shared memory within 160 KB, for heads narrower than 128) fails the call before that step's first launch, naming
 * the text: the carried tail grows without bound when the model predicts no comma and no sentence end.  NULL on error
 * (fa_offline_last_error()).
 * Concurrent calls on one handle pool: a call's texts join the lockstep walk of the calls already running at the next step boundary
 * (in arrival order, while the step's device buffers stay within 1 GiB; a call alone always runs), and every step scores one window
 * of every active text of every call as one batch.  A window's punctuation depends on that window only, so each call gets exactly
 * what it gets alone: its texts, ids and steps.  An over-long window fails only its own call, with the message it gets alone; a
 * failure of a step's forward fails every call that had a window in that step. */
void* fa_punc_init(const char* model_file, int32_t device);
void* fa_punc_infer(void* punc, const char* const* texts, int32_t n);
/* text i (NUL-terminated UTF-8; NULL for an out-of-range index) / its n punctuation ids (NULL with 0 for an empty text) */
const char* fa_punc_result_text(const void* result, int32_t index);
const int32_t* fa_punc_result_ids(const void* result, int32_t index, int32_t* n);
/* the lockstep steps the call had a window in (its longest text's window count, pooled or alone) */
int64_t fa_punc_result_steps(const void* result);
void fa_punc_free_result(void* result);
void fa_punc_uninit(void* punc);
/* Calls the punctuation handle's pool has admitted since init, and the lockstep steps it ran them in (steps below the calls' own step
 * counts summed: calls shared steps).  A call whose texts are all empty never enters the pool.  0, or FA_ERR_ARG for a NULL argument. */
int fa_punc_pool_stats(const void* punc, int64_t* calls, int64_t* steps);
/* Host only: the same walk with a caller's scorer in place of the network.  score_fn(ctx, ids [batch, t_max], lens [batch], batch,
 * t_max, punc_out [batch, t_max]) scores one lockstep step (row b valid for its first lens[b] entries, padding ids 0) and returns 0,
 * or nonzero to fail the call.  tokens [n_tokens] / punc_list [n_punc]: the vocabulary and the punctuation classes; split_size words per
 * window; max_window > 0 refuses longer windows as fa_punc_infer does.  Returns a result for the fa_punc_result_* accessors, NULL on
 * error (fa_offline_last_error()). */
typedef int32_t (*fa_punc_score_fn)(void* ctx, const int32_t* ids, const int32_t* lens, int32_t batch, int32_t t_max, int32_t* punc_out);
void* fa_punc_walk_host(const char* const* texts, int32_t n, const char* const* tokens, int32_t n_tokens, const char* const* punc_list,
                        int32_t n_punc, int32_t sentence_end_id, int32_t split_size, int64_t max_window, fa_punc_score_fn score_fn, void* ctx);
/* Host only: a punctuation handle whose steps call score_fn(ctx, ...) in place of the network, with the vocabulary, split_size and
 * max_window of fa_punc_walk_host and its refusals.  fa_punc_infer, fa_punc_pool_stats and fa_punc_uninit take it, and concurrent
 * calls pool exactly as on a fa_punc_init handle: a step's scorer call holds every admitted call's windows.  score_fn is called from
 * whichever calling thread leads the step, one call at a time.  NULL on error (fa_offline_last_error()). */
void* fa_punc_init_host(const char* const* tokens, int32_t n_tokens, const char* const* punc_list, int32_t n_punc, int32_t sentence_end_id,
                        int32_t split_size, int64_t max_window, fa_punc_score_fn score_fn, void* ctx);

#ifdef __cplusplus
}
#endif
#endif /* FUNASR_B200_H_ */
