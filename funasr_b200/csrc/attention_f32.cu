// fp32 SIMT fused multi-head attention with key-padding mask (flash-style, online softmax).
//
// Replaces the scores -> masked_fill(-inf) -> softmax -> masked_fill(0) -> @V -> merge-heads chain of
// MultiHeadedAttentionSANM.forward_attention (sanm/attention.py:288-304, scores from :324-325) and
// MultiHeadedAttentionCrossAtt (:760-794, :811-812).  q is pre-scaled by d_k^-0.5 exactly like :324.
// The [B,H,Tq,Tk] score tensor (256 MB at B=64,T=500) never touches HBM.
// One CTA = 64 queries of one (utterance, head); keys/values streamed in tiles of 64.
#include "common.cuh"
#include "kernels.h"
#include <math.h>

namespace fa {

constexpr int ATT_D = 128, ATT_BQ = 64, ATT_BK = 64;

struct AttSmem {
  float Qt[ATT_D][ATT_BQ + 4];   // transposed: [d][query]
  float Kt[ATT_D][ATT_BK + 4];   // transposed: [d][key]
  float Vs[ATT_BK][ATT_D];       // [key][d]
};
// Probabilities alias the K tile (dead once S is in registers): 102 KB per CTA -> two CTAs per SM.
typedef float PsRow[ATT_BK + 1];
static_assert(sizeof(PsRow) * ATT_BQ <= sizeof(float) * ATT_D * (ATT_BK + 4), "Ps must fit in Kt");

__global__ void __launch_bounds__(256)
attention_f32_kernel(const float* __restrict__ q, int64_t ldq, const float* __restrict__ k, int64_t ldk,
                     const float* __restrict__ v, int64_t ldv, const int32_t* __restrict__ key_lens, int tq, int tk,
                     float* __restrict__ ctx, int64_t ldc, float qscale, int kv_shared, const int32_t* __restrict__ kv_index) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  AttSmem& s = *reinterpret_cast<AttSmem*>(smem_raw);
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * ATT_BQ;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int klen = min(key_lens[b], tk);
  PsRow* Ps = reinterpret_cast<PsRow*>(&s.Kt[0][0]);
  const float* qb = q + ((int64_t)b * tq) * ldq + h * ATT_D;
  const int bkv = kv_index ? kv_index[b] : kv_shared ? 0 : b;   // hotword memory: one k / v entry shared by every utterance, or one per group
  const float* kb = k + ((int64_t)bkv * tk) * ldk + h * ATT_D;
  const float* vb = v + ((int64_t)bkv * tk) * ldv + h * ATT_D;

  // stage Q (scaled) transposed: 64 rows x 32 float4
  for (int idx = tid; idx < ATT_BQ * (ATT_D / 4); idx += 256) {
    const int r = idx >> 5, c4 = idx & 31;
    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < tq) val = __ldg(reinterpret_cast<const float4*>(qb + (int64_t)(q0 + r) * ldq + 4 * c4));
    s.Qt[4 * c4 + 0][r] = __fmul_rn(val.x, qscale);
    s.Qt[4 * c4 + 1][r] = __fmul_rn(val.y, qscale);
    s.Qt[4 * c4 + 2][r] = __fmul_rn(val.z, qscale);
    s.Qt[4 * c4 + 3][r] = __fmul_rn(val.w, qscale);
  }

  float o[4][8];
  float mrow[4], lrow[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    mrow[i] = -INFINITY;
    lrow[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) o[i][j] = 0.f;
  }

  for (int k0 = 0; k0 < klen; k0 += ATT_BK) {
    __syncthreads();  // previous tile fully consumed (also orders the Q staging before first use)
    for (int idx = tid; idx < ATT_BK * (ATT_D / 4); idx += 256) {
      const int r = idx >> 5, c4 = idx & 31;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (k0 + r < klen) {
        kv = __ldg(reinterpret_cast<const float4*>(kb + (int64_t)(k0 + r) * ldk + 4 * c4));
        vv = __ldg(reinterpret_cast<const float4*>(vb + (int64_t)(k0 + r) * ldv + 4 * c4));
      }
      s.Kt[4 * c4 + 0][r] = kv.x; s.Kt[4 * c4 + 1][r] = kv.y; s.Kt[4 * c4 + 2][r] = kv.z; s.Kt[4 * c4 + 3][r] = kv.w;
      *reinterpret_cast<float4*>(&s.Vs[r][4 * c4]) = vv;
    }
    __syncthreads();

    // S = Q K^T for rows ty*4..+3, keys tx*4..+3
    float sc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) sc[i][j] = 0.f;
#pragma unroll 8
    for (int d = 0; d < ATT_D; ++d) {
      const float4 a = *reinterpret_cast<const float4*>(&s.Qt[d][ty * 4]);
      const float4 c = *reinterpret_cast<const float4*>(&s.Kt[d][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, cv[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) sc[i][j] = fmaf(av[i], cv[j], sc[i][j]);
    }
    __syncthreads();  // every thread is done reading Kt before it is reused for the probabilities
    // mask keys beyond the utterance, online softmax update per row (16 lanes share a row group)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (k0 + tx * 4 + j >= klen) sc[i][j] = -INFINITY;
        mx = fmaxf(mx, sc[i][j]);
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      const float mnew = fmaxf(mrow[i], mx);      // finite: every tile has >= 1 valid key
      const float corr = expf(mrow[i] - mnew);    // exp(-inf) = 0 on the first tile
      float ps = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float p = expf(sc[i][j] - mnew);
        Ps[ty * 4 + i][tx * 4 + j] = p;
        ps += p;
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, off);
      lrow[i] = lrow[i] * corr + ps;
      mrow[i] = mnew;
#pragma unroll
      for (int j = 0; j < 8; ++j) o[i][j] *= corr;
    }
    __syncthreads();
    // O += P V : rows ty*4..+3, dims tx*4..+3 and 64+tx*4..+3
#pragma unroll 4
    for (int kk = 0; kk < ATT_BK; ++kk) {
      const float4 v0 = *reinterpret_cast<const float4*>(&s.Vs[kk][tx * 4]);
      const float4 v1 = *reinterpret_cast<const float4*>(&s.Vs[kk][64 + tx * 4]);
      const float vv[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float p = Ps[ty * 4 + i][kk];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[i][j] = fmaf(p, vv[j], o[i][j]);
      }
    }
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = q0 + ty * 4 + i;
    if (r >= tq) continue;
    const float inv = lrow[i] > 0.f ? 1.0f / lrow[i] : 0.f;   // klen == 0 -> zeros (softmax(all -inf) masked to 0)
    float* dst = ctx + ((int64_t)b * tq + r) * ldc + h * ATT_D;
    *reinterpret_cast<float4*>(dst + tx * 4) = make_float4(o[i][0] * inv, o[i][1] * inv, o[i][2] * inv, o[i][3] * inv);
    *reinterpret_cast<float4*>(dst + 64 + tx * 4) = make_float4(o[i][4] * inv, o[i][5] * inv, o[i][6] * inv, o[i][7] * inv);
  }
}

// Generic head dimension (a multiple of 32 up to 128, or 80) for the small SAN-M stacks around the hot path — CT-Transformer
// punctuation: 8 heads x 32 (ct_transformer/template.yaml:31-45) over a few dozen tokens — and the fp32 parity path of the fa-zh
// aligner (4 heads x 80).  One warp per (utterance, head, query): scores of all
// keys into shared memory, max, exp / sum, weighted sum of v.  Same mask semantics as the tiled kernel above.
__global__ void __launch_bounds__(128)
attention_small_kernel(const float* __restrict__ q, int64_t ldq, const float* __restrict__ k, int64_t ldk, const float* __restrict__ v,
                       int64_t ldv, const int32_t* __restrict__ key_lens, int heads, int hd, int tq, int tk, float* __restrict__ ctx,
                       int64_t ldc, float qscale, int kv_shared, const int32_t* __restrict__ kv_index, int64_t n_rows) {
  extern __shared__ float s_sc[];                       // [4 warps][tk]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 4 + warp;   // ((b * heads) + h) * tq + n
  if (row >= n_rows) return;
  const int n = (int)(row % tq);
  const int h = (int)((row / tq) % heads);
  const int b = (int)(row / ((int64_t)tq * heads));
  const int klen = min(key_lens[b], tk);
  const int bkv = kv_index ? kv_index[b] : kv_shared ? 0 : b;
  const int per = (hd + 31) >> 5;                       // dims per lane (1..4); lane + 32 j < hd holds a dim
  float* sc = s_sc + warp * tk;
  const float* qr = q + ((int64_t)b * tq + n) * ldq + h * hd;
  float qv[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j = 0; j < per; ++j) qv[j] = lane + 32 * j < hd ? __fmul_rn(qr[lane + 32 * j], qscale) : 0.f;
  float mx = -INFINITY;
  for (int t = 0; t < klen; ++t) {
    const float* kr = k + ((int64_t)bkv * tk + t) * ldk + h * hd;
    float acc = 0.f;
    for (int j = 0; j < per; ++j)
      if (lane + 32 * j < hd) acc = fmaf(qv[j], kr[lane + 32 * j], acc);
    acc = warp_sum(acc);
    if (lane == 0) sc[t] = acc;
    mx = fmaxf(mx, acc);
  }
  __syncwarp();
  float sum = 0.f;
  for (int t = lane; t < klen; t += 32) { const float e = expf(sc[t] - mx); sc[t] = e; sum += e; }
  sum = warp_sum(sum);
  __syncwarp();
  float o[4] = {0.f, 0.f, 0.f, 0.f};
  for (int t = 0; t < klen; ++t) {
    const float p = sc[t] / sum;
    const float* vr = v + ((int64_t)bkv * tk + t) * ldv + h * hd;
    for (int j = 0; j < per; ++j)
      if (lane + 32 * j < hd) o[j] = fmaf(p, vr[lane + 32 * j], o[j]);
  }
  float* dst = ctx + ((int64_t)b * tq + n) * ldc + h * hd;
  for (int j = 0; j < per; ++j)
    if (lane + 32 * j < hd) dst[lane + 32 * j] = klen > 0 ? o[j] : 0.f;
}

static int attention_small_launch(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, const AttnShape& s,
                                  const int32_t* key_lens, const AttnOut& out, cudaStream_t st) {
  if (s.head_dim < 32 || s.head_dim > 128 || ((s.head_dim & 31) && s.head_dim != 80)) return FA_ERR_UNSUPPORTED;
  const size_t smem = (size_t)4 * s.tk * sizeof(float);
  if (smem > 160 * 1024) return FA_ERR_UNSUPPORTED;
  if (smem > 48 * 1024) FA_CUDA_OK(cudaFuncSetAttribute(attention_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t rows = (int64_t)s.batch * s.heads * s.tq;
  attention_small_kernel<<<(unsigned)((rows + 3) / 4), 128, smem, st>>>(q, ldq, k, ldk, v, ldv, key_lens, s.heads, s.head_dim, s.tq, s.tk,
                                                                       out.ctx, out.ldc, attn_qscale(s.head_dim), s.kv_shared ? 1 : 0, s.kv_index, rows);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

static int attention_f32_launch(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, const AttnShape& s,
                                const int32_t* key_lens, const AttnOut& out, cudaStream_t st) {
  if ((ldq | ldk | ldv | out.ldc) & 3) return FA_ERR_UNSUPPORTED;
  static PerDeviceOnce once;
  FA_RETURN_IF_ERR(ensure_dyn_smem(attention_f32_kernel, sizeof(AttSmem), once));
  dim3 grid((s.tq + ATT_BQ - 1) / ATT_BQ, s.heads, s.batch);
  attention_f32_kernel<<<grid, 256, sizeof(AttSmem), st>>>(q, ldq, k, ldk, v, ldv, key_lens, s.tq, s.tk, out.ctx, out.ldc,
                                                           attn_qscale(ATT_D), s.kv_shared ? 1 : 0, s.kv_index);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

// attention_rows in fp32 mode: the tiled kernel for 128-wide heads, the warp-per-query one otherwise
int attention_f32_rows(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, const AttnShape& s,
                       const int32_t* key_lens, const AttnOut& out, cudaStream_t st) {
  if (s.batch <= 0 || s.tq <= 0) return FA_OK;
  if (!q || !k || !v || !key_lens || !out.ctx || s.tk <= 0) return FA_ERR_ARG;
  if (s.head_dim == ATT_D) return attention_f32_launch(q, ldq, k, ldk, v, ldv, s, key_lens, out, st);
  return attention_small_launch(q, ldq, k, ldk, v, ldv, s, key_lens, out, st);
}

}  // namespace fa

extern "C" int fa_attention(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv,
                            const int32_t* key_lens, int32_t batch, int32_t heads, int32_t tq, int32_t tk, float* ctx,
                            int64_t ld_ctx, fa_stream_t stream) {
  return fa::attention_rows(q, ldq, k, ldk, v, ldv, fa::AttnShape{batch, heads, fa::ATT_D, tq, tk, 0}, key_lens, fa::AttnOut().to(ctx, ld_ctx),
                            FA_GEMM_F32_SIMT, nullptr, (cudaStream_t)stream);
}

extern "C" int fa_attention_f32_ex(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv,
                                   const int32_t* key_lens, int32_t batch, int32_t heads, int32_t head_dim, int32_t tq, int32_t tk,
                                   float* ctx, int64_t ld_ctx, int32_t kv_shared, fa_stream_t stream) {
  if (heads < 1) return FA_ERR_ARG;
  return fa::attention_rows(q, ldq, k, ldk, v, ldv, fa::AttnShape{batch, heads, head_dim, tq, tk, kv_shared}, key_lens,
                            fa::AttnOut().to(ctx, ld_ctx), FA_GEMM_F32_SIMT, nullptr, (cudaStream_t)stream);
}
