// Output-side kernels of the greedy decode: row arg-max with log-sum-exp (log_softmax value of the arg-max,
// paraformer/model.py:345,642-644), optional in-place log_softmax of the full logits for parity checks, the
// {blank,sos,eos} filter (:655-666), and the fp32 -> fp16 plane split used by the tensor-core GEMM weights.
#include "common.cuh"
#include "tc_common.cuh"
#include <math.h>

namespace fa {

// One CTA per row of logits [rows, vocab].  Ties resolve to the lowest index (torch.argmax).
// The row is read ONCE into registers (NV float4 per thread) and the three sweeps — maximum, sum of exponentials, lowest index whose
// rounded log-prob equals the maximum's — run on the registers: the first version swept global memory three times with 4-byte
// loads and took 300 us for 10^4 rows x 8404 (336 MB per sweep); one 16-byte sweep is ~60 us of HBM time.
template <int THREADS, int NV>
__global__ void __launch_bounds__(THREADS)
argmax_lse_kernel(float* __restrict__ logits, int vocab, int64_t ld, int32_t* __restrict__ ids,
                  float* __restrict__ best_logp, int write_log_softmax) {
  constexpr int NW = THREADS / 32;
  __shared__ float s_val[NW];
  __shared__ int s_idx[NW];
  __shared__ float s_sum[NW];
  const int64_t row = blockIdx.x;
  float* x = logits + row * ld;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool vec = ((ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0);
  float v[NV][4];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i0 = 4 * (threadIdx.x + THREADS * k);
    if (vec && i0 + 3 < vocab) {
      const float4 t = *reinterpret_cast<const float4*>(x + i0);
      v[k][0] = t.x; v[k][1] = t.y; v[k][2] = t.z; v[k][3] = t.w;
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) v[k][e] = i0 + e < vocab ? x[i0 + e] : -INFINITY;
    }
  }
  float best = -INFINITY;
  int bi = 0x7fffffff;
#pragma unroll
  for (int k = 0; k < NV; ++k)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int i = 4 * (threadIdx.x + THREADS * k) + e;          // increasing within a thread: strict > keeps the lowest index
      if (v[k][e] > best) { best = v[k][e]; bi = i; }
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) { s_val[warp] = best; s_idx[warp] = bi; }
  __syncthreads();
  best = s_val[0]; bi = s_idx[0];
#pragma unroll
  for (int w = 1; w < NW; ++w) {
    if (s_val[w] > best || (s_val[w] == best && s_idx[w] < bi)) { best = s_val[w]; bi = s_idx[w]; }
  }
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k)
#pragma unroll
    for (int e = 0; e < 4; ++e) sum += expf(v[k][e] - best);       // padding holds -inf: exp = 0
  sum = warp_sum(sum);
  if (lane == 0) s_sum[warp] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int w = 0; w < NW; ++w) sum += s_sum[w];
  // torch log_softmax: (x - max) - log(sum exp(x - max)); arg-max is taken over those rounded values (model.py:642),
  // so an element whose log-prob rounds to the same float as the maximum's wins if its index is lower.
  const float lsum = logf(sum);
  const float best_lp = __fsub_rn(0.f, lsum);
  int tie = bi;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i0 = 4 * (threadIdx.x + THREADS * k);
    float lp[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      lp[e] = __fsub_rn(__fsub_rn(v[k][e], best), lsum);
      if (lp[e] == best_lp && i0 + e < tie) tie = i0 + e;
    }
    if (write_log_softmax) {
      if (vec && i0 + 3 < vocab) *reinterpret_cast<float4*>(x + i0) = make_float4(lp[0], lp[1], lp[2], lp[3]);
      else {
#pragma unroll
        for (int e = 0; e < 4; ++e) if (i0 + e < vocab) x[i0 + e] = lp[e];
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) tie = min(tie, __shfl_xor_sync(0xffffffffu, tie, o));
  __syncthreads();
  if (lane == 0) s_idx[warp] = tie;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = s_idx[0];
#pragma unroll
    for (int w = 1; w < NW; ++w) t = min(t, s_idx[w]);
    ids[row] = t;
    best_logp[row] = best_lp;
  }
}

// One warp per utterance: ordered compaction of ids not in {blank, sos, eos}.
__global__ void greedy_filter_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ tok_lens, int n_max,
                                     int sos, int eos, int blank, int32_t* __restrict__ out_ids,
                                     int32_t* __restrict__ out_lens) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const int len = min(tok_lens[b], n_max);
  int count = 0;
  for (int base = 0; base < n_max; base += 32) {
    const int k = base + lane;
    const int id = k < len ? ids[(int64_t)b * n_max + k] : -1;
    const bool keep = k < len && id != sos && id != eos && id != blank;
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (keep) out_ids[(int64_t)b * n_max + count + __popc(m & ((1u << lane) - 1))] = id;
    count += __popc(m);
  }
  for (int k = count + lane; k < n_max; k += 32) out_ids[(int64_t)b * n_max + k] = -1;
  if (lane == 0) out_lens[b] = count;
}

// One warp per utterance: torch.unique_consecutive over the frame arg-max ids, then drop blank
// (sense_voice/model.py:1015-1025).  Ordered compaction with ballots.
__global__ void ctc_filter_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ lens, int t_max, int blank,
                                  int32_t* __restrict__ out_ids, int32_t* __restrict__ out_lens) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const int len = min(lens[b], t_max);
  const int32_t* row = ids + (int64_t)b * t_max;
  int count = 0;
  for (int base = 0; base < t_max; base += 32) {
    const int t = base + lane;
    const int id = t < len ? row[t] : -1;
    const int prev = (t > 0 && t < len) ? row[t - 1] : -2;
    const bool keep = t < len && id != prev && id != blank;
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (keep) out_ids[(int64_t)b * t_max + count + __popc(m & ((1u << lane) - 1))] = id;
    count += __popc(m);
  }
  for (int k = count + lane; k < t_max; k += 32) out_ids[(int64_t)b * t_max + k] = -1;
  if (lane == 0) out_lens[b] = count;
}

__global__ void broadcast_rows_kernel(const float* __restrict__ rows, int n_rows, int cols, float* __restrict__ dst,
                                      int64_t batch_stride_rows) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_rows * cols) dst[(int64_t)b * batch_stride_rows * cols + i] = rows[i];
}

// dst[b, r, :] = embed[q(b, r), :] with q(b, .) = {ids[2b], 1, 2, ids[2b + 1]}: SenseVoice's per-utterance query rows.  Ids are
// clamped to the table (the callers validate them on the host first).
__global__ void sv_query_rows_kernel(const float* __restrict__ embed, int n_embed, int cols, const int32_t* __restrict__ ids,
                                     float* __restrict__ dst, int64_t batch_stride_rows) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 4 * cols) return;
  const int r = i / cols, c = i - r * cols;
  int q = r == 0 ? ids[2 * b] : r == 3 ? ids[2 * b + 1] : r;
  q = min(max(q, 0), n_embed - 1);
  dst[(int64_t)b * batch_stride_rows * cols + i] = embed[(int64_t)q * cols + c];
}

int ctc_filter_launch(const int32_t* ids, const int32_t* lens, int batch, int t_max, int blank, int32_t* out_ids,
                      int32_t* out_lens, cudaStream_t st) {
  ctc_filter_kernel<<<batch, 32, 0, st>>>(ids, lens, t_max, blank, out_ids, out_lens);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

// x = hi + mid + lo with hi = f16(x), mid = f16(x - hi), lo = f16(x - hi - mid) (fp16 planes, tc_common.cuh); planes [3][rows][cols_pad].
__global__ void __launch_bounds__(256)
split_planes_kernel(const float* __restrict__ src, int64_t ld, int64_t rows, int cols, int cols_pad,
                  plane_t* __restrict__ planes) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = rows * cols_pad;
  if (i >= total) return;
  const int64_t r = i / cols_pad;
  const int c = (int)(i - r * cols_pad);
  const float x = c < cols ? src[r * ld + c] : 0.f;
  const plane_t h = to_plane(x);
  const float r1 = x - plane_to_float(h);
  const plane_t m = to_plane(r1);
  const float r2 = r1 - plane_to_float(m);
  planes[i] = h;
  planes[total + i] = m;
  planes[2 * total + i] = to_plane(r2);
}

int argmax_lse_launch(float* logits, int64_t rows, int vocab, int64_t ld, int32_t* ids, float* best_logp,
                      int write_log_softmax, cudaStream_t st) {
  if (rows <= 0) return FA_OK;
  // registers per thread hold the row: 256 x 36 = 9216 (Paraformer 8404), 1024 x 28 = 28672 (SenseVoice 25055), 512 x 120 = 61440
  if (vocab <= 256 * 36) argmax_lse_kernel<256, 9><<<(unsigned)rows, 256, 0, st>>>(logits, vocab, ld, ids, best_logp, write_log_softmax);
  else if (vocab <= 1024 * 28) argmax_lse_kernel<1024, 7><<<(unsigned)rows, 1024, 0, st>>>(logits, vocab, ld, ids, best_logp, write_log_softmax);
  else if (vocab <= 512 * 120) argmax_lse_kernel<512, 30><<<(unsigned)rows, 512, 0, st>>>(logits, vocab, ld, ids, best_logp, write_log_softmax);
  else return FA_ERR_UNSUPPORTED;
  FA_CHECK_LAUNCH();
  return FA_OK;
}

}  // namespace fa

extern "C" int fa_greedy_filter(const int32_t* argmax_ids, const int32_t* tok_lens, int32_t batch, int32_t n_max,
                                int32_t sos, int32_t eos, int32_t blank, int32_t* out_ids, int32_t* out_lens,
                                fa_stream_t stream) {
  if (!argmax_ids || !tok_lens || !out_ids || !out_lens || batch <= 0 || n_max <= 0) return FA_ERR_ARG;
  fa::greedy_filter_kernel<<<batch, 32, 0, (cudaStream_t)stream>>>(argmax_ids, tok_lens, n_max, sos, eos, blank, out_ids, out_lens);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" int fa_broadcast_rows(const float* rows, int32_t n_rows, int32_t cols, float* dst, int64_t dst_batch_stride_rows,
                                 int32_t batch, fa_stream_t stream) {
  if (!rows || !dst || n_rows <= 0 || cols <= 0 || batch <= 0 || dst_batch_stride_rows < n_rows) return FA_ERR_ARG;
  dim3 grid((n_rows * cols + 255) / 256, batch);
  fa::broadcast_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(rows, n_rows, cols, dst, dst_batch_stride_rows);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" int fa_sv_query_rows(const float* embed, int32_t n_embed, int32_t cols, const int32_t* ids, int32_t batch, float* dst,
                                int64_t dst_batch_stride_rows, fa_stream_t stream) {
  if (!embed || !ids || !dst || n_embed < 3 || cols <= 0 || batch <= 0 || batch > 65535 || dst_batch_stride_rows < 4) return FA_ERR_ARG;
  dim3 grid((4 * cols + 255) / 256, batch);
  fa::sv_query_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(embed, n_embed, cols, ids, dst, dst_batch_stride_rows);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" int fa_split_planes(const float* src, int64_t ld_src, int64_t rows, int32_t cols, int32_t cols_pad,
                             void* planes, fa_stream_t stream) {
  if (!src || !planes || rows <= 0 || cols <= 0 || cols_pad < cols) return FA_ERR_ARG;
  const int64_t total = rows * cols_pad;
  fa::split_planes_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      src, ld_src, rows, cols, cols_pad, reinterpret_cast<fa::plane_t*>(planes));
  FA_CHECK_LAUNCH();
  return FA_OK;
}
