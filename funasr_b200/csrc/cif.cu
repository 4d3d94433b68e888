// CIF predictor tail: im2col for the k=3 conv, alpha head, tail threshold, fp64 prefix scan, fire detection and
// the weight-integrate ("continuous integrate-and-fire") segment sums — CifPredictorV2.forward inference branch
// (funasr/models/paraformer/cif_predictor.py:253-314), tail_process_fn (:414-446), cif_wo_hidden_v1 (:818-850)
// and cif_v1 (:853-908).  No host synchronisation: fires are compacted on the device, the token count per
// utterance is written to token_num and read by the host once per batch.
//
// Arithmetic follows the reference's rounding order: alpha prefix sums in fp64 then cast to fp32 (:835),
// fires = (fire + ps) - floor(ps) (:846-847), the per-channel running sum of the fp32 products alpha*h kept in fp64 and
// rounded to fp32 where it is read (:878: torch's CPU cumsum of a float32 tensor accumulates in double,
// acc_type<float> = double), frame = ((PH[t_k] - PH[t_{k-1}]) + rem_{k-1} h_{k-1}) - rem_k h_k (:896).  The acoustic
// embeddings therefore equal the reference's bit for bit.
#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"
#include <math.h>

namespace fa {

// Xc[(b,t), k*D + c] = enc[b, t+k-1, c], zero outside [0, ext[b])  (ConstantPad1d((1,1)) + Conv1d(k=3), :275-276).  ext (NULL: t_max
// for every row) is the padded length the row's batch had in the reference: its conv at t = len - 1 reads frame len when len < ext.
__global__ void __launch_bounds__(256)
cif_im2col_kernel(const float* __restrict__ enc, int t_max, const int32_t* __restrict__ ext, int d, float* __restrict__ xc, int64_t total4) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const int d4 = d >> 2;
  const int c4 = (int)(i % d4);
  const int64_t rk = i / d4;
  const int k = (int)(rk % 3);
  const int64_t row = rk / 3;
  const int t = (int)(row % t_max) + k - 1;
  const int te = ext ? ext[row / t_max] : t_max;
  float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
  if (t >= 0 && t < te) val = __ldg(reinterpret_cast<const float4*>(enc + (row + k - 1) * d) + c4);
  reinterpret_cast<float4*>(xc)[i] = val;
}

// The k = 3 conv as ONE GEMM without an im2col copy (tensor-core path): the encoder output goes to fp16 planes with one zero row in
// front of and behind every utterance, P[b][0] = 0, P[b][1 + t] = enc[b, t], P[b][T + 1] = 0 (row pitch d).  The im2col row of
// (b, t) — enc[b, t-1] | enc[b, t] | enc[b, t+1] — is then the 3 d CONTIGUOUS elements starting at P[b][t], i.e. the im2col matrix is
// the overlapping 2-D view {rows b (T + 2) + t, 3 d columns, row pitch d}, which a TMA tensor map describes directly.  Rows
// b (T + 2) + T and + T + 1 of that view mix two utterances: their outputs are computed and never read.  Frames at or past ext[b]
// (NULL: t_max) are zero planes, as in im2col above.
__global__ void __launch_bounds__(256)
cif_pad_planes_kernel(const float* __restrict__ enc, int t_max, const int32_t* __restrict__ ext, int d, int nplanes, int64_t rows_alloc,
                      int64_t rows_valid, plane_t* __restrict__ planes) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int d4 = d >> 2;
  if (i >= rows_alloc * d4) return;
  const int64_t r = i / d4;
  const int c = (int)(i - r * d4) * 4;
  const int tp = t_max + 2;
  const int64_t b = r / tp;
  const int t = (int)(r - b * tp) - 1;
  float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
  if (r < rows_valid && t >= 0 && t < (ext ? ext[b] : t_max)) x = __ldg(reinterpret_cast<const float4*>(enc + (b * t_max + t) * d + c));
  float v[4] = {x.x, x.y, x.z, x.w};
  const int64_t plane = rows_alloc * d;
  for (int pl = 0; pl < nplanes; ++pl) {
    uint2 pk;
    pk.x = pack_planes2(v[0], v[1]);
    pk.y = pack_planes2(v[2], v[3]);
    *reinterpret_cast<uint2*>(planes + pl * plane + r * d + c) = pk;
    const float2 a = unpack_planes2(pk.x), bb = unpack_planes2(pk.y);
    v[0] -= a.x; v[1] -= a.y; v[2] -= bb.x; v[3] -= bb.y;
  }
}

// alpha[b,t] = relu(sigmoid(c . w + b0) * smooth - noise) * mask     (:280-285); one warp per row.  c_tb: rows of c per utterance
// (t_max, or t_max + 2 when c comes from the padded-view GEMM above)
__global__ void __launch_bounds__(256)
cif_alpha_kernel(const float* __restrict__ c, int d, const float* __restrict__ w, const float* __restrict__ b0,
                 const int32_t* __restrict__ lens, int t_max, int64_t rows, float smooth, float noise,
                 float* __restrict__ alpha_rows, int c_tb) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int64_t crow = (row / t_max) * c_tb + (row % t_max);
  const float4* cr = reinterpret_cast<const float4*>(c + crow * d);
  const float4* w4 = reinterpret_cast<const float4*>(w);
  float acc = 0.f;
  for (int i = lane; i < (d >> 2); i += 32) {
    const float4 a = __ldg(cr + i), ww = __ldg(w4 + i);
    acc += (a.x * ww.x + a.y * ww.y) + (a.z * ww.z + a.w * ww.w);
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    const int b = (int)(row / t_max), t = (int)(row % t_max);
    const float z = acc + __ldg(b0);
    float a = 1.0f / (1.0f + expf(-z));
    a = fmaxf(__fsub_rn(__fmul_rn(a, smooth), noise), 0.f);
    alpha_rows[row] = t < lens[b] ? a : 0.f;
  }
}

// torch's CPU fp32 `x.sum(-1)` of one contiguous row, bit for bit (ATen/native/cpu/SumKernel.cpp: cascade_sum ->
// vectorized_inner_sum -> row_sum -> multi_row_sum).  The x86 builds of torch 2.x run this kernel with 8 fp32 SIMD lanes
// under every CPU capability (DEFAULT / AVX2 / AVX512 — verified against torch.sum for row lengths 1..9001 by
// tests/test_oracle_golden.py::test_torch_row_sum_emulation), so the order is machine independent:
//   the row is viewed as vectors of 8 lanes; vectors are dealt round-robin to 4 ILP accumulators (vector 4i+k -> accumulator k);
//   each accumulator is a 4-level cascade that flushes level 0 into level 1 every 16 vectors (level 1 into 2 every 256, ...);
//   then  p0 += leftover vectors;  p0 += p1; p0 += p2; p0 += p3;  result = (((tail scalars summed left to right) + lane0) + lane1) ...
// The integer outcome floor(sum alpha) (cif_predictor.py:443-444) and the timestamp rescale token_num / sum(alpha2)
// (bicif_paraformer/cif_predictor.py:343-345) follow the reference's rounding exactly.  Warp-collective (all 32 lanes of one
// warp call it): thread (k = lane / 8, l = lane % 8) owns lane l of ILP accumulator k.  Every lane returns the sum.
__device__ float torch_row_sum_f32(const float* __restrict__ x, int n) {
  const int lane = threadIdx.x & 31, k = lane >> 3, l = lane & 7;
  if (n < 8) {                                   // scalar_inner_sum: the same scheme with one lane
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int ilp = n >> 2;
    for (int i = 0; i < ilp; ++i)
      for (int kk = 0; kk < 4; ++kk) acc[kk] = __fadd_rn(acc[kk], x[4 * i + kk]);
    for (int i = ilp * 4; i < n; ++i) acc[0] = __fadd_rn(acc[0], x[i]);
    return __fadd_rn(__fadd_rn(__fadd_rn(acc[0], acc[1]), acc[2]), acc[3]);
  }
  const int vec_size = n >> 3, size_ilp = vec_size >> 2;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  int i = 0;
  while (i + 16 <= size_ilp) {                   // level_step = 16 (level_power = max(4, ceil_log2(size_ilp) / 4) = 4 up to 2^19 vectors)
    for (int j = 0; j < 16; ++j, ++i) a0 = __fadd_rn(a0, x[((i << 2) + k) * 8 + l]);
    a1 = __fadd_rn(a1, a0); a0 = 0.f;
    if ((i & (15 << 4)) == 0) {
      a2 = __fadd_rn(a2, a1); a1 = 0.f;
      if ((i & (15 << 8)) == 0) { a3 = __fadd_rn(a3, a2); a2 = 0.f; }
    }
  }
  for (; i < size_ilp; ++i) a0 = __fadd_rn(a0, x[((i << 2) + k) * 8 + l]);
  a0 = __fadd_rn(__fadd_rn(__fadd_rn(a0, a1), a2), a3);
  if (k == 0)
    for (int v = size_ilp * 4; v < vec_size; ++v) a0 = __fadd_rn(a0, x[v * 8 + l]);
  const float p1 = __shfl_sync(0xffffffffu, a0, 8 + l), p2 = __shfl_sync(0xffffffffu, a0, 16 + l), p3 = __shfl_sync(0xffffffffu, a0, 24 + l);
  a0 = __fadd_rn(__fadd_rn(__fadd_rn(a0, p1), p2), p3);            // meaningful in lanes 0..7
  float f = 0.f;
  for (int t = vec_size * 8; t < n; ++t) f = __fadd_rn(f, x[t]);
#pragma unroll
  for (int ll = 0; ll < 8; ++ll) f = __fadd_rn(f, __shfl_sync(0xffffffffu, a0, ll));
  return f;
}

// One CTA per (utterance, group of CIF_CH channels), one thread per channel.
//   phase 1 (thread 0): alpha' = [alpha, 0], alpha'[len] += tail; token_num = floor(sum alpha'); fp64 prefix
//                       sums -> fires / remainders / fire ordinals into shared memory (every channel group of an utterance
//                       repeats this scalar scan — 500 steps, all groups run concurrently; group 0 writes the per-utterance outputs).
//   phase 2 (all threads): channel-wise running sum of alpha'*h' over time, emitting one acoustic frame per fire.  The sum is a
//                       sequential cumsum per channel in fp64 over the fp32 products, rounded to fp32 at each fire (torch's CPU
//                       cumsum, which accumulates float32 in double), so the kernel is bound by the latency of its
//                       loads, not by bytes: 64 channels per CTA put 8 CTAs on every utterance (512 CTAs at B = 64 instead of 64 —
//                       round 2 launch list: 189 us for 65 MB with one 512-thread CTA per utterance), and the time loop fetches
//                       CIF_UNROLL frames ahead of the dependent adds.
// ext[b] (NULL: t_max) is the row's padded length in the reference's batch: the token count sums the ext[b] + 1 weights of that row
// and the hidden frames past ext[b] read zero.  The weights past ext[b] are zero, so nothing fires there.
constexpr int CIF_CH = 64;
constexpr int CIF_UNROLL = 16;
__global__ void __launch_bounds__(CIF_CH)
cif_fire_kernel(const float* __restrict__ enc, const float* __restrict__ alpha_rows, const int32_t* __restrict__ lens,
                const int32_t* __restrict__ ext, int t_max, int d, float tail, float* __restrict__ acoustic, int n_cap, int32_t* __restrict__ token_num,
                float* __restrict__ alphas_out, float* __restrict__ peaks_out) {
  extern __shared__ float sm[];
  float* s_alpha = sm;                    // [T+1]
  float* s_rem = sm + (t_max + 1);        // [T+1]
  int* s_ord = reinterpret_cast<int*>(sm + 2 * (t_max + 1));  // [T+1] fire ordinal or -1
  const int b = blockIdx.x;
  const bool first_group = blockIdx.y == 0;
  const int T1 = t_max + 1;
  const int te = ext ? ext[b] : t_max, T1e = te + 1;
  const int len = min(lens[b], t_max);
  for (int t = threadIdx.x; t < T1; t += blockDim.x) {
    float a = t < t_max ? alpha_rows[(int64_t)b * t_max + t] : 0.f;
    if (t == len) a = __fadd_rn(a, tail);           // mask_2 - mask_1 is 1 exactly at index len (:426-433)
    s_alpha[t] = a;
  }
  __syncthreads();
  __shared__ float s_total;
  if ((threadIdx.x >> 5) == 1) {                    // warp 1, beside thread 0's scan: token_num = floor(alphas.sum(-1)) in torch's fp32 order
    const float tot = torch_row_sum_f32(s_alpha, T1e);
    if ((threadIdx.x & 31) == 0) s_total = tot;
  }
  if (threadIdx.x == 0) {
    double ps = 0.0;
    float prev_floor = 0.f;
    int ord = 0;
    for (int t = 0; t < T1; ++t) {
      ps += (double)s_alpha[t];                     // cumsum(dtype=float64) :835
      const float psf = (float)ps;
      const float fl = floorf(psf);
      const bool fire = (fl - prev_floor) > 0.f;    // :838-845 (prefix_sum_floor - shifted floor, [:,0] := 0)
      prev_floor = fl;
      const float fires = __fsub_rn(__fadd_rn(fire ? 1.f : 0.f, psf), fl);   // :846-847
      s_rem[t] = __fsub_rn(fires, floorf(fires));   // :889
      s_ord[t] = fire ? ord++ : -1;
      if (first_group) {
        peaks_out[(int64_t)b * T1 + t] = fires;
        alphas_out[(int64_t)b * T1 + t] = s_alpha[t];
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && first_group) token_num[b] = (int32_t)floorf(s_total);   // floor(alphas.sum(-1)) (:443-444), torch's own summation order
  const float* hb = enc + (int64_t)b * t_max * d;
  float* ob = acoustic + (int64_t)b * n_cap * d;
  const int c = blockIdx.y * CIF_CH + threadIdx.x;
  if (c < d) {
    double acc = 0.0;                     // PH[t] before its rounding to fp32
    float prev_ph = 0.f, prev_rh = 0.f;
    for (int t0 = 0; t0 < T1e; t0 += CIF_UNROLL) {
      float hh[CIF_UNROLL];
#pragma unroll
      for (int u = 0; u < CIF_UNROLL; ++u) {                              // the loads of CIF_UNROLL frames go out before the first dependent add
        const int t = t0 + u;
        hh[u] = t < te ? __ldg(hb + (int64_t)t * d + c) : 0.f;            // hidden gets one zero frame appended (:441-442)
      }
#pragma unroll
      for (int u = 0; u < CIF_UNROLL; ++u) {
        const int t = t0 + u;
        if (t < T1e) {
          const float h = hh[u];
          acc = __dadd_rn(acc, (double)__fmul_rn(s_alpha[t], h));         // cumsum(alphas * hidden) :878
          const int k = s_ord[t];
          if (k >= 0) {
            const float ph = __double2float_rn(acc);                      // the cumsum's fp32 output PH[t]
            const float rh = __fmul_rn(s_rem[t], h);
            if (k < n_cap) ob[(int64_t)k * d + c] = __fsub_rn(__fadd_rn(__fsub_rn(ph, prev_ph), prev_rh), rh);   // :896
            prev_ph = ph;
            prev_rh = rh;
          }
        }
      }
    }
  }
}


// BiCif flavour (CifPredictorV3.forward -> `cif`, funasr/models/bicif_paraformer/cif_predictor.py:37-84): the integrate-and-fire
// recurrence runs sequentially in fp32 (no fp64 prefix sums), a fire subtracts exactly 1.0, and a frame is the running
// fp32 sum  frame += cur * h  (multiply, then add) that restarts at  remainds * h  after every fire.  Same launch geometry
// as cif_fire_kernel: thread 0 resolves the scalar recurrence into shared memory, then one thread per channel.  ext as there.
__global__ void __launch_bounds__(512)
cif_fire_loop_kernel(const float* __restrict__ enc, const float* __restrict__ alpha_rows, const int32_t* __restrict__ lens,
                     const int32_t* __restrict__ ext, int t_max, int d, float tail, float threshold, float* __restrict__ acoustic, int n_cap,
                     int32_t* __restrict__ token_num, float* __restrict__ alphas_out, float* __restrict__ peaks_out) {
  extern __shared__ float sm[];
  float* s_cur = sm;                      // [T+1] weight of frame t inside the token being integrated
  float* s_rem = sm + (t_max + 1);        // [T+1] weight carried into the next token when t fires
  int* s_ord = reinterpret_cast<int*>(sm + 2 * (t_max + 1));  // [T+1] fire ordinal or -1
  const int b = blockIdx.x;
  const int T1 = t_max + 1;
  const int te = ext ? ext[b] : t_max, T1e = te + 1;
  const int len = min(lens[b], t_max);
  for (int t = threadIdx.x; t < T1; t += blockDim.x) {
    float a = t < t_max ? alpha_rows[(int64_t)b * t_max + t] : 0.f;
    if (t == len) a = __fadd_rn(a, tail);           // tail_process_fn (:352-377): mask_2 - mask_1 is 1 exactly at index len
    s_cur[t] = a;
  }
  __syncthreads();
  __shared__ float s_total;
  float total_w1 = 0.f;
  if ((threadIdx.x >> 5) == 1) total_w1 = torch_row_sum_f32(s_cur, T1e);   // before thread 0 overwrites s_cur with the per-frame weights
  __syncthreads();
  if (threadIdx.x == 32) s_total = total_w1;
  if (threadIdx.x == 0) {
    float integrate = 0.f;
    int ord = 0;
    for (int t = 0; t < T1; ++t) {
      const float alpha = s_cur[t];
      const float completion = __fsub_rn(1.0f, integrate);      // :54
      integrate = __fadd_rn(integrate, alpha);                   // :56
      peaks_out[(int64_t)b * T1 + t] = integrate;                // list_fires (:57)
      alphas_out[(int64_t)b * T1 + t] = alpha;
      const bool fire = integrate >= threshold;                  // :59
      if (fire) integrate = __fsub_rn(integrate, 1.0f);          // :60-62 (minus ones, not minus threshold)
      const float cur = fire ? completion : alpha;               // :63
      s_cur[t] = cur;
      s_rem[t] = __fsub_rn(alpha, cur);                          // :64
      s_ord[t] = fire ? ord++ : -1;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) token_num[b] = (int32_t)floorf(s_total);  // tail_process_fn: floor(alphas.sum(-1)) (:380-381), torch's summation order
  const float* hb = enc + (int64_t)b * t_max * d;
  float* ob = acoustic + (int64_t)b * n_cap * d;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float frame = 0.f;
    for (int t = 0; t < T1e; ++t) {
      const float h = t < te ? __ldg(hb + (int64_t)t * d + c) : 0.f;      // hidden gets one zero frame appended (:371-372)
      frame = __fadd_rn(frame, __fmul_rn(s_cur[t], h));                   // :66
      const int k = s_ord[t];
      if (k >= 0) {
        if (k < n_cap) ob[(int64_t)k * d + c] = frame;                    // :67, :78
        frame = __fmul_rn(s_rem[t], h);                                   // :68-70
      }
    }
  }
}

// Upsampled timestamp head of CifPredictorV3.get_upsample_timestamp (:300-352), after the BLSTM: per utterance
//   alphas2 *= token_num / sum(alphas2);  us_peaks = cif_wo_hidden(alphas2, threshold - 1e-4)  (fp32, sequential).
// The sum runs over the row's padded length ext_up[b] (NULL: t3); the weights past it are zero.
__global__ void cif_upsample_scan_kernel(float* __restrict__ alphas2, const int32_t* __restrict__ token_num, const int32_t* __restrict__ ext_up,
                                         int t3, float thr, float* __restrict__ us_peaks) {
  const int b = blockIdx.x;
  float* a = alphas2 + (int64_t)b * t3;
  __shared__ float s_scale;
  if (threadIdx.x < 32) {
    const float tot = torch_row_sum_f32(a, ext_up ? ext_up[b] : t3);                  // _token_num = alphas2.sum(-1) (:343), torch's fp32 summation order
    if (threadIdx.x == 0) s_scale = __fdiv_rn((float)token_num[b], tot);       // (token_num / _token_num) :345
  }
  __syncthreads();
  const float scale = s_scale;
  for (int t = threadIdx.x; t < t3; t += blockDim.x) a[t] = __fmul_rn(a[t], scale);
  __syncthreads();
  if (threadIdx.x == 0) {
    float integrate = 0.f;
    for (int t = 0; t < t3; ++t) {
      integrate = __fadd_rn(integrate, a[t]);
      us_peaks[(int64_t)b * t3 + t] = integrate;
      if (integrate >= thr) integrate = __fsub_rn(integrate, thr);
    }
  }
}

// op-level entry for the parity tests: out[r] = torch-order fp32 sum of row r
__global__ void row_sum_f32_kernel(const float* __restrict__ x, int64_t ld, int n, float* __restrict__ out) {
  const float s = torch_row_sum_f32(x + (int64_t)blockIdx.x * ld, n);
  if (threadIdx.x == 0) out[blockIdx.x] = s;
}

int cif_im2col_launch(const float* enc, int64_t rows, int t_max, const int32_t* ext, int d, float* xc, cudaStream_t st) {
  const int64_t total4 = rows * 3 * (d / 4);
  if (total4 <= 0) return FA_OK;
  cif_im2col_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, st>>>(enc, t_max, ext, d, xc, total4);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

int cif_alpha_launch(const float* c, int d, const float* w, const float* b0, const int32_t* lens, int t_max,
                     int64_t rows, float smooth, float noise, float* alpha_rows, cudaStream_t st, int c_rows_per_batch) {
  if (rows <= 0) return FA_OK;
  cif_alpha_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(c, d, w, b0, lens, t_max, rows, smooth, noise, alpha_rows,
                                                               c_rows_per_batch > 0 ? c_rows_per_batch : t_max);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

int cif_pad_planes_launch(const float* enc, int batch, int t_max, const int32_t* ext, int d, int nplanes, int64_t rows_alloc, plane_t* planes,
                          cudaStream_t st) {
  if ((d & 3) || nplanes < 1 || nplanes > 3) return FA_ERR_UNSUPPORTED;
  const int64_t total = rows_alloc * (d / 4);
  cif_pad_planes_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(enc, t_max, ext, d, nplanes, rows_alloc, (int64_t)batch * (t_max + 2),
                                                                         planes);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

int cif_fire_launch(const float* enc, const float* alpha_rows, const int32_t* lens, const int32_t* ext, int batch, int t_max, int d,
                    float tail, float* acoustic, int n_cap, int32_t* token_num, float* alphas, float* peaks,
                    cudaStream_t st) {
  const size_t smem = (size_t)3 * (t_max + 1) * sizeof(float);
  if (smem > 200 * 1024) return FA_ERR_UNSUPPORTED;
  if (smem > 48 * 1024) FA_CUDA_OK(cudaFuncSetAttribute(cif_fire_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cif_fire_kernel<<<dim3(batch, (d + CIF_CH - 1) / CIF_CH), CIF_CH, smem, st>>>(enc, alpha_rows, lens, ext, t_max, d, tail, acoustic, n_cap, token_num,
                                                                                alphas, peaks);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

int cif_fire_loop_launch(const float* enc, const float* alpha_rows, const int32_t* lens, const int32_t* ext, int batch, int t_max, int d,
                         float tail, float threshold, float* acoustic, int n_cap, int32_t* token_num, float* alphas, float* peaks,
                         cudaStream_t st) {
  const size_t smem = (size_t)3 * (t_max + 1) * sizeof(float);
  if (smem > 200 * 1024) return FA_ERR_UNSUPPORTED;
  if (smem > 48 * 1024) FA_CUDA_OK(cudaFuncSetAttribute(cif_fire_loop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cif_fire_loop_kernel<<<batch, 512, smem, st>>>(enc, alpha_rows, lens, ext, t_max, d, tail, threshold, acoustic, n_cap, token_num, alphas,
                                                 peaks);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

int cif_upsample_scan_launch(float* alphas2, const int32_t* token_num, const int32_t* ext_up, int batch, int t3, float thr, float* us_peaks,
                             cudaStream_t st) {
  cif_upsample_scan_kernel<<<batch, 256, 0, st>>>(alphas2, token_num, ext_up, t3, thr, us_peaks);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

}  // namespace fa

extern "C" int fa_row_sum_f32(const float* x, int64_t ld, int32_t rows, int32_t n, float* out, fa_stream_t stream) {
  if (!x || !out || rows < 0 || n < 0 || n >= (8 << 19)) return FA_ERR_ARG;
  if (rows == 0) return FA_OK;
  fa::row_sum_f32_kernel<<<rows, 32, 0, (cudaStream_t)stream>>>(x, ld, n, out);
  FA_CHECK_LAUNCH();
  return FA_OK;
}
