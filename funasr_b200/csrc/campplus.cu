// CAM++ speaker embedding (funasr/models/campplus/model.py, components.py) on the GPU: fbank + CMN features -> [B, 192].
//
// Activations are time-major.  The FCM front end keeps channels last ([chunk][F][T][32]) and its last conv writes the
// [chunk * T, 320] layout (channel index c * 10 + f) straight into the zero-padded input of the TDNN layer, whose k=5 / stride 2
// Conv1d is ONE GEMM over an overlapping 2-D view of that buffer (row pitch 2 * 320, 1600 columns; cif.cu uses the same view for
// its k=3 conv).  Every 1x1 conv is an nn.Linear GEMM (gemm_f32 / gemm_tc in the engine's gemm_mode).  Eval-mode BatchNorm that
// follows a conv is folded into the conv on the host; BatchNorm that precedes ReLU + conv is a per-channel affine applied by
// bn_relu_kernel while it writes the GEMM's A operand (fp32 rows or fp16 planes).  The dense blocks own one [rows, C_final]
// buffer each: every layer reads a column prefix and writes its 32 new channels into the next column slice (no concatenation).
//
// Every kernel that walks time takes the rows' extents on the device (NULL: every row has the batch's T): row b then computes exactly
// what a batch padded to ext[b] frames computes, reading and writing nothing at or past its extent (fa_campplus_forward_ext).
#include "kernels.h"
#include "tc_common.cuh"
#include <vector>

namespace fa {

constexpr int kCamBn = 128, kCamOut = 32, kCamHid = 64, kCamSeg = 100;
constexpr int kCamTile = 32;                  // output rows per tile of the local conv
constexpr int kCamMaxDil = 8;
// cam_gate_kernel holds every segment mean of a chunk in (non-opt-in) shared memory: nseg <= 94, i.e. t <= 9 400 TDNN frames
// (18 800 feature frames, ~188 s)
constexpr size_t kCamGateSmemMax = 48 * 1024;
static size_t cam_gate_smem(int nseg) { return ((size_t)nseg * kCamBn + kCamBn + kCamHid) * sizeof(float); }

// ------------------------------------------------------------------------------------------------ FCM 2-D convolutions
// in (b, f, t, c) at in[b * isb + f * isf + t * ist + c]; out (b, f, t, o) at out[b * osb + f * osf + t * ost + o * osc]; res (the
// residual branch) in out's layout with osc == 1.  w [KS * KS][CIN][32] (tap-major, output channels contiguous), BN folded.
// Direct convolution in fp32 (every gemm_mode).  A thread owns a register tile of kConvTP consecutive time positions x 16 output
// channels of one (chunk, frequency) row, so each weight it reads from shared memory (one 16-byte load per 4 channels) feeds kConvTP
// FMAs and each input it reads (one 16-byte load per 4 input channels) feeds 16; the two channel halves of a tile sit in adjacent
// lanes and share their input loads through L1.  EXT: ext [B] holds chunk b's frame count; taps at or past it read zero, and nothing
// is written there.  Without it every chunk has T frames, and the kernel compiles to what it compiled to before extents existed.
constexpr int kConvTP = 4;
template <int KS, int CIN, bool EXT>
__global__ void __launch_bounds__(128)
fcm_conv_kernel(const float* __restrict__ in, int64_t isb, int64_t isf, int64_t ist, int f_in, const float* __restrict__ w,
                const float* __restrict__ bias, const float* __restrict__ res, float* __restrict__ out, int64_t osb, int64_t osf,
                int64_t ost, int osc, int f_out, int T, const int32_t* __restrict__ ext, int stride_f, int relu, int64_t total) {
  __shared__ __align__(16) float ws[KS * KS * CIN * 32];
  for (int j = threadIdx.x; j < KS * KS * CIN * 32; j += blockDim.x) ws[j] = w[j];
  __syncthreads();
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int half = (int)(idx & 1);
  const int64_t rest = idx >> 1;
  const int n_tb = (T + kConvTP - 1) / kConvTP;
  const int t0 = (int)(rest % n_tb) * kConvTP;
  const int64_t bf = rest / n_tb;
  const int fo = (int)(bf % f_out);
  const int b = (int)(bf / f_out);
  const int Tb = EXT ? __ldg(ext + b) : T;
  if (EXT && t0 >= Tb) return;
  float acc[kConvTP][16];
#pragma unroll
  for (int p = 0; p < kConvTP; ++p)
#pragma unroll
    for (int o = 0; o < 16; ++o) acc[p][o] = 0.f;
  constexpr int PAD = KS / 2;
  const float* ib = in + (int64_t)b * isb;
  const float* wh = ws + half * 16;
#pragma unroll
  for (int kf = 0; kf < KS; ++kf) {
    const int fi = fo * stride_f + kf - PAD;
    if (fi < 0 || fi >= f_in) continue;
#pragma unroll
    for (int kt = 0; kt < KS; ++kt) {
      const float* wt = wh + (kf * KS + kt) * CIN * 32;
      int64_t off[kConvTP];
      bool ok[kConvTP];
#pragma unroll
      for (int p = 0; p < kConvTP; ++p) {
        const int ti = t0 + p + kt - PAD;
        ok[p] = ti >= 0 && ti < Tb;
        off[p] = (int64_t)fi * isf + (int64_t)(ok[p] ? ti : 0) * ist;
      }
      if (CIN == 1) {
        float xv[kConvTP];
#pragma unroll
        for (int p = 0; p < kConvTP; ++p) xv[p] = ok[p] ? __ldg(ib + off[p]) : 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 wv = *reinterpret_cast<const float4*>(wt + 4 * q);
#pragma unroll
          for (int p = 0; p < kConvTP; ++p) {
            acc[p][4 * q] = fmaf(xv[p], wv.x, acc[p][4 * q]);
            acc[p][4 * q + 1] = fmaf(xv[p], wv.y, acc[p][4 * q + 1]);
            acc[p][4 * q + 2] = fmaf(xv[p], wv.z, acc[p][4 * q + 2]);
            acc[p][4 * q + 3] = fmaf(xv[p], wv.w, acc[p][4 * q + 3]);
          }
        }
      } else {
#pragma unroll 2
        for (int c4 = 0; c4 < CIN; c4 += 4) {
          float4 xv[kConvTP];
#pragma unroll
          for (int p = 0; p < kConvTP; ++p)
            xv[p] = ok[p] ? __ldg(reinterpret_cast<const float4*>(ib + off[p] + c4)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int cc = 0; cc < 4; ++cc) {
            const float* wc = wt + (c4 + cc) * 32;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float4 wv = *reinterpret_cast<const float4*>(wc + 4 * q);
#pragma unroll
              for (int p = 0; p < kConvTP; ++p) {
                const float x = cc == 0 ? xv[p].x : (cc == 1 ? xv[p].y : (cc == 2 ? xv[p].z : xv[p].w));
                acc[p][4 * q] = fmaf(x, wv.x, acc[p][4 * q]);
                acc[p][4 * q + 1] = fmaf(x, wv.y, acc[p][4 * q + 1]);
                acc[p][4 * q + 2] = fmaf(x, wv.z, acc[p][4 * q + 2]);
                acc[p][4 * q + 3] = fmaf(x, wv.w, acc[p][4 * q + 3]);
              }
            }
          }
        }
      }
    }
  }
#pragma unroll
  for (int p = 0; p < kConvTP; ++p) {
    const int t = t0 + p;
    if (t >= Tb) break;
    const int64_t ooff = (int64_t)b * osb + (int64_t)fo * osf + (int64_t)t * ost;
#pragma unroll
    for (int o = 0; o < 16; ++o) {
      const int oc = half * 16 + o;
      float v = acc[p][o] + __ldg(bias + oc);
      if (res) v += res[ooff + oc];
      if (relu) v = fmaxf(v, 0.f);
      out[ooff + (int64_t)oc * osc] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------ BN + ReLU operand pass
// y = relu(x[:, :C] * scale + shift) -> fp32 rows [rows, C] (planes == nullptr) or fp16 planes [npl][rows][cpad] (zero columns
// C..cpad), the A operand of the following GEMM.  One thread per 4 columns.
__global__ void bn_relu_kernel(const float* __restrict__ x, int64_t ldx, int64_t rows, int C, int cpad, const float* __restrict__ scale,
                               const float* __restrict__ shift, float* __restrict__ out, plane_t* __restrict__ planes, int npl) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int c4n = (planes ? cpad : C) >> 2;
  if (i >= rows * c4n) return;
  const int64_t r = i / c4n;
  const int c = (int)(i - r * c4n) * 4;
  float v[4];
  if (c < C) {   // C % 4 == 0
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x + r * ldx + c));
    const float4 s = __ldg(reinterpret_cast<const float4*>(scale + c)), h = __ldg(reinterpret_cast<const float4*>(shift + c));
    v[0] = fmaxf(fmaf(xv.x, s.x, h.x), 0.f); v[1] = fmaxf(fmaf(xv.y, s.y, h.y), 0.f);
    v[2] = fmaxf(fmaf(xv.z, s.z, h.z), 0.f); v[3] = fmaxf(fmaf(xv.w, s.w, h.w), 0.f);
  } else {
    v[0] = v[1] = v[2] = v[3] = 0.f;
  }
  if (!planes) {
    *reinterpret_cast<float4*>(out + r * C + c) = make_float4(v[0], v[1], v[2], v[3]);
    return;
  }
  const int64_t plane = rows * cpad;
  for (int pl = 0; pl < npl; ++pl) {
    uint2 pk;
    pk.x = pack_planes2(v[0], v[1]);
    pk.y = pack_planes2(v[2], v[3]);
    *reinterpret_cast<uint2*>(planes + pl * plane + r * cpad + c) = pk;
    const float2 a = unpack_planes2(pk.x), b = unpack_planes2(pk.y);
    v[0] -= a.x; v[1] -= a.y; v[2] -= b.x; v[3] -= b.y;
  }
}

// ------------------------------------------------------------------------------------------------ TDNN output compaction
// The overlapping-view GEMM yields P / 2 rows per chunk of which the first t_out are the conv's outputs: copy those into the
// block buffer's first 128 columns; ext_out [B] (NULL: t_out): chunk b copies its first ext_out[b] rows only.
__global__ void tdnn_compact_kernel(const float* __restrict__ src, int rows_per_chunk, int t_out, const int32_t* __restrict__ ext_out,
                                    int batch, float* __restrict__ dst, int64_t ldd) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = (int64_t)batch * t_out * (kCamBn / 4);
  if (i >= total) return;
  const int c = (int)(i % (kCamBn / 4)) * 4;
  const int64_t r = i / (kCamBn / 4);
  const int b = (int)(r / t_out), t = (int)(r % t_out);
  if (ext_out && t >= __ldg(ext_out + b)) return;
  const float4 v = *reinterpret_cast<const float4*>(src + ((int64_t)b * rows_per_chunk + t) * kCamBn + c);
  *reinterpret_cast<float4*>(dst + r * ldd + c) = v;
}

// ------------------------------------------------------------------------------------------------ CAM layer
// Context gates (CAMLayer.forward, components.py:216-276): per chunk, mean over T plus the ceil-mode 100-frame segment means
// (avg_pool1d divides a short last window by its own length), then sigmoid(W2 relu(W1 ctx + b1) + b2) per segment.
// h [B * T, 128] -> gates [B][nseg][32].  One CTA of 128 threads (one per channel) per chunk; sums run in time order.  ext [B]
// (NULL: T): chunk b's means run over its first ext[b] rows, and it writes the gates of its own ceil(ext[b] / 100) segments only.
__global__ void __launch_bounds__(kCamBn)
cam_gate_kernel(const float* __restrict__ h, int T, const int32_t* __restrict__ ext, int nseg, const float* __restrict__ w1,
                const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2, float* __restrict__ gates) {
  extern __shared__ float sm[];
  float* seg = sm;                          // [nseg][128]
  float* ctx = sm + nseg * kCamBn;          // [128]
  float* z = ctx + kCamBn;                  // [64]
  const int b = blockIdx.x, c = threadIdx.x;
  const float* hb = h + (int64_t)b * T * kCamBn + c;
  const int Tb = ext ? __ldg(ext + b) : T;
  const int nsb = (Tb + kCamSeg - 1) / kCamSeg;
  float tot = 0.f, sacc = 0.f;
  for (int t = 0; t < Tb; ++t) {
    const float v = __ldg(hb + (int64_t)t * kCamBn);
    tot += v;
    sacc += v;
    if (t % kCamSeg == kCamSeg - 1 || t == Tb - 1) {
      const int s = t / kCamSeg;
      seg[s * kCamBn + c] = sacc / (float)(t - s * kCamSeg + 1);
      sacc = 0.f;
    }
  }
  const float mean = tot / (float)Tb;
  for (int s = 0; s < nsb; ++s) {
    __syncthreads();
    ctx[c] = mean + seg[s * kCamBn + c];
    __syncthreads();
    if (c < kCamHid) {
      float a = __ldg(b1 + c);
      for (int k = 0; k < kCamBn; ++k) a = fmaf(__ldg(w1 + c * kCamBn + k), ctx[k], a);
      z[c] = fmaxf(a, 0.f);
    }
    __syncthreads();
    if (c < kCamOut) {
      float a = __ldg(b2 + c);
      for (int k = 0; k < kCamHid; ++k) a = fmaf(__ldg(w2 + c * kCamHid + k), z[k], a);
      gates[((int64_t)b * nseg + s) * kCamOut + c] = 1.f / (1.f + expf(-a));
    }
  }
}

// Local dilated k=3 conv 128 -> 32 (zero padding inside each chunk) times the gate of the row's segment, written into the block
// buffer's column slice: out[(b T + t) * ldo + o].  wl [3][128][32].  Grid (ceil(T / rows_per_cta), B), 256 threads: lane = output
// channel, each warp owns 4 rows of a 32-row tile; the h rows of the tile (plus the dilation halo) are staged in shared memory.
// ext [B] (NULL: T): chunk b's halo reads zero at or past ext[b], and nothing is written there.
__global__ void __launch_bounds__(256)
cam_local_kernel(const float* __restrict__ h, int T, const int32_t* __restrict__ ext, int dil, int rows_per_cta, const float* __restrict__ wl,
                 const float* __restrict__ gates, int nseg, float* __restrict__ out, int64_t ldo) {
  extern __shared__ __align__(16) float sm[];
  float* ws = sm;                                        // [3 * 128][32]
  float* hs = sm + 3 * kCamBn * kCamOut;                 // [kCamTile + 2 dil][128]
  const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int Tb = ext ? __ldg(ext + b) : T;
  const int r_beg = blockIdx.x * rows_per_cta, r_end = min(Tb, r_beg + rows_per_cta);
  if (r_beg >= r_end) return;
  for (int j = threadIdx.x; j < 3 * kCamBn * kCamOut / 4; j += blockDim.x)
    reinterpret_cast<float4*>(ws)[j] = __ldg(reinterpret_cast<const float4*>(wl) + j);
  const float* hb = h + (int64_t)b * T * kCamBn;
  const int halo_rows = kCamTile + 2 * dil;
  for (int t0 = r_beg; t0 < r_end; t0 += kCamTile) {
    __syncthreads();
    for (int j = threadIdx.x; j < halo_rows * (kCamBn / 4); j += blockDim.x) {
      const int r = j / (kCamBn / 4), c = (j % (kCamBn / 4)) * 4;
      const int t = t0 - dil + r;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t >= 0 && t < Tb) v = __ldg(reinterpret_cast<const float4*>(hb + (int64_t)t * kCamBn + c));
      *reinterpret_cast<float4*>(hs + r * kCamBn + c) = v;
    }
    __syncthreads();
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int rw = warp * 4;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float* hk = hs + (rw + k * dil) * kCamBn;
      const float* wk = ws + k * kCamBn * kCamOut + lane;
#pragma unroll 8
      for (int c = 0; c < kCamBn; ++c) {
        const float wv = wk[c * kCamOut];
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] = fmaf(wv, hk[i * kCamBn + c], acc[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int t = t0 + rw + i;
      if (t < r_end) out[((int64_t)b * T + t) * ldo + lane] = acc[i] * __ldg(gates + ((int64_t)b * nseg + t / kCamSeg) * kCamOut + lane);
    }
  }
}

// ------------------------------------------------------------------------------------------------ statistics pooling
// out_nonlinear (BN + ReLU) then StatsPool (components.py statistics_pooling): stats[b] = [mean_T(y) || std_T(y, unbiased)], y =
// relu(x * scale + shift).  Grid (C / 128, B), one thread per channel, two passes over T, or over chunk b's first ext[b] rows (ext
// [B], NULL: T).
__global__ void __launch_bounds__(128)
stats_pool_kernel(const float* __restrict__ x, int T, const int32_t* __restrict__ ext, int C, const float* __restrict__ scale,
                  const float* __restrict__ shift, float* __restrict__ stats) {
  const int b = blockIdx.y, c = blockIdx.x * 128 + threadIdx.x;
  if (c >= C) return;
  const int Tb = ext ? __ldg(ext + b) : T;
  const float s = __ldg(scale + c), sh = __ldg(shift + c);
  const float* xb = x + (int64_t)b * T * C + c;
  float sum = 0.f;
  for (int t = 0; t < Tb; ++t) sum += fmaxf(fmaf(__ldg(xb + (int64_t)t * C), s, sh), 0.f);
  const float mean = sum / (float)Tb;
  float sq = 0.f;
  for (int t = 0; t < Tb; ++t) {
    const float d = fmaxf(fmaf(__ldg(xb + (int64_t)t * C), s, sh), 0.f) - mean;
    sq = fmaf(d, d, sq);
  }
  stats[(int64_t)b * 2 * C + c] = mean;
  stats[(int64_t)b * 2 * C + C + c] = sqrtf(sq / (float)(Tb - 1));
}

// CMN of the CAM++ frontend (campplus/utils.py extract_feature): feats[b, t, :] -= mean over the utterance's own frames; padded rows
// stay zero.  One thread per (utterance, mel bin), sequential time-order sum (deterministic).  An utterance longer than t_max has only
// t_max rows in feats: the mean is over those, and no row of the next utterance (or past the buffer) is touched.
__global__ void cmn_kernel(float* __restrict__ feats, const int32_t* __restrict__ lens, int t_max, int batch) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch * 80) return;
  const int b = i / 80, c = i % 80;
  const int n = min(lens[b], t_max);
  float* f = feats + (int64_t)b * t_max * 80 + c;
  float s = 0.f;
  for (int t = 0; t < n; ++t) s += f[(int64_t)t * 80];
  const float m = s / (float)n;
  for (int t = 0; t < n; ++t) f[(int64_t)t * 80] -= m;
}

// ------------------------------------------------------------------------------------------------ launchers
// ext: each chunk's frame count on the device, NULL for T everywhere
template <int KS, int CIN, typename... A>
static void fcm_conv_launch(unsigned grid, cudaStream_t st, bool ext, A... a) {
  if (ext) fcm_conv_kernel<KS, CIN, true><<<grid, 128, 0, st>>>(a...);
  else fcm_conv_kernel<KS, CIN, false><<<grid, 128, 0, st>>>(a...);
}

static int conv_launch(const FaCamConv2d& cv, const float* in, int64_t isb, int64_t isf, int64_t ist, int f_in, const float* res,
                       float* out, int64_t osb, int64_t osf, int64_t ost, int osc, int batch, int T, const int32_t* ext, int relu,
                       cudaStream_t st) {
  if (!cv.w || !cv.b || cv.c_out != 32 || (cv.stride_f != 1 && cv.stride_f != 2)) return FA_ERR_ARG;
  const int f_out = (f_in + 2 * (cv.ksize / 2) - cv.ksize) / cv.stride_f + 1;
  const int64_t total = (int64_t)batch * f_out * ((T + kConvTP - 1) / kConvTP) * 2;
  if (total <= 0) return FA_OK;
  if ((cv.c_in & 3) && cv.c_in != 1) return FA_ERR_UNSUPPORTED;
  const unsigned grid = (unsigned)((total + 127) / 128);
  if (cv.ksize == 3 && cv.c_in == 1)
    fcm_conv_launch<3, 1>(grid, st, ext, in, isb, isf, ist, f_in, cv.w, cv.b, res, out, osb, osf, ost, osc, f_out, T, ext, cv.stride_f, relu, total);
  else if (cv.ksize == 3 && cv.c_in == 32)
    fcm_conv_launch<3, 32>(grid, st, ext, in, isb, isf, ist, f_in, cv.w, cv.b, res, out, osb, osf, ost, osc, f_out, T, ext, cv.stride_f, relu, total);
  else if (cv.ksize == 1 && cv.c_in == 32)
    fcm_conv_launch<1, 32>(grid, st, ext, in, isb, isf, ist, f_in, cv.w, cv.b, res, out, osb, osf, ost, osc, f_out, T, ext, cv.stride_f, relu, total);
  else
    return FA_ERR_UNSUPPORTED;
  FA_CHECK_LAUNCH();
  return FA_OK;
}

static int bn_relu_launch(const float* x, int64_t ldx, int64_t rows, int C, int cpad, const float* scale, const float* shift, float* out,
                          plane_t* planes, int npl, cudaStream_t st) {
  if (rows <= 0) return FA_OK;
  if ((C & 3) || (ldx & 3) || (cpad & 3) || !scale || !shift) return FA_ERR_UNSUPPORTED;
  const int64_t total = rows * ((planes ? cpad : C) / 4);
  bn_relu_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, ldx, rows, C, cpad, scale, shift, out, planes, npl);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

static int cam_launch(const float* h, int batch, int T, const int32_t* ext, int dil, const float* local_w, const float* w1, const float* b1, const float* w2,
                      const float* b2, float* gates, float* out, int64_t ldo, cudaStream_t st) {
  if (batch <= 0 || T <= 0) return FA_OK;
  if (dil < 1 || dil > kCamMaxDil || !local_w || !w1 || !b1 || !w2 || !b2) return FA_ERR_ARG;
  const int nseg = (T + kCamSeg - 1) / kCamSeg;
  const size_t gsm = cam_gate_smem(nseg);
  if (gsm > kCamGateSmemMax) return FA_ERR_UNSUPPORTED;
  cam_gate_kernel<<<batch, kCamBn, gsm, st>>>(h, T, ext, nseg, w1, b1, w2, b2, gates);
  FA_CHECK_LAUNCH();
  const size_t lsm = (size_t)(3 * kCamBn * kCamOut + (kCamTile + 2 * kCamMaxDil) * kCamBn) * sizeof(float);
  static PerDeviceOnce once;
  FA_RETURN_IF_ERR(ensure_dyn_smem(cam_local_kernel, lsm, once));
  const int rows_per_cta = 2 * kCamTile;
  dim3 grid((T + rows_per_cta - 1) / rows_per_cta, batch);
  cam_local_kernel<<<grid, 256, lsm, st>>>(h, T, ext, dil, rows_per_cta, local_w, gates, nseg, out, ldo);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

static int stats_launch(const float* x, int batch, int T, const int32_t* ext, int C, const float* scale, const float* shift, float* stats,
                        cudaStream_t st) {
  if (batch <= 0) return FA_OK;
  if (T < 1 || C <= 0 || !scale || !shift) return FA_ERR_ARG;
  stats_pool_kernel<<<dim3((C + 127) / 128, batch), 128, 0, st>>>(x, T, ext, C, scale, shift, stats);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

// Shapes of one forward: T feature frames -> t_out = ceil(T / 2) TDNN frames; P = padded TDNN input rows per chunk (even).
struct CamShapes {
  int B, T, t_out, P, nseg;
  int64_t rows, pad_rows;
  int c_final[3];
};
// FA_ERR_ARG for a null model, batch < 1 or T < 2; FA_ERR_UNSUPPORTED for more CAM segments than cam_launch accepts (T > 18 800),
// so that the forward refuses such an input before its first launch and the workspace query returns 0 for it.
static int cam_shapes(const FaCampplus* m, int batch, int T, CamShapes* s) {
  if (!m || batch <= 0 || T < 2) return FA_ERR_ARG;
  s->B = batch; s->T = T;
  s->t_out = (T - 1) / 2 + 1;
  s->P = (T + 4 + 1) / 2 * 2;
  s->nseg = (s->t_out + kCamSeg - 1) / kCamSeg;
  if (cam_gate_smem(s->nseg) > kCamGateSmemMax) return FA_ERR_UNSUPPORTED;
  s->rows = (int64_t)batch * s->t_out;
  s->pad_rows = (int64_t)batch * s->P + 4;
  int c = 128;
  for (int i = 0; i < 3; ++i) { s->c_final[i] = c + 32 * m->n_layers[i]; c = s->c_final[i] / 2; }
  return FA_OK;
}

struct CamBufs {
  float *x80, *x40a, *x40b, *x40c, *pad, *tdnn, *buf[3], *h, *gates, *op, *stats;
  plane_t *pad_planes, *op_planes;
  Arena scratch{nullptr, 0};   // the dense layer's GEMM
  int32_t* ext = nullptr;      // with extents: [B] feature frames, then [B] TDNN frames
};

static void cam_carve(Arena& a, const CamShapes& s, int mode, bool ext, CamBufs* out) {
  const int64_t BT = (int64_t)s.B * s.T;
  const bool tc = mode != FA_GEMM_F32_SIMT;
  const int npl = gemm_planes(mode);
  const int cmax = s.c_final[1] > s.c_final[2] ? s.c_final[1] : s.c_final[2];
  out->x80 = a.take<float>(BT * 80 * 32);
  out->x40a = a.take<float>(BT * 40 * 32);
  out->x40b = a.take<float>(BT * 40 * 32);
  out->x40c = a.take<float>(BT * 40 * 32);
  out->pad = a.take<float>(s.pad_rows * 320);
  out->tdnn = a.take<float>((int64_t)s.B * (s.P / 2) * kCamBn);
  for (int i = 0; i < 3; ++i) out->buf[i] = a.take<float>(s.rows * s.c_final[i]);
  out->h = a.take<float>(s.rows * kCamBn);
  out->gates = a.take<float>((int64_t)s.B * s.nseg * kCamOut);
  out->stats = a.take<float>((int64_t)s.B * 1024);
  out->op = tc ? nullptr : a.take<float>(s.rows * cmax);
  out->pad_planes = tc ? a.take<plane_t>((size_t)npl * s.pad_rows * 320) : nullptr;
  out->op_planes = tc ? a.take<plane_t>((size_t)npl * s.rows * ((cmax + 63) / 64 * 64)) : nullptr;
  if (tc) out->scratch = a.sub(gemm_tc_scratch_bytes(s.B, 1024, mode));
  if (ext) out->ext = a.take<int32_t>((size_t)2 * s.B);       // last: the carve above is unchanged without it
}

// y[rows, out_f] (ldy) = act(A W^T + b) with A = relu(x[:, :in_f] * scale + shift) (fp32 rows or fp16 planes)
static int bn_relu_linear(const float* x, int64_t ldx, int64_t rows, const float* scale, const float* shift, const FaLinear& lin,
                          int relu, float* y, int64_t ldy, int mode, const CamBufs& bf, cudaStream_t st) {
  if (mode == FA_GEMM_F32_SIMT) {
    FA_RETURN_IF_ERR(bn_relu_launch(x, ldx, rows, lin.in_f, lin.in_f, scale, shift, bf.op, nullptr, 0, st));
    return gemm_f32_launch(bf.op, lin.in_f, rows, lin.w, lin.out_f, lin.in_f, lin.b, GemmEpi().relu(relu).to(y, ldy), st);
  }
  FA_RETURN_IF_ERR(bn_relu_launch(x, ldx, rows, lin.in_f, lin.in_pad, scale, shift, nullptr, bf.op_planes, gemm_planes(mode), st));
  return gemm_tc_planes_launch(bf.op_planes, rows, lin, GemmEpi().relu(relu).to(y, ldy), mode, st);
}

// ext_h: each row's padded length (host, checked by the caller; NULL: T for every row), copied into the workspace with each row's
// TDNN frame count
static int campplus_forward(const FaCampplus* m, const float* feats, int batch, int T, float* emb, int mode, void* ws, size_t ws_bytes,
                            cudaStream_t st, const int32_t* ext_h) {
  CamShapes s;
  if (!feats || !emb) return FA_ERR_ARG;
  FA_RETURN_IF_ERR(cam_shapes(m, batch, T, &s));
  if (mode != FA_GEMM_F32_SIMT && mode != FA_GEMM_F16X1 && mode != FA_GEMM_F16X3 && mode != FA_GEMM_F16X6) return FA_ERR_ARG;
  const bool tc = mode != FA_GEMM_F32_SIMT;
  if (tc && (!m->tdnn.w_planes || !m->dense.w_planes || m->tdnn.in_pad != 1600)) return FA_ERR_ARG;
  if (m->tdnn.in_f != 1600 || m->tdnn.out_f != kCamBn || m->dense.in_f != 1024) return FA_ERR_UNSUPPORTED;
  // every layer's shape is checked before the first launch: a malformed layer enqueues nothing
  {
    const FaCamLayer* L = m->layers;
    for (int blk = 0; blk < 3; ++blk) {
      const int cf = s.c_final[blk];
      for (int l = 0; l < m->n_layers[blk]; ++l, ++L) {
        if (L->linear1.in_f != cf - 32 * (m->n_layers[blk] - l) || L->linear1.out_f != kCamBn) return FA_ERR_ARG;
        if (tc && !L->linear1.w_planes) return FA_ERR_ARG;
      }
      const FaCamTransit& tr = m->transit[blk];
      if (tr.linear.in_f != cf || tr.linear.out_f != cf / 2) return FA_ERR_ARG;
      if (tc && !tr.linear.w_planes) return FA_ERR_ARG;
    }
    if (2 * (s.c_final[2] / 2) != m->dense.in_f) return FA_ERR_ARG;
  }
  Arena a(ws, ws_bytes);
  CamBufs bf;
  cam_carve(a, s, mode, ext_h != nullptr, &bf);
  if (!a.ok()) return FA_ERR_WORKSPACE;
  const int B = s.B;
  const int32_t *ext = nullptr, *ext_out = nullptr;
  if (ext_h) {
    std::vector<int32_t> e(ext_h, ext_h + B);
    for (int b = 0; b < B; ++b) e.push_back((ext_h[b] - 1) / 2 + 1);
    FA_CUDA_OK(cudaMemcpyAsync(bf.ext, e.data(), e.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    ext = bf.ext;
    ext_out = bf.ext + B;
  }
  const int64_t F80 = 80LL * T * 32, F40 = 40LL * T * 32, F20 = 20LL * T * 32;
  const FaCamConv2d* c = m->fcm;
  // FCM (components.py FCM.forward): feats [B, T, 80] read as (b, f, t) with one input channel
  FA_RETURN_IF_ERR(conv_launch(c[0], feats, (int64_t)T * 80, 1, 80, 80, nullptr, bf.x80, F80, (int64_t)T * 32, 32, 1, B, T, ext, 1, st));
  // layer1.0 (stride 2): shortcut, conv1, conv2 + shortcut
  FA_RETURN_IF_ERR(conv_launch(c[3], bf.x80, F80, (int64_t)T * 32, 32, 80, nullptr, bf.x40a, F40, (int64_t)T * 32, 32, 1, B, T, ext, 0, st));
  FA_RETURN_IF_ERR(conv_launch(c[1], bf.x80, F80, (int64_t)T * 32, 32, 80, nullptr, bf.x40b, F40, (int64_t)T * 32, 32, 1, B, T, ext, 1, st));
  FA_RETURN_IF_ERR(conv_launch(c[2], bf.x40b, F40, (int64_t)T * 32, 32, 40, bf.x40a, bf.x40c, F40, (int64_t)T * 32, 32, 1, B, T, ext, 1, st));
  // layer1.1
  FA_RETURN_IF_ERR(conv_launch(c[4], bf.x40c, F40, (int64_t)T * 32, 32, 40, nullptr, bf.x40a, F40, (int64_t)T * 32, 32, 1, B, T, ext, 1, st));
  FA_RETURN_IF_ERR(conv_launch(c[5], bf.x40a, F40, (int64_t)T * 32, 32, 40, bf.x40c, bf.x40b, F40, (int64_t)T * 32, 32, 1, B, T, ext, 1, st));
  // layer2.0 (stride 2), F = 20 (x80 is free again)
  FA_RETURN_IF_ERR(conv_launch(c[8], bf.x40b, F40, (int64_t)T * 32, 32, 40, nullptr, bf.x80, F20, (int64_t)T * 32, 32, 1, B, T, ext, 0, st));
  FA_RETURN_IF_ERR(conv_launch(c[6], bf.x40b, F40, (int64_t)T * 32, 32, 40, nullptr, bf.x40a, F20, (int64_t)T * 32, 32, 1, B, T, ext, 1, st));
  FA_RETURN_IF_ERR(conv_launch(c[7], bf.x40a, F20, (int64_t)T * 32, 32, 20, bf.x80, bf.x40c, F20, (int64_t)T * 32, 32, 1, B, T, ext, 1, st));
  // layer2.1
  FA_RETURN_IF_ERR(conv_launch(c[9], bf.x40c, F20, (int64_t)T * 32, 32, 20, nullptr, bf.x40a, F20, (int64_t)T * 32, 32, 1, B, T, ext, 1, st));
  FA_RETURN_IF_ERR(conv_launch(c[10], bf.x40a, F20, (int64_t)T * 32, 32, 20, bf.x40c, bf.x40b, F20, (int64_t)T * 32, 32, 1, B, T, ext, 1, st));
  // conv2 (stride 2) -> the TDNN input [b * P + 2 + t][c * 10 + f], two zero rows either side of every chunk
  FA_CUDA_OK(cudaMemsetAsync(bf.pad, 0, (size_t)s.pad_rows * 320 * sizeof(float), st));
  FA_RETURN_IF_ERR(conv_launch(c[11], bf.x40b, F20, (int64_t)T * 32, 32, 20, nullptr, bf.pad + 2 * 320, (int64_t)s.P * 320, 1, 320, 10, B,
                               T, ext, 1, st));
  // TDNN: Conv1d(320 -> 128, k 5, stride 2, pad 2) + folded BN + ReLU as one GEMM over the overlapping view (row pitch 640)
  const int64_t Mt = (int64_t)B * (s.P / 2);
  if (!tc) {
    FA_RETURN_IF_ERR(gemm_f32_launch(bf.pad, 640, Mt, m->tdnn.w, kCamBn, 1600, m->tdnn.b, GemmEpi().relu().to(bf.tdnn, kCamBn), st));
  } else {
    FA_RETURN_IF_ERR(split_rows_launch(bf.pad, 320, s.pad_rows, 320, 320, gemm_planes(mode), bf.pad_planes, st));
    FA_RETURN_IF_ERR(gemm_tc_planes_launch(bf.pad_planes, Mt, m->tdnn, GemmEpi().relu().to(bf.tdnn, kCamBn), mode, st, 640, s.pad_rows / 2));
  }
  {
    const int64_t total = s.rows * (kCamBn / 4);
    tdnn_compact_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(bf.tdnn, s.P / 2, s.t_out, ext_out, B, bf.buf[0], s.c_final[0]);
    FA_CHECK_LAUNCH();
  }
  // dense CAM blocks and transits
  const FaCamLayer* L = m->layers;
  for (int blk = 0; blk < 3; ++blk) {
    const int cf = s.c_final[blk];
    float* buf = bf.buf[blk];
    for (int l = 0; l < m->n_layers[blk]; ++l, ++L) {
      const int c_in = cf - 32 * (m->n_layers[blk] - l);
      FA_RETURN_IF_ERR(bn_relu_linear(buf, cf, s.rows, L->bn1_scale, L->bn1_shift, L->linear1, 1, bf.h, kCamBn, mode, bf, st));
      FA_RETURN_IF_ERR(cam_launch(bf.h, B, s.t_out, ext_out, m->dilation[blk], L->local_w, L->w1, L->b1, L->w2, L->b2, bf.gates, buf + c_in, cf, st));
    }
    const FaCamTransit& tr = m->transit[blk];
    float* dst = blk < 2 ? bf.buf[blk + 1] : bf.buf[0];
    const int64_t ldd = blk < 2 ? s.c_final[blk + 1] : cf / 2;
    FA_RETURN_IF_ERR(bn_relu_linear(buf, cf, s.rows, tr.scale, tr.shift, tr.linear, 0, dst, ldd, mode, bf, st));
  }
  const int c_out = s.c_final[2] / 2;
  FA_RETURN_IF_ERR(stats_launch(bf.buf[0], B, s.t_out, ext_out, c_out, m->out_scale, m->out_shift, bf.stats, st));
  return gemm_rows(bf.stats, 2 * c_out, B, m->dense, GemmEpi().to(emb, m->dense.out_f), mode, &bf.scratch, st);
}

}  // namespace fa

using namespace fa;

extern "C" int fa_campplus_features(const float* wav, const int32_t* wav_lens, int32_t batch, int64_t wav_stride, const float* tables,
                                    float* feats, int32_t* feat_lens, int32_t t_max, fa_stream_t stream) {
  if (!wav || !wav_lens || !tables || !feats || !feat_lens || batch <= 0 || t_max <= 0) return FA_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  FA_RETURN_IF_ERR(fbank_unscaled_launch(wav, wav_lens, batch, wav_stride, tables, feats, feat_lens, t_max, st));
  cmn_kernel<<<(batch * 80 + 127) / 128, 128, 0, st>>>(feats, feat_lens, t_max, batch);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

static size_t campplus_ws_bytes(const FaCampplus* model, int32_t batch, int32_t t, int32_t gemm_mode, bool ext) {
  CamShapes s;
  if (cam_shapes(model, batch, t, &s) != FA_OK) return 0;
  Arena m = Arena::measuring();
  CamBufs bf;
  cam_carve(m, s, gemm_mode, ext, &bf);
  return m.bytes();
}

extern "C" size_t fa_campplus_workspace_bytes(const FaCampplus* model, int32_t batch, int32_t t, int32_t gemm_mode) {
  return campplus_ws_bytes(model, batch, t, gemm_mode, false);
}

extern "C" size_t fa_campplus_ext_workspace_bytes(const FaCampplus* model, int32_t batch, int32_t t, int32_t gemm_mode) {
  return campplus_ws_bytes(model, batch, t, gemm_mode, true);
}

extern "C" int fa_campplus_forward(const FaCampplus* model, const float* feats, int32_t batch, int32_t t, float* emb, int32_t gemm_mode,
                                   void* workspace, size_t ws_bytes, fa_stream_t stream) {
  return campplus_forward(model, feats, batch, t, emb, gemm_mode, workspace, ws_bytes, (cudaStream_t)stream, nullptr);
}

extern "C" int fa_campplus_forward_ext(const FaCampplus* model, const float* feats, int32_t batch, int32_t t, float* emb, int32_t gemm_mode,
                                       void* workspace, size_t ws_bytes, fa_stream_t stream, const int32_t* ext_h) {
  if (!ext_h || batch <= 0) return FA_ERR_ARG;
  for (int32_t b = 0; b < batch; ++b)
    if (ext_h[b] < 2 || ext_h[b] > t) return FA_ERR_ARG;
  return campplus_forward(model, feats, batch, t, emb, gemm_mode, workspace, ws_bytes, (cudaStream_t)stream, ext_h);
}

extern "C" int fa_campplus_conv2d(const FaCamConv2d* conv, const float* x, int32_t batch, int32_t f_in, int32_t t, const float* res,
                                  float* y, int32_t relu, fa_stream_t stream) {
  if (!conv || !x || !y || batch <= 0 || f_in <= 0 || t <= 0) return FA_ERR_ARG;
  const int f_out = (f_in + 2 * (conv->ksize / 2) - conv->ksize) / (conv->stride_f > 0 ? conv->stride_f : 1) + 1;
  const int64_t ci = conv->c_in;
  return conv_launch(*conv, x, (int64_t)f_in * t * ci, (int64_t)t * ci, ci, f_in, res, y, (int64_t)f_out * t * 32, (int64_t)t * 32, 32, 1,
                     batch, t, nullptr, relu, (cudaStream_t)stream);
}

extern "C" int fa_campplus_cam(const float* h, int32_t batch, int32_t t, int32_t dilation, const float* local_w, const float* w1,
                               const float* b1, const float* w2, const float* b2, float* gates, float* out, int64_t ld_out,
                               fa_stream_t stream) {
  if (!h || !gates || !out || ld_out < 32) return FA_ERR_ARG;
  return cam_launch(h, batch, t, nullptr, dilation, local_w, w1, b1, w2, b2, gates, out, ld_out, (cudaStream_t)stream);
}

extern "C" int fa_campplus_stats_pool(const float* x, int32_t batch, int32_t t, int32_t channels, const float* scale, const float* shift,
                                      float* stats, fa_stream_t stream) {
  if (!x || !stats) return FA_ERR_ARG;
  return stats_launch(x, batch, t, nullptr, channels, scale, shift, stats, (cudaStream_t)stream);
}
