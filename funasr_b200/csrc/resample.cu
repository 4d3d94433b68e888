// Polyphase sinc resampler: the GPU counterpart of torchaudio.functional.resample as FunASR's loader applies it when the input
// rate differs from the model's (funasr/utils/load_utils.py:176-178, torchaudio.transforms.Resample defaults: sinc_interp_hann,
// lowpass_filter_width 6, rolloff 0.99).  torchaudio pads the waveform by (width, width + orig) zeros and runs a conv1d with
// `new` output channels and stride `orig` (orig / new already divided by their gcd); output sample n = i*new + j is therefore
//   y[n] = sum_k x[i*orig + k - width] * kernel[j][k],   k < 2*width + orig,   x = 0 outside [0, len),
// truncated to ceil(new * len / orig) samples.  The kernel table is computed on the host (funasr_b200/resample.py restates
// torchaudio's _get_sinc_resample_kernel).  One thread per output sample, table rows through the read-only cache.
#include "common.cuh"

namespace fa {

__global__ void __launch_bounds__(256)
resample_kernel(const float* __restrict__ x, const int32_t* __restrict__ lens, int64_t x_stride, const float* __restrict__ table,
                int orig, int nnew, int width, int taps, float* __restrict__ y, int64_t y_stride, int y_cap, int32_t* __restrict__ out_lens) {
  const int b = blockIdx.y;
  const int len = lens[b];
  const int64_t out_len64 = ((int64_t)nnew * len + orig - 1) / orig;         // ceil(new * len / orig)
  const int out_len = (int)(out_len64 < y_cap ? out_len64 : y_cap);
  if (blockIdx.x == 0 && threadIdx.x == 0) out_lens[b] = out_len;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= y_cap) return;
  float acc = 0.f;
  if (n < out_len) {
    const int i = n / nnew, j = n - i * nnew;
    const float* xr = x + (int64_t)b * x_stride;
    const float* tr = table + (int64_t)j * taps;
    const int base = i * orig - width;
    const int k_lo = base < 0 ? -base : 0;
    const int k_hi = min(taps, len - base);
    for (int k = k_lo; k < k_hi; ++k) acc = fmaf(__ldg(xr + base + k), __ldg(tr + k), acc);
  }
  y[(int64_t)b * y_stride + n] = acc;                                         // rows are zero filled beyond out_len
}

// Interleaved PCM frames -> mono fp32 in [-1, 1): the sample decode of the loader (funasr/utils/load_utils.py:48-179 ->
// torchaudio.load(normalize=True) semantics: u8 -> (x - 128) / 128, s16 -> x / 2^15, s24 (packed, little endian) -> x / 2^23,
// s32 -> x / 2^31, f32 unchanged; load_utils.py:168-170 / extract_fbank average the channels).  Every scale is a power of two, so
// each decoded sample is exact.  pcm_frame is the one definition: pcm_decode_kernel and the ingest both use it.
__device__ __forceinline__ float pcm_frame(const unsigned char* __restrict__ pcm, int fmt, int channels, int64_t i) {
  float acc = 0.f;
  for (int c = 0; c < channels; ++c) {
    const int64_t k = i * channels + c;
    float v;
    switch (fmt) {
      case 0: v = reinterpret_cast<const float*>(pcm)[k]; break;
      case 1: v = (float)reinterpret_cast<const int16_t*>(pcm)[k] * (1.0f / 32768.0f); break;
      case 2: {
        const unsigned char* p = pcm + 3 * k;
        int32_t x = (int32_t)p[0] | ((int32_t)p[1] << 8) | ((int32_t)(signed char)p[2] << 16);
        v = (float)x * (1.0f / 8388608.0f);
        break;
      }
      case 3: v = (float)reinterpret_cast<const int32_t*>(pcm)[k] * (1.0f / 2147483648.0f); break;
      default: v = ((float)pcm[k] - 128.0f) * (1.0f / 128.0f); break;
    }
    acc += v;
  }
  return channels > 1 ? acc / (float)channels : acc;
}

// One thread per frame.
__global__ void __launch_bounds__(256)
pcm_decode_kernel(const unsigned char* __restrict__ pcm, int fmt, int channels, int64_t frames, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= frames) return;
  out[i] = pcm_frame(pcm, fmt, channels, i);
}

// The handle's ingest: raw PCM rows -> 16 kHz mono fp32 rows [B, stride], one thread per output sample, one CTA per 256 outputs of
// one row.  A CTA first decodes the input frames its outputs read (the window [lo, hi) between its first and last output's taps)
// into shared memory with pcm_frame, so each frame is decoded once per CTA rather than once per tap; a tap outside the window (a
// window wider than the staging buffer) is decoded from the bytes directly, with the same result.
//   kDecode   16 kHz input: y[t] = pcm_frame(t).
//   kLoader   resample_kernel's sum over the same table, in the same fmaf order over k: bit for bit fa_pcm_decode + fa_resample
//             (for finite samples when the table's zero taps are skipped).
//   kRuntime  LinearResample: output t in unit t / out_unit, phase p = t % out_unit, taps from first[p] + unit * in_unit, weights row
//             p; w * x summed from tap 0 with indices outside [0, n) skipped, every product and add rounded on its own (the
//             reference is plain C++ without contraction).
enum { kDecode = -1, kLoader = 0, kRuntime = 1 };
constexpr int kIngestThreads = 256, kIngestWindow = 4096;   // 16 KB of staged frames: a 192 kHz CTA needs about 3 300

template <int MODE>
__global__ void __launch_bounds__(kIngestThreads)
ingest_kernel(const unsigned char* __restrict__ raw, const int64_t* __restrict__ rows, int fmt, int channels, FaIngestTable tab,
              float* __restrict__ y, int64_t stride) {
  const int b = blockIdx.y;
  const int64_t t0 = (int64_t)blockIdx.x * kIngestThreads, t = t0 + threadIdx.x;
  const unsigned char* pcm = raw + rows[3 * b];
  const int64_t n = rows[3 * b + 1], out_len = rows[3 * b + 2];
  float* yr = y + (int64_t)b * stride;
  if (MODE == kDecode) {
    if (t < stride) yr[t] = t < out_len ? pcm_frame(pcm, fmt, channels, t) : 0.f;
    return;
  }
  __shared__ float xs[kIngestWindow];
  auto first_tap = [&](int64_t s) -> int64_t {             // the input index of output s's tap 0
    const int64_t u = s / tab.out_unit, p = s - u * tab.out_unit;
    return MODE == kLoader ? u * tab.in_unit - tab.width : (int64_t)__ldg(tab.first + p) + u * tab.in_unit;
  };
  int64_t lo = 0, w = 0;
  if (t0 < out_len) {
    const int64_t t1 = min(t0 + kIngestThreads - 1, out_len - 1);
    lo = max(first_tap(t0), (int64_t)0);
    const int64_t hi = min(first_tap(t1) + tab.taps, n);
    w = hi > lo ? hi - lo : 0;
  }
  const bool staged = w <= kIngestWindow;
  if (staged)
    for (int64_t i = threadIdx.x; i < w; i += kIngestThreads) xs[i] = pcm_frame(pcm, fmt, channels, lo + i);
  __syncthreads();
  if (t >= stride) return;
  auto x_at = [&](int64_t idx) -> float {
    const int64_t s = idx - lo;
    return staged && s >= 0 && s < w ? xs[s] : pcm_frame(pcm, fmt, channels, idx);
  };
  float acc = 0.f;
  if (t < out_len) {
    const int64_t u = t / tab.out_unit, p = t - u * tab.out_unit, base = first_tap(t);
    const float* wr = tab.weights + p * tab.taps;
    if (MODE == kLoader) {
      // with spans (first / n_taps: the row's nonzero taps) the exact zeros outside are skipped: fmaf(x, 0, acc) is acc for a finite
      // x, and acc, which starts at +0, is never -0
      int64_t k_lo = base < 0 ? -base : 0, k_hi = min((int64_t)tab.taps, n - base);
      if (tab.first) {
        const int64_t z0 = __ldg(tab.first + p);
        k_lo = max(k_lo, z0);
        k_hi = min(k_hi, z0 + __ldg(tab.n_taps + p));
      }
      for (int64_t k = k_lo; k < k_hi; ++k) acc = fmaf(x_at(base + k), __ldg(wr + k), acc);
    } else {
      const int nt = __ldg(tab.n_taps + p);
      for (int j = 0; j < nt; ++j) {
        const int64_t idx = base + j;
        if (idx < 0 || idx >= n) continue;
        acc = __fadd_rn(acc, __fmul_rn(__ldg(wr + j), x_at(idx)));
      }
    }
  }
  yr[t] = acc;                                                // zero past the row's output length
}

}  // namespace fa

extern "C" int fa_pcm_decode(const void* pcm, int32_t sample_format, int32_t channels, int64_t frames, float* out, fa_stream_t stream) {
  if (!pcm || !out || sample_format < 0 || sample_format > 4 || channels < 1 || channels > 64 || frames < 0) return FA_ERR_ARG;
  if (frames == 0) return FA_OK;
  fa::pcm_decode_kernel<<<(unsigned)((frames + 255) / 256), 256, 0, (cudaStream_t)stream>>>(static_cast<const unsigned char*>(pcm), sample_format, channels,
                                                                                          frames, out);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" int fa_resample(const float* x, const int32_t* lens, int32_t batch, int64_t x_stride, const float* table, int32_t orig,
                           int32_t nnew, int32_t width, float* y, int64_t y_stride, int32_t y_cap, int32_t* out_lens, fa_stream_t stream) {
  if (!x || !lens || !table || !y || !out_lens || batch <= 0 || orig <= 0 || nnew <= 0 || width <= 0 || y_cap <= 0 || y_stride < y_cap)
    return FA_ERR_ARG;
  const int taps = 2 * width + orig;
  dim3 grid((y_cap + 255) / 256, batch);
  fa::resample_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, lens, x_stride, table, orig, nnew, width, taps, y, y_stride, y_cap, out_lens);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" int fa_ingest_pcm(const void* raw, const int64_t* rows, int32_t batch, int32_t sample_format, int32_t channels, const FaIngestTable* table,
                             float* y, int64_t stride, fa_stream_t stream) {
  if (!raw || !rows || !table || !y || batch < 1 || batch > 65535 || sample_format < 0 || sample_format > 4 || channels < 1 || channels > 64 ||
      stride < 1)
    return FA_ERR_ARG;
  const FaIngestTable& t = *table;
  if (t.mode != fa::kDecode && (!t.weights || t.in_unit < 1 || t.out_unit < 1 || t.taps < 1 || t.width < 0)) return FA_ERR_ARG;
  if ((t.mode == fa::kRuntime && (!t.first || !t.n_taps)) || (t.mode == fa::kLoader && !t.first != !t.n_taps)) return FA_ERR_ARG;
  if (t.mode != fa::kDecode && t.mode != fa::kLoader && t.mode != fa::kRuntime) return FA_ERR_ARG;
  const int64_t blocks = (stride + fa::kIngestThreads - 1) / fa::kIngestThreads;
  if (blocks > 0x7fffffffLL) return FA_ERR_ARG;
  const dim3 grid((unsigned)blocks, (unsigned)batch);
  const unsigned char* p = static_cast<const unsigned char*>(raw);
  cudaStream_t st = (cudaStream_t)stream;
  if (t.mode == fa::kDecode) fa::ingest_kernel<fa::kDecode><<<grid, fa::kIngestThreads, 0, st>>>(p, rows, sample_format, channels, t, y, stride);
  else if (t.mode == fa::kLoader) fa::ingest_kernel<fa::kLoader><<<grid, fa::kIngestThreads, 0, st>>>(p, rows, sample_format, channels, t, y, stride);
  else fa::ingest_kernel<fa::kRuntime><<<grid, fa::kIngestThreads, 0, st>>>(p, rows, sample_format, channels, t, y, stride);
  FA_CHECK_LAUNCH();
  return FA_OK;
}
