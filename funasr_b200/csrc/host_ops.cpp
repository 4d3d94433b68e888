// Small host-side (no CUDA) sequential routines of the timestamp post-processing, in the library so that the per-utterance host
// work keeps up with the GPU (64 utterances per ~40 ms step).
#include "../../include/funasr_b200.h"

#include <vector>

// Integrate-and-fire trace of one utterance, funasr/utils/timestamp_tools.py:14-34 (`cif_wo_hidden`): fp32 running sum of the
// weights, reduced by `threshold` right after every frame where it reaches it; trace[t] holds the value BEFORE the reduction.
// ts_prediction_lfr6_standard re-integrates the renormalised weights with it whenever the fire count differs from tokens + 1 (:67-72)
// — for BiCif / SeACo Paraformer that is every utterance (the head fires once per token).  Plain fp32 adds in program order
// (compiled with -ffp-contract=off), identical to the numpy loop in funasr_b200/timestamps.py (1 ms per 1500 frames there).
extern "C" int fa_cif_wo_hidden_host(const float* alphas, int64_t n, float threshold, float* trace) {
  if (n < 0 || (n > 0 && (!alphas || !trace))) return FA_ERR_ARG;
  float level = 0.0f;
  for (int64_t t = 0; t < n; ++t) {
    level = level + alphas[t];
    trace[t] = level;
    if (level >= threshold) level = level - 1.0f * threshold;
  }
  return FA_OK;
}

namespace {

// numpy's float32 pairwise summation (numpy/_core/src/umath/loops_utils.h.src: @TYPE@_pairwise_sum), the order
// `weights.sum(dtype=np.float32)` adds in: below 8 elements a plain loop, up to 128 eight interleaved partial sums, above that the
// two halves (the first one a multiple of 8 long) summed recursively.
float pairwise_sum_f32(const float* a, int64_t n) {
  if (n < 8) {
    float res = 0.f;
    for (int64_t i = 0; i < n; ++i) res += a[i];
    return res;
  }
  if (n <= 128) {
    float r[8];
    for (int k = 0; k < 8; ++k) r[k] = a[k];
    int64_t i;
    for (i = 8; i < n - (n % 8); i += 8)
      for (int k = 0; k < 8; ++k) r[k] += a[i + k];
    float res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += a[i];
    return res;
  }
  int64_t n2 = n / 2;
  n2 -= n2 % 8;
  return pairwise_sum_f32(a, n2) + pairwise_sum_f32(a + n2, n - n2);
}

// np.add.reduce over a contiguous 1-D float32 array (numpy 2): the identity 0 plus one pairwise sum over every element
float numpy_sum_f32(const float* a, int64_t n) { return 0.f + pairwise_sum_f32(a, n); }

}  // namespace

// [start_ms, end_ms] stamps of one utterance, funasr/utils/timestamp_tools.py:37-123 (ts_prediction_lfr6_standard) by the route of
// funasr_b200/timestamps.py:_stamps_only, which remains the specification: fires where the trace reaches 1 - 1e-4 (fp32), shifted by
// force_time_shift -1.5 frames; when their count is not n_tokens + 1 the weights are rescaled to sum to n_tokens + 1 (fp32 sum in
// numpy's order, fp32 division) and re-integrated (fa_cif_wo_hidden_host); one span between consecutive fires, cut at 12 frames;
// the trailing-edge rule on the last span (unless it was cut: then it applies to the <sil> span after the cut, which is no stamp);
// every value in double, + vad_offset_ms / 1000 s, then int(x * 1000) with truncation toward zero.
extern "C" int64_t fa_ts_stamps_host(const float* us_alphas, const float* us_peaks, int64_t n_frames, int64_t n_tokens, int32_t upsample_rate,
                                     double vad_offset_ms, int32_t* out, int64_t max_out) {
  if (n_frames < 0 || n_tokens < 0 || upsample_rate < 1 || max_out < 0 || (n_frames > 0 && (!us_alphas || !us_peaks)) ||
      (max_out > 0 && !out))
    return FA_ERR_ARG;
  if (n_tokens == 0) return 0;                                        // :46-47: an empty token list has no stamp
  const int kMaxTokenFrames = 12, kEdgeSilenceFrames = 5;
  const double shift = -1.5, sec_per_frame = 10.0 * 6 / 1000 / upsample_rate;
  const float fire_level = (float)(1.0 - 1e-4);
  std::vector<double> fires;
  auto find_fires = [&](const float* trace) {
    fires.clear();
    for (int64_t t = 0; t < n_frames; ++t)
      if (trace[t] >= fire_level) fires.push_back((double)t + shift);
  };
  find_fires(us_peaks);
  if ((int64_t)fires.size() != n_tokens + 1) {                        // :67-72
    const float div = numpy_sum_f32(us_alphas, n_frames) / (float)(n_tokens + 1);
    std::vector<float> w((size_t)n_frames), trace((size_t)n_frames);
    for (int64_t t = 0; t < n_frames; ++t) w[t] = us_alphas[t] / div;      // all-zero weights: NaN, and no fire below
    fa_cif_wo_hidden_host(w.data(), n_frames, fire_level, trace.data());
    find_fires(trace.data());
  }
  const int64_t n_span = (int64_t)fires.size() - 1;
  if (n_span < 1) return 0;                                           // no fire, or only edge <sil> spans
  const double shift_s = vad_offset_ms / 1000.0;
  for (int64_t i = 0; i < n_span && i < max_out; ++i) {
    const double lo = fires[i], hi = fires[i + 1];
    const bool cut = hi - lo > kMaxTokenFrames;
    double start = lo * sec_per_frame, end = (cut ? lo + kMaxTokenFrames : hi) * sec_per_frame;
    if (i == n_span - 1 && !cut) {
      const double last = fires[n_span];
      end = ((double)n_frames - last > kEdgeSilenceFrames) ? (((double)n_frames + last) * 0.5) * sec_per_frame : (double)n_frames * sec_per_frame;
    }
    if (vad_offset_ms != 0.0) { start += shift_s; end += shift_s; }
    out[2 * i] = (int32_t)(int64_t)(start * 1000);
    out[2 * i + 1] = (int32_t)(int64_t)(end * 1000);
  }
  return n_span;
}
