// Small host-side (no CUDA) sequential routines of the timestamp post-processing, in the library so that the per-utterance host
// work keeps up with the GPU (64 utterances per ~40 ms step).
#include "../../include/funasr_b200.h"

#include <algorithm>
#include <cmath>
#include <utility>
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

namespace {

// torch's CPU sum over an outer (strided) dimension, float32 accumulation (aten/src/ATen/native/cpu/SumKernel.cpp): one column of
// `size` values `stride` apart.  multi_row_sum is a four-level cascade: 16-element blocks (2^level_power, level_power = max(4,
// ceil(log2 size) / 4)) summed left to right into level 0, each finished block added one level up, a level carried further up whenever
// the position is a multiple of the next level's span; the tail then goes into level 0, and the levels are added 0 + 1 + 2 + 3.
int64_t ceil_log2(int64_t n) {
  int64_t r = 0;
  while (((int64_t)1 << r) < n) ++r;
  return r;
}

float cascade_sum(const float* a, int64_t stride, int64_t size) {
  const int64_t level_power = std::max<int64_t>(4, ceil_log2(size) / 4), level_step = (int64_t)1 << level_power, mask = level_step - 1;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  int64_t i = 0;
  while (i + level_step <= size) {
    for (int64_t j = 0; j < level_step; ++j) acc[0] += a[(i + j) * stride];
    i += level_step;
    for (int j = 1; j < 4; ++j) {
      acc[j] += acc[j - 1];
      acc[j - 1] = 0.f;
      if (i & (mask << (j * level_power))) break;
    }
  }
  for (; i < size; ++i) acc[0] += a[i * stride];
  return ((acc[0] + acc[1]) + acc[2]) + acc[3];
}

// row_sum: the column read as [size / 4, 4], four interleaved cascades, the tail added to the first, then the four added in order
float interleaved_sum(const float* a, int64_t stride, int64_t size) {
  const int64_t q = size / 4;
  float p[4];
  for (int k = 0; k < 4; ++k) p[k] = cascade_sum(a + k * stride, 4 * stride, q);
  for (int64_t i = 4 * q; i < size; ++i) p[0] += a[i * stride];
  return ((p[0] + p[1]) + p[2]) + p[3];
}

// x.sum(0) of a contiguous [size0, size1] float32 tensor: the vectorised outer-reduction path cascades columns in blocks of 32 (four
// vectors of 8 lanes); the columns after the last whole block go through row_sum.  Worker threads split the columns at multiples of
// 128 bytes (32 columns), which leaves every column's path, and so every bit of the result, as in one thread.
void torch_sum_dim0(const float* x, int64_t size0, int64_t size1, float* out) {
  const int64_t blocked = size1 / 32 * 32;
  for (int64_t j = 0; j < size1; ++j) out[j] = j < blocked ? cascade_sum(x + j, size1, size0) : interleaved_sum(x + j, size1, size0);
}

}  // namespace

// SeACo's attention-score filter on the host (seaco_paraformer/model.py:320-343 as funasr_b200/engine.py:seaco_decode computes it with
// torch on the CPU): scores = probs.sum(0).sum(0) over probs [heads, n_rows, n_hw] in torch's summation order, then
// torch.topk(scores, k = min(nfilter, n_hw - 1)) in its order among equal scores (std::partial_sort when 64 k <= n_hw, else
// std::nth_element and a sort of the first k - 1, on (score, index) pairs in index order, greater-than), followed by n_hw - 1.
extern "C" int32_t fa_seaco_asf_select_host(const float* probs, int32_t heads, int32_t n_rows, int32_t n_hw, int32_t nfilter, int32_t* picked) {
  if (!probs || !picked || heads < 1 || n_rows < 1 || n_hw < 2 || nfilter < 1) return FA_ERR_ARG;
  const int64_t cols = (int64_t)n_rows * n_hw;
  std::vector<float> per_row((size_t)cols), scores((size_t)n_hw);
  torch_sum_dim0(probs, heads, cols, per_row.data());
  torch_sum_dim0(per_row.data(), n_rows, n_hw, scores.data());
  const int64_t k = std::min<int64_t>(nfilter, n_hw - 1);
  typedef std::pair<float, int64_t> elem_t;
  std::vector<elem_t> queue((size_t)n_hw);
  for (int64_t j = 0; j < n_hw; ++j) queue[j] = elem_t(scores[j], j);
  auto greater = [](const elem_t& x, const elem_t& y) -> bool { return (std::isnan(x.first) && !std::isnan(y.first)) || (x.first > y.first); };
  if (k * 64 <= n_hw) {
    std::partial_sort(queue.begin(), queue.begin() + k, queue.end(), greater);
  } else {
    std::nth_element(queue.begin(), queue.begin() + k - 1, queue.end(), greater);
    std::sort(queue.begin(), queue.begin() + k - 1, greater);
  }
  for (int64_t j = 0; j < k; ++j) picked[j] = (int32_t)queue[j].second;
  picked[k] = n_hw - 1;
  return (int32_t)(k + 1);
}
