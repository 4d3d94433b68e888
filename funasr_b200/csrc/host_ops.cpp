// Small host-side (no CUDA) sequential routines of the timestamp post-processing, in the library so that the per-utterance host
// work keeps up with the GPU (64 utterances per ~40 ms step).
#include "../../include/funasr_b200.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
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

// ------------------------------------------------------------------------------------------------ speaker clustering, host side
// The parts of ClusterBackend / campplus utils.py that are small or sequential (funasr_b200/diarization.py is the specification): the
// tridiagonal eigenproblem left by fa_spk_tridiagonalize, k-means, merge_by_cos and the label post-processing.
namespace {

// eigenvalues of T below x (Sturm sequence of the LDL^T pivots; a pivot below pivmin counts as -pivmin)
int64_t sturm_count(const double* d, const double* e, int64_t n, double x, double pivmin) {
  int64_t c = 0;
  double q = d[0] - x;
  if (std::fabs(q) < pivmin) q = -pivmin;
  if (q < 0) ++c;
  for (int64_t i = 1; i < n; ++i) {
    q = d[i] - x - e[i - 1] * e[i - 1] / q;
    if (std::fabs(q) < pivmin) q = -pivmin;
    if (q < 0) ++c;
  }
  return c;
}

// deterministic generator of the host routines (splitmix64)
struct SplitMix {
  uint64_t s;
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};

// T - lambda I = P L U with partial pivoting (LAPACK dlagtf's elimination): U has two superdiagonals
struct TridiagLU {
  std::vector<double> u0, u1, u2, l;
  std::vector<char> piv;
  void factor(const double* d, const double* e, int64_t n, double lambda, double tiny) {
    u0.assign(n, 0.0); u1.assign(n, 0.0); u2.assign(n, 0.0); l.assign(n, 0.0); piv.assign(n, 0);
    double r0 = d[0] - lambda, r1 = n > 1 ? e[0] : 0.0, r2 = 0.0;
    for (int64_t i = 0; i + 1 < n; ++i) {
      const double s0 = e[i], s1 = d[i + 1] - lambda, s2 = i + 2 < n ? e[i + 1] : 0.0;
      double n0, n1;
      if (std::fabs(s0) > std::fabs(r0)) {
        piv[i] = 1;
        u0[i] = s0; u1[i] = s1; u2[i] = s2;
        l[i] = r0 / s0;
        n0 = r1 - l[i] * s1; n1 = r2 - l[i] * s2;
      } else {
        if (r0 == 0.0) r0 = tiny;
        u0[i] = r0; u1[i] = r1; u2[i] = r2;
        l[i] = s0 / r0;
        n0 = s1 - l[i] * r1; n1 = s2 - l[i] * r2;
      }
      if (std::fabs(u0[i]) < tiny) u0[i] = std::copysign(tiny, u0[i]);
      r0 = n0; r1 = n1; r2 = 0.0;
    }
    u0[n - 1] = std::fabs(r0) < tiny ? std::copysign(tiny, r0) : r0;
  }
  void solve(double* b, int64_t n) const {
    for (int64_t i = 0; i + 1 < n; ++i) {
      if (piv[i]) std::swap(b[i], b[i + 1]);
      b[i + 1] -= l[i] * b[i];
    }
    for (int64_t i = n - 1; i >= 0; --i) {
      double s = b[i];
      if (i + 1 < n) s -= u1[i] * b[i + 1];
      if (i + 2 < n) s -= u2[i] * b[i + 2];
      b[i] = s / u0[i];
    }
  }
};

double norm2(const double* x, int64_t n) {
  double s = 0.0;
  for (int64_t i = 0; i < n; ++i) s += x[i] * x[i];
  return std::sqrt(s);
}

double sq_dist(const double* a, const double* b, int32_t dim) {
  double s = 0.0;
  for (int32_t c = 0; c < dim; ++c) {
    const double t = a[c] - b[c];
    s += t * t;
  }
  return s;
}

// Python's round(x, 2): correctly rounded, ties to even on the exact binary value (glibc's %.2f rounds the same way)
double round2(double x) {
  char buf[64];
  snprintf(buf, sizeof buf, "%.2f", x);
  return strtod(buf, nullptr);
}

struct Turn { double st, ed; int32_t spk; };

// merge_seque: consecutive turns of one speaker that touch or overlap become one
std::vector<Turn> merge_seque(const std::vector<Turn>& res) {
  std::vector<Turn> out;
  for (const Turn& r : res) {
    if (out.empty() || r.spk != out.back().spk || r.st > out.back().ed) out.push_back(r);
    else out.back().ed = r.ed;
  }
  return out;
}

}  // namespace

// The m smallest eigenvalues w[m] (ascending) of the symmetric tridiagonal T (d [n], e [n - 1]) by bisection on Sturm counts, and
// the eigenvectors of the first k as rows of z [k, n] by inverse iteration on T - w_j I (four solves from a fixed pseudo-random
// start), orthogonalised by Gram-Schmidt against the earlier vectors of the same cluster (eigenvalues closer than 1e-3 ||T||): a
// Laplacian with several connected components has a repeated eigenvalue 0.  The vectors span the eigenspaces scipy's would; within a
// cluster the basis may differ by a rotation, and a vector by its sign.  Returns FA_OK or FA_ERR_ARG.
extern "C" int fa_sym_tridiag_smallest_host(const double* d, const double* e, int32_t n, int32_t m, int32_t k, double* w, double* z) {
  if (!d || n < 1 || (n > 1 && !e) || m < 1 || m > n || k < 0 || k > m || !w || (k > 0 && !z)) return FA_ERR_ARG;
  double lo = d[0], hi = d[0], emax2 = 0.0;
  for (int32_t i = 0; i < n; ++i) {
    const double r = (i > 0 ? std::fabs(e[i - 1]) : 0.0) + (i + 1 < n ? std::fabs(e[i]) : 0.0);
    lo = std::min(lo, d[i] - r);
    hi = std::max(hi, d[i] + r);
    if (i + 1 < n) emax2 = std::max(emax2, e[i] * e[i]);
  }
  const double eps = 2.220446049250313e-16, tnorm = std::max(std::fabs(lo), std::fabs(hi));
  const double pivmin = 2.2250738585072014e-308 * std::max(1.0, emax2);
  lo -= 2 * eps * tnorm + pivmin;
  hi += 2 * eps * tnorm + pivmin;
  for (int32_t i = 0; i < m; ++i) {                // the (i + 1)-th smallest: count(a) <= i < count(b)
    double a = i > 0 ? w[i - 1] - 4 * eps * tnorm - pivmin : lo, b = hi;
    if (sturm_count(d, e, n, a, pivmin) > i) a = lo;
    for (int it = 0; it < 200 && b - a > 2 * eps * std::max(std::fabs(a), std::fabs(b)) + pivmin; ++it) {
      const double mid = 0.5 * (a + b);
      if (mid <= a || mid >= b) break;
      if (sturm_count(d, e, n, mid, pivmin) > i) b = mid;
      else a = mid;
    }
    w[i] = 0.5 * (a + b);
  }
  const double ortol = 1e-3 * tnorm, tiny = eps * std::max(tnorm, 1e-300);
  TridiagLU lu;
  int32_t first = 0;                               // the current cluster's first vector
  for (int32_t j = 0; j < k; ++j) {
    if (j > 0 && w[j] - w[j - 1] > ortol) first = j;
    double* x = z + (int64_t)j * n;
    SplitMix rng{0x5eedull + (uint64_t)j};
    for (int32_t i = 0; i < n; ++i) x[i] = 2.0 * rng.uniform() - 1.0;
    lu.factor(d, e, n, w[j], tiny);
    for (int it = 0; it < 5; ++it) {
      for (int pass = 0; pass < 2; ++pass)
        for (int32_t q = first; q < j; ++q) {
          const double* y = z + (int64_t)q * n;
          double s = 0.0;
          for (int32_t i = 0; i < n; ++i) s += x[i] * y[i];
          for (int32_t i = 0; i < n; ++i) x[i] -= s * y[i];
        }
      double nx = norm2(x, n);
      if (!(nx > 0.0)) { x[j % n] = 1.0; nx = 1.0; }
      for (int32_t i = 0; i < n; ++i) x[i] /= nx;
      if (it == 4) break;
      lu.solve(x, n);
      const double big = norm2(x, n);
      if (std::isfinite(big) && big > 0.0)
        for (int32_t i = 0; i < n; ++i) x[i] /= big;
    }
  }
  return FA_OK;
}

// k-means on x [n, dim] (float64): k-means++ seeding and Lloyd iterations (at most max_iter, until the assignment repeats), the best
// inertia of n_init starts (diarization.kmeans; the generator is this library's, so only the partition is comparable).  An empty
// cluster keeps its centre.  labels [n] in 0 .. k - 1.  Returns FA_OK or FA_ERR_ARG.
extern "C" int fa_spk_kmeans_host(const double* x, int64_t n, int32_t dim, int32_t k, uint64_t seed, int32_t n_init, int32_t max_iter,
                                  int32_t* labels) {
  if (!x || !labels || n < 1 || dim < 1 || k < 1 || k > n || n_init < 1 || max_iter < 1) return FA_ERR_ARG;
  SplitMix rng{seed};
  std::vector<double> centers((size_t)k * dim), d2((size_t)n), sums((size_t)k * dim);
  std::vector<int32_t> lab((size_t)n), cnt((size_t)k);
  double best = INFINITY;
  bool have = false;
  for (int32_t run = 0; run < n_init; ++run) {
    const int64_t i0 = (int64_t)(rng.next() % (uint64_t)n);
    std::copy(x + i0 * dim, x + (i0 + 1) * dim, centers.begin());
    for (int64_t i = 0; i < n; ++i) d2[i] = sq_dist(x + i * dim, centers.data(), dim);
    for (int32_t j = 1; j < k; ++j) {
      double tot = 0.0;
      for (int64_t i = 0; i < n; ++i) tot += d2[i];
      int64_t pick = (int64_t)(rng.next() % (uint64_t)n);
      if (tot > 0.0) {
        const double r = rng.uniform() * tot;
        double c = 0.0;
        for (int64_t i = 0; i < n; ++i) {
          if (d2[i] > 0.0) pick = i;
          c += d2[i];
          if (c > r && d2[i] > 0.0) break;
        }
      }
      std::copy(x + pick * dim, x + (pick + 1) * dim, centers.begin() + (size_t)j * dim);
      for (int64_t i = 0; i < n; ++i) d2[i] = std::min(d2[i], sq_dist(x + i * dim, centers.data() + (size_t)j * dim, dim));
    }
    for (int32_t it = 0; it < max_iter; ++it) {
      bool changed = it == 0;
      for (int64_t i = 0; i < n; ++i) {
        int32_t arg = 0;
        double dm = INFINITY;
        for (int32_t j = 0; j < k; ++j) {
          const double t = sq_dist(x + i * dim, centers.data() + (size_t)j * dim, dim);
          if (t < dm) { dm = t; arg = j; }
        }
        if (lab[i] != arg) changed = true;
        lab[i] = arg;
      }
      if (!changed) break;
      std::fill(sums.begin(), sums.end(), 0.0);
      std::fill(cnt.begin(), cnt.end(), 0);
      for (int64_t i = 0; i < n; ++i) {
        ++cnt[lab[i]];
        for (int32_t c = 0; c < dim; ++c) sums[(size_t)lab[i] * dim + c] += x[i * dim + c];
      }
      for (int32_t j = 0; j < k; ++j)
        if (cnt[j] > 0)
          for (int32_t c = 0; c < dim; ++c) centers[(size_t)j * dim + c] = sums[(size_t)j * dim + c] / cnt[j];
    }
    double inertia = 0.0;
    for (int64_t i = 0; i < n; ++i) inertia += sq_dist(x + i * dim, centers.data() + (size_t)lab[i] * dim, dim);
    if (!have || inertia < best) {
      best = inertia;
      have = true;
      std::copy(lab.begin(), lab.end(), labels);
    }
  }
  return FA_OK;
}

// ClusterBackend.merge_by_cos: while two clusters' mean embeddings (emb [n, dim] fp32) have a cosine of at least thr, the pair with
// the largest cosine (first in row-major order) merges into the lower label and the labels above close up.  labels in place.
extern "C" int fa_spk_merge_by_cos_host(int32_t* labels, const float* emb, int64_t n, int32_t dim, double thr) {
  if (!labels || !emb || n < 1 || dim < 1) return FA_ERR_ARG;
  for (;;) {
    int32_t spk = 0;
    for (int64_t i = 0; i < n; ++i) {
      if (labels[i] < 0) return FA_ERR_ARG;
      spk = std::max(spk, labels[i] + 1);
    }
    if (spk <= 1) break;
    std::vector<double> c((size_t)spk * dim, 0.0);
    std::vector<int64_t> cnt((size_t)spk, 0);
    for (int64_t i = 0; i < n; ++i) {
      ++cnt[labels[i]];
      for (int32_t t = 0; t < dim; ++t) c[(size_t)labels[i] * dim + t] += emb[i * dim + t];
    }
    for (int32_t s = 0; s < spk; ++s) {              // an empty label's centre is NaN, as numpy's mean of nothing
      double nn = 0.0;
      for (int32_t t = 0; t < dim; ++t) c[(size_t)s * dim + t] /= (double)cnt[s];
      for (int32_t t = 0; t < dim; ++t) nn += c[(size_t)s * dim + t] * c[(size_t)s * dim + t];
      nn = std::sqrt(nn);
      for (int32_t t = 0; t < dim; ++t) c[(size_t)s * dim + t] /= nn;
    }
    int32_t a = 0, b = 0;
    double bestv = 0.0;                              // np.triu(aff, 1): the zeroed entries take part in the arg-max
    bool nan = false;
    for (int32_t i = 0; i < spk && !nan; ++i)
      for (int32_t j = i + 1; j < spk; ++j) {
        double v = 0.0;
        for (int32_t t = 0; t < dim; ++t) v += c[(size_t)i * dim + t] * c[(size_t)j * dim + t];
        if (std::isnan(v)) { a = i; b = j; nan = true; break; }   // np.argmax stops at the first NaN, and NaN < thr is false
        if (v > bestv) { bestv = v; a = i; b = j; }
      }
    if (!nan && (a == b ? 0.0 : bestv) < thr) break;
    if (a == b) break;
    for (int64_t i = 0; i < n; ++i) {
      if (labels[i] == b) labels[i] = a;
      else if (labels[i] > b) labels[i] -= 1;
    }
  }
  return FA_OK;
}

// postprocess (campplus utils.py): chunks [n][2] seconds in time order with their labels -> speaker turns [<= n][3] (start_s, end_s,
// speaker): labels renumbered in order of first appearance (correct_labels), merge_seque, overlapping turns meet at the midpoint,
// then smooth (times rounded to 2 decimals as Python's round, turns shorter than 0.7 s take a neighbour's speaker, merge_seque
// again).  Returns the number of turns, or FA_ERR_ARG.
extern "C" int64_t fa_spk_postprocess_host(const double* chunks, const int32_t* labels, int64_t n, double* turns) {
  if (n < 1 || !chunks || !labels || !turns) return FA_ERR_ARG;
  std::vector<int32_t> seen;
  std::vector<Turn> res;
  for (int64_t i = 0; i < n; ++i) {
    auto it = std::find(seen.begin(), seen.end(), labels[i]);
    const int32_t l = (int32_t)(it - seen.begin());
    if (it == seen.end()) seen.push_back(labels[i]);
    res.push_back(Turn{chunks[2 * i], chunks[2 * i + 1], l});
  }
  res = merge_seque(res);
  for (size_t i = 1; i < res.size(); ++i)
    if (res[i - 1].ed > res[i].st + 1e-4) {
      const double p = (res[i].st + res[i - 1].ed) / 2;
      res[i].st = p;
      res[i - 1].ed = p;
    }
  if (res.size() >= 2) {                             // smooth; a single turn is returned unrounded
    const double mindur = 0.7;
    const size_t m = res.size();
    for (size_t i = 0; i < m; ++i) {
      res[i].st = round2(res[i].st);
      res[i].ed = round2(res[i].ed);
      if (res[i].ed - res[i].st < mindur) {
        if (i == 0) res[i].spk = res[i + 1].spk;
        else if (i == m - 1) res[i].spk = res[i - 1].spk;
        else if (res[i].st - res[i - 1].ed <= res[i + 1].st - res[i].ed) res[i].spk = res[i - 1].spk;
        else res[i].spk = res[i + 1].spk;
      }
    }
    res = merge_seque(res);
  }
  for (size_t i = 0; i < res.size(); ++i) {
    turns[3 * i] = res[i].st;
    turns[3 * i + 1] = res[i].ed;
    turns[3 * i + 2] = res[i].spk;
  }
  return (int64_t)res.size();
}

// distribute_spk: every sentence {start_ms, end_ms} (sentences [ns][2]) takes the speaker whose turns (turns [nt][3], seconds) overlap
// it most, with the reference's running tally (a turn of the leading speaker adds its overlap again).  spk [ns].
extern "C" int fa_spk_distribute_host(const int32_t* sentences, int64_t ns, const double* turns, int64_t nt, int32_t* spk) {
  if (ns < 0 || nt < 0 || (ns > 0 && (!sentences || !spk)) || (nt > 0 && !turns)) return FA_ERR_ARG;
  for (int64_t s = 0; s < ns; ++s) {
    const double s0 = sentences[2 * s], s1 = sentences[2 * s + 1];
    int32_t best = 0;
    double max_ov = 0.0;
    for (int64_t t = 0; t < nt; ++t) {
      const double st = turns[3 * t] * 1000, ed = turns[3 * t + 1] * 1000;
      const int32_t sp = (int32_t)turns[3 * t + 2];
      const double ov = std::max(std::min(s1, ed) - std::max(s0, st), 0.0);
      if (ov > max_ov) { max_ov = ov; best = sp; }
      if (ov > 0 && best == sp) max_ov += ov;
    }
    spk[s] = best;
  }
  return FA_OK;
}

// ------------------------------------------------------------------------------------------------ resampling tables (to 16 kHz)
namespace {

const int64_t kMaxTableFloats = (32ll << 20) / 4;   // 32 MiB of weights

int32_t gcd32(int32_t a, int32_t b) {
  while (b) { const int32_t t = a % b; a = b; b = t; }
  return a;
}

bool rate_ok(int32_t rate, int32_t new_rate) { return rate >= 1000 && rate <= 192000 && new_rate >= 1000 && new_rate <= 192000; }

// LinearResample's phase p < out_unit (kaldi feat/resample.cc SetIndexesAndWeights): output time p / out_rate, the input indices
// within num_zeros / (2 cutoff) seconds of it (ceil of the lower edge, floor of the upper), weight FilterFunc(float(dt)) / in_rate.
// The arithmetic mixes float and double as the definition does: the cutoff is a float, FilterFunc takes and returns a float, its
// window and sinc are evaluated in double.
struct LinearResampleDef {
  int32_t in_rate, out_rate, in_unit, out_unit;
  float cutoff;
  int32_t zeros = 6;
  LinearResampleDef(int32_t in, int32_t out) : in_rate(in), out_rate(out) {
    const int32_t g = gcd32(in, out);
    in_unit = in / g; out_unit = out / g;
    const float min_freq = (float)std::min(in, out);
    cutoff = (float)(0.99 * 0.5 * min_freq);
  }
  double window_width() const { return zeros / (2.0 * cutoff); }
  float filter(float t) const {
    const double two_pi = 6.283185307179586476925286766559005, pi = 3.1415926535897932384626433832795;
    float window, f;
    if (std::fabs(t) < zeros / (2.0 * cutoff)) window = (float)(0.5 * (1 + std::cos(two_pi * cutoff / zeros * t)));
    else window = 0.0f;
    if (t != 0) f = (float)(std::sin(two_pi * cutoff * t) / (pi * t));
    else f = 2 * cutoff;
    return f * window;
  }
  void span(int32_t p, int32_t* first, int32_t* n) const {
    const double ww = window_width(), out_t = p / (double)out_rate;
    const double min_t = out_t - ww, max_t = out_t + ww;
    const int32_t lo = (int32_t)std::ceil(min_t * in_rate), hi = (int32_t)std::floor(max_t * in_rate);
    *first = lo; *n = hi - lo + 1;
  }
  float weight(int32_t p, int32_t index) const {
    const double out_t = p / (double)out_rate, in_t = index / (double)in_rate, dt = in_t - out_t;
    return filter((float)dt) / in_rate;
  }
};

}  // namespace

// resample.sinc_resample_table (torchaudio's _get_sinc_resample_kernel, lowpass width 6, rolloff 0.99): the shift j / new rounded to
// float32 (torch divides an int64 arange by an int there), the grid in float64, the window cos(t pi / 6 / 2) squared, sin(pi t) /
// (pi t) with 1 at 0, times base / orig, rounded to float32.  glibc's sin / cos are numpy's on x86-64.
extern "C" int64_t fa_loader_resample_table_host(int32_t rate, int32_t new_rate, int32_t* orig_out, int32_t* nnew_out, int32_t* width_out,
                                                 float* table, int64_t cap) {
  if (!rate_ok(rate, new_rate)) return FA_ERR_ARG;
  const int32_t g = gcd32(rate, new_rate), orig = rate / g, nw = new_rate / g;
  const double lpw = 6, base = std::min(orig, nw) * 0.99;
  const int32_t width = (int32_t)std::ceil(6 * orig / base);
  const int64_t taps = 2 * (int64_t)width + orig, need = (int64_t)nw * taps;
  if (need > kMaxTableFloats) return FA_ERR_UNSUPPORTED;
  if (orig_out) *orig_out = orig;
  if (nnew_out) *nnew_out = nw;
  if (width_out) *width_out = width;
  if (!table) return need;
  if (cap < need) return FA_ERR_ARG;
  const double scale = base / orig, pi = 3.141592653589793;
  for (int32_t j = 0; j < nw; ++j) {
    const double shift = (double)((float)(-j) / (float)nw);
    for (int64_t k = 0; k < taps; ++k) {
      const double idx = (double)(k - width) / orig;
      double t = (shift + idx) * base;
      t = std::min(std::max(t, -lpw), lpw);
      double w = std::cos(t * pi / lpw / 2);
      w = w * w;
      t = t * pi;
      const double kern = t == 0 ? 1.0 : std::sin(t) / t;
      table[(int64_t)j * taps + k] = (float)(kern * w * scale);
    }
  }
  return need;
}

extern "C" int64_t fa_runtime_resample_table_host(int32_t rate, int32_t new_rate, int32_t* in_unit, int32_t* out_unit, int32_t* max_taps,
                                                  int32_t* first, int32_t* n_taps, float* weights, int64_t cap) {
  if (!rate_ok(rate, new_rate)) return FA_ERR_ARG;
  const LinearResampleDef d(rate, new_rate);
  int32_t longest = 0;
  for (int32_t p = 0; p < d.out_unit; ++p) {
    int32_t lo, n;
    d.span(p, &lo, &n);
    longest = std::max(longest, n);
  }
  const int64_t need = (int64_t)d.out_unit * longest;
  if (need > kMaxTableFloats) return FA_ERR_UNSUPPORTED;
  if (in_unit) *in_unit = d.in_unit;
  if (out_unit) *out_unit = d.out_unit;
  if (max_taps) *max_taps = longest;
  if (!weights) return need;
  if (cap < need || !first || !n_taps) return FA_ERR_ARG;
  for (int32_t p = 0; p < d.out_unit; ++p) {
    d.span(p, &first[p], &n_taps[p]);
    float* row = weights + (int64_t)p * longest;
    for (int32_t j = 0; j < longest; ++j) row[j] = j < n_taps[p] ? d.weight(p, first[p] + j) : 0.0f;
  }
  return need;
}

// the largest count c with (c - 1) / out_rate inside [0, n / in_rate), in ticks of 1 / lcm(in_rate, out_rate)
extern "C" int64_t fa_runtime_resample_out_len_host(int32_t rate, int32_t new_rate, int64_t n) {
  if (!rate_ok(rate, new_rate) || n < 0) return FA_ERR_ARG;
  const int64_t tick = (int64_t)rate / gcd32(rate, new_rate) * new_rate;
  const int64_t ticks = n * (tick / rate), per_out = tick / new_rate;
  if (ticks <= 0) return 0;
  int64_t last = ticks / per_out;
  if (last * per_out == ticks) --last;
  return last + 1;
}
