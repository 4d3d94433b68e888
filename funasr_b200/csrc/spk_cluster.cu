// Speaker clustering on the device: the O(N^2 d) and O(N^3) parts of the reference's SpectralCluster
// (campplus/cluster_backend.py; funasr_b200/diarization.py is the specification).
//
//   fa_spk_laplacian        embeddings [n, dim] -> unnormalised Laplacian [n, n] float64: row L2 norm, cosine similarity (fp32),
//                           p-pruning (one CTA sorts each row), 0.5 (P + P^T), zero diagonal, D - M
//   fa_spk_tridiagonalize   unblocked Householder reduction of the Laplacian to T = Q^T L Q (float64), three ordinary launches per
//                           column (reflector, symmetric mat-vec, rank-2 update); the reflectors stay in the matrix
//   fa_spk_back_transform   Q z for the few tridiagonal eigenvectors the clustering uses
//
// Each has a _batch form over a ragged set of independent problems (a group's recordings), and the single entry is its one-set case.
// The set is a grid dimension and a CTA past its set's extent returns at once, so the batch makes the launches of its largest set
// (at most kSetsPerLaunch sets per launch) and every set does the same IEEE operations, in the same order, as it does alone.
//
// The small tridiagonal eigenproblem, the k-means and the post-processing run on the host (host_ops.cpp).  No launch waits on another
// CTA: there is no cooperative launch and no grid-wide barrier, every dependency is a kernel boundary on the caller's stream.
#include "common.cuh"
#include <vector>

namespace {

constexpr int kMaxRows = 2047;          // the spectral path's largest input (ClusterBackend: fewer than 2048 chunks)
constexpr int kSortKeys = 2048;
constexpr int kMaxDim = 1024;
constexpr int kSetsPerLaunch = 64;      // sets per launch of a batch: Sets<64> is a 2.5 KB kernel parameter, read in place (__grid_constant__)

// Sets [first, first + count) of a batch, concatenated in set order: set s has n[s] rows, starts at row row[s] of the embeddings and
// of d / e / tau / v / p, at entry mat[s] of the matrices, at partial part[s] of the symv partials and at entry z[s] of z
template <int C>
struct Sets {
  int count;
  int n[C];
  int aux[C];                           // the Laplacian: the entries pruned per row; the back-transform: k
  int64_t row[C], mat[C], part[C], z[C];
  int max_n() const { int m = 0; for (int i = 0; i < count; ++i) m = n[i] > m ? n[i] : m; return m; }
  int max_aux() const { int m = 0; for (int i = 0; i < count; ++i) m = aux[i] > m ? aux[i] : m; return m; }
};

// the batch's sets in launches of C, with their offsets (aux: NULL = 0; k: the back-transform's vectors per set)
template <int C>
std::vector<Sets<C>> make_sets(const int32_t* n, int32_t count, const int32_t* aux, const int32_t* k) {
  std::vector<Sets<C>> out;
  int64_t row = 0, mat = 0, part = 0, z = 0;
  for (int i = 0; i < count; ++i) {
    if (i % C == 0) out.push_back(Sets<C>{});
    Sets<C>& s = out.back();
    const int c = s.count++;
    s.n[c] = n[i]; s.aux[c] = aux ? aux[i] : 0;
    s.row[c] = row; s.mat[c] = mat; s.part[c] = part; s.z[c] = z;
    row += n[i]; mat += (int64_t)n[i] * n[i]; part += (n[i] + 7) / 8; z += k ? (int64_t)k[i] * n[i] : 0;
  }
  return out;
}

// f(sets) -> status for each launch group of the batch, the first failure returned.  A one-set batch (the single entries) passes a
// one-set parameter block, so its launches carry no larger parameters than the single entries always had.
template <class F>
int for_sets(const int32_t* n, int32_t count, const int32_t* aux, const int32_t* k, F f) {
  if (count == 1) return f(make_sets<1>(n, count, aux, k)[0]);
  for (const Sets<kSetsPerLaunch>& c : make_sets<kSetsPerLaunch>(n, count, aux, k)) {
    const int rc = f(c);
    if (rc != FA_OK) return rc;
  }
  return FA_OK;
}

// FA_OK, FA_ERR_ARG (NULL n, count < 1, an n[s] < 1) or FA_ERR_UNSUPPORTED (an n[s] > kMaxRows): the single entries' codes for n
int check_sizes(const int32_t* n, int32_t count) {
  if (!n || count < 1) return FA_ERR_ARG;
  bool big = false;
  for (int i = 0; i < count; ++i) {
    if (n[i] < 1) return FA_ERR_ARG;
    big = big || n[i] > kMaxRows;
  }
  return big ? FA_ERR_UNSUPPORTED : FA_OK;
}

int64_t sum_n(const int32_t* n, int32_t count, bool squares) {
  int64_t t = 0;
  for (int i = 0; i < count; ++i) t += squares ? (int64_t)n[i] * n[i] : n[i];
  return t;
}

// ---- Laplacian

// xn[i] = x[i] / ||x[i]|| (a zero norm counts as 1, _normalize_rows), one warp per row
__global__ void __launch_bounds__(256) normalize_rows_kernel(const float* __restrict__ x, int n, int dim, float* __restrict__ xn) {
  const int row = blockIdx.x * 8 + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (row >= n) return;
  const float* r = x + (int64_t)row * dim;
  float s = 0.f;
  for (int c = lane; c < dim; c += 32) s += r[c] * r[c];
  s = fa::warp_sum(s);
  float nrm = sqrtf(s);
  if (nrm == 0.f) nrm = 1.f;
  for (int c = lane; c < dim; c += 32) xn[(int64_t)row * dim + c] = r[c] / nrm;
}

// s = xn xn^T in fp32 per set (blockIdx.z): 64 x 64 output tiles, 4 x 4 per thread, 16-wide slices of the inner dimension
template <class S>
__global__ void __launch_bounds__(256) cosine_kernel(const float* __restrict__ xn, int dim, float* __restrict__ s, const __grid_constant__ S sets) {
  __shared__ float a[16][64 + 1], b[16][64 + 1];
  const int n = sets.n[blockIdx.z];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  if (r0 >= n || c0 >= n) return;
  xn += sets.row[blockIdx.z] * dim;
  s += sets.mat[blockIdx.z];
  float acc[4][4] = {};
  for (int k0 = 0; k0 < dim; k0 += 16) {
    for (int e = threadIdx.x; e < 16 * 64; e += 256) {
      const int rr = e / 16, kk = e % 16, k = k0 + kk;
      a[kk][rr] = (r0 + rr < n && k < dim) ? xn[(int64_t)(r0 + rr) * dim + k] : 0.f;
      b[kk][rr] = (c0 + rr < n && k < dim) ? xn[(int64_t)(c0 + rr) * dim + k] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk)
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += a[kk][ty * 4 + i] * b[kk][tx * 4 + j];
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = r0 + ty * 4 + i, c = c0 + tx * 4 + j;
      if (r < n && c < n) s[(int64_t)r * n + c] = acc[i][j];
    }
}

__device__ __forceinline__ uint32_t ordered_bits(float f) {     // ascending float order as unsigned order
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// p_pruning: the n_elems smallest entries of row blockIdx.x of set blockIdx.y become 0, in place.  Keys (value, column) sorted ascending
// in shared memory by a bitonic network, so equal values go in column order (numpy's argsort is unstable: the one place the two may
// differ).
template <class S>
__global__ void __launch_bounds__(1024) prune_rows_kernel(float* __restrict__ s, const __grid_constant__ S sets) {
  __shared__ unsigned long long keys[kSortKeys];
  __shared__ unsigned char drop[kSortKeys];
  const int n = sets.n[blockIdx.y], n_elems = sets.aux[blockIdx.y];
  if ((int)blockIdx.x >= n || n_elems <= 0) return;
  float* row = s + sets.mat[blockIdx.y] + (int64_t)blockIdx.x * n;
  for (int c = threadIdx.x; c < kSortKeys; c += blockDim.x) {
    keys[c] = c < n ? ((unsigned long long)ordered_bits(row[c]) << 32) | (unsigned)c : ~0ull;
    drop[c] = 0;
  }
  __syncthreads();
  for (int size = 2; size <= kSortKeys; size <<= 1)
    for (int stride = size / 2; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < kSortKeys / 2; t += blockDim.x) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        const bool up = (lo & size) == 0;
        const unsigned long long x = keys[lo], y = keys[hi];
        if ((x > y) == up) { keys[lo] = y; keys[hi] = x; }
      }
      __syncthreads();
    }
  for (int r = threadIdx.x; r < n_elems; r += blockDim.x) drop[keys[r] & 0xffffffffu] = 1;
  __syncthreads();
  for (int c = threadIdx.x; c < n; c += blockDim.x)
    if (drop[c]) row[c] = 0.f;
}

__device__ __forceinline__ double block_sum(double v, double* red) {   // every thread gets the sum; fixed order
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x / 32, nw = blockDim.x / 32;
  __syncthreads();
  if (threadIdx.x % 32 == 0) red[w] = v;
  __syncthreads();
  double t = 0.0;
  for (int k = 0; k < nw; ++k) t += red[k];
  return t;
}

// m = 0.5 (p + p^T) (fp32) with a zero diagonal; lap row i = diag(sum_j |m_ij|) - m, float64.  One CTA per row (blockIdx.x) of
// each set (blockIdx.y).
template <class S>
__global__ void __launch_bounds__(256) laplacian_kernel(const float* __restrict__ p, double* __restrict__ lap, const __grid_constant__ S sets) {
  __shared__ double red[8];
  const int i = blockIdx.x, n = sets.n[blockIdx.y];
  if (i >= n) return;
  p += sets.mat[blockIdx.y];
  lap += sets.mat[blockIdx.y];
  double deg = 0.0;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const float m = j == i ? 0.f : 0.5f * (p[(int64_t)i * n + j] + p[(int64_t)j * n + i]);
    deg += fabs((double)m);
    lap[(int64_t)i * n + j] = j == i ? 0.0 : (double)(0.f - m);
  }
  deg = block_sum(deg, red);
  if (threadIdx.x == 0) lap[(int64_t)i * n + i] = (double)(float)deg;
}

// ---- Householder tridiagonalisation (LAPACK dsytd2, lower, unblocked)

// Column j: the reflector H = I - tau v v^T with H a[j+1:, j] = (beta, 0, ...).  Reads row j (the matrix is kept exactly symmetric);
// writes d[j], e[j], tau[j], v (v[0] = 1) to vbuf, and keeps v[1:] in lap below the subdiagonal of column j and right of the
// superdiagonal of row j (the back-transform reads the row).  j == n - 1 only writes d[n - 1]; a set with j >= n is done.  One CTA per
// set (blockIdx.x).
template <class S>
__global__ void __launch_bounds__(1024) reflector_kernel(double* __restrict__ lap, int j, double* __restrict__ d, double* __restrict__ e,
                                                         double* __restrict__ tau, double* __restrict__ vbuf, const __grid_constant__ S sets) {
  __shared__ double red[32];
  const int n = sets.n[blockIdx.x];
  if (j >= n) return;
  const int64_t o = sets.row[blockIdx.x];
  lap += sets.mat[blockIdx.x]; d += o; e += o; tau += o; vbuf += o;
  double* row = lap + (int64_t)j * n;
  const int m = n - j - 1;
  if (threadIdx.x == 0) d[j] = row[j];
  if (m <= 0) return;
  double ss = 0.0;
  for (int t = 1 + threadIdx.x; t < m; t += blockDim.x) ss += row[j + 1 + t] * row[j + 1 + t];
  ss = block_sum(ss, red);
  const double alpha = row[j + 1];
  double beta = alpha, tj = 0.0, scale = 0.0;
  if (ss != 0.0) {
    beta = -copysign(sqrt(alpha * alpha + ss), alpha);
    tj = (beta - alpha) / beta;
    scale = 1.0 / (alpha - beta);
  }
  __syncthreads();                                            // every thread read row[j + 1] before it is overwritten
  for (int t = threadIdx.x; t < m; t += blockDim.x) {
    const double v = t == 0 ? 1.0 : (ss != 0.0 ? row[j + 1 + t] * scale : 0.0);
    vbuf[t] = v;
    const double kept = t == 0 ? beta : v;
    row[j + 1 + t] = kept;
    lap[(int64_t)(j + 1 + t) * n + j] = kept;
  }
  if (threadIdx.x == 0) { e[j] = beta; tau[j] = tj; }
}

// p = tau A22 v over the trailing block A22 = lap[j+1:, j+1:], one warp per row; partial[blockIdx.x] = sum of p_t v_t over the block's
// rows (fixed order, so the rank-2 update is deterministic).  Set blockIdx.y has (m + 7) / 8 blocks.
template <class S>
__global__ void __launch_bounds__(256) symv_kernel(const double* __restrict__ lap, int j, const double* __restrict__ tau,
                                                   const double* __restrict__ vbuf, double* __restrict__ p, double* __restrict__ partial,
                                                   const __grid_constant__ S sets) {
  __shared__ double v[kMaxRows];
  __shared__ double pv[8];
  const int n = sets.n[blockIdx.y], m = n - j - 1, off = j + 1;
  if (m <= 0 || (int)blockIdx.x >= (m + 7) / 8) return;
  const int64_t o = sets.row[blockIdx.y];
  lap += sets.mat[blockIdx.y]; tau += o; vbuf += o; p += o; partial += sets.part[blockIdx.y];
  for (int t = threadIdx.x; t < m; t += blockDim.x) v[t] = vbuf[t];
  __syncthreads();
  const int w = threadIdx.x / 32, lane = threadIdx.x % 32, r = blockIdx.x * 8 + w;
  const double tj = tau[j];
  double mine = 0.0;
  if (r < m) {
    const double* a = lap + (int64_t)(off + r) * n + off;
    double s = 0.0;
    for (int c = lane; c < m; c += 32) s += a[c] * v[c];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const double pr = tj * s;
    if (lane == 0) p[r] = pr;
    mine = pr * v[r];
  }
  if (lane == 0) pv[w] = mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += pv[k];
    partial[blockIdx.x] = t;
  }
}

// A22 -= v w^T + w v^T with w = p - (tau / 2)(p^T v) v.  Each entry's two products are rounded and added without contraction, so the
// updated matrix stays exactly symmetric.  32 x 32 tiles, 4 rows per thread; set blockIdx.z has (m + 31) / 32 tiles a side.
template <class S>
__global__ void __launch_bounds__(256) rank2_kernel(double* __restrict__ lap, int j, const double* __restrict__ tau,
                                                    const double* __restrict__ vbuf, const double* __restrict__ p,
                                                    const double* __restrict__ partial, const __grid_constant__ S sets) {
  __shared__ double c_sh;
  const int n = sets.n[blockIdx.z], m = n - j - 1, off = j + 1, n_partial = (m + 7) / 8;
  if (m <= 0 || (int)blockIdx.x * 32 >= m || (int)blockIdx.y * 32 >= m) return;
  const int64_t o = sets.row[blockIdx.z];
  lap += sets.mat[blockIdx.z]; tau += o; vbuf += o; p += o; partial += sets.part[blockIdx.z];
  if (threadIdx.x == 0) {
    double pv = 0.0;
    for (int k = 0; k < n_partial; ++k) pv += partial[k];
    c_sh = __dmul_rn(0.5 * tau[j], pv);
  }
  __syncthreads();
  const double c = c_sh;
  const int col = blockIdx.x * 32 + threadIdx.x % 32;
  if (col >= m) return;
  const double vc = vbuf[col], wc = __dsub_rn(p[col], __dmul_rn(c, vc));
  for (int k = 0; k < 4; ++k) {
    const int r = blockIdx.y * 32 + threadIdx.x / 32 + 8 * k;
    if (r >= m) break;
    const double vr = vbuf[r], wr = __dsub_rn(p[r], __dmul_rn(c, vr));
    double* a = lap + (int64_t)(off + r) * n + off + col;
    *a = __dsub_rn(*a, __dadd_rn(__dmul_rn(vr, wc), __dmul_rn(wr, vc)));
  }
}

// z (row blockIdx.x of set blockIdx.y's z [k, n]) := H(0) H(1) ... H(n-2) z, applied last reflector first.  One CTA per (vector, set),
// z in shared memory; n == 1 leaves z as it is.
template <class S>
__global__ void __launch_bounds__(512) back_transform_kernel(const double* __restrict__ lap, const double* __restrict__ tau, double* __restrict__ z,
                                                             const __grid_constant__ S sets) {
  __shared__ double zs[kMaxRows];
  __shared__ double red[16];
  const int n = sets.n[blockIdx.y];
  if ((int)blockIdx.x >= sets.aux[blockIdx.y] || n == 1) return;
  lap += sets.mat[blockIdx.y];
  tau += sets.row[blockIdx.y];
  double* zr = z + sets.z[blockIdx.y] + (int64_t)blockIdx.x * n;
  for (int t = threadIdx.x; t < n; t += blockDim.x) zs[t] = zr[t];
  __syncthreads();
  for (int j = n - 2; j >= 0; --j) {
    const double tj = tau[j];
    if (tj == 0.0) continue;
    const double* row = lap + (int64_t)j * n;
    const int m = n - j - 1, off = j + 1;
    double s = 0.0;
    for (int t = threadIdx.x; t < m; t += blockDim.x) s += (t == 0 ? 1.0 : row[off + t]) * zs[off + t];
    s = block_sum(s, red) * tj;
    for (int t = threadIdx.x; t < m; t += blockDim.x) zs[off + t] -= s * (t == 0 ? 1.0 : row[off + t]);
    __syncthreads();
  }
  for (int t = threadIdx.x; t < n; t += blockDim.x) zr[t] = zs[t];
}

// Laplacian workspace: the normalised rows [sum n, dim] and the similarities [sum n^2], fp32
fa::Arena lap_carve(fa::Arena a, const int32_t* n, int32_t count, int dim, float** xn, float** s) {
  *xn = a.take<float>((size_t)sum_n(n, count, false) * dim);
  *s = a.take<float>((size_t)sum_n(n, count, true));
  return a;
}

// tridiagonalisation workspace: v [sum n], p [sum n], one partial per symv block of each set
fa::Arena tri_carve(fa::Arena a, const int32_t* n, int32_t count, double** v, double** p, double** partial) {
  int64_t parts = 0;
  for (int i = 0; i < count; ++i) parts += (n[i] + 7) / 8;
  *v = a.take<double>((size_t)sum_n(n, count, false));
  *p = a.take<double>((size_t)sum_n(n, count, false));
  *partial = a.take<double>((size_t)parts);
  return a;
}

}  // namespace

extern "C" double fa_spk_effective_pval(int32_t n, double pval) { return n * pval < 6 ? 6.0 / n : pval; }

extern "C" size_t fa_spk_laplacian_batch_workspace_bytes(const int32_t* n, int32_t count, int32_t dim) {
  if (check_sizes(n, count) != FA_OK || dim < 1 || dim > kMaxDim) return 0;
  float *xn, *s;
  return lap_carve(fa::Arena::measuring(), n, count, dim, &xn, &s).bytes();
}

extern "C" size_t fa_spk_laplacian_workspace_bytes(int32_t n, int32_t dim) { return fa_spk_laplacian_batch_workspace_bytes(&n, 1, dim); }

extern "C" int fa_spk_laplacian_batch(const float* emb, const int32_t* n, int32_t count, int32_t dim, double pval, double* lap, void* workspace,
                                      size_t ws_bytes, fa_stream_t stream) {
  const int sizes = check_sizes(n, count);
  if (!emb || !lap || sizes == FA_ERR_ARG || dim < 1 || !(pval >= 0.0 && pval <= 1.0)) return FA_ERR_ARG;
  if (sizes != FA_OK || dim > kMaxDim) return FA_ERR_UNSUPPORTED;
  float *xn, *s;
  const fa::Arena a = lap_carve(fa::Arena(workspace, ws_bytes), n, count, dim, &xn, &s);
  if (!a.ok() || !xn || !s) return FA_ERR_WORKSPACE;
  std::vector<int32_t> n_elems((size_t)count);
  for (int i = 0; i < count; ++i) {
    const double pv = fa_spk_effective_pval(n[i], pval);
    n_elems[i] = (int)((1 - pv) * n[i]);                    // int((1 - pval) * n): float64, truncated
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t rows = sum_n(n, count, false);
  normalize_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(emb, (int)rows, dim, xn);
  FA_CHECK_LAUNCH();
  return for_sets(n, count, n_elems.data(), nullptr, [&](const auto& c) {
    const int nmax = c.max_n(), tiles = (nmax + 63) / 64;
    cosine_kernel<<<dim3(tiles, tiles, c.count), 256, 0, st>>>(xn, dim, s, c);
    FA_CHECK_LAUNCH();
    if (c.max_aux() > 0) {
      prune_rows_kernel<<<dim3(nmax, c.count), 1024, 0, st>>>(s, c);
      FA_CHECK_LAUNCH();
    }
    laplacian_kernel<<<dim3(nmax, c.count), 256, 0, st>>>(s, lap, c);
    FA_CHECK_LAUNCH();
    return FA_OK;
  });
}

extern "C" int fa_spk_laplacian(const float* emb, int32_t n, int32_t dim, double pval, double* lap, void* workspace, size_t ws_bytes,
                                fa_stream_t stream) {
  return fa_spk_laplacian_batch(emb, &n, 1, dim, pval, lap, workspace, ws_bytes, stream);
}

extern "C" size_t fa_spk_tridiagonalize_batch_workspace_bytes(const int32_t* n, int32_t count) {
  if (check_sizes(n, count) != FA_OK) return 0;
  double *v, *p, *partial;
  return tri_carve(fa::Arena::measuring(), n, count, &v, &p, &partial).bytes();
}

extern "C" size_t fa_spk_tridiagonalize_workspace_bytes(int32_t n) { return fa_spk_tridiagonalize_batch_workspace_bytes(&n, 1); }

// Column j runs for every set with j < n in one launch each of the reflector, symv and rank-2 kernels: 3 (max n - 1) + 1 launches
extern "C" int fa_spk_tridiagonalize_batch(double* lap, const int32_t* n, int32_t count, double* d, double* e, double* tau, void* workspace,
                                           size_t ws_bytes, fa_stream_t stream) {
  const int sizes = check_sizes(n, count);
  if (!lap || !d || sizes == FA_ERR_ARG) return FA_ERR_ARG;
  for (int i = 0; i < count; ++i)
    if (n[i] > 1 && (!e || !tau)) return FA_ERR_ARG;
  if (sizes != FA_OK) return FA_ERR_UNSUPPORTED;
  double *v, *p, *partial;
  const fa::Arena a = tri_carve(fa::Arena(workspace, ws_bytes), n, count, &v, &p, &partial);
  if (!a.ok() || !v || !p || !partial) return FA_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  return for_sets(n, count, nullptr, nullptr, [&](const auto& c) {
    const int nmax = c.max_n();
    for (int j = 0; j < nmax - 1; ++j) {
      const int m = nmax - j - 1, blocks = (m + 7) / 8, tiles = (m + 31) / 32;
      reflector_kernel<<<c.count, 1024, 0, st>>>(lap, j, d, e, tau, v, c);
      FA_CHECK_LAUNCH();
      symv_kernel<<<dim3(blocks, c.count), 256, 0, st>>>(lap, j, tau, v, p, partial, c);
      FA_CHECK_LAUNCH();
      rank2_kernel<<<dim3(tiles, tiles, c.count), 256, 0, st>>>(lap, j, tau, v, p, partial, c);
      FA_CHECK_LAUNCH();
    }
    reflector_kernel<<<c.count, 1024, 0, st>>>(lap, nmax - 1, d, e, tau, v, c);
    FA_CHECK_LAUNCH();
    return FA_OK;
  });
}

extern "C" int fa_spk_tridiagonalize(double* lap, int32_t n, double* d, double* e, double* tau, void* workspace, size_t ws_bytes,
                                     fa_stream_t stream) {
  return fa_spk_tridiagonalize_batch(lap, &n, 1, d, e, tau, workspace, ws_bytes, stream);
}

extern "C" int fa_spk_back_transform_batch(const double* lap, const double* tau, const int32_t* n, const int32_t* k, int32_t count, double* z,
                                           fa_stream_t stream) {
  const int sizes = check_sizes(n, count);
  if (!lap || !z || !k || sizes == FA_ERR_ARG) return FA_ERR_ARG;
  bool any = false;                                          // a set with n > 1: n == 1 leaves its z as it is
  for (int i = 0; i < count; ++i) {
    if (k[i] < 1 || k[i] > n[i] || (n[i] > 1 && !tau)) return FA_ERR_ARG;
    any = any || n[i] > 1;
  }
  if (sizes != FA_OK) return FA_ERR_UNSUPPORTED;
  if (!any) return FA_OK;
  return for_sets(n, count, k, k, [&](const auto& c) {
    back_transform_kernel<<<dim3(c.max_aux(), c.count), 512, 0, (cudaStream_t)stream>>>(lap, tau, z, c);
    FA_CHECK_LAUNCH();
    return FA_OK;
  });
}

extern "C" int fa_spk_back_transform(const double* lap, const double* tau, int32_t n, double* z, int32_t k, fa_stream_t stream) {
  return fa_spk_back_transform_batch(lap, tau, &n, &k, 1, z, stream);
}
