// Speaker clustering on the device: the O(N^2 d) and O(N^3) parts of the reference's SpectralCluster
// (campplus/cluster_backend.py; funasr_b200/diarization.py is the specification).
//
//   fa_spk_laplacian        embeddings [n, dim] -> unnormalised Laplacian [n, n] float64: row L2 norm, cosine similarity (fp32),
//                           p-pruning (one CTA sorts each row), 0.5 (P + P^T), zero diagonal, D - M
//   fa_spk_tridiagonalize   unblocked Householder reduction of the Laplacian to T = Q^T L Q (float64), three ordinary launches per
//                           column (reflector, symmetric mat-vec, rank-2 update); the reflectors stay in the matrix
//   fa_spk_back_transform   Q z for the few tridiagonal eigenvectors the clustering uses
//
// The small tridiagonal eigenproblem, the k-means and the post-processing run on the host (host_ops.cpp).  No launch waits on another
// CTA: there is no cooperative launch and no grid-wide barrier, every dependency is a kernel boundary on the caller's stream.
#include "common.cuh"

namespace {

constexpr int kMaxRows = 2047;          // the spectral path's largest input (ClusterBackend: fewer than 2048 chunks)
constexpr int kSortKeys = 2048;
constexpr int kMaxDim = 1024;

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

// s = xn xn^T in fp32: 64 x 64 output tiles, 4 x 4 per thread, 16-wide slices of the inner dimension
__global__ void __launch_bounds__(256) cosine_kernel(const float* __restrict__ xn, int n, int dim, float* __restrict__ s) {
  __shared__ float a[16][64 + 1], b[16][64 + 1];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
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

// p_pruning: the n_elems smallest entries of row blockIdx.x become 0, in place.  Keys (value, column) sorted ascending in shared
// memory by a bitonic network, so equal values go in column order (numpy's argsort is unstable: the one place the two may differ).
__global__ void __launch_bounds__(1024) prune_rows_kernel(float* __restrict__ s, int n, int n_elems) {
  __shared__ unsigned long long keys[kSortKeys];
  __shared__ unsigned char drop[kSortKeys];
  float* row = s + (int64_t)blockIdx.x * n;
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

// m = 0.5 (p + p^T) (fp32) with a zero diagonal; lap row i = diag(sum_j |m_ij|) - m, float64.  One CTA per row.
__global__ void __launch_bounds__(256) laplacian_kernel(const float* __restrict__ p, int n, double* __restrict__ lap) {
  __shared__ double red[8];
  const int i = blockIdx.x;
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
// superdiagonal of row j (the back-transform reads the row).  j == n - 1 only writes d[n - 1].
__global__ void __launch_bounds__(1024) reflector_kernel(double* __restrict__ lap, int n, int j, double* __restrict__ d, double* __restrict__ e,
                                                         double* __restrict__ tau, double* __restrict__ vbuf) {
  __shared__ double red[32];
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
// rows (fixed order, so the rank-2 update is deterministic)
__global__ void __launch_bounds__(256) symv_kernel(const double* __restrict__ lap, int n, int j, const double* __restrict__ tau,
                                                   const double* __restrict__ vbuf, double* __restrict__ p, double* __restrict__ partial) {
  __shared__ double v[kMaxRows];
  __shared__ double pv[8];
  const int m = n - j - 1, off = j + 1;
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
// updated matrix stays exactly symmetric.  32 x 32 tiles, 4 rows per thread.
__global__ void __launch_bounds__(256) rank2_kernel(double* __restrict__ lap, int n, int j, const double* __restrict__ tau,
                                                    const double* __restrict__ vbuf, const double* __restrict__ p,
                                                    const double* __restrict__ partial, int n_partial) {
  __shared__ double c_sh;
  const int m = n - j - 1, off = j + 1;
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

// z (row blockIdx.x of z [k, n]) := H(0) H(1) ... H(n-2) z, applied last reflector first.  One CTA per vector, z in shared memory.
__global__ void __launch_bounds__(512) back_transform_kernel(const double* __restrict__ lap, const double* __restrict__ tau, int n,
                                                             double* __restrict__ z) {
  __shared__ double zs[kMaxRows];
  __shared__ double red[16];
  double* zr = z + (int64_t)blockIdx.x * n;
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

// tridiagonalisation workspace: v [n], p [n], one partial per symv block
fa::Arena tri_carve(fa::Arena a, int n, double** v, double** p, double** partial) {
  *v = a.take<double>(n);
  *p = a.take<double>(n);
  *partial = a.take<double>((n + 7) / 8);
  return a;
}

}  // namespace

extern "C" double fa_spk_effective_pval(int32_t n, double pval) { return n * pval < 6 ? 6.0 / n : pval; }

extern "C" size_t fa_spk_laplacian_workspace_bytes(int32_t n, int32_t dim) {
  if (n < 1 || n > kMaxRows || dim < 1 || dim > kMaxDim) return 0;
  fa::Arena a = fa::Arena::measuring();
  a.take<float>((size_t)n * dim);
  a.take<float>((size_t)n * n);
  return a.bytes();
}

extern "C" int fa_spk_laplacian(const float* emb, int32_t n, int32_t dim, double pval, double* lap, void* workspace, size_t ws_bytes,
                                fa_stream_t stream) {
  if (!emb || !lap || n < 1 || dim < 1 || !(pval >= 0.0 && pval <= 1.0)) return FA_ERR_ARG;
  if (n > kMaxRows || dim > kMaxDim) return FA_ERR_UNSUPPORTED;
  fa::Arena a(workspace, ws_bytes);
  float* xn = a.take<float>((size_t)n * dim);
  float* s = a.take<float>((size_t)n * n);
  if (!a.ok() || !xn || !s) return FA_ERR_WORKSPACE;
  const double pv = fa_spk_effective_pval(n, pval);
  const int n_elems = (int)((1 - pv) * n);                  // int((1 - pval) * n): float64, truncated
  cudaStream_t st = (cudaStream_t)stream;
  normalize_rows_kernel<<<(n + 7) / 8, 256, 0, st>>>(emb, n, dim, xn);
  FA_CHECK_LAUNCH();
  cosine_kernel<<<dim3((n + 63) / 64, (n + 63) / 64), 256, 0, st>>>(xn, n, dim, s);
  FA_CHECK_LAUNCH();
  if (n_elems > 0) {
    prune_rows_kernel<<<n, 1024, 0, st>>>(s, n, n_elems);
    FA_CHECK_LAUNCH();
  }
  laplacian_kernel<<<n, 256, 0, st>>>(s, n, lap);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" size_t fa_spk_tridiagonalize_workspace_bytes(int32_t n) {
  if (n < 1 || n > kMaxRows) return 0;
  double *v, *p, *partial;
  return tri_carve(fa::Arena::measuring(), n, &v, &p, &partial).bytes();
}

extern "C" int fa_spk_tridiagonalize(double* lap, int32_t n, double* d, double* e, double* tau, void* workspace, size_t ws_bytes,
                                     fa_stream_t stream) {
  if (!lap || !d || n < 1 || (n > 1 && (!e || !tau))) return FA_ERR_ARG;
  if (n > kMaxRows) return FA_ERR_UNSUPPORTED;
  double *v, *p, *partial;
  const fa::Arena a = tri_carve(fa::Arena(workspace, ws_bytes), n, &v, &p, &partial);
  if (!a.ok() || !v || !p || !partial) return FA_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  for (int j = 0; j < n - 1; ++j) {
    const int m = n - j - 1, blocks = (m + 7) / 8, tiles = (m + 31) / 32;
    reflector_kernel<<<1, 1024, 0, st>>>(lap, n, j, d, e, tau, v);
    FA_CHECK_LAUNCH();
    symv_kernel<<<blocks, 256, 0, st>>>(lap, n, j, tau, v, p, partial);
    FA_CHECK_LAUNCH();
    rank2_kernel<<<dim3(tiles, tiles), 256, 0, st>>>(lap, n, j, tau, v, p, partial, blocks);
    FA_CHECK_LAUNCH();
  }
  reflector_kernel<<<1, 1024, 0, st>>>(lap, n, n - 1, d, e, tau, v);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" int fa_spk_back_transform(const double* lap, const double* tau, int32_t n, double* z, int32_t k, fa_stream_t stream) {
  if (!lap || !z || n < 1 || k < 1 || k > n || (n > 1 && !tau)) return FA_ERR_ARG;
  if (n > kMaxRows || k > 65535) return FA_ERR_UNSUPPORTED;
  if (n == 1) return FA_OK;
  back_transform_kernel<<<k, 512, 0, (cudaStream_t)stream>>>(lap, tau, n, z);
  FA_CHECK_LAUNCH();
  return FA_OK;
}
