// fp32 SIMT GEMM with fused nn.Linear epilogue:  Y = act(X W^T + b) (+ res1) (+ res2).
//
// This is the parity-reference contraction path (FA_GEMM_F32_SIMT): plain FFMA accumulation in fp32, the
// arithmetic closest to the reference's MKL/cuBLAS sgemm (attention.py:256,306; positionwise_feed_forward.py:34).
// The tensor-core path (gemm_tc.cu) is validated against it on the device.
// 128x128x16 tiles, 256 threads, 8x8 outputs per thread, register-prefetch double buffering.
#include "common.cuh"
#include "kernels.h"

namespace fa {

constexpr int BM = 128, BN = 128, BK = 16, PADM = 4;

__global__ void __launch_bounds__(256)
gemm_f32_kernel(const float* __restrict__ A, int64_t lda, const float* __restrict__ W, int64_t ldw,
                const float* __restrict__ bias, int relu, const float* __restrict__ r1, int64_t ldr1,
                const float* __restrict__ r2, int64_t ldr2, float* __restrict__ C, int64_t ldc, int64_t M, int N,
                int K) {
  __shared__ __align__(16) float As[2][BK][BM + PADM];
  __shared__ __align__(16) float Bs[2][BK][BN + PADM];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (int64_t)blockIdx.y * BM;
  const int n0 = blockIdx.x * BN;
  const int lrow = tid >> 2, lkq = tid & 3;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra[2], rb[2];
  auto gload = [&](int k0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t m = m0 + lrow + 64 * h;
      ra[h] = m < M ? __ldg(reinterpret_cast<const float4*>(A + m * lda + k0 + 4 * lkq)) : make_float4(0.f, 0.f, 0.f, 0.f);
      const int n = n0 + lrow + 64 * h;
      rb[h] = n < N ? __ldg(reinterpret_cast<const float4*>(W + (int64_t)n * ldw + k0 + 4 * lkq)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = lrow + 64 * h;
      As[buf][4 * lkq + 0][r] = ra[h].x; As[buf][4 * lkq + 1][r] = ra[h].y;
      As[buf][4 * lkq + 2][r] = ra[h].z; As[buf][4 * lkq + 3][r] = ra[h].w;
      Bs[buf][4 * lkq + 0][r] = rb[h].x; Bs[buf][4 * lkq + 1][r] = rb[h].y;
      Bs[buf][4 * lkq + 2][r] = rb[h].z; Bs[buf][4 * lkq + 3][r] = rb[h].w;
    }
  };

  const int nk = K / BK;
  gload(0);
  sstore(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) gload((kt + 1) * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      sstore(buf ^ 1);
      __syncthreads();
    }
  }

  // epilogue: bias -> relu -> residuals
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int n = n0 + jh * 64 + tx * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int nn = n + j;
        if (nn >= N) continue;
        float v = acc[i][jh * 4 + j];
        if (bias) v += __ldg(bias + nn);
        if (relu) v = fmaxf(v, 0.f);
        if (r1) v += __ldg(r1 + m * ldr1 + nn);
        if (r2) v += __ldg(r2 + m * ldr2 + nn);
        C[m * ldc + nn] = v;
      }
    }
  }
}

int gemm_f32_launch(const float* A, int64_t lda, int64_t M, const float* W, int N, int K, const float* bias, const GemmEpi& epi, cudaStream_t st) {
  if (M <= 0 || N <= 0) return FA_OK;
  if (!A || !W || !epi.y || epi.planes || epi.att) return FA_ERR_ARG;
  if (K % BK != 0 || lda % 4 != 0 || (((uintptr_t)A) & 15) || (((uintptr_t)W) & 15)) return FA_ERR_UNSUPPORTED;
  dim3 grid((N + BN - 1) / BN, (unsigned)((M + BM - 1) / BM));
  gemm_f32_kernel<<<grid, 256, 0, st>>>(A, lda, W, K, bias, epi.relu_on, epi.r1, epi.ld1, epi.r2, epi.ld2, epi.y, epi.ldy, M, N, K);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

}  // namespace fa
