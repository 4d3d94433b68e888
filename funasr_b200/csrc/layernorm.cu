// Row LayerNorm (funasr/models/transformer/layer_norm.py:13-39, eps = 1e-12), one warp per row, the row
// held in registers (two-pass mean / variance in fp32), float4 loads and stores.
// Optional fused prologue for the first encoder layer: x*sqrt(d_model) + sinusoidal position encoding
// (SANMEncoder.forward encoder.py:409,428; SinusoidalPositionEncoder embedding.py:396-432).
// Optional fused epilogue for the tensor-core path: the normalised row is written as fp16 planes (hi, mid, lo) — the A
// operand of the following tensor-core GEMM — instead of / in addition to fp32.
// HBM-bound: algorithmic bytes = 8 B per element (read + write).
#include "common.cuh"
#include "tc_common.cuh"

namespace fa {

template <int NV, int NPL>  // NV: float4 per lane (row length <= 128*NV); NPL: fp16 planes written (0 = fp32 output only)
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* x, int64_t rows, int n, const float* __restrict__ g,
                 const float* __restrict__ bta, float eps, float* y,   // x may alias y (in-place)
                 const float* __restrict__ pe_inv, float xscale, int rows_per_batch,
                 plane_t* __restrict__ planes, int nplanes, int cols_pad, float* __restrict__ emb_out) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = n >> 2;
  const float4* xr = reinterpret_cast<const float4*>(x + row * n);
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c4 = lane + 32 * i;
    v[i] = c4 < nvec ? xr[c4] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (pe_inv != nullptr) {
    const float pos = (float)((int)(row % rows_per_batch) + 1);
    const int half = n >> 1;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c4 = lane + 32 * i;
      if (c4 < nvec) {
        float* e = reinterpret_cast<float*>(&v[i]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int c = 4 * c4 + k;
          const float pe = c < half ? sinf(__fmul_rn(pos, __ldg(pe_inv + c))) : cosf(__fmul_rn(pos, __ldg(pe_inv + c - half)));
          e[k] = __fadd_rn(__fmul_rn(e[k], xscale), pe);
        }
        // the embedded row itself: the residual of a first layer whose in_size == size (encoder.py:120-126; CT-Transformer)
        if (emb_out != nullptr) reinterpret_cast<float4*>(emb_out + row * n)[c4] = v[i];
      }
    }
  }
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(sum) / (float)n;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c4 = lane + 32 * i;
    if (c4 < nvec) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      sq += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = 1.0f / sqrtf(warp_sum(sq) / (float)n + eps);
  float4* yr = y ? reinterpret_cast<float4*>(y + row * n) : nullptr;
  const int64_t plane_elems = rows * cols_pad;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const float4* b4 = reinterpret_cast<const float4*>(bta);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c4 = lane + 32 * i;
    if (c4 < nvec) {
      const float4 gg = __ldg(g4 + c4), bb = __ldg(b4 + c4);
      float4 o;
      o.x = (v[i].x - mean) * rstd * gg.x + bb.x;
      o.y = (v[i].y - mean) * rstd * gg.y + bb.y;
      o.z = (v[i].z - mean) * rstd * gg.z + bb.z;
      o.w = (v[i].w - mean) * rstd * gg.w + bb.w;
      if (yr) yr[c4] = o;
      if (NPL > 0) {
        float e0 = o.x, e1 = o.y, e2 = o.z, e3 = o.w;
        plane_t* dst = planes + row * cols_pad + 4 * c4;
#pragma unroll
        for (int pl = 0; pl < NPL; ++pl) {           // packed cvt.rn.satfinite.f16x2 per plane (tc_common.cuh: operand planes)
          uint2 pk;
          pk.x = pack_planes2(e0, e1);
          pk.y = pack_planes2(e2, e3);
          *reinterpret_cast<uint2*>(dst) = pk;
          if (pl + 1 < NPL) {
            dst += plane_elems;
            const float2 a = unpack_planes2(pk.x), b = unpack_planes2(pk.y);
            e0 -= a.x; e1 -= a.y; e2 -= b.x; e3 -= b.y;
          }
        }
      }
    } else if (NPL > 0 && 4 * c4 < cols_pad) {         // zero the K padding (e.g. 560 -> 576)
#pragma unroll
      for (int pl = 0; pl < NPL; ++pl) {
        *reinterpret_cast<uint2*>(planes + pl * plane_elems + row * cols_pad + 4 * c4) = make_uint2(0u, 0u);
      }
    }
  }
}

int layernorm_launch(const float* x, int64_t rows, const FaNorm& nm, float* y, const float* pe_inv, float xscale,
                     int rows_per_batch, cudaStream_t st, plane_t* planes, int nplanes, int cols_pad, float* emb_out) {
  if (rows <= 0) return FA_OK;
  if (!x || (!y && !planes) || !nm.g || !nm.b) return FA_ERR_ARG;
  const int n = nm.n;
  if (n <= 0 || (n & 3) || n > 2048) return FA_ERR_UNSUPPORTED;
  if (planes && (cols_pad < n || (cols_pad & 3) || cols_pad > 2048)) return FA_ERR_UNSUPPORTED;
  const int need = ((planes ? cols_pad : n) / 4 + 31) / 32;
  const unsigned blocks = (unsigned)((rows + 7) / 8);
  const int npl = planes ? nplanes : 0;
  if (npl < 0 || npl > 3 || (planes && npl == 0)) return FA_ERR_ARG;
#define FA_LN_LAUNCH(NV, NPL)                                                                                \
  layernorm_kernel<NV, NPL><<<blocks, 256, 0, st>>>(x, rows, n, nm.g, nm.b, nm.eps, y, pe_inv, xscale,                   \
                                                   rows_per_batch > 0 ? rows_per_batch : 1, planes, nplanes, cols_pad, emb_out)
#define FA_LN_CASE(NV)                                                                                       \
  do {                                                                                                       \
    if (npl == 0) FA_LN_LAUNCH(NV, 0); else if (npl == 1) FA_LN_LAUNCH(NV, 1);                               \
    else if (npl == 2) FA_LN_LAUNCH(NV, 2); else FA_LN_LAUNCH(NV, 3);                                        \
  } while (0)
  if (need <= 4) FA_LN_CASE(4);
  else if (need <= 5) FA_LN_CASE(5);
  else if (need <= 8) FA_LN_CASE(8);
  else FA_LN_CASE(16);
#undef FA_LN_CASE
#undef FA_LN_LAUNCH
  FA_CHECK_LAUNCH();
  return FA_OK;
}

}  // namespace fa

extern "C" int fa_layernorm(const float* x, int64_t rows, const FaNorm* norm, float* y, const float* pe_inv,
                            float xscale, int32_t rows_per_batch, fa_stream_t stream) {
  if (!norm) return FA_ERR_ARG;
  return fa::layernorm_launch(x, rows, *norm, y, pe_inv, xscale, rows_per_batch, (cudaStream_t)stream, nullptr, 0, 0, nullptr);
}

// The same LayerNorm with the tensor-core path's fused outputs: fp16 planes [nplanes][rows][cols_pad] (columns [n, cols_pad) zeroed)
// and, with pe_inv, the embedded rows x * xscale + PE in emb_out.  y may be NULL when planes is set.
extern "C" int fa_layernorm_planes(const float* x, int64_t rows, const FaNorm* norm, float* y, void* planes, int32_t nplanes,
                                   int32_t cols_pad, const float* pe_inv, float xscale, int32_t rows_per_batch, float* emb_out,
                                   fa_stream_t stream) {
  if (!norm || rows < 0 || (planes && (nplanes < 1 || nplanes > 3)) || (!planes && nplanes != 0)) return FA_ERR_ARG;
  if (emb_out && !pe_inv) return FA_ERR_ARG;                       // the embedded rows exist only with the PE prologue
  if (pe_inv && rows_per_batch <= 0) return FA_ERR_ARG;
  // rows are read and written as float4, planes as uint2
  if ((((uintptr_t)x) & 15) || (((uintptr_t)y) & 15) || (((uintptr_t)emb_out) & 15) || (((uintptr_t)planes) & 7)) return FA_ERR_UNSUPPORTED;
  return fa::layernorm_launch(x, rows, *norm, y, pe_inv, xscale, rows_per_batch, (cudaStream_t)stream, reinterpret_cast<fa::plane_t*>(planes),
                              nplanes, cols_pad, emb_out);
}
