// wgmma / TMA GEMM with fp16 operand splitting and a fused nn.Linear epilogue (sm_90a).
//
//   Y[M,N] = act( sum_{(p,q) in terms} A_p[M,K] * W_q[N,K]^T + b ) (+ res1) (+ res2)
//
// A_p / W_q are the fp16 planes of the fp32 operands (x = hi + mid + lo, made by split kernels), accumulation is
// fp32 in registers.  Modes: F16X1 = {(0,0)} (fast), F16X3 = {(0,0),(0,1),(1,0)} (~2^-17 relative, the default
// parity mode on tensor cores), F16X6 = X3 + {(1,1),(0,2),(2,0)} (~fp32).  This replaces the torch.nn.Linear calls
// of the hot path (sanm/attention.py:256,306, transformer/positionwise_feed_forward.py:34,
// sanm/positionwise_feed_forward.py:33, paraformer/decoder.py:444, cif conv as GEMM).
//
// Structure (one persistent CTA per SM, 384 threads, 128 x BN output tiles, "ping-pong" schedule):
//   warpgroup 0    : TMA producer — one elected lane of warp 0 issues cp.async.bulk.tensor.2d (SWIZZLE_128B) of the A/W plane
//                    tiles into a shared-memory ring, in the order the MMAs consume them; the warpgroup gives its registers back
//   warpgroups 1, 2: consumers — each owns whole 128 x BN tiles and takes every second tile of the CTA's persistent sequence.  An
//                    ordering barrier pair hands the tensor pipe from one to the other: while one issues its tile's
//                    wgmma.mma_async (two m64nBNk16 per K=16 slice and split term, one k-block of MMAs in flight), the other
//                    runs the epilogue of its previous tile straight from its accumulator registers (bias/ReLU/residuals ->
//                    fp32 rows to HBM, or fp16 planes for a following GEMM).
#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"
#include <stdlib.h>
#include <unordered_map>

namespace fa {

constexpr int TC_BM = 128;      // tile rows: two wgmma M = 64 halves, both issued by one consumer warpgroup
constexpr int TC_BK = 64;       // one 128-byte swizzle span of fp16
constexpr int TC_UK = 16;       // wgmma K for 16-bit inputs
constexpr uint32_t TC_TILE_BYTES_A = TC_BM * TC_BK * 2;   // 16 KB per plane tile
constexpr uint32_t TC_PRODUCER_REGS = 40, TC_CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 64 K registers
constexpr uint32_t TC_ORDER_BAR = 1;   // named barriers 1, 2: "consumer warpgroup 0 / 1 may issue its tile's MMAs"

// ------------------------------------------------------------------------------------------------ kernel
struct TcParams {
  int64_t M;
  int N, Kp;            // Kp: K padded to a multiple of 64 (planes are zero padded)
  int64_t a_plane_rows; // rows between consecutive A planes in the 2D tensor map (= M)
  int w_plane_rows;     // = N
  int n_terms;          // 1, 3 or 6
  int relu;
  const float* bias;
  const float* r1; int64_t ldr1;
  const float* r2; int64_t ldr2;
  float* C; int64_t ldc;                 // fp32 output (or null)
  plane_t* out_planes;             // fp16 plane output [3][M][ldo] (or null)
  int64_t ldo; int out_nplanes;
  int tiles_m, tiles_n;
  AttnSinks att;                          // optional: route column ranges to attention operand planes
  // The tensor cores accumulate in fp32 with truncation: every 16-wide k-step shrinks the running sum by a fraction of an ulp, a
  // SYSTEMATIC relative error that grows linearly in K (tools/noise_probe.py measures it against the fp32 SIMT GEMM).  The epilogue
  // multiplies the accumulator by 1 + (K / 16) * c (rz_comp_scale; c measured on an H100, DESIGN.md §2) before the bias: the expected
  // shrink is undone, what remains is the random part.  FA_RZ_COMP=0 disables it (A/B).
  float acc_scale;
};

static float rz_comp_scale(int kp, int n_terms) {
  static const bool on = [] { const char* e = getenv("FA_RZ_COMP"); return !(e && e[0] == '0'); }();
  if (!on) return 1.0f;
  return 1.0f + (float)(kp / 16) * (n_terms >= 3 ? 5.3e-8f : 3.4e-8f);
}

__constant__ int c_term_a[6] = {0, 0, 1, 1, 0, 2};
__constant__ int c_term_w[6] = {0, 1, 0, 1, 2, 0};

// Accumulators of one 128 x BN tile in a consumer warpgroup: d[h] is the m64 MMA over the tile's 8-row groups h, h + 2, h + 4, ..
// (descriptor stride 2048 B), so warp q holds exactly rows [32 q, +32): lane l has rows 32 q + 16 e + 8 h + l / 4 (e = 0: registers
// 4 j, 4 j + 1; e = 1: 4 j + 2, 4 j + 3) at columns 8 j + 2 (l % 4) + {0, 1}.
//
// Epilogue of one tile: warp q drains its 32 rows one 16-column chunk at a time.
//   phase 1  the chunk's 16 accumulators per lane -> a padded per-warp shared-memory tile [32][20] (row = 32-row offset)
//   phase 2  re-read with the warp laid out as 8 rows x 4 float4 columns, so bias / residual loads and every store are
//            coalesced 16-byte (fp32) or 8-byte (fp16 plane) accesses; V columns of the attention sink take a
//            column-per-lane path that writes the per-head transposed planes as 4 consecutive keys (8 bytes) per store.
// The chunk loops are fully unrolled: the accumulator registers are indexed by compile-time constants only.
constexpr int EPI_CH = 16;                       // columns per chunk
constexpr int EPI_LD = 20;                       // padded row pitch (floats): 16-byte aligned float4 rows
constexpr int EPI_WARP_FLOATS = 32 * EPI_LD;     // 2.5 KB per consumer warp
constexpr int EPI_WARPS = 8;

template <int BN>
__device__ __forceinline__ void acc_chunk_to_stage(const float (&d)[2][BN / 2], const int c0, float* stage, int lane) {
  float* s = stage + (lane >> 2) * EPI_LD + 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const int j = c0 / 8 + jj;
      *reinterpret_cast<float2*>(s + 8 * h * EPI_LD + 8 * jj) = make_float2(d[h][4 * j], d[h][4 * j + 1]);
      *reinterpret_cast<float2*>(s + (16 + 8 * h) * EPI_LD + 8 * jj) = make_float2(d[h][4 * j + 2], d[h][4 * j + 3]);
    }
}

// row `lane` (16 consecutive fp32 columns) of the staged chunk -> 16 registers
__device__ __forceinline__ void acc_ld_32x16(const float* src, uint32_t (&r)[16]) {
#pragma unroll
  for (int j = 0; j < 16; j += 4) {
    const uint4 v = *reinterpret_cast<const uint4*>(src + j);
    r[j] = v.x; r[j + 1] = v.y; r[j + 2] = v.z; r[j + 3] = v.w;
  }
}

// x = hi + mid + lo split of 4 values into fp16 planes: packed converts (cvt.rn.satfinite.f16x2.f32), packed unpack.  NPL is a compile-
// time constant: with a runtime plane count the loop compiles to a branchy 4x-unrolled body.
template <int NPL>
__device__ __forceinline__ void store_planes4(plane_t* dst, int64_t plane_stride, float x0, float x1, float x2, float x3) {
#pragma unroll
  for (int pl = 0; pl < NPL; ++pl) {
    uint2 pk;
    pk.x = pack_planes2(x0, x1);
    pk.y = pack_planes2(x2, x3);
    *reinterpret_cast<uint2*>(dst) = pk;
    if (pl + 1 < NPL) {
      dst += plane_stride;
      const float2 a = unpack_planes2(pk.x), b = unpack_planes2(pk.y);
      x0 -= a.x; x1 -= a.y; x2 -= b.x; x3 -= b.y;
    }
  }
}

// per-head transposed V planes straight from the row-per-lane registers: for a fixed head dim the 32 lanes hold 32
// consecutive keys, so every 2-byte store instruction covers one 64-byte run.  The value is fmaf(acc, acc_scale, bias), rounded
// once, as in every other output of the epilogue (the fp32 V rows the FSMN reads, the staged transpose).
template <int NPL>
__device__ __forceinline__ void store_vt16(plane_t* dst, int64_t t_pad, int64_t plane, const uint32_t (&r)[16], const float* bias, float acc_scale) {
#pragma unroll
  for (int j = 0; j < 16; j += 2) {
    const float b0 = bias ? __ldg(bias + j) : 0.f, b1 = bias ? __ldg(bias + j + 1) : 0.f;
    float x0 = fmaf(__uint_as_float(r[j]), acc_scale, b0), x1 = fmaf(__uint_as_float(r[j + 1]), acc_scale, b1);
    plane_t* d0 = dst + (int64_t)j * t_pad;
#pragma unroll
    for (int pl = 0; pl < NPL; ++pl) {
      const uint32_t hb = pack_planes2(x0, x1);
      d0[0] = __ushort_as_half((unsigned short)(hb & 0xFFFFu));
      d0[t_pad] = __ushort_as_half((unsigned short)(hb >> 16));
      if (pl + 1 < NPL) { d0 += plane; const float2 a = unpack_planes2(hb); x0 -= a.x; x1 -= a.y; }
    }
  }
}

// The same through shared memory, for key counts that are a multiple of 4 (rows of one utterance then start at a multiple of 4,
// so groups of four consecutive keys stay inside one utterance and are 8-byte aligned in the transposed planes): the warp's
// 32 x 16 chunk is staged at pitch 17 (conflict free for the row-per-lane writes AND for the column reads below), then lane
// (g = lane & 7, c = lane >> 3) packs keys 4g..4g+3 of columns c, c+4, c+8, c+12 and stores 8 bytes per plane — 8 store
// instructions per lane and chunk instead of 32 two-byte ones.
constexpr int VT_LD = 17;
template <int NPL>
__device__ __forceinline__ void store_vt_staged(plane_t* __restrict__ dst_g /* this lane's key group, column 0 of the chunk */, int64_t t_pad,
                                                int64_t plane, const float (&x)[16], float* stage, int lane) {
  float* srow = stage + lane * VT_LD;
#pragma unroll
  for (int j = 0; j < 16; ++j) srow[j] = x[j];
  __syncwarp();
  const int g = lane & 7, c = lane >> 3;
  const float* sp = stage + (4 * g) * VT_LD + c;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float k0 = sp[4 * i], k1 = sp[4 * i + VT_LD], k2 = sp[4 * i + 2 * VT_LD], k3 = sp[4 * i + 3 * VT_LD];
    plane_t* d = dst_g + (int64_t)(c + 4 * i) * t_pad;
#pragma unroll
    for (int pl = 0; pl < NPL; ++pl) {
      uint2 pk;
      pk.x = pack_planes2(k0, k1);
      pk.y = pack_planes2(k2, k3);
      *reinterpret_cast<uint2*>(d) = pk;
      if (pl + 1 < NPL) {
        d += plane;
        const float2 a = unpack_planes2(pk.x), b = unpack_planes2(pk.y);
        k0 -= a.x; k1 -= a.y; k2 -= b.x; k3 -= b.y;
      }
    }
  }
  __syncwarp();
}

// EPI selects the output kind at compile time so the inner loops carry no runtime branching on it:
//   EPI_F32    fp32 rows (+ bias, ReLU, up to two residuals; ragged N tail supported)
//   EPI_PLANES fp16 planes for a following GEMM (+ bias, ReLU)
//   EPI_ATT    attention operands: scaled q planes / k planes / per-head transposed v planes (+ fp32 v for FSMN)
//   EPI_F32R2  EPI_F32 with TWO residuals (only reachable through the C ABI; its interior path keeps the one-chunk-ahead pipeline of
//              both residual streams in a kernel instantiation of its own, so the common one-residual kernel can spend those
//              registers on a deeper ring)
constexpr int EPI_F32 = 0, EPI_PLANES = 1, EPI_ATT = 2, EPI_F32R2 = 3;

// fp32-output interior tiles with two residuals: the residual rows do not depend on the accumulator, so their loads are software
// pipelined one chunk ahead (out-projection / FFN-w_2 epilogues are bound by memory-level parallelism).
template <int BN>
__device__ __forceinline__ void epilogue_fast_f32(const TcParams& p, const float (&d)[2][BN / 2], int64_t row0, int tile_col0, float* stage,
                                                  int lane) {
  const int rr0 = lane >> 2, c4 = (lane & 3) * 4;
  const int64_t rfirst = row0 + rr0;
  const float* sp = stage + rr0 * EPI_LD + c4;
  float* c_row = p.C + rfirst * p.ldc + c4 + tile_col0;
  const float* r1_row = p.r1 ? p.r1 + rfirst * p.ldr1 + c4 + tile_col0 : nullptr;
  const float* r2_row = p.r2 ? p.r2 + rfirst * p.ldr2 + c4 + tile_col0 : nullptr;
  const int64_t sc = 8 * p.ldc, s1 = 8 * p.ldr1, s2 = 8 * p.ldr2;
  const bool c_vec = (p.ldc & 3) == 0;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 nv1[4], nv2[4];
  auto prefetch = [&](int c0) {
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      nv1[it] = r1_row ? __ldg(reinterpret_cast<const float4*>(r1_row + c0 + it * s1)) : z4;
      nv2[it] = r2_row ? __ldg(reinterpret_cast<const float4*>(r2_row + c0 + it * s2)) : z4;
    }
  };
  prefetch(0);
#pragma unroll
  for (int c0 = 0; c0 < BN; c0 += EPI_CH) {
    float4 rv1[4], rv2[4];
#pragma unroll
    for (int it = 0; it < 4; ++it) { rv1[it] = nv1[it]; rv2[it] = nv2[it]; }
    if (c0 + EPI_CH < BN) prefetch(c0 + EPI_CH);
    acc_chunk_to_stage<BN>(d, c0, stage, lane);
    __syncwarp();
    float4 bias4 = z4;
    if (p.bias) bias4 = __ldg(reinterpret_cast<const float4*>(p.bias + tile_col0 + c0 + c4));
    float* pc = c_row + c0;
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const float4 acc = *reinterpret_cast<const float4*>(sp + it * 8 * EPI_LD);
      float v0 = fmaf(acc.x, p.acc_scale, bias4.x), v1 = fmaf(acc.y, p.acc_scale, bias4.y), v2 = fmaf(acc.z, p.acc_scale, bias4.z), v3 = fmaf(acc.w, p.acc_scale, bias4.w);
      if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
      v0 += rv1[it].x; v1 += rv1[it].y; v2 += rv1[it].z; v3 += rv1[it].w;
      v0 += rv2[it].x; v1 += rv2[it].y; v2 += rv2[it].z; v3 += rv2[it].w;
      if (c_vec) *reinterpret_cast<float4*>(pc) = make_float4(v0, v1, v2, v3);
      else { pc[0] = v0; pc[1] = v1; pc[2] = v2; pc[3] = v3; }
      pc += sc;
    }
    __syncwarp();
  }
}

// The same for at most ONE residual (every fp32-output GEMM of the model: out-projection + x, FFN w_2 + x): the registers the second
// residual's pipeline would hold become a RING-deep ring of the first's, so each warp keeps RING 16-column chunks of residual rows
// in flight instead of one.
template <int BN>
__device__ __forceinline__ void epilogue_fast_f32_r1(const TcParams& p, const float (&d)[2][BN / 2], int64_t row0, int tile_col0, float* stage,
                                                     int lane) {
  const int rr0 = lane >> 2, c4 = (lane & 3) * 4;
  const int64_t rfirst = row0 + rr0;
  const float* sp = stage + rr0 * EPI_LD + c4;
  float* c_row = p.C + rfirst * p.ldc + c4 + tile_col0;
  const float* r_row = p.r1 ? p.r1 + rfirst * p.ldr1 + c4 + tile_col0 : nullptr;
  const int64_t sc = 8 * p.ldc, s1 = 8 * p.ldr1;
  const bool c_vec = (p.ldc & 3) == 0;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  constexpr int RING = 4;
  constexpr int NCH = BN / EPI_CH;
  float4 ring[RING][4];
  auto fetch = [&](float4 (&dst)[4], int c0) {
#pragma unroll
    for (int it = 0; it < 4; ++it) dst[it] = r_row ? __ldg(reinterpret_cast<const float4*>(r_row + c0 + it * s1)) : z4;
  };
#pragma unroll
  for (int i = 0; i < RING && i < NCH; ++i) fetch(ring[i], EPI_CH * i);
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c0 = EPI_CH * i;
    acc_chunk_to_stage<BN>(d, c0, stage, lane);
    __syncwarp();
    float4 bias4 = z4;
    if (p.bias) bias4 = __ldg(reinterpret_cast<const float4*>(p.bias + tile_col0 + c0 + c4));
    float* pc = c_row + c0;
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const float4 acc = *reinterpret_cast<const float4*>(sp + it * 8 * EPI_LD);
      const float4 rv = ring[i % RING][it];
      float v0 = fmaf(acc.x, p.acc_scale, bias4.x), v1 = fmaf(acc.y, p.acc_scale, bias4.y), v2 = fmaf(acc.z, p.acc_scale, bias4.z), v3 = fmaf(acc.w, p.acc_scale, bias4.w);
      if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
      v0 += rv.x; v1 += rv.y; v2 += rv.z; v3 += rv.w;
      if (c_vec) *reinterpret_cast<float4*>(pc) = make_float4(v0, v1, v2, v3);
      else { pc[0] = v0; pc[1] = v1; pc[2] = v2; pc[3] = v3; }
      pc += sc;
    }
    __syncwarp();
    if (i + RING < NCH) fetch(ring[i % RING], c0 + EPI_CH * RING);
  }
}

// Interior tiles (all 32 rows and all BN columns in range): straight-line code, no bounds predicates, every row base
// computed once per tile and advanced by constant strides.
template <int BN, int EPI, int NPL>
__device__ __forceinline__ void epilogue_fast(const TcParams& p, const float (&d)[2][BN / 2], int64_t row0, int tile_col0, float* stage, int lane) {
  const AttnSinks& a = p.att;
  constexpr int QPL = NPL < 2 ? NPL : 2;             // attention operands carry at most two planes
  const int rr0 = lane >> 2, c4 = (lane & 3) * 4;
  const int64_t rfirst = row0 + rr0;
  float* srow = stage + lane * EPI_LD;
  const float* sp = stage + rr0 * EPI_LD + c4;
  float* c_row = (EPI != EPI_PLANES && p.C) ? p.C + rfirst * p.ldc + c4 : nullptr;
  plane_t* o_row = EPI == EPI_PLANES ? p.out_planes + rfirst * p.ldo + c4 : nullptr;
  plane_t* q_row = EPI == EPI_ATT ? a.q_planes + rfirst * a.width + c4 : nullptr;
  plane_t* k_row = EPI == EPI_ATT ? a.k_planes + rfirst * a.width + c4 : nullptr;
  const int64_t sc = 8 * p.ldc, so = 8 * p.ldo, sq = 8 * (int64_t)a.width;
  const int64_t plane_o = p.M * p.ldo, plane_q = p.M * (int64_t)a.width;
  const bool c_vec = (p.ldc & 3) == 0;
  plane_t* vt_row = nullptr;
  plane_t* vt_grp = nullptr;                          // staged path: this lane's group of four keys (rows row0 + 4 (lane & 7) ..)
  int64_t vt_plane = 0;
  const bool vt_staged = EPI == EPI_ATT && (a.t_rows & 3) == 0 && (a.t_pad & 3) == 0 && (reinterpret_cast<uintptr_t>(a.vt_planes) & 7) == 0;
  if (EPI == EPI_ATT) {
    const int64_t rw = row0 + lane;
    const int b2 = (int)(rw / a.t_rows), t2 = (int)(rw - (int64_t)b2 * a.t_rows);
    vt_row = a.vt_planes + (int64_t)b2 * a.width * a.t_pad + t2;
    vt_plane = (p.M / a.t_rows) * (int64_t)a.width * a.t_pad;
    const int64_t rg = row0 + 4 * (lane & 7);
    const int bg = (int)(rg / a.t_rows), tg = (int)(rg - (int64_t)bg * a.t_rows);
    vt_grp = a.vt_planes + (int64_t)bg * a.width * a.t_pad + tg;
  }
#pragma unroll
  for (int c0 = 0; c0 < BN; c0 += EPI_CH) {
    const int col0 = tile_col0 + c0;
    const bool v_sink = EPI == EPI_ATT && col0 >= a.v0 && col0 < a.v0 + a.width;
    acc_chunk_to_stage<BN>(d, c0, stage, lane);
    __syncwarp();
    if (EPI == EPI_ATT && v_sink) {
      uint32_t r[16];
      acc_ld_32x16(srow, r);
      if (vt_staged) {
        float x[16];
#pragma unroll
        for (int j = 0; j < 16; j += 4) {
          float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
          if (p.bias) b4 = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + j));      // same address in every lane: one broadcast
          x[j] = fmaf(__uint_as_float(r[j]), p.acc_scale, b4.x); x[j + 1] = fmaf(__uint_as_float(r[j + 1]), p.acc_scale, b4.y);
          x[j + 2] = fmaf(__uint_as_float(r[j + 2]), p.acc_scale, b4.z); x[j + 3] = fmaf(__uint_as_float(r[j + 3]), p.acc_scale, b4.w);
        }
        __syncwarp();                                  // every lane has its row: the transpose may overwrite the stage
        store_vt_staged<QPL>(vt_grp + (int64_t)(col0 - a.v0) * a.t_pad, a.t_pad, vt_plane, x, stage, lane);   // ends with __syncwarp
        if (c_row) {
#pragma unroll
          for (int j = 0; j < 16; j += 4) *reinterpret_cast<uint4*>(srow + j) = make_uint4(r[j], r[j + 1], r[j + 2], r[j + 3]);
          __syncwarp();
        }
      } else {
        store_vt16<QPL>(vt_row + (int64_t)(col0 - a.v0) * a.t_pad, a.t_pad, vt_plane, r, p.bias ? p.bias + col0 : nullptr, p.acc_scale);
      }
    }
    float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.bias) bias4 = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + c4));
    if (EPI == EPI_PLANES) {
      plane_t* po = o_row + col0;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const float4 acc = *reinterpret_cast<const float4*>(sp + it * 8 * EPI_LD);
        float v0 = fmaf(acc.x, p.acc_scale, bias4.x), v1 = fmaf(acc.y, p.acc_scale, bias4.y), v2 = fmaf(acc.z, p.acc_scale, bias4.z), v3 = fmaf(acc.w, p.acc_scale, bias4.w);
        if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
        store_planes4<NPL>(po, plane_o, v0, v1, v2, v3);
        po += so;
      }
    } else {
      const bool q_sink = col0 >= a.q0 && col0 < a.q0 + a.width;
      const bool k_sink = col0 >= a.k0 && col0 < a.k0 + a.width;
      if (q_sink || k_sink) {
        plane_t* pq = q_sink ? q_row + (col0 - a.q0) : k_row + (col0 - a.k0);
        const float qs = q_sink ? a.qscale : 1.0f;
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const float4 acc = *reinterpret_cast<const float4*>(sp + it * 8 * EPI_LD);
          store_planes4<QPL>(pq, plane_q, __fmul_rn(fmaf(acc.x, p.acc_scale, bias4.x), qs), __fmul_rn(fmaf(acc.y, p.acc_scale, bias4.y), qs),
                             __fmul_rn(fmaf(acc.z, p.acc_scale, bias4.z), qs), __fmul_rn(fmaf(acc.w, p.acc_scale, bias4.w), qs));
          pq += sq;
        }
      } else if (v_sink && c_row) {                    // fp32 V rows feed the FSMN memory block
        float* pc = c_row + col0;
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const float4 acc = *reinterpret_cast<const float4*>(sp + it * 8 * EPI_LD);
          const float4 o = make_float4(fmaf(acc.x, p.acc_scale, bias4.x), fmaf(acc.y, p.acc_scale, bias4.y), fmaf(acc.z, p.acc_scale, bias4.z),
                                       fmaf(acc.w, p.acc_scale, bias4.w));
          if (c_vec) *reinterpret_cast<float4*>(pc) = o;
          else { pc[0] = o.x; pc[1] = o.y; pc[2] = o.z; pc[3] = o.w; }
          pc += sc;
        }
      }
    }
    __syncwarp();
  }
}

// Edge tiles (row tail of M, ragged N such as vocab 8404 / 25055): one staged 16-column chunk, every access bounds checked.
// Out of line: edge tiles are rare, and the call keeps the interior paths' code compact.
template <int EPI, int NPL>
__device__ __noinline__ void epilogue_edge_chunk(const TcParams& p, int64_t row0, int col0, float* stage, int lane) {
  const AttnSinks& a = p.att;
  constexpr int QPL = NPL < 2 ? NPL : 2;
  if (EPI == EPI_ATT && col0 >= a.v0 && col0 < a.v0 + a.width && row0 + lane < p.M) {
    uint32_t r[16];
    acc_ld_32x16(stage + lane * EPI_LD, r);
    const int64_t rw = row0 + lane;
    const int b2 = (int)(rw / a.t_rows), t2 = (int)(rw - (int64_t)b2 * a.t_rows);
    store_vt16<QPL>(a.vt_planes + ((int64_t)b2 * a.width + (col0 - a.v0)) * a.t_pad + t2, a.t_pad,
                    (p.M / a.t_rows) * (int64_t)a.width * a.t_pad, r, p.bias ? p.bias + col0 : nullptr, p.acc_scale);
  }
  if (col0 < p.N && row0 < p.M) {
    const bool full = col0 + EPI_CH <= p.N;
    const bool v_sink = EPI == EPI_ATT && col0 >= a.v0 && col0 < a.v0 + a.width;
    const bool q_sink = EPI == EPI_ATT && col0 >= a.q0 && col0 < a.q0 + a.width;
    const bool k_sink = EPI == EPI_ATT && col0 >= a.k0 && col0 < a.k0 + a.width;
    const bool want_c = EPI == EPI_F32 ? true : (EPI == EPI_ATT ? (p.C != nullptr && v_sink) : false);
    if (EPI != EPI_ATT || want_c || q_sink || k_sink) {
      const int rr0 = lane >> 2, c4 = (lane & 3) * 4;
      const int col = col0 + c4;
      const int64_t rfirst = row0 + rr0;
      const int rows_left = (int)((p.M - rfirst + 7) >> 3);        // passes (of 8 rows) with a valid row for this lane
      float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p.bias) {
        if (full) bias4 = __ldg(reinterpret_cast<const float4*>(p.bias + col));
        else { float* bp = reinterpret_cast<float*>(&bias4); for (int e = 0; e < 4; ++e) if (col + e < p.N) bp[e] = __ldg(p.bias + col + e); }
      }
      const float* sp = stage + rr0 * EPI_LD + c4;
      const bool c_vec = (p.ldc & 3) == 0;
      for (int it = 0; it < 4 && it < rows_left; ++it) {
        const int64_t row = rfirst + 8 * it;
        const float4 acc = *reinterpret_cast<const float4*>(sp + it * 8 * EPI_LD);
        float vv[4] = {fmaf(acc.x, p.acc_scale, bias4.x), fmaf(acc.y, p.acc_scale, bias4.y), fmaf(acc.z, p.acc_scale, bias4.z), fmaf(acc.w, p.acc_scale, bias4.w)};
        if (p.relu) { for (int e = 0; e < 4; ++e) vv[e] = fmaxf(vv[e], 0.f); }
        if (full) {
          if (EPI == EPI_F32) {
            for (int e = 0; e < 4; ++e) {
              if (p.r1) vv[e] += __ldg(p.r1 + row * p.ldr1 + col + e);
              if (p.r2) vv[e] += __ldg(p.r2 + row * p.ldr2 + col + e);
            }
          }
          if (want_c) {
            float* pc = p.C + row * p.ldc + col;
            if (c_vec) *reinterpret_cast<float4*>(pc) = make_float4(vv[0], vv[1], vv[2], vv[3]);
            else { pc[0] = vv[0]; pc[1] = vv[1]; pc[2] = vv[2]; pc[3] = vv[3]; }
          }
          if (EPI == EPI_PLANES) store_planes4<NPL>(p.out_planes + row * p.ldo + col, p.M * p.ldo, vv[0], vv[1], vv[2], vv[3]);
          if (q_sink) store_planes4<QPL>(a.q_planes + row * a.width + (col - a.q0), p.M * (int64_t)a.width, __fmul_rn(vv[0], a.qscale),
                                         __fmul_rn(vv[1], a.qscale), __fmul_rn(vv[2], a.qscale), __fmul_rn(vv[3], a.qscale));
          if (k_sink) store_planes4<QPL>(a.k_planes + row * a.width + (col - a.k0), p.M * (int64_t)a.width, vv[0], vv[1], vv[2], vv[3]);
        } else {                                                   // ragged N tail: scalar (fp32 output only)
          for (int e = 0; e < 4; ++e) {
            if (col + e >= p.N) break;
            float x = vv[e];
            if (p.r1) x += __ldg(p.r1 + row * p.ldr1 + col + e);
            if (p.r2) x += __ldg(p.r2 + row * p.ldr2 + col + e);
            if (want_c) p.C[row * p.ldc + col + e] = x;
          }
        }
      }
    }
  }
}

// row0: the warp's first row (32 rows per warp); tile_col0: the tile's first column
template <int BN, int EPI, int NPL>
__device__ __forceinline__ void epilogue_warp(const TcParams& p, const float (&d)[2][BN / 2], int64_t row0, int tile_col0, float* stage, int lane) {
  constexpr int EPIB = EPI == EPI_F32R2 ? EPI_F32 : EPI;
  const bool interior = row0 + 32 <= p.M && tile_col0 + BN <= p.N;
  if (!interior) {
#pragma unroll
    for (int c0 = 0; c0 < BN; c0 += EPI_CH) {
      acc_chunk_to_stage<BN>(d, c0, stage, lane);
      __syncwarp();
      epilogue_edge_chunk<EPIB, NPL>(p, row0, tile_col0 + c0, stage, lane);
      __syncwarp();
    }
  } else if constexpr (EPI == EPI_F32) {
    epilogue_fast_f32_r1<BN>(p, d, row0, tile_col0, stage, lane);
  } else if constexpr (EPI == EPI_F32R2) {
    epilogue_fast_f32<BN>(p, d, row0, tile_col0, stage, lane);
  } else {
    epilogue_fast<BN, EPI, NPL>(p, d, row0, tile_col0, stage, lane);
  }
}

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  if constexpr (BN == 128) wgmma_m64n128_ss(d, a_desc, b_desc, accumulate);
  else wgmma_m64n64_ss(d, a_desc, b_desc, accumulate);
}

// Tile order and hand-offs.  The CTA's tiles are j = 0 .. T-1 (tile blockIdx.x + j gridDim.x); consumer warpgroup c takes
// j = c, c + 2, ..; the producer loads every tile's k-blocks in j order, so the ring slot of (j, kb) is (j k_blocks + kb) % STAGES.
// Ordering barrier ORDER_BAR + c ("c may issue"): before tile j > 0 its consumer waits on it (bar.sync), after issuing tile j's MMAs
// its consumer signals the other's (bar.arrive) only if tile j + 1 exists.  So every wait is matched by exactly one signal and no
// signal is left unmatched, for any T >= 1 (T = 1: consumer 1 has no tile and never touches the barriers; odd T: consumer 0's
// last tile signals nothing).  A barrier cannot be signalled twice before it is waited on: the two consumers strictly alternate.
template <int BN, int STAGES, int APL, int WPL, int EPI>  // APL / WPL: A / W planes resident per stage
__global__ void __launch_bounds__(384, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, const __grid_constant__ TcParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  constexpr uint32_t TILE_W_BYTES = BN * TC_BK * 2;
  constexpr uint32_t STAGE_BYTES = APL * TC_TILE_BYTES_A + WPL * TILE_W_BYTES;
  // align to 1024 B WITHOUT leaving the shared address space (a uintptr_t round trip makes every access a generic LD/ST)
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* epi_stage = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);          // 8 x [32][20] floats
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(epi_stage + EPI_WARPS * EPI_WARP_FLOATS);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = p.tiles_m * p.tiles_n;
  const int k_blocks = p.Kp / TC_BK;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_w);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }   // emptied by the 4 warps of one consumer
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (warp == 0 && elect_one_sync()) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int tm = tile / p.tiles_n, tn = tile - tm * p.tiles_n;
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          unsigned char* st = smem + stage * STAGE_BYTES;
#pragma unroll
          for (int pl = 0; pl < APL; ++pl)
            tma_load_2d(st + pl * TC_TILE_BYTES_A, &map_a, &full_bar[stage], kb * TC_BK, (int)(pl * p.a_plane_rows + (int64_t)tm * TC_BM));
#pragma unroll
          for (int pl = 0; pl < WPL; ++pl)
            tma_load_2d(st + APL * TC_TILE_BYTES_A + pl * TILE_W_BYTES, &map_w, &full_bar[stage], kb * TC_BK, pl * p.w_plane_rows + tn * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup cw owns tiles j = cw, cw + 2, ..; warp q drains rows [32 q, +32) =====================
    setmaxnreg_inc<TC_CONSUMER_REGS>();
    const int cw = (warp >> 2) - 1, q = warp & 3;
    const int n_local = (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1;     // grid <= n_tiles: every CTA has a tile
    float* stage_w = epi_stage + (warp - 4) * EPI_WARP_FLOATS;
    for (int j = cw; j < n_local; j += 2) {
      const int tile = blockIdx.x + j * gridDim.x;
      const int tm = tile / p.tiles_n, tn = tile - tm * p.tiles_n;
      const int it0 = j * k_blocks;
      int stage = it0 % STAGES; uint32_t phase = (uint32_t)(it0 / STAGES) & 1u;
      float d[2][BN / 2];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) d[h][i] = 0.f;
      if (j > 0) named_bar(TC_ORDER_BAR + cw, 256);    // the other consumer has issued tile j - 1
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t st = smem_u32(smem + stage * STAGE_BYTES);
        wgmma_fence();
        for (int t = 0; t < p.n_terms; ++t) {
          const uint64_t da = make_sw128_desc(st + c_term_a[t] * TC_TILE_BYTES_A, 2048);    // 8-row groups 0, 2, ..; + 64 (1024 B): 1, 3, ..
          const uint64_t dw = make_sw128_desc(st + APL * TC_TILE_BYTES_A + c_term_w[t] * TILE_W_BYTES);
#pragma unroll
          for (int k = 0; k < TC_BK / TC_UK; ++k) {
            const uint32_t acc = (kb | t | k) != 0 ? 1u : 0u;
            wgmma_tile<BN>(d[0], da + 2 * k, dw + 2 * k, acc);
            wgmma_tile<BN>(d[1], da + 64 + 2 * k, dw + 2 * k, acc);
          }
        }
        wgmma_commit();
        wgmma_wait_pending1();                         // the previous k-block's MMAs have retired: its ring slot is free
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if (j + 1 < n_local) named_bar_arrive(TC_ORDER_BAR + (cw ^ 1), 256);   // tile j + 1 may queue its MMAs behind this tile's last k-block
      wgmma_wait_all();
      wgmma_fence_regs(d[0]);
      wgmma_fence_regs(d[1]);
      if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
      epilogue_warp<BN, EPI, APL>(p, d, (int64_t)tm * TC_BM + q * 32, tn * BN, stage_w, lane);
    }
  }
}

// fp32 rows [rows, cols] (ld) -> fp16 planes [nplanes][rows][cols_pad]; 4 elements per thread.
__global__ void __launch_bounds__(256)
split_rows_kernel(const float* __restrict__ src, int64_t ld, int64_t rows, int cols, int cols_pad, int nplanes,
                  plane_t* __restrict__ planes) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int c4n = cols_pad >> 2;
  const int64_t total = rows * c4n;
  if (i >= total) return;
  const int64_t r = i / c4n;
  const int c = (int)(i - r * c4n) * 4;
  float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c + 3 < cols) x = __ldg(reinterpret_cast<const float4*>(src + r * ld + c));
  else {
    float* e = reinterpret_cast<float*>(&x);
    for (int k = 0; k < 4; ++k) if (c + k < cols) e[k] = __ldg(src + r * ld + c + k);
  }
  float v[4] = {x.x, x.y, x.z, x.w};
  const int64_t plane = rows * cols_pad;
  for (int pl = 0; pl < nplanes; ++pl) {
    uint2 pk;
    pk.x = pack_planes2(v[0], v[1]);
    pk.y = pack_planes2(v[2], v[3]);
    *reinterpret_cast<uint2*>(planes + pl * plane + r * cols_pad + c) = pk;
    const float2 a = unpack_planes2(pk.x), b = unpack_planes2(pk.y);
    v[0] -= a.x; v[1] -= a.y; v[2] -= b.x; v[3] -= b.y;
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static const PFN_encodeTiled fn = []() -> PFN_encodeTiled {       // thread-safe one-time lookup
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      return reinterpret_cast<PFN_encodeTiled>(p);
    return nullptr;
  }();
  return fn;
}

// 2D fp16 tensor [rows, cols] (row pitch ld elements), box {64 cols, box_rows}, 128B swizzle.
// A forward pass encodes ~570 maps over a few dozen distinct (pointer, shape) pairs — the workspace slices and the weight
// planes are the same every layer and every step — so the encoded descriptors are kept in a small per-thread cache
// (no locking; a descriptor depends only on the key).
struct MapKey {
  const void* base; uint64_t rows, cols, ld; uint32_t box;
  bool operator==(const MapKey& o) const { return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && box == o.box; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    uint64_t h = (uint64_t)(uintptr_t)k.base * 0x9E3779B97F4A7C15ull;
    h ^= (k.rows + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    h ^= (k.cols * 31 + k.ld * 131 + k.box + (h << 6) + (h >> 2));
    return (size_t)h;
  }
};
int make_plane_map(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  static thread_local std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  const MapKey key{base, rows, cols, ld, box_rows};
  auto it = cache.find(key);
  if (it != cache.end()) { *m = it->second; return FA_OK; }
  PFN_encodeTiled enc = get_encode();
  if (!enc) return FA_ERR_CUDA;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)TC_BK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return FA_ERR_CUDA;
  if (cache.size() >= 4096) cache.clear();
  cache.emplace(key, *m);
  return FA_OK;
}

// gemm_rows' scratch: the fp16 planes of the fp32 A operand (none on the fp32 SIMT path, which takes no scratch)
static plane_t* gemm_carve(Arena& a, int64_t rows, int k_pad, int mode) {
  return mode == FA_GEMM_F32_SIMT ? nullptr : a.take<plane_t>((size_t)gemm_planes(mode) * rows * k_pad);
}

size_t gemm_tc_scratch_bytes(int64_t max_rows, int max_k, int mode) {
  Arena m = Arena::measuring();
  gemm_carve(m, max_rows, (max_k + 63) / 64 * 64, mode);
  return m.bytes();
}

template <int BN, int STAGES, int APL, int WPL, int EPI>
static int launch_cfg_e(const CUtensorMap& ma, const CUtensorMap& mw, const TcParams& p, cudaStream_t st) {
  constexpr size_t smem = (size_t)STAGES * (APL * TC_TILE_BYTES_A + WPL * BN * TC_BK * 2) + 1024 + EPI_WARPS * EPI_WARP_FLOATS * 4 +
                          2 * STAGES * 8;
  static_assert(smem <= 227 * 1024, "shared memory per block");
  static PerDeviceOnce once;
  FA_RETURN_IF_ERR(ensure_dyn_smem(gemm_tc_kernel<BN, STAGES, APL, WPL, EPI>, smem, once));
  const int n_sm = sm_count();
  const int tiles = p.tiles_m * p.tiles_n;
  const int grid = tiles < n_sm ? tiles : n_sm;
  gemm_tc_kernel<BN, STAGES, APL, WPL, EPI><<<grid, 384, smem, st>>>(ma, mw, p);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

static inline int epi_kind(const TcParams& p) { return p.att.enabled ? EPI_ATT : (p.out_planes ? EPI_PLANES : (p.r2 ? EPI_F32R2 : EPI_F32)); }

template <int BN, int STAGES, int APL, int WPL>
static int launch_cfg(const CUtensorMap& ma, const CUtensorMap& mw, const TcParams& p, cudaStream_t st) {
  switch (epi_kind(p)) {
    case EPI_ATT: return launch_cfg_e<BN, STAGES, APL, WPL, EPI_ATT>(ma, mw, p, st);
    case EPI_PLANES: return launch_cfg_e<BN, STAGES, APL, WPL, EPI_PLANES>(ma, mw, p, st);
    case EPI_F32R2: return launch_cfg_e<BN, STAGES, APL, WPL, EPI_F32R2>(ma, mw, p, st);
    default: return launch_cfg_e<BN, STAGES, APL, WPL, EPI_F32>(ma, mw, p, st);
  }
}

// A planes already split: a_planes [npl][M][Kp]
int gemm_tc_planes_launch(const plane_t* a_planes, int64_t M, const FaLinear& lin, const GemmEpi& epi, int mode, cudaStream_t st,
                          int64_t a_ld, int64_t a_plane_rows) {
  if (M <= 0) return FA_OK;
  const uint64_t lda = a_ld > 0 ? (uint64_t)a_ld : (uint64_t)lin.in_pad;          // A row pitch (overlapping view: < K_pad)
  const int64_t apr = a_plane_rows > 0 ? a_plane_rows : M;                         // rows between consecutive A planes
  if (lda & 7) return FA_ERR_UNSUPPORTED;
  if (!lin.w_planes || !a_planes) return FA_ERR_ARG;
  const int N = lin.out_f, Kp = lin.in_pad;
  if (N <= 0) return FA_ERR_ARG;
  if (Kp % TC_BK != 0 || M * 3 > 0x7fffffffLL) return FA_ERR_UNSUPPORTED;
  if (epi.y && (epi.ldy & 3) == 0 && (((uintptr_t)epi.y) & 15)) return FA_ERR_UNSUPPORTED;
  if ((epi.r1 && (epi.ld1 & 3)) || (epi.r2 && (epi.ld2 & 3))) return FA_ERR_UNSUPPORTED;
  // the epilogue reads bias and residual rows as float4 and writes output planes as uint2 (store_planes4)
  if ((lin.b && (((uintptr_t)lin.b) & 15)) || (epi.r1 && (((uintptr_t)epi.r1) & 15)) || (epi.r2 && (((uintptr_t)epi.r2) & 15))) return FA_ERR_UNSUPPORTED;
  if (epi.planes && ((epi.ldp & 3) || (((uintptr_t)epi.planes) & 7))) return FA_ERR_UNSUPPORTED;
  if ((epi.y && epi.ldy < N) || (epi.r1 && epi.ld1 < N) || (epi.r2 && epi.ld2 < N) || (epi.planes && epi.ldp < N)) return FA_ERR_ARG;
  const int npl = gemm_planes(mode);
  // 128 x 128 tiles with a 6 (x1) / 3 (x3) stage ring; 128 x 64 for x6 (three planes per operand: two 72 KB stages, a third does
  // not fit beside the epilogue staging in 227 KB).
  // Ragged N (the vocabulary projections: 8404, 25055): the last column tile's W box reaches past row N of a plane — into the next
  // plane's first rows or, for the last plane, out of the tensor map (zero fill) — so its surplus accumulator columns hold finite
  // garbage that the bounds-checked edge epilogue never stores.
  const int BN = npl == 3 ? 64 : 128;
  CUtensorMap ma, mw;
  const uint64_t a_rows1 = (uint64_t)apr * npl - (lda < (uint64_t)Kp ? ((uint64_t)Kp - lda + lda - 1) / lda : 0);
  FA_RETURN_IF_ERR(make_plane_map(&ma, a_planes, a_rows1, (uint64_t)Kp, lda, TC_BM));
  FA_RETURN_IF_ERR(make_plane_map(&mw, lin.w_planes, (uint64_t)N * 3, (uint64_t)Kp, (uint64_t)Kp, BN));
  TcParams p;
  p.M = M; p.N = N; p.Kp = Kp; p.a_plane_rows = apr; p.w_plane_rows = N;
  p.n_terms = mode == FA_GEMM_F16X1 ? 1 : (mode == FA_GEMM_F16X3 ? 3 : 6);
  p.relu = epi.relu_on; p.bias = lin.b; p.r1 = epi.r1; p.ldr1 = epi.ld1; p.r2 = epi.r2; p.ldr2 = epi.ld2; p.C = epi.y; p.ldc = epi.ldy;
  p.out_planes = epi.planes; p.ldo = epi.ldp; p.out_nplanes = npl;
  p.tiles_m = (int)((M + TC_BM - 1) / TC_BM); p.tiles_n = (N + BN - 1) / BN;
  p.acc_scale = rz_comp_scale(Kp, p.n_terms);
  if (epi.att) { p.att = *epi.att; p.att.enabled = 1; } else { p.att = AttnSinks{}; }
  if (epi.att && (N % 32 != 0 || epi.att->width % 32 != 0 || epi.att->t_rows <= 0 || M % epi.att->t_rows != 0)) return FA_ERR_UNSUPPORTED;
  if (epi.planes && (N % 32 != 0)) return FA_ERR_UNSUPPORTED;
  switch (npl) {
    case 1: return launch_cfg<128, 6, 1, 1>(ma, mw, p, st);
    case 2: return launch_cfg<128, 3, 2, 2>(ma, mw, p, st);
    default: return launch_cfg<64, 2, 3, 3>(ma, mw, p, st);
  }
}

int split_rows_launch(const float* x, int64_t ldx, int64_t rows, int cols, int cols_pad, int nplanes, plane_t* planes,
                      cudaStream_t st) {
  if (rows <= 0) return FA_OK;
  if ((ldx & 3) || (((uintptr_t)x) & 15) || (cols_pad & 3)) return FA_ERR_UNSUPPORTED;
  const int64_t total = rows * (cols_pad / 4);
  split_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, ldx, rows, cols, cols_pad, nplanes, planes);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

int gemm_rows(const float* x, int64_t ldx, int64_t rows, const FaLinear& lin, const GemmEpi& epi, int mode, Arena* scratch, cudaStream_t st) {
  if (!lin.w) return FA_ERR_ARG;
  if (mode == FA_GEMM_F32_SIMT) return gemm_f32_launch(x, ldx, rows, lin.w, lin.out_f, lin.in_f, lin.b, epi, st);
  if (rows <= 0) return FA_OK;
  if (mode != FA_GEMM_F16X1 && mode != FA_GEMM_F16X3 && mode != FA_GEMM_F16X6) return FA_ERR_ARG;
  if (!scratch) return FA_ERR_WORKSPACE;
  Arena local(scratch->base, scratch->cap);   // scratch is reused by every call (stream ordered)
  plane_t* planes = gemm_carve(local, rows, lin.in_pad, mode);
  if (!local.ok()) return FA_ERR_WORKSPACE;
  FA_RETURN_IF_ERR(split_rows_launch(x, ldx, rows, lin.in_f, lin.in_pad, gemm_planes(mode), planes, st));
  return gemm_tc_planes_launch(planes, rows, lin, epi, mode, st);
}

}  // namespace fa
