// wgmma / TMA fused multi-head attention with fp16 operand splitting (sm_90a).
//
// Same contract as attention_f32.cu (sanm/attention.py:288-304 with scores from :324-325; cross-attention :760-794,
// :811-812): ctx = softmax(mask(q d_k^-0.5 . k^T)) v per head, key-padding mask, heads merged.  Score and context
// contractions run on the tensor cores (wgmma) with fp32 accumulation in registers; operands are fp16 planes (hi, lo) of the
// fp32 tensors so that S = Qh.Kh + Qh.Kl + Ql.Kh and O = Ph.Vh + Ph.Vl + Pl.Vh carry ~2^-17 relative error (x3 mode),
// or one plane (x1 mode).  The [B,H,Tq,Tk] score tensor never leaves the SM.
//
// One CTA = 128 queries of one (utterance, head), keys in chunks of 64, two passes over the keys:
//   pass A: S~ = Qh.Kh (one MMA term) -> per-row max m   (softmax is invariant to the choice of m)
//   pass B: S (all terms) -> p = exp(s - m), l += sum p, P planes in registers (the A operand of the next wgmma),
//           O += P.V accumulated in registers with no rescaling; finally O / l -> fp16 planes (A operand of the
//           out-projection GEMM) and/or fp32.
#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"
#include <math.h>
#include <stdlib.h>
#include <vector>

namespace fa {

constexpr int AT_BQ = 128, AT_BKEY = 64, AT_D = 128;
constexpr uint32_t AT_Q_KBLK = AT_BQ * 128;      // 16 KB: 128 rows x 64 fp16
constexpr uint32_t AT_BOX = 8192;                // every K / V box: 64 rows x 128 B
// K/V ring slots: as many as fit next to the Q planes in 227 KB of shared memory
#define AT_NSLOT(npl) ((npl) == 1 ? 8 : 5)

struct AttTcParams {
  int tq, tk, heads, batch;
  float o_scale;                                       // truncation compensation of the P.V accumulation, per k-step (gemm_tc.cu: acc_scale)
  int kv_shared;                                       // 1: every utterance attends over the SAME keys / values (hotword memory): K/V planes hold one batch entry
  const int32_t* kv_index;                             // or: utterance b attends over K/V entry kv_index[b] (AttnShape)
  const int32_t* key_lens;
  int64_t q_plane_rows, k_plane_rows, v_plane_rows;   // rows between planes in the respective 2D maps
  float* ctx; int64_t ldc;                             // fp32 output (or null)
  plane_t* ctx_planes; int64_t ldp; int out_nplanes;   // fp16 planes [npl][B*tq][ldp] (or null)
};

// NPL: operand planes (1 | 2); OPL: context planes written (0 = fp32 context only); HD: head dim, 128 or 80.
// An 80-wide head is read as two 64-dim boxes like a 128-wide one (same 128B swizzle, same descriptors): the score MMAs use only
// the first 16-dim k-step of the second box, and P.V (n = 80) only its first 16 d-rows.  The rest of that box is the neighbouring
// head's columns, or the map's zero fill after the last head.
// One CTA = 128 queries of one (utterance, head), 384 threads: warp 0 is the TMA producer, warps 4-11 are two consumer
// warpgroups of 64 query rows each.  K and V chunks share ONE shared-memory ring, filled in the order the consumers read them
//   pass A: Khi(0) .. Khi(nc-1)          pass B: K(0), V(0), K(1), V(1), ..., K(nc-1), V(nc-1)
// and each slot is released by the eight consumer warps once their MMAs on it have retired.
template <int NPL, int OPL, int HD>
__global__ void __launch_bounds__(384, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                    const __grid_constant__ CUtensorMap map_v, const AttTcParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  constexpr uint32_t Q_BYTES = NPL * 2 * AT_Q_KBLK;       // Q planes, two 64-dim boxes each, read by the score MMAs in place
  constexpr uint32_t SLOT_BYTES = NPL * 2 * AT_BOX;       // one K chunk (NPL planes x 2 d-blocks) or one V chunk (NPL x 2 row halves)
  constexpr int NSLOT = AT_NSLOT(NPL);
  constexpr int NT = NPL == 1 ? 1 : 3;
  // align to 1024 B WITHOUT leaving the shared address space (a uintptr_t round trip makes every access a generic LD/ST)
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* sQ = smem;
  unsigned char* sRing = sQ + Q_BYTES;
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sRing + NSLOT * SLOT_BYTES);
  uint64_t* r_full = q_full + 1;      // [NSLOT]
  uint64_t* r_empty = r_full + NSLOT; // [NSLOT] 8 arrivals: every consumer warp is done with the slot

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AT_BQ, h = blockIdx.y, b = blockIdx.z;

  if (warp == 0 && lane == 0) { tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_k); tma_prefetch_desc(&map_v); }
  if (warp == 1 && lane == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < NSLOT; ++s) { mbar_init(&r_full[s], 1); mbar_init(&r_empty[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  const int klen = min(p.key_lens[b], p.tk);
  const int bkv = p.kv_index ? p.kv_index[b] : p.kv_shared ? 0 : b;
  const int nc = (klen + AT_BKEY - 1) / AT_BKEY;     // key chunks with at least one valid key

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (nc > 0 && elect_one_sync()) {
      mbar_expect_tx(q_full, Q_BYTES);
#pragma unroll
      for (int pl = 0; pl < NPL; ++pl)
#pragma unroll
        for (int kb = 0; kb < 2; ++kb)
          tma_load_2d(sQ + (pl * 2 + kb) * AT_Q_KBLK, &map_q, q_full, h * HD + kb * 64,
                      (int)(pl * p.q_plane_rows + (int64_t)b * p.tq + q0));
      uint32_t n = 0;                                       // ring sequence number
      auto load_chunk = [&](bool is_v, int idx, int nb) {  // nb boxes of 8 KB: box bi = plane bi / 2, half bi % 2
        const uint32_t slot = n % NSLOT;
        mbar_wait(&r_empty[slot], ((n / NSLOT) & 1u) ^ 1u);
        mbar_expect_tx(&r_full[slot], (uint32_t)nb * AT_BOX);
        unsigned char* dst = sRing + slot * SLOT_BYTES;
        for (int bi = 0; bi < nb; ++bi) {
          const int pl = bi >> 1, sub = bi & 1;
          if (is_v) tma_load_2d(dst + bi * AT_BOX, &map_v, &r_full[slot], idx * AT_BKEY, (int)(pl * p.v_plane_rows + ((int64_t)bkv * p.heads + h) * HD + sub * 64));
          else tma_load_2d(dst + bi * AT_BOX, &map_k, &r_full[slot], h * HD + sub * 64, (int)(pl * p.k_plane_rows + (int64_t)bkv * p.tk + idx * AT_BKEY));
        }
        ++n;
      };
      for (int i = 0; i < nc; ++i) load_chunk(false, i, 2);            // pass A: hi plane only
      for (int t = 0; t < nc; ++t) {
        load_chunk(false, t, NPL * 2);
        load_chunk(true, t, NPL * 2);
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: warpgroup wg owns query rows [64 wg, +64) =====================
    // accumulator layout (tc_common.cuh): this thread holds rows r0 and r0 + 8, columns 8 j + cq + {0, 1}
    const int wg = (warp - 4) >> 2;
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
    const int ta[3] = {0, 0, 1}, tb[3] = {0, 1, 0};
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    if (nc > 0) {
      const uint32_t q_addr = smem_u32(sQ) + wg * (64 * 128), ring_addr = smem_u32(sRing);
      uint32_t n = 0;                                       // ring sequence number
      auto acquire = [&]() -> uint32_t {
        const uint32_t slot = n % NSLOT;
        mbar_wait(&r_full[slot], (n / NSLOT) & 1u);
        return ring_addr + slot * SLOT_BYTES;
      };
      auto release = [&]() {                                // after wgmma_wait_all: this warp's MMAs on the slot have retired
        __syncwarp();
        if (lane == 0) mbar_arrive(&r_empty[n % NSLOT]);
        ++n;
      };
      // S[64 x 64] = sum over the first nterm terms of Q plane ta . K plane tb^T
      auto scores = [&](float (&s)[32], uint32_t k_addr, int nterm) {
        wgmma_fence();
        for (int term = 0; term < nterm; ++term) {
#pragma unroll
          for (int k = 0; k < HD / 16; ++k) {
            const uint64_t da = make_sw128_desc(q_addr + (ta[term] * 2 + (k >> 2)) * AT_Q_KBLK) + 2 * (k & 3);
            const uint64_t db = make_sw128_desc(k_addr + (tb[term] * 2 + (k >> 2)) * AT_BOX) + 2 * (k & 3);
            wgmma_m64n64_ss(s, da, db, (term | k) != 0 ? 1u : 0u);
          }
        }
        wgmma_commit();
        wgmma_wait_all();
        wgmma_fence_regs(s);
      };
      mbar_wait(q_full, 0);
      // ---- pass A: approximate row max (softmax is invariant to the choice of m; an approximate maximum only has to keep
      //      exp(s - m) in range, so the hi . hi term suffices)
      for (int i = 0; i < nc; ++i) {
        float s[32];
        scores(s, acquire(), 1);
        release();
        const int kbase = i * AT_BKEY + cq;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (kbase + 8 * j + e < klen) { m0 = fmaxf(m0, s[4 * j + e]); m1 = fmaxf(m1, s[4 * j + 2 + e]); }
      }
#pragma unroll
      for (int o2 = 1; o2 <= 2; o2 <<= 1) {                 // the four lanes of a quad share a row
        m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o2));
        m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o2));
      }
      // probabilities are formed as p' = 2^10 exp(s - m): the common factor cancels in O / l, and it keeps probabilities down to
      // 6e-8 inside the fp16 planes' NORMAL range (p' <= ~1100 with the approximate maximum of pass A; fp16 holds 65504)
      const float mp0 = m0 - 6.931471805599453f, mp1 = m1 - 6.931471805599453f;
      // ---- pass B: S (all terms) -> p -> fp16 planes in registers (the A operand of P.V) -> O += P . V
      for (int t = 0; t < nc; ++t) {
        float s[32];
        scores(s, acquire(), NT);
        release();
        uint32_t ph[4][4], plo[4][4];                       // [16-key step][A fragment register]
        const int kbase = t * AT_BKEY + cq;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const bool v0 = kbase + 8 * j < klen, v1 = kbase + 8 * j + 1 < klen;
          const float a = v0 ? __expf(s[4 * j] - mp0) : 0.f, bb = v1 ? __expf(s[4 * j + 1] - mp0) : 0.f;
          const float c = v0 ? __expf(s[4 * j + 2] - mp1) : 0.f, dd = v1 ? __expf(s[4 * j + 3] - mp1) : 0.f;
          l0 += a; l0 += bb; l1 += c; l1 += dd;
          const uint32_t h01 = pack_planes2(a, bb), h23 = pack_planes2(c, dd);
          ph[j >> 1][(j & 1) * 2] = h01;
          ph[j >> 1][(j & 1) * 2 + 1] = h23;
          if (NPL > 1) {
            const float2 u = unpack_planes2(h01), w = unpack_planes2(h23);
            plo[j >> 1][(j & 1) * 2] = pack_planes2(a - u.x, bb - u.y);
            plo[j >> 1][(j & 1) * 2 + 1] = pack_planes2(c - w.x, dd - w.y);
          }
        }
        const uint32_t v_addr = acquire();
        wgmma_fence();
#pragma unroll
        for (int term = 0; term < NT; ++term) {
          const uint64_t db = make_sw128_desc(v_addr + tb[term] * 2 * AT_BOX);
#pragma unroll
          for (int kk = 0; kk < AT_BKEY / 16; ++kk) {
            if constexpr (HD == 128) wgmma_m64n128_rs(o, ta[term] == 0 ? ph[kk] : plo[kk], db + 2 * kk, 1u);
            else wgmma_m64n80_rs(o, ta[term] == 0 ? ph[kk] : plo[kk], db + 2 * kk, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait_all();
        wgmma_fence_regs(o);
        release();
      }
#pragma unroll
      for (int o2 = 1; o2 <= 2; o2 <<= 1) {
        l0 += __shfl_xor_sync(0xffffffffu, l0, o2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, o2);
      }
    }
    // ---- epilogue: O / l -> fp32 context and / or fp16 planes (the A operand of the out-projection GEMM)
    const float comp = 1.0f + (float)(nc * (AT_BKEY / 16)) * p.o_scale;     // nc key chunks x 4 k-steps were accumulated into O
    const float inv0 = l0 > 0.f ? comp / l0 : 0.f, inv1 = l1 > 0.f ? comp / l1 : 0.f;
    const int64_t plane = (int64_t)p.batch * p.tq * p.ldp;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int row = q0 + r0 + 8 * half;
      if (row >= p.tq) continue;
      const int64_t grow = (int64_t)b * p.tq + row;
      const float inv = half ? inv1 : inv0;
#pragma unroll
      for (int j = 0; j < HD / 8; ++j) {
        float x0 = o[4 * j + 2 * half] * inv, x1 = o[4 * j + 2 * half + 1] * inv;
        const int col = h * HD + 8 * j + cq;
        if (p.ctx) *reinterpret_cast<float2*>(p.ctx + grow * p.ldc + col) = make_float2(x0, x1);
        if (OPL > 0) {
          plane_t* dst = p.ctx_planes + grow * p.ldp + col;
#pragma unroll
          for (int pl = 0; pl < OPL; ++pl) {
            const uint32_t pk = pack_planes2(x0, x1);
            *reinterpret_cast<uint32_t*>(dst) = pk;
            if (pl + 1 < OPL) {
              dst += plane;
              const float2 u = unpack_planes2(pk);
              x0 -= u.x; x1 -= u.y;
            }
          }
        }
      }
    }
  }
}

// V [B, tk, ldv] (head h at column h*128) -> Vt planes [npl][B*H*128][tkp] (keys contiguous), via a 64x64 smem transpose.
__global__ void __launch_bounds__(256)
vt_planes_kernel(const float* __restrict__ v, int64_t ldv, int tk, int tkp, int heads, int nplanes, int64_t plane_elems,
                 plane_t* __restrict__ vt) {
  __shared__ float tile[64][65];
  const int t0 = blockIdx.x * 64, dblk = blockIdx.y, b = blockIdx.z;   // dblk over heads*2 (64-wide d blocks)
  const int tid = threadIdx.x;
  for (int idx = tid; idx < 64 * 16; idx += 256) {
    const int tr = idx >> 4, c4 = idx & 15;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t0 + tr < tk) x = __ldg(reinterpret_cast<const float4*>(v + ((int64_t)b * tk + t0 + tr) * ldv + dblk * 64 + 4 * c4));
    tile[tr][4 * c4 + 0] = x.x; tile[tr][4 * c4 + 1] = x.y; tile[tr][4 * c4 + 2] = x.z; tile[tr][4 * c4 + 3] = x.w;
  }
  __syncthreads();
  // each thread writes 2 consecutive keys for one d: 64 d x 32 key-pairs = 2048 items / 256 threads
  for (int idx = tid; idx < 64 * 32; idx += 256) {
    const int d = idx >> 5, kp = (idx & 31) * 2;
    if (t0 + kp >= tkp) continue;
    float a = tile[kp][d], bb = tile[kp + 1][d];
    plane_t* dst = vt + ((int64_t)b * heads * AT_D + dblk * 64 + d) * tkp + t0 + kp;
    for (int pl = 0; pl < nplanes; ++pl) {
      const uint32_t pk = pack_planes2(a, bb);
      *reinterpret_cast<uint32_t*>(dst + pl * plane_elems) = pk;
      const float2 u = unpack_planes2(pk);
      a -= u.x; bb -= u.y;
    }
  }
}

// fp32 [rows, cols] (ld) * scale -> fp16 planes [nplanes][rows][cols]
__global__ void __launch_bounds__(256)
scale_split_kernel(const float* __restrict__ src, int64_t ld, int64_t rows, int cols, float scale, int nplanes,
                   plane_t* __restrict__ planes) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int c4n = cols >> 2;
  if (i >= rows * c4n) return;
  const int64_t r = i / c4n;
  const int c = (int)(i - r * c4n) * 4;
  const float4 x = __ldg(reinterpret_cast<const float4*>(src + r * ld + c));
  float v[4] = {__fmul_rn(x.x, scale), __fmul_rn(x.y, scale), __fmul_rn(x.z, scale), __fmul_rn(x.w, scale)};
  const int64_t plane = rows * cols;
  for (int pl = 0; pl < nplanes; ++pl) {
    uint2 pk;
    pk.x = pack_planes2(v[0], v[1]);
    pk.y = pack_planes2(v[2], v[3]);
    *reinterpret_cast<uint2*>(planes + pl * plane + r * cols + c) = pk;
    const float2 ua = unpack_planes2(pk.x), ub = unpack_planes2(pk.y);
    v[0] -= ua.x; v[1] -= ua.y; v[2] -= ub.x; v[3] -= ub.y;
  }
}

static int key_pitch(int tk) { return (tk + 63) / 64 * 64; }   // the V^T planes' keys, padded to whole 64-key chunks

AttnPlanes attn_carve(Arena& a, int batch, int tq, int kv_batch, int tk, int width, int mode) {
  AttnPlanes p;
  p.npl = attn_planes(mode);
  p.t_pad = key_pitch(tk);
  p.q = a.take<plane_t>((size_t)p.npl * batch * tq * width);
  p.k = a.take<plane_t>((size_t)p.npl * kv_batch * tk * width);
  p.vt = a.take<plane_t>((size_t)p.npl * kv_batch * width * p.t_pad);
  return p;
}

AttnSinks attn_sinks(const AttnPlanes& p, int q0, int k0, int v0, int width, int t_rows, float qscale) {
  AttnSinks s;
  if (q0 >= 0) s.q0 = q0;
  if (k0 >= 0) s.k0 = k0;
  if (v0 >= 0) s.v0 = v0;
  s.width = width; s.npl = p.npl; s.t_rows = t_rows; s.t_pad = p.t_pad; s.qscale = qscale;
  s.q_planes = p.q; s.k_planes = p.k; s.vt_planes = p.vt;
  return s;
}

// attention_rows' scratch in the tensor-core modes: the planes of a 128-wide head over kv_batch K / V entries
size_t attention_tc_scratch_bytes(int batch, int heads, int tq, int kv_batch, int tk, int mode) {
  if (mode == FA_GEMM_F32_SIMT) return 0;
  Arena m = Arena::measuring();
  attn_carve(m, batch, tq, kv_batch, tk, heads * AT_D, mode);
  return m.bytes();
}

// the fp32 mode of attention_rows (attention_f32.cu)
int attention_f32_rows(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, const AttnShape& s,
                       const int32_t* key_lens, const AttnOut& out, cudaStream_t st);

int attention_rows(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, const AttnShape& s,
                   const int32_t* key_lens, const AttnOut& out, int mode, Arena* scratch, cudaStream_t st) {
  if (mode == FA_GEMM_F32_SIMT) return attention_f32_rows(q, ldq, k, ldk, v, ldv, s, key_lens, out, st);
  if (s.head_dim != AT_D) return FA_ERR_UNSUPPORTED;
  if (s.batch <= 0 || s.tq <= 0) return FA_OK;
  if (!q || !k || !v || !key_lens || s.tk <= 0 || !scratch) return FA_ERR_ARG;
  if ((ldq | ldk | ldv) & 3) return FA_ERR_UNSUPPORTED;
  const int d = s.heads * AT_D;
  const int kvb = s.kv_entries();
  const int64_t mq = (int64_t)s.batch * s.tq, mk = (int64_t)kvb * s.tk, mv = (int64_t)kvb * d;
  Arena local(scratch->base, scratch->cap);
  const AttnPlanes p = attn_carve(local, s.batch, s.tq, kvb, s.tk, d, mode);
  if (!local.ok()) return FA_ERR_WORKSPACE;
  const int64_t tot = mq * (d / 4);
  scale_split_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(q, ldq, mq, d, attn_qscale(AT_D), p.npl, p.q);
  FA_CHECK_LAUNCH();
  const int64_t totk = mk * (d / 4);
  scale_split_kernel<<<(unsigned)((totk + 255) / 256), 256, 0, st>>>(k, ldk, mk, d, 1.0f, p.npl, p.k);
  FA_CHECK_LAUNCH();
  dim3 g(p.t_pad / 64, s.heads * 2, kvb);
  vt_planes_kernel<<<g, 256, 0, st>>>(v, ldv, s.tk, p.t_pad, s.heads, p.npl, mv * p.t_pad, p.vt);
  FA_CHECK_LAUNCH();
  return attention_planes(p, s, key_lens, out, st);
}

template <int NPL, int OPL, int HD>
static int launch_att(dim3 grid, const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, const AttTcParams& p, cudaStream_t st) {
  constexpr size_t smem = (size_t)NPL * 2 * AT_Q_KBLK + (size_t)AT_NSLOT(NPL) * NPL * 2 * AT_BOX + 1024 + (1 + 2 * AT_NSLOT(NPL)) * 8;
  static_assert(smem <= 227 * 1024, "shared memory per block");
  static PerDeviceOnce once;
  FA_RETURN_IF_ERR(ensure_dyn_smem(attention_tc_kernel<NPL, OPL, HD>, smem, once));
  attention_tc_kernel<NPL, OPL, HD><<<grid, 384, smem, st>>>(mq, mk, mv, p);
  return FA_OK;
}

template <int HD>
static int launch_att_planes(int npl, int opl, dim3 grid, const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                             const AttTcParams& p, cudaStream_t st) {
  if (npl == 1) {
    if (opl > 1) return FA_ERR_UNSUPPORTED;
    return opl == 0 ? launch_att<1, 0, HD>(grid, mq, mk, mv, p, st) : launch_att<1, 1, HD>(grid, mq, mk, mv, p, st);
  }
  if (opl == 1) return FA_ERR_UNSUPPORTED;
  return opl == 0 ? launch_att<2, 0, HD>(grid, mq, mk, mv, p, st)
         : opl == 2 ? launch_att<2, 2, HD>(grid, mq, mk, mv, p, st)
                    : launch_att<2, 3, HD>(grid, mq, mk, mv, p, st);
}

// Operand planes already in place (written by the producing GEMMs' epilogues, gemm_tc.cu AttnSinks, or by attention_rows)
int attention_planes(const AttnPlanes& pl, const AttnShape& s, const int32_t* key_lens, const AttnOut& out, cudaStream_t st) {
  if (s.head_dim != 128 && s.head_dim != 80) return FA_ERR_UNSUPPORTED;
  if (s.batch <= 0 || s.tq <= 0) return FA_OK;
  if (!pl.q || !pl.k || !pl.vt || !key_lens || s.tk <= 0) return FA_ERR_ARG;
  const int npl = pl.npl;
  const int d = s.heads * s.head_dim;
  const int kvb = s.kv_entries();
  const int64_t mq = (int64_t)s.batch * s.tq, mk = (int64_t)kvb * s.tk, mv = (int64_t)kvb * d;
  CUtensorMap mq_map, mk_map, mv_map;
  FA_RETURN_IF_ERR(make_plane_map(&mq_map, pl.q, (uint64_t)mq * npl, (uint64_t)d, (uint64_t)d, AT_BQ));
  FA_RETURN_IF_ERR(make_plane_map(&mk_map, pl.k, (uint64_t)mk * npl, (uint64_t)d, (uint64_t)d, AT_BKEY));
  FA_RETURN_IF_ERR(make_plane_map(&mv_map, pl.vt, (uint64_t)mv * npl, (uint64_t)s.tk, (uint64_t)pl.t_pad, 64));   // 8 KB boxes: 64 d-rows x 64 keys
  AttTcParams p;
  p.tq = s.tq; p.tk = s.tk; p.heads = s.heads; p.batch = s.batch; p.key_lens = key_lens; p.kv_shared = s.kv_shared ? 1 : 0; p.kv_index = s.kv_index;
  {
    static const bool rz_on = [] { const char* e = getenv("FA_RZ_COMP"); return !(e && e[0] == '0'); }();
    p.o_scale = rz_on ? (npl > 1 ? 5.3e-8f : 3.4e-8f) : 0.f;                                   // relative shrink per 16-key k-step
  }
  p.q_plane_rows = mq; p.k_plane_rows = mk; p.v_plane_rows = mv;
  p.ctx = out.ctx; p.ldc = out.ldc; p.ctx_planes = out.planes; p.ldp = out.ldp; p.out_nplanes = out.nplanes;
  dim3 grid((s.tq + AT_BQ - 1) / AT_BQ, s.heads, s.batch);
  const int opl = out.planes ? out.nplanes : 0;
  if (out.planes && (opl < 1 || opl > 3)) return FA_ERR_ARG;
  FA_RETURN_IF_ERR(s.head_dim == 128 ? launch_att_planes<128>(npl, opl, grid, mq_map, mk_map, mv_map, p, st)
                                      : launch_att_planes<80>(npl, opl, grid, mq_map, mk_map, mv_map, p, st));
  FA_CHECK_LAUNCH();
  return FA_OK;
}

}  // namespace fa


extern "C" size_t fa_attention_tc_workspace_bytes(int32_t batch, int32_t heads, int32_t tq, int32_t tk, int32_t gemm_mode) {
  return fa::attention_tc_scratch_bytes(batch, heads, tq, batch, tk, gemm_mode);
}

extern "C" int fa_attention_tc(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv,
                               const int32_t* key_lens, int32_t batch, int32_t heads, int32_t tq, int32_t tk, float* ctx,
                               int64_t ld_ctx, int32_t gemm_mode, void* workspace, size_t ws_bytes, fa_stream_t stream) {
  if (!ctx || heads * fa::AT_D > 4096 || (ld_ctx & 3)) return FA_ERR_ARG;
  if (gemm_mode == FA_GEMM_F32_SIMT) return FA_ERR_ARG;
  fa::Arena scratch(workspace, ws_bytes);
  return fa::attention_rows(q, ldq, k, ldk, v, ldv, fa::AttnShape{batch, heads, fa::AT_D, tq, tk, 0}, key_lens, fa::AttnOut().to(ctx, ld_ctx),
                            gemm_mode, &scratch, (cudaStream_t)stream);
}

// utterance b over K / V entry kv_index_h[b]: the index in the workspace's first ints, then attention_rows' planes (tensor-core modes)
static fa::Arena attn_grouped_carve(fa::Arena& a, int batch, int heads, int tq, int kv_batch, int tk, int mode, int32_t** idx) {
  *idx = a.take<int32_t>(batch);
  return a.sub(fa::attention_tc_scratch_bytes(batch, heads, tq, kv_batch, tk, mode));
}

extern "C" size_t fa_attention_grouped_workspace_bytes(int32_t batch, int32_t heads, int32_t tq, int32_t kv_batch, int32_t tk, int32_t gemm_mode) {
  if (batch < 1 || heads < 1 || tq < 1 || kv_batch < 1 || tk < 1) return 0;
  fa::Arena m = fa::Arena::measuring();
  int32_t* idx;
  attn_grouped_carve(m, batch, heads, tq, kv_batch, tk, gemm_mode, &idx);
  return m.bytes();
}

extern "C" int fa_attention_grouped(const float* q, int64_t ldq, const float* k, int64_t ldk, const float* v, int64_t ldv, const int32_t* key_lens,
                                    const int32_t* kv_index_h, int32_t kv_batch, int32_t batch, int32_t heads, int32_t head_dim, int32_t tq,
                                    int32_t tk, float* ctx, int64_t ld_ctx, int32_t gemm_mode, void* workspace, size_t ws_bytes,
                                    fa_stream_t stream) {
  if (gemm_mode != FA_GEMM_F32_SIMT && gemm_mode != FA_GEMM_F16X1 && gemm_mode != FA_GEMM_F16X3 && gemm_mode != FA_GEMM_F16X6) return FA_ERR_ARG;
  if (!q || !k || !v || !key_lens || !kv_index_h || !ctx || batch < 1 || heads < 1 || tq < 1 || tk < 1 || kv_batch < 1 || head_dim < 1 ||
      heads * head_dim > 4096 || ld_ctx < heads * head_dim || (ld_ctx & 3))
    return FA_ERR_ARG;
  for (int32_t b = 0; b < batch; ++b)
    if (kv_index_h[b] < 0 || kv_index_h[b] >= kv_batch) return FA_ERR_ARG;
  if (gemm_mode != FA_GEMM_F32_SIMT && head_dim != fa::AT_D) return FA_ERR_UNSUPPORTED;
  fa::Arena a(workspace, ws_bytes);
  int32_t* idx;
  fa::Arena scratch = attn_grouped_carve(a, batch, heads, tq, kv_batch, tk, gemm_mode, &idx);
  if (!a.ok()) return FA_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  // staged through pageable memory of this frame, which the copy has read when it returns: the caller may reuse kv_index_h at once,
  // whatever memory it lives in
  const std::vector<int32_t> staged(kv_index_h, kv_index_h + batch);
  FA_CUDA_OK(cudaMemcpyAsync(idx, staged.data(), (size_t)batch * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  fa::AttnShape s{batch, heads, head_dim, tq, tk, 0};
  s.kv_batch = kv_batch; s.kv_index = idx;
  return fa::attention_rows(q, ldq, k, ldk, v, ldv, s, key_lens, fa::AttnOut().to(ctx, ld_ctx), gemm_mode, &scratch, st);
}

extern "C" int fa_attention_tc_planes_ex(const void* q_planes, const void* k_planes, const void* vt_planes, const int32_t* key_lens,
                                         int32_t batch, int32_t heads, int32_t head_dim, int32_t tq, int32_t tk, float* ctx, int64_t ld_ctx,
                                         void* ctx_planes, int64_t ld_planes, int32_t out_nplanes, int32_t gemm_mode, int32_t kv_shared,
                                         fa_stream_t stream) {
  if (gemm_mode != FA_GEMM_F16X1 && gemm_mode != FA_GEMM_F16X3 && gemm_mode != FA_GEMM_F16X6) return FA_ERR_ARG;
  if (head_dim != 128 && head_dim != 80) return FA_ERR_UNSUPPORTED;
  if (heads < 1 || heads * head_dim > 4096 || (!ctx && !ctx_planes)) return FA_ERR_ARG;
  if (ctx && (ld_ctx < heads * head_dim || (ld_ctx & 3))) return FA_ERR_ARG;          // float2 stores
  if (ctx_planes && (ld_planes < heads * head_dim || (ld_planes & 1))) return FA_ERR_ARG;   // 4-byte stores of two fp16
  auto in = [](const void* p) { return static_cast<fa::plane_t*>(const_cast<void*>(p)); };   // read only
  const fa::AttnPlanes pl{in(q_planes), in(k_planes), in(vt_planes), fa::attn_planes(gemm_mode), fa::key_pitch(tk)};
  return fa::attention_planes(pl, fa::AttnShape{batch, heads, head_dim, tq, tk, kv_shared}, key_lens,
                              fa::AttnOut().to(ctx, ld_ctx).to(static_cast<fa::plane_t*>(ctx_planes), ld_planes, out_nplanes),
                              (cudaStream_t)stream);
}

extern "C" int fa_attention_tc_planes(const void* q_planes, const void* k_planes, const void* vt_planes, const int32_t* key_lens,
                                      int32_t batch, int32_t heads, int32_t tq, int32_t tk, float* ctx, int64_t ld_ctx, void* ctx_planes,
                                      int64_t ld_planes, int32_t out_nplanes, int32_t gemm_mode, int32_t kv_shared, fa_stream_t stream) {
  return fa_attention_tc_planes_ex(q_planes, k_planes, vt_planes, key_lens, batch, heads, fa::AT_D, tq, tk, ctx, ld_ctx, ctx_planes,
                                   ld_planes, out_nplanes, gemm_mode, kv_shared, stream);
}
