// Persistent bidirectional LSTM recurrence (one layer, batch_first, no packing) — the BLSTM of CifPredictorV3's timestamp head
// (funasr/models/bicif_paraformer/cif_predictor.py:187-190, :318-320: `output2, _ = self.blstm(output2)` on the 3x upsampled
// encoder output).  cuDNN needs 34 ms for [64, 1500, 512] in fp32; the recurrence is 1500 strictly sequential steps of a
// [B,512] x [512,2048] product per direction, so the design goal is the shortest possible step:
//   * the input projections x W_ih^T + b_ih + b_hh of ALL steps are one tensor-core GEMM of this library (fa_linear), outside;
//   * weight-stationary recurrence: 2 directions x 64 CTAs, CTA c keeps the 4 gate rows of hidden units [8c, 8c+8) of W_hh in
//     shared memory for the whole sequence;
//   * per step: gather h_{t-1} (published by the 64 CTAs of this direction) -> the recurrent product on tensor cores (below)
//     -> gates, c, h -> write the h slice -> per-direction grid barrier (monotone atomic counter).
// Launched cooperatively so all 128 CTAs are co-resident (the barrier would deadlock otherwise).
#include "common.cuh"
#include <cuda_bf16.h>

namespace fa {

// Hidden sizes H: 512 (Paraformer-large family: 64 CTAs per direction) and 320 (fa-zh MonotonicAligner: 40 CTAs per direction).
constexpr int LS_HMAX = 512;       // largest hidden size: sizes the exchange tensor of fa_blstm_tc_scratch_bytes
constexpr int LS_UNITS = 8;        // hidden units per CTA
constexpr int LS_ROWS = 4 * LS_UNITS;    // 32 gate rows per CTA
constexpr int LS_BT = 64;          // sequences per batch tile (4 warps x 16 sequences)

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// Tensor-core recurrence: the [64 seq] x [32 gate rows] x [H] product of a step
// on warp-level bf16 MMAs (mma.sync.m16n8k16) with the 3-product operand split used everywhere else in this library
// (h = hi + lo, w = hi + lo; hi.hi + hi.lo + lo.hi, fp32 accumulate, ~2^-17 relative per product).  W_hh planes stay in shared
// memory for all steps; every CTA publishes its slice of h_t as bf16 hi / lo planes into a double-buffered exchange tensor that
// the other CTAs copy straight into shared memory (cp.async) in the row pitch ldmatrix wants.  Fragment layout does the rest:
// local gate row n = 8 g + u makes n-tile g of the m16n8 accumulator hold gate g of the CTA's 8 units, so one thread ends up
// with all four gates of its (2 sequences x 2 units) cells.

// bytes per bf16 row in shared memory (1040 at H = 512, 656 at 320): an odd number of 16-byte units, so 16-byte rows of 8 lanes
// hit 8 distinct bank groups
template <int H>
constexpr int lt_pitch() { return H * 2 + 16; }

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// hx: exchange tensor [2 parity][2 dir][2 plane][batch_pad][H] bf16 (batch_pad = tiles * 64).  xproj and out hold t_ld steps per
// sequence.  ext[b] (NULL: T for every sequence) is sequence b's own length: the grid runs T = max(ext) steps in lockstep, sequence b's
// forward direction reads and writes t = step and its backward direction t = ext[b] - 1 - step, both from a zero state, and both stop
// writing at step ext[b] (a sequence past its length computes finite values nobody reads)
template <int H>
__global__ void __launch_bounds__(128, 1)
blstm_tc_kernel(const float* __restrict__ xproj, const float* __restrict__ w_hh_f, const float* __restrict__ w_hh_b, int batch, int T,
                int t_ld, const int32_t* __restrict__ ext, float* __restrict__ out, __nv_bfloat16* __restrict__ hx,
                unsigned int* __restrict__ counters) {
  constexpr int LS_H = H, LS_NC = H / LS_UNITS, LT_PITCH = lt_pitch<H>();
  extern __shared__ __align__(16) unsigned char smb[];
  unsigned char* sWp = smb;                                   // [2 planes][32 rows][LT_PITCH]
  unsigned char* sHp = smb + 2 * LS_ROWS * LT_PITCH;          // [2 planes][64 seq][LT_PITCH]
  const int dir = blockIdx.x / LS_NC, c = blockIdx.x % LS_NC;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* whh = dir == 0 ? w_hh_f : w_hh_b;
  // W_hh slice -> bf16 hi / lo planes, local row n = g*8 + u  <->  row g*512 + 8c + u
  for (int idx = tid; idx < LS_ROWS * (LS_H / 2); idx += blockDim.x) {
    const int r = idx / (LS_H / 2), k2 = idx % (LS_H / 2);
    const int g = r / LS_UNITS, u = r % LS_UNITS;
    const float2 w = __ldg(reinterpret_cast<const float2*>(whh + ((int64_t)g * LS_H + c * LS_UNITS + u) * LS_H) + k2);
    const __nv_bfloat162 h2 = __floats2bfloat162_rn(w.x, w.y);
    const uint32_t hb = *reinterpret_cast<const uint32_t*>(&h2);
    const __nv_bfloat162 l2 = __floats2bfloat162_rn(w.x - __uint_as_float(hb << 16), w.y - __uint_as_float(hb & 0xFFFF0000u));
    *reinterpret_cast<uint32_t*>(sWp + r * LT_PITCH + 4 * k2) = hb;
    *reinterpret_cast<uint32_t*>(sWp + LS_ROWS * LT_PITCH + r * LT_PITCH + 4 * k2) = *reinterpret_cast<const uint32_t*>(&l2);
  }
  const int n_tiles = (batch + LS_BT - 1) / LS_BT;
  const int batch_pad = n_tiles * LS_BT;
  // accumulator ownership (m16n8 D fragment): rows r0 = lane/4 and r0+8 of the warp's 16 sequences, columns 2*(lane%4), +1
  const int r0 = lane >> 2, cu = 2 * (lane & 3);
  float cst[4][2][2];
#pragma unroll
  for (int i = 0; i < 4; ++i) { cst[i][0][0] = cst[i][0][1] = cst[i][1][0] = cst[i][1][1] = 0.f; }
  __syncthreads();
  unsigned int* counter = counters + dir;
  const int64_t out_ld = 2 * LS_H, xp_ld = 2 * 4 * LS_H;
  const uint32_t sW_addr = (uint32_t)__cvta_generic_to_shared(sWp), sH_addr = (uint32_t)__cvta_generic_to_shared(sHp);
  // ldmatrix lane addressing.  A (16 seq x 16 k): matrices (rows 0-7,k 0-7), (rows 8-15,k 0-7), (rows 0-7,k 8-15), (rows 8-15,k 8-15)
  const uint32_t a_lane = (uint32_t)((warp * 16 + (lane & 15)) * LT_PITCH + (lane >> 4) * 16);
  // B (two n-tiles x 16 k per x4): matrices (n 0-7,k 0-7), (n 0-7,k 8-15), (n 8-15,k 0-7), (n 8-15,k 8-15)
  const uint32_t b_lane = (uint32_t)(((lane & 7) + ((lane >> 4) << 3)) * LT_PITCH + ((lane >> 3) & 1) * 16);
  const int64_t plane_stride = (int64_t)batch_pad * LS_H;                 // elements between hi and lo plane
  const int64_t dir_stride = 2 * plane_stride, par_stride = 2 * dir_stride;
  for (int step = 0; step < T; ++step) {
    const __nv_bfloat16* hx_rd = hx + (int64_t)((step + 1) & 1) * par_stride + dir * dir_stride;   // written during step-1
    __nv_bfloat16* hx_wr = hx + (int64_t)(step & 1) * par_stride + dir * dir_stride;
    if (step > 0) {
      if (tid == 0) {
        const unsigned int want = (unsigned int)step * LS_NC;
        while (*reinterpret_cast<volatile unsigned int*>(counter) < want) { }
        __threadfence();
      }
      __syncthreads();
    }
#pragma unroll
    for (int bt = 0; bt < 4; ++bt) {
      if (bt >= n_tiles) break;
      const int b0 = bt * LS_BT;
      // x projections (+ biases) of this thread's 2 sequences x 2 units x 4 gates
      float acc[4][4];                     // [gate][d-fragment element: (r0,cu) (r0,cu+1) (r0+8,cu) (r0+8,cu+1)]
      int ts[2];                           // the time index of this thread's 2 sequences; -1 past their length
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int b = min(b0 + warp * 16 + r0 + 8 * hh, batch - 1);
        const int eb = ext ? ext[b] : T;
        const int t = dir == 0 ? step : eb - 1 - step;
        ts[hh] = step < eb ? t : -1;
        const float* xp = xproj + ((int64_t)b * t_ld + max(t, 0)) * xp_ld + dir * 4 * LS_H + c * LS_UNITS + cu;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const float2 x2 = __ldg(reinterpret_cast<const float2*>(xp + g * LS_H));
          acc[g][2 * hh] = x2.x; acc[g][2 * hh + 1] = x2.y;
        }
      }
      if (step > 0) {
        // h_{t-1} planes of this tile: [64][512] bf16 hi and lo, L2 -> shared memory
        for (int idx = tid; idx < 2 * LS_BT * (LS_H / 8); idx += blockDim.x) {
          const int pl = idx / (LS_BT * (LS_H / 8)), rem = idx % (LS_BT * (LS_H / 8));
          const int b = rem / (LS_H / 8), k8 = rem % (LS_H / 8);
          const uint32_t dst = sH_addr + (uint32_t)(pl * LS_BT * LT_PITCH + b * LT_PITCH + 16 * k8);
          const __nv_bfloat16* src = hx_rd + pl * plane_stride + (int64_t)(b0 + b) * LS_H + 8 * k8;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
        float d[4][4];
#pragma unroll
        for (int g = 0; g < 4; ++g) { d[g][0] = d[g][1] = d[g][2] = d[g][3] = 0.f; }
#pragma unroll 4
        for (int k = 0; k < LS_H / 16; ++k) {
          uint32_t ah[4], al[4], bh01[4], bh23[4], bl01[4], bl23[4];
          ldmatrix_x4(ah, sH_addr + a_lane + 32 * k);
          ldmatrix_x4(al, sH_addr + LS_BT * LT_PITCH + a_lane + 32 * k);
          ldmatrix_x4(bh01, sW_addr + b_lane + 32 * k);                                   // gates 0,1 (hi)
          ldmatrix_x4(bh23, sW_addr + 16 * LT_PITCH + b_lane + 32 * k);                  // gates 2,3 (hi)
          ldmatrix_x4(bl01, sW_addr + LS_ROWS * LT_PITCH + b_lane + 32 * k);             // gates 0,1 (lo)
          ldmatrix_x4(bl23, sW_addr + LS_ROWS * LT_PITCH + 16 * LT_PITCH + b_lane + 32 * k);
          mma_bf16_16816(d[0], ah, bh01[0], bh01[1]); mma_bf16_16816(d[1], ah, bh01[2], bh01[3]);
          mma_bf16_16816(d[2], ah, bh23[0], bh23[1]); mma_bf16_16816(d[3], ah, bh23[2], bh23[3]);
          mma_bf16_16816(d[0], ah, bl01[0], bl01[1]); mma_bf16_16816(d[1], ah, bl01[2], bl01[3]);
          mma_bf16_16816(d[2], ah, bl23[0], bl23[1]); mma_bf16_16816(d[3], ah, bl23[2], bl23[3]);
          mma_bf16_16816(d[0], al, bh01[0], bh01[1]); mma_bf16_16816(d[1], al, bh01[2], bh01[3]);
          mma_bf16_16816(d[2], al, bh23[0], bh23[1]); mma_bf16_16816(d[3], al, bh23[2], bh23[3]);
        }
#pragma unroll
        for (int g = 0; g < 4; ++g)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[g][e] += d[g][e];
      }
      // cells: element e = 2*hh + uu  <->  sequence r0 + 8 hh, unit cu + uu
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int bseq = b0 + warp * 16 + r0 + 8 * hh;
        float hv[2];
#pragma unroll
        for (int uu = 0; uu < 2; ++uu) {
          const int e = 2 * hh + uu;
          const float ig = sigmoidf_(acc[0][e]), fg = sigmoidf_(acc[1][e]), gg = tanhf(acc[2][e]), og = sigmoidf_(acc[3][e]);
          const float cn = fg * cst[bt][hh][uu] + ig * gg;
          cst[bt][hh][uu] = cn;
          hv[uu] = og * tanhf(cn);
        }
        if (bseq < batch && ts[hh] >= 0) *reinterpret_cast<float2*>(out + ((int64_t)bseq * t_ld + ts[hh]) * out_ld + dir * LS_H + c * LS_UNITS + cu) = make_float2(hv[0], hv[1]);
        // publish bf16 planes of h_t for the next step (padded sequences publish finite garbage that nobody reads back into results)
        const __nv_bfloat162 h2 = __floats2bfloat162_rn(hv[0], hv[1]);
        const uint32_t hb = *reinterpret_cast<const uint32_t*>(&h2);
        const __nv_bfloat162 l2 = __floats2bfloat162_rn(hv[0] - __uint_as_float(hb << 16), hv[1] - __uint_as_float(hb & 0xFFFF0000u));
        const int64_t off = (int64_t)bseq * LS_H + c * LS_UNITS + cu;
        *reinterpret_cast<uint32_t*>(hx_wr + off) = hb;
        *reinterpret_cast<uint32_t*>(hx_wr + plane_stride + off) = *reinterpret_cast<const uint32_t*>(&l2);
      }
      __syncthreads();                               // sHp is reused by the next batch tile
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) atomicAdd(counter, 1u);
  }
}

// 256 bytes of step counters, then the bf16 hi / lo planes of h for both directions, double buffered
static size_t blstm_scratch_bytes(int batch, int H) {
  const int batch_pad = (batch + LS_BT - 1) / LS_BT * LS_BT;
  return 256 + (size_t)2 * 2 * 2 * batch_pad * H * sizeof(__nv_bfloat16);
}

template <int H>
static int blstm_tc_launch_h(const float* xproj, const float* w_hh_f, const float* w_hh_b, int batch, int T, int t_ld, const int32_t* ext,
                             float* out, void* scratch, size_t scratch_bytes, cudaStream_t st) {
  const size_t need = blstm_scratch_bytes(batch, H);
  if (scratch_bytes < need) return FA_ERR_WORKSPACE;
  const size_t smem = (size_t)2 * LS_ROWS * lt_pitch<H>() + (size_t)2 * LS_BT * lt_pitch<H>();
  static PerDeviceOnce once;
  FA_RETURN_IF_ERR(ensure_dyn_smem(blstm_tc_kernel<H>, smem, once));
  unsigned int* counters = static_cast<unsigned int*>(scratch);
  __nv_bfloat16* hx = reinterpret_cast<__nv_bfloat16*>(static_cast<char*>(scratch) + 256);
  FA_CUDA_OK(cudaMemsetAsync(scratch, 0, need, st));
  void* args[] = {(void*)&xproj, (void*)&w_hh_f, (void*)&w_hh_b, (void*)&batch, (void*)&T, (void*)&t_ld, (void*)&ext, (void*)&out, (void*)&hx,
                  (void*)&counters};
  FA_CUDA_OK(cudaLaunchCooperativeKernel((const void*)blstm_tc_kernel<H>, dim3(2 * (H / LS_UNITS)), dim3(128), args, smem, st));
  count_launch();
  return FA_OK;
}

// T steps of sequences t_ld long; ext: their lengths on the device (NULL: T = t_ld for all)
int blstm_tc_launch(const float* xproj, const float* w_hh_f, const float* w_hh_b, int batch, int T, int t_ld, const int32_t* ext, int hidden,
                    float* out, void* scratch, size_t scratch_bytes, cudaStream_t st) {
  if (batch <= 0 || T <= 0) return FA_OK;
  if (!xproj || !w_hh_f || !w_hh_b || !out || !scratch) return FA_ERR_ARG;
  if ((hidden != 512 && hidden != 320) || batch > 4 * LS_BT) return FA_ERR_UNSUPPORTED;
  return hidden == 512 ? blstm_tc_launch_h<512>(xproj, w_hh_f, w_hh_b, batch, T, t_ld, ext, out, scratch, scratch_bytes, st)
                       : blstm_tc_launch_h<320>(xproj, w_hh_f, w_hh_b, batch, T, t_ld, ext, out, scratch, scratch_bytes, st);
}

// the per-sequence lengths ext_h [batch] (host, 1 <= ext_h[b] <= t_len) after the recurrence's scratch, 256-byte aligned
static size_t blstm_ext_scratch_bytes(int batch) {
  return blstm_scratch_bytes(batch, LS_HMAX) + (size_t)(batch > 0 ? batch : 0) * sizeof(int32_t);
}

}  // namespace fa

// One-layer bidirectional LSTM over [B, T, H], H = 512 or 320, given the input projections of both directions:
//   xproj [B*T, 2*4H] = x W_ih^T + b_ih + b_hh, columns [0,4H) forward gates (i,f,g,o), [4H,8H) reverse.
// scratch >= fa_blstm_tc_scratch_bytes(batch) (sized for H = 512, which covers 320).
extern "C" size_t fa_blstm_tc_scratch_bytes(int32_t batch) { return fa::blstm_scratch_bytes(batch, fa::LS_HMAX); }
extern "C" int fa_blstm_forward_tc(const float* xproj, const float* w_hh_fwd, const float* w_hh_bwd, int32_t batch, int32_t t_len,
                                   int32_t hidden, float* out, void* scratch, size_t scratch_bytes, fa_stream_t stream) {
  return fa::blstm_tc_launch(xproj, w_hh_fwd, w_hh_bwd, batch, t_len, t_len, nullptr, hidden, out, scratch, scratch_bytes, (cudaStream_t)stream);
}

extern "C" size_t fa_blstm_tc_ext_scratch_bytes(int32_t batch) { return fa::blstm_ext_scratch_bytes(batch); }
extern "C" int fa_blstm_forward_tc_ext(const float* xproj, const float* w_hh_fwd, const float* w_hh_bwd, int32_t batch, int32_t t_len,
                                       int32_t hidden, float* out, void* scratch, size_t scratch_bytes, fa_stream_t stream, const int32_t* ext_h) {
  if (!ext_h || batch < 0 || t_len < 0) return FA_ERR_ARG;
  int32_t t_run = 0;
  for (int32_t b = 0; b < batch; ++b) {
    if (ext_h[b] < 1 || ext_h[b] > t_len) return FA_ERR_ARG;
    t_run = ext_h[b] > t_run ? ext_h[b] : t_run;
  }
  if (batch == 0 || t_len == 0) return FA_OK;
  if (!xproj || !w_hh_fwd || !w_hh_bwd || !out || !scratch) return FA_ERR_ARG;
  if ((hidden != 512 && hidden != 320) || batch > 4 * fa::LS_BT) return FA_ERR_UNSUPPORTED;
  if (scratch_bytes < fa::blstm_ext_scratch_bytes(batch)) return FA_ERR_WORKSPACE;
  const size_t lstm_bytes = fa::blstm_scratch_bytes(batch, fa::LS_HMAX);
  int32_t* ext_d = reinterpret_cast<int32_t*>(static_cast<char*>(scratch) + lstm_bytes);
  FA_CUDA_OK(cudaMemcpyAsync(ext_d, ext_h, (size_t)batch * sizeof(int32_t), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return fa::blstm_tc_launch(xproj, w_hh_fwd, w_hh_bwd, batch, t_run, t_len, ext_d, hidden, out, scratch, lstm_bytes, (cudaStream_t)stream);
}
