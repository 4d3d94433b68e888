// FSMN memory block: out[b,t,c] = m[t] * ( v[t]m[t] + sum_j w[c,j] v[t+j-L]m[t+j-L] ) (+ res[b,t,c]),
// m[t] = 1[t < lens[b]], L = (k-1)/2, zero outside [0, t_max) — the depthwise Conv1d(groups=C, no bias)
// of MultiHeadedAttentionSANM.forward_fsmn (sanm/attention.py:216-239) and of the decoder's
// MultiHeadedAttentionSANMDecoder.forward (:583-631); `res` fuses DecoderLayerSANM's `residual + x`
// (paraformer/decoder.py:107).  HBM-bound (reads v once + halo, writes once): channels are the
// coalesced axis, each thread slides a k-wide register window down a strip of time steps.
//
// Two kernels compute it (bit-identical results, same fma order):
//  * fsmn_kernel      — plain SIMT strips: every thread slides a K-wide register window down 32 time steps of one channel;
//                       the K-1 halo rows of a strip are re-read through L2 (+31 % reads at K = 11).
//  * fsmn_tma_kernel  — the TMA-staged, warp-specialised form: persistent CTAs (one per SM); a producer warp streams
//                       [64 + K - 1 time steps] x [128 channels] boxes of v (and the matching 64-row box of the residual) into a
//                       3-stage shared-memory ring with cp.async.bulk.tensor (3-D tensor map {channel, time, utterance}: the zero
//                       padding of the convolution at the utterance edges IS the map's out-of-bounds fill), 8 consumer warps slide
//                       their windows over shared memory (each v element crosses L2->SM once) and store the result rows coalesced.
//                       Used wherever its shape rules hold (k = 11 / 21, channels % 128 == 0, t_max >= 64, 16-byte aligned rows);
//                       the SIMT kernel covers every other shape.  A/B at the encoder shape (DESIGN.md §6): 48.1 -> 39.9 us.
#include "common.cuh"
#include "tc_common.cuh"
#include <unordered_map>

namespace fa {

constexpr int FSMN_TT = 32;     // time steps per thread strip
constexpr int FSMN_KMAX = 31;

// K taps, the window of output t covers inputs t - L .. t - L + K - 1: L = (K-1)/2 is the centred SAN-M memory block, L = K - 1
// the causal memory of the FSMN-VAD encoder (FSMNBlock.conv_left over zero LEFT padding, fsmn_vad_streaming/encoder.py:136-160).
template <int K, int L>
__global__ void __launch_bounds__(128)
fsmn_kernel(const float* __restrict__ v, int64_t ldv, const int32_t* __restrict__ lens, int t_max, int channels,
            const float* __restrict__ w, const float* __restrict__ res, int64_t ldr, float* __restrict__ out,
            int64_t ldo) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int t0 = blockIdx.y * FSMN_TT;
  const int b = blockIdx.z;
  if (c >= channels) return;
  const int len = min(lens[b], t_max);
  float wk[K];
#pragma unroll
  for (int j = 0; j < K; ++j) wk[j] = __ldg(w + c * K + j);
  const float* vb = v + (int64_t)b * t_max * ldv + c;
  auto load = [&](int t) -> float { return (t >= 0 && t < len) ? __ldg(vb + (int64_t)t * ldv) : 0.f; };  // v*m, zero pad
  float win[K];
#pragma unroll
  for (int j = 0; j < K - 1; ++j) win[j + 1] = load(t0 - L + j);
  const int t_end = min(t0 + FSMN_TT, t_max);
  for (int t = t0; t < t_end; ++t) {
#pragma unroll
    for (int j = 0; j < K - 1; ++j) win[j] = win[j + 1];
    win[K - 1] = load(t + K - 1 - L);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < K; ++j) acc = fmaf(wk[j], win[j], acc);
    float o = t < len ? __fadd_rn(acc, win[L]) : 0.f;     // (conv + inputs) * mask
    const int64_t row = (int64_t)b * t_max + t;
    if (res) o = __fadd_rn(__ldg(res + row * ldr + c), o);
    out[row * ldo + c] = o;
  }
}

// ------------------------------------------------------------------------------------------------ TMA-staged variant
constexpr int FT_TT = 64;          // output time steps per tile
constexpr int FT_CH = 128;         // channels per tile (512 B rows in shared memory)
constexpr int FT_STAGES = 3;
constexpr int FT_CONSUMER_WARPS = 8;
constexpr int FT_THREADS = 32 * (1 + FT_CONSUMER_WARPS);

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

template <int K>
__global__ void __launch_bounds__(FT_THREADS, 1)
fsmn_tma_kernel(const __grid_constant__ CUtensorMap vmap, const __grid_constant__ CUtensorMap rmap, int has_res,
                const int32_t* __restrict__ lens, int t_max, int t_tiles, int ch_tiles, int n_tiles,
                const float* __restrict__ w, float* __restrict__ out, int64_t ldo) {
  constexpr int L = (K - 1) / 2;
  constexpr int VROWS = FT_TT + K - 1;
  constexpr uint32_t V_BYTES = VROWS * FT_CH * 4, R_BYTES = FT_TT * FT_CH * 4, STAGE_BYTES = V_BYTES + R_BYTES;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + FT_STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + FT_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&vmap);
    if (has_res) tma_prefetch_desc(&rmap);
    for (int s = 0; s < FT_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], FT_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ===================== producer: one lane issues the bulk tensor copies =====================
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int ct = tile % ch_tiles, rest = tile / ch_tiles;
        const int tt = rest % t_tiles, b = rest / t_tiles;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_expect_tx(&full_bar[stage], has_res ? STAGE_BYTES : V_BYTES);
        unsigned char* sp = smem + stage * STAGE_BYTES;
        // rows t0 - L .. t0 - L + VROWS - 1 of utterance b: rows outside [0, t_max) arrive as zeros (the conv's zero padding)
        tma_load_3d(sp, &vmap, &full_bar[stage], ct * FT_CH, tt * FT_TT - L, b);
        if (has_res) tma_load_3d(sp + V_BYTES, &rmap, &full_bar[stage], ct * FT_CH, tt * FT_TT, b);
        if (++stage == FT_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ===================== consumers: 2 threads per channel, 32 output rows each =====================
    const int ctid = threadIdx.x - 32;
    const int c = ctid & (FT_CH - 1), half = ctid >> 7;
    const int r0 = half * (FT_TT / 2);
    int stage = 0; uint32_t phase = 0;
    float wk[K];
    int wk_ct = -1;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const int ct = tile % ch_tiles, rest = tile / ch_tiles;
      const int tt = rest % t_tiles, b = rest / t_tiles;
      const int t0 = tt * FT_TT;
      const int len = min(lens[b], t_max);
      if (ct != wk_ct) {
#pragma unroll
        for (int j = 0; j < K; ++j) wk[j] = __ldg(w + (ct * FT_CH + c) * K + j);
        wk_ct = ct;
      }
      mbar_wait(&full_bar[stage], phase);
      const float* sv = reinterpret_cast<const float*>(smem + stage * STAGE_BYTES) + c;
      const float* sr = reinterpret_cast<const float*>(smem + stage * STAGE_BYTES + V_BYTES) + c;
      // shared row i holds input time t0 - L + i; times >= len are masked (v * m), times < 0 / >= t_max were zero-filled
      auto load = [&](int i) -> float { return (t0 - L + i < len) ? sv[i * FT_CH] : 0.f; };
      float win[K];
#pragma unroll
      for (int j = 0; j < K - 1; ++j) win[j + 1] = load(r0 + j);
      float* orow = out + ((int64_t)b * t_max + t0 + r0) * ldo + ct * FT_CH + c;
#pragma unroll 4
      for (int r = r0; r < r0 + FT_TT / 2; ++r) {
#pragma unroll
        for (int j = 0; j < K - 1; ++j) win[j] = win[j + 1];
        win[K - 1] = load(r + K - 1);
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < K; ++j) acc = fmaf(wk[j], win[j], acc);
        const int t = t0 + r;
        float o = t < len ? __fadd_rn(acc, win[L]) : 0.f;     // (conv + inputs) * mask
        if (has_res) o = __fadd_rn(sr[r * FT_CH], o);
        if (t < t_max) *orow = o;
        orow += ldo;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);          // this warp is done reading the stage
      if (++stage == FT_STAGES) { stage = 0; phase ^= 1; }
    }
  }
}

// 3-D fp32 tensor map {cols (contiguous), rows, batch}: row pitch ld floats, batch pitch rows * ld floats; box {box_cols, box_rows, 1};
// no swizzle (rows of the box are 512 B, consumers read them conflict-free along the channel axis); out-of-bounds elements read 0.
static int make_f32_map3(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t batch, uint64_t ld, uint32_t box_cols,
                         uint32_t box_rows) {
  typedef CUresult (*PFN_enc)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                              const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static const PFN_enc enc = []() -> PFN_enc {                     // thread-safe one-time lookup (two handles / two threads share this TU)
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
    return reinterpret_cast<PFN_enc>(p);
  }();
  if (!enc) return FA_ERR_CUDA;
  struct Key {
    const void* base; uint64_t cols, rows, batch, ld; uint32_t bc, br;
    bool operator==(const Key& o) const { return base == o.base && cols == o.cols && rows == o.rows && batch == o.batch && ld == o.ld && bc == o.bc && br == o.br; }
  };
  struct Hash {
    size_t operator()(const Key& k) const {
      uint64_t h = (uint64_t)(uintptr_t)k.base * 0x9E3779B97F4A7C15ull;
      h ^= k.rows * 1315423911ull + k.batch * 2654435761ull + k.ld * 97 + k.cols * 31 + k.bc * 7 + k.br + (h << 6) + (h >> 2);
      return (size_t)h;
    }
  };
  static thread_local std::unordered_map<Key, CUtensorMap, Hash> cache;   // the workspace slices repeat every layer and every step
  const Key key{base, cols, rows, batch, ld, box_cols, box_rows};
  auto it = cache.find(key);
  if (it != cache.end()) { *m = it->second; return FA_OK; }
  cuuint64_t dims[3] = {cols, rows, batch};
  cuuint64_t strides[2] = {ld * 4, rows * ld * 4};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  if (enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return FA_ERR_CUDA;
  if (cache.size() >= 1024) cache.clear();
  cache.emplace(key, *m);
  return FA_OK;
}

static bool fsmn_tma_supported(const float* v, int64_t ldv, int channels, int ksize, const float* res, int64_t ldr) {
  if (ksize != 11 && ksize != 21) return false;
  if (channels % FT_CH != 0) return false;
  if ((reinterpret_cast<uintptr_t>(v) & 15) || (ldv & 3) || ldv < channels) return false;             // TMA: 16-byte base and pitches
  if (res && ((reinterpret_cast<uintptr_t>(res) & 15) || (ldr & 3) || ldr < channels)) return false;
  return true;
}

template <int K>
static int fsmn_tma_launch_k(const float* v, int64_t ldv, const int32_t* lens, int batch, int t_max, int channels, const float* w,
                             const float* res, int64_t ldr, float* out, int64_t ldo, cudaStream_t st) {
  constexpr size_t smem = (size_t)FT_STAGES * ((FT_TT + K - 1) * FT_CH * 4 + FT_TT * FT_CH * 4) + 1024 + 64;
  static PerDeviceOnce once;
  FA_RETURN_IF_ERR(ensure_dyn_smem(fsmn_tma_kernel<K>, smem, once));
  CUtensorMap vm, rm;
  FA_RETURN_IF_ERR(make_f32_map3(&vm, v, (uint64_t)channels, (uint64_t)t_max, (uint64_t)batch, (uint64_t)ldv, FT_CH, FT_TT + K - 1));
  if (res) FA_RETURN_IF_ERR(make_f32_map3(&rm, res, (uint64_t)channels, (uint64_t)t_max, (uint64_t)batch, (uint64_t)ldr, FT_CH, FT_TT));
  else rm = vm;
  const int t_tiles = (t_max + FT_TT - 1) / FT_TT, ch_tiles = channels / FT_CH;
  const int64_t n_tiles64 = (int64_t)batch * t_tiles * ch_tiles;
  if (n_tiles64 > 0x7fffffffLL) return FA_ERR_UNSUPPORTED;
  const int n_tiles = (int)n_tiles64;
  const int n_sm = sm_count();
  const int grid = n_tiles < n_sm ? n_tiles : n_sm;
  fsmn_tma_kernel<K><<<grid, FT_THREADS, smem, st>>>(vm, rm, res ? 1 : 0, lens, t_max, t_tiles, ch_tiles, n_tiles, w, out, ldo);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

int fsmn_tma_launch(const float* v, int64_t ldv, const int32_t* lens, int batch, int t_max, int channels, const float* w, int ksize,
                    const float* res, int64_t ldr, float* out, int64_t ldo, cudaStream_t st) {
  if (batch <= 0 || t_max <= 0) return FA_OK;
  if (!v || !lens || !w || !out) return FA_ERR_ARG;
  if (!fsmn_tma_supported(v, ldv, channels, ksize, res, ldr)) return FA_ERR_UNSUPPORTED;
  if (ksize == 11) return fsmn_tma_launch_k<11>(v, ldv, lens, batch, t_max, channels, w, res, ldr, out, ldo, st);
  return fsmn_tma_launch_k<21>(v, ldv, lens, batch, t_max, channels, w, res, ldr, out, ldo, st);
}

// the TMA-staged kernel wherever its shape rules hold, SIMT strips otherwise (tools/fsmn_probe.py compares the two)
int fsmn_simt_launch(const float* v, int64_t ldv, const int32_t* lens, int batch, int t_max, int channels, const float* w,
                     int ksize, const float* res, int64_t ldr, float* out, int64_t ldo, cudaStream_t st, int causal);

int fsmn_launch(const float* v, int64_t ldv, const int32_t* lens, int batch, int t_max, int channels, const float* w,
                int ksize, const float* res, int64_t ldr, float* out, int64_t ldo, cudaStream_t st, int causal) {
  if (batch <= 0 || t_max <= 0) return FA_OK;
  if (!v || !lens || !w || !out) return FA_ERR_ARG;
  if (!causal && t_max >= FT_TT && fsmn_tma_supported(v, ldv, channels, ksize, res, ldr))
    return fsmn_tma_launch(v, ldv, lens, batch, t_max, channels, w, ksize, res, ldr, out, ldo, st);
  return fsmn_simt_launch(v, ldv, lens, batch, t_max, channels, w, ksize, res, ldr, out, ldo, st, causal);
}

int fsmn_simt_launch(const float* v, int64_t ldv, const int32_t* lens, int batch, int t_max, int channels, const float* w,
                     int ksize, const float* res, int64_t ldr, float* out, int64_t ldo, cudaStream_t st, int causal) {
  if (batch <= 0 || t_max <= 0) return FA_OK;
  if (!v || !lens || !w || !out) return FA_ERR_ARG;
  dim3 grid((channels + 127) / 128, (t_max + FSMN_TT - 1) / FSMN_TT, batch);
  if (causal) {
    if (ksize != 20) return FA_ERR_UNSUPPORTED;
    fsmn_kernel<20, 19><<<grid, 128, 0, st>>>(v, ldv, lens, t_max, channels, w, res, ldr, out, ldo);
    FA_CHECK_LAUNCH();
    return FA_OK;
  }
  switch (ksize) {
    case 11: fsmn_kernel<11, 5><<<grid, 128, 0, st>>>(v, ldv, lens, t_max, channels, w, res, ldr, out, ldo); break;
    case 21: fsmn_kernel<21, 10><<<grid, 128, 0, st>>>(v, ldv, lens, t_max, channels, w, res, ldr, out, ldo); break;
    case 31: fsmn_kernel<31, 15><<<grid, 128, 0, st>>>(v, ldv, lens, t_max, channels, w, res, ldr, out, ldo); break;
    default: return FA_ERR_UNSUPPORTED;
  }
  FA_CHECK_LAUNCH();
  return FA_OK;
}

}  // namespace fa

extern "C" int fa_fsmn(const float* v, int64_t ldv, const int32_t* lens, int32_t batch, int32_t t_max, int32_t channels,
                       const float* w, int32_t ksize, const float* res, int64_t ld_res, float* out, int64_t ld_out,
                       fa_stream_t stream) {
  return fa::fsmn_launch(v, ldv, lens, batch, t_max, channels, w, ksize, res, ld_res, out, ld_out, (cudaStream_t)stream, 0);
}

extern "C" int fa_fsmn_simt(const float* v, int64_t ldv, const int32_t* lens, int32_t batch, int32_t t_max, int32_t channels,
                            const float* w, int32_t ksize, const float* res, int64_t ld_res, float* out, int64_t ld_out,
                            fa_stream_t stream) {
  return fa::fsmn_simt_launch(v, ldv, lens, batch, t_max, channels, w, ksize, res, ld_res, out, ld_out, (cudaStream_t)stream, 0);
}

extern "C" int fa_fsmn_tma(const float* v, int64_t ldv, const int32_t* lens, int32_t batch, int32_t t_max, int32_t channels,
                           const float* w, int32_t ksize, const float* res, int64_t ld_res, float* out, int64_t ld_out,
                           fa_stream_t stream) {
  return fa::fsmn_tma_launch(v, ldv, lens, batch, t_max, channels, w, ksize, res, ld_res, out, ld_out, (cudaStream_t)stream);
}
