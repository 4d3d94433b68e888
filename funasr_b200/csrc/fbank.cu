// Fused Fbank + LFR + CMVN frontend (one kernel): wav[B, N] -> feats[B, T, 560].
//
// Replaces WavFrontend.forward (funasr/frontends/wav_frontend.py:149-196): per utterance
//   x32768 (:169) -> torchaudio.compliance.kaldi.fbank(dither=0, hamming, 25/10 ms, 80 mel, snip_edges)
//   (kaldi.py:514-647) -> apply_lfr m=7 n=6 (:63-86) -> apply_cmvn (:46-60) -> pad_sequence(0.0) (:195).
//
// HBM-bound by design: algorithmic bytes = 4 B/sample in + 4*560 B/LFR-row out (3.04 MB per 30 s).
// The per-configuration constants (window, FFT twiddles, mel filter taps) are computed once by fa_fbank_make_tables.
// One CTA owns kRows consecutive LFR rows of one utterance: it copies the tables into shared memory, each warp reads
// its frames' samples straight from global memory (coalesced 8-byte loads; the 2.5x overlap between frames hits L1)
// and turns them into log-mel rows with a register-resident 256-point complex FFT (radix 8 in registers x 32-point
// across the lanes on shuffles; real 512-point FFT by even/odd packing), and the CTA then writes its LFR rows
// (7 stacked log-mel frames, CMVN applied) with fully coalesced stores.
// Adjacent CTAs recompute one overlapping frame (1/48 redundancy) instead of round-tripping log-mel
// through HBM.
#include "common.cuh"

namespace fa {

constexpr int kWin = 400, kShift = 160, kFft = 512, kBins = 257, kMel = 80;
constexpr int kFramesMax = 49;                         // frames one CTA turns into log-mel rows: 6*(8-1)+7 (ASR, LFR 7/6) or 1*(44-1)+5 (VAD, LFR 5/1)
constexpr int kWarps = 8;
constexpr int kMelPackMax = 1024;
// Precomputed tables (fa_fbank_make_tables): constants of the configuration that every CTA would otherwise rebuild — the
// sparse support of the 80 triangular mel filters, the FFT twiddles, the window, and the mel TAP SCHEDULE: the ~514 non-zero
// filter taps dealt to the 32 lanes filter by filter (longest first, each to the least loaded lane), so that a warp applies all
// 80 filters in max-load (~18) uniform iterations instead of three lane-per-filter passes of up to 4 + 14 + 18 dependent ones.
// Layout in floats:
constexpr int kTapMax = 40;                            // iterations of the tap loop (average load 16, longest filter 18)
constexpr int kTabStart = 0, kTabLen = kMel, kTabOff = 2 * kMel, kTabW = 3 * kMel, kTabTw = kTabW + kMelPackMax,
              kTabWin = kTabTw + 512, kTabTapN = kTabWin + kWin, kTabTapMeta = kTabTapN + 8, kTabTapW = kTabTapMeta + kTapMax * 32,
              kTabFloats = kTabTapW + kTapMax * 32;
constexpr int kTapFlush = 1 << 16;                     // tap meta: bin | filter << 9 | kTapFlush on a filter's last tap
constexpr int kZs = 36;                                // spectrum row pitch (float2): at most 2-way bank conflicts on the strided reads

// Shared memory of fbank_tab_kernel (no waveform staging: 4 CTAs per SM instead of 2).
struct FbankSmemT {
  float logmel[kFramesMax * kMel];
  float2 zs[kWarps][8 * kZs];      // per warp: the 256-point spectrum as [k1 = 0..7][k2] rows of pitch kZs
  float pw[kWarps][264];           // per warp: power spectrum P[0..256]
  float macc[kWarps][kMel];        // per warp: mel energies of the frame in flight
  float2 tw[256];
  float win[kWin];
  int tap_meta[kTapMax * 32];
  float tap_w[kTapMax * 32];
};

// Per-lane constants of the register FFT (hoisted out of the frame loop).
struct LaneTw { float2 tw8[8]; float2 twl[5]; int rev; };

// One frame -> its 256-point complex spectrum Z (of z[n] = y[2n] + i y[2n+1], y = the DC-removed, pre-emphasised, windowed and
// zero-padded 512-sample frame) in Zs[k1 * kZs + k2] = Z[k1 + 8 k2].  Warp-collective.  x: the frame's first sample,
// vec2: x is 8-byte aligned.
__device__ __forceinline__ void frame_spectrum(const float* __restrict__ x, const float scl, const bool vec2, const float* __restrict__ s_win,
                                               const LaneTw& lt, const int lane, float2* __restrict__ Zs) {
  const float kR = 0.70710678118654752f;
  // samples 2(L + 32 r), +1 of the frame (zero beyond the 400-sample window) and their predecessors
  float xe[8], xo[8], xp[8];
  float part = 0.f;
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int j0 = 2 * lane + 64 * r;
    if (j0 < kWin) {
      float2 v;
      if (vec2) v = *reinterpret_cast<const float2*>(x + j0); else v = make_float2(x[j0], x[j0 + 1]);
      xe[r] = v.x * scl; xo[r] = v.y * scl;                      // scl = 32768 (exact) when x is the raw waveform
      xp[r] = x[j0 > 0 ? j0 - 1 : 0] * scl;                      // replicate pad, kaldi.py:193-198
      part += xe[r] + xo[r];
    } else { xe[r] = xo[r] = xp[r] = 0.f; }
  }
  const float mean = warp_sum(part) / (float)kWin;               // remove_dc_offset kaldi.py:183-186
  float2 v[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int j0 = 2 * lane + 64 * r;
    if (j0 < kWin) {
      const float ce = __fsub_rn(xe[r], mean), co = __fsub_rn(xo[r], mean), cp = __fsub_rn(xp[r], mean);
      const float2 w2 = *reinterpret_cast<const float2*>(s_win + j0);
      v[r].x = __fmul_rn(__fsub_rn(ce, __fmul_rn(0.97f, cp)), w2.x);      // pre-emphasis then window (:193-204)
      v[r].y = __fmul_rn(__fsub_rn(co, __fmul_rn(0.97f, ce)), w2.y);
    } else { v[r] = make_float2(0.f, 0.f); }
  }
  // (1) 8-point DFT over r (two 4-point DFTs on the even / odd r, then the W_8 combine)
  {
    float2 e[4], o[4];
    {
      const float2 t0 = make_float2(v[0].x + v[4].x, v[0].y + v[4].y), t1 = make_float2(v[0].x - v[4].x, v[0].y - v[4].y);
      const float2 t2 = make_float2(v[2].x + v[6].x, v[2].y + v[6].y), t3 = make_float2(v[2].x - v[6].x, v[2].y - v[6].y);
      e[0] = make_float2(t0.x + t2.x, t0.y + t2.y); e[2] = make_float2(t0.x - t2.x, t0.y - t2.y);
      e[1] = make_float2(t1.x + t3.y, t1.y - t3.x); e[3] = make_float2(t1.x - t3.y, t1.y + t3.x);    // t1 -/+ i t3
    }
    {
      const float2 t0 = make_float2(v[1].x + v[5].x, v[1].y + v[5].y), t1 = make_float2(v[1].x - v[5].x, v[1].y - v[5].y);
      const float2 t2 = make_float2(v[3].x + v[7].x, v[3].y + v[7].y), t3 = make_float2(v[3].x - v[7].x, v[3].y - v[7].y);
      o[0] = make_float2(t0.x + t2.x, t0.y + t2.y); o[2] = make_float2(t0.x - t2.x, t0.y - t2.y);
      o[1] = make_float2(t1.x + t3.y, t1.y - t3.x); o[3] = make_float2(t1.x - t3.y, t1.y + t3.x);
    }
    // W_8^1 = (1 - i)/sqrt2, W_8^2 = -i, W_8^3 = (-1 - i)/sqrt2
    const float2 o1 = make_float2(kR * (o[1].x + o[1].y), kR * (o[1].y - o[1].x));
    const float2 o2 = make_float2(o[2].y, -o[2].x);
    const float2 o3 = make_float2(kR * (o[3].y - o[3].x), -kR * (o[3].x + o[3].y));
    v[0] = make_float2(e[0].x + o[0].x, e[0].y + o[0].y); v[4] = make_float2(e[0].x - o[0].x, e[0].y - o[0].y);
    v[1] = make_float2(e[1].x + o1.x, e[1].y + o1.y);     v[5] = make_float2(e[1].x - o1.x, e[1].y - o1.y);
    v[2] = make_float2(e[2].x + o2.x, e[2].y + o2.y);     v[6] = make_float2(e[2].x - o2.x, e[2].y - o2.y);
    v[3] = make_float2(e[3].x + o3.x, e[3].y + o3.y);     v[7] = make_float2(e[3].x - o3.x, e[3].y - o3.y);
  }
  // (2) twiddle W_256^{lane k1}
#pragma unroll
  for (int k1 = 1; k1 < 8; ++k1) v[k1] = make_float2(v[k1].x * lt.tw8[k1].x - v[k1].y * lt.tw8[k1].y, v[k1].x * lt.tw8[k1].y + v[k1].y * lt.tw8[k1].x);
  // (3) 32-point DFT across the lanes (decimation in frequency: lane L ends with output index rev5(L))
#pragma unroll
  // One butterfly for both halves, no selects: r = partner + sgn * own (sgn = +1 in the lower lane: the sum; -1 in the upper lane:
  // lower - upper), then r * w with w = the stage twiddle in the upper lane and exactly (1, 0) in the lower lane (lt.twl holds that).
  // The last stage (pairs of adjacent lanes) has w = 1 everywhere.  Bit-identical to the select form: +-1 and (1, 0) are exact.
  for (int st = 0; st < 5; ++st) {
    const int mm = 16 >> st;
    const float sgn = (lane & mm) ? -1.f : 1.f;
    const float2 w = lt.twl[st];
#pragma unroll
    for (int k1 = 0; k1 < 8; ++k1) {
      const float px = __shfl_xor_sync(0xffffffffu, v[k1].x, mm), py = __shfl_xor_sync(0xffffffffu, v[k1].y, mm);
      const float rx = fmaf(sgn, v[k1].x, px), ry = fmaf(sgn, v[k1].y, py);
      v[k1] = st == 4 ? make_float2(rx, ry) : make_float2(rx * w.x - ry * w.y, rx * w.y + ry * w.x);
    }
  }
#pragma unroll
  for (int k1 = 0; k1 < 8; ++k1) Zs[k1 * kZs + lt.rev] = v[k1];                  // Z[k1 + 8 rev5(lane)]
  __syncwarp();
}

// fa_fbank_lfr_cmvn_tables: kLfrM / kLfrN is the low-frame-rate stacking (7/6 for Paraformer & SenseVoice, 5/1 for the FSMN-VAD,
// 1/1 for CAM++), kRows the LFR rows per CTA.
//   * no waveform staging: every warp reads its frame's 400 samples straight from global memory (coalesced 8-byte loads; the 2.5x
//     overlap between frames hits L1).  Staging the CTA's samples in shared memory first put 32 dependent global-load rounds in
//     front of a barrier and its 32 KB of shared memory held the kernel at 2 CTAs per SM;
//   * power spectrum in pairs: X[k] and X[256 - k] of the real 512-point transform share E_k and O_k, so a lane computes both
//     from one pair of spectrum loads (4 iterations instead of 9);
//   * mel filters through the balanced tap schedule of the tables (see kTapMax).
template <int kLfrM, int kLfrN, int kRows>
__global__ void __launch_bounds__(kWarps * 32, 3)
fbank_tab_kernel(const float* __restrict__ wav, const int32_t* __restrict__ wav_lens, int64_t wav_stride, const float* __restrict__ cmvn,
                 const float* __restrict__ tables, float* __restrict__ feats, int32_t* __restrict__ feat_lens, int t_max,
                 int64_t batch_stride_rows, float wav_scale) {
  constexpr int kFeat = kMel * kLfrM;
  static_assert(kLfrN * (kRows - 1) + kLfrM <= kFramesMax, "too many frames per CTA");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FbankSmemT& s = *reinterpret_cast<FbankSmemT*>(smem_raw);
  const int b = blockIdx.y, i0 = blockIdx.x * kRows;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = wav_lens[b];
  const int m = n >= kWin ? 1 + (n - kWin) / kShift : 0;      // kaldi.py:_get_strided, snip_edges
  const int t_b = (m + kLfrN - 1) / kLfrN;                    // wav_frontend.py:73
  if (blockIdx.x == 0 && tid == 0) feat_lens[b] = t_b;

  float* out = feats + ((int64_t)b * batch_stride_rows + i0) * kFeat;
  if (i0 >= t_b) {  // pure padding rows
    const int rows = min(kRows, t_max - i0);
    for (int idx = tid; idx < rows * kFeat; idx += blockDim.x) out[idx] = 0.f;
    return;
  }
  const int f_lo = max(0, kLfrN * i0 - (kLfrM - 1) / 2);
  const int f_hi = min(m - 1, kLfrN * (i0 + kRows - 1) + (kLfrM - 1) / 2);
  const int nfr = f_hi - f_lo + 1;

  const int n_taps = min(__ldg(reinterpret_cast<const int*>(tables) + kTabTapN), kTapMax);
  for (int j = tid; j < 256; j += blockDim.x) s.tw[j] = make_float2(__ldg(tables + kTabTw + 2 * j), __ldg(tables + kTabTw + 2 * j + 1));
  for (int j = tid; j < kWin; j += blockDim.x) s.win[j] = __ldg(tables + kTabWin + j);
  for (int j = tid; j < n_taps * 32; j += blockDim.x) {
    s.tap_meta[j] = __ldg(reinterpret_cast<const int*>(tables) + kTabTapMeta + j);
    s.tap_w[j] = __ldg(tables + kTabTapW + j);
  }
  __syncthreads();

  float2* Zs = s.zs[warp];
  float* P = s.pw[warp];
  float* macc = s.macc[warp];
  auto twid = [&](int idx) -> float2 {                            // e^{-2 pi i idx / 512}, idx in [0, 512)
    const float2 w = s.tw[idx & 255];
    return idx < 256 ? w : make_float2(-w.x, -w.y);
  };
  LaneTw lt;
#pragma unroll
  for (int k1 = 1; k1 < 8; ++k1) lt.tw8[k1] = twid(2 * lane * k1);   // W_256^{lane k1}
  lt.tw8[0] = make_float2(1.f, 0.f);
#pragma unroll
  for (int st = 0; st < 5; ++st) {                                   // W_{2m}^{lane mod m} in the upper lane of a butterfly, 1 in the lower
    const int mm = 16 >> st;
    lt.twl[st] = (lane & mm) ? twid((lane & (mm - 1)) * (256 / mm)) : make_float2(1.f, 0.f);
  }
  lt.rev = (int)(__brev((unsigned)lane) >> 27);
  const float* wb = wav + (int64_t)b * wav_stride;
  const bool vec2 = ((reinterpret_cast<uintptr_t>(wb) & 7) == 0);     // frames start at multiples of 160 samples
  for (int f = warp; f < nfr; f += kWarps) {
    frame_spectrum(wb + (int64_t)(f_lo + f) * kShift, wav_scale, vec2, s.win, lt, lane, Zs);
    // power spectrum of the real signal: P[k] and P[256 - k] from the same Z[k], Z[256 - k]
    auto Z = [&](int k) -> float2 { return Zs[(k & 7) * kZs + (k >> 3)]; };
    auto pair = [&](int k) {
      const float2 zk = Z(k), zc = Z((256 - k) & 255);
      const float er = 0.5f * (zk.x + zc.x), ei = 0.5f * (zk.y - zc.y);
      const float orr = 0.5f * (zk.y + zc.y), oi = -0.5f * (zk.x - zc.x);
      const float2 w = s.tw[k];
      const float a = w.x * orr - w.y * oi, c = w.x * oi + w.y * orr;            // W_512^k O_k
      const float re1 = er + a, im1 = ei + c, re2 = er - a, im2 = ei - c;          // X[k] = E + W O, X[256-k] = conj(E - W O)
      // |X|^2 directly: the reference's abs().pow(2.0) (:616-618) rounds twice more; the difference (<= 1.5 ulp of P) is two orders
      // below the rounding noise of the transform itself and saves two square-root sequences per pair
      P[k] = re1 * re1 + im1 * im1;
      P[256 - k] = re2 * re2 + im2 * im2;
    };
#pragma unroll
    for (int i = 0; i < 4; ++i) pair(lane + 32 * i);             // k = 0..127 (k = 0 gives P[0] and P[256])
    if (lane == 0) pair(128);
    __syncwarp();
    // mel filters: every lane walks its own tap list; a filter's energy is complete (and stored) on its last tap
    {
      float acc = 0.f;
#pragma unroll 4
      for (int t = 0; t < n_taps; ++t) {
        const int mt = s.tap_meta[t * 32 + lane];
        acc = fmaf(P[mt & 511], s.tap_w[t * 32 + lane], acc);
        if (mt & kTapFlush) { macc[(mt >> 9) & 127] = acc; acc = 0.f; }
      }
    }
    __syncwarp();
    // __logf = lg2.approx * ln 2: <= 2 ulp outside [0.5, 2], 2^-21.4 absolute inside — far inside the 2e-5 log-mel tolerance
    for (int j = lane; j < kMel; j += 32) s.logmel[f * kMel + j] = __logf(fmaxf(macc[j], 1.1920929e-07f));    // :632-633
    __syncwarp();
  }
  __syncthreads();

  // ---- LFR stacking + CMVN, coalesced row stores ----
  const int rows = min(kRows, t_max - i0);
  for (int idx = tid; idx < rows * kFeat; idx += blockDim.x) {
    const int r = idx / kFeat, col = idx - r * kFeat;
    const int i = i0 + r;
    float v = 0.f;
    if (i < t_b) {
      const int j = col / kMel, c = col - j * kMel;
      int fsrc = kLfrN * i - (kLfrM - 1) / 2 + j;
      fsrc = min(max(fsrc, 0), m - 1);
      v = s.logmel[(fsrc - f_lo) * kMel + c];
      if (cmvn != nullptr) v = __fmul_rn(__fadd_rn(v, __ldg(cmvn + col)), __ldg(cmvn + kFeat + col));
    }
    out[idx] = v;
  }
}

// fa_fbank_make_tables: the per-configuration constants, computed once: the non-zero support of each mel filter, its packed
// weights, the FFT twiddles, the window and the tap schedule that fbank_tab_kernel walks
__global__ void fbank_tables_kernel(const float* __restrict__ mel_banks, const float* __restrict__ window, float* __restrict__ tables) {
  __shared__ int s_start[kMel], s_len[kMel], s_off[kMel];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int* ti = reinterpret_cast<int*>(tables);
  for (int j = warp; j < kMel; j += kWarps) {
    const float* row = mel_banks + j * kBins;
    int st = kBins, en = -1;
    for (int k = lane; k < kBins; k += 32) {
      if (row[k] != 0.f) { st = min(st, k); en = max(en, k); }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      st = min(st, __shfl_xor_sync(0xffffffffu, st, o));
      en = max(en, __shfl_xor_sync(0xffffffffu, en, o));
    }
    if (lane == 0) { s_start[j] = en < 0 ? 0 : st; s_len[j] = en < 0 ? 0 : en - st + 1; }
  }
  __syncthreads();
  if (tid == 0) {
    int off = 0;
    for (int j = 0; j < kMel; ++j) { s_off[j] = off; off += s_len[j]; if (off > kMelPackMax) { s_len[j] = 0; off = s_off[j]; } }
  }
  __syncthreads();
  for (int j = tid; j < kMelPackMax; j += blockDim.x) tables[kTabW + j] = 0.f;
  __syncthreads();
  if (tid < kMel) {
    ti[kTabStart + tid] = s_start[tid]; ti[kTabLen + tid] = s_len[tid]; ti[kTabOff + tid] = s_off[tid];
    const float* row = mel_banks + tid * kBins + s_start[tid];
    for (int k = 0; k < s_len[tid]; ++k) tables[kTabW + s_off[tid] + k] = row[k];
  }
  for (int k = tid; k < 256; k += blockDim.x) {
    float sn, cs;
    sincospif((float)k * (1.0f / 256.0f), &sn, &cs);        // e^{-2 pi i k / 512}
    tables[kTabTw + 2 * k] = cs; tables[kTabTw + 2 * k + 1] = -sn;
  }
  for (int j = tid; j < kWin; j += blockDim.x) tables[kTabWin + j] = window[j];
  // tap schedule: filters longest first, each to the least loaded lane (ties: lowest lane); a lane's list = its filters' taps in
  // bin order, the last tap of a filter carries kTapFlush.  Unused slots: bin 0, weight 0.
  for (int j = tid; j < kTapMax * 32; j += blockDim.x) { ti[kTabTapMeta + j] = 0; tables[kTabTapW + j] = 0.f; }
  __syncthreads();
  if (tid == 0) {
    int load[32];
    for (int l = 0; l < 32; ++l) load[l] = 0;
    bool used[kMel];
    for (int j = 0; j < kMel; ++j) used[j] = s_len[j] == 0;        // empty filters: energy 0 -> log(eps), written below
    int max_load = 0;
    for (int it = 0; it < kMel; ++it) {
      int best = -1;
      for (int j = 0; j < kMel; ++j) if (!used[j] && (best < 0 || s_len[j] > s_len[best])) best = j;
      if (best < 0) break;
      used[best] = true;
      int lane = 0;
      for (int l = 1; l < 32; ++l) if (load[l] < load[lane]) lane = l;
      const int len = min(s_len[best], kTapMax - load[lane]);       // a schedule that does not fit drops taps (never with kaldi's banks)
      const float* row = mel_banks + best * kBins + s_start[best];
      for (int k = 0; k < len; ++k) {
        const int slot = (load[lane] + k) * 32 + lane;
        ti[kTabTapMeta + slot] = (s_start[best] + k) | (best << 9) | (k == len - 1 ? kTapFlush : 0);
        tables[kTabTapW + slot] = row[k];
      }
      load[lane] += len;
      max_load = max(max_load, load[lane]);
    }
    // empty filters (none in kaldi's banks) still need their energy written: one zero-weight flush tap each
    for (int j = 0; j < kMel; ++j) {
      if (s_len[j] != 0) continue;
      int lane = 0;
      for (int l = 1; l < 32; ++l) if (load[l] < load[lane]) lane = l;
      if (load[lane] >= kTapMax) continue;
      ti[kTabTapMeta + load[lane] * 32 + lane] = 0 | (j << 9) | kTapFlush;
      load[lane] += 1;
      max_load = max(max_load, load[lane]);
    }
    ti[kTabTapN] = max_load;
  }
}

template <int M, int N, int ROWS>
static int fbank_tab_launch(const float* wav, const int32_t* wav_lens, int batch, int64_t wav_stride, const float* cmvn, const float* tables,
                            float* feats, int64_t stride_rows, int32_t* feat_lens, int t_max, cudaStream_t st, float wav_scale = 32768.0f) {
  const size_t smem = sizeof(FbankSmemT);
  static PerDeviceOnce once;
  FA_RETURN_IF_ERR(ensure_dyn_smem(fbank_tab_kernel<M, N, ROWS>, smem, once));
  dim3 grid((t_max + ROWS - 1) / ROWS, batch);
  fbank_tab_kernel<M, N, ROWS><<<grid, kWarps * 32, smem, st>>>(wav, wav_lens, wav_stride, cmvn, tables, feats, feat_lens, t_max, stride_rows,
                                                                wav_scale);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

// Utterances shorter than one 25 ms frame: the reference shrinks the window to the whole utterance (wav_frontend.py:174:
// frame_length = min(25 ms, len / fs) => window = n samples, ONE frame, FFT size = next power of two of n; kaldi.py:514-647) and the
// LFR stacking of a single frame is that frame repeated lfr_m times.  One CTA, a direct DFT in fp64 (<= 257 bins x 399 samples):
// this is an edge case of a few microseconds, kept off the frame-per-warp kernel whose constants assume the 400 / 512 geometry.
__global__ void __launch_bounds__(256)
fbank_short_kernel(const float* __restrict__ wav, int n, const float* __restrict__ window, const float* __restrict__ mel, int pad,
                   const float* __restrict__ cmvn, int lfr_m, float* __restrict__ out) {
  __shared__ float xs[512], ys[512], pw[257], lm[kMel];
  __shared__ double red[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double part = 0.0;
  for (int j = tid; j < pad; j += blockDim.x) {
    const float v = j < n ? wav[j] * 32768.0f : 0.f;
    xs[j] = v;
    part += (double)v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (lane == 0) red[warp] = part;
  __syncthreads();
  double tot = 0.0;
  for (int w = 0; w < 8; ++w) tot += red[w];
  const float mean = (float)(tot / (double)n);                       // remove_dc_offset kaldi.py:183-186
  for (int j = tid; j < pad; j += blockDim.x) {
    float y = 0.f;
    if (j < n) {
      const float c = __fsub_rn(xs[j], mean), cp = __fsub_rn(xs[j > 0 ? j - 1 : 0], mean);
      y = __fmul_rn(__fsub_rn(c, __fmul_rn(0.97f, cp)), window[j]);  // pre-emphasis (replicate pad) then window :193-204
    }
    ys[j] = y;
  }
  __syncthreads();
  const int bins = pad / 2 + 1;
  for (int k = tid; k < bins; k += blockDim.x) {
    double re = 0.0, im = 0.0;
    for (int j = 0; j < n; ++j) {
      double sn, cs;
      sincospi(2.0 * (double)((k * j) % pad) / (double)pad, &sn, &cs);
      re += (double)ys[j] * cs;
      im -= (double)ys[j] * sn;
    }
    pw[k] = (float)(re * re + im * im);
  }
  __syncthreads();
  for (int j = tid; j < kMel; j += blockDim.x) {
    const float* row = mel + (size_t)j * bins;
    float acc = 0.f;
    for (int k = 0; k < bins; ++k) acc = fmaf(pw[k], row[k], acc);
    lm[j] = logf(fmaxf(acc, 1.1920929e-07f));
  }
  __syncthreads();
  for (int idx = tid; idx < lfr_m * kMel; idx += blockDim.x) {
    float v = lm[idx % kMel];
    if (cmvn != nullptr) v = __fmul_rn(__fadd_rn(v, cmvn[idx]), cmvn[lfr_m * kMel + idx]);
    out[idx] = v;
  }
}

// CAM++ frontend (campplus/utils.py extract_feature: torchaudio kaldi.fbank with its defaults): the waveform is NOT scaled by 32768,
// no LFR stacking (1 / 1), no CMVN; the window (povey) comes with the tables.  feats [B, t_max, 80].
int fbank_unscaled_launch(const float* wav, const int32_t* wav_lens, int batch, int64_t wav_stride, const float* tables, float* feats,
                          int32_t* feat_lens, int t_max, cudaStream_t st) {
  return fbank_tab_launch<1, 1, 48>(wav, wav_lens, batch, wav_stride, nullptr, tables, feats, t_max, feat_lens, t_max, st, 1.0f);
}

}  // namespace fa

extern "C" int fa_fbank_short(const float* wav, int32_t n_samples, const float* window, const float* mel_banks, int32_t padded_fft,
                              const float* cmvn, int32_t lfr_m, float* feats_row, fa_stream_t stream) {
  if (!wav || !window || !mel_banks || !feats_row || n_samples < 2 || n_samples >= fa::kWin || lfr_m < 1 || lfr_m > 16) return FA_ERR_ARG;
  if (padded_fft < n_samples || padded_fft > 512 || (padded_fft & (padded_fft - 1))) return FA_ERR_ARG;
  fa::fbank_short_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(wav, n_samples, window, mel_banks, padded_fft, cmvn, lfr_m, feats_row);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" size_t fa_fbank_tables_bytes(void) { return (size_t)fa::kTabFloats * sizeof(float); }

extern "C" int fa_fbank_make_tables(const float* mel_banks, const float* window, float* tables, fa_stream_t stream) {
  if (!mel_banks || !window || !tables) return FA_ERR_ARG;
  fa::fbank_tables_kernel<<<1, fa::kWarps * 32, 0, (cudaStream_t)stream>>>(mel_banks, window, tables);
  FA_CHECK_LAUNCH();
  return FA_OK;
}

extern "C" int fa_fbank_lfr_cmvn_tables(const float* wav, const int32_t* wav_lens, int32_t batch, int64_t wav_stride, const float* cmvn,
                                        const float* tables, int32_t lfr_m, int32_t lfr_n, float* feats,
                                        int64_t feats_batch_stride_rows, int32_t* feat_lens, int32_t t_max, fa_stream_t stream) {
  if (!wav || !wav_lens || !tables || !feats || !feat_lens || batch <= 0 || t_max <= 0 || feats_batch_stride_rows < t_max) return FA_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (lfr_m == 7 && lfr_n == 6)
    return fa::fbank_tab_launch<7, 6, 8>(wav, wav_lens, batch, wav_stride, cmvn, tables, feats, feats_batch_stride_rows, feat_lens, t_max, st);
  if (lfr_m == 5 && lfr_n == 1)
    return fa::fbank_tab_launch<5, 1, 44>(wav, wav_lens, batch, wav_stride, cmvn, tables, feats, feats_batch_stride_rows, feat_lens, t_max, st);
  return FA_ERR_UNSUPPORTED;
}
