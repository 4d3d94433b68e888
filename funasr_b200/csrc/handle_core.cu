// Core of the handle-style C API (handle.h): the model-file loader, the SAN-M stack binder, the checked audio layout and the upload
// of host PCM in it, and the device gather of recording segments.
#include "handle.h"
#include <stdio.h>
#include <string.h>

namespace {

bool read_exact(FILE* f, void* dst, size_t n) { return fread(dst, 1, n, f) == n; }

__global__ void pcm16_to_f32_kernel(const int16_t* __restrict__ src, float* __restrict__ dst, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (float)src[i] * (1.0f / 32768.0f);     // exact; the frontend multiplies by 32768 again (wav_frontend.py:169)
}

// four consecutive output columns per thread: scalar reads (a segment starts anywhere), one 16-byte store
__global__ void __launch_bounds__(256)
gather_segments_kernel(const float* __restrict__ rec, int64_t n_rec, const int64_t* __restrict__ starts, const int32_t* __restrict__ lens,
                       int64_t stride, float* __restrict__ out) {
  const int r = blockIdx.y;
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (c >= stride) return;
  const int64_t s = starts[r];
  const int32_t len = lens[r];
  float v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int64_t j = c + k, src = s + j;
    v[k] = (j < len && src >= 0 && src < n_rec) ? rec[src] : 0.f;
  }
  *reinterpret_cast<float4*>(out + (int64_t)r * stride + c) = make_float4(v[0], v[1], v[2], v[3]);
}

}  // namespace

namespace fa_handle {

thread_local std::string g_err;

bool sync_stream(cudaStream_t st) {
  if (cudaStreamSynchronize(st) == cudaSuccess) return true;
  set_err(std::string("CUDA error: ") + cudaGetErrorString(cudaGetLastError()));
  return false;
}

bool load_file(std::map<std::string, Tensor>& tensors, const char* path, bool to_device) {
  FILE* f = fopen(path, "rb");
  if (!f) { set_err(std::string("cannot open ") + path); return false; }
  char magic[8];
  uint32_t n = 0;
  long fsize = 0;
  if (fseek(f, 0, SEEK_END) == 0) fsize = ftell(f);
  rewind(f);
  bool ok = fsize > 0 && read_exact(f, magic, 8) && memcmp(magic, "FAB2MDL1", 8) == 0 && read_exact(f, &n, 4);
  std::vector<float> host;
  for (uint32_t i = 0; ok && i < n; ++i) {
    uint32_t nl = 0, nd = 0;
    uint64_t nbytes = 0;
    ok = read_exact(f, &nl, 4) && nl < 4096;
    std::string name(ok ? nl : 0, '\0');
    ok = ok && read_exact(f, &name[0], nl) && read_exact(f, &nd, 4) && nd <= 8;
    Tensor tt;
    tt.shape.resize(nd);
    ok = ok && (nd == 0 || read_exact(f, tt.shape.data(), 8 * nd)) && read_exact(f, &nbytes, 8);
    if (!ok) break;
    const long pos = ftell(f);
    const long pad = (16 - pos % 16) % 16;
    ok = fseek(f, pad, SEEK_CUR) == 0 && nbytes == (uint64_t)tt.numel() * 4 &&
         pos + pad <= fsize && nbytes <= (uint64_t)(fsize - (pos + pad));   // the payload lies inside the file: a corrupt size cannot drive an allocation
    if (!ok) break;
    if (name.compare(0, 2, "__") == 0) {
      tt.host.resize(nbytes / 4);
      ok = read_exact(f, tt.host.data(), nbytes);
    } else if (!to_device) {
      ok = fseek(f, (long)nbytes, SEEK_CUR) == 0;
    } else {
      host.resize(nbytes / 4);
      ok = read_exact(f, host.data(), nbytes);
      if (!ok) break;
      if (cudaMalloc(&tt.dev, nbytes ? nbytes : 4) != cudaSuccess) { ok = false; set_err("cudaMalloc failed for " + name); break; }
      cudaMemcpy(tt.dev, host.data(), nbytes, cudaMemcpyHostToDevice);
    }
    if (!ok) break;
    tensors[name] = tt;
  }
  fclose(f);
  if (!ok && g_err.empty()) set_err(std::string("malformed model file ") + path);
  return ok;
}

// SANMEncoder keeps its first layer (input width -> d_model) apart as encoders0.0 (sanm/encoder.py:188-461); SenseVoice's
// tp_encoders are one plain list
std::string enc_layer_prefix(bool tp, int i) {
  if (tp) return "encoder.tp_encoders." + std::to_string(i);
  return i == 0 ? "encoder.encoders0.0" : "encoder.encoders." + std::to_string(i - 1);
}

// QKV [3D, in], FSMN [D, 1, K] with layer 0's K in every layer, FFN [F, D] / [D, F] with F <= 2048 (enc_carve's bound).  The main
// stack takes the position encoding and ends in encoder.after_norm; SenseVoice's tp stack (D in, possibly empty) in encoder.tp_norm.
void bind_stack(Builder& b, bool tp, int n, int in, int D, int heads, std::vector<FaEncLayer>& L, FaEncoder& e) {
  auto norm = [&](const std::string& p, int64_t w) {
    b.shaped(p + ".weight", {w}); b.shaped(p + ".bias", {w});
    return b.norm(p);
  };
  auto lin = [&](const std::string& p, int64_t out, int64_t k) {
    b.shaped(p + ".weight", {out, k}); b.shaped(p + ".bias", {out});
    return b.lin(p);
  };
  const Tensor* k0 = n > 0 ? b.get(enc_layer_prefix(tp, 0) + ".self_attn.fsmn_block.weight") : nullptr;
  const int64_t K = k0 && k0->shape.size() == 3 ? k0->shape[2] : 0;
  L.assign(n > 0 ? n : 1, FaEncLayer{});
  for (int i = 0; i < n; ++i) {
    const std::string p = enc_layer_prefix(tp, i);
    const int64_t x = i == 0 ? in : D;
    const Tensor* w1 = b.get(p + ".feed_forward.w_1.weight");
    const int64_t F = w1 && w1->shape.size() == 2 ? w1->shape[0] : 0;
    if (w1 && (F < 1 || F > 2048)) b.refuse("bad shape of " + p + ".feed_forward.w_1.weight (at most 2048 units)");
    L[i].norm1 = norm(p + ".norm1", x); L[i].norm2 = norm(p + ".norm2", D);
    L[i].qkv = lin(p + ".self_attn.linear_q_k_v", 3 * D, x); L[i].out = lin(p + ".self_attn.linear_out", D, D);
    b.shaped(p + ".self_attn.fsmn_block.weight", {D, 1, K});
    L[i].fsmn_w = b.ptr(p + ".self_attn.fsmn_block.weight");
    L[i].w1 = lin(p + ".feed_forward.w_1", F, D); L[i].w2 = lin(p + ".feed_forward.w_2", D, F);
  }
  e = FaEncoder{};
  e.layers = L.data(); e.n_layers = n; e.heads = heads; e.fsmn_k = (int)K;
  if (n > 0) e.after_norm = norm(tp ? "encoder.tp_norm" : "encoder.after_norm", D);
  if (!tp) {
    b.shaped("encoder.pe_inv_timescales", {in / 2});
    e.pe_inv_timescales = b.ptr("encoder.pe_inv_timescales");
  }
}

void bind_ts_head(Builder& b, int D, FaTimestampHead& h) {
  const Tensor* tc = b.opt("__ts_config__");
  if (!tc || tc->host.size() < 3) { b.refuse("missing __ts_config__"); return; }
  const float* c = tc->host.data();
  if (c[0] != 3.f) { b.refuse("upsample_times " + std::to_string(c[0]) + " in __ts_config__, only 3 is supported"); return; }
  b.shaped("predictor.upsample_cnn.gemm_weight", {3 * D, D}); b.shaped("predictor.upsample_cnn.gemm_bias", {3 * D});
  b.shaped("predictor.blstm.ih_gemm_weight", {8 * D, D});     b.shaped("predictor.blstm.ih_gemm_bias", {8 * D});
  b.shaped("predictor.blstm.weight_hh_l0", {4 * D, D});       b.shaped("predictor.blstm.weight_hh_l0_reverse", {4 * D, D});
  b.shaped("predictor.cif_output2.weight", {1, 2 * D});       b.shaped("predictor.cif_output2.bias", {1});
  h.up_times = 3; h.smooth2 = c[1]; h.noise2 = c[2];
  h.upsample = b.lin("predictor.upsample_cnn", true, "predictor.upsample_cnn.gemm_weight", "predictor.upsample_cnn.gemm_bias");
  h.blstm_ih = b.lin("predictor.blstm.ih", true, "predictor.blstm.ih_gemm_weight", "predictor.blstm.ih_gemm_bias");
  h.w_hh_fwd = b.ptr("predictor.blstm.weight_hh_l0"); h.w_hh_bwd = b.ptr("predictor.blstm.weight_hh_l0_reverse");
  h.out2_w = b.ptr("predictor.cif_output2.weight"); h.out2_b = b.ptr("predictor.cif_output2.bias");
}

int64_t Audio::frame_bytes() const {
  static const int kBytes[5] = {4, 2, 3, 4, 1};
  return (int64_t)kBytes[fmt.sample_format] * fmt.channels;
}

int64_t Audio::len16(int64_t frames) const {
  if (!tab) return frames;
  if (tab->t.mode == FA_RESAMPLE_LOADER) return ((int64_t)tab->t.out_unit * frames + tab->t.in_unit - 1) / tab->t.in_unit;   // fa_resample's
  return fa_runtime_resample_out_len_host(fmt.sample_rate, 16000, frames);
}

double Audio::seconds(const int64_t* n, int B) const {
  double s = 0.0;
  for (int i = 0; i < B; ++i) s += (double)n[i] / fmt.sample_rate;
  return s;
}

bool plan_audio(const FaAudioFormat* fmt, ResampleCache& cache, Audio& a) {
  if (!fmt) { set_err("audio format is NULL"); return false; }
  const FaAudioFormat f = *fmt;
  if (f.sample_format < 0 || f.sample_format > 4) {
    set_err("bad sample_format " + std::to_string(f.sample_format) + " (0 f32, 1 s16le, 2 s24le, 3 s32le, 4 u8)");
    return false;
  }
  if (f.channels < 1 || f.channels > 64) { set_err("channels " + std::to_string(f.channels) + " outside 1..64"); return false; }
  if (f.resampler != FA_RESAMPLE_LOADER && f.resampler != FA_RESAMPLE_RUNTIME) {
    set_err("bad resampler " + std::to_string(f.resampler) + " (0 FA_RESAMPLE_LOADER, 1 FA_RESAMPLE_RUNTIME)");
    return false;
  }
  if (f.sample_rate < 1000 || f.sample_rate > 192000) {
    set_err("sample rate " + std::to_string(f.sample_rate) + " Hz outside 1000..192000 Hz");
    return false;
  }
  a.fmt = f;
  a.tab = nullptr;
  if (f.sample_rate == 16000) return true;
  const std::pair<int32_t, int32_t> key(f.sample_rate, f.resampler);
  std::lock_guard<std::mutex> lock(cache.mu);        // entries are never removed: a table found stays where it is
  auto it = cache.tables.find(key);
  if (it != cache.tables.end()) { a.tab = &it->second; return true; }
  ResampleTable t;
  FaIngestTable& d = t.t;
  d.mode = f.resampler;
  int64_t need = 0;
  if (f.resampler == FA_RESAMPLE_LOADER) {
    need = fa_loader_resample_table_host(f.sample_rate, 16000, &d.in_unit, &d.out_unit, &d.width, nullptr, 0);
    if (need > 0) {
      d.taps = 2 * d.width + d.in_unit;
      t.weights.resize((size_t)need);
      need = fa_loader_resample_table_host(f.sample_rate, 16000, &d.in_unit, &d.out_unit, &d.width, t.weights.data(), need);
      t.first.assign(d.out_unit, 0); t.n_taps.assign(d.out_unit, 0);
      for (int32_t j = 0; j < d.out_unit; ++j) {     // each row's nonzero span: 34 of 475 taps at 44.1 kHz
        const float* row = t.weights.data() + (size_t)j * d.taps;
        int32_t k0 = 0, k1 = d.taps;
        while (k0 < k1 && row[k0] == 0.0f) ++k0;
        while (k1 > k0 && row[k1 - 1] == 0.0f) --k1;
        t.first[j] = k0; t.n_taps[j] = k1 - k0;
      }
    }
  } else {
    need = fa_runtime_resample_table_host(f.sample_rate, 16000, &d.in_unit, &d.out_unit, &d.taps, nullptr, nullptr, nullptr, 0);
    if (need > 0) {
      t.weights.resize((size_t)need); t.first.resize(d.out_unit); t.n_taps.resize(d.out_unit);
      need = fa_runtime_resample_table_host(f.sample_rate, 16000, &d.in_unit, &d.out_unit, &d.taps, t.first.data(), t.n_taps.data(),
                                            t.weights.data(), need);
    }
  }
  if (need <= 0) {
    set_err("sample rate " + std::to_string(f.sample_rate) + " Hz: its " + (f.resampler == FA_RESAMPLE_LOADER ? "loader" : "runtime") +
            " resampling table to 16 kHz exceeds 32 MiB");
    return false;
  }
  a.tab = &(cache.tables[key] = std::move(t));
  return true;
}

const FaAudioFormat* pcm16k_format(int32_t pcm_format, FaAudioFormat& f) {
  f = FaAudioFormat{pcm_format, 1, 16000, FA_RESAMPLE_LOADER};
  return pcm_format == 0 || pcm_format == 1 ? &f : nullptr;
}

bool upload(const void* const* bufs, const int64_t* n, int B, int64_t stride, const Audio& au, ResampleCache& cache, DevBuf& buf,
            cudaStream_t st, float** wav, float* into) {
  const int64_t tot = (int64_t)B * stride;
  if (au.direct()) {
    const int32_t pcm_format = au.fmt.sample_format;
    int16_t* p16 = nullptr;
    if (!carve(buf, "waveforms", [&](fa::Arena& a) {
          *wav = into ? into : a.take<float>((size_t)(tot > 0 ? tot : 4));
          if (pcm_format == 1) p16 = a.take<int16_t>((size_t)tot);
        }))
      return false;
    if (tot == 0) return true;
    if (pcm_format == 1) {
      for (int i = 0; i < B; ++i) cudaMemcpyAsync(p16 + (int64_t)i * stride, bufs[i], (size_t)n[i] * 2, cudaMemcpyHostToDevice, st);
      pcm16_to_f32_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(p16, *wav, tot);
    } else {
      for (int i = 0; i < B; ++i) cudaMemcpyAsync(*wav + (int64_t)i * stride, bufs[i], (size_t)n[i] * 4, cudaMemcpyHostToDevice, st);
    }
    return true;
  }
  // rows {byte offset, frames, 16 kHz length}; each row's bytes start 16-byte aligned
  std::vector<int64_t>& rows = cache.rows;
  rows.resize((size_t)3 * B);
  int64_t bytes = 0;
  for (int i = 0; i < B; ++i) {
    rows[3 * i] = bytes; rows[3 * i + 1] = n[i]; rows[3 * i + 2] = au.len16(n[i]);
    bytes += (n[i] * au.frame_bytes() + 15) / 16 * 16;
  }
  FaIngestTable t = au.tab ? au.tab->t : FaIngestTable{};
  if (!au.tab) t.mode = -1;
  unsigned char* raw;
  int64_t* rows_d;
  float* w = nullptr;
  int32_t *first = nullptr, *n_taps = nullptr;
  if (!carve(buf, "waveforms", [&](fa::Arena& a) {
        *wav = into ? into : a.take<float>((size_t)(tot > 0 ? tot : 4));
        raw = a.take<unsigned char>((size_t)(bytes > 0 ? bytes : 16));
        rows_d = a.take<int64_t>((size_t)3 * B);
        if (au.tab) w = a.take<float>(au.tab->weights.size());
        if (au.tab && !au.tab->first.empty()) { first = a.take<int32_t>(au.tab->first.size()); n_taps = a.take<int32_t>(au.tab->n_taps.size()); }
      }))
    return false;
  if (tot == 0) return true;
  // pageable host sources: each copy returns once its bytes are staged, so rows and the cached tables may change after it
  for (int i = 0; i < B; ++i) cudaMemcpyAsync(raw + rows[3 * i], bufs[i], (size_t)(n[i] * au.frame_bytes()), cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(rows_d, rows.data(), rows.size() * 8, cudaMemcpyHostToDevice, st);
  if (au.tab) {
    cudaMemcpyAsync(w, au.tab->weights.data(), au.tab->weights.size() * 4, cudaMemcpyHostToDevice, st);
    t.weights = w;
    if (first) {
      cudaMemcpyAsync(first, au.tab->first.data(), au.tab->first.size() * 4, cudaMemcpyHostToDevice, st);
      cudaMemcpyAsync(n_taps, au.tab->n_taps.data(), au.tab->n_taps.size() * 4, cudaMemcpyHostToDevice, st);
      t.first = first; t.n_taps = n_taps;
    }
  }
  const int rc = fa_ingest_pcm(raw, rows_d, B, au.fmt.sample_format, au.fmt.channels, &t, *wav, stride, st);
  if (rc != FA_OK) { set_err(std::string("fa_ingest_pcm: ") + fa_status_string(rc)); return false; }
  return true;
}

bool gather(const float* rec, int64_t n, const int64_t* starts, const int32_t* lens, int rows, int64_t stride, int64_t* starts_d,
            int32_t* lens_d, float* out, cudaStream_t st) {
  cudaMemcpyAsync(starts_d, starts, (size_t)rows * 8, cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(lens_d, lens, (size_t)rows * 4, cudaMemcpyHostToDevice, st);
  const int rc = fa_gather_segments(rec, n, starts_d, lens_d, rows, stride, out, st);
  if (rc != FA_OK) { set_err(std::string("fa_gather_segments: ") + fa_status_string(rc)); return false; }
  return true;
}

}  // namespace fa_handle

extern "C" const char* fa_offline_last_error(void) { return fa_handle::g_err.c_str(); }

extern "C" int fa_gather_segments(const float* rec, int64_t n_rec, const int64_t* starts, const int32_t* lens, int32_t rows, int64_t stride,
                                  float* out, fa_stream_t stream) {
  if (rows < 0 || rows > 65535 || n_rec < 0 || (rows > 0 && (!rec || !starts || !lens || !out || stride <= 0))) return FA_ERR_ARG;
  if (rows == 0) return FA_OK;
  if (stride % 4 || reinterpret_cast<uintptr_t>(out) % 16) return FA_ERR_UNSUPPORTED;
  const int64_t blocks = (stride / 4 + 255) / 256;
  if (blocks > 0x7fffffffLL) return FA_ERR_ARG;
  gather_segments_kernel<<<dim3((unsigned)blocks, (unsigned)rows), 256, 0, (cudaStream_t)stream>>>(rec, n_rec, starts, lens, stride, out);
  FA_CHECK_LAUNCH();
  return FA_OK;
}
