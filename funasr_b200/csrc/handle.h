// Internal core of the handle-style C API (never included by include/): the error string every handle kind reports through
// fa_offline_last_error, the model-file loader, the two-pass Builder, the grow-only device buffers each call carves its memory from,
// and the handle structs and functions that cross files (long audio runs the recogniser, the VAD and the speaker model).
//
//   handle_core.cu   file loader, Builder, plan_audio / upload (pcm16_to_f32_kernel, fa_ingest_pcm), fa_gather_segments
//   offline_asr.cu   recogniser (Paraformer, contextual, BiCif, SeACo, SenseVoice): fa_offline_*
//   offline_vad.cu   FSMN-VAD: fa_vad_*
//   offline_spk.cu   CAM++ speaker embeddings, clustering, diarization, and the speaker handle's request pool: fa_spk_*
//   offline_long.cu  long audio: fa_offline_infer_vad*, fa_offline_result_{segments,spk}
//   offline_pool.cu  the recogniser's request pool: every decoding call's passes, GPU packs and scatter; fa_offline_pool_stats
//   offline_punc.cu  CT-Transformer punctuation and its request pool (concurrent calls share lockstep steps): fa_punc_*
//   offline_align.cu MonotonicAligner (fa-zh) forced alignment: fa_align_*
#pragma once
#include "common.cuh"
#include "request_pool.h"
#include <algorithm>
#include <atomic>
#include <exception>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

// hidden: nothing here is part of the library's exported interface (include/funasr_b200.h)
namespace __attribute__((visibility("hidden"))) fa_handle {

extern thread_local std::string g_err;
inline void set_err(const std::string& s) { g_err = s; }
inline std::nullptr_t fail(const std::string& s) { set_err(s); return nullptr; }

// f() with every C++ exception turned into an error message: none may cross the C ABI (a malformed file can ask for an absurd
// allocation)
template <typename F>
bool no_throw(const char* what, F f) {
  try {
    return f();
  } catch (const std::exception& e) {
    set_err(std::string(what) + e.what());
    return false;
  }
}

// the stream's work finished, or "CUDA error: ..." set
bool sync_stream(cudaStream_t st);

inline bool valid_gemm_mode(int mode) {
  return mode == FA_GEMM_F32_SIMT || mode == FA_GEMM_F16X1 || mode == FA_GEMM_F16X3 || mode == FA_GEMM_F16X6;
}

struct Tensor {
  float* dev = nullptr;              // weights
  std::vector<float> host;           // the payload of the "__" configuration tensors, which stay on the host
  std::vector<int64_t> shape;
  int64_t numel() const { int64_t n = 1; for (auto d : shape) n *= d; return n; }
};

// Grow-only device allocation.  Growing frees the old block, so each DevBuf is carved by exactly one function (carve below); a callee
// that needs memory carves a DevBuf of its own, and device data passes between functions as pointers.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  bool reserve(size_t n) {
    if (n <= cap) return true;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    const size_t want = n + n / 8 + 4096;
    if (cudaMalloc(&p, want) != cudaSuccess) { cudaGetLastError(); return false; }
    cap = want;
    return true;
  }
  ~DevBuf() { if (p) cudaFree(p); }
};

// One stage's device buffers out of d: c(Arena&) takes them, run once measuring, d grown to that size, then once over d.  false:
// "device allocation failed (<stage>)" set.
template <typename C>
bool carve(DevBuf& d, const char* stage, C c) {
  fa::Arena m = fa::Arena::measuring();
  c(m);
  if (!d.reserve(m.bytes())) { set_err(std::string("device allocation failed (") + stage + ")"); return false; }
  fa::Arena a(d.p, d.cap);
  c(a);
  return true;
}

// File layout (funasr_b200/pack.py): "FAB2MDL1", u32 n_tensors, then per tensor:
//   u32 name_len, name, u32 ndim, i64 dims[ndim], u64 nbytes, zero padding to a 16-byte file offset, fp32 data
// The payload of a "__" configuration tensor is read into Tensor::host.  to_device = false skips the weights (names and shapes
// only): what can be checked before any device is touched.
bool load_file(std::map<std::string, Tensor>& tensors, const char* path, bool to_device = true);

// One model file loaded onto one device: its tensors, what the handle allocates beside them (weight planes, padded weights, the
// fbank tables), and the handle's stream
struct Loaded {
  int device = 0;
  std::map<std::string, Tensor> t;
  std::vector<void*> owned;
  cudaStream_t st = nullptr;
  float* fbank_tables = nullptr;
  bool open(const char* path, int dev) {
    if (cudaSetDevice(dev) != cudaSuccess) { cudaGetLastError(); set_err("no such CUDA device (this library has no CPU path)"); return false; }
    device = dev;
    if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) { set_err("cudaStreamCreate failed"); return false; }
    return load_file(t, path);
  }
  // device memory freed with the handle; nullptr if cudaMalloc fails
  void* alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr;
    owned.push_back(p);
    return p;
  }
  ~Loaded() {
    for (auto& kv : t) if (kv.second.dev) cudaFree(kv.second.dev);
    for (void* p : owned) cudaFree(p);
    if (st) cudaStreamDestroy(st);
  }
};

// One model kind's description, run twice: over the file's index (f == nullptr: names and shapes only, nothing touches a device),
// then over the loaded file.  A file the index pass accepts is refused later only for a device failure.
struct Builder {
  const std::map<std::string, Tensor>& t;
  Loaded* f;                                         // nullptr: the index pass
  int mode = FA_GEMM_F32_SIMT;
  float ln_eps = 0.f;
  std::string what;                                  // prefix of every message: the model kind or the part being bound
  bool ok = true;                                    // the first refusal is the one reported
  bool refuse(const std::string& s) {
    if (ok) set_err(what + s);
    ok = false;
    return false;
  }
  const Tensor* opt(const std::string& k) const {
    auto it = t.find(k);
    return it == t.end() ? nullptr : &it->second;
  }
  const Tensor* get(const std::string& k) {
    const Tensor* x = opt(k);
    if (!x) refuse("missing tensor " + k);
    return x;
  }
  const Tensor* shaped(const std::string& k, std::initializer_list<int64_t> dims) {
    const Tensor* x = get(k);
    if (x && !std::equal(dims.begin(), dims.end(), x->shape.begin(), x->shape.end())) refuse("bad shape of " + k);
    return x;
  }
  const float* ptr(const std::string& k) { const Tensor* x = get(k); return x ? x->dev : nullptr; }   // nullptr on the index
  FaNorm norm(const std::string& p) {
    FaNorm nm{};
    const Tensor* w = get(p + ".weight");
    nm.g = w ? w->dev : nullptr; nm.b = ptr(p + ".bias"); nm.n = w ? (int32_t)w->numel() : 0; nm.eps = ln_eps;
    return nm;
  }
  FaLinear lin(const std::string& p, bool bias = true, const char* weight_key = nullptr, const char* bias_key = nullptr) {
    FaLinear L{};
    const Tensor* w = get(weight_key ? std::string(weight_key) : p + ".weight");
    // [out, in] or a k = 1 Conv1d weight [out, in, 1] (bias_output, contextual_paraformer/decoder.py:287)
    if (!w || !(w->shape.size() == 2 || (w->shape.size() == 3 && w->shape[2] == 1))) { if (w) refuse("bad weight " + p); return L; }
    L.w = w->dev; L.b = bias ? ptr(bias_key ? std::string(bias_key) : p + ".bias") : nullptr;
    L.out_f = (int32_t)w->shape[0]; L.in_f = (int32_t)w->shape[1]; L.in_pad = (L.in_f + 63) / 64 * 64;
    if (mode != FA_GEMM_F32_SIMT && f) split_planes(L);
    return L;
  }
  // L's fp16 planes for the tensor-core GEMMs, owned by the loaded file
  void split_planes(FaLinear& L) {
    void* planes = f->alloc((size_t)3 * L.out_f * L.in_pad * 2);
    if (!planes) { refuse("cudaMalloc planes"); return; }
    if (fa_split_planes(L.w, L.in_f, L.out_f, L.in_f, L.in_pad, planes, f->st) != FA_OK) refuse("fa_split_planes failed");
    L.w_planes = planes;
  }
  // the frontend's fbank tables (fa_fbank_make_tables) from frontend.mel_banks and frontend.window
  void fbank_tables() {
    const Tensor* mel = get("frontend.mel_banks");
    const Tensor* win = get("frontend.window");
    if (!mel || !win || !f) return;
    f->fbank_tables = static_cast<float*>(f->alloc(fa_fbank_tables_bytes()));
    if (!f->fbank_tables) { refuse("cudaMalloc fbank tables"); return; }
    if (fa_fbank_make_tables(mel->dev, win->dev, f->fbank_tables, f->st) != FA_OK) refuse("fa_fbank_make_tables failed");
  }
};

// fa_offline_init / fa_vad_init / fa_punc_init / fa_spk_init: build() over the file's index into a throwaway handle (every refusal
// before any device work, naming the piece), then over the loaded file into the handle returned
template <typename H>
H* open_handle(const char* path, int device, int mode, bool (*build)(H&, Builder&)) {
  if (!path) return fail("model_file is NULL");
  std::unique_ptr<H> h;
  const bool ok = no_throw("model file rejected: ", [&] {
    std::map<std::string, Tensor> index;
    H probe;
    Builder on_index{index, nullptr, mode};
    if (!load_file(index, path, false) || !build(probe, on_index)) return false;
    h.reset(new H());
    Builder on_device{h->file.t, &h->file, mode};
    return h->file.open(path, device) && build(*h, on_device) && sync_stream(h->file.st);
  });
  return ok ? h.release() : nullptr;
}

// LFR frames of n 16 kHz samples (wav_frontend.py:73 after kaldi.py snip_edges framing)
inline int num_lfr_frames(int64_t n) {
  const int64_t mfr = n >= 400 ? 1 + (n - 400) / 160 : 0;
  return (int)((mfr + 5) / 6);
}

// SANMEncoder's layer names: encoders0.0 then encoders.{i - 1}; SenseVoice's tp_encoders one plain list
std::string enc_layer_prefix(bool tp, int i);

// A SAN-M stack of n layers over `in` input features into e and L, in the shapes fa_sanm_encoder_forward takes (the recogniser's
// encoders and punctuation's)
void bind_stack(Builder& b, bool tp, int n, int in, int D, int heads, std::vector<FaEncLayer>& L, FaEncoder& e);

// CifPredictorV3's upsampled timestamp head at width D into h: __ts_config__ (upsample_times 3, smooth_factor2, noise_threshold2) and
// the tensors pack.py:timestamp_head_tensors writes, in their shapes; h.threshold is the caller's.  Every refusal is prefixed by b.what
// (the BiCif recogniser's and the aligner's).
void bind_ts_head(Builder& b, int D, FaTimestampHead& h);

// ------------------------------------------------------------------------------------------------ audio in (FaAudioFormat)
// One (rate, resampler)'s host tables; fa_ingest_pcm reads their device copy
struct ResampleTable {
  FaIngestTable t{};                                 // the shape; the device pointers are set per upload
  std::vector<float> weights;
  std::vector<int32_t> first, n_taps;                // runtime: each phase's first input index and taps; loader: each row's nonzero span
};

// A handle's resampling tables keyed by (rate, resampler), built on the host when first needed and kept (grow-only, like its
// buffers), and the host rows of the last upload
struct ResampleCache {
  std::mutex mu;                                     // plan_audio's lookup and insertion: callers check their format concurrently
  std::map<std::pair<int32_t, int32_t>, ResampleTable> tables;
  std::vector<int64_t> rows;                         // written by upload, under the handle's device lock
};

// The caller's audio layout, checked, with its table (nullptr at 16 kHz)
struct Audio {
  FaAudioFormat fmt{};
  const ResampleTable* tab = nullptr;
  // 16 kHz mono f32 / s16: the upload the 16 kHz entries always had (a copy, or the s16 conversion kernel)
  bool direct() const { return fmt.sample_rate == 16000 && fmt.channels == 1 && (fmt.sample_format == 0 || fmt.sample_format == 1); }
  int64_t frame_bytes() const;
  int64_t len16(int64_t frames) const;               // the 16 kHz samples of `frames` frames
  double seconds(const int64_t* n, int B) const;     // the caller's frames at the caller's rate
  std::string at16k() const { return fmt.sample_rate == 16000 ? "" : " at 16 kHz"; }
};

// fmt checked (NULL, sample_format, channels 1..64, resampler, rate 1 000..192 000, a table above 32 MiB) and its table built or
// found in cache; false: the refusal set, nothing touched a device
bool plan_audio(const FaAudioFormat* fmt, ResampleCache& cache, Audio& a);
// f = the descriptor of a 16 kHz entry's pcm_format; &f for 0 (f32) and 1 (s16le), NULL for any other value (a bad argument)
const FaAudioFormat* pcm16k_format(int32_t pcm_format, FaAudioFormat& f);

// B host recordings bufs[i] of n[i] frames in a's layout into 16 kHz rows of `stride` floats, *wav, carved from buf with the staged
// bytes and the table: direct() as the 16 kHz entries always did, otherwise one fa_ingest_pcm launch.  into: write the rows there
// ([B, stride] on the device) instead, buf holding only the staged bytes and the table.
bool upload(const void* const* bufs, const int64_t* n, int B, int64_t stride, const Audio& a, ResampleCache& cache, DevBuf& buf,
            cudaStream_t st, float** wav, float* into = nullptr);

// rows segments of the device recording rec [n]: the host starts / lengths (samples) copied into starts_d / lens_d, then
// fa_gather_segments into out [rows, stride] with zero tails.  The caller keeps the host arrays alive until the stream passes them.
bool gather(const float* rec, int64_t n, const int64_t* starts, const int32_t* lens, int rows, int64_t stride, int64_t* starts_d,
            int32_t* lens_d, float* out, cudaStream_t st);

// rows[index] with *n = its size / width; a NULL result or an index out of range: *n = 0 and NULL, an empty row as well unless
// keep_empty
template <typename T>
const T* result_row(const std::vector<std::vector<T>>* rows, int32_t index, int32_t* n, int width, bool keep_empty) {
  if (!rows || index < 0 || index >= (int32_t)rows->size() || ((*rows)[index].empty() && !keep_empty)) { if (n) *n = 0; return nullptr; }
  if (n) *n = (int32_t)((*rows)[index].size() / width);
  return (*rows)[index].data();
}

// ------------------------------------------------------------------------------------------------ handles that cross files
// Any handle may be shared by many threads.  Each handle has a device lock (`mu`), held by a call for all of its work on the handle's
// stream and buffers; argument checks run before it is taken.  A call that needs several handles takes their locks in one order,
// recogniser -> VAD -> speaker (-> punctuation, aligner: never held with another), so two recognisers sharing a VAD cannot deadlock.
// The recogniser's decoding calls, speaker-only calls (fa_spk_embed*, fa_spk_cluster) and punctuation calls do not take `mu`
// themselves: they post a ticket to their handle's request pool (request_pool.h), whose leading thread runs rounds over every
// caller's tickets, each round taking the device locks it needs.  A recogniser round is one pass that decodes the queued compatible
// calls in shared GPU packs under the recogniser, VAD and speaker locks (offline_pool.cu); a speaker round is one pass under the
// speaker lock alone (offline_spk.cu); a punctuation round is one lockstep step under the punctuation lock (offline_punc.cu).  A
// recogniser's diarized pass takes the speaker lock directly (diarize), after the recogniser and VAD locks, so it and the speaker
// pool's passes interleave at pass boundaries and cannot deadlock.
struct Vad;
struct Spk;
struct SpkTicket;
struct Result;

// One call of fa_offline_infer* (an utterance batch) or fa_offline_infer_vad* (long audio), its arguments checked, waiting in the pool
struct Ticket : PoolTicket {
  const void* const* bufs = nullptr;
  const int64_t* n_samples = nullptr;                // the caller's frames
  int batch = 0;
  Audio au;
  std::vector<int64_t> n16;                          // 16 kHz samples per buffer
  const float* hw_embed = nullptr;                   // hotword rows [n_hotwords, 512] on the host
  int32_t n_hotwords = 0;
  int hw_set = -1;                                   // the pass's index of its hotword rows (identical rows: one set), -1 without
  const int32_t *lang = nullptr, *tn = nullptr;      // SenseVoice queries per buffer (NULL: the defaults)
  bool long_audio = false;                           // fa_offline_infer_vad*: VAD, then packs of each recording's segments
  Vad* vad = nullptr;
  FaLongAudioOptions opts{};
  Spk* spk = nullptr;                                // diarized: shares a pass only with the same speaker handle, or none
  int32_t preset_spk_num = 0;
  std::unique_ptr<Result> res;                       // written by the pass, read by the owner once done
};

struct Model {
  std::mutex mu;
  Loaded file;
  int mode = 3;
  int enc_layers = 0, dec_layers = 0, d_model = 512, heads = 4, kernel = 11, vocab = 0, feat_dim = 560;
  float ln_eps = 1e-12f, cif_threshold = 1.f, tail_threshold = 0.45f;
  std::vector<FaEncLayer> enc_l;
  std::vector<FaDecLayer> dec_l;
  FaEncoder enc{};
  FaPredictor pred{};
  FaDecoder dec{};
  const float* cmvn = nullptr;
  bool contextual = false;                           // ContextualParaformer: decoder with a hotword bias branch
  bool ts = false;                                   // BiCifParaformer: CifPredictorV3's upsampled timestamp head
  FaTimestampHead head{};
  std::mutex host_cache_mu;                          // host_cache alone: host readers do not wait for a decode on the handle
  std::map<std::string, std::vector<float>> host_cache;   // fa_offline_host_tensor
  bool sv = false;                                   // SenseVoiceSmall (__sv_config__): query rows, the SAN-M and tp stacks, the CTC head
  int tp_layers = 0, n_embed = 0, blank = 0;
  std::vector<FaEncLayer> tp_l;
  FaEncoder tp{};
  FaLinear ctc{};
  const float* embed = nullptr;
  bool seaco = false;                                // SeacoParaformer (__seaco_config__): hotword encoder, SeACo decoder, NO_BIAS merge
  int no_bias = 0, nfilter = 0;
  std::vector<FaDecLayer> seaco_l;
  FaDecoder seaco_dec{};
  FaLinear hw_out{};
  std::vector<FaLinear> hw_ih, hw_hh;
  FaHotwordEncoder hw_enc{};
  // device memory, each DevBuf carved by the function it is named after
  ResampleCache resample;
  DevBuf upload;                                     // the host batch of fa_offline_infer*, the recording of long audio
  DevBuf encode, decode, seaco_bias, decode_sv;      // decode_batch before and after its token-count sync; seaco_bias; decode_sv
  DevBuf hotword_embed;                              // fa_offline_hotword_embed's rows
  DevBuf pool_recs;                                  // a pass's recordings and utterances, one row each (pool_group)
  DevBuf pack;                                       // pool_group: one GPU pack's gather offsets and padded rows
  DevBuf ws;                                         // the GEMM workspace every stage above uses in turn
  RequestPool<Ticket> pool;                          // each round one pass (offline_pool.cu)
  std::atomic<int64_t> pool_packs{0};                // GPU packs decoded since init
};

struct Result {
  std::vector<std::vector<int32_t>> ids;
  std::vector<int32_t> token_num;
  std::vector<std::vector<int32_t>> segs;            // fa_offline_infer_vad: {start_ms, end_ms, n_tokens} per segment, per recording
  bool ts = false;                                   // the model has the timestamp head: stamps[i] = {start_ms, end_ms} pairs
  std::vector<std::vector<int32_t>> stamps;
  std::vector<std::vector<int32_t>> spk;             // fa_offline_infer_vad_spk: one speaker per segment of a diarized recording
  float audio_seconds = 0.f;
};

const int32_t kSvAuto = 0, kSvWoItn = 15;            // SenseVoiceSmall.inference's defaults: language "auto", text norm "woitn"

// a contextual model's hotword memory (at least the <s> entry) or a SeACo model's rows, as the caller passed them
bool check_hotword_rows(const Model& m, const float* hw_embed, int32_t n_hotwords);
// every query id inside the embedding table; `what` names the unit ("utterance", "recording")
bool check_queries(const Model& m, const int32_t* lang, const int32_t* tn, int n, const char* what);
// A GPU pack's hotword rows: its distinct host row sets, and per reference pack (rows the reference decodes as one batch, contiguous
// in the GPU pack) its first row, row count and set (-1: the call passed none, a SeACo call decoded without biasing)
struct PackHotwords {
  std::vector<const float*> rows;                    // per set: [n[s], 512] on the host
  std::vector<int32_t> n;
  struct Ref { int first, count, set; };
  std::vector<Ref> refs;
};
// one padded batch on the device (wav [B, stride], lens_h >= 400 samples each) decoded by the handle's model kind: the hotword memories
// reach a contextual or SeACo Paraformer (hw: NULL or no reference pack with a set = none), the queries (per row, NULL = the defaults)
// a SenseVoice model.  ext_h [B]: each row's padded length in LFR frames, the t_max of the batch the reference decodes it in
// (num_lfr_frames(lens_h[b]) <= ext_h[b]); the CIF predictor and the timestamp head give row b exactly what that batch gives it, and
// each reference pack's hotword biasing is the one the reference gives that batch.
std::unique_ptr<Result> decode_pack(Model& m, const float* wav, int64_t stride, const std::vector<int32_t>& lens_h, const std::vector<int32_t>& ext_h,
                                    const PackHotwords* hw, const int32_t* lang, const int32_t* tn);
// t's call through the recogniser's request pool: queued, decoded by whichever thread leads the pass that admits it -> its result, or
// nullptr with its own message set as this thread's error
void* pool_call(Model& m, Ticket& t);

struct Vad {
  std::mutex mu;
  Loaded file;
  std::vector<FaVadLayer> layers;
  FaVadEncoder enc{};
  FaVadOptions opts{};
  const float* cmvn = nullptr;
  ResampleCache resample;
  DevBuf upload;                                     // fa_vad_infer's recording
  DevBuf vad_run;
};

struct VadResult {
  std::vector<int32_t> seg;                          // {start_ms, end_ms} pairs
  std::vector<float> frames;                         // [2][frames]: silence posterior, frame energy
  float audio_seconds = 0.f;
};

FaVadRunOptions default_vad_run();
// VAD of one device-resident recording wav [n] fp32 on stream st (the VAD's own, or the recogniser's in long audio)
bool vad_run(Vad& v, const float* wav, int64_t n, cudaStream_t st, const FaVadRunOptions& ro, VadResult& out);
// The same for B device-resident recordings wav [B, stride] of n[i] samples in one batched pass (fa_fsmn_vad_forward_batch,
// fa_frame_decibels_batch, one copy back), each recording's end points then walked on its own -> out[i], equal to vad_run on it
bool vad_run_batch(Vad& v, const float* wav, int64_t stride, const int64_t* n, int B, cudaStream_t st, const FaVadRunOptions& ro,
                   std::vector<VadResult>& out);

struct Spk {
  std::mutex mu;
  Loaded file;
  int mode = FA_GEMM_F32_SIMT;
  FaCampplus model{};
  std::vector<FaCamLayer> layers;
  ResampleCache resample;
  DevBuf upload;                                     // fa_spk_embed's batch
  DevBuf embed, cluster_input;                       // a pass's lengths and embeddings; its clustering calls' embeddings
  DevBuf pool_recs;                                  // one embedding pack's recordings when it holds several calls, one row each
  DevBuf spk_embed_rows, diarize, spk_cluster;
  RequestPool<SpkTicket> pool;                       // each round one pass of speaker-only calls (offline_spk.cu)
  std::atomic<int64_t> pool_passes{0};               // passes run since init
};

// One recording of the speaker stage: recs[off, off + n) of the stage's device buffer, its {start_ms, end_ms, n_tokens} segments and
// its preset count (<= 0: none) -> one speaker per segment in *spk, or its own refusal in err (named by the prefix what)
struct SpkJob {
  int64_t off = 0, n = 0;
  const std::vector<int32_t>* segs = nullptr;
  int preset = 0;
  std::string what;
  std::vector<int32_t>* spk = nullptr;
  std::string err;
};
// LongAudioPipeline.generate's diarization of many device-resident recordings at once (recs [n_recs], complete), on the speaker
// handle's stream: every recording gets what it gets alone, and a refusal (a preset above the chunk count, 2048 or more chunks without
// one) fails only its own job.  false: a device failure, with the message set.
bool diarize(Spk& s, const float* recs, int64_t n_recs, std::vector<SpkJob>& jobs);

}  // namespace fa_handle
