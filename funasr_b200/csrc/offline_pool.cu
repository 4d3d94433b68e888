// The recogniser's request pool: concurrent calls on one handle decoded in shared GPU packs, each call getting exactly what it gets alone.
//
// The reference decodes a call's utterances as one batch, and a long recording's VAD segments in packs of its own (fa_merge_vad,
// fa_pack_segments).  Its CIF predictor and timestamp head read past a row's end, up to the padded length of the batch the row is in
// (DESIGN §6), so a row's result is a function of its audio and of that one number, its extent ext.  decode_pack takes ext per row.
// Rows of many calls can therefore share one pack: each row carries the extent of the batch the reference would decode it in, its
// "reference pack".
//
// A call posts a Ticket to the handle's request pool (request_pool.h).  Each round of the pool's leader is one pass: it admits the
// head of the queue and the later compatible tickets in arrival order (up to an hour of padded audio), takes the device locks and,
// per group of rows:
//   uploads every recording and utterance batch into one buffer, runs one batched VAD pass over the long-audio recordings,
//   forms each call's reference packs and their extents, merges reference packs of different calls into GPU packs (sorted by extent,
//   at most kPackSamples of padded audio, a larger reference pack alone), decodes each, and scatters the rows back.
// Pack-level rules of the reference (a long-audio pack without a token empties its recording) apply per reference pack.  Every ticket
// of a pass ends with it.
//
// Hotword calls (contextual and SeACo Paraformer) pool like any other: the reference gives every utterance of a batch the same hotword
// memory, and for SeACo with more rows than nfilter the attention-score filter of the batch's utterance 0, so the memory belongs to the
// reference pack.  decode_pack takes each reference pack's rows and set; identical sets within a pass (the same count and the same
// bytes: a server-wide list) are one set, projected once per GPU pack.
//
// Diarized calls pool too: their reference packs merge like any other, and once a group's recordings are assembled one speaker stage
// (diarize) embeds and clusters all of its diarized recordings together; each recording is still clustered on its own, as the
// reference's ClusterBackend does, and a refusal of the stage fails only its own call.
#include "handle.h"
#include <string.h>

using namespace fa_handle;

namespace {

// padded 16 kHz samples a pass drains and one group uploads at once: an hour of audio (230 MB of fp32 rows)
const int64_t kVadGroupSamples = 3600LL * 16000;
// padded 16 kHz samples of a GPU pack merged from several calls' reference packs: 300 s, the reference's default batch_size_s
const int64_t kPackSamples = 300LL * 16000;
// hotword memory rows of a GPU pack: (distinct sets + reference packs the SeACo filter runs on) x the longest set.  A reference pack
// over it decodes alone; 4096 rows are 16 MB of bias k|v.
const int64_t kPackHotwordRows = 4096;

int64_t padded(int64_t n) { return (n + 3) / 4 * 4; }

bool same_opts(const FaLongAudioOptions& a, const FaLongAudioOptions& b) {
  return a.batch_size_s == b.batch_size_s && a.batch_size_threshold_s == b.batch_size_threshold_s && a.merge_vad == b.merge_vad &&
         a.merge_length_s == b.merge_length_s && a.vad.dynamic_silence == b.vad.dynamic_silence &&
         a.vad.max_end_silence_time == b.vad.max_end_silence_time && memcmp(&a.vad.speech_noise_thres, &b.vad.speech_noise_thres, sizeof(double)) == 0;
}

int64_t ticket_samples(const Ticket& t) {
  int64_t s = 0;
  for (int64_t n : t.n16) s += padded(n);
  return s;
}

// A pass's admission: the head of the queue and every later ticket that may share its packs, in arrival order, until an hour of padded
// audio.  Long-audio tickets share a pass only with the same VAD handle and options, diarized tickets only with the same speaker handle
// (a pass takes at most one speaker lock); the others stay queued for a later pass.
void admit(std::deque<Ticket*>& queue, std::vector<Ticket*>& pass) {
  const Ticket* key = nullptr;
  Spk* spk = nullptr;
  int64_t samples = 0;
  for (auto it = queue.begin(); it != queue.end();) {
    Ticket* c = *it;
    if ((c->long_audio && key && (c->vad != key->vad || !same_opts(c->opts, key->opts))) || (c->spk && spk && c->spk != spk)) { ++it; continue; }
    const int64_t s = ticket_samples(*c);
    if (!pass.empty() && samples + s > kVadGroupSamples) break;
    samples += s;
    if (c->long_audio && !key) key = c;
    if (c->spk && !spk) spk = c->spk;
    pass.push_back(c);
    it = queue.erase(it);
  }
}

// rows the reference decodes together: a call's utterance batch, or one pack of one recording's VAD segments
struct RefPack {
  Ticket* t;
  std::vector<int64_t> starts;                       // in the group's buffer
  std::vector<int32_t> lens, lang, tn;               // 16 kHz samples, SenseVoice queries
  int ext = 0;                                       // LFR frames of its longest row
  int64_t lmax = 0;
  int set = -1;                                      // its call's hotword set in the pass (-1: none)
  std::string bad;                                   // long audio: a segment under 400 samples, reported if the recording reaches it
  std::unique_ptr<Result> out;                       // its rows, scattered from the GPU pack
};

// a long-audio recording of a group: its segments, their pack order and its reference packs in the reference's order
struct LongRec {
  Ticket* t;
  int i, row;
  std::vector<int32_t> segs, order;
  std::vector<int> packs;
};

// a slice of one ticket's buffers: a whole utterance batch, or one long-audio recording
struct Unit { Ticket* t; int first, count; };

bool pool_group(Model& m, const std::vector<Unit>& units, int64_t stride, const PackHotwords& sets) {
  cudaStream_t st = m.file.st;
  // rows: long-audio recordings first (one batched VAD pass reads them as [nl, stride]), then the utterance batches
  std::vector<int> row(units.size());
  int rows = 0, nl = 0;
  for (int pass_long = 1; pass_long >= 0; --pass_long)
    for (size_t u = 0; u < units.size(); ++u)
      if (units[u].t->long_audio == (pass_long == 1)) { row[u] = rows; rows += units[u].count; nl += pass_long ? units[u].count : 0; }
  // one unit (a lone caller): its upload is the group's buffer, as the take-turns path decoded from it; several: each written into it
  float* recs = nullptr;
  if (units.size() > 1 &&
      !carve(m.pool_recs, "recordings", [&](fa::Arena& a) { recs = a.take<float>((size_t)std::max<int64_t>((int64_t)rows * stride, 4)); }))
    return false;
  std::vector<int64_t> n_long;
  Vad* vad = nullptr;
  FaVadRunOptions vro{};
  for (size_t u = 0; u < units.size(); ++u) {
    const Unit& un = units[u];
    float* into = recs ? recs + (int64_t)row[u] * stride : nullptr;
    float* wav;
    if (!upload(&un.t->bufs[un.first], &un.t->n_samples[un.first], un.count, stride, un.t->au, m.resample, m.upload, st, &wav, into)) return false;
    if (!recs) recs = wav;
    if (un.t->long_audio) { vad = un.t->vad; vro = un.t->opts.vad; }
  }
  for (size_t u = 0; u < units.size(); ++u)
    if (units[u].t->long_audio) n_long.push_back(units[u].t->n16[units[u].first]);      // rows 0..nl-1 in unit order
  std::vector<VadResult> vr;
  if (nl > 0 && !vad_run_batch(*vad, recs, stride, n_long.data(), nl, st, vro, vr)) return false;
  // reference packs
  std::vector<RefPack> packs;
  std::vector<LongRec> longs;
  std::vector<int> utt_pack(units.size(), -1);
  int li = 0;
  for (size_t u = 0; u < units.size(); ++u) {
    Ticket& t = *units[u].t;
    if (!t.long_audio) {
      RefPack p{&t};
      p.set = t.hw_set;
      for (int j = 0; j < t.batch; ++j) {
        p.starts.push_back((int64_t)(row[u] + j) * stride);
        p.lens.push_back((int32_t)t.n16[j]);
        p.lang.push_back(t.lang ? t.lang[j] : kSvAuto);
        p.tn.push_back(t.tn ? t.tn[j] : kSvWoItn);
        p.ext = std::max(p.ext, num_lfr_frames(t.n16[j]));
        p.lmax = std::max<int64_t>(p.lmax, t.n16[j]);
      }
      utt_pack[u] = (int)packs.size();
      packs.push_back(std::move(p));
      continue;
    }
    const VadResult& v = vr[li++];
    if (!t.err.empty()) continue;                            // failed in an earlier group
    const FaLongAudioOptions& o = t.opts;
    const int i = units[u].first;
    const int64_t n = t.n16[i];
    LongRec lr{&t, i, row[u], v.seg, {}, {}};
    if (o.merge_vad) {                                       // inference_with_vad (auto_model.py:852-1035)
      lr.segs.resize(2 * v.seg.size() + 2);
      const int64_t k = fa_merge_vad(v.seg.data(), (int64_t)v.seg.size() / 2, o.merge_length_s * 1000, 0, lr.segs.data());
      if (k < 0) { set_err("fa_merge_vad failed"); return false; }
      lr.segs.resize((size_t)(2 * k));
    }
    const int64_t ns = (int64_t)lr.segs.size() / 2;
    if (ns > 0) {
      const std::vector<int32_t>& segs = lr.segs;
      std::vector<int32_t> bounds((size_t)(2 * ns));
      lr.order.resize((size_t)ns);
      const int64_t np = fa_pack_segments(segs.data(), ns, o.batch_size_s, o.batch_size_threshold_s, lr.order.data(), bounds.data());
      if (np < 0) { set_err("fa_pack_segments failed"); return false; }
      for (int64_t q = 0; q < np; ++q) {
        RefPack p{&t};
        p.set = t.hw_set;
        for (int j = bounds[2 * q]; j < bounds[2 * q + 1]; ++j) {     // slice_padding_audio_samples (utils/vad_utils.py:44-51)
          const int s = lr.order[j];
          const int64_t b0 = (int64_t)segs[2 * s] * 16, b1 = std::min<int64_t>((int64_t)segs[2 * s + 1] * 16, n), len = b1 - b0;
          if (len < 400) {
            p.bad = "recording " + std::to_string(i) + ": VAD segment " + std::to_string(s) + " [" + std::to_string(segs[2 * s]) + ", " +
                    std::to_string(segs[2 * s + 1]) + "] ms has " + std::to_string(len > 0 ? len : 0) + " samples; the recogniser needs >= 400 (25 ms)";
            break;
          }
          p.starts.push_back((int64_t)row[u] * stride + b0);
          p.lens.push_back((int32_t)len);
          p.lang.push_back(t.lang ? t.lang[i] : kSvAuto);
          p.tn.push_back(t.tn ? t.tn[i] : kSvWoItn);
          p.ext = std::max(p.ext, num_lfr_frames(len));
          p.lmax = std::max(p.lmax, len);
        }
        lr.packs.push_back((int)packs.size());
        const bool bad = !p.bad.empty();
        packs.push_back(std::move(p));
        if (bad) break;                                      // the recording either fails here or emptied earlier: later packs are never read
      }
    }
    longs.push_back(std::move(lr));
  }
  // GPU packs: reference packs by extent, merged while the padded audio fits kPackSamples and the hotword memories kPackHotwordRows;
  // two packs of one call never share a GPU pack, so a lone caller decodes exactly its reference packs
  std::vector<int> by_ext;
  for (size_t p = 0; p < packs.size(); ++p)
    if (packs[p].bad.empty()) by_ext.push_back((int)p);
  std::stable_sort(by_ext.begin(), by_ext.end(), [&](int a, int b) { return packs[a].ext < packs[b].ext; });
  std::vector<std::vector<int>> gpu;
  int64_t g_rows = 0, g_lmax = 0, g_hw_max = 0, g_memories = 0;
  std::vector<char> g_sets(sets.n.size(), 0);
  for (int p : by_ext) {
    const RefPack& rp = packs[p];
    const int64_t n = rp.set >= 0 ? sets.n[rp.set] : 0;
    const int64_t memories = g_memories + (rp.set >= 0 && !g_sets[rp.set]) + (m.seaco && m.nfilter > 0 && m.nfilter < n);
    bool join = !gpu.empty() && (g_rows + (int64_t)rp.lens.size()) * padded(std::max(g_lmax, rp.lmax)) <= kPackSamples &&
                memories * std::max(g_hw_max, n) <= kPackHotwordRows;
    for (size_t k = 0; join && k < (gpu.empty() ? 0 : gpu.back().size()); ++k) join = packs[gpu.back()[k]].t != rp.t;
    if (!join) {
      gpu.emplace_back(); g_rows = 0; g_lmax = 0; g_hw_max = 0; g_memories = 0;
      std::fill(g_sets.begin(), g_sets.end(), 0);
    }
    gpu.back().push_back(p);
    g_rows += (int64_t)rp.lens.size();
    g_lmax = std::max(g_lmax, rp.lmax);
    g_hw_max = std::max(g_hw_max, n);
    g_memories += (rp.set >= 0 && !g_sets[rp.set]) + (m.seaco && m.nfilter > 0 && m.nfilter < n);
    if (rp.set >= 0) g_sets[rp.set] = 1;
  }
  for (const std::vector<int>& g : gpu) {
    std::vector<int64_t> starts;
    std::vector<int32_t> lens, ext, lang, tn;
    int64_t lmax = 0;
    PackHotwords hw;                                         // the pack's sets, numbered in the pack
    std::vector<int> local(sets.n.size(), -1);
    for (int p : g) {
      const RefPack& rp = packs[p];
      int set = -1;
      if (rp.set >= 0) {
        if (local[rp.set] < 0) {
          local[rp.set] = (int)hw.n.size();
          hw.rows.push_back(sets.rows[rp.set]);
          hw.n.push_back(sets.n[rp.set]);
        }
        set = local[rp.set];
      }
      hw.refs.push_back({(int)lens.size(), (int)rp.lens.size(), set});
      starts.insert(starts.end(), rp.starts.begin(), rp.starts.end());
      lens.insert(lens.end(), rp.lens.begin(), rp.lens.end());
      ext.insert(ext.end(), rp.lens.size(), rp.ext);
      lang.insert(lang.end(), rp.lang.begin(), rp.lang.end());
      tn.insert(tn.end(), rp.tn.begin(), rp.tn.end());
      lmax = std::max(lmax, rp.lmax);
    }
    const int B = (int)lens.size();
    int64_t pstride = padded(lmax);
    float* wav;
    if (g.size() == 1 && packs[g[0]].t->batch == B && !packs[g[0]].t->long_audio) {
      wav = recs + packs[g[0]].starts[0];                   // a call's whole batch alone: its rows are already padded in place
      pstride = stride;
    } else {
      int64_t* starts_d;
      int32_t* lens_d;
      if (!carve(m.pack, "segments", [&](fa::Arena& a) {
            starts_d = a.take<int64_t>(B); lens_d = a.take<int32_t>(B); wav = a.take<float>((size_t)B * pstride);
          }))
        return false;
      if (!gather(recs, (int64_t)rows * stride, starts.data(), lens.data(), B, pstride, starts_d, lens_d, wav, st)) return false;
    }
    std::unique_ptr<Result> r = decode_pack(m, wav, pstride, lens, ext, &hw, lang.data(), tn.data());
    if (!r) return false;
    ++m.pool_packs;
    int j = 0;
    for (int p : g) {                                        // scatter: each reference pack's rows
      RefPack& rp = packs[p];
      rp.out.reset(new Result());
      for (size_t k = 0; k < rp.lens.size(); ++k, ++j) {
        rp.out->ids.push_back(std::move(r->ids[j]));
        rp.out->token_num.push_back(r->token_num[j]);
        rp.out->stamps.push_back(r->ts ? std::move(r->stamps[j]) : std::vector<int32_t>());
      }
    }
  }
  // the calls' results
  for (size_t u = 0; u < units.size(); ++u) {
    if (units[u].t->long_audio) continue;
    Ticket& t = *units[u].t;
    RefPack& rp = packs[utt_pack[u]];
    t.res->ids.swap(rp.out->ids);
    t.res->token_num.swap(rp.out->token_num);
    if (m.ts) t.res->stamps.swap(rp.out->stamps);
  }
  // each recording's own failure, decided in recording order once the speaker stage has run: a short VAD segment where the reference
  // reaches it, or a refusal of the speaker stage.  A ticket's later recordings in the group (consecutive in longs) are not assembled
  // after its first.
  std::vector<std::string> rec_err(longs.size());
  std::vector<int> job_of(longs.size(), -1);
  const Ticket* stopped = nullptr;
  std::vector<SpkJob> jobs;
  Spk* spk = nullptr;
  for (size_t li = 0; li < longs.size(); ++li) {
    LongRec& lr = longs[li];
    Ticket& t = *lr.t;
    if (!t.err.empty() || &t == stopped) continue;
    const int64_t ns = (int64_t)lr.segs.size() / 2;
    std::vector<std::vector<int32_t>> seg_ids((size_t)ns), seg_stamps((size_t)ns);
    bool emptied = false;
    int beg = 0;
    for (int p : lr.packs) {                                 // the reference's pack loop: a bad segment fails the call where it is reached
      RefPack& rp = packs[p];
      if (!rp.bad.empty()) { rec_err[li] = rp.bad; stopped = &t; break; }
      int tmax = 0;
      for (int32_t k : rp.out->token_num) tmax = std::max(tmax, k);
      // no token in the whole pack: the recording's result is empty (:990-999).  SenseVoiceSmall.inference returns a result for every
      // utterance, empty or not, so its packs never empty a recording.
      if (tmax < 1 && !m.sv) { emptied = true; break; }
      for (size_t k = 0; k < rp.lens.size(); ++k) {
        seg_ids[lr.order[beg + k]].swap(rp.out->ids[k]);
        seg_stamps[lr.order[beg + k]].swap(rp.out->stamps[k]);
      }
      beg += (int)rp.lens.size();
    }
    if (stopped == &t) continue;
    std::vector<int32_t>&ids = t.res->ids[lr.i], &segs_out = t.res->segs[lr.i], &stamps = t.res->stamps[lr.i];
    for (int64_t s = 0; s < ns; ++s) {
      const int32_t k = emptied ? 0 : (int32_t)seg_ids[s].size();
      segs_out.insert(segs_out.end(), {lr.segs[2 * s], lr.segs[2 * s + 1], k});
      if (emptied) continue;
      ids.insert(ids.end(), seg_ids[s].begin(), seg_ids[s].end());
      for (int32_t v : seg_stamps[s]) stamps.push_back(v + lr.segs[2 * s]);      // absolute ms (auto_model.py:1008-1022)
    }
    t.res->token_num[lr.i] = (int32_t)ids.size();
    if (t.spk && !ids.empty()) {                             // diarize every recording that decoded a token
      SpkJob jb;
      jb.off = (int64_t)lr.row * stride; jb.n = t.n16[lr.i]; jb.segs = &segs_out; jb.preset = t.preset_spk_num;
      jb.what = "recording " + std::to_string(lr.i) + ": "; jb.spk = &t.res->spk[lr.i];
      job_of[li] = (int)jobs.size();
      jobs.push_back(std::move(jb));
      spk = t.spk;                                           // one speaker handle per pass (admit)
    }
  }
  // one speaker stage over the group's diarized recordings.  The recogniser's stream is idle here (its results are on the host); the
  // speaker work runs on the speaker handle's stream.
  if (!jobs.empty() && !diarize(*spk, recs, (int64_t)rows * stride, jobs)) return false;
  for (size_t li = 0; li < longs.size(); ++li) {
    Ticket& t = *longs[li].t;
    if (!t.err.empty()) continue;
    t.err = !rec_err[li].empty() ? rec_err[li] : (job_of[li] >= 0 ? jobs[job_of[li]].err : rec_err[li]);
  }
  return true;
}

// One pass over the admitted tickets under the device locks (recogniser -> VAD -> speaker): every ticket ends with a result or a message
void run_pass(Model& m, const std::vector<Ticket*>& pass) {
  std::lock_guard<std::mutex> dev(m.mu);
  Vad* vad = nullptr;
  Spk* spk = nullptr;
  for (Ticket* t : pass) {
    if (t->long_audio) vad = t->vad;
    if (t->spk) spk = t->spk;
  }
  std::unique_lock<std::mutex> vad_lock, spk_lock;
  if (vad) vad_lock = std::unique_lock<std::mutex>(vad->mu);
  if (spk) spk_lock = std::unique_lock<std::mutex>(spk->mu);
  cudaSetDevice(m.file.device);
  PackHotwords sets;                                         // the pass's distinct hotword sets: the same count and the same bytes
  for (Ticket* t : pass) {
    t->hw_set = -1;
    if (!(m.contextual || m.seaco) || !t->hw_embed || t->n_hotwords < 1) continue;   // the other models ignore rows
    const size_t bytes = (size_t)t->n_hotwords * 512 * sizeof(float);
    for (size_t k = 0; k < sets.n.size() && t->hw_set < 0; ++k)
      if (sets.n[k] == t->n_hotwords && (sets.rows[k] == t->hw_embed || memcmp(sets.rows[k], t->hw_embed, bytes) == 0)) t->hw_set = (int)k;
    if (t->hw_set < 0) {
      t->hw_set = (int)sets.n.size();
      sets.rows.push_back(t->hw_embed);
      sets.n.push_back(t->n_hotwords);
    }
  }
  const bool ok = no_throw(pass[0]->long_audio ? "fa_offline_infer_vad: " : "fa_offline_infer: ", [&] {
    std::vector<Unit> units;
    for (Ticket* t : pass) {
      t->res.reset(new Result());
      Result& r = *t->res;
      r.ids.resize(t->batch);
      r.token_num.assign(t->batch, 0);
      r.ts = m.ts;
      if (m.ts || t->long_audio) r.stamps.resize(t->batch);
      if (t->long_audio) {
        r.segs.resize(t->batch);
        r.spk.resize(t->batch);
        for (int i = 0; i < t->batch; ++i) units.push_back({t, i, 1});
      } else {
        units.push_back({t, 0, t->batch});
      }
      r.audio_seconds = (float)t->au.seconds(t->n_samples, t->batch);
    }
    // groups of units in arrival order, at most kVadGroupSamples padded samples each (a larger unit is a group of its own)
    for (size_t g0 = 0, g1; g0 < units.size(); g0 = g1) {
      auto width = [&](const Unit& u) {
        int64_t w = 0;
        for (int i = u.first; i < u.first + u.count; ++i) w = std::max(w, padded(u.t->n16[i]));
        return w;
      };
      int64_t stride = width(units[g0]);
      int rows = units[g0].count;
      for (g1 = g0 + 1; g1 < units.size(); ++g1) {
        const int64_t w = std::max(stride, width(units[g1]));
        if ((rows + units[g1].count) * w > kVadGroupSamples) break;
        stride = w;
        rows += units[g1].count;
      }
      if (!pool_group(m, std::vector<Unit>(units.begin() + g0, units.begin() + g1), stride, sets)) return false;
    }
    return true;
  });
  if (!ok)                                                   // a device failure: every ticket of the pass gets its message
    for (Ticket* t : pass) t->err = g_err;
}

}  // namespace

namespace fa_handle {

void* pool_call(Model& m, Ticket& t) {
  m.pool.call(t, admit, [&](std::vector<Ticket*>& pass, std::vector<Ticket*>& ended) {
    run_pass(m, pass);
    ended.swap(pass);
  }, "fa_offline_infer: ");
  if (!t.err.empty()) return fail(t.err);
  g_err.clear();
  return t.res.release();
}

}  // namespace fa_handle

extern "C" int fa_offline_pool_stats(const void* handle, int64_t* calls, int64_t* packs) {
  const Model* m = static_cast<const Model*>(handle);
  if (!m || !calls || !packs) return FA_ERR_ARG;
  *calls = m->pool.calls.load();
  *packs = m->pool_packs.load();
  return FA_OK;
}
