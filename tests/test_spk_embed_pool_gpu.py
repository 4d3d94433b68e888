"""GPU (-m gpu): the CAM++ forward with a padded length per row, and the speaker handle's request pool.

- fa_campplus_forward_ext: every row equals fa_campplus_forward on its own first ext[b] frames, bit for bit, in every GEMM mode, over
  a NaN-filled workspace and with large values past every extent (a read past an extent would show); all extents at t is
  fa_campplus_forward on the whole batch.
- Pooled calls: embedding calls (mixed batches, lengths, sample formats and rates) and clustering calls posted from many threads equal
  the same calls made one at a time on another handle, bit for bit, and the pool shows fewer passes than calls; a refused clustering
  set fails only its own call, with its own message; speaker-only calls and diarized long-audio calls on one speaker handle do not
  deadlock and give what they give alone; a lone call launches what one call launched before calls were pooled."""
import ctypes as C
import threading
import time

import numpy as np
import pytest
import torch

from funasr_b200 import _abi, pack, synth
from funasr_b200.offline import OfflineRecognizer, OfflineSpeaker, OfflineVad
from test_campplus_entries_gpu import DEV, MODES, _engine, _st, _voice_feats
from test_spk_host import SPK_CASES, campplus_state_dict

pytestmark = pytest.mark.gpu

WAIT = 600.0
# extents covering the TDNN parity (odd / even frame counts) and the 100-frame CAM segment edges (t_out 100, 101, 201)
EXTS = [2, 3, 4, 5, 147, 148, 199, 200, 201, 202, 401, 7, 60, 250, 333, 399, 402, 523]
T_EXT = 600
# kernel launches of a lone fa_spk_embed call (one 16 kHz f32 recording of 2 s), counted on the parent commit's fa_spk_embed:
# fa_campplus_features and the CAM++ forward (FCM, TDNN, 52 CAM layers, transits, statistics pooling, dense layer)
LONE_LAUNCHES = {"fp32": 232, "fp16x3": 234}


def _ws(nbytes):
    """A workspace of exactly nbytes, every byte 0xff (NaN as fp32)."""
    return torch.full((max(int(nbytes), 1),), 255, dtype=torch.uint8, device=DEV)


def _forward(eng, feats, ext=None):
    """fa_campplus_forward (ext None) or fa_campplus_forward_ext over NaN-filled workspace and output -> [B, 192] on the host."""
    lib = eng.lib
    B, T, _ = feats.shape
    emb = torch.full((B, 192), float("nan"), device=DEV)
    q = lib.fa_campplus_workspace_bytes if ext is None else lib.fa_campplus_ext_workspace_bytes
    ws = _ws(q(C.byref(eng.model), B, T, eng.mode))
    fd = feats.contiguous().to(DEV)
    torch.cuda.synchronize()
    if ext is None:
        rc = lib.fa_campplus_forward(C.byref(eng.model), fd.data_ptr(), B, T, emb.data_ptr(), eng.mode, ws.data_ptr(), ws.numel(), _st())
    else:
        e = (C.c_int32 * B)(*ext)
        rc = lib.fa_campplus_forward_ext(C.byref(eng.model), fd.data_ptr(), B, T, emb.data_ptr(), eng.mode, ws.data_ptr(), ws.numel(),
                                         _st(), e)
    torch.cuda.synchronize()
    assert rc == 0, rc
    return emb.cpu()


def _ragged(feats, ext, seed):
    """feats with every frame at or past row b's extent replaced by large random values."""
    g = torch.Generator().manual_seed(seed)
    out = feats.clone()
    for b, e in enumerate(ext):
        out[b, e:] = 1e4 * torch.randn(out.shape[1] - e, out.shape[2], generator=g)
    return out


def _same(a, b):
    return torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(torch.nan_to_num(a), torch.nan_to_num(b))


@pytest.mark.parametrize("mode", MODES)
def test_forward_ext_rows_equal_each_row_alone(mode):
    eng = _engine(mode)
    ext = EXTS + [T_EXT]
    feats = _voice_feats(T_EXT, len(ext))
    got = _forward(eng, _ragged(feats, ext, 1), ext)
    for b, e in enumerate(ext):
        alone = _forward(eng, feats[b:b + 1, :e])[0]
        assert _same(got[b], alone), (mode, b, e)
        assert torch.isnan(alone).all() if e == 2 else not torch.isnan(alone).any(), (mode, e)
    whole = _forward(eng, feats)
    assert torch.equal(_forward(eng, feats, [T_EXT] * len(ext)), whole)


def test_forward_ext_longest_row_among_short_rows():
    """fp16x3: one 18 800-frame row (94 CAM segments) among short rows."""
    eng = _engine("fp16x3")
    T = 18800
    long_row = _voice_feats(T, 1)
    short = _voice_feats(401, 3)
    ext = [148, T, 3, 401]
    feats = torch.zeros(4, T, 80)
    feats[1] = long_row[0]
    for b, e in ((0, 148), (2, 3), (3, 401)):
        feats[b, :e] = short[b - (b > 1), :e]
    got = _forward(eng, _ragged(feats, ext, 2), ext)
    for b, e in enumerate(ext):
        assert torch.equal(got[b], _forward(eng, feats[b:b + 1, :e])[0]), (b, e)


# ------------------------------------------------------------------------------------------------ the speaker handle's pool
@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("spk_pool")
    cfg = synth.PARAFORMER_TINY
    out = {"asr": str(d / "asr.fab2"), "vad": str(d / "vad.fab2"), "spk": str(d / "spk.fab2")}
    pack.write_model_file(out["asr"], synth.make_state_dict(cfg, 3), cfg, synth.make_cmvn(cfg, 1))
    pack.write_vad_model_file(out["vad"], synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    pack.write_campplus_model_file(campplus_state_dict(), out["spk"])
    return out


def _run_threads(jobs, n_threads, first=None):
    """jobs (callables) shared out over n_threads daemon threads (first, if given, started alone just before them) -> results in job
    order; a thread that does not finish within WAIT fails the test instead of hanging it."""
    out, errs = [None] * len(jobs), []

    def run(idx):
        try:
            for k in idx:
                out[k] = jobs[k]()
        except Exception as e:                                  # noqa: BLE001 - reported below
            errs.append(e)
    groups = [list(range(j, len(jobs), n_threads)) for j in range(n_threads)]
    ts = []
    if first is not None:
        groups = [[first]] + [[k for k in g if k != first] for g in groups]
    for g in groups:
        ts.append(threading.Thread(target=run, args=(g,), daemon=True))
        ts[-1].start()
        if first is not None and len(ts) == 1:
            time.sleep(0.05)
    t0 = time.time()
    for t in ts:
        t.join(max(1.0, WAIT - (time.time() - t0)))
        assert not t.is_alive(), "a call did not return: deadlock or hang"
    assert not errs, errs
    return out


_BASE = []


def _voice(seconds, seed):
    """seconds of one of three synthetic 61 s voices (synthesised once), from a seeded offset and at a seeded gain."""
    if not _BASE:
        _BASE.extend(synth.make_voice_wav([(v, 61.0, 0.2)], 500 + v, lead_s=0.0).numpy() for v in range(3))
    base = _BASE[seed % 3]
    n = int(seconds * 16000)
    off = (seed * 7919) % (base.size - n + 1)
    return np.ascontiguousarray(base[off:off + n] * (0.5 + (seed % 17) / 32), dtype=np.float32)


def _embed_requests(seed, count):
    """Seeded embedding calls: batches of 1-8, 0.5-60 s, f32 / s16 at 16 kHz, 8 kHz and 44.1 kHz through either resampler."""
    rng = np.random.default_rng(seed)
    reqs = []
    for k in range(count):
        b = int(rng.integers(1, 9))
        secs = [float(rng.uniform(0.5, 60.0)) if rng.random() < 0.15 else float(rng.uniform(0.5, 12.0)) for _ in range(b)]
        wavs = [_voice(s, 1000 * seed + 10 * k + i) for i, s in enumerate(secs)]
        kind = k % 4
        if kind == 1:
            wavs = [(w * 32767).astype(np.int16) for w in wavs]
            reqs.append((wavs, 16000, "loader"))
        elif kind == 2:
            reqs.append(([np.ascontiguousarray(w[::2]) for w in wavs], 8000, "loader" if k % 8 < 4 else "runtime"))
        elif kind == 3:
            idx = [np.arange(0, w.size, 16000 / 44100.0).astype(np.int64) for w in wavs]
            reqs.append(([np.ascontiguousarray(w[i]) for w, i in zip(wavs, idx)], 44100, "runtime" if k % 8 < 4 else "loader"))
        else:
            reqs.append((wavs, 16000, "loader"))
    return reqs


@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_pooled_embed_calls_equal_each_call_alone(files, mode):
    spk, ref = OfflineSpeaker(files["spk"], 0, mode), OfflineSpeaker(files["spk"], 0, mode)
    long_call = ([_voice(60.0, 90 + i) for i in range(64)], 16000, "loader")
    reqs = [long_call] + _embed_requests(7, 48)
    want = [ref.embed(w, fs=fs, resampler=r) for w, fs, r in reqs]
    c0, p0 = spk.pool_stats()
    got = _run_threads([lambda q=q: spk.embed(q[0], fs=q[1], resampler=q[2]) for q in reqs], 16, first=0)
    calls, passes = (a - b for a, b in zip(spk.pool_stats(), (c0, p0)))
    for k, (g, w) in enumerate(zip(got, want)):
        assert g.tobytes() == w.tobytes(), (mode, k)
    assert calls == len(reqs) and passes < calls, (calls, passes)
    spk.close()
    ref.close()


def test_a_pooled_pass_needs_no_more_device_memory_than_its_calls_alone(files):
    """2 048 rows of 1 s and one 60 s row posted together, while a long call holds the pool, share a pass.  Each pack is uploaded at
    its own row pitch, so once every call has run alone on the handle the pooled pass grows none of its buffers (uploading the short
    call at the 60 s pitch would take about 8 GB).  Both equal the calls alone."""
    spk, ref = OfflineSpeaker(files["spk"], 0, "fp32"), OfflineSpeaker(files["spk"], 0, "fp32")
    blocker = [_voice(60.0, 300 + i) for i in range(16)]
    short = [_voice(1.0, 400 + i) for i in range(2048)]
    long_row = [_voice(60.0, 401)]
    want = [ref.embed(w) for w in (blocker, short, long_row)]
    for w in (blocker, short, long_row):                       # the handle's buffers grown to what each call needs alone
        spk.embed(w)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    c0, p0 = spk.pool_stats()
    got = _run_threads([lambda w=w: spk.embed(w) for w in (blocker, short, long_row)], 3, first=0)
    torch.cuda.synchronize()
    grown = free0 - torch.cuda.mem_get_info()[0]
    calls, passes = (a - b for a, b in zip(spk.pool_stats(), (c0, p0)))
    for g, w in zip(got, want):
        assert g.tobytes() == w.tobytes()
    assert calls == 3 and passes < calls, (calls, passes)
    assert grown < (1 << 30), grown
    spk.close()
    ref.close()


def _mixture(n, k, seed):
    rng = np.random.RandomState(seed)
    centers = rng.randn(k, 192)
    lab = rng.randint(0, k, size=n)
    return np.ascontiguousarray((centers[lab] + 0.3 * rng.randn(n, 192)).astype(np.float32))


def _cluster(spk, x, preset):
    lab = np.full(x.shape[0], -1, np.int32)
    rc = spk.lib.fa_spk_cluster(spk.handle, x.ctypes.data, x.shape[0], preset, lab.ctypes.data)
    return rc, (lab.tolist() if rc == 0 else spk.lib.fa_offline_last_error().decode())


def test_pooled_cluster_calls_equal_each_call_alone(files):
    spk, ref = OfflineSpeaker(files["spk"], 0, "fp32"), OfflineSpeaker(files["spk"], 0, "fp32")
    calls = []
    for i, n in enumerate((5, 19, 20, 120, 700, 2047)):
        x = _mixture(n, 3 + i % 3, 40 + i)
        calls += [(x, 0), (x, 2 + i % 4)]
    calls.append((_mixture(2100, 4, 99), 4))                     # k-means on the normalised rows
    calls.append((_mixture(30, 2, 98), 31))                      # a preset above n: refused, alone
    want = [_cluster(ref, x, p) for x, p in calls]
    assert want[-1][0] != 0 and "exceeds" in want[-1][1]
    assert all(w[0] == 0 for w in want[:-1])
    c0, p0 = spk.pool_stats()
    got = _run_threads([lambda c=c: _cluster(spk, *c) for c in calls], 12)
    assert got == want
    calls_n, passes = (a - b for a, b in zip(spk.pool_stats(), (c0, p0)))
    assert calls_n == len(calls) and passes < calls_n, (calls_n, passes)
    spk.close()
    ref.close()


def test_mixed_traffic_on_one_speaker_handle(files):
    """4 threads diarize the fixtures' recordings (fa_offline_infer_vad_spk) while 8 threads post embedding calls, all on one speaker
    handle: nothing deadlocks, and every result equals the same call alone."""
    rec, vad = OfflineRecognizer(files["asr"], 0, "fp32"), OfflineVad(files["vad"], 0)
    spk, ref = OfflineSpeaker(files["spk"], 0, "fp32"), OfflineSpeaker(files["spk"], 0, "fp32")
    long_jobs = []
    for name, (pattern, seed, kw) in SPK_CASES.items():
        wav = synth.make_voice_wav(pattern, seed).numpy()
        long_jobs.append((wav, kw.get("preset_spk_num")))
    reqs = _embed_requests(11, 24)
    want_long = [rec.infer_long([w], vad, spk=ref, preset_spk_num=p)[0] for w, p in long_jobs]
    want_emb = [ref.embed(w, fs=fs, resampler=r) for w, fs, r in reqs]
    jobs = [lambda j=j: rec.infer_long([j[0]], vad, spk=spk, preset_spk_num=j[1])[0] for j in long_jobs * 2]
    emb_jobs = [lambda q=q: spk.embed(q[0], fs=q[1], resampler=q[2]) for q in reqs]
    results = {}

    def longs():
        results["long"] = _run_threads(jobs, 4)

    def embeds():
        results["emb"] = _run_threads(emb_jobs, 8)
    ts = [threading.Thread(target=f, daemon=True) for f in (longs, embeds)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(WAIT)
        assert not t.is_alive(), "deadlock or hang"
    assert results["long"] == want_long * 2
    for k, (g, w) in enumerate(zip(results["emb"], want_emb)):
        assert g.tobytes() == w.tobytes(), k
    for h in (rec, vad, spk, ref):
        h.close()


@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_a_lone_call_launches_what_the_parent_launches(files, mode):
    spk = OfflineSpeaker(files["spk"], 0, mode)
    w = [_voice(2.0, 5)]
    first = spk.embed(w)                                         # buffers grown
    for _ in range(2):
        l0 = spk.lib.fa_launch_count()
        again = spk.embed(w)
        assert spk.lib.fa_launch_count() - l0 == LONE_LAUNCHES[mode]
        assert again.tobytes() == first.tobytes()
    spk.close()
