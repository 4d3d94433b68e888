"""GPU: audio at any sample rate and PCM layout through the C handle API (FaAudioFormat).  fa_ingest_pcm against fa_pcm_decode +
fa_resample (loader mode, bit for bit) and against the reference runtime's LinearResample (runtime mode); the four `_audio` entries
against their 16 kHz counterparts fed the matching reference's 16 kHz rows; refusals before any launch; and the runtime shim at
8 kHz against the 16 kHz buffer LinearResample produces."""
import ctypes as C
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import torch

import linres_ref
from audio_in_ref import RATES, linres_rows
from conftest import ROOT
from funasr_b200 import _abi, pack, synth
from funasr_b200.offline import OfflineRecognizer, OfflineSpeaker, OfflineVad
from funasr_b200.resample import resample, sinc_resample_table
from test_offline_vad_gpu import LONG_CASES, _vocab_dir
from test_spk_host import SPK_CASES, campplus_state_dict

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CFG = synth.PARAFORMER_TINY
BYTES = {0: 4, 1: 2, 2: 3, 3: 4, 4: 1}


def _lib():
    return _abi.load()


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _raw(fmt, frames, channels, seed):
    """Random interleaved PCM of one sample format as bytes (uint8 array)."""
    g = np.random.default_rng(seed)
    n = frames * channels
    if fmt == 0:
        return (g.standard_normal(n) * 0.3).astype(np.float32).view(np.uint8)
    if fmt == 1:
        return g.integers(-32768, 32768, n).astype(np.int16).view(np.uint8)
    if fmt == 2:
        return g.integers(0, 256, 3 * n).astype(np.uint8)
    if fmt == 3:
        return g.integers(-2 ** 31, 2 ** 31, n).astype(np.int32).view(np.uint8)
    return g.integers(0, 256, n).astype(np.uint8)


def _decode(raw, fmt, channels, frames):
    """fa_pcm_decode of one row -> mono float32 on the device"""
    src = torch.from_numpy(np.ascontiguousarray(raw)).to(DEV)
    out = torch.empty(max(frames, 1), dtype=torch.float32, device=DEV)
    _abi.check(_lib().fa_pcm_decode(src.data_ptr(), fmt, channels, frames, out.data_ptr(), _stream()), "fa_pcm_decode")
    return out[:frames]


class _Table:
    """A resampling table of the host functions, uploaded with torch, as FaIngestTable.  Loader mode: with spans (each row's nonzero
    taps, what the handle passes) or the full rows."""

    def __init__(self, rate, mode, spans=True):
        lib = _lib()
        self.keep = []
        if rate == 16000:
            self.t = _abi.FaIngestTable(-1)
            self.len16 = lambda n: n
            return
        if mode == _abi.RESAMPLE_LOADER:
            tab, orig, new, width = sinc_resample_table(rate, 16000)
            nz = tab != 0
            k0 = np.where(nz.any(1), nz.argmax(1), 0).astype(np.int32)
            k1 = np.where(nz.any(1), tab.shape[1] - nz[:, ::-1].argmax(1), 0).astype(np.int32)
            self.keep = [torch.from_numpy(a).to(DEV) for a in (tab, k0, k1 - k0)]
            first, n_taps = (self.keep[1].data_ptr(), self.keep[2].data_ptr()) if spans else (None, None)
            self.t = _abi.FaIngestTable(0, orig, new, width, 2 * width + orig, 0, self.keep[0].data_ptr(), first, n_taps)
            self.len16 = lambda n: -(-new * n // orig)
        else:
            iu, ou, mt = C.c_int32(), C.c_int32(), C.c_int32()
            need = lib.fa_runtime_resample_table_host(rate, 16000, C.byref(iu), C.byref(ou), C.byref(mt), None, None, None, 0)
            first, n_taps, w = np.zeros(ou.value, np.int32), np.zeros(ou.value, np.int32), np.zeros(need, np.float32)
            lib.fa_runtime_resample_table_host(rate, 16000, C.byref(iu), C.byref(ou), C.byref(mt), first.ctypes.data, n_taps.ctypes.data,
                                               w.ctypes.data, need)
            self.keep = [torch.from_numpy(a).to(DEV) for a in (w, first, n_taps)]
            self.t = _abi.FaIngestTable(1, iu.value, ou.value, 0, mt.value, 0, *[k.data_ptr() for k in self.keep])
            self.len16 = lambda n: int(lib.fa_runtime_resample_out_len_host(rate, 16000, n))


def _ingest(raws, frames, fmt, channels, rate, mode, spans=True):
    """fa_ingest_pcm over a ragged batch -> (rows [B, stride] on the host, 16 kHz lengths); one launch, NaN-filled output first."""
    lib = _lib()
    tab = _Table(rate, mode, spans)
    offs, buf = [], []
    pos = 0
    for r in raws:
        offs.append(pos)
        pad = (-r.size) % 16
        buf.append(np.concatenate([r, np.zeros(pad, np.uint8)]))
        pos += r.size + pad
    raw = torch.from_numpy(np.concatenate(buf)).to(DEV)
    lens = [tab.len16(n) for n in frames]
    rows = torch.tensor([[o, n, l] for o, n, l in zip(offs, frames, lens)], dtype=torch.int64).to(DEV)
    stride = max(4, (max(lens) + 3) // 4 * 4)
    y = torch.full((len(raws), stride), float("nan"), dtype=torch.float32, device=DEV)
    torch.cuda.synchronize()
    before = lib.fa_launch_count()
    _abi.check(lib.fa_ingest_pcm(raw.data_ptr(), rows.data_ptr(), len(raws), fmt, channels, C.byref(tab.t), y.data_ptr(), stride, _stream()),
               "fa_ingest_pcm")
    assert lib.fa_launch_count() - before == 1
    torch.cuda.synchronize()
    return y.cpu().numpy(), lens


def _same(a, b):
    return a.shape == b.shape and np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("rate", RATES + (16000,))
def test_ingest_runtime_mode_equals_linear_resample(rate):
    """Ragged mono f32 rows at the edge lengths (1, under one filter, unit boundaries +-1) and 3 s of noise: each row equals the
    reference's Resample(flush=true) of the same samples, zero past its length."""
    tab = _Table(rate, _abi.RESAMPLE_RUNTIME)
    iu = tab.t.in_unit if rate != 16000 else 1
    edges = linres_ref.edge_lengths(iu, max(tab.t.taps, 1)) + [3 * rate]
    x = linres_ref.noise(rate, 3.0, seed=2)
    raws = [x[:n].view(np.uint8) for n in edges]
    y, lens = _ingest(raws, edges, 0, 1, rate, _abi.RESAMPLE_RUNTIME)
    for i, n in enumerate(edges):
        want = linres_rows(x[:n], rate)
        assert lens[i] == want.size, (rate, n)
        assert _same(y[i, :lens[i]], want), (rate, n)
        assert not y[i, lens[i]:].any()


@pytest.mark.parametrize("rate", RATES + (16000, 1000, 192000))
@pytest.mark.parametrize("fmt", [0, 1, 2, 3, 4])
def test_ingest_loader_mode_is_decode_then_fa_resample(rate, fmt):
    """Every sample format, 1, 2 and 6 channels: bit for bit fa_pcm_decode followed by fa_resample (funasr_b200.resample), with the
    rows' nonzero spans and with full rows, zero past their lengths; runtime mode on the same bytes equals LinearResample of
    fa_pcm_decode's samples."""
    for channels in (1, 2, 6):
        frames = [1, 37, 2 * rate // 100 + 3, rate // 3]
        raws = [_raw(fmt, n, channels, 100 * fmt + 10 * channels + i) for i, n in enumerate(frames)]
        y, lens = _ingest(raws, frames, fmt, channels, rate, _abi.RESAMPLE_LOADER)
        y_full, _ = _ingest(raws, frames, fmt, channels, rate, _abi.RESAMPLE_LOADER, spans=False)
        assert _same(y, y_full)
        yr, lens_r = _ingest(raws, frames, fmt, channels, rate, _abi.RESAMPLE_RUNTIME)
        for i, n in enumerate(frames):
            dec = _decode(raws[i], fmt, channels, n)
            if rate == 16000:
                want = dec.cpu().numpy()
            else:
                out, ol = resample(dec[None].contiguous(), torch.tensor([n], dtype=torch.int32, device=DEV), rate, 16000)
                want = out[0, :int(ol[0])].cpu().numpy()
            assert lens[i] == want.size and _same(y[i, :lens[i]], want), (rate, fmt, channels, n)
            assert not y[i, lens[i]:].any()
            if rate in RATES or rate == 16000:
                assert _same(yr[i, :lens_r[i]], linres_rows(dec.cpu().numpy(), rate)), (rate, fmt, channels, n)
                assert not yr[i, lens_r[i]:].any()


# ------------------------------------------------------------------------------------------------ the handle entries
@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("audio_in")
    out = {k: str(d / (k + ".fab2")) for k in ("asr", "bicif", "vad", "spk", "seaco")}
    cmvn = synth.make_cmvn(CFG, 1)
    pack.write_model_file(out["asr"], synth.make_state_dict(CFG, 3), CFG, cmvn)
    pack.write_model_file(out["bicif"], synth.make_bicif_state_dict(CFG, 8), CFG, cmvn)
    pack.write_vad_model_file(out["vad"], synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    pack.write_campplus_model_file(campplus_state_dict(), out["spk"])
    pack.write_seaco_model_file(out["seaco"], synth.make_seaco_state_dict(CFG, 5), CFG, cmvn, no_bias=synth.seaco_no_bias_id(CFG), nfilter=4)
    return out


def _ptrs(arrs):
    n = len(arrs)
    return (C.c_void_p * n)(*[a.ctypes.data for a in arrs]), (C.c_int64 * n)(*[a.shape[0] for a in arrs])


def _result(lib, res, stamped=False):
    assert res, lib.fa_offline_last_error().decode()
    try:
        out = []
        cnt = C.c_int32(0)
        for i in range(lib.fa_offline_result_count(res)):
            p = lib.fa_offline_result_ids(res, i, C.byref(cnt))
            ids = [int(p[k]) for k in range(cnt.value)]
            if stamped:
                s = lib.fa_offline_result_stamps(res, i, C.byref(cnt))
                ids = (ids, [int(s[k]) for k in range(2 * cnt.value)])
            out.append(ids)
        return out, float(lib.fa_offline_result_audio_seconds(res))
    finally:
        lib.fa_offline_free_result(res)


# (name, sample format, channels, rate, frames per utterance): 8 kHz s16, 44.1 kHz stereo s24, 48 kHz f32
INPUTS = [("8k_s16", 1, 1, 8000, (16000, 9001, 24000)), ("44k1_s24_stereo", 2, 2, 44100, (88200, 50000)), ("48k_f32", 0, 1, 48000, (96000, 60001))]


def _speechlike(fmt, channels, rate, frames, seed):
    """Speech-like synthetic audio at `rate` in the given layout (the channels carry scaled copies)."""
    w = synth.make_wav(int(frames), seed, "speechlike").numpy().astype(np.float32)
    x = np.stack([w * (0.9 - 0.1 * c) for c in range(channels)], axis=1) if channels > 1 else w
    if fmt == 0:
        return np.ascontiguousarray(x, np.float32)
    if fmt == 1:
        return np.clip(np.round(x * 32767), -32768, 32767).astype(np.int16)
    s = np.clip(np.round(x.reshape(-1) * 8388607), -8388608, 8388607).astype(np.int32)     # s24 packed: the low three bytes
    return np.ascontiguousarray(s.view(np.uint8).reshape(-1, 4)[:, :3].reshape(x.shape[0], -1))


def _rows16(arr, fmt, channels, rate, mode):
    """The matching reference's 16 kHz float32 rows: the Python route (fa_pcm_decode -> funasr_b200.resample) for the loader, the
    reference LinearResample of the decoded samples for the runtime."""
    n = arr.shape[0]
    dec = _decode(arr.reshape(-1).view(np.uint8), fmt, channels, n)
    if mode == _abi.RESAMPLE_RUNTIME:
        return np.ascontiguousarray(linres_rows(dec.cpu().numpy(), rate))
    out, ol = resample(dec[None].contiguous(), torch.tensor([n], dtype=torch.int32, device=DEV), rate, 16000)
    return np.ascontiguousarray(out[0, :int(ol[0])].cpu().numpy())


@pytest.mark.parametrize("mode", [_abi.RESAMPLE_LOADER, _abi.RESAMPLE_RUNTIME])
def test_offline_infer_audio_equals_16k_rows(files, mode):
    """Ids and BiCif stamps of fa_offline_infer_audio equal fa_offline_infer_hw on the reference's 16 kHz rows; audio_seconds counts
    the caller's frames at the caller's rate."""
    lib = _lib()
    for key in ("asr", "bicif"):
        h = lib.fa_offline_init(files[key].encode(), 0, _abi.GEMM_F16X3)
        assert h, lib.fa_offline_last_error()
        for name, fmt, ch, rate, frames in INPUTS:
            arrs = [_speechlike(fmt, ch, rate, n, 20 + i) for i, n in enumerate(frames)]
            p, l = _ptrs(arrs)
            d = _abi.FaAudioFormat(fmt, ch, rate, mode)
            got, secs = _result(lib, lib.fa_offline_infer_audio(h, p, l, len(arrs), C.byref(d), None, 0, None, None), stamped=True)
            rows = [_rows16(a, fmt, ch, rate, mode) for a in arrs]
            p16, l16 = _ptrs(rows)
            want, _ = _result(lib, lib.fa_offline_infer_hw(h, p16, l16, len(rows), 0, None, 0), stamped=True)
            assert got == want and any(g[0] for g in got), (key, name, mode)
            assert abs(secs - sum(frames) / rate) < 1e-4
        lib.fa_offline_uninit(h)


def test_loader_mode_equals_paraformer_inference_fs():
    """Loader mode gives ParaformerB200.inference(fs=...)'s ids (its loader resamples with the same table and kernel)."""
    import tempfile
    import funasr_b200
    from test_abi_host import _tiny_conf
    m = funasr_b200.ParaformerB200(**_tiny_conf())
    m.load_state_dict(synth.make_state_dict(CFG, 3), strict=True)
    m.to(DEV).eval()
    cmvn = synth.make_cmvn(CFG, 1)
    fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0,
                                     cmvn=cmvn)
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "m.fab2")
        pack.write_model_file(path, synth.make_state_dict(CFG, 3), CFG, cmvn)
        rec = OfflineRecognizer(path, 0, "fp32")                # the plugin's default gemm_mode
        for rate in (8000, 48000):
            wavs = [_speechlike(0, 1, rate, n, 40 + i) for i, n in enumerate((rate * 2, rate + 777))]
            res, _ = m.inference(wavs, key=["a", "b"], tokenizer=None, frontend=fe, device=DEV, fs=rate)
            assert rec.infer(wavs, fs=rate) == [r["token_int"] for r in res], rate
        rec.close()


@pytest.mark.parametrize("mode", [_abi.RESAMPLE_LOADER, _abi.RESAMPLE_RUNTIME])
def test_sensevoice_queries_and_seaco_hotwords(tmp_path, files, mode):
    from conftest import load_sv_case
    cfg, wseed, _, cmvn, _ = load_sv_case("sv_tiny_ragged3")
    sv_path = str(tmp_path / "sv.fab2")
    pack.write_sensevoice_model_file(sv_path, synth.make_sensevoice_state_dict(cfg, wseed), cfg, cmvn)
    name, fmt, ch, rate, frames = INPUTS[0]
    arrs = [_speechlike(fmt, ch, rate, n, 60 + i) for i, n in enumerate(frames)]
    rows = [_rows16(a, fmt, ch, rate, mode) for a in arrs]
    sv = OfflineRecognizer(sv_path, 0, "fp16x3")
    for lang, itn in (("zh", True), (["en", "yue", "auto"], False)):
        got = sv.infer(arrs, language=lang, use_itn=itn, fs=rate, resampler=["loader", "runtime"][mode])
        assert got == sv.infer(rows, language=lang, use_itn=itn) and all(got)
    sv.close()
    se = OfflineRecognizer(files["seaco"], 0, "fp16x3")
    hw = se.hotword_embeddings([[5, 6, 7], [9, 10], [11, 12, 13, 14], [20, 21], [30, 31, 32], [1]])
    got = se.infer(arrs, hotword_embeddings=hw, fs=rate, resampler=["loader", "runtime"][mode])
    assert got == se.infer(rows, hotword_embeddings=hw) and all(got)
    se.close()


@pytest.mark.parametrize("mode", ["loader", "runtime"])
def test_long_audio_vad_and_speaker_at_8k(files, mode):
    """fa_offline_infer_vad_audio at 8 kHz s16: the segments, ids and `spk` labels of the 16 kHz call on the matching rows; the same
    for fa_vad_infer_audio and fa_spk_embed_audio."""
    rec, vad, spk = OfflineRecognizer(files["asr"], 0, "fp16x3"), OfflineVad(files["vad"], 0), OfflineSpeaker(files["spk"], 0, "fp32")
    m = _abi.RESAMPLERS[mode]
    recs = {"longaudio_40s": synth.make_vad_wav(*LONG_CASES["longaudio_40s"][:3]).numpy(),
            "spk_two_voices": synth.make_voice_wav(*SPK_CASES["spk_two_voices"][:2]).numpy()}
    for name, w16 in recs.items():
        x8 = np.clip(np.round(w16[::2] * 32767), -32768, 32767).astype(np.int16)
        rows = _rows16(x8, 1, 1, 8000, m)
        got = rec.infer_long([x8], vad, spk=spk, fs=8000, resampler=mode)[0]
        want = rec.infer_long([rows], vad, spk=spk)[0]
        assert got == want and got["vad_segments"], name
        assert abs(rec.last_audio_seconds - x8.size / 8000) < 1e-4
        assert vad.segments(x8, fs=8000, resampler=mode) == vad.segments(rows)
    chunks = [_speechlike(1, 1, 8000, n, 80 + i) for i, n in enumerate((12000, 8000, 30001))]
    assert np.array_equal(spk.embed(chunks, fs=8000, resampler=mode), spk.embed([_rows16(c, 1, 1, 8000, m) for c in chunks]))
    for h in (rec, vad, spk):
        h.close()


def test_16k_mono_entries_are_the_old_ones(files):
    """At 16 kHz mono f32 / s16 the new entries give the old entries' outputs with the same fa_launch_count delta."""
    lib = _lib()
    h = lib.fa_offline_init(files["bicif"].encode(), 0, _abi.GEMM_F16X3)
    v = lib.fa_vad_init(files["vad"].encode(), 0)
    s = lib.fa_spk_init(files["spk"].encode(), 0, _abi.GEMM_F32_SIMT)
    w = synth.make_vad_wav(*LONG_CASES["longaudio_40s"][:3]).numpy()
    for fmt, arrs in ((0, [w[:48000], w[5000:40000]]), (1, [np.round(w[:48000] * 32767).astype(np.int16), np.round(w[7:30000] * 32767).astype(np.int16)])):
        p, l = _ptrs(arrs)
        d = _abi.FaAudioFormat(fmt, 1, 16000, _abi.RESAMPLE_RUNTIME)

        def counted(f):
            torch.cuda.synchronize()
            before = lib.fa_launch_count()
            out = f()
            return out, lib.fa_launch_count() - before
        old = counted(lambda: _result(lib, lib.fa_offline_infer_hw(h, p, l, 2, fmt, None, 0), True))
        new = counted(lambda: _result(lib, lib.fa_offline_infer_audio(h, p, l, 2, C.byref(d), None, 0, None, None), True))
        assert old == new
        o = _abi.FaLongAudioOptions(300, 60, 0, 15, _abi.FaVadRunOptions(1, 0, float("nan")))
        old = counted(lambda: _result(lib, lib.fa_offline_infer_vad(h, v, p, l, 2, fmt, None, 0, C.byref(o)), True))
        new = counted(lambda: _result(lib, lib.fa_offline_infer_vad_audio(h, v, None, p, l, 2, C.byref(d), None, 0, None, None, C.byref(o), 0), True))
        assert old == new
        e_old, e_new = np.zeros((2, 192), np.float32), np.zeros((2, 192), np.float32)
        n_old = counted(lambda: lib.fa_spk_embed(s, p, l, 2, fmt, e_old.ctypes.data))
        n_new = counted(lambda: lib.fa_spk_embed_audio(s, p, l, 2, C.byref(d), e_new.ctypes.data))
        assert n_old == n_new and np.array_equal(e_old, e_new)

        def vad_segs(r):
            assert r
            n = C.c_int64(0)
            q = lib.fa_vad_result_segments(r, C.byref(n))
            out = [int(q[k]) for k in range(2 * n.value)], float(lib.fa_vad_result_audio_seconds(r))
            lib.fa_vad_free_result(r)
            return out
        old = counted(lambda: vad_segs(lib.fa_vad_infer(v, arrs[0].ctypes.data, arrs[0].shape[0], fmt, None)))
        new = counted(lambda: vad_segs(lib.fa_vad_infer_audio(v, arrs[0].ctypes.data, arrs[0].shape[0], C.byref(d), None)))
        assert old == new
    lib.fa_offline_uninit(h), lib.fa_vad_uninit(v), lib.fa_spk_uninit(s)


def test_refusals_before_any_launch(files):
    lib = _lib()
    h = lib.fa_offline_init(files["asr"].encode(), 0, _abi.GEMM_F16X3)
    v = lib.fa_vad_init(files["vad"].encode(), 0)
    s = lib.fa_spk_init(files["spk"].encode(), 0, _abi.GEMM_F32_SIMT)
    x = np.zeros(16000, np.int16)
    p, l = _ptrs([x])
    cases = [((5, 1, 8000, 0), b"bad sample_format 5"), ((1, 0, 8000, 0), b"channels 0 outside 1..64"), ((1, 65, 8000, 0), b"channels 65"),
             ((1, 1, 999, 0), b"sample rate 999 Hz outside"), ((1, 1, 16001, 0), b"sample rate 16001 Hz: its loader resampling table"),
             ((1, 1, 8000, 2), b"bad resampler 2")]
    o = _abi.FaLongAudioOptions(300, 60, 0, 15, _abi.FaVadRunOptions(1, 0, float("nan")))
    emb = np.zeros((1, 192), np.float32)
    torch.cuda.synchronize()
    before = lib.fa_launch_count()
    for desc, msg in cases + [(None, b"audio format is NULL")]:
        d = None if desc is None else C.byref(_abi.FaAudioFormat(*desc))
        assert not lib.fa_offline_infer_audio(h, p, l, 1, d, None, 0, None, None)
        assert msg in lib.fa_offline_last_error(), (desc, lib.fa_offline_last_error())
        assert not lib.fa_offline_infer_vad_audio(h, v, s, p, l, 1, d, None, 0, None, None, C.byref(o), 0)
        assert msg in lib.fa_offline_last_error()
        assert not lib.fa_vad_infer_audio(v, x.ctypes.data, x.size, d, None)
        assert msg in lib.fa_offline_last_error()
        assert lib.fa_spk_embed_audio(s, p, l, 1, d, emb.ctypes.data) != 0
        assert msg in lib.fa_offline_last_error()
    # 199 frames at 8 kHz are 398 samples at 16 kHz: under the 400 the recogniser and CAM++ need
    short = np.zeros(199, np.int16)
    ps, ls = _ptrs([short])
    d = C.byref(_abi.FaAudioFormat(1, 1, 8000, 0))
    assert not lib.fa_offline_infer_audio(h, ps, ls, 1, d, None, 0, None, None)
    assert b">= 400 samples (25 ms) at 16 kHz" in lib.fa_offline_last_error()
    assert lib.fa_spk_embed_audio(s, ps, ls, 1, d, emb.ctypes.data) != 0
    assert b"input 0 has 398 samples at 16 kHz" in lib.fa_offline_last_error()
    assert not lib.fa_offline_infer_audio(h, p, l, 1, C.byref(_abi.FaAudioFormat(1, 1, 8000, 0)), None, 0, (C.c_int32 * 1)(0), None)
    assert b"need a SenseVoice model file" in lib.fa_offline_last_error()
    assert lib.fa_launch_count() == before
    lib.fa_offline_uninit(h), lib.fa_vad_uninit(v), lib.fa_spk_uninit(s)


# ------------------------------------------------------------------------------------------------ the runtime shim
_CLIENT = r'''
#include <stdio.h>
#include <fstream>
#include <sstream>
#include <string>
#include "funasrruntime_b200.h"
static std::string slurp(const char* p) { std::ifstream f(p, std::ios::binary); std::stringstream s; s << f.rdbuf(); return s.str(); }
static void show(const char* tag, FUNASR_RESULT r) {
  if (!r) { printf("%s ERROR %s\n", tag, FunB200LastError()); return; }
  printf("%s %s|%s|%.4f\n", tag, FunASRGetResult(r, 0), FunASRGetStamp(r), FunASRGetRetSnippetTime(r));
  FunASRFreeResult(r);
}
static void vad(const char* tag, FUNASR_RESULT r) {
  if (!r) { printf("%s ERROR %s\n", tag, FunB200LastError()); return; }
  printf("%s", tag);
  for (auto& s : *FsmnVadGetResult(r, 0)) printf(" %d,%d", s[0], s[1]);
  printf("\n");
  FsmnVadFreeResult(r);
}
// argv: asr-dir vad-dir pcm8k wav8k wav16k(f32)
int main(int argc, char** argv) {
  std::vector<std::vector<float>> hw;
  const std::string pcm = slurp(argv[3]), w16 = slurp(argv[5]);
  for (int with_vad = 0; with_vad < 2; ++with_vad) {
    std::map<std::string, std::string> mp{{"model-dir", argv[1]}};
    if (with_vad) mp["vad-dir"] = argv[2];
    FUNASR_HANDLE h = FunOfflineInit(mp, 1, true, 1);
    if (!h) { printf("init ERROR %s\n", FunB200LastError()); return 1; }
    const char* t = with_vad ? "vad_" : "";
    std::string tag = std::string(t);
    show((tag + "pcm8k").c_str(), FunOfflineInferBuffer(h, pcm.data(), (int)pcm.size(), RASR_NONE, nullptr, hw, 8000, "pcm", true, nullptr));
    show((tag + "file8k").c_str(), FunOfflineInfer(h, argv[4], RASR_NONE, nullptr, hw, 16000, true, nullptr));
    show((tag + "ref16k").c_str(), FunOfflineInferBuffer(h, w16.data(), (int)w16.size(), RASR_NONE, nullptr, hw, 16000, "wav", true, nullptr));
    FunOfflineUninit(h);
  }
  std::map<std::string, std::string> vp{{"model-dir", argv[2]}};
  FUNASR_HANDLE v = FsmnVadInit(vp, 1);
  vad("fsmn_pcm8k", FsmnVadInferBuffer(v, pcm.data(), (int)pcm.size(), nullptr, true, 8000, "pcm"));
  vad("fsmn_ref16k", FsmnVadInferBuffer(v, w16.data(), (int)w16.size(), nullptr, true, 16000, "wav"));
  FsmnVadUninit(v);
  return 0;
}
'''


def _wav(data, tag, bits, rate):
    fmt_chunk = struct.pack("<HHIIHH", tag, 1, rate, rate * bits // 8, bits // 8, bits)
    return b"RIFF" + struct.pack("<I", 4 + 8 + len(fmt_chunk) + 8 + len(data)) + b"WAVE" + b"fmt " + struct.pack("<I", len(fmt_chunk)) + \
        fmt_chunk + b"data" + struct.pack("<I", len(data)) + data


def test_runtime_shim_at_8k(tmp_path, files):
    """FunOfflineInferBuffer (8 kHz "pcm"), FunOfflineInfer (an 8 kHz WAV file), with and without vad-dir, and FsmnVadInferBuffer
    return the text, stamps and segments of the 16 kHz float buffer the reference LinearResample makes of the same audio."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    src = tmp_path / "client.cpp"
    src.write_text(_CLIENT)
    exe = str(tmp_path / "client")
    libdir = os.path.join(ROOT, "funasr_b200")
    r = subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), str(src), "-L" + libdir, "-lfunasr_b200",
                        "-Wl,-rpath," + libdir, "-o", exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    asr_dir, vad_dir = _vocab_dir(tmp_path, files["vad"], files["bicif"], CFG.vocab)
    w16 = synth.make_vad_wav(*LONG_CASES["longaudio_40s"][:3]).numpy()
    x8 = np.clip(np.round(w16[::2] * 32767), -32768, 32767).astype(np.int16)
    ref = linres_rows(x8.astype(np.float32) / np.float32(32768), 8000)
    (tmp_path / "a.pcm").write_bytes(x8.tobytes())
    (tmp_path / "a8k.wav").write_bytes(_wav(x8.tobytes(), 1, 16, 8000))
    (tmp_path / "ref16k.wav").write_bytes(_wav(ref.astype(np.float32).tobytes(), 3, 32, 16000))
    p = subprocess.run([exe, asr_dir, vad_dir, str(tmp_path / "a.pcm"), str(tmp_path / "a8k.wav"), str(tmp_path / "ref16k.wav")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-2000:]
    out = dict(ln.split(" ", 1) if " " in ln else (ln, "") for ln in p.stdout.splitlines())
    assert not any(v.startswith("ERROR") for v in out.values()), p.stdout
    for pre in ("", "vad_"):
        want = out[pre + "ref16k"].rsplit("|", 1)[0]
        assert want.split("|")[0] and want.split("|")[1], (pre, want)
        for k in ("pcm8k", "file8k"):
            text_stamp, secs = out[pre + k].rsplit("|", 1)
            assert text_stamp == want, (pre, k)
            assert abs(float(secs) - x8.size / 8000) < 1e-3
    assert out["fsmn_pcm8k"] == out["fsmn_ref16k"] and out["fsmn_pcm8k"].strip()
