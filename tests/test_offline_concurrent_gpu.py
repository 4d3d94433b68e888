"""GPU: one handle shared by many threads, as the reference's servers share one FunOfflineInit handle among their decoder threads.
Every call's result equals the same call made alone; a malformed call fails on its own thread with its own message.  The batched
FSMN-VAD of long audio over many recordings (fa_fsmn_vad_forward_batch, fa_frame_decibels_batch) equals the single-recording
entries bit for bit."""
import ctypes as C
import os
import shutil
import subprocess
import threading

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

from funasr_b200 import _abi, pack, synth
from funasr_b200.offline import OfflineRecognizer, OfflineVad
from test_offline_punc_host import ENC_CONF as PUNC_ENC_CONF
from test_offline_seaco_gpu import _seaco_file
from test_offline_stamps_gpu import BICIF_SEED, _bicif_file
from test_offline_sv_gpu import _sv_file
from test_offline_vad_gpu import LONG_CASES, _s16, _wav_bytes
from test_vad_host import VAD_CASES

CFG = synth.PARAFORMER_TINY
DEV = "cuda:0"


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("conc")
    cmvn = synth.make_cmvn(CFG, 1)
    out = {"vad": str(d / "vad.fab2"), "asr": str(d / "asr.fab2"), "bicif": str(d / "bicif.fab2"), "seaco": str(d / "seaco.fab2")}
    pack.write_vad_model_file(out["vad"], synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    pack.write_model_file(out["asr"], synth.make_state_dict(CFG, 3), CFG, cmvn)
    _bicif_file(out["bicif"], CFG, BICIF_SEED, cmvn)
    _seaco_file(out["seaco"], 5, 8, cmvn)
    return out


def _long_wavs():
    wavs = [synth.make_vad_wav(*LONG_CASES[k][:3]).numpy() for k in ("longaudio_40s", "longaudio_25s_onebatch")]
    return wavs + [synth.make_vad_wav(18.0, 21).numpy()]


def _utts(k):
    return [synth.make_wav(8000 + 1237 * ((k * 3 + j) % 11), 40 + k * 3 + j, "speechlike").numpy() for j in range(1 + k % 3)]


def _threads(n, fn):
    """fn(k) on n threads released together -> results by k; the first exception raised on a thread is re-raised here."""
    out, errs = [None] * n, []
    bar = threading.Barrier(n)

    def run(k):
        try:
            bar.wait()
            out[k] = fn(k)
        except BaseException as e:                                      # noqa: BLE001 - re-raised below
            errs.append(e)
    ts = [threading.Thread(target=run, args=(k,)) for k in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errs:
        raise errs[0]
    return out


@pytest.mark.gpu
def test_sixteen_threads_on_one_handle(tmp_path_factory, files):
    """16 threads share one recogniser and one VAD handle, a few calls each (short batches and long audio): plain, BiCif, SeACo with
    two hotword sets, SenseVoice with a query per thread.  Every result equals the call made alone."""
    vad = OfflineVad(files["vad"], 0)
    lw = _long_wavs()
    for key in ("asr", "bicif"):
        rec = OfflineRecognizer(files[key], 0, "fp16x3")
        solo = [rec.infer_stamped(_utts(k)) for k in range(16)]
        solo_long = [rec.infer_long([lw[k % 3]], vad, batch_size_s=6) for k in range(16)]
        got = _threads(16, lambda k: [rec.infer_stamped(_utts(k)), rec.infer_long([lw[k % 3]], vad, batch_size_s=6), rec.infer_stamped(_utts(k))])
        assert got == [[solo[k], solo_long[k], solo[k]] for k in range(16)]
        rec.close()
    sea = OfflineRecognizer(files["seaco"], 0, "fp16x3")
    sets = [sea.hotword_embeddings(synth.make_hotwords(4 + 20 * s, CFG.vocab, seed=s) + [[1]]) for s in (0, 1)]
    solo = [sea.infer(_utts(k), hotword_embeddings=sets[k % 2]) for k in range(16)]
    solo_long = [sea.infer_long([lw[k % 3]], vad, batch_size_s=6, hotword_embeddings=sets[k % 2]) for k in range(16)]
    got = _threads(16, lambda k: [sea.infer(_utts(k), hotword_embeddings=sets[k % 2]),
                                  sea.infer_long([lw[k % 3]], vad, batch_size_s=6, hotword_embeddings=sets[k % 2]),
                                  sea.hotword_embeddings([[5 + k, 7], [9]])])
    assert [g[:2] for g in got] == [[solo[k], solo_long[k]] for k in range(16)]
    assert all(np.array_equal(g[2], sea.hotword_embeddings([[5 + k, 7], [9]])) for k, g in enumerate(got))
    sea.close()
    sv = OfflineRecognizer(_sv_file(tmp_path_factory, "sv_tiny_ragged3")[0], 0, "fp16x3")
    langs = ["zh", "en", "yue", "ja"]
    solo = [sv.infer(_utts(k), language=langs[k % 4], use_itn=bool(k % 2)) for k in range(16)]
    solo_long = [sv.infer_long([lw[k % 3]], vad, batch_size_s=6, language=langs[k % 4]) for k in range(16)]
    got = _threads(16, lambda k: [sv.infer(_utts(k), language=langs[k % 4], use_itn=bool(k % 2)),
                                  sv.infer_long([lw[k % 3]], vad, batch_size_s=6, language=langs[k % 4])])
    assert got == [[solo[k], solo_long[k]] for k in range(16)]
    sv.close()
    segs = [vad.segments(w) for w in lw]
    assert _threads(9, lambda k: vad.segments(lw[k % 3])) == [segs[k % 3] for k in range(9)]
    vad.close()


@pytest.mark.gpu
def test_bad_request_among_good_ones(files):
    """A malformed call (a buffer under 400 samples, a pcm_format that does not exist) fails on its own thread with its own message;
    the calls around it succeed with their solo results."""
    rec = OfflineRecognizer(files["asr"], 0, "fp16x3")
    solo = [rec.infer(_utts(k)) for k in range(8)]

    def call(k):
        if k == 3:
            with pytest.raises(_abi.FunasrB200Error, match="400 samples"):
                rec.infer([np.zeros(100, np.float32)])
            return "refused"
        if k == 5:
            w = np.zeros(4000, np.float32)
            ptrs, lens = (C.c_void_p * 1)(w.ctypes.data), (C.c_int64 * 1)(w.size)
            assert not rec.lib.fa_offline_infer(rec.handle, ptrs, lens, 1, 7)
            assert rec.lib.fa_offline_last_error() == b"bad argument"
            return "refused"
        return rec.infer(_utts(k))
    got = _threads(8, call)
    assert got == [("refused" if k in (3, 5) else solo[k]) for k in range(8)]
    rec.close()


@pytest.mark.gpu
def test_rtf_client_eight_threads_equal_one(files, tmp_path):
    """examples/offline_rtf_client.cpp with vad-dir and punc-dir: 8 threads on one FunOfflineInit handle print the texts 1 thread
    prints."""
    inc = os.path.join(ROOT, "include")
    exe = str(tmp_path / "rtf_client")
    r = subprocess.run(["g++", "-std=c++17", "-pthread", '-DFUNASR_RUNTIME_HEADER="funasrruntime_b200.h"', "-I" + inc,
                        os.path.join(ROOT, "examples", "offline_rtf_client.cpp"), "-L" + os.path.join(ROOT, "funasr_b200"), "-lfunasr_b200",
                        "-Wl,-rpath," + os.path.join(ROOT, "funasr_b200"), "-o", exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    asr_dir, vad_dir, punc_dir = tmp_path / "asr", tmp_path / "vad", tmp_path / "punc"
    for d in (asr_dir, vad_dir, punc_dir):
        d.mkdir()
    shutil.copy(files["asr"], asr_dir / "model.fab2")
    (asr_dir / "tokens.txt").write_text("\n".join(chr(0x4E00 + i) for i in range(CFG.vocab)) + "\n", encoding="utf-8")
    shutil.copy(files["vad"], vad_dir / "vad.fab2")
    pack.write_punc_model_file(str(punc_dir / "punc.fab2"), synth.make_punc_state_dict(0), synth.PUNC_LIST, synth.punc_token_list(), 3,
                               PUNC_ENC_CONF)
    lines = []
    for k, w in enumerate(_long_wavs() + [synth.make_vad_wav(9.0 + k, 60 + k).numpy() for k in range(9)]):
        p = tmp_path / ("w%d.wav" % k)
        p.write_bytes(_wav_bytes(_s16(w), "s16"))
        lines.append("u%d %s" % (k, p))
    (tmp_path / "list.txt").write_text("\n".join(lines) + "\n")

    def run(n):
        r = subprocess.run([exe, str(asr_dir), str(tmp_path / "list.txt"), str(n), str(vad_dir), str(punc_dir)], stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:]
        out = r.stdout.strip().splitlines()
        assert out[-1].startswith("threads %d files 12 failed 0" % n), out[-1]
        return out[:-1]
    one = run(1)
    assert len(one) == 12 and sum(len(x.split(" ", 1)) > 1 for x in one) >= 3
    assert run(8) == one


def _st():
    return torch.cuda.current_stream().cuda_stream


@pytest.mark.gpu
def test_batched_vad_forward_and_decibels_equal_single_entries():
    """Ragged rows (0, 1, 19, 20, 33, 301 and 700 frames) in one fa_fsmn_vad_forward_batch equal fa_fsmn_vad_forward on each row alone,
    bit for bit, over a workspace and output full of NaN; fa_frame_decibels_batch on ragged recordings (one under 400 samples, the
    vad_130s and vad_silence recordings) equals fa_frame_decibels on each."""
    from funasr_b200.vad_model import VadEngine
    lib = _abi.load()
    eng = VadEngine(synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), DEV, synth.make_vad_cmvn(0))   # owns the weights enc points to
    enc = eng.enc
    frames = [301, 0, 19, 700, 1, 20, 33]
    B, T = len(frames), max(frames)
    g = torch.Generator().manual_seed(4)
    feats = torch.full((B, T, 400), float("nan"))
    for b, t in enumerate(frames):
        lvl = 4 * torch.sin(torch.arange(t, dtype=torch.float32) / 37.0)
        feats[b, :t] = torch.randn(t, 400, generator=g) + lvl[:, None]
    feats = feats.to(DEV)
    need = int(lib.fa_fsmn_vad_batch_workspace_bytes(C.byref(enc), B, T))
    ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
    sil = torch.full((B, T), float("nan"), device=DEV)
    fr = (C.c_int32 * B)(*frames)
    assert lib.fa_fsmn_vad_forward_batch(C.byref(enc), feats.data_ptr(), 400, fr, B, T, sil.data_ptr(), ws.data_ptr(), need, _st()) == 0
    for b, t in enumerate(frames):
        if t == 0:
            continue
        one = torch.full((t,), float("nan"), device=DEV)
        n1 = int(lib.fa_fsmn_vad_workspace_bytes(C.byref(enc), t))
        w1 = torch.zeros((n1,), dtype=torch.uint8, device=DEV)
        x = feats[b, :t].contiguous()
        assert lib.fa_fsmn_vad_forward(C.byref(enc), x.data_ptr(), 400, t, one.data_ptr(), None, w1.data_ptr(), n1, _st()) == 0
        torch.cuda.synchronize()
        assert torch.equal(sil[b, :t], one), b
    bad = (C.c_int32 * B)(*[T + 1] * B)
    assert lib.fa_fsmn_vad_forward_batch(C.byref(enc), feats.data_ptr(), 400, bad, B, T, sil.data_ptr(), ws.data_ptr(), need, _st()) == -1
    wavs = [synth.make_vad_wav(*VAD_CASES[k][:3]) for k in ("vad_130s", "vad_silence")] + [synth.make_wav(399, 3), synth.make_wav(4567, 5)]
    n = [w.numel() for w in wavs]
    nf = [(x - 400) // 160 + 1 if x >= 400 else 0 for x in n]
    stride, T = (max(n) + 3) // 4 * 4, max(nf)
    rows = torch.full((len(wavs), stride), float("nan"))
    for b, w in enumerate(wavs):
        rows[b, : w.numel()] = w
    rows = rows.to(DEV)
    db = torch.full((len(wavs), T), float("nan"), device=DEV)
    nf_d = torch.tensor(nf, dtype=torch.int32, device=DEV)
    assert lib.fa_frame_decibels_batch(rows.data_ptr(), stride, nf_d.data_ptr(), len(wavs), T, db.data_ptr(), _st()) == 0
    for b, t in enumerate(nf):
        one = torch.full((max(t, 1),), float("nan"), device=DEV)
        x = rows[b, : n[b]].contiguous()
        assert lib.fa_frame_decibels(x.data_ptr(), n[b], t, one.data_ptr(), _st()) == 0
        torch.cuda.synchronize()
        assert torch.equal(db[b, :t], one[:t]), b
        assert torch.isnan(db[b, t:]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_long_audio_batched_vad_equals_each_recording_alone(files, mode):
    """fa_offline_infer_vad over many recordings (one upload, one batched VAD pass) equals each recording alone and fa_vad_infer's
    segments, and the reference's golden ids: the long-audio goldens with the vad_130s and vad_silence recordings, a recording under
    400 samples and silence."""
    wavs = [synth.make_vad_wav(*LONG_CASES[k][:3]).numpy() for k in ("longaudio_40s", "longaudio_25s_onebatch")]
    wavs += [synth.make_vad_wav(*VAD_CASES[k][:3]).numpy() for k in ("vad_130s", "vad_silence")]
    wavs += [np.zeros(399, np.float32), np.zeros(32000, np.float32)]
    rec, vad = OfflineRecognizer(files["asr"], 0, mode), OfflineVad(files["vad"], 0)
    for kw, gold, i in (({"batch_size_s": 6}, "longaudio_40s", 0), ({"batch_size_s": 300}, "longaudio_25s_onebatch", 1)):
        many = rec.infer_long(wavs, vad, **kw)
        assert many == [rec.infer_long([w], vad, **kw)[0] for w in wavs]
        assert many[i]["token_int"] == np.load(os.path.join(GOLDEN, gold + ".npz"))["ids"].tolist()
        assert [m["vad_segments"] for m in many] == [vad.segments(w) for w in wavs]
    rec.close()
    vad.close()
