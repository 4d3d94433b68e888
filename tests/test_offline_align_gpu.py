"""GPU: forced alignment through the C handle API (fa_align_init / fa_align_infer) for the fa-zh MonotonicAligner shape -- the
reference's golden stamps, equality with MonotonicAlignerB200.inference in every gemm mode (the same kernels on the same planes),
audio at other rates and layouts, the refusals of fa_align_infer before any launch, grow-then-shrink batches, and the C client."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from funasr_b200 import _abi, pack, synth
from funasr_b200.offline import OfflineAligner
from test_aligner_gpu import ALIGNER_GOLDENS, _CharTok, _model
from test_audio_in_gpu import _rows16, _speechlike

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TOKENS = synth.aligner_token_list(400)
EOS = TOKENS.index("</s>")


def _golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    ids = [r.tolist() for r in np.split(z["ids_flat"], np.cumsum(z["ids_len"])[:-1])]
    split = lambda flat, lens: [s.tolist() for s in np.split(z[flat].reshape(-1, 2), np.cumsum(z[lens])[:-1])]   # noqa: E731
    wavs = [synth.make_aligner_wav(float(sec), int(s)).numpy() for sec, s in z["wav_spec"]]
    return wavs, ids, split("stamps_flat", "stamps_len"), split("final_flat", "final_len")


def _file(tmp_path_factory, cfg_name, seed):
    cfg = getattr(synth, cfg_name)
    path = str(tmp_path_factory.mktemp("aligner") / ("%s.fab2" % cfg_name))
    pack.write_aligner_model_file(path, synth.make_aligner_state_dict(cfg, seed), cfg, synth.make_cmvn(cfg, seed=1), token_list=TOKENS)
    return path


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    return {name: _file(tmp_path_factory, *spec) for name, spec in ALIGNER_GOLDENS.items()}


def _align_raw(lib, h, arrs, ids, fmt):
    """fa_align_infer -> (stamps per utterance, ids per utterance, audio seconds), or None with the error."""
    n = len(arrs)
    toks = [np.ascontiguousarray(t, np.int32) for t in ids]
    p = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
    l = (C.c_int64 * n)(*[a.shape[0] for a in arrs])
    rows = (C.c_void_p * n)(*[t.ctypes.data if t.size else None for t in toks])
    k = (C.c_int32 * n)(*[t.size for t in toks])
    res = lib.fa_align_infer(h, p, l, n, C.byref(fmt), rows, k)
    if not res:
        return None, lib.fa_offline_last_error()
    cnt = C.c_int32(0)
    st, kept = [], []
    for i in range(lib.fa_offline_result_count(res)):
        s = lib.fa_offline_result_stamps(res, i, C.byref(cnt))
        st.append([[int(s[2 * j]), int(s[2 * j + 1])] for j in range(cnt.value)])
        q = lib.fa_offline_result_ids(res, i, C.byref(cnt))
        kept.append([int(q[j]) for j in range(cnt.value)])
    secs = float(lib.fa_offline_result_audio_seconds(res))
    lib.fa_offline_free_result(res)
    return (st, kept, secs), None


@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("name", list(ALIGNER_GOLDENS))
def test_handle_stamps_vs_reference_golden(files, name, mode):
    """The reference's stamps (ts_prediction_lfr6_standard and after sentence_postprocess) exactly, and the transcript as the ids."""
    wavs, ids, stamps, final = _golden(name)
    lib = _abi.load()
    h = lib.fa_align_init(files[name].encode(), 0, _abi.GEMM_MODES[mode])
    assert h, lib.fa_offline_last_error()
    (got, kept, secs), err = _align_raw(lib, h, wavs, ids, _abi.FaAudioFormat(0, 1, 16000, 0))
    assert err is None, err
    assert got == stamps == final
    assert kept == ids
    assert abs(secs - sum(w.size for w in wavs) / 16000) < 1e-3
    lib.fa_align_uninit(h)


def _python(cfg_name, seed, mode, wavs, ids):
    from funasr_b200.modules import WavFrontendB200
    import torch
    cfg = getattr(synth, cfg_name)
    model = _model(cfg, seed, mode)
    fe = WavFrontendB200(cmvn=synth.make_cmvn(cfg, seed=1), lfr_m=7, lfr_n=6, dither=0.0)
    pairs = [(torch.from_numpy(w), list(t)) for w, t in zip(wavs, ids)]
    res, _ = model.inference(pairs, key=["u%d" % i for i in range(len(pairs))], tokenizer=_CharTok(TOKENS), frontend=fe, device=DEV,
                             data_type=("sound", "text"))
    return [r["timestamp"] for r in res]


@pytest.mark.parametrize("mode", ["fp32", "fp16", "fp16x3", "fp16x6"])
def test_handle_equals_python_class(files, mode):
    """Stamps equal MonotonicAlignerB200.inference on the same waveforms and ids: a transcript ending in </s>, the transcript [</s>]
    (no token after the drop), an empty transcript, one longer than the audio fires for, and a batch of one."""
    wavs, ids, _, _ = _golden("aligner_tiny_ragged3")
    g = np.random.default_rng(3)
    batch_ids = [ids[0] + [EOS], [EOS], [], [int(t) for t in g.integers(3, 403, 60)]]
    batch_wavs = [wavs[0], wavs[2], wavs[1], wavs[1]]
    al = OfflineAligner(files["aligner_tiny_ragged3"], 0, mode)
    got = al.align(batch_wavs, batch_ids)
    want = _python("ALIGNER_TINY", 5, mode, batch_wavs, batch_ids)
    assert got == want
    assert len(got[0]) == len(ids[0]) and got[1] == [] and got[2] == [] and got[3]
    one = al.align([wavs[0]], [ids[0]])
    assert one == _python("ALIGNER_TINY", 5, mode, [wavs[0]], [ids[0]]) == [got[0]]
    al.close()


@pytest.mark.parametrize("rate", [8000, 44100])
def test_audio_formats_equal_16k_rows(files, rate):
    """s16 stereo at 8 kHz and 44.1 kHz (loader resampler) give the stamps of the handle fed the 16 kHz rows of the same audio."""
    al = OfflineAligner(files["aligner_tiny_ragged3"], 0, "fp16x3")
    _, ids, _, _ = _golden("aligner_tiny_ragged3")
    arrs = [_speechlike(1, 2, rate, n, 60 + i) for i, n in enumerate((rate * 3, rate * 2 + 999, rate))]
    got = al.align(arrs, ids, fs=rate, resampler="loader")
    secs = al.last_audio_seconds
    rows = [_rows16(a, 1, 2, rate, _abi.RESAMPLE_LOADER) for a in arrs]
    assert got == al.align(rows, ids) and any(got)
    assert abs(secs - sum(a.shape[0] for a in arrs) / rate) < 1e-4
    al.close()


def test_refusals_before_any_launch_and_growing_buffers(files):
    """Each fa_align_infer refusal launches nothing and leaves the handle usable; batches that grow then shrink give identical stamps."""
    lib = _abi.load()
    h = lib.fa_align_init(files["aligner_tiny_ragged3"].encode(), 0, _abi.GEMM_F16X3)
    assert h, lib.fa_offline_last_error()
    wavs, ids, stamps, _ = _golden("aligner_tiny_ragged3")
    f16 = _abi.FaAudioFormat(0, 1, 16000, 0)
    (first, _, _), _ = _align_raw(lib, h, wavs, ids, f16)
    assert first == stamps
    w = np.ascontiguousarray(wavs[0])
    p = (C.c_void_p * 2)(w.ctypes.data, w.ctypes.data)
    l = (C.c_int64 * 2)(w.size, w.size)
    t = np.array(ids[0], np.int32)
    rows = (C.c_void_p * 2)(t.ctypes.data, t.ctypes.data)
    k = (C.c_int32 * 2)(t.size, t.size)
    fmt = C.byref(f16)
    short = np.zeros(399, np.float32)
    cases = [
        ("NULL handle", lambda: lib.fa_align_infer(None, p, l, 2, fmt, rows, k), b"bad argument"),
        ("NULL bufs", lambda: lib.fa_align_infer(h, None, l, 2, fmt, rows, k), b"bad argument"),
        ("NULL n_frames", lambda: lib.fa_align_infer(h, p, None, 2, fmt, rows, k), b"bad argument"),
        ("NULL fmt", lambda: lib.fa_align_infer(h, p, l, 2, None, rows, k), b"bad argument"),
        ("NULL n_ids", lambda: lib.fa_align_infer(h, p, l, 2, fmt, rows, None), b"bad argument"),
        ("batch 0", lambda: lib.fa_align_infer(h, p, l, 0, fmt, rows, k), b"bad argument"),
        ("n_ids < 0", lambda: lib.fa_align_infer(h, p, l, 2, fmt, rows, (C.c_int32 * 2)(3, -1)), b"utterance 1"),
        ("NULL ids", lambda: lib.fa_align_infer(h, p, l, 2, fmt, None, k), b"utterance 0"),
        ("NULL ids[1]", lambda: lib.fa_align_infer(h, p, l, 2, fmt, (C.c_void_p * 2)(t.ctypes.data, None), k), b"utterance 1"),
        ("short", lambda: lib.fa_align_infer(h, (C.c_void_p * 2)(w.ctypes.data, short.ctypes.data), (C.c_int64 * 2)(w.size, 399), 2, fmt,
                                             rows, k), b"utterance 1"),
        ("short at 8 kHz", lambda: lib.fa_align_infer(h, p, (C.c_int64 * 2)(w.size, 199), 2, C.byref(_abi.FaAudioFormat(0, 1, 8000, 0)),
                                                      rows, k), b"at 16 kHz"),
        ("bad format", lambda: lib.fa_align_infer(h, p, l, 2, C.byref(_abi.FaAudioFormat(9, 1, 16000, 0)), rows, k), b"sample_format"),
        ("bad channels", lambda: lib.fa_align_infer(h, p, l, 2, C.byref(_abi.FaAudioFormat(0, 0, 16000, 0)), rows, k), b"channels"),
        ("bad rate", lambda: lib.fa_align_infer(h, p, l, 2, C.byref(_abi.FaAudioFormat(0, 1, 500, 0)), rows, k), b"sample rate"),
        ("bad resampler", lambda: lib.fa_align_infer(h, p, l, 2, C.byref(_abi.FaAudioFormat(0, 1, 16000, 7)), rows, k), b"resampler"),
        ("huge table", lambda: lib.fa_align_infer(h, p, l, 2, C.byref(_abi.FaAudioFormat(0, 1, 16001, 0)), rows, k), b"32 MiB"),
    ]
    for name, call, needle in cases:
        before = lib.fa_launch_count()
        assert not call(), name
        assert needle in lib.fa_offline_last_error(), (name, lib.fa_offline_last_error())
        assert lib.fa_launch_count() == before, name
    # the handle still works, and a grown then shrunk batch reuses the grown buffers with the same stamps
    (again, _, _), _ = _align_raw(lib, h, wavs, ids, f16)
    assert again == first
    (big, _, _), _ = _align_raw(lib, h, wavs * 6, ids * 6, f16)
    assert big == first * 6
    (small, _, _), _ = _align_raw(lib, h, wavs[:1], ids[:1], f16)
    assert small == first[:1]
    (again, _, _), _ = _align_raw(lib, h, wavs, ids, f16)
    assert again == first
    lib.fa_align_uninit(h)


def test_c_client_prints_the_golden_stamps(tmp_path, files):
    """examples/offline_align_client.c on the tiny golden's first utterance (a tokens.txt, the space-separated transcript): its float32
    samples give the golden stamps; as s16le PCM (rounded, so a fire may move by one upsampled frame) the stamps the handle gives for
    the same samples."""
    exe = str(tmp_path / "offline_align_client")
    libdir = os.path.join(ROOT, "funasr_b200")
    r = subprocess.run(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "offline_align_client.c"),
                        "-L" + libdir, "-lfunasr_b200", "-Wl,-rpath," + libdir, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    wavs, ids, stamps, _ = _golden("aligner_tiny_ragged3")
    (tmp_path / "tokens.txt").write_text("\n".join(TOKENS) + "\n", encoding="utf-8")
    (tmp_path / "t.txt").write_text(" ".join(TOKENS[i] for i in ids[0]) + "\n", encoding="utf-8")
    pcm = np.clip(np.round(wavs[0] * 32768), -32768, 32767).astype(np.int16)
    al = OfflineAligner(files["aligner_tiny_ragged3"], 0, "fp16x3")
    for kind, samples, want in (("f32", wavs[0].astype(np.float32), stamps[0]), ("s16", pcm, al.align([pcm], [ids[0]])[0])):
        (tmp_path / "a.pcm").write_bytes(samples.tobytes())
        run = subprocess.run([exe, files["aligner_tiny_ragged3"], str(tmp_path / "tokens.txt"), str(tmp_path / "a.pcm"), str(tmp_path / "t.txt"),
                              "16000", kind], capture_output=True, text=True)
        assert run.returncode == 0, run.stderr
        assert run.stdout.strip().split("\n") == ["%s %d %d" % (TOKENS[i], s, e) for i, (s, e) in zip(ids[0], want)], kind
        assert len(want) == len(ids[0])
    al.close()
