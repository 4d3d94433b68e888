"""GPU: FSMN-VAD and long-audio recognition through the C handle API (fa_vad_*, fa_offline_infer_vad, fa_gather_segments) and the
C++ runtime surface (FsmnVad*, FunOfflineInit with "vad-dir"), against the reference's golden segments / ids and against
LongAudioPipeline run in the same mode."""
import ctypes as C
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

import funasr_b200
from funasr_b200 import _abi, pack, synth, vad as V
from funasr_b200.offline import OfflineRecognizer, OfflineVad
from test_abi_host import _tiny_conf
from test_vad_host import VAD_CASES

DEV = "cuda:0"
# must match tests/test_gpu_parity.py:test_long_audio_pipeline_vs_reference_golden
LONG_CASES = {"longaudio_40s": (40.0, 7, [(3.0, 2.5), (1.5, 2.2), (4.0, 3.0), (2.0, 2.2), (6.0, 2.4)], {"batch_size_s": 6}),
              "longaudio_25s_onebatch": (25.0, 8, [(2.0, 2.5), (3.0, 2.1)], {"batch_size_s": 300})}


def _gold(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


@pytest.fixture(scope="module")
def vad_file(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("vad") / "vad.fab2")
    pack.write_vad_model_file(path, synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    return path


@pytest.fixture(scope="module")
def asr_file(tmp_path_factory):
    cfg = synth.PARAFORMER_TINY
    path = str(tmp_path_factory.mktemp("asr") / "model.fab2")
    pack.write_model_file(path, synth.make_state_dict(cfg, 3), cfg, synth.make_cmvn(cfg, 1))
    return path


def _vad_plugin():
    c = synth.VAD_DEFAULT
    vad = funasr_b200.FsmnVADStreamingB200(encoder="FSMN", encoder_conf=dict(
        input_dim=c.input_dim, input_affine_dim=c.input_affine_dim, fsmn_layers=c.fsmn_layers, linear_dim=c.linear_dim, proj_dim=c.proj_dim,
        lorder=c.lorder, rorder=0, lstride=1, rstride=0, output_affine_dim=c.output_affine_dim, output_dim=c.output_dim))
    vad.load_state_dict(synth.make_vad_state_dict(c, 0), strict=True)
    vad.to(DEV).eval()
    fe = funasr_b200.WavFrontendOnlineB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=5, lfr_n=1,
                                           dither=0.0, cmvn=synth.make_vad_cmvn(0))
    return vad, fe


class _CountingAsr:
    """Wraps the ASR plugin to record each segment's token count by key ("<key>_<segment index>", long_audio.py)."""

    def __init__(self, m):
        self.m, self.seen = m, {}

    def inference(self, batch, key=None, **kw):
        res, meta = self.m.inference(batch, key=key, **kw)
        for r in res:
            self.seen[r["key"]] = len(r["token_int"])
        return res, meta


def _pipeline(mode, state=None, contextual=False):
    cfg = synth.PARAFORMER_TINY
    conf = _tiny_conf()
    conf["gemm_mode"] = mode
    if contextual:
        conf["decoder"] = "ContextualParaformerDecoderB200"
        asr = funasr_b200.ContextualParaformerB200(**conf)
    else:
        asr = funasr_b200.ParaformerB200(**conf)
    asr.load_state_dict(state if state is not None else synth.make_state_dict(cfg, 3), strict=True)
    asr.to(DEV).eval()
    asr_fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0,
                                         cmvn=synth.make_cmvn(cfg, 1))
    vad, vad_fe = _vad_plugin()
    counting = _CountingAsr(asr)
    return funasr_b200.LongAudioPipeline(counting, asr_fe, vad, vad_fe, device=DEV), counting, asr


def _python_result(pipe, counting, wav, **kw):
    counting.seen.clear()
    out = pipe.generate(wav, key="rec", **kw)
    segs = out["vad_segments"]
    ids = out.get("token_int", [])
    n_tok = [counting.seen.get("rec_%d" % i, 0) for i in range(len(segs))] if ids else [0] * len(segs)
    return {"token_int": ids, "vad_segments": segs, "n_tokens": n_tok}


def _wav_bytes(x, fmt):
    if fmt == "f32":
        data, tag, bits = np.ascontiguousarray(x, np.float32).tobytes(), 3, 32
    else:
        data, tag, bits = np.ascontiguousarray(x, np.int16).tobytes(), 1, 16
    fmt_chunk = struct.pack("<HHIIHH", tag, 1, 16000, 16000 * bits // 8, bits // 8, bits)
    return b"RIFF" + struct.pack("<I", 4 + 8 + len(fmt_chunk) + 8 + len(data)) + b"WAVE" + b"fmt " + struct.pack("<I", len(fmt_chunk)) + \
        fmt_chunk + b"data" + struct.pack("<I", len(data)) + data


def _s16(x):
    return np.clip(np.round(np.asarray(x, np.float32) * 32768.0), -32768, 32767).astype(np.int16)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(VAD_CASES))
def test_vad_handle_vs_reference_golden(vad_file, name):
    """fa_vad_infer on the reference's golden recordings (float32 PCM): segments bit-exact, and equal to the walk over the handle's
    own per-frame values."""
    seconds, seed, pattern, kw = VAD_CASES[name]
    g = _gold(name)
    wav = synth.make_vad_wav(seconds, seed, pattern).numpy()
    v = OfflineVad(vad_file, 0)
    segs, frames = v.segments(wav, want_frames=True, **kw)
    assert segs == g["segments"].tolist()
    assert frames.shape == (2, g["sil_prob"].shape[0])
    if frames.shape[1]:
        assert np.abs(frames[0] - g["sil_prob"]).max() <= 1e-4
    assert V.detect_segments(frames[0].tolist(), frames[1].tolist(), wav.size, **kw) == segs
    assert v.segments(wav[:399]) == []                                   # shorter than one frame
    v.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("name", list(LONG_CASES))
def test_long_audio_handle_vs_reference_golden_and_pipeline(vad_file, asr_file, name, mode):
    """fa_offline_infer_vad reproduces the unmodified reference's AutoModel(vad_model=...).generate ids, and equals LongAudioPipeline in
    the same mode: ids, segments and tokens per segment, with and without merge_vad; s16 input equals the pipeline on the dequantised
    audio."""
    seconds, seed, pattern, kw = LONG_CASES[name]
    g = _gold(name)
    wav = synth.make_vad_wav(seconds, seed, pattern).numpy()
    assert wav.size == int(g["n_samples"])
    rec, vad = OfflineRecognizer(asr_file, 0, mode), OfflineVad(vad_file, 0)
    got = rec.infer_long([wav], vad, **kw)[0]
    assert got["token_int"] == g["ids"].tolist()
    assert abs(rec.last_audio_seconds - wav.size / 16000.0) < 1e-3
    pipe, counting, _ = _pipeline(mode)
    want = _python_result(pipe, counting, wav, **kw)
    assert got == want and len(got["vad_segments"]) >= 2 and sum(got["n_tokens"]) == len(got["token_int"])
    for merge_s in (5, 15):
        got_m = rec.infer_long([wav], vad, merge_vad=True, merge_length_s=merge_s, **kw)[0]
        assert got_m == _python_result(pipe, counting, wav, merge_vad=True, merge_length_s=merge_s, **kw)
    pcm = _s16(wav)
    assert rec.infer_long([pcm], vad, **kw)[0] == _python_result(pipe, counting, pcm.astype(np.float32) / 32768.0, **kw)
    assert rec.infer_long([wav], vad, **kw)[0] == got                   # the second call at this size reuses every buffer
    rec.close()
    vad.close()


@pytest.mark.gpu
def test_long_audio_three_recordings_equal_three_calls_and_fixed_silence(vad_file, asr_file):
    rec, vad = OfflineRecognizer(asr_file, 0, "fp16x3"), OfflineVad(vad_file, 0)
    wavs = [synth.make_vad_wav(*LONG_CASES["longaudio_40s"][:3]).numpy(), synth.make_vad_wav(*LONG_CASES["longaudio_25s_onebatch"][:3]).numpy(),
            synth.make_vad_wav(18.0, 21).numpy()]
    for kw in ({"batch_size_s": 6}, {"batch_size_s": 6, "max_end_silence_time": 500}, {"dynamic_silence": False, "speech_noise_thres": 0.7}):
        many = rec.infer_long(wavs, vad, **kw)
        assert many == [rec.infer_long([w], vad, **kw)[0] for w in wavs]
        assert [m["vad_segments"] for m in many] == [vad.segments(w, **{k: v for k, v in kw.items() if k != "batch_size_s"}) for w in wavs]
    # silence only: no segment, no id; a recording shorter than one frame as well
    quiet = rec.infer_long([np.zeros(48000, np.float32), np.zeros(100, np.float32)], vad)
    assert quiet == [{"token_int": [], "vad_segments": [], "n_tokens": []}] * 2
    rec.close()
    vad.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_long_audio_contextual_hotwords_vs_pipeline(vad_file, tmp_path, mode):
    """ContextualParaformer: the same hotword memory biases every segment, as in the reference."""
    cfg = synth.PARAFORMER_TINY
    state = synth.make_contextual_state_dict(cfg, 6)
    path = str(tmp_path / "ctx.fab2")
    pack.write_model_file(path, state, cfg, synth.make_cmvn(cfg, 1))
    hw = synth.make_hotwords(8, cfg.vocab, seed=11)
    pipe, counting, asr = _pipeline(mode, state, contextual=True)
    emb = asr.encode_hotwords(hw).float().cpu().numpy()
    wav = synth.make_vad_wav(*LONG_CASES["longaudio_40s"][:3]).numpy()
    rec, vad = OfflineRecognizer(path, 0, mode), OfflineVad(vad_file, 0)
    got = rec.infer_long([wav], vad, batch_size_s=6, hotword_embeddings=emb)[0]
    assert got == _python_result(pipe, counting, wav, batch_size_s=6, hotword_ids=hw)
    assert got["token_int"]
    with pytest.raises(_abi.FunasrB200Error):
        rec.infer_long([wav], vad, batch_size_s=6)                      # a contextual model needs the hotword memory
    rec.close()
    vad.close()


@pytest.mark.gpu
def test_gather_segments_bit_exact():
    """fa_gather_segments against torch slicing + zero padding: ragged rows, a segment clipped at the end of the recording, pad columns
    zero even over a dirty buffer."""
    lib = _abi.load()
    g = torch.Generator().manual_seed(5)
    n = 100003
    rec = torch.randn(n, generator=g).to(DEV)
    starts = [0, 17, 99000, 50001, 3, 100000]
    lens = [400, 12345, 1003, 0, 7, 3]                                   # the last one ends exactly at n; one empty row
    stride = (max(lens) + 3) // 4 * 4
    out = torch.full((len(starts), stride), float("nan"), device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    s_d = torch.tensor(starts, dtype=torch.int64, device=DEV)
    l_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    assert lib.fa_gather_segments(rec.data_ptr(), n, s_d.data_ptr(), l_d.data_ptr(), len(starts), stride, out.data_ptr(), st) == 0
    want = torch.zeros_like(out)
    for r, (s, ln) in enumerate(zip(starts, lens)):
        want[r, :ln] = rec[s: s + ln]
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    # a row reaching past the recording reads zeros there
    l_d2 = torch.tensor([10], dtype=torch.int32, device=DEV)
    s_d2 = torch.tensor([n - 4], dtype=torch.int64, device=DEV)
    out2 = torch.full((1, 12), 7.0, device=DEV)
    assert lib.fa_gather_segments(rec.data_ptr(), n, s_d2.data_ptr(), l_d2.data_ptr(), 1, 12, out2.data_ptr(), st) == 0
    torch.cuda.synchronize()
    assert torch.equal(out2[0, :4], rec[n - 4:]) and not out2[0, 4:].any()
    assert lib.fa_gather_segments(rec.data_ptr(), n, s_d.data_ptr(), l_d.data_ptr(), 1, 6, out.data_ptr(), st) == -4   # stride % 4


@pytest.mark.gpu
def test_vad_handle_refuses_malformed_files(tmp_path, vad_file):
    lib = _abi.load()
    blob = open(vad_file, "rb").read()
    (tmp_path / "trunc.fab2").write_bytes(blob[: len(blob) // 2])
    (tmp_path / "magic.fab2").write_bytes(b"XXXXXXXX" + blob[8:])
    assert not lib.fa_vad_init(str(tmp_path / "missing.fab2").encode(), 0) and b"cannot open" in lib.fa_offline_last_error()
    for p in ("trunc.fab2", "magic.fab2"):
        assert not lib.fa_vad_init(str(tmp_path / p).encode(), 0) and b"malformed" in lib.fa_offline_last_error()


def _vocab_dir(tmp_path, vad_file, asr_file, vocab):
    """A model directory with one CJK character per token, so that the concatenated segment texts map back to ids."""
    d = tmp_path / "asr"
    d.mkdir()
    os.symlink(asr_file, str(d / "model.fab2"))
    (d / "tokens.txt").write_text("\n".join(chr(0x4E00 + i) for i in range(vocab)) + "\n", encoding="utf-8")
    vd = tmp_path / "vad"
    vd.mkdir()
    os.symlink(vad_file, str(vd / "vad.fab2"))
    return str(d), str(vd)


@pytest.mark.gpu
def test_runtime_vad_client(tmp_path, vad_file, asr_file):
    """examples/offline_vad_client.cpp: FsmnVadInfer / FsmnVadInferBuffer give the golden segments on vad_fixed800 (float32 WAV) and the
    detector's fixed-silence segments over the handle's own posteriors elsewhere; FunOfflineInfer with "vad-dir" gives text that maps back
    to fa_offline_infer_vad's ids under the fixed end silence, for float32 and s16 WAV."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    inc, libdir = os.path.join(ROOT, "include"), os.path.join(ROOT, "funasr_b200")
    exe = str(tmp_path / "vad_client")
    r = subprocess.run(["g++", "-std=c++17", '-DFUNASR_RUNTIME_HEADER="funasrruntime_b200.h"', "-I" + inc,
                        os.path.join(ROOT, "examples", "offline_vad_client.cpp"), "-L" + libdir, "-lfunasr_b200", "-Wl,-rpath," + libdir, "-o", exe],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    cfg = synth.PARAFORMER_TINY
    asr_dir, vad_dir = _vocab_dir(tmp_path, vad_file, asr_file, cfg.vocab)

    def run(wav_path, *extra):
        p = subprocess.run([exe, vad_dir, wav_path, *extra], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert p.returncode == 0, p.stdout[-2000:]
        return dict(ln.split(" ", 1) if " " in ln else (ln, "") for ln in p.stdout.splitlines())

    def segs(line):
        return [[int(a), int(b)] for a, b in (t.strip("[]").split(",") for t in line.split())]

    # the golden fixed-silence case
    seconds, seed, pattern, kw = VAD_CASES["vad_fixed800"]
    w = synth.make_vad_wav(seconds, seed, pattern).numpy()
    path = str(tmp_path / "fixed800.wav")
    open(path, "wb").write(_wav_bytes(w, "f32"))
    out = run(path)
    want = _gold("vad_fixed800")["segments"].tolist()
    assert segs(out["file_segments"]) == want and segs(out["buffer_segments"]) == want
    vad = OfflineVad(vad_file, 0)
    rec = OfflineRecognizer(asr_file, 0, "fp16x3")
    for name in ("vad_30s", "vad_random45"):
        seconds, seed, pattern, _ = VAD_CASES[name]
        w = synth.make_vad_wav(seconds, seed, pattern).numpy()
        path = str(tmp_path / (name + ".wav"))
        open(path, "wb").write(_wav_bytes(w, "f32"))
        out = run(path)
        _, frames = vad.segments(w, want_frames=True)
        assert segs(out["file_segments"]) == V.detect_segments(frames[0].tolist(), frames[1].tolist(), w.size, max_end_silence_time=800)
    # recognition through "vad-dir"
    w = synth.make_vad_wav(*LONG_CASES["longaudio_40s"][:3]).numpy()
    for fmt, arr in (("f32", w), ("s16", _s16(w))):
        path = str(tmp_path / ("long_%s.wav" % fmt))
        open(path, "wb").write(_wav_bytes(arr, fmt))
        out = run(path, asr_dir, "fp16x3")
        ids = [ord(ch) - 0x4E00 for ch in out["asr_result"]]
        want = rec.infer_long([arr], vad, dynamic_silence=False)[0]
        assert ids == want["token_int"] and ids
        assert abs(float(out["asr_seconds"]) - w.size / 16000.0) < 1e-3
    rec.close()
    vad.close()
