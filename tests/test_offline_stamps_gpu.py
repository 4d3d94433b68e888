"""GPU: per-token timestamps through the C handle API for a BiCifParaformer model file — fa_offline_infer against the reference's
golden ids and stamps, fa_offline_infer_vad against the reference's AutoModel(model="BiCifParaformer", vad_model=...) and against
LongAudioPipeline, plain Paraformer files unchanged, and FunASRGetStamp of the C++ runtime surface."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, gold_stamps, load_bicif_case, load_case, state_dict_for

import funasr_b200
from funasr_b200 import pack, synth
from funasr_b200.offline import OfflineRecognizer, OfflineVad
from test_abi_host import _tiny_conf
from test_offline_vad_gpu import LONG_CASES, _vad_plugin, _wav_bytes

DEV = "cuda:0"
BICIF_SEED = 8                     # the weights of bicif_tiny_ragged3 and of longaudio_bicif_40s (oracle/make_bicif_long_golden.py)
LONG = "longaudio_bicif_40s"


def _bicif_file(path, cfg, wseed, cmvn):
    pack.write_model_file(path, synth.make_bicif_state_dict(cfg, wseed), cfg, cmvn)
    return path


@pytest.fixture(scope="module")
def bicif_file(tmp_path_factory):
    cfg = synth.PARAFORMER_TINY
    return _bicif_file(str(tmp_path_factory.mktemp("bicif") / "model.fab2"), cfg, BICIF_SEED, synth.make_cmvn(cfg, 1))


@pytest.fixture(scope="module")
def vad_file(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("vad") / "vad.fab2")
    pack.write_vad_model_file(path, synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    return path


def _long_wav():
    return synth.make_vad_wav(*LONG_CASES["longaudio_40s"][:3]).numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("name", ["bicif_tiny_ragged3", "bicif_large_single"])
def test_handle_stamps_vs_reference_golden(tmp_path, name, mode):
    """fa_offline_infer on a BiCif file: the reference's greedy ids (CifPredictorV3's sequential fp32 `cif` on the token branch) and
    its per-token stamps (bicif_paraformer/model.py:402-407), integer ms exact, for the same batch the golden ran."""
    cfg, wseed, wavs, cmvn, g = load_bicif_case(name)
    rec = OfflineRecognizer(_bicif_file(str(tmp_path / "m.fab2"), cfg, wseed, cmvn), 0, mode)
    assert rec.has_timestamps
    got = rec.infer_stamped([w.numpy() for w in wavs])
    assert [t for r in got for t in r["token_int"]] == g["ids_flat"].tolist()
    assert [r["timestamp"] for r in got] == gold_stamps(g)
    assert [len(r["timestamp"]) for r in got] == [len(r["token_int"]) for r in got]
    assert rec.infer([w.numpy() for w in wavs]) == [r["token_int"] for r in got]
    rec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_long_audio_stamps_vs_reference_golden_and_pipeline(bicif_file, vad_file, mode):
    """fa_offline_infer_vad on the 40 s recording in 6 s packs: ids and absolute stamps equal the unmodified reference's, and equal
    LongAudioPipeline over BiCifParaformerB200 in the same mode; a recording without speech gives no stamp."""
    g = dict(np.load(os.path.join(GOLDEN, LONG + ".npz")))
    wav = _long_wav()
    assert wav.size == int(g["n_samples"])
    rec, vad = OfflineRecognizer(bicif_file, 0, mode), OfflineVad(vad_file, 0)
    got = rec.infer_long([wav], vad, batch_size_s=6)[0]
    assert got["token_int"] == g["ids"].tolist()
    assert got["timestamp"] == g["timestamp"].tolist()
    assert len(got["vad_segments"]) >= 2 and sum(got["n_tokens"]) == len(got["token_int"])
    cfg = synth.PARAFORMER_TINY
    conf = _tiny_conf()
    conf["gemm_mode"] = mode
    conf["predictor"] = "CifPredictorV3B200"
    conf["predictor_conf"] = dict(idim=512, threshold=1.0, l_order=1, r_order=1, tail_threshold=cfg.tail_threshold, smooth_factor2=0.25,
                                  noise_threshold2=0.01, upsample_times=3, use_cif1_cnn=False, upsample_type="cnn_blstm")
    asr = funasr_b200.BiCifParaformerB200(**conf)
    asr.load_state_dict(synth.make_bicif_state_dict(cfg, BICIF_SEED), strict=True)
    asr.to(DEV).eval()
    asr_fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0,
                                         cmvn=synth.make_cmvn(cfg, 1))
    v, v_fe = _vad_plugin()
    pipe = funasr_b200.LongAudioPipeline(asr, asr_fe, v, v_fe, device=DEV, tokenizer=None)
    want = pipe.generate(wav, key="rec", batch_size_s=6)
    assert got["token_int"] == want["token_int"] and got["timestamp"] == want["timestamp"]
    assert got["vad_segments"] == want["vad_segments"]
    quiet = rec.infer_long([np.zeros(48000, np.float32)], vad)[0]
    assert quiet == {"token_int": [], "vad_segments": [], "n_tokens": [], "timestamp": []}
    assert rec.infer_long([wav], vad, batch_size_s=6)[0] == got            # buffers reused
    rec.close()
    vad.close()


@pytest.mark.gpu
def test_plain_paraformer_file_gives_the_same_ids_and_no_stamps(tmp_path, vad_file):
    cfg, wseed, wavs, cmvn, g = load_case("tiny_ragged3")
    path = str(tmp_path / "plain.fab2")
    pack.write_model_file(path, state_dict_for(cfg, wseed), cfg, cmvn)
    rec = OfflineRecognizer(path, 0, "fp16x3")
    assert not rec.has_timestamps
    got = rec.infer_stamped([w.numpy() for w in wavs])
    assert [t for r in got for t in r["token_int"]] == g["ids_flat"].tolist()
    assert all(r["timestamp"] == [] for r in got)
    vad = OfflineVad(vad_file, 0)
    assert "timestamp" not in rec.infer_long([_long_wav()], vad, batch_size_s=6)[0]
    rec.close()
    vad.close()


CLIENT = r'''
#include <stdio.h>
#include "funasrruntime_b200.h"
int main(int argc, char** argv) {
  std::map<std::string, std::string> mp;
  mp["model-dir"] = argv[1];
  mp["gemm-mode"] = "fp16x3";
  if (argc > 3) mp["vad-dir"] = argv[3];
  FUNASR_HANDLE h = FunOfflineInit(mp, 1);
  if (!h) { printf("init failed\n"); return 1; }
  std::vector<std::vector<float>> hw;
  FUNASR_RESULT r = FunOfflineInfer(h, argv[2], RASR_NONE, nullptr, hw, 16000);
  if (!r) { printf("infer failed\n"); return 1; }
  printf("stamp %s\nsents [%s]\n", FunASRGetStamp(r), FunASRGetStampSents(r));
  FunASRFreeResult(r);
  FunOfflineUninit(h);
  return 0;
}
'''


def _render(stamps):
    return "[" + ",".join("[%d,%d]" % (a, b) for a, b in stamps) + "]" if stamps else ""


@pytest.mark.gpu
def test_runtime_get_stamp(tmp_path, bicif_file, vad_file):
    """FunOfflineInit on a BiCif model-dir, with and without vad-dir: FunASRGetStamp is the runtime's "[[b,e],...]" rendering of the
    handle's stamps (the runtime's fixed end silence with vad-dir); FunASRGetStampSents stays empty."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    inc, libdir = os.path.join(ROOT, "include"), os.path.join(ROOT, "funasr_b200")
    src, exe = tmp_path / "stamp_client.cpp", str(tmp_path / "stamp_client")
    src.write_text(CLIENT)
    r = subprocess.run(["g++", "-std=c++17", "-I" + inc, str(src), "-L" + libdir, "-lfunasr_b200", "-Wl,-rpath," + libdir, "-o", exe],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    d, vd = tmp_path / "asr", tmp_path / "vad"
    d.mkdir()
    vd.mkdir()
    os.symlink(bicif_file, str(d / "model.fab2"))
    os.symlink(vad_file, str(vd / "vad.fab2"))
    rec, vad = OfflineRecognizer(bicif_file, 0, "fp16x3"), OfflineVad(vad_file, 0)

    def run(wav_path, *extra):
        p = subprocess.run([exe, str(d), wav_path, *extra], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert p.returncode == 0, p.stdout[-2000:]
        return dict(ln.split(" ", 1) if " " in ln else (ln, "") for ln in p.stdout.splitlines())

    _, _, wavs, _, _ = load_bicif_case("bicif_tiny_ragged3")
    short = wavs[0].numpy()
    path = str(tmp_path / "short.wav")
    open(path, "wb").write(_wav_bytes(short, "f32"))
    out = run(path)
    want = rec.infer_stamped([short])[0]["timestamp"]
    assert want and out["stamp"] == _render(want) and out["sents"] == "[]"
    long = _long_wav()
    path = str(tmp_path / "long.wav")
    open(path, "wb").write(_wav_bytes(long, "f32"))
    out = run(path, str(vd))
    want = rec.infer_long([long], vad, dynamic_silence=False)[0]["timestamp"]
    assert want and out["stamp"] == _render(want)
    rec.close()
    vad.close()
