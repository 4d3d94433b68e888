"""GPU: CT-Transformer punctuation through the C handle API -- fa_punc_infer against the reference's goldens, many texts in one lockstep
call against one call per text and against CTTransformerB200.inference, the refusal of a window too long for the attention kernel,
and the C++ runtime surface: FunOfflineInit with "punc-dir" (with a BiCif model and "vad-dir") and CTTransformerInfer."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

import funasr_b200
from funasr_b200 import _abi, pack, synth
from funasr_b200.offline import OfflinePunc
from test_offline_punc_host import ENC_CONF, CharTokenizer
from test_offline_stamps_gpu import BICIF_SEED, _bicif_file, _long_wav
from test_offline_vad_gpu import _wav_bytes
import stampsent_ref

DEV = "cuda:0"
CASES = ["punc_short", "punc_long", "punc_english_tail"]


@pytest.fixture(scope="module")
def punc_file(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("punc") / "punc.fab2")
    pack.write_punc_model_file(path, synth.make_punc_state_dict(0), synth.PUNC_LIST, synth.punc_token_list(), 3, ENC_CONF)
    return path


@pytest.mark.gpu
def test_punc_handle_reproduces_the_reference_goldens(punc_file):
    p = OfflinePunc(punc_file, 0)
    gs = [np.load(os.path.join(GOLDEN, n + ".npz")) for n in CASES]
    for g in gs:                                                       # alone
        (r,) = p.infer([str(g["text_in"])])
        assert r["text"] == str(g["text_out"]) and r["punc_array"] == g["punc_array"].tolist()
    got = p.infer([str(g["text_in"]) for g in gs])                     # together, in lockstep
    assert [(r["text"], r["punc_array"]) for r in got] == [(str(g["text_out"]), g["punc_array"].tolist()) for g in gs]
    assert p.infer(["", "  \t"]) == [{"text": "", "punc_array": []}] * 2 and p.last_steps == 0
    p.close()


@pytest.mark.gpu
def test_batched_equals_one_by_one_and_the_engine(punc_file):
    """48 seeded texts of 1 to 1 200 words in one call: texts and punctuation arrays identical to one call per text and to
    CTTransformerB200.inference (the Python engine over the same kernels) per text."""
    rng = np.random.default_rng(5)
    n_words = [1, 2, 19, 20, 21, 1200] + [int(v) for v in rng.integers(1, 1201, 42)]
    texts = [synth.make_punc_text(n, 100 + i) for i, n in enumerate(n_words)]
    p = OfflinePunc(punc_file, 0)
    lib = _abi.load()
    c0 = lib.fa_launch_count()
    batched = p.infer(texts)
    launches = lib.fa_launch_count() - c0
    steps = p.last_steps
    alone = [p.infer([t])[0] for t in texts]
    assert batched == alone
    assert steps >= 60 and launches > 0
    m = funasr_b200.CTTransformerB200(encoder="SANMEncoder", encoder_conf=dict(ENC_CONF), vocab_size=len(synth.punc_token_list()),
                                      punc_list=synth.PUNC_LIST, punc_weight=[1.0] * len(synth.PUNC_LIST), embed_unit=synth.PUNC_DIM,
                                      att_unit=synth.PUNC_DIM, sentence_end_id=3)
    m.load_state_dict(synth.make_punc_state_dict(0), strict=True)
    m.to(DEV).eval()
    tok = CharTokenizer(synth.punc_token_list())
    for t, b in zip(texts, batched):
        r = m.inference([t], key=["k"], tokenizer=tok, device=DEV)[0][0]
        assert b == {"text": r["text"], "punc_array": r["punc_array"].tolist()}, t
    assert p.infer(texts) == batched                                   # grow-only buffers reused
    p.close()


@pytest.mark.gpu
def test_window_too_long_for_the_attention_kernel_fails_naming_the_text(tmp_path):
    """A model that never predicts a comma or a sentence end carries every window into the next; with 2 000-word windows the sixth
    step would hold 12 000 words, past the 10 240 keys of the fp32 attention kernel: the call fails before that step, naming the text,
    and the handle keeps working."""
    st = synth.make_punc_state_dict(0)
    st["decoder.bias"] = st["decoder.bias"].clone()
    st["decoder.bias"][:] = -100.0
    st["decoder.bias"][1] = 100.0                                      # always "_"
    t = pack.punc_model_tensors(st, synth.PUNC_LIST, synth.punc_token_list(), 3, ENC_CONF)
    t["__punc_config__"] = t["__punc_config__"].copy()
    t["__punc_config__"][5] = 2000
    path = str(tmp_path / "blank.fab2")
    pack._write(path, t)
    p = OfflinePunc(path, 0)
    short = synth.make_punc_text(30, 1)
    with pytest.raises(_abi.FunasrB200Error, match="text 1: window 5 holds 12000 words"):
        p.infer([short, "你" * 13000])
    (r,) = p.infer([short])
    assert r["punc_array"] == [1] * (len(r["punc_array"]) - 1) + [3] and r["text"][-1] in "。."
    p.close()


RUNTIME_CLIENT = r'''
#include <stdio.h>
#include "funasrruntime_b200.h"
int main(int argc, char** argv) {
  std::map<std::string, std::string> mp;
  mp["model-dir"] = argv[1];
  mp["vad-dir"] = argv[3];
  if (argc > 4) mp["punc-dir"] = argv[4];
  FUNASR_HANDLE h = FunOfflineInit(mp, 1);
  if (!h) { printf("init failed %s\n", FunB200LastError()); return 1; }
  std::vector<std::vector<float>> hw;
  FUNASR_RESULT r = FunOfflineInfer(h, argv[2], RASR_NONE, nullptr, hw, 16000);
  if (!r) { printf("infer failed %s\n", FunB200LastError()); return 1; }
  printf("text %s\nstamp %s\nsents [%s]\n", FunASRGetResult(r, 0), FunASRGetStamp(r), FunASRGetStampSents(r));
  FunASRFreeResult(r);
  FunOfflineUninit(h);
  std::map<std::string, std::string> pp;
  pp["model-dir"] = argv[4 < argc ? 4 : 1];
  printf("online %s\n", CTTransformerInit(pp, 1, PUNC_ONLINE) ? "accepted" : FunB200LastError());
  return 0;
}
'''


@pytest.mark.gpu
def test_runtime_punc_dir_with_bicif_and_vad(tmp_path, punc_file):
    """FunOfflineInit with model-dir (tiny BiCif) + vad-dir + punc-dir on a 40 s recording: the text is fa_punc_infer of the same
    call's text without punc-dir, the stamps are unchanged, FunASRGetStampSents is TimestampSentence (tests/stampsent_ref.py) of those two
    strings; PUNC_ONLINE is refused with a message."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    cfg = synth.PARAFORMER_TINY
    d, vd, pd = tmp_path / "asr", tmp_path / "vad", tmp_path / "punc"
    for x in (d, vd, pd):
        x.mkdir()
    _bicif_file(str(d / "model.fab2"), cfg, BICIF_SEED, synth.make_cmvn(cfg, 1))
    cjk = synth.punc_token_list()[3:synth.PUNC_VOCAB - 17]
    (d / "tokens.txt").write_text("\n".join(["<blank>", "<s>", "</s>"] + [cjk[i % len(cjk)] for i in range(3, cfg.vocab)]) + "\n",
                                  encoding="utf-8")
    pack.write_vad_model_file(str(vd / "vad.fab2"), synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    os.symlink(punc_file, str(pd / "punc.fab2"))
    wav = str(tmp_path / "long.wav")
    open(wav, "wb").write(_wav_bytes(_long_wav(), "f32"))
    inc, libdir = os.path.join(ROOT, "include"), os.path.join(ROOT, "funasr_b200")
    src, exe = tmp_path / "client.cpp", str(tmp_path / "client")
    src.write_text(RUNTIME_CLIENT)
    r = subprocess.run(["g++", "-std=c++17", "-I" + inc, str(src), "-L" + libdir, "-lfunasr_b200", "-Wl,-rpath," + libdir, "-o", exe],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]

    def run(*extra):
        p = subprocess.run([exe, str(d), wav, str(vd), *extra], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        out = p.stdout.decode("utf-8")
        assert p.returncode == 0, out[-2000:]
        return dict(ln.split(" ", 1) if " " in ln else (ln, "") for ln in out.splitlines())

    plain, punc = run(), run(str(pd))
    assert len(plain["text"]) > 20 and plain["stamp"].startswith("[[")
    p = OfflinePunc(punc_file, 0)
    want = p.infer([plain["text"]])[0]["text"]
    assert punc["text"] == want and want != plain["text"]
    assert punc["stamp"] == plain["stamp"]
    assert plain["sents"] == "[]"                                       # without punc-dir it stays empty
    sents = punc["sents"][1:-1]
    assert sents == stampsent_ref.timestamp_sentence(punc["text"], punc["stamp"]) and sents.count('"punc":') > 3
    assert "PUNC_OFFLINE" in punc["online"]
    p.close()


@pytest.mark.gpu
def test_cttransformer_entry_points_give_the_goldens(tmp_path, punc_file):
    """examples/offline_punc_client.cpp (the runtime's offline punctuation client): CTTransformerInfer line by line gives the goldens'
    texts."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    pd = tmp_path / "punc"
    pd.mkdir()
    os.symlink(punc_file, str(pd / "punc.fab2"))
    gs = [np.load(os.path.join(GOLDEN, n + ".npz")) for n in CASES]
    (tmp_path / "in.txt").write_text("\n".join(str(g["text_in"]) for g in gs) + "\n", encoding="utf-8")
    inc, libdir = os.path.join(ROOT, "include"), os.path.join(ROOT, "funasr_b200")
    exe = str(tmp_path / "punc_client")
    r = subprocess.run(["g++", "-std=c++17", "-I" + inc, os.path.join(ROOT, "examples", "offline_punc_client.cpp"), "-L" + libdir,
                        "-lfunasr_b200", "-Wl,-rpath," + libdir, "-o", exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    p = subprocess.run([exe, str(pd), str(tmp_path / "in.txt")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    out = p.stdout.decode("utf-8")
    assert p.returncode == 0, out[-2000:]
    got = [ln[len("punc_result "):] for ln in out.splitlines() if ln.startswith("punc_result ")]
    assert got == [str(g["text_out"]) for g in gs]
