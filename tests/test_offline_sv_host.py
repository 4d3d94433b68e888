"""CPU: SenseVoiceSmall in the C library without a GPU -- the SenseVoice model file, fa_offline_init's refusals, the runtime's CTCSearch
text (fa_sv_ctc_text_host) against a Python restatement of sensevoice-small.cpp:305-355, the query mapping and the example client's
runtime symbols."""
import ctypes as C
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

from funasr_b200 import _abi, pack, synth
from funasr_b200.modules import SenseVoiceSmallB200
from funasr_b200.offline import sv_query_ids

CFG = synth.SENSEVOICE_TINY


@pytest.fixture(scope="module")
def sv_state():
    return synth.make_sensevoice_state_dict(CFG, 4)


def test_sensevoice_model_file_round_trip(tmp_path, sv_state):
    cmvn = synth.make_cmvn(synth.PARAFORMER_LARGE, seed=1)
    path = str(tmp_path / "sv.fab2")
    pack.write_sensevoice_model_file(path, sv_state, CFG, cmvn)
    back = pack.read_model_file(path)
    c = back["__sv_config__"]
    assert c.tolist()[:7] == [CFG.enc_layers, CFG.tp_layers, CFG.d_model, CFG.heads, CFG.kernel, CFG.vocab, CFG.feat_dim]
    assert c[7] == np.float32(1e-5) and c[8] == 0                         # SenseVoice's LayerNorm eps travels in the file
    assert "__config__" not in back
    for k, v in sv_state.items():
        assert np.array_equal(back[k], v.numpy()) and back[k].shape == tuple(v.shape), k
    assert np.array_equal(back["frontend.cmvn"], cmvn.numpy())
    assert np.array_equal(back["encoder.pe_inv_timescales"], synth.sinusoid_inv_timescales(CFG.feat_dim).numpy())
    para = pack.model_tensors(synth.make_state_dict(synth.PARAFORMER_TINY, 3), synth.PARAFORMER_TINY, cmvn)
    for k in ("frontend.mel_banks", "frontend.window", "encoder.pe_inv_timescales"):   # the same derived tables as the Paraformer file
        assert np.array_equal(back[k], para[k]), k
    with pytest.raises(ValueError, match="not a SenseVoiceSmall"):
        pack.write_sensevoice_model_file(path, {k: v for k, v in sv_state.items() if k != "embed.weight"}, CFG)


def _refused(tmp_path, sv_state, edit) -> str:
    t = pack.sensevoice_model_tensors(sv_state, CFG, None)
    edit(t)
    path = str(tmp_path / "bad.fab2")
    pack._write(path, t)
    lib = _abi.load()
    assert not lib.fa_offline_init(path.encode(), 0, _abi.GEMM_MODES["fp16x3"])
    return lib.fa_offline_last_error().decode()


def _set_cfg(i, v):
    def f(t):
        t["__sv_config__"] = t["__sv_config__"].copy()
        t["__sv_config__"][i] = v
    return f


def test_sensevoice_init_refusals_name_the_piece_without_a_device(tmp_path, sv_state):
    """Decided on the file's index alone, so the message names the piece (not the missing device) on any machine."""
    para = pack.model_tensors(synth.make_state_dict(synth.PARAFORMER_TINY, 3), synth.PARAFORMER_TINY, None)
    assert "both __config__" in _refused(tmp_path, sv_state, lambda t: t.__setitem__("__config__", para["__config__"]))
    assert "missing tensor encoder.tp_encoders.1.feed_forward.w_2.bias" in _refused(
        tmp_path, sv_state, lambda t: t.pop("encoder.tp_encoders.1.feed_forward.w_2.bias"))
    assert "missing tensor embed.weight" in _refused(tmp_path, sv_state, lambda t: t.pop("embed.weight"))
    assert "missing tensor encoder.tp_norm.weight" in _refused(tmp_path, sv_state, lambda t: t.pop("encoder.tp_norm.weight"))
    assert "missing tensor encoder.encoders.1.norm1.weight" in _refused(tmp_path, sv_state, lambda t: t.pop("encoder.encoders.1.norm1.weight"))
    assert "d_model 768" in _refused(tmp_path, sv_state, _set_cfg(2, 768))
    assert "8 heads" in _refused(tmp_path, sv_state, _set_cfg(3, 8))
    assert "vocabulary of 70000" in _refused(tmp_path, sv_state, _set_cfg(5, 70000))
    assert "bad shape of ctc.ctc_lo.weight" in _refused(tmp_path, sv_state, _set_cfg(5, 1300))
    assert "bad shape of embed.weight" in _refused(tmp_path, sv_state, lambda t: t.__setitem__("embed.weight", t["embed.weight"][:2]))
    assert "bad __sv_config__" in _refused(tmp_path, sv_state, lambda t: t.__setitem__("__sv_config__", t["__sv_config__"][:8]))
    w1 = "encoder.tp_encoders.1.feed_forward.w_1.weight"
    assert "bad shape of " + w1 in _refused(tmp_path, sv_state, lambda t: t.__setitem__(w1, t[w1][:, :256]))
    path = str(tmp_path / "sv.fab2")                                         # a well-formed file fails only for want of a device
    pack.write_sensevoice_model_file(path, sv_state, CFG)
    lib = _abi.load()
    h = lib.fa_offline_init(path.encode(), 0, _abi.GEMM_MODES["fp16x3"])
    assert h or lib.fa_offline_last_error() == b"no such CUDA device (this library has no CPU path)"
    lib.fa_offline_uninit(h)


# ------------------------------------------------------------------------------------------------------------ CTCSearch text
def ctc_search_text(ids, vocab):
    """SenseVoiceSmall::CTCSearch (runtime/onnxruntime/src/sensevoice-small.cpp:305-355) after its arg-max and collapse, restated in
    Python over the ids, with the one difference the library documents: with exactly 3 tokens the fourth tag is empty (the runtime
    reads tokens[3] one past the end there).  An id outside the vocabulary reads as its decimal number."""
    piece = lambda i: vocab[i] if 0 <= i < len(vocab) else str(i)       # noqa: E731
    lang = emo = event = itn = ""
    if len(ids) >= 3:
        lang, emo, event = piece(ids[0]), piece(ids[1]), piece(ids[2])
        if len(ids) > 3:
            itn = piece(ids[3])
    text = ""
    for i in ids[4:]:
        w = piece(i).encode("utf-8")
        text += " " + w[3:].decode("utf-8", "surrogateescape") if "▁".encode() in w else w.decode("utf-8", "surrogateescape")
    if itn == "<|withitn|>":
        text += "。" if lang == "<|zh|>" else "."
    return lang + emo + event + " " + text


def sv_ctc_text_host(ids, vocab) -> str:
    lib = _abi.load()
    arr = np.ascontiguousarray(ids, dtype=np.int32)
    enc = [v.encode("utf-8") for v in vocab]
    toks = (C.c_char_p * max(len(enc), 1))(*enc)
    n = lib.fa_sv_ctc_text_host(arr.ctypes.data, len(arr), toks, len(enc), None, 0)
    assert n >= 0
    buf = C.create_string_buffer(n + 1)
    assert lib.fa_sv_ctc_text_host(arr.ctypes.data, len(arr), toks, len(enc), buf, n + 1) == n
    return buf.raw[:n].decode("utf-8", "surrogateescape")


VOCAB = ["<blank>", "<|zh|>", "<|en|>", "<|yue|>", "<|NEUTRAL|>", "<|HAPPY|>", "<|Speech|>", "<|BGM|>", "<|withitn|>", "<|woitn|>",
         "▁hello", "▁world", "lo", "ing", "你", "好", "▁世界", "a▁b", "été", "▁", "x▁"]


def test_ctc_search_text_equals_the_runtime_restatement():
    rng = random.Random(5)
    seen = set()
    for _ in range(3000):
        n = rng.randint(0, 6)
        ids = [rng.choice([rng.randrange(len(VOCAB)), rng.randrange(len(VOCAB) + 5)]) for _ in range(n)]
        if n >= 4 and rng.random() < 0.5:
            ids[0], ids[3] = rng.choice([1, 2, 3]), 8                   # <|withitn|> after <|zh|> and after another language
        want = ctc_search_text(ids, VOCAB)
        assert sv_ctc_text_host(ids, VOCAB) == want, ids
        seen.add((n, n >= 4 and ids[3] == 8 and ids[0] == 1, n >= 4 and ids[3] == 8 and ids[0] != 1))
    assert {n for n, _, _ in seen} == set(range(7)) and any(z for _, z, _ in seen) and any(o for _, _, o in seen)
    assert sv_ctc_text_host([1, 4, 6, 8, 14, 15, 10], VOCAB) == "<|zh|><|NEUTRAL|><|Speech|> 你好 hello。"
    assert sv_ctc_text_host([2, 4, 6, 8, 10, 11], VOCAB) == "<|en|><|NEUTRAL|><|Speech|>  hello world."
    assert sv_ctc_text_host([2, 4, 6], VOCAB) == "<|en|><|NEUTRAL|><|Speech|> "            # exactly 3 tokens: the fourth tag is empty
    assert sv_ctc_text_host([2, 4], VOCAB) == " "
    assert sv_ctc_text_host([7, 8, 9, 10, 99], []) == "789 99"                             # no token list: decimal ids
    lib = _abi.load()
    assert lib.fa_sv_ctc_text_host(None, 2, None, 0, None, 0) == -1


# ------------------------------------------------------------------------------------------------------------ queries
RUNTIME_LID_MAP = {"auto": 0, "zh": 3, "en": 4, "yue": 7, "ja": 11, "ko": 12, "nospeech": 13}   # sensevoice-small.h:110-118


def test_query_mapping():
    assert SenseVoiceSmallB200.lid_dict == RUNTIME_LID_MAP
    assert SenseVoiceSmallB200.textnorm_dict == {"withitn": 14, "woitn": 15}
    lid, tn = sv_query_ids(3)
    assert lid.tolist() == [0, 0, 0] and tn.tolist() == [15, 15, 15]                     # SenseVoiceSmall.inference's defaults
    lid, tn = sv_query_ids(3, ["zh", "klingon", "yue"], [True, False, True])
    assert lid.tolist() == [3, 0, 7] and tn.tolist() == [14, 15, 14]                    # an unknown language is "auto"
    lid, tn = sv_query_ids(2, "en", True)
    assert lid.tolist() == [4, 4] and tn.tolist() == [14, 14] and lid.dtype == np.int32
    with pytest.raises(_abi.FunasrB200Error):
        sv_query_ids(2, ["zh"])
    src = open(os.path.join(ROOT, "funasr_b200", "csrc", "runtime_shim.cpp")).read()   # the shim's table is the runtime's
    for k, v in RUNTIME_LID_MAP.items():
        assert '{"%s", %d}' % (k, v) in src
    assert "svs_itn ? 14 : 15" in src


def test_sv_client_links_against_the_reference_header(tmp_path):
    """examples/offline_sv_client.cpp (bin/funasr-onnx-offline.cpp's calls with svs_lang / svs_itn) compiled against
    include/funasrruntime_b200.h needs exactly the runtime symbols it needs against the reference's own funasrruntime.h
    (tests/golden/sv_client_symbols.txt, oracle/make_sv_client_symbols_golden.py); the library exports them all, and the client links
    and fails cleanly without a model."""
    if shutil.which("g++") is None or shutil.which("nm") is None:
        pytest.skip("no g++ / nm")
    import make_sv_client_symbols_golden as mk
    inc = os.path.join(ROOT, "include")
    with open(os.path.join(GOLDEN, "sv_client_symbols.txt")) as f:
        want = f.read().split()
    assert len(want) == 8 and any("FunOfflineInferBuffer" in s for s in want) and any("CompileHotwordEmbedding" in s for s in want)
    assert mk.client_runtime_symbols('"funasrruntime_b200.h"', inc) == want
    lib = os.path.join(ROOT, "funasr_b200", "libfunasr_b200.so")
    exported = {ln.split()[-1] for ln in subprocess.run(["nm", "-D", "--defined-only", lib], check=True, stdout=subprocess.PIPE,
                                                        text=True).stdout.splitlines() if ln.strip()}
    assert not [s for s in want if s not in exported]
    exe = str(tmp_path / "sv_client")
    r = subprocess.run(["g++", "-std=c++17", '-DFUNASR_RUNTIME_HEADER="funasrruntime_b200.h"', "-I" + inc,
                        os.path.join(ROOT, "examples", "offline_sv_client.cpp"), "-L" + os.path.join(ROOT, "funasr_b200"), "-lfunasr_b200",
                        "-Wl,-rpath," + os.path.join(ROOT, "funasr_b200"), "-o", exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    r = subprocess.run([exe, str(tmp_path), str(tmp_path / "none.wav"), "zh", "1"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 1 and "asr init failed" in r.stdout
