"""CPU: CT-Transformer punctuation in the C library without a GPU -- the punctuation model file, fa_punc_init's refusals, and the host
text walk (fa_punc_walk_host) against the reference's goldens (with the oracle network as its scorer) and against
CTTransformerB200.inference (funasr_b200/punc.py, the specification) driven by the same scripted scorers on random texts."""
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN

import punc_oracle as PO
from funasr_b200 import _abi, pack, synth
from funasr_b200.offline import punc_walk_host
from funasr_b200.punc import CTTransformerB200, split_words
from punc_scripted import random_text, scripted

CASES = ["punc_short", "punc_long", "punc_english_tail"]
ENC_CONF = dict(input_size=synth.PUNC_DIM, output_size=synth.PUNC_DIM, attention_heads=synth.PUNC_HEADS, linear_units=synth.PUNC_FFN,
                num_blocks=synth.PUNC_LAYERS, kernel_size=11, sanm_shfit=0, input_layer="pe", normalize_before=True)


class CharTokenizer:
    """CharTokenizer.encode for a list of words (abs_tokenizer.py:118-124): exact lookup, unknown -> <unk>."""

    def __init__(self, toks):
        self.t2i = {t: i for i, t in enumerate(toks)}
        self.unk = self.t2i["<unk>"]

    def encode(self, words):
        return [self.t2i.get(w, self.unk) for w in words]


def punc_model():
    return CTTransformerB200(encoder="SANMEncoder", encoder_conf=dict(ENC_CONF), vocab_size=len(synth.punc_token_list()),
                             punc_list=synth.PUNC_LIST, punc_weight=[1.0] * len(synth.PUNC_LIST), embed_unit=synth.PUNC_DIM,
                             att_unit=synth.PUNC_DIM, sentence_end_id=3)


class ScriptedEngine:
    def __init__(self, seed, probs):
        self.seed, self.probs = seed, probs

    def punc_ids(self, ids):
        return scripted(np.asarray(ids, np.int64)[None], self.seed, self.probs)[0]


def spec(texts, engine):
    """CTTransformerB200.inference, one text at a time, with `engine` as its network."""
    m = punc_model()
    m.engine = lambda device: engine
    tok = CharTokenizer(synth.punc_token_list())
    out = []
    for t in texts:
        r = m.inference([t], key=["k"], tokenizer=tok)[0][0]
        out.append((r["text"], [] if r["punc_array"] is None else [int(v) for v in r["punc_array"].tolist()]))
    return out


def walk(texts, score, **kw):
    res = punc_walk_host(texts, synth.punc_token_list(), synth.PUNC_LIST, 3, score, **kw)
    return [(r["text"], r["punc_array"]) for r in res]


# ------------------------------------------------------------------------------------------------------------------ model file
def test_punc_model_file_round_trip(tmp_path):
    st = synth.make_punc_state_dict(0)
    path = str(tmp_path / "punc.fab2")
    toks = synth.punc_token_list()
    pack.write_punc_model_file(path, st, synth.PUNC_LIST, toks, 3, ENC_CONF)
    back = pack.read_model_file(path)
    cfg = pack.read_punc_config(back)
    assert cfg == {"layers": synth.PUNC_LAYERS, "d_model": synth.PUNC_DIM, "heads": synth.PUNC_HEADS, "kernel": 11, "sentence_end_id": 3,
                   "split_size": 20, "punc_list": synth.PUNC_LIST, "token_list": toks}
    for k, v in st.items():
        assert np.array_equal(back[k], v.numpy()) and back[k].shape == tuple(v.shape), k
    assert np.array_equal(back["encoder.pe_inv_timescales"], synth.sinusoid_inv_timescales(synth.PUNC_DIM).numpy())
    assert back["__punc_tokens__"].dtype == np.float32 and back["__punc_list__"].size * 4 % 4 == 0
    with pytest.raises(ValueError):
        pack.write_punc_model_file(path, st, synth.PUNC_LIST, toks[:-1], 3, ENC_CONF)          # no <unk>
    with pytest.raises(ValueError):
        pack.write_punc_model_file(path, st, synth.PUNC_LIST, toks[:5] + ["a\nb"] + toks[5:], 3, ENC_CONF)
    with pytest.raises(ValueError):
        pack.write_punc_model_file(path, st, synth.PUNC_LIST, toks, 6, ENC_CONF)
    for bad in ({"sanm_shfit": 5}, {"input_layer": "embed"}, {"normalize_before": False}):
        with pytest.raises(ValueError, match="sanm_shfit 0"):
            pack.write_punc_model_file(path, st, synth.PUNC_LIST, toks, 3, dict(ENC_CONF, **bad))


def _refused(tmp_path, edit) -> str:
    t = pack.punc_model_tensors(synth.make_punc_state_dict(0), synth.PUNC_LIST, synth.punc_token_list(), 3, ENC_CONF)
    edit(t)
    path = str(tmp_path / "bad.fab2")
    pack._write(path, t)
    lib = _abi.load()
    assert not lib.fa_punc_init(path.encode(), 0)
    return lib.fa_offline_last_error().decode()


def _set_cfg(i, v):
    def f(t):
        t["__punc_config__"] = t["__punc_config__"].copy()
        t["__punc_config__"][i] = v
    return f


def test_punc_init_refusals_name_the_piece_without_a_device(tmp_path):
    """Decided on the file's index alone, so the message names the piece (not the missing device) on any machine."""
    assert "d_model 768" in _refused(tmp_path, _set_cfg(1, 768))
    assert "head dim" in _refused(tmp_path, _set_cfg(2, 16))                 # 256 / 16 = 16-wide heads
    assert "head dim" in _refused(tmp_path, _set_cfg(2, 3))                  # 256 / 3 is not whole
    assert "head dim" in _refused(tmp_path, _set_cfg(2, 5))
    assert "missing tensor decoder.bias" in _refused(tmp_path, lambda t: t.pop("decoder.bias"))
    assert "missing tensor encoder.encoders.2.feed_forward.w_1.weight" in _refused(tmp_path, lambda t: t.pop("encoder.encoders.2.feed_forward.w_1.weight"))
    assert "missing tensor __punc_tokens__" in _refused(tmp_path, lambda t: t.pop("__punc_tokens__"))
    assert "bad shape of decoder.weight" in _refused(tmp_path, lambda t: t.__setitem__("decoder.weight", t["decoder.weight"][:5]))
    assert "no <unk>" in _refused(tmp_path, lambda t: t.__setitem__("__punc_tokens__", pack._text_blob(synth.punc_token_list()[:-1])))
    assert "sentence_end_id" in _refused(tmp_path, _set_cfg(4, 9))
    for k in (7, 13):                                                         # the fp32 FSMN kernel is built for 11, 21 and 31 taps
        def kern(t, k=k):
            for name in list(t):
                if name.endswith("fsmn_block.weight"):
                    t[name] = np.zeros((synth.PUNC_DIM, 1, k), np.float32)
            _set_cfg(3, k)(t)
        assert "FSMN kernel %d" % k in _refused(tmp_path, kern)
    fsmn = "encoder.encoders.1.self_attn.fsmn_block.weight"                  # one layer with 21 taps in an 11-tap stack
    assert "bad shape of " + fsmn in _refused(tmp_path, lambda t: t.__setitem__(fsmn, np.zeros((synth.PUNC_DIM, 1, 21), np.float32)))
    lib = _abi.load()
    path = str(tmp_path / "punc.fab2")                                       # a well-formed file fails only for want of a device
    pack.write_punc_model_file(path, synth.make_punc_state_dict(0), synth.PUNC_LIST, synth.punc_token_list(), 3, ENC_CONF)
    h = lib.fa_punc_init(path.encode(), 0)
    assert h or lib.fa_offline_last_error() == b"no such CUDA device (this library has no CPU path)"
    lib.fa_punc_uninit(h)
    assert not lib.fa_punc_init(None, 0) and lib.fa_offline_last_error() == b"model_file is NULL"
    assert not lib.fa_punc_init(str(tmp_path / "missing.fab2").encode(), 0) and b"cannot open" in lib.fa_offline_last_error()
    assert not lib.fa_punc_infer(None, None, 0) and lib.fa_offline_last_error() == b"bad argument"
    assert lib.fa_punc_result_text(None, 0) is None and lib.fa_punc_result_steps(None) == 0
    lib.fa_punc_free_result(None)
    lib.fa_punc_uninit(None)


# ------------------------------------------------------------------------------------------------------------------ the walk
@pytest.mark.parametrize("name", CASES)
def test_walk_with_the_oracle_network_reproduces_the_reference(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    p = synth.make_punc_state_dict(0)

    def score(ids, lens):
        out = np.zeros_like(ids)
        for b in range(ids.shape[0]):
            out[b, :lens[b]] = PO.punc_ids([int(i) for i in ids[b, :lens[b]]], p, synth.PUNC_LAYERS, synth.PUNC_HEADS).numpy()
        return out

    (text, arr), = walk([str(g["text_in"])], score)
    assert text == str(g["text_out"])
    assert arr == g["punc_array"].tolist()


# scripted scorers: (seed, cumulative probabilities of <unk>, ，, 。, ？, 、)
SCORERS = [
    (1, (0.0, 0.10, 0.05, 0.02, 0.03)),          # ordinary text
    (2, (0.0, 0.08, 0.002, 0.0, 0.02)),         # sentence ends rare enough for the carry to pass 200 words, with commas
    (3, (0.0, 0.0, 0.0, 0.0, 0.0)),             # no comma and no sentence end at all: the whole text is carried
    (4, (0.01, 0.2, 0.15, 0.1, 0.1)),           # every class, <unk> included
    (5, (0.0, 0.0, 0.01, 0.0, 0.3)),            # 、 but no comma: long carries cannot be cut
]


@pytest.mark.parametrize("seed,probs", SCORERS)
def test_walk_equals_the_specification_on_random_texts(seed, probs):
    """At least 500 texts over all scorers: 0 to 2 000 words of mixed CJK / ASCII, repeated and non-ASCII whitespace, ASCII glued to
    CJK, unknown and 4-byte words; all of a scorer's texts go through one lockstep walk."""
    rng = random.Random(1000 + seed)
    lens = [0, 1, 2, 19, 20, 21, 40, 41] + [rng.choice([rng.randint(0, 60), rng.randint(0, 400), rng.randint(0, 2000)]) for _ in range(100)]
    texts = [random_text(rng, n) for n in lens] + ["", "   ", "　\t", "hello", "hello world", "你", "ok,", "Ab"]
    want = spec(texts, ScriptedEngine(seed, probs))
    got = walk(texts, lambda ids, ln: scripted(ids, seed, probs))
    for t, w, g in zip(texts, want, got):
        assert g == w, t
    if seed == 3:
        assert max(len(a) for _, a in want) > 1000                        # the carry did grow past the 200-word trigger


def test_walk_branches_and_steps():
    """The branches the scripted scorers must reach, and the lockstep itself: texts of different lengths in one call, one step per
    window of the longest."""
    rng = random.Random(7)
    texts = [random_text(rng, n) for n in (5, 45, 260, 1300)]
    probs = (0.0, 0.08, 0.002, 0.0, 0.02)
    got = walk(texts, lambda ids, ln: scripted(ids, 2, probs))
    assert got == spec(texts, ScriptedEngine(2, probs))
    calls = []

    def score(ids, lens):
        calls.append((ids.shape[0], ids.shape[1], lens.tolist()))
        return scripted(ids, 2, probs)

    walk(texts, score)
    windows = [-(-len(split_words(t)) // 20) for t in texts]
    assert len(calls) == max(windows) and windows[-1] > 60                # one step per window of the longest text
    assert [c[0] for c in calls[:3]] == [4, 3, 3] and calls[-1][0] == 1
    assert all(c[1] == max(c[2]) for c in calls)
    # English only, and final windows that end in ，, 、, "," or a Latin word
    eng = " ".join(synth.punc_token_list()[-17:-1]) * 3
    for probs2 in [(0, 0, 0, 0, 0), (0, 1.0, 0, 0, 0), (0, 0, 0, 0, 1.0), (0, 0.3, 0.1, 0, 0)]:
        ts = [eng, "你好" * 15, eng + " 你", "你 " + eng]
        assert walk(ts, lambda ids, ln: scripted(ids, 9, probs2)) == spec(ts, ScriptedEngine(9, probs2))


def test_walk_refusals():
    """A window longer than max_window fails the call and names the text; a scorer's failure or an out-of-range id fails it too."""
    texts = ["你好" * 30, "好" * 300]
    with pytest.raises(_abi.FunasrB200Error, match="text 1: window 5 holds 120 words"):
        walk(texts, lambda ids, ln: np.ones_like(ids), max_window=100)
    with pytest.raises(_abi.FunasrB200Error, match="outside the list"):
        walk(texts, lambda ids, ln: np.full_like(ids, 6))
    with pytest.raises(ZeroDivisionError):
        walk(texts, lambda ids, ln: 1 // 0)
    assert walk(["", " 　 "], lambda ids, ln: 1 // 0) == [("", []), ("", [])]      # no window: the scorer is never called
    with pytest.raises(_abi.FunasrB200Error, match="duplicated"):
        punc_walk_host(["a"], ["<unk>", "a", "a"], synth.PUNC_LIST, 3, lambda i, n: np.ones_like(i))


def test_punc_client_links_against_the_reference_header(tmp_path):
    """examples/offline_punc_client.cpp (the call sequence of bin/funasr-onnx-offline-punc.cpp plus FunOfflineInit with "punc-dir")
    compiled against include/funasrruntime_b200.h needs exactly the runtime symbols it needs against the reference's own
    funasrruntime.h (tests/golden/punc_client_symbols.txt, oracle/make_punc_client_symbols_golden.py); the library exports them all, and
    the client links and fails cleanly without a model."""
    import shutil
    import subprocess
    from conftest import ROOT
    if shutil.which("g++") is None or shutil.which("nm") is None:
        pytest.skip("no g++ / nm")
    import make_punc_client_symbols_golden as mk
    inc = os.path.join(ROOT, "include")
    with open(os.path.join(GOLDEN, "punc_client_symbols.txt")) as f:
        want = f.read().split()
    assert len(want) >= 10 and sum("CTTransformer" in s for s in want) == 5
    assert mk.client_runtime_symbols('"funasrruntime_b200.h"', inc) == want
    lib = os.path.join(ROOT, "funasr_b200", "libfunasr_b200.so")
    exported = {ln.split()[-1] for ln in subprocess.run(["nm", "-D", "--defined-only", lib], check=True, stdout=subprocess.PIPE,
                                                        text=True).stdout.splitlines() if ln.strip()}
    assert not [s for s in want if s not in exported]
    exe = str(tmp_path / "punc_client")
    r = subprocess.run(["g++", "-std=c++17", '-DFUNASR_RUNTIME_HEADER="funasrruntime_b200.h"', "-I" + inc,
                        os.path.join(ROOT, "examples", "offline_punc_client.cpp"), "-L" + os.path.join(ROOT, "funasr_b200"), "-lfunasr_b200",
                        "-Wl,-rpath," + os.path.join(ROOT, "funasr_b200"), "-o", exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    (tmp_path / "in.txt").write_text("你好\n")
    r = subprocess.run([exe, str(tmp_path), str(tmp_path / "in.txt")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 1 and "punc init failed" in r.stdout


def test_walk_reproduces_the_reference_walk_with_scripted_scorers():
    """tests/golden/punc_walk_cases.npz (oracle/make_punc_walk_golden.py): the unmodified reference's CTTransformer.inference with its
    punc_forward replaced by scripted scorers, on texts that reach the comma cut past 200 words, windows carried whole, English-only
    text and final windows ending in ，, 、, "," or a Latin word.  The C++ walk and punc.py both reproduce every case exactly."""
    g = np.load(os.path.join(GOLDEN, "punc_walk_cases.npz"))
    names = set()
    longest = 0
    for i in range(int(g["n"])):
        text, seed, probs = str(g["text_in_%d" % i]), int(g["seed_%d" % i]), tuple(g["probs_%d" % i].tolist())
        want = (str(g["text_out_%d" % i]), g["punc_array_%d" % i].tolist())
        seen = []

        def score(ids, lens, seed=seed, probs=probs):
            seen.append(int(lens.max()))
            return scripted(ids, seed, probs)

        assert walk([text], score) == [want], str(g["name_%d" % i])
        assert spec([text], ScriptedEngine(seed, probs)) == [want]
        names.add(str(g["name_%d" % i]))
        longest = max(longest, max(seen))
        if str(g["name_%d" % i]) == "rare_ends_with_commas":
            assert max(seen) > 200 and want[1].count(3) > 0                    # the cut at the last comma happened
    assert longest > 200 and {"no_comma_no_end", "english_only", "ends_in_comma_cjk", "ends_in_dun", "ends_in_comma_latin",
                              "ends_in_latin_word"} <= names
