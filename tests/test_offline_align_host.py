"""CPU: the forced-alignment side of the handle API that needs no GPU -- the MonotonicAligner model file (the repacked timestamp head,
__aligner_config__ and its eos_id), fa_align_init's refusals (all in the index pass, before any device work), the NULL and argument
cases of fa_align_infer, fa_offline_init refusing an aligner file, and the C client compiling against the plain C header."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

from funasr_b200 import _abi, pack, synth
from test_offline_stamps_host import HEAD_NAMES

CFG = synth.ALIGNER_TINY


def _state():
    return synth.make_aligner_state_dict(CFG, 5)


def test_aligner_model_file_round_trips(tmp_path):
    st = _state()
    path = str(tmp_path / "aligner.fab2")
    pack.write_aligner_model_file(path, st, CFG, synth.make_cmvn(CFG, 1), token_list=synth.aligner_token_list(400),
                                  smooth_factor2=0.3, noise_threshold2=0.02)
    back = pack.read_model_file(path)
    head = pack.timestamp_head_tensors(st)
    assert set(head) == set(HEAD_NAMES)
    for k in HEAD_NAMES:
        assert back[k].shape == tuple(head[k].shape) and np.array_equal(back[k], head[k].numpy()), k
    assert back["predictor.upsample_cnn.gemm_weight"].shape == (3 * 320, 320)
    assert back["__ts_config__"].tolist() == [3.0, float(np.float32(0.3)), float(np.float32(0.02))]
    cfg = back["__aligner_config__"].tolist()
    assert cfg == [CFG.enc_layers, 320, 4, 560, float(np.float32(CFG.ln_eps)), 1.0, 2]
    assert back["frontend.cmvn"].shape == (2, 560) and back["encoder.pe_inv_timescales"].shape == (280,)
    for k, v in st.items():                                     # the encoder under its own names, unchanged
        if k.startswith("encoder."):
            assert np.array_equal(back[k], v.numpy()), k
    assert not [k for k in back if "cif_conv1d" in k or k.startswith("predictor.cif_output.")]
    assert not [k for k in back if k in ("__config__", "__sv_config__")]
    # eos_id: -1 without a token list or without "</s>" in it
    assert pack.aligner_model_tensors(st, CFG, None)["__aligner_config__"][6] == -1
    assert pack.aligner_model_tensors(st, CFG, None, token_list=["<blank>", "a", "<unk>"])["__aligner_config__"][6] == -1
    with pytest.raises(ValueError):
        pack.aligner_model_tensors(synth.make_state_dict(synth.PARAFORMER_TINY, 3), CFG, None)


def _variant(tmp_path, name, edit):
    t = pack.aligner_model_tensors(_state(), CFG, synth.make_cmvn(CFG, 1), synth.aligner_token_list(400))
    edit(t)
    path = str(tmp_path / name)
    pack._write(path, t)
    return path


def _cfg(**kw):
    idx = {"enc_layers": 0, "d_model": 1, "heads": 2, "feat_dim": 3}

    def edit(t):
        c = t["__aligner_config__"].copy()
        for k, v in kw.items():
            c[idx[k]] = v
        t["__aligner_config__"] = c
    return edit


def test_align_init_refusals_name_the_piece(tmp_path):
    """Every refusal of fa_align_init comes from the index pass: NULL and a message naming the piece, with or without a GPU."""
    lib = _abi.load()

    def drop(*names):
        return lambda t: [t.pop(n) for n in names]

    def put(name, value):
        return lambda t: t.__setitem__(name, np.asarray(value, np.float32))

    cases = [
        ("no_cfg", drop("__aligner_config__"), [b"__aligner_config__"]),
        ("short_cfg", put("__aligner_config__", [3, 320, 4]), [b"__aligner_config__"]),
        ("with_config", put("__config__", np.zeros(10)), [b"__config__"]),
        ("with_sv", put("__sv_config__", np.zeros(9)), [b"__sv_config__"]),
        ("d384", _cfg(d_model=384, heads=4), [b"d_model 384"]),
        ("hd64", _cfg(d_model=320, heads=5), [b"d_model 320 with 5 heads"]),
        ("d512_h8", _cfg(d_model=512, heads=8), [b"d_model 512 with 8 heads"]),
        ("feat400", _cfg(feat_dim=400), [b"feat_dim 400"]),
        ("cmvn", put("frontend.cmvn", np.zeros((2, 400))), [b"frontend.cmvn"]),
        ("cmvn_flat", put("frontend.cmvn", np.zeros(1120)), [b"frontend.cmvn"]),
        ("up5", put("__ts_config__", [5, 0.25, 0.01]), [b"upsample_times", b"timestamp head"]),
        ("no_ts_cfg", drop("__ts_config__"), [b"__ts_config__", b"timestamp head"]),
        ("no_ih", drop("predictor.blstm.ih_gemm_bias"), [b"predictor.blstm.ih_gemm_bias", b"timestamp head"]),
        ("no_hh", drop("predictor.blstm.weight_hh_l0_reverse"), [b"predictor.blstm.weight_hh_l0_reverse", b"timestamp head"]),
        ("head512", put("predictor.upsample_cnn.gemm_weight", np.zeros((1536, 512))), [b"predictor.upsample_cnn.gemm_weight"]),
        ("out2", put("predictor.cif_output2.weight", np.zeros((1, 1024))), [b"predictor.cif_output2.weight"]),
        ("no_enc", drop("encoder.encoders.1.self_attn.linear_out.weight"), [b"encoder.encoders.1.self_attn.linear_out.weight"]),
        ("enc_shape", put("encoder.encoders0.0.feed_forward.w_2.weight", np.zeros((320, 1000))),
         [b"encoder.encoders0.0.feed_forward.w_2.weight"]),
        ("no_pe", drop("encoder.pe_inv_timescales"), [b"encoder.pe_inv_timescales"]),
        ("no_mel", drop("frontend.mel_banks"), [b"frontend.mel_banks"]),
    ]
    for name, edit, needles in cases:
        path = _variant(tmp_path, name + ".fab2", edit)
        assert not lib.fa_align_init(path.encode(), 0, 3), name
        msg = lib.fa_offline_last_error()
        assert all(n in msg for n in needles), (name, msg)
        if name not in ("with_config", "with_sv"):
            assert b"MonotonicAligner" in msg, (name, msg)
    assert not lib.fa_align_init(None, 0, 3) and b"NULL" in lib.fa_offline_last_error()
    assert not lib.fa_align_init(_variant(tmp_path, "ok.fab2", lambda t: None).encode(), 0, 5)
    assert b"gemm_mode" in lib.fa_offline_last_error()
    assert not lib.fa_align_init(str(tmp_path / "absent.fab2").encode(), 0, 3)
    assert b"cannot open" in lib.fa_offline_last_error()


def test_recogniser_refuses_an_aligner_file(tmp_path):
    lib = _abi.load()
    path = _variant(tmp_path, "aligner.fab2", lambda t: None)
    assert not lib.fa_offline_init(path.encode(), 0, 3)
    assert b"fa_align_init" in lib.fa_offline_last_error()
    # and the aligner refuses a recogniser file
    p2 = str(tmp_path / "para.fab2")
    pack.write_model_file(p2, synth.make_state_dict(synth.PARAFORMER_TINY, 3), synth.PARAFORMER_TINY, None)
    assert not lib.fa_align_init(p2.encode(), 0, 3)
    assert b"__aligner_config__" in lib.fa_offline_last_error()


def test_null_handle_and_arguments():
    lib = _abi.load()
    wav = np.zeros(16000, np.float32)
    bufs = (C.c_void_p * 1)(wav.ctypes.data)
    n = (C.c_int64 * 1)(16000)
    fmt = _abi.FaAudioFormat(0, 1, 16000, 0)
    ids = np.array([5, 6], np.int32)
    rows = (C.c_void_p * 1)(ids.ctypes.data)
    n_ids = (C.c_int32 * 1)(2)
    assert not lib.fa_align_infer(None, bufs, n, 1, C.byref(fmt), rows, n_ids)
    assert b"bad argument" in lib.fa_offline_last_error()
    lib.fa_align_uninit(None)
    cnt = C.c_int32(7)
    assert lib.fa_offline_result_count(None) == 0
    assert not lib.fa_offline_result_stamps(None, 0, C.byref(cnt)) and cnt.value == 0


def test_align_client_compiles_as_c99(tmp_path):
    """examples/offline_align_client.c is plain C99 against include/funasr_b200.h and links; without a model file it fails cleanly."""
    exe = str(tmp_path / "offline_align_client")
    libdir = os.path.join(ROOT, "funasr_b200")
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I" + os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "examples", "offline_align_client.c"), "-L" + libdir, "-lfunasr_b200", "-Wl,-rpath," + libdir,
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    run = subprocess.run([exe], capture_output=True, text=True)
    assert run.returncode == 2 and "usage" in run.stderr
    tokens = tmp_path / "tokens.txt"
    tokens.write_text("\n".join(synth.aligner_token_list(4)) + "\n", encoding="utf-8")
    (tmp_path / "t.txt").write_text("一", encoding="utf-8")
    (tmp_path / "a.pcm").write_bytes(np.zeros(800, np.int16).tobytes())
    run = subprocess.run([exe, str(tmp_path / "absent.fab2"), str(tokens), str(tmp_path / "a.pcm"), str(tmp_path / "t.txt")],
                         capture_output=True, text=True)
    assert run.returncode == 1 and "init failed" in run.stderr
