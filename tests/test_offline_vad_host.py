"""CPU: the host routines of long-audio recognition in the C library against their Python specifications (segment packing,
merge_vad), the FSMN-VAD model file, the handle API's refusals without a GPU and the link surface of the VAD client."""
import ctypes as C
import os
import random
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

from funasr_b200 import _abi, pack, synth
from funasr_b200.long_audio import pack_segments
from funasr_b200.vad import VadOptions, merge_vad


def _native_pack(segs, batch_size_s, threshold_s):
    lib = _abi.load()
    n = len(segs)
    arr = np.ascontiguousarray(np.array(segs, dtype=np.int32).reshape(-1, 2))
    order = np.zeros(max(n, 1), np.int32)
    packs = np.zeros((max(n, 1), 2), np.int32)
    k = lib.fa_pack_segments(arr.ctypes.data, n, batch_size_s, threshold_s, order.ctypes.data, packs.ctypes.data)
    assert k >= 0
    return order[:n].tolist(), [tuple(p) for p in packs[:k].tolist()]


def _native_merge(segs, max_length_ms, min_length_ms=0):
    lib = _abi.load()
    n = len(segs)
    arr = np.ascontiguousarray(np.array(segs, dtype=np.int32).reshape(-1, 2))
    out = np.zeros((max(2 * n, 1), 2), np.int32)
    k = lib.fa_merge_vad(arr.ctypes.data, n, max_length_ms, min_length_ms, out.ctypes.data)
    assert k >= 0
    return out[:k].tolist()


def _random_segments(rng, n):
    segs, t = [], rng.randint(0, 3000)
    for _ in range(n):
        kind = rng.random()
        if kind < 0.2:
            d = rng.choice([1000, 2000, 5000])                        # ties
        elif kind < 0.3:
            d = rng.choice([59990, 60000, 60010, 70000])               # around the 60 s threshold and beyond batch_size_s
        else:
            d = rng.randint(30, 20000)
        segs.append([t, t + d])
        t += d + rng.randint(0, 4000)
    return segs


def test_pack_segments_matches_the_python_specification():
    rng = random.Random(1234)
    cases = [([], 300, 60), ([[0, 500]], 300, 60), ([[0, 400000]], 300, 60), ([[0, 60000], [61000, 121000]], 300, 60),
             ([[0, 1000], [2000, 3000], [4000, 5000]], 1, 60), ([[0, 3000], [4000, 7000]], 6, 60), ([[0, 2000]] * 5, 6, 60)]
    for _ in range(2400):
        n = rng.choice([1, 2, 3, rng.randint(1, 12), rng.randint(1, 80)])
        cases.append((_random_segments(rng, n), rng.choice([0, 1, 6, 30, 60, 300]), rng.choice([0, 1, 10, 60])))
    for segs, bs, th in cases:
        assert _native_pack(segs, bs, th) == pack_segments(segs, bs, th), (segs, bs, th)


def test_merge_vad_matches_the_python_specification():
    rng = random.Random(99)
    cases = [([], 15000), ([[100, 900]], 15000), ([[0, 1000], [1000, 2000]], 15000), ([[0, 20000], [21000, 22000]], 15000)]
    for _ in range(2000):
        cases.append((_random_segments(rng, rng.randint(1, 40)), rng.choice([0, 1000, 5000, 15000, 60000])))
    for segs, ml in cases:
        assert _native_merge(segs, ml) == merge_vad(segs, ml), (segs, ml)
    assert _native_merge([[0, 1000], [1200, 1500], [9000, 9100]], 1000, 250) == merge_vad([[0, 1000], [1200, 1500], [9000, 9100]], 1000, 250)


def test_vad_model_file_round_trip(tmp_path):
    st = synth.make_vad_state_dict(synth.VAD_DEFAULT, 0)
    cmvn = synth.make_vad_cmvn(0)
    path = str(tmp_path / "vad.fab2")
    conf = {"max_end_silence_time": 500, "speech_noise_thres": 0.6, "fe_prior_thres": 1e-4, "snr_thres": -100.0, "sil_pdf_ids": [0, 3],
            "speech_2_noise_ratio": 1.0 / 3.0}
    pack.write_vad_model_file(path, st, cmvn, conf)
    back = pack.read_model_file(path)
    cfg = pack.read_vad_config(back)
    want = VadOptions.from_conf(conf)
    for name in pack.VAD_INT_FIELDS + pack.VAD_REAL_FIELDS:
        assert cfg[name] == getattr(want, name) and type(cfg[name])(getattr(want, name)) == cfg[name], name
    assert cfg["speech_noise_thres"] == 0.6 and cfg["fe_prior_thres"] == 1e-4          # exact doubles, not their fp32 roundings
    assert cfg["speech_2_noise_ratio"] == 1.0 / 3.0
    assert cfg["lorder"] == 20 and cfg["sil_pdf_ids"] == [0, 3]
    for k, v in st.items():
        assert np.array_equal(back[k], v.numpy()) and back[k].shape == tuple(v.shape), k
    assert np.array_equal(back["frontend.cmvn"], cmvn.numpy()) and back["frontend.mel_banks"].shape == (80, 257)
    # defaults
    pack.write_vad_model_file(path, st, cmvn, {})
    d = pack.read_vad_config(pack.read_model_file(path))
    assert d["speech_noise_thres"] == 0.6 and d["fe_prior_thres"] == 1e-4 and d["max_end_silence_time"] == 800 and d["sil_pdf_ids"] == [0]


def test_vad_model_file_refuses_unsupported_shapes(tmp_path):
    st = synth.make_vad_state_dict(synth.VAD_DEFAULT, 0)
    path = str(tmp_path / "vad.fab2")
    bad = dict(st)
    bad["encoder.fsmn.0.fsmn_block.conv_right.weight"] = torch.zeros(128, 1, 2, 1)
    with pytest.raises(ValueError):
        pack.write_vad_model_file(path, bad, None, {})
    short = dict(st)
    short["encoder.fsmn.1.fsmn_block.conv_left.weight"] = torch.zeros(128, 1, 10, 1)
    with pytest.raises(ValueError):
        pack.write_vad_model_file(path, short, None, {})
    with pytest.raises(ValueError):
        pack.write_vad_model_file(path, st, None, {"max_end_silence_time": 800.5})
    with pytest.raises(ValueError):
        pack.write_vad_model_file(path, st, None, {"sil_pdf_ids": [0, 1, 2, 3, 4]})
    with pytest.raises(Exception):
        pack.write_vad_model_file(path, st, None, {"encoder_conf": dict(input_dim=400, input_affine_dim=140, fsmn_layers=4, linear_dim=250,
                                                                        proj_dim=128, lorder=20, rorder=1, lstride=1, rstride=0,
                                                                        output_affine_dim=140, output_dim=248)})


def test_vad_handle_refuses_bad_files_and_null_handles(tmp_path):
    """Missing, truncated or wrong-magic files, files with a bad piece and NULL handles: NULL plus a message, never an exception across
    the ABI.  A file is checked on its index before any device work, so the message names the piece on any machine."""
    lib = _abi.load()
    good = str(tmp_path / "vad.fab2")
    pack.write_vad_model_file(good, synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    blob = open(good, "rb").read()
    (tmp_path / "trunc.fab2").write_bytes(blob[: len(blob) // 2])
    (tmp_path / "magic.fab2").write_bytes(b"XXXXXXXX" + blob[8:])
    (tmp_path / "empty.fab2").write_bytes(b"")
    assert not lib.fa_vad_init(str(tmp_path / "missing.fab2").encode(), 0) and b"cannot open" in lib.fa_offline_last_error()
    for p in ("trunc.fab2", "magic.fab2", "empty.fab2"):
        assert not lib.fa_vad_init(str(tmp_path / p).encode(), 0)
        assert b"malformed" in lib.fa_offline_last_error()

    def refused(edit):
        t = pack.vad_model_tensors(synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
        edit(t)
        path = str(tmp_path / "bad.fab2")
        pack._write(path, t)
        assert not lib.fa_vad_init(path.encode(), 0)
        return lib.fa_offline_last_error().decode()

    def set_cfg(i, v):
        def f(t):
            c = t["__vad_config__"].view("<f8").copy()
            c[i] = v
            t["__vad_config__"] = c.view("<f4")
        return f

    assert "right-context" in refused(lambda t: t.__setitem__("encoder.fsmn.1.fsmn_block.conv_right.weight", np.zeros((128, 1, 2, 1), np.float32)))
    assert refused(lambda t: t.pop("encoder.out_linear2.linear.weight")) == "missing tensor encoder.out_linear2.linear.weight"
    assert refused(lambda t: t.__setitem__("__vad_config__", t["__vad_config__"][:48])) == "bad __vad_config__"
    assert refused(set_cfg(19, 10)) == "unsupported VAD config"                     # lorder
    assert refused(set_cfg(21, 248)) == "sil_pdf_ids outside the output"            # out_linear2 has 248 outputs
    h = lib.fa_vad_init(good.encode(), 0)
    assert h or lib.fa_offline_last_error() == b"no such CUDA device (this library has no CPU path)"
    lib.fa_vad_uninit(h)
    assert not lib.fa_vad_init(None, 0)
    assert lib.fa_offline_last_error() == b"model_file is NULL"
    x = np.zeros(16000, np.float32)
    assert not lib.fa_vad_infer(None, x.ctypes.data, x.size, 0, None)
    assert lib.fa_offline_last_error() == b"bad argument"
    ptrs = (C.c_void_p * 1)(x.ctypes.data)
    lens = (C.c_int64 * 1)(x.size)
    assert not lib.fa_offline_infer_vad(None, None, ptrs, lens, 1, 0, None, 0, None)
    assert lib.fa_offline_last_error() == b"bad argument"
    n = C.c_int64(7)
    assert not lib.fa_vad_result_segments(None, C.byref(n)) and n.value == 0
    m = C.c_int32(7)
    assert not lib.fa_offline_result_segments(None, 0, C.byref(m)) and m.value == 0
    lib.fa_vad_free_result(None)
    lib.fa_vad_uninit(None)
    assert lib.fa_pack_segments(None, 3, 300, 60, None, None) == -1
    assert lib.fa_merge_vad(None, 3, 15000, 0, None) == -1
    assert lib.fa_gather_segments(None, 10, None, None, 1, 4, None, None) == -1


def test_vad_client_links_against_the_reference_header(tmp_path):
    """examples/offline_vad_client.cpp (the call sequence of bin/funasr-onnx-offline-vad.cpp plus FunOfflineInit with "vad-dir")
    compiled against include/funasrruntime_b200.h needs exactly the runtime symbols it needs against the reference's own
    funasrruntime.h (tests/golden/fsmnvad_client_symbols.txt, oracle/make_vad_client_symbols_golden.py); the library exports them all,
    and the client links and fails cleanly without a GPU / model."""
    if shutil.which("g++") is None or shutil.which("nm") is None:
        pytest.skip("no g++ / nm")
    import make_vad_client_symbols_golden as mk
    inc = os.path.join(ROOT, "include")
    with open(os.path.join(GOLDEN, "fsmnvad_client_symbols.txt")) as f:
        want = f.read().split()
    assert len(want) >= 10 and any("FsmnVadGetResult" in s for s in want)
    assert mk.client_runtime_symbols('"funasrruntime_b200.h"', inc) == want
    lib = os.path.join(ROOT, "funasr_b200", "libfunasr_b200.so")
    exported = {ln.split()[-1] for ln in subprocess.run(["nm", "-D", "--defined-only", lib], check=True, stdout=subprocess.PIPE,
                                                        text=True).stdout.splitlines() if ln.strip()}
    assert not [s for s in want if s not in exported]
    exe = str(tmp_path / "vad_client")
    r = subprocess.run(["g++", "-std=c++17", '-DFUNASR_RUNTIME_HEADER="funasrruntime_b200.h"', "-I" + inc,
                        os.path.join(ROOT, "examples", "offline_vad_client.cpp"), "-L" + os.path.join(ROOT, "funasr_b200"), "-lfunasr_b200",
                        "-Wl,-rpath," + os.path.join(ROOT, "funasr_b200"), "-o", exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    r = subprocess.run([exe, str(tmp_path), str(tmp_path / "none.wav")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 1 and "init failed" in r.stdout
