"""CPU: the float64 CAM++ restatement (tests/campplus_ref.py) that the GPU parity tests compare against, pinned to the reference:
to the embeddings the unmodified reference computed for the fixtures' chunks (oracle/make_spk_golden.py stores them as cb_in) and,
where the reference tree is present, to its CAMPPlus class run live in float64.  Also the frame-count limits of the forward's
workspace query (host code)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from campplus_ref import campplus_ref, emb_err
from test_spk_host import SPK_CASES, campplus_state_dict, load_spk_case

# Worst over the 4 stored chunks of each fixture (T = 148), measured on an x86-64 CPU with torch 2.11: the restatement (float64)
# against the reference's fp32 CAMPPlus run.  "matrix": max |d| / max |ref| over the fixture's [4, 192] block; "utt": the same per
# utterance (campplus_ref.emb_err).  What remains is the reference's own fp32 rounding.  Bars: 4 x the worst of all fixtures.
MEASURED_VS_STORED = {"spk_two_voices": (7.65e-6, 1.54e-5), "spk_three_preset": (3.82e-6, 1.10e-5), "spk_few_chunks": (6.57e-6, 1.29e-5),
                      "spk_short_segment": (8.46e-6, 1.17e-5)}
BAR_MATRIX, BAR_UTT = 3.4e-5, 6.2e-5
# The live reference in float64 against the restatement: 4.3e-14 worst per utterance at T = 3, 201 and 401
BAR_LIVE64 = 1e-12
LIVE_T = (2, 3, 201, 401)


@pytest.mark.parametrize("name", list(SPK_CASES))
def test_restatement_matches_the_stored_reference_embeddings(name):
    g = load_spk_case(name)
    ref = g["cb_in"][:4].astype(np.float64)                 # the chunks the features were extracted from, in time order
    got = campplus_ref(campplus_state_dict(), torch.from_numpy(g["features"])).numpy()
    matrix = float(np.abs(got - ref).max() / np.abs(ref).max())
    utt = float(emb_err(ref, got)[0].max())
    print("restatement vs stored reference %s: matrix %.3e, worst utterance %.3e" % (name, matrix, utt))
    assert matrix <= BAR_MATRIX and utt <= BAR_UTT


def _live_inputs(T):
    """Two utterances of T frames cut from the fixtures' stored chunk features (real CMN'd fbank, calibrated BN statistics)."""
    f = np.concatenate([load_spk_case(n)["features"].reshape(-1, 80) for n in ("spk_two_voices", "spk_few_chunks")])
    return np.stack([f[:T], f[100:100 + T]])


_LIVE = """
import sys
import numpy as np
import torch
import ref_shim
ref_shim.import_reference()
from funasr.models.campplus.model import CAMPPlus
from test_spk_host import campplus_state_dict
m = CAMPPlus(feat_dim=80, embedding_size=192, growth_rate=32, bn_size=4, init_channels=128, config_str="batchnorm-relu",
             memory_efficient=True, output_level="segment")
m.load_state_dict(campplus_state_dict(), strict=True)
m.double().eval()
z = np.load(sys.argv[1])
with torch.no_grad():
    np.savez(sys.argv[2], **{k: m(torch.from_numpy(z[k])).numpy() for k in z.files})
"""


def test_restatement_matches_the_live_reference(tmp_path):
    """The reference's CAMPPlus, in float64, on T = 2, 3, 201 and 401 frames (the smallest inputs, a one-frame last CAM segment, three
    segments): equal to the restatement within float64 rounding, and NaN exactly where it is (T = 2: the unbiased std of one TDNN
    frame).  Run in a child process: importing the reference registers its classes into process-wide tables other tests read."""
    import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("reference tree not present")
    inp, out = tmp_path / "in.npz", tmp_path / "out.npz"
    np.savez(inp, **{"T%d" % T: _live_inputs(T).astype(np.float64) for T in LIVE_T})
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, "-c", _LIVE, str(inp), str(out)], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                       env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    live = np.load(out)
    sd = campplus_state_dict()
    for T in LIVE_T:
        ref = live["T%d" % T]
        mine = campplus_ref(sd, torch.from_numpy(_live_inputs(T))).numpy()
        if T == 2:
            assert np.isnan(ref).all() and np.isnan(mine).all()
            continue
        err = float(emb_err(mine, ref)[0].max())
        print("restatement vs live reference (float64) T%d: %.3e" % (T, err))
        assert err <= BAR_LIVE64, (T, err)


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_workspace_query_names_the_frame_limits(mode):
    """fa_campplus_workspace_bytes returns 0 for every input the forward refuses: fewer than 2 frames, or more than 18 800 (94 CAM
    segments of 100 TDNN frames, the segment means the context gate holds in shared memory); the Python engine's message names the
    same limit."""
    from funasr_b200 import _abi
    from funasr_b200.campplus import MAX_FEAT_FRAMES
    lib = _abi.load()
    m = _abi.FaCampplus()
    m.n_layers[0], m.n_layers[1], m.n_layers[2] = 12, 24, 16
    q = lambda b, t: int(lib.fa_campplus_workspace_bytes(C.byref(m), b, t, mode))
    assert MAX_FEAT_FRAMES == 18800
    assert q(1, 1) == 0 and q(1, 2) > 0
    for b in (1, 4):
        assert q(b, 18800) > q(b, 18799) > 0
        assert q(b, 18801) == 0 and q(b, 20000) == 0 and q(b, 1 << 30) == 0
