"""CPU: the MonotonicAligner (fa-zh) goldens against the oracle's restatement, the aligner's transcript forms, its drop-in key and
the plane-fed attention entry with an explicit head dim in the C ABI."""
import os

import numpy as np
import pytest
import torch

import aligner_oracle
from conftest import GOLDEN
from funasr_b200 import _abi, registry, synth
from funasr_b200.modules import MonotonicAlignerB200, _aligner_tokens
from funasr_b200.timestamps import ts_prediction_lfr6_standard

CASES = {"aligner_tiny_ragged3": (synth.ALIGNER_TINY, 5), "aligner_fa_zh_single": (synth.ALIGNER_FA_ZH, 6)}
TOKENS = synth.aligner_token_list(400)


def _split(flat, lens, width=1):
    return np.split(flat.reshape(-1, width) if width > 1 else flat, np.cumsum(lens)[:-1])


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    name = request.param
    cfg, seed = CASES[name]
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    ids = [[int(t) for t in r] for r in _split(z["ids_flat"], z["ids_len"])]
    wavs = [synth.make_aligner_wav(float(sec), int(s)) for sec, s in z["wav_spec"]]
    out = aligner_oracle.aligner_forward(wavs, ids, synth.make_aligner_state_dict(cfg, seed), synth.make_cmvn(cfg, seed=1), cfg.enc_layers)
    return name, z, ids, out


def test_oracle_reproduces_aligner_golden(case):
    name, z, ids, out = case
    assert out["enc_lens"].tolist() == z["enc_lens"].tolist()
    assert torch.allclose(out["enc"][:, z["enc_rows"]], torch.from_numpy(z["enc"]), rtol=0, atol=1e-4)
    for b, n in enumerate(z["enc_lens"].tolist()):
        ref = torch.from_numpy(z["us_alphas"][b, :3 * n])
        assert float((out["us_alphas"][b, :3 * n] - ref).abs().max() / ref.abs().max()) <= 1e-5
    stamps = _split(z["stamps_flat"], z["stamps_len"], 2)
    for b, n in enumerate(z["enc_lens"].tolist()):
        _, st = ts_prediction_lfr6_standard(out["us_alphas"][b, :3 * n].numpy(), out["us_peaks"][b, :3 * n].numpy(),
                                            [TOKENS[t] for t in ids[b]], want_text=False)
        assert st == stamps[b].tolist(), (name, b)
    # the fire decisions sit far from the threshold, so fp32 reorderings cannot move a stamp
    assert float(z["fire_margin"]) > 1e-4


def test_golden_stamps_are_not_uniform():
    z = np.load(os.path.join(GOLDEN, "aligner_fa_zh_single.npz"))
    starts = z["stamps_flat"].reshape(-1, 2)[:, 0]
    gaps = np.diff(starts)
    assert gaps.max() >= 4 * max(gaps.min(), 20)


def test_tiny_golden_covers_reintegration_and_single_char():
    z = np.load(os.path.join(GOLDEN, "aligner_tiny_ragged3.npz"))
    lens, elens = z["ids_len"].tolist(), z["enc_lens"].tolist()
    assert 1 in lens and len(set(lens)) == 3
    # more characters than the scan fires for: ts_prediction_lfr6_standard re-integrates
    fires = [int((z["us_peaks"][b, :3 * n] >= 1.0 - 1e-4).sum()) for b, n in enumerate(elens)]
    assert any(f < n + 1 for f, n in zip(fires, lens)), (fires, lens)


def test_sentence_postprocess_of_oracle_stamps_equals_golden_final():
    """The reference's sentence_postprocess on the golden pre-postprocessing stamps gives the golden final (text, timestamp).  Run in
    a child process: importing the reference registers its classes into process-wide tables other tests read."""
    import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("reference tree not present")
    code = """
import json, sys
import numpy as np
import ref_shim
ref_shim.import_reference()
from funasr.utils import postprocess_utils
from funasr_b200 import synth
toks = synth.aligner_token_list(400)
z = np.load(sys.argv[1])
ids = np.split(z["ids_flat"], np.cumsum(z["ids_len"])[:-1])
st = np.split(z["stamps_flat"].reshape(-1, 2), np.cumsum(z["stamps_len"])[:-1])
fin = np.split(z["final_flat"].reshape(-1, 2), np.cumsum(z["final_len"])[:-1])
ok = []
for b in range(len(ids)):
    text, ts, _ = postprocess_utils.sentence_postprocess([toks[t] for t in ids[b]], st[b].tolist())
    ok.append(text == str(z["final_text"][b]) and [list(p) for p in ts] == fin[b].tolist())
print(json.dumps(ok))
"""
    import json
    import subprocess
    import sys
    from conftest import ROOT
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "oracle")]))
    for name in CASES:
        r = subprocess.run([sys.executable, "-c", code, os.path.join(GOLDEN, name + ".npz")], stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True, env=env, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        assert json.loads(r.stdout.strip().splitlines()[-1]) == [True] * len(np.load(os.path.join(GOLDEN, name + ".npz"))["ids_len"])


class _Tok:
    def encode(self, text):
        return [TOKENS.index(t) for t in text.strip().split(" ")]


def test_transcript_forms(tmp_path):
    text = " ".join(TOKENS[3:9])
    want = list(range(3, 9))
    assert _aligner_tokens(text, _Tok()) == want
    p = tmp_path / "t.txt"
    p.write_text(text + "\n")
    assert _aligner_tokens(str(p), _Tok()) == want
    assert _aligner_tokens(want, None) == want
    assert _aligner_tokens(np.array(want), None) == want
    with pytest.raises(_abi.FunasrB200Error):
        _aligner_tokens(text, None)


def test_aligner_drop_in_key_and_params():
    assert registry.DROP_IN_KEYS[("model_classes", "MonotonicAligner")] == "MonotonicAlignerB200"
    cfg = synth.ALIGNER_TINY
    m = MonotonicAlignerB200(
        encoder="SANMEncoder", encoder_conf=dict(output_size=320, attention_heads=4, linear_units=1280, num_blocks=cfg.enc_layers,
                                                 kernel_size=11, input_layer="pe", normalize_before=True, selfattention_layer_type="sanm"),
        predictor="CifPredictorV3", predictor_conf=dict(idim=320, threshold=1.0, l_order=1, r_order=1, tail_threshold=0.45, smooth_factor2=0.25,
                                                        noise_threshold2=0.01, upsample_times=3, use_cif1_cnn=False, upsample_type="cnn_blstm"),
        input_size=560, predictor_bias=1, length_normalized_loss=False, specaug="SpecAugLFR")
    # the reference's state_dict names, predictor.cif_conv1d / cif_output included
    m.load_state_dict(synth.make_aligner_state_dict(cfg, 5), strict=True)
    with pytest.raises(_abi.FunasrB200Error):
        m.engine("cpu")


def test_plane_attention_ex_in_header_and_mirror():
    hdr = open(os.path.join(os.path.dirname(_abi.__file__), "..", "include", "funasr_b200.h")).read()
    assert "int fa_attention_tc_planes_ex(" in hdr
    assert len(_abi.SIGNATURES["fa_attention_tc_planes_ex"][1]) == len(_abi.SIGNATURES["fa_attention_tc_planes"][1]) + 1
