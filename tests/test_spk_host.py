"""Speaker diarization host routines (funasr_b200.diarization, long_audio.speaker_chunks) against the reference's stored results, and the
CAM++ surface that needs no GPU (ABI symbols, state_dict names).  Fixtures: oracle/make_spk_golden.py."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

# name: (pattern [(voice, speech_s, silence_s)], wav seed, generate kwargs) — must match oracle/make_spk_golden.py:SPK_CASES
SPK_CASES = {
    "spk_two_voices": ([(v, 3.0, 2.5) for v in (0, 1) * 4], 1, {}),
    "spk_three_preset": ([(v, 3.0, 2.5) for v in (0, 1, 2) * 3], 2, {"preset_spk_num": 3, "return_spk_center": True}),
    "spk_few_chunks": ([(0, 3.0, 2.5), (1, 3.0, 2.5)], 3, {}),
    "spk_short_segment": ([(0, 3.0, 2.5), (1, 1.0, 2.5), (0, 3.0, 2.5), (1, 3.0, 2.5)] * 2, 4, {}),
}
SPK_SEED = 0
HOST_CLUSTER_CASES = ["spectral_k3", "spectral_preset4", "merge_by_cos", "kmeans_2048", "few_rows"]


def load_spk_case(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    g["sentence_info"] = json.loads(str(g["sentence_info"]))
    g["kwargs"] = json.loads(str(g["kwargs"]))
    return g


def campplus_state_dict():
    """The fixtures' CAM++ weights: the seeded synthetic weights with the calibrated BatchNorm statistics overlaid."""
    from funasr_b200 import synth
    stats = dict(np.load(os.path.join(GOLDEN, "spk_campplus_bn.npz")))
    return synth.make_campplus_state_dict(SPK_SEED, stats)


def vad_segments(g):
    return [[s["start"], s["end"]] for s in g["sentence_info"]]


@pytest.mark.parametrize("name", list(SPK_CASES))
def test_chunk_bounds_match_reference(name):
    """sv_chunk over every VAD segment's samples: chunk times bit-equal, chunk samples (zero-padded tails) sum-equal."""
    from funasr_b200 import synth
    from funasr_b200.long_audio import speaker_chunks
    pattern, seed, _ = SPK_CASES[name]
    g = load_spk_case(name)
    wav = synth.make_voice_wav(pattern, seed).numpy()
    assert wav.size == int(g["n_samples"])
    ch = speaker_chunks(vad_segments(g), wav.size)
    assert [[a, b] for a, b, _, _ in ch] == g["chunk_times"].tolist()
    sums = [float(np.sum(np.pad(wav[s:s + n], (0, 24000 - n)), dtype=np.float64)) for _, _, s, n in ch]
    assert sums == g["chunk_waves_sum"].tolist()


@pytest.mark.parametrize("name", list(SPK_CASES))
def test_labels_and_sentence_info_match_reference(name):
    """ClusterBackend on the reference's embeddings -> the reference's labels (incl. the eigengap count); postprocess + distribute_spk
    -> its sentence_info speakers; return_spk_center -> its centres within fp32 rounding."""
    from funasr_b200 import diarization as D
    g = load_spk_case(name)
    kw = g["kwargs"]
    labels = D.ClusterBackend()(g["cb_in"], oracle_num=kw.get("preset_spk_num"))
    assert D.correct_labels(labels).tolist() == D.correct_labels(g["labels"]).tolist()
    segs = [[a, b] for a, b in g["chunk_times"].tolist()]
    if kw.get("return_spk_center"):
        sv, centers = D.postprocess(segs, None, labels, g["cb_in"], return_spk_center=True)
        np.testing.assert_allclose(centers, g["spk_embedding_center"], rtol=0, atol=1e-6 * np.abs(g["spk_embedding_center"]).max())
    else:
        sv = D.postprocess(segs, None, labels, g["cb_in"])
    sentences = [{k: v for k, v in s.items() if k != "spk"} for s in g["sentence_info"]]
    D.distribute_spk(sentences, sv)
    assert [s["spk"] for s in sentences] == [s["spk"] for s in g["sentence_info"]]


def test_two_voice_fixture_alternates():
    """The fixture is a real diarization case: the two synthetic voices alternate and the reference labels the sentences so."""
    g = load_spk_case("spk_two_voices")
    assert [s["spk"] for s in g["sentence_info"]] == [0, 1] * 4
    assert g["labels"].max() >= 1 and len(g["labels"]) >= 20        # spectral path, speaker count from the eigengap


@pytest.mark.parametrize("case", HOST_CLUSTER_CASES)
def test_cluster_backend_matches_reference(case):
    from funasr_b200 import diarization as D
    g = np.load(os.path.join(GOLDEN, "spk_host_routines.npz"))
    k = int(g[case + "__k"])
    labels = D.ClusterBackend()(g[case + "__x"], oracle_num=None if k < 0 else k)
    assert D.correct_labels(labels).tolist() == D.correct_labels(g[case + "__labels"]).tolist()


@pytest.mark.parametrize("i", range(6))
def test_postprocess_and_distribute_match_reference(i):
    from funasr_b200 import diarization as D
    g = np.load(os.path.join(GOLDEN, "spk_host_routines.npz"))
    segs = g["post%d__segs" % i].tolist()
    sv, centers = D.postprocess([list(s) for s in segs], None, g["post%d__labels" % i].copy(), g["post%d__emb" % i], return_spk_center=True)
    assert np.array_equal(np.array([[a, b, s] for a, b, s in sv], dtype=np.float64), g["post%d__sv" % i])
    np.testing.assert_allclose(centers, g["post%d__centers" % i], rtol=0, atol=1e-6)
    ref = json.loads(str(g["post%d__sentences" % i]))
    sentences = [{"start": d["start"], "end": d["end"]} for d in ref]
    D.distribute_spk(sentences, sv)
    assert [d["spk"] for d in sentences] == [d["spk"] for d in ref]


def test_umap_path_raises():
    from funasr_b200 import diarization as D
    x = np.random.RandomState(0).randn(D.SPECTRAL_MAX_CHUNKS, 8).astype(np.float32)
    with pytest.raises(NotImplementedError, match="2048"):
        D.ClusterBackend()(x)
    assert len(D.ClusterBackend()(x, oracle_num=2)) == D.SPECTRAL_MAX_CHUNKS


def test_sv_chunk_shapes():
    from funasr_b200 import diarization as D
    segs = D.sv_chunk([[1.0, 1.5, np.ones(8000, np.float32)], [3.0, 6.1, np.ones(49600, np.float32)]])
    assert [round(s[0], 4) for s in segs] == [1.0, 3.0, 3.75, 4.5, 4.6]
    assert all(s[2].shape == (24000,) for s in segs) and segs[0][2][8000:].sum() == 0


def test_campplus_abi_symbols_exported():
    from funasr_b200 import _abi
    lib = C.CDLL(_abi.LIB_PATH)
    header = open(os.path.join(ROOT, "include", "funasr_b200.h")).read()
    for name in ("fa_campplus_features", "fa_campplus_workspace_bytes", "fa_campplus_forward", "fa_campplus_conv2d", "fa_campplus_cam",
                 "fa_campplus_stats_pool"):
        assert hasattr(lib, name) and name + "(" in header and name in _abi.SIGNATURES
    assert (C.sizeof(_abi.FaCampplus), C.sizeof(_abi.FaCamLayer), C.sizeof(_abi.FaCamConv2d)) == (680, 96, 32)    # include/funasr_b200.h on x86-64
    _abi.load()
    m = _abi.FaCampplus()
    assert _abi.load().fa_campplus_workspace_bytes(C.byref(m), 0, 148, 0) == 0      # invalid shape -> 0, no crash


def test_campplus_state_dict_names():
    """CAMPPlusB200 holds the reference's state_dict names and shapes; the fixtures' statistics load into it."""
    import torch
    from funasr_b200 import get_tables
    from funasr_b200.campplus import CAMPPlusB200, campplus_specs
    m = CAMPPlusB200()
    sd = campplus_state_dict()
    assert list(m.state_dict().keys()) == list(campplus_specs().keys()) == list(sd.keys())
    m.load_state_dict(sd, strict=True)
    assert sum(v.numel() for k, v in m.state_dict().items() if "running" not in k and "num_batches" not in k) == 6_848_544
    assert get_tables().model_classes["CAMPPlusB200"] is CAMPPlusB200
    with pytest.raises(Exception):
        m.engine("cpu")
    assert torch.equal(m.state_dict()["xvector.dense.nonlinear.batchnorm.running_var"], sd["xvector.dense.nonlinear.batchnorm.running_var"])
