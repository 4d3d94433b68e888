import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")

# name: (config name, weight seed, [(n_samples, wav seed, kind)], use_cmvn) — must match oracle/make_golden.py:CASES
GOLDEN_CASES = {
    "tiny_ragged3": ("tiny", 3, [(48000, 1, "speechlike"), (27200, 2, "noise"), (38437, 3, "speechlike")], True),
    "tiny_single": ("tiny", 3, [(16000, 4, "speechlike")], False),
    "large_ragged2": ("large", 0, [(480000, 0, "speechlike"), (196800, 5, "speechlike")], True),
}


# (n_samples, wav seed, kind) of tests/golden/knf_fbank.npz — must match oracle/make_knf_golden.py:CASES
KNF_CASES = [(16000, 31, "speechlike"), (8123, 32, "noise"), (400, 33, "noise"), (559, 34, "noise"), (48000, 35, "speechlike"), (27200, 36, "noise")]


def knf_logmel_cases():
    """-> [(wav fp32 tensor, golden log-mel [frames, 80] of the reference's compiled kaldi-native-fbank, live log-mel or None)].
    The live column re-runs oracle/_ref/libknf_ref.so when it is present (oracle/knf/Makefile builds it where the reference tree is)."""
    from funasr_b200 import synth
    import knf_ref
    g = np.load(os.path.join(GOLDEN, "knf_fbank.npz"))
    assert g["cases"].tolist() == [[n, s, 0 if k == "speechlike" else 1] for n, s, k in KNF_CASES]
    have = knf_ref.build()
    out = []
    for i, (n, s, k) in enumerate(KNF_CASES):
        w = synth.make_wav(n, s, k)
        out.append((w, g["logmel_%d" % i], knf_ref.fbank(w.numpy()) if have else None))
    return out


def knf_bound(ref_logmel, scale=1.0):
    """|d log-mel| allowed against kaldi-native-fbank: both sides are fp32 FFTs at their rounding floor in near-empty mel bins
    (its Ooura radix-4 FFT is ~4x noisier there than pocketfft): 4e-5 + 8e-6 * sqrt(E_frame_max / E_bin)."""
    r = np.asarray(ref_logmel, dtype=np.float64)
    return scale * (4e-5 + 8e-6 * np.exp(0.5 * (r.max(-1, keepdims=True) - r)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    # a fresh checkout has no built library (it is git-ignored): build it once (nvcc cross-compiles sm_90a without a GPU)
    if not os.path.exists(os.path.join(ROOT, "funasr_b200", "libfunasr_b200.so")):
        import __graft_entry__
        __graft_entry__.build()


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_case(name):
    from funasr_b200 import synth
    cfg_name, wseed, specs, use_cmvn = GOLDEN_CASES[name]
    cfg = synth.PARAFORMER_TINY if cfg_name == "tiny" else synth.PARAFORMER_LARGE
    gold = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    wavs = [synth.make_wav(n, s, k) for (n, s, k) in specs]
    cmvn = synth.make_cmvn(cfg, seed=1) if use_cmvn else None
    if cmvn is not None:
        # the golden run passed CMVN through an am.mvn text file written with %.9g (lossless for fp32)
        cmvn = torch.tensor(np.array([[float("%.9g" % v) for v in row] for row in cmvn.tolist()], dtype=np.float32))
    return cfg, wseed, wavs, cmvn, gold


_STATE_CACHE = {}


def state_dict_for(cfg, seed):
    from funasr_b200 import synth
    key = (cfg.enc_layers, cfg.dec_layers, cfg.vocab, seed)
    if key not in _STATE_CACHE:
        _STATE_CACHE.clear()            # at most one (large ~880 MB) dict alive
        _STATE_CACHE[key] = synth.make_state_dict(cfg, seed)
    return _STATE_CACHE[key]


def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


# SenseVoiceSmall golden cases — must match oracle/make_golden.py:SV_CASES
SV_CASES = {
    "sv_tiny_ragged3": ("tiny", 4, [(48000, 11, "speechlike"), (27200, 12, "noise"), (38437, 13, "speechlike")]),
    "sv_large_single": ("large", 1, [(160000, 14, "speechlike")]),
}


def load_sv_case(name):
    from funasr_b200 import synth
    cfg_name, wseed, specs = SV_CASES[name]
    cfg = synth.SENSEVOICE_TINY if cfg_name == "tiny" else synth.SENSEVOICE_SMALL
    gold = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    wavs = [synth.make_wav(n, s, k) for (n, s, k) in specs]
    cmvn = synth.make_cmvn(synth.PARAFORMER_LARGE, seed=1)
    cmvn = torch.tensor(np.array([[float("%.9g" % v) for v in row] for row in cmvn.tolist()], dtype=np.float32))
    return cfg, wseed, wavs, cmvn, gold


# ContextualParaformer golden cases — must match oracle/make_golden.py:CTX_CASES
CTX_CASES = {
    "ctx_tiny_ragged3": ("tiny", 6, [(48000, 21, "speechlike"), (27200, 22, "noise"), (38437, 23, "speechlike")], 5),
    "ctx_large_single": ("large", 2, [(240000, 24, "speechlike")], 32),
}


def load_ctx_case(name):
    from funasr_b200 import synth
    cfg_name, wseed, specs, n_hot = CTX_CASES[name]
    cfg = synth.PARAFORMER_TINY if cfg_name == "tiny" else synth.PARAFORMER_LARGE
    gold = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    wavs = [synth.make_wav(n, s, k) for (n, s, k) in specs]
    cmvn = synth.make_cmvn(cfg, seed=1)
    cmvn = torch.tensor(np.array([[float("%.9g" % v) for v in row] for row in cmvn.tolist()], dtype=np.float32))
    return cfg, wseed, wavs, cmvn, synth.make_hotwords(n_hot, cfg.vocab, seed=7), gold


# BiCifParaformer golden cases — must match oracle/make_golden.py:BICIF_CASES
BICIF_CASES = {
    "bicif_tiny_ragged3": ("tiny", 8, [(48000, 31, "speechlike"), (27200, 32, "noise"), (38437, 33, "speechlike")]),
    "bicif_large_single": ("large", 3, [(160000, 34, "speechlike")]),
}


def load_bicif_case(name):
    from funasr_b200 import synth
    cfg_name, wseed, specs = BICIF_CASES[name]
    cfg = synth.PARAFORMER_TINY if cfg_name == "tiny" else synth.PARAFORMER_LARGE
    gold = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    wavs = [synth.make_wav(n, s, k) for (n, s, k) in specs]
    cmvn = synth.make_cmvn(cfg, seed=1)
    cmvn = torch.tensor(np.array([[float("%.9g" % v) for v in row] for row in cmvn.tolist()], dtype=np.float32))
    return cfg, wseed, wavs, cmvn, gold


def gold_stamps(g):
    """[[[s, e], ...] per utterance] from the flat golden arrays."""
    out, pos = [], 0
    for n in g["stamps_len"].tolist():
        flat = g["stamps_flat"][pos: pos + 2 * n].tolist()
        out.append([[flat[2 * i], flat[2 * i + 1]] for i in range(n)])
        pos += 2 * n
    return out


# SeacoParaformer golden cases — must match oracle/make_golden.py:SEACO_CASES (name: cfg, weight seed, wavs, n hotwords, nfilter)
SEACO_CASES = {
    "seaco_tiny_ragged3": ("tiny", 10, [(48000, 41, "speechlike"), (27200, 42, "noise"), (38437, 43, "speechlike")], 6, 50),
    "seaco_tiny_asf": ("tiny", 11, [(40000, 44, "speechlike"), (30000, 45, "speechlike")], 24, 8),
}


def load_seaco_case(name):
    from funasr_b200 import synth
    cfg_name, wseed, specs, n_hot, nfilter = SEACO_CASES[name]
    cfg = synth.PARAFORMER_TINY if cfg_name == "tiny" else synth.PARAFORMER_LARGE
    gold = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    wavs = [synth.make_wav(n, s, k) for (n, s, k) in specs]
    cmvn = synth.make_cmvn(cfg, seed=1)
    cmvn = torch.tensor(np.array([[float("%.9g" % v) for v in row] for row in cmvn.tolist()], dtype=np.float32))
    return cfg, wseed, wavs, cmvn, synth.make_hotwords(n_hot, cfg.vocab, seed=9), nfilter, gold
