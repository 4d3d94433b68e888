"""GPU (-m gpu): fa_campplus_forward, the whole CAM++ forward of csrc/campplus.cu (FCM convs, TDNN GEMM, 52 CAM dense layers,
transits, statistics pooling, dense layer), against the float64 restatement tests/campplus_ref.py, per utterance, in every GEMM mode,
at the frame counts where the kernels change behaviour.

Inputs: features of synthetic voices (synth.make_voice_wav) made by fa_campplus_features (pinned to float64 by test_frontend_gpu.py),
copied to the host, and the fixtures' stored chunk features; the library and the restatement take the same float32 features.  Real
features matter: the fixtures' BatchNorm statistics were calibrated on real chunks, and i.i.d. noise drives the activations elsewhere.

Metric: per utterance, err = max_c |got - ref| / max_c |ref| over the 192 outputs (campplus_ref.emb_err); 1 - cos(got, ref), what the
clustering consumes, is reported next to it.  Each split-mode case also reruns its inputs in single-plane fp16 and requires that
output to miss the fp16x3 bar by 10 x or more: a bar that a lost operand plane could pass is too loose.

BARS: at most 4 x the worst error measured over all cases of a mode on an NVIDIA H100 80GB HBM3 (700 W power limit); MEASURED holds
those worst values.  Every case prints its worst utterance with -s.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from campplus_ref import campplus_ref, emb_err
from test_spk_host import SPK_CASES, campplus_state_dict, load_spk_case

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MODES = ["fp32", "fp16", "fp16x3", "fp16x6"]
SPLIT = ("fp16x3", "fp16x6")

# Worst per mode over every case below, on an NVIDIA H100 80GB HBM3 at its 700 W power limit (worst case in brackets).  The fp32
# bar is 4 x its worst.  The split-mode bars sit at 1.9 - 2 x: 4 x would let single-plane fp16 come within 10 x of them (its
# smallest error, 1.44e-3 at T18800, is 10.3 x the fp16x3 bar).  fp16x6 measures like fp16x3: the FCM convs, the CAM layers and
# the statistics pooling run in fp32 in every mode, and what the GEMMs' third A plane adds sits below their fp32 accumulation.
# 1 - cos, what the clustering sees, stays below 1.4e-10 (fp32), 5e-5 (fp16) and 1.1e-9 (fp16x3, fp16x6).
MEASURED = {"fp32": 2.31e-5,      # spk_three_preset
            "fp16": 1.08e-2,      # T201
            "fp16x3": 7.21e-5,    # T202
            "fp16x6": 6.87e-5}    # T202
BARS = {"fp32": 9.2e-5, "fp16": 4.3e-2, "fp16x3": 1.4e-4, "fp16x6": 1.4e-4}

# name: (T feature frames, batch); t_out = (T - 1) // 2 + 1 TDNN frames, CAM segments of 100 TDNN frames
CASES = {
    "T3": (3, 4),            # t_out 2: the smallest valid inputs, odd and even padded pitch P = (T + 5) // 2 * 2
    "T4": (4, 4),
    "T5": (5, 4),            # t_out 3
    "T148_B1": (148, 1),     # the diarization chunk (1.5 s, t_out 74)
    "T148_B17": (148, 17),
    "T148_B64": (148, 64),
    "T199": (199, 2),        # t_out 100: exactly one full segment
    "T200": (200, 2),
    "T201": (201, 2),        # t_out 101: a one-frame last segment
    "T202": (202, 2),
    "T401": (401, 2),        # t_out 201: three segments
    "T3000": (3000, 2),      # 30 s
    "T18800": (18800, 1),    # t_out 9 400, 94 segments: the longest input the forward takes
}
FIXTURES = list(SPK_CASES)   # their 4 stored chunk features each (T = 148)


def _st(stream=None):
    return (stream or torch.cuda.current_stream()).cuda_stream


_ENG, _FEATS, _REF, _SD = {}, {}, {}, {}


def _engine(mode):
    if mode not in _ENG:
        from funasr_b200.campplus import CampplusEngine
        _ENG[mode] = CampplusEngine(campplus_state_dict(), DEV, mode)
    return _ENG[mode]


def _voice_feats(T, B):
    """[B, T, 80] float32 on the host: fa_campplus_features of B synthetic recordings, voices alternating in 2 s bursts."""
    from funasr_b200 import synth
    n = 400 + 160 * (T - 1)
    wavs = []
    for b in range(B):
        pattern, dur = [], 0.0
        while dur * 16000 < n + 800 * b:
            pattern.append(((b + len(pattern)) % 3, 2.0, 0.3))
            dur += 2.3
        w = synth.make_voice_wav(pattern, 100 * T + b, lead_s=0.0)
        wavs.append(w[800 * b:800 * b + n])
    eng = _engine("fp32")
    wav = torch.stack(wavs).float().contiguous().to(DEV)
    feats, flens = eng.features(wav, torch.full((B,), n, dtype=torch.int32, device=DEV), T)
    assert flens.tolist() == [T] * B
    return feats.cpu()


def _feats(name):
    if name not in _FEATS:
        _FEATS[name] = torch.from_numpy(load_spk_case(name)["features"]) if name in SPK_CASES else _voice_feats(*CASES[name])
    return _FEATS[name]


def _ref(name):
    if name not in _REF:
        if not _SD:
            _SD["sd"] = campplus_state_dict()
        _REF[name] = campplus_ref(_SD["sd"], _feats(name)).numpy()
    return _REF[name]


def _run(eng, feats, stream=None):
    """fa_campplus_forward in a workspace of exactly the queried size -> [B, 192] on the host."""
    lib = eng.lib
    B, T, _ = feats.shape
    emb = torch.full((B, 192), float("nan"), device=DEV)
    ws = torch.empty(int(lib.fa_campplus_workspace_bytes(C.byref(eng.model), B, T, eng.mode)), dtype=torch.uint8, device=DEV)
    fd = feats.contiguous().to(DEV)
    torch.cuda.synchronize()
    rc = lib.fa_campplus_forward(C.byref(eng.model), fd.data_ptr(), B, T, emb.data_ptr(), eng.mode, ws.data_ptr(), ws.numel(), _st(stream))
    torch.cuda.synchronize()
    assert rc == 0
    return emb.cpu()


def _err(name, mode):
    return emb_err(_run(_engine(mode), _feats(name)), _ref(name))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(CASES) + FIXTURES)
def test_embeddings_vs_float64(name, mode):
    rel, cos = _err(name, mode)
    b = int(np.argmax(rel))
    print("MEASURED campplus %s %s %.3e  worst utt %d of %d, 1 - cos %.2e (worst 1 - cos %.2e)" % (
        mode, name, rel[b], b, rel.shape[0], cos[b], cos.max()))
    assert rel.max() <= BARS[mode]
    if mode in SPLIT:
        e16 = float(_err(name, "fp16")[0].max())
        bar = BARS["fp16x3"]
        print("TEETH campplus %s fp16 %.3e = %.1f x the fp16x3 bar %.1e" % (name, e16, e16 / bar, bar))
        assert e16 >= 10 * bar, "fp16 passes within 10 x of the fp16x3 bar: the bar cannot see a lost plane"


@pytest.mark.parametrize("mode", MODES)
def test_two_frames_give_nan_like_the_reference(mode):
    """T = 2: one TDNN frame, whose unbiased std over time is 0 / 0.  The reference's StatsPool (x.std(unbiased=True)) gives NaN
    there, and the dense layer spreads it to all 192 outputs; the forward does the same, in every mode."""
    feats = _voice_feats(2, 3)
    ref = campplus_ref(campplus_state_dict(), feats).numpy()
    got = _run(_engine(mode), feats).numpy()
    assert np.isnan(ref).all()
    assert np.array_equal(np.isnan(got), np.isnan(ref))


@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_longer_than_18800_frames_is_refused_before_any_launch(mode):
    """T = 18 801 would need a 95th CAM segment: the workspace query returns 0, the forward returns FA_ERR_UNSUPPORTED with nothing
    enqueued even given more workspace than any such input needs, and the engine names the limit."""
    from funasr_b200 import _abi
    eng = _engine(mode)
    lib = eng.lib
    T = 18801
    assert lib.fa_campplus_workspace_bytes(C.byref(eng.model), 1, T, eng.mode) == 0
    ws = torch.empty(2 * int(lib.fa_campplus_workspace_bytes(C.byref(eng.model), 1, T - 1, eng.mode)), dtype=torch.uint8, device=DEV)
    feats = torch.zeros(1, T, 80, device=DEV)
    emb = torch.empty(1, 192, device=DEV)
    torch.cuda.synchronize()
    n0 = lib.fa_launch_count()
    rc = lib.fa_campplus_forward(C.byref(eng.model), feats.data_ptr(), 1, T, emb.data_ptr(), eng.mode, ws.data_ptr(), ws.numel(), _st())
    torch.cuda.synchronize()
    assert rc == -4 and lib.fa_launch_count() == n0
    with pytest.raises(_abi.FunasrB200Error, match="2 ... 18800 feature frames"):
        eng.embed_feats(feats)
    assert lib.fa_launch_count() == n0


@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("T", [148, 201])
def test_chunks_are_independent_and_runs_repeat(T, mode):
    """A batch of 17: every chunk run alone equals its row of the batch, bit for bit (nothing crosses chunks: FCM time padding, the
    TDNN view's zero rows, CAM halos and segment means, statistics pooling); a second run and a run on another stream are
    bit-identical; embed_feats with its workspace cap lowered so that the batch runs in slices of 5 equals one call."""
    eng = _engine(mode)
    feats = _voice_feats(T, 17)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    out = _run(eng, feats, s1)
    assert not torch.isnan(out).any()
    assert torch.equal(_run(eng, feats, s2), out)
    assert torch.equal(_run(eng, feats, s1), out)
    for b in range(17):
        assert torch.equal(_run(eng, feats[b:b + 1])[0], out[b]), b
    per = int(eng.lib.fa_campplus_workspace_bytes(C.byref(eng.model), 1, T, eng.mode))
    eng.WORKSPACE_CAP = 5 * per + per // 2
    try:
        fd = feats.to(DEV)
        sliced = eng.embed_feats(fd)
        del eng.WORKSPACE_CAP
        whole = eng.embed_feats(fd)
    finally:
        eng.__dict__.pop("WORKSPACE_CAP", None)
    torch.cuda.synchronize()
    assert torch.equal(sliced.cpu(), out) and torch.equal(whole.cpu(), out)
