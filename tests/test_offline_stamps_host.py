"""CPU: the timestamp side of the handle API — the native stamp routine (fa_ts_stamps_host) against its Python specification
(timestamps.ts_prediction_lfr6_standard, stamps only), the BiCifParaformer model file (the repacked timestamp head and __ts_config__),
and the handle's refusals of incomplete heads, which need no GPU."""
import ctypes as C
import json
import os

import numpy as np
import torch

from conftest import GOLDEN

from funasr_b200 import _abi, pack, synth
from funasr_b200 import timestamps as TS

HEAD_NAMES = ("predictor.upsample_cnn.gemm_weight", "predictor.upsample_cnn.gemm_bias", "predictor.blstm.ih_gemm_weight",
              "predictor.blstm.ih_gemm_bias", "predictor.blstm.weight_hh_l0", "predictor.blstm.weight_hh_l0_reverse",
              "predictor.cif_output2.weight", "predictor.cif_output2.bias")


def _native(first, second, n_tokens, upsample_rate=3, vad_offset=0.0, max_out=None):
    a = np.ascontiguousarray(first, np.float32)
    p = np.ascontiguousarray(second, np.float32)
    assert a.size == p.size
    cap = max(a.size, 1) if max_out is None else max_out
    out = np.zeros((max(cap, 1), 2), np.int32)
    k = _abi.load().fa_ts_stamps_host(a.ctypes.data, p.ctypes.data, a.size, n_tokens, upsample_rate, float(vad_offset), out.ctypes.data, cap)
    assert k >= 0
    return out[: min(k, cap)].tolist(), k


def _python(first, second, n_tokens, **kw):
    return TS.ts_prediction_lfr6_standard(first, second, ["c%d" % i for i in range(n_tokens)], want_text=False, **kw)[1]


def test_native_stamps_equal_the_python_routine_on_the_reference_golden():
    """Every case of tests/golden/timestamps.json (made by the reference's own ts_prediction_lfr6_standard): the token count without a
    trailing </s> (the Python routine pops it), upsample rates 1 and 3, VAD offsets."""
    with open(os.path.join(GOLDEN, "timestamps.json")) as f:
        cases = json.load(f)
    n = 0
    for c in cases:
        chars = list(c["chars"])
        assert "<sil>" not in chars
        if not chars:
            assert _native(c["first"], c["second"], 0)[0] == [] == c["res"]
            continue
        n_tok = len(chars) - (chars[-1] == "</s>")
        got, k = _native(c["first"], c["second"], n_tok, c["upsample_rate"], c["vad_offset"])
        want = TS.ts_prediction_lfr6_standard(np.array(c["first"], np.float32), np.array(c["second"], np.float32), chars,
                                              vad_offset=c["vad_offset"], upsample_rate=c["upsample_rate"], want_text=False)[1]
        assert got == want == c["res"] and k == len(want)
        n += 1
    assert n >= 100


def test_native_stamps_equal_the_python_routine_on_random_cases():
    """2 400 random utterances over every regime of the routine: fire count equal to tokens + 1 or not (re-integration, with the
    weights' fp32 sum in numpy's order up to 12 000 frames), all-zero weights, no fire at all, a token cut at 12 frames as the last
    span, and both trailing-edge rules; the stamp count on its own when it is not the token count."""
    rng = np.random.default_rng(2024)
    seen = dict(reint=0, zero=0, no_fire=0, cut_last=0, edge_mid=0, edge_end=0, count_ne_tokens=0)
    for trial in range(2400):
        T = int(rng.integers(1, 600)) if trial % 10 else int(rng.integers(600, 12000))
        dens = float(rng.choice([0.02, 0.1, 0.3, 0.6]))
        a = (rng.random(T) ** int(rng.choice([1, 2])) * np.float32(2 * dens)).astype(np.float32)
        if trial % 7 == 0:
            a[: T // 3] = 0
        if trial % 5 == 0:
            a[-(T // 4):] = 0
        if trial % 11 == 0 and T > 60:
            a[-40:] = 0
            a[-41] = 1.0                                      # a fire followed by a long gap: the last span is cut at 12 frames
        if trial % 17 == 0:
            a[:] = 0
        peaks = TS.cif_wo_hidden(a, 1.0)
        n_fire = int((peaks >= np.float32(1 - 1e-4)).sum())
        n_tok = max(1, n_fire - 1 + int(rng.integers(-3, 4)) * int(trial % 3 == 0))
        off = float(rng.choice([0.0, 0.0, 130.0, 12340.0]))
        rate = int(rng.choice([3, 3, 1]))
        for first, second in ((a, peaks), (peaks, a)):        # the BiCif call order and the Paraformer one
            want = _python(first, second, n_tok, vad_offset=off, upsample_rate=rate)
            got, k = _native(first, second, n_tok, rate, off)
            assert got == want and k == len(want), (trial, T, n_tok)
        seen["reint"] += n_fire != n_tok + 1
        seen["zero"] += not a.any()
        seen["no_fire"] += not want
        seen["count_ne_tokens"] += bool(want) and len(want) != n_tok
        fires = np.flatnonzero(peaks >= np.float32(1 - 1e-4))
        if n_fire == n_tok + 1 and fires.size >= 2:
            last = fires[-1] - 1.5
            seen["cut_last"] += fires[-1] - fires[-2] > 12
            seen["edge_mid"] += fires[-1] - fires[-2] <= 12 and T - last > 5
            seen["edge_end"] += fires[-1] - fires[-2] <= 12 and T - last <= 5
    assert all(v > 5 for v in seen.values()), seen
    # out is bounded by max_out; the count is returned whole
    a = np.full(60, 0.5, np.float32)
    full, k = _native(a, TS.cif_wo_hidden(a, 1.0), 29)
    part, k2 = _native(a, TS.cif_wo_hidden(a, 1.0), 29, max_out=3)
    assert k == k2 == len(full) and part == full[:3]


def _bicif_state():
    return synth.make_bicif_state_dict(synth.PARAFORMER_TINY, 8)


def test_bicif_model_file_round_trips_the_head(tmp_path):
    cfg = synth.PARAFORMER_TINY
    st = _bicif_state()
    path = str(tmp_path / "bicif.fab2")
    pack.write_model_file(path, st, cfg, synth.make_cmvn(cfg, 1), smooth_factor2=0.3, noise_threshold2=0.02)
    back = pack.read_model_file(path)
    head = pack.timestamp_head_tensors(st)
    assert set(head) == set(HEAD_NAMES)
    for k in HEAD_NAMES:
        assert back[k].dtype == np.float32 and back[k].shape == tuple(head[k].shape) and np.array_equal(back[k], head[k].numpy()), k
    assert back["__ts_config__"].tolist() == [3.0, float(np.float32(0.3)), float(np.float32(0.02))]
    assert back["__config__"].shape == (10,)
    # the repack itself: W[k*512 + o, c] = w[c, o, k], the bias repeated 3x, both input projections stacked with b_ih + b_hh
    uw = st["predictor.upsample_cnn.weight"].numpy()
    W = back["predictor.upsample_cnn.gemm_weight"]
    assert W.shape == (1536, 512) and np.array_equal(W[512 * 2 + 7], uw[:, 7, 2])
    assert np.array_equal(back["predictor.upsample_cnn.gemm_bias"], np.tile(st["predictor.upsample_cnn.bias"].numpy(), 3))
    assert np.array_equal(back["predictor.blstm.ih_gemm_weight"][2048:], st["predictor.blstm.weight_ih_l0_reverse"].numpy())
    assert np.array_equal(back["predictor.blstm.ih_gemm_bias"][:2048],
                          st["predictor.blstm.bias_ih_l0"].numpy() + st["predictor.blstm.bias_hh_l0"].numpy())
    for k, v in st.items():                                   # every state tensor under its own name, unchanged
        assert np.array_equal(back[k], v.numpy()), k


def test_engine_head_struct_holds_the_packers_tensors():
    """The engine's timestamp head (fp32 mode needs no device for its weights) holds exactly the tensors the model file holds."""
    from funasr_b200.engine import _EngineBase
    st = _bicif_state()
    e = _EngineBase()
    e._init_base(st, "cpu", "fp32", 1e-12)
    e._init_timestamp_head("predictor.", 0.25, 0.01, 1.0)
    kept = {t.data_ptr(): t for t in e._keep}
    head = pack.timestamp_head_tensors(st)
    h = e.ts_head
    assert h.up_times == 3
    used = {"predictor.upsample_cnn.gemm_weight": h.upsample.w, "predictor.upsample_cnn.gemm_bias": h.upsample.b,
            "predictor.blstm.ih_gemm_weight": h.blstm_ih.w, "predictor.blstm.ih_gemm_bias": h.blstm_ih.b,
            "predictor.blstm.weight_hh_l0": h.w_hh_fwd, "predictor.blstm.weight_hh_l0_reverse": h.w_hh_bwd,
            "predictor.cif_output2.weight": h.out2_w, "predictor.cif_output2.bias": h.out2_b}
    for k, ptr in used.items():
        assert torch.equal(kept[ptr].reshape(head[k].shape), head[k]), k
    assert (h.upsample.out_f, h.upsample.in_f, h.blstm_ih.out_f, h.blstm_ih.in_f) == (1536, 512, 4096, 512)
    assert (h.smooth2, h.noise2, h.threshold) == (0.25, np.float32(0.01), 1.0)


def test_plain_paraformer_file_is_unchanged():
    cfg = synth.PARAFORMER_TINY
    st = synth.make_state_dict(cfg, 3)
    t = pack.model_tensors(st, cfg, synth.make_cmvn(cfg, 1))
    want = ["__config__", "frontend.mel_banks", "frontend.window", "frontend.cmvn", "encoder.pe_inv_timescales"] + \
        [k for k in st if k.startswith(("encoder.", "predictor.", "decoder."))] + ["predictor.cif_conv1d.gemm_weight"]
    assert list(t) == want
    for k in st:
        assert np.array_equal(t[k], st[k].numpy())


def _write_variant(tmp_path, name, edit):
    cfg = synth.PARAFORMER_TINY
    t = pack.model_tensors(_bicif_state(), cfg, None)
    edit(t)
    path = str(tmp_path / name)
    pack._write(path, t)
    return path


def test_handle_refuses_incomplete_heads_before_any_device_work(tmp_path):
    """A head without __ts_config__ (a file packed before the handle read the head), with a missing or misshapen tensor, or with an
    upsampling factor other than 3: NULL and a message that names the piece, with or without a GPU."""
    lib = _abi.load()

    def drop(*names):
        return lambda t: [t.pop(n) for n in names]

    def set_cfg(v):
        return lambda t: t.__setitem__("__ts_config__", np.array(v, np.float32))

    old = {k: v for k, v in pack.model_tensors(_bicif_state(), synth.PARAFORMER_TINY, None).items()
           if k != "__ts_config__" and "gemm" not in k or k == "predictor.cif_conv1d.gemm_weight"}
    cases = [("old.fab2", lambda t: (t.clear(), t.update(old)), b"__ts_config__"),
             ("no_cfg.fab2", drop("__ts_config__"), b"__ts_config__"),
             ("no_ih.fab2", drop("predictor.blstm.ih_gemm_bias"), b"predictor.blstm.ih_gemm_bias"),
             ("no_hh.fab2", drop("predictor.blstm.weight_hh_l0_reverse"), b"predictor.blstm.weight_hh_l0_reverse"),
             ("no_out2.fab2", drop("predictor.cif_output2.weight"), b"predictor.cif_output2.weight"),
             ("shape.fab2", lambda t: t.__setitem__("predictor.upsample_cnn.gemm_weight", np.zeros((512, 512), np.float32)),
              b"predictor.upsample_cnn.gemm_weight"),
             ("up5.fab2", set_cfg([5, 0.25, 0.01]), b"upsample_times"),
             ("short_cfg.fab2", set_cfg([3]), b"__ts_config__")]
    for name, edit, needle in cases:
        path = _write_variant(tmp_path, name, edit)
        assert not lib.fa_offline_init(path.encode(), 0, 3), name
        msg = lib.fa_offline_last_error()
        assert needle in msg and b"timestamp head" in msg, (name, msg)


def test_null_results_handles_and_arguments():
    lib = _abi.load()
    assert lib.fa_offline_has_timestamps(None) == 0
    n = C.c_int32(7)
    assert not lib.fa_offline_result_stamps(None, 0, C.byref(n)) and n.value == 0
    assert not lib.fa_offline_result_stamps(None, -1, None)
    x = np.zeros(4, np.float32)
    out = np.zeros(8, np.int32)
    assert lib.fa_ts_stamps_host(None, None, 4, 2, 3, 0.0, out.ctypes.data, 4) == -1
    assert lib.fa_ts_stamps_host(x.ctypes.data, x.ctypes.data, 4, 2, 0, 0.0, out.ctypes.data, 4) == -1
    assert lib.fa_ts_stamps_host(x.ctypes.data, x.ctypes.data, 4, -1, 3, 0.0, out.ctypes.data, 4) == -1
    assert lib.fa_ts_stamps_host(x.ctypes.data, x.ctypes.data, 4, 2, 3, 0.0, None, 4) == -1
    assert lib.fa_ts_stamps_host(x.ctypes.data, x.ctypes.data, 4, 2, 3, 0.0, None, 0) == 0      # all-zero weights: nothing fires
    assert lib.fa_ts_stamps_host(None, None, 0, 0, 3, 0.0, None, 0) == 0
