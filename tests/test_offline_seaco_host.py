"""SeacoParaformer in the C handle API, host side: the model file (pack.write_seaco_model_file), fa_offline_init's refusals of a bad
SeACo file before any device work, the attention-score filter's host selection (fa_seaco_asf_select_host) against torch, and the
hotword encoder's argument checks, which all run before a launch."""
import ctypes as C

import numpy as np
import pytest
import torch

from funasr_b200 import _abi, pack, synth

CFG = synth.PARAFORMER_TINY


def _seaco_state():
    return synth.make_seaco_state_dict(CFG, 10)


def test_seaco_model_file_round_trips(tmp_path):
    """Everything write_model_file writes (the BiCif head included), the SeACo decoder, hotword_output_layer, every bias_encoder
    tensor, the folded GEMM biases and __seaco_config__ [no_bias, nfilter, layers]."""
    st = _seaco_state()
    path = str(tmp_path / "seaco.fab2")
    pack.write_seaco_model_file(path, st, CFG, synth.make_cmvn(CFG, 1), no_bias=synth.seaco_no_bias_id(CFG), nfilter=8)
    t = pack.read_model_file(path)
    base = pack.model_tensors(st, CFG, synth.make_cmvn(CFG, 1))
    for k, v in base.items():
        assert np.array_equal(t[k], v), k
    assert "predictor.upsample_cnn.gemm_weight" in t and "__ts_config__" in t
    for k, v in st.items():
        if k.startswith(("seaco_decoder.", "hotword_output_layer.", "bias_encoder.", "decoder.embed.")):
            assert np.array_equal(t[k], v.float().numpy()), k
    for layer in (0, 1):
        want = (st["bias_encoder.bias_ih_l%d" % layer] + st["bias_encoder.bias_hh_l%d" % layer]).numpy()
        assert np.array_equal(t["bias_encoder.gemm_bias_l%d" % layer], want)
    assert t["__seaco_config__"].tolist() == [synth.seaco_no_bias_id(CFG), 8, 2]
    # write_model_file itself is unchanged: a SeACo state packed by it stays a BiCif file without the SeACo parts
    plain = str(tmp_path / "plain.fab2")
    pack.write_model_file(plain, st, CFG)
    p = pack.read_model_file(plain)
    assert "__seaco_config__" not in p and not any(k.startswith(("seaco_decoder.", "hotword_output_layer.")) for k in p)


def test_seaco_model_file_refusals(tmp_path):
    st = _seaco_state()
    bid = dict(st, **{"lstm_proj.weight": torch.zeros(512, 1024), "lstm_proj.bias": torch.zeros(512)})
    with pytest.raises(ValueError, match="bias_encoder_bid"):
        pack.write_seaco_model_file(str(tmp_path / "a.fab2"), bid, CFG)
    mean = {k: v for k, v in st.items() if not k.startswith("bias_encoder.")}
    mean["bias_embed.weight"] = torch.zeros(CFG.vocab, 512)
    with pytest.raises(ValueError, match="mean"):
        pack.write_seaco_model_file(str(tmp_path / "b.fab2"), mean, CFG)
    with pytest.raises(ValueError, match="no_bias"):
        pack.write_seaco_model_file(str(tmp_path / "c.fab2"), st, CFG, no_bias=CFG.vocab)


def _variant(tmp_path, name, edit):
    t = pack.seaco_model_tensors(_seaco_state(), CFG, None, no_bias=synth.seaco_no_bias_id(CFG), nfilter=8)
    edit(t)
    path = str(tmp_path / name)
    pack._write(path, t)
    return path


def test_handle_refuses_bad_seaco_files_before_any_device_work(tmp_path):
    """NULL and a message naming the piece, from the index pass (so the same with or without a GPU)."""
    lib = _abi.load()

    def drop(*names):
        return lambda t: [t.pop(n) for n in names]

    def put(name, arr):
        return lambda t: t.__setitem__(name, arr)

    cases = [("no_out.fab2", drop("hotword_output_layer.weight"), b"hotword_output_layer.weight"),
             ("hh1.fab2", put("bias_encoder.weight_hh_l1", np.zeros((2048, 256), np.float32)), b"bias_encoder.weight_hh_l1"),
             ("nobias.fab2", put("__seaco_config__", np.array([CFG.vocab, 8, 2], np.float32)), b"no_bias"),
             ("ctx.fab2", put("decoder.bias_decoder.norm3.weight", np.ones(512, np.float32)), b"bias_decoder"),
             ("emb.fab2", put("decoder.embed.0.weight", np.zeros((CFG.vocab, 256), np.float32)), b"decoder.embed.0.weight"),
             ("layers.fab2", drop(*[k for k in _seaco_state() if k.startswith("seaco_decoder.decoders.5.")]),
              b"seaco_decoder"),
             ("nfilter.fab2", put("__seaco_config__", np.array([100, -1, 2], np.float32)), b"nfilter"),
             ("cfg.fab2", put("__seaco_config__", np.array([100, 8], np.float32)), b"__seaco_config__"),
             ("l2.fab2", put("__seaco_config__", np.array([100, 8, 3], np.float32)), b"bias_encoder")]
    for name, edit, needle in cases:
        path = _variant(tmp_path, name, edit)
        assert not lib.fa_offline_init(path.encode(), 0, 3), name
        msg = lib.fa_offline_last_error()
        assert needle in msg and b"SeACo" in msg, (name, msg)
    # a well-formed file opens a handle, or fails only for the missing device
    ok = _variant(tmp_path, "ok.fab2", lambda t: None)
    h = lib.fa_offline_init(ok.encode(), 0, 3)
    if h:
        assert lib.fa_offline_is_seaco(h) == 1 and lib.fa_offline_has_timestamps(h) == 1
        lib.fa_offline_uninit(h)
    else:
        assert b"no such CUDA device" in lib.fa_offline_last_error()


def _asf_torch(p, nfilter):
    n = p.shape[2]
    return torch.topk(torch.from_numpy(p).sum(0).sum(0), min(nfilter, n - 1))[1].tolist() + [n - 1]


def _asf_native(p, nfilter):
    lib = _abi.load()
    out = np.full(p.shape[2], -7, np.int32)
    k = lib.fa_seaco_asf_select_host(np.ascontiguousarray(p).ctypes.data, p.shape[0], p.shape[1], p.shape[2], nfilter, out.ctypes.data)
    assert k == min(nfilter, p.shape[2] - 1) + 1
    return out[:k].tolist()


def test_asf_selection_equals_torch_on_random_cases():
    """2 200 cases, heads 1-8, rows 1-400, hotwords 2-600, nfilter 1 .. n - 1 (and above): softmax-like rows, and quantised rows whose
    scores tie exactly, so that torch.topk's order among equal scores (partial_sort for 64 k <= n, nth_element + sort otherwise) is
    restated too.  Both column paths of torch's outer-dimension sum (32-column cascade blocks, row_sum for the rest) are reached."""
    rng = np.random.default_rng(2024)
    for case in range(2200):
        H, R, N = int(rng.integers(1, 9)), int(rng.integers(1, 401)), int(rng.integers(2, 601))
        if case % 3 == 0:
            p = (rng.integers(0, 4, size=(H, R, N)) / 8).astype(np.float32)
        else:
            p = rng.random((H, R, N)).astype(np.float32) ** 3
            p /= p.sum(-1, keepdims=True)
        nfilter = int(rng.integers(1, N + 2)) if case % 5 else int(rng.integers(1, max(2, N // 64 + 1)))
        assert _asf_native(p, nfilter) == _asf_torch(p, nfilter), (case, H, R, N, nfilter)


def test_asf_selection_edges_and_refusals():
    p = np.zeros((4, 3, 5), np.float32)                     # all scores tie
    for nf in (1, 2, 4, 50):
        assert _asf_native(p, nf) == _asf_torch(p, nf)
    lib = _abi.load()
    out = np.zeros(8, np.int32)
    assert lib.fa_seaco_asf_select_host(None, 4, 3, 5, 2, out.ctypes.data) == -1
    assert lib.fa_seaco_asf_select_host(p.ctypes.data, 4, 3, 1, 2, out.ctypes.data) == -1
    assert lib.fa_seaco_asf_select_host(p.ctypes.data, 4, 3, 5, 0, out.ctypes.data) == -1
    assert lib.fa_seaco_asf_select_host(p.ctypes.data, 0, 3, 5, 2, out.ctypes.data) == -1
    assert lib.fa_seaco_asf_select_host(p.ctypes.data, 4, 3, 5, 2, None) == -1


def _fake_encoder(mode):
    """An encoder struct whose pointers are never read: every refusal below comes before the first launch."""
    fake = C.c_void_p(16)
    lin = lambda bias: _abi.FaLinear(fake, fake if bias else None, fake if mode else None, 2048, 512, 512, 0)   # noqa: E731
    ih, hh = (_abi.FaLinear * 2)(lin(True), lin(True)), (_abi.FaLinear * 2)(lin(False), lin(False))
    return _abi.FaHotwordEncoder(fake, 100, 2, ih, hh), (ih, hh)


@pytest.mark.parametrize("mode", [0, 3])
def test_hotword_encoder_refuses_before_any_launch(mode):
    lib = _abi.load()
    enc, _keep = _fake_encoder(mode)
    ids = np.array([5, 6, 7, 1], np.int32)
    lens = np.array([3, 1], np.int32)
    rows, ws = C.c_void_p(256), C.c_void_p(256)
    call = lambda e, i, ln, n, r=rows: lib.fa_hotword_encoder_forward(C.byref(e), i, ln, n, r, mode, ws, 1 << 30, None)   # noqa: E731
    l0 = lib.fa_launch_count()
    bad = ids.copy()
    bad[1] = 100                                            # one past the vocabulary
    assert call(enc, bad.ctypes.data, lens.ctypes.data, 2) == -1
    bad[1] = -1
    assert call(enc, bad.ctypes.data, lens.ctypes.data, 2) == -1
    assert call(enc, ids.ctypes.data, lens.ctypes.data, 0) == -1
    assert call(enc, None, lens.ctypes.data, 2) == -1 and call(enc, ids.ctypes.data, None, 2) == -1
    assert call(enc, ids.ctypes.data, lens.ctypes.data, 2, None) == -1
    zero = np.array([3, 0], np.int32)
    assert call(enc, ids.ctypes.data, zero.ctypes.data, 2) == -1
    assert lib.fa_hotword_encoder_forward(None, ids.ctypes.data, lens.ctypes.data, 2, rows, mode, ws, 1 << 30, None) == -1
    enc.n_layers = 0
    assert call(enc, ids.ctypes.data, lens.ctypes.data, 2) == -1
    enc.n_layers = 2
    assert lib.fa_hotword_encoder_forward(C.byref(enc), ids.ctypes.data, lens.ctypes.data, 2, rows, mode, ws, 16, None) == -3   # workspace
    assert lib.fa_launch_count() == l0
    need = lib.fa_hotword_encoder_workspace_bytes(2, 4, mode)
    assert need > 0 and lib.fa_hotword_encoder_workspace_bytes(0, 4, mode) == 0 and lib.fa_hotword_encoder_workspace_bytes(2, 1, mode) == 0
    assert lib.fa_hotword_encoder_workspace_bytes(2, 4000, mode) > need


def test_null_handles_and_arguments():
    lib = _abi.load()
    assert lib.fa_offline_is_seaco(None) == 0
    rows = np.zeros((1, 512), np.float32)
    ids, lens = np.array([5], np.int32), np.array([1], np.int32)
    assert lib.fa_offline_hotword_embed(None, ids.ctypes.data, lens.ctypes.data, 1, rows.ctypes.data) == -1
    assert b"bad argument" in lib.fa_offline_last_error()
