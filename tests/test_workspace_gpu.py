"""Every entry point that takes a caller workspace, on every path and GEMM mode it supports, run in a buffer of exactly the size its
query returns: the call succeeds, and its outputs do not depend on what the workspace held before (a buffer the carve dropped
cannot be read before it is written).  The same buffer passed as one byte shorter is refused with FA_ERR_WORKSPACE before anything
is enqueued."""
import ctypes as C

import pytest
import torch

from test_spk_host import campplus_state_dict

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MODES = ["fp32", "fp16", "fp16x3", "fp16x6"]
TC_MODES = MODES[1:]
FA_ERR_WORKSPACE = -3


def _st():
    return torch.cuda.current_stream().cuda_stream


def _lib():
    from funasr_b200 import _abi
    return _abi.load()


def _check(need, call, outputs, refuses_short=True):
    """call(ws_ptr, ws_bytes) -> status.  (a) exactly `need` bytes pre-filled with 0x00, then with 0x3C (finite in fp16 and fp32):
    FA_OK and bit-identical outputs.  (b) the same buffer as need - 1 bytes: FA_ERR_WORKSPACE, and no launch (refuses_short=False
    where the query is an upper bound over a selector it cannot see)."""
    lib = _lib()
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    ptr = ws.data_ptr() if need else None
    runs = []
    for fill in (0x00, 0x3C):
        ws.fill_(fill)
        for o in outputs:
            o.zero_()
        assert call(ptr, need) == 0, fill
        torch.cuda.synchronize()
        runs.append([o.clone() for o in outputs])
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    if need > 0 and refuses_short:
        n0 = lib.fa_launch_count()
        assert call(ptr, need - 1) == FA_ERR_WORKSPACE
        assert lib.fa_launch_count() == n0


_STATES = {}


def _state(kind):
    from funasr_b200 import synth
    if kind not in _STATES:
        cfg = synth.PARAFORMER_TINY
        make = {"plain": synth.make_state_dict, "contextual": synth.make_contextual_state_dict, "bicif": synth.make_bicif_state_dict,
                "seaco": synth.make_seaco_state_dict}
        if kind == "aligner":
            _STATES[kind] = synth.make_aligner_state_dict(synth.ALIGNER_TINY, 3)
        elif kind == "sensevoice":
            _STATES[kind] = synth.make_sensevoice_state_dict(synth.SENSEVOICE_TINY, 3)
        else:
            _STATES[kind] = make[kind](cfg, 3)
    return _STATES[kind]


def _engine(kind, mode):
    from funasr_b200 import synth
    from funasr_b200.engine import AlignerEngine, ParaformerEngine, SenseVoiceEngine
    if kind == "aligner":
        return AlignerEngine(_state(kind), synth.ALIGNER_TINY, DEV, gemm_mode=mode)
    if kind == "sensevoice":
        return SenseVoiceEngine(_state(kind), synth.SENSEVOICE_TINY, DEV, gemm_mode=mode)
    cfg = synth.PARAFORMER_TINY
    return ParaformerEngine(_state(kind), cfg, DEV, gemm_mode=mode, contextual=kind == "contextual", bicif=kind == "bicif",
                            seaco=kind == "seaco", no_bias=synth.seaco_no_bias_id(cfg))


def _randn(*shape, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, generator=g, device=DEV)


B, T, N = 3, 37, 9
LENS = [37, 20, 29]


def _lens(vals):
    return torch.tensor(vals, dtype=torch.int32, device=DEV)


# ------------------------------------------------------------------------------------------------ encoder
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", ["pe", "plain_stack", "aligner"])
def test_encoder_workspace(kind, mode):
    from funasr_b200 import _abi
    lib = _lib()
    eng = _engine({"pe": "plain", "plain_stack": "sensevoice", "aligner": "aligner"}[kind], mode)
    enc = eng.tp if kind == "plain_stack" else eng.enc
    d = 320 if kind == "aligner" else 512
    feats = _randn(B, T, 512 if kind == "plain_stack" else 560, seed=1)
    lens = _lens(LENS)
    out = torch.empty(B, T, d, device=DEV)
    need = lib.fa_sanm_encoder_workspace_bytes(B, T, _abi.GEMM_MODES[mode])
    _check(need, lambda p, n: lib.fa_sanm_encoder_forward(C.byref(enc), feats.data_ptr(), lens.data_ptr(), B, T, out.data_ptr(),
                                                          eng.mode, p, n, _st()), [out])


# ---------------------------------------------------------------------------------------------- predictor
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", ["v2", "v3"])
def test_predictor_workspace(kind, mode):
    lib = _lib()
    eng = _engine("plain" if kind == "v2" else "bicif", mode)
    enc = _randn(B, T, 512, seed=2)
    lens = _lens(LENS)
    acoustic, tok = torch.empty(B, T + 1, 512, device=DEV), torch.empty(B, dtype=torch.int32, device=DEV)
    alphas, peaks = torch.empty(B, T + 1, device=DEV), torch.empty(B, T + 1, device=DEV)
    need = lib.fa_cif_predictor_workspace_bytes(B, T, eng.mode)
    _check(need, lambda p, n: lib.fa_cif_predictor_forward(C.byref(eng.pred), enc.data_ptr(), lens.data_ptr(), B, T, acoustic.data_ptr(),
                                                           T + 1, tok.data_ptr(), alphas.data_ptr(), peaks.data_ptr(), eng.mode, p, n,
                                                           _st()), [acoustic, tok, alphas, peaks])


# ------------------------------------------------------------------------------------------------ decoder
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", ["plain", "contextual", "hidden"])
def test_decoder_workspace(kind, mode):
    lib = _lib()
    eng = _engine("contextual" if kind == "contextual" else "plain", mode)
    V = eng.cfg.vocab
    enc = _randn(B, T, 512, seed=3)
    acoustic = _randn(B, N + 2, 512, seed=4)
    enc_lens, tok = _lens(LENS), _lens([9, 4, 7])
    nh = 0
    if kind == "contextual":
        nh = 5
        hw = _randn(nh, 512, seed=5)
        hw_lens = _lens([nh] * B)
        eng.dec.has_bias, eng.dec.n_hotwords, eng.dec.hw_embed, eng.dec.hw_lens = 1, nh, hw.data_ptr(), hw_lens.data_ptr()
    ids, best = torch.empty(B, N, dtype=torch.int32, device=DEV), torch.empty(B, N, device=DEV)
    logits = torch.empty(B, N, V, device=DEV)
    hidden = torch.empty(B, N, 512, device=DEV)
    need = lib.fa_paraformer_decoder_workspace_bytes_hw(B, T, N, V, eng.mode, nh)
    args = (C.byref(eng.dec), enc.data_ptr(), enc_lens.data_ptr(), B, T, acoustic.data_ptr(), N + 2, tok.data_ptr(), N, ids.data_ptr(),
            best.data_ptr(), logits.data_ptr(), 1)
    if kind == "hidden":
        _check(need, lambda p, n: lib.fa_paraformer_decoder_forward_hidden(*args, hidden.data_ptr(), eng.mode, p, n, _st()),
               [ids, best, logits, hidden])
    else:
        _check(need, lambda p, n: lib.fa_paraformer_decoder_forward(*args, eng.mode, p, n, _st()), [ids, best, logits])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", ["finish", "attn_probs"])
def test_decoder_stack_workspace(kind, mode):
    lib = _lib()
    eng = _engine("seaco", mode)
    dec = eng.seaco_dec
    t_mem = 6
    memory = _randn(t_mem, 512, seed=6)
    x = _randn(B, N, 512, seed=7)
    mem_lens, tok = _lens([t_mem] * B), _lens([9, 4, 7])
    hidden = torch.empty(B, N, 512, device=DEV)
    probs = torch.empty(dec.heads, N, t_mem, device=DEV)
    need = lib.fa_sanm_decoder_stack_workspace_bytes(B, t_mem, N, eng.mode)
    if kind == "finish":
        outs, h, pr = [hidden], hidden.data_ptr(), None
    else:
        outs, h, pr = [probs], None, probs.data_ptr()
    _check(need, lambda p, n: lib.fa_sanm_decoder_stack_forward(C.byref(dec), memory.data_ptr(), mem_lens.data_ptr(), 1, B, t_mem, x.data_ptr(),
                                                                N, tok.data_ptr(), N, dec.n_layers, 1 if kind == "finish" else 0, h, pr,
                                                                eng.mode, p, n, _st()), outs)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", ["bicif", "aligner"])
def test_timestamp_head_workspace(kind, mode):
    lib = _lib()
    eng = _engine(kind, mode)
    d = 320 if kind == "aligner" else 512
    enc = _randn(B, T, d, seed=20)
    lens, tok = _lens(LENS), _lens([9, 4, 7])
    us_alphas, us_peaks = torch.empty(B, 3 * T, device=DEV), torch.empty(B, 3 * T, device=DEV)
    need = lib.fa_timestamp_head_workspace_bytes(B, T, d, 3, eng.mode)
    _check(need, lambda p, n: lib.fa_timestamp_head_forward(C.byref(eng.ts_head), enc.data_ptr(), lens.data_ptr(), tok.data_ptr(), B, T,
                                                            us_alphas.data_ptr(), us_peaks.data_ptr(), eng.mode, p, n, _st()),
           [us_alphas, us_peaks])


# ------------------------------------------------------------------------------------------- output heads
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("with_b", [False, True])
def test_linear_argmax_workspace(with_b, mode):
    lib = _lib()
    eng = _engine("seaco", mode)
    rows, V = B * N, eng.cfg.vocab
    a, b = _randn(rows, 512, seed=8), _randn(rows, 512, seed=9)
    ids, best, logp = torch.empty(rows, dtype=torch.int32, device=DEV), torch.empty(rows, device=DEV), torch.empty(rows, V, device=DEV)
    need = lib.fa_linear_argmax_workspace_bytes(rows, V, eng.mode)
    _check(need, lambda p, n: lib.fa_linear_argmax(C.byref(eng.hw_out), a.data_ptr(), b.data_ptr() if with_b else None, rows, ids.data_ptr(),
                                                   best.data_ptr(), logp.data_ptr(), eng.mode, p, n, _st()), [ids, best, logp])


@pytest.mark.parametrize("mode", MODES)
def test_ctc_workspace(mode):
    lib = _lib()
    eng = _engine("sensevoice", mode)
    V = eng.ctc.out_f
    enc = _randn(B, T, 512, seed=10)
    lens = _lens(LENS)
    am = torch.empty(B, T, dtype=torch.int32, device=DEV)
    out_ids, out_lens = torch.empty(B, T, dtype=torch.int32, device=DEV), torch.empty(B, dtype=torch.int32, device=DEV)
    need = lib.fa_ctc_greedy_workspace_bytes(B, T, V, eng.mode)
    _check(need, lambda p, n: lib.fa_ctc_greedy_forward(C.byref(eng.ctc), enc.data_ptr(), lens.data_ptr(), B, T, 0, am.data_ptr(),
                                                        out_ids.data_ptr(), out_lens.data_ptr(), None, eng.mode, p, n, _st()),
           [am, out_ids, out_lens])


# ------------------------------------------------------------------------------------------- VAD, CAM++
def test_vad_workspace():
    from funasr_b200 import synth
    from funasr_b200.vad_model import VadEngine
    lib = _lib()
    eng = VadEngine(synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), DEV, synth.make_vad_cmvn(0))
    t = 301
    feats = _randn(t, 400, seed=11)
    sil = torch.empty(t, device=DEV)
    scores = torch.empty(t, eng.enc.out2.out_f, device=DEV)
    need = lib.fa_fsmn_vad_workspace_bytes(C.byref(eng.enc), t)
    _check(need, lambda p, n: lib.fa_fsmn_vad_forward(C.byref(eng.enc), feats.data_ptr(), 400, t, sil.data_ptr(), scores.data_ptr(), p, n,
                                                      _st()), [sil, scores])


@pytest.mark.parametrize("mode", MODES)
def test_campplus_workspace(mode):
    from funasr_b200.campplus import CampplusEngine
    lib = _lib()
    eng = CampplusEngine(campplus_state_dict(), DEV, mode)
    b, t = 2, 148
    feats = _randn(b, t, 80, seed=12)
    emb = torch.empty(b, 192, device=DEV)
    need = lib.fa_campplus_workspace_bytes(C.byref(eng.model), b, t, eng.mode)
    _check(need, lambda p, n: lib.fa_campplus_forward(C.byref(eng.model), feats.data_ptr(), b, t, emb.data_ptr(), eng.mode, p, n, _st()), [emb])


# ------------------------------------------------------------------------------------------- op level
@pytest.mark.parametrize("mode", TC_MODES)
def test_attention_tc_workspace(mode):
    from funasr_b200 import _abi
    lib = _lib()
    H, tq, tk = 4, 9, 37
    q, k, v = _randn(B, tq, 512, seed=13), _randn(B, tk, 512, seed=14), _randn(B, tk, 512, seed=15)
    lens = _lens(LENS)
    ctx = torch.empty(B, tq, 512, device=DEV)
    gm = _abi.GEMM_MODES[mode]
    need = lib.fa_attention_tc_workspace_bytes(B, H, tq, tk, gm)
    _check(need, lambda p, n: lib.fa_attention_tc(q.data_ptr(), 512, k.data_ptr(), 512, v.data_ptr(), 512, lens.data_ptr(), B, H, tq, tk,
                                                  ctx.data_ptr(), 512, gm, p, n, _st()), [ctx])


@pytest.mark.parametrize("mode", MODES)
def test_linear_workspace_on_the_head_projection(mode):
    lib = _lib()
    eng = _engine("bicif", mode)
    lin = eng.ts_head.blstm_ih
    rows = B * T
    x = _randn(rows, lin.in_f, seed=16)
    y = torch.empty(rows, lin.out_f, device=DEV)
    need = lib.fa_linear_workspace_bytes(rows, lin.in_f, eng.mode)
    _check(need, lambda p, n: lib.fa_linear(x.data_ptr(), lin.in_f, rows, C.byref(lin), 0, None, 0, None, 0, y.data_ptr(), lin.out_f, eng.mode,
                                            p, n, _st()), [y])


@pytest.mark.parametrize("hidden", [512, 320])
def test_blstm_workspace(hidden):
    lib = _lib()
    b, t = 3, 7
    xp = _randn(b * t, 8 * hidden, seed=17) * 0.5
    wf, wb = _randn(4 * hidden, hidden, seed=18) * 0.05, _randn(4 * hidden, hidden, seed=19) * 0.05
    out = torch.empty(b, t, 2 * hidden, device=DEV)
    need = lib.fa_blstm_tc_scratch_bytes(b)      # sized for H = 512: exact there, an upper bound for 320
    _check(need, lambda p, n: lib.fa_blstm_forward_tc(xp.data_ptr(), wf.data_ptr(), wb.data_ptr(), b, t, hidden, out.data_ptr(), p, n, _st()),
           [out], refuses_short=hidden == 512)
