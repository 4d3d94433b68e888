"""GPU (-m gpu): the fa-zh MonotonicAligner shape (d = 320, 4 x 80 heads, BLSTM hidden 320) through every layer it runs.

  * MonotonicAlignerB200.inference against the reference's goldens (tests/golden/aligner_*.npz) in fp32 and fp16x3: the same
    integer-ms stamps, upsampled CIF weights within 1e-4 relative, fires at the same frames.
  * The 80-wide tensor-core attention (fa_attention_tc_planes_ex) against float64, its 128-wide instantiation against
    fa_attention_tc_planes bit for bit; the fp32 warp-per-query kernel at hd = 80 against float64.
  * The QKV GEMM's attention sinks at D = 320 (tiles straddling the q | k and k | v boundaries) against the CPU split.
  * The BLSTM recurrence at hidden 320 against a float64 restatement, and batch independence bit for bit.
  * The encoder at (320, 80): fp16x3 against fp32.
The attention bars are those of the 128-wide kernel (tests/test_attention_gpu.py): the 80-wide instantiation runs the same
arithmetic with fewer k-steps.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from test_attention_gpu import DEV, F16, NAN, QPL, NPL, _Linear, _a_planes, _lib, _ref64, _same, _split, _st, _vt

pytestmark = pytest.mark.gpu

HD80, D320 = 80, 320
QSCALE80 = float(np.float32(80 ** -0.5))
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# plane-fed attention against float64 (max |d ctx| / max |V|); the same bars as the 128-wide kernel (test_attention_gpu.py)
F64_TOL = {"fp16x3": 3e-6, "fp16": 5e-4}
F32_TOL = 1e-6
FA_ERR_UNSUPPORTED = -4      # include/funasr_b200.h


def _planes_attention_ex(abi, lib, qp, kp, vt, lens, B, H, hd, tq, tk, mode, kv_shared=0):
    d = H * hd
    ctx = torch.full((B * tq, d), NAN, device=DEV)
    qd, kd, vd = qp.to(DEV), kp.to(DEV), vt.to(DEV)
    ld = torch.tensor(lens, dtype=torch.int32, device=DEV)
    st = lib.fa_attention_tc_planes_ex(qd.data_ptr(), kd.data_ptr(), vd.data_ptr(), ld.data_ptr(), B, H, hd, tq, tk, ctx.data_ptr(), d,
                                       None, 0, 0, abi.GEMM_MODES[mode], kv_shared, _st())
    assert st == 0, st
    torch.cuda.synchronize()
    return ctx.cpu()


def _rand(B, H, tq, tk, seed, kb=None, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    d = H * HD80
    q = torch.randn(B * tq, d, generator=g) * QSCALE80 * scale
    k = torch.randn((kb or B) * tk, d, generator=g)
    v = torch.randn((kb or B) * tk, d, generator=g)
    return q, k, v


ATT_CASES = [   # (B, H, tq, tk, lens)
    (2, 4, 100, 100, [100, 37]),
    (1, 4, 130, 4100, [4100]),                 # the longest key range, two query tiles
    (3, 4, 64, 192, [64, 128, 192]),           # key counts exactly at 64-key chunk edges
    (3, 4, 70, 200, [65, 63, 1]),              # one past / one short of a chunk edge, a single key
    (2, 1, 33, 129, [129, 0]),                 # one head; an utterance without keys -> zeros
]


@pytest.mark.parametrize("mode", ["fp16", "fp16x3", "fp16x6"])
@pytest.mark.parametrize("case", ATT_CASES, ids=[str(c[:4]) for c in ATT_CASES])
def test_attention_hd80_vs_float64(case, mode):
    B, H, tq, tk, lens = case
    abi, lib = _lib()
    q, k, v = _rand(B, H, tq, tk, seed=tq * 7 + tk)
    npl = QPL[mode]
    qp, kp = _split(q, npl), _split(k, npl)
    tkp = (tk + 63) // 64 * 64
    got = _planes_attention_ex(abi, lib, qp, kp, _vt(v, B, tk, tkp, npl), lens, B, H, HD80, tq, tk, mode)
    rec = lambda p: p.float().sum(0)
    want, _, _ = _ref64(rec(qp), rec(kp), rec(_split(v, npl)), lens, B, H, tq, tk, hd=HD80)
    err = float((got.double() - want).abs().max() / v.abs().max())
    assert err <= F64_TOL["fp16" if mode == "fp16" else "fp16x3"], err


@pytest.mark.parametrize("mode", ["fp16", "fp16x3"])
def test_attention_hd80_peaked_rows(mode):
    """Scores in the tens (probability concentrated on a few keys)."""
    B, H, tq, tk, lens = 2, 4, 64, 300, [300, 211]
    abi, lib = _lib()
    q, k, v = _rand(B, H, tq, tk, seed=5, scale=6.0)
    npl = QPL[mode]
    qp, kp = _split(q, npl), _split(k, npl)
    got = _planes_attention_ex(abi, lib, qp, kp, _vt(v, B, tk, 320, npl), lens, B, H, HD80, tq, tk, mode)
    want, _, _ = _ref64(qp.float().sum(0), kp.float().sum(0), _split(v, npl).float().sum(0), lens, B, H, tq, tk, hd=HD80)
    err = float((got.double() - want).abs().max() / v.abs().max())
    assert err <= (5e-4 if mode == "fp16" else 4e-5), err


def test_attention_hd80_kv_shared_and_independence():
    """A shared K/V equals the same K/V replicated per utterance; an utterance and a head do not depend on their neighbours."""
    abi, lib = _lib()
    B, H, tq, tk, mode = 3, 4, 50, 90, "fp16x3"
    q, k, v = _rand(B, H, tq, tk, seed=11, kb=1)
    lens = [90, 90, 90]
    shared = _planes_attention_ex(abi, lib, _split(q, 2), _split(k, 2), _vt(v, 1, tk, 128, 2), lens, B, H, HD80, tq, tk, mode, kv_shared=1)
    kr, vr = k.repeat(B, 1), v.repeat(B, 1)
    rep = _planes_attention_ex(abi, lib, _split(q, 2), _split(kr, 2), _vt(vr, B, tk, 128, 2), lens, B, H, HD80, tq, tk, mode)
    assert torch.equal(shared, rep)
    # utterance 1 alone, then head 2 of utterance 1 alone
    one = _planes_attention_ex(abi, lib, _split(q[tq:2 * tq], 2), _split(k, 2), _vt(v, 1, tk, 128, 2), [90], 1, H, HD80, tq, tk, mode)
    assert torch.equal(one, rep[tq:2 * tq])
    cols = slice(2 * HD80, 3 * HD80)
    head = _planes_attention_ex(abi, lib, _split(q[tq:2 * tq, cols].contiguous(), 2), _split(k[:, cols].contiguous(), 2),
                                _vt(v[:, cols].contiguous(), 1, tk, 128, 2), [90], 1, 1, HD80, tq, tk, mode)
    assert torch.equal(head, rep[tq:2 * tq, cols])


@pytest.mark.parametrize("mode", ["fp16", "fp16x3"])
def test_plane_entry_hd128_equals_fa_attention_tc_planes(mode):
    abi, lib = _lib()
    B, H, tq, tk, lens = 2, 4, 70, 150, [150, 77]
    g = torch.Generator().manual_seed(3)
    q, k, v = (torch.randn(B * n, H * 128, generator=g) for n in (tq, tk, tk))
    npl = QPL[mode]
    qp, kp, vt = _split(q * 0.088, npl).to(DEV), _split(k, npl).to(DEV), _vt(v, B, tk, 192, npl).to(DEV)
    ld = torch.tensor(lens, dtype=torch.int32, device=DEV)
    a = torch.full((B * tq, H * 128), NAN, device=DEV)
    b = torch.full((B * tq, H * 128), NAN, device=DEV)
    gm = abi.GEMM_MODES[mode]
    assert lib.fa_attention_tc_planes(qp.data_ptr(), kp.data_ptr(), vt.data_ptr(), ld.data_ptr(), B, H, tq, tk, a.data_ptr(), H * 128,
                                      None, 0, 0, gm, 0, _st()) == 0
    assert lib.fa_attention_tc_planes_ex(qp.data_ptr(), kp.data_ptr(), vt.data_ptr(), ld.data_ptr(), B, H, 128, tq, tk, b.data_ptr(),
                                         H * 128, None, 0, 0, gm, 0, _st()) == 0
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_attention_status_codes_other_head_dims():
    abi, lib = _lib()
    buf = torch.zeros(1 << 20, dtype=F16, device=DEV)
    ld = torch.tensor([8], dtype=torch.int32, device=DEV)
    ctx = torch.zeros(8, 1024, device=DEV)
    for hd in (64, 96, 112, 256):
        st = lib.fa_attention_tc_planes_ex(buf.data_ptr(), buf.data_ptr(), buf.data_ptr(), ld.data_ptr(), 1, 4, hd, 8, 8, ctx.data_ptr(),
                                           1024, None, 0, 0, abi.GEMM_MODES["fp16x3"], 0, _st())
        assert st == FA_ERR_UNSUPPORTED, (hd, st)


@pytest.mark.parametrize("kv_shared", [0, 1])
def test_f32_attention_hd80_vs_float64(kv_shared):
    abi, lib = _lib()
    B, H, tq, tk, lens = 3, 4, 40, 300, [300, 123, 1]
    q, k, v = _rand(B, H, tq, tk, seed=9, kb=1 if kv_shared else None)
    q = q / QSCALE80                                   # the kernel scales q itself
    qd, kd, vd = q.to(DEV), k.to(DEV), v.to(DEV)
    ctx = torch.full((B * tq, D320), NAN, device=DEV)
    ld = torch.tensor(lens, dtype=torch.int32, device=DEV)
    abi.check(lib.fa_attention_f32_ex(qd.data_ptr(), D320, kd.data_ptr(), D320, vd.data_ptr(), D320, ld.data_ptr(), B, H, HD80, tq, tk,
                                      ctx.data_ptr(), D320, kv_shared, _st()), "fa_attention_f32_ex")
    torch.cuda.synchronize()
    want, _, _ = _ref64(q * torch.tensor(QSCALE80), k, v, lens, B, H, tq, tk, hd=HD80, kv_shared=bool(kv_shared))
    err = float((ctx.cpu().double() - want).abs().max() / v.abs().max())
    assert err <= F32_TOL, err


# ---------------------------------------------------------------------------------------------------- QKV sinks at D = 320
@pytest.mark.parametrize("mode", list(NPL))
@pytest.mark.parametrize("T,t_pad", [(100, 128), (37, 64)], ids=["staged_vt", "vt16"])
def test_attn_sinks_d320_equal_split(T, t_pad, mode):
    """N = 960: 128-wide tiles straddle column 320 (q | k) and 640 (k | v); the sinks split each 16-column chunk on its own."""
    abi, lib = _lib()
    B, N, W, in_f = 3, 3 * D320, D320, 320
    M = B * T
    L = _Linear(abi, lib, N, in_f, seed=77)
    x = torch.randn(M, in_f, generator=torch.Generator().manual_seed(M))
    ap = _a_planes(abi, lib, x.to(DEV), NPL[mode], L.in_pad)
    gm = abi.GEMM_MODES[mode]
    y = torch.full((M, N), NAN, device=DEV)
    abi.check(lib.fa_linear_planes(ap.data_ptr(), M, C.byref(L.lin), 0, None, 0, None, 0, y.data_ptr(), N, gm, _st()), "fp32 epilogue")
    qp = torch.full((3, M, W), NAN, dtype=F16, device=DEV)
    kp = torch.full((3, M, W), NAN, dtype=F16, device=DEV)
    vt = torch.full((3, B * W, t_pad), NAN, dtype=F16, device=DEV)
    abi.check(lib.fa_linear_attn_sinks(ap.data_ptr(), M, C.byref(L.lin), 0, W, 2 * W, W, T, t_pad, QSCALE80, qp.data_ptr(), kp.data_ptr(),
                                       vt.data_ptr(), None, N, gm, _st()), "attn sinks")
    torch.cuda.synchronize()
    y, qp, kp, vt = y.cpu(), qp.cpu(), kp.cpu(), vt.cpu()
    npl = QPL[mode]
    _same(qp[:npl], _split(y[:, :W] * torch.tensor(QSCALE80), npl), "q planes")
    _same(kp[:npl], _split(y[:, W:2 * W], npl), "k planes")
    yt = y[:, 2 * W:].reshape(B, T, W).transpose(1, 2).reshape(B * W, T)
    _same(vt[:npl, :, :T], _split(yt, npl), "v^T planes")


# ---------------------------------------------------------------------------------------------------- BLSTM at hidden 320
def _blstm_run(abi, lib, xproj, whf, whb, B, T, H):
    out = torch.full((B, T, 2 * H), NAN, device=DEV)
    nb = int(lib.fa_blstm_tc_scratch_bytes(B))
    scr = torch.empty(nb, dtype=torch.uint8, device=DEV)
    st = lib.fa_blstm_forward_tc(xproj.data_ptr(), whf.data_ptr(), whb.data_ptr(), B, T, H, out.data_ptr(), scr.data_ptr(), nb, _st())
    torch.cuda.synchronize()
    return st, out


def _blstm_inputs(B, T, H, seed):
    g = torch.Generator().manual_seed(seed)
    xproj = torch.randn(B * T, 8 * H, generator=g) * 0.8
    whf, whb = (torch.randn(4 * H, H, generator=g) / H ** 0.5 for _ in range(2))
    return xproj, whf, whb


def _blstm_ref64(xproj, whf, whb, B, T, H):
    x = xproj.double().reshape(B, T, 2, 4 * H)
    out = torch.zeros(B, T, 2 * H, dtype=torch.float64)
    for d, w in enumerate((whf.double(), whb.double())):
        h = torch.zeros(B, H, dtype=torch.float64)
        c = torch.zeros(B, H, dtype=torch.float64)
        for s in range(T):
            t = s if d == 0 else T - 1 - s
            gt = x[:, t, d] + h @ w.T
            i, f, gg, o = gt.split(H, -1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(o) * torch.tanh(c)
            out[:, t, d * H:(d + 1) * H] = h
    return out


def test_blstm_h320_vs_float64():
    abi, lib = _lib()
    B, T, H = 70, 150, 320                       # two batch tiles, the second partly padded
    xproj, whf, whb = _blstm_inputs(B, T, H, 1)
    st, out = _blstm_run(abi, lib, xproj.to(DEV), whf.to(DEV), whb.to(DEV), B, T, H)
    assert st == 0, st
    err = float((out.cpu().double() - _blstm_ref64(xproj, whf, whb, B, T, H)).abs().max())
    assert err <= 2e-4, err                      # h in (-1, 1): bf16 hi / lo split of h and W_hh (~2^-17 relative per product)


def test_blstm_h320_batch_independence_and_status():
    abi, lib = _lib()
    T, H = 40, 320
    xproj, whf, whb = _blstm_inputs(256, T, H, 2)
    xd, wf, wb = xproj.to(DEV), whf.to(DEV), whb.to(DEV)
    st, full = _blstm_run(abi, lib, xd, wf, wb, 256, T, H)
    assert st == 0
    for b in (0, 131, 255):
        st, one = _blstm_run(abi, lib, xd[b * T:(b + 1) * T].contiguous(), wf, wb, 1, T, H)
        assert st == 0 and torch.equal(one[0].view(torch.int32), full[b].view(torch.int32)), b
    st, _ = _blstm_run(abi, lib, xd, wf, wb, 1, T, 256)
    assert st == FA_ERR_UNSUPPORTED, st


# ---------------------------------------------------------------------------------------------------- encoder and model
def test_encoder_320_fp16x3_vs_fp32():
    """(320, 80) encoder, 30 blocks: fp16x3 against fp32.  Both carry ~2^-22 relative per product and every block is LayerNorm-
    bounded.  The bar, 1e-4, is ten times tighter than the 1e-3 test_gpu_parity.py holds the 512-wide encoder output to."""
    from funasr_b200 import synth
    from funasr_b200.engine import AlignerEngine
    cfg = synth.ALIGNER_FA_ZH
    sd = synth.make_aligner_state_dict(cfg, 6)
    g = torch.Generator().manual_seed(4)
    B, T = 3, 180
    feats = torch.randn(B, T, 560, generator=g).to(DEV)
    lens = torch.tensor([180, 97, 5], dtype=torch.int32, device=DEV)
    outs = {m: AlignerEngine(sd, cfg, DEV, gemm_mode=m).encode(feats, lens) for m in ("fp32", "fp16x3")}
    torch.cuda.synchronize()
    for b, n in enumerate(lens.tolist()):
        assert rel_err(outs["fp16x3"][b, :n].cpu(), outs["fp32"][b, :n].cpu()) <= 1e-4


class _CharTok:
    """The CharTokenizer surface the aligner uses (split_with_space), over the synthetic token list."""

    def __init__(self, tokens):
        self.tokens = tokens
        self.ids = {t: i for i, t in enumerate(tokens)}

    def encode(self, text):
        return [self.ids.get(t, len(self.tokens) - 1) for t in text.strip().split(" ")]

    def ids2tokens(self, ids):
        return [self.tokens[i] for i in ids]

    def tokens2text(self, tokens):
        return "".join(tokens)


def _model(cfg, seed, mode):
    from funasr_b200 import synth
    from funasr_b200.modules import MonotonicAlignerB200
    m = MonotonicAlignerB200(
        encoder="SANMEncoder", encoder_conf=dict(output_size=cfg.d_model, attention_heads=cfg.heads, linear_units=cfg.ffn,
                                                 num_blocks=cfg.enc_layers, kernel_size=cfg.kernel, input_layer="pe",
                                                 normalize_before=True, selfattention_layer_type="sanm"),
        predictor="CifPredictorV3", predictor_conf=dict(idim=cfg.d_model, threshold=1.0, l_order=1, r_order=1, tail_threshold=0.45,
                                                        smooth_factor2=0.25, noise_threshold2=0.01, upsample_times=3, use_cif1_cnn=False,
                                                        upsample_type="cnn_blstm"),
        input_size=560, predictor_bias=1, length_normalized_loss=False, gemm_mode=mode)
    m.load_state_dict(synth.make_aligner_state_dict(cfg, seed), strict=True)
    return m.to(DEV)


ALIGNER_GOLDENS = {"aligner_tiny_ragged3": ("ALIGNER_TINY", 5), "aligner_fa_zh_single": ("ALIGNER_FA_ZH", 6)}


@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("name", list(ALIGNER_GOLDENS))
def test_aligner_model_vs_golden(name, mode):
    from funasr_b200 import synth
    from funasr_b200.modules import WavFrontendB200
    z = np.load(os.path.join(GOLD, name + ".npz"))
    cfg_name, seed = ALIGNER_GOLDENS[name]
    cfg = getattr(synth, cfg_name)
    model = _model(cfg, seed, mode)
    fe = WavFrontendB200(cmvn=synth.make_cmvn(cfg, seed=1), lfr_m=7, lfr_n=6, dither=0.0)
    tok = _CharTok(synth.aligner_token_list(400))
    ids = np.split(z["ids_flat"], np.cumsum(z["ids_len"])[:-1])
    wavs = [synth.make_aligner_wav(float(sec), int(s)) for sec, s in z["wav_spec"]]
    pairs = [(w, [int(t) for t in i]) for w, i in zip(wavs, ids)]
    res, _ = model.inference(pairs, key=["u%d" % i for i in range(len(pairs))], tokenizer=tok, frontend=fe, device=DEV,
                             data_type=("sound", "text"))
    stamps = np.split(z["stamps_flat"].reshape(-1, 2), np.cumsum(z["stamps_len"])[:-1])
    for r, st in zip(res, stamps):
        assert r["timestamp"] == st.tolist()
    # the timestamp head's weights and fires
    eng = model.engine(DEV)
    feats, flens = fe(torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True), [w.numel() for w in wavs], device=DEV)
    lens = flens.to(DEV, torch.int32)
    assert lens.cpu().tolist() == z["enc_lens"].tolist()
    ua, up = eng.upsample_timestamp(eng.encode(feats, lens), lens, torch.tensor([len(i) + 1 for i in ids], dtype=torch.int32))
    ua, up = ua.cpu(), up.cpu()
    for b, n in enumerate(z["enc_lens"].tolist()):
        ref = torch.from_numpy(z["us_alphas"][b, :3 * n])
        assert float((ua[b, :3 * n] - ref).abs().max() / ref.abs().max()) <= 1e-4
        fires_got = (up[b, :3 * n] >= 1.0 - 1e-4).nonzero().flatten().tolist()
        fires_want = (torch.from_numpy(z["us_peaks"][b, :3 * n]) >= 1.0 - 1e-4).nonzero().flatten().tolist()
        assert fires_got == fires_want
