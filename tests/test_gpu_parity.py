"""GPU (-m gpu): the CUDA path, called through the C ABI, against the oracle on the same seeded inputs, against the
committed golden vectors of the reference, and — at BASELINE sizes — through size-independent properties.

Bars: integer outcomes (frame counts, token counts, greedy ids) bit-exact; floating point within 1e-3 relative of the
fp32 reference (rel = max|a-b| / max|b|), the tolerance the north star states for logits.  Frontend: log-mel values
agree to 2e-5 except where a mel bin sits far below the frame's strongest bin — there BOTH fp32 FFTs (ours and the
reference's pocketfft) are at their rounding-noise floor (torch fp32 vs fp64 differs by up to 1e-3 on these inputs),
so the bound is |d logmel| <= 2e-5 + 2e-6 * sqrt(E_frame_max / E_bin); mean |d| <= 2e-5.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import CTX_CASES, GOLDEN, GOLDEN_CASES, SV_CASES, load_case, load_ctx_case, load_sv_case, rel_err, state_dict_for

import paraformer_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _lib():
    from funasr_b200 import _abi
    return _abi, _abi.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


# ----------------------------------------------------------------------------------------------- frontend
def _run_frontend(wavs, cmvn):
    from funasr_b200.engine import FrontendEngine, num_lfr_frames
    eng = FrontendEngine(cmvn, DEV)
    lens = [w.numel() for w in wavs]
    pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
    t_max = max(num_lfr_frames(n) for n in lens)
    feats, fl = eng(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), t_max)
    torch.cuda.synchronize()
    return feats.cpu(), fl.cpu()


def _assert_feats_close(got, ref, cmvn):
    """got/ref: [T, 560] LFR+CMVN features of one utterance; bound stated in the module docstring."""
    g, r = got.double(), ref.double()
    if cmvn is not None:                                   # undo CMVN -> stacked log-mel
        g, r = g / cmvn[1].double() - cmvn[0].double(), r / cmvn[1].double() - cmvn[0].double()
    g, r = g.reshape(-1, 7, 80), r.reshape(-1, 7, 80)
    frame_max = r.max(dim=-1, keepdim=True).values
    tol = 2e-5 + 2e-6 * torch.exp(0.5 * (frame_max - r))
    d = (g - r).abs()
    assert bool((d <= tol).all()), "log-mel diff %.3e exceeds noise-floor bound (worst excess %.3e)" % (float(d.max()), float((d - tol).max()))
    assert float(d.mean()) <= 2e-5


@pytest.mark.parametrize("lens,use_cmvn", [([16000, 400, 8123, 559, 560, 1359, 1360], True), ([48000, 27200], False), ([480000], True)])
def test_fbank_lfr_cmvn_vs_oracle(lens, use_cmvn):
    from funasr_b200 import synth
    wavs = [synth.make_wav(n, 20 + i, "speechlike" if i % 2 == 0 else "noise") for i, n in enumerate(lens)]
    cmvn = synth.make_cmvn(synth.PARAFORMER_LARGE, 2) if use_cmvn else None
    ref, ref_len = O.frontend(wavs, cmvn)
    got, got_len = _run_frontend(wavs, cmvn)
    assert got_len.tolist() == ref_len.tolist()                    # integer: exact
    assert got.shape == ref.shape
    for b, n in enumerate(ref_len.tolist()):
        _assert_feats_close(got[b, :n], ref[b, :n], cmvn)
        assert float(got[b, n:].abs().max()) == 0.0 if n < got.shape[1] else True   # pad_sequence(0.0)


def test_fbank_vs_the_reference_runtimes_compiled_kaldi_native_fbank():
    """The CUDA frontend against the reference's OTHER Fbank: kaldi-native-fbank compiled from the reference tree
    (oracle/_ref/libknf_ref.so when it travelled, else its committed outputs tests/golden/knf_fbank.npz), stacked 7/6 by the
    oracle's LFR.  Frame counts exact; log-mel inside the rounding floor of two different fp32 FFTs (2 x conftest.knf_bound: the oracle alone uses 0.94 of it)."""
    from conftest import knf_bound, knf_logmel_cases
    cases = knf_logmel_cases()
    got, got_len = _run_frontend([w for w, _, _ in cases], None)
    for b, (w, gold, live) in enumerate(cases):
        ref = O.apply_lfr(torch.from_numpy(live if live is not None else gold), 7, 6).double().numpy()
        n = int(got_len[b])
        assert n == ref.shape[0]
        g, r = got[b, :n].double().numpy().reshape(n, 7, 80), ref.reshape(n, 7, 80)
        d = np.abs(g - r)
        assert (d <= knf_bound(r, 2.0)).all(), float((d / knf_bound(r, 2.0)).max())
        assert d.mean() <= 2e-5


def test_fbank_silence_and_clipping_edges():
    """All-zero audio hits the log floor (log eps); full-scale square wave exercises large magnitudes."""
    z = torch.zeros(3200)
    sq = torch.sign(torch.sin(torch.arange(4000.0) * 0.3)).float()
    ref, _ = O.frontend([z, sq], None)
    got, _ = _run_frontend([z, sq], None)
    assert np.abs(got[0, :4].numpy() - ref[0, :4].numpy()).max() <= 1e-5      # log(eps) floor everywhere
    _assert_feats_close(got[1], ref[1], None)


# ------------------------------------------------------------------------------------------- operator level
def test_layernorm_vs_oracle():
    abi, lib = _lib()
    g = torch.Generator().manual_seed(0)
    for n, rows in [(512, 1000), (560, 333), (2048, 77)]:
        x = torch.randn(rows, n, generator=g) * 3 + 0.5
        w, b = 1 + 0.1 * torch.randn(n, generator=g), 0.1 * torch.randn(n, generator=g)
        xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
        y = torch.empty_like(xd)
        nm = abi.FaNorm(wd.data_ptr(), bd.data_ptr(), n, 1e-12)
        abi.check(lib.fa_layernorm(xd.data_ptr(), rows, C.byref(nm), y.data_ptr(), None, 1.0, 1, _st()), "ln")
        assert rel_err(y.cpu().numpy(), O.layer_norm(x, w, b).numpy()) <= 1e-5
    # fused x*sqrt(512)+PE prologue (encoder.py:409,428)
    from funasr_b200 import synth
    B, T, n = 2, 97, 560
    x = torch.randn(B, T, n, generator=g)
    w, b = 1 + 0.1 * torch.randn(n, generator=g), 0.1 * torch.randn(n, generator=g)
    inv = synth.sinusoid_inv_timescales(n).to(DEV)
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    y = torch.empty_like(xd)
    nm = abi.FaNorm(wd.data_ptr(), bd.data_ptr(), n, 1e-12)
    abi.check(lib.fa_layernorm(xd.data_ptr(), B * T, C.byref(nm), y.data_ptr(), inv.data_ptr(), 512 ** 0.5, T, _st()), "ln+pe")
    ref = O.layer_norm(x * 512 ** 0.5 + O.sinusoid_pe(T, n), w, b)
    assert rel_err(y.cpu().numpy(), ref.numpy()) <= 1e-5


@pytest.mark.parametrize("rows,out_f,in_f", [(1000, 1536, 560), (777, 512, 2048), (130, 8404, 512), (64, 1000, 512)])
def test_linear_fp32_vs_oracle(rows, out_f, in_f):
    abi, lib = _lib()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(rows, in_f, generator=g)
    w = torch.randn(out_f, in_f, generator=g) / in_f ** 0.5
    b = torch.randn(out_f, generator=g) * 0.1
    r1 = torch.randn(rows, out_f, generator=g)
    xd, wd, bd, r1d = x.to(DEV), w.to(DEV), b.to(DEV), r1.to(DEV)
    y = torch.empty(rows, out_f, device=DEV)
    lin = abi.FaLinear(wd.data_ptr(), bd.data_ptr(), None, out_f, in_f, (in_f + 63) // 64 * 64, 0)
    abi.check(lib.fa_linear(xd.data_ptr(), in_f, rows, C.byref(lin), 1, r1d.data_ptr(), out_f, None, 0, y.data_ptr(), out_f,
                            abi.GEMM_F32_SIMT, None, 0, _st()), "linear")
    ref = torch.relu(torch.nn.functional.linear(x, w, b)) + r1
    assert rel_err(y.cpu().numpy(), ref.numpy()) <= 2e-6


@pytest.mark.parametrize("mode,tol", [("fp16x6", 1e-5), ("fp16x3", 3e-5), ("fp16", 2e-2)])
@pytest.mark.parametrize("rows,out_f,in_f", [(1000, 1536, 560), (300, 512, 2048), (130, 8404, 512), (129, 1000, 512), (32000, 512, 512),
                                             (1000, 8404, 512), (700, 25060, 512)])    # ragged N (vocabulary projections) through the edge epilogue; residual rows need a pitch % 4 == 0
def test_linear_tcgen05_vs_oracle(rows, out_f, in_f, mode, tol):
    """wgmma/TMA GEMM with fp16 operand splitting against the CPU fp32 nn.Linear (ragged M/N/K tails)."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(rows, in_f, generator=g)
    w = torch.randn(out_f, in_f, generator=g) / in_f ** 0.5
    b = torch.randn(out_f, generator=g) * 0.1
    r1 = torch.randn(rows, out_f, generator=g)
    r2 = torch.randn(rows, out_f, generator=g)
    xd, wd, bd, r1d, r2d = x.to(DEV), w.to(DEV), b.to(DEV), r1.to(DEV), r2.to(DEV)
    in_pad = (in_f + 63) // 64 * 64
    planes = torch.empty(3, out_f, in_pad, dtype=torch.float16, device=DEV)
    abi.check(lib.fa_split_planes(wd.data_ptr(), in_f, out_f, in_f, in_pad, planes.data_ptr(), _st()), "split")
    torch.cuda.synchronize()
    # three fp16 planes: hi is exact to 2^-11 of |w|, the remainders sit in fp16's subnormal range for weights of this size, whose
    # spacing is 2^-24 — reconstruction within half of that (3e-8 absolute, ~2e-7 of max |w| here)
    assert np.abs((planes[0].float() + planes[1].float() + planes[2].float())[:, :in_f].cpu().numpy() - w.numpy()).max() <= 2.0 ** -25 + 1e-12
    y = torch.full((rows, out_f), float("nan"), device=DEV)
    lin = abi.FaLinear(wd.data_ptr(), bd.data_ptr(), planes.data_ptr(), out_f, in_f, in_pad, 0)
    ws = torch.empty(3 * rows * in_pad * 2 + 4096, dtype=torch.uint8, device=DEV)
    abi.check(lib.fa_linear(xd.data_ptr(), in_f, rows, C.byref(lin), 1, r1d.data_ptr(), out_f, r2d.data_ptr(), out_f, y.data_ptr(),
                            out_f, abi.GEMM_MODES[mode], ws.data_ptr(), ws.numel(), _st()), "linear tc")
    torch.cuda.synchronize()
    ref = torch.relu(torch.nn.functional.linear(x, w, b)) + r1 + r2
    assert not torch.isnan(y).any()
    err = rel_err(y.cpu().numpy(), ref.numpy())
    print("linear wgmma %s rows=%d out=%d in=%d: rel err %.2e (tol %.0e)" % (mode, rows, out_f, in_f, err, tol))
    assert err <= tol


def test_fsmn_vs_oracle():
    abi, lib = _lib()
    g = torch.Generator().manual_seed(2)
    B, T, Cn = 3, 150, 512
    lens = torch.tensor([150, 1, 77], dtype=torch.int32)
    qkv = torch.randn(B, T, 1536, generator=g)
    w = torch.randn(Cn, 1, 11, generator=g) * 0.2
    res = torch.randn(B, T, Cn, generator=g)
    mask = (torch.arange(T)[None, :] < lens[:, None]).float()[:, :, None]
    ref = O.fsmn(qkv[:, :, 1024:], w, mask)
    qd, wd, ld, rd = qkv.to(DEV), w.to(DEV), lens.to(DEV), res.to(DEV)
    out = torch.empty(B, T, Cn, device=DEV)
    abi.check(lib.fa_fsmn(qd.data_ptr() + 1024 * 4, 1536, ld.data_ptr(), B, T, Cn, wd.data_ptr(), 11, None, 0, out.data_ptr(), Cn, _st()), "fsmn")
    assert rel_err(out.cpu().numpy(), ref.numpy()) <= 1e-6
    abi.check(lib.fa_fsmn(qd.data_ptr() + 1024 * 4, 1536, ld.data_ptr(), B, T, Cn, wd.data_ptr(), 11, rd.data_ptr(), Cn, out.data_ptr(), Cn, _st()), "fsmn+res")
    assert rel_err(out.cpu().numpy(), (res + ref).numpy()) <= 1e-6


@pytest.mark.parametrize("B,T,Cn,ld,K,lens", [(3, 150, 512, 1536, 11, [150, 1, 77]), (5, 500, 512, 1536, 11, [500, 83, 0, 499, 321]),
                                               (2, 64, 128, 128, 21, [64, 9]), (300, 70, 256, 256, 21, None)])
def test_fsmn_tma_staged_variant_is_bit_identical(B, T, Cn, ld, K, lens):
    """fa_fsmn_tma (persistent, warp-specialised, cp.async.bulk.tensor ring; utterance edges = the tensor map's zero fill) against the
    SIMT kernel bit for bit and against the oracle — with and without the fused residual, a strided v view, partial last time tiles,
    empty / one-frame utterances and more tiles than SMs."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(21)
    lens = torch.tensor(lens if lens is not None else [int(x) for x in torch.randint(0, T + 1, (B,), generator=g)], dtype=torch.int32)
    off = ld - Cn
    src = torch.randn(B, T, ld, generator=g)
    w = torch.randn(Cn, 1, K, generator=g) * 0.2
    res = torch.randn(B, T, Cn, generator=g)
    mask = (torch.arange(T)[None, :] < lens[:, None]).float()[:, :, None]
    ref = O.fsmn(src[:, :, off:], w, mask)
    sd, wd, ld_dev, rd = src.to(DEV), w.to(DEV), lens.to(DEV), res.to(DEV)
    for r in (None, rd):
        a, b = torch.full((B, T, Cn), 7.0, device=DEV), torch.full((B, T, Cn), -7.0, device=DEV)
        args = (sd.data_ptr() + off * 4, ld, ld_dev.data_ptr(), B, T, Cn, wd.data_ptr(), K, None if r is None else r.data_ptr(), Cn)
        d = torch.full((B, T, Cn), 3.0, device=DEV)
        abi.check(lib.fa_fsmn_simt(*args, a.data_ptr(), Cn, _st()), "fa_fsmn_simt")
        abi.check(lib.fa_fsmn_tma(*args, b.data_ptr(), Cn, _st()), "fa_fsmn_tma")
        abi.check(lib.fa_fsmn(*args, d.data_ptr(), Cn, _st()), "fa_fsmn")          # the default route (either kernel)
        torch.cuda.synchronize()
        assert torch.equal(a, b) and torch.equal(a, d)
        assert rel_err(b.cpu().numpy(), (ref if r is None else res + ref).numpy()) <= 1e-6
    # unsupported shapes answer with a status code, never a wrong result
    assert lib.fa_fsmn_tma(sd.data_ptr() + off * 4, ld, ld_dev.data_ptr(), B, T, Cn, wd.data_ptr(), 31, None, 0, a.data_ptr(), Cn, _st()) == -4
    assert lib.fa_fsmn_tma(sd.data_ptr() + 4, ld, ld_dev.data_ptr(), B, T, Cn, wd.data_ptr(), K, None, 0, a.data_ptr(), Cn, _st()) == -4


@pytest.mark.parametrize("tq,tk,lens", [(130, 130, [130, 1, 65]), (37, 211, [211, 64, 129])])
def test_attention_vs_oracle(tq, tk, lens):
    abi, lib = _lib()
    g = torch.Generator().manual_seed(3)
    B, H, D = 3, 4, 512
    q = torch.randn(B, tq, D, generator=g) * 1.5
    k = torch.randn(B, tk, D, generator=g) * 1.5
    v = torch.randn(B, tk, D, generator=g)
    kl = torch.tensor(lens, dtype=torch.int32)
    mask = (torch.arange(tk)[None, :] < kl[:, None])[:, None, :]
    ref = O.mh_attention(q, k, v, mask, H)
    qd, kd, vd, ld = q.to(DEV), k.to(DEV), v.to(DEV), kl.to(DEV)
    ctx = torch.empty(B, tq, D, device=DEV)
    abi.check(lib.fa_attention(qd.data_ptr(), D, kd.data_ptr(), D, vd.data_ptr(), D, ld.data_ptr(), B, H, tq, tk, ctx.data_ptr(), D, _st()), "attn")
    assert rel_err(ctx.cpu().numpy(), ref.numpy()) <= 1e-5


@pytest.mark.parametrize("mode,tol", [("fp16x3", 5e-5), ("fp16", 2e-2)])
@pytest.mark.parametrize("tq,tk,lens", [(130, 130, [130, 1, 65]), (37, 211, [211, 64, 129]), (500, 500, [500, 83, 499]),
                                        (300, 300, [300, 0, 17]),                                    # an utterance without keys: zero context
                                        (260, 200, [200, 3, 64, 65, 199] * 10)])                     # 600 query tiles: several waves of one-tile CTAs
def test_attention_tcgen05_vs_oracle(tq, tk, lens, mode, tol):
    """Tensor-core attention (two-pass softmax, fp16 operand planes, register accumulators) vs the CPU reference chain."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(6)
    B, H, D = len(lens), 4, 512
    q = torch.randn(B, tq, D, generator=g) * 1.5
    k = torch.randn(B, tk, D, generator=g) * 1.5
    v = torch.randn(B, tk, D, generator=g)
    kl = torch.tensor(lens, dtype=torch.int32)
    mask = (torch.arange(tk)[None, :] < kl[:, None])[:, None, :]
    ref = O.mh_attention(q, k, v, mask, H)
    qd, kd, vd, ld = q.to(DEV), k.to(DEV), v.to(DEV), kl.to(DEV)
    ctx = torch.full((B, tq, D), float("nan"), device=DEV)
    gm = abi.GEMM_MODES[mode]
    ws = torch.empty(lib.fa_attention_tc_workspace_bytes(B, H, tq, tk, gm), dtype=torch.uint8, device=DEV)
    abi.check(lib.fa_attention_tc(qd.data_ptr(), D, kd.data_ptr(), D, vd.data_ptr(), D, ld.data_ptr(), B, H, tq, tk, ctx.data_ptr(), D,
                                  gm, ws.data_ptr(), ws.numel(), _st()), "attn tc")
    torch.cuda.synchronize()
    assert not torch.isnan(ctx).any()
    assert rel_err(ctx.cpu().numpy(), ref.numpy()) <= tol


# ------------------------------------------------------------------------------------------------ model level
def _engine(cfg, wseed, mode="fp32"):
    from funasr_b200.engine import ParaformerEngine
    return ParaformerEngine(state_dict_for(cfg, wseed), cfg, DEV, gemm_mode=mode)


def _run_model(cfg, wseed, wavs, cmvn, mode="fp32"):
    from funasr_b200.engine import FrontendEngine, num_lfr_frames
    fe = FrontendEngine(cmvn, DEV)
    lens = [w.numel() for w in wavs]
    pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
    feats, fl = fe(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), max(num_lfr_frames(n) for n in lens))
    eng = _engine(cfg, wseed, mode)
    out = eng.forward_feats(feats, fl, want_taps=True)
    torch.cuda.synchronize()
    out["feats"], out["feat_lens"] = feats, fl
    return out


def _sub(cfg, t, step):
    return t[:, ::step] if cfg.enc_layers > 10 else t


@pytest.mark.parametrize("mode", ["fp32", "fp16x3", "fp16x6"])
@pytest.mark.parametrize("name", list(GOLDEN_CASES))
def test_paraformer_vs_reference_golden(name, mode):
    """End-to-end against the UNMODIFIED reference's outputs (tests/golden, made by oracle/make_golden.py), with the
    contractions on the fp32 SIMT path and on the wgmma fp16x3 split path."""
    cfg, wseed, wavs, cmvn, g = load_case(name)
    o = _run_model(cfg, wseed, wavs, cmvn, mode)
    assert o["feat_lens"].cpu().tolist() == g["feat_lens"].tolist()
    fd = np.abs(_sub(cfg, o["feats"].cpu(), 7).numpy() - g["feats"])
    assert fd.max() <= 1e-2 and fd.mean() <= 2e-5          # FFT-noise-floor bins dominate the max (see docstring)
    assert rel_err(_sub(cfg, o["enc"].cpu(), 7).numpy(), g["enc"]) <= 1e-3
    assert np.abs(o["alphas"].cpu().numpy() - g["alphas"]).max() <= 1e-4
    assert o["token_num"].tolist() == g["token_num"].tolist()                      # integer: exact
    n = int(g["token_num"].max())
    assert rel_err(_sub(cfg, o["acoustic"][:, :n].cpu(), 5).numpy(), g["acoustic"]) <= 1e-3
    lp = o["logp"][:, g["logp_rows"].tolist(), :].cpu().numpy()
    assert rel_err(lp, g["logp_sel"]) <= 1e-3                                      # contract tolerance
    valid = np.arange(n)[None, :] < g["token_num"][:, None]
    assert (o["argmax"].cpu().numpy()[valid] == g["argmax"][valid]).all()
    ids_flat = [t for r in o["ids"] for t in r]
    assert ids_flat == g["ids_flat"].tolist()                                      # greedy ids: bit-exact
    assert [len(r) for r in o["ids"]] == g["ids_len"].tolist()


def test_paraformer_vs_oracle_fresh_inputs():
    """Same seeded inputs through the oracle and the CUDA path (inputs not in the golden set, ragged batch of 5)."""
    from funasr_b200 import synth
    cfg = synth.PARAFORMER_TINY
    wavs = [synth.make_wav(n, 40 + i, "speechlike") for i, n in enumerate([64000, 9000, 33333, 400, 20480])]
    cmvn = synth.make_cmvn(cfg, 3)
    p = state_dict_for(cfg, 9)
    ref = O.paraformer_forward(wavs, p, cmvn, cfg.enc_layers, cfg.dec_layers)
    o = _run_model(cfg, 9, wavs, cmvn)
    assert o["token_num"].tolist() == ref["token_num"].tolist()
    assert rel_err(o["enc"].cpu().numpy(), ref["enc"].numpy()) <= 1e-3
    assert rel_err(o["logp"].cpu().numpy(), ref["logp"].numpy()) <= 1e-3
    assert o["ids"] == ref["ids"]


def test_properties_at_baseline_size():
    """BASELINE config 2 shape (B=64 x 30 s, T=500) with a 3+2-layer stack: size-independent properties —
    determinism (bit-identical reruns), permutation equivariance over utterances (bit-exact: utterances are
    independent), zero-filled feature padding, token counts within the CIF bound T+1."""
    from funasr_b200 import synth
    from funasr_b200.engine import FrontendEngine
    cfg = synth.PARAFORMER_TINY
    B, N = 64, 480000
    g = torch.Generator().manual_seed(77)
    base = [synth.make_wav(N, 60 + i, "speechlike") for i in range(4)]
    gains = 0.3 + 0.7 * torch.rand(B, generator=g)
    wav = torch.stack([base[i % 4].roll(137 * i) * gains[i] for i in range(B)])
    lens = torch.full((B,), N, dtype=torch.int32)
    lens[5], lens[17] = 80000, 400 + 160 * 6 * 100
    fe = FrontendEngine(synth.make_cmvn(cfg, 1), DEV)
    eng = _engine(cfg, 5)
    feats, fl = fe(wav.to(DEV), lens.to(DEV), 500)
    assert fl.cpu().tolist() == [500 if i not in (5, 17) else (83 if i == 5 else 101) for i in range(B)]
    assert float(feats[5, 83:].abs().max()) == 0.0
    a = eng.forward_feats(feats, fl, want_taps=True)
    b = eng.forward_feats(feats, fl, want_taps=True)
    assert a["ids"] == b["ids"] and torch.equal(a["enc"], b["enc"]) and torch.equal(a["logp"], b["logp"])
    assert all(0 <= int(t) <= 501 for t in a["token_num"].tolist())
    perm = torch.randperm(B, generator=g)
    c = eng.forward_feats(feats[perm.to(DEV)].contiguous(), fl[perm.to(DEV)].contiguous(), want_taps=True)
    assert [a["ids"][int(i)] for i in perm] == c["ids"]
    assert torch.equal(a["enc"][perm.to(DEV)], c["enc"])


def test_plugin_inference_contract():
    """ParaformerB200.inference keeps Paraformer.inference's contract (model.py:534-697): results with key/token_int,
    meta_data['batch_data_time'] in audio seconds; ids identical to the golden reference ids."""
    import funasr_b200
    cfg, wseed, wavs, cmvn, g = load_case("tiny_ragged3")
    from test_abi_host import _tiny_conf
    m = funasr_b200.ParaformerB200(**_tiny_conf())
    m.load_state_dict(state_dict_for(cfg, wseed), strict=True)
    m.to(DEV).eval()
    fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6,
                                     dither=0.0, cmvn=cmvn)
    res, meta = m.inference([w.numpy() for w in wavs], key=["a", "b", "c"], tokenizer=None, frontend=fe, device=DEV)
    assert [r["key"] for r in res] == ["a", "b", "c"]
    assert [t for r in res for t in r["token_int"]] == g["ids_flat"].tolist()
    assert abs(meta["batch_data_time"] - float(g["batch_data_time"])) < 1e-6
    # pred_timestamp (model.py:558,673-680): CIF fires -> [start_ms, end_ms] per token.  Expected values: the reference-pinned
    # host routine (tests/test_timestamps.py) applied to the ORACLE's CIF weights / fires for the same batch.
    from funasr_b200.timestamps import paraformer_timestamps
    res_t, _ = m.inference([w.numpy() for w in wavs], key=["a", "b", "c"], tokenizer=None, frontend=fe, device=DEV, pred_timestamp=True)
    ora = O.paraformer_forward(wavs, state_dict_for(cfg, wseed), cmvn, cfg.enc_layers, cfg.dec_layers)
    for i, r in enumerate(res_t):
        want = paraformer_timestamps(ora["peaks"][i].numpy(), ora["alphas"][i].numpy(), [str(t) for t in ora["ids"][i]])[1]
        assert len(r["timestamp"]) == len(r["token_int"]) and len(want) == len(r["timestamp"])
        assert all(a <= b for a, b in r["timestamp"])
        # this tiny fixture is exact (tools/parity_diag.py: 11/11 in both modes); the routine re-integrates the rescaled fire trace
        # with a hard threshold, so on long utterances a weight that differs from the CPU's in its last fp32 bits can move a stamp by
        # one 60 ms frame (full-depth fixture: 218/222 exact in fp32, 208/222 in the split mode — reported, not asserted to be 100 %)
        assert r["timestamp"] == want


# ------------------------------------------------------------------------------------------------ SenseVoiceSmall
@pytest.mark.parametrize("mode", ["fp32", "fp16x3", "fp16x6"])
@pytest.mark.parametrize("name", list(SV_CASES))
def test_sensevoice_vs_reference_golden(name, mode):
    """BASELINE config 4: query-frame prepend + 50+20 SAN-M blocks (eps 1e-5) + CTC greedy vs the reference's outputs."""
    from funasr_b200 import synth
    from funasr_b200.engine import SenseVoiceEngine
    cfg, wseed, wavs, cmvn, g = load_sv_case(name)
    eng = SenseVoiceEngine(synth.make_sensevoice_state_dict(cfg, wseed), cfg, DEV, gemm_mode=mode, cmvn=cmvn)
    lens = [w.numel() for w in wavs]
    pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
    o = eng.forward_wav(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), lens, language_id=0, textnorm_id=15, want_taps=True)
    torch.cuda.synchronize()
    step = 7 if cfg.enc_layers > 10 else 1
    assert o["enc_lens"].cpu().tolist() == g["enc_lens"].tolist()
    assert rel_err(o["enc"][:, ::step].cpu().numpy(), g["enc"]) <= 1e-3
    assert rel_err(o["logp"][:, g["logp_rows"].tolist()].cpu().numpy(), g["logp_sel"]) <= 1e-3
    valid = np.arange(g["argmax"].shape[1])[None, :] < g["enc_lens"][:, None]
    assert (o["argmax"].cpu().numpy()[valid] == g["argmax"][valid]).all()
    assert [t for r in o["ids"] for t in r] == g["ids_flat"].tolist()            # CTC greedy ids: bit-exact
    assert [len(r) for r in o["ids"]] == g["ids_len"].tolist()


def test_sensevoice_plugin_inference():
    import funasr_b200
    from funasr_b200 import synth
    cfg, wseed, wavs, cmvn, g = load_sv_case("sv_tiny_ragged3")
    m = funasr_b200.SenseVoiceSmallB200(encoder="SenseVoiceEncoderSmallB200",
                                        encoder_conf=dict(output_size=512, attention_heads=4, linear_units=2048, num_blocks=cfg.enc_layers,
                                                          tp_blocks=cfg.tp_layers, input_layer="pe", kernel_size=11, sanm_shfit=0,
                                                          selfattention_layer_type="sanm"), input_size=560, vocab_size=cfg.vocab)
    m.load_state_dict(synth.make_sensevoice_state_dict(cfg, wseed), strict=True)
    m.to(DEV).eval()
    fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0, cmvn=cmvn)
    res, meta = m.inference([w.numpy() for w in wavs], key=["a", "b", "c"], tokenizer=None, frontend=fe, device=DEV, language="auto", use_itn=False)
    assert [t for r in res for t in r["token_int"]] == g["ids_flat"].tolist()


# ------------------------------------------------------------------------------------------- ContextualParaformer
@pytest.mark.parametrize("mode", ["fp32", "fp16x3", "fp16x6"])
@pytest.mark.parametrize("name", list(CTX_CASES))
def test_contextual_vs_reference_golden(name, mode):
    """BASELINE config 5 through the plugin class: hotword memory (torch LSTM, O(#hotwords)) + CUDA bias decoder."""
    import funasr_b200
    from funasr_b200 import synth
    from test_abi_host import _tiny_conf
    cfg, wseed, wavs, cmvn, hw, g = load_ctx_case(name)
    conf = _tiny_conf()
    conf["encoder_conf"]["num_blocks"] = cfg.enc_layers
    conf["decoder_conf"].update(num_blocks=cfg.dec_layers, att_layer_num=cfg.dec_layers)
    conf.update(decoder="ContextualParaformerDecoderB200", vocab_size=cfg.vocab, gemm_mode=mode)
    m = funasr_b200.ContextualParaformerB200(**conf)
    m.load_state_dict(synth.make_contextual_state_dict(cfg, wseed), strict=True)
    m.to(DEV).eval()
    hw_embed = m.encode_hotwords(hw)
    assert rel_err(hw_embed.cpu().numpy(), g["hw_embed"]) <= 1e-4
    fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0, cmvn=cmvn)
    res, meta = m.inference([w.numpy() for w in wavs], key=["u%d" % i for i in range(len(wavs))], tokenizer=None, frontend=fe,
                            device=DEV, hotword_ids=hw)
    assert [t for r in res for t in r["token_int"]] == g["ids_flat"].tolist()       # bit-exact greedy ids
    # log-probs through the stage API
    eng = m.engine(DEV)
    from funasr_b200.engine import num_lfr_frames
    lens = [w.numel() for w in wavs]
    pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
    feats, fl = fe.engine(DEV)(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), max(num_lfr_frames(n) for n in lens))
    out = eng.forward_feats(feats, fl, want_taps=True)
    assert out["token_num"].tolist() == g["token_num"].tolist()
    assert rel_err(out["logp"][:, g["logp_rows"].tolist()].cpu().numpy(), g["logp_sel"]) <= 1e-3


# fp16 (x1: one fp16 plane per operand, one P plane in attention) is the fast mode and does not meet the 1e-3 contract, so its ids
# are not asserted; these bounds catch a broken single-plane path (a wrong plane count or layout gives O(1) errors).  Worst case
# measured on an H100 80GB HBM3 (700 W): encoder 1.0e-3 (Paraformer; contextual 7.2e-4), selected log-probs 1.4e-3 (contextual;
# Paraformer 1.1e-3).
X1_ENC_TOL, X1_LOGP_TOL = 4e-3, 5e-3


@pytest.mark.parametrize("model", ["paraformer", "contextual"])
def test_fp16_single_plane_mode_stays_bounded(model):
    """The tiny Paraformer and contextual fixtures in fp16 (x1): outputs finite, encoder output against the golden encoder (the
    contextual fixture has none: against the same model in fp32) and the selected log-probs against the golden ones."""
    from funasr_b200.engine import num_lfr_frames
    if model == "paraformer":
        cfg, wseed, wavs, cmvn, g = load_case("tiny_ragged3")
        o = _run_model(cfg, wseed, wavs, cmvn, "fp16")
        enc, enc_ref = o["enc"].cpu().numpy(), g["enc"]
    else:
        import funasr_b200
        from funasr_b200 import synth
        from test_abi_host import _tiny_conf
        cfg, wseed, wavs, cmvn, hw, g = load_ctx_case("ctx_tiny_ragged3")
        lens = [w.numel() for w in wavs]
        pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
        fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0,
                                         cmvn=cmvn)
        feats, fl = fe.engine(DEV)(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), max(num_lfr_frames(n) for n in lens))
        outs = {}
        for mode in ("fp16", "fp32"):
            conf = _tiny_conf()
            conf["encoder_conf"]["num_blocks"] = cfg.enc_layers
            conf["decoder_conf"].update(num_blocks=cfg.dec_layers, att_layer_num=cfg.dec_layers)
            conf.update(decoder="ContextualParaformerDecoderB200", vocab_size=cfg.vocab, gemm_mode=mode)
            m = funasr_b200.ContextualParaformerB200(**conf)
            m.load_state_dict(synth.make_contextual_state_dict(cfg, wseed), strict=True)
            m.to(DEV).eval()
            eng = m.engine(DEV)
            eng.set_hotwords(m.encode_hotwords(hw))
            outs[mode] = eng.forward_feats(feats, fl, want_taps=True)
            torch.cuda.synchronize()
        o = outs["fp16"]
        enc, enc_ref = o["enc"].cpu().numpy(), outs["fp32"]["enc"].cpu().numpy()
    lp = o["logp"][:, g["logp_rows"].tolist()].cpu().numpy()
    assert np.isfinite(enc).all() and np.isfinite(o["logp"].cpu().numpy()).all()
    e_enc, e_lp = rel_err(enc, enc_ref), rel_err(lp, g["logp_sel"])
    print("fp16 %s: encoder rel err %.2e (bar %.0e), selected log-probs %.2e (bar %.0e)" % (model, e_enc, X1_ENC_TOL, e_lp, X1_LOGP_TOL))
    assert e_enc <= X1_ENC_TOL and e_lp <= X1_LOGP_TOL


# ------------------------------------------------------------------------------------------- config 3: ragged buckets
def test_config3_bucketed_ragged_vs_oracle():
    """BASELINE config 3 in miniature: a ragged list is length-bucketed (funasr_b200.batching), every bucket runs as one
    padded batch, results come back in input order and equal the oracle run on the same buckets (padded-batch semantics
    of the reference, incl. what the CIF conv reads at the first padded frame)."""
    from funasr_b200 import synth
    from funasr_b200.batching import bucket_by_length, run_bucketed
    from funasr_b200.engine import FrontendEngine, num_lfr_frames
    cfg = synth.PARAFORMER_TINY
    g = torch.Generator().manual_seed(99)
    lens = [int(x) for x in (8000 + 56000 * torch.rand(12, generator=g)).tolist()]
    wavs = [synth.make_wav(n, 70 + i, "speechlike") for i, n in enumerate(lens)]
    cmvn = synth.make_cmvn(cfg, 1)
    p = state_dict_for(cfg, 5)
    fe, eng = FrontendEngine(cmvn, DEV), _engine(cfg, 5, "fp16x3")

    def infer(batch):
        ln = [w.numel() for w in batch]
        pad = torch.nn.utils.rnn.pad_sequence(batch, batch_first=True).to(DEV)
        feats, fl = fe(pad, torch.tensor(ln, dtype=torch.int32, device=DEV), max(num_lfr_frames(n) for n in ln))
        return eng.forward_feats(feats, fl)["ids"]

    got = run_bucketed(wavs, infer, max_batch=4, max_frames=4 * 100)
    ref = run_bucketed(wavs, lambda b: O.paraformer_forward(b, p, cmvn, cfg.enc_layers, cfg.dec_layers)["ids"], max_batch=4, max_frames=4 * 100)
    assert got == ref
    assert len(bucket_by_length(lens, 4, 400)) >= 3


# ------------------------------------------------------------------------------------------------- edge cases
def test_long_utterance_60s_vs_oracle():
    """Maximum practical size of one VAD segment (60 s -> T = 1000 LFR frames, 8 query tiles, 16 key chunks): both
    precision paths against the oracle."""
    from funasr_b200 import synth
    cfg = synth.PARAFORMER_TINY
    wavs = [synth.make_wav(960000, 81, "speechlike"), synth.make_wav(700001, 82, "speechlike")]
    cmvn = synth.make_cmvn(cfg, 2)
    p = state_dict_for(cfg, 12)
    ref = O.paraformer_forward(wavs, p, cmvn, cfg.enc_layers, cfg.dec_layers)
    for mode in ("fp32", "fp16x3"):
        o = _run_model(cfg, 12, wavs, cmvn, mode)
        assert o["feat_lens"].cpu().tolist() == [1000, 729]
        assert o["token_num"].tolist() == ref["token_num"].tolist()
        assert rel_err(o["logp"].cpu().numpy(), ref["logp"].numpy()) <= 1e-3
        assert o["ids"] == ref["ids"]


def test_silence_and_minimum_length():
    """All-zero audio (log floor everywhere) and the shortest supported utterance (one 25 ms frame -> one LFR frame):
    token counts and ids follow the oracle; a batch whose largest token count is 0 yields empty results like
    Paraformer.inference (model.py:615-616)."""
    import funasr_b200
    from funasr_b200 import synth
    from test_abi_host import _tiny_conf
    cfg = synth.PARAFORMER_TINY
    wavs = [torch.zeros(16000), synth.make_wav(400, 83, "noise"), synth.make_wav(24000, 84, "speechlike")]
    cmvn = synth.make_cmvn(cfg, 2)
    p = state_dict_for(cfg, 12)
    ref = O.paraformer_forward(wavs, p, cmvn, cfg.enc_layers, cfg.dec_layers)
    o = _run_model(cfg, 12, wavs, cmvn, "fp16x3")
    assert o["token_num"].tolist() == ref["token_num"].tolist()
    assert o["ids"] == ref["ids"]
    # a predictor that never fires: bias -> very negative => alpha ~ 0, tail 0.45 < 1 => zero tokens everywhere
    p2 = dict(p)
    p2["predictor.cif_output.bias"] = torch.full((1,), -30.0)
    m = funasr_b200.ParaformerB200(**_tiny_conf())
    m.load_state_dict(p2, strict=True)
    m.to(DEV).eval()
    fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0, cmvn=cmvn)
    results, meta = m.inference([w.numpy() for w in wavs], key=["a", "b", "c"], tokenizer=None, frontend=fe, device=DEV)
    assert results == []                                   # model.py:615-616: `return []` when no utterance has a token
    assert abs(meta["batch_data_time"] - sum(max(1, -(-(1 + (w.numel() - 400) // 160) // 6)) for w in wavs) * 0.06) < 1e-9
    ref2 = O.paraformer_forward(wavs, p2, cmvn, cfg.enc_layers, cfg.dec_layers)
    assert int(ref2["token_num"].max()) == 0 and ref2["ids"] == [[], [], []]


def test_abi_status_codes():
    """The C ABI reports problems as negative status codes (no exceptions, no silent fallback): bad arguments (-1),
    workspace too small (-3), unsupported shapes (-4); the Python layer turns them into FunasrB200Error."""
    abi, lib = _lib()
    from funasr_b200 import synth
    cfg = synth.PARAFORMER_TINY
    eng = _engine(cfg, 5, "fp16x3")
    B, T = 2, 40
    feats = torch.randn(B, T, 560, device=DEV)
    lens = torch.tensor([40, 17], dtype=torch.int32, device=DEV)
    out = torch.empty(B, T, 512, device=DEV)
    need = lib.fa_sanm_encoder_workspace_bytes(B, T, eng.mode)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    ok = lib.fa_sanm_encoder_forward(C.byref(eng.enc), feats.data_ptr(), lens.data_ptr(), B, T, out.data_ptr(), eng.mode, ws.data_ptr(), need, _st())
    assert ok == 0
    assert lib.fa_sanm_encoder_forward(C.byref(eng.enc), feats.data_ptr(), lens.data_ptr(), B, T, out.data_ptr(), eng.mode, ws.data_ptr(), need // 4, _st()) == -3
    assert lib.fa_sanm_encoder_forward(C.byref(eng.enc), None, lens.data_ptr(), B, T, out.data_ptr(), eng.mode, ws.data_ptr(), need, _st()) == -1
    assert lib.fa_sanm_encoder_forward(C.byref(eng.enc), feats.data_ptr(), lens.data_ptr(), 0, T, out.data_ptr(), eng.mode, ws.data_ptr(), need, _st()) == -1
    nm = abi.FaNorm(feats.data_ptr(), feats.data_ptr(), 4100, 1e-12)       # rows longer than the kernel supports
    assert lib.fa_layernorm(feats.data_ptr(), 4, C.byref(nm), out.data_ptr(), None, 1.0, 1, _st()) == -4
    assert lib.fa_fbank_lfr_cmvn_tables(None, None, 1, 0, None, None, 7, 6, None, 1, None, 1, _st()) == -1
    with pytest.raises(abi.FunasrB200Error):
        abi.check(-3, "demo")
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_offline_handle_api_vs_reference_golden(tmp_path, mode):
    """fa_offline_init / fa_offline_infer (the funasrruntime.h-style C handle API: no torch on the data path, weights from the
    flat file written by pack.py) reproduces the unmodified reference's greedy ids on the ragged golden batch — float32 and
    int16 PCM input."""
    from funasr_b200 import pack
    from funasr_b200.offline import OfflineRecognizer
    cfg, wseed, wavs, cmvn, g = load_case("tiny_ragged3")
    path = str(tmp_path / "m.fab2")
    pack.write_model_file(path, state_dict_for(cfg, wseed), cfg, cmvn)
    rec = OfflineRecognizer(path, 0, mode)
    ids = rec.infer([w.numpy() for w in wavs])
    assert [t for r in ids for t in r] == g["ids_flat"].tolist()
    assert [len(r) for r in ids] == g["ids_len"].tolist()
    assert abs(rec.last_audio_seconds - sum(w.numel() for w in wavs) / 16000.0) < 1e-3
    # second call on the same handle (buffers are reused), different batch composition
    ids2 = rec.infer([wavs[1].numpy()])
    assert ids2[0] == ids[1]
    # int16 PCM: identical to the float path on the dequantised waveform
    pcm = [np.clip(np.round(w.numpy() * 32768.0), -32768, 32767).astype(np.int16) for w in wavs]
    deq = [p.astype(np.float32) / 32768.0 for p in pcm]
    assert rec.infer(pcm) == rec.infer(deq)
    rec.close()
    with pytest.raises(Exception):
        OfflineRecognizer(str(tmp_path / "missing.fab2"), 0, mode)


# ------------------------------------------------------------------------------------------------ BiCifParaformer
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("name", ["bicif_tiny_ragged3", "bicif_large_single"])
def test_bicif_vs_reference_golden(name, mode):
    """BiCifParaformer (SURVEY §8f rank 1) against the unmodified reference: CifPredictorV3's sequential fp32 `cif` on the token
    branch (fa_cif_predictor_forward, cif_variant 1), the upsampled timestamp head (ConvTranspose1d as a GEMM of this library,
    the BLSTM fa_blstm_forward_tc, fa_cif_upsample_alphas) and the per-token [start_ms, end_ms] the reference derives from it."""
    from conftest import gold_stamps, load_bicif_case
    from funasr_b200 import synth
    from funasr_b200.engine import FrontendEngine, ParaformerEngine
    from funasr_b200.timestamps import ts_prediction_lfr6_standard
    cfg, wseed, wavs, cmvn, g = load_bicif_case(name)
    eng = ParaformerEngine(synth.make_bicif_state_dict(cfg, wseed), cfg, DEV, gemm_mode=mode, bicif=True)
    fe = FrontendEngine(cmvn, DEV)
    lens = [w.numel() for w in wavs]
    pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
    from funasr_b200.engine import num_lfr_frames
    feats, fl = fe(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), max(num_lfr_frames(n) for n in lens))
    o = eng.forward_feats(feats, fl, want_taps=True)
    assert o["token_num"].tolist() == g["token_num"].tolist()
    assert np.abs(o["alphas"].cpu().numpy() - g["alphas"]).max() <= 1e-4
    assert np.abs(o["peaks"].cpu().numpy() - g["peaks"]).max() <= 2e-3          # running fp32 integral of ~T alphas
    n = int(g["token_num"].max())
    assert rel_err(o["acoustic"][:, :n, ::5].cpu().numpy(), g["acoustic"]) <= 1e-3
    assert rel_err(o["logp"][:, g["logp_rows"].tolist(), :].cpu().numpy(), g["logp_sel"]) <= 1e-3
    assert [t for r in o["ids"] for t in r] == g["ids_flat"].tolist()           # greedy ids: bit-exact
    tok = torch.tensor(g["token_num"], dtype=torch.int32, device=DEV)
    us_alphas, us_peaks = eng.upsample_timestamp(o["enc"], fl, tok)
    assert rel_err(us_alphas.cpu().numpy(), g["us_alphas"]) <= 1e-3
    want = gold_stamps(g)
    ua, up = us_alphas.cpu().numpy(), us_peaks.cpu().numpy()
    for i, ids in enumerate(o["ids"]):
        m = int(g["enc_lens"][i]) * 3
        got = ts_prediction_lfr6_standard(ua[i][:m], up[i][:m], ["t%d" % (t - 3) for t in ids])[1]
        # integer milliseconds: bit-exact in both precision modes (round 2: the timestamp rescale token_num / alphas2.sum(-1) now
        # follows torch's fp32 summation order, which removed the one-frame differences round 1 tolerated)
        assert got == want[i], (i, [(a, b) for a, b in zip(got, want[i]) if a != b][:3])


@pytest.mark.gpu
def test_bicif_plugin_inference_timestamps():
    """BiCifParaformerB200.inference keeps BiCifParaformer.inference's contract: token ids + "timestamp" per token."""
    import funasr_b200
    from conftest import gold_stamps, load_bicif_case
    from funasr_b200 import synth
    from test_abi_host import _tiny_conf
    cfg, wseed, wavs, cmvn, g = load_bicif_case("bicif_tiny_ragged3")
    conf = _tiny_conf()
    conf["predictor"] = "CifPredictorV3B200"
    conf["predictor_conf"] = dict(idim=512, threshold=1.0, l_order=1, r_order=1, tail_threshold=cfg.tail_threshold, smooth_factor2=0.25,
                                  noise_threshold2=0.01, upsample_times=3, use_cif1_cnn=False, upsample_type="cnn_blstm")
    m = funasr_b200.BiCifParaformerB200(**conf)
    m.load_state_dict(synth.make_bicif_state_dict(cfg, wseed), strict=True)
    m.to(DEV).eval()
    fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6,
                                     dither=0.0, cmvn=cmvn)
    res, _ = m.inference([w.numpy() for w in wavs], key=["a", "b", "c"], tokenizer=None, frontend=fe, device=DEV)
    assert [t for r in res for t in r["token_int"]] == g["ids_flat"].tolist()
    want = gold_stamps(g)
    for r, w in zip(res, want):
        assert r["timestamp"] == w                                  # integer milliseconds: exact


@pytest.mark.gpu
@pytest.mark.parametrize("rates", [(8000, 16000), (48000, 16000), (44100, 16000)])
def test_resample_matches_torchaudio_algorithm(rates):
    """fa_resample against the torchaudio algorithm (pad (width, width + orig) zeros, conv1d with stride orig, truncate to
    ceil(new * len / orig)) evaluated on the CPU with the same table — ragged batch, per-row lengths."""
    from funasr_b200.resample import resample, sinc_resample_table
    o, n = rates
    tab, orig, new, width = sinc_resample_table(o, n)
    g = torch.Generator().manual_seed(5)
    lens = [o * 2 + 37, o + 1, 5000]
    wav = torch.zeros(len(lens), max(lens))
    for i, ln in enumerate(lens):
        wav[i, :ln] = torch.randn(ln, generator=g) * 0.3
    got, got_lens = resample(wav.to(DEV), torch.tensor(lens, dtype=torch.int32), o, n)
    kern = torch.from_numpy(tab)[:, None, :]
    for i, ln in enumerate(lens):
        x = torch.nn.functional.pad(wav[i:i + 1, :ln], (width, width + orig))
        ref = torch.nn.functional.conv1d(x[:, None], kern, stride=orig).transpose(1, 2).reshape(1, -1)
        tl = -(-new * ln // orig)
        assert int(got_lens[i]) == tl
        assert torch.allclose(got[i, :tl].cpu(), ref[0, :tl], atol=2e-6, rtol=1e-5)
        assert float(got[i, tl:].abs().max() if got.shape[1] > tl else 0.0) == 0.0
    try:
        import torchaudio
        # transforms.Resample precomputes the table in float64 like the reference's loader does (functional.resample on a float32
        # waveform would build it in float32)
        ta = torchaudio.transforms.Resample(o, n)(wav[0:1, :lens[0]])
        assert torch.allclose(got[0, :ta.shape[1]].cpu(), ta[0], atol=2e-6, rtol=1e-5)
    except ImportError:
        pass


@pytest.mark.gpu
def test_plugin_resamples_8k_input_like_the_reference_loader():
    """inference(fs=8000): the waveform is resampled on the GPU (load_utils.py:176-178 semantics) before the frontend; ids equal
    those obtained by resampling with the same algorithm on the CPU first."""
    import funasr_b200
    from funasr_b200.resample import sinc_resample_table
    from test_abi_host import _tiny_conf
    cfg, wseed, wavs, cmvn, g = load_case("tiny_ragged3")
    m = funasr_b200.ParaformerB200(**_tiny_conf())
    m.load_state_dict(state_dict_for(cfg, wseed), strict=True)
    m.to(DEV).eval()
    fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0, cmvn=cmvn)
    w8 = [w[::2].contiguous() for w in wavs]                       # pretend 8 kHz recordings
    res8, _ = m.inference([w.numpy() for w in w8], tokenizer=None, frontend=fe, device=DEV, fs=8000)
    tab, orig, new, width = sinc_resample_table(8000, 16000)
    kern = torch.from_numpy(tab)[:, None, :]
    up = []
    for w in w8:
        x = torch.nn.functional.pad(w[None], (width, width + orig))
        y = torch.nn.functional.conv1d(x[:, None], kern, stride=orig).transpose(1, 2).reshape(-1)
        up.append(y[: -(-new * w.numel() // orig)].contiguous())
    res16, _ = m.inference([w.numpy() for w in up], tokenizer=None, frontend=fe, device=DEV)
    assert [r["token_int"] for r in res8] == [r["token_int"] for r in res16]


def test_row_sum_matches_torch_cpu_order_bit_exact():
    """fa_row_sum_f32 (the summation order the CIF kernels use for floor(alphas.sum(-1)), cif_predictor.py:443-444, and for the
    timestamp rescale token_num / alphas2.sum(-1), bicif cif_predictor.py:343-345) equals torch's CPU fp32 sum bit for bit,
    including rows whose sum is within an ulp of an integer (where floor() flips with the order)."""
    abi, lib = _lib()
    g = np.random.default_rng(3)
    for n in [1, 5, 8, 33, 84, 101, 501, 502, 1001, 1500, 3001]:
        rows = 64
        x = (g.random((rows, n)) * 0.5).astype(np.float32)
        if n >= 84:        # drive every row's exact sum onto an integer
            s64 = x.astype(np.float64).sum(-1, keepdims=True)
            x = (x.astype(np.float64) * (np.round(s64) / s64)).astype(np.float32)
        want = torch.from_numpy(x).sum(-1)
        xd = torch.from_numpy(x).to(DEV)
        out = torch.empty(rows, device=DEV)
        abi.check(lib.fa_row_sum_f32(xd.data_ptr(), n, rows, n, out.data_ptr(), _st()), "fa_row_sum_f32")
        assert torch.equal(out.cpu(), want), n
        assert torch.equal(torch.floor(out.cpu()), torch.floor(want))


# ------------------------------------------------------------------------------------ the benchmark configuration itself
def test_full_depth_b64_30s_ids_equal_oracle():
    """BASELINE config 2 exactly as bench.py runs it — the full 50 + 16-layer model, 64 x 30 s, fp16x3 — against the oracle on the
    same 64 utterances: token counts and greedy ids of ALL 64 bit-exact, log-probs of two utterances within 1e-3."""
    import bench
    from funasr_b200 import synth
    from funasr_b200.engine import FrontendEngine, ParaformerEngine
    cfg = synth.PARAFORMER_LARGE
    wavs_map, n_all = bench.job_waveforms(2, 0, 1)
    wavs = [wavs_map[i] for i in range(64)]
    cmvn = synth.make_cmvn(cfg, 1)
    p = state_dict_for(cfg, 0)
    eng = ParaformerEngine(p, cfg, DEV, gemm_mode="fp16x3")
    fe = FrontendEngine(cmvn, DEV)
    pad = torch.stack(wavs).to(DEV)
    lens = torch.full((64,), 480000, dtype=torch.int32, device=DEV)
    feats, fl = fe(pad, lens, 500)
    out = eng.forward_feats(feats, fl)
    torch.cuda.synchronize()
    want_ids, want_tok, ref_lp, min_margin, max_abs_lp = [], [], None, [], 0.0
    torch.set_num_threads(max(1, min(32, bench.usable_cpus())))
    for b0 in range(0, 64, 8):                              # equal lengths: a batch of 8 is 8 independent utterances (no padding)
        o = O.paraformer_forward(wavs[b0:b0 + 8], p, cmvn, cfg.enc_layers, cfg.dec_layers)
        want_ids += o["ids"]
        want_tok += o["token_num"].tolist()
        top2 = torch.topk(o["logp"], 2, dim=-1).values
        for k in range(8):
            nk = int(o["token_num"][k])
            min_margin.append(float((top2[k, :nk, 0] - top2[k, :nk, 1]).min()))
        max_abs_lp = max(max_abs_lp, float(o["logp"].abs().max()))
        if b0 == 0:
            ref_lp = o["logp"][:2]
    assert out["token_num"].tolist() == want_tok             # CIF token counts: exact for all 64
    assert sum(len(r) for r in want_ids) > 64 * 100          # a meaningful number of tokens (synthetic weights: ~160 per utterance)
    taps = eng.forward_feats(feats[:2].contiguous(), fl[:2].contiguous(), want_taps=True)
    n = min(ref_lp.shape[1], taps["logp"].shape[1])
    assert rel_err(taps["logp"][:, :n].cpu().numpy(), ref_lp[:, :n].numpy()) <= 1e-3
    # greedy ids, token by token over all ~10 000 tokens.  An arg-max is only a well-defined function of the input where the
    # reference's own top-2 margin exceeds the floating-point deviation the contract allows (1e-3 of max |logp|); the reference
    # itself moves log-probs by 3e-5 between 1 and 8 MKL threads.  So: every utterance whose smallest margin is above that bound
    # must match exactly, any difference must sit on a token whose oracle margin is inside the bound, and there must be few.
    bound = 2e-3 * max_abs_lp
    bad = [i for i in range(64) if out["ids"][i] != want_ids[i]]
    print("B=64 parity: %d tokens, %d utterances differ %s; min margins of those: %s (bound %.3g)" % (
        sum(len(r) for r in want_ids), len(bad), bad, ["%.2e" % min_margin[i] for i in bad], bound))
    flipped = 0
    for i in bad:
        assert min_margin[i] <= bound, "utterance %d differs although its smallest top-2 margin is %.3g" % (i, min_margin[i])
        assert len(out["ids"][i]) == len(want_ids[i])
        k = sum(a != b for a, b in zip(out["ids"][i], want_ids[i]))
        assert k <= 2
        flipped += k
    # measured: the tensor-core path's log-probs deviate by up to ~1e-2 absolute (3e-4 of max |logp|, against the 1e-3 the contract
    # allows) — dominated by the tensor cores' accumulation rounding, not by the fp16 operand split (tools/noise_probe.py) — and the
    # top-2 margins of random-weight logits are exponentially distributed from zero, so ~1 token per 1000 sits inside the noise
    assert flipped <= 0.003 * sum(len(r) for r in want_ids), "more near-tie flips than the arithmetic noise explains: %s" % bad


def test_two_handles_two_threads_and_shared_hotword_memory(tmp_path):
    """The handle API as a server uses the reference's (one recogniser per worker thread): two fa_offline handles driven
    concurrently from two host threads (each on its own stream; the encoder's side-stream fork/join is per caller stream) give
    the same ids as sequential calls."""
    import threading
    from funasr_b200 import pack
    from funasr_b200.offline import OfflineRecognizer
    cfg, wseed, wavs, cmvn, g = load_case("tiny_ragged3")
    path = str(tmp_path / "m.fab2")
    pack.write_model_file(path, state_dict_for(cfg, wseed), cfg, cmvn)
    recs = [OfflineRecognizer(path, 0, "fp16x3") for _ in range(2)]
    want = recs[0].infer([w.numpy() for w in wavs])
    assert [t for r in want for t in r] == g["ids_flat"].tolist()
    results, errors = [None, None], []

    def work(k):
        try:
            for _ in range(6):
                got = recs[k].infer([w.numpy() for w in wavs])
                if got != want:
                    errors.append((k, got))
            results[k] = got
        except Exception as e:  # pragma: no cover
            errors.append((k, repr(e)))

    th = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors[:1]
    assert results[0] == want and results[1] == want
    for r in recs:
        r.close()


def test_contextual_many_hotwords_short_utterance():
    """More hotwords than encoder frames (a 100-entry list with a 2 s utterance, T = 33): the hotword memory is attended as ONE
    shared k/v copy, so its size is independent of t_max (the round-1 kernel replicated it per utterance and refused this)."""
    import funasr_b200
    from funasr_b200 import synth
    from test_abi_host import _tiny_conf
    cfg = synth.PARAFORMER_TINY
    wavs = [synth.make_wav(32000, 91, "speechlike"), synth.make_wav(20000, 92, "speechlike")]
    cmvn = synth.make_cmvn(cfg, 1)
    p = synth.make_contextual_state_dict(cfg, 6)
    hw = synth.make_hotwords(100, cfg.vocab, seed=11)
    ref = O.contextual_forward(wavs, p, cmvn, cfg.enc_layers, cfg.dec_layers, hw)
    for mode in ("fp32", "fp16x3"):
        conf = _tiny_conf()
        conf.update(decoder="ContextualParaformerDecoderB200", gemm_mode=mode)
        m = funasr_b200.ContextualParaformerB200(**conf)
        m.load_state_dict(p, strict=True)
        m.to(DEV).eval()
        fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0, cmvn=cmvn)
        res, _ = m.inference([w.numpy() for w in wavs], key=["a", "b"], tokenizer=None, frontend=fe, device=DEV, hotword_ids=hw)
        assert [r["token_int"] for r in res] == ref["ids"], mode


# ------------------------------------------------------------------------------------------------ SeacoParaformer
@pytest.mark.parametrize("mode", ["fp32", "fp16x3", "fp16x6"])
@pytest.mark.parametrize("name", ["seaco_tiny_ragged3", "seaco_tiny_asf"])
def test_seaco_vs_reference_golden(name, mode):
    """SeacoParaformer (SURVEY §8f rank 1) on the GPU against the UNMODIFIED reference's `_seaco_decode_with_ASF` outputs
    (tests/golden/seaco_*.npz) and the oracle's stage taps: decoder hidden exit, 2-layer hotword LSTM, the SeACo decoder over the
    shared hotword memory (FFN 1024, FSMN k = 21), attention-score filtering (second case: 25 hotwords, nfilter 8), the
    hotword_output_layer and the NO_BIAS merge.  Greedy ids bit-exact; merged log-probs within 1e-3."""
    from conftest import load_seaco_case
    from funasr_b200 import synth
    from funasr_b200.engine import FrontendEngine, ParaformerEngine, num_lfr_frames
    cfg, wseed, wavs, cmvn, hw, nfilter, g = load_seaco_case(name)
    p = synth.make_seaco_state_dict(cfg, wseed)
    ora = O.seaco_forward(wavs, p, cmvn, cfg.enc_layers, cfg.dec_layers, hw, synth.seaco_no_bias_id(cfg), nfilter=nfilter)
    eng = ParaformerEngine(p, cfg, DEV, gemm_mode=mode, seaco=True, no_bias=synth.seaco_no_bias_id(cfg))
    fe = FrontendEngine(cmvn, DEV)
    lens = [w.numel() for w in wavs]
    pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
    feats, fl = fe(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), max(num_lfr_frames(n) for n in lens))
    o = eng.forward_feats_seaco(feats, fl, hw, nfilter=nfilter, want_taps=True)
    torch.cuda.synchronize()
    assert o["token_num"].tolist() == g["token_num"].tolist()
    assert rel_err(o["hw_selected_all"].cpu().numpy(), g["hw_selected"]) <= 1e-4
    assert rel_err(o["dec_hidden"].cpu().numpy(), ora["dec_hidden"].numpy()) <= 1e-3
    if nfilter < len(hw):
        assert o["asf_picked"] == ora["asf_picked"]                                  # the same hotwords survive the filter, same order
    n = int(g["token_num"].max())
    assert rel_err(o["dha_pred"][:, :n].cpu().numpy(), ora["dha_pred"].numpy()) <= 1e-3
    assert rel_err(o["merged"][:, g["logp_rows"].tolist()].cpu().numpy(), g["merged_sel"]) <= 1e-3
    valid = np.arange(n)[None, :] < g["token_num"][:, None]
    assert (o["merged"][:, :n].argmax(-1).cpu().numpy()[valid] == g["argmax"][:, :n][valid]).all()
    assert [t for r in o["ids"] for t in r] == g["ids_flat"].tolist() and [len(r) for r in o["ids"]] == g["ids_len"].tolist()
    assert any(int(t) != 0 for t in (o["dha_ids"].cpu().numpy()[valid] != synth.seaco_no_bias_id(cfg)).tolist())    # the bias path is exercised


def test_seaco_plugin_inference_with_timestamps():
    """SeacoParaformerB200.inference keeps SeacoParaformer.inference's contract (model.py:422-581): token ids under hotword biasing
    plus per-token timestamps from the BiCif head; without hotwords it reduces to the plain decoder distribution (:381-382)."""
    import funasr_b200
    from conftest import load_seaco_case
    from funasr_b200 import synth
    from test_abi_host import _tiny_conf
    cfg, wseed, wavs, cmvn, hw, nfilter, g = load_seaco_case("seaco_tiny_asf")
    conf = _tiny_conf()
    conf["predictor"] = "CifPredictorV3B200"
    conf["predictor_conf"] = dict(idim=512, threshold=1.0, l_order=1, r_order=1, tail_threshold=cfg.tail_threshold, smooth_factor2=0.25,
                                  noise_threshold2=0.01, upsample_times=3, use_cif1_cnn=False, upsample_type="cnn_blstm")
    m = funasr_b200.SeacoParaformerB200(**conf, seaco_decoder="ParaformerSANMDecoder", inner_dim=512, NO_BIAS=synth.seaco_no_bias_id(cfg),
                                        seaco_decoder_conf=dict(attention_heads=4, linear_units=synth.SEACO_FFN, num_blocks=4,
                                                                kernel_size=synth.SEACO_KERNEL, sanm_shfit=0, use_output_layer=False,
                                                                wo_input_layer=True))
    p = synth.make_seaco_state_dict(cfg, wseed)
    m.load_state_dict(p, strict=True)
    m.to(DEV).eval()
    fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0, cmvn=cmvn)
    res, _ = m.inference([w.numpy() for w in wavs], key=["a", "b"], tokenizer=None, frontend=fe, device=DEV, hotword_ids=hw, nfilter=nfilter)
    assert [t for r in res for t in r["token_int"]] == g["ids_flat"].tolist()
    assert all(len(r["timestamp"]) == len(r["token_int"]) and all(a <= b for a, b in r["timestamp"]) for r in res)
    plain, _ = m.inference([w.numpy() for w in wavs], key=["a", "b"], tokenizer=None, frontend=fe, device=DEV)
    ref = O.bicif_forward(wavs, p, cmvn, cfg.enc_layers, cfg.dec_layers)
    assert [r["token_int"] for r in plain] == ref["ids"]


# ------------------------------------------------------------------------------------------------ FSMN-VAD + long audio
@pytest.mark.parametrize("name", ["vad_30s", "vad_130s", "vad_fixed800", "vad_random45", "vad_short", "vad_silence"])
def test_fsmn_vad_vs_reference_golden(name):
    """FSMN-VAD (SURVEY §8f rank 2) on the GPU against the UNMODIFIED reference (tests/golden/vad_*.npz from FsmnVADStreaming +
    WavFrontendOnline through AutoModel.generate): fused Fbank + LFR 5/1 + CMVN, the FSMN encoder and the frame energies in one pass
    over the whole waveform, the end-point detector on the host — silence posteriors within 1e-4, segment boundaries (integer
    milliseconds) bit-exact, through the plugin class."""
    import funasr_b200
    from funasr_b200 import synth
    from test_vad_host import VAD_CASES
    g = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz")))
    seconds, seed, pattern, kw = VAD_CASES[name]
    wav = synth.make_vad_wav(seconds, seed, pattern)
    c = synth.VAD_DEFAULT
    m = funasr_b200.FsmnVADStreamingB200(encoder="FSMN", encoder_conf=dict(
        input_dim=c.input_dim, input_affine_dim=c.input_affine_dim, fsmn_layers=c.fsmn_layers, linear_dim=c.linear_dim, proj_dim=c.proj_dim,
        lorder=c.lorder, rorder=0, lstride=1, rstride=0, output_affine_dim=c.output_affine_dim, output_dim=c.output_dim))
    m.load_state_dict(synth.make_vad_state_dict(c, 0), strict=True)
    m.to(DEV).eval()
    fe = funasr_b200.WavFrontendOnlineB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=5, lfr_n=1, dither=0.0,
                                           cmvn=synth.make_vad_cmvn(0))
    eng = m.engine(DEV, fe.cmvn)
    sil, db, sc = eng.scores(wav.to(DEV), want_scores=True)
    assert sil.numel() == g["sil_prob"].shape[0]
    if sil.numel():
        assert np.abs(sil.cpu().numpy() - g["sil_prob"]).max() <= 1e-4
        assert np.abs(sc[g["score_rows"].tolist()].cpu().numpy() - g["score_sel"]).max() <= 1e-4
        assert np.abs(db.cpu().numpy() - g["decibel"]).max() <= 1e-3
    res, meta = m.inference(wav.numpy(), key=["k"], frontend=fe, device=DEV, **kw)
    assert res[0]["key"] == "k" and res[0]["value"] == g["segments"].tolist()


@pytest.mark.parametrize("name", ["longaudio_40s", "longaudio_25s_onebatch"])
def test_long_audio_pipeline_vs_reference_golden(name):
    """The whole long-audio path against the UNMODIFIED reference's AutoModel(model=Paraformer, vad_model=FsmnVADStreaming)
    .generate() (inference_with_vad, auto_model.py:852-1035): VAD segments -> duration-sorted dynamic batches (batch_size_s) ->
    padded-batch decoding -> results restored to time order and concatenated; greedy ids of the whole recording bit-exact."""
    import funasr_b200
    from funasr_b200 import synth
    from test_abi_host import _tiny_conf
    sys_path_cases = {"longaudio_40s": (40.0, 7, [(3.0, 2.5), (1.5, 2.2), (4.0, 3.0), (2.0, 2.2), (6.0, 2.4)], {"batch_size_s": 6}),
                      "longaudio_25s_onebatch": (25.0, 8, [(2.0, 2.5), (3.0, 2.1)], {"batch_size_s": 300})}
    seconds, seed, pattern, kw = sys_path_cases[name]
    g = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz")))
    wav = synth.make_vad_wav(seconds, seed, pattern)
    assert wav.numel() == int(g["n_samples"])
    cfg = synth.PARAFORMER_TINY
    asr = funasr_b200.ParaformerB200(**_tiny_conf())
    asr.load_state_dict(synth.make_state_dict(cfg, 3), strict=True)
    asr.to(DEV).eval()
    asr_fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0,
                                         cmvn=synth.make_cmvn(cfg, 1))
    c = synth.VAD_DEFAULT
    vad = funasr_b200.FsmnVADStreamingB200(encoder="FSMN", encoder_conf=dict(
        input_dim=c.input_dim, input_affine_dim=c.input_affine_dim, fsmn_layers=c.fsmn_layers, linear_dim=c.linear_dim, proj_dim=c.proj_dim,
        lorder=c.lorder, rorder=0, lstride=1, rstride=0, output_affine_dim=c.output_affine_dim, output_dim=c.output_dim))
    vad.load_state_dict(synth.make_vad_state_dict(c, 0), strict=True)
    vad.to(DEV).eval()
    vad_fe = funasr_b200.WavFrontendOnlineB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=5, lfr_n=1,
                                               dither=0.0, cmvn=synth.make_vad_cmvn(0))
    pipe = funasr_b200.LongAudioPipeline(asr, asr_fe, vad, vad_fe, device=DEV)
    out = pipe.generate(wav.numpy(), key="rec", pred_timestamp=True, **kw)
    assert len(out["vad_segments"]) >= 2
    assert out["token_int"] == g["ids"].tolist()
    # timestamps of every segment are shifted by its start and stay inside it (auto_model.py:1008-1022)
    assert len(out["timestamp"]) == len(out["token_int"])
    assert all(a <= b for a, b in out["timestamp"]) and out["timestamp"][0][0] >= out["vad_segments"][0][0]
    assert out["timestamp"][-1][1] <= out["vad_segments"][-1][1] + 1000     # the last stamp ends with the segment's last (padded) LFR frame


# ------------------------------------------------------------------------------------ FunOffline* (C++ runtime surface)
def _cjk_tokens(vocab):
    return ["<blank>", "<s>", "</s>"] + [chr(0x4E00 + i) for i in range(3, vocab)]


def _write_wav16(path, wav):
    import struct
    pcm = np.clip(np.round(wav.numpy() * 32768.0), -32768, 32767).astype("<i2")
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 36 + pcm.nbytes) + b"WAVEfmt " + struct.pack("<IHHIIHH", 16, 1, 1, 16000, 32000, 2, 16))
        f.write(b"data" + struct.pack("<I", pcm.nbytes) + pcm.tobytes())
    return pcm


@pytest.mark.parametrize("contextual", [False, True])
def test_funoffline_cpp_client_end_to_end(tmp_path, contextual):
    """The C++ client (examples/offline_runtime_client.cpp: FunOfflineInit / CompileHotwordEmbedding / FunOfflineInfer /
    FunOfflineInferBuffer / FunASRGetResult ... with the reference runtime's signatures) on a model directory written by pack.py:
    the text it prints maps back to exactly the ids of the Python path on the same 16-bit audio — plain Paraformer, and
    ContextualParaformer with multi-token hotwords compiled by the shim's host LSTM (hw_emb -> the CUDA bias decoder)."""
    import subprocess
    import funasr_b200
    from funasr_b200 import pack, synth
    from test_abi_host import _tiny_conf
    cfg = synth.PARAFORMER_TINY
    cmvn = synth.make_cmvn(cfg, 1)
    wav = synth.make_wav(48000, 21 if contextual else 1, "speechlike")
    state = synth.make_contextual_state_dict(cfg, 6) if contextual else synth.make_state_dict(cfg, 3)
    mdir = tmp_path / "model"
    mdir.mkdir()
    pack.write_model_file(str(mdir / "model.fab2"), state, cfg, cmvn)
    toks = _cjk_tokens(cfg.vocab)
    (mdir / "tokens.txt").write_text("\n".join(toks) + "\n", encoding="utf-8")
    pcm = _write_wav16(str(tmp_path / "a.wav"), wav)
    deq = torch.from_numpy(pcm.astype(np.float32) / 32768.0)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "client")
    r = subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(root, "include"), os.path.join(root, "examples", "offline_runtime_client.cpp"),
                        "-L" + os.path.join(root, "funasr_b200"), "-lfunasr_b200", "-Wl,-rpath," + os.path.join(root, "funasr_b200"), "-o", exe],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-1500:]
    hw = synth.make_hotwords(5, cfg.vocab, seed=7)
    hot_str = " ".join("".join(toks[t] for t in h) for h in hw[:-1]) if contextual else ""
    r = subprocess.run([exe, str(mdir), str(tmp_path / "a.wav"), "fp16x3", hot_str], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-1500:]
    out = dict(ln.split(" ", 1) for ln in r.stdout.strip().splitlines() if " " in ln)
    ids_file = [toks.index(c) for c in out["file_result"].strip()]
    ids_buf = [toks.index(c) for c in out["buffer_result"].strip()]
    assert ids_file == ids_buf and len(ids_file) > 0
    assert abs(float(out["audio_seconds"]) - 2 * 3.0) < 1e-3
    # the Python path on the same dequantised audio
    conf = _tiny_conf()
    conf["gemm_mode"] = "fp16x3"
    fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0, cmvn=cmvn)
    if contextual:
        conf["decoder"] = "ContextualParaformerDecoderB200"
        m = funasr_b200.ContextualParaformerB200(**conf)
        m.load_state_dict(state, strict=True)
        m.to(DEV).eval()
        res, _ = m.inference([deq.numpy()], key=["a"], tokenizer=None, frontend=fe, device=DEV, hotword_ids=hw)
        assert int(out["hotword_rows"]) == len(hw)
    else:
        m = funasr_b200.ParaformerB200(**conf)
        m.load_state_dict(state, strict=True)
        m.to(DEV).eval()
        res, _ = m.inference([deq.numpy()], key=["a"], tokenizer=None, frontend=fe, device=DEV)
    assert ids_file == res[0]["token_int"]


def test_audio_decode_matches_host_decoding(tmp_path):
    """funasr_b200.audio (SURVEY §8f rank 4): WAV containers (PCM 8 / 16 / 24 / 32 bit, float32, stereo) decoded, mixed down and
    resampled on the GPU against the same decode done with numpy on the host (torchaudio.load(normalize=True) scaling, channel mean,
    load_utils.py:168-178) — and against torchaudio.load itself when its backend can read the file."""
    import struct
    from funasr_b200 import audio
    from funasr_b200.resample import sinc_resample_table
    g = np.random.default_rng(7)
    n = 8000
    x = np.clip(g.standard_normal((n, 2)) * 0.3, -0.99, 0.99)

    def wav_bytes(tag, bits, ch, rate, payload):
        blk = ch * bits // 8
        return (b"RIFF" + struct.pack("<I", 36 + len(payload)) + b"WAVEfmt " + struct.pack("<IHHIIHH", 16, tag, ch, rate, rate * blk, blk, bits) +
                b"data" + struct.pack("<I", len(payload)) + payload)

    cases = []
    s16 = np.round(x * 32767).astype("<i2")
    cases.append(("s16 stereo", wav_bytes(1, 16, 2, 16000, s16.tobytes()), s16.astype(np.float32).mean(1) / 32768.0, 16000))
    s32 = np.round(x[:, :1] * (2 ** 31 - 1)).astype("<i4")
    cases.append(("s32 mono", wav_bytes(1, 32, 1, 16000, s32.tobytes()), (s32[:, 0].astype(np.float64) / 2 ** 31).astype(np.float32), 16000))
    s24v = np.round(x[:, 0] * (2 ** 23 - 1)).astype(np.int32)
    s24 = b"".join(struct.pack("<i", int(v))[:3] for v in s24v)
    cases.append(("s24 mono", wav_bytes(1, 24, 1, 16000, s24), (s24v.astype(np.float64) / 2 ** 23).astype(np.float32), 16000))
    u8 = np.round(x[:, 0] * 127 + 128).astype(np.uint8)
    cases.append(("u8 mono", wav_bytes(1, 8, 1, 16000, u8.tobytes()), (u8.astype(np.float32) - 128.0) / 128.0, 16000))
    f32 = x.astype("<f4")
    cases.append(("f32 stereo 8k", wav_bytes(3, 32, 2, 8000, f32.tobytes()), f32.mean(1), 8000))
    for name, data, want, rate in cases:
        got = audio.load_audio(data, fs=16000, device=DEV)
        if rate == 16000:
            assert got.numel() == want.shape[0], name
            assert np.abs(got.cpu().numpy() - want).max() <= 1e-6, name
        else:                                                       # + resample (torchaudio's polyphase kernel, restated bit-exactly)
            tab, orig, new, width = sinc_resample_table(rate, 16000)
            xp = torch.nn.functional.pad(torch.from_numpy(want)[None], (width, width + orig))
            ref = torch.nn.functional.conv1d(xp[:, None], torch.from_numpy(tab)[:, None, :], stride=orig).transpose(1, 2).reshape(-1)
            tl = -(-new * want.shape[0] // orig)
            assert got.numel() == tl and torch.allclose(got.cpu(), ref[:tl], atol=2e-6, rtol=1e-5), name
    # a file path, and torchaudio as an independent decoder when available
    p = tmp_path / "a.wav"
    p.write_bytes(cases[0][1])
    got = audio.load_audio(str(p), device=DEV)
    try:
        import torchaudio
        ta, sr = torchaudio.load(str(p))
        assert sr == 16000 and torch.allclose(got.cpu(), ta.mean(0), atol=1e-6)
    except Exception:
        pass
    with pytest.raises(Exception):
        audio.load_audio(b"RIFFxxxxWAVEjunk", device=DEV)


# ------------------------------------------------------------------------------------------------ CT-Transformer punctuation

@pytest.mark.parametrize("name", ["punc_short", "punc_long", "punc_english_tail"])
def test_ct_transformer_vs_reference_golden(name):
    """CTTransformerB200.inference on the GPU (fa_embedding -> SANM encoder with 32-wide heads -> fa_linear_argmax) against the
    unmodified reference's AutoModel(model="CTTransformer").generate() for the same seeded weights and text: the punctuated text and
    the punctuation id per token are equal (integer outputs, bit-exact bar)."""
    import funasr_b200
    from funasr_b200 import synth
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    toks = synth.punc_token_list()
    t2i = {t: i for i, t in enumerate(toks)}

    class Tok:
        def encode(self, words):
            return [t2i.get(w, t2i["<unk>"]) for w in words]

    m = funasr_b200.CTTransformerB200(
        encoder="SANMEncoder",
        encoder_conf=dict(input_size=synth.PUNC_DIM, output_size=synth.PUNC_DIM, attention_heads=synth.PUNC_HEADS, linear_units=synth.PUNC_FFN,
                          num_blocks=synth.PUNC_LAYERS, kernel_size=11, sanm_shfit=0, input_layer="pe", normalize_before=True),
        vocab_size=len(toks), punc_list=synth.PUNC_LIST, punc_weight=[1.0] * len(synth.PUNC_LIST), embed_unit=synth.PUNC_DIM, att_unit=synth.PUNC_DIM,
        sentence_end_id=3)
    m.load_state_dict(synth.make_punc_state_dict(0), strict=True)
    m.to(DEV).eval()
    res, _ = m.inference([str(g["text_in"])], key=["k"], tokenizer=Tok(), device=DEV)
    assert res[0]["text"] == str(g["text_out"])
    assert res[0]["punc_array"].tolist() == g["punc_array"].tolist()


def test_utterances_shorter_than_one_frame_follow_the_reference_window_rule():
    """2 <= n < 400 samples: WavFrontend.forward passes frame_length = min(25 ms, len / fs) (wav_frontend.py:174), i.e. ONE window over
    the whole utterance, FFT size = next power of two.  The GPU frontend (fa_fbank_short beside the batched kernel) against the oracle's
    restatement of exactly that call — and against torchaudio's kaldi.fbank itself when it is importable — in a batch that mixes short
    and ordinary utterances; feat_lens = 1 for the short ones."""
    from funasr_b200 import synth
    from funasr_b200.engine import FrontendEngine, num_lfr_frames
    cfg = synth.PARAFORMER_TINY
    cmvn = synth.make_cmvn(cfg, 1)
    lens = [399, 3200, 256, 255, 100, 17, 2, 400]
    wavs = [synth.make_wav(n, 10 + i) for i, n in enumerate(lens)]
    ref_feats, ref_lens = O.frontend(wavs, cmvn)
    assert ref_lens.tolist() == [num_lfr_frames(n) for n in lens] == [1, 3, 1, 1, 1, 1, 1, 1]
    fe = FrontendEngine(cmvn, DEV)
    pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
    feats, fl = fe(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), max(num_lfr_frames(n) for n in lens), host_lens=lens)
    torch.cuda.synchronize()
    assert fl.tolist() == ref_lens.tolist()
    for b, n in enumerate(lens):
        t = int(ref_lens[b])
        got, want = feats[b, :t].cpu().numpy(), ref_feats[b, :t].numpy()
        # log-mel of near-empty bins sits on the transform's rounding floor (DESIGN.md §2): absolute 2e-3 there, 3e-5 relative elsewhere
        assert np.abs(got - want).max() <= 3e-5 * np.abs(want).max() + 2e-3, (n, np.abs(got - want).max())
        assert (feats[b, t:] == 0).all()
    try:
        import torchaudio.compliance.kaldi as K
    except Exception:
        return
    for b, n in enumerate(lens):
        if n >= 400:
            continue
        m = K.fbank(wavs[b][None] * 32768.0, num_mel_bins=80, frame_length=min(25, torch.tensor(n) / 16000 * 1000), frame_shift=10, dither=0.0,
                    energy_floor=0.0, window_type="hamming", sample_frequency=16000, snip_edges=True)
        want = ((m.repeat(1, 7) + cmvn[0]) * cmvn[1]).numpy()
        got = feats[b, :1].cpu().numpy()
        assert np.abs(got - want).max() <= 3e-5 * np.abs(want).max() + 2e-3, (n, np.abs(got - want).max())
