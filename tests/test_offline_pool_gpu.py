"""GPU: rows with their own padded extent, and the recogniser's request pool.

The CIF predictor, the timestamp head and its BLSTM with a padded length ext per row (the _ext entries) give each row exactly what
the existing entries give it in a batch padded to ext.  Concurrent calls on one handle decoded in shared GPU packs give every call
exactly what it gets alone on a fresh handle, and the pool's counters show that calls shared packs."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from funasr_b200 import _abi
from funasr_b200.offline import OfflineRecognizer, OfflineVad
from test_decode_kernels_gpu import _blstm_weights, _blstm_xproj, _predictor_struct, _random_predictor
from test_offline_concurrent_gpu import _long_wavs, _utts, files  # noqa: F401 - the model files fixture

DEV = "cuda:0"
D = 512


def _st():
    return torch.cuda.current_stream().cuda_stream


def _i32(v):
    return (C.c_int32 * len(v))(*v)


def _cif(lib, pred, mode, enc, lens, ext=None):
    """fa_cif_predictor_forward (ext None) or fa_cif_predictor_forward_ext over NaN-filled outputs and workspace -> CPU tensors."""
    B, T, _ = enc.shape
    m = _abi.GEMM_MODES[mode]
    acoustic = torch.full((B, T + 1, D), float("nan"), device=DEV)
    tok = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    alphas = torch.full((B, T + 1), float("nan"), device=DEV)
    peaks = torch.full((B, T + 1), float("nan"), device=DEV)
    need = lib.fa_cif_predictor_workspace_bytes(B, T, m) if ext is None else lib.fa_cif_predictor_ext_workspace_bytes(B, T, m)
    ws = torch.full((int(need),), 255, dtype=torch.uint8, device=DEV)
    encd, lensd = enc.to(DEV).contiguous(), torch.tensor(lens, dtype=torch.int32, device=DEV)
    args = [C.byref(pred), encd.data_ptr(), lensd.data_ptr(), B, T, acoustic.data_ptr(), T + 1, tok.data_ptr(), alphas.data_ptr(),
            peaks.data_ptr(), m, ws.data_ptr(), ws.numel(), _st()]
    if ext is None:
        _abi.check(lib.fa_cif_predictor_forward(*args), "fa_cif_predictor_forward")
    else:
        _abi.check(lib.fa_cif_predictor_forward_ext(*args, _i32(lens), _i32(ext)), "fa_cif_predictor_forward_ext")
    torch.cuda.synchronize()
    return acoustic.cpu(), tok.cpu(), alphas.cpu(), peaks.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("variant", [0, 1])
def test_cif_predictor_ext_equals_batch_padded_to_ext(variant, mode):
    """Ragged rows with ext in [len, t_max] and nonzero encoder frames past every length: row b of fa_cif_predictor_forward_ext equals
    fa_cif_predictor_forward on a batch of that row padded to ext[b] frames (token count, alphas and peaks over ext + 1, the fired
    embeddings), bit for bit; ext = t_max everywhere equals fa_cif_predictor_forward."""
    lib = _abi.load()
    pred, keep = _predictor_struct(_abi, lib, mode, variant, *_random_predictor())
    g = torch.Generator().manual_seed(17)
    T = 61
    lens = [61, 13, 37, 1, 25, 40, 8]
    ext = [61, 20, 37, 9, 44, 61, 8]
    enc = torch.randn(len(lens), T, D, generator=g)
    got = _cif(lib, pred, mode, enc, lens, ext)
    for b, (n, e) in enumerate(zip(lens, ext)):
        one = _cif(lib, pred, mode, enc[b:b + 1, :e].contiguous(), [n])
        k = int(one[1][0])
        assert int(got[1][b]) == k, b
        assert torch.equal(got[2][b, :e + 1].view(torch.int32), one[2][0].view(torch.int32)), b
        assert torch.equal(got[3][b, :e + 1].view(torch.int32), one[3][0].view(torch.int32)), b
        assert torch.equal(got[0][b, :k].view(torch.int32), one[0][0, :k].view(torch.int32)), b
    full = _cif(lib, pred, mode, enc, lens, [T] * len(lens))
    ref = _cif(lib, pred, mode, enc, lens)
    for a, r in zip(full, ref):
        assert torch.equal(a.view(torch.int32), r.view(torch.int32))
    del keep


@pytest.mark.gpu
def test_blstm_ext_equals_each_sequence_alone():
    """fa_blstm_forward_tc_ext over ragged lengths (both directions from a zero state at each sequence's own end) equals
    fa_blstm_forward_tc on each sequence's first ext[b] steps alone, bit for bit; all lengths T equals fa_blstm_forward_tc; more than
    256 sequences and a length outside [1, T] are refused."""
    lib = _abi.load()
    wf, wb = [w.to(DEV) for w in _blstm_weights(1.0)]
    B, T = 70, 45
    ext = [45, 7, 23, 1, 45, 30] + [1 + (5 * b) % 45 for b in range(B - 6)]
    xp = _blstm_xproj(B, T, 1.0, 5).to(DEV).contiguous()
    scratch = torch.full((int(lib.fa_blstm_tc_ext_scratch_bytes(B)),), 255, dtype=torch.uint8, device=DEV)
    out = torch.full((B, T, 2 * D), float("nan"), device=DEV)
    assert lib.fa_blstm_forward_tc_ext(xp.data_ptr(), wf.data_ptr(), wb.data_ptr(), B, T, D, out.data_ptr(), scratch.data_ptr(),
                                       scratch.numel(), _st(), _i32(ext)) == 0
    for b in range(B):
        e = ext[b]
        x1 = xp[b:b + 1, :e].contiguous()
        one = torch.full((1, e, 2 * D), float("nan"), device=DEV)
        assert lib.fa_blstm_forward_tc(x1.data_ptr(), wf.data_ptr(), wb.data_ptr(), 1, e, D, one.data_ptr(), scratch.data_ptr(),
                                       scratch.numel(), _st()) == 0
        torch.cuda.synchronize()
        assert torch.equal(out[b, :e].view(torch.int32), one[0].view(torch.int32)), b
        assert torch.isnan(out[b, e:]).all(), b
    ref = torch.full((B, T, 2 * D), float("nan"), device=DEV)
    assert lib.fa_blstm_forward_tc(xp.data_ptr(), wf.data_ptr(), wb.data_ptr(), B, T, D, ref.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                   _st()) == 0
    assert lib.fa_blstm_forward_tc_ext(xp.data_ptr(), wf.data_ptr(), wb.data_ptr(), B, T, D, out.data_ptr(), scratch.data_ptr(),
                                       scratch.numel(), _st(), _i32([T] * B)) == 0
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int32), ref.view(torch.int32))
    assert lib.fa_blstm_forward_tc_ext(xp.data_ptr(), wf.data_ptr(), wb.data_ptr(), 257, 1, D, out.data_ptr(), scratch.data_ptr(),
                                       scratch.numel(), _st(), _i32([1] * 257)) == -4
    assert lib.fa_blstm_forward_tc_ext(xp.data_ptr(), wf.data_ptr(), wb.data_ptr(), 2, T, D, out.data_ptr(), scratch.data_ptr(),
                                       scratch.numel(), _st(), _i32([T + 1, 3])) == -1


def _stats(lib, rec):
    c, p = C.c_int64(-1), C.c_int64(-1)
    assert lib.fa_offline_pool_stats(rec.handle, C.byref(c), C.byref(p)) == 0
    return c.value, p.value


def _requests(k):
    """Request k of the mix: an utterance batch as s16 16 kHz, f32 44.1 kHz stereo or s16 8 kHz, or long audio with VAD."""
    utts = _utts(k)
    kind = k % 4
    if kind == 0:
        return ("utt", [np.clip(u * 32767, -32768, 32767).astype(np.int16) for u in utts], 16000)
    if kind == 1:
        return ("utt", [np.stack([u, 0.5 * u], 1).astype(np.float32) for u in utts], 44100)
    if kind == 2:
        return ("utt", [np.clip(u[::2] * 32767, -32768, 32767).astype(np.int16) for u in utts], 8000)
    return ("long", [_long_wavs()[k % 3]], 16000)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("key", ["asr", "bicif"])
def test_pooled_calls_equal_each_call_alone(files, key, mode):  # noqa: F811 - the fixture
    """One thread holds the handle with a long call while 16 others post mixed requests, so the next leader drains them together:
    every call's ids, stamps, segments and audio seconds equal the same call made alone on a fresh handle, and the pool decoded the
    calls in fewer GPU packs than the calls take alone."""
    lib = _abi.load()
    vad = OfflineVad(files["vad"], 0)
    reqs = [_requests(k) for k in range(16)]
    big = [w for w in _long_wavs()] * 3

    def call(rec, r):
        kind, wavs, fs = r
        if kind == "utt":
            return rec.infer_stamped(wavs, fs=fs)
        return rec.infer_long(wavs, vad, batch_size_s=6, fs=fs)
    alone, packs_alone = [], 0
    for r in reqs + [("long", big, 16000)]:
        fresh = OfflineRecognizer(files[key], 0, mode)
        alone.append(call(fresh, r))
        packs_alone += _stats(lib, fresh)[1]
        fresh.close()
    big_alone = alone.pop()
    rec = OfflineRecognizer(files[key], 0, mode)
    got = [None] * 16
    first = {}
    started = threading.Event()

    def lead():
        started.set()
        first["r"] = rec.infer_long(big, vad, batch_size_s=6)

    def run(k):
        got[k] = call(rec, reqs[k])
    t0 = threading.Thread(target=lead)
    t0.start()
    started.wait()
    ts = [threading.Thread(target=run, args=(k,)) for k in range(16)]
    for t in ts:
        t.start()
    for t in ts + [t0]:
        t.join()
    assert first["r"] == big_alone
    assert got == alone
    calls, packs = _stats(lib, rec)
    assert calls == 17 and packs < packs_alone, (calls, packs, packs_alone)
    rec.close()
    vad.close()


@pytest.mark.gpu
def test_bad_request_among_pooled_ones_fails_alone(files):  # noqa: F811 - the fixture
    """A call with a buffer under 400 samples fails on its own thread with its own message while pooled calls around it succeed with
    their alone results."""
    lib = _abi.load()
    rec = OfflineRecognizer(files["asr"], 0, "fp16x3")
    alone = [rec.infer(_utts(k)) for k in range(8)]
    errs = [None] * 8
    got = [None] * 8

    def run(k):
        if k == 3:
            buf = np.zeros(100, np.float32)
            ptrs = (C.c_void_p * 1)(buf.ctypes.data)
            lens = (C.c_int64 * 1)(100)
            r = lib.fa_offline_infer(rec.handle, ptrs, lens, 1, 0)
            errs[k] = (r, lib.fa_offline_last_error().decode())
            return
        got[k] = rec.infer(_utts(k))
    ts = [threading.Thread(target=run, args=(k,)) for k in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs[3][0] and "400 samples" in errs[3][1]
    assert [g for k, g in enumerate(got) if k != 3] == [a for k, a in enumerate(alone) if k != 3]
    rec.close()


def _engine(kind, mode):
    from funasr_b200 import synth
    from funasr_b200.engine import ParaformerEngine
    cfg = synth.PARAFORMER_LARGE if kind == "large" else synth.PARAFORMER_TINY
    sd = synth.make_bicif_state_dict(cfg, 5) if kind == "bicif" else synth.make_state_dict(cfg, 3)
    return ParaformerEngine(sd, cfg, DEV, gemm_mode=mode, bicif=kind == "bicif")


def _head_ext(lib, eng, enc, lens, tok, ext=None):
    """fa_timestamp_head_forward (ext None) or fa_timestamp_head_forward_ext over NaN-filled outputs and workspace -> CPU tensors."""
    B, T, _ = enc.shape
    U = eng.ts_head.up_times
    ua = torch.full((B, T * U), float("nan"), device=DEV)
    up = torch.full((B, T * U), float("nan"), device=DEV)
    q = lib.fa_timestamp_head_workspace_bytes if ext is None else lib.fa_timestamp_head_ext_workspace_bytes
    ws = torch.full((int(q(B, T, D, U, eng.mode)),), 255, dtype=torch.uint8, device=DEV)
    ld, td = torch.tensor(lens, dtype=torch.int32, device=DEV), torch.tensor(tok, dtype=torch.int32, device=DEV)
    args = [C.byref(eng.ts_head), enc.data_ptr(), ld.data_ptr(), td.data_ptr(), B, T, ua.data_ptr(), up.data_ptr(), eng.mode,
            ws.data_ptr(), ws.numel(), _st()]
    if ext is None:
        _abi.check(lib.fa_timestamp_head_forward(*args), "fa_timestamp_head_forward")
    else:
        _abi.check(lib.fa_timestamp_head_forward_ext(*args, _i32(lens), _i32(ext)), "fa_timestamp_head_forward_ext")
    torch.cuda.synchronize()
    return ua.cpu(), up.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_timestamp_head_ext_equals_batch_padded_to_ext(mode):
    """fa_timestamp_head_forward_ext over 260 ragged rows (two BLSTM launches, the second starting at row 256) with nonzero encoder
    frames past every length: each row's us_alphas / us_peaks over U * ext equal fa_timestamp_head_forward on that row padded to its
    ext, bit for bit; ext = t_max everywhere equals fa_timestamp_head_forward on the whole batch."""
    lib = _abi.load()
    eng = _engine("bicif", mode)
    U = eng.ts_head.up_times
    g = torch.Generator().manual_seed(23)
    B, T = 260, 40
    lens = torch.randint(1, T + 1, (B,), generator=g).tolist()
    ext = [n + int(torch.randint(0, T - n + 1, (1,), generator=g)) for n in lens]
    ext[-1] = lens[-1]                                      # the last launch's longest row shorter than T in most draws
    tok = torch.randint(1, 9, (B,), generator=g).tolist()
    enc = torch.randn(B, T, D, generator=g).to(DEV)
    ua, up = _head_ext(lib, eng, enc, lens, tok, ext)
    for b in range(B):
        e = ext[b]
        oa, op = _head_ext(lib, eng, enc[b:b + 1, :e].contiguous(), [lens[b]], [tok[b]])
        assert torch.equal(ua[b, :U * e].view(torch.int32), oa[0].view(torch.int32)), b
        assert torch.equal(up[b, :U * e].view(torch.int32), op[0].view(torch.int32)), b
    fa, fp = _head_ext(lib, eng, enc, lens, tok, [T] * B)
    ra, rp = _head_ext(lib, eng, enc, lens, tok)
    assert torch.equal(fa.view(torch.int32), ra.view(torch.int32)) and torch.equal(fp.view(torch.int32), rp.view(torch.int32))


def _stage_taps(lib, eng, feats, lens, ext):
    """The pooled decode of decode_batch, stage by stage: encoder, CIF predictor with per-row extents, decoder log-probs and, for BiCif,
    the timestamp head with per-row extents -> CPU tensors."""
    B, T, _ = feats.shape
    ld = torch.tensor(lens, dtype=torch.int32, device=DEV)
    enc = eng.encode(feats.to(DEV).contiguous(), ld)
    acoustic, tok, alphas, peaks = _cif(lib, eng.pred, eng.mode_name, enc, lens, ext)
    n_max = max(1, int(tok.max()))
    _, _, logp = eng.decode(enc, ld, acoustic.to(DEV).contiguous(), tok.to(DEV), n_max, want_logp=True)
    out = {"enc": enc.cpu(), "tok": tok, "alphas": alphas, "peaks": peaks, "acoustic": acoustic, "logp": logp.cpu()}
    if getattr(eng, "ts_head", None) is not None:
        out["us_alphas"], out["us_peaks"] = _head_ext(lib, eng, enc, lens, tok.tolist(), ext)
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind,mode", [("tiny", "fp32"), ("tiny", "fp16x3"), ("bicif", "fp32"), ("bicif", "fp16x3"), ("large", "fp16x3")])
def test_premise_row_alone_equals_row_in_pooled_packs(kind, mode):
    """The premise of the pool: a row decoded in its own reference pack (padded to ext) and the same row inside larger pooled packs
    (beside longer rows, shorter rows and a mix, extents up to 1000 frames) give the same encoder output over [0, ext), alphas, peaks,
    token count, acoustic embeddings, decoder log-probs and BiCif us_alphas / us_peaks, bit for bit."""
    lib = _abi.load()
    eng = _engine(kind, mode)
    eng.mode_name = mode
    g = torch.Generator().manual_seed(31)
    F = eng.cfg.feat_dim

    def feats_of(ns, T):
        x = torch.zeros(len(ns), T, F)
        for b, n in enumerate(ns):
            x[b, :n] = torch.randn(n, F, generator=g)
        return x
    for L, E in ((83, 121), (610, 1000), (400, 400)):
        own = feats_of([L, E], E)                           # the reference pack: the row beside a row of length E
        rows = {"longer": [1000, 1000], "shorter": [17, 5], "mixed": [3, 1000]}
        alone = _stage_taps(lib, eng, own, [L, E], [E, E])
        k = int(alone["tok"][0])
        for name, extra in rows.items():
            Tb = max(E, max(extra))
            x = torch.zeros(4, Tb, F)
            x[0, :E] = own[1]                              # the companion row, then the target row, then the other call's rows
            x[1, :E] = own[0]
            x[2:] = feats_of(extra, Tb)
            got = _stage_taps(lib, eng, x, [E, L] + extra, [E, E] + extra)
            where = (kind, mode, L, E, name)
            assert torch.equal(got["enc"][1, :E].view(torch.int32), alone["enc"][0, :E].view(torch.int32)), where
            assert int(got["tok"][1]) == k, where
            for key in ("alphas", "peaks"):
                assert torch.equal(got[key][1, :E + 1].view(torch.int32), alone[key][0, :E + 1].view(torch.int32)), (where, key)
            assert torch.equal(got["acoustic"][1, :k].view(torch.int32), alone["acoustic"][0, :k].view(torch.int32)), where
            assert torch.equal(got["logp"][1, :k].view(torch.int32), alone["logp"][0, :k].view(torch.int32)), where
            if "us_alphas" in alone:
                U = eng.ts_head.up_times
                for key in ("us_alphas", "us_peaks"):
                    assert torch.equal(got[key][1, :U * E].view(torch.int32), alone[key][0, :U * E].view(torch.int32)), (where, key)
