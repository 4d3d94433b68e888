"""GPU: diarized calls in the recogniser's request pool.  The ragged-batch spectral-clustering entries equal the single entries run set
by set, bit for bit; diarized calls pooled with plain long-audio and utterance calls get exactly what each gets alone; the reference
fixtures still hold through the pooled path; a speaker-stage refusal fails only its own call."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from funasr_b200 import _abi, pack, synth
from funasr_b200.offline import OfflineRecognizer, OfflineSpeaker, OfflineVad
from test_offline_concurrent_gpu import _long_wavs, _utts
from test_offline_stamps_gpu import BICIF_SEED, _bicif_file
from test_spk_host import SPK_CASES, campplus_state_dict, load_spk_case

CFG = synth.PARAFORMER_TINY
DEV = "cuda:0"
NS = [1, 2, 19, 20, 63, 64, 65, 200, 2047]
KS = [1, 2, 16, 7, 16, 3, 12, 16, 5]                 # vectors back-transformed per set (at most n)


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("pool_spk")
    cmvn = synth.make_cmvn(CFG, 1)
    out = {"asr": str(d / "asr.fab2"), "bicif": str(d / "bicif.fab2"), "vad": str(d / "vad.fab2"), "spk": str(d / "spk.fab2")}
    pack.write_model_file(out["asr"], synth.make_state_dict(CFG, 3), CFG, cmvn)
    _bicif_file(out["bicif"], CFG, BICIF_SEED, cmvn)
    pack.write_vad_model_file(out["vad"], synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    pack.write_campplus_model_file(campplus_state_dict(), out["spk"])
    return out


def _i32(v):
    return (C.c_int32 * len(v))(*v)


def _three_voices(n, seed):
    rng = np.random.RandomState(seed)
    centers = rng.randn(3, 192)
    return (centers[rng.randint(0, 3, size=n)] + 2.0 * rng.randn(n, 192)).astype(np.float32)


def _nan(n, dtype=torch.float64):
    return torch.full((n,), float("nan"), dtype=dtype, device=DEV)


def _ws(nbytes):
    return torch.full((int(nbytes) // 4 + 1,), float("nan"), dtype=torch.float32, device=DEV)


@pytest.mark.gpu
def test_batched_kernels_equal_single_entries_bit_for_bit():
    lib = _abi.load()
    st = torch.cuda.current_stream().cuda_stream
    ks = [min(k, n) for k, n in zip(KS, NS)]
    embs = [_three_voices(n, 100 + i) for i, n in enumerate(NS)]
    rng = np.random.RandomState(5)
    zs = [rng.randn(k, n) for k, n in zip(ks, NS)]
    # the single entries, set by set
    single = []
    for x, n, k, z in zip(embs, NS, ks, zs):
        emb = torch.from_numpy(x).to(DEV)
        lap = _nan(n * n)
        ws = _ws(max(lib.fa_spk_laplacian_workspace_bytes(n, 192), lib.fa_spk_tridiagonalize_workspace_bytes(n)))
        _abi.check(lib.fa_spk_laplacian(emb.data_ptr(), n, 192, 0.022, lap.data_ptr(), ws.data_ptr(), ws.numel() * 4, st), "fa_spk_laplacian")
        lap0 = lap.clone()
        d, e, tau = _nan(n), _nan(n), _nan(n)
        ws.fill_(float("nan"))
        _abi.check(lib.fa_spk_tridiagonalize(lap.data_ptr(), n, d.data_ptr(), e.data_ptr(), tau.data_ptr(), ws.data_ptr(), ws.numel() * 4, st),
                   "fa_spk_tridiagonalize")
        zd = torch.from_numpy(z).to(DEV).contiguous()
        _abi.check(lib.fa_spk_back_transform(lap.data_ptr(), tau.data_ptr(), n, zd.data_ptr(), k, st), "fa_spk_back_transform")
        single.append([t.cpu().numpy() for t in (lap0, lap, d, e, tau, zd.flatten())])
    # the batch
    S, rows, sq = len(NS), sum(NS), sum(n * n for n in NS)
    n_arr, k_arr = _i32(NS), _i32(ks)
    emb = torch.from_numpy(np.concatenate(embs)).to(DEV)
    lap = _nan(sq)
    ws = _ws(max(lib.fa_spk_laplacian_batch_workspace_bytes(n_arr, S, 192), lib.fa_spk_tridiagonalize_batch_workspace_bytes(n_arr, S)))
    _abi.check(lib.fa_spk_laplacian_batch(emb.data_ptr(), n_arr, S, 192, 0.022, lap.data_ptr(), ws.data_ptr(), ws.numel() * 4, st),
               "fa_spk_laplacian_batch")
    lap0 = lap.clone()
    d, e, tau = _nan(rows), _nan(rows), _nan(rows)
    ws.fill_(float("nan"))
    torch.cuda.synchronize()
    before = lib.fa_launch_count()
    _abi.check(lib.fa_spk_tridiagonalize_batch(lap.data_ptr(), n_arr, S, d.data_ptr(), e.data_ptr(), tau.data_ptr(), ws.data_ptr(), ws.numel() * 4, st),
               "fa_spk_tridiagonalize_batch")
    assert lib.fa_launch_count() - before == 3 * (max(NS) - 1) + 1
    zd = torch.from_numpy(np.concatenate([z.flatten() for z in zs])).to(DEV)
    _abi.check(lib.fa_spk_back_transform_batch(lap.data_ptr(), tau.data_ptr(), n_arr, k_arr, S, zd.data_ptr(), st), "fa_spk_back_transform_batch")
    got = [t.cpu().numpy() for t in (lap0, lap, d, e, tau, zd)]
    mo = vo = zo = 0
    for i, (n, k) in enumerate(zip(NS, ks)):
        s_lap0, s_lap, s_d, s_e, s_tau, s_z = single[i]
        assert np.array_equal(got[0][mo:mo + n * n], s_lap0), ("laplacian", n)
        assert np.array_equal(got[1][mo:mo + n * n], s_lap), ("reflectors", n)
        assert np.array_equal(got[2][vo:vo + n], s_d), ("d", n)
        assert np.array_equal(got[3][vo:vo + n - 1], s_e[:n - 1]), ("e", n)
        assert np.array_equal(got[4][vo:vo + n - 1], s_tau[:n - 1]), ("tau", n)
        assert np.array_equal(got[5][zo:zo + k * n], s_z), ("z", n, k)
        mo, vo, zo = mo + n * n, vo + n, zo + k * n
    torch.cuda.synchronize()


def _spk_wav(name):
    pattern, seed, _ = SPK_CASES[name]
    return synth.make_voice_wav(pattern, seed).numpy()


def _requests():
    """16 calls: diarized calls on each fixture recording with and without a preset count, one diarized call over several recordings,
    plain long-audio calls and utterance calls."""
    names = list(SPK_CASES)
    reqs = []
    for k in range(16):
        kind = k % 4
        if kind == 0:
            name = names[(k // 4) % len(names)]
            reqs.append(("spk", [_spk_wav(name)], SPK_CASES[name][2].get("preset_spk_num"), name))
        elif kind == 1:
            name = names[(k // 4 + 1) % len(names)]
            reqs.append(("spk", [_spk_wav(name)], 2 + k % 3, None))
        elif kind == 2:
            reqs.append(("long", [_long_wavs()[k % 3]], None, None))
        else:
            reqs.append(("utt", _utts(k), None, None))
    reqs[5] = ("spk", [_spk_wav(n) for n in names], None, None)
    return reqs


def _call(rec, vad, spk, r):
    kind, wavs, preset, _ = r
    if kind == "utt":
        return rec.infer_stamped(wavs)
    if kind == "long":
        return rec.infer_long(wavs, vad)
    return rec.infer_long(wavs, vad, spk=spk, preset_spk_num=preset)


def _stats(lib, rec):
    c, p = C.c_int64(-1), C.c_int64(-1)
    assert lib.fa_offline_pool_stats(rec.handle, C.byref(c), C.byref(p)) == 0
    return c.value, p.value


def _pooled(rec, first_call, calls):
    """first_call holds the handle while the calls are posted on threads of their own, so the next leader drains them together ->
    (first result, results or exceptions by call)."""
    out, first = [None] * len(calls), {}
    started = threading.Event()

    def lead():
        started.set()
        first["r"] = first_call()

    def run(k):
        try:
            out[k] = calls[k]()
        except _abi.FunasrB200Error as e:
            out[k] = e
    t0 = threading.Thread(target=lead)
    t0.start()
    started.wait()
    ts = [threading.Thread(target=run, args=(k,)) for k in range(len(calls))]
    for t in ts:
        t.start()
    for t in ts + [t0]:
        t.join()
    return first["r"], out


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("key", ["asr", "bicif"])
def test_pooled_diarized_calls_equal_each_call_alone(files, key, mode):
    lib = _abi.load()
    vad, spk = OfflineVad(files["vad"], 0), OfflineSpeaker(files["spk"], 0, mode)
    reqs = _requests()
    big = _long_wavs() * 3
    alone, packs_alone = [], 0
    for r in reqs + [("long", big, None, None)]:
        fresh = OfflineRecognizer(files[key], 0, mode)
        alone.append(_call(fresh, vad, spk, r))
        packs_alone += _stats(lib, fresh)[1]
        fresh.close()
    big_alone = alone.pop()
    rec = OfflineRecognizer(files[key], 0, mode)
    first, got = _pooled(rec, lambda: rec.infer_long(big, vad), [lambda r=r: _call(rec, vad, spk, r) for r in reqs])
    assert first == big_alone
    for k, (g, a) in enumerate(zip(got, alone)):
        assert g == a, (k, reqs[k][0], reqs[k][3])
    calls, packs = _stats(lib, rec)
    assert calls == 17 and packs < packs_alone, (calls, packs, packs_alone)
    # the reference fixtures through the pooled path
    for (kind, _, _, name), g in zip(reqs, got):
        if name is not None:
            gold = load_spk_case(name)
            assert g[0]["vad_segments"] == gold["segments"].tolist(), name
            assert g[0]["spk"] == [s["spk"] for s in gold["sentence_info"]], (name, g[0]["spk"])
    for h in (rec, vad, spk):
        h.close()


@pytest.mark.gpu
def test_speaker_refusal_among_pooled_calls_fails_alone(files):
    """A diarized call whose preset count exceeds its recording's chunk count fails on its own thread with the message it gets alone,
    and so does a call over several recordings whose second one is refused; the calls pooled with them get their alone results."""
    lib = _abi.load()
    vad, spk = OfflineVad(files["vad"], 0), OfflineSpeaker(files["spk"], 0, "fp16x3")
    bad = [("spk", [_spk_wav("spk_two_voices")], 1000, None),
           ("spk", [_spk_wav("spk_few_chunks"), _spk_wav("spk_two_voices"), _spk_wav("spk_three_preset")], 1000, None)]
    reqs = _requests()[:6] + bad
    alone = []
    for r in reqs:
        fresh = OfflineRecognizer(files["asr"], 0, "fp16x3")
        try:
            alone.append(_call(fresh, vad, spk, r))
        except _abi.FunasrB200Error as e:
            alone.append(e)
        fresh.close()
    assert all(isinstance(a, _abi.FunasrB200Error) for a in alone[6:])
    assert "recording 0: preset_spk_num 1000 exceeds the" in str(alone[6])
    assert "recording 1: preset_spk_num 1000 exceeds the" in str(alone[7])
    rec = OfflineRecognizer(files["asr"], 0, "fp16x3")
    _, got = _pooled(rec, lambda: rec.infer_long(_long_wavs() * 3, vad), [lambda r=r: _call(rec, vad, spk, r) for r in reqs])
    for k in range(6):
        assert got[k] == alone[k], k
    for k in (6, 7):
        assert isinstance(got[k], _abi.FunasrB200Error) and str(got[k]) == str(alone[k]), (got[k], alone[k])
    assert _stats(lib, rec)[0] == len(reqs) + 1
    for h in (rec, vad, spk):
        h.close()
