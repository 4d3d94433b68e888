"""Speaker diarization in the C handle API on the GPU: fa_spk_embed against CampplusEngine (bit for bit), the clustering kernels
(fa_spk_laplacian, fa_spk_tridiagonalize, fa_spk_back_transform) against numpy, fa_spk_cluster against ClusterBackend, and
fa_offline_infer_vad_spk against the reference's diarization fixtures."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from funasr_b200 import _abi, pack, synth
from funasr_b200 import diarization as D
from funasr_b200.long_audio import speaker_chunks
from funasr_b200.offline import OfflineRecognizer, OfflineSpeaker, OfflineVad
from test_spk_host import HOST_CLUSTER_CASES, SPK_CASES, campplus_state_dict, load_spk_case, vad_segments

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("spk")
    cfg = synth.PARAFORMER_TINY
    out = {"asr": str(d / "asr.fab2"), "vad": str(d / "vad.fab2"), "spk": str(d / "spk.fab2")}
    pack.write_model_file(out["asr"], synth.make_state_dict(cfg, 3), cfg, synth.make_cmvn(cfg, 1))
    pack.write_vad_model_file(out["vad"], synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    pack.write_campplus_model_file(campplus_state_dict(), out["spk"])
    return out


def _engine(mode):
    from funasr_b200.campplus import CAMPPlusB200
    m = CAMPPlusB200(gemm_mode=mode)
    m.load_state_dict(campplus_state_dict(), strict=True)
    return m


def _chunk_batch(name):
    pattern, seed, _ = SPK_CASES[name]
    wav = synth.make_voice_wav(pattern, seed).numpy()
    ch = speaker_chunks(vad_segments(load_spk_case(name)), wav.size)
    return [np.pad(wav[s:s + n], (0, 24000 - n)).astype(np.float32) for _, _, s, n in ch]


@pytest.mark.parametrize("mode", ["fp32", "fp16x3", "fp16"])
def test_embed_is_bit_identical_to_campplus_engine(files, mode):
    spk = OfflineSpeaker(files["spk"], 0, mode)
    m = _engine(mode)
    eng = m.engine(DEV)
    for name in SPK_CASES:
        chunks = _chunk_batch(name)
        batch = torch.from_numpy(np.stack(chunks)).to(DEV)
        n = len(chunks)
        want = eng.embed_wav(batch, torch.full((n,), 24000, dtype=torch.int32, device=DEV), [24000] * n).cpu().numpy()
        got = spk.embed(chunks)
        assert np.array_equal(got, want), (name, mode, np.abs(got - want).max())
    rng = np.random.RandomState(3)
    ragged = [(rng.randn(k) * 0.1).astype(np.float32) for k in (400, 7001, 24000, 51234, 16000)]
    want = m.inference(ragged, device=DEV)[0][0]["spk_embedding"].cpu().numpy()
    assert np.array_equal(spk.embed(ragged), want), mode
    pcm = [(w * 32767).astype(np.int16) for w in ragged]
    want16 = m.inference([p.astype(np.float32) / 32768.0 for p in pcm], device=DEV)[0][0]["spk_embedding"].cpu().numpy()
    assert np.array_equal(spk.embed(pcm), want16), mode
    spk.close()


def test_embed_refusals_happen_before_any_launch(files):
    spk = OfflineSpeaker(files["spk"], 0, "fp32")
    lib = spk.lib
    before = lib.fa_launch_count()
    with pytest.raises(_abi.FunasrB200Error, match="input 1 has 399 samples"):
        spk.embed([np.zeros(8000, np.float32), np.zeros(399, np.float32)])
    with pytest.raises(_abi.FunasrB200Error, match="input 0 has 18801 feature frames"):
        spk.embed([np.zeros(400 + 160 * 18800, np.float32), np.zeros(8000, np.float32)])
    assert lib.fa_launch_count() == before
    spk.close()


def _numpy_laplacian(x):
    sc = D.SpectralCluster()
    sim = sc.sim_mat(x)
    pruned = sc.p_pruning(sim.copy())
    return sc.laplacian(0.5 * (pruned + pruned.T))


def _device_laplacian(lib, x):
    n, dim = x.shape
    emb = torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(DEV)
    lap = torch.empty((n, n), dtype=torch.float64, device=DEV)
    ws = torch.empty(int(lib.fa_spk_laplacian_workspace_bytes(n, dim)), dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    _abi.check(lib.fa_spk_laplacian(emb.data_ptr(), n, dim, 0.022, lap.data_ptr(), ws.data_ptr(), ws.numel(), st), "fa_spk_laplacian")
    return lap


def _mixture(n, k, dim, seed, spread=1.0):
    rng = np.random.RandomState(seed)
    centers = rng.randn(k, dim)
    lab = rng.randint(0, k, size=n)
    return (centers[lab] + spread * rng.randn(n, dim)).astype(np.float32)


@pytest.mark.parametrize("n", [20, 120, 700, 2047])
def test_laplacian_matches_numpy(n):
    lib = _abi.load()
    x = _mixture(n, 3, 192, n, spread=3.0)
    lap = _device_laplacian(lib, x).cpu().numpy()
    ref = _numpy_laplacian(x).astype(np.float64)
    off = ~np.eye(n, dtype=bool)
    assert np.array_equal(lap[off] == 0, ref[off] == 0)        # the same entries pruned
    assert np.abs(lap - ref).max() <= 1e-6 * max(1.0, np.abs(ref).max())


def _device_eig(lib, lap_np, m=16, k=None):
    n = lap_np.shape[0]
    lap = torch.from_numpy(np.ascontiguousarray(lap_np, np.float64)).to(DEV)
    tri = torch.zeros(3 * n, dtype=torch.float64, device=DEV)
    ws = torch.empty(int(lib.fa_spk_tridiagonalize_workspace_bytes(n)), dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    _abi.check(lib.fa_spk_tridiagonalize(lap.data_ptr(), n, tri.data_ptr(), tri[n:].data_ptr(), tri[2 * n:].data_ptr(), ws.data_ptr(), ws.numel(), st),
               "fa_spk_tridiagonalize")
    de = tri.cpu().numpy()
    d, e = np.ascontiguousarray(de[:n]), np.ascontiguousarray(de[n:2 * n - 1])
    w = np.zeros(m)
    lib.fa_sym_tridiag_smallest_host(d.ctypes.data, e.ctypes.data, n, m, 0, w.ctypes.data, None)
    if k is None:
        k = int(np.argmax(np.diff(w))) + 1
    z = np.zeros((k, n))
    assert lib.fa_sym_tridiag_smallest_host(d.ctypes.data, e.ctypes.data, n, m, k, w.ctypes.data, z.ctypes.data) == 0
    zd = torch.from_numpy(z).to(DEV)
    _abi.check(lib.fa_spk_back_transform(lap.data_ptr(), tri[2 * n:].data_ptr(), n, zd.data_ptr(), k, st), "fa_spk_back_transform")
    return w, k, zd.cpu().numpy()


@pytest.mark.parametrize("n", [20, 120, 800, 2047])
def test_eigendecomposition_matches_numpy_eigh(n):
    lib = _abi.load()
    x = _mixture(n, 4, 192, 7 + n, spread=2.0)
    lap = _numpy_laplacian(x).astype(np.float64)
    w, k, z = _device_eig(lib, lap)
    ref_w, ref_v = np.linalg.eigh(lap)
    lnorm = np.abs(lap).sum(1).max()
    assert np.abs(w - ref_w[:16]).max() <= 1e-9 * lnorm, (n, np.abs(w - ref_w[:16]).max() / lnorm)
    assert k == int(np.argmax(np.diff(ref_w[:16]))) + 1
    V = ref_v[:, :k]
    assert np.abs(z.T @ z - V @ V.T).max() <= 1e-6, (n, np.abs(z.T @ z - V @ V.T).max())


@pytest.mark.parametrize("case", HOST_CLUSTER_CASES)
def test_cluster_matches_cluster_backend(files, case):
    g = np.load(os.path.join(GOLDEN, "spk_host_routines.npz"))
    x = np.ascontiguousarray(g[case + "__x"], np.float32)
    k = int(g[case + "__k"])
    if x.shape[1] != 192:                        # the handle's rows are 192 wide: zero columns change no norm or cosine
        x = np.ascontiguousarray(np.pad(x, ((0, 0), (0, 192 - x.shape[1]))))
    spk = OfflineSpeaker(files["spk"], 0, "fp32")
    lab = np.zeros(x.shape[0], np.int32)
    assert spk.lib.fa_spk_cluster(spk.handle, x.ctypes.data, x.shape[0], k if k > 0 else 0, lab.ctypes.data) == 0, spk.lib.fa_offline_last_error()
    assert D.correct_labels(lab).tolist() == D.correct_labels(g[case + "__labels"]).tolist()
    assert D.correct_labels(lab).tolist() == D.correct_labels(D.ClusterBackend()(x, oracle_num=k if k > 0 else None)).tolist()
    if x.shape[0] >= 2048:
        assert spk.lib.fa_spk_cluster(spk.handle, x.ctypes.data, x.shape[0], 0, lab.ctypes.data) != 0
        assert b"UMAP" in spk.lib.fa_offline_last_error()
    spk.close()


@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_infer_vad_spk_matches_reference_fixtures(files, mode):
    rec, vad, spk = OfflineRecognizer(files["asr"], 0, mode), OfflineVad(files["vad"], 0), OfflineSpeaker(files["spk"], 0, mode)
    for name, (pattern, seed, kw) in SPK_CASES.items():
        g = load_spk_case(name)
        wav = synth.make_voice_wav(pattern, seed).numpy()
        plain = rec.infer_long([wav], vad, batch_size_s=300)[0]
        got = rec.infer_long([wav], vad, batch_size_s=300, spk=spk, preset_spk_num=kw.get("preset_spk_num"))[0]
        assert got["vad_segments"] == g["segments"].tolist(), name
        assert got["spk"] == [s["spk"] for s in g["sentence_info"]], (name, got["spk"])
        assert {k: v for k, v in got.items() if k != "spk"} == plain, name
        assert rec.infer_long([wav], vad, batch_size_s=300)[0] == plain, name
    # two recordings in one call: each diarized on its own
    w0 = synth.make_voice_wav(*SPK_CASES["spk_two_voices"][:2]).numpy()
    w1 = synth.make_voice_wav(*SPK_CASES["spk_few_chunks"][:2]).numpy()
    both = rec.infer_long([w0, w1], vad, spk=spk)
    assert [b["spk"] for b in both] == [[s["spk"] for s in load_spk_case(n)["sentence_info"]] for n in ("spk_two_voices", "spk_few_chunks")]
    for h in (rec, vad, spk):
        h.close()
