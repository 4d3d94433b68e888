"""Speaker diarization in the C handle API, host side: the CAM++ model file (pack.write_campplus_model_file) and fa_spk_init's refusals
before any device work, and the host routines of the clustering (fa_sym_tridiag_smallest_host, fa_spk_kmeans_host,
fa_spk_merge_by_cos_host, fa_spk_postprocess_host, fa_spk_distribute_host) against funasr_b200.diarization and scipy."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import scipy.linalg

from conftest import GOLDEN
from funasr_b200 import _abi, pack
from funasr_b200 import diarization as D
from test_spk_host import campplus_state_dict

NO_DEVICE = b"no such CUDA device"


def _ptr(a):
    return a.ctypes.data


def test_campplus_model_file_round_trips(tmp_path):
    from funasr_b200.campplus import campplus_specs, povey_window
    from funasr_b200.engine import kaldi_mel_banks
    st = campplus_state_dict()
    path = str(tmp_path / "spk.fab2")
    pack.write_campplus_model_file(st, path)
    t = pack.read_model_file(path)
    names = [k for k in campplus_specs() if not k.endswith("num_batches_tracked")]
    for k in names:
        assert np.array_equal(t[k], st[k].float().numpy()), k
    assert not any(k.endswith("num_batches_tracked") for k in t)
    assert np.array_equal(t["frontend.mel_banks"], kaldi_mel_banks().numpy())
    assert np.array_equal(t["frontend.window"], povey_window().numpy())
    assert t["__spk_config__"].tolist() == [80, 192, 32, 4, 128]
    assert set(t) == set(names) | {"frontend.mel_banks", "frontend.window", "__spk_config__"}


def test_campplus_model_file_refuses_other_shapes(tmp_path):
    st = campplus_state_dict()
    missing = {k: v for k, v in st.items() if k != "xvector.dense.linear.weight"}
    with pytest.raises(ValueError, match="xvector.dense.linear.weight"):
        pack.write_campplus_model_file(missing, str(tmp_path / "a.fab2"))
    wide = dict(st)
    wide["head.conv1.weight"] = wide["head.conv1.weight"].repeat(2, 1, 1, 1)
    with pytest.raises(ValueError, match="head.conv1.weight"):
        pack.write_campplus_model_file(wide, str(tmp_path / "b.fab2"))


def _variant(tmp_path, name, edit):
    t = pack.campplus_model_tensors(campplus_state_dict())
    edit(t)
    path = str(tmp_path / name)
    pack._write(path, t)
    return path


def test_handle_refuses_bad_speaker_files_before_any_device_work(tmp_path):
    """NULL and a message naming the piece, from the index pass (so the same with or without a GPU)."""
    lib = _abi.load()

    def drop(name):
        return lambda t: t.pop(name)

    def put(name, arr):
        return lambda t: t.__setitem__(name, arr)

    cases = [("no_dense.fab2", drop("xvector.dense.linear.weight"), b"missing tensor xvector.dense.linear.weight"),
             ("no_var.fab2", drop("xvector.block2.tdnnd7.nonlinear1.batchnorm.running_var"), b"xvector.block2.tdnnd7.nonlinear1.batchnorm.running_var"),
             ("shape.fab2", put("xvector.block3.tdnnd2.linear1.weight", np.zeros((128, 99, 1), np.float32)), b"bad shape of xvector.block3.tdnnd2.linear1.weight"),
             ("window.fab2", put("frontend.window", np.zeros(512, np.float32)), b"bad shape of frontend.window"),
             ("cfg.fab2", put("__spk_config__", np.array([80, 512, 32, 4, 128], np.float32)), b"__spk_config__"),
             ("nocfg.fab2", drop("__spk_config__"), b"missing tensor __spk_config__"),
             ("sv.fab2", put("__sv_config__", np.zeros(9, np.float32)), b"__sv_config__"),
             ("seaco.fab2", put("__seaco_config__", np.zeros(3, np.float32)), b"__seaco_config__")]
    for name, edit, want in cases:
        h = lib.fa_spk_init(_variant(tmp_path, name, edit).encode(), 0, 0)
        assert not h, name
        msg = lib.fa_offline_last_error()
        assert msg.startswith(b"model file rejected: CAM++ model: ") or msg.startswith(b"CAM++ model: "), msg
        assert want in msg, (name, msg)
        assert NO_DEVICE not in msg
    assert not lib.fa_spk_init(str(tmp_path / "absent.fab2").encode(), 0, 0)
    assert not lib.fa_spk_init(_variant(tmp_path, "ok.fab2", lambda t: None).encode(), 0, 2)
    assert b"gemm_mode" in lib.fa_offline_last_error()
    good = _variant(tmp_path, "good.fab2", lambda t: None).encode()
    h = lib.fa_spk_init(good, 0, 0)
    if h:
        lib.fa_spk_uninit(h)
    else:
        assert NO_DEVICE in lib.fa_offline_last_error()


def _tridiag_smallest(d, e, m, k):
    lib = _abi.load()
    n = d.size
    w = np.zeros(m)
    z = np.zeros((max(k, 1), n))
    assert lib.fa_sym_tridiag_smallest_host(_ptr(d), _ptr(e), n, m, k, _ptr(w), _ptr(z)) == 0
    return w, z[:k]


def _check_tridiag(d, e, m=16, k=15):
    w, z = _tridiag_smallest(d, e, m, k)
    ref_w, ref_v = scipy.linalg.eigh_tridiagonal(d, e)
    tnorm = np.abs(d).max() + 2 * np.abs(e).max()
    assert np.abs(w - ref_w[:m]).max() <= 1e-10 * tnorm
    V = ref_v[:, :k]
    assert np.abs(z @ z.T - np.eye(k)).max() <= 1e-8
    assert np.abs(z.T @ z - V @ V.T).max() <= 1e-8
    return w


@pytest.mark.parametrize("n", [20, 57, 300, 2047])
def test_tridiagonal_eigensolver_matches_scipy_on_random_matrices(n):
    rng = np.random.RandomState(n)
    d = rng.rand(n) * 10
    e = rng.randn(n - 1)
    w = _check_tridiag(d, e, k=min(15, n))
    # the 15th eigenvalue must be separated from the 16th for the projector to be defined
    assert w[14] < w[15]


@pytest.mark.parametrize("n,blocks", [(40, 3), (500, 4), (2047, 5)])
def test_tridiagonal_eigensolver_matches_scipy_on_block_degenerate_matrices(n, blocks):
    """Several connected components: zero couplings between blocks, each block the Laplacian of a path (eigenvalue 0 once per block)."""
    rng = np.random.RandomState(blocks)
    cuts = np.sort(rng.choice(np.arange(5, n - 5), blocks - 1, replace=False))
    wts = rng.rand(n - 1) + 0.5
    wts[cuts - 1] = 0.0
    d = np.zeros(n)
    d[:-1] += wts
    d[1:] += wts
    e = -wts
    w = _check_tridiag(d, e, k=blocks)
    assert np.abs(w[:blocks]).max() < 1e-10 and w[blocks] > 1e-8


def _kmeans_host(x, k):
    x = np.ascontiguousarray(x, dtype=np.float64)
    lab = np.zeros(x.shape[0], np.int32)
    assert _abi.load().fa_spk_kmeans_host(_ptr(x), x.shape[0], x.shape[1], int(k), 0, 10, 300, _ptr(lab)) == 0
    return lab


def _merge_host(labels, emb):
    lab = np.ascontiguousarray(labels, dtype=np.int32).copy()
    emb = np.ascontiguousarray(emb, dtype=np.float32)
    assert _abi.load().fa_spk_merge_by_cos_host(_ptr(lab), _ptr(emb), emb.shape[0], emb.shape[1], 0.78) == 0
    return lab


def _same_partition(a, b):
    return D.correct_labels(np.asarray(a)).tolist() == D.correct_labels(np.asarray(b)).tolist()


def test_kmeans_and_merge_match_reference_routines():
    g = np.load(os.path.join(GOLDEN, "spk_host_routines.npz"))
    # >= 2048 chunks with a preset count: k-means on the normalised rows
    x, k = g["kmeans_2048__x"], int(g["kmeans_2048__k"])
    lab = _kmeans_host(D._normalize_rows(x), k)
    assert _same_partition(lab, g["kmeans_2048__labels"])
    assert _same_partition(lab, D.kmeans(D._normalize_rows(x), k))
    # the spectral embedding (scipy here; the device path is tests/test_offline_spk_gpu.py), k-means, then merge_by_cos
    for case in ("merge_by_cos", "spectral_k3"):
        x = g[case + "__x"]
        sc = D.SpectralCluster()
        emb, kk = sc.spec_embs(sc.laplacian(0.5 * (lambda p: p + p.T)(sc.p_pruning(sc.sim_mat(x)))), None)
        lab = _kmeans_host(emb, kk)
        assert _same_partition(lab, D.kmeans(emb, kk)), case
        merged = _merge_host(lab, x)
        assert _same_partition(merged, D.ClusterBackend.merge_by_cos(D.kmeans(emb, kk), x, 0.78)), case
        assert _same_partition(merged, g[case + "__labels"]), case
    x = g["few_rows__x"]
    assert _same_partition(_kmeans_host(x, 2), D.kmeans(x, 2))


@pytest.mark.parametrize("seed", range(8))
def test_kmeans_and_merge_on_separated_mixtures(seed):
    rng = np.random.RandomState(100 + seed)
    k, dim = rng.randint(2, 7), rng.choice([3, 16, 192])
    centers = rng.randn(k, dim) * 10
    sizes = rng.randint(5, 60, size=k)
    x = np.concatenate([c + rng.randn(s, dim) for c, s in zip(centers, sizes)]).astype(np.float32)
    x = x[rng.permutation(len(x))]
    lab = _kmeans_host(x, k)
    ref = D.kmeans(x, k)
    assert _same_partition(lab, ref)
    # two clusters sharing a direction merge; the rest stay apart
    assert _same_partition(_merge_host(lab, x), D.ClusterBackend.merge_by_cos(ref, x, 0.78))
    y = np.concatenate([x, x[: sizes.min()] * 2.0]).astype(np.float32)
    two = np.concatenate([lab, np.full(sizes.min(), k, np.int32)])
    assert _same_partition(_merge_host(two, y), D.ClusterBackend.merge_by_cos(two.astype(np.int64), y, 0.78))


def _postprocess_host(segs, labels):
    segs = np.ascontiguousarray(segs, dtype=np.float64)
    labels = np.ascontiguousarray(labels, dtype=np.int32)
    turns = np.zeros((len(labels), 3))
    n = _abi.load().fa_spk_postprocess_host(_ptr(segs), _ptr(labels), len(labels), _ptr(turns))
    assert n > 0
    return turns[:n]


def _distribute_host(sent, turns):
    sent = np.ascontiguousarray(sent, dtype=np.int32)
    turns = np.ascontiguousarray(turns, dtype=np.float64)
    out = np.zeros(len(sent), np.int32)
    assert _abi.load().fa_spk_distribute_host(_ptr(sent), len(sent), _ptr(turns), len(turns), _ptr(out)) == 0
    return out.tolist()


@pytest.mark.parametrize("i", range(6))
def test_postprocess_and_distribute_equal_reference(i):
    g = np.load(os.path.join(GOLDEN, "spk_host_routines.npz"))
    turns = _postprocess_host(g["post%d__segs" % i], g["post%d__labels" % i])
    assert np.array_equal(turns, g["post%d__sv" % i])
    ref = json.loads(str(g["post%d__sentences" % i]))
    assert _distribute_host([[d["start"], d["end"]] for d in ref], turns) == [d["spk"] for d in ref]


def test_postprocess_rounds_like_python_on_half_cases():
    """smooth's round(x, 2) on values whose decimal expansion ends in 5 (ties resolved on the exact binary value), random turns."""
    rng = np.random.RandomState(7)
    for trial in range(300):
        n = rng.randint(1, 30)
        st = np.cumsum(rng.choice([0.005, 0.015, 0.125, 0.375, 0.745, 1.005, 0.7, 0.75, 1.5], size=n))
        ed = st + rng.choice([0.3, 0.695, 0.705, 1.5, 2.675, 0.745], size=n)
        segs = np.stack([st, ed], 1)
        labels = rng.randint(0, 3, size=n)
        want = D.postprocess([list(s) for s in segs.tolist()], None, labels.copy(), np.zeros((n, 2), np.float32))
        got = _postprocess_host(segs, labels)
        assert np.array_equal(got, np.array([[a, b, s] for a, b, s in want], dtype=np.float64)), trial
        sent = [[int(a * 1000), int(b * 1000) + 300] for a, b in segs[: rng.randint(1, n + 1)].tolist()]
        ref = D.distribute_spk([{"start": a, "end": b} for a, b in sent], want)
        assert _distribute_host(sent, got) == [d["spk"] for d in ref], trial


def test_speaker_symbols_are_exported_and_declared():
    lib = C.CDLL(_abi.LIB_PATH)
    header = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "funasr_b200.h")).read()
    for name in ("fa_spk_init", "fa_spk_uninit", "fa_spk_embed", "fa_spk_cluster", "fa_offline_infer_vad_spk", "fa_offline_result_spk",
                 "fa_spk_effective_pval", "fa_spk_laplacian_workspace_bytes", "fa_spk_laplacian", "fa_spk_tridiagonalize_workspace_bytes",
                 "fa_spk_tridiagonalize", "fa_spk_back_transform", "fa_sym_tridiag_smallest_host", "fa_spk_kmeans_host",
                 "fa_spk_merge_by_cos_host", "fa_spk_postprocess_host", "fa_spk_distribute_host"):
        assert hasattr(lib, name) and name + "(" in header and name in _abi.SIGNATURES, name
    lib = _abi.load()
    assert lib.fa_spk_effective_pval(100, 0.022) == 0.06 and lib.fa_spk_effective_pval(1000, 0.022) == 0.022
    assert lib.fa_spk_laplacian_workspace_bytes(2048, 192) == 0 and lib.fa_spk_tridiagonalize_workspace_bytes(2048) == 0
    assert lib.fa_spk_laplacian_workspace_bytes(2047, 192) > 2047 * 2047 * 4
    # the long-audio entry refuses a missing speaker handle, and the result accessor a NULL result
    cnt = C.c_int32(5)
    assert not lib.fa_offline_result_spk(None, 0, C.byref(cnt)) and cnt.value == 0
    assert not lib.fa_offline_infer_vad_spk(None, None, None, None, None, 1, 0, None, 0, None, None, None, 0)
    assert b"spk" in lib.fa_offline_last_error()
