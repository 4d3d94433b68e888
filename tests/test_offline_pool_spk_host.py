"""CPU: the ragged-batch spectral-clustering entries (Laplacian, tridiagonalisation, back-transform over many independent sets) are
exported and declared, refuse every bad argument with the single entries' codes before any launch, and size their workspaces from the
same carve as the single entries."""
import ctypes as C

import pytest

from funasr_b200 import _abi

NEW = ["fa_spk_laplacian_batch_workspace_bytes", "fa_spk_laplacian_batch", "fa_spk_tridiagonalize_batch_workspace_bytes",
       "fa_spk_tridiagonalize_batch", "fa_spk_back_transform_batch"]
FAKE = C.c_void_p(256)                           # never dereferenced: every call below is refused first
BIG = 1 << 40
ARG, WORKSPACE, UNSUPPORTED = -1, -3, -4


def _i32(v):
    return (C.c_int32 * len(v))(*v)


def test_new_symbols_exported_and_declared():
    lib = _abi.load()
    for name in NEW:
        assert name in _abi.SIGNATURES, name
        assert hasattr(lib, name), name


def _lap(lib, n, count=None, dim=192, pval=0.022, emb=FAKE, lap=FAKE, ws_bytes=BIG):
    count = len(n) if count is None and n is not None else (count or 0)
    return lib.fa_spk_laplacian_batch(emb, _i32(n) if n is not None else None, count, dim, pval, lap, FAKE, ws_bytes, None)


def _tri(lib, n, count=None, lap=FAKE, d=FAKE, e=FAKE, tau=FAKE, ws_bytes=BIG):
    count = len(n) if count is None and n is not None else (count or 0)
    return lib.fa_spk_tridiagonalize_batch(lap, _i32(n) if n is not None else None, count, d, e, tau, FAKE, ws_bytes, None)


def _back(lib, n, k, count=None, lap=FAKE, tau=FAKE, z=FAKE):
    count = len(n) if count is None and n is not None else (count or 0)
    return lib.fa_spk_back_transform_batch(lap, tau, _i32(n) if n is not None else None, _i32(k) if k is not None else None, count, z, None)


def test_laplacian_batch_refusals_before_any_launch():
    lib = _abi.load()
    before = lib.fa_launch_count()
    assert _lap(lib, None, count=2) == ARG
    assert _lap(lib, [20, 30], emb=None) == ARG
    assert _lap(lib, [20, 30], lap=None) == ARG
    assert _lap(lib, [20, 30], count=0) == ARG
    assert _lap(lib, [20, 30], count=-1) == ARG
    assert _lap(lib, [20, 0, 30]) == ARG
    assert _lap(lib, [20, -5]) == ARG
    assert _lap(lib, [20, 30], dim=0) == ARG
    assert _lap(lib, [20, 30], pval=-0.1) == ARG
    assert _lap(lib, [20, 30], pval=float("nan")) == ARG
    assert _lap(lib, [20, 2048]) == UNSUPPORTED
    assert _lap(lib, [20, 30], dim=1025) == UNSUPPORTED
    assert _lap(lib, [20, 2048], dim=0) == ARG                     # a bad argument is reported before an unsupported size
    ws = lib.fa_spk_laplacian_batch_workspace_bytes(_i32([20, 30]), 2, 192)
    assert _lap(lib, [20, 30], ws_bytes=ws - 1) == WORKSPACE
    assert lib.fa_launch_count() == before


def test_tridiagonalize_batch_refusals_before_any_launch():
    lib = _abi.load()
    before = lib.fa_launch_count()
    assert _tri(lib, None, count=2) == ARG
    assert _tri(lib, [20, 30], lap=None) == ARG
    assert _tri(lib, [20, 30], d=None) == ARG
    assert _tri(lib, [20, 30], e=None) == ARG
    assert _tri(lib, [20, 30], tau=None) == ARG
    assert _tri(lib, [20, 30], count=0) == ARG
    assert _tri(lib, [20, 0]) == ARG
    assert _tri(lib, [2048, 30]) == UNSUPPORTED
    ws = lib.fa_spk_tridiagonalize_batch_workspace_bytes(_i32([20, 30]), 2)
    assert _tri(lib, [20, 30], ws_bytes=ws - 1) == WORKSPACE
    assert lib.fa_launch_count() == before


def test_back_transform_batch_refusals_before_any_launch():
    lib = _abi.load()
    before = lib.fa_launch_count()
    assert _back(lib, None, [1, 1], count=2) == ARG
    assert _back(lib, [20, 30], None) == ARG
    assert _back(lib, [20, 30], [1, 1], lap=None) == ARG
    assert _back(lib, [20, 30], [1, 1], z=None) == ARG
    assert _back(lib, [20, 30], [1, 1], tau=None) == ARG
    assert _back(lib, [20, 30], [1, 1], count=0) == ARG
    assert _back(lib, [20, 0], [1, 1]) == ARG
    assert _back(lib, [20, 30], [0, 1]) == ARG                     # k < 1
    assert _back(lib, [20, 30], [1, 31]) == ARG                    # k > n
    assert _back(lib, [20, 2048], [1, 2]) == UNSUPPORTED
    assert lib.fa_launch_count() == before


def test_single_entries_keep_their_codes():
    """The single entries are the count = 1 case: the same refusals, with the same codes."""
    lib = _abi.load()
    before = lib.fa_launch_count()
    assert lib.fa_spk_laplacian(FAKE, 0, 192, 0.022, FAKE, FAKE, BIG, None) == ARG
    assert lib.fa_spk_laplacian(FAKE, 2048, 192, 0.022, FAKE, FAKE, BIG, None) == UNSUPPORTED
    assert lib.fa_spk_laplacian(FAKE, 20, 1025, 0.022, FAKE, FAKE, BIG, None) == UNSUPPORTED
    assert lib.fa_spk_laplacian(FAKE, 20, 192, 0.022, FAKE, FAKE, 16, None) == WORKSPACE
    assert lib.fa_spk_tridiagonalize(FAKE, 20, FAKE, None, FAKE, FAKE, BIG, None) == ARG
    assert lib.fa_spk_tridiagonalize(FAKE, 2048, FAKE, FAKE, FAKE, FAKE, BIG, None) == UNSUPPORTED
    assert lib.fa_spk_tridiagonalize(FAKE, 20, FAKE, FAKE, FAKE, FAKE, 16, None) == WORKSPACE
    assert lib.fa_spk_back_transform(FAKE, FAKE, 20, FAKE, 21, None) == ARG
    assert lib.fa_spk_back_transform(FAKE, FAKE, 2048, FAKE, 2, None) == UNSUPPORTED
    assert lib.fa_launch_count() == before


@pytest.mark.parametrize("n", [1, 2, 19, 20, 64, 65, 200, 2047])
def test_batch_workspace_at_count_one_equals_the_single_entry(n):
    lib = _abi.load()
    assert lib.fa_spk_laplacian_batch_workspace_bytes(_i32([n]), 1, 192) == lib.fa_spk_laplacian_workspace_bytes(n, 192) > 0
    assert lib.fa_spk_tridiagonalize_batch_workspace_bytes(_i32([n]), 1) == lib.fa_spk_tridiagonalize_workspace_bytes(n) > 0


def test_batch_workspace_queries():
    lib = _abi.load()
    for bad in ([0], [2048], [20, 0], [20, 2048]):
        assert lib.fa_spk_laplacian_batch_workspace_bytes(_i32(bad), len(bad), 192) == 0, bad
        assert lib.fa_spk_tridiagonalize_batch_workspace_bytes(_i32(bad), len(bad)) == 0, bad
    assert lib.fa_spk_laplacian_batch_workspace_bytes(None, 1, 192) == 0
    assert lib.fa_spk_laplacian_batch_workspace_bytes(_i32([20]), 0, 192) == 0
    assert lib.fa_spk_laplacian_batch_workspace_bytes(_i32([20]), 1, 0) == 0
    assert lib.fa_spk_laplacian_batch_workspace_bytes(_i32([20]), 1, 1025) == 0
    assert lib.fa_spk_tridiagonalize_batch_workspace_bytes(None, 1) == 0
    assert lib.fa_spk_tridiagonalize_batch_workspace_bytes(_i32([20]), 0) == 0
    # a batch needs at least what each of its sets needs alone, and grows with every set
    ns = [1, 2, 19, 20, 63, 64, 65, 200, 2047]
    lap = lib.fa_spk_laplacian_batch_workspace_bytes(_i32(ns), len(ns), 192)
    tri = lib.fa_spk_tridiagonalize_batch_workspace_bytes(_i32(ns), len(ns))
    assert lap >= 4 * (sum(ns) * 192 + sum(n * n for n in ns))
    assert tri >= 8 * (2 * sum(ns) + sum((n + 7) // 8 for n in ns))
    assert lap > lib.fa_spk_laplacian_batch_workspace_bytes(_i32(ns[:-1]), len(ns) - 1, 192)
    assert tri > lib.fa_spk_tridiagonalize_batch_workspace_bytes(_i32(ns[:-1]), len(ns) - 1)
