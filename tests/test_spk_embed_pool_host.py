"""CPU: the CAM++ forward with a padded length per row (fa_campplus_forward_ext) and the speaker pool's counters are exported and
declared, every bad argument of the forward is refused with its code before any launch, and its workspace query sizes from the same
carve as fa_campplus_forward's."""
import ctypes as C
import os

import pytest

from conftest import ROOT
from funasr_b200 import _abi

NEW = ["fa_campplus_ext_workspace_bytes", "fa_campplus_forward_ext", "fa_spk_pool_stats"]
FAKE = C.c_void_p(256)                           # never dereferenced: every call below is refused first
BIG = 1 << 40
ARG, UNSUPPORTED = -1, -4


def _i32(v):
    return (C.c_int32 * len(v))(*v)


def _model():
    m = _abi.FaCampplus()
    m.n_layers[0], m.n_layers[1], m.n_layers[2] = 12, 24, 16
    return m


def test_new_symbols_exported_and_declared():
    lib = _abi.load()
    header = open(os.path.join(ROOT, "include", "funasr_b200.h")).read()
    for name in NEW:
        assert name in _abi.SIGNATURES, name
        assert hasattr(lib, name), name
        assert " %s(" % name in header, name


@pytest.mark.parametrize("mode", [0, 2])
def test_forward_ext_refusals_before_any_launch(mode):
    lib = _abi.load()
    m = _model()
    before = lib.fa_launch_count()

    def fwd(batch, t, ext):
        return lib.fa_campplus_forward_ext(C.byref(m), FAKE, batch, t, FAKE, mode, FAKE, BIG, None, ext)
    assert fwd(2, 148, None) == ARG
    assert fwd(2, 148, _i32([148, 1])) == ARG                 # ext < 2
    assert fwd(2, 148, _i32([0, 148])) == ARG
    assert fwd(2, 148, _i32([149, 148])) == ARG               # ext > t
    assert fwd(0, 148, _i32([148])) == ARG                    # batch < 1
    assert fwd(-1, 148, _i32([148])) == ARG
    assert fwd(1, 18801, _i32([18801])) == UNSUPPORTED        # a 95th CAM segment
    assert fwd(2, 18801, _i32([148, 200])) == UNSUPPORTED     # the padded length decides, whatever the rows' extents
    assert fwd(1, 18801, _i32([1])) == ARG                    # a bad argument is reported before an unsupported size
    assert lib.fa_launch_count() == before


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_ext_workspace_query(mode):
    lib = _abi.load()
    m = _model()
    q = lambda b, t: int(lib.fa_campplus_workspace_bytes(C.byref(m), b, t, mode))
    qe = lambda b, t: int(lib.fa_campplus_ext_workspace_bytes(C.byref(m), b, t, mode))
    for b, t in ((0, 148), (-1, 148), (1, 1), (1, 0), (1, 18801), (4, 20000)):
        assert qe(b, t) == 0, (b, t)
    for b in (1, 4, 64):
        for t in (2, 3, 148, 201, 18800):
            assert qe(b, t) >= q(b, t) > 0, (b, t)
            assert qe(b, t) - q(b, t) <= 2 * 4 * b + 256, (b, t)   # the rows' two extent arrays and their alignment


def test_pool_stats_refuses_null():
    lib = _abi.load()
    c, p = C.c_int64(7), C.c_int64(7)
    assert lib.fa_spk_pool_stats(None, C.byref(c), C.byref(p)) == ARG
    assert lib.fa_spk_pool_stats(FAKE, None, C.byref(p)) == ARG
    assert lib.fa_spk_pool_stats(FAKE, C.byref(c), None) == ARG
    assert (c.value, p.value) == (7, 7)
