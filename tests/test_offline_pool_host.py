"""CPU: the per-row extent entries and the request pool's query are exported and declared, and every _ext entry refuses bad extents
and NULL arguments before any device work."""
import ctypes as C

from funasr_b200 import _abi

NEW = ["fa_cif_predictor_ext_workspace_bytes", "fa_cif_predictor_forward_ext", "fa_timestamp_head_ext_workspace_bytes",
       "fa_timestamp_head_forward_ext", "fa_blstm_tc_ext_scratch_bytes", "fa_blstm_forward_tc_ext", "fa_offline_pool_stats"]


def _i32(v):
    return (C.c_int32 * len(v))(*v)


def test_new_symbols_exported_and_declared():
    lib = _abi.load()
    for name in NEW:
        assert name in _abi.SIGNATURES, name
        assert hasattr(lib, name), name


def test_cif_and_timestamp_ext_refusals():
    lib = _abi.load()
    fake = C.c_void_p(256)                       # never dereferenced: every call below is refused first
    pred = _abi.FaPredictor()
    head = _abi.FaTimestampHead()
    head.up_times = 3                            # so that only the extents (or the NULL arrays) can refuse below
    lens = [5, 3, 7]
    for ext, ok in (([5, 3, 7], True), ([4, 3, 7], False), ([5, 3, 8], False), ([5, 2, 7], False)):
        if ok:
            continue
        assert lib.fa_cif_predictor_forward_ext(C.byref(pred), fake, fake, 3, 7, fake, 8, fake, fake, fake, 0, fake, 1 << 30, None,
                                                _i32(lens), _i32(ext)) == -1, ext
        assert lib.fa_timestamp_head_forward_ext(C.byref(head), fake, fake, fake, 3, 7, fake, fake, 0, fake, 1 << 30, None,
                                                 _i32(lens), _i32(ext)) == -1, ext
    for lh, eh in ((None, _i32(lens)), (_i32(lens), None)):
        assert lib.fa_cif_predictor_forward_ext(C.byref(pred), fake, fake, 3, 7, fake, 8, fake, fake, fake, 0, fake, 1 << 30, None,
                                                lh, eh) == -1
        assert lib.fa_timestamp_head_forward_ext(C.byref(head), fake, fake, fake, 3, 7, fake, fake, 0, fake, 1 << 30, None, lh, eh) == -1
    assert lib.fa_cif_predictor_forward_ext(None, fake, fake, 3, 7, fake, 8, fake, fake, fake, 0, fake, 1 << 30, None,
                                            _i32(lens), _i32(lens)) == -1
    # the extent entries carve ext after the existing buffers
    for m in (0, 3):
        assert lib.fa_cif_predictor_ext_workspace_bytes(3, 37, m) >= lib.fa_cif_predictor_workspace_bytes(3, 37, m) + 12
        assert lib.fa_timestamp_head_ext_workspace_bytes(3, 37, 512, 3, m) >= lib.fa_timestamp_head_workspace_bytes(3, 37, 512, 3, m) + 24
    assert lib.fa_blstm_tc_ext_scratch_bytes(3) == lib.fa_blstm_tc_scratch_bytes(3) + 12


def test_blstm_ext_refusals():
    lib = _abi.load()
    fake = C.c_void_p(256)
    for ext in ([0, 3], [4, 5], [-1, 2]):
        assert lib.fa_blstm_forward_tc_ext(fake, fake, fake, 2, 4, 512, fake, fake, 1 << 30, None, _i32(ext)) == -1, ext
    assert lib.fa_blstm_forward_tc_ext(fake, fake, fake, 2, 4, 512, fake, fake, 1 << 30, None, None) == -1
    assert lib.fa_blstm_forward_tc_ext(None, fake, fake, 2, 4, 512, fake, fake, 1 << 30, None, _i32([1, 4])) == -1


def test_pool_stats_refuses_null():
    lib = _abi.load()
    c, p = C.c_int64(), C.c_int64()
    assert lib.fa_offline_pool_stats(None, C.byref(c), C.byref(p)) == -1
    assert lib.fa_offline_pool_stats(C.c_void_p(256), None, C.byref(p)) == -1
