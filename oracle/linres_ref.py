"""TEST INFRASTRUCTURE: loader for oracle/_ref/liblinres_ref.so, the reference C++ runtime's LinearResample
(runtime/onnxruntime/src/resample.cpp) compiled by oracle/linres/Makefile and constructed as Audio::WavResample constructs it.  It
pins FA_RESAMPLE_RUNTIME: the phase tables, the flushed output count and Resample(flush=true).  tests/golden/linres_cases.npz
(oracle/make_linres_golden.py) holds the same for checkouts without the reference tree.
Only tests/, tools/ and __graft_entry__.build() may import this module."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "_ref", "liblinres_ref.so")
REFERENCE_ROOT = "/root/reference"
RATES = (8000, 11025, 12000, 22050, 24000, 32000, 44100, 48000)


def build(force: bool = False) -> bool:
    """Compile from the reference tree when it is present; elsewhere the prebuilt file (or the committed golden) is used."""
    if os.path.exists(SO) and not force:
        return True
    if not os.path.isfile(os.path.join(REFERENCE_ROOT, "runtime", "onnxruntime", "src", "resample.cpp")):
        return False
    r = subprocess.run(["make", "-C", os.path.join(HERE, "linres"), "REF=" + REFERENCE_ROOT] + (["-B"] if force else []),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/linres build failed:\n" + r.stdout[-2000:])
    return os.path.exists(SO)


def available() -> bool:
    return os.path.exists(SO)


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(SO)
        lib.linres_new.restype = C.c_void_p
        lib.linres_new.argtypes = [C.c_int32, C.c_int32]
        lib.linres_free.argtypes = [C.c_void_p]
        lib.linres_units.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.linres_row.restype = C.c_int32
        lib.linres_row.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32]
        lib.linres_out_len.restype = C.c_int64
        lib.linres_out_len.argtypes = [C.c_void_p, C.c_int64]
        lib.linres_resample.restype = C.c_int64
        lib.linres_resample.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]
        _lib = lib
    return _lib


class LinearResample:
    """LinearResample(rate, new_rate, 0.99 * 0.5 * min rate, 6) of the reference runtime."""

    def __init__(self, rate: int, new_rate: int = 16000):
        self.lib = _load()
        self.h = self.lib.linres_new(int(rate), int(new_rate))

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.linres_free(self.h)

    def tables(self):
        """-> (in_unit, out_unit, first [out_unit] int32, n_taps [out_unit] int32, weights [out_unit, max_taps] float32 zero padded)"""
        iu, ou = C.c_int32(), C.c_int32()
        self.lib.linres_units(self.h, C.byref(iu), C.byref(ou))
        first = np.zeros(ou.value, np.int32)
        n_taps = np.zeros(ou.value, np.int32)
        rows = []
        for p in range(ou.value):
            f = C.c_int32()
            n = self.lib.linres_row(self.h, p, C.byref(f), None, 0)
            w = np.zeros(n, np.float32)
            self.lib.linres_row(self.h, p, C.byref(f), w.ctypes.data, n)
            first[p], n_taps[p] = f.value, n
            rows.append(w)
        weights = np.zeros((ou.value, int(n_taps.max())), np.float32)
        for p, w in enumerate(rows):
            weights[p, :w.size] = w
        return iu.value, ou.value, first, n_taps, weights

    def out_len(self, n: int) -> int:
        return int(self.lib.linres_out_len(self.h, int(n)))

    def resample(self, x: np.ndarray) -> np.ndarray:
        a = np.ascontiguousarray(x, dtype=np.float32)
        y = np.zeros(self.out_len(a.size), np.float32)
        k = self.lib.linres_resample(self.h, a.ctypes.data, a.size, y.ctypes.data, y.size)
        assert k == y.size
        return y


def edge_lengths(in_unit: int, max_taps: int):
    """1, shorter than one filter, exactly at unit boundaries and one either side, around the filter length."""
    ls = {1, 2, max(1, max_taps // 2), max_taps - 1, max_taps, max_taps + 1}
    for k in (1, 2, 3, 7):
        ls.update({k * in_unit - 1, k * in_unit, k * in_unit + 1})
    return sorted(v for v in ls if v >= 1)


def noise(rate: int, seconds: float = 60.0, seed: int = 0) -> np.ndarray:
    return (np.random.default_rng(seed + rate).standard_normal(int(rate * seconds)) * 0.1).astype(np.float32)
