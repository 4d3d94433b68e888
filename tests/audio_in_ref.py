"""References of the audio-in path (FaAudioFormat) shared by tests/test_audio_in_host.py and tests/test_audio_in_gpu.py.

FA_RESAMPLE_RUNTIME is pinned to the reference runtime's LinearResample: the compiled library (oracle/linres_ref.py) where
oracle/_ref/liblinres_ref.so was built, the committed tests/golden/linres_cases.npz otherwise.  `linres_numpy` restates its sum
order in float32 (each product and each add rounded on its own, taps from 0, indices outside the input skipped); the host test pins
it to the oracle, so checkouts without the library can still produce the runtime's 16 kHz rows."""
import hashlib
import os

import numpy as np

import linres_ref
from conftest import GOLDEN

RATES = linres_ref.RATES


def golden():
    return np.load(os.path.join(GOLDEN, "linres_cases.npz"))


def have_oracle() -> bool:
    return linres_ref.build()


def runtime_tables(rate: int):
    """-> (in_unit, out_unit, first, n_taps, weights [out_unit, max_taps]) of the reference, from the library or the golden."""
    if have_oracle():
        return linres_ref.LinearResample(rate).tables()
    g = golden()
    iu, ou = g["r%d_units" % rate].tolist()
    return iu, ou, g["r%d_first" % rate], g["r%d_n_taps" % rate], g["r%d_weights" % rate]


def linres_numpy(x: np.ndarray, rate: int) -> np.ndarray:
    """LinearResample(rate, 16000).Resample(x, flush=true) restated in numpy float32."""
    iu, ou, first, n_taps, w = runtime_tables(rate)
    x = np.asarray(x, np.float32)
    n = x.size
    m = -(-16000 * n // rate) if n else 0
    t = np.arange(m, dtype=np.int64)
    u, p = t // ou, t % ou
    base = first[p].astype(np.int64) + u * iu
    acc = np.zeros(m, np.float32)
    for j in range(w.shape[1]):
        idx = base + j
        ok = (j < n_taps[p]) & (idx >= 0) & (idx < n)
        prod = w[p, j] * x[np.clip(idx, 0, max(n - 1, 0))] if n else np.zeros(m, np.float32)
        acc = np.where(ok, acc + prod, acc).astype(np.float32)
    return acc


def linres_rows(x: np.ndarray, rate: int) -> np.ndarray:
    """The runtime's 16 kHz samples of mono float32 x at `rate`: the compiled reference where built, the restatement otherwise."""
    if rate == 16000:
        return np.asarray(x, np.float32)
    if have_oracle():
        return linres_ref.LinearResample(rate).resample(x)
    return linres_numpy(x, rate)


def sha256(a: np.ndarray) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).digest(), np.uint8)
