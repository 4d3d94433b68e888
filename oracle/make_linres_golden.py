"""Writes tests/golden/linres_cases.npz from the compiled reference LinearResample (oracle/_ref/liblinres_ref.so, see linres_ref.py)
for checkouts without the reference tree.  Per rate r in linres_ref.RATES, to 16 kHz:
  r{r}_units [in_unit, out_unit], r{r}_first, r{r}_n_taps, r{r}_weights (zero padded);
  r{r}_lens / r{r}_out_lens: the flushed output count of 2 000 seeded random lengths;
  r{r}_edge_lens, r{r}_edge_out: Resample(flush=true) of seeded noise at each edge length (linres_ref.edge_lengths), concatenated;
  r{r}_noise_sha256: sha256 of the float32 output bytes for 60 s of linres_ref.noise(r) (the output itself is too large to commit)."""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import linres_ref as L  # noqa: E402


def main():
    assert L.build(), "needs the reference tree (oracle/linres/Makefile)"
    out = {}
    rng = np.random.default_rng(7)
    for r in L.RATES:
        lr = L.LinearResample(r)
        iu, ou, first, n_taps, w = lr.tables()
        out["r%d_units" % r] = np.array([iu, ou], np.int32)
        out["r%d_first" % r], out["r%d_n_taps" % r], out["r%d_weights" % r] = first, n_taps, w
        lens = rng.integers(1, 3_000_000, 2000).astype(np.int64)
        out["r%d_lens" % r] = lens
        out["r%d_out_lens" % r] = np.array([lr.out_len(int(n)) for n in lens], np.int64)
        edges = L.edge_lengths(iu, int(n_taps.max()))
        x = L.noise(r, 1.0, seed=1)
        out["r%d_edge_lens" % r] = np.array(edges, np.int64)
        out["r%d_edge_out" % r] = np.concatenate([lr.resample(x[:n]) for n in edges])
        out["r%d_noise_sha256" % r] = np.frombuffer(hashlib.sha256(lr.resample(L.noise(r)).tobytes()).digest(), np.uint8)
    path = os.path.join(HERE, "..", "tests", "golden", "linres_cases.npz")
    np.savez_compressed(path, **out)
    print("wrote", os.path.normpath(path), os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
