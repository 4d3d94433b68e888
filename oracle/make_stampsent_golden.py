"""Writes tests/golden/stampsent_cases.npz: the C++ runtime's own TimestampSentence (oracle/_ref/libstampsent_ref.so, built from the
reference's util.cpp by oracle/stampsent/Makefile) on seeded random (text, stamp) pairs (tests/stampsent_cases.py), so checkouts
without the reference tree still pin tests/stampsent_ref.py.  Run where the reference tree is present:
python oracle/make_stampsent_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [HERE, os.path.join(ROOT, "tests")]
import stampsent_lib  # noqa: E402
from stampsent_cases import pairs  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "stampsent_cases.npz")
SEED, N = 20261017, 600


def main():
    if not stampsent_lib.build():
        sys.exit("the reference tree is needed to build oracle/_ref/libstampsent_ref.so")
    ps = pairs(SEED, N)
    out = [stampsent_lib.timestamp_sentence(t, s) for t, s in ps]
    np.savez_compressed(GOLDEN, seed=np.array(SEED), text=np.array([t for t, _ in ps]), stamp=np.array([s for _, s in ps]), sents=np.array(out))
    print("wrote", GOLDEN, len(out), "cases;", sum(o != "[]" for o in out), "non-empty")


if __name__ == "__main__":
    main()
