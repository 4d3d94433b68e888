"""Scripted punctuation scorers and random texts shared by tests/test_offline_punc_host.py and oracle/make_punc_walk_golden.py: a
scorer is punctuation as a fixed function of (token id, position in the window), so it can steer the mini-sentence walk into branches
seeded weights do not reach, and the same function drives the reference's CTTransformer.inference, punc.py and the C++ walk."""
import random

import numpy as np

from funasr_b200 import synth


def scripted(ids: np.ndarray, seed: int, probs) -> np.ndarray:
    """Punctuation as a fixed function of (token id, position in the window): a hash of both picks a class by the cumulative
    probabilities `probs` over PUNC_LIST (<unk>, _, ，, 。, ？, 、); what is left over is "_"."""
    pos = np.broadcast_to(np.arange(ids.shape[-1], dtype=np.uint64), ids.shape)
    h = (ids.astype(np.uint64) * np.uint64(2654435761) + (pos + np.uint64(1)) * np.uint64(40503) + np.uint64(seed * 977 + 13)) % np.uint64(1 << 32)
    h = (h * np.uint64(2246822519)) % np.uint64(1 << 32)
    u = h.astype(np.float64) / float(1 << 32)
    out = np.ones(ids.shape, np.int32)
    acc = 0.0
    for cls, p in zip((0, 2, 3, 4, 5), probs):                     # <unk>, ，, 。, ？, 、
        out[(u >= acc) & (u < acc + p)] = cls
        acc += p
    return out


def random_text(rng: random.Random, n_words: int) -> str:
    toks = synth.punc_token_list()
    cjk, eng = toks[3:synth.PUNC_VOCAB - 17], toks[synth.PUNC_VOCAB - 17:-1]
    extra = ["😀", "𠀀", "é", "ж", "龥", "ｱ"]                    # 2-, 3- and 4-byte characters outside the vocabulary
    out = []
    for _ in range(n_words):
        k = rng.random()
        if k < 0.55:
            w = rng.choice(cjk)
        elif k < 0.75:
            w = rng.choice(eng)
            w = w.upper() if rng.random() < 0.1 else (w.capitalize() if rng.random() < 0.1 else w)
        elif k < 0.85:
            w = "".join(rng.choice("abcxyzQ0129'-") for _ in range(rng.randint(1, 6)))    # unknown ASCII words
        else:
            w = rng.choice(extra)
        sep = rng.choice(["", "", "", " ", "  ", "\t", "　", " \n "]) if out else rng.choice(["", " "])
        out.append(sep + w)
    return "".join(out) + rng.choice(["", " ", "  "])
