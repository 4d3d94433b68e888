"""Random (punctuated text, stamp string) pairs for TimestampSentence: shared by oracle/make_stampsent_golden.py and
tests/test_stampsent_host.py."""
import random

PIECES = ["你", "好", "世", "界", "㐀", "乙", "hello", "World", "gpu", "a", "it's", "x-ray", "R&D", "42", "7", "，", "。", "？", "、", ",", ".",
          "?", "!", ";", ":", "—", "「", "」", "…", "é", "ж", "😀", "ｱ", " ", "  ", "\t"]


def random_pair(rng: random.Random):
    n = rng.choice([0, 1, 3, rng.randint(0, 30), rng.randint(0, 120)])
    text = "".join(rng.choice(PIECES) for _ in range(n))
    if rng.random() < 0.15:
        text = "".join(c for c in text if c not in "，。？、,?")        # no punctuation at all
    k = max(0, len(text) + rng.randint(-10, 10)) if rng.random() < 0.8 else rng.randint(0, 5)   # counts that match or not
    t, stamps = rng.randint(0, 5000), []
    for _ in range(k):
        b = t + rng.randint(0, 300)
        t = b + rng.randint(1, 600)
        stamps.append((b, t))
    stamp = "[" + ",".join("[%d,%d]" % p for p in stamps) + "]" if stamps else ""
    return text, stamp


def pairs(seed: int, n: int):
    rng = random.Random(seed)
    return [random_pair(rng) for _ in range(n)]
