"""CT-Transformer punctuation through the C handle API (fa_punc_infer): many texts in one lockstep call against one call per text.
Usage: punc_probe.py [--texts 64] [--words 1600] [--reps 5] [--out DIR]

--texts seeded synthetic transcripts (synth.make_punc_text, about 3 000 characters at 1 600 words) and the synthetic CT-Transformer
weights (d = 256, 8 x 32 heads, 4 layers).  After one warm-up of each, the two ways run alternately --reps times; each time is a host
clock around the call, which ends in a device synchronise.  Reports per way the median ms, the lockstep steps and the kernel launches
(fa_launch_count), checks that both give the same results, and prints the card and its power limit read in the same run.
--out DIR writes the JSON there."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--texts", type=int, default=64)
    ap.add_argument("--words", type=int, default=1600)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from funasr_b200 import _abi, pack, synth
    from funasr_b200.offline import OfflinePunc
    lib = _abi.load()
    texts = [synth.make_punc_text(a.words, 7000 + i) for i in range(a.texts)]
    conf = dict(attention_heads=synth.PUNC_HEADS, kernel_size=11)
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "punc.fab2")
        pack.write_punc_model_file(path, synth.make_punc_state_dict(0), synth.PUNC_LIST, synth.punc_token_list(), 3, conf)
        p = OfflinePunc(path, 0)

    def batched():
        return p.infer(texts), p.last_steps

    def one_by_one():
        out, steps = [], 0
        for t in texts:
            out += p.infer([t])
            steps += p.last_steps
        return out, steps

    ways = {"one_call": batched, "one_call_per_text": one_by_one}
    res = {k: {"ms": []} for k in ways}
    outs = {}
    for k, fn in ways.items():                                  # warm-up: grow-only buffers, first-launch costs
        outs[k] = fn()[0]
    for _ in range(a.reps):
        for k, fn in ways.items():
            c0 = lib.fa_launch_count()
            t0 = time.perf_counter()
            out, steps = fn()
            res[k]["ms"].append((time.perf_counter() - t0) * 1e3)
            res[k]["launches"] = int(lib.fa_launch_count() - c0)
            res[k]["steps"] = int(steps)
            assert out == outs[k]
    for k in ways:
        res[k]["median_ms"] = round(statistics.median(res[k]["ms"]), 2)
        res[k]["ms"] = [round(v, 2) for v in res[k]["ms"]]
    report = {"card": card(), "texts": a.texts, "words_per_text": a.words,
              "mean_chars_per_text": round(sum(len(t) for t in texts) / len(texts), 1),
              "same_results": outs["one_call"] == outs["one_call_per_text"], **res,
              "speedup": round(res["one_call_per_text"]["median_ms"] / res["one_call"]["median_ms"], 2)}
    s = json.dumps(report, ensure_ascii=False)
    print(s)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "punc_probe.json"), "w") as f:
            f.write(s + "\n")
    p.close()


if __name__ == "__main__":
    main()
