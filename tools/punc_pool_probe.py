"""Throughput of the punctuation pool: T threads on one CT-Transformer handle, each sending seeded punctuation requests.
Usage: punc_pool_probe.py --libs NEW.so [OLD.so] [--threads 1,4,16,64] [--calls 512] [--reps 3] [--out DIR]

Each library named by --libs (for example this build and the parent commit's, built from their own trees) runs in a worker process of
its own, the libraries alternating, --reps times.  A worker opens one handle on the synthetic CT-Transformer (d 256, 4 layers; weights
written once by funasr_b200.pack), then for each T: a warm-up, then --calls fa_punc_infer calls shared out over T threads released
together.  Request k is seeded: one text of 20-150 characters (one utterance's result), or with probability 1/16 one of 1 000-3 000
characters (a long recording's result), mixed CJK and Latin (synth.make_punc_text).  Per (library, T), as medians over the reps: texts/s and
characters/s (over the wall time of the window, which ends when every call has returned), p50 and p99 call latency, lockstep steps
per call (fa_punc_pool_stats where the library has it, otherwise the calls' own fa_punc_result_steps summed) and kernel launches per
call (fa_launch_count).  Also checks that every library gives the same texts and ids for every request, and prints the card and its
power limit read in the same run.  --out DIR writes the JSON there."""
import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

NAMES = ["fa_punc_init", "fa_punc_infer", "fa_punc_result_text", "fa_punc_result_ids", "fa_punc_result_steps", "fa_punc_free_result",
         "fa_punc_uninit", "fa_punc_pool_stats", "fa_offline_last_error", "fa_launch_count"]


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def request(k):
    """Request k: one text of 20-150 characters, or with probability 1/16 of 1 000-3 000 (seeded, so the long requests spread over
    the threads)."""
    from funasr_b200 import synth
    rng = np.random.default_rng(3000 + k)
    n = int(rng.integers(1000, 3001)) if rng.random() < 1 / 16 else int(rng.integers(20, 151))
    return synth.make_punc_text(n, 8000 + k)[:n]


def load(path):
    from funasr_b200 import _abi
    lib = C.CDLL(path)
    for name in NAMES:
        if hasattr(lib, name):
            res, args = _abi.SIGNATURES[name]
            getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


def worker(a):
    lib = load(a.lib)
    h = lib.fa_punc_init(a.model.encode(), 0)
    assert h, lib.fa_offline_last_error()
    stats = hasattr(lib, "fa_punc_pool_stats")
    texts = [request(k) for k in range(a.calls)]
    chars = sum(len(t) for t in texts)
    arrs = [(C.c_char_p * 1)(t.encode("utf-8")) for t in texts]

    def one(k):
        t0 = time.perf_counter()
        r = lib.fa_punc_infer(h, arrs[k], 1)
        assert r, lib.fa_offline_last_error()
        lat = time.perf_counter() - t0
        n = C.c_int32()
        p = lib.fa_punc_result_ids(r, 0, C.byref(n))
        ids = np.asarray([p[i] for i in range(n.value)], np.int32).tobytes()
        digest = hashlib.sha1(lib.fa_punc_result_text(r, 0) + b"\0" + ids).hexdigest()[:16]
        steps = int(lib.fa_punc_result_steps(r))
        lib.fa_punc_free_result(r)
        return lat, digest, steps

    def pool():
        if not stats:
            return 0
        c, s = C.c_int64(), C.c_int64()
        lib.fa_punc_pool_stats(h, C.byref(c), C.byref(s))
        return s.value
    out = {}
    for T in a.threads:
        for k in range(min(16, a.calls)):                   # warm-up: a long text grows the buffers
            one(k)
        lat, hashes, own = [None] * a.calls, [None] * a.calls, [0] * a.calls
        bar = threading.Barrier(T + 1)

        def run(j):
            bar.wait()
            for k in range(j, a.calls, T):
                lat[k], hashes[k], own[k] = one(k)
        ts = [threading.Thread(target=run, args=(j,)) for j in range(T)]
        for t in ts:
            t.start()
        s0 = pool()
        l0 = lib.fa_launch_count()
        bar.wait()
        t0 = time.perf_counter()
        for t in ts:
            t.join()
        wall = time.perf_counter() - t0
        steps = pool() - s0 if stats else sum(own)
        ls = sorted(lat)
        out[str(T)] = {"texts_per_s": a.calls / wall, "chars_per_s": chars / wall, "p50_ms": 1e3 * ls[len(ls) // 2],
                       "p99_ms": 1e3 * ls[min(len(ls) - 1, int(0.99 * len(ls)))], "steps_per_call": steps / a.calls,
                       "launches_per_call": (lib.fa_launch_count() - l0) / a.calls, "ids": hashes}
    lib.fa_punc_uninit(h)
    json.dump(out, open(a.json, "w"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="+", default=[os.path.join(ROOT, "funasr_b200", "libfunasr_b200.so")])
    ap.add_argument("--threads", default="1,4,16,64")
    ap.add_argument("--calls", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--lib", default=None)
    ap.add_argument("--model", default=None)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    a.threads = [int(x) for x in a.threads.split(",")]
    if a.worker:
        return worker(a)
    from funasr_b200 import pack, synth
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_offline_punc_host import ENC_CONF
    tmp = tempfile.mkdtemp(prefix="punc_pool_probe_")
    model = os.path.join(tmp, "punc.fab2")
    pack.write_punc_model_file(model, synth.make_punc_state_dict(0), synth.PUNC_LIST, synth.punc_token_list(), 3, ENC_CONF)
    runs = {lib: [] for lib in a.libs}
    for rep in range(a.reps):
        for lib in a.libs:                                  # alternating
            js = os.path.join(tmp, "r%d_%d.json" % (rep, a.libs.index(lib)))
            subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--lib", lib, "--model", model, "--json", js,
                            "--threads", ",".join(map(str, a.threads)), "--calls", str(a.calls)], check=True)
            runs[lib].append(json.load(open(js)))
    res = {"card": card(), "calls": a.calls, "reps": a.reps, "libs": a.libs, "table": {}}
    ids = []
    for lib in a.libs:
        for key in runs[lib][0]:
            rs = [r[key] for r in runs[lib]]
            med = {f: statistics.median(r[f] for r in rs) for f in ("texts_per_s", "chars_per_s", "p50_ms", "p99_ms", "steps_per_call",
                                                                     "launches_per_call")}
            med["texts_per_s_reps"] = [r["texts_per_s"] for r in rs]
            res["table"]["%s T=%s" % (os.path.relpath(lib, ROOT), key)] = med
            ids += [r["ids"] for r in rs]
    res["results_equal"] = all(x == ids[0] for x in ids)
    print("card:", res["card"])
    for k, v in res["table"].items():
        print("%-48s %8.1f texts/s %9.0f chars/s  p50 %7.2f ms  p99 %7.2f ms  steps/call %.3f  launches/call %.1f  reps %s" % (
            k, v["texts_per_s"], v["chars_per_s"], v["p50_ms"], v["p99_ms"], v["steps_per_call"], v["launches_per_call"],
            ["%.0f" % x for x in v["texts_per_s_reps"]]))
    print("texts and ids equal across libraries, reps and thread counts:", res["results_equal"])
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(res, open(os.path.join(a.out, "punc_pool_probe.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
