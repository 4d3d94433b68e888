"""Throughput of the request pool for hotword calls: T threads on one SeACo handle, each sending seeded 5-15 s requests with hotword rows.
Usage: offline_hotword_pool_probe.py --libs NEW.so [OLD.so] [--threads 1,4,16,64] [--cases shared,distinct,sos] [--calls 128] [--reps 2]
                                     [--mode fp16x3] [--out DIR]

Each library named by --libs (for example this build and the parent commit's, built from their own trees) runs in a worker process of
its own, the libraries alternating, --reps times.  A worker opens one SeACo Paraformer handle at PARAFORMER_LARGE shape (synthetic
weights, nfilter 8, written once by funasr_b200.pack), then for each hotword case and each T: a warm-up, then --calls
fa_offline_infer_hw requests shared out over T threads released together.  A request is one seeded 5-15 s utterance with seeded rows:
  shared    one list of 50 rows, the same bytes in every request (a server-wide hotword list; the filter runs on every batch)
  distinct  a list of its own of 1-50 rows per request
  sos       the <s> row only (what CompileHotwordEmbedding gives for an empty hotword string)
The same request numbers give the same audio and rows in every worker.  Per (library, case, T), as medians over the reps: audio-s/s
(request seconds / wall time of the window, which ends when every call has returned its host result), p50 and p99 call latency, and
calls per GPU pack (fa_offline_pool_stats).  Also checks that every library gives the same ids for every request, and prints the card
and its power limit read in the same run.  --out DIR writes the JSON there."""
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

NAMES = ["fa_offline_init", "fa_offline_infer_hw", "fa_offline_result_count", "fa_offline_result_ids", "fa_offline_free_result",
         "fa_offline_uninit", "fa_offline_last_error", "fa_offline_pool_stats"]
CASES = ("shared", "distinct", "sos")


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def request(k):
    """Request k: one seeded utterance of 5-15 s, speech-like."""
    from funasr_b200 import synth
    n = int(np.random.default_rng(1000 + k).integers(5 * 16000, 15 * 16000 + 1))
    return synth.make_wav(n, 7000 + k, "speechlike").numpy().astype(np.float32)


def rows(case, k):
    """Request k's hotword rows [n, 512] for a case (seeded; the last row stands for <s>)."""
    n = 50 if case == "shared" else 1 if case == "sos" else int(np.random.default_rng(2000 + k).integers(1, 51))
    seed = 3000 if case == "shared" else 4000 if case == "sos" else 5000 + k
    return (np.random.default_rng(seed).standard_normal((n, 512)) * 0.5).astype(np.float32)


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
    from funasr_b200 import _abi
    h = lib.fa_offline_init(a.model.encode(), 0, _abi.GEMM_MODES[a.mode])
    assert h, lib.fa_offline_last_error()
    wavs = [request(k) for k in range(a.calls)]

    def one(hw, k):
        w = wavs[k]
        ptrs = (C.c_void_p * 1)(w.ctypes.data)
        lens = (C.c_int64 * 1)(w.size)
        t0 = time.perf_counter()
        r = lib.fa_offline_infer_hw(h, ptrs, lens, 1, 0, hw[k].ctypes.data, hw[k].shape[0])
        assert r, lib.fa_offline_last_error()
        n = C.c_int32()
        p = lib.fa_offline_result_ids(r, 0, C.byref(n))
        ids = [p[i] for i in range(n.value)]
        lib.fa_offline_free_result(r)
        return time.perf_counter() - t0, hashlib.sha1(np.asarray(ids, np.int32).tobytes()).hexdigest()[:16]

    def pool():
        c, p = C.c_int64(), C.c_int64()
        lib.fa_offline_pool_stats(h, C.byref(c), C.byref(p))
        return c.value, p.value
    out = {}
    for case in a.cases:
        hw = [rows(case, k) for k in range(a.calls)]
        for T in a.threads:
            for k in range(min(4, a.calls)):                # warm-up: every shape class the window sees
                one(hw, k)
            lat, hashes = [None] * a.calls, [None] * a.calls
            bar = threading.Barrier(T + 1)

            def run(j):
                bar.wait()
                for k in range(j, a.calls, T):
                    lat[k], hashes[k] = one(hw, k)
            ts = [threading.Thread(target=run, args=(j,)) for j in range(T)]
            for t in ts:
                t.start()
            c0, p0 = pool()
            bar.wait()
            t0 = time.perf_counter()
            for t in ts:
                t.join()
            wall = time.perf_counter() - t0
            c1, p1 = pool()
            seconds = sum(w.size for w in wavs) / 16000.0
            ls = sorted(lat)
            out["%s/%d" % (case, T)] = {"audio_s_per_s": seconds / wall, "p50_ms": 1e3 * ls[len(ls) // 2],
                                        "p99_ms": 1e3 * ls[min(len(ls) - 1, int(0.99 * len(ls)))],
                                        "calls_per_pack": (c1 - c0) / (p1 - p0) if p1 > p0 else None, "ids": hashes}
    lib.fa_offline_uninit(h)
    json.dump(out, open(a.json, "w"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="+", default=[os.path.join(ROOT, "funasr_b200", "libfunasr_b200.so")])
    ap.add_argument("--threads", default="1,4,16,64")
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--calls", type=int, default=128)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--mode", default="fp16x3")
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--lib", default=None)
    ap.add_argument("--model", default=None)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    a.threads = [int(x) for x in a.threads.split(",")]
    a.cases = a.cases.split(",")
    assert all(c in CASES for c in a.cases), a.cases
    if a.worker:
        return worker(a)
    from funasr_b200 import pack, synth
    tmp = tempfile.mkdtemp(prefix="hotword_pool_probe_")
    cfg = synth.PARAFORMER_LARGE
    model = os.path.join(tmp, "seaco_large.fab2")
    pack.write_seaco_model_file(model, synth.make_seaco_state_dict(cfg, 0), cfg, synth.make_cmvn(cfg, 1), no_bias=synth.seaco_no_bias_id(cfg),
                                nfilter=8)
    runs = {lib: [] for lib in a.libs}
    for rep in range(a.reps):
        for lib in a.libs:                                  # alternating
            js = os.path.join(tmp, "r%d_%d.json" % (rep, a.libs.index(lib)))
            subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--lib", lib, "--model", model, "--json", js,
                            "--threads", ",".join(map(str, a.threads)), "--cases", ",".join(a.cases), "--calls", str(a.calls), "--mode", a.mode], check=True)
            runs[lib].append(json.load(open(js)))
    res = {"card": card(), "mode": a.mode, "calls": a.calls, "reps": a.reps, "libs": a.libs, "cases": a.cases, "table": {}}
    ids = {}
    for lib in a.libs:
        for key in runs[lib][0]:
            rs = [r[key] for r in runs[lib]]
            med = {f: statistics.median(r[f] for r in rs) if rs[0][f] is not None else None
                   for f in ("audio_s_per_s", "p50_ms", "p99_ms", "calls_per_pack")}
            res["table"]["%s %s" % (os.path.relpath(lib, ROOT), key)] = med
            for r in rs:
                ids.setdefault(key.split("/")[0], []).append(r["ids"])      # per case: every library, rep and T
    res["results_equal"] = all(all(x == v[0] for x in v) for v in ids.values())
    print("card:", res["card"])
    for k, v in res["table"].items():
        print("%-60s %9.1f audio-s/s  p50 %7.1f ms  p99 %7.1f ms  calls/pack %s" % (k, v["audio_s_per_s"], v["p50_ms"], v["p99_ms"],
                                                                                   "-" if v["calls_per_pack"] is None else "%.2f" % v["calls_per_pack"]))
    print("results equal across libraries, reps and thread counts:", res["results_equal"])
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(res, open(os.path.join(a.out, "offline_hotword_pool_probe.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
