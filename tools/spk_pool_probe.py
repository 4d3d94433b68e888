"""Throughput of the speaker pool: T threads on one CAM++ handle, each sending seeded fa_spk_embed requests.
Usage: spk_pool_probe.py --libs NEW.so [OLD.so] [--threads 1,4,16,64] [--calls 256] [--reps 2] [--mode fp16x3] [--out DIR]

Each library named by --libs (for example this build and the parent commit's, built from their own trees) runs in a worker process of
its own, the libraries alternating, --reps times.  A worker opens one handle on the CAM++ fixture weights (tests/test_spk_host.py,
written once by funasr_b200.pack) in --mode, then for each T: a warm-up, then --calls fa_spk_embed calls shared out over T threads
released together.  Request k is seeded: one utterance of 1-20 s, or with probability 1/16 a batch of 8 such utterances or one 60 s
input (16 kHz f32 cut from one synthetic voice).  Per (library, T), as medians over the reps: calls/s and audio seconds per second
(over the wall time of the window, which ends when every call has returned), p50 and p99 call latency, pool passes per call
(fa_spk_pool_stats where the library has it; 1 otherwise, every call running alone) and kernel launches per call (fa_launch_count).
Also checks that every library gives the same embedding bits for every request.

Then, on this build only: fa_campplus_forward_ext with every extent equal to t against fa_campplus_forward, at B = 64 and
t in {148, 1 000, 6 000}, timed with CUDA events (alternating, medians over --fwd-iters runs each), and their outputs compared bit for
bit.  The card's name and power limit are read in the same run.  --out DIR writes the JSON there."""
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

NAMES = ["fa_spk_init", "fa_spk_uninit", "fa_spk_embed", "fa_spk_pool_stats", "fa_offline_last_error", "fa_launch_count"]


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def requests(n):
    """n seeded requests, each a list of float32 recordings cut from one 61 s synthetic voice."""
    from funasr_b200 import synth
    base = synth.make_voice_wav([(0, 61.0, 0.2)], 11, lead_s=0.0).numpy()
    out = []
    for k in range(n):
        rng = np.random.default_rng(5000 + k)
        r = rng.random()
        secs = [60.0] if r < 1 / 32 else [float(rng.uniform(1.0, 20.0)) for _ in range(8 if r < 1 / 16 else 1)]
        wavs = []
        for s in secs:
            m = int(s * 16000)
            off = int(rng.integers(0, base.size - m + 1))
            wavs.append(np.ascontiguousarray(base[off:off + m] * float(rng.uniform(0.3, 1.0)), dtype=np.float32))
        out.append(wavs)
    return out


def load(path):
    from funasr_b200 import _abi
    lib = C.CDLL(path)
    for name in NAMES:
        if hasattr(lib, name):
            res, args = _abi.SIGNATURES[name]
            getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


def worker(a):
    from funasr_b200 import _abi
    lib = load(a.lib)
    h = lib.fa_spk_init(a.model.encode(), 0, _abi.GEMM_MODES[a.mode])
    assert h, lib.fa_offline_last_error()
    stats = hasattr(lib, "fa_spk_pool_stats")
    reqs = requests(a.calls)
    secs = sum(w.size for r in reqs for w in r) / 16000
    args = [((C.c_void_p * len(r))(*[w.ctypes.data for w in r]), (C.c_int64 * len(r))(*[w.size for w in r])) for r in reqs]

    def one(k):
        out = np.empty((len(reqs[k]), 192), np.float32)
        t0 = time.perf_counter()
        rc = lib.fa_spk_embed(h, args[k][0], args[k][1], len(reqs[k]), 0, out.ctypes.data)
        lat = time.perf_counter() - t0
        assert rc == 0, lib.fa_offline_last_error()
        return lat, hashlib.sha1(out.tobytes()).hexdigest()[:16]

    def passes():
        if not stats:
            return 0
        c, p = C.c_int64(), C.c_int64()
        lib.fa_spk_pool_stats(h, C.byref(c), C.byref(p))
        return p.value
    out = {}
    for T in a.threads:
        for k in range(min(16, a.calls)):                   # warm-up: grows the buffers
            one(k)
        lat, hashes = [None] * a.calls, [None] * a.calls
        bar = threading.Barrier(T + 1)

        def run(j):
            bar.wait()
            for k in range(j, a.calls, T):
                lat[k], hashes[k] = one(k)
        ts = [threading.Thread(target=run, args=(j,)) for j in range(T)]
        for t in ts:
            t.start()
        p0 = passes()
        l0 = lib.fa_launch_count()
        bar.wait()
        t0 = time.perf_counter()
        for t in ts:
            t.join()
        wall = time.perf_counter() - t0
        npass = passes() - p0 if stats else a.calls
        ls = sorted(lat)
        out[str(T)] = {"calls_per_s": a.calls / wall, "audio_s_per_s": secs / wall, "p50_ms": 1e3 * ls[len(ls) // 2],
                       "p99_ms": 1e3 * ls[min(len(ls) - 1, int(0.99 * len(ls)))], "passes_per_call": npass / a.calls,
                       "launches_per_call": (lib.fa_launch_count() - l0) / a.calls, "emb": hashes}
    lib.fa_spk_uninit(h)
    json.dump(out, open(a.json, "w"))


def time_forward(a):
    """fa_campplus_forward_ext (every extent t) against fa_campplus_forward at B = 64 in --mode, CUDA events, this build."""
    import torch
    from funasr_b200.campplus import CampplusEngine
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_spk_host import campplus_state_dict
    dev = "cuda:0"
    eng = CampplusEngine(campplus_state_dict(), dev, a.mode)
    lib, B = eng.lib, 64
    st = torch.cuda.current_stream().cuda_stream
    out = {}
    for t in (148, 1000, 6000):
        g = torch.Generator(device=dev).manual_seed(t)
        feats = torch.randn(B, t, 80, device=dev, generator=g)
        ext = (C.c_int32 * B)(*([t] * B))
        ws = torch.empty(int(lib.fa_campplus_ext_workspace_bytes(C.byref(eng.model), B, t, eng.mode)), dtype=torch.uint8, device=dev)
        embs = {k: torch.empty(B, 192, device=dev) for k in ("forward", "forward_ext")}

        def run(k):
            if k == "forward":
                rc = lib.fa_campplus_forward(C.byref(eng.model), feats.data_ptr(), B, t, embs[k].data_ptr(), eng.mode, ws.data_ptr(),
                                             ws.numel(), st)
            else:
                rc = lib.fa_campplus_forward_ext(C.byref(eng.model), feats.data_ptr(), B, t, embs[k].data_ptr(), eng.mode, ws.data_ptr(),
                                                 ws.numel(), st, ext)
            assert rc == 0, rc
        times = {"forward": [], "forward_ext": []}
        for k in times:                                     # warm-up
            run(k)
        for _ in range(a.fwd_iters):
            for k in times:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run(k)
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1))
        out[str(t)] = {k: statistics.median(v) for k, v in times.items()}
        out[str(t)]["bit_identical"] = bool(torch.equal(embs["forward"], embs["forward_ext"]))
        del ws
    json.dump(out, open(a.json, "w"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="+", default=[os.path.join(ROOT, "funasr_b200", "libfunasr_b200.so")])
    ap.add_argument("--threads", default="1,4,16,64")
    ap.add_argument("--calls", type=int, default=256)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--mode", default="fp16x3", choices=["fp32", "fp16", "fp16x3", "fp16x6"])
    ap.add_argument("--fwd-iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--forward", action="store_true")
    ap.add_argument("--lib", default=None)
    ap.add_argument("--model", default=None)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    a.threads = [int(x) for x in a.threads.split(",")]
    if a.worker:
        return worker(a)
    if a.forward:
        return time_forward(a)
    from funasr_b200 import pack
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_spk_host import campplus_state_dict
    tmp = tempfile.mkdtemp(prefix="spk_pool_probe_")
    model = os.path.join(tmp, "spk.fab2")
    pack.write_campplus_model_file(campplus_state_dict(), model)
    common = ["--threads", ",".join(map(str, a.threads)), "--calls", str(a.calls), "--mode", a.mode]
    runs = {lib: [] for lib in a.libs}
    for rep in range(a.reps):
        for lib in a.libs:                                  # alternating
            js = os.path.join(tmp, "r%d_%d.json" % (rep, a.libs.index(lib)))
            subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--lib", lib, "--model", model, "--json", js] + common,
                           check=True)
            runs[lib].append(json.load(open(js)))
    fj = os.path.join(tmp, "forward.json")
    subprocess.run([sys.executable, os.path.abspath(__file__), "--forward", "--json", fj, "--mode", a.mode, "--fwd-iters", str(a.fwd_iters)],
                   check=True)
    res = {"card": card(), "mode": a.mode, "calls": a.calls, "reps": a.reps, "libs": a.libs, "table": {}, "forward": json.load(open(fj))}
    embs = []
    for lib in a.libs:
        for key in runs[lib][0]:
            rs = [r[key] for r in runs[lib]]
            med = {f: statistics.median(r[f] for r in rs) for f in ("calls_per_s", "audio_s_per_s", "p50_ms", "p99_ms", "passes_per_call",
                                                                     "launches_per_call")}
            med["calls_per_s_reps"] = [r["calls_per_s"] for r in rs]
            res["table"]["%s T=%s" % (os.path.relpath(lib, ROOT), key)] = med
            embs += [r["emb"] for r in rs]
    res["embeddings_equal"] = all(x == embs[0] for x in embs)
    print("card:", res["card"], " mode:", a.mode)
    for k, v in res["table"].items():
        print("%-44s %7.1f calls/s %8.0f audio-s/s  p50 %8.2f ms  p99 %8.2f ms  passes/call %.3f  launches/call %.1f  reps %s" % (
            k, v["calls_per_s"], v["audio_s_per_s"], v["p50_ms"], v["p99_ms"], v["passes_per_call"], v["launches_per_call"],
            ["%.1f" % x for x in v["calls_per_s_reps"]]))
    print("embeddings bit-identical across libraries, reps and thread counts:", res["embeddings_equal"])
    for t, v in res["forward"].items():
        print("B=64 t=%-5s fa_campplus_forward %8.3f ms  fa_campplus_forward_ext (every extent t) %8.3f ms  (%+.1f %%)  bit-identical %s" % (
            t, v["forward"], v["forward_ext"], 100 * (v["forward_ext"] / v["forward"] - 1), v["bit_identical"]))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(res, open(os.path.join(a.out, "spk_pool_probe.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
