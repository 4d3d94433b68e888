"""Throughput of the recogniser's request pool: T threads on one handle, each sending seeded 5-15 s requests.
Usage: offline_pool_probe.py --libs NEW.so [OLD.so] [--threads 1,4,16,64] [--calls 128] [--reps 2] [--mode fp16x3] [--diarized] [--out DIR]

Each library named by --libs (for example this build and the parent commit's, built from their own trees) runs in a worker process of
its own, the libraries alternating, --reps times.  A worker opens one PARAFORMER_LARGE handle (synthetic weights written once by
funasr_b200.pack) and one synthetic FSMN-VAD handle, then for fa_offline_infer and fa_offline_infer_vad and each T: a warm-up, then
--calls requests shared out over T threads released together.  A request is one seeded 5-15 s utterance; the same request numbers give
the same audio in every worker.  Per (library, entry, T), as medians over the reps: audio-s/s (request seconds / wall time of the
window, which ends when every call has returned its host result), p50 and p99 call latency, and calls per GPU pack
(fa_offline_pool_stats, where the library has it).  Also checks that every library gives the same ids for every request, and prints the
card and its power limit read in the same run.  --out DIR writes the JSON there.

--diarized: the entry is fa_offline_infer_vad_spk instead, with the CAM++ fixture weights (tests/golden/spk_campplus_bn.npz) in the
same mode.  Request k is a seeded 2-5 min recording of turns of three synthetic voices (synth.make_voice_wav); even requests are
diarized, odd ones are plain fa_offline_infer_vad calls on the same handles.  Per (library, T) it adds the launches per call
(fa_launch_count) and, over the diarized requests' chunk counts (their VAD segments' sv_chunk windows), the device time and launch
count of the spectral stage of one pass: per recording fa_spk_laplacian + fa_spk_tridiagonalize + fa_spk_back_transform (k = 4), and
where the library has them the same sets through the _batch entries (CUDA events, medians of 5).  Ids and speakers are compared across
libraries."""
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

NAMES = ["fa_offline_init", "fa_offline_infer", "fa_offline_infer_vad", "fa_offline_result_count", "fa_offline_result_ids",
         "fa_offline_free_result", "fa_offline_uninit", "fa_offline_last_error", "fa_vad_init", "fa_vad_uninit", "fa_offline_pool_stats",
         "fa_offline_infer_vad_spk", "fa_offline_result_spk", "fa_offline_result_segments", "fa_spk_init", "fa_spk_uninit", "fa_launch_count",
         "fa_spk_laplacian_workspace_bytes", "fa_spk_laplacian", "fa_spk_tridiagonalize_workspace_bytes", "fa_spk_tridiagonalize",
         "fa_spk_back_transform", "fa_spk_laplacian_batch_workspace_bytes", "fa_spk_laplacian_batch",
         "fa_spk_tridiagonalize_batch_workspace_bytes", "fa_spk_tridiagonalize_batch", "fa_spk_back_transform_batch"]


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def request(k):
    """Request k: one seeded utterance of 5-15 s, speech-like."""
    from funasr_b200 import synth
    n = int(np.random.default_rng(1000 + k).integers(5 * 16000, 15 * 16000 + 1))
    return synth.make_wav(n, 7000 + k, "speechlike").numpy().astype(np.float32)


def voice_bank():
    """Twelve seeded speech turns, four for each of the three synthetic voices (synth.make_voice_wav), 2-6 s each."""
    from funasr_b200 import synth
    rng = np.random.default_rng(5000)
    return [synth.make_voice_wav([(v, float(rng.uniform(2, 6)), 0.0)], 9000 + 4 * v + i, lead_s=0.0).numpy().astype(np.float32)
            for v in range(3) for i in range(4)]


def voice_request(k, bank):
    """Request k of --diarized: a seeded 2-5 min recording of turns from the bank (three voices) with 0.3-2 s pauses."""
    rng = np.random.default_rng(6000 + k)
    target, parts, total = rng.uniform(120, 300) * 16000, [np.zeros(8000, np.float32)], 8000
    while total < target:
        turn = bank[int(rng.integers(0, len(bank)))]
        gap = np.zeros(int(rng.uniform(0.3, 2) * 16000), np.float32)
        parts += [turn, gap]
        total += turn.size + gap.size
    return np.concatenate(parts)


def spectral_stage(lib, ns):
    """Device ms and launches of one pass's spectral stage over sets of ns rows: per set with the single entries, and with the _batch
    entries where lib has them (CUDA events around the work, medians of 5 after a warm-up)."""
    import torch
    st = torch.cuda.current_stream()
    rng = np.random.default_rng(1)
    embs = [torch.from_numpy(rng.standard_normal((n, 192)).astype(np.float32)).cuda() for n in ns]
    ks = [min(4, n) for n in ns]
    out = {}

    def single():
        for e, n, k in zip(embs, ns, ks):
            ws = torch.empty(max(lib.fa_spk_laplacian_workspace_bytes(n, 192), lib.fa_spk_tridiagonalize_workspace_bytes(n)), dtype=torch.uint8, device="cuda")
            lap, tri, z = (torch.empty(n * n, dtype=torch.float64, device="cuda"), torch.empty(3 * n, dtype=torch.float64, device="cuda"),
                           torch.ones(k * n, dtype=torch.float64, device="cuda"))
            assert lib.fa_spk_laplacian(e.data_ptr(), n, 192, 0.022, lap.data_ptr(), ws.data_ptr(), ws.numel(), st.cuda_stream) == 0
            assert lib.fa_spk_tridiagonalize(lap.data_ptr(), n, tri.data_ptr(), tri[n:].data_ptr(), tri[2 * n:].data_ptr(), ws.data_ptr(),
                                             ws.numel(), st.cuda_stream) == 0
            assert lib.fa_spk_back_transform(lap.data_ptr(), tri[2 * n:].data_ptr(), n, z.data_ptr(), k, st.cuda_stream) == 0
    emb_all = torch.cat(embs)
    n_arr, k_arr = (C.c_int32 * len(ns))(*ns), (C.c_int32 * len(ns))(*ks)
    rows, sq = sum(ns), sum(n * n for n in ns)

    def batch():
        ws = torch.empty(max(lib.fa_spk_laplacian_batch_workspace_bytes(n_arr, len(ns), 192),
                             lib.fa_spk_tridiagonalize_batch_workspace_bytes(n_arr, len(ns))), dtype=torch.uint8, device="cuda")
        lap, tri = torch.empty(sq, dtype=torch.float64, device="cuda"), torch.empty(3 * rows, dtype=torch.float64, device="cuda")
        z = torch.ones(sum(k * n for k, n in zip(ks, ns)), dtype=torch.float64, device="cuda")
        assert lib.fa_spk_laplacian_batch(emb_all.data_ptr(), n_arr, len(ns), 192, 0.022, lap.data_ptr(), ws.data_ptr(), ws.numel(), st.cuda_stream) == 0
        assert lib.fa_spk_tridiagonalize_batch(lap.data_ptr(), n_arr, len(ns), tri.data_ptr(), tri[rows:].data_ptr(), tri[2 * rows:].data_ptr(),
                                               ws.data_ptr(), ws.numel(), st.cuda_stream) == 0
        assert lib.fa_spk_back_transform_batch(lap.data_ptr(), tri[2 * rows:].data_ptr(), n_arr, k_arr, len(ns), z.data_ptr(), st.cuda_stream) == 0
    for name, fn in (("single", single), ("batch", batch)):
        if name == "batch" and not hasattr(lib, "fa_spk_laplacian_batch"):
            continue
        fn()
        torch.cuda.synchronize()
        ms, launches = [], 0
        for _ in range(5):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            l0 = lib.fa_launch_count()
            a.record()
            fn()
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
            launches = lib.fa_launch_count() - l0
        out[name] = {"device_ms": statistics.median(ms), "launches": launches}
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
    lib = load(a.lib)
    from funasr_b200 import _abi
    h = lib.fa_offline_init(a.model.encode(), 0, _abi.GEMM_MODES[a.mode])
    v = lib.fa_vad_init(a.vad.encode(), 0)
    assert h and v, lib.fa_offline_last_error()
    s = lib.fa_spk_init(a.spk.encode(), 0, _abi.GEMM_MODES[a.mode]) if a.diarized else None
    assert h and v and (s or not a.diarized), lib.fa_offline_last_error()
    stats = hasattr(lib, "fa_offline_pool_stats")
    if a.diarized:
        bank = np.load(os.path.join(os.path.dirname(a.model), "voices.npz"))
        bank = [bank["t%d" % i] for i in range(len(bank.files))]
    wavs = [voice_request(k, bank) if a.diarized else request(k) for k in range(a.calls)]
    segs = {}

    def one(entry, k):
        w = wavs[k]
        ptrs = (C.c_void_p * 1)(w.ctypes.data)
        lens = (C.c_int64 * 1)(w.size)
        t0 = time.perf_counter()
        if entry == "infer":
            r = lib.fa_offline_infer(h, ptrs, lens, 1, 0)
        elif entry == "infer_vad_spk" and k % 2 == 0:
            r = lib.fa_offline_infer_vad_spk(h, v, s, ptrs, lens, 1, 0, None, 0, None, None, None, 0)
        else:
            r = lib.fa_offline_infer_vad(h, v, ptrs, lens, 1, 0, None, 0, None)
        assert r, lib.fa_offline_last_error()
        n = C.c_int32()
        p = lib.fa_offline_result_ids(r, 0, C.byref(n))
        ids = [p[i] for i in range(n.value)]
        if entry == "infer_vad_spk":
            p = lib.fa_offline_result_spk(r, 0, C.byref(n))
            ids += [-1] + [p[i] for i in range(n.value)]
            p = lib.fa_offline_result_segments(r, 0, C.byref(n))
            segs[k] = [(p[3 * i], p[3 * i + 1]) for i in range(n.value)]
        lib.fa_offline_free_result(r)
        return time.perf_counter() - t0, hashlib.sha1(np.asarray(ids, np.int32).tobytes()).hexdigest()[:16]

    def pool():
        if not stats:
            return 0, 0
        c, p = C.c_int64(), C.c_int64()
        lib.fa_offline_pool_stats(h, C.byref(c), C.byref(p))
        return c.value, p.value
    out = {}
    for entry in (("infer_vad_spk",) if a.diarized else ("infer", "infer_vad")):
        for T in a.threads:
            for k in range(min(4, a.calls)):                # warm-up: every shape class the window sees
                one(entry, k)
            lat, hashes = [None] * a.calls, [None] * a.calls
            bar = threading.Barrier(T + 1)

            def run(j):
                bar.wait()
                for k in range(j, a.calls, T):
                    lat[k], hashes[k] = one(entry, k)
            ts = [threading.Thread(target=run, args=(j,)) for j in range(T)]
            for t in ts:
                t.start()
            c0, p0 = pool()
            l0 = lib.fa_launch_count()
            bar.wait()
            t0 = time.perf_counter()
            for t in ts:
                t.join()
            wall = time.perf_counter() - t0
            c1, p1 = pool()
            launches = (lib.fa_launch_count() - l0) / a.calls
            seconds = sum(w.size for w in wavs) / 16000.0
            ls = sorted(lat)
            out["%s/%d" % (entry, T)] = {"audio_s_per_s": seconds / wall, "p50_ms": 1e3 * ls[len(ls) // 2],
                                         "p99_ms": 1e3 * ls[min(len(ls) - 1, int(0.99 * len(ls)))],
                                         "calls_per_pack": (c1 - c0) / (p1 - p0) if p1 > p0 else None, "launches_per_call": launches,
                                         "ids": hashes}
    if a.diarized:                                          # the diarized requests' chunk counts on the spectral path
        from funasr_b200.long_audio import speaker_chunks
        ns = [len(speaker_chunks(segs[k], wavs[k].size)) for k in sorted(segs)]
        ns = [n for n in ns if 20 <= n < 2048][:8]
        out["spectral"] = {"n": ns, **spectral_stage(lib, ns)}
        lib.fa_spk_uninit(s)
    lib.fa_offline_uninit(h)
    lib.fa_vad_uninit(v)
    json.dump(out, open(a.json, "w"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="+", default=[os.path.join(ROOT, "funasr_b200", "libfunasr_b200.so")])
    ap.add_argument("--threads", default="1,4,16,64")
    ap.add_argument("--calls", type=int, default=128)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--mode", default="fp16x3")
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--lib", default=None)
    ap.add_argument("--model", default=None)
    ap.add_argument("--vad", default=None)
    ap.add_argument("--json", default=None)
    ap.add_argument("--diarized", action="store_true")
    ap.add_argument("--spk", default=None)
    a = ap.parse_args()
    a.threads = [int(x) for x in a.threads.split(",")]
    if a.worker:
        return worker(a)
    from funasr_b200 import pack, synth
    tmp = tempfile.mkdtemp(prefix="pool_probe_")
    cfg = synth.PARAFORMER_LARGE
    model, vad = os.path.join(tmp, "large.fab2"), os.path.join(tmp, "vad.fab2")
    pack.write_model_file(model, synth.make_state_dict(cfg, 0), cfg, synth.make_cmvn(cfg, 1))
    pack.write_vad_model_file(vad, synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    spk = os.path.join(tmp, "spk.fab2")
    if a.diarized:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from test_spk_host import campplus_state_dict
        pack.write_campplus_model_file(campplus_state_dict(), spk)
        np.savez(os.path.join(tmp, "voices.npz"), **{"t%d" % i: t for i, t in enumerate(voice_bank())})
    runs = {lib: [] for lib in a.libs}
    for rep in range(a.reps):
        for lib in a.libs:                                  # alternating
            js = os.path.join(tmp, "r%d_%d.json" % (rep, a.libs.index(lib)))
            subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--lib", lib, "--model", model, "--vad", vad, "--json", js,
                            "--threads", ",".join(map(str, a.threads)), "--calls", str(a.calls), "--mode", a.mode, "--spk", spk]
                           + (["--diarized"] if a.diarized else []), check=True)
            runs[lib].append(json.load(open(js)))
    res = {"card": card(), "mode": a.mode, "calls": a.calls, "reps": a.reps, "libs": a.libs, "table": {}}
    ids = {}
    for lib in a.libs:
        for key in runs[lib][0]:
            rs = [r[key] for r in runs[lib]]
            if key == "spectral":
                res.setdefault("spectral", {})[os.path.relpath(lib, ROOT)] = {
                    "n": rs[0]["n"], **{w: {f: statistics.median(r[w][f] for r in rs) for f in ("device_ms", "launches")} for w in rs[0] if w != "n"}}
                continue
            med = {f: statistics.median(r[f] for r in rs) if rs[0][f] is not None else None
                   for f in ("audio_s_per_s", "p50_ms", "p99_ms", "calls_per_pack", "launches_per_call")}
            med["audio_s_per_s_reps"] = [r["audio_s_per_s"] for r in rs]
            res["table"]["%s %s" % (os.path.relpath(lib, ROOT), key)] = med
            for r in rs:
                ids.setdefault(key.split("/")[0], []).append(r["ids"])
    res["results_equal"] = all(all(x == v[0] for x in v) for v in ids.values())
    print("card:", res["card"])
    for k, v in res["table"].items():
        print("%-60s %9.1f audio-s/s  p50 %7.1f ms  p99 %7.1f ms  calls/pack %s  launches/call %.0f" % (
            k, v["audio_s_per_s"], v["p50_ms"], v["p99_ms"], "-" if v["calls_per_pack"] is None else "%.2f" % v["calls_per_pack"], v["launches_per_call"]))
    for lib, v in res.get("spectral", {}).items():
        print("%s spectral stage over n = %s:" % (lib, v["n"]), {w: v[w] for w in v if w != "n"})
    print("results equal across libraries, reps and thread counts:", res["results_equal"])
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(res, open(os.path.join(a.out, "offline_pool_probe.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
