"""Speaker diarization through the C handle API: where the time goes.
Usage: offline_spk_probe.py [--reps 5] [--seconds 600] [--out DIR]

For N = 200, 800 and 2 047 speaker chunks (seeded three-voice mixtures of 192-wide embeddings), medians of --reps runs after a warm-up:
  device: fa_spk_laplacian + fa_spk_tridiagonalize, and fa_spk_back_transform (CUDA events);
  host:   fa_sym_tridiag_smallest_host (16 eigenvalues, the eigengap's vectors), fa_spk_kmeans_host, fa_spk_merge_by_cos_host and
          fa_spk_postprocess_host (host clock);
  scipy:  scipy.linalg.eigh of the same float32 Laplacian, the reference's dense solve (host clock, for comparison).
Then one --seconds two-voice recording (synthetic voices, PARAFORMER_TINY + FSMN-VAD + the CAM++ fixture weights, fp32) through
fa_offline_infer_vad and fa_offline_infer_vad_spk, alternating (host clock around calls that end in a synchronise).
Prints the card and its power limit read in the same call; --out DIR writes the JSON there."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import scipy.linalg  # noqa: E402
import torch  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def median(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        ts.append(fn())
    return statistics.median(ts)


def clustering(lib, n, reps):
    from funasr_b200 import _abi
    from funasr_b200 import diarization as D
    rng = np.random.RandomState(n)
    centers = rng.randn(3, 192)
    x = (centers[rng.randint(0, 3, size=n)] + 2.0 * rng.randn(n, 192)).astype(np.float32)
    dev = torch.device("cuda:0")
    emb = torch.from_numpy(x).to(dev)
    lap = torch.empty((n, n), dtype=torch.float64, device=dev)
    tri = torch.empty(3 * n, dtype=torch.float64, device=dev)
    ws = torch.empty(max(int(lib.fa_spk_laplacian_workspace_bytes(n, 192)), int(lib.fa_spk_tridiagonalize_workspace_bytes(n))),
                     dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    state = {}

    def device_part():
        ev[0].record()
        _abi.check(lib.fa_spk_laplacian(emb.data_ptr(), n, 192, 0.022, lap.data_ptr(), ws.data_ptr(), ws.numel(), st), "laplacian")
        _abi.check(lib.fa_spk_tridiagonalize(lap.data_ptr(), n, tri.data_ptr(), tri[n:].data_ptr(), tri[2 * n:].data_ptr(), ws.data_ptr(),
                                             ws.numel(), st), "tridiagonalize")
        ev[1].record()
        de = tri.cpu().numpy()
        state["d"], state["e"] = np.ascontiguousarray(de[:n]), np.ascontiguousarray(de[n:2 * n - 1])
        t0 = time.perf_counter()
        w = np.zeros(16)
        lib.fa_sym_tridiag_smallest_host(state["d"].ctypes.data, state["e"].ctypes.data, n, 16, 0, w.ctypes.data, None)
        k = int(np.argmax(np.diff(w))) + 1
        z = np.zeros((k, n))
        lib.fa_sym_tridiag_smallest_host(state["d"].ctypes.data, state["e"].ctypes.data, n, 16, k, w.ctypes.data, z.ctypes.data)
        state["host_eig"] = time.perf_counter() - t0
        zd = torch.from_numpy(z).to(dev)
        ev[1].synchronize()
        t1 = torch.cuda.Event(enable_timing=True)
        t1.record()
        _abi.check(lib.fa_spk_back_transform(lap.data_ptr(), tri[2 * n:].data_ptr(), n, zd.data_ptr(), k, st), "back_transform")
        ev[2].record()
        ev[2].synchronize()
        state["vecs"] = np.ascontiguousarray(zd.cpu().numpy().T)
        state["k"] = k
        state["back"] = t1.elapsed_time(ev[2]) / 1e3
        return ev[0].elapsed_time(ev[1]) / 1e3

    lap_tri = median(device_part, reps)
    back = state["back"]
    host_eig = state["host_eig"]

    def host_rest():
        t0 = time.perf_counter()
        lab = np.zeros(n, np.int32)
        lib.fa_spk_kmeans_host(state["vecs"].ctypes.data, n, state["k"], state["k"], 0, 10, 300, lab.ctypes.data)
        lib.fa_spk_merge_by_cos_host(lab.ctypes.data, x.ctypes.data, n, 192, 0.78)
        times = np.ascontiguousarray(np.stack([np.arange(n) * 0.75, np.arange(n) * 0.75 + 1.5], 1))
        turns = np.zeros((n, 3))
        lib.fa_spk_postprocess_host(times.ctypes.data, lab.ctypes.data, n, turns.ctypes.data)
        return time.perf_counter() - t0

    host_rest_s = median(host_rest, reps)
    ref_lap = D.SpectralCluster().laplacian(0.5 * (lambda p: p + p.T)(D.SpectralCluster().p_pruning(D.SpectralCluster.sim_mat(x))))

    def scipy_eigh():
        t0 = time.perf_counter()
        scipy.linalg.eigh(ref_lap)
        return time.perf_counter() - t0

    return {"n": n, "k": state["k"], "device_laplacian_tridiagonalize_ms": lap_tri * 1e3, "device_back_transform_ms": back * 1e3,
            "host_bisection_inverse_iteration_ms": host_eig * 1e3, "host_kmeans_merge_post_ms": host_rest_s * 1e3,
            "scipy_eigh_float32_ms": median(scipy_eigh, max(1, reps // 2)) * 1e3}


def long_audio(seconds, reps):
    from funasr_b200 import pack, synth
    from funasr_b200.offline import OfflineRecognizer, OfflineSpeaker, OfflineVad
    from test_spk_host import campplus_state_dict
    d = tempfile.mkdtemp()
    cfg = synth.PARAFORMER_TINY
    asr_f, vad_f, spk_f = (os.path.join(d, n) for n in ("asr.fab2", "vad.fab2", "spk.fab2"))
    pack.write_model_file(asr_f, synth.make_state_dict(cfg, 3), cfg, synth.make_cmvn(cfg, 1))
    pack.write_vad_model_file(vad_f, synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    pack.write_campplus_model_file(campplus_state_dict(), spk_f)
    rec, vad, spk = OfflineRecognizer(asr_f, 0, "fp32"), OfflineVad(vad_f, 0), OfflineSpeaker(spk_f, 0, "fp32")
    turns = max(2, int(seconds / 10))
    wav = synth.make_voice_wav([(v, 6.0, 4.0) for v in (0, 1) * (turns // 2)], 1).numpy()
    plain = rec.infer_long([wav], vad)[0]
    with_spk = rec.infer_long([wav], vad, spk=spk)[0]
    ta, tb = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        rec.infer_long([wav], vad)
        ta.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        rec.infer_long([wav], vad, spk=spk)
        tb.append(time.perf_counter() - t0)
    return {"seconds": wav.size / 16000, "segments": len(plain["vad_segments"]), "speakers": sorted(set(with_spk["spk"])),
            "same_ids_and_segments": {k: v for k, v in with_spk.items() if k != "spk"} == plain,
            "infer_vad_ms": statistics.median(ta) * 1e3, "infer_vad_spk_ms": statistics.median(tb) * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=600)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from funasr_b200 import _abi
    lib = _abi.load()
    out = {"card": card(), "clustering": [clustering(lib, n, a.reps) for n in (200, 800, 2047)], "long_audio": long_audio(a.seconds, a.reps)}
    out["card_after"] = card()
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "offline_spk_probe.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
