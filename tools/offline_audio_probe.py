"""Cost of audio at other rates and PCM layouts in the C handle API: the fa_ingest_pcm kernel alone, and the whole
fa_offline_infer_audio call against fa_offline_infer on the same audio already resampled to 16 kHz.
Usage: offline_audio_probe.py [--batch 64] [--seconds 30] [--reps 7] [--mode fp16x3] [--out DIR]

PARAFORMER_LARGE synthetic weights.  Three inputs of --batch speech-like utterances of --seconds each: 8 kHz s16 mono, 44.1 kHz s16
stereo and 48 kHz f32 mono, each in both resamplers (loader, runtime).  The ingest time is CUDA events around --reps x 10
launches of fa_ingest_pcm on the staged batch (median per launch).  The whole-call comparison alternates fa_offline_infer_audio on the
raw batch with fa_offline_infer_hw on its 16 kHz rows (the rows fa_ingest_pcm produced, copied to the host) --reps times; each time is a
host clock around a call that ends in the handle's own synchronisation; medians and spreads are reported.  The card's name and power
limit are read in the same run.  --out DIR writes the JSON there."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


INPUTS = [("8k_s16_mono", 1, 1, 8000), ("44k1_s16_stereo", 1, 2, 44100), ("48k_f32_mono", 0, 1, 48000)]


def make_batch(fmt, ch, rate, batch, seconds):
    from funasr_b200 import synth
    n = int(seconds * rate)
    out = []
    for i in range(batch):
        w = synth.make_wav(n, 300 + i, "speechlike").numpy()
        x = np.stack([w, w * 0.8], axis=1) if ch == 2 else w
        out.append(np.ascontiguousarray(x, np.float32) if fmt == 0 else np.clip(np.round(x * 32767), -32768, 32767).astype(np.int16))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--mode", default="fp16x3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("offline_audio_probe: no CUDA device (this measurement has no CPU path)")
    from funasr_b200 import _abi, pack, synth
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    from test_audio_in_gpu import _Table
    lib = _abi.load()
    info = card()
    cfg = synth.PARAFORMER_LARGE
    path = os.path.join(tempfile.mkdtemp(), "model.fab2")
    pack.write_model_file(path, synth.make_state_dict(cfg, 0), cfg, synth.make_cmvn(cfg, 1))
    h = lib.fa_offline_init(path.encode(), 0, _abi.GEMM_MODES[a.mode])
    assert h, lib.fa_offline_last_error()
    dev = "cuda:0"
    st = torch.cuda.current_stream(dev).cuda_stream
    results = {"card": info, "batch": a.batch, "seconds": a.seconds, "gemm_mode": a.mode, "cases": []}

    def result_ids(res):
        assert res, lib.fa_offline_last_error().decode()
        cnt = C.c_int32(0)
        ids = []
        for i in range(lib.fa_offline_result_count(res)):
            p = lib.fa_offline_result_ids(res, i, C.byref(cnt))
            ids.append([int(p[k]) for k in range(cnt.value)])
        lib.fa_offline_free_result(res)
        return ids

    for name, fmt, ch, rate in INPUTS:
        arrs = make_batch(fmt, ch, rate, a.batch, a.seconds)
        ptrs = (C.c_void_p * a.batch)(*[x.ctypes.data for x in arrs])
        lens = (C.c_int64 * a.batch)(*[x.shape[0] for x in arrs])
        for resampler in ("loader", "runtime"):
            mode = _abi.RESAMPLERS[resampler]
            # the kernel alone on the staged batch
            tab = _Table(rate, mode)
            raw = torch.from_numpy(np.concatenate([x.reshape(-1).view(np.uint8) for x in arrs])).to(dev)
            n = arrs[0].shape[0]
            per = arrs[0].nbytes
            L = tab.len16(n)
            stride = (L + 3) // 4 * 4
            rows = torch.tensor([[i * per, n, L] for i in range(a.batch)], dtype=torch.int64, device=dev)
            y = torch.empty((a.batch, stride), dtype=torch.float32, device=dev)

            def launch():
                _abi.check(lib.fa_ingest_pcm(raw.data_ptr(), rows.data_ptr(), a.batch, fmt, ch, C.byref(tab.t), y.data_ptr(), stride, st),
                           "fa_ingest_pcm")
            for _ in range(3):
                launch()
            ms = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(10):
                    launch()
                e1.record()
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1) / 10)
            rows16 = [np.ascontiguousarray(r[:L]) for r in y.cpu().numpy()]
            p16 = (C.c_void_p * a.batch)(*[x.ctypes.data for x in rows16])
            l16 = (C.c_int64 * a.batch)(*[x.shape[0] for x in rows16])
            d = _abi.FaAudioFormat(fmt, ch, rate, mode)

            def call_new():
                t0 = time.perf_counter()
                ids = result_ids(lib.fa_offline_infer_audio(h, ptrs, lens, a.batch, C.byref(d), None, 0, None, None))
                return ids, time.perf_counter() - t0

            def call_old():
                t0 = time.perf_counter()
                ids = result_ids(lib.fa_offline_infer_hw(h, p16, l16, a.batch, 0, None, 0))
                return ids, time.perf_counter() - t0
            ids_new, _ = call_new()
            ids_old, _ = call_old()
            same = ids_new == ids_old
            t_new, t_old = [], []
            for _ in range(a.reps):
                t_new.append(call_new()[1] * 1e3)
                t_old.append(call_old()[1] * 1e3)
            case = {"input": name, "resampler": resampler, "ingest_ms_median": statistics.median(ms), "ingest_ms_range": [min(ms), max(ms)],
                    "call_ms_median": statistics.median(t_new), "call_ms_range": [min(t_new), max(t_new)],
                    "preresampled_call_ms_median": statistics.median(t_old), "preresampled_call_ms_range": [min(t_old), max(t_old)],
                    "ingest_share_of_call": statistics.median(ms) / statistics.median(t_new), "same_ids": same}
            results["cases"].append(case)
            print(json.dumps(case))
    lib.fa_offline_uninit(h)
    print("card:", info)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "offline_audio_probe.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
