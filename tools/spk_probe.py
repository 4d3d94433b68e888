"""CAM++ speaker-embedding throughput on the GPU.  Usage: spk_probe.py [--chunks 800] [--reps 5] [--out DIR]

Prints the card, its power limit and clocks, then for each gemm_mode the time to embed --chunks 1.5 s chunks (about 10 min of speech
at sv_chunk's 0.75 s shift) from a device-resident waveform batch (CUDA events around features + forward, median of --reps after a
warm-up) and the rate of algorithmic work at 1.67 GFLOP per chunk; a torch.profiler per-kernel table of one fp16x3 call (--out DIR:
kernels.txt); and the whole LongAudioPipeline (VAD + tiny Paraformer) on a synthetic multi-speaker recording with and without
spk_model."""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

GFLOP_PER_CHUNK = 1.67
DEV = "cuda:0"


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts), min(ts), max(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=800)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spk_probe needs a CUDA device")
    from funasr_b200 import synth
    from funasr_b200.campplus import CampplusEngine
    from test_spk_host import campplus_state_dict
    print("card:", card())
    sd = campplus_state_dict()
    rec = synth.make_voice_wav([(v % 3, 8.0, 0.2) for v in range(8)], 11)                    # ~66 s of three voices
    starts = (np.arange(a.chunks) * 12000) % (rec.numel() - 24000)
    wav = torch.stack([rec[s:s + 24000] for s in starts]).to(DEV)
    lens = torch.full((a.chunks,), 24000, dtype=torch.int32, device=DEV)
    res = {"card": card(), "chunks": a.chunks}
    for mode in ("fp32", "fp16x3", "fp16"):
        eng = CampplusEngine(sd, DEV, mode)
        med, lo, hi = timed(lambda: eng.embed_wav(wav, lens, [24000] * a.chunks), a.reps)
        rate = GFLOP_PER_CHUNK * a.chunks / (med / 1e3) / 1e3
        print("%-7s %d chunks: median %.2f ms (min %.2f, max %.2f) -> %.1f TFLOP/s algorithmic, %.0f chunks/s" % (
            mode, a.chunks, med, lo, hi, rate, a.chunks / (med / 1e3)))
        res[mode] = {"median_ms": med, "min_ms": lo, "max_ms": hi, "tflops": rate}
    # per-kernel split (separate run: tracing slows the host)
    eng = CampplusEngine(sd, DEV, "fp16x3")
    eng.embed_wav(wav, lens, [24000] * a.chunks)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.embed_wav(wav, lens, [24000] * a.chunks)
        torch.cuda.synchronize()
    us, calls = collections.Counter(), collections.Counter()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name.split("(")[0].split("<")[0]
            us[name] += e.device_time if hasattr(e, "device_time") else e.cuda_time
            calls[name] += 1
    total = sum(us.values())
    lines = ["%-8s %10s %7s  %s" % ("calls", "total_ms", "share", "kernel")]
    for k, v in us.most_common():
        lines.append("%-8d %10.3f %6.1f%%  %s" % (calls[k], v / 1e3, 100.0 * v / total, k))
    print("\n".join(lines))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "kernels.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")
    # the whole long-audio pipeline with and without diarization
    from test_campplus_gpu import _pipeline
    import funasr_b200
    pipe, parts = _pipeline("fp16x3")
    plain = funasr_b200.LongAudioPipeline(*parts, device=DEV)
    long_wav = synth.make_voice_wav([(v % 2, 3.0, 2.5) for v in range(110)], 12).numpy()          # ~10 min
    for name, p in (("without spk_model", plain), ("with spk_model", pipe)):
        med, lo, hi = timed(lambda: p.generate(long_wav, key="rec", pred_timestamp=True), max(2, a.reps // 2))
        print("LongAudioPipeline %s: %.1f s of audio, median %.1f ms (min %.1f, max %.1f)" % (name, long_wav.size / 16000, med, lo, hi))
        res["pipeline " + name] = {"median_ms": med, "audio_s": long_wav.size / 16000}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
