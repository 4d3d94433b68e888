"""Cost of the BiCif timestamp head in the C handle API: fa_offline_infer on the same batch with and without the head.
Usage: offline_stamps_probe.py [--batch 64] [--seconds 30] [--reps 7] [--mode fp16x3] [--out DIR]

PARAFORMER_LARGE synthetic BiCif weights (synth.make_bicif_state_dict) packed twice: with the timestamp head (a BiCifParaformer file:
CifPredictorV3's token branch + upsample GEMM, BLSTM, upsampled CIF, host stamps) and without it (the same state minus the head, a plain
Paraformer file).  One batch of --batch synthetic speech-like utterances of --seconds each.  After a warm-up of both handles, the two
calls run alternately --reps times; each time is a host clock around a call that ends in the handle's own synchronisation.  Reports the
medians, their spread, the added ms and share per call, and the card and its power limit read in the same run.  --out DIR writes the
JSON there."""
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
import torch  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--mode", default="fp16x3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("offline_stamps_probe: no CUDA device (this measurement has no CPU path)")
    from funasr_b200 import pack, synth
    from funasr_b200.offline import OfflineRecognizer
    info = card()
    cfg = synth.PARAFORMER_LARGE
    state = synth.make_bicif_state_dict(cfg, 0)
    cmvn = synth.make_cmvn(cfg, 1)
    td = tempfile.mkdtemp()
    with_head, without = os.path.join(td, "bicif.fab2"), os.path.join(td, "plain.fab2")
    pack.write_model_file(with_head, state, cfg, cmvn)
    pack.write_model_file(without, {k: v for k, v in state.items()
                                    if not k.startswith(("predictor.upsample_cnn.", "predictor.blstm.", "predictor.cif_output2."))}, cfg, cmvn)
    del state
    n = int(a.seconds * 16000)
    wavs = [synth.make_wav(n, 100 + i, "speechlike").numpy() for i in range(a.batch)]
    recs = {"with_head": OfflineRecognizer(with_head, 0, a.mode), "without_head": OfflineRecognizer(without, 0, a.mode)}
    assert recs["with_head"].has_timestamps and not recs["without_head"].has_timestamps

    def call(name):
        t0 = time.perf_counter()
        out = recs[name].infer_stamped(wavs)                   # returns after the handle's device synchronisation and host stamps
        return out, time.perf_counter() - t0

    for name in recs:                                          # warm-up: every buffer grows to this batch
        call(name)
        call(name)
    t = {k: [] for k in recs}
    for _ in range(a.reps):
        for name in recs:
            out, dt = call(name)
            t[name].append(dt)
            if name == "with_head":
                tokens = sum(len(r["token_int"]) for r in out)
                stamps = sum(len(r["timestamp"]) for r in out)
    med = {k: statistics.median(v) for k, v in t.items()}
    res = {"card": info, "mode": a.mode, "batch": a.batch, "seconds_each": a.seconds, "reps": a.reps,
           "with_head_ms": 1e3 * med["with_head"], "without_head_ms": 1e3 * med["without_head"],
           "head_added_ms": 1e3 * (med["with_head"] - med["without_head"]),
           "head_share_of_call": (med["with_head"] - med["without_head"]) / med["with_head"],
           "spread": {k: (max(v) - min(v)) / statistics.median(v) for k, v in t.items()},
           "audio_s_per_s": {k: a.batch * a.seconds / v for k, v in med.items()},
           "tokens": tokens, "stamps": stamps}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "offline_stamps_probe_b%d_%s.json" % (a.batch, a.mode)), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
