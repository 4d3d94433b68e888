"""SeacoParaformer through the C handle API, PARAFORMER_LARGE synthetic SeACo weights.
Usage: offline_seaco_probe.py [--batch 64] [--utt-seconds 30] [--reps 5] [--mode fp16x3] [--out DIR]

Two measurements, medians of --reps runs after a warm-up (a host clock around a call that ends in a device synchronise):
  embed: fa_offline_hotword_embed for 10, 100, 1 000 and 5 000 hotwords of 2-6 tokens (the hotword encoder on the GPU, rows copied back);
  step:  one fa_offline_infer_hw call on --batch utterances of --utt-seconds with no hotword rows, with 7 hotwords + <s> (no filter)
         and with 300 + <s> (the attention-score filter active at nfilter 50).
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
import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def median_seconds(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--utt-seconds", type=float, default=30.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--mode", default="fp16x3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from funasr_b200 import pack, synth
    from funasr_b200.offline import OfflineRecognizer
    cfg = synth.PARAFORMER_LARGE
    res = {"card": card(), "mode": a.mode, "batch": a.batch, "utt_seconds": a.utt_seconds}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "seaco.fab2")
        pack.write_seaco_model_file(path, synth.make_seaco_state_dict(cfg, 0), cfg, synth.make_cmvn(cfg, 1),
                                    no_bias=synth.seaco_no_bias_id(cfg), nfilter=50)
        rec = OfflineRecognizer(path, 0, a.mode)
    embed = {}
    for n in (10, 100, 1000, 5000):
        hw = synth.make_hotwords(n, cfg.vocab, seed=n)
        embed[n] = median_seconds(lambda: rec.hotword_embeddings(hw), a.reps) * 1e3
        print("embed %5d hotwords: %.3f ms" % (n + 1, embed[n]), flush=True)
    res["embed_ms"] = embed
    wavs = [synth.make_wav(int(a.utt_seconds * 16000), 100 + i).numpy() for i in range(a.batch)]
    step = {}
    for n in (0, 7, 300):
        rows = rec.hotword_embeddings(synth.make_hotwords(n, cfg.vocab, seed=5)) if n else None
        step[n] = median_seconds(lambda: rec.infer(wavs, hotword_embeddings=rows), a.reps) * 1e3
        print("step %dx%.0fs, %d hotwords: %.2f ms" % (a.batch, a.utt_seconds, n, step[n]), flush=True)
    res["step_ms"] = step
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "offline_seaco_probe.json"), "w") as f:
            json.dump(res, f, indent=1)
    rec.close()


if __name__ == "__main__":
    main()
