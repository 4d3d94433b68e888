"""Forced alignment through the C handle API against the Python class: one fa_align_infer call (host waveforms and token ids in,
stamps out) and one MonotonicAlignerB200.inference call on the same batch, at the full fa-zh shape (synthetic ALIGNER_FA_ZH weights,
30 blocks of d = 320).  B utterances x S seconds with 7 tokens per second of transcript (210 at 30 s).  Per gemm mode: medians of
--reps alternating calls after a warm-up, host clock around calls that end in a synchronise; the stamps of both must be equal.
Prints one JSON line with the card name and power limit read in the same run; --out DIR writes it to DIR/offline_align_probe.json.

    python tools/offline_align_probe.py [--batch 64] [--seconds 30] [--reps 7] [--out DIR]
"""
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
import torch  # noqa: E402

from funasr_b200 import pack, synth  # noqa: E402
from funasr_b200.modules import WavFrontendB200  # noqa: E402
from funasr_b200.offline import OfflineAligner  # noqa: E402
from test_aligner_gpu import _CharTok, _model  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1000.0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("offline_align_probe needs a CUDA device")
    dev = "cuda:0"
    cfg, seed = synth.ALIGNER_FA_ZH, 6
    tokens = synth.aligner_token_list(400)
    wavs = [synth.make_aligner_wav(a.seconds, s).numpy() for s in range(a.batch)]
    n_tok = int(7 * a.seconds)
    rng = np.random.default_rng(0)
    ids = [[int(t) for t in rng.integers(3, 403, n_tok)] for _ in range(a.batch)]
    fe = WavFrontendB200(cmvn=synth.make_cmvn(cfg, seed=1), lfr_m=7, lfr_n=6, dither=0.0)
    tok = _CharTok(tokens)
    res = {"card": card(), "batch": a.batch, "seconds": a.seconds, "tokens": n_tok, "reps": a.reps, "modes": {}}
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "aligner.fab2")
        pack.write_aligner_model_file(path, synth.make_aligner_state_dict(cfg, seed), cfg, synth.make_cmvn(cfg, seed=1), token_list=tokens)
        for mode in ("fp32", "fp16x3"):
            al = OfflineAligner(path, 0, mode)
            model = _model(cfg, seed, mode)
            pairs = [(torch.from_numpy(w), t) for w, t in zip(wavs, ids)]

            def handle():
                return al.align(wavs, ids)

            def python():
                r, _ = model.inference(pairs, tokenizer=tok, frontend=fe, device=dev, data_type=("sound", "text"))
                return [x["timestamp"] for x in r]

            _, h_out = timed(handle)
            _, p_out = timed(python)
            th, tp = [], []
            for _ in range(a.reps):
                th.append(timed(handle)[0])
                tp.append(timed(python)[0])
            mh, mp = statistics.median(th), statistics.median(tp)
            res["modes"][mode] = {"handle_ms": round(mh, 2), "python_ms": round(mp, 2), "equal_stamps": h_out == p_out,
                                  "handle_audio_s_per_s": round(a.batch * a.seconds / (mh / 1000.0), 1)}
            al.close()
            del model
            torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "offline_align_probe.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
