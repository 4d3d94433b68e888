"""MonotonicAligner (fa-zh, synthetic weights) throughput on the GPU: B utterances x S seconds with ~7 characters per second of
transcript, waveforms resident on the device.  Per precision: median of N timed runs (CUDA events, after a warm-up) of the whole
alignment (frontend -> encoder -> upsample + BLSTM -> scan) and of each stage; then a torch.profiler kernel table in a run of its
own.  Prints one JSON line with the card name, power limit and SM clock read in the same run.  With --out DIR it also writes
DIR/aligner_probe.json and the kernel table to DIR/aligner_kernels.txt (without it the table goes to stdout).

    python tools/aligner_probe.py [--batch 64] [--seconds 30] [--runs 5] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from funasr_b200 import synth  # noqa: E402
from funasr_b200.engine import AlignerEngine, FrontendEngine, num_lfr_frames  # noqa: E402
from funasr_b200.timestamps import ts_prediction_lfr6_standard  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("aligner_probe needs a CUDA device")
    dev = "cuda:0"
    cfg = synth.ALIGNER_FA_ZH
    sd = synth.make_aligner_state_dict(cfg, 6)
    n = int(a.seconds * 16000)
    wav = torch.stack([synth.make_aligner_wav(a.seconds, s) for s in range(a.batch)]).to(dev)
    wl = torch.full((a.batch,), n, dtype=torch.int32, device=dev)
    tmax = num_lfr_frames(n)
    n_chars = int(7 * a.seconds)
    tokens = [synth.aligner_token_list()[3 + (i % 400)] for i in range(n_chars)]
    tok = torch.full((a.batch,), n_chars + 1, dtype=torch.int32)
    fe = FrontendEngine(synth.make_cmvn(cfg, seed=1), dev)
    res = {"card": card(), "batch": a.batch, "seconds": a.seconds, "chars": n_chars, "runs": a.runs, "modes": {}}
    for mode in ("fp32", "fp16x3", "fp16"):
        eng = AlignerEngine(sd, cfg, dev, gemm_mode=mode)

        def stages():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
            feats, lens = fe(wav, wl, tmax)
            enc = eng.encode(feats, lens)
            ev[1].record()
            ua, up = eng.upsample_timestamp(enc, lens, tok)
            ev[2].record()
            ua, up, el = ua.cpu().numpy(), up.cpu().numpy(), lens.cpu().tolist()
            for i in range(a.batch):
                ts_prediction_lfr6_standard(ua[i][:3 * el[i]], up[i][:3 * el[i]], tokens, want_text=False)
            ev[3].record()
            torch.cuda.synchronize()
            return [ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3]), ev[0].elapsed_time(ev[3])]

        stages()
        stages()
        cols = zip(*[stages() for _ in range(a.runs)])            # per stage: the a.runs timings
        med = [sorted(col)[len(col) // 2] for col in cols]
        res["modes"][mode] = {"frontend_encoder_ms": med[0], "upsample_blstm_alphas_ms": med[1], "scan_host_ms": med[2], "total_ms": med[3],
                              "audio_s_per_s": a.batch * a.seconds / (med[3] / 1000.0)}
        if mode == "fp16x3":
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                stages()
            table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=25)
            if a.out:
                os.makedirs(a.out, exist_ok=True)
                with open(os.path.join(a.out, "aligner_kernels.txt"), "w") as f:
                    f.write(table)
            else:
                print(table)
        del eng
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "aligner_probe.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
