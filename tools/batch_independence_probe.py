"""Does a Paraformer row depend on the other rows of its batch or on the padded length?  Decodes utterance x alone and inside
batches with other utterances (longer, shorter, several), through FrontendEngine + ParaformerEngine.forward_feats(want_taps=True),
and compares x's row stage by stage over its valid region: features, encoder output, CIF alphas, acoustic embeddings, decoder
log-probs, ids.  Prints, per gemm mode and batch composition, each stage's max |difference| (0 = bit for bit) and the first stage that
differs.  Synthetic weights (PARAFORMER_TINY, the long-audio goldens' seed) and synthetic speech; needs a GPU.

    python tools/batch_independence_probe.py [--modes fp32,fp16x3] [--out DIR]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from funasr_b200 import synth  # noqa: E402
from funasr_b200.engine import FrontendEngine, ParaformerEngine, num_lfr_frames  # noqa: E402


def run(fe, eng, wavs, dev):
    lens = [w.numel() for w in wavs]
    pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(dev)
    feats, fl = fe(pad, torch.tensor(lens, dtype=torch.int32, device=dev), max(num_lfr_frames(n) for n in lens))
    out = eng.forward_feats(feats, fl, want_taps=True)
    torch.cuda.synchronize()
    return feats, out


def row_stages(feats, out, r, t, n_tok):
    return {"feats": feats[r, :t].float().cpu(), "enc": out["enc"][r, :t].float().cpu(), "alphas": out["alphas"][r, :t].float().cpu(),
            "acoustic": out["acoustic"][r, :n_tok].float().cpu(), "logp": out["logp"][r, :n_tok].float().cpu()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="fp32,fp16x3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = "cuda:0"
    cfg = synth.PARAFORMER_TINY
    p, cmvn = synth.make_state_dict(cfg, 3), synth.make_cmvn(cfg, 1)
    fe = FrontendEngine(cmvn, dev)
    x = synth.make_wav(40000, 11, "speechlike")
    others = {"alone": [], "+longer": [synth.make_wav(160000, 12, "speechlike")], "+shorter": [synth.make_wav(12000, 13, "speechlike")],
              "+7 mixed": [synth.make_wav(8000 + 9000 * k, 20 + k, "speechlike") for k in range(7)]}
    t = num_lfr_frames(x.numel())
    report = []
    for mode in a.modes.split(","):
        eng = ParaformerEngine(p, cfg, dev, gemm_mode=mode)
        base = None
        for name, extra in others.items():
            feats, out = run(fe, eng, [x] + extra, dev)
            n_tok = int(out["token_num"][0])
            st = row_stages(feats, out, 0, t, n_tok)
            st_ids = out["ids"][0]
            if base is None:
                base = (st, st_ids, n_tok)
                continue
            diffs = {k: (float((v - base[0][k]).abs().max()) if v.shape == base[0][k].shape else float("inf")) for k, v in st.items()}
            first = next((k for k, d in diffs.items() if d != 0.0), None)
            row = {"mode": mode, "batch": name, "token_num_equal": n_tok == base[2], "ids_equal": st_ids == base[1], "max_abs": diffs,
                   "first_stage_that_differs": first}
            report.append(row)
            print(json.dumps(row))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "batch_independence_probe.json"), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
