"""Parity diagnostics on the GPU (writes gpurun_out/parity_diag.json):
  1. BiCif timestamps: exact rate of the per-token [start_ms, end_ms] against the unmodified reference's golden values, per
     precision mode, with the largest us_alphas difference;
  2. pred_timestamp (CIF fires of CifPredictorV2) exact rate against the oracle;
  3. seed sweep: >= 8 weight seeds of the full 50+16-layer model: smallest top-1/top-2 log-prob margin over the emitted tokens vs
     the arithmetic noise of the fp16x3 path (max |logp_fp16x3 - logp_fp32|), and whether the greedy ids of the two modes agree.
usage: python tools/parity_diag.py [bicif] [predts] [seeds N]"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
DEV = "cuda:0"


def bicif():
    from conftest import BICIF_CASES, gold_stamps, load_bicif_case
    from funasr_b200 import synth
    from funasr_b200.engine import FrontendEngine, ParaformerEngine, num_lfr_frames
    from funasr_b200.timestamps import ts_prediction_lfr6_standard
    out = {}
    for name in BICIF_CASES:
        cfg, wseed, wavs, cmvn, g = load_bicif_case(name)
        for mode in ("fp32", "fp16x3"):
            eng = ParaformerEngine(synth.make_bicif_state_dict(cfg, wseed), cfg, DEV, gemm_mode=mode, bicif=True)
            fe = FrontendEngine(cmvn, DEV)
            lens = [w.numel() for w in wavs]
            pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
            feats, fl = fe(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), max(num_lfr_frames(n) for n in lens))
            o = eng.forward_feats(feats, fl, want_taps=True)
            tok = torch.tensor(g["token_num"], dtype=torch.int32, device=DEV)
            ua, up = eng.upsample_timestamp(o["enc"], fl, tok)
            ua, up = ua.cpu().numpy(), up.cpu().numpy()
            want = gold_stamps(g)
            exact = total = 0
            worst = 0
            for i, ids in enumerate(o["ids"]):
                m = int(g["enc_lens"][i]) * 3
                got = ts_prediction_lfr6_standard(ua[i][:m], up[i][:m], ["t%d" % (t - 3) for t in ids])[1]
                for a, b in zip(got, want[i]):
                    total += 1
                    exact += a == b
                    worst = max(worst, abs(a[0] - b[0]), abs(a[1] - b[1]))
            out["%s/%s" % (name, mode)] = {
                "stamps": total, "exact": exact, "worst_ms": worst, "us_alphas_maxdiff": float(np.abs(ua - g["us_alphas"]).max()),
                "us_peaks_maxdiff": float(np.abs(up - g["us_peaks"]).max()), "ids_equal": [t for r in o["ids"] for t in r] == g["ids_flat"].tolist(),
                "alphas_maxdiff": float(np.abs(o["alphas"].cpu().numpy() - g["alphas"]).max())}
            print(name, mode, out["%s/%s" % (name, mode)], flush=True)
    return out


def predts():
    import paraformer_oracle as O
    from conftest import load_case, state_dict_for
    from funasr_b200 import synth
    from funasr_b200.engine import FrontendEngine, ParaformerEngine, num_lfr_frames
    from funasr_b200.timestamps import paraformer_timestamps
    out = {}
    for name in ("tiny_ragged3", "large_ragged2"):
        cfg, wseed, wavs, cmvn, g = load_case(name)
        p = state_dict_for(cfg, wseed)
        ora = O.paraformer_forward(wavs, p, cmvn, cfg.enc_layers, cfg.dec_layers)
        for mode in ("fp32", "fp16x3"):
            eng = ParaformerEngine(p, cfg, DEV, gemm_mode=mode)
            fe = FrontendEngine(cmvn, DEV)
            lens = [w.numel() for w in wavs]
            pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
            feats, fl = fe(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), max(num_lfr_frames(n) for n in lens))
            o = eng.forward_feats(feats, fl, want_taps=True)
            al, pk = o["alphas"].cpu().numpy(), o["peaks"].cpu().numpy()
            exact = total = worst = 0
            for i in range(len(wavs)):
                want = paraformer_timestamps(ora["peaks"][i].numpy(), ora["alphas"][i].numpy(), [str(t) for t in ora["ids"][i]])[1]
                got = paraformer_timestamps(pk[i], al[i], [str(t) for t in o["ids"][i]])[1]
                for a, b in zip(got, want):
                    total += 1
                    exact += a == b
                    worst = max(worst, abs(a[0] - b[0]), abs(a[1] - b[1]))
            out["%s/%s" % (name, mode)] = {"stamps": total, "exact": exact, "worst_ms": worst,
                                           "alphas_maxdiff": float(np.abs(al - ora["alphas"].numpy()).max()),
                                           "fires_equal": bool(((pk >= 1.0 - 1e-4) == (ora["peaks"].numpy() >= 1.0 - 1e-4)).all())}
            print(name, mode, out["%s/%s" % (name, mode)], flush=True)
    return out


def seeds(n):
    from funasr_b200 import synth
    from funasr_b200.engine import FrontendEngine, ParaformerEngine
    cfg = synth.PARAFORMER_LARGE
    cmvn = synth.make_cmvn(cfg, 1)
    fe = FrontendEngine(cmvn, DEV)
    rows = []
    for s in range(n):
        wavs = [synth.make_wav(480000, 500 + 2 * s, "speechlike"), synth.make_wav(480000, 501 + 2 * s, "speechlike") * 0.6]
        pad = torch.stack(wavs).to(DEV)
        feats, fl = fe(pad, torch.full((2,), 480000, dtype=torch.int32, device=DEV), 500)
        p = synth.make_state_dict(cfg, 100 + s)
        res = {}
        for mode in ("fp32", "fp16x3"):
            eng = ParaformerEngine(p, cfg, DEV, gemm_mode=mode)
            o = eng.forward_feats(feats, fl, want_taps=True)
            res[mode] = (o["logp"].double().cpu(), o["token_num"].tolist(), o["ids"])
            del eng
            torch.cuda.empty_cache()
        lp32, tok, ids32 = res["fp32"]
        lp3, tok3, ids3 = res["fp16x3"]
        n_c = min(lp32.shape[1], lp3.shape[1])
        valid = torch.arange(n_c)[None, :] < torch.tensor(tok)[:, None]
        top2 = torch.topk(lp32[:, :n_c], 2, dim=-1).values
        margin = (top2[..., 0] - top2[..., 1])[valid]
        diff = (lp3[:, :n_c] - lp32[:, :n_c]).abs()
        rows.append({"weight_seed": 100 + s, "tokens": tok, "token_num_equal": tok == tok3, "ids_equal": ids32 == ids3,
                     "min_top2_margin": float(margin.min()), "p01_top2_margin": float(margin.kthvalue(max(1, int(0.01 * margin.numel()))).values),
                     "max_abs_logp_diff": float(diff[valid].max()), "rel_logp_err": float(diff[valid].max() / lp32[:, :n_c][valid].abs().max()),
                     "argmax_noise_at_valid": float(torch.gather(diff, 2, lp32[:, :n_c].argmax(-1, keepdim=True)).squeeze(-1)[valid].max())})
        print(rows[-1], flush=True)
    return rows


if __name__ == "__main__":
    args = sys.argv[1:] or ["bicif", "predts", "seeds", "8"]
    out = {}
    if "bicif" in args:
        out["bicif_timestamps"] = bicif()
    if "predts" in args:
        out["pred_timestamp"] = predts()
    if "seeds" in args:
        k = args.index("seeds")
        out["seed_sweep"] = seeds(int(args[k + 1]) if k + 1 < len(args) and args[k + 1].isdigit() else 8)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    path = os.path.join(ROOT, "gpurun_out", "parity_diag.json")
    prev = {}
    if os.path.exists(path):
        try:
            prev = json.load(open(path))
        except Exception:
            prev = {}
    prev.update(out)
    json.dump(prev, open(path, "w"), indent=1)
    print("wrote", path)
