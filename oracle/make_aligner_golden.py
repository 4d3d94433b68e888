"""Generate tests/golden/aligner_*.npz by running the UNMODIFIED reference MonotonicAligner (fa-zh) on CPU.

Run where the reference tree is present:   python oracle/make_aligner_golden.py
The reference is driven through its own plugin surface: AutoModel(model="MonotonicAligner", ..., init_param=<synthetic .pt>)
-> model.inference(data_in=[(wav, text), ...], data_type=("sound", "text"), tokenizer=CharTokenizer).  Weights, waveforms and
transcripts come from funasr_b200/synth.py (seeded), so only outputs are stored.
"""
import copy
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import ref_shim  # noqa: E402
import aligner_oracle  # noqa: E402
from make_golden import GOLD, write_cmvn_file  # noqa: E402
from funasr_b200 import synth  # noqa: E402

N_CHARS = 400
CASES = {
    # name: (cfg, weight seed, [(seconds, wav seed, n_chars, text seed)])
    # tiny: texts of different lengths; the second has more characters than its 1.5 s can fire for (the re-integration branch of
    # ts_prediction_lfr6_standard); the third is one character
    "aligner_tiny_ragged3": (synth.ALIGNER_TINY, 5, [(4.0, 1, 14, 1), (1.5, 2, 90, 2), (2.5, 3, 1, 3)]),
    "aligner_fa_zh_single": (synth.ALIGNER_FA_ZH, 6, [(25.0, 4, 80, 4)]),
}


def make_text(n: int, seed: int) -> str:
    """n space-separated characters of the synthetic token list (CharTokenizer split_with_space)."""
    g = torch.Generator().manual_seed(31 * seed + 7)
    toks = synth.aligner_token_list(N_CHARS)
    return " ".join(toks[3 + int(i)] for i in torch.randint(0, N_CHARS, (n,), generator=g))


def build_reference(cfg, wseed, cmvn_file, tmp):
    from funasr import AutoModel
    pt = os.path.join(tmp, "aligner_%d_%d.pt" % (cfg.enc_layers, wseed))
    torch.save(synth.make_aligner_state_dict(cfg, wseed), pt)
    return AutoModel(
        model="MonotonicAligner",
        model_conf=dict(length_normalized_loss=False, predictor_bias=1),
        encoder="SANMEncoder",
        encoder_conf=dict(output_size=cfg.d_model, attention_heads=cfg.heads, linear_units=cfg.ffn, num_blocks=cfg.enc_layers,
                          dropout_rate=0.1, positional_dropout_rate=0.1, attention_dropout_rate=0.1, input_layer="pe",
                          pos_enc_class="SinusoidalPositionEncoder", normalize_before=True, kernel_size=cfg.kernel, sanm_shfit=0,
                          selfattention_layer_type="sanm"),
        predictor="CifPredictorV3",
        predictor_conf=dict(idim=cfg.d_model, threshold=1.0, l_order=1, r_order=1, tail_threshold=cfg.tail_threshold, smooth_factor2=0.25,
                            noise_threshold2=0.01, upsample_times=3, use_cif1_cnn=False, upsample_type="cnn_blstm"),
        frontend="WavFrontend",
        frontend_conf=dict(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0,
                           cmvn_file=cmvn_file),
        tokenizer="CharTokenizer", tokenizer_conf=dict(token_list=synth.aligner_token_list(N_CHARS), unk_symbol="<unk>", split_with_space=True),
        device="cpu", ncpu=os.cpu_count(), disable_update=True, disable_pbar=True, init_param=pt,
    )


def run_case(name, cfg, wseed, specs, tmp):
    from funasr.utils.load_utils import extract_fbank
    from funasr.utils.timestamp_tools import ts_prediction_lfr6_standard
    cmvn_file = os.path.join(tmp, "am_%s.mvn" % name)
    write_cmvn_file(cmvn_file, synth.make_cmvn(cfg, seed=1))
    am = build_reference(cfg, wseed, cmvn_file, tmp)
    model, frontend, tokenizer = am.model, am.kwargs["frontend"], am.kwargs["tokenizer"]
    wavs = [synth.make_aligner_wav(sec, s) for (sec, s, _, _) in specs]
    texts = [make_text(n, ts) for (_, _, n, ts) in specs]
    with torch.no_grad():
        res, _ = model.inference(data_in=[(w.numpy(), t) for w, t in zip(wavs, texts)], key=["u%d" % i for i in range(len(wavs))],
                                 tokenizer=tokenizer, frontend=frontend, device="cpu", data_type=("sound", "text"))
        feats, flens = extract_fbank([w for w in wavs], frontend=frontend)
        enc, elens = model.encode(feats, flens)
        ids = [tokenizer.encode(t) for t in texts]
        tok = torch.tensor([len(i) + 1 for i in ids])
        _, _, us_alphas, us_peaks = model.calc_predictor_timestamp(enc, elens, tok)
    stamps = []
    for i in range(len(wavs)):
        n = int(elens[i]) * 3
        _, st = ts_prediction_lfr6_standard(us_alphas[i][:n].clone(), us_peaks[i][:n].clone(), copy.copy(tokenizer.ids2tokens(ids[i])))
        stamps.append(st)
    stride = 7 if cfg.enc_layers > 10 else 1
    margin = aligner_oracle.fire_margin(us_alphas, elens)
    out = dict(
        ids_flat=np.array([t for r in ids for t in r], dtype=np.int32), ids_len=np.array([len(r) for r in ids], dtype=np.int32),
        wav_spec=np.array([[sec, s] for (sec, s, _, _) in specs], dtype=np.float64),
        enc_lens=elens.numpy().astype(np.int32), enc_rows=np.arange(0, enc.shape[1], stride, dtype=np.int32),
        enc=enc[:, ::stride, :].numpy().astype(np.float32), us_alphas=us_alphas.numpy(), us_peaks=us_peaks.numpy(),
        stamps_flat=np.array([v for st in stamps for pair in st for v in pair], dtype=np.int32),
        stamps_len=np.array([len(st) for st in stamps], dtype=np.int32),
        final_text=np.array([r["text"] for r in res]),
        final_flat=np.array([v for r in res for pair in r["timestamp"] for v in pair], dtype=np.int32),
        final_len=np.array([len(r["timestamp"]) for r in res], dtype=np.int32),
        fire_margin=np.float64(margin),
    )
    np.savez_compressed(os.path.join(GOLD, name + ".npz"), **out)
    for st, r in zip(stamps, res):
        d = np.diff(np.array(st)[:, 0]) if len(st) > 1 else np.zeros(1)
        print("%s: %d chars, enc_len %s, stamp start gaps min/max %d/%d ms, text %r..." % (
            name, len(st), elens.tolist(), d.min(), d.max(), r["text"][:12]))
    print("%s: fire margin %.3e" % (name, margin))


if __name__ == "__main__":
    ref_shim.import_reference()
    with tempfile.TemporaryDirectory() as tmp:
        for name, (cfg, wseed, specs) in CASES.items():
            if len(sys.argv) > 1 and name not in sys.argv[1:]:
                continue
            run_case(name, cfg, wseed, specs, tmp)
