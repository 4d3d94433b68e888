"""Writes tests/golden/live_reference.json and tests/golden/live_reference_components.npz: what the unmodified reference's own
functions return on the seeded inputs of four host tests, so that those tests compare with the reference wherever they run:
  * funasr.utils.vad_utils.merge_vad on 50 random segment lists                    (tests/test_vad_host.py)
  * the C++ runtime's end-point detector (oracle/_ref/libvad_ref.so) on 60 random posterior tracks and on the Python reference's
    scores of three golden VAD cases                                               (tests/test_vad_host.py)
  * ContextualParaformer.generate_hotwords_list on a string and a .txt source      (tests/test_properties_host.py)
  * the SANMEncoder / CifPredictorV2 classes on random features                    (tests/test_oracle_golden.py)
  * funasr.utils.timestamp_tools.ts_prediction_lfr6_standard on 50 random traces   (tests/test_timestamps.py)
The inputs are regenerated from the same seeds by the tests.  Run where the reference tree is present:
python oracle/make_live_golden.py"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import knf_ref  # noqa: E402
import make_vad_cpp_golden as mk  # noqa: E402
import ref_shim  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def merge_vad_cases():
    """The 50 seeded segment lists of test_merge_vad_matches_reference_function."""
    g = np.random.default_rng(0)
    return [np.sort(g.integers(0, 200000, size=2 * int(g.integers(1, 12)))).reshape(-1, 2).tolist() for _ in range(50)]


def vad_detector_cases():
    """The 60 seeded posterior tracks of test_detector_matches_the_reference_runtimes_compiled_cpp_detector."""
    rng = np.random.default_rng(7)
    return [mk.random_case(rng, 40.0 if it < 50 else 150.0) for it in range(60)]


# (seconds, seed, pattern) of three tests/golden/vad_*.npz cases — must match oracle/make_vad_golden.py:VAD_CASES
NAMED_VAD_CASES = {
    "vad_fixed800": (30.0, 3, [(2.0, 1.0), (3.0, 0.5), (1.0, 1.5)]),
    "vad_short": (1.2, 5, [(5.0, 0.1)]),
    "vad_silence": (3.0, 6, [(0.0, 9.0)]),
}

def timestamp_cases():
    """(peaks, alphas, chars) of the 50 seeded traces of test_timestamps_against_live_reference."""
    from funasr_b200 import timestamps as TS
    rng = np.random.default_rng(7)
    out = []
    for trial in range(50):
        T = int(rng.integers(6, 120))
        a = (rng.random(T).astype(np.float32) ** 2 * 0.8).astype(np.float32)
        peaks = TS.cif_wo_hidden(a, 1.0)
        chars = ["c%d" % i for i in range(max(1, int((peaks >= 1 - 1e-4).sum()) - 1 + trial % 2))]
        out.append((peaks, a, chars))
    return out


HOTWORD_SEG_DICT = "hello he@@ llo\n你 你\n好 好\n7 7\ngpu gpu\n"
HOTWORD_TXT = "hello 你好\ngpu\n"
HOTWORD_VOCAB = {"<unk>": 9, "he@@": 3, "llo": 4, "你": 5, "好": 6, "7": 7, "gpu": 8}


def encoder_inputs():
    """Features / lengths of test_oracle_matches_live_reference_components (weights: synth.make_state_dict(TINY, 11))."""
    g = torch.Generator().manual_seed(5)
    feats = torch.randn(3, 41, 560, generator=g)
    lens = torch.tensor([41, 17, 30], dtype=torch.int32)
    for b in range(3):
        feats[b, lens[b]:] = 0
    return feats, lens


def main():
    ref_shim.import_reference()
    assert knf_ref.build(), "needs the reference tree for oracle/_ref"
    from funasr.utils.vad_utils import merge_vad as ref_merge
    from funasr.models.contextual_paraformer.model import ContextualParaformer
    from funasr.register import tables
    from funasr.utils.timestamp_tools import ts_prediction_lfr6_standard
    from funasr_b200 import synth
    out = {"merge_vad": [ref_merge([list(x) for x in t], 15000) for t in merge_vad_cases()]}
    out["vad_detector"] = [knf_ref.vad_segments(sp, wav, mes, 60000, thr) for n, sp, wav, mes, thr in vad_detector_cases()]
    named = {}
    for name, (seconds, seed, pattern) in NAMED_VAD_CASES.items():     # the Python reference's scores through the C++ detector
        gg = np.load(os.path.join(GOLDEN, name + ".npz"))
        named[name] = knf_ref.vad_segments(gg["sil_prob"], synth.make_vad_wav(seconds, seed, pattern).numpy(), 800, 60000, 0.6)
    out["vad_detector_named"] = named

    class Tok:
        vocab = HOTWORD_VOCAB

        def tokens2ids(self, toks):
            return [self.vocab.get(t, self.vocab["<unk>"]) for t in toks]

    class Fe:
        cmvn_file = None

    class Dummy:
        sos = 1

    with tempfile.TemporaryDirectory() as td:
        open(os.path.join(td, "am.mvn"), "w").write("x")
        open(os.path.join(td, "seg_dict"), "w", encoding="utf8").write(HOTWORD_SEG_DICT)
        txt = os.path.join(td, "hw.txt")
        open(txt, "w", encoding="utf8").write(HOTWORD_TXT)
        fe = Fe()
        fe.cmvn_file = os.path.join(td, "am.mvn")
        out["hotwords"] = {"string": ContextualParaformer.generate_hotwords_list(Dummy(), "Hello 你好 GPU xyz", tokenizer=Tok(), frontend=fe),
                           "txt": ContextualParaformer.generate_hotwords_list(Dummy(), txt, tokenizer=Tok(), frontend=fe)}
    ts = []
    for peaks, a, chars in timestamp_cases():
        try:
            txt, res = ts_prediction_lfr6_standard(torch.tensor(peaks.copy()), torch.tensor(a.copy()), list(chars), upsample_rate=1)
        except IndexError:
            txt, res = "", []
        ts.append([txt, res])
    out["timestamps"] = ts
    with open(os.path.join(GOLDEN, "live_reference.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))

    cfg = synth.PARAFORMER_TINY
    p = synth.make_state_dict(cfg, 11)
    enc = tables.encoder_classes["SANMEncoder"](input_size=560, output_size=512, attention_heads=4, linear_units=2048,
                                                num_blocks=cfg.enc_layers, input_layer="pe", kernel_size=11, sanm_shfit=0,
                                                selfattention_layer_type="sanm").eval()
    enc.load_state_dict({k[len("encoder."):]: v for k, v in p.items() if k.startswith("encoder.")}, strict=True)
    pred = tables.predictor_classes["CifPredictorV2"](idim=512, threshold=1.0, l_order=1, r_order=1, tail_threshold=0.45).eval()
    pred.load_state_dict({k[len("predictor."):]: v for k, v in p.items() if k.startswith("predictor.")}, strict=True)
    feats, lens = encoder_inputs()
    with torch.no_grad():
        r_enc, r_len, _ = enc(feats, lens)
        mask = (torch.arange(41)[None, :] < lens[:, None])[:, None, :]
        r_emb, r_tok, r_al, r_pk = pred(r_enc, None, mask, ignore_id=-1)
    np.savez_compressed(os.path.join(GOLDEN, "live_reference_components.npz"), enc=r_enc.numpy(), enc_lens=r_len.numpy(),
                        token_num=r_tok.numpy(), alphas=r_al.numpy(), peaks=r_pk.numpy(), acoustic=r_emb.numpy())
    for fn in ("live_reference.json", "live_reference_components.npz"):
        print("wrote", fn, os.path.getsize(os.path.join(GOLDEN, fn)), "bytes")


if __name__ == "__main__":
    main()
