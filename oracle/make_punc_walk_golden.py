"""Writes tests/golden/punc_walk_cases.npz: the unmodified reference's CTTransformer.inference (ct_transformer/model.py:290-473) on
long texts, with its `punc_forward` replaced by a scripted scorer -- punctuation as a fixed function of (token id, position in the
window), tests/punc_scripted.py:scripted -- so the mini-sentence walk reaches branches that seeded weights do not: the comma cut past
200 words with its relabelling to sentence_end_id, windows with neither comma nor sentence end (carried whole), English-only text and
final windows ending in ，, 、, "," or a Latin word.  Each case stores its text, the scorer's seed and class probabilities, and the
reference's text and punc_array.  tests/test_offline_punc_host.py runs fa_punc_walk_host against it.
Run where the reference tree is present:  python oracle/make_punc_walk_golden.py"""
import os
import random
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [ROOT, HERE, os.path.join(ROOT, "tests")]
import ref_shim  # noqa: E402
from funasr_b200 import synth  # noqa: E402
from punc_scripted import random_text, scripted  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "punc_walk_cases.npz")
ENGLISH = " ".join(synth.punc_token_list()[synth.PUNC_VOCAB - 17:-1])


def cases():
    """(name, text, seed, probabilities of <unk>, ，, 。, ？, 、)"""
    rng = random.Random(4242)
    return [
        ("rare_ends_with_commas", random_text(rng, 900), 2, (0.0, 0.08, 0.002, 0.0, 0.02)),
        ("no_comma_no_end", random_text(rng, 400), 3, (0.0, 0.0, 0.0, 0.0, 0.0)),
        ("dun_only_long", random_text(rng, 500), 5, (0.0, 0.0, 0.01, 0.0, 0.3)),
        ("every_class", random_text(rng, 300), 4, (0.01, 0.2, 0.15, 0.1, 0.1)),
        ("english_only", " ".join([ENGLISH] * 6), 1, (0.0, 0.1, 0.05, 0.02, 0.0)),
        ("ends_in_comma_cjk", "你好" * 23, 9, (0.0, 1.0, 0.0, 0.0, 0.0)),
        ("ends_in_dun", "世界" * 17, 9, (0.0, 0.0, 0.0, 0.0, 1.0)),
        ("ends_in_comma_latin", ENGLISH + " " + ENGLISH, 9, (0.0, 1.0, 0.0, 0.0, 0.0)),
        ("ends_in_latin_word", "你 " + ENGLISH * 2, 9, (0.0, 0.0, 0.0, 0.0, 0.0)),
    ]


def main():
    ref_shim.import_reference()
    from funasr import AutoModel
    toks = synth.punc_token_list()
    with tempfile.TemporaryDirectory() as tmp:
        pt = os.path.join(tmp, "punc.pt")
        torch.save(synth.make_punc_state_dict(0), pt)
        am = AutoModel(model="CTTransformer",
                       model_conf=dict(ignore_id=0, embed_unit=synth.PUNC_DIM, att_unit=synth.PUNC_DIM, dropout_rate=0.1, punc_list=synth.PUNC_LIST,
                                       punc_weight=[1.0] * len(synth.PUNC_LIST), sentence_end_id=3),
                       encoder="SANMEncoder",
                       encoder_conf=dict(input_size=synth.PUNC_DIM, output_size=synth.PUNC_DIM, attention_heads=synth.PUNC_HEADS,
                                         linear_units=synth.PUNC_FFN, num_blocks=synth.PUNC_LAYERS, dropout_rate=0.1, positional_dropout_rate=0.1,
                                         attention_dropout_rate=0.0, input_layer="pe", pos_enc_class="SinusoidalPositionEncoder",
                                         normalize_before=True, kernel_size=11, sanm_shfit=0, selfattention_layer_type="sanm", padding_idx=0),
                       tokenizer="CharTokenizer", tokenizer_conf=dict(token_list=toks, unk_symbol="<unk>"),
                       device="cpu", ncpu=os.cpu_count(), disable_update=True, disable_pbar=True, init_param=pt)
        out = {}
        for i, (name, text, seed, probs) in enumerate(cases()):
            def punc_forward(text, text_lengths, _seed=seed, _probs=probs):     # model.py:112-125's (logits, lengths), one-hot
                ids = scripted(text.cpu().numpy().astype(np.int64), _seed, _probs)
                return torch.nn.functional.one_hot(torch.from_numpy(ids.astype(np.int64)), len(synth.PUNC_LIST)).float(), text_lengths
            am.model.punc_forward = punc_forward
            r = am.generate(input=text, disable_pbar=True)[0]
            arr = np.asarray(r["punc_array"]).astype(np.int64)
            out["name_%d" % i] = np.array(name)
            out["text_in_%d" % i] = np.array(text)
            out["seed_%d" % i] = np.array(seed)
            out["probs_%d" % i] = np.array(probs, np.float64)
            out["text_out_%d" % i] = np.array(r["text"])
            out["punc_array_%d" % i] = arr
            print("%s: %d ids -> %r  punc %s" % (name, arr.size, r["text"][-40:], np.bincount(arr, minlength=6).tolist()))
        out["n"] = np.array(len(cases()))
        np.savez_compressed(GOLDEN, **out)
    print("wrote", GOLDEN)


if __name__ == "__main__":
    main()
