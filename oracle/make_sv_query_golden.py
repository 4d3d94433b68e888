"""Generate the SenseVoiceSmall query and long-audio goldens by running the UNMODIFIED reference on CPU (build container only):

    python oracle/make_sv_query_golden.py

- sv_tiny_en_itn / sv_tiny_yue_woitn: SenseVoiceSmall.inference on the sv_tiny_ragged3 waveforms and weights with language="en",
  use_itn=True and language="yue", use_itn=False (the sv_* goldens of make_golden.py cover only "auto" without ITN).  Stored: the ids
  and enc_lens.
- longaudio_sv_40s: AutoModel(model="SenseVoiceSmall", vad_model=FsmnVADStreaming).generate(language="zh", use_itn=True, batch_size_s=6)
  on the longaudio_40s recording with tiny SenseVoice weights of seed 6: every decoded frame's top-2 log-prob margin is >= 1.2e-3 there
  (with the sv_tiny_ragged3 weights, seed 4, one frame of the first segment has a margin of 8.6e-6, which a reordered fp32 sum flips).  Stored: the VAD segments (recorded by wrapping the AutoModel
  instance's bound `inference` method; the reference's code is untouched) and the ids of all segments in time order, read back from
  the joined text: the token list names id k "t{k-1}" (and the last id "<unk>"), so the CharTokenizer's decoded pieces spell the ids,
  and inference_with_vad joins segment texts with " " (auto_model.py:1028-1032)."""
import os
import re
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_golden  # noqa: E402
import make_vad_golden  # noqa: E402
import ref_runner  # noqa: E402
import ref_shim  # noqa: E402
from funasr_b200 import synth  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")

# name: (language, use_itn) on the sv_tiny_ragged3 waveforms and weights
QUERY_CASES = {"sv_tiny_en_itn": ("en", True), "sv_tiny_yue_woitn": ("yue", False)}
# name: (seconds, wav seed, pattern, generate kwargs): the longaudio_40s recording; LONG_SV_WEIGHT_SEED: its SENSEVOICE_TINY weights
LONG_SV_CASES = {"longaudio_sv_40s": (40.0, 7, [(3.0, 2.5), (1.5, 2.2), (4.0, 3.0), (2.0, 2.2), (6.0, 2.4)],
                                      {"batch_size_s": 6, "language": "zh", "use_itn": True})}
LONG_SV_WEIGHT_SEED = 6


class IdTokenizer:
    """SenseVoiceSmall.inference needs tokenizer.decode(token_int) (model.py:1027); record the ids verbatim."""

    def decode(self, ids):
        return " ".join(str(int(i)) for i in ids)


def sv_kwargs(cfg, wseed, tmp):
    cmvn_file = os.path.join(tmp, "am_sv.mvn")
    make_golden.write_cmvn_file(cmvn_file, synth.make_cmvn(synth.PARAFORMER_LARGE, seed=1))
    pt = os.path.join(tmp, "sv_%d.pt" % wseed)
    torch.save(synth.make_sensevoice_state_dict(cfg, wseed), pt)
    tokens = ["<blank>"] + ["t%d" % i for i in range(cfg.vocab - 2)] + ["<unk>"]
    return dict(
        model="SenseVoiceSmall", model_conf=dict(length_normalized_loss=True, sos=1, eos=2, ignore_id=-1),
        encoder="SenseVoiceEncoderSmall",
        encoder_conf=dict(output_size=cfg.d_model, attention_heads=cfg.heads, linear_units=cfg.ffn, num_blocks=cfg.enc_layers,
                          tp_blocks=cfg.tp_layers, dropout_rate=0.1, positional_dropout_rate=0.1, attention_dropout_rate=0.1,
                          input_layer="pe", pos_enc_class="SinusoidalPositionEncoder", normalize_before=True, kernel_size=cfg.kernel,
                          sanm_shfit=0, selfattention_layer_type="sanm"),
        frontend="WavFrontend",
        frontend_conf=dict(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0,
                           cmvn_file=cmvn_file),
        tokenizer="CharTokenizer", tokenizer_conf=dict(token_list=tokens, unk_symbol="<unk>", split_with_space=True),
        device="cpu", ncpu=os.cpu_count(), disable_update=True, disable_pbar=True, init_param=pt)


def run_query_cases(tmp):
    from funasr import AutoModel
    cfg, wseed, specs, _ = make_golden.SV_CASES["sv_tiny_ragged3"]
    am = AutoModel(**sv_kwargs(cfg, wseed, tmp))
    model, frontend = am.model, am.kwargs["frontend"]
    wavs = [synth.make_wav(n, s, k) for (n, s, k) in specs]
    for name, (language, use_itn) in QUERY_CASES.items():
        with torch.no_grad():
            res, _ = model.inference(data_in=[w.numpy() for w in wavs], key=["u%d" % i for i in range(len(wavs))], tokenizer=IdTokenizer(),
                                     frontend=frontend, device="cpu", language=language, use_itn=use_itn)
            from funasr.utils.load_utils import extract_fbank
            _, flens = extract_fbank([w for w in wavs], frontend=frontend)
        ids = [[int(t) for t in r["text"].split()] for r in res]
        np.savez_compressed(os.path.join(GOLD, name + ".npz"), enc_lens=(flens + 4).numpy().astype(np.int32),
                            ids_flat=np.array([t for r in ids for t in r], dtype=np.int32), ids_len=np.array([len(r) for r in ids], dtype=np.int32))
        print("%s: ctc tokens %s, ids[0][:8] %s" % (name, [len(r) for r in ids], ids[0][:8]))


def run_long_sv_case(name, seconds, seed, pattern, gen_kw, tmp):
    from funasr import AutoModel
    cfg, wseed = synth.SENSEVOICE_TINY, LONG_SV_WEIGHT_SEED
    vad_cmvn = os.path.join(tmp, "vad_sv.mvn")
    ref_runner.write_cmvn_file(vad_cmvn, synth.make_vad_cmvn(0))
    vpt = os.path.join(tmp, "vad_sv.pt")
    torch.save(synth.make_vad_state_dict(synth.VAD_DEFAULT, make_vad_golden.VAD_WEIGHT_SEED), vpt)
    vc = make_vad_golden.vad_conf(vad_cmvn)
    kw = sv_kwargs(cfg, wseed, tmp)
    am = AutoModel(**kw, vad_model=vc["model"],
                   vad_kwargs=dict(model_conf=vc["model_conf"], encoder=vc["encoder"], encoder_conf=vc["encoder_conf"], frontend=vc["frontend"],
                                   frontend_conf=vc["frontend_conf"], init_param=vpt))
    segs = []
    infer = am.inference

    def recorded(*a, **k):
        r = infer(*a, **k)
        if k.get("model") is am.vad_model:
            segs.extend([list(map(int, s)) for s in r[0]["value"]])
        return r

    am.inference = recorded
    wav = synth.make_vad_wav(seconds, seed, pattern)
    # a torch.device (not the string "cpu") keeps the reference's batching over the duration-sorted segments (auto_model.py:929-930)
    res = am.generate(input=wav.numpy(), disable_pbar=True, device=torch.device("cpu"), **gen_kw)
    ids = [int(t) + 1 if t else cfg.vocab - 1 for t, _ in re.findall(r"t(\d+)|(<unk>)", res[0]["text"])]
    np.savez_compressed(os.path.join(GOLD, name + ".npz"), segments=np.array(segs, dtype=np.int64).reshape(-1, 2), ids=np.array(ids, dtype=np.int64),
                        n_samples=np.int64(wav.numel()))
    print("%s: %d segments %s, %d ids %s" % (name, len(segs), segs, len(ids), ids[:12]))


def main():
    ref_shim.import_reference()
    with tempfile.TemporaryDirectory() as tmp:
        run_query_cases(tmp)
        for name, (seconds, seed, pattern, kw) in LONG_SV_CASES.items():
            run_long_sv_case(name, seconds, seed, pattern, kw, tmp)


if __name__ == "__main__":
    main()
