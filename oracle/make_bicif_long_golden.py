"""Generate tests/golden/longaudio_bicif_40s.npz by running the UNMODIFIED reference on CPU: AutoModel(model="BiCifParaformer",
vad_model=FsmnVADStreaming).generate() -> inference_with_vad, with per-token timestamps.  Writes only this fixture.
Run in the build container only:   python oracle/make_bicif_long_golden.py

The recording, the VAD model and its configuration are those of make_vad_golden.py's longaudio_40s case; the recogniser is the tiny
BiCifParaformer of synth.make_bicif_state_dict (the weights of make_golden.py's bicif_tiny_ragged3)."""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import ref_runner  # noqa: E402
import ref_shim  # noqa: E402
from funasr_b200 import synth  # noqa: E402
from make_vad_golden import GOLD, LONG_CASES, VAD_WEIGHT_SEED, vad_conf  # noqa: E402

# name: (seconds, wav seed, pattern, generate kwargs, BiCif weight seed) — the recording of longaudio_40s, in 6 s packs
BICIF_LONG_CASES = {
    "longaudio_bicif_40s": LONG_CASES["longaudio_40s"][:3] + ({"batch_size_s": 6}, 8),
}
CJK0 = 0x4E00


def cjk_token_list(cfg):
    """The tN vocabulary with one CJK character per token: BiCifParaformer.inference passes its stamps through
    sentence_postprocess, which keeps one stamp per token for an all-CJK token list and none for "t12"-style tokens."""
    return ["<blank>", "<s>", "</s>"] + [chr(CJK0 + i) for i in range(cfg.vocab - 4)] + ["<unk>"]


def run_bicif_long_case(name, seconds, seed, pattern, gen_kw, wseed, tmp):
    from funasr import AutoModel
    cfg = synth.PARAFORMER_TINY
    asr_cmvn = os.path.join(tmp, "bicif.mvn")
    ref_runner.write_cmvn_file(asr_cmvn, synth.make_cmvn(cfg, 1))
    vad_cmvn = os.path.join(tmp, "vad.mvn")
    ref_runner.write_cmvn_file(vad_cmvn, synth.make_vad_cmvn(0))
    pt = os.path.join(tmp, "bicif.pt")
    torch.save(synth.make_bicif_state_dict(cfg, wseed), pt)
    vpt = os.path.join(tmp, "vad.pt")
    torch.save(synth.make_vad_state_dict(synth.VAD_DEFAULT, VAD_WEIGHT_SEED), vpt)
    vc = vad_conf(vad_cmvn)
    am = AutoModel(model="BiCifParaformer",
                   model_conf=dict(ctc_weight=0.0, lsm_weight=0.1, length_normalized_loss=True, predictor_weight=1.0, predictor_bias=1, sampling_ratio=0.75),
                   encoder="SANMEncoder", encoder_conf=ref_runner._enc_conf(cfg), decoder="ParaformerSANMDecoder", decoder_conf=ref_runner._dec_conf(cfg),
                   predictor="CifPredictorV3",
                   predictor_conf=dict(idim=cfg.d_model, threshold=1.0, l_order=1, r_order=1, tail_threshold=cfg.tail_threshold, smooth_factor2=0.25,
                                       noise_threshold2=0.01, upsample_times=3, use_cif1_cnn=False, upsample_type="cnn_blstm"),
                   frontend="WavFrontend", frontend_conf=ref_runner._frontend_conf(asr_cmvn), tokenizer="CharTokenizer",
                   tokenizer_conf=dict(token_list=cjk_token_list(cfg), unk_symbol="<unk>", split_with_space=True),
                   init_param=pt, vad_model=vc["model"],
                   vad_kwargs=dict(model_conf=vc["model_conf"], encoder=vc["encoder"], encoder_conf=vc["encoder_conf"], frontend=vc["frontend"],
                                   frontend_conf=vc["frontend_conf"], init_param=vpt),
                   device="cpu", ncpu=os.cpu_count(), disable_update=True, disable_pbar=True)
    wav = synth.make_vad_wav(seconds, seed, pattern)
    # a torch.device, not the string "cpu": the reference's dynamic batching over the duration-sorted segments runs (auto_model.py:929-930)
    res = am.generate(input=wav.numpy(), disable_pbar=True, device=torch.device("cpu"), **gen_kw)
    r = res[0]
    text = r.get("text", "")
    ids = [ord(ch) - CJK0 + 3 for ch in text if ch != " "]
    ts = r.get("timestamp", [])
    assert all(0 <= i - 3 < cfg.vocab - 4 for i in ids), text
    assert len(ts) == len(ids) and ids, (len(ts), len(ids))          # one stamp per id
    np.savez_compressed(os.path.join(GOLD, name + ".npz"), ids=np.array(ids, dtype=np.int64), timestamp=np.array(ts, dtype=np.int64).reshape(-1, 2),
                        n_samples=np.int64(wav.numel()), text=np.array(text))
    print("%s: %d ids, %d stamps, first stamps %s" % (name, len(ids), len(ts), ts[:4]))


def main():
    ref_shim.import_reference()
    os.makedirs(GOLD, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        for name, (seconds, seed, pattern, kw, wseed) in BICIF_LONG_CASES.items():
            run_bicif_long_case(name, seconds, seed, pattern, kw, wseed, tmp)


if __name__ == "__main__":
    main()
