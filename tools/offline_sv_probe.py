"""SenseVoiceSmall through the C handle API against the Python path, SENSEVOICE_SMALL synthetic weights.
Usage: offline_sv_probe.py [--batch 64] [--utt-seconds 30] [--long-seconds 600] [--reps 5] [--mode fp16x3] [--out DIR]

Two measurements, each with host waveforms in and ids out, after a warm-up of both sides, the two sides run alternately --reps times
(a host clock around work that ends in a device synchronise), medians reported:
  batch: fa_offline_infer_sv on --batch utterances of --utt-seconds against SenseVoiceEngine.forward_wav (waveforms copied to the
         device and padded by torch, ids copied back);
  long:  fa_offline_infer_vad_sv on one --long-seconds recording against LongAudioPipeline with SenseVoiceSmallB200.
Both sides must give identical ids.  Prints the card and its power limit read in the same call; --out DIR writes the JSON there."""
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

DEV = "cuda:0"


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def alternate(a, b, reps):
    ta, tb, oa, ob = [], [], None, None
    for _ in range(reps):
        oa, t = clock(a)
        ta.append(t)
        ob, t = clock(b)
        tb.append(t)
    return oa, ob, statistics.median(ta), statistics.median(tb)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--utt-seconds", type=float, default=30.0)
    ap.add_argument("--long-seconds", type=float, default=600.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--mode", default="fp16x3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("offline_sv_probe: no CUDA device (this measurement has no CPU path)")
    import funasr_b200
    from funasr_b200 import pack, synth
    from funasr_b200.engine import SenseVoiceEngine
    from funasr_b200.offline import OfflineRecognizer, OfflineVad
    info = card()
    cfg = synth.SENSEVOICE_SMALL
    state = synth.make_sensevoice_state_dict(cfg, 1)
    cmvn = synth.make_cmvn(synth.PARAFORMER_LARGE, 1)
    vc = synth.VAD_DEFAULT
    vstate, vcmvn = synth.make_vad_state_dict(vc, 0), synth.make_vad_cmvn(0)
    td = tempfile.mkdtemp()
    asr_path, vad_path = os.path.join(td, "model.fab2"), os.path.join(td, "vad.fab2")
    pack.write_sensevoice_model_file(asr_path, state, cfg, cmvn)
    pack.write_vad_model_file(vad_path, vstate, vcmvn, {})
    rec, vad = OfflineRecognizer(asr_path, 0, a.mode), OfflineVad(vad_path, 0)
    out = {"card": info, "mode": a.mode, "reps": a.reps}

    # ---- batch: 64 x 30 s
    n = int(a.utt_seconds * 16000)
    wavs = [synth.make_wav(n - 160 * i, 100 + i).numpy().astype(np.float32) for i in range(a.batch)]
    eng = SenseVoiceEngine(state, cfg, DEV, gemm_mode=a.mode, cmvn=cmvn)

    def handle_batch():
        return rec.infer(wavs, language="zh", use_itn=True)

    def engine_batch():
        lens = [w.size for w in wavs]
        pad = torch.nn.utils.rnn.pad_sequence([torch.from_numpy(w) for w in wavs], batch_first=True).to(DEV)
        return eng.forward_wav(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), lens, language_id=3, textnorm_id=14)["ids"]

    handle_batch(), engine_batch()
    h_ids, e_ids, th, te = alternate(handle_batch, engine_batch, a.reps)
    assert h_ids == e_ids, "batch: the handle and the engine disagree"
    audio = sum(w.size for w in wavs) / 16000.0
    out["batch"] = {"utterances": a.batch, "audio_s": audio, "handle_s": th, "engine_s": te, "handle_audio_s_per_s": audio / th,
                    "engine_audio_s_per_s": audio / te}
    del eng
    torch.cuda.empty_cache()

    # ---- long: one recording through VAD
    wav = synth.make_vad_wav(a.long_seconds, 12).numpy()
    asr = funasr_b200.SenseVoiceSmallB200(encoder="SenseVoiceEncoderSmallB200",
                                          encoder_conf=dict(output_size=512, attention_heads=4, linear_units=2048, num_blocks=cfg.enc_layers,
                                                            tp_blocks=cfg.tp_layers, input_layer="pe", kernel_size=11, sanm_shfit=0,
                                                            selfattention_layer_type="sanm"), input_size=560, vocab_size=cfg.vocab, gemm_mode=a.mode)
    asr.load_state_dict(state, strict=True)
    asr.to(DEV).eval()
    asr_fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0, cmvn=cmvn)
    pv = funasr_b200.FsmnVADStreamingB200(encoder="FSMN", encoder_conf=dict(
        input_dim=vc.input_dim, input_affine_dim=vc.input_affine_dim, fsmn_layers=vc.fsmn_layers, linear_dim=vc.linear_dim, proj_dim=vc.proj_dim,
        lorder=vc.lorder, rorder=0, lstride=1, rstride=0, output_affine_dim=vc.output_affine_dim, output_dim=vc.output_dim))
    pv.load_state_dict(vstate, strict=True)
    pv.to(DEV).eval()
    vad_fe = funasr_b200.WavFrontendOnlineB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=5, lfr_n=1, dither=0.0,
                                               cmvn=vcmvn)
    pipe = funasr_b200.LongAudioPipeline(asr, asr_fe, pv, vad_fe, device=DEV)

    def handle_long():
        return rec.infer_long([wav], vad, language="zh", use_itn=True)[0]["token_int"]

    def pipeline_long():
        return pipe.generate(wav, key="rec", language="zh", use_itn=True)["token_int"]

    handle_long(), pipeline_long()
    h_ids, p_ids, th, tp = alternate(handle_long, pipeline_long, a.reps)
    assert h_ids == p_ids, "long: the handle and the pipeline disagree"
    out["long"] = {"audio_s": wav.size / 16000.0, "ids": len(h_ids), "handle_s": th, "pipeline_s": tp,
                   "handle_audio_s_per_s": wav.size / 16000.0 / th, "pipeline_audio_s_per_s": wav.size / 16000.0 / tp}
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "offline_sv_probe.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
