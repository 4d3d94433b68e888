"""Long-audio recognition through the C handle API (fa_offline_infer_vad) against LongAudioPipeline on the same recording.
Usage: offline_vad_probe.py [--seconds 600] [--reps 5] [--mode fp16x3] [--batch-size-s 300] [--out DIR]

One synthetic recording (synth.make_vad_wav: speech-like bursts and pauses), PARAFORMER_LARGE synthetic weights, the synthetic FSMN-VAD.
After a warm-up of both, the two paths run alternately --reps times; each time is a host clock around work that ends in a device
synchronise.  Per path: VAD alone (fa_vad_infer / the VAD plugin's inference), the whole call, decode = whole - VAD, and the host CPU
time of the whole call (process time), as medians; audio-s/s = recording seconds / whole-call median.  Also checks that both paths give
the same ids and segments, and prints the card and its power limit read in the same call.  --out DIR writes the JSON there."""
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
    w0, c0 = time.perf_counter(), time.process_time()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - w0, time.process_time() - c0


def paraformer_conf(cfg, mode):
    return dict(
        encoder="SANMEncoderB200",
        encoder_conf=dict(output_size=512, attention_heads=4, linear_units=2048, num_blocks=cfg.enc_layers, dropout_rate=0.1, input_layer="pe",
                          pos_enc_class="SinusoidalPositionEncoder", normalize_before=True, kernel_size=11, sanm_shfit=0, selfattention_layer_type="sanm"),
        decoder="ParaformerSANMDecoderB200",
        decoder_conf=dict(attention_heads=4, linear_units=2048, num_blocks=cfg.dec_layers, att_layer_num=cfg.dec_layers, kernel_size=11, sanm_shfit=0),
        predictor="CifPredictorV2B200",
        predictor_conf=dict(idim=512, threshold=1.0, l_order=1, r_order=1, tail_threshold=0.45),
        input_size=560, vocab_size=cfg.vocab, gemm_mode=mode)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=600.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--mode", default="fp16x3")
    ap.add_argument("--batch-size-s", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("offline_vad_probe: no CUDA device (this measurement has no CPU path)")
    import funasr_b200
    from funasr_b200 import pack, synth
    from funasr_b200.offline import OfflineRecognizer, OfflineVad
    info = card()
    cfg = synth.PARAFORMER_LARGE
    state = synth.make_state_dict(cfg, 0)
    cmvn = synth.make_cmvn(cfg, 1)
    vc = synth.VAD_DEFAULT
    vstate, vcmvn = synth.make_vad_state_dict(vc, 0), synth.make_vad_cmvn(0)
    td = tempfile.mkdtemp()
    asr_path, vad_path = os.path.join(td, "model.fab2"), os.path.join(td, "vad.fab2")
    pack.write_model_file(asr_path, state, cfg, cmvn)
    pack.write_vad_model_file(vad_path, vstate, vcmvn, {})
    wav = synth.make_vad_wav(a.seconds, 12).numpy()
    seconds = wav.size / 16000.0

    rec, vad = OfflineRecognizer(asr_path, 0, a.mode), OfflineVad(vad_path, 0)
    asr = funasr_b200.ParaformerB200(**paraformer_conf(cfg, a.mode))
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

    def handle_vad():
        return vad.segments(wav)

    def handle_all():
        return rec.infer_long([wav], vad, batch_size_s=a.batch_size_s)[0]

    def pipe_vad():
        return pv.inference(torch.from_numpy(wav).to(DEV), key=["rec"], frontend=vad_fe, device=DEV)[0][0]["value"]

    def pipe_all():
        return pipe.generate(wav, key="rec", batch_size_s=a.batch_size_s)

    for fn in (handle_vad, handle_all, pipe_vad, pipe_all):                 # warm-up: every shape of the timed window
        clock(fn)
    t = {k: [] for k in ("handle_vad", "handle_total", "handle_host", "pipe_vad", "pipe_total", "pipe_host")}
    same = True
    for _ in range(a.reps):
        _, dv, _ = clock(handle_vad)
        h, dt, hc = clock(handle_all)
        t["handle_vad"].append(dv); t["handle_total"].append(dt); t["handle_host"].append(hc)
        _, dv, _ = clock(pipe_vad)
        p, dt, pc = clock(pipe_all)
        t["pipe_vad"].append(dv); t["pipe_total"].append(dt); t["pipe_host"].append(pc)
        same = same and h["token_int"] == p.get("token_int", []) and h["vad_segments"] == p["vad_segments"]
    med = {k: statistics.median(v) for k, v in t.items()}
    spread = {k: (max(v) - min(v)) / statistics.median(v) for k, v in t.items() if k.endswith("total")}
    res = {"card": info, "mode": a.mode, "audio_seconds": seconds, "segments": len(h["vad_segments"]), "tokens": len(h["token_int"]),
           "identical_outputs": same, "reps": a.reps}
    for side in ("handle", "pipe"):
        res[side] = {"vad_ms": 1e3 * med[side + "_vad"], "decode_ms": 1e3 * (med[side + "_total"] - med[side + "_vad"]),
                     "total_ms": 1e3 * med[side + "_total"], "host_cpu_ms": 1e3 * med[side + "_host"],
                     "audio_s_per_s": seconds / med[side + "_total"], "total_spread": spread[side + "_total"]}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "offline_vad_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
