"""Generate tests/golden/spk_*.npz by running the UNMODIFIED reference's speaker path on the CPU.  Build container only:
    python oracle/make_spk_golden.py

1. Calibration: the synthetic CAM++ weights (synth.make_campplus_state_dict) get BatchNorm running statistics from ONE train-mode
   forward (momentum=None) of the reference CAMPPlus over the 1.5 s chunks (sv_chunk) of the two-voice recording's speech bursts.
   With identity statistics random-weight embeddings of different voices collapse into one speaker; calibrated, they separate.  The
   statistics are stored (spk_campplus_bn.npz); tests rebuild the weights from the seed and overlay them.
2. Pipelines: AutoModel(model=Paraformer, vad_model=FsmnVADStreaming, spk_model=CAMPPlus).generate() (inference_with_vad with the
   spk branch, vad_segment mode since there is no punctuation model).  The chunk waveforms the speaker model saw, its embeddings and the
   ClusterBackend's labels are recorded by wrapping bound methods of the model INSTANCES; sentence_info comes from generate().
3. Host routines: stored embedding matrices through the reference ClusterBackend (incl. >= 2048 rows with preset_spk_num and
   merge_by_cos merges) and randomised postprocess / distribute_spk cases.
np.random is seeded before every call that clusters: the reference's k_means draws from the global RNG."""
import json
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

GOLD = os.path.join(ROOT, "tests", "golden")
SPK_SEED = 0
CALIB_PATTERN = [(v, 3.0, 2.5) for v in (0, 1) * 4]       # the two-voice case's layout (~45 s)

# name: (pattern [(voice, speech_s, silence_s)], wav seed, generate kwargs)
SPK_CASES = {
    "spk_two_voices": (CALIB_PATTERN, 1, {}),
    "spk_three_preset": ([(v, 3.0, 2.5) for v in (0, 1, 2) * 3], 2, {"preset_spk_num": 3, "return_spk_center": True}),
    "spk_few_chunks": ([(0, 3.0, 2.5), (1, 3.0, 2.5)], 3, {}),
    "spk_short_segment": ([(0, 3.0, 2.5), (1, 1.0, 2.5), (0, 3.0, 2.5), (1, 3.0, 2.5)] * 2, 4, {}),
}
CAMPPLUS_CONF = dict(feat_dim=80, embedding_size=192, growth_rate=32, bn_size=4, init_channels=128, config_str="batchnorm-relu",
                     memory_efficient=True, output_level="segment")


def ground_truth_segments(pattern, lead_s=0.5):
    out, pos = [], lead_s
    for _, sp, sl in pattern:
        out.append((pos, pos + sp))
        pos += sp + sl
    return out


def calibrate(chunk_waves, voice):
    """BatchNorm running statistics of one train-mode forward (momentum=None) over chunk_waves; voice: ground-truth voice per chunk."""
    from funasr.models.campplus.model import CAMPPlus
    from funasr.models.campplus.utils import extract_feature
    feats, _, _ = extract_feature([torch.from_numpy(c) for c in chunk_waves])
    m = CAMPPlus(**CAMPPLUS_CONF)
    m.load_state_dict(synth.make_campplus_state_dict(SPK_SEED), strict=True)
    for mod in m.modules():
        if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
            mod.momentum = None
            mod.reset_running_stats()
    m.train()
    with torch.no_grad():
        m(feats)
    m.eval()
    stats = {k: v.clone() for k, v in m.state_dict().items() if k.endswith("running_mean") or k.endswith("running_var")}
    with torch.no_grad():
        e = torch.nn.functional.normalize(m(feats), dim=1)
    cos = (e @ e.T).numpy()
    same = voice[:, None] == voice[None, :]
    print("calibration: %d chunks, cosine within %.3f / between %.3f" % (len(chunk_waves), cos[same & ~np.eye(len(voice), dtype=bool)].mean(),
                                                                         cos[~same].mean()))
    np.savez_compressed(os.path.join(GOLD, "spk_campplus_bn.npz"), **{k: v.numpy() for k, v in stats.items()})
    return stats


def voice_at(pattern, t, lead_s=0.5):
    """Voice of the burst nearest to time t (s)."""
    best, pos, v_best = None, lead_s, 0
    for v, sp, sl in pattern:
        d = 0.0 if pos <= t <= pos + sp else min(abs(t - pos), abs(t - pos - sp))
        if best is None or d < best:
            best, v_best = d, v
        pos += sp + sl
    return v_best


def build_pipeline(tmp, stats):
    from funasr import AutoModel
    from make_vad_golden import VAD_WEIGHT_SEED, vad_conf
    cfg = synth.PARAFORMER_TINY
    asr_cmvn = os.path.join(tmp, "asr.mvn")
    ref_runner.write_cmvn_file(asr_cmvn, synth.make_cmvn(cfg, 1))
    vad_cmvn = os.path.join(tmp, "vad.mvn")
    ref_runner.write_cmvn_file(vad_cmvn, synth.make_vad_cmvn(0))
    pt, vpt, spt = (os.path.join(tmp, n) for n in ("asr.pt", "vad.pt", "spk.pt"))
    torch.save(synth.make_state_dict(cfg, 3), pt)
    torch.save(synth.make_vad_state_dict(synth.VAD_DEFAULT, VAD_WEIGHT_SEED), vpt)
    torch.save(synth.make_campplus_state_dict(SPK_SEED, stats), spt)
    vc = vad_conf(vad_cmvn)
    return AutoModel(model="Paraformer",
                     model_conf=dict(ctc_weight=0.0, lsm_weight=0.1, length_normalized_loss=True, predictor_weight=1.0, predictor_bias=1,
                                     sampling_ratio=0.75),
                     encoder="SANMEncoder", encoder_conf=ref_runner._enc_conf(cfg), decoder="ParaformerSANMDecoder",
                     decoder_conf=ref_runner._dec_conf(cfg),
                     predictor="CifPredictorV2", predictor_conf=dict(idim=cfg.d_model, threshold=1.0, l_order=1, r_order=1,
                                                                     tail_threshold=cfg.tail_threshold),
                     frontend="WavFrontend", frontend_conf=ref_runner._frontend_conf(asr_cmvn), tokenizer="CharTokenizer",
                     tokenizer_conf=dict(token_list=ref_runner.token_list(cfg), unk_symbol="<unk>", split_with_space=True),
                     init_param=pt, vad_model=vc["model"],
                     vad_kwargs=dict(model_conf=vc["model_conf"], encoder=vc["encoder"], encoder_conf=vc["encoder_conf"],
                                     frontend=vc["frontend"], frontend_conf=vc["frontend_conf"], init_param=vpt),
                     spk_model="CAMPPlus", spk_kwargs=dict(model_conf=CAMPPLUS_CONF, init_param=spt), spk_mode="vad_segment",
                     device="cpu", ncpu=os.cpu_count(), disable_update=True, disable_pbar=True)


def run_case(am, name, pattern, seed, kw, save=True):
    from funasr.models.campplus.utils import extract_feature
    wav = synth.make_voice_wav(pattern, seed)
    rec = {"chunks": [], "emb": [], "labels": None, "cb_in": None, "times": []}
    spk_inf = am.spk_model.inference
    cb_fwd = am.cb_model.forward

    def spk_wrapped(data_in, *a, **k):
        res, meta = spk_inf(data_in, *a, **k)
        rec["chunks"].extend(np.asarray(x) for x in data_in)
        rec["emb"].append(res[0]["spk_embedding"].detach().clone())
        return res, meta

    def cb_wrapped(X, **params):
        labels = cb_fwd(X, **params)
        rec["labels"] = np.array(labels)
        rec["cb_in"] = X.detach().clone().numpy()
        return labels

    sv_chunk_mod = sys.modules["funasr.auto.auto_model"]
    sv_chunk_fn = sv_chunk_mod.sv_chunk

    def sv_chunk_wrapped(vad_segments, *a, **k):
        segs = sv_chunk_fn(vad_segments, *a, **k)
        rec["times"].extend((c[0], c[1]) for c in segs)
        return segs

    am.spk_model.inference = spk_wrapped
    am.cb_model.forward = cb_wrapped
    sv_chunk_mod.sv_chunk = sv_chunk_wrapped
    np.random.seed(0)
    try:
        res = am.generate(input=wav.numpy(), disable_pbar=True, device=torch.device("cpu"), pred_timestamp=True, **kw)
    finally:
        am.spk_model.inference = spk_inf
        am.cb_model.forward = cb_fwd
        sv_chunk_mod.sv_chunk = sv_chunk_fn
    if save is False:
        return rec
    r = res[0]
    info = r["sentence_info"]
    order = np.argsort([a for a, _ in rec["times"]], kind="stable")            # time order, like all_segments and the embeddings
    chunks = [rec["chunks"][i] for i in order]
    feats, _, _ = extract_feature([torch.from_numpy(c) for c in chunks[:4]])
    out = dict(n_samples=np.int64(wav.numel()), segments=np.array([[s["start"], s["end"]] for s in info], dtype=np.int64),
               chunk_times=np.array([rec["times"][i] for i in order], dtype=np.float64),
               chunk_waves_sum=np.array([float(np.sum(c, dtype=np.float64)) for c in chunks]),
               features=feats.numpy(), cb_in=rec["cb_in"], labels=rec["labels"].astype(np.int64),
               sentence_info=np.array(json.dumps([{k: (v if k != "timestamp" else [list(map(int, t)) for t in v]) for k, v in s.items()}
                                                  for s in info])),
               kwargs=np.array(json.dumps(kw)))
    if "spk_embedding_center" in r:
        out["spk_embedding_center"] = np.asarray(r["spk_embedding_center"], dtype=np.float32)
    np.savez_compressed(os.path.join(GOLD, name + ".npz"), **out)
    print("%s: %.1f s, %d segments, %d chunks, labels %s, spk per sentence %s" % (
        name, wav.numel() / 16000, len(info), len(rec["labels"]), rec["labels"].tolist()[:40], [s["spk"] for s in info]))


def cluster_cases():
    """Stored embedding matrices through the reference ClusterBackend; randomised postprocess / distribute_spk cases."""
    from funasr.models.campplus.cluster_backend import ClusterBackend
    from funasr.models.campplus.utils import distribute_spk, postprocess
    rng = np.random.RandomState(11)
    cases = {}

    def blobs(n, k, dim=192, spread=0.35, centers=None):
        c = rng.randn(k, dim) if centers is None else centers
        lab = rng.randint(0, k, size=n)
        return (c[lab] + spread * rng.randn(n, dim)).astype(np.float32)

    cases["spectral_k3"] = (blobs(120, 3), None)
    cases["spectral_preset4"] = (blobs(90, 4), 4)
    base = rng.randn(4, 192)
    near = np.stack([base[0], base[1], base[0] + 0.25 * rng.randn(192), base[3]])
    cases["merge_by_cos"] = (blobs(160, 4, centers=near, spread=0.5), None)
    cases["kmeans_2048"] = (blobs(2100, 3, dim=16, spread=0.6), 3)
    cases["few_rows"] = (blobs(12, 2), None)
    out = {}
    for name, (x, k) in cases.items():
        np.random.seed(0)
        lab = ClusterBackend()(torch.from_numpy(x), oracle_num=k)
        out[name + "__x"] = x
        out[name + "__k"] = np.int64(-1 if k is None else k)
        out[name + "__labels"] = np.asarray(lab).astype(np.int64)
        print("cluster %s: n=%d k=%s -> %d speakers" % (name, x.shape[0], k, len(set(np.asarray(lab).tolist()))))
    # postprocess / distribute_spk on random chunk layouts and labels
    for i in range(6):
        segs, t = [], 0.3
        for _ in range(rng.randint(3, 9)):
            dur = float(rng.choice([0.4, 1.0, 2.3, 3.7, 6.1]))
            for st, ed in [(0.0, min(1.5, dur))] + [(s, s + 1.5) for s in np.arange(0.75, max(dur - 1.5, 0) + 1e-9, 0.75)]:
                segs.append([float(t + st), float(t + ed)])         # Python floats, as sv_chunk's times are
            t += dur + float(rng.choice([0.2, 0.9, 2.0]))
        lab = rng.randint(0, 3, size=len(segs))
        emb = rng.randn(len(segs), 8).astype(np.float32)
        sv, centers = postprocess([list(s) for s in segs], None, lab.copy(), emb, return_spk_center=True)
        sentences = [{"start": int(a * 1000), "end": int(b * 1000)} for a, b in
                     sorted(set((round(s[0], 1), round(s[0], 1) + float(rng.choice([0.5, 1.2, 3.0]))) for s in segs[::2]))]
        distribute_spk(sentences, sv)
        out["post%d__segs" % i] = np.array(segs)
        out["post%d__labels" % i] = lab.astype(np.int64)
        out["post%d__emb" % i] = emb
        out["post%d__sv" % i] = np.array([[a, b, c] for a, b, c in sv], dtype=np.float64)
        out["post%d__centers" % i] = centers.astype(np.float32)
        out["post%d__sentences" % i] = np.array(json.dumps(sentences))
    np.savez_compressed(os.path.join(GOLD, "spk_host_routines.npz"), **out)


def main():
    ref_shim.import_reference()
    os.makedirs(GOLD, exist_ok=True)
    which = sys.argv[1:] or ["pipeline", "host"]
    if "pipeline" in which:
        with tempfile.TemporaryDirectory() as tmp:
            # calibrate on the chunks the reference pipeline itself cuts from the two-voice recording
            pattern, seed, kw = SPK_CASES["spk_two_voices"]
            rec = run_case(build_pipeline(tmp, None), "spk_two_voices", pattern, seed, kw, save=False)
            voice = np.array([voice_at(pattern, 0.5 * (a + b)) for a, b in sorted(rec["times"])])
            order = np.argsort([a for a, _ in rec["times"]], kind="stable")
            stats = calibrate([rec["chunks"][i] for i in order], voice)
            am = build_pipeline(tmp, stats)
            for name, (pattern, seed, kw) in SPK_CASES.items():
                run_case(am, name, pattern, seed, kw)
    if "host" in which:
        cluster_cases()


if __name__ == "__main__":
    main()
