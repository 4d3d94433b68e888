"""Times the host-side (CPU) routines that sit behind the GPU path — the VAD end-point walk and the timestamp post-processing — in
their Python-specification form and in the form the model classes run (library host code / vectorised).  No GPU needed.
    python tools/host_probe.py > host_routines.json"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from funasr_b200 import timestamps as TS, vad  # noqa: E402


def per_call_ms(fn, n):
    fn()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    return (time.perf_counter() - t0) / n * 1e3


g = np.load(os.path.join(ROOT, "tests", "golden", "vad_130s.npz"))
sp, db, n = g["sil_prob"], g["decibel"], int(g["n_samples"])
sp_l, db_l = sp.tolist(), db.tolist()
rep = {"cpu": open("/proc/cpuinfo").read().split("model name")[1].split("\n")[0].strip(": \t") if os.path.exists("/proc/cpuinfo") else "?",
       "vad_detector_130s_recording_ms": {"python_walk": per_call_ms(lambda: vad.detect_segments(sp_l, db_l, n), 5),
                                          "library_host_code": per_call_ms(lambda: vad.detect_segments_native(sp, db, n), 200)}}
rep["vad_detector_130s_recording_ms"]["x_realtime_python"] = 130e3 / rep["vad_detector_130s_recording_ms"]["python_walk"]
rep["vad_detector_130s_recording_ms"]["x_realtime_library"] = 130e3 / rep["vad_detector_130s_recording_ms"]["library_host_code"]
d = np.load(os.path.join(ROOT, "tests", "golden", "bicif_large_single.npz"))
ua, up = d["us_alphas"][0], d["us_peaks"][0]
toks = ["t%d" % i for i in range(int(d["ids_len"][0]))]
rng = np.random.default_rng(0)
al = rng.uniform(0, 0.22, 1500).astype(np.float32)
rep["timestamps_per_utterance_ms"] = {
    "bicif_golden_501_frames_13_tokens": {"labelled_walk_with_text": per_call_ms(lambda: TS.ts_prediction_lfr6_standard(ua, up, toks), 200),
                                           "stamps_only": per_call_ms(lambda: TS.ts_prediction_lfr6_standard(ua, up, toks, want_text=False), 500)},
    "re_integration_1500_frames": {"python_loop": per_call_ms(lambda: TS.cif_wo_hidden_py(al, 0.9999), 20),
                                   "library_host_code": per_call_ms(lambda: TS.cif_wo_hidden(al, 0.9999), 2000)}}
tr = TS.cif_wo_hidden(al * np.float32(161 / al.sum()), 0.9999)
toks2 = ["t%d" % i for i in range(int((tr >= np.float32(0.9999)).sum()) - 1)]
a2 = al * np.float32(161 / al.sum())
rep["timestamps_per_utterance_ms"]["synthetic_1500_frames_%d_tokens" % len(toks2)] = {
    "labelled_walk_with_text": per_call_ms(lambda: TS.ts_prediction_lfr6_standard(a2, tr, toks2), 100),
    "stamps_only": per_call_ms(lambda: TS.ts_prediction_lfr6_standard(a2, tr, toks2, want_text=False), 500)}
print(json.dumps(rep, indent=1))
