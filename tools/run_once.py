"""Runs the hot path a few times (for ncu launch lists / captures). Usage: run_once.py --mode fp16x3 --B 16 --iters 2

--profile DIR: one untimed warm-up forward, then the timed iterations under torch.profiler with CUDA activities; writes
DIR/trace.pt.trace.json and DIR/kernels.txt (per kernel: calls, total ms, share of the summed step time; gemm_tc_kernel rows
carry their output kind, the last template argument)."""
import argparse, collections, json, os, re, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from funasr_b200 import synth
from funasr_b200.engine import FrontendEngine, ParaformerEngine
ap = argparse.ArgumentParser()
ap.add_argument("--mode", default="fp16x3"); ap.add_argument("--B", type=int, default=16); ap.add_argument("--iters", type=int, default=2)
ap.add_argument("--layers", type=int, default=50)
ap.add_argument("--profile", metavar="DIR", default=None)
a = ap.parse_args()
dev = "cuda:0"
cfg = synth.ParaformerConfig(enc_layers=a.layers, dec_layers=16 if a.layers == 50 else 2)
p = synth.make_state_dict(cfg, 0)
fe = FrontendEngine(synth.make_cmvn(cfg, 1), dev)
eng = ParaformerEngine(p, cfg, dev, gemm_mode=a.mode)
base = [synth.make_wav(480000, 100 + i) for i in range(4)]
wav = torch.stack([base[i % 4].roll(977 * i) for i in range(a.B)]).to(dev)
lens = torch.full((a.B,), 480000, dtype=torch.int32, device=dev)
torch.cuda.synchronize()

# gemm_tc_kernel<BN, STAGES, APL, WPL, EPI>: EPI names the output kind (gemm_tc.cu)
EPI_KINDS = {"0": "EPI_F32 (out-proj / w_2 / decoder)", "1": "EPI_PLANES (w_1)", "2": "EPI_ATT (QKV)", "3": "EPI_F32R2 (two residuals)"}


def kernel_table(trace_path, step_ms):
    with open(trace_path) as f:
        events = json.load(f)["traceEvents"]
    calls, us = collections.Counter(), collections.Counter()
    for e in events:
        if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset"):
            calls[e["name"]] += 1
            us[e["name"]] += e["dur"]
    lines = ["# %d iteration(s), summed step time %.3f ms (CUDA events around frontend + forward)" % (a.iters, step_ms),
             "%-8s %10s %7s  %s" % ("calls", "total_ms", "share", "kernel")]
    gemm_ms, by_kind = 0.0, collections.Counter()
    for name, t in us.most_common():
        ms = t / 1e3
        m = re.search(r"gemm_tc_kernel<([^>]*)>", name)
        label = name
        if m:
            kind = EPI_KINDS.get(m.group(1).split(",")[-1].strip(), "?")
            label = "%s  [%s]" % (name, kind)
            gemm_ms += ms
            by_kind[kind] += ms
        lines.append("%-8d %10.3f %6.1f%%  %s" % (calls[name], ms, 100 * ms / step_ms, label[:200]))
    lines.append("")
    lines.append("gemm_tc_kernel total: %.3f ms = %.1f%% of the step" % (gemm_ms, 100 * gemm_ms / step_ms))
    for kind, ms in by_kind.most_common():
        lines.append("  %-40s %10.3f ms %6.1f%%" % (kind, ms, 100 * ms / step_ms))
    lines.append("all kernels + copies: %.3f ms = %.1f%% of the step" % (sum(us.values()) / 1e3, 100 * sum(us.values()) / 1e3 / step_ms))
    return "\n".join(lines) + "\n"


def step(it):
    t0 = time.perf_counter()
    e0, e1, e2 = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    e0.record()
    feats, fl = fe(wav, lens, 500)
    t1 = time.perf_counter()
    e1.record()
    out = eng.forward_feats(feats, fl)
    e2.record()
    torch.cuda.synchronize()
    print("iter %d: host fe call %.3f ms, gpu frontend %.3f ms, gpu rest %.3f ms, wall %.3f ms, tokens %d" % (
        it, (t1 - t0) * 1e3, e0.elapsed_time(e1), e1.elapsed_time(e2), (time.perf_counter() - t0) * 1e3, int(out["token_num"].sum())), flush=True)
    return e0.elapsed_time(e2)


if a.profile is None:
    for it in range(a.iters):
        step(it)
else:
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(a.profile, exist_ok=True)
    step(-1)                                          # warm-up: module loads, tensor-map cache, allocator
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        step_ms = sum(step(it) for it in range(a.iters))
    trace = os.path.join(a.profile, "trace.pt.trace.json")
    prof.export_chrome_trace(trace)
    table = kernel_table(trace, step_ms)
    with open(os.path.join(a.profile, "kernels.txt"), "w") as f:
        f.write(table)
    print(table)
