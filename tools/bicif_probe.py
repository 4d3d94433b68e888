"""Times the BiCifParaformer additions at the benchmark shape (B=64 x 30 s): token path vs the upsampled timestamp head, and this
library's BLSTM recurrence against cuDNN's."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from funasr_b200 import synth
from funasr_b200.engine import FrontendEngine, ParaformerEngine

B = 64
dev = "cuda:0"
cfg = synth.ParaformerConfig()
state = synth.make_bicif_state_dict(cfg, 0)
eng = ParaformerEngine(state, cfg, dev, gemm_mode="fp16x3", bicif=True)
fe = FrontendEngine(synth.make_cmvn(cfg, 1), dev)
base = [synth.make_wav(480000, 100 + i) for i in range(4)]
wav = torch.stack([base[i % 4].roll(977 * i) for i in range(B)]).to(dev)
wl = torch.full((B,), 480000, dtype=torch.int32, device=dev)


def timeit(fn, n=5):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


feats, fl = fe(wav, wl, 500)
out = eng.forward_feats(feats, fl)
t_tok = timeit(lambda: eng.forward_feats(fe(wav, wl, 500)[0], fl))
enc, lens, tok = out["enc_dev"], out["lens_dev"], out["tok_dev"]
t_ts = timeit(lambda: eng.upsample_timestamp(enc, lens, tok))
# the recurrence alone: fa_blstm_forward_tc against torch.nn.LSTM (cuDNN, TF32 off) with the same weights and input
bp = "predictor.blstm."
lstm = torch.nn.LSTM(512, 512, 1, bias=True, batch_first=True, bidirectional=True).to(dev)
lstm.load_state_dict({k[len(bp):]: v for k, v in state.items() if k.startswith(bp)})
lstm.eval().requires_grad_(False)
x = torch.randn(B, 1500, 512, device=dev) * 0.5
torch.backends.cuda.matmul.allow_tf32 = False
with torch.no_grad(), torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
    xproj = torch.cat([x @ lstm.weight_ih_l0.T + (lstm.bias_ih_l0 + lstm.bias_hh_l0),
                       x @ lstm.weight_ih_l0_reverse.T + (lstm.bias_ih_l0_reverse + lstm.bias_hh_l0_reverse)], -1).reshape(B * 1500, 4096)
    t_lstm = timeit(lambda: lstm(x))
    ref, _ = lstm(x)
from funasr_b200 import _abi
st = torch.cuda.current_stream().cuda_stream
nbs = int(eng.lib.fa_blstm_tc_scratch_bytes(B))
scr = torch.empty(nbs, dtype=torch.uint8, device=dev)
feat_tc = torch.empty(B, 1500, 1024, device=dev)
t_tc = timeit(lambda: _abi.check(eng.lib.fa_blstm_forward_tc(xproj.data_ptr(), eng.ts_head.w_hh_fwd, eng.ts_head.w_hh_bwd, B, 1500, 512,
                                                            feat_tc.data_ptr(), scr.data_ptr(), nbs, st), "blstm tc"))
torch.cuda.synchronize()
print(f"fa_blstm_forward_tc (mma.sync bf16 x3) alone (recurrence, B={B}, T=1500): {t_tc:.2f} ms = {t_tc / 1500 * 1000:.2f} us per step; "
      f"max |tc - cuDNN| = {float((feat_tc - ref).abs().max()):.3e}")
print(f"B={B}: token path (frontend+encoder+CIF(v3)+decoder) {t_tok:.2f} ms; timestamp head {t_ts:.2f} ms; cuDNN BLSTM [64,1500,512] {t_lstm:.2f} ms")
