"""GPU (-m gpu): kernel-level parity of the decode-side kernels whose outputs are integers or decide integers — the BiLSTM
recurrence of the timestamp head, CIF integrate-and-fire (both variants), the timestamp re-integration, the arg-max / log-softmax
head, the CTC and greedy filters and the SeACo merge — each against a plain restatement of the same operation on the CPU, at the
batch shapes, lengths and vocabularies where these kernels change code path.

Two things make bit-exact comparisons possible here.
  * Crafted inputs whose arithmetic is exact on both sides.  One caveat shapes every construction that goes through the tensor-core
    GEMM: its epilogue multiplies the accumulator by 1 + (K / 16) c (the compensation for the tensor cores' truncating fp32
    accumulation, gemm_tc.cu), so in the fp16x* modes a GEMM output is exact only where the accumulator is 0 and the value comes
    from the bias.  The crafted CIF alphas therefore take their per-frame value from the conv bias and the ReLU.  The arg-max
    rows keep their designed maxima, ties and near-ties in columns whose activation is 0, so those values are the bias exactly.
  * Where the input of a kernel is itself the output of a GEMM, the reference starts from the GPU's own values (returned alphas,
    or the logits of a separate fa_linear call with the same weights, which is the GEMM fa_linear_argmax runs).  Then only the
    kernel under test stands between the two sides.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import paraformer_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
D = 512
H = 512


def _lib():
    from funasr_b200 import _abi
    return _abi, _abi.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    """Bit pattern of an fp32 tensor: torch.equal on it also tells -0.0 from 0.0."""
    return t.contiguous().view(torch.int32)


def _planes(lib, abi, w):
    """fp16 planes [3][out_f][in_pad] of a device weight [out_f, in_f] for the tensor-core modes."""
    out_f, in_f = w.shape
    in_pad = (in_f + 63) // 64 * 64
    p = torch.empty(3, out_f, in_pad, dtype=torch.float16, device=DEV)
    abi.check(lib.fa_split_planes(w.data_ptr(), in_f, out_f, in_f, in_pad, p.data_ptr(), _st()), "fa_split_planes")
    return p, in_pad


# ============================================================================================== BiLSTM recurrence
# Bound on |h_gpu - h_ref|.  The kernel's recurrent product runs on bf16 hi / lo planes with three products: each operand is
# x = hi + lo + e, |e| <= 2^-18 |x|, and the dropped lo * lo term is <= 2^-18 |x w|, so each product carries <= ~2^-16 relative
# error, accumulated in fp32.  A gate pre-activation sum_k w_k h_k (512 terms, |w| <= 1/sqrt(512) at PyTorch's default init) then
# carries a random-signed error of ~2^-16 * sqrt(512) * rms|w h| ~ 1e-6 per step, and the cell state carries it forward damped by
# the forget gate, so the error does not grow with T.  The ×4 set scales weights and input projections by 4: each gate sees 4x
# larger products and the saturated cells hold larger values, ~16x the error in all.
# Measured on an H100 80GB HBM3 (700 W): worst |d h| 1.2e-6 at the default init (B = 64, T = 300; 1.2e-6 also at B = 16,
# T = 1500) and 1.9e-5 with the ×4 weights (B = 16, T = 1500): the bound keeps a factor 5 over the worst case.
BLSTM_TOL = 1e-4
BLSTM_SHAPES = [(1, 1), (3, 2), (64, 300), (65, 97), (130, 64), (256, 40), (16, 1500)]


def _blstm_weights(scale, seed=11):
    """w_hh of both directions with PyTorch's default nn.LSTM init U(-1/sqrt(512), 1/sqrt(512)), times `scale`."""
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / math.sqrt(H)
    return [((torch.rand(4 * H, H, generator=g) * 2 - 1) * (k * scale)).contiguous() for _ in range(2)]


def _blstm_xproj(B, T, scale, seed):
    """Input projections x W_ih^T + b_ih + b_hh of both directions, [B, T, 4096] fp32: for x ~ N(0, 1) and the default init the
    per-gate pre-activation has std sqrt(512 / (3 * 512)) ~ 0.58."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, T, 8 * H, generator=g) * (0.58 * scale)


def _blstm_ref(xproj, w_f, w_b):
    """float64 one-layer bidirectional nn.LSTM recurrence from the same fp32 input projections: gate order i, f, g, o, zero initial
    state, no packing (the reverse direction starts at t = T - 1 of the padded length) -> [B, T, 1024] float64 (forward | reverse)."""
    B, T, _ = xproj.shape
    out = torch.empty(B, T, 2 * H, dtype=torch.float64)
    for d, w in enumerate((w_f, w_b)):
        wt = w.double().t().contiguous()
        h = torch.zeros(B, H, dtype=torch.float64)
        c = torch.zeros(B, H, dtype=torch.float64)
        for s in range(T):
            t = s if d == 0 else T - 1 - s
            z = xproj[:, t, d * 4 * H:(d + 1) * 4 * H].double() + h @ wt
            i, f, g, o = z.split(H, dim=1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
            h = torch.sigmoid(o) * torch.tanh(c)
            out[:, t, d * H:(d + 1) * H] = h
    return out


def _blstm_run(lib, xp_dev, wf_dev, wb_dev, B, T, scratch):
    out = torch.full((B, T, 2 * H), float("nan"), device=DEV)
    st = lib.fa_blstm_forward_tc(xp_dev.data_ptr(), wf_dev.data_ptr(), wb_dev.data_ptr(), B, T, H, out.data_ptr(),
                                 scratch.data_ptr(), scratch.numel(), _st())
    assert st == 0, st
    torch.cuda.synchronize()
    return out


def test_blstm_reference_is_torch_lstm():
    """The float64 restatement above is nn.LSTM(512, 512, bidirectional=True, batch_first=True): same gate order, bias split and
    reverse-direction indexing."""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(3, 7, H, generator=g, dtype=torch.float64)
    lstm = torch.nn.LSTM(H, H, 1, batch_first=True, bidirectional=True).double()
    with torch.no_grad():
        want, _ = lstm(x)
        xp = torch.cat([x @ lstm.weight_ih_l0.t() + lstm.bias_ih_l0 + lstm.bias_hh_l0,
                        x @ lstm.weight_ih_l0_reverse.t() + lstm.bias_ih_l0_reverse + lstm.bias_hh_l0_reverse], -1)
        got = _blstm_ref(xp, lstm.weight_hh_l0, lstm.weight_hh_l0_reverse)
    assert float((got - want).abs().max()) < 1e-12


@pytest.mark.parametrize("scale", [1, 4])
@pytest.mark.parametrize("B,T", BLSTM_SHAPES)
def test_blstm_recurrence_vs_float64_lstm(B, T, scale):
    """fa_blstm_forward_tc against the float64 LSTM at batch tiles 1 to 4 (B = 65..256 spans 2..4 tiles of 64 sequences, with a
    ragged last tile), t_len = 1 and the 3 x 500 frames of a 30 s utterance."""
    abi, lib = _lib()
    w_f, w_b = _blstm_weights(scale)
    xp = _blstm_xproj(B, T, scale, seed=B * 7919 + T)
    scratch = torch.empty(int(lib.fa_blstm_tc_scratch_bytes(B)), dtype=torch.uint8, device=DEV)
    out = _blstm_run(lib, xp.to(DEV), w_f.to(DEV), w_b.to(DEV), B, T, scratch).cpu()
    ref = _blstm_ref(xp, w_f, w_b)
    assert not torch.isnan(out).any()
    err_f = float((out[..., :H].double() - ref[..., :H]).abs().max())
    err_b = float((out[..., H:].double() - ref[..., H:]).abs().max())
    print("blstm B=%d T=%d x%d: max |dh| forward %.2e reverse %.2e (bound %.0e)" % (B, T, scale, err_f, err_b, BLSTM_TOL))
    assert err_f <= BLSTM_TOL and err_b <= BLSTM_TOL


def test_blstm_batch_composition_and_dirty_scratch_are_bit_exact():
    """Each MMA row is one sequence, so a sequence's output cannot depend on which tile or row it occupies: sequences at the tile
    edges of a B = 256 run equal the same input rows run alone, bit for bit.  A second call on the same, now dirty, scratch (the
    exchange planes and barrier counters of the previous call) repeats the first bit for bit."""
    abi, lib = _lib()
    B, T = 256, 40
    w_f, w_b = [w.to(DEV) for w in _blstm_weights(1)]
    xp = _blstm_xproj(B, T, 1, seed=5).to(DEV)
    scratch = torch.empty(int(lib.fa_blstm_tc_scratch_bytes(B)), dtype=torch.uint8, device=DEV)
    full = _blstm_run(lib, xp, w_f, w_b, B, T, scratch)
    for b in (0, 63, 64, 127, 128, 255):
        one = _blstm_run(lib, xp[b:b + 1].contiguous(), w_f, w_b, 1, T, scratch)
        assert torch.equal(_bits(one[0]), _bits(full[b])), b
    again = _blstm_run(lib, xp, w_f, w_b, B, T, scratch)
    assert torch.equal(_bits(again), _bits(full))


def test_blstm_status_codes():
    abi, lib = _lib()
    T = 4
    xp = torch.zeros(257 * T * 8 * H, device=DEV)
    w = torch.zeros(4 * H, H, device=DEV)
    out = torch.empty(257 * T * 2 * H, device=DEV)
    big = int(lib.fa_blstm_tc_scratch_bytes(256))
    scratch = torch.empty(big, dtype=torch.uint8, device=DEV)
    args = lambda x, b, hid, nbytes: (x, w.data_ptr(), w.data_ptr(), b, T, hid, out.data_ptr(), scratch.data_ptr(), nbytes, _st())
    assert lib.fa_blstm_forward_tc(*args(xp.data_ptr(), 257, H, big)) == -4          # more than 4 batch tiles
    assert lib.fa_blstm_forward_tc(*args(xp.data_ptr(), 2, 256, big)) == -4          # hidden != 512
    assert lib.fa_blstm_forward_tc(*args(xp.data_ptr(), 65, H, int(lib.fa_blstm_tc_scratch_bytes(65)) - 1)) == -3
    assert lib.fa_blstm_forward_tc(*args(None, 2, H, big)) == -1
    assert lib.fa_blstm_forward_tc(*args(xp.data_ptr(), 0, H, big)) == 0              # nothing to do
    torch.cuda.synchronize()


# ============================================================================================== CIF predictor
CIF_MODES = ["fp32", "fp16x3", "fp16x6"]
TAIL = 0.45
# |alpha_gpu - alpha_oracle|: the k = 3 conv is a GEMM in the engine's mode, then a 512-wide dot product and a sigmoid (slope
# <= 1/4) in fp32.  In the tensor-core modes the conv's accumulation rounding dominates (fp16x3 and fp16x6 measure the same).
# Crafted alphas are exact except the ~0.6 frame, which carries the tensor-core epilogue's scale.
# Measured on an H100 (random weights, worst over T = 37 / 500 / 4100): fp32 8.3e-7, fp16x3 2.3e-6, fp16x6 2.3e-6; crafted: 0 in
# fp32, 4.8e-7 in the tensor-core modes.
ALPHA_TOL = {"fp32": 2e-6, "fp16x3": 5e-6, "fp16x6": 5e-6}

# channel-0 encoder values of the crafted predictor (see _crafted_predictor) and the alpha each one gives
X_ONE, X_HALF, X_ZERO, X_06 = -40.0, 0.0, 20.0, -0.40625


def _predictor_struct(abi, lib, mode, variant, conv_w, conv_b, out_w, out_b):
    """FaPredictor for Conv1d weight conv_w [512, 512, 3] (repacked to the GEMM weight W[n, k*512 + c] = w[n, c, k]), bias conv_b,
    cif_output weight out_w [512] and bias out_b [1]; threshold 1, tail 0.45, smooth 1, noise 0.  -> (struct, tensors to keep)."""
    W = conv_w.permute(0, 2, 1).reshape(D, 3 * D).contiguous().to(DEV)
    keep = [W, conv_b.to(DEV), out_w.contiguous().to(DEV), out_b.to(DEV)]
    planes, in_pad = (None, 3 * D)
    if mode != "fp32":
        planes, in_pad = _planes(lib, abi, W)
        keep.append(planes)
    conv = abi.FaLinear(W.data_ptr(), keep[1].data_ptr(), planes.data_ptr() if planes is not None else None, D, 3 * D, in_pad, 0)
    return abi.FaPredictor(conv, keep[2].data_ptr(), keep[3].data_ptr(), 1.0, TAIL, 1.0, 0.0, variant, 0), keep


def _crafted_predictor():
    """alpha = sigmoid(20 - relu(enc[t, 0] + 20)) through the real conv / alpha head: conv centre tap of channel 0 -> output
    channel 0 with bias 20, out_w = -e0, out_b = 20.  enc[t, 0] <= -20 gives exactly 1.0 (relu -> 0, sigmoid(20) rounds to 1),
    enc[t, 0] = 0 gives exactly 0.5 (the accumulator is 0, so the conv output is its bias 20 in every mode), 20 gives ~2e-9 and
    -0.40625 gives ~0.6002."""
    conv_w = torch.zeros(D, D, 3)
    conv_w[0, 0, 1] = 1.0
    conv_b = torch.zeros(D)
    conv_b[0] = 20.0
    out_w = torch.zeros(D)
    out_w[0] = -1.0
    return conv_w, conv_b, out_w, torch.tensor([20.0])


def _random_predictor(seed=3):
    """The seeded predictor weights funasr_b200.synth gives a Paraformer (about one token per five frames)."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(D, D, 3, generator=g) / math.sqrt(3 * D), torch.randn(D, generator=g) * 0.02,
            torch.randn(D, generator=g) * (1.2 / math.sqrt(D)), torch.tensor([-1.6]))


def _crafted_enc(T, lens, seed):
    """[B, T, 512]: random N(0, 1) channels (they weigh 0 in the crafted alpha, but they are the hidden states the acoustic
    embeddings integrate) and a channel 0 that spells alpha sequences whose fp64 prefix sums land exactly on integers."""
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    enc = torch.randn(B, T, D, generator=g)
    pat = [
        [X_ONE],                                                    # 1.0 every frame: a fire on every frame, sums 1, 2, 3, ...
        [X_HALF],                                                   # 0.5 runs: every second frame lands on an integer
        [X_HALF, X_ONE, X_HALF, X_ZERO, X_HALF, X_HALF, X_ONE, X_ONE, X_ZERO, X_ZERO, X_HALF],   # mixed, with ~0 frames
        [X_ZERO, X_ZERO, X_HALF, X_ONE, X_HALF, X_ONE, X_ONE, X_HALF, X_ZERO, X_HALF],
    ]
    for b in range(B):
        p = pat[b % len(pat)]
        ch0 = torch.tensor([p[t % len(p)] for t in range(T)])
        n = min(int(lens[b]), T)
        if b % 2 == 0 and n >= 3:                                   # ... 0.5, 0.6 before the end: the 0.45 tail completes a token
            ch0[n - 3], ch0[n - 2], ch0[n - 1] = X_HALF, X_HALF, X_06
        enc[b, :, 0] = ch0
    return enc


def _cif_run(abi, lib, pred, mode, enc, lens, n_cap, guard=4096):
    """fa_cif_predictor_forward into a sentinel-filled acoustic buffer with `guard` floats behind it -> CPU tensors."""
    B, T, _ = enc.shape
    SENT = 12345.0
    acoustic = torch.full((B * n_cap * D + guard,), SENT, device=DEV)
    tok = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    alphas = torch.full((B, T + 1), float("nan"), device=DEV)
    peaks = torch.full((B, T + 1), float("nan"), device=DEV)
    m = abi.GEMM_MODES[mode]
    ws = torch.empty(int(lib.fa_cif_predictor_workspace_bytes(B, T, m)), dtype=torch.uint8, device=DEV)
    encd, lensd = enc.to(DEV).contiguous(), torch.tensor(lens, dtype=torch.int32, device=DEV)
    abi.check(lib.fa_cif_predictor_forward(C.byref(pred), encd.data_ptr(), lensd.data_ptr(), B, T, acoustic.data_ptr(), n_cap,
                                           tok.data_ptr(), alphas.data_ptr(), peaks.data_ptr(), m, ws.data_ptr(), ws.numel(), _st()),
              "fa_cif_predictor_forward")
    torch.cuda.synchronize()
    acoustic = acoustic.cpu()
    assert bool((acoustic[B * n_cap * D:] == SENT).all()), "acoustic written past batch * n_cap rows"
    return acoustic[:B * n_cap * D].view(B, n_cap, D), tok.cpu(), alphas.cpu(), peaks.cpu()


def _cif_reference(variant, enc, alphas):
    """From the GPU's own alphas [B, T+1]: (fire positions [B, T+1] bool, peaks, frames [B, >= fires, 512]) — cif_wo_hidden_v1 +
    cif_v1 (fp64 prefix sums, torch's cumsum of alphas * hidden) for variant 0, the sequential fp32 `cif` for variant 1."""
    B, T, _ = enc.shape
    hidden = torch.cat([enc, torch.zeros(B, 1, D)], dim=1)
    if variant == 0:
        peaks, fire = O.cif_fires(alphas)
        frames, _ = O.cif_v1(hidden, alphas)
    else:
        frames, peaks = O.cif_loop(hidden, alphas, 1.0)
        fire = peaks >= 1.0
    return fire, peaks, frames


def _check_cif(variant, enc, lens, out, n_cap, ref_alphas=None, mode="fp32"):
    acoustic, tok, alphas, peaks = out
    B, T, _ = enc.shape
    fire, want_peaks, frames = _cif_reference(variant, enc, alphas)
    assert torch.equal(tok, torch.floor(alphas.sum(-1)).to(torch.int32))           # floor(alphas.sum(-1)) in torch's fp32 order
    assert torch.equal(_bits(peaks), _bits(want_peaks))
    worst = 0.0
    for b in range(B):
        n = int(fire[b].sum())
        k = min(n, n_cap)
        assert frames.shape[1] >= k
        got, want = acoustic[b, :k], frames[b, :k]
        if not torch.equal(_bits(got), _bits(want)):
            d = (got.double() - want.double()).abs().max() / want.double().abs().max()
            worst = max(worst, float(d))
        assert bool((acoustic[b, k:] == 0).all()), "row %d: rows at or beyond the fire count must be zero" % b
    assert worst == 0.0, "acoustic embeddings differ from the reference's, max relative %.2e" % worst
    err = None
    if ref_alphas is not None:
        err = float((alphas.double() - ref_alphas.double()).abs().max())
        assert err <= ALPHA_TOL[mode], err
    return err


def _oracle_alphas(enc, lens, conv_w, conv_b, out_w, out_b):
    """alphas after tail_process_fn, [B, T+1], from the oracle's CifPredictorV2 head."""
    B, T, _ = enc.shape
    p = {"predictor.cif_conv1d.weight": conv_w, "predictor.cif_conv1d.bias": conv_b,
         "predictor.cif_output.weight": out_w[None], "predictor.cif_output.bias": out_b}
    mask = (torch.arange(T)[None, :] < torch.tensor(lens)[:, None])[:, None, :]
    al = O.cif_alphas(enc, mask, p)
    _, al2, _ = O.cif_tail(enc, al, mask.squeeze(1).float(), TAIL)
    return al2


@pytest.mark.parametrize("mode", CIF_MODES)
@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("T", [64, 500, 4100])
def test_cif_crafted_exact_alphas(T, variant, mode):
    """Alphas of exactly 1.0 and 0.5 (and ~2e-9, and one ~0.6 frame before the tail): prefix sums land exactly on integers and the
    0.45 tail completes a token.  T = 4100 takes the > 48 KB dynamic shared-memory path.  Token counts, fire positions, peaks and
    the acoustic embeddings equal the reference's arithmetic bit for bit; rows at or beyond the fire count are zero."""
    abi, lib = _lib()
    weights = _crafted_predictor()
    pred, keep = _predictor_struct(abi, lib, mode, variant, *weights)
    lens = [T, T - 3, T, 1, 0, T // 2]
    enc = _crafted_enc(T, lens, seed=T + variant)
    out = _cif_run(abi, lib, pred, mode, enc, lens, T + 1)
    alphas = out[2]
    assert set(alphas[:, :-1].flatten().tolist()) >= {1.0, 0.5, 0.0}             # the construction holds in this mode
    err = _check_cif(variant, enc, lens, out, T + 1, _oracle_alphas(enc, lens, *weights), mode)
    print("cif crafted T=%d variant %d %s: tokens %s, alpha err %.2e" % (T, variant, mode, out[1].tolist(), err))


@pytest.mark.parametrize("mode", CIF_MODES)
@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("T", [37, 500, 4100])
def test_cif_random_ragged(T, variant, mode):
    """Random encoder output and the synthetic predictor weights over a ragged batch: lens T, 0, 1, T - 1, T + 5 (clamped to
    T by the kernel, all-ones mask in the reference) and random lengths."""
    abi, lib = _lib()
    weights = _random_predictor()
    pred, keep = _predictor_struct(abi, lib, mode, variant, *weights)
    g = torch.Generator().manual_seed(100 + T)
    lens = [T, 0, 1, T - 1, T + 5] + torch.randint(1, T + 1, (3,), generator=g).tolist()
    enc = torch.randn(len(lens), T, D, generator=g)
    out = _cif_run(abi, lib, pred, mode, enc, lens, T + 1)
    err = _check_cif(variant, enc, lens, out, T + 1, _oracle_alphas(enc, lens, *weights), mode)
    print("cif random T=%d variant %d %s: tokens %s, alpha err %.2e" % (T, variant, mode, out[1].tolist(), err))


@pytest.mark.parametrize("variant", [0, 1])
def test_cif_n_cap_below_fire_count(variant):
    """With n_cap smaller than the number of fires the first n_cap rows are those of an uncapped run and nothing is written past
    them: not into the next utterance's rows, not behind the buffer."""
    abi, lib = _lib()
    mode, T = "fp16x3", 64
    weights = _crafted_predictor()
    pred, keep = _predictor_struct(abi, lib, mode, variant, *weights)
    lens = [T, T, T - 3]
    enc = _crafted_enc(T, lens, seed=9)
    full = _cif_run(abi, lib, pred, mode, enc, lens, T + 1)
    assert int(full[1].min()) > 5
    for n_cap in (1, 5):
        capped = _cif_run(abi, lib, pred, mode, enc, lens, n_cap)
        assert torch.equal(capped[1], full[1]) and torch.equal(_bits(capped[3]), _bits(full[3]))
        assert torch.equal(_bits(capped[0]), _bits(full[0][:, :n_cap]))
        _check_cif(variant, enc, lens, capped, n_cap)


@pytest.mark.parametrize("variant", [0, 1])
def test_cif_t_max_limit(variant):
    """Three [T + 1] arrays in shared memory: t_max = 17065 is the largest that fits 200 KB; 17066 returns -4."""
    abi, lib = _lib()
    pred, keep = _predictor_struct(abi, lib, "fp16x3", variant, *_crafted_predictor())
    m = abi.GEMM_MODES["fp16x3"]
    T = 17066
    enc = torch.zeros(1, T, D, device=DEV)
    lens = torch.tensor([T], dtype=torch.int32, device=DEV)
    acoustic = torch.empty(T + 1, D, device=DEV)
    tok = torch.empty(1, dtype=torch.int32, device=DEV)
    al, pk = torch.empty(1, T + 1, device=DEV), torch.empty(1, T + 1, device=DEV)
    ws = torch.empty(int(lib.fa_cif_predictor_workspace_bytes(1, T, m)), dtype=torch.uint8, device=DEV)
    st = lib.fa_cif_predictor_forward(C.byref(pred), enc.data_ptr(), lens.data_ptr(), 1, T, acoustic.data_ptr(), T + 1, tok.data_ptr(),
                                      al.data_ptr(), pk.data_ptr(), m, ws.data_ptr(), ws.numel(), _st())
    assert st == -4
    st = lib.fa_cif_predictor_forward(C.byref(pred), enc.data_ptr(), lens.data_ptr(), 1, T - 1, acoustic.data_ptr(), T, tok.data_ptr(),
                                      al.data_ptr(), pk.data_ptr(), m, ws.data_ptr(), ws.numel(), _st())
    assert st == 0
    torch.cuda.synchronize()


# ============================================================================================== timestamp re-integration
def _upsample_run(abi, lib, feat, w, b, lens_up, tok, smooth2, noise2, threshold):
    B, T3, dz = feat.shape
    us_a = torch.full((B, T3), float("nan"), device=DEV)
    us_p = torch.full((B, T3), float("nan"), device=DEV)
    fd, wd, bd = feat.to(DEV).contiguous(), w.to(DEV), b.to(DEV)
    ld = torch.tensor(lens_up, dtype=torch.int32, device=DEV)
    td = torch.tensor(tok, dtype=torch.int32, device=DEV)
    abi.check(lib.fa_cif_upsample_alphas(fd.data_ptr(), dz, wd.data_ptr(), bd.data_ptr(), ld.data_ptr(), td.data_ptr(), B, T3,
                                         smooth2, noise2, threshold, us_a.data_ptr(), us_p.data_ptr(), _st()), "fa_cif_upsample_alphas")
    torch.cuda.synchronize()
    return us_a.cpu(), us_p.cpu()


def _upsample_ref(z, lens_up, tok, smooth2, noise2, threshold):
    """CifPredictorV3.get_upsample_timestamp after the BLSTM, in fp32 on the CPU: alphas2 = relu(sigmoid(z) * smooth2 - noise2) *
    mask, rescaled by token_num / alphas2.sum(-1), then cif_wo_hidden with threshold - 1e-4 (the kernel's fp32 threshold)."""
    T3 = z.shape[1]
    mask = (torch.arange(T3)[None, :] < torch.tensor(lens_up)[:, None]).float()
    a2 = torch.relu(torch.sigmoid(z) * smooth2 - noise2) * mask
    a2 = a2 * (torch.tensor(tok, dtype=torch.float32) / a2.sum(-1))[:, None]
    thr = float(np.float32(float(np.float32(threshold)) - 1e-4))
    return a2, O.cif_wo_hidden_loop(a2, thr), thr


def _crafted_feat(z0, seed):
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(z0.shape[0], z0.shape[1], 1024, generator=g)
    feat[..., 0] = z0
    w = torch.zeros(1024)
    w[0] = 1.0
    return feat, w, torch.zeros(1)


@pytest.mark.parametrize("T3", [300, 1500])
def test_upsample_scan_crafted_bit_exact(T3):
    """feat . w + b in {-30, 0, 30} (w = e0, b = 0): with smooth 0.25 and noise 0.01 the alphas are exactly 0, 0.125 - 0.01 and
    0.25 - 0.01 in fp32 on both sides, so us_alphas (the rescale by token_num / sum) and us_peaks equal the CPU's bit for bit."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(T3)
    B = 4
    z = torch.tensor([-30.0, 0.0, 30.0])[torch.randint(0, 3, (B, T3), generator=g)]
    z[:, 0] = 30.0
    lens_up = [T3, T3 - 3, 3 * (T3 // 6), 3]
    a_unscaled = torch.relu(torch.sigmoid(z) * 0.25 - 0.01) * (torch.arange(T3)[None, :] < torch.tensor(lens_up)[:, None])
    tok = [max(1, int(round(float(s) * 1.1))) for s in a_unscaled.sum(-1)]
    feat, w, b = _crafted_feat(z, seed=T3 + 1)
    us_a, us_p = _upsample_run(abi, lib, feat, w, b, lens_up, tok, 0.25, 0.01, 1.0)
    a2, peaks, _ = _upsample_ref(z, lens_up, tok, 0.25, 0.01, 1.0)
    assert torch.equal(_bits(us_a), _bits(a2))
    assert torch.equal(_bits(us_p), _bits(peaks))


def test_upsample_scan_exact_threshold_crossings():
    """Dyadic alphas 0.25 / 0.5 (smooth 0.5, noise 1e-10), token_num equal to their sum (rescale by exactly 1) and a threshold whose
    fp32 threshold - 1e-4 is exactly 1.0: the running integral lands exactly on the threshold, where `>=` decides."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(4)
    B, T3 = 3, 96
    z = torch.tensor([0.0, 30.0])[torch.randint(0, 2, (B, T3), generator=g)]
    z[:, -4:] = torch.tensor([0.0, 0.0, 0.0, 0.0])
    lens_up = [T3, T3, T3]
    a = torch.where(z > 0, 0.5, 0.25)
    for r in range(B):                                              # make each row's sum an integer: the tail of four 0.25s absorbs the rest
        frac = float(a[r].sum()) % 1.0
        for k in range(int(round(frac / 0.25))):
            z[r, -1 - k] = -30.0
    a = torch.relu(torch.sigmoid(z) * 0.5 - 1e-10)
    tot = a.sum(-1)
    assert torch.equal(tot, torch.round(tot))
    tok = [int(t) for t in tot]
    feat, w, b = _crafted_feat(z, seed=5)
    threshold = 1.0001
    us_a, us_p = _upsample_run(abi, lib, feat, w, b, lens_up, tok, 0.5, 1e-10, threshold)
    a2, peaks, thr = _upsample_ref(z, lens_up, tok, 0.5, 1e-10, threshold)
    assert thr == 1.0 and torch.equal(a2, a) and bool((peaks == 1.0).any())
    assert torch.equal(_bits(us_a), _bits(a2))
    assert torch.equal(_bits(us_p), _bits(peaks))


def test_upsample_scan_random():
    """Random features and head weights: us_alphas within fp32 rounding of the float64 head (1e-6; measured on an H100: 6.0e-8),
    and us_peaks bit-exact against the sequential loop run on the GPU's own us_alphas."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(8)
    B, T3 = 5, 1500
    feat = torch.randn(B, T3, 1024, generator=g)
    w = torch.randn(1024, generator=g) * (3.0 / 32)
    b = torch.tensor([-0.3])
    lens_up = [T3, 3, T3 - 3, 300, 999]
    z = (feat.double() @ w.double() + b.double()).float()
    a_unscaled = torch.relu(torch.sigmoid(z) * 0.25 - 0.01) * (torch.arange(T3)[None, :] < torch.tensor(lens_up)[:, None])
    tok = [max(1, int(float(s))) for s in a_unscaled.sum(-1)]
    us_a, us_p = _upsample_run(abi, lib, feat, w, b, lens_up, tok, 0.25, 0.01, 1.0)
    a2, _, thr = _upsample_ref(z, lens_up, tok, 0.25, 0.01, 1.0)
    err = float((us_a.double() - a2.double()).abs().max())
    print("upsample random: us_alphas max |d| %.2e" % err)
    assert err <= 1e-6
    assert torch.equal(_bits(us_p), _bits(O.cif_wo_hidden_loop(us_a, thr)))


def _head_composed(abi, lib, head, mode, enc, lens, tok):
    """The timestamp head as the handle and the engine each launched it before fa_timestamp_head_forward, from public entries: the
    upsample fa_linear, the input-projection fa_linear, fa_blstm_forward_tc over at most 256 sequences per launch, lens x U (torch),
    fa_cif_upsample_alphas."""
    st = _st()
    B, T, d = enc.shape
    U = head.up_times
    ws = torch.empty(lib.fa_linear_workspace_bytes(B * T * U, d, mode) + 1, dtype=torch.uint8, device=DEV)
    up = torch.empty(B * T * U, d, device=DEV)
    xproj = torch.empty(B * T * U, 8 * d, device=DEV)
    feat = torch.empty(B * T * U, 2 * d, device=DEV)
    abi.check(lib.fa_linear(enc.data_ptr(), d, B * T, C.byref(head.upsample), 0, None, 0, None, 0, up.data_ptr(), U * d, mode, ws.data_ptr(),
                            ws.numel(), st), "fa_linear(upsample)")
    abi.check(lib.fa_linear(up.data_ptr(), d, B * T * U, C.byref(head.blstm_ih), 0, None, 0, None, 0, xproj.data_ptr(), 8 * d, mode,
                            ws.data_ptr(), ws.numel(), st), "fa_linear(blstm ih)")
    scratch = torch.empty(lib.fa_blstm_tc_scratch_bytes(min(B, 256)), dtype=torch.uint8, device=DEV)
    for b0 in range(0, B, 256):
        bn = min(256, B - b0)
        abi.check(lib.fa_blstm_forward_tc(xproj[b0 * T * U:].data_ptr(), head.w_hh_fwd, head.w_hh_bwd, bn, T * U, d, feat[b0 * T * U:].data_ptr(),
                                          scratch.data_ptr(), scratch.numel(), st), "fa_blstm_forward_tc")
    lens_up = (lens * U).to(torch.int32)
    us_a, us_p = torch.empty(B, T * U, device=DEV), torch.empty(B, T * U, device=DEV)
    abi.check(lib.fa_cif_upsample_alphas(feat.data_ptr(), 2 * d, head.out2_w, head.out2_b, lens_up.data_ptr(), tok.data_ptr(), B, T * U, head.smooth2,
                                         head.noise2, head.threshold, us_a.data_ptr(), us_p.data_ptr(), st), "fa_cif_upsample_alphas")
    return us_a, us_p


@pytest.mark.parametrize("mode", ["fp32", "fp16", "fp16x3", "fp16x6"])
@pytest.mark.parametrize("kind", ["bicif", "aligner"])
def test_timestamp_head_entry_is_the_composed_sequence(kind, mode):
    """fa_timestamp_head_forward (through the engine's upsample_timestamp) gives bit for bit what the composed public entries give,
    at D 512 (BiCif) and 320 (the aligner), B = 300 so that the recurrence runs as a 256- and a 44-sequence launch; the entry counts
    exactly one launch more (lens x U, which the composition does in torch)."""
    from funasr_b200 import synth
    from funasr_b200.engine import AlignerEngine, ParaformerEngine
    abi, lib = _lib()
    if kind == "aligner":
        eng = AlignerEngine(synth.make_aligner_state_dict(synth.ALIGNER_TINY, 3), synth.ALIGNER_TINY, DEV, gemm_mode=mode)
    else:
        eng = ParaformerEngine(synth.make_bicif_state_dict(synth.PARAFORMER_TINY, 3), synth.PARAFORMER_TINY, DEV, gemm_mode=mode, bicif=True)
    g = torch.Generator(device=DEV).manual_seed(21)
    B, T, d = 300, 7, eng.cfg.d_model
    enc = torch.randn(B, T, d, generator=g, device=DEV)
    lens = torch.randint(1, T + 1, (B,), generator=g, device=DEV, dtype=torch.int32)
    lens[::5] = T
    tok = torch.randint(0, 6, (B,), generator=g, device=DEV, dtype=torch.int32)
    n0 = lib.fa_launch_count()
    us_a, us_p = eng.upsample_timestamp(enc, lens, tok)
    n1 = lib.fa_launch_count()
    ref_a, ref_p = _head_composed(abi, lib, eng.ts_head, eng.mode, enc, lens, tok)
    n2 = lib.fa_launch_count()
    torch.cuda.synchronize()
    assert torch.equal(_bits(us_a), _bits(ref_a)) and torch.equal(_bits(us_p), _bits(ref_p))
    assert float(us_p.sum()) > 0
    assert n1 - n0 == n2 - n1 + 1


# ============================================================================================== arg-max / log-softmax
ARGMAX_MODES = ["fp32", "fp16x3", "fp16"]
VOCABS = [1, 5, 9216, 9217, 25055, 28672, 28673, 61440]
K_IN = 512
TOP = 2.0 ** -6                 # the designed maximum; one ulp below it is 2^-30, far below half an ulp of any log-sum >= log 2
# |logp - float64 log_softmax of the same fp32 logits| / max |logp| of the row.  The ids follow torch's fp32 CPU log_softmax (the
# reference's rule), but its values are no yardstick at this bar: at V = 25055 with many comparable terms, its fp32 sum of
# exponentials puts it 1.6e-6 of max |logp| from float64, while the kernel's shorter, blocked sum stays within that of float64.
# Measured on an H100: worst 8.8e-8 over every vocabulary and mode here, 3.5e-8 in the CTC test.
LOGP_TOL = 1e-6


def _onehot_linear(abi, lib, mode, V, bias):
    """W[v] = e_(v mod 512): logits[r, v] = x[r, v mod 512] (+ the epilogue's scale in tensor-core modes) + b[v]."""
    W = torch.zeros(V, K_IN, device=DEV)
    W[torch.arange(V, device=DEV), torch.arange(V, device=DEV) % K_IN] = 1.0
    bd = bias.to(DEV).contiguous()
    keep = [W, bd]
    planes = None
    if mode != "fp32":
        planes, _ = _planes(lib, abi, W)
        keep.append(planes)
    return abi.FaLinear(W.data_ptr(), bd.data_ptr(), planes.data_ptr() if planes is not None else None, V, K_IN, K_IN, 0), keep


def _fp16_grid(g, shape, lo, hi, step=1.0 / 16):
    """Random values on a grid of `step` in [lo, hi]: exact in fp16 and in the fp16 planes of every mode."""
    n = int(round((hi - lo) / step))
    return lo + torch.randint(0, n + 1, shape, generator=g).float() * step


def _argmax_design(V, kind, g, rows=8):
    """-> (x [rows, 512], b [V], expected id per row or -1).  The designed entries sit in columns whose activation is 0, so their
    logits are the bias exactly in every mode; every other column is pushed down by a random negative activation.
      'near': b[j] = TOP at j = V - 1 and b[i] = TOP - 2^-30 at i = V // 3 < j — both log-probs round to the same value, so the
              lower index wins although it is not the strict maximum;
      'tie' : b[t1] = b[t2] = TOP (t1 = V // 4 < t2 = V - 2), an exact tie: the lower index wins;
      'wide': generic rows, half of them with a huge dynamic range (one class at +30000, the rest at -30000).  b = 0, so equal
              activations give exactly tied logits and unequal ones differ by far more than an ulp of the log-sum, also after the
              tensor-core epilogue's scale."""
    b = _fp16_grid(g, (V,), -6.0, -2.0)
    x = -_fp16_grid(g, (rows, K_IN), 0.0, 4.0)
    want = [-1] * rows
    if kind == "wide":
        x = _fp16_grid(g, (rows, K_IN), -3.0, 3.0)
        for r in range(0, rows, 2):
            x[r] = -30000.0
            x[r, (r * 37) % K_IN] = 30000.0
        return x, torch.zeros(V), want
    if V < 3:
        b[0] = TOP
        return x, b, [0] * rows
    i, j = (V // 3, V - 1) if kind == "near" else (V // 4, V - 2)
    b[i], b[j] = (TOP - 2.0 ** -30, TOP) if kind == "near" else (TOP, TOP)
    for v in (i, j):
        x[:, v % K_IN] = 0.0
        members = torch.arange(v % K_IN, V, K_IN)
        b[members[(members != i) & (members != j)]] = -8.0                  # the rest of those classes stays far below
    return x, b, [i] * rows


def _run_linear_argmax(abi, lib, lin, mode, a, b2, V, want_logp, logp_offset=0):
    rows = a.shape[0]
    m = abi.GEMM_MODES[mode]
    ids = torch.full((rows,), -9, dtype=torch.int32, device=DEV)
    best = torch.full((rows,), float("nan"), device=DEV)
    lp_buf = torch.full((rows * V + logp_offset,), float("nan"), device=DEV) if want_logp else None
    ws = torch.empty(int(lib.fa_linear_argmax_workspace_bytes(rows, V, m)), dtype=torch.uint8, device=DEV)
    ad = a.to(DEV).contiguous()
    bd = b2.to(DEV).contiguous() if b2 is not None else None
    st = lib.fa_linear_argmax(C.byref(lin), ad.data_ptr(), bd.data_ptr() if bd is not None else None, rows, ids.data_ptr(),
                              best.data_ptr(), lp_buf.data_ptr() + 4 * logp_offset if want_logp else None, m, ws.data_ptr(),
                              ws.numel(), _st())
    torch.cuda.synchronize()
    logp = lp_buf[logp_offset:].view(rows, V).cpu() if want_logp else None
    return st, ids.cpu(), best.cpu(), logp


def _gpu_logits(abi, lib, lin, mode, x, V):
    """The GEMM fa_linear_argmax runs, called on its own: its logits, bit for bit."""
    rows = x.shape[0]
    m = abi.GEMM_MODES[mode]
    y = torch.empty(rows, V, device=DEV)
    ws = torch.empty(int(lib.fa_linear_argmax_workspace_bytes(rows, V, m)), dtype=torch.uint8, device=DEV)
    xd = x.to(DEV).contiguous()
    abi.check(lib.fa_linear(xd.data_ptr(), K_IN, rows, C.byref(lin), 0, None, 0, None, 0, y.data_ptr(), V, m, ws.data_ptr(),
                            ws.numel(), _st()), "fa_linear")
    torch.cuda.synchronize()
    return y.cpu()


@pytest.mark.parametrize("mode", ARGMAX_MODES)
@pytest.mark.parametrize("V", VOCABS)
def test_linear_argmax_ties_and_tiers(V, mode):
    """fa_linear_argmax over the three register tiers of argmax_lse_kernel (<= 9216, <= 28672, <= 61440) and their boundaries,
    odd vocabularies (scalar loads) beside multiples of 4 (float4 loads): ids equal torch.log_softmax(logits, -1).argmax(-1) on
    the CPU (lowest index among equal rounded log-probs, the reference's rule), best_logp and the full log-softmax within LOGP_TOL
    of max |logp| of the float64 log-softmax.  The 'wide' rows go through the a + b input path."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(V)
    worst = 0.0
    for kind, want_logp in (("near", False), ("tie", True), ("wide", True)):
        x, b, want = _argmax_design(V, kind, g)
        lin, keep = _onehot_linear(abi, lib, mode, V, b)
        if kind == "wide":                                          # a + b with an exact fp32 sum: the GEMM sees x
            b2 = _fp16_grid(g, x.shape, -1.0, 1.0)
            a, b2 = x - b2, b2
            assert torch.equal(a + b2, x)
        else:
            a, b2 = x, None
        st, ids, best, logp = _run_linear_argmax(abi, lib, lin, mode, a, b2, V, want_logp)
        assert st == 0, st
        logits = _gpu_logits(abi, lib, lin, mode, x, V)
        if mode == "fp32":                                          # the one-hot GEMM is exact here: logits = fp32(x + b)
            assert torch.equal(logits, x[:, torch.arange(V) % K_IN] + b)
        ref_ids = torch.log_softmax(logits, -1).argmax(-1).to(torch.int32)
        for r, w in enumerate(want):                                # the design really produces its tie / near-tie
            if w >= 0:
                assert int(ref_ids[r]) == w, (kind, r)
        assert torch.equal(ids, ref_ids), (kind, ids.tolist(), ref_ids.tolist())
        ref_lp = torch.log_softmax(logits.double(), -1)
        scale = ref_lp.abs().amax(-1).clamp_min(1e-30)                       # per row: max |logp|
        err = float(((best.double() - ref_lp.gather(1, ref_ids.long()[:, None])[:, 0]).abs() / scale).max())
        if logp is not None:
            err = max(err, float(((logp.double() - ref_lp).abs().amax(-1) / scale).max()))
        worst = max(worst, err)
        assert err <= LOGP_TOL, (kind, err)
    print("linear_argmax V=%d %s: logp err %.2e of max |logp|" % (V, mode, worst))


def test_linear_argmax_vector_and_scalar_paths_agree():
    """The same logits through the aligned float4 path and, with the output pointer one float off, the scalar path (fp32 mode: the
    SIMT GEMM takes any alignment): identical ids, best_logp and log-softmax."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(17)
    for V in (9216, 28672, 61440):
        x, b, _ = _argmax_design(V, "near", g)
        lin, keep = _onehot_linear(abi, lib, "fp32", V, b)
        r0 = _run_linear_argmax(abi, lib, lin, "fp32", x, None, V, True, 0)
        r1 = _run_linear_argmax(abi, lib, lin, "fp32", x, None, V, True, 1)
        assert r0[0] == 0 and r1[0] == 0
        assert torch.equal(r0[1], r1[1]) and torch.equal(_bits(r0[2]), _bits(r1[2])) and torch.equal(_bits(r0[3]), _bits(r1[3]))


def test_linear_argmax_vocab_limit():
    abi, lib = _lib()
    g = torch.Generator().manual_seed(1)
    V = 61441
    lin, keep = _onehot_linear(abi, lib, "fp16x3", V, _fp16_grid(g, (V,), -1.0, 1.0))
    st, *_ = _run_linear_argmax(abi, lib, lin, "fp16x3", _fp16_grid(g, (4, K_IN), -1.0, 1.0), None, V, False)
    assert st == -4


# ============================================================================================== CTC head and greedy filter
CTC_V = 25055


def _ctc_classes():
    """One candidate id per activation class c: cand[c] = c + 512 * (7 c mod 48) spreads them over [0, 24576); cand[0] = 0 is blank."""
    c = torch.arange(K_IN)
    return c + K_IN * ((7 * c) % 48)


def _ctc_design(t_max, g):
    """Designed per-frame classes [B, t_max] and lens: all blank, repeats, repeats across a blank, random over a small alphabet
    (blank frequent); lens 0, 1, t_max, t_max - 1 and t_max + 3 (clamped to t_max)."""
    alphabet = torch.tensor([0, 0, 1, 2, 3, 100, 511])
    rep = [5, 5, 5, 7, 7, 0, 0, 3, 0, 3, 3, 0, 0, 0, 5]
    across = [9, 0, 9, 0, 0, 9, 9, 0, 4]
    rows = [torch.zeros(t_max, dtype=torch.long),
            torch.tensor([rep[i % len(rep)] for i in range(t_max)]),
            torch.tensor([across[i % len(across)] for i in range(t_max)])]
    rows += [alphabet[torch.randint(0, len(alphabet), (t_max,), generator=g)] for _ in range(4)]
    lens = [t_max, t_max, t_max, 0, 1, max(t_max - 1, 0), t_max + 3]
    return torch.stack(rows), lens


@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("t_max", [1, 31, 32, 33, 500])
def test_ctc_greedy_designed_frames(t_max, mode):
    """fa_ctc_greedy_forward with a one-hot projection whose per-frame arg-max is designed: argmax_ids equal the design on every
    frame (padding included), out_ids / out_lens equal torch.unique_consecutive with blank dropped, padded with -1.  t_max around
    32 crosses the filter's ballot boundary.  With a log-prob buffer the logits rows are dense (V = 25055, scalar loads), without
    one they are pitched to 25056 (float4 loads): both give the same ids."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(t_max)
    cand = _ctc_classes()
    bias = torch.full((CTC_V,), -1.0)
    bias[cand] = 0.0
    lin, keep = _onehot_linear(abi, lib, mode, CTC_V, bias)
    cls, lens = _ctc_design(t_max, g)
    B = cls.shape[0]
    enc = torch.zeros(B, t_max, K_IN)
    enc.scatter_(2, cls[..., None], 4.0)
    design = cand[cls].to(torch.int32)
    m = abi.GEMM_MODES[mode]
    encd, lensd = enc.to(DEV), torch.tensor(lens, dtype=torch.int32, device=DEV)
    ws = torch.empty(int(lib.fa_ctc_greedy_workspace_bytes(B, t_max, CTC_V, m)), dtype=torch.uint8, device=DEV)
    results = []
    for with_logp in (True, False):
        am = torch.full((B, t_max), -9, dtype=torch.int32, device=DEV)
        out_ids = torch.full((B, t_max), 7777, dtype=torch.int32, device=DEV)
        out_lens = torch.full((B,), -9, dtype=torch.int32, device=DEV)
        logp = torch.full((B, t_max, CTC_V), float("nan"), device=DEV) if with_logp else None
        abi.check(lib.fa_ctc_greedy_forward(C.byref(lin), encd.data_ptr(), lensd.data_ptr(), B, t_max, 0, am.data_ptr(), out_ids.data_ptr(),
                                            out_lens.data_ptr(), logp.data_ptr() if with_logp else None, m, ws.data_ptr(), ws.numel(), _st()),
                  "fa_ctc_greedy_forward")
        torch.cuda.synchronize()
        results.append((am.cpu(), out_ids.cpu(), out_lens.cpu()))
        if with_logp:
            logits = _gpu_logits(abi, lib, lin, mode, enc.view(B * t_max, K_IN), CTC_V)
            ref_lp = torch.log_softmax(logits.double(), -1)
            err = float((logp.cpu().view(-1, CTC_V).double() - ref_lp).abs().max() / ref_lp.abs().max())
            print("ctc t_max=%d %s: logp err %.2e of max |logp|" % (t_max, mode, err))
            assert err <= LOGP_TOL, err
    assert torch.equal(results[0][0], results[1][0]) and torch.equal(results[0][1], results[1][1])
    am, out_ids, out_lens = results[0]
    assert torch.equal(am, design)
    for b in range(B):
        seq = torch.unique_consecutive(design[b, :min(lens[b], t_max)])
        seq = seq[seq != 0].tolist()
        assert int(out_lens[b]) == len(seq), b
        assert out_ids[b, :len(seq)].tolist() == seq, b
        assert bool((out_ids[b, len(seq):] == -1).all()), b


@pytest.mark.parametrize("n_max", [1, 32, 33, 501])
def test_greedy_filter(n_max):
    """fa_greedy_filter on ids in [0, 10) (blank 0, sos 1, eos 2 frequent) with tok_lens 0, 1, n_max, beyond n_max and random:
    the reference's filter of yseq[:tok_len] (paraformer/model.py:655-666), padded with -1."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(n_max)
    lens = [0, 1, n_max, n_max + 5, max(n_max - 1, 0)] + torch.randint(0, n_max + 1, (4,), generator=g).tolist()
    B = len(lens)
    ids = torch.randint(0, 10, (B, n_max), generator=g, dtype=torch.int32)
    out_ids = torch.full((B, n_max), 7777, dtype=torch.int32, device=DEV)
    out_lens = torch.full((B,), -9, dtype=torch.int32, device=DEV)
    idsd, lensd = ids.to(DEV), torch.tensor(lens, dtype=torch.int32, device=DEV)
    abi.check(lib.fa_greedy_filter(idsd.data_ptr(), lensd.data_ptr(), B, n_max, 1, 2, 0, out_ids.data_ptr(), out_lens.data_ptr(), _st()),
              "fa_greedy_filter")
    torch.cuda.synchronize()
    out_ids, out_lens = out_ids.cpu(), out_lens.cpu()
    for b in range(B):
        keep = [x for x in ids[b, :lens[b]].tolist() if x not in (0, 1, 2)]
        assert int(out_lens[b]) == len(keep), b
        assert out_ids[b].tolist() == keep + [-1] * (n_max - len(keep)), b


# ============================================================================================== SeACo merge
def test_seaco_merge():
    """Per row the decoder's arg-max, its log-prob and its log-prob row where the hotword decoder's arg-max is NO_BIAS, else the
    hotword decoder's: merged rows are bit-identical copies of the chosen source (seaco_weight = 1)."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(6)
    rows, V, no_bias = 300, 8405, 8377
    dec_ids = torch.randint(0, V, (rows,), generator=g, dtype=torch.int32)
    dha_ids = torch.randint(0, V, (rows,), generator=g, dtype=torch.int32)
    dha_ids[torch.rand(rows, generator=g) < 0.5] = no_bias
    dha_ids[:2] = torch.tensor([no_bias, 3], dtype=torch.int32)
    dec_best, dha_best = -torch.rand(rows, generator=g) * 5, -torch.rand(rows, generator=g) * 5
    dec_lp, dha_lp = -torch.rand(rows, V, generator=g) * 20, -torch.rand(rows, V, generator=g) * 20
    dec_lp[:, 0], dha_lp[:, 1] = -0.0, -0.0
    dev = [t.to(DEV) for t in (dec_ids, dec_best, dha_ids, dha_best, dec_lp, dha_lp)]
    keep_dec = dha_ids == no_bias
    for with_rows in (True, False):
        out_ids = torch.full((rows,), -9, dtype=torch.int32, device=DEV)
        out_best = torch.full((rows,), float("nan"), device=DEV)
        merged = torch.full((rows, V), float("nan"), device=DEV) if with_rows else None
        abi.check(lib.fa_seaco_merge(dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(), dev[3].data_ptr(), rows, no_bias,
                                     out_ids.data_ptr(), out_best.data_ptr(), dev[4].data_ptr(), dev[5].data_ptr(),
                                     merged.data_ptr() if with_rows else None, V, _st()), "fa_seaco_merge")
        torch.cuda.synchronize()
        assert torch.equal(out_ids.cpu(), torch.where(keep_dec, dec_ids, dha_ids))
        assert torch.equal(_bits(out_best.cpu()), _bits(torch.where(keep_dec, dec_best, dha_best)))
        if with_rows:
            assert torch.equal(_bits(merged.cpu()), _bits(torch.where(keep_dec[:, None], dec_lp, dha_lp)))
    out = torch.empty(rows, dtype=torch.int32, device=DEV)
    assert lib.fa_seaco_merge(dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(), dev[3].data_ptr(), rows, no_bias, out.data_ptr(),
                              out.data_ptr(), None, dev[5].data_ptr(), out.data_ptr(), V, _st()) == -1
    assert lib.fa_seaco_merge(dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(), dev[3].data_ptr(), 0, no_bias, out.data_ptr(),
                              out.data_ptr(), None, None, None, V, _st()) == 0
    torch.cuda.synchronize()
