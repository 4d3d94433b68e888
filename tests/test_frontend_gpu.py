"""GPU (-m gpu): kernel-level parity of the frontend kernels — the fused Fbank + LFR + CMVN kernel in its three instantiations
(7/6 for Paraformer and SenseVoice, 5/1 for the FSMN-VAD, 1/1 for CAM++), the short-utterance Fbank, CAM++'s per-utterance mean
subtraction, the FSMN-VAD scorer and the frame energies — each against a float64 restatement of the same operation on the CPU.

The restatements live here: the oracles under oracle/ are fp32 and stay as they are.  tests/test_frontend_host.py holds them against
torchaudio's kaldi.fbank on float64 input and against the fp32 oracles, without a GPU.

Tolerances.  The log-mel bound is |d| <= 1e-5 + 1e-6 sqrt(E_frame_max / E_bin): the fp32 FFT leaves an absolute error of a few
ulp of the frame's largest amplitude in every bin, so a bin far below the frame's peak carries a relative error that grows as the
square root of the energy ratio (the bound between two fp32 FFTs in tests/conftest.py:knf_bound is four times this constant and
eight times this slope; one side is now exact).  Every test prints its worst ratio to its bound.  Measured on an H100 80GB HBM3
(700 W): worst ratio 0.31 for the batched kernel and mean |d log-mel| 1.0e-6 .. 2.0e-6, except the pure tones at 9.5e-6 — there most
mel bins sit 60 dB and more below the tone's band, so the sqrt term, not the constant, sets their error.
"""
import ctypes as C
import functools
import math

import numpy as np
import pytest
import torch

import paraformer_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
EPS = float(np.finfo(np.float32).eps)       # kaldi's energy floor: float32 epsilon, whatever the input dtype (kaldi.py:_get_epsilon)
U = 2.0 ** -24                              # unit roundoff of fp32
WIN, SHIFT = 400, 160
LFRS = [(7, 6), (5, 1)]


# ============================================================================================== float64 restatement
@functools.lru_cache(maxsize=None)
def mel_banks64(padded=512):
    """kaldi.get_mel_banks (paraformer_oracle.get_mel_banks) with the zero Nyquist column, as float64 [80, padded / 2 + 1].  torchaudio
    builds the filters in the default dtype and casts them to the input's dtype, so on float64 input it applies these fp32 values —
    the same ones the kernels get."""
    return np.pad(O.get_mel_banks(80, padded).double().numpy(), ((0, 0), (0, 1)))


def window64(kind, n):
    if kind == "hamming":
        return torch.hamming_window(n, periodic=False, alpha=0.54, beta=0.46, dtype=torch.float64).numpy()
    return torch.hann_window(n, periodic=False, dtype=torch.float64).pow(0.85).numpy()      # povey


def num_frames(n):
    return 1 + (n - WIN) // SHIFT if n >= WIN else 0


def fbank64(wav, window="hamming", scale=32768.0):
    """kaldi.fbank(wav * scale, 80 mel, 25 / 10 ms, snip_edges, dither 0, energy_floor 0) in float64 -> log-mel [frames, 80]: framing,
    DC offset removed, pre-emphasis 0.97 with the first sample replicated, window, 512-point rfft power, mel filters,
    log(max(e, eps_f32)).  Below one 400-sample window the utterance is ONE frame of all n samples with an FFT of the next power of
    two (wav_frontend.py:174 passes frame_length = min(25 ms, n / fs))."""
    x = np.asarray(wav, dtype=np.float64) * scale
    n = x.size
    win, m = (WIN, num_frames(n)) if n >= WIN else (n, 1)
    pad = 1 << (win - 1).bit_length()
    fr = np.lib.stride_tricks.sliding_window_view(x, win)[::SHIFT][:m]
    fr = fr - fr.mean(1, keepdims=True)
    prev = np.concatenate([fr[:, :1], fr[:, :-1]], 1)
    y = (fr - 0.97 * prev) * window64(window, win)
    power = np.abs(np.fft.rfft(y, n=pad)) ** 2
    return np.log(np.maximum(power @ mel_banks64(pad).T, EPS))


def lfr64(lm, m, n):
    """Low-frame-rate stacking as the clamped gather it is (wav_frontend.py:63-86): row i = frames n i - (m - 1) / 2 + j, j < m, clamped
    to [0, T - 1], for i < ceil(T / n)."""
    T = lm.shape[0]
    idx = np.clip(np.arange((T + n - 1) // n)[:, None] * n - (m - 1) // 2 + np.arange(m)[None, :], 0, T - 1)
    return lm[idx].reshape(idx.shape[0], -1)


def cmvn64(x, cmvn):
    c = np.asarray(cmvn, dtype=np.float64)
    return (x + c[0]) * c[1]


def logmel_bound(lm, c0=1e-5, c1=1e-6):
    """c0 + c1 sqrt(E_frame_max / E_bin) from float64 log-mel rows."""
    return c0 + c1 * np.exp(0.5 * (lm.max(-1, keepdims=True) - lm))


def vad_logits64(x, p):
    """FSMN.forward (fsmn_vad_streaming/encoder.py:355-377) in float64 up to the logits: in_linear1 -> in_linear2 -> ReLU ->
    4 x [linear (no bias) -> q + causal memory sum_k w[:, k] q[t - 19 + k] (zero before the first frame) -> affine -> ReLU] ->
    out_linear1 -> out_linear2."""
    w = {k: v.double().numpy() for k, v in p.items()}
    lin = lambda name, v, bias=True: v @ w[name + ".linear.weight"].T + (w[name + ".linear.bias"] if bias else 0.0)
    h = np.maximum(lin("encoder.in_linear2", lin("encoder.in_linear1", np.asarray(x, dtype=np.float64))), 0.0)
    i = 0
    while ("encoder.fsmn.%d.linear.linear.weight" % i) in w:
        pre = "encoder.fsmn.%d" % i
        q = lin(pre + ".linear", h, bias=False)
        cw = w[pre + ".fsmn_block.conv_left.weight"][:, 0, :, 0]                 # [128, lorder]; tap lorder - 1 = the current frame
        lo, T = cw.shape[1], q.shape[0]
        qp = np.concatenate([np.zeros((lo - 1, q.shape[1])), q])
        mem = sum(cw[:, k] * qp[k:k + T] for k in range(lo))
        h = np.maximum(lin(pre + ".affine", q + mem), 0.0)
        i += 1
    return lin("encoder.out_linear2", lin("encoder.out_linear1", h))


def softmax64(z):
    e = np.exp(z - z.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


# ============================================================================================== device helpers
def _lib():
    from funasr_b200 import _abi
    return _abi, _abi.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.fixture(scope="module")
def tables():
    """Device tables of both windows: hamming (ASR and VAD frontends) and povey (CAM++)."""
    from funasr_b200.campplus import povey_window
    from funasr_b200.engine import kaldi_mel_banks
    abi, lib = _lib()
    out = {}
    mel = kaldi_mel_banks().to(DEV)
    for kind, win in (("hamming", torch.hamming_window(400, periodic=False, alpha=0.54, beta=0.46)), ("povey", povey_window())):
        win = win.float().to(DEV).contiguous()
        t = torch.empty(int(lib.fa_fbank_tables_bytes()) // 4, dtype=torch.float32, device=DEV)
        abi.check(lib.fa_fbank_make_tables(mel.data_ptr(), win.data_ptr(), t.data_ptr(), _st()), "fa_fbank_make_tables")
        torch.cuda.synchronize()
        out[kind] = t
    return out


def _rows(n, lfr_n):
    return (num_frames(n) + lfr_n - 1) // lfr_n


def _padded(wavs):
    """[B, width] on the device, width = the longest utterance rounded up to a multiple of 4 (every row 16-byte aligned); lens int32."""
    lens = [len(w) for w in wavs]
    width = (max(lens) + 3) // 4 * 4
    buf = torch.zeros(len(wavs), width, dtype=torch.float32)
    for b, w in enumerate(wavs):
        buf[b, :len(w)] = torch.as_tensor(np.asarray(w, dtype=np.float32))
    return buf.to(DEV), torch.tensor(lens, dtype=torch.int32, device=DEV)


def _fbank_call(lib, tab, wav_ptr, lens, wav_stride, lfr, cmvn, feats_ptr, stride_rows, t_max):
    B = lens.numel()
    flens = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    st = lib.fa_fbank_lfr_cmvn_tables(wav_ptr, lens.data_ptr(), B, wav_stride, _ptr(cmvn), tab.data_ptr(), lfr[0], lfr[1], feats_ptr,
                                      stride_rows, flens.data_ptr(), t_max, _st())
    assert st == 0, st
    return flens


def _fbank(tab, wavs, lfr, cmvn=None, t_max=None):
    """Compact run: feats [B, t_max, 80 lfr_m] (NaN beforehand, so an unwritten element shows), feat_lens."""
    abi, lib = _lib()
    wav, lens = _padded(wavs)
    t_max = t_max or max(_rows(len(w), lfr[1]) for w in wavs)
    feats = torch.full((len(wavs), t_max, 80 * lfr[0]), float("nan"), device=DEV)
    flens = _fbank_call(lib, tab, wav.data_ptr(), lens, wav.stride(0), lfr, cmvn, feats.data_ptr(), t_max, t_max)
    torch.cuda.synchronize()
    return feats, flens


def _cmvn(lfr_m, seed=1):
    from funasr_b200 import synth
    if lfr_m == 5:
        return synth.make_vad_cmvn(seed)
    return synth.make_cmvn(synth.PARAFORMER_TINY, seed)


def _check_features(tag, feats, flens, wavs, lfr, cmvn, window="hamming", scale=32768.0, mean_bound=1e-5):
    """Every utterance against the float64 restatement: |d| <= |cmvn scale| * logmel_bound + 2u |feature| (the fp32 add and multiply of
    the CMVN step each round once), mean |d| / |cmvn scale| <= 1e-5; feature lengths and padding rows exact."""
    feats = feats.cpu().numpy()
    scl = np.ones(80 * lfr[0]) if cmvn is None else np.abs(cmvn[1].double().numpy())
    worst, worst_at, d_sum, d_cnt = 0.0, None, 0.0, 0
    for b, w in enumerate(wavs):
        lm = fbank64(w, window, scale)
        want = lfr64(lm, *lfr)
        bound = lfr64(logmel_bound(lm), *lfr)
        if cmvn is not None:
            want = cmvn64(want, cmvn)
        t = want.shape[0]
        assert int(flens[b]) == t, (tag, b, int(flens[b]), t)
        got = feats[b, :t].astype(np.float64)
        assert np.isfinite(got).all(), (tag, b)
        d = np.abs(got - want)
        r = d / (scl * bound + 2 * U * np.abs(want))
        if r.max() > worst:
            worst, worst_at = float(r.max()), (b, len(w)) + np.unravel_index(int(r.argmax()), r.shape)
        d_sum += float((d / scl).sum())
        d_cnt += d.size
        assert (feats[b, t:] == 0).all() and not np.signbit(feats[b, t:]).any(), (tag, b)      # padding rows: +0.0 exactly
    mean = d_sum / d_cnt
    print("%s: worst |d| / bound %.3f at (utt, n, row, col) %s, mean |d log-mel| %.2e (bound %.0e)" % (tag, worst, worst_at, mean, mean_bound))
    assert worst <= 1.0 and mean <= mean_bound


# ============================================================================================== Fbank + LFR + CMVN
def _n(frames, extra=0):
    return WIN + SHIFT * (frames - 1) + extra


# frame count changes at 400 / 560; LFR-7/6 row counts change at frame counts = 1 and 5 mod 6 (47 -> 8 rows, 48 -> 8, 49 -> 9, 96 -> 16,
# 97 -> 17, 101 -> 17); CTA edges at 8 / 9 / 16 / 17 rows (7/6) and 44 / 45 / 88 / 89 rows (5/1)
BOUNDARY_LENS = [400, 559, 560, 561, _n(5), _n(6, 159), _n(7, 1), _n(44), _n(45, 80), _n(47), _n(48, 159), _n(49), _n(88, 3), _n(89),
                 _n(96), _n(97, 17), _n(101)]
SIGNALS = ["speech", "noise", "impulse", "square", "tiny", "zeros", "const"]


def _signal(kind, n, seed):
    from funasr_b200 import synth
    if kind in ("speech", "noise"):
        return synth.make_wav(n, seed, "speechlike" if kind == "speech" else "noise").numpy()
    i = np.arange(n)
    if kind == "impulse":
        x = np.zeros(n)
        x[(3 * n) // 7] = 1.0
    elif kind == "square":                                      # full scale, 400 Hz
        x = np.where((i // 20) % 2 == 0, 1.0, -1.0)
    elif kind == "tiny":                                        # amplitude 1e-7: mel energies down towards the eps floor
        x = 1e-7 * np.random.default_rng(seed).standard_normal(n)
    elif kind == "zeros":
        x = np.zeros(n)
    else:                                                       # "const": DC removal leaves exactly zero
        x = np.full(n, 0.25)
    return x.astype(np.float32)


@pytest.mark.parametrize("cmvn_on", [False, True])
@pytest.mark.parametrize("lfr", LFRS)
@pytest.mark.parametrize("kind", SIGNALS)
def test_fbank_lfr_cmvn_vs_float64(tables, kind, lfr, cmvn_on):
    """fa_fbank_lfr_cmvn_tables against the float64 Fbank, LFR gather and CMVN, in one ragged batch over the lengths where the frame
    count, the LFR row count and the CTA tiling change."""
    cmvn = _cmvn(lfr[0]) if cmvn_on else None
    wavs = [_signal(kind, n, 100 + i) for i, n in enumerate(BOUNDARY_LENS)]
    feats, flens = _fbank(tables["hamming"], wavs, lfr, None if cmvn is None else cmvn.to(DEV))
    _check_features("fbank %s lfr %d/%d cmvn %s" % (kind, lfr[0], lfr[1], cmvn_on), feats, flens, wavs, lfr, cmvn)


TONE_BINS = [1, 2, 3, 5, 8, 16, 31, 32, 33, 63, 64, 65, 96, 127, 128, 129, 160, 192, 200, 223, 224, 240, 254, 255]


@pytest.mark.parametrize("lfr", LFRS)
def test_fbank_pure_tones_at_bin_centres_vs_float64(tables, lfr):
    """Tones at exact bin centres k * 31.25 Hz: all of a frame's energy sits in one bin of the 512-point transform (plus the window's
    leakage), so a wrong twiddle or bit-reversal index for one k moves a whole mel band, which broadband noise would average away."""
    n = _n(49)
    i = np.arange(n)
    wavs = [(0.5 * np.cos(2 * math.pi * k * i / 512.0 + 0.1 * k)).astype(np.float32) for k in TONE_BINS]
    feats, flens = _fbank(tables["hamming"], wavs, lfr)
    _check_features("tones lfr %d/%d" % lfr, feats, flens, wavs, lfr, None)


@pytest.mark.parametrize("lfr", LFRS)
def test_fbank_long_utterance_vs_float64(tables, lfr):
    """A 30 s utterance (2998 frames: 500 LFR-7/6 rows over 63 CTAs, 2998 LFR-5/1 rows over 69) beside a two-frame one."""
    from funasr_b200 import synth
    wavs = [synth.make_wav(480000, 7, "speechlike").numpy(), _signal("noise", 561, 8)]
    cmvn = _cmvn(lfr[0])
    feats, flens = _fbank(tables["hamming"], wavs, lfr, cmvn.to(DEV))
    _check_features("long lfr %d/%d" % lfr, feats, flens, wavs, lfr, cmvn)


@pytest.mark.parametrize("lfr", LFRS)
def test_fbank_constant_input_sits_on_the_log_floor(tables, lfr):
    """A constant 0.25 (8192 after the x32768 scale) has an exact frame mean, so after the DC removal the frame is exactly zero and every
    log-mel value is the floor the kernel writes for zero energy, __logf(eps), bit for bit — the value an all-zero waveform gives,
    whose frames are zero without any arithmetic.  Any other value means a non-zero residue reached the FFT.  That floor is within
    __logf's 2 ulp of log(eps) (measured on an H100 80GB HBM3 at 700 W: 1.45 ulp, the same for both signals)."""
    wavs = [_signal("const", n, 0) for n in BOUNDARY_LENS]
    feats, flens = _fbank(tables["hamming"], wavs, lfr)
    zeros, zlens = _fbank(tables["hamming"], [_signal("zeros", n, 0) for n in BOUNDARY_LENS], lfr)
    assert torch.equal(flens, zlens)
    floor = math.log(EPS)
    ulp = float(np.spacing(np.float32(abs(floor))))
    for b, n in enumerate(BOUNDARY_LENS):
        t = _rows(n, lfr[1])
        assert int(flens[b]) == t
        assert torch.equal(_bits(feats[b, :t]), _bits(zeros[b, :t])), b
    values = torch.unique(zeros[:, :1]).cpu().double()
    assert values.numel() == 1
    off = abs(float(values[0]) - floor)
    print("constant lfr %d/%d: every value on the zero-energy floor, %.2e (%.2f ulp) from log(eps)" % (lfr + (off, off / ulp)))
    assert off <= 2 * ulp


# ============================================================================================== layout and load paths, bit for bit
LAYOUT_LENS = [_n(49), _n(9, 77), _n(97, 1), 561, _n(17, 3)]


@pytest.mark.parametrize("lfr", LFRS)
def test_fbank_scalar_and_vector_loads_agree(tables, lfr):
    """A frame is loaded with 8-byte loads when its utterance starts 8-byte aligned and with scalar loads otherwise.  With an odd
    wav_stride every other utterance starts misaligned, and a base pointer one float further swaps which ones, so each utterance
    takes the scalar path in one of the two runs: both must equal the aligned layout bit for bit.  FrontendEngine passes
    wav.stride(0) through, so a padded batch whose longest utterance has an odd length runs this path too."""
    from funasr_b200.engine import FrontendEngine
    abi, lib = _lib()
    tab = tables["hamming"]
    cmvn = _cmvn(lfr[0]).to(DEV)
    wavs = [_signal("speech", n, 40 + i) for i, n in enumerate(LAYOUT_LENS)]
    ref, ref_lens = _fbank(tab, wavs, lfr, cmvn)
    B, t_max, S = len(wavs), ref.shape[1], (max(LAYOUT_LENS) + 2) | 1                     # odd stride
    for off in (0, 1):
        flat = torch.zeros(off + B * S + 8, dtype=torch.float32)
        for b, w in enumerate(wavs):
            flat[off + b * S: off + b * S + len(w)] = torch.as_tensor(w)
        flat = flat.to(DEV)
        _, lens = _padded(wavs)
        feats = torch.full_like(ref, float("nan"))
        flens = _fbank_call(lib, tab, flat.data_ptr() + 4 * off, lens, S, lfr, cmvn, feats.data_ptr(), t_max, t_max)
        torch.cuda.synchronize()
        assert torch.equal(flens, ref_lens)
        assert torch.equal(_bits(feats), _bits(ref)), off
    # the engine on a padded batch of odd width
    odd = wavs + [_signal("noise", _n(98, 2) + 1, 9)]
    assert len(odd[-1]) % 2 == 1 and len(odd[-1]) == max(len(w) for w in odd)
    pad = torch.nn.utils.rnn.pad_sequence([torch.as_tensor(w) for w in odd], batch_first=True).to(DEV)
    assert pad.stride(0) % 2 == 1
    fe = FrontendEngine(cmvn, DEV, lfr_m=lfr[0], lfr_n=lfr[1])
    t_odd = max(_rows(len(w), lfr[1]) for w in odd)
    got, got_lens = fe(pad, torch.tensor([len(w) for w in odd], dtype=torch.int32, device=DEV), t_odd)
    want, want_lens = _fbank(tab, odd, lfr, cmvn)
    torch.cuda.synchronize()
    assert torch.equal(got_lens, want_lens) and torch.equal(_bits(got), _bits(want))


@pytest.mark.parametrize("lfr", LFRS)
def test_fbank_batch_composition_is_bit_exact(tables, lfr):
    """A CTA owns rows of one utterance, so an utterance's features cannot depend on its neighbours: each utterance alone equals the same
    utterance inside the ragged batch, bit for bit, and the batch's rows past its length are zero."""
    tab = tables["hamming"]
    cmvn = _cmvn(lfr[0]).to(DEV)
    wavs = [_signal("speech" if i % 2 else "noise", n, 60 + i) for i, n in enumerate(LAYOUT_LENS)]
    full, flens = _fbank(tab, wavs, lfr, cmvn)
    for b, w in enumerate(wavs):
        one, one_lens = _fbank(tab, [w], lfr, cmvn)
        t = int(one_lens[0])
        assert t == int(flens[b]) == one.shape[1]
        assert torch.equal(_bits(one[0]), _bits(full[b, :t])), b
        assert torch.equal(_bits(full[b, t:]), torch.zeros_like(_bits(full[b, t:]))), b


@pytest.mark.parametrize("lfr", LFRS)
def test_fbank_t_max_below_an_utterance_truncates_it(tables, lfr):
    """t_max below an utterance's row count: the kernel writes its first t_max rows — the same values as an untruncated run, since a
    CTA's frames are clamped to the utterance, not to t_max — and nothing after feats [B, t_max, F].  feat_lens still reports the
    utterance's full row count (the caller learns that the utterance did not fit)."""
    abi, lib = _lib()
    tab = tables["hamming"]
    cmvn = _cmvn(lfr[0]).to(DEV)
    wavs = [_signal("speech", n, 70 + i) for i, n in enumerate(LAYOUT_LENS)]
    full, full_lens = _fbank(tab, wavs, lfr, cmvn)
    t_max = 12 if lfr == (7, 6) else 60
    rows = [_rows(len(w), lfr[1]) for w in wavs]
    assert min(rows) < t_max < max(rows)
    B, F = len(wavs), 80 * lfr[0]
    slack = 3 * F
    sentinel = -1234.5
    buf = torch.full((B * t_max * F + slack,), sentinel, device=DEV)
    wav, lens = _padded(wavs)
    flens = _fbank_call(lib, tab, wav.data_ptr(), lens, wav.stride(0), lfr, cmvn, buf.data_ptr(), t_max, t_max)
    torch.cuda.synchronize()
    assert flens.tolist() == full_lens.tolist() == rows
    feats = buf[:B * t_max * F].view(B, t_max, F)
    for b in range(B):
        k = min(rows[b], t_max)
        assert torch.equal(_bits(feats[b, :k]), _bits(full[b, :k])), b
        assert (feats[b, k:] == 0).all(), b
    assert (buf[B * t_max * F:] == sentinel).all()


@pytest.mark.parametrize("lfr", LFRS)
def test_fbank_strided_output_and_broadcast_rows(tables, lfr):
    """SenseVoice's forward_wav layout: utterance b's features start at row 4 of a block of t_max + 4 rows (feats_batch_stride_rows =
    t_max + 4, base at row 4), then fa_broadcast_rows writes the 4 query rows in front of every utterance.  With the whole buffer set to
    a sentinel first, the feature call leaves the 4 prefix rows and everything past the last utterance untouched and writes exactly the
    compact run's values; the broadcast then fills exactly the prefix rows."""
    abi, lib = _lib()
    tab = tables["hamming"]
    cmvn = _cmvn(lfr[0]).to(DEV)
    wavs = [_signal("speech", n, 80 + i) for i, n in enumerate(LAYOUT_LENS)]
    ref, ref_lens = _fbank(tab, wavs, lfr, cmvn)
    B, t_max, F = ref.shape
    P, sentinel = 4, -777.25
    blk = torch.full((B * (t_max + P) + 2, F), sentinel, device=DEV)          # 2 guard rows after the last utterance
    wav, lens = _padded(wavs)
    flens = _fbank_call(lib, tab, wav.data_ptr(), lens, wav.stride(0), lfr, cmvn, blk.data_ptr() + P * F * 4, t_max + P, t_max)
    torch.cuda.synchronize()
    assert torch.equal(flens, ref_lens)
    x = blk[:B * (t_max + P)].view(B, t_max + P, F)
    assert (x[:, :P] == sentinel).all()
    assert torch.equal(_bits(x[:, P:]), _bits(ref))
    assert (blk[B * (t_max + P):] == sentinel).all()
    before = blk.clone()
    q = torch.randn(P, F, generator=torch.Generator().manual_seed(3)).to(DEV)
    assert lib.fa_broadcast_rows(q.data_ptr(), P, F, blk.data_ptr(), t_max + P, B, _st()) == 0
    torch.cuda.synchronize()
    assert torch.equal(_bits(x[:, :P]), _bits(q.expand(B, P, F)))
    assert torch.equal(_bits(x[:, P:]), _bits(before[:B * (t_max + P)].view(B, t_max + P, F)[:, P:]))
    assert (blk[B * (t_max + P):] == sentinel).all()


SHORT_N = [2, 3, 129, 256, 257, 399]


def test_fbank_short_vs_float64_short_window_rule(tables):
    """fa_fbank_short (2 <= n < 400: one window of all n samples, FFT of the next power of two, the frame repeated lfr_m times, CMVN)
    against the float64 rule.  Its transform is a float64 DFT, so what is left is the fp32 framing arithmetic and the fp32 mel sum:
    |d| <= |cmvn scale| (5e-6 + 1e-6 sqrt(E_frame_max / E_bin)) + 2u |feature|."""
    from funasr_b200.engine import kaldi_mel_banks
    abi, lib = _lib()
    cmvn = _cmvn(7)
    cmvn_dev = cmvn.to(DEV)
    scl = np.abs(cmvn[1].double().numpy())
    worst, worst_n = 0.0, None
    for i, n in enumerate(SHORT_N):
        w = _signal("speech", 400, 90 + i)[:n]
        pad = 1 << (n - 1).bit_length()
        win = torch.hamming_window(n, periodic=False, alpha=0.54, beta=0.46, dtype=torch.float32).to(DEV)
        mel = kaldi_mel_banks(n_fft=pad).to(DEV)
        wd = torch.as_tensor(w).to(DEV)
        out = torch.full((7 * 80,), float("nan"), device=DEV)
        abi.check(lib.fa_fbank_short(wd.data_ptr(), n, win.data_ptr(), mel.data_ptr(), pad, cmvn_dev.data_ptr(), 7, out.data_ptr(), _st()),
                  "fa_fbank_short")
        torch.cuda.synchronize()
        lm = fbank64(w)
        assert lm.shape == (1, 80)
        want = cmvn64(np.tile(lm, (1, 7))[0], cmvn)
        bound = scl * np.tile(logmel_bound(lm, 5e-6, 1e-6), (1, 7))[0] + 2 * U * np.abs(want)
        r = float((np.abs(out.cpu().double().numpy() - want) / bound).max())
        if r > worst:
            worst, worst_n = r, n
    print("fbank_short: worst |d| / bound %.3f at n = %s" % (worst, worst_n))
    assert worst <= 1.0


# ============================================================================================== CAM++ features and CMN
def _campplus_ref(w, t_keep=None):
    """float64 features of fa_campplus_features: kaldi.fbank with torchaudio's defaults (povey, no x32768, no LFR), then the mean over
    the kept frames subtracted.  Also returns the log-mel rows for the bound."""
    lm = fbank64(w, "povey", 1.0)[:t_keep]
    return lm - lm.mean(0), lm


def _cmn_bound(lm):
    """Bound on |d| of the mean-subtracted features of one utterance (T frames, per mel bin c).  The log-mel error e_t is at most
    B_t = logmel_bound(lm).  The kernel subtracts m = fl(fl(sum) / T), its sum sequential in time order in fp32: each partial sum S_k
    is rounded once, so the sum is off by at most u sum_k |S_k| beyond the B_t it inherits, the division adds u |m| and the
    subtraction u |y|.  So |d y_t| <= B_t + mean_k(B_k) + u (sum_k |S_k| / T + |m| + |y_t|), with S_k, m and y from float64 — the
    sequential-sum term grows with T, which is why a 1500-frame utterance is the case where this mean is least accurate."""
    T = lm.shape[0]
    b = logmel_bound(lm)
    S = np.abs(np.cumsum(lm, 0)).sum(0) / T
    m = lm.mean(0)
    y = lm - m
    return b + b.mean(0) + U * (S + np.abs(m) + np.abs(y))


def _campplus_call(lib, tab, wavs, t_max, slack_rows=0, sentinel=0.0):
    wav, lens = _padded(wavs)
    B = len(wavs)
    buf = torch.full(((B * t_max + slack_rows) * 80,), sentinel, device=DEV)
    flens = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    st = lib.fa_campplus_features(wav.data_ptr(), lens.data_ptr(), B, wav.stride(0), tab.data_ptr(), buf.data_ptr(), flens.data_ptr(),
                                  t_max, _st())
    assert st == 0, st
    torch.cuda.synchronize()
    return buf, flens


@pytest.mark.parametrize("case", ["ragged", "long"])
def test_campplus_features_vs_float64(tables, case):
    """fa_campplus_features (the 1/1 instantiation with the povey window and no x32768, then per-utterance mean subtraction) against
    float64, on frame counts around the kernel's 48-row CTAs and on one ~1500-frame utterance."""
    abi, lib = _lib()
    frames = [47, 48, 49, 95, 96, 97] if case == "ragged" else [1500]
    wavs = [_signal("speech" if i % 2 == 0 else "noise", _n(f, 13 * i), 20 + i) for i, f in enumerate(frames)]
    t_max = max(frames)
    buf, flens = _campplus_call(lib, tables["povey"], wavs, t_max)
    assert flens.tolist() == frames
    feats = buf.view(len(wavs), t_max, 80).cpu().double().numpy()
    worst, at = 0.0, None
    for b, w in enumerate(wavs):
        want, lm = _campplus_ref(w)
        r = np.abs(feats[b, :frames[b]] - want) / _cmn_bound(lm)
        if r.max() > worst:
            worst, at = float(r.max()), (b,) + np.unravel_index(int(r.argmax()), r.shape)
        assert (feats[b, frames[b]:] == 0).all()
    print("campplus %s: worst |d| / bound %.3f at (utt, row, col) %s" % (case, worst, at))
    assert worst <= 1.0


def test_campplus_t_max_below_the_frame_count_stays_in_its_rows(tables):
    """t_max below an utterance's frame count: the feature kernel writes its first t_max frames, and the mean subtraction must use
    those rows only — the mean over the rows that exist — and write nothing outside feats [B, t_max, 80].  The allocation has slack
    after B * t_max rows, all of it set to a sentinel, so a stray write lands in memory the test owns and shows as a changed
    sentinel.  feat_lens still reports the full frame counts."""
    abi, lib = _lib()
    frames, t_max, slack = [60, 30, 70], 40, 64
    wavs = [_signal("speech", _n(f, 5), 30 + i) for i, f in enumerate(frames)]
    sentinel = 4321.0
    buf, flens = _campplus_call(lib, tables["povey"], wavs, t_max, slack, sentinel)
    assert flens.tolist() == frames
    B = len(wavs)
    feats = buf[:B * t_max * 80].view(B, t_max, 80).cpu().double().numpy()
    assert (buf[B * t_max * 80:] == sentinel).all()
    worst = 0.0
    for b, w in enumerate(wavs):
        k = min(frames[b], t_max)
        want, lm = _campplus_ref(w, k)
        worst = max(worst, float((np.abs(feats[b, :k] - want) / _cmn_bound(lm)).max()))
        assert (feats[b, k:] == 0).all(), b
    print("campplus truncated: worst |d| / bound %.3f" % worst)
    assert worst <= 1.0


# ============================================================================================== FSMN-VAD scorer
VAD_T = [1, 2, 19, 20, 21, 31, 32, 33, 64, 6000, 6001, 13000]
SIL_SETS = [(0,), (0, 5), (0, 5, 17, 247)]
# out_linear2 scaled so the logits span about -14 .. 24 on the inputs below: some posteriors come within 1e-6 of 0 or of 1, where the
# detector's thresholds bite
VAD_LOGIT_SCALE = 3.0
# Bound on the logit error of the fp32 SIMT GEMM chain (K = 400, 144, 256, 128, 256, 144).  Perturbing every logit by at most dz moves
# each posterior by a factor within e^(+-2 dz), and the same holds for 1 - p, so |dp| <= 2 dz min(p, 1 - p).  The softmax's own fp32
# rounding is relative to p: expf (<= 2 ulp, 4u), the row sum (8 terms per lane, then a 5-level shuffle tree: <= 13u), the division
# (u) and the silence sum (u per id): (18 + n_sil) u p, taken as (20 + n_sil) u p.  Near p = 1 this term, not dz, is what limits
# the kernel: the 247 other terms of the sum are each below half an ulp of it.
# Measured on an H100 80GB HBM3 (700 W): the largest logit error the posteriors imply is 2.5e-5 (t = 6000), worst ratio to the bound
# 0.42.  A flat 2e-6 on |dp| would not hold: the largest |dp| is 5.5e-6, at posteriors near 1/2, where p (1 - p) times that logit
# error is what any fp32 GEMM chain of these widths leaves (an fp32 CPU evaluation of the same network is off by 4.5e-5 in the
# logits); at the ends, where the thresholds act, the bound is a few ulp of p or of 1 - p.
VAD_DZ = 2e-4
VAD_ROUND = 20


def _vad_state():
    from funasr_b200 import synth
    p = synth.make_vad_state_dict(seed=0)
    for k in ("encoder.out_linear2.linear.weight", "encoder.out_linear2.linear.bias"):
        p[k] = p[k] * VAD_LOGIT_SCALE
    return p


def _vad_feats(t, seed):
    """[t, 400] CMVN-scale features whose mean level (the synthetic model's energy channel) swings slowly between silence and speech."""
    g = torch.Generator().manual_seed(seed)
    s = torch.arange(t, dtype=torch.float32)
    level = 4 * torch.sin(2 * math.pi * s / 397.0) + 2 * torch.sin(2 * math.pi * s / 89.0)
    return torch.randn(t, 400, generator=g) + level[:, None]


@pytest.fixture(scope="module")
def vad():
    from funasr_b200.vad_model import VadEngine
    p = _vad_state()
    return p, {ids: VadEngine(p, DEV, None, sil_pdf_ids=ids) for ids in SIL_SETS}


def _vad_forward(lib, enc, feats, ld, t, ws_fill=0, want_scores=True, out_dim=248):
    need = int(lib.fa_fsmn_vad_workspace_bytes(C.byref(enc), t))
    ws = torch.full((need,), ws_fill, dtype=torch.uint8, device=DEV)
    sil = torch.full((t,), float("nan"), device=DEV)
    sc = torch.full((t, out_dim), float("nan"), device=DEV) if want_scores else None
    st = lib.fa_fsmn_vad_forward(C.byref(enc), feats.data_ptr(), ld, t, sil.data_ptr(), _ptr(sc), ws.data_ptr(), need, _st())
    torch.cuda.synchronize()
    return st, sil, sc


@pytest.mark.parametrize("t", VAD_T)
def test_fsmn_vad_forward_vs_float64(vad, t):
    """fa_fsmn_vad_forward (fp32 GEMMs, the causal 20-tap memory, softmax and silence sum) against the float64 FSMN, scores and
    sil_prob, with 1, 2 and 4 silence ids, at t around the memory's 20 frames, the 32-frame SIMT strip and the reference's 60 s
    chunk.  |dp| <= 2 VAD_DZ min(p, 1 - p) + (VAD_ROUND + n_sil) u p, n_sil = 0 for the scores."""
    abi, lib = _lib()
    p, engines = vad
    x = _vad_feats(t, seed=t)
    z = vad_logits64(x.numpy(), p)
    want = softmax64(z)
    xd = x.to(DEV)
    worst, worst_abs, dz_seen = 0.0, 0.0, 0.0
    for ids, eng in engines.items():
        st, sil, sc = _vad_forward(lib, eng.enc, xd, 400, t)
        assert st == 0, st
        got = sc.cpu().double().numpy()
        gsil = sil.cpu().double().numpy()
        wsil = want[:, list(ids)].sum(-1)
        for g_, w_, k in ((got, want, 0), (gsil, wsil, len(ids))):
            d = np.abs(g_ - w_)
            tail = np.minimum(w_, 1 - w_)
            rnd = (VAD_ROUND + k) * U * w_
            r = d / (2 * VAD_DZ * tail + rnd)
            worst, worst_abs = max(worst, float(r.max())), max(worst_abs, float(d.max()))
            dz_seen = max(dz_seen, float((np.maximum(d - rnd, 0) / np.maximum(2 * tail, 1e-300)).max()))
    near = int(((want[:, 0] < 1e-6) | (want[:, 0] > 1 - 1e-6)).sum())
    print("fsmn_vad t=%d: logits %.1f .. %.1f, %d sil posteriors within 1e-6 of 0 or 1; worst |dp| / bound %.3f, max |dp| %.2e, implied "
          "logit error %.2e (bound %.0e)" % (t, z.min(), z.max(), near, worst, worst_abs, dz_seen, VAD_DZ))
    assert worst <= 1.0


def test_fsmn_vad_strided_input_and_dirty_workspace_are_bit_exact(vad):
    """ld_feats > 400 with NaN in the extra columns reads only the 400 feature columns, and a workspace full of NaN before the call
    gives the same bits as a zeroed one: the zero-fill of the padded activation columns covers every buffer the GEMMs read."""
    abi, lib = _lib()
    p, engines = vad
    enc = engines[SIL_SETS[-1]].enc
    t = 1000
    x = _vad_feats(t, seed=5).to(DEV)
    st, sil0, sc0 = _vad_forward(lib, enc, x, 400, t)
    assert st == 0
    for ld in (404, 512):
        wide = torch.full((t, ld), float("nan"), device=DEV)
        wide[:, :400] = x
        st, sil, sc = _vad_forward(lib, enc, wide, ld, t)
        assert st == 0
        assert torch.equal(_bits(sil), _bits(sil0)) and torch.equal(_bits(sc), _bits(sc0)), ld
    st, sil, sc = _vad_forward(lib, enc, x, 400, t, ws_fill=0xFF)          # 0xFFFFFFFF: a NaN in every fp32 slot
    assert st == 0
    assert torch.equal(_bits(sil), _bits(sil0)) and torch.equal(_bits(sc), _bits(sc0))
    st, sil, _ = _vad_forward(lib, enc, x, 400, t, ws_fill=0xFF, want_scores=False)
    assert st == 0 and torch.equal(_bits(sil), _bits(sil0))


def test_fsmn_vad_status_codes(vad):
    """n_sil outside 1..4 -> FA_ERR_ARG; a memory layer other than 128 wide, or an input width not a multiple of 16 ->
    FA_ERR_UNSUPPORTED; a workspace one byte short -> FA_ERR_WORKSPACE."""
    abi, lib = _lib()
    p, engines = vad
    base = engines[SIL_SETS[0]].enc
    t = 40
    x = _vad_feats(t, seed=6).to(DEV)

    def run(enc, ws_less=0):
        need = int(lib.fa_fsmn_vad_workspace_bytes(C.byref(base), t))
        ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
        sil = torch.empty(t, device=DEV)
        st = lib.fa_fsmn_vad_forward(C.byref(enc), x.data_ptr(), 400, t, sil.data_ptr(), None, ws.data_ptr(), need - ws_less, _st())
        torch.cuda.synchronize()
        return st

    assert run(base) == 0
    for n_sil in (0, 5):
        e = abi.FaVadEncoder.from_buffer_copy(base)
        e.n_sil = n_sil
        assert run(e) == -1, n_sil
    e = abi.FaVadEncoder.from_buffer_copy(base)
    layers = (abi.FaVadLayer * base.n_layers)(*[abi.FaVadLayer.from_buffer_copy(base.layers[i]) for i in range(base.n_layers)])
    layers[1].lin.out_f = 64
    e.layers = layers
    assert run(e) == -4
    e = abi.FaVadEncoder.from_buffer_copy(base)
    e.in1.in_f = 392 + 4                                                   # 396: not a multiple of 16
    assert run(e) == -4
    assert run(base, ws_less=1) == -3


# ============================================================================================== frame energies
def test_frame_decibels_vs_float64():
    """fa_frame_decibels against float64 10 log10(sum x^2 + 1e-6) on n = (T - 1) 160 + 400 samples exactly (the last frame ends on the
    last sample), with an all-zero frame (-60 dB) and a full-scale one; frames one past the end is FA_ERR_ARG.  |d| <= 1e-4 dB."""
    from funasr_b200 import synth
    abi, lib = _lib()
    T = 1000
    n = (T - 1) * SHIFT + WIN
    x = synth.make_wav(n, 3, "speechlike").numpy().copy()
    x[10 * SHIFT: 10 * SHIFT + WIN] = 0.0                                   # frame 10 all zero
    x[20 * SHIFT: 20 * SHIFT + WIN] = np.where(np.arange(WIN) % 2 == 0, 1.0, -1.0)   # frame 20 full scale
    xd = torch.as_tensor(x).to(DEV)
    db = torch.full((T,), float("nan"), device=DEV)
    abi.check(lib.fa_frame_decibels(xd.data_ptr(), n, T, db.data_ptr(), _st()), "fa_frame_decibels")
    torch.cuda.synchronize()
    fr = np.lib.stride_tricks.sliding_window_view(x.astype(np.float64), WIN)[::SHIFT][:T]
    want = 10 * np.log10((fr * fr).sum(-1) + 1e-6)
    got = db.cpu().double().numpy()
    d = np.abs(got - want)
    print("frame_decibels: max |d| %.2e dB (bound 1e-4), zero frame %.6f dB, full-scale frame %.4f dB" % (d.max(), got[10], got[20]))
    assert abs(want[10] + 60.0) < 1e-12 and abs(got[10] + 60.0) <= 1e-4
    assert abs(want[20] - 10 * math.log10(400 + 1e-6)) < 1e-12
    assert d.max() <= 1e-4
    assert lib.fa_frame_decibels(xd.data_ptr(), n, T + 1, db.data_ptr(), _st()) == -1
    assert lib.fa_frame_decibels(xd.data_ptr(), n, 0, db.data_ptr(), _st()) == 0
