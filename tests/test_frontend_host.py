"""The float64 restatements that tests/test_frontend_gpu.py holds the frontend kernels against, checked on the CPU: the Fbank against
torchaudio's kaldi.fbank on float64 input (both windows, the short-utterance rule), the LFR gather against the fp32 oracle's
apply_lfr, and the FSMN-VAD scorer against the fp32 oracle."""
import math

import numpy as np
import pytest
import torch

import paraformer_oracle as O
import test_frontend_gpu as G
import vad_oracle as VO


@pytest.mark.parametrize("window,scale", [("hamming", 32768.0), ("povey", 1.0)])
def test_fbank64_is_torchaudio_kaldi_fbank(window, scale):
    """fbank64 is kaldi.fbank(wav * scale, 80 mel, 25 / 10 ms, dither 0, energy_floor 0, snip_edges) on float64 input to ~1e-9:
    framing, DC removal, pre-emphasis with the replicated first sample, the window, the power spectrum, the mel filters and the eps
    floor — and, below 400 samples, one window of all n samples with the FFT of the next power of two."""
    K = pytest.importorskip("torchaudio.compliance.kaldi")
    from funasr_b200 import synth
    worst = 0.0
    for i, n in enumerate([2, 3, 129, 256, 257, 399, 400, 559, 560, 561, 8123, 48000]):
        w = synth.make_wav(n, 50 + i, "speechlike" if i % 2 else "noise").double()
        got = G.fbank64(w.numpy(), window, scale)
        want = K.fbank(w[None] * scale, num_mel_bins=80, frame_length=25.0 if n >= 400 else n / 16000 * 1000, frame_shift=10, dither=0.0,
                       energy_floor=0.0, window_type=window, sample_frequency=16000, snip_edges=True).numpy()
        assert got.shape == want.shape == (max(1, G.num_frames(n)), 80), n
        worst = max(worst, float(np.abs(got - want).max()))
    # tones, an impulse and silence reach the eps floor and the single-bin spectra
    n = 8080
    i = np.arange(n)
    for x in [np.cos(2 * math.pi * 128 * i / 512.0), np.eye(1, n, 3000)[0], np.zeros(n), np.full(n, 0.25)]:
        got = G.fbank64(x, window, scale)
        want = K.fbank(torch.tensor(x)[None] * scale, num_mel_bins=80, dither=0.0, energy_floor=0.0, window_type=window).numpy()
        worst = max(worst, float(np.abs(got - want).max()))
    print("fbank64 (%s) vs torchaudio float64: max |d| %.1e" % (window, worst))
    assert worst <= 1e-9


@pytest.mark.parametrize("m,n", [(7, 6), (5, 1), (1, 1)])
def test_lfr64_is_the_oracle_gather(m, n):
    """lfr64 equals paraformer_oracle.apply_lfr (pinned against the reference's goldens) for frame counts around the row changes."""
    g = torch.Generator().manual_seed(m * 10 + n)
    for T in [1, 2, 5, 6, 7, 11, 12, 13, 47, 48, 49]:
        x = torch.randn(T, 80, generator=g, dtype=torch.float64)
        assert np.array_equal(G.lfr64(x.numpy(), m, n), O.apply_lfr(x, m, n).numpy()), T


def test_vad_logits64_is_the_fp32_oracle():
    """softmax(vad_logits64) equals vad_oracle.fsmn_scores (fp32) to its rounding, on the scaled weights and energy-swinging inputs of
    the GPU test, at lengths shorter and longer than the 20-frame memory."""
    p = G._vad_state()
    for t in [1, 19, 21, 300]:
        x = G._vad_feats(t, seed=t)
        got = G.softmax64(G.vad_logits64(x.numpy(), p))
        with torch.no_grad():
            want = VO.fsmn_scores(x, p).double().numpy()
        assert np.abs(got - want).max() <= 2e-5, t
