"""The float64 restatement of the model entry points (tests/model_entries_ref.py) checked without a GPU: it reproduces the
reference's committed goldens within fp32 rounding, equals the oracle's own functions when run in fp32, and the per-row metric
behaves on hand-made arrays."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_case, load_ctx_case, load_sv_case, state_dict_for

import model_entries_ref as R
import paraformer_oracle as O

# float64 restatement against the fp32 reference goldens: what separates them is the reference's own fp32 rounding.  Worst
# measured: encoder rows 1.2e-6 (tiny Paraformer), 2.6e-6 (SenseVoice), 2.0e-6 (aligner); selected log-probs 2.1e-5 absolute
# (SenseVoice, |logp| up to ~15).  Bars: about 5 x or more.
GOLD_ROW, GOLD_ALPHA, GOLD_LOGP = 3e-5, 1e-6, 1e-4


@pytest.mark.parametrize("name", ["tiny_ragged3", "tiny_single"])
def test_paraformer_restatement_reproduces_goldens(name):
    cfg, wseed, _, _, g = load_case(name)
    p = R.to64(state_dict_for(cfg, wseed))
    feats, lens = torch.from_numpy(g["feats"]).double(), g["feat_lens"]
    T = feats.shape[1]
    enc = R.encoder(feats, lens, p, R.paraformer_encoder_names(cfg.enc_layers), "encoder.after_norm", cfg.heads, cfg.ln_eps)[cfg.enc_layers]
    e = R.worst(R.row_err(enc.numpy(), g["enc"]), R.len_mask(lens, T))
    print(R.describe("enc", e))
    assert e[0] <= GOLD_ROW
    al, asum, fires = R.predictor(enc, lens, p, cfg.tail_threshold)
    assert np.abs(al.numpy() - g["alphas"]).max() <= GOLD_ALPHA
    tok = np.floor(asum.numpy()).astype(np.int32)
    assert tok.tolist() == g["token_num"].tolist()
    n = int(g["token_num"].max())
    acoustic = np.zeros((len(lens), n, enc.shape[2]))
    for b, (frames, _, _, _) in enumerate(fires):
        k = min(frames.shape[0], int(tok[b]))
        acoustic[b, :k] = frames[:k]
    assert R.worst(R.row_err(acoustic, g["acoustic"]))[0] <= GOLD_ROW
    _, logits = R.decoder_hidden(enc, lens, torch.from_numpy(acoustic), torch.from_numpy(tok), p, cfg.dec_layers, cfg.heads, cfg.ln_eps)
    lp = torch.log_softmax(logits, -1)[:, g["logp_rows"].tolist()].numpy()
    assert np.abs(lp - g["logp_sel"]).max() <= GOLD_LOGP


def test_contextual_restatement_reproduces_goldens():
    cfg, wseed, wavs, cmvn, _, g = load_ctx_case("ctx_tiny_ragged3")
    from funasr_b200 import synth
    p = R.to64(synth.make_contextual_state_dict(cfg, wseed))
    feats, lens = O.frontend(wavs, cmvn)
    enc = R.encoder(feats.double(), lens, p, R.paraformer_encoder_names(cfg.enc_layers), "encoder.after_norm", cfg.heads,
                    cfg.ln_eps)[cfg.enc_layers]
    al, asum, fires = R.predictor(enc, lens, p, cfg.tail_threshold)
    tok = np.floor(asum.numpy()).astype(np.int64)
    assert tok.tolist() == g["token_num"].tolist()
    n = int(tok.max())
    acoustic = torch.zeros(len(wavs), n, 512, dtype=torch.float64)
    for b, (frames, _, _, _) in enumerate(fires):
        k = min(frames.shape[0], int(tok[b]))
        acoustic[b, :k] = torch.from_numpy(frames[:k])
    logits = O.contextual_decoder(enc, lens, acoustic, torch.from_numpy(tok), torch.from_numpy(g["hw_embed"]).double(), p, cfg.dec_layers)
    lp = torch.log_softmax(logits, -1)[:, g["logp_rows"].tolist()].numpy()
    assert np.abs(lp - g["logp_sel"]).max() <= GOLD_LOGP


def _sv_inputs(name):
    from funasr_b200 import synth
    cfg, wseed, wavs, cmvn, g = load_sv_case(name)
    p = synth.make_sensevoice_state_dict(cfg, wseed)
    feats, flens = O.frontend(wavs, cmvn)
    emb = p["embed.weight"]
    q = torch.stack([emb[0], emb[1], emb[2], emb[15]])[None].repeat(feats.shape[0], 1, 1)
    return cfg, p, torch.cat([q, feats], dim=1), flens + 4, g


def test_sensevoice_restatement_reproduces_goldens():
    cfg, p, x, lens, g = _sv_inputs("sv_tiny_ragged3")
    p = R.to64(p)
    names = R.paraformer_encoder_names(cfg.enc_layers)
    h = R.encoder(x.double(), lens, p, names, "encoder.after_norm", cfg.heads, cfg.ln_eps)[cfg.enc_layers]
    enc = R.encoder(h, lens, p, ["encoder.tp_encoders.%d" % i for i in range(cfg.tp_layers)], "encoder.tp_norm", cfg.heads, cfg.ln_eps,
                    embed=False)[cfg.tp_layers]
    e = R.worst(R.row_err(enc.numpy(), g["enc"]), R.len_mask(lens, x.shape[1]))
    print(R.describe("sv enc", e))
    assert e[0] <= GOLD_ROW
    lp = torch.log_softmax(F.linear(enc, p["ctc.ctc_lo.weight"], p["ctc.ctc_lo.bias"]), -1)[:, g["logp_rows"].tolist()].numpy()
    assert np.abs(lp - g["logp_sel"]).max() <= GOLD_LOGP


def test_aligner_restatement_reproduces_goldens():
    from funasr_b200 import synth
    g = dict(np.load(R.__file__.replace("model_entries_ref.py", "golden/aligner_tiny_ragged3.npz")))
    cfg = synth.ALIGNER_TINY
    p = R.to64(synth.make_aligner_state_dict(cfg, 5))
    wavs = [synth.make_aligner_wav(float(sec), int(s)) for sec, s in g["wav_spec"].tolist()]
    feats, lens = O.frontend(wavs, synth.make_cmvn(cfg, seed=1))
    assert lens.tolist() == g["enc_lens"].tolist()
    enc = R.encoder(feats.double(), lens, p, R.paraformer_encoder_names(cfg.enc_layers), "encoder.after_norm", cfg.heads,
                    cfg.ln_eps)[cfg.enc_layers]
    e = R.worst(R.row_err(enc[:, g["enc_rows"]].numpy(), g["enc"]), R.len_mask(lens, enc.shape[1])[:, g["enc_rows"]])
    print(R.describe("aligner enc", e))
    assert e[0] <= GOLD_ROW


# ------------------------------------------------------------------------------------------------ fp32: the oracle itself
def test_restatement_in_fp32_is_the_oracle():
    """Run in fp32, every restated piece equals the oracle function it stands for bit for bit; the integrate-and-fire restatement
    (the oracle's runs in fp32 whatever its input) agrees with cif_v1 and cif_loop within fp32 rounding."""
    cfg, wseed, _, _, g = load_case("tiny_ragged3")
    p = state_dict_for(cfg, wseed)
    feats, lens = torch.from_numpy(g["feats"]), torch.from_numpy(g["feat_lens"])
    T = feats.shape[1]
    assert torch.equal(R.sinusoid_pe(T, 560, torch.float32), O.sinusoid_pe(T, 560))
    enc_o, _ = O.encoder(feats, lens, p, cfg.enc_layers, cfg.heads, cfg.ln_eps)
    enc = R.encoder(feats, lens, p, R.paraformer_encoder_names(cfg.enc_layers), "encoder.after_norm", cfg.heads, cfg.ln_eps)[cfg.enc_layers]
    assert torch.equal(enc, enc_o)
    emb_o, tok_o, al_o, peaks_o = O.predictor(enc_o, lens, p, cfg.tail_threshold)
    al, asum, fires = R.predictor(enc, lens, p, cfg.tail_threshold)
    assert torch.equal(al, al_o) and torch.equal(torch.floor(asum), tok_o)
    for b, (frames, peaks, _, _) in enumerate(fires):
        k = int(tok_o[b])
        assert np.abs(frames[:k] - emb_o[b, :k].numpy()).max() <= 1e-5 * max(1.0, np.abs(frames).max())
        assert np.abs(peaks - peaks_o[b].numpy()).max() <= 1e-5
    mask = (torch.arange(T)[None, :] < lens[:, None].long())[:, None, :]
    hidden, al2, _ = O.cif_tail(enc_o, O.cif_alphas(enc_o, mask, p), mask.squeeze(1).float(), cfg.tail_threshold)
    emb_l, fires_l = O.cif_loop(hidden, al2)
    for b, (frames, peaks, _, _) in enumerate(fires):
        assert np.abs(frames - emb_l[b, :frames.shape[0]].numpy()).max() <= 1e-5 * max(1.0, np.abs(frames).max())
        assert np.abs(peaks - fires_l[b].numpy()).max() <= 1e-5
    tok = tok_o.long()
    n = int(tok.max())
    h, logits = R.decoder_hidden(enc_o, lens, emb_o, tok, p, cfg.dec_layers, cfg.heads, cfg.ln_eps)
    assert torch.equal(logits, O.decoder(enc_o, lens, emb_o[:, :n], tok, p, cfg.dec_layers, cfg.heads, cfg.ln_eps))


# ------------------------------------------------------------------------------------------------ the metric
def test_row_metric_on_hand_made_arrays():
    ref = np.array([[[1.0, -2.0, 0.5], [0.0, 0.0, 0.0], [1e-4, 0.0, -1e-4]]])     # [1, 3, 3]: a normal row, an all-zero row, a tiny row
    got = ref + np.array([[[0.0, 2e-3, 0.0], [0.0, -5e-4, 0.0], [0.0, 1e-4, 0.0]]])
    e = R.row_err(got, ref)
    assert e.shape == (1, 3)
    assert e[0, 0] == pytest.approx(1e-3)                     # 2e-3 / max |ref| = 2
    assert e[0, 1] == pytest.approx(5e-4 / R.FLOOR)           # all-zero reference row: the floor normalises, no division by zero
    assert e[0, 2] == pytest.approx(1e-4 / R.FLOOR)           # a small row is not judged against a larger row's scale
    assert np.isfinite(e).all()
    # a global max-normalised error would hide the small row's error behind the large row's scale
    assert np.abs(got - ref)[0, 2].max() / np.abs(ref).max() < e[0, 2]
    valid = np.array([[True, False, True]])
    v, idx, ok = R.worst(e, valid)
    assert v == pytest.approx(5e-2) and idx == (0, 1) and ok is False
    assert "padded" in R.describe("x", (v, idx, ok)) and "utt 0, row 1" in R.describe("x", (v, idx, ok))
    assert R.row_err(ref, ref).max() == 0.0


def test_decision_rule_on_hand_made_rows():
    ref = np.array([[0.0, 5.0, 4.0], [0.0, 5.0, 4.999], [3.0, 1.0, 2.9995]])
    bound = np.array([1e-3, 1e-3, 1e-3])
    assert R.decision_ok(np.array([1, 1, 0]), ref, bound).all()
    assert R.decision_ok(np.array([1, 2, 2]), ref, bound).tolist() == [True, True, True]   # rows 2 and 3 are near ties: either id
    assert R.decision_ok(np.array([2, 0, 1]), ref, bound).tolist() == [False, False, False]


def test_cif_fire_on_hand_made_alphas():
    h = np.eye(4)
    frames, peaks, fires, integ = R.cif_fire(h, np.array([0.6, 0.6, 0.9, 0.3]))
    assert fires == [1, 2] and np.allclose(peaks, [0.6, 1.2, 1.1, 0.4])
    assert np.allclose(frames, [[0.6, 0.4, 0, 0], [0, 0.2, 0.8, 0]]) and np.allclose(integ, [0.6, 1.2, 2.1, 2.4])
