"""Seeded synthetic Paraformer weights, waveforms and configs.

No pretrained Paraformer weights exist offline (SURVEY.md §8c), so parity and the
benchmark run on a deterministic, well-conditioned synthetic ``state_dict`` whose
key names and shapes are exactly the reference's (SURVEY.md §8 row a21:
``encoder.encoders0.0.self_attn.linear_q_k_v.weight`` ...), so the very same dict
loads into the reference ``Paraformer`` through ``load_pretrained_model`` and into
this backend.  Everything is generated on the CPU with ``torch.Generator`` so it
is identical on every machine with this torch version.
"""
from __future__ import annotations

import math
from collections import OrderedDict
from dataclasses import dataclass, asdict

import torch


@dataclass(frozen=True)
class ParaformerConfig:
    """Architecture constants of Paraformer-large (funasr/models/paraformer/template.yaml:9-66)."""
    n_mels: int = 80
    lfr_m: int = 7
    lfr_n: int = 6
    d_model: int = 512
    heads: int = 4
    ffn: int = 2048
    enc_layers: int = 50      # encoder_conf.num_blocks (1 x encoders0 + 49 x encoders)
    dec_layers: int = 16      # decoder_conf.num_blocks == att_layer_num
    kernel: int = 11          # FSMN kernel_size, sanm_shfit = 0
    vocab: int = 8404
    cif_threshold: float = 1.0
    tail_threshold: float = 0.45
    ln_eps: float = 1e-12     # funasr/models/transformer/layer_norm.py:24

    @property
    def feat_dim(self) -> int:
        return self.n_mels * self.lfr_m

    def to_dict(self):
        return asdict(self)


PARAFORMER_LARGE = ParaformerConfig()
# Same operator shapes, fewer layers: the oracle finishes in well under a second.
PARAFORMER_TINY = ParaformerConfig(enc_layers=3, dec_layers=2, vocab=1000)


def _randn(g, *shape, std=1.0):
    return torch.randn(*shape, generator=g, dtype=torch.float32) * std


def make_state_dict(cfg: ParaformerConfig = PARAFORMER_LARGE, seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """Well-conditioned synthetic weights under the reference's parameter names."""
    g = torch.Generator().manual_seed(1000003 * seed + 17)
    D, F, V, K, Din = cfg.d_model, cfg.ffn, cfg.vocab, cfg.kernel, cfg.feat_dim
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()

    def linear(prefix, out_f, in_f, bias=True, gain=1.0):
        sd[prefix + ".weight"] = _randn(g, out_f, in_f, std=gain / math.sqrt(in_f))
        if bias:
            sd[prefix + ".bias"] = _randn(g, out_f, std=0.02)

    def norm(prefix, n):
        sd[prefix + ".weight"] = 1.0 + _randn(g, n, std=0.1)
        sd[prefix + ".bias"] = _randn(g, n, std=0.05)

    # Gains chosen so that (a) frames/tokens stay distinct through 50+16 layers (diverse greedy ids) and (b) the
    # network is well conditioned: 1e-6 relative input noise moves log-probs by ~5e-4 while the smallest top-1/top-2
    # margin is ~1e-2, so greedy ids are a meaningful bit-exact parity target.
    def enc_layer(prefix, in_size):
        res = 0.7 if in_size != D else 0.3
        linear(prefix + ".self_attn.linear_out", D, D, gain=res)
        linear(prefix + ".self_attn.linear_q_k_v", 3 * D, in_size, gain=1.5)
        sd[prefix + ".self_attn.linear_q_k_v.weight"][: 2 * D] *= 1.5   # sharper q.k scores -> frame-specific context
        sd[prefix + ".self_attn.fsmn_block.weight"] = _randn(g, D, 1, K, std=0.15)
        linear(prefix + ".feed_forward.w_1", F, D)
        linear(prefix + ".feed_forward.w_2", D, F, gain=res)
        norm(prefix + ".norm1", in_size)
        norm(prefix + ".norm2", D)

    enc_layer("encoder.encoders0.0", Din)
    for i in range(cfg.enc_layers - 1):
        enc_layer("encoder.encoders.%d" % i, D)
    norm("encoder.after_norm", D)

    # CIF predictor (paraformer/cif_predictor.py:241-242)
    sd["predictor.cif_conv1d.weight"] = _randn(g, D, D, 3, std=1.0 / math.sqrt(3 * D))
    sd["predictor.cif_conv1d.bias"] = _randn(g, D, std=0.02)
    sd["predictor.cif_output.weight"] = _randn(g, 1, D, std=1.2 / math.sqrt(D))
    # sigmoid(-1.6) ~ 0.17 per 60 ms LFR frame -> a few tokens per second
    sd["predictor.cif_output.bias"] = torch.full((1,), -1.6)

    sd["decoder.embed.0.weight"] = _randn(g, V, D, std=0.1)  # unused at inference
    norm("decoder.after_norm", D)
    linear("decoder.output_layer", V, D, gain=3.0)

    def dec_ffn(prefix, res=0.3):
        linear(prefix + ".feed_forward.w_1", F, D)
        sd[prefix + ".feed_forward.w_2.weight"] = _randn(g, D, F, std=res / math.sqrt(F))
        norm(prefix + ".feed_forward.norm", F)

    for i in range(cfg.dec_layers):
        p = "decoder.decoders.%d" % i
        dec_ffn(p)
        sd[p + ".self_attn.fsmn_block.weight"] = _randn(g, D, 1, K, std=0.15)
        linear(p + ".src_attn.linear_q", D, D, gain=1.5)
        linear(p + ".src_attn.linear_k_v", 2 * D, D, gain=1.5)
        linear(p + ".src_attn.linear_out", D, D, gain=0.3)
        norm(p + ".norm1", D)
        norm(p + ".norm2", D)
        norm(p + ".norm3", D)
    dec_ffn("decoder.decoders3.0", res=0.7)
    norm("decoder.decoders3.0.norm1", D)
    return sd


def make_contextual_state_dict(cfg: ParaformerConfig = PARAFORMER_LARGE, seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """ContextualParaformer (BASELINE config 5; funasr/models/contextual_paraformer): the Paraformer dict with the last
    attention decoder layer renamed `decoder.last_decoder`, plus `decoder.bias_decoder.*`, `decoder.bias_output.weight`
    (Conv1d 1024->512, k=1, no bias), the hotword LSTM `bias_encoder.*` and `bias_embed.weight` (inner_dim 512)."""
    base = make_state_dict(cfg, seed)
    g = torch.Generator().manual_seed(1000003 * seed + 41)
    D, V = cfg.d_model, cfg.vocab
    last = cfg.dec_layers - 1
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for k, v in base.items():
        sd[k.replace("decoder.decoders.%d." % last, "decoder.last_decoder.")] = v
    sd["decoder.bias_decoder.norm3.weight"] = 1.0 + _randn(g, D, std=0.1)
    sd["decoder.bias_decoder.norm3.bias"] = _randn(g, D, std=0.05)
    for name, shape, gain in (("linear_q", (D, D), 1.5), ("linear_k_v", (2 * D, D), 1.5), ("linear_out", (D, D), 0.3)):
        sd["decoder.bias_decoder.src_attn.%s.weight" % name] = _randn(g, *shape, std=gain / math.sqrt(D))
        sd["decoder.bias_decoder.src_attn.%s.bias" % name] = _randn(g, shape[0], std=0.02)
    sd["decoder.bias_output.weight"] = _randn(g, D, 2 * D, 1, std=1.0 / math.sqrt(2 * D))
    sd["bias_encoder.weight_ih_l0"] = _randn(g, 4 * D, D, std=1.0 / math.sqrt(D))
    sd["bias_encoder.weight_hh_l0"] = _randn(g, 4 * D, D, std=1.0 / math.sqrt(D))
    sd["bias_encoder.bias_ih_l0"] = _randn(g, 4 * D, std=0.05)
    sd["bias_encoder.bias_hh_l0"] = _randn(g, 4 * D, std=0.05)
    sd["bias_embed.weight"] = _randn(g, V, D, std=1.0)
    return sd


def make_bicif_state_dict(cfg: ParaformerConfig = PARAFORMER_LARGE, seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """BiCifParaformer (funasr/models/bicif_paraformer; predictor CifPredictorV3, upsample_type cnn_blstm, template.yaml:52-63):
    the Paraformer dict plus the timestamp head `predictor.upsample_cnn` (ConvTranspose1d 512->512, k=s=3), `predictor.blstm`
    (1-layer bidirectional LSTM 512->512) and `predictor.cif_output2` (Linear 1024->1)."""
    sd = make_state_dict(cfg, seed)
    g = torch.Generator().manual_seed(1000003 * seed + 77)
    D = cfg.d_model
    sd["predictor.upsample_cnn.weight"] = _randn(g, D, D, 3, std=1.0 / math.sqrt(D))
    sd["predictor.upsample_cnn.bias"] = _randn(g, D, std=0.05)
    for suf in ("", "_reverse"):
        sd["predictor.blstm.weight_ih_l0" + suf] = _randn(g, 4 * D, D, std=1.5 / math.sqrt(D))
        sd["predictor.blstm.weight_hh_l0" + suf] = _randn(g, 4 * D, D, std=1.0 / math.sqrt(D))
        sd["predictor.blstm.bias_ih_l0" + suf] = _randn(g, 4 * D, std=0.05)
        sd["predictor.blstm.bias_hh_l0" + suf] = _randn(g, 4 * D, std=0.05)
    sd["predictor.cif_output2.weight"] = _randn(g, 1, 2 * D, std=3.0 / math.sqrt(2 * D))
    sd["predictor.cif_output2.bias"] = torch.full((1,), -0.3)
    return sd



# MonotonicAligner fa-zh (monotonic_aligner/template.yaml): SAN-M encoder d = 320, 4 x 80 heads, FFN 1280, 30 blocks, CifPredictorV3
# idim 320 (BLSTM hidden 320).  vocab only sizes the unused decoder-side tensors make_state_dict also draws.
ALIGNER_FA_ZH = ParaformerConfig(d_model=320, heads=4, ffn=1280, enc_layers=30, dec_layers=1, kernel=11, vocab=64)
ALIGNER_TINY = ParaformerConfig(d_model=320, heads=4, ffn=1280, enc_layers=3, dec_layers=1, kernel=11, vocab=64)


def aligner_token_list(n_chars: int = 400):
    """CharTokenizer token list of the synthetic aligner: <blank> <s> </s>, n_chars CJK characters, <unk>."""
    return ["<blank>", "<s>", "</s>"] + [chr(0x4E00 + i) for i in range(n_chars)] + ["<unk>"]


def make_aligner_state_dict(cfg: ParaformerConfig = ALIGNER_FA_ZH, seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """MonotonicAligner (funasr/models/monotonic_aligner/model.py): `encoder.*` and CifPredictorV3's `predictor.*` — cif_conv1d /
    cif_output (loaded, unused at inference) plus the timestamp head.  The timestamp head's gains make the upsampled CIF weights
    follow the audio (their spread across frames is several times their mean), so speech and pauses produce uneven stamps;
    with untuned random weights the weights come out near-constant and the stamps evenly spaced."""
    base = make_state_dict(cfg, seed)
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict((k, v) for k, v in base.items() if k.startswith(("encoder.", "predictor.")))
    g = torch.Generator().manual_seed(1000003 * seed + 91)
    D = cfg.d_model
    sd["predictor.upsample_cnn.weight"] = _randn(g, D, D, 3, std=1.0 / math.sqrt(D))
    sd["predictor.upsample_cnn.bias"] = _randn(g, D, std=0.05)
    for suf in ("", "_reverse"):
        sd["predictor.blstm.weight_ih_l0" + suf] = _randn(g, 4 * D, D, std=1.5 / math.sqrt(D))
        sd["predictor.blstm.weight_hh_l0" + suf] = _randn(g, 4 * D, D, std=1.0 / math.sqrt(D))
        sd["predictor.blstm.bias_ih_l0" + suf] = _randn(g, 4 * D, std=0.05)
        sd["predictor.blstm.bias_hh_l0" + suf] = _randn(g, 4 * D, std=0.05)
    sd["predictor.cif_output2.weight"] = _randn(g, 1, 2 * D, std=8.0 / math.sqrt(2 * D))
    sd["predictor.cif_output2.bias"] = torch.full((1,), -1.0)
    return sd


def make_aligner_wav(seconds: float, seed: int = 0) -> torch.Tensor:
    """Speech-like stretches (0.6-2.0 s) separated by quiet pauses (0.2-0.8 s), 16 kHz: the aligner's stamps then have gaps."""
    g = torch.Generator().manual_seed(7727 * seed + 3)
    n, parts, k = int(seconds * 16000), [], 0
    while sum(p.numel() for p in parts) < n:
        m = int(16000 * (0.6 + 1.4 * float(torch.rand(1, generator=g))))
        parts.append(make_wav(m, 100 * seed + k))
        q = int(16000 * (0.2 + 0.6 * float(torch.rand(1, generator=g))))
        parts.append(0.01 * make_wav(q, 100 * seed + k + 50, "noise"))
        k += 1
    return torch.cat(parts)[:n].contiguous()


SEACO_FFN, SEACO_KERNEL, SEACO_LAYERS = 1024, 21, 6      # seaco_paraformer/template.yaml:57-69 (num_blocks 4 < att_layer_num 6 -> 6 layers)


def seaco_no_bias_id(cfg: ParaformerConfig) -> int:
    """The `NO_BIAS` token id (8377 of 8404 in the released model): the same distance from the end of the synthetic vocabulary."""
    return cfg.vocab - 27


def make_seaco_state_dict(cfg: ParaformerConfig = PARAFORMER_LARGE, seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """SeacoParaformer (funasr/models/seaco_paraformer/model.py:50-120): the BiCif dict plus the 2-layer hotword LSTM
    `bias_encoder`, the `seaco_decoder` (ParaformerSANMDecoder over the hotword memory: 6 attention layers, FFN 1024, FSMN k=21, no
    input / output layer) and `hotword_output_layer`.  `decoder.embed` (the hotword embedding table here) gets unit variance."""
    sd = make_bicif_state_dict(cfg, seed)
    g = torch.Generator().manual_seed(1000003 * seed + 91)
    D, V = cfg.d_model, cfg.vocab
    sd["decoder.embed.0.weight"] = _randn(g, V, D, std=1.0)
    for layer in (0, 1):
        sd["bias_encoder.weight_ih_l%d" % layer] = _randn(g, 4 * D, D, std=1.0 / math.sqrt(D))
        sd["bias_encoder.weight_hh_l%d" % layer] = _randn(g, 4 * D, D, std=1.0 / math.sqrt(D))
        sd["bias_encoder.bias_ih_l%d" % layer] = _randn(g, 4 * D, std=0.05)
        sd["bias_encoder.bias_hh_l%d" % layer] = _randn(g, 4 * D, std=0.05)

    def linear(prefix, out_f, in_f, gain=1.0, bias=True):
        sd[prefix + ".weight"] = _randn(g, out_f, in_f, std=gain / math.sqrt(in_f))
        if bias:
            sd[prefix + ".bias"] = _randn(g, out_f, std=0.02)

    def norm(prefix, n):
        sd[prefix + ".weight"] = 1.0 + _randn(g, n, std=0.1)
        sd[prefix + ".bias"] = _randn(g, n, std=0.05)

    def ffn(prefix, res):
        linear(prefix + ".feed_forward.w_1", SEACO_FFN, D)
        sd[prefix + ".feed_forward.w_2.weight"] = _randn(g, D, SEACO_FFN, std=res / math.sqrt(SEACO_FFN))
        norm(prefix + ".feed_forward.norm", SEACO_FFN)

    for i in range(SEACO_LAYERS):
        p = "seaco_decoder.decoders.%d" % i
        sd[p + ".self_attn.fsmn_block.weight"] = _randn(g, D, 1, SEACO_KERNEL, std=0.1)
        linear(p + ".src_attn.linear_q", D, D, gain=1.5)
        linear(p + ".src_attn.linear_k_v", 2 * D, D, gain=1.5)
        linear(p + ".src_attn.linear_out", D, D, gain=0.5)
        ffn(p, 0.3)
        norm(p + ".norm1", D)
        norm(p + ".norm2", D)
        norm(p + ".norm3", D)
    norm("seaco_decoder.after_norm", D)
    ffn("seaco_decoder.decoders3.0", 0.7)
    norm("seaco_decoder.decoders3.0.norm1", D)
    linear("hotword_output_layer", V, D, gain=3.0)
    sd["hotword_output_layer.bias"][seaco_no_bias_id(cfg)] = 3.0     # most positions vote NO_BIAS, some pick a hotword token
    return sd


def make_hotwords(n: int, vocab: int, seed: int = 7, sos: int = 1):
    """n random hotword token-id sequences (len 2..6) + the trailing [sos] entry generate_hotwords_list appends
    (contextual_paraformer/model.py:606-607)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        ln = int(torch.randint(2, 7, (1,), generator=g))
        out.append(torch.randint(3, vocab - 1, (ln,), generator=g).tolist())
    return out + [[sos]]


@dataclass(frozen=True)
class SenseVoiceConfig:
    """SenseVoiceSmall (funasr/models/sense_voice/model.py:489-1034; runtime/triton_gpu/.../config.yaml): the same SAN-M
    encoder (50 blocks) + 20 "tp" blocks, LayerNorm eps 1e-5, CTC head over 25055 tokens, 4 prepended query frames."""
    n_mels: int = 80
    lfr_m: int = 7
    lfr_n: int = 6
    d_model: int = 512
    heads: int = 4
    ffn: int = 2048
    enc_layers: int = 50
    tp_layers: int = 20
    kernel: int = 11
    vocab: int = 25055
    n_embed: int = 16          # 7 + len(lid_dict) + len(textnorm_dict), model.py:735
    ln_eps: float = 1e-5       # torch.nn.LayerNorm default, model.py:300-322

    @property
    def feat_dim(self) -> int:
        return self.n_mels * self.lfr_m


SENSEVOICE_SMALL = SenseVoiceConfig()
SENSEVOICE_TINY = SenseVoiceConfig(enc_layers=3, tp_layers=2, vocab=1200)


def make_sensevoice_state_dict(cfg: SenseVoiceConfig = SENSEVOICE_SMALL, seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """Synthetic SenseVoiceSmall weights under the reference's names (encoder.*, ctc.ctc_lo.*, embed.weight)."""
    g = torch.Generator().manual_seed(1000003 * seed + 29)
    D, F, V, K, Din = cfg.d_model, cfg.ffn, cfg.vocab, cfg.kernel, cfg.feat_dim
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()

    def linear(prefix, out_f, in_f, gain=1.0):
        sd[prefix + ".weight"] = _randn(g, out_f, in_f, std=gain / math.sqrt(in_f))
        sd[prefix + ".bias"] = _randn(g, out_f, std=0.02)

    def norm(prefix, n):
        sd[prefix + ".weight"] = 1.0 + _randn(g, n, std=0.1)
        sd[prefix + ".bias"] = _randn(g, n, std=0.05)

    def enc_layer(prefix, in_size):
        res = 0.7 if in_size != D else 0.3
        linear(prefix + ".self_attn.linear_out", D, D, gain=res)
        linear(prefix + ".self_attn.linear_q_k_v", 3 * D, in_size, gain=1.5)
        sd[prefix + ".self_attn.linear_q_k_v.weight"][: 2 * D] *= 1.5
        sd[prefix + ".self_attn.fsmn_block.weight"] = _randn(g, D, 1, K, std=0.15)
        linear(prefix + ".feed_forward.w_1", F, D)
        linear(prefix + ".feed_forward.w_2", D, F, gain=res)
        norm(prefix + ".norm1", in_size)
        norm(prefix + ".norm2", D)

    enc_layer("encoder.encoders0.0", Din)
    for i in range(cfg.enc_layers - 1):
        enc_layer("encoder.encoders.%d" % i, D)
    for i in range(cfg.tp_layers):
        enc_layer("encoder.tp_encoders.%d" % i, D)
    norm("encoder.after_norm", D)
    norm("encoder.tp_norm", D)
    linear("ctc.ctc_lo", V, D, gain=3.0)
    sd["ctc.ctc_lo.bias"][0] += 2.0       # CTC blank gets a head start so that blanks / repeats actually occur
    sd["embed.weight"] = _randn(g, cfg.n_embed, Din, std=1.0)
    return sd


def make_cmvn(cfg: ParaformerConfig = PARAFORMER_LARGE, seed: int = 0) -> torch.Tensor:
    """A plausible [2, 560] (shift, scale) pair.  Log-mel energies of 16-bit-scaled synthetic audio sit
    near 13 (low bins) .. 21 (high bins) with unit-ish spread, so shift ~ -(that), scale ~ 1."""
    g = torch.Generator().manual_seed(7919 * seed + 5)
    mel = torch.arange(cfg.n_mels, dtype=torch.float32) / (cfg.n_mels - 1)
    mean = (14.0 + 5.0 * mel).repeat(cfg.lfr_m)
    shift = -(mean + _randn(g, cfg.feat_dim, std=0.3))
    scale = 0.8 + 0.4 * torch.rand(cfg.feat_dim, generator=g)
    return torch.stack([shift, scale]).float()


def make_wav(n_samples: int, seed: int = 0, kind: str = "speechlike") -> torch.Tensor:
    """float32 waveform in [-1, 1], 16 kHz (SURVEY.md §8d synthetic input recipe).

    ``noise``: 0.1*N(0,1).  ``speechlike``: band-limited noise bursts with independent slowly varying
    envelopes per band ("formants") plus an amplitude-modulated harmonic stack ("voicing"), so spectra
    change from frame to frame and CIF weights vary over time.
    """
    g = torch.Generator().manual_seed(104729 * seed + 11)
    noise = torch.randn(n_samples, generator=g, dtype=torch.float32)
    if kind == "noise":
        return (0.1 * noise).clamp_(-1, 1)
    spec = torch.fft.rfft(noise.double())
    freqs = torch.arange(spec.numel(), dtype=torch.float64) * (16000.0 / n_samples)
    edges = [60.0, 300.0, 600.0, 1000.0, 1500.0, 2200.0, 3000.0, 4200.0, 6000.0, 8000.0]
    n_ctrl = max(4, int(n_samples / 16000.0 * 7.0) + 2)        # ~7 envelope control points per second
    x = torch.zeros(n_samples, dtype=torch.float64)
    for lo, hi in zip(edges[:-1], edges[1:]):
        band = torch.fft.irfft(spec * ((freqs >= lo) & (freqs < hi)), n=n_samples)
        band = band / (band.std() + 1e-9)
        ctrl = torch.rand(n_ctrl, generator=g, dtype=torch.float32).double() ** 3
        env = torch.nn.functional.interpolate(ctrl[None, None, :], size=n_samples, mode="linear", align_corners=True)[0, 0]
        x += (0.02 + 0.3 * float(torch.rand(1, generator=g))) * env * band
    t = torch.arange(n_samples, dtype=torch.float64) / 16000.0
    f0 = 100.0 + 120.0 * float(torch.rand(1, generator=g))
    vib = 1.0 + 0.08 * torch.sin(2 * math.pi * 0.7 * t)
    ctrl = torch.rand(n_ctrl, generator=g, dtype=torch.float32).double() ** 2
    env = torch.nn.functional.interpolate(ctrl[None, None, :], size=n_samples, mode="linear", align_corners=True)[0, 0]
    phase = 2 * math.pi * torch.cumsum(f0 * vib / 16000.0, dim=0)
    for h in range(1, 9):
        x += (0.25 / h) * env * torch.sin(h * phase)
    x = x + 0.003 * noise.double()
    return (0.6 * x / x.abs().max()).float()


def sinusoid_inv_timescales(depth: int) -> torch.Tensor:
    """inv_timescales of SinusoidalPositionEncoder.encode (transformer/embedding.py:409-414), fp32 ops in the same order."""
    inc = torch.log(torch.tensor([10000], dtype=torch.float32)) / (depth / 2 - 1)
    return torch.exp(torch.arange(depth / 2).type(torch.float32) * (-inc))


# ------------------------------------------------------------------------------------------------------------------
# FSMN-VAD (funasr/models/fsmn_vad_streaming: encoder FSMN, template.yaml:40-52)
# ------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class VadConfig:
    input_dim: int = 400          # 80 mel x LFR 5 (lfr_n = 1)
    input_affine_dim: int = 140
    fsmn_layers: int = 4
    linear_dim: int = 250
    proj_dim: int = 128
    lorder: int = 20
    rorder: int = 0
    output_affine_dim: int = 140
    output_dim: int = 248
    lfr_m: int = 5
    lfr_n: int = 1
    n_mels: int = 80


VAD_DEFAULT = VadConfig()


def make_vad_cmvn(seed: int = 0) -> torch.Tensor:
    """[2, 400] (shift, scale) for the VAD frontend (80 mel x LFR 5)."""
    g = torch.Generator().manual_seed(6007 * seed + 3)
    mel = torch.arange(80, dtype=torch.float32) / 79
    mean = (14.0 + 5.0 * mel).repeat(5)
    shift = -(mean + _randn(g, 400, std=0.3))
    scale = 0.8 + 0.4 * torch.rand(400, generator=g)
    return torch.stack([shift, scale]).float()


def make_vad_state_dict(cfg: VadConfig = VAD_DEFAULT, seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """Synthetic FSMN-VAD weights under the reference's names (encoder.in_linear1.linear.weight ...).  Random weights alone give a
    silence posterior unrelated to the audio, so one hidden unit per layer carries a smoothed frame-energy signal from the
    features to the silence logit (silence when the CMVN-normalised log-mel energy is low); every other weight is seeded noise at a
    gain that perturbs but does not drown that signal.  The result segments bursty synthetic audio into several speech regions —
    enough for the end-point logic, the 60 s chunking and the dynamic silence schedule to be exercised."""
    g = torch.Generator().manual_seed(1000003 * seed + 131)
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    A, L, P, O, V = cfg.input_affine_dim, cfg.linear_dim, cfg.proj_dim, cfg.output_affine_dim, cfg.output_dim

    def lin(name, out_f, in_f, gain, bias=True):
        sd[name + ".linear.weight"] = _randn(g, out_f, in_f, std=gain / math.sqrt(in_f))
        if bias:
            sd[name + ".linear.bias"] = _randn(g, out_f, std=0.05)

    lin("encoder.in_linear1", A, cfg.input_dim, 0.5)
    sd["encoder.in_linear1.linear.weight"][0] = 1.0 / cfg.input_dim                 # unit 0: mean normalised log-mel energy
    sd["encoder.in_linear1.linear.bias"][0] = 0.0
    lin("encoder.in_linear2", L, A, 0.5)
    sd["encoder.in_linear2.linear.weight"][0] = 0.0
    sd["encoder.in_linear2.linear.weight"][0, 0] = 1.0
    sd["encoder.in_linear2.linear.bias"][0] = 4.0                                   # silence (~ -7) -> 0 after ReLU, speech (~ 0) -> ~4
    for i in range(cfg.fsmn_layers):
        p = "encoder.fsmn.%d" % i
        lin(p + ".linear", P, L, 0.4, bias=False)
        sd[p + ".linear.linear.weight"][0] = 0.0
        sd[p + ".linear.linear.weight"][0, 0] = 1.0
        sd[p + ".fsmn_block.conv_left.weight"] = _randn(g, P, 1, cfg.lorder, 1, std=0.03)
        sd[p + ".fsmn_block.conv_left.weight"][0] = 0.025                           # energy channel: 20-frame smoothing
        lin(p + ".affine", L, P, 0.5)
        sd[p + ".affine.linear.weight"][0] = 0.0
        sd[p + ".affine.linear.weight"][0, 0] = 0.66
        sd[p + ".affine.linear.bias"][0] = 0.0
    lin("encoder.out_linear1", O, L, 0.5)
    sd["encoder.out_linear1.linear.weight"][0] = 0.0
    sd["encoder.out_linear1.linear.weight"][0, 0] = 1.0
    sd["encoder.out_linear1.linear.bias"][0] = 0.0
    lin("encoder.out_linear2", V, O, 0.4)
    sd["encoder.out_linear2.linear.weight"][:, 0] = 0.0
    sd["encoder.out_linear2.linear.weight"][0, 0] = -1.4                            # silence logit falls with energy
    sd["encoder.out_linear2.linear.bias"][0] = 8.0
    return sd


def make_vad_wav(seconds: float, seed: int = 0, pattern=None) -> torch.Tensor:
    """Bursty 16 kHz test audio: speech-like stretches separated by near-silence.  pattern: [(speech_s, silence_s), ...] repeated
    until `seconds`; default durations are drawn from the seed."""
    n = int(seconds * 16000)
    g = torch.Generator().manual_seed(7001 * seed + 19)
    base = make_wav(min(n, 480000), 900 + seed, "speechlike")
    reps = (n + base.numel() - 1) // base.numel()
    x = base.repeat(reps)[:n].clone()
    env = torch.zeros(n)
    pos, k = int(0.3 * 16000 * float(torch.rand(1, generator=g))), 0
    while pos < n:
        if pattern:
            sp, sl = pattern[k % len(pattern)]
        else:
            sp, sl = 0.6 + 5.0 * float(torch.rand(1, generator=g)), 0.15 + 2.8 * float(torch.rand(1, generator=g)) ** 2
        a, b = pos, min(n, pos + int(sp * 16000))
        env[a:b] = 1.0
        pos = b + int(sl * 16000)
        k += 1
    ramp = 160
    kern = torch.ones(1, 1, ramp) / ramp
    env = torch.nn.functional.conv1d(torch.nn.functional.pad(env[None, None], (ramp // 2, ramp - ramp // 2 - 1)), kern)[0, 0]
    noise = torch.randn(n, generator=g) * 0.0015
    return (x * env + noise).clamp_(-1, 1).float().contiguous()


# ------------------------------------------------------------------------------------------------------------------
# CT-Transformer punctuation (funasr/models/ct_transformer: template.yaml:9-45)
# ------------------------------------------------------------------------------------------------------------------
PUNC_LIST = ["<unk>", "_", "，", "。", "？", "、"]
PUNC_VOCAB, PUNC_DIM, PUNC_HEADS, PUNC_FFN, PUNC_LAYERS = 600, 256, 8, 1024, 4


def punc_token_list():
    """Synthetic vocabulary: CJK characters plus a few lower-case English words (the model sees both kinds)."""
    words = ["the", "a", "of", "hello", "world", "speech", "model", "is", "fast", "gpu", "we", "test", "it", "now", "today", "and"]
    return ["<blank>", "<s>", "</s>"] + [chr(0x4E00 + i) for i in range(PUNC_VOCAB - 4 - len(words))] + words + ["<unk>"]


def make_punc_state_dict(seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """CTTransformer weights under the reference's names: embed.weight [V, 256], encoder.* (SANMEncoder d=256, 8 heads, FFN 1024, 4 blocks),
    decoder.{weight [6, 256], bias}; decoder gain / bias chosen so that all punctuation classes occur."""
    g = torch.Generator().manual_seed(1000003 * seed + 211)
    D, F, K = PUNC_DIM, PUNC_FFN, 11
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    sd["embed.weight"] = _randn(g, PUNC_VOCAB, D, std=1.0)

    def layer(p):
        sd[p + ".self_attn.linear_q_k_v.weight"] = _randn(g, 3 * D, D, std=1.2 / math.sqrt(D))
        sd[p + ".self_attn.linear_q_k_v.bias"] = _randn(g, 3 * D, std=0.02)
        sd[p + ".self_attn.linear_out.weight"] = _randn(g, D, D, std=0.5 / math.sqrt(D))
        sd[p + ".self_attn.linear_out.bias"] = _randn(g, D, std=0.02)
        sd[p + ".self_attn.fsmn_block.weight"] = _randn(g, D, 1, K, std=0.1)
        sd[p + ".feed_forward.w_1.weight"] = _randn(g, F, D, std=1.0 / math.sqrt(D))
        sd[p + ".feed_forward.w_1.bias"] = _randn(g, F, std=0.02)
        sd[p + ".feed_forward.w_2.weight"] = _randn(g, D, F, std=0.5 / math.sqrt(F))
        sd[p + ".feed_forward.w_2.bias"] = _randn(g, D, std=0.02)
        for n in ("norm1", "norm2"):
            sd[p + ".%s.weight" % n] = 1.0 + _randn(g, D, std=0.1)
            sd[p + ".%s.bias" % n] = _randn(g, D, std=0.05)

    layer("encoder.encoders0.0")
    for i in range(PUNC_LAYERS - 1):
        layer("encoder.encoders.%d" % i)
    sd["encoder.after_norm.weight"] = 1.0 + _randn(g, D, std=0.1)
    sd["encoder.after_norm.bias"] = _randn(g, D, std=0.05)
    sd["decoder.weight"] = _randn(g, len(PUNC_LIST), D, std=2.0 / math.sqrt(D))
    sd["decoder.bias"] = torch.tensor([-6.0, 2.2, 0.6, 0.0, -0.6, -0.3])
    return sd


def make_punc_text(n_words: int, seed: int = 0) -> str:
    """Unpunctuated mixed Chinese / English text: characters run together, English words separated by spaces."""
    g = torch.Generator().manual_seed(31337 * seed + 7)
    toks = punc_token_list()
    out, prev_latin = [], False
    for _ in range(n_words):
        if float(torch.rand(1, generator=g)) < 0.2:
            w = toks[PUNC_VOCAB - 1 - 16 + int(torch.randint(0, 16, (1,), generator=g))]
            out.append((" " if out else "") + w + " ")
        else:
            out.append(toks[3 + int(torch.randint(0, PUNC_VOCAB - 4 - 16, (1,), generator=g))])
    return "".join(out).replace("  ", " ").strip()


# ------------------------------------------------------------------------------------------------------------------
# CAM++ speaker model (funasr/models/campplus: template.yaml) and multi-speaker recordings
# ------------------------------------------------------------------------------------------------------------------
def make_campplus_state_dict(seed: int = 0, bn_stats=None) -> "OrderedDict[str, torch.Tensor]":
    """CAMPPlus weights under the reference's names (campplus_specs): kaiming-normal convs (the reference's own init for Conv1d),
    BatchNorm affines near identity, running statistics mean 0 / var 1.  bn_stats: {name: tensor} overlaid on the running statistics
    (the calibrated ones the fixtures store: with identity statistics random-weight embeddings of different voices collapse)."""
    from .campplus import campplus_specs
    g = torch.Generator().manual_seed(60013 * seed + 5)
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for name, shape in campplus_specs().items():
        leaf = name.rsplit(".", 1)[1]
        if leaf == "num_batches_tracked":
            sd[name] = torch.tensor(0, dtype=torch.long)
        elif leaf == "running_mean":
            sd[name] = torch.zeros(shape)
        elif leaf == "running_var":
            sd[name] = torch.ones(shape)
        elif len(shape) == 1:       # BN affine or conv bias
            is_bn_w = leaf == "weight"
            sd[name] = (1.0 + _randn(g, *shape, std=0.1)) if is_bn_w else _randn(g, *shape, std=0.05)
        else:
            fan_in = int(math.prod(shape[1:]))
            sd[name] = _randn(g, *shape, std=math.sqrt(2.0 / fan_in))
    for k, v in (bn_stats or {}).items():
        sd[k] = torch.as_tensor(v).to(sd[k].dtype).reshape(sd[k].shape).clone()
    return sd


# (f0 Hz, formant Hz, syllable rate Hz) of the synthetic voices
VOICES = [(110.0, 700.0, 2.5), (230.0, 1800.0, 7.0), (160.0, 1200.0, 4.5)]


def make_voice_wav(pattern, seed: int = 0, lead_s: float = 0.5) -> torch.Tensor:
    """Multi-speaker 16 kHz test audio: pattern [(voice index, speech_s, silence_s), ...].  Every voice is a harmonic stack on its own
    f0 with intonation, shaped by one formant resonance that moves with the voice's own syllable rhythm; bursts are separated by
    near-silence so a VAD cuts them apart.  The voices differ in how their spectra change over time, which survives the per-utterance
    mean subtraction of a speaker model's frontend (a static spectral difference would not)."""
    g = torch.Generator().manual_seed(7919 * seed + 3)
    total = lead_s + sum(sp + sl for _, sp, sl in pattern)
    n = int(total * 16000)
    x = torch.zeros(n, dtype=torch.float64)
    pos = int(lead_s * 16000)
    for v, sp, sl in pattern:
        f0, fm, rate = VOICES[v]
        m = int(sp * 16000)
        t = torch.arange(m, dtype=torch.float64) / 16000.0
        phase0 = 2 * math.pi * float(torch.rand(1, generator=g))
        syl = torch.sin(math.pi * rate * t + phase0) ** 2                         # one syllable per half period
        inst = f0 * (1.0 + 0.08 * torch.sin(2 * math.pi * 0.5 * rate * t + phase0))
        phase = 2 * math.pi * torch.cumsum(inst, 0) / 16000.0
        form = fm * (1.0 + 0.25 * (syl - 0.5))
        y = torch.zeros(m, dtype=torch.float64)
        for h in range(1, int(4000 // f0) + 1):
            amp = torch.exp(-0.5 * ((h * inst - form) / (0.2 * fm)) ** 2) + 0.1 / h
            y += amp * torch.sin(h * phase + float(torch.rand(1, generator=g)) * 6.283)
        # breath noise in the formant band, strongest between syllables
        nz = torch.fft.rfft(torch.randn(m, generator=g, dtype=torch.float64))
        fr = torch.arange(nz.numel(), dtype=torch.float64) * (16000.0 / m)
        nz = torch.fft.irfft(nz * torch.exp(-0.5 * ((fr - 1.5 * fm) / (0.4 * fm)) ** 2), n=m)
        y = y / (y.abs().max() + 1e-9) + 0.15 * v * nz / (nz.std() + 1e-9) * (1.0 - syl)
        ramp = torch.clamp(torch.minimum(t, sp - t) / 0.02, 0.0, 1.0)
        y = y * (0.25 + 0.75 * syl) * ramp
        x[pos:pos + m] = 0.25 * y / (y.abs().max() + 1e-9)
        pos += m + int(sl * 16000)
    x += torch.randn(n, generator=g, dtype=torch.float64) * 0.0015
    return x.clamp_(-1, 1).float().contiguous()
