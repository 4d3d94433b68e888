"""Flat model file for the handle-style C API (csrc/offline_asr.cu: fa_offline_init).

One file = every tensor the path needs under FunASR's own state_dict names (so it can be produced from an unmodified
model.pt + am.mvn), plus the derived tables the kernels take as inputs:

    __config__                         [10] enc_layers, dec_layers, d_model, heads, fsmn kernel, vocab, feat_dim, ln_eps,
                                            cif threshold, tail threshold
    frontend.mel_banks [80,257], frontend.window [400], frontend.cmvn [2,560] (optional)
    encoder.pe_inv_timescales [280]    SinusoidalPositionEncoder timescales (transformer/embedding.py:409-414)
    predictor.cif_conv1d.gemm_weight   Conv1d(512,512,3) weight repacked to a [512, 3*512] GEMM weight

A BiCifParaformer (CifPredictorV3 with the upsampled timestamp head, recognised by predictor.upsample_cnn.weight) also carries
the head in the form the library's launches take it (`timestamp_head_tensors`, the one owner of this repack):

    predictor.upsample_cnn.gemm_weight [3*512, 512] ConvTranspose1d(512,512,3,stride 3) weight as a GEMM weight, W[k*512+o, c] = w[c,o,k]
    predictor.upsample_cnn.gemm_bias   [3*512]      its bias repeated 3x
    predictor.blstm.ih_gemm_weight     [8*512, 512] [weight_ih_l0; weight_ih_l0_reverse]: both input projections as one GEMM
    predictor.blstm.ih_gemm_bias       [8*512]      [bias_ih_l0 + bias_hh_l0; bias_ih_l0_reverse + bias_hh_l0_reverse]
    predictor.blstm.weight_hh_l0 / weight_hh_l0_reverse [4*512, 512], predictor.cif_output2.weight [1, 1024] / .bias [1]
                                                    (the reference's names, copied like every predictor.* tensor)
    __ts_config__                      [3] upsample_times, smooth_factor2, noise_threshold2

A SeacoParaformer file (`write_seaco_model_file`, recognised by __seaco_config__) adds seaco_decoder.*, hotword_output_layer.* and
bias_encoder.* under the reference's names, and

    bias_encoder.gemm_bias_l{k} [2048]  bias_ih_l{k} + bias_hh_l{k}: the hotword LSTM's input-projection GEMM bias
    __seaco_config__                    [3] no_bias, nfilter, LSTM layers

The FSMN-VAD file (csrc/offline_vad.cu: fa_vad_init) uses the same layout: the encoder's weights under the reference's names
(encoder.in_linear1.linear.weight, encoder.fsmn.{i}.fsmn_block.conv_left.weight, ...), frontend.mel_banks / window / cmvn [2, 400]
and

    __vad_config__                     [50] the bytes of 25 float64 values: the VADXOptions fields in FaVadOptions order (14 integer
                                            fields, then speech_2_noise_ratio, snr_thres, decibel_thres, speech_noise_thres,
                                            fe_prior_thres), lorder, len(sil_pdf_ids), sil_pdf_ids padded to 4

The detector compares posteriors in double precision against speech_noise_thres and fe_prior_thres, so the options travel as float64.

The CT-Transformer punctuation file (csrc/offline_punc.cu: fa_punc_init) holds embed.weight, encoder.encoders0.0.*, encoder.encoders.{i}.*,
encoder.after_norm.* and decoder.* under the reference's names, the derived encoder.pe_inv_timescales [embed_unit / 2], and

    __punc_config__                    [6] layers, d_model, heads, fsmn kernel, sentence_end_id, split_size (20)
    __punc_list__ / __punc_tokens__    the UTF-8 bytes of punc_list / token_list, newline-joined, zero-padded to a multiple of 4 and
                                       stored as the bytes of an fp32 tensor (like __vad_config__); the handle keeps them on the host

The SenseVoiceSmall file (csrc/offline_asr.cu: fa_offline_init, recognised by __sv_config__) holds encoder.encoders0.0.*,
encoder.encoders.{i}.*, encoder.after_norm.*, encoder.tp_encoders.{i}.*, encoder.tp_norm.*, ctc.ctc_lo.* and embed.weight under the
reference's names, the frontend tables and encoder.pe_inv_timescales of the Paraformer file, and

    __sv_config__                      [9] enc_layers, tp_layers, d_model, heads, fsmn kernel, vocab, feat_dim, ln_eps, blank_id

The CAM++ speaker file (csrc/offline_spk.cu: fa_spk_init, recognised by __spk_config__) holds every CAMPPlus state_dict tensor
(head.*, xvector.*) under the reference's names, unfolded and without num_batches_tracked, frontend.mel_banks [80, 257] and the povey
window frontend.window [400] (torchaudio kaldi.fbank's defaults), and

    __spk_config__                     [5] feat_dim 80, embedding 192, growth 32, bn_size 4, init_channels 128

The handle folds the BatchNorms itself, in float64, the same way CampplusEngine does.

The MonotonicAligner (fa-zh) file (csrc/offline_align.cu: fa_align_init, recognised by __aligner_config__) holds encoder.* under the
reference's names, the timestamp head as `timestamp_head_tensors` repacks it (at the model's width: 320 for fa-zh), __ts_config__ with
its BiCif meaning, the frontend tables and encoder.pe_inv_timescales of the Paraformer file, and

    __aligner_config__                 [7] enc_layers, d_model, heads, feat_dim, ln_eps, cif threshold, eos_id (the index of "</s>" in the
                                           token list, -1 without one)

predictor.cif_conv1d / cif_output are left out: get_upsample_timestamp does not read them.

Layout: b"FAB2MDL1", u32 n_tensors, then per tensor: u32 name_len, name (utf-8), u32 ndim, i64 dims[ndim], u64 nbytes,
zero padding to a 16-byte file offset, little-endian fp32 data.
"""
from __future__ import annotations

import struct
from typing import Dict, Optional

import numpy as np
import torch

from .synth import ParaformerConfig, sinusoid_inv_timescales

MAGIC = b"FAB2MDL1"


def _frontend_tensors(out: Dict[str, np.ndarray], cmvn: Optional[torch.Tensor], feat_dim: int) -> None:
    """The derived tables of a recogniser file: mel banks, window, optional CMVN and the encoder's PE timescales."""
    from .engine import kaldi_mel_banks
    out["frontend.mel_banks"] = kaldi_mel_banks().numpy()
    out["frontend.window"] = torch.hamming_window(400, periodic=False, alpha=0.54, beta=0.46, dtype=torch.float32).numpy()
    if cmvn is not None:
        out["frontend.cmvn"] = cmvn.detach().float().cpu().numpy()
    out["encoder.pe_inv_timescales"] = sinusoid_inv_timescales(feat_dim).float().numpy()


def model_tensors(state: Dict[str, torch.Tensor], cfg: ParaformerConfig, cmvn: Optional[torch.Tensor], smooth_factor2: float = 0.25,
                  noise_threshold2: float = 0.01) -> Dict[str, np.ndarray]:
    out: Dict[str, np.ndarray] = {}
    out["__config__"] = np.array([cfg.enc_layers, cfg.dec_layers, cfg.d_model, cfg.heads, cfg.kernel, cfg.vocab, cfg.feat_dim,
                                  cfg.ln_eps, cfg.cif_threshold, cfg.tail_threshold], dtype=np.float32)
    _frontend_tensors(out, cmvn, cfg.feat_dim)
    for k, v in state.items():
        if k.startswith(("encoder.", "predictor.", "decoder.", "bias_encoder.", "bias_embed.")) and torch.is_floating_point(v):
            out[k] = v.detach().float().cpu().contiguous().numpy()
    cw = state["predictor.cif_conv1d.weight"].detach().float().cpu()
    out["predictor.cif_conv1d.gemm_weight"] = cw.permute(0, 2, 1).reshape(cw.shape[0], -1).contiguous().numpy()
    if "predictor." + TS_HEAD_KEY in state:
        for k, v in timestamp_head_tensors(state).items():
            out[k] = v.cpu().numpy()
        up_times = int(state["predictor." + TS_HEAD_KEY].shape[2])
        out["__ts_config__"] = np.array([up_times, smooth_factor2, noise_threshold2], dtype=np.float32)
    return out


def write_model_file(path: str, state: Dict[str, torch.Tensor], cfg: ParaformerConfig, cmvn: Optional[torch.Tensor] = None,
                     smooth_factor2: float = 0.25, noise_threshold2: float = 0.01) -> int:
    """smooth_factor2 / noise_threshold2: CifPredictorV3's predictor_conf values (paraformer-large-vad-punc's by default); used only
    when the state dict has the BiCif timestamp head."""
    return _write(path, model_tensors(state, cfg, cmvn, smooth_factor2, noise_threshold2))


def seaco_model_tensors(state: Dict[str, torch.Tensor], cfg: ParaformerConfig, cmvn: Optional[torch.Tensor] = None, no_bias: int = 8377,
                        nfilter: int = 50, smooth_factor2: float = 0.25, noise_threshold2: float = 0.01) -> Dict[str, np.ndarray]:
    """The tensors of a SeacoParaformer model file: everything `model_tensors` writes (the BiCif timestamp head included; decoder.embed.0
    is the hotword embedding table), seaco_decoder.*, hotword_output_layer.* and bias_encoder.* under the reference's names, plus
    bias_encoder.gemm_bias_l{k} = bias_ih_l{k} + bias_hh_l{k} (the input projection's GEMM bias) and __seaco_config__ [no_bias, nfilter,
    lstm layers].  nfilter travels with the file because it is a model choice: the attention-score filter keeps that many hotwords."""
    if any(k.startswith("lstm_proj.") for k in state):
        raise ValueError("SeACo with bias_encoder_bid (a bidirectional hotword LSTM and lstm_proj) is not supported: the handle runs the "
                         "unidirectional bias_encoder")
    if any(k.startswith("bias_embed.") for k in state) or "bias_encoder.weight_ih_l0" not in state:
        raise ValueError("SeACo with bias_encoder_type 'mean' (bias_embed, no LSTM) is not supported: the handle runs the 'lstm' "
                         "bias_encoder")
    if "hotword_output_layer.weight" not in state or not any(k.startswith("seaco_decoder.") for k in state):
        raise ValueError("not a SeacoParaformer state_dict (seaco_decoder / hotword_output_layer missing)")
    if not 0 <= int(no_bias) < cfg.vocab or int(nfilter) < 0:
        raise ValueError("no_bias must lie inside the vocabulary and nfilter must be >= 0")
    out = model_tensors(state, cfg, cmvn, smooth_factor2, noise_threshold2)
    for k, v in state.items():
        if k.startswith(("seaco_decoder.", "hotword_output_layer.")) and torch.is_floating_point(v):
            out[k] = v.detach().float().cpu().contiguous().numpy()
    layers = 0
    while "bias_encoder.weight_ih_l%d" % layers in state:
        f = lambda n: state["bias_encoder.%s_l%d" % (n, layers)].detach().float().cpu()      # noqa: E731
        out["bias_encoder.gemm_bias_l%d" % layers] = (f("bias_ih") + f("bias_hh")).contiguous().numpy()
        layers += 1
    out["__seaco_config__"] = np.array([int(no_bias), int(nfilter), layers], dtype=np.float32)
    return out


def write_seaco_model_file(path: str, state: Dict[str, torch.Tensor], cfg: ParaformerConfig, cmvn: Optional[torch.Tensor] = None,
                           no_bias: int = 8377, nfilter: int = 50, smooth_factor2: float = 0.25, noise_threshold2: float = 0.01) -> int:
    """A SeacoParaformer (`paraformer-zh`) model file for the handle: `seaco_model_tensors`.  no_bias: the model's NO_BIAS token id;
    nfilter: the attention-score filter's hotword count (SeacoParaformer.inference's default 50)."""
    return _write(path, seaco_model_tensors(state, cfg, cmvn, no_bias, nfilter, smooth_factor2, noise_threshold2))


def sensevoice_model_tensors(state: Dict[str, torch.Tensor], cfg, cmvn: Optional[torch.Tensor], blank_id: int = 0) -> Dict[str, np.ndarray]:
    """The tensors of a SenseVoiceSmall model file.  state: SenseVoiceSmall's state_dict; cfg: synth.SenseVoiceConfig (its ln_eps, 1e-5,
    travels in the file: the handle's Paraformer default is 1e-12)."""
    if "embed.weight" not in state or "ctc.ctc_lo.weight" not in state or "encoder.encoders0.0.norm1.weight" not in state:
        raise ValueError("not a SenseVoiceSmall state_dict (embed.weight / ctc.ctc_lo / encoder.encoders0.0 missing)")
    out: Dict[str, np.ndarray] = {}
    out["__sv_config__"] = np.array([cfg.enc_layers, cfg.tp_layers, cfg.d_model, cfg.heads, cfg.kernel, cfg.vocab, cfg.feat_dim, cfg.ln_eps,
                                     blank_id], dtype=np.float32)
    _frontend_tensors(out, cmvn, cfg.feat_dim)
    for k, v in state.items():
        if k.startswith(("encoder.", "ctc.", "embed.")) and torch.is_floating_point(v):
            out[k] = v.detach().float().cpu().contiguous().numpy()
    return out


def aligner_model_tensors(state: Dict[str, torch.Tensor], cfg: ParaformerConfig, cmvn: Optional[torch.Tensor], token_list=None,
                          smooth_factor2: float = 0.25, noise_threshold2: float = 0.01) -> Dict[str, np.ndarray]:
    """The tensors of a MonotonicAligner model file.  state: MonotonicAligner's state_dict (synth.make_aligner_state_dict uses the same
    names); cfg: its encoder shape and CIF threshold; cmvn: am.mvn as [2, 560]; token_list: the tokenizer's list, which only gives
    eos_id; smooth_factor2 / noise_threshold2: CifPredictorV3's predictor_conf values."""
    if "encoder.encoders0.0.norm1.weight" not in state or "predictor." + TS_HEAD_KEY not in state:
        raise ValueError("not a MonotonicAligner state_dict (encoder.encoders0.0 / predictor.upsample_cnn missing)")
    eos_id = list(token_list).index("</s>") if token_list is not None and "</s>" in token_list else -1
    out: Dict[str, np.ndarray] = {}
    out["__aligner_config__"] = np.array([cfg.enc_layers, cfg.d_model, cfg.heads, cfg.feat_dim, cfg.ln_eps, cfg.cif_threshold, eos_id],
                                         dtype=np.float32)
    _frontend_tensors(out, cmvn, cfg.feat_dim)
    for k, v in state.items():
        if k.startswith("encoder.") and torch.is_floating_point(v):
            out[k] = v.detach().float().cpu().contiguous().numpy()
    for k, v in timestamp_head_tensors(state).items():
        out[k] = v.cpu().numpy()
    up_times = int(state["predictor." + TS_HEAD_KEY].shape[2])
    out["__ts_config__"] = np.array([up_times, smooth_factor2, noise_threshold2], dtype=np.float32)
    return out


def write_aligner_model_file(path: str, state: Dict[str, torch.Tensor], cfg: ParaformerConfig, cmvn: Optional[torch.Tensor] = None,
                             token_list=None, smooth_factor2: float = 0.25, noise_threshold2: float = 0.01) -> int:
    """A MonotonicAligner (fa-zh) model file for the forced-alignment handle (fa_align_init): `aligner_model_tensors`."""
    return _write(path, aligner_model_tensors(state, cfg, cmvn, token_list, smooth_factor2, noise_threshold2))


def campplus_model_tensors(state: Dict[str, torch.Tensor]) -> Dict[str, np.ndarray]:
    """The CAM++ speaker file's tensors; refuses any state_dict that is not CAMPPlusB200's template.yaml shape."""
    from .campplus import BN_CH, EMB_DIM, FEAT_DIM, GROWTH, INIT_CH, campplus_specs, povey_window
    from .engine import kaldi_mel_banks
    out: Dict[str, np.ndarray] = {}
    for name, shape in campplus_specs().items():
        if name.endswith("num_batches_tracked"):
            continue
        if name not in state:
            raise ValueError("CAM++ state_dict lacks %s (CAMPPlusB200 is built for the template.yaml shape: feat 80, embedding 192, "
                             "growth 32, bn_size 4, init 128)" % name)
        v = state[name]
        if tuple(v.shape) != tuple(shape):
            raise ValueError("CAM++ tensor %s has shape %s, the template.yaml shape needs %s" % (name, tuple(v.shape), tuple(shape)))
        out[name] = v.detach().float().cpu().contiguous().numpy()
    out["frontend.mel_banks"] = kaldi_mel_banks().numpy()
    out["frontend.window"] = povey_window().numpy()
    out["__spk_config__"] = np.array([FEAT_DIM, EMB_DIM, GROWTH, BN_CH // GROWTH, INIT_CH], dtype=np.float32)
    return out


def write_campplus_model_file(state: Dict[str, torch.Tensor], path: str) -> int:
    """CAMPPlus state_dict -> the speaker handle's model file (fa_spk_init)."""
    return _write(path, campplus_model_tensors(state))


def write_sensevoice_model_file(path: str, state: Dict[str, torch.Tensor], cfg, cmvn: Optional[torch.Tensor] = None, blank_id: int = 0) -> int:
    return _write(path, sensevoice_model_tensors(state, cfg, cmvn, blank_id))


TS_HEAD_KEY = "upsample_cnn.weight"


def timestamp_head_tensors(state: Dict[str, torch.Tensor], prefix: str = "predictor.") -> Dict[str, torch.Tensor]:
    """CifPredictorV3's timestamp head (bicif_paraformer/cif_predictor.py:121-352, upsample_type "cnn_blstm") repacked for this
    library's launches, on the device the state lives on: {name: fp32 tensor} under the names of the module docstring.  Both the
    engine (engine.py:_init_timestamp_head) and the model file take the head from here."""
    uw = state[prefix + TS_HEAD_KEY].detach().float()                     # ConvTranspose1d weight [in, out, k], stride == k
    up_times = int(uw.shape[2])
    bp = prefix + "blstm."
    f = lambda k: state[k].detach().float()                               # noqa: E731
    return {
        # out[b, 3t+k, o] = sum_c x[b,t,c] w[c,o,k] + bias[o]  ==  one GEMM with W[(k,o), c], rows viewed as [B, 3T, D]
        prefix + "upsample_cnn.gemm_weight": uw.permute(2, 1, 0).reshape(-1, uw.shape[0]).contiguous(),
        prefix + "upsample_cnn.gemm_bias": f(prefix + "upsample_cnn.bias").repeat(up_times).contiguous(),
        bp + "ih_gemm_weight": torch.cat([f(bp + "weight_ih_l0"), f(bp + "weight_ih_l0_reverse")], 0).contiguous(),
        bp + "ih_gemm_bias": torch.cat([f(bp + "bias_ih_l0") + f(bp + "bias_hh_l0"),
                                        f(bp + "bias_ih_l0_reverse") + f(bp + "bias_hh_l0_reverse")], 0).contiguous(),
        bp + "weight_hh_l0": f(bp + "weight_hh_l0").contiguous(),
        bp + "weight_hh_l0_reverse": f(bp + "weight_hh_l0_reverse").contiguous(),
        prefix + "cif_output2.weight": f(prefix + "cif_output2.weight").contiguous(),
        prefix + "cif_output2.bias": f(prefix + "cif_output2.bias").contiguous(),
    }


VAD_INT_FIELDS = ("sample_rate", "detect_mode", "max_end_silence_time", "max_start_silence_time", "window_size_ms", "sil_to_speech_time_thres",
                  "speech_to_sil_time_thres", "do_extend", "lookback_time_start_point", "lookahead_time_end_point", "max_single_segment_time",
                  "noise_frame_num_used_for_snr", "frame_in_ms", "frame_length_ms")
VAD_REAL_FIELDS = ("speech_2_noise_ratio", "snr_thres", "decibel_thres", "speech_noise_thres", "fe_prior_thres")


def vad_model_tensors(state: Dict[str, torch.Tensor], cmvn: Optional[torch.Tensor], vad_conf: Optional[dict] = None) -> Dict[str, np.ndarray]:
    """The tensors of a FSMN-VAD model file.  state: FsmnVADStreaming's state_dict (encoder.* names); vad_conf: its model_conf
    (VADXOptions, `VadOptions.from_conf`), optionally with the "encoder_conf" of the model's config.  Refuses what FSMNB200 / VadEngine
    refuse."""
    from .engine import kaldi_mel_banks
    from .vad import VadOptions
    conf = dict(vad_conf or {})
    enc_conf = conf.pop("encoder_conf", None)
    if enc_conf is not None:
        from .vad_model import FSMNB200
        FSMNB200(**enc_conf)                                         # raises for the shapes the kernels are not built for
    o = VadOptions.from_conf(conf)
    if any(k.endswith("fsmn_block.conv_right.weight") for k in state):
        raise ValueError("FSMN-VAD with a right-context memory (rorder > 0) is not supported")
    n_layers = 0
    while "encoder.fsmn.%d.linear.linear.weight" % n_layers in state:
        n_layers += 1
    if n_layers == 0 or "encoder.in_linear1.linear.weight" not in state:
        raise ValueError("not an FSMN-VAD state_dict (encoder.in_linear1 / encoder.fsmn.{i} missing)")
    if tuple(state["encoder.in_linear1.linear.weight"].shape)[1:] != (400,):
        raise ValueError("the VAD frontend is 80 mel x LFR 5: in_linear1 must take 400 inputs")
    lorder = 20
    for i in range(n_layers):
        cw = state["encoder.fsmn.%d.fsmn_block.conv_left.weight" % i]
        if tuple(cw.shape) != (128, 1, lorder, 1) or state["encoder.fsmn.%d.linear.linear.weight" % i].shape[0] != 128:
            raise ValueError("FSMN-VAD layer %d: need proj 128 and lorder 20 (conv_left weight [128, 1, 20, 1])" % i)
    sil = [int(v) for v in o.sil_pdf_ids]
    if not 1 <= len(sil) <= 4:
        raise ValueError("sil_pdf_ids must hold 1 to 4 ids")
    ints = []
    for name in VAD_INT_FIELDS:
        v = getattr(o, name)
        if float(v) != int(v):
            raise ValueError("VAD option %s = %r is not a whole number" % (name, v))
        ints.append(int(v))
    if o.frame_in_ms <= 0 or o.window_size_ms < o.frame_in_ms:
        raise ValueError("VAD options need frame_in_ms > 0 and window_size_ms >= frame_in_ms")
    cfg = np.array(ints + [float(getattr(o, n)) for n in VAD_REAL_FIELDS] + [lorder, len(sil)] + sil + [0] * (4 - len(sil)), dtype="<f8")
    out: Dict[str, np.ndarray] = {"__vad_config__": cfg.view("<f4")}
    out["frontend.mel_banks"] = kaldi_mel_banks().numpy()
    out["frontend.window"] = torch.hamming_window(400, periodic=False, alpha=0.54, beta=0.46, dtype=torch.float32).numpy()
    if cmvn is not None:
        c = cmvn.detach().float().cpu().numpy()
        if c.shape != (2, 400):
            raise ValueError("the VAD's cmvn must be [2, 400]")
        out["frontend.cmvn"] = c
    for k, v in state.items():
        if k.startswith("encoder.") and torch.is_floating_point(v):
            out[k] = v.detach().float().cpu().contiguous().numpy()
    return out


def write_vad_model_file(path: str, state: Dict[str, torch.Tensor], cmvn: Optional[torch.Tensor] = None, vad_conf: Optional[dict] = None) -> int:
    return _write(path, vad_model_tensors(state, cmvn, vad_conf))


def read_vad_config(tensors: Dict[str, np.ndarray]) -> dict:
    """The options of a VAD model file read back (tests): {field: value, ..., "lorder", "sil_pdf_ids"}."""
    c = np.ascontiguousarray(tensors["__vad_config__"], dtype="<f4").view("<f8")
    n_int = len(VAD_INT_FIELDS)
    out = {n: int(c[i]) for i, n in enumerate(VAD_INT_FIELDS)}
    out.update({n: float(c[n_int + i]) for i, n in enumerate(VAD_REAL_FIELDS)})
    base = n_int + len(VAD_REAL_FIELDS)
    out["lorder"] = int(c[base])
    out["sil_pdf_ids"] = [int(v) for v in c[base + 2: base + 2 + int(c[base + 1])]]
    return out


PUNC_SPLIT_SIZE = 20


def _text_blob(items) -> np.ndarray:
    for s in items:
        if "\n" in s or "\0" in s or not s:
            raise ValueError("list entry %r: entries must be non-empty and hold no newline or NUL" % (s,))
    b = "\n".join(items).encode("utf-8")
    return np.frombuffer(b + b"\0" * ((4 - len(b) % 4) % 4), dtype="<f4").copy()


def _blob_text(arr: np.ndarray) -> list:
    return np.ascontiguousarray(arr, dtype="<f4").tobytes().rstrip(b"\0").decode("utf-8").split("\n")


def punc_model_tensors(state: Dict[str, torch.Tensor], punc_list, token_list, sentence_end_id: int, encoder_conf: dict) -> Dict[str, np.ndarray]:
    """The tensors of a CT-Transformer punctuation model file.  state: CTTransformer's state_dict; encoder_conf: its SANMEncoder conf
    (attention_heads, kernel_size; the layer count and widths are read from the weights)."""
    layers = 0
    while "encoder.encoders.%d.norm1.weight" % layers in state:
        layers += 1
    if "embed.weight" not in state or "encoder.encoders0.0.norm1.weight" not in state:
        raise ValueError("not a CT-Transformer state_dict (embed.weight / encoder.encoders0.0 missing)")
    if "<unk>" not in token_list:
        raise ValueError("token_list has no <unk> entry")
    if not 0 <= int(sentence_end_id) < len(punc_list):
        raise ValueError("sentence_end_id outside punc_list")
    layout = {k: encoder_conf.get(k, v) for k, v in (("sanm_shfit", 0), ("input_layer", "pe"), ("normalize_before", True),
                                                       ("selfattention_layer_type", "sanm"))}
    if layout != {"sanm_shfit": 0, "input_layer": "pe", "normalize_before": True, "selfattention_layer_type": "sanm"}:
        raise ValueError("the punctuation encoder runs sanm_shfit 0, input_layer \"pe\", normalize_before, \"sanm\" attention; got %r" % layout)
    d_model = int(state["encoder.after_norm.weight"].numel())
    heads = int(encoder_conf.get("attention_heads", 8))
    kernel = int(state["encoder.encoders0.0.self_attn.fsmn_block.weight"].shape[-1])
    d_in = int(state["embed.weight"].shape[1])
    out: Dict[str, np.ndarray] = {}
    out["__punc_config__"] = np.array([layers + 1, d_model, heads, kernel, int(sentence_end_id), PUNC_SPLIT_SIZE], dtype=np.float32)
    out["__punc_list__"] = _text_blob(list(punc_list))
    out["__punc_tokens__"] = _text_blob(list(token_list))
    out["encoder.pe_inv_timescales"] = sinusoid_inv_timescales(d_in).float().numpy()
    for k, v in state.items():
        if k.startswith(("embed.", "encoder.", "decoder.")) and torch.is_floating_point(v):
            out[k] = v.detach().float().cpu().contiguous().numpy()
    return out


def write_punc_model_file(path: str, state: Dict[str, torch.Tensor], punc_list, token_list, sentence_end_id: int, encoder_conf: dict) -> int:
    return _write(path, punc_model_tensors(state, punc_list, token_list, sentence_end_id, encoder_conf))


def read_punc_config(tensors: Dict[str, np.ndarray]) -> dict:
    """The configuration and both lists of a punctuation model file read back (tests)."""
    c = [int(v) for v in tensors["__punc_config__"]]
    return {"layers": c[0], "d_model": c[1], "heads": c[2], "kernel": c[3], "sentence_end_id": c[4], "split_size": c[5],
            "punc_list": _blob_text(tensors["__punc_list__"]), "token_list": _blob_text(tensors["__punc_tokens__"])}


def _write(path: str, tensors: Dict[str, np.ndarray]) -> int:
    with open(path, "wb") as f:
        f.write(MAGIC)
        f.write(struct.pack("<I", len(tensors)))
        for name, arr in tensors.items():
            arr = np.ascontiguousarray(arr, dtype="<f4")
            nb = name.encode("utf-8")
            f.write(struct.pack("<I", len(nb)))
            f.write(nb)
            f.write(struct.pack("<I", arr.ndim))
            f.write(struct.pack("<%dq" % arr.ndim, *arr.shape))
            f.write(struct.pack("<Q", arr.nbytes))
            f.write(b"\0" * ((16 - f.tell() % 16) % 16))
            f.write(arr.tobytes())
    return len(tensors)


def read_model_file(path: str) -> Dict[str, np.ndarray]:
    """Python reader of the same layout (tests; mirrors load_file() in csrc/handle_core.cu)."""
    out: Dict[str, np.ndarray] = {}
    with open(path, "rb") as f:
        if f.read(8) != MAGIC:
            raise ValueError("not a funasr_b200 model file")
        (n,) = struct.unpack("<I", f.read(4))
        for _ in range(n):
            (nl,) = struct.unpack("<I", f.read(4))
            name = f.read(nl).decode("utf-8")
            (nd,) = struct.unpack("<I", f.read(4))
            shape = struct.unpack("<%dq" % nd, f.read(8 * nd)) if nd else ()
            (nbytes,) = struct.unpack("<Q", f.read(8))
            f.seek((16 - f.tell() % 16) % 16, 1)
            out[name] = np.frombuffer(f.read(nbytes), dtype="<f4").reshape(shape)
    return out
