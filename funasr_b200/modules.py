"""Reference-shaped plugin classes backed by the CUDA library.

Each class mirrors the constructor arguments, the parameter names (state_dict keys) and the call contract of the
reference class it replaces, so FunASR's own AutoModel.build_model / load_pretrained_model drive it unchanged:

  WavFrontendB200             <- funasr/frontends/wav_frontend.py:91-196        (WavFrontend)
  SANMEncoderB200             <- funasr/models/sanm/encoder.py:188-461          (SANMEncoder)
  CifPredictorV2B200          <- funasr/models/paraformer/cif_predictor.py:209-314
  ParaformerSANMDecoderB200   <- funasr/models/paraformer/decoder.py:234-449
  ParaformerB200              <- funasr/models/paraformer/model.py:30-697       (Paraformer, inference path)

The modules are torch.nn.Module only as *parameter containers* (so load_state_dict(strict=True), .to(device) and
.eval() work as the reference expects); no torch.nn op runs on the hot path, and there is no CPU fallback —
calling them without CUDA or without the built library raises.
"""
from __future__ import annotations

import time
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import _abi
from .engine import AlignerEngine, FrontendEngine, ParaformerEngine, SenseVoiceEngine, num_lfr_frames
from .hotwords import generate_hotwords_list
from .registry import get_tables, register
from .synth import ParaformerConfig, SenseVoiceConfig


class _Container(nn.Module):
    """Plain container so dotted parameter names reproduce the reference's state_dict keys."""


def _add_param(root: nn.Module, dotted: str, shape) -> None:
    parts = dotted.split(".")
    mod = root
    for p in parts[:-1]:
        if not hasattr(mod, p):
            mod.add_module(p, _Container())
        mod = getattr(mod, p)
    mod.register_parameter(parts[-1], nn.Parameter(torch.zeros(*shape), requires_grad=False))


class _ParamHolder(nn.Module):
    def _specs(self) -> Dict[str, tuple]:
        raise NotImplementedError

    def _build(self):
        for name, shape in self._specs().items():
            _add_param(self, name, shape)

    def forward(self, *a, **k):  # pragma: no cover
        raise _abi.FunasrB200Error("%s runs only inside ParaformerB200 on a CUDA device" % type(self).__name__)


def load_cmvn(cmvn_file: str) -> torch.Tensor:
    """Kaldi-nnet text `am.mvn` -> [2, dim] (shift, scale); same parse as load_cmvn (wav_frontend.py:15-43):
    the row after <AddShift>/<Rescale> starting with <LearnRateCoef>, tokens [3:-1]."""
    with open(cmvn_file, "r", encoding="utf-8") as f:
        lines = f.readlines()
    means, scales = [], []
    for i, line in enumerate(lines):
        item = line.split()
        if not item:
            continue
        if item[0] in ("<AddShift>", "<Rescale>") and i + 1 < len(lines):
            nxt = lines[i + 1].split()
            if nxt and nxt[0] == "<LearnRateCoef>":
                vals = nxt[3:len(nxt) - 1]
                if item[0] == "<AddShift>":
                    means = vals
                else:
                    scales = vals
    return torch.as_tensor(np.array([np.array(means).astype(np.float32), np.array(scales).astype(np.float32)]), dtype=torch.float32)


@register("frontend_classes", "WavFrontendB200")
class WavFrontendB200(nn.Module):
    """Drop-in for WavFrontend: forward(input [B,Nmax] fp32, input_lengths) -> (feats [B,Tmax,560], lens int64)."""

    def __init__(self, cmvn_file: str = None, fs: int = 16000, window: str = "hamming", n_mels: int = 80,
                 frame_length: int = 25, frame_shift: int = 10, filter_length_min: int = -1, filter_length_max: int = -1,
                 lfr_m: int = 1, lfr_n: int = 1, dither: float = 1.0, snip_edges: bool = True, upsacle_samples: bool = True,
                 device: str = "cuda", cmvn: Optional[torch.Tensor] = None, **kwargs):
        super().__init__()
        self.fs, self.window, self.n_mels = fs, window, n_mels
        self.frame_length, self.frame_shift = frame_length, frame_shift
        self.lfr_m, self.lfr_n, self.dither = lfr_m, lfr_n, dither
        self.snip_edges, self.upsacle_samples, self.cmvn_file = snip_edges, upsacle_samples, cmvn_file
        self.cmvn = cmvn if cmvn is not None else (None if cmvn_file is None else load_cmvn(cmvn_file))
        if (fs, window, n_mels, frame_length, frame_shift, lfr_m, lfr_n, snip_edges, upsacle_samples) != \
                (16000, "hamming", 80, 25, 10, 7, 6, True, True):
            raise _abi.FunasrB200Error("WavFrontendB200 is built for the Paraformer/SenseVoice frontend config "
                                       "(16 kHz, hamming 25/10 ms, 80 mel, LFR 7/6, snip_edges)")
        # dither: the reference default 1.0 adds torch.randn noise per frame (kaldi.py:179-181), which cannot be
        # reproduced bit-for-bit by construction; this backend is deterministic (== dither 0.0).
        self._device = device
        self._engine: Optional[FrontendEngine] = None

    def output_size(self) -> int:
        return self.n_mels * self.lfr_m

    def engine(self, device=None) -> FrontendEngine:
        dev = torch.device(device or self._device)
        if self._engine is None or self._engine.device != dev:
            self._engine = FrontendEngine(self.cmvn, dev)
        return self._engine

    def forward(self, input: torch.Tensor, input_lengths, device=None, **kwargs) -> Tuple[torch.Tensor, torch.Tensor]:
        eng = self.engine(device if device is not None else (input.device if input.is_cuda else None))
        lens = [int(x) for x in (input_lengths.tolist() if torch.is_tensor(input_lengths) else input_lengths)]
        if min(lens) < 2:
            raise _abi.FunasrB200Error("an utterance needs at least 2 samples (kaldi.fbank asserts 2 <= window_size)")
        t_max = max(num_lfr_frames(n) for n in lens)
        wav = input.to(eng.device, torch.float32, non_blocking=True).contiguous()
        wl = torch.tensor(lens, dtype=torch.int32).to(eng.device, non_blocking=True)
        feats, flens = eng(wav, wl, t_max, host_lens=lens)
        return feats, flens.to(torch.int64)


@register("encoder_classes", "SANMEncoderB200")
class SANMEncoderB200(_ParamHolder):
    def __init__(self, input_size: int, output_size: int = 256, attention_heads: int = 4, linear_units: int = 2048,
                 num_blocks: int = 6, kernel_size: int = 11, sanm_shfit: int = 0, input_layer: str = "pe",
                 normalize_before: bool = True, selfattention_layer_type: str = "sanm", **kwargs):
        super().__init__()
        head_dim = output_size // attention_heads if attention_heads else 0
        if (input_layer, normalize_before, selfattention_layer_type, sanm_shfit) != ("pe", True, "sanm", 0) or input_size > 560 or \
                output_size % 16 or output_size > 512 or head_dim * attention_heads != output_size or head_dim not in (32, 64, 80, 96, 128) or \
                linear_units > 2048 or input_size % 16:
            raise _abi.FunasrB200Error("SANMEncoderB200 supports input_layer='pe', sanm, normalize_before, d <= 512 (head dim 32..128), "
                                       "linear_units <= 2048 — d=512 / 4 heads (Paraformer, SenseVoice) and d=320 / 4 heads (fa-zh) run "
                                       "on the tensor cores, other shapes (CT-Transformer: d=256 / 8 heads) on the fp32 path")
        self.input_size, self._output_size = input_size, output_size
        self.heads, self.ffn, self.num_blocks, self.kernel_size = attention_heads, linear_units, num_blocks, kernel_size
        self._build()

    def output_size(self) -> int:
        return self._output_size

    def _specs(self):
        D, F, K = self._output_size, self.ffn, self.kernel_size
        s = {}

        def layer(p, in_size):
            s[p + ".self_attn.linear_out.weight"] = (D, D)
            s[p + ".self_attn.linear_out.bias"] = (D,)
            s[p + ".self_attn.linear_q_k_v.weight"] = (3 * D, in_size)
            s[p + ".self_attn.linear_q_k_v.bias"] = (3 * D,)
            s[p + ".self_attn.fsmn_block.weight"] = (D, 1, K)
            s[p + ".feed_forward.w_1.weight"] = (F, D)
            s[p + ".feed_forward.w_1.bias"] = (F,)
            s[p + ".feed_forward.w_2.weight"] = (D, F)
            s[p + ".feed_forward.w_2.bias"] = (D,)
            s[p + ".norm1.weight"] = (in_size,)
            s[p + ".norm1.bias"] = (in_size,)
            s[p + ".norm2.weight"] = (D,)
            s[p + ".norm2.bias"] = (D,)

        layer("encoders0.0", self.input_size)
        for i in range(self.num_blocks - 1):
            layer("encoders.%d" % i, D)
        s["after_norm.weight"] = (D,)
        s["after_norm.bias"] = (D,)
        return s


@register("predictor_classes", "CifPredictorV2B200")
class CifPredictorV2B200(_ParamHolder):
    def __init__(self, idim, l_order, r_order, threshold=1.0, dropout=0.1, smooth_factor=1.0, noise_threshold=0,
                 tail_threshold=0.0, tail_mask=True, **kwargs):
        super().__init__()
        if (idim, l_order, r_order, smooth_factor, noise_threshold, tail_mask) != (512, 1, 1, 1.0, 0, True) or tail_threshold <= 0:
            raise _abi.FunasrB200Error("CifPredictorV2B200 supports idim=512, l_order=r_order=1, tail_threshold>0, tail_mask")
        self.idim, self.threshold, self.tail_threshold = idim, threshold, tail_threshold
        self._build()

    def _specs(self):
        D = self.idim
        return {"cif_conv1d.weight": (D, D, 3), "cif_conv1d.bias": (D,), "cif_output.weight": (1, D), "cif_output.bias": (1,)}


@register("predictor_classes", "CifPredictorV3B200")
class CifPredictorV3B200(_ParamHolder):
    """Parameter container for CifPredictorV3 (funasr/models/bicif_paraformer/cif_predictor.py:121-352) in the configuration
    BiCifParaformer ships with (template.yaml:52-63): upsample_type "cnn_blstm", use_cif1_cnn False, upsample_times 3."""

    def __init__(self, idim, l_order, r_order, threshold=1.0, dropout=0.1, smooth_factor=1.0, noise_threshold=0, tail_threshold=0.0,
                 smooth_factor2=1.0, noise_threshold2=0, upsample_times=5, upsample_type="cnn", use_cif1_cnn=True, tail_mask=True, **kwargs):
        super().__init__()
        if idim not in (512, 320) or (l_order, r_order, smooth_factor, noise_threshold, tail_mask) != (1, 1, 1.0, 0, True) or tail_threshold <= 0:
            raise _abi.FunasrB200Error("CifPredictorV3B200 supports idim=512 or 320, l_order=r_order=1, tail_threshold>0, tail_mask")
        if upsample_type != "cnn_blstm" or use_cif1_cnn or upsample_times != 3:
            raise _abi.FunasrB200Error("CifPredictorV3B200 supports upsample_type='cnn_blstm', use_cif1_cnn=False, upsample_times=3")
        self.idim, self.threshold, self.tail_threshold = idim, threshold, tail_threshold
        self.smooth_factor2, self.noise_threshold2, self.upsample_times = float(smooth_factor2), float(noise_threshold2), upsample_times
        self._build()

    def _specs(self):
        D, U = self.idim, self.upsample_times
        s = {"cif_conv1d.weight": (D, D, 3), "cif_conv1d.bias": (D,), "cif_output.weight": (1, D), "cif_output.bias": (1,),
             "upsample_cnn.weight": (D, D, U), "upsample_cnn.bias": (D,), "cif_output2.weight": (1, 2 * D), "cif_output2.bias": (1,)}
        for suf in ("", "_reverse"):
            s["blstm.weight_ih_l0" + suf] = (4 * D, D)
            s["blstm.weight_hh_l0" + suf] = (4 * D, D)
            s["blstm.bias_ih_l0" + suf] = (4 * D,)
            s["blstm.bias_hh_l0" + suf] = (4 * D,)
        return s


@register("decoder_classes", "ParaformerSANMDecoderB200")
class ParaformerSANMDecoderB200(_ParamHolder):
    def __init__(self, vocab_size: int, encoder_output_size: int, attention_heads: int = 4, linear_units: int = 2048,
                 num_blocks: int = 6, att_layer_num: int = 6, kernel_size: int = 21, sanm_shfit: int = 0, **kwargs):
        super().__init__()
        if encoder_output_size != 512 or attention_heads != 4 or att_layer_num != num_blocks or sanm_shfit != 0:
            raise _abi.FunasrB200Error("ParaformerSANMDecoderB200 supports d=512, 4 heads, att_layer_num == num_blocks, sanm_shfit=0")
        self.vocab_size, self.D, self.ffn = vocab_size, encoder_output_size, linear_units
        self.num_blocks, self.kernel_size = num_blocks, kernel_size
        self._build()

    def _specs(self):
        D, F, K, V = self.D, self.ffn, self.kernel_size, self.vocab_size
        s = {"embed.0.weight": (V, D), "after_norm.weight": (D,), "after_norm.bias": (D,),
             "output_layer.weight": (V, D), "output_layer.bias": (V,)}

        def ffn(p):
            s[p + ".feed_forward.w_1.weight"] = (F, D)
            s[p + ".feed_forward.w_1.bias"] = (F,)
            s[p + ".feed_forward.w_2.weight"] = (D, F)
            s[p + ".feed_forward.norm.weight"] = (F,)
            s[p + ".feed_forward.norm.bias"] = (F,)

        for i in range(self.num_blocks):
            p = "decoders.%d" % i
            ffn(p)
            s[p + ".self_attn.fsmn_block.weight"] = (D, 1, K)
            for nme, shp in (("linear_q", (D, D)), ("linear_k_v", (2 * D, D)), ("linear_out", (D, D))):
                s[p + ".src_attn.%s.weight" % nme] = shp
                s[p + ".src_attn.%s.bias" % nme] = (shp[0],)
            for n in ("norm1", "norm2", "norm3"):
                s[p + ".%s.weight" % n] = (D,)
                s[p + ".%s.bias" % n] = (D,)
        ffn("decoders3.0")
        s["decoders3.0.norm1.weight"] = (D,)
        s["decoders3.0.norm1.bias"] = (D,)
        return s


def _as_wave_list(data_in, fs: int, frontend=None, audio_fs: int = 16000, **kwargs) -> List[torch.Tensor]:
    """ndarray / tensor / list thereof -> list of 1-D fp32 tensors.  Paths, bytes and urls are delegated to the
    reference's own loader (funasr.utils.load_utils.load_audio_text_image_video, model.py:578) when FunASR is
    installed; that part of the pipeline (audio decode / resample) is outside this backend's scope."""
    items = data_in if isinstance(data_in, (list, tuple)) else [data_in]
    out = []
    for x in items:
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(x)
        if not torch.is_tensor(x):
            try:
                from funasr.utils.load_utils import load_audio_text_image_video
            except Exception as e:  # pragma: no cover
                raise _abi.FunasrB200Error("only ndarray / tensor waveforms are accepted without FunASR installed") from e
            x = load_audio_text_image_video(x, fs=fs, audio_fs=audio_fs, data_type=kwargs.get("data_type", "sound"))
        x = x.to(torch.float32)
        if x.dim() > 1:
            x = x.mean(dim=0) if x.shape[0] > 1 else x[0]     # mono (load_utils.py:extract_fbank)
        out.append(x.contiguous())
    return out


@register("model_classes", "ParaformerB200")
class ParaformerB200(nn.Module):
    """Drop-in for funasr.models.paraformer.model.Paraformer on the offline greedy inference path."""

    def __init__(self, specaug=None, specaug_conf=None, normalize=None, normalize_conf=None, encoder: str = None,
                 encoder_conf: dict = None, decoder: str = None, decoder_conf: dict = None, ctc=None, ctc_conf=None,
                 predictor: str = None, predictor_conf: dict = None, ctc_weight: float = 0.0, input_size: int = 80,
                 vocab_size: int = -1, ignore_id: int = -1, blank_id: int = 0, sos: int = 1, eos: int = 2,
                 gemm_mode: str = "fp32", **kwargs):
        super().__init__()
        tables = get_tables()
        enc_cls = tables.encoder_classes.get(encoder) if isinstance(encoder, str) else encoder
        dec_cls = tables.decoder_classes.get(decoder) if isinstance(decoder, str) else decoder
        pred_cls = tables.predictor_classes.get(predictor) if isinstance(predictor, str) else predictor
        # an unmodified reference config names the reference classes; they map onto this backend's components
        enc_cls = enc_cls if (enc_cls is not None and issubclass(enc_cls, _ParamHolder)) else SANMEncoderB200
        dec_cls = dec_cls if (dec_cls is not None and issubclass(dec_cls, _ParamHolder)) else ParaformerSANMDecoderB200
        pred_cls = pred_cls if (pred_cls is not None and issubclass(pred_cls, _ParamHolder)) else CifPredictorV2B200
        self.encoder = enc_cls(input_size=input_size, **(encoder_conf or {}))                       # model.py:131-132
        self.decoder = dec_cls(vocab_size=vocab_size, encoder_output_size=self.encoder.output_size(), **(decoder_conf or {}))
        self.predictor = pred_cls(**(predictor_conf or {}))                                         # model.py:149-150
        self.vocab_size, self.ignore_id = vocab_size, ignore_id
        self.blank_id, self.sos, self.eos = blank_id, sos, eos
        self.gemm_mode = gemm_mode
        self.cfg = ParaformerConfig(enc_layers=self.encoder.num_blocks, dec_layers=self.decoder.num_blocks, vocab=vocab_size,
                                    kernel=self.encoder.kernel_size, tail_threshold=self.predictor.tail_threshold,
                                    cif_threshold=self.predictor.threshold)
        self._engine: Optional[ParaformerEngine] = None

    # -- weights enter through load_pretrained_model -> load_state_dict(strict=True) -> this hook
    #    (funasr/train_utils/load_pretrained_model.py:104-113)
    def on_pretrained_model_loaded(self, loaded_keys=None):
        self._engine = None

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    def engine(self, device=None) -> ParaformerEngine:
        dev = torch.device(device) if device is not None else next(self.parameters()).device
        if dev.type != "cuda":
            raise _abi.FunasrB200Error("ParaformerB200 needs a CUDA device (got %s); there is no CPU path" % dev)
        if self._engine is None or self._engine.device != dev:
            self._engine = ParaformerEngine(self.state_dict(), self.cfg, dev, gemm_mode=self.gemm_mode)
        return self._engine

    # -- stage methods with the reference's names (model.py:286-346), tensors in / tensors out
    def encode(self, speech: torch.Tensor, speech_lengths: torch.Tensor, **kwargs):
        eng = self.engine(speech.device)
        lens = speech_lengths.to(speech.device, torch.int32)
        return eng.encode(speech.contiguous(), lens), lens

    def calc_predictor(self, encoder_out, encoder_out_lens):
        eng = self.engine(encoder_out.device)
        acoustic, tok, alphas, peaks = eng.predict(encoder_out, encoder_out_lens.to(torch.int32))
        n = int(tok.max().item())
        return acoustic[:, :n, :], tok.to(torch.float32), alphas, peaks

    def cal_decoder_with_predictor(self, encoder_out, encoder_out_lens, sematic_embeds, ys_pad_lens):
        eng = self.engine(encoder_out.device)
        n_max = sematic_embeds.shape[1]
        tok = ys_pad_lens.to(torch.int32)
        _, _, logp = eng.decode(encoder_out, encoder_out_lens.to(torch.int32), sematic_embeds.contiguous(), tok, n_max, want_logp=True)
        return logp, ys_pad_lens

    def _features(self, data_in, data_lengths, frontend, device, kwargs, meta_data):
        """model.py:572-600: load -> pad -> frontend, all on the device: (speech [B,T,560], lens [B] int32)."""
        if isinstance(data_in, torch.Tensor) and kwargs.get("data_type", "sound") == "fbank":
            speech = data_in if data_in.dim() == 3 else data_in[None]
            speech_lengths = data_lengths.reshape(-1) if data_lengths is not None else torch.tensor([speech.shape[1]])
            speech = speech.to(device, torch.float32).contiguous()
            lens = speech_lengths.to(device, torch.int32)
        else:
            t1 = time.perf_counter()
            # kwargs["fs"] is the rate of the GIVEN audio (model.py:578 passes it to the loader as audio_fs)
            wavs = _as_wave_list(data_in, fs=getattr(frontend, "fs", 16000), audio_fs=int(kwargs.get("fs", 16000)),
                                 **{k: v for k, v in kwargs.items() if k not in ("fs", "audio_fs", "frontend")})
            t2 = time.perf_counter()
            meta_data["load_data"] = f"{t2 - t1:0.3f}"
            if not isinstance(frontend, WavFrontendB200):
                raise _abi.FunasrB200Error("ParaformerB200 needs frontend='WavFrontendB200' (the fused CUDA frontend)")
            wl = [int(w.numel()) for w in wavs]
            if min(wl) < 2:
                raise _abi.FunasrB200Error("an utterance needs at least 2 samples (kaldi.fbank asserts 2 <= window_size)")
            nmax = max(wl)
            # pad_sequence (load_utils.py:412) done on the device: each utterance is copied host->device straight into its
            # row (truly asynchronous when the caller's buffers are pinned), no host-side staging copy
            ragged = min(wl) != nmax
            wav_dev = (torch.zeros if ragged else torch.empty)((len(wavs), nmax), dtype=torch.float32, device=device)
            for i, w in enumerate(wavs):
                wav_dev[i, : wl[i]].copy_(w, non_blocking=True)
            wl_dev = torch.tensor(wl, dtype=torch.int32).to(device, non_blocking=True)
            audio_fs = int(kwargs.get("fs", frontend.fs))          # rate of the given waveforms (load_utils.py:176-178 resamples)
            if audio_fs != frontend.fs and all(isinstance(x, (np.ndarray, torch.Tensor)) for x in
                                               (data_in if isinstance(data_in, (list, tuple)) else [data_in])):
                from .resample import resample, sinc_resample_table
                wav_dev, wl_dev = resample(wav_dev, wl_dev, audio_fs, frontend.fs)
                _, o_r, n_r, _ = sinc_resample_table(audio_fs, frontend.fs)
                wl = [-(-n_r * n // o_r) for n in wl]
                if min(wl) < 2:
                    raise _abi.FunasrB200Error("an utterance needs at least 2 samples (kaldi.fbank asserts 2 <= window_size)")
            speech, lens = frontend.engine(device)(wav_dev, wl_dev, max(num_lfr_frames(n) for n in wl), host_lens=wl)
            meta_data["extract_feat"] = f"{time.perf_counter() - t2:0.3f}"
            meta_data["batch_data_time"] = sum(num_lfr_frames(n) for n in wl) * frontend.frame_shift * frontend.lfr_n / 1000
        return speech, lens

    def _forward(self, eng, speech, lens, kwargs):
        """features -> greedy ids; subclasses with a different decode (SeACo) override this."""
        return eng.forward_feats(speech, lens, sos=self.sos, eos=self.eos, blank=self.blank_id)

    def infer_ids_device(self, data_in, frontend=None, **kwargs):
        """The hot path of inference() with the result left ON THE DEVICE: (ids [B, n] int32 padded with -1, lens [B] int32) —
        what funasr_b200.sharding.ShardedRunner exchanges between GPUs (no per-utterance host lists on the way)."""
        device = torch.device(kwargs.get("device", "cuda"))
        if device.type != "cuda":
            raise _abi.FunasrB200Error("%s needs device='cuda' (no CPU fallback)" % type(self).__name__)
        speech, lens = self._features(data_in, None, frontend, device, kwargs, {})
        out = self.engine(device).forward_feats(speech, lens, sos=self.sos, eos=self.eos, blank=self.blank_id, host_lists=False)
        if "ids_dev" not in out:                                  # no utterance produced a token
            b = speech.shape[0]
            return torch.full((b, 1), -1, dtype=torch.int32, device=device), torch.zeros((b,), dtype=torch.int32, device=device)
        return out["ids_dev"], out["ids_lens_dev"]

    def inference(self, data_in, data_lengths=None, key: list = None, tokenizer=None, frontend=None, **kwargs):
        """Same contract as Paraformer.inference (model.py:534-697): returns (results, meta_data)."""
        device = torch.device(kwargs.get("device", "cuda"))
        if device.type != "cuda":
            raise _abi.FunasrB200Error("ParaformerB200.inference needs device='cuda' (no CPU fallback)")
        meta_data = {}
        eng = self.engine(device)
        speech, lens = self._features(data_in, data_lengths, frontend, device, kwargs, meta_data)
        out = self._forward(eng, speech, lens, kwargs)
        if kwargs.get("_keep_taps"):
            self._last_out = out                  # BiCifParaformerB200 reads enc / lens / token counts for its timestamp head
        ids = out["ids"]
        if max((int(t) for t in out["token_num"].tolist()), default=0) < 1:
            return [], meta_data                              # model.py:615-616
        b = len(ids)
        if key is None:
            key = ["utt%d" % i for i in range(b)]
        if isinstance(key[0], (list, tuple)):
            key = key[0]
        if len(key) < b:
            key = key * b
        results = []
        pred_timestamp = bool(kwargs.get("pred_timestamp", False))            # model.py:558
        if pred_timestamp:
            from .timestamps import paraformer_timestamps
            alphas_h, peaks_h = out["alphas"].cpu().numpy(), out["peaks"].cpu().numpy()
        for i in range(b):
            token_int = ids[i]
            if tokenizer is not None:                         # CPU string work stays the reference's (model.py:668-687)
                token = tokenizer.ids2tokens(token_int)
                text = tokenizer.tokens2text(token)
                stamp = None
                if pred_timestamp:                            # model.py:673-680: CIF fires -> [start_ms, end_ms] per token
                    _, stamp = paraformer_timestamps(peaks_h[i], alphas_h[i], list(token), kwargs.get("begin_time", 0), want_text=False)
                if not hasattr(tokenizer, "bpemodel"):
                    try:
                        from funasr.utils import postprocess_utils
                        if stamp is not None:
                            text, stamp, _ = postprocess_utils.sentence_postprocess(token, stamp)
                        else:
                            text, _ = postprocess_utils.sentence_postprocess(token)
                    except ImportError:
                        pass
                res_i = {"key": key[i], "text": text}
                if stamp is not None:
                    res_i["timestamp"] = stamp
                results.append(res_i)
            else:
                res_i = {"key": key[i], "token_int": token_int}
                if pred_timestamp:                            # extension: the reference only time-stamps when it has a tokenizer
                    res_i["timestamp"] = paraformer_timestamps(peaks_h[i], alphas_h[i], [str(t) for t in token_int],
                                                               kwargs.get("begin_time", 0), want_text=False)[1]
                results.append(res_i)
        return results, meta_data


# ------------------------------------------------------------------------------------------------------------------
# SenseVoiceSmall (BASELINE config 4)
# ------------------------------------------------------------------------------------------------------------------
@register("encoder_classes", "SenseVoiceEncoderSmallB200")
class SenseVoiceEncoderSmallB200(SANMEncoderB200):
    """Parameter container for SenseVoiceEncoderSmall (funasr/models/sense_voice/model.py:489-656): the SANMEncoder
    layout plus `tp_encoders.{i}` and `tp_norm`."""

    def __init__(self, input_size: int, tp_blocks: int = 0, **kwargs):
        self.tp_blocks = tp_blocks
        super().__init__(input_size=input_size, **kwargs)

    def _specs(self):
        s = super()._specs()
        D = self._output_size
        proto = {k[len("encoders.0"):]: v for k, v in s.items() if k.startswith("encoders.0.")} if self.num_blocks > 1 else None
        if proto is None:
            proto = {k[len("encoders0.0"):]: (v if "norm1" not in k and "linear_q_k_v.weight" not in k else
                                               ((D,) if "norm1" in k else (3 * D, D))) for k, v in s.items() if k.startswith("encoders0.0.")}
        for i in range(self.tp_blocks):
            for suffix, shape in proto.items():
                s["tp_encoders.%d%s" % (i, suffix)] = shape
        s["tp_norm.weight"] = (D,)
        s["tp_norm.bias"] = (D,)
        return s


class _CTCHolder(_ParamHolder):
    def __init__(self, odim, eprojs):
        super().__init__()
        self.odim, self.eprojs = odim, eprojs
        self._build()

    def _specs(self):
        return {"ctc_lo.weight": (self.odim, self.eprojs), "ctc_lo.bias": (self.odim,)}


@register("model_classes", "SenseVoiceSmallB200")
class SenseVoiceSmallB200(nn.Module):
    """Drop-in for SenseVoiceSmall's greedy CTC inference (funasr/models/sense_voice/model.py:659-1034)."""

    lid_dict = {"auto": 0, "zh": 3, "en": 4, "yue": 7, "ja": 11, "ko": 12, "nospeech": 13}
    textnorm_dict = {"withitn": 14, "woitn": 15}

    def __init__(self, encoder: str = None, encoder_conf: dict = None, ctc_conf: dict = None, input_size: int = 80,
                 vocab_size: int = -1, blank_id: int = 0, gemm_mode: str = "fp32", **kwargs):
        super().__init__()
        tables = get_tables()
        enc_cls = tables.encoder_classes.get(encoder) if isinstance(encoder, str) else encoder
        if enc_cls is None or not issubclass(enc_cls, _ParamHolder):
            enc_cls = SenseVoiceEncoderSmallB200
        self.encoder = enc_cls(input_size=input_size, **(encoder_conf or {}))
        self.ctc = _CTCHolder(vocab_size, self.encoder.output_size())
        self.embed = nn.Embedding(7 + len(self.lid_dict) + len(self.textnorm_dict), input_size)   # parameter container only
        self.embed.weight.requires_grad_(False)
        self.vocab_size, self.blank_id, self.gemm_mode = vocab_size, blank_id, gemm_mode
        self.cfg = SenseVoiceConfig(enc_layers=self.encoder.num_blocks, tp_layers=self.encoder.tp_blocks, vocab=vocab_size,
                                    kernel=self.encoder.kernel_size)
        self._engine = None

    def on_pretrained_model_loaded(self, loaded_keys=None):
        self._engine = None

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    def engine(self, device, cmvn) -> SenseVoiceEngine:
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _abi.FunasrB200Error("SenseVoiceSmallB200 needs a CUDA device; there is no CPU path")
        if self._engine is None or self._engine.device != dev:
            self._engine = SenseVoiceEngine(self.state_dict(), self.cfg, dev, gemm_mode=self.gemm_mode, cmvn=cmvn)
        return self._engine

    def infer_ids_device(self, data_in, frontend=None, **kwargs):
        """CTC greedy ids left on the device: (ids [B, T] int32 padded with -1, lens [B] int32) for ShardedRunner."""
        out = self._run(data_in, frontend, {}, host_lists=False, **kwargs)
        return out["ids_dev"], out["ids_lens_dev"]

    def inference(self, data_in, data_lengths=None, key: list = ["wav_file_tmp_name"], tokenizer=None, frontend=None, **kwargs):
        meta_data = {}
        out = self._run(data_in, frontend, meta_data, **kwargs)
        b = len(out["ids"])
        if isinstance(key[0], (list, tuple)):
            key = key[0]
        if len(key) < b:
            key = key * b
        results = []
        for i in range(b):
            ids = out["ids"][i]
            results.append({"key": key[i], "text": tokenizer.decode(ids)} if tokenizer is not None else {"key": key[i], "token_int": ids})
        return results, meta_data

    def _run(self, data_in, frontend, meta_data, host_lists=True, **kwargs):
        device = torch.device(kwargs.get("device", "cuda"))
        if not isinstance(frontend, WavFrontendB200):
            raise _abi.FunasrB200Error("SenseVoiceSmallB200 needs frontend='WavFrontendB200'")
        eng = self.engine(device, frontend.cmvn)
        wavs = _as_wave_list(data_in, fs=frontend.fs, audio_fs=int(kwargs.get("fs", 16000)),
                             **{k: v for k, v in kwargs.items() if k not in ("fs", "audio_fs", "frontend")})
        wl = [int(w.numel()) for w in wavs]
        if min(wl) < 2:
            raise _abi.FunasrB200Error("an utterance needs at least 2 samples (kaldi.fbank asserts 2 <= window_size)")
        nmax = max(wl)
        wav_dev = (torch.zeros if min(wl) != nmax else torch.empty)((len(wavs), nmax), dtype=torch.float32, device=device)
        for i, w in enumerate(wavs):
            wav_dev[i, : wl[i]].copy_(w, non_blocking=True)
        wl_dev = torch.tensor(wl, dtype=torch.int32).to(device, non_blocking=True)
        meta_data["batch_data_time"] = sum(num_lfr_frames(n) for n in wl) * frontend.frame_shift * frontend.lfr_n / 1000
        language = kwargs.get("language", "auto")
        textnorm = kwargs.get("text_norm", None) or ("withitn" if kwargs.get("use_itn", False) else "woitn")
        return eng.forward_wav(wav_dev, wl_dev, wl, self.lid_dict.get(language, 0), self.textnorm_dict[textnorm], self.blank_id,
                               host_lists=host_lists)


# ------------------------------------------------------------------------------------------------------------------
# ContextualParaformer (BASELINE config 5)
# ------------------------------------------------------------------------------------------------------------------
@register("decoder_classes", "ContextualParaformerDecoderB200")
class ContextualParaformerDecoderB200(ParaformerSANMDecoderB200):
    """Parameter container for ContextualParaformerDecoder (funasr/models/contextual_paraformer/decoder.py:133-290)."""

    def _specs(self):
        s = super()._specs()
        D = self.D
        last = "decoders.%d." % (self.num_blocks - 1)
        for k in [k for k in s if k.startswith(last)]:
            s["last_decoder." + k[len(last):]] = s.pop(k)
        s["bias_decoder.norm3.weight"] = (D,)
        s["bias_decoder.norm3.bias"] = (D,)
        for nme, shp in (("linear_q", (D, D)), ("linear_k_v", (2 * D, D)), ("linear_out", (D, D))):
            s["bias_decoder.src_attn.%s.weight" % nme] = shp
            s["bias_decoder.src_attn.%s.bias" % nme] = (shp[0],)
        s["bias_output.weight"] = (D, 2 * D, 1)
        return s


@register("model_classes", "ContextualParaformerB200")
class ContextualParaformerB200(ParaformerB200):
    """Drop-in for ContextualParaformer's greedy inference with hotwords (contextual_paraformer/model.py:46-520).
    The hotword encoder (Embedding + 1-layer LSTM over a few short token sequences, O(#hotwords) and independent of the
    audio) runs in torch as the scope contract allows (SURVEY.md §7 item 9); everything per audio frame/token is CUDA."""

    def __init__(self, *args, inner_dim: int = 512, **kwargs):
        if not isinstance(kwargs.get("decoder"), type) and kwargs.get("decoder") not in ("ContextualParaformerDecoderB200",):
            kwargs["decoder"] = "ContextualParaformerDecoderB200"
        super().__init__(*args, **kwargs)
        if inner_dim != 512:
            raise _abi.FunasrB200Error("ContextualParaformerB200 supports inner_dim=512")
        self.bias_encoder = nn.LSTM(inner_dim, inner_dim, 1, batch_first=True)
        self.bias_embed = nn.Embedding(self.vocab_size, inner_dim)
        for p_ in list(self.bias_encoder.parameters()) + list(self.bias_embed.parameters()):
            p_.requires_grad_(False)

    def engine(self, device=None) -> ParaformerEngine:
        dev = torch.device(device) if device is not None else next(self.parameters()).device
        if dev.type != "cuda":
            raise _abi.FunasrB200Error("ContextualParaformerB200 needs a CUDA device; there is no CPU path")
        if self._engine is None or self._engine.device != dev:
            self._engine = ParaformerEngine(self.state_dict(), self.cfg, dev, gemm_mode=self.gemm_mode, contextual=True)
        return self._engine

    @torch.no_grad()
    def encode_hotwords(self, hw_list) -> torch.Tensor:
        """bias_embed -> LSTM -> h_n: [Nhw, 512] (model.py:350-372); hw_list=None -> the single [sos] entry (:350-358)."""
        dev = self.bias_embed.weight.device
        if hw_list is None:
            hw_list = [[1]]
        lens = [len(h) for h in hw_list]
        pad = torch.zeros((len(hw_list), max(lens)), dtype=torch.long, device=dev)
        for i, h in enumerate(hw_list):
            pad[i, : len(h)] = torch.tensor(h, device=dev)
        packed = torch.nn.utils.rnn.pack_padded_sequence(self.bias_embed(pad), lens, batch_first=True, enforce_sorted=False)
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):     # cuDNN RNNs default to TF32: keep fp32
            _, (h_n, _) = self.bias_encoder(packed)
        return h_n[0]

    def infer_ids_device(self, data_in, frontend=None, **kwargs):
        hw = kwargs.pop("hotword_ids", None)    # the reference re-encodes the hotword list on every call too (model.py:350-372)
        self.engine(kwargs.get("device", "cuda")).set_hotwords(self.encode_hotwords(hw))
        return super().infer_ids_device(data_in, frontend=frontend, **kwargs)

    def inference(self, data_in, data_lengths=None, key: list = None, tokenizer=None, frontend=None, **kwargs):
        hw = kwargs.get("hotword_ids")          # list of token-id lists (+ trailing [sos]); text hotwords need the tokenizer
        if hw is None and kwargs.get("hotword") and tokenizer is not None:      # .txt file or string; seg_dict aware (model.py:528-660)
            hw = generate_hotwords_list(kwargs["hotword"], tokenizer, frontend, self.sos)
        self.engine(kwargs.get("device", "cuda")).set_hotwords(self.encode_hotwords(hw))
        return super().inference(data_in, data_lengths, key, tokenizer, frontend, **kwargs)


# ------------------------------------------------------------------------------------------------------------------
# BiCifParaformer (SURVEY.md §8f rank 1: timestamps)
# ------------------------------------------------------------------------------------------------------------------
@register("model_classes", "BiCifParaformerB200")
class BiCifParaformerB200(ParaformerB200):
    """Drop-in for BiCifParaformer's greedy inference (funasr/models/bicif_paraformer/model.py:271-428): the Paraformer path with
    CifPredictorV3 (sequential fp32 `cif` on the token branch) plus the upsampled CIF timestamp head; results carry
    "timestamp": [[start_ms, end_ms], ...] per token."""

    def __init__(self, *args, **kwargs):
        if not isinstance(kwargs.get("predictor"), type) and kwargs.get("predictor") != "CifPredictorV3B200":
            kwargs["predictor"] = "CifPredictorV3B200"
        super().__init__(*args, **kwargs)

    def engine(self, device=None) -> ParaformerEngine:
        dev = torch.device(device) if device is not None else next(self.parameters()).device
        if dev.type != "cuda":
            raise _abi.FunasrB200Error("BiCifParaformerB200 needs a CUDA device; there is no CPU path")
        if self._engine is None or self._engine.device != dev:
            self._engine = ParaformerEngine(self.state_dict(), self.cfg, dev, gemm_mode=self.gemm_mode, bicif=True,
                                            smooth_factor2=self.predictor.smooth_factor2, noise_threshold2=self.predictor.noise_threshold2)
        return self._engine

    def calc_predictor_timestamp(self, encoder_out, encoder_out_lens, token_num):
        """model.py:177-191 -> (ds_alphas=None, ds_cif_peak=None, us_alphas, us_peaks)."""
        us_alphas, us_peaks = self.engine(encoder_out.device).upsample_timestamp(encoder_out, encoder_out_lens.to(torch.int32), token_num)
        return None, None, us_alphas, us_peaks

    def inference(self, data_in, data_lengths=None, key: list = None, tokenizer=None, frontend=None, **kwargs):
        from .timestamps import ts_prediction_lfr6_standard
        kwargs.pop("pred_timestamp", None)                      # BiCif always time-stamps, from its own head
        results, meta_data = super().inference(data_in, data_lengths, key, tokenizer, frontend, _keep_taps=True, **kwargs)
        out = getattr(self, "_last_out", None)
        if not results or out is None:
            return results, meta_data
        eng = self.engine(kwargs.get("device", "cuda"))
        us_alphas, us_peaks = eng.upsample_timestamp(out["enc_dev"], out["lens_dev"], out["tok_dev"])
        ua, up, lens = us_alphas.cpu().numpy(), us_peaks.cpu().numpy(), out["lens_dev"].cpu().tolist()
        for i, r in enumerate(results):
            ids = out["ids"][i]
            token = tokenizer.ids2tokens(ids) if tokenizer is not None else [str(t) for t in ids]
            n = int(lens[i]) * eng.ts_head.up_times
            _, stamp = ts_prediction_lfr6_standard(ua[i][:n], up[i][:n], list(token), vad_offset=kwargs.get("begin_time", 0),
                                                   want_text=False)                                                                 # model.py:402-407
            if tokenizer is not None:
                try:
                    from funasr.utils import postprocess_utils
                    r["text"], stamp, _ = postprocess_utils.sentence_postprocess(token, stamp)
                except ImportError:
                    pass
            r["timestamp"] = stamp
        self._last_out = None
        return results, meta_data


# ------------------------------------------------------------------------------------------------------------------
# MonotonicAligner (fa-zh): timestamps for a transcript the caller already has
# ------------------------------------------------------------------------------------------------------------------
def _aligner_tokens(text, tokenizer) -> List[int]:
    """One transcript as token ids, the way load_audio_text_image_video (load_utils.py:144-146, :148-149) reads data_type "text":
    a path to an existing text file is read and encoded, any other string is encoded, a sequence of ids is taken as is."""
    import os
    if isinstance(text, str):
        if tokenizer is None:
            raise _abi.FunasrB200Error("MonotonicAlignerB200 needs a tokenizer to encode a text transcript")
        if os.path.exists(text):
            with open(text, "r") as f:
                text = f.read().strip()
        return [int(t) for t in tokenizer.encode(text)]
    if torch.is_tensor(text) or isinstance(text, np.ndarray):
        text = text.tolist()
    return [int(t) for t in text]


@register("model_classes", "MonotonicAlignerB200")
class MonotonicAlignerB200(nn.Module):
    """Drop-in for funasr.models.monotonic_aligner.model.MonotonicAligner.inference (model.py:182-267): given (audio, transcript)
    pairs, the SAN-M encoder and CifPredictorV3's upsampled timestamp head give [start_ms, end_ms] per transcript character."""

    def __init__(self, input_size: int = 80, specaug=None, specaug_conf=None, normalize=None, normalize_conf=None, encoder: str = None,
                 encoder_conf: dict = None, predictor: str = None, predictor_conf: dict = None, predictor_bias: int = 0,
                 length_normalized_loss: bool = False, gemm_mode: str = "fp32", **kwargs):
        super().__init__()
        # specaug, predictor_bias and length_normalized_loss only act in training (model.py:100-146)
        tables = get_tables()
        enc_cls = tables.encoder_classes.get(encoder) if isinstance(encoder, str) else encoder
        pred_cls = tables.predictor_classes.get(predictor) if isinstance(predictor, str) else predictor
        enc_cls = enc_cls if (enc_cls is not None and issubclass(enc_cls, _ParamHolder)) else SANMEncoderB200
        pred_cls = pred_cls if (pred_cls is not None and issubclass(pred_cls, _ParamHolder)) else CifPredictorV3B200
        self.encoder = enc_cls(input_size=input_size, **(encoder_conf or {}))
        self.predictor = pred_cls(**(predictor_conf or {}))
        if self.predictor.idim != self.encoder.output_size():
            raise _abi.FunasrB200Error("MonotonicAlignerB200: predictor idim %d != encoder output size %d"
                                       % (self.predictor.idim, self.encoder.output_size()))
        self.predictor_bias = predictor_bias
        self.gemm_mode = gemm_mode
        self.cfg = ParaformerConfig(d_model=self.encoder.output_size(), heads=self.encoder.heads, ffn=self.encoder.ffn,
                                    enc_layers=self.encoder.num_blocks, dec_layers=0, kernel=self.encoder.kernel_size,
                                    tail_threshold=self.predictor.tail_threshold, cif_threshold=self.predictor.threshold)
        self._engine: Optional[AlignerEngine] = None

    def on_pretrained_model_loaded(self, loaded_keys=None):
        self._engine = None

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    def engine(self, device=None) -> AlignerEngine:
        dev = torch.device(device) if device is not None else next(self.parameters()).device
        if dev.type != "cuda":
            raise _abi.FunasrB200Error("MonotonicAlignerB200 needs a CUDA device (got %s); there is no CPU path" % dev)
        if self._engine is None or self._engine.device != dev:
            self._engine = AlignerEngine(self.state_dict(), self.cfg, dev, gemm_mode=self.gemm_mode,
                                         smooth_factor2=self.predictor.smooth_factor2, noise_threshold2=self.predictor.noise_threshold2)
        return self._engine

    def encode(self, speech: torch.Tensor, speech_lengths: torch.Tensor, **kwargs):
        eng = self.engine(speech.device)
        lens = speech_lengths.to(speech.device, torch.int32)
        return eng.encode(speech.contiguous(), lens), lens

    def calc_predictor_timestamp(self, encoder_out, encoder_out_lens, token_num):
        """model.py:156-168 -> (ds_alphas=None, ds_cif_peak=None, us_alphas, us_peaks)."""
        us_alphas, us_peaks = self.engine(encoder_out.device).upsample_timestamp(encoder_out, encoder_out_lens.to(torch.int32), token_num)
        return None, None, us_alphas, us_peaks

    def inference(self, data_in, data_lengths=None, key: list = None, tokenizer=None, frontend=None, **kwargs):
        """Same contract as MonotonicAligner.inference: data_in is one (audio, text) pair or a list of them, data_type
        ("sound", "text"); returns ([{"key", "text", "timestamp"}, ...], meta_data)."""
        from .timestamps import ts_prediction_lfr6_standard
        device = torch.device(kwargs.get("device", "cuda"))
        if device.type != "cuda":
            raise _abi.FunasrB200Error("MonotonicAlignerB200.inference needs device='cuda' (no CPU fallback)")
        data_type = kwargs.get("data_type", ("sound", "text"))
        if tuple(data_type) != ("sound", "text"):
            raise _abi.FunasrB200Error("MonotonicAlignerB200 takes data_type=('sound', 'text') (audio, transcript) pairs")
        pairs = [data_in] if (isinstance(data_in, tuple) and len(data_in) == 2) else list(data_in)
        token_lists = [_aligner_tokens(t, tokenizer) for _, t in pairs]
        kw = {k: v for k, v in kwargs.items() if k != "data_type"}
        meta_data = {}
        eng = self.engine(device)
        speech, lens = ParaformerB200._features(self, [a for a, _ in pairs], data_lengths, frontend, device, kw, meta_data)
        enc = eng.encode(speech, lens)
        text_lengths = torch.tensor([len(t) + 1 for t in token_lists], dtype=torch.int32)          # model.py:226-228
        us_alphas, us_peaks = eng.upsample_timestamp(enc, lens, text_lengths)
        ua, up, elens = us_alphas.cpu().numpy(), us_peaks.cpu().numpy(), lens.cpu().tolist()
        b = len(pairs)
        if key is None:
            key = ["utt%d" % i for i in range(b)]
        if isinstance(key[0], (list, tuple)):
            key = key[0]
        results = []
        for i, token_int in enumerate(token_lists):
            token = tokenizer.ids2tokens(token_int) if tokenizer is not None else [str(t) for t in token_int]
            n = int(elens[i]) * eng.ts_head.up_times
            _, stamp = ts_prediction_lfr6_standard(ua[i][:n], up[i][:n], list(token), want_text=False)       # model.py:243-247
            text = tokenizer.tokens2text(token) if tokenizer is not None else " ".join(token)
            try:
                from funasr.utils import postprocess_utils
                text, stamp, _ = postprocess_utils.sentence_postprocess(token, stamp)                        # model.py:248-250
            except ImportError:
                pass
            results.append({"key": key[i], "text": text, "timestamp": stamp})
        return results, meta_data


# ------------------------------------------------------------------------------------------------------------------
# SeacoParaformer (SURVEY.md §8f rank 1: the `paraformer-zh` default alias)
# ------------------------------------------------------------------------------------------------------------------
class _SeacoDecoderHolder(_ParamHolder):
    """Parameter container for the SeACo decoder: ParaformerSANMDecoder(use_output_layer=False, wo_input_layer=True)
    (seaco_paraformer/model.py:100-110) — `decoders.{i}` (att_layer_num layers), `decoders3.0`, `after_norm`."""

    def __init__(self, attention_heads: int = 4, linear_units: int = 1024, num_blocks: int = 4, att_layer_num: int = 6, kernel_size: int = 21,
                 sanm_shfit: int = 0, **kwargs):
        super().__init__()
        if attention_heads != 4 or sanm_shfit != 0 or linear_units > 2048 or att_layer_num < 6:
            raise _abi.FunasrB200Error("the SeACo decoder supports 4 heads, sanm_shfit=0, linear_units <= 2048, att_layer_num >= 6 "
                                       "(forward_asf6 addresses decoders[0..5], paraformer/decoder.py:507-512)")
        self.ffn, self.layers, self.kernel_size = linear_units, att_layer_num, kernel_size
        self._build()

    def _specs(self):
        D, F, K = 512, self.ffn, self.kernel_size
        s = {"after_norm.weight": (D,), "after_norm.bias": (D,)}

        def ffn(p):
            s[p + ".feed_forward.w_1.weight"] = (F, D)
            s[p + ".feed_forward.w_1.bias"] = (F,)
            s[p + ".feed_forward.w_2.weight"] = (D, F)
            s[p + ".feed_forward.norm.weight"] = (F,)
            s[p + ".feed_forward.norm.bias"] = (F,)

        for i in range(self.layers):
            p = "decoders.%d" % i
            ffn(p)
            s[p + ".self_attn.fsmn_block.weight"] = (D, 1, K)
            for nme, shp in (("linear_q", (D, D)), ("linear_k_v", (2 * D, D)), ("linear_out", (D, D))):
                s[p + ".src_attn.%s.weight" % nme] = shp
                s[p + ".src_attn.%s.bias" % nme] = (shp[0],)
            for n in ("norm1", "norm2", "norm3"):
                s[p + ".%s.weight" % n] = (D,)
                s[p + ".%s.bias" % n] = (D,)
        ffn("decoders3.0")
        s["decoders3.0.norm1.weight"] = (D,)
        s["decoders3.0.norm1.bias"] = (D,)
        return s


@register("model_classes", "SeacoParaformerB200")
class SeacoParaformerB200(BiCifParaformerB200):
    """Drop-in for SeacoParaformer's greedy inference with hotwords (funasr/models/seaco_paraformer/model.py:50-581): the BiCif path
    (CifPredictorV3 tokens + upsampled timestamps) with `_seaco_decode_with_ASF` in place of the plain decoder call — decoder
    hidden states, the SeACo decoder over the hotword memory (twice), attention-score filtering when the hotword list is longer than
    `nfilter`, hotword_output_layer, NO_BIAS merge.  The hotword encoder (Embedding + 2-layer LSTM, O(#hotwords)) runs in torch."""

    def __init__(self, *args, inner_dim: int = 512, bias_encoder_type: str = "lstm", bias_encoder_bid: bool = False, seaco_decoder: str = None,
                 seaco_decoder_conf: dict = None, NO_BIAS: int = 8377, **kwargs):
        super().__init__(*args, **kwargs)
        if inner_dim != 512 or bias_encoder_type != "lstm" or bias_encoder_bid:
            raise _abi.FunasrB200Error("SeacoParaformerB200 supports inner_dim=512, bias_encoder_type='lstm', unidirectional")
        conf = {k: v for k, v in (seaco_decoder_conf or {}).items() if k in ("attention_heads", "linear_units", "num_blocks", "att_layer_num",
                                                                             "kernel_size", "sanm_shfit")}
        self.seaco_decoder = _SeacoDecoderHolder(**conf)
        self.bias_encoder = nn.LSTM(inner_dim, inner_dim, 2, batch_first=True)
        self.hotword_output_layer = nn.Linear(inner_dim, self.vocab_size)
        for p_ in list(self.bias_encoder.parameters()) + list(self.hotword_output_layer.parameters()):
            p_.requires_grad_(False)
        self.NO_BIAS = int(NO_BIAS)

    def engine(self, device=None) -> ParaformerEngine:
        dev = torch.device(device) if device is not None else next(self.parameters()).device
        if dev.type != "cuda":
            raise _abi.FunasrB200Error("SeacoParaformerB200 needs a CUDA device; there is no CPU path")
        if self._engine is None or self._engine.device != dev:
            self._engine = ParaformerEngine(self.state_dict(), self.cfg, dev, gemm_mode=self.gemm_mode, seaco=True, no_bias=self.NO_BIAS,
                                            smooth_factor2=self.predictor.smooth_factor2, noise_threshold2=self.predictor.noise_threshold2)
        return self._engine

    def _forward(self, eng, speech, lens, kwargs):
        hw = kwargs.get("hotword_ids")          # list of token-id lists incl. the trailing [sos] entry (generate_hotwords_list)
        tok = kwargs.get("_tokenizer")
        if hw is None and kwargs.get("hotword") and tok is not None:            # seaco_paraformer/model.py:583-690
            hw = generate_hotwords_list(kwargs["hotword"], tok, kwargs.get("_frontend"), self.sos)
        return eng.forward_feats_seaco(speech, lens, hw, nfilter=int(kwargs.get("nfilter", 50)), sos=self.sos, eos=self.eos, blank=self.blank_id)

    def inference(self, data_in, data_lengths=None, key: list = None, tokenizer=None, frontend=None, **kwargs):
        return super().inference(data_in, data_lengths, key, tokenizer, frontend, _tokenizer=tokenizer, _frontend=frontend, **kwargs)
