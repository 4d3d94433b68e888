"""CAM++ speaker embeddings on the GPU behind the reference's plugin surface (funasr/models/campplus).

  CAMPPlusB200     <- model.py CAMPPlus: same state_dict names (head.*, xvector.*); inference() -> [{"spk_embedding": [B, 192]}]
  CampplusEngine   folded / repacked weights and the two kernel calls: fa_campplus_features (kaldi fbank with torchaudio's defaults +
                   per-utterance mean subtraction) and fa_campplus_forward (FCM, TDNN, 52 CAM dense layers, transits, statistics
                   pooling, dense layer).

Eval-mode BatchNorm that follows a conv is folded into that conv here, once; BatchNorm in front of ReLU + conv becomes a per-channel
affine the kernels apply while they build the GEMM operand.  No torch.nn op on the path; no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import time
from collections import OrderedDict
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import _abi
from .engine import _EngineBase, kaldi_mel_banks
from .modules import _as_wave_list
from .registry import register

BN_EPS = 1e-5
BLOCK_LAYERS, BLOCK_DILATION = (12, 24, 16), (1, 2, 2)
GROWTH, BN_CH, INIT_CH, FEAT_DIM, EMB_DIM = 32, 128, 128, 80, 192
# order of FaCampplus.fcm
FCM_CONVS = ["conv1", "layer1.0.conv1", "layer1.0.conv2", "layer1.0.shortcut.0", "layer1.1.conv1", "layer1.1.conv2",
             "layer2.0.conv1", "layer2.0.conv2", "layer2.0.shortcut.0", "layer2.1.conv1", "layer2.1.conv2", "conv2"]
FCM_BNS = ["bn1", "layer1.0.bn1", "layer1.0.bn2", "layer1.0.shortcut.1", "layer1.1.bn1", "layer1.1.bn2",
           "layer2.0.bn1", "layer2.0.bn2", "layer2.0.shortcut.1", "layer2.1.bn1", "layer2.1.bn2", "bn2"]
FCM_STRIDE = [1, 2, 1, 2, 1, 1, 2, 1, 2, 1, 1, 2]
# fa_campplus_forward's longest input (~188 s): the CAM context gate keeps at most 94 segment means of 100 TDNN frames per chunk
MAX_FEAT_FRAMES = 18800


def campplus_specs() -> "OrderedDict[str, tuple]":
    """name -> shape of every entry of the reference CAMPPlus state_dict (template.yaml configuration)."""
    s: "OrderedDict[str, tuple]" = OrderedDict()

    def bn(p, n, affine=True):
        if affine:
            s[p + ".weight"], s[p + ".bias"] = (n,), (n,)
        s[p + ".running_mean"], s[p + ".running_var"], s[p + ".num_batches_tracked"] = (n,), (n,), ()

    for conv, bnn in zip(FCM_CONVS, FCM_BNS):
        cin = 1 if conv == "conv1" else 32
        k = 1 if conv.endswith("shortcut.0") else 3
        s["head." + conv + ".weight"] = (32, cin, k, k)
        bn("head." + bnn, 32)
    s["xvector.tdnn.linear.weight"] = (INIT_CH, 320, 5)
    bn("xvector.tdnn.nonlinear.batchnorm", INIT_CH)
    c = INIT_CH
    for i, n_layers in enumerate(BLOCK_LAYERS):
        for l in range(n_layers):
            p = "xvector.block%d.tdnnd%d." % (i + 1, l + 1)
            cin = c + l * GROWTH
            bn(p + "nonlinear1.batchnorm", cin)
            s[p + "linear1.weight"] = (BN_CH, cin, 1)
            bn(p + "nonlinear2.batchnorm", BN_CH)
            s[p + "cam_layer.linear_local.weight"] = (GROWTH, BN_CH, 3)
            s[p + "cam_layer.linear1.weight"], s[p + "cam_layer.linear1.bias"] = (BN_CH // 2, BN_CH, 1), (BN_CH // 2,)
            s[p + "cam_layer.linear2.weight"], s[p + "cam_layer.linear2.bias"] = (GROWTH, BN_CH // 2, 1), (GROWTH,)
        c += n_layers * GROWTH
        bn("xvector.transit%d.nonlinear.batchnorm" % (i + 1), c)
        s["xvector.transit%d.linear.weight" % (i + 1)] = (c // 2, c, 1)
        c //= 2
    bn("xvector.out_nonlinear.batchnorm", c)
    s["xvector.dense.linear.weight"] = (EMB_DIM, 2 * c, 1)
    bn("xvector.dense.nonlinear.batchnorm", EMB_DIM, affine=False)
    return s


def povey_window(n: int = 400) -> torch.Tensor:
    """torchaudio.compliance.kaldi's default window: hann(periodic=False) ** 0.85."""
    return torch.hann_window(n, periodic=False, dtype=torch.float32).pow(0.85)


def num_fbank_frames(n_samples: int) -> int:
    return 1 + (n_samples - 400) // 160 if n_samples >= 400 else 0


class CampplusEngine(_EngineBase):
    """Folded weights + ctypes structs of one CAM++ model on one device, in one gemm_mode."""

    # the forward's workspace grows ~5 MB per 1.5 s chunk; larger batches run in slices of this many bytes
    WORKSPACE_CAP = 1 << 30

    def __init__(self, state: Dict[str, torch.Tensor], device, gemm_mode: str = "fp32"):
        self._init_base(state, device, gemm_mode, BN_EPS)
        self.mel = kaldi_mel_banks().to(self.device)
        self.window = povey_window().to(self.device)
        self.tables = torch.empty(int(self.lib.fa_fbank_tables_bytes()) // 4, dtype=torch.float32, device=self.device)
        _abi.check(self.lib.fa_fbank_make_tables(self.mel.data_ptr(), self.window.data_ptr(), self.tables.data_ptr(), self._stream()),
                   "fa_fbank_make_tables")
        m = _abi.FaCampplus()
        for i, (conv, bnn, stride) in enumerate(zip(FCM_CONVS, FCM_BNS, FCM_STRIDE)):
            m.fcm[i] = self.conv2d(state["head." + conv + ".weight"], self._bn(state, "head." + bnn), stride)
        s, t = self._bn(state, "xvector.tdnn.nonlinear.batchnorm")
        w = state["xvector.tdnn.linear.weight"].double().permute(0, 2, 1).reshape(INIT_CH, -1)      # [o][k * 320 + c]
        m.tdnn = self._folded(w, s, t)
        self.layers = (_abi.FaCamLayer * sum(BLOCK_LAYERS))()
        k = 0
        for i, n_layers in enumerate(BLOCK_LAYERS):
            m.n_layers[i], m.dilation[i] = n_layers, BLOCK_DILATION[i]
            for l in range(n_layers):
                p = "xvector.block%d.tdnnd%d." % (i + 1, l + 1)
                L = self.layers[k]
                k += 1
                L.bn1_scale, L.bn1_shift = self._affine(state, p + "nonlinear1.batchnorm")
                s, t = self._bn(state, p + "nonlinear2.batchnorm")
                L.linear1 = self._folded(state[p + "linear1.weight"].double()[:, :, 0], s, t)
                L.local_w = self._keep_ptr(state[p + "cam_layer.linear_local.weight"].permute(2, 1, 0))       # [k][c][o]
                L.w1 = self._keep_ptr(state[p + "cam_layer.linear1.weight"][:, :, 0])
                L.b1 = self._keep_ptr(state[p + "cam_layer.linear1.bias"])
                L.w2 = self._keep_ptr(state[p + "cam_layer.linear2.weight"][:, :, 0])
                L.b2 = self._keep_ptr(state[p + "cam_layer.linear2.bias"])
            p = "xvector.transit%d." % (i + 1)
            tr = m.transit[i]
            tr.scale, tr.shift = self._affine(state, p + "nonlinear.batchnorm")
            w = self._dev(state[p + "linear.weight"][:, :, 0])
            tr.linear = self._lin("", bias=False, weight=w)
        m.layers = self.layers
        m.out_scale, m.out_shift = self._affine(state, "xvector.out_nonlinear.batchnorm")
        s, t = self._bn(state, "xvector.dense.nonlinear.batchnorm", affine=False)
        m.dense = self._folded(state["xvector.dense.linear.weight"].double()[:, :, 0], s, t)
        self.model = m
        torch.cuda.current_stream(self.device).synchronize()

    # ---- weight folding
    @staticmethod
    def _bn(state, p, affine=True):
        """eval BatchNorm as y = x * s + t (float64)."""
        var, mean = state[p + ".running_var"].double(), state[p + ".running_mean"].double()
        s = 1.0 / torch.sqrt(var + BN_EPS)
        if affine:
            s = s * state[p + ".weight"].double()
            return s, state[p + ".bias"].double() - mean * s
        return s, -mean * s

    def _keep_ptr(self, t: torch.Tensor) -> int:
        return self._dev(t.float()).data_ptr()

    def _affine(self, state, p):
        s, t = self._bn(state, p)
        return self._keep_ptr(s), self._keep_ptr(t)

    def _folded(self, w: torch.Tensor, s: torch.Tensor, t: torch.Tensor) -> _abi.FaLinear:
        """conv (as [out, in]) followed by BN -> one Linear with bias."""
        wf = self._dev((w * s[:, None]).float())
        return self._lin("", weight=wf, bias_tensor=self._dev(t.float()))

    def conv2d(self, w: torch.Tensor, bn, stride: int) -> _abi.FaCamConv2d:
        s, t = bn
        cout, cin, k, _ = w.shape
        wf = (w.double() * s[:, None, None, None]).permute(2, 3, 1, 0).reshape(k * k, cin, cout)     # [kf * k + kt][ci][o]
        return _abi.FaCamConv2d(self._keep_ptr(wf), self._keep_ptr(t), cin, cout, k, stride)

    # ---- forward
    def features(self, wav: torch.Tensor, wav_lens: torch.Tensor, t_max: int):
        """wav [B, Nmax] fp32 on the device, wav_lens [B] int32 on the device -> feats [B, t_max, 80], feat_lens [B]."""
        assert wav.is_cuda and wav.dtype == torch.float32 and wav.stride(1) == 1
        B = wav.shape[0]
        feats = torch.empty((B, t_max, FEAT_DIM), dtype=torch.float32, device=self.device)
        flens = torch.empty((B,), dtype=torch.int32, device=self.device)
        _abi.check(self.lib.fa_campplus_features(wav.data_ptr(), wav_lens.data_ptr(), B, wav.stride(0), self.tables.data_ptr(),
                                                 feats.data_ptr(), flens.data_ptr(), t_max, self._stream()), "fa_campplus_features")
        return feats, flens

    def embed_feats(self, feats: torch.Tensor) -> torch.Tensor:
        """feats [B, T, 80] (every frame counts, like the reference's unmasked forward) -> [B, 192]."""
        feats = feats.contiguous()
        B, T, _ = feats.shape
        out = torch.empty((B, EMB_DIM), dtype=torch.float32, device=self.device)
        per = int(self.lib.fa_campplus_workspace_bytes(C.byref(self.model), 1, T, self.mode))
        if per == 0:
            raise _abi.FunasrB200Error("CAM++ takes 2 ... %d feature frames per input (got %d)" % (MAX_FEAT_FRAMES, T))
        step = max(1, min(B, self.WORKSPACE_CAP // per))
        for b0 in range(0, B, step):
            nb = min(step, B - b0)
            ws = self._workspace(int(self.lib.fa_campplus_workspace_bytes(C.byref(self.model), nb, T, self.mode)))
            _abi.check(self.lib.fa_campplus_forward(C.byref(self.model), feats[b0:b0 + nb].data_ptr(), nb, T, out[b0].data_ptr(), self.mode,
                                                    ws.data_ptr(), ws.numel(), self._stream()), "fa_campplus_forward")
        return out

    def embed_wav(self, wav: torch.Tensor, wav_lens: torch.Tensor, host_lens: List[int]) -> torch.Tensor:
        if min(host_lens) < 400:
            raise _abi.FunasrB200Error("CAM++ needs at least 400 samples (one 25 ms frame) per input")
        t_max = max(num_fbank_frames(n) for n in host_lens)
        feats, _ = self.features(wav, wav_lens, t_max)
        return self.embed_feats(feats)


def _add_tensor(root: nn.Module, dotted: str, shape) -> None:
    parts = dotted.split(".")
    mod = root
    for p in parts[:-1]:
        if not hasattr(mod, p):
            mod.add_module(p, nn.Module())
        mod = getattr(mod, p)
    if parts[-1] in ("running_mean", "running_var", "num_batches_tracked"):
        mod.register_buffer(parts[-1], torch.zeros(shape, dtype=torch.long if parts[-1] == "num_batches_tracked" else torch.float32))
    else:
        mod.register_parameter(parts[-1], nn.Parameter(torch.zeros(*shape), requires_grad=False))


@register("model_classes", "CAMPPlusB200")
class CAMPPlusB200(nn.Module):
    """Drop-in for CAMPPlus (campplus/model.py) on the inference path: same constructor arguments and state_dict names."""

    def __init__(self, feat_dim=80, embedding_size=192, growth_rate=32, bn_size=4, init_channels=128, config_str="batchnorm-relu",
                 memory_efficient=True, output_level="segment", gemm_mode: str = "fp32", **kwargs):
        super().__init__()
        if (feat_dim, embedding_size, growth_rate, bn_size, init_channels, config_str, output_level) != \
                (FEAT_DIM, EMB_DIM, GROWTH, BN_CH // GROWTH, INIT_CH, "batchnorm-relu", "segment"):
            raise _abi.FunasrB200Error("CAMPPlusB200 is built for the template.yaml shape (feat 80, embedding 192, growth 32, bn_size 4, "
                                       "init 128, batchnorm-relu, segment output)")
        self.gemm_mode = gemm_mode
        for name, shape in campplus_specs().items():
            _add_tensor(self, name, shape)
        self._engine: Optional[CampplusEngine] = None

    def on_pretrained_model_loaded(self, loaded_keys=None):
        self._engine = None

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    def forward(self, *a, **k):  # pragma: no cover
        raise _abi.FunasrB200Error("CAMPPlusB200 runs through inference() / engine() on a CUDA device")

    def engine(self, device) -> CampplusEngine:
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _abi.FunasrB200Error("CAMPPlusB200 needs a CUDA device; there is no CPU path")
        if self._engine is None or self._engine.device != dev:
            self._engine = CampplusEngine({k: v.detach().cpu() for k, v in self.state_dict().items()}, dev, self.gemm_mode)
        return self._engine

    def inference(self, data_in, data_lengths=None, key: list = None, tokenizer=None, frontend=None, **kwargs):
        """list of waveforms (ragged allowed) -> ([{"spk_embedding": [B, 192]}], meta_data) like CAMPPlus.inference: features of shorter
        inputs are zero-padded to the longest (pad_list) and the padded frames take part in every mean."""
        device = torch.device(kwargs.get("device", "cuda"))
        meta_data = {}
        t1 = time.perf_counter()
        wavs = _as_wave_list(data_in, fs=16000, audio_fs=int(kwargs.get("fs", 16000)))
        meta_data["load_data"] = f"{time.perf_counter() - t1:0.3f}"
        eng = self.engine(device)
        lens = [int(w.numel()) for w in wavs]
        pad = torch.nn.utils.rnn.pad_sequence([w.reshape(-1) for w in wavs], batch_first=True).to(device, torch.float32, non_blocking=True)
        emb = eng.embed_wav(pad.contiguous(), torch.tensor(lens, dtype=torch.int32).to(device, non_blocking=True), lens)
        meta_data["batch_data_time"] = float(np.sum(lens)) / 16000.0
        return [{"spk_embedding": emb}], meta_data
