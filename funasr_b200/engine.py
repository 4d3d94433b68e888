"""Host-side driver of the C ABI: packs weights into the FaEncoder/FaPredictor/FaDecoder structs, owns the
device workspace, and sequences frontend -> encoder -> CIF predictor -> decoder -> greedy ids on the current
CUDA stream.  PyTorch is used for device memory, streams and H2D/D2H copies only; every arithmetic op on the hot
path is a kernel in libfunasr_b200.so.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _abi
from .synth import ParaformerConfig, sinusoid_inv_timescales


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def kaldi_mel_banks(n_mels=80, n_fft=512, fs=16000.0, low=20.0, high=0.0) -> torch.Tensor:
    """Triangular mel filters exactly as torchaudio.compliance.kaldi.get_mel_banks (kaldi.py:436-511, vtln 1.0)
    builds them, right-padded with one zero column (kaldi.py:621-627): [n_mels, n_fft/2 + 1] fp32.
    Host-side table construction (a constant of the configuration), same torch ops in the same order."""
    nyq = 0.5 * fs
    if high <= 0.0:
        high += nyq
    bw = fs / n_fft
    ml = 1127.0 * math.log(1.0 + low / 700.0)
    mh = 1127.0 * math.log(1.0 + high / 700.0)
    delta = (mh - ml) / (n_mels + 1)
    b = torch.arange(n_mels).unsqueeze(1)
    left, center, right = ml + b * delta, ml + (b + 1.0) * delta, ml + (b + 2.0) * delta
    mel = (1127.0 * (1.0 + (bw * torch.arange(n_fft / 2)) / 700.0).log()).unsqueeze(0)
    up = (mel - left) / (center - left)
    down = (right - mel) / (right - center)
    banks = torch.max(torch.zeros(1), torch.min(up, down))
    return torch.nn.functional.pad(banks, (0, 1), value=0.0).float().contiguous()


def num_lfr_frames(n_samples: int, win=400, shift=160, lfr_n=6) -> int:
    """LFR rows of an utterance.  Below one 25 ms window the reference shrinks the window to the utterance (wav_frontend.py:174):
    one frame as long as kaldi.fbank accepts it (window >= 2 samples)."""
    m = 1 + (n_samples - win) // shift if n_samples >= win else (1 if n_samples >= 2 else 0)
    return (m + lfr_n - 1) // lfr_n


class FrontendEngine:
    """Fused Fbank+LFR+CMVN (fa_fbank_lfr_cmvn_tables).  lfr_m / lfr_n: 7 / 6 (Paraformer, SenseVoice) or 5 / 1 (FSMN-VAD)."""

    def __init__(self, cmvn: Optional[torch.Tensor], device, lfr_m: int = 7, lfr_n: int = 6):
        self.lib = _abi.load()
        self.device = torch.device(device)
        self.lfr_m, self.lfr_n = int(lfr_m), int(lfr_n)
        self.feat_dim = 80 * self.lfr_m
        self.cmvn = None if cmvn is None else cmvn.to(self.device, torch.float32).contiguous()
        if self.cmvn is not None and tuple(self.cmvn.shape) != (2, self.feat_dim):
            raise _abi.FunasrB200Error("cmvn must be [2, %d] for lfr_m=%d" % (self.feat_dim, self.lfr_m))
        self.mel = kaldi_mel_banks().to(self.device)
        self.window = torch.hamming_window(400, periodic=False, alpha=0.54, beta=0.46, dtype=torch.float32).to(self.device)
        # per-configuration constants (sparse mel support, twiddles, window), built once on the device
        self._short_mel = {}
        self.tables = torch.empty(int(self.lib.fa_fbank_tables_bytes()) // 4, dtype=torch.float32, device=self.device)
        st = torch.cuda.current_stream(self.device).cuda_stream
        _abi.check(self.lib.fa_fbank_make_tables(self.mel.data_ptr(), self.window.data_ptr(), self.tables.data_ptr(), st), "fa_fbank_make_tables")

    def __call__(self, wav: torch.Tensor, wav_lens: torch.Tensor, t_max: int, host_lens=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """wav [B, Nmax] fp32 on device, wav_lens [B] int32 on device -> feats [B, t_max, 560], feat_lens [B] int32.
        host_lens: the same lengths on the host; needed only when some utterance is shorter than 400 samples."""
        assert wav.is_cuda and wav.dtype == torch.float32 and wav.stride(1) == 1
        B = wav.shape[0]
        feats = torch.empty((B, t_max, self.feat_dim), dtype=torch.float32, device=self.device)
        flens = torch.empty((B,), dtype=torch.int32, device=self.device)
        st = torch.cuda.current_stream(self.device).cuda_stream
        _abi.check(self.lib.fa_fbank_lfr_cmvn_tables(wav.data_ptr(), wav_lens.data_ptr(), B, wav.stride(0), _ptr(self.cmvn),
                                                     self.tables.data_ptr(), self.lfr_m, self.lfr_n, feats.data_ptr(), t_max,
                                                     flens.data_ptr(), t_max, st), "fa_fbank_lfr_cmvn_tables")
        if host_lens is not None and min(host_lens) < 400:
            self._short_rows(wav, host_lens, feats, flens, st)
        return feats, flens

    def _short_rows(self, wav, host_lens, feats, flens, st):
        """Utterances below one 25 ms frame (the batched kernel left their rows empty): one frame over the whole utterance each,
        like kaldi.fbank(frame_length=len / fs) in wav_frontend.py:171-181."""
        for b, n in enumerate(host_lens):
            if n >= 400:
                continue
            if n < 2:
                raise _abi.FunasrB200Error("an utterance needs at least 2 samples (kaldi.fbank asserts 2 <= window_size)")
            pad = 1 << (n - 1).bit_length()
            if pad not in self._short_mel:
                self._short_mel[pad] = kaldi_mel_banks(n_fft=pad).to(self.device)
            win = torch.hamming_window(n, periodic=False, alpha=0.54, beta=0.46, dtype=torch.float32).to(self.device)
            _abi.check(self.lib.fa_fbank_short(wav[b].data_ptr(), n, win.data_ptr(), self._short_mel[pad].data_ptr(), pad, _ptr(self.cmvn),
                                               self.lfr_m, feats[b, 0].data_ptr(), st), "fa_fbank_short")
        idx = torch.tensor([b for b, n in enumerate(host_lens) if n < 400], dtype=torch.long).to(self.device)
        flens.index_fill_(0, idx, 1)


class _EngineBase:
    """Weight packing (device copies, fp16 planes, ctypes structs), workspace and the encoder call."""

    def _init_base(self, state, device, gemm_mode, ln_eps):
        self.lib = _abi.load()
        self.device = torch.device(device)
        self.mode = _abi.GEMM_MODES[gemm_mode] if isinstance(gemm_mode, str) else int(gemm_mode)
        self._keep: List[torch.Tensor] = []   # keeps every packed tensor alive
        self._ws: Optional[torch.Tensor] = None
        self._state = state
        self._eps = ln_eps

    def _g(self, k):
        return self._dev(self._state[k])

    def _lin(self, prefix, bias=True, weight=None, bias_tensor=None) -> _abi.FaLinear:
        w = self._dev(self._state[prefix + ".weight"]) if weight is None else weight
        b = bias_tensor if bias_tensor is not None else (self._dev(self._state[prefix + ".bias"]) if bias else None)
        out_f, in_f = w.shape
        in_pad = (in_f + 63) // 64 * 64
        planes = None
        if self.mode != _abi.GEMM_F32_SIMT:
            planes = torch.empty((3, out_f, in_pad), dtype=torch.float16, device=self.device)
            st = torch.cuda.current_stream(self.device).cuda_stream
            _abi.check(self.lib.fa_split_planes(w.data_ptr(), in_f, out_f, in_f, in_pad, planes.data_ptr(), st), "fa_split_planes")
            self._keep.append(planes)
        return _abi.FaLinear(w.data_ptr(), _ptr(b), _ptr(planes), out_f, in_f, in_pad, 0)

    def _norm(self, prefix) -> _abi.FaNorm:
        w, b = self._g(prefix + ".weight"), self._g(prefix + ".bias")
        return _abi.FaNorm(w.data_ptr(), b.data_ptr(), w.numel(), self._eps)

    def _enc_stack(self, layer_prefixes, after_norm_prefix, heads, fsmn_k, pe_depth):
        """FaEncoder over the given layer name prefixes; pe_depth None -> plain 512->512 stack (no x*sqrt(d)+PE)."""
        layers = (_abi.FaEncLayer * len(layer_prefixes))()
        for L, p in zip(layers, layer_prefixes):
            L.norm1, L.norm2 = self._norm(p + ".norm1"), self._norm(p + ".norm2")
            L.qkv, L.out = self._lin(p + ".self_attn.linear_q_k_v"), self._lin(p + ".self_attn.linear_out")
            L.fsmn_w = self._g(p + ".self_attn.fsmn_block.weight").data_ptr()     # [512,1,11] contiguous == [512,11]
            L.w1, L.w2 = self._lin(p + ".feed_forward.w_1"), self._lin(p + ".feed_forward.w_2")
        pe = self._dev(sinusoid_inv_timescales(pe_depth)) if pe_depth else None
        fsmn_k = int(self._state[layer_prefixes[0] + ".self_attn.fsmn_block.weight"].shape[-1])    # taps come from the weights
        enc = _abi.FaEncoder(layers, len(layer_prefixes), heads, fsmn_k, 0, self._norm(after_norm_prefix), _ptr(pe))
        self._keep_structs = getattr(self, "_keep_structs", []) + [layers]
        return enc

    def _dev(self, t: torch.Tensor) -> torch.Tensor:
        t = t.detach().to(self.device, torch.float32).contiguous()
        self._keep.append(t)
        return t

    def _workspace(self, nbytes: int) -> torch.Tensor:
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty((int(nbytes * 1.1) + 4096,), dtype=torch.uint8, device=self.device)
            self._invalidate_graphs()           # every captured launch baked the old workspace address in
        return self._ws

    def _invalidate_graphs(self):
        """Captured CUDA graphs hold raw device addresses: whenever an engine-owned buffer or the workspace is replaced, every
        graph is dropped (a stale graph would write into freed memory)."""
        self.__dict__["_buf_gen"] = self.__dict__.get("_buf_gen", 0) + 1
        g = self.__dict__.get("_dec_graphs")
        if g:
            g.clear()

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _persist(self, name: str, shape, dtype=torch.float32) -> torch.Tensor:
        """Engine-owned buffer that keeps its address across calls with the same shape (CUDA-graph replay needs stable
        pointers).  Only the fused forward path uses these; the public per-stage methods return fresh tensors."""
        bufs = self.__dict__.setdefault("_pbufs", {})
        t = bufs.get(name)
        if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
            t = torch.empty(tuple(shape), dtype=dtype, device=self.device)
            bufs[name] = t
            self._invalidate_graphs()
        return t

    def _encode(self, enc_struct, x: torch.Tensor, lens: torch.Tensor, d_model: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        B, T, _ = x.shape
        if out is None:
            out = torch.empty((B, T, d_model), dtype=torch.float32, device=self.device)
        ws = self._workspace(self.lib.fa_sanm_encoder_workspace_bytes(B, T, self.mode))
        _abi.check(self.lib.fa_sanm_encoder_forward(C.byref(enc_struct), x.data_ptr(), lens.data_ptr(), B, T, out.data_ptr(),
                                                    self.mode, ws.data_ptr(), ws.numel(), self._stream()), "fa_sanm_encoder_forward")
        return out

    def _init_timestamp_head(self, prefix_pred, smooth_factor2, noise_threshold2, threshold):
        """CifPredictorV3 timestamp head (bicif_paraformer/cif_predictor.py:121-352, upsample_type "cnn_blstm", use_cif1_cnn False),
        shared by BiCifParaformer / SeacoParaformer and the MonotonicAligner."""
        from .pack import timestamp_head_tensors
        head = {k[len(prefix_pred):]: self._dev(v) for k, v in timestamp_head_tensors(self._state, prefix_pred).items()}
        self.ts_head = _abi.FaTimestampHead(
            self._lin("upsample_cnn", weight=head["upsample_cnn.gemm_weight"], bias_tensor=head["upsample_cnn.gemm_bias"]),
            self._lin("blstm.ih", weight=head["blstm.ih_gemm_weight"], bias_tensor=head["blstm.ih_gemm_bias"]),
            head["blstm.weight_hh_l0"].data_ptr(), head["blstm.weight_hh_l0_reverse"].data_ptr(),
            head["cif_output2.weight"].data_ptr(), head["cif_output2.bias"].data_ptr(),
            int(self._state[prefix_pred + "upsample_cnn.weight"].shape[2]),   # ConvTranspose1d weight [in, out, k], stride == k
            float(smooth_factor2), float(noise_threshold2), float(threshold))

    def upsample_timestamp(self, enc: torch.Tensor, lens: torch.Tensor, token_num: torch.Tensor):
        """CifPredictorV3.get_upsample_timestamp (bicif_paraformer/cif_predictor.py:300-352): enc [B,T,D] (D = 512 or 320), lens [B] i32,
        token_num [B] i32 (rounded) -> (us_alphas [B,3T], us_peaks [B,3T]), one fa_timestamp_head_forward.  Its workspace is the
        engine's: it grows once to the head's size, after which the head and the decoder graphs keep the same address."""
        if getattr(self, "ts_head", None) is None:
            raise _abi.FunasrB200Error("engine was not built with the CifPredictorV3 timestamp head (bicif=True)")
        B, T, D = enc.shape
        U = self.ts_head.up_times
        us_alphas = torch.empty((B, T * U), dtype=torch.float32, device=self.device)
        us_peaks = torch.empty_like(us_alphas)
        lens = lens.to(self.device, torch.int32).contiguous()
        tok = token_num.to(self.device, torch.int32).contiguous()
        ws = self._workspace(self.lib.fa_timestamp_head_workspace_bytes(B, T, D, U, self.mode))
        _abi.check(self.lib.fa_timestamp_head_forward(C.byref(self.ts_head), enc.data_ptr(), lens.data_ptr(), tok.data_ptr(), B, T,
                                                      us_alphas.data_ptr(), us_peaks.data_ptr(), self.mode, ws.data_ptr(), ws.numel(),
                                                      self._stream()), "fa_timestamp_head_forward")
        return us_alphas, us_peaks


class AlignerEngine(_EngineBase):
    """MonotonicAligner (monotonic_aligner/model.py): the SAN-M encoder plus CifPredictorV3's timestamp head — no token
    predictor, no decoder (`predictor.cif_conv1d` / `cif_output` are not used by get_upsample_timestamp)."""

    def __init__(self, state: Dict[str, torch.Tensor], cfg: ParaformerConfig, device, gemm_mode: str = "fp32",
                 smooth_factor2: float = 0.25, noise_threshold2: float = 0.01):
        self._init_base(state, device, gemm_mode, cfg.ln_eps)
        self.cfg = cfg
        K = int(state["encoder.encoders0.0.self_attn.fsmn_block.weight"].shape[-1])
        names = ["encoder." + ("encoders0.0" if i == 0 else "encoders.%d" % (i - 1)) for i in range(cfg.enc_layers)]
        self.enc = self._enc_stack(names, "encoder.after_norm", cfg.heads, K, cfg.feat_dim)
        self._init_timestamp_head("predictor.", smooth_factor2, noise_threshold2, cfg.cif_threshold)
        torch.cuda.current_stream(self.device).synchronize()
        self._state = None

    def encode(self, feats: torch.Tensor, lens: torch.Tensor) -> torch.Tensor:
        """SANMEncoder.forward: feats [B,T,560], lens [B] int32 -> [B,T,D]."""
        return self._encode(self.enc, feats, lens, self.cfg.d_model)


class ParaformerEngine(_EngineBase):
    """Packed weights + workspace + the encoder/predictor/decoder ABI calls."""

    def __init__(self, state: Dict[str, torch.Tensor], cfg: ParaformerConfig, device, gemm_mode: str = "fp32",
                 prefix_enc="encoder.", prefix_pred="predictor.", prefix_dec="decoder.", contextual: bool = False, bicif: bool = False,
                 smooth_factor2: float = 0.25, noise_threshold2: float = 0.01, seaco: bool = False, no_bias: int = 8377):
        self._init_base(state, device, gemm_mode, cfg.ln_eps)
        self.cfg = cfg
        self.contextual = contextual
        self.bicif = bicif or seaco          # SeacoParaformer derives from BiCifParaformer (CifPredictorV3 + timestamp head)
        bicif = self.bicif
        self.seaco = seaco
        self.no_bias = int(no_bias)
        g, lin, norm = self._g, self._lin, self._norm
        D = cfg.d_model
        # FSMN tap counts come from each stack's own weights [512, 1, K]: encoder and decoder kernel_size are independent
        # constructor arguments (decoder default 21, paraformer/decoder.py:234)
        K = int(state[prefix_enc + "encoders0.0.self_attn.fsmn_block.weight"].shape[-1])
        first_dec = prefix_dec + ("decoders.0" if (cfg.dec_layers > 1 or not contextual) else "last_decoder")
        Kd = int(state[first_dec + ".self_attn.fsmn_block.weight"].shape[-1])
        # ---- encoder
        names = [prefix_enc + ("encoders0.0" if i == 0 else "encoders.%d" % (i - 1)) for i in range(cfg.enc_layers)]
        self.enc = self._enc_stack(names, prefix_enc + "after_norm", cfg.heads, K, cfg.feat_dim)
        self.enc_layers = self._keep_structs[-1]
        # ---- predictor: Conv1d(512,512,3) weight [out, in, k] -> GEMM weight [out, k*512 + in]
        cw = state[prefix_pred + "cif_conv1d.weight"]
        cw = self._dev(cw.permute(0, 2, 1).reshape(cw.shape[0], -1))
        conv = lin(prefix_pred + "cif_conv1d", weight=cw)
        self.pred = _abi.FaPredictor(conv, g(prefix_pred + "cif_output.weight").data_ptr(),
                                     g(prefix_pred + "cif_output.bias").data_ptr(), cfg.cif_threshold,
                                     cfg.tail_threshold, 1.0, 0.0, 1 if bicif else 0, 0)
        if bicif:
            self._init_timestamp_head(prefix_pred, smooth_factor2, noise_threshold2, cfg.cif_threshold)
        # ---- decoder
        def dec_layer(L, p, full=True):
            L.norm1 = norm(p + ".norm1")
            L.ffn_w1, L.ffn_norm = lin(p + ".feed_forward.w_1"), norm(p + ".feed_forward.norm")
            L.ffn_w2 = lin(p + ".feed_forward.w_2", bias=False)
            if full:
                L.norm2, L.norm3 = norm(p + ".norm2"), norm(p + ".norm3")
                L.fsmn_w = g(p + ".self_attn.fsmn_block.weight").data_ptr()
                L.q, L.kv, L.out = lin(p + ".src_attn.linear_q"), lin(p + ".src_attn.linear_k_v"), lin(p + ".src_attn.linear_out")

        n_plain = cfg.dec_layers - 1 if contextual else cfg.dec_layers
        self.dec_layers = (_abi.FaDecLayer * max(n_plain, 1))()
        for i in range(n_plain):
            dec_layer(self.dec_layers[i], prefix_dec + "decoders.%d" % i)
        self.dec = _abi.FaDecoder()
        self.dec.layers = self.dec_layers
        self.dec.n_layers, self.dec.heads, self.dec.fsmn_k, self.dec.vocab = n_plain, cfg.heads, Kd, cfg.vocab
        self.dec.has_bias = 0
        if contextual:   # ContextualParaformerDecoder (contextual_paraformer/decoder.py:133-352)
            dec_layer(self.dec.bias_last, prefix_dec + "last_decoder")
            self.dec.bias_norm3 = norm(prefix_dec + "bias_decoder.norm3")
            self.dec.bias_q = lin(prefix_dec + "bias_decoder.src_attn.linear_q")
            self.dec.bias_kv = lin(prefix_dec + "bias_decoder.src_attn.linear_k_v")
            self.dec.bias_out = lin(prefix_dec + "bias_decoder.src_attn.linear_out")
            bw = state[prefix_dec + "bias_output.weight"]
            self.dec.bias_output = lin(prefix_dec + "bias_output", bias=False, weight=self._dev(bw.reshape(bw.shape[0], -1)))
            self.dec.clas_scale = 1.0
            self._hw = None
        dec_layer(self.dec.last, prefix_dec + "decoders3.0", full=False)
        self.dec.after_norm = norm(prefix_dec + "after_norm")
        self.dec.output = lin(prefix_dec + "output_layer")
        if seaco:   # SeacoParaformer (seaco_paraformer/model.py:50-120): hotword LSTM, SeACo decoder over the hotword memory, hotword_output_layer
            sp = "seaco_decoder."
            n_s = 0
            while (sp + "decoders.%d.norm1.weight" % n_s) in state:
                n_s += 1
            self.seaco_layers = (_abi.FaDecLayer * n_s)()
            for i in range(n_s):
                dec_layer(self.seaco_layers[i], sp + "decoders.%d" % i)
            self.seaco_dec = _abi.FaDecoder()
            self.seaco_dec.layers, self.seaco_dec.n_layers, self.seaco_dec.heads = self.seaco_layers, n_s, cfg.heads
            self.seaco_dec.fsmn_k = int(state[sp + "decoders.0.self_attn.fsmn_block.weight"].shape[-1])
            self.seaco_dec.vocab, self.seaco_dec.has_bias = 0, 0
            dec_layer(self.seaco_dec.last, sp + "decoders3.0", full=False)
            self.seaco_dec.after_norm = norm(sp + "after_norm")
            self.hw_out = lin("hotword_output_layer")
            # the hotword encoder (Embedding + 2-layer LSTM over a handful of short token sequences) is O(#hotwords), independent of
            # the audio: torch (cuDNN, TF32 off), as the scope contract allows for the hotword side (SURVEY.md §7 item 9)
            self.hw_embed_table = g(prefix_dec + "embed.0.weight")
            self.hw_lstm = torch.nn.LSTM(D, D, 2, batch_first=True).to(self.device)
            self.hw_lstm.load_state_dict({k[len("bias_encoder."):]: v for k, v in state.items() if k.startswith("bias_encoder.")})
            self.hw_lstm.eval().requires_grad_(False)
        torch.cuda.current_stream(self.device).synchronize()
        self._state = None

    # ------------------------------------------------------------------------------------------
    def encode(self, feats: torch.Tensor, lens: torch.Tensor) -> torch.Tensor:
        """SANMEncoder.forward: feats [B,T,560], lens [B] int32 -> [B,T,512]."""
        return self._encode(self.enc, feats, lens, self.cfg.d_model)

    def predict(self, enc: torch.Tensor, lens: torch.Tensor, persistent: bool = False):
        """CifPredictorV2.forward -> (acoustic [B,T+1,512] zero padded, token_num [B] i32, alphas [B,T+1], peaks [B,T+1])."""
        B, T, D = enc.shape
        n_cap = T + 1
        new = (lambda name, shape, dt: self._persist("pred_" + name, shape, dt)) if persistent else \
            (lambda name, shape, dt: torch.empty(shape, dtype=dt, device=self.device))
        acoustic = new("acoustic", (B, n_cap, D), torch.float32)
        tok = new("tok", (B,), torch.int32)
        alphas = new("alphas", (B, T + 1), torch.float32)
        peaks = new("peaks", (B, T + 1), torch.float32)
        ws = self._workspace(self.lib.fa_cif_predictor_workspace_bytes(B, T, self.mode))
        _abi.check(self.lib.fa_cif_predictor_forward(C.byref(self.pred), enc.data_ptr(), lens.data_ptr(), B, T, acoustic.data_ptr(),
                                                     n_cap, tok.data_ptr(), alphas.data_ptr(), peaks.data_ptr(), self.mode,
                                                     ws.data_ptr(), ws.numel(), self._stream()), "fa_cif_predictor_forward")
        return acoustic, tok, alphas, peaks

    def set_hotwords(self, hw_embed: torch.Tensor):
        """Hotword memory [Nhw, 512] (LSTM last hidden states) for the contextual bias decoder."""
        if not self.contextual:
            raise _abi.FunasrB200Error("engine was not built with contextual=True")
        self._hw = hw_embed.detach().to(self.device, torch.float32).contiguous()
        self._hw_lens = None

    def decode(self, enc: torch.Tensor, enc_lens: torch.Tensor, acoustic: torch.Tensor, tok_lens: torch.Tensor, n_max: int,
               want_logp: bool = False, out: Optional[tuple] = None):
        """ParaformerSANMDecoder.forward + arg-max -> (argmax ids [B,n_max] i32, best logp [B,n_max], logp or None)."""
        B, T, D = enc.shape
        if self.contextual:
            if self._hw is None:
                raise _abi.FunasrB200Error("call set_hotwords() first")
            if self._hw_lens is None or self._hw_lens.numel() != B:
                self._hw_lens = torch.full((B,), self._hw.shape[0], dtype=torch.int32, device=self.device)
            self.dec.has_bias, self.dec.n_hotwords = 1, self._hw.shape[0]
            self.dec.hw_embed, self.dec.hw_lens = self._hw.data_ptr(), self._hw_lens.data_ptr()
        if out is not None:
            ids, best = out
        else:
            ids = torch.empty((B, n_max), dtype=torch.int32, device=self.device)
            best = torch.empty((B, n_max), dtype=torch.float32, device=self.device)
        logp = torch.empty((B, n_max, self.cfg.vocab), dtype=torch.float32, device=self.device) if want_logp else None
        ws = self._workspace(self.lib.fa_paraformer_decoder_workspace_bytes_hw(B, T, n_max, self.cfg.vocab, self.mode,
                                                                               self._hw.shape[0] if self.contextual else 0))
        _abi.check(self.lib.fa_paraformer_decoder_forward(
            C.byref(self.dec), enc.data_ptr(), enc_lens.data_ptr(), B, T, acoustic.data_ptr(), acoustic.shape[1],
            tok_lens.data_ptr(), n_max, ids.data_ptr(), best.data_ptr(), _ptr(logp), 1, self.mode, ws.data_ptr(), ws.numel(),
            self._stream()), "fa_paraformer_decoder_forward")
        return ids, best, logp

    # ------------------------------------------------------------------------------------------ SeacoParaformer
    @torch.no_grad()
    def seaco_hotword_representation(self, hw_list) -> torch.Tensor:
        """_hotword_representation (seaco_paraformer/model.py:384-416): decoder.embed -> 2-layer LSTM over the packed padded
        batch -> each hotword's output at its last token: [n_hw, 512]."""
        lens = [len(h) for h in hw_list]
        pad = torch.zeros((len(hw_list), max(lens)), dtype=torch.long, device=self.device)
        for i, h in enumerate(hw_list):
            pad[i, : len(h)] = torch.tensor(h, device=self.device)
        emb = torch.nn.functional.embedding(pad, self.hw_embed_table)
        packed = torch.nn.utils.rnn.pack_padded_sequence(emb, torch.tensor(lens, dtype=torch.int64), batch_first=True, enforce_sorted=False)
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            out, _ = self.hw_lstm(packed)
        out = torch.nn.utils.rnn.pad_packed_sequence(out, batch_first=True)[0]
        return out[torch.arange(len(hw_list), device=self.device), torch.tensor(lens, device=self.device) - 1].contiguous()

    def _seaco_stack(self, memory, x, ld_x_rows, tok, B, n_max, n_run, finish, hidden=None, attn=None):
        n_hw = memory.shape[0]
        mem_lens = torch.full((B,), n_hw, dtype=torch.int32, device=self.device)
        ws = self._workspace(self.lib.fa_sanm_decoder_stack_workspace_bytes(B, n_hw, n_max, self.mode))
        _abi.check(self.lib.fa_sanm_decoder_stack_forward(
            C.byref(self.seaco_dec), memory.data_ptr(), mem_lens.data_ptr(), 1, B, n_hw, x.data_ptr(), ld_x_rows, tok.data_ptr(), n_max,
            n_run, finish, _ptr(hidden), _ptr(attn), self.mode, ws.data_ptr(), ws.numel(), self._stream()), "fa_sanm_decoder_stack_forward")

    def seaco_decode(self, enc, enc_lens, acoustic, tok, n_max, hw_list, nfilter: int = 50, want_logp: bool = False):
        """_seaco_decode_with_ASF (seaco_paraformer/model.py:271-382) + arg-max: -> (ids [B,n_max] i32, best logp, taps)."""
        if not self.seaco:
            raise _abi.FunasrB200Error("engine was not built with seaco=True")
        B, T, D = enc.shape
        V = self.cfg.vocab
        new = lambda *shape, dt=torch.float32: torch.empty(shape, dtype=dt, device=self.device)
        dec_ids, dec_best, hidden = new(B, n_max, dt=torch.int32), new(B, n_max), new(B, n_max, D)
        dec_logp = new(B, n_max, V) if want_logp else None
        ws = self._workspace(self.lib.fa_paraformer_decoder_workspace_bytes_hw(B, T, n_max, V, self.mode, 0))
        _abi.check(self.lib.fa_paraformer_decoder_forward_hidden(
            C.byref(self.dec), enc.data_ptr(), enc_lens.data_ptr(), B, T, acoustic.data_ptr(), acoustic.shape[1], tok.data_ptr(), n_max,
            dec_ids.data_ptr(), dec_best.data_ptr(), _ptr(dec_logp), 1, hidden.data_ptr(), self.mode, ws.data_ptr(), ws.numel(),
            self._stream()), "fa_paraformer_decoder_forward_hidden")
        taps = {"dec_hidden": hidden}
        if hw_list is None:                                   # model.py:381-382: plain decoder distribution
            return dec_ids, dec_best, dict(taps, merged=dec_logp)
        selected = self.seaco_hotword_representation(hw_list)
        taps["hw_selected_all"] = selected
        n_hw = selected.shape[0]
        if 0 < nfilter < n_hw:                                # ASF (model.py:320-343): keep the hotwords utterance 0 attends to most
            probs = new(self.seaco_dec.heads, n_max, n_hw)
            self._seaco_stack(selected, hidden, n_max, tok, 1, n_max, self.seaco_dec.n_layers, 0, attn=probs)
            scores = probs.cpu().sum(0).sum(0)                # the reference's own reduction order, on the host (hotword_scores[0].sum(0).sum(0))
            picked = torch.topk(scores, min(nfilter, n_hw - 1))[1].tolist() + [len(hw_list) - 1]
            selected = selected[torch.tensor(picked, device=self.device)].contiguous()
            taps["asf_picked"] = picked
        taps["hw_selected"] = selected
        cif_att, dec_att = new(B, n_max, D), new(B, n_max, D)
        self._seaco_stack(selected, acoustic, acoustic.shape[1], tok, B, n_max, self.seaco_dec.n_layers, 1, hidden=cif_att)
        self._seaco_stack(selected, hidden, n_max, tok, B, n_max, self.seaco_dec.n_layers, 1, hidden=dec_att)
        dha_ids, dha_best = new(B, n_max, dt=torch.int32), new(B, n_max)
        dha_logp = new(B, n_max, V) if want_logp else None
        rows = B * n_max
        ws = self._workspace(self.lib.fa_linear_argmax_workspace_bytes(rows, V, self.mode))
        _abi.check(self.lib.fa_linear_argmax(C.byref(self.hw_out), cif_att.data_ptr(), dec_att.data_ptr(), rows, dha_ids.data_ptr(),
                                             dha_best.data_ptr(), _ptr(dha_logp), self.mode, ws.data_ptr(), ws.numel(), self._stream()),
                   "fa_linear_argmax")
        ids, best = new(B, n_max, dt=torch.int32), new(B, n_max)
        merged = new(B, n_max, V) if want_logp else None
        _abi.check(self.lib.fa_seaco_merge(dec_ids.data_ptr(), dec_best.data_ptr(), dha_ids.data_ptr(), dha_best.data_ptr(), rows, self.no_bias,
                                           ids.data_ptr(), best.data_ptr(), _ptr(dec_logp), _ptr(dha_logp), _ptr(merged), V, self._stream()),
                   "fa_seaco_merge")
        taps.update(merged=merged, dha_pred=dha_logp, dha_ids=dha_ids)
        return ids, best, taps

    def forward_feats_seaco(self, feats: torch.Tensor, lens: torch.Tensor, hw_list, nfilter: int = 50, want_taps: bool = False,
                            sos=1, eos=2, blank=0):
        """SeacoParaformer.inference (model.py:422-581) from features to greedy ids."""
        enc = self._encode(self.enc, feats, lens, self.cfg.d_model)
        acoustic, tok, alphas, peaks = self.predict(enc, lens)
        tok_host = tok.cpu()
        n_max = int(tok_host.max()) if tok_host.numel() else 0
        out = {"token_num": tok_host, "alphas": alphas, "peaks": peaks, "enc_dev": enc, "lens_dev": lens, "tok_dev": tok}
        if want_taps:
            out.update(enc=enc, acoustic=acoustic)
        if n_max < 1:
            out["ids"] = [[] for _ in range(feats.shape[0])]
            return out
        ids, best, taps = self.seaco_decode(enc, lens, acoustic, tok, n_max, hw_list, nfilter, want_logp=want_taps)
        fids, flens = self.greedy_filter(ids, tok, sos, eos, blank)
        fids_h, flens_h = fids.cpu(), flens.cpu()
        out["ids"] = [fids_h[b, : int(flens_h[b])].tolist() for b in range(fids_h.shape[0])]
        out["ids_dev"], out["ids_lens_dev"] = fids, flens
        if want_taps:
            out.update(taps)
        return out

    def greedy_filter(self, ids: torch.Tensor, tok_lens: torch.Tensor, sos=1, eos=2, blank=0, out: Optional[tuple] = None):
        B, n_max = ids.shape
        if out is not None:
            out, out_lens = out
        else:
            out = torch.empty_like(ids)
            out_lens = torch.empty((B,), dtype=torch.int32, device=self.device)
        _abi.check(self.lib.fa_greedy_filter(ids.data_ptr(), tok_lens.data_ptr(), B, n_max, sos, eos, blank, out.data_ptr(),
                                             out_lens.data_ptr(), self._stream()), "fa_greedy_filter")
        return out, out_lens

    def forward_feats(self, feats: torch.Tensor, lens: torch.Tensor, want_taps: bool = False, sos=1, eos=2, blank=0, host_lists: bool = True):
        """feats -> greedy ids.  One host synchronisation (the token counts), like the reference's `.item()`
        (cif_predictor.py:311) — every other reference sync is gone.

        Without taps the stage outputs live in engine-owned buffers (stable addresses) and the decoder + arg-max + filter launch
        sequence (~190 mostly small kernels) is replayed from a CUDA graph once the same (shape, n_max) has been seen twice —
        measured 9.4 -> 8.2 ms at B=64; the encoder (few large kernels, launches already hidden) gains nothing from a graph
        and is launched directly."""
        B, T, _ = feats.shape
        fused = not want_taps
        enc = self._encode(self.enc, feats, lens, self.cfg.d_model, out=self._persist("enc", (B, T, self.cfg.d_model)) if fused else None)
        if fused:
            lens_p = self._persist("lens", (B,), torch.int32)
            lens_p.copy_(lens)
            lens = lens_p
        acoustic, tok, alphas, peaks = self.predict(enc, lens, persistent=fused)
        tok_host = tok.cpu()                       # D2H + sync: B int32
        n_max = int(tok_host.max()) if tok_host.numel() else 0
        out = {"enc": enc, "alphas": alphas, "peaks": peaks, "token_num": tok_host, "acoustic": acoustic} if want_taps else \
            {"token_num": tok_host, "alphas": alphas, "peaks": peaks, "enc_dev": enc, "lens_dev": lens, "tok_dev": tok}   # device refs (timestamps)
        if n_max < 1:                              # paraformer/model.py:615-616
            out["ids"] = [[] for _ in range(feats.shape[0])]
            return out
        if fused:
            fids, flens = self._decode_filter_fused(enc, lens, acoustic, tok, n_max, sos, eos, blank)
            ids = best = logp = None
        else:
            ids, best, logp = self.decode(enc, lens, acoustic, tok, n_max, want_logp=want_taps)
            fids, flens = self.greedy_filter(ids, tok, sos, eos, blank)
        out["ids_dev"], out["ids_lens_dev"] = fids, flens        # device copies (multi-GPU all-gather consumes these)
        if host_lists:
            fids_h, flens_h = fids.cpu(), flens.cpu()  # D2H of the result
            out["ids"] = [fids_h[b, : int(flens_h[b])].tolist() for b in range(fids_h.shape[0])]
            out["ids_padded"], out["ids_lens"] = fids_h, flens_h
        if want_taps:
            out.update(argmax=ids, best_logp=best, logp=logp)
        return out

    # ---- decoder + arg-max + sos/eos/blank filter, replayed from a CUDA graph when the shape repeats ---------------------
    _GRAPH_CAP = 16

    def _decode_filter_fused(self, enc, lens, acoustic, tok, n_max, sos, eos, blank):
        B, T, _ = enc.shape
        # four output buffers sized ONCE for the CIF bound (n_max <= T + 1) and viewed as [B, n_max]: their addresses do not depend
        # on n_max, nothing grows with the number of distinct n_max values, and the graph key below covers every pointer a capture
        # bakes in (all four buffers, the stage inputs, the workspace) plus the buffer generation
        cap = B * (T + 1)
        flat = (self._persist("dec_ids", (cap,), torch.int32), self._persist("dec_best", (cap,)),
                self._persist("dec_fids", (cap,), torch.int32), self._persist("dec_flens", (B,), torch.int32))
        bufs = (flat[0][: B * n_max].view(B, n_max), flat[1][: B * n_max].view(B, n_max), flat[2][: B * n_max].view(B, n_max), flat[3])

        def run():
            ids, _, _ = self.decode(enc, lens, acoustic, tok, n_max, out=(bufs[0], bufs[1]))
            self.greedy_filter(ids, tok, sos, eos, blank, out=(bufs[2], bufs[3]))

        if self.contextual:
            run()
            return bufs[2], bufs[3]
        # size the workspace BEFORE the key is formed: a growth replaces it (and drops every graph)
        self._workspace(self.lib.fa_paraformer_decoder_workspace_bytes_hw(B, T, n_max, self.cfg.vocab, self.mode, 0))
        key = (B, T, n_max, sos, eos, blank, enc.data_ptr(), lens.data_ptr(), acoustic.data_ptr(), tok.data_ptr(),
               bufs[0].data_ptr(), bufs[1].data_ptr(), bufs[2].data_ptr(), bufs[3].data_ptr(), self._ws.data_ptr(),
               self.__dict__.get("_buf_gen", 0))
        graphs = self.__dict__.setdefault("_dec_graphs", {})
        ent = graphs.get(key)
        if ent is None:
            if len(graphs) >= self._GRAPH_CAP:                      # drop the oldest entry (dict keeps insertion order)
                graphs.pop(next(iter(graphs)))
            ent = graphs[key] = {"seen": 0, "graph": None}
        ent["seen"] += 1
        if ent["graph"] is not None:
            ent["graph"].replay()
            self.replayed_launches = getattr(self, "replayed_launches", 0) + ent["n_launch"]
        elif ent["seen"] < 2:
            run()                                                   # first sighting: plain launches (also the warm-up)
        else:
            cur = torch.cuda.current_stream(self.device)
            side = self.__dict__.setdefault("_cap_stream", torch.cuda.Stream(device=self.device))
            side.wait_stream(cur)
            g = torch.cuda.CUDAGraph()
            l0 = self.lib.fa_launch_count()
            with torch.cuda.graph(g, stream=side):
                run()
            ent["n_launch"] = int(self.lib.fa_launch_count() - l0)    # kernels recorded into the graph (counted once here)
            cur.wait_stream(side)
            if self.__dict__.get("_buf_gen", 0) != key[-1]:              # a buffer / the workspace was replaced during capture: pointers are stale
                run()
                graphs.pop(key, None)
            else:
                ent["graph"] = g
                g.replay()                                          # the capture itself was counted by fa_launch_count
        return bufs[2], bufs[3]


class SenseVoiceEngine(_EngineBase):
    """SenseVoiceSmall (BASELINE config 4): 4 query frames + fused frontend -> 50 SAN-M blocks -> after_norm -> 20 tp
    blocks -> tp_norm -> CTC greedy (funasr/models/sense_voice/model.py:623-656, :918-1034)."""

    def __init__(self, state: Dict[str, torch.Tensor], cfg, device, gemm_mode: str = "fp32", cmvn: Optional[torch.Tensor] = None):
        self._init_base(state, device, gemm_mode, cfg.ln_eps)
        self.cfg = cfg
        names = ["encoder." + ("encoders0.0" if i == 0 else "encoders.%d" % (i - 1)) for i in range(cfg.enc_layers)]
        self.enc = self._enc_stack(names, "encoder.after_norm", cfg.heads, cfg.kernel, cfg.feat_dim)
        self.tp = self._enc_stack(["encoder.tp_encoders.%d" % i for i in range(cfg.tp_layers)], "encoder.tp_norm", cfg.heads,
                                  cfg.kernel, None) if cfg.tp_layers > 0 else None
        self.ctc = self._lin("ctc.ctc_lo")
        self.embed = self._g("embed.weight")
        self.frontend = FrontendEngine(cmvn, device)
        self._queries = {}
        torch.cuda.current_stream(self.device).synchronize()
        self._state = None

    def query_rows(self, language_id: int, textnorm_id: int) -> torch.Tensor:
        """[language, event(1), emo(2), textnorm] embedding rows (model.py:971-995); built once per combination."""
        key = (language_id, textnorm_id)
        if key not in self._queries:
            idx = torch.tensor([language_id, 1, 2, textnorm_id], device=self.device)
            self._queries[key] = self.embed.index_select(0, idx).contiguous()
        return self._queries[key]

    def forward_wav(self, wav: torch.Tensor, wav_lens: torch.Tensor, host_lens: Sequence[int], language_id: int = 0,
                    textnorm_id: int = 15, blank: int = 0, want_taps: bool = False, host_lists: bool = True):
        """wav [B, Nmax] fp32 on device -> CTC greedy ids.  No host synchronisation before the final D2H."""
        B = wav.shape[0]
        t_feat = max(num_lfr_frames(int(n)) for n in host_lens)
        T = t_feat + 4
        x = torch.empty((B, T, self.cfg.feat_dim), dtype=torch.float32, device=self.device)
        flens = torch.empty((B,), dtype=torch.int32, device=self.device)
        fe = self.frontend
        _abi.check(self.lib.fa_fbank_lfr_cmvn_tables(wav.data_ptr(), wav_lens.data_ptr(), B, wav.stride(0), _ptr(fe.cmvn), fe.tables.data_ptr(),
                                                     7, 6, x.data_ptr() + 4 * self.cfg.feat_dim * 4, T, flens.data_ptr(),
                                                     t_feat, self._stream()), "fa_fbank_lfr_cmvn_tables")
        if min(int(n) for n in host_lens) < 400:
            fe._short_rows(wav, [int(n) for n in host_lens], x[:, 4:], flens, self._stream())
        q = self.query_rows(language_id, textnorm_id)
        _abi.check(self.lib.fa_broadcast_rows(q.data_ptr(), 4, self.cfg.feat_dim, x.data_ptr(), T, B, self._stream()), "fa_broadcast_rows")
        lens = torch.tensor([num_lfr_frames(int(n)) + 4 for n in host_lens], dtype=torch.int32).to(self.device, non_blocking=True)
        enc = self._encode(self.enc, x, lens, self.cfg.d_model)
        if self.tp is not None:
            enc = self._encode(self.tp, enc, lens, self.cfg.d_model)
        V = self.cfg.vocab
        am = torch.empty((B, T), dtype=torch.int32, device=self.device)
        ids = torch.empty((B, T), dtype=torch.int32, device=self.device)
        olens = torch.empty((B,), dtype=torch.int32, device=self.device)
        logp = torch.empty((B, T, V), dtype=torch.float32, device=self.device) if want_taps else None
        ws = self._workspace(self.lib.fa_ctc_greedy_workspace_bytes(B, T, V, self.mode))
        _abi.check(self.lib.fa_ctc_greedy_forward(C.byref(self.ctc), enc.data_ptr(), lens.data_ptr(), B, T, blank, am.data_ptr(), ids.data_ptr(),
                                                  olens.data_ptr(), _ptr(logp), self.mode, ws.data_ptr(), ws.numel(), self._stream()),
                   "fa_ctc_greedy_forward")
        out = {"enc_lens": lens, "ids_dev": ids, "ids_lens_dev": olens}
        if host_lists:
            ids_h, olens_h = ids.cpu(), olens.cpu()
            out["ids"] = [ids_h[b, : int(olens_h[b])].tolist() for b in range(B)]
        if want_taps:
            out.update(enc=enc, logp=logp, argmax=am)
        return out
