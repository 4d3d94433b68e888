"""ctypes binding of the handle-style C API (include/funasr_b200.h: fa_offline_*), the counterpart of FunASR's C++ runtime
FunOfflineInit / FunOfflineInferBuffer / FunASRGetResult (runtime/onnxruntime/include/funasrruntime.h:100-116).
Nothing here touches torch on the data path: host PCM buffers in, token ids out.  `OfflineVad` binds the FSMN-VAD handle
(fa_vad_*) and `OfflineRecognizer.infer_long` the long-audio entry (fa_offline_infer_vad): VAD segments packed by duration and decoded
batch by batch, the same results as LongAudioPipeline.generate.  A BiCifParaformer model file adds per-token [start_ms, end_ms] stamps
(`infer_stamped`, and "timestamp" in `infer_long`'s results); a SeacoParaformer model file takes hotword rows from
`hotword_embeddings` (its hotword encoder on the GPU).  `OfflinePunc` binds the CT-Transformer punctuation handle (fa_punc_*),
and `punc_walk_host` its text walk with any scorer in place of the network.  `OfflineSpeaker` binds the CAM++ speaker handle (fa_spk_*);
passed to `infer_long(spk=...)` it diarizes long audio (fa_offline_infer_vad_spk).  `OfflineAligner` binds the MonotonicAligner's
forced-alignment handle (fa_align_*): per-token stamps for transcripts the caller already has."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import numpy as np

from . import _abi


_SAMPLE_FORMATS = {np.dtype(np.float32): 0, np.dtype(np.int16): 1, np.dtype(np.int32): 3, np.dtype(np.uint8): 4}


def _pcm_batch(wavs, fs: int = 16000, resampler: str = "loader"):
    """-> (contiguous arrays, pcm_format, FaAudioFormat or None).  None: 16 kHz mono float32 / int16, which the 16 kHz entries take;
    otherwise the descriptor of the `_audio` entries.  Arrays are 1-D (mono) or 2-D [frames, channels] of one dtype: float32 in
    [-1, 1], int16, int32 or uint8 PCM (s24 only through the C API)."""
    arrs = [np.ascontiguousarray(w) for w in wavs]
    kinds = {a.dtype for a in arrs}
    if len(kinds) != 1 or next(iter(kinds)) not in _SAMPLE_FORMATS:
        raise _abi.FunasrB200Error("waveforms must all be float32, all int16, all int32 or all uint8, got %s" % kinds)
    if any(a.ndim not in (1, 2) for a in arrs) or len({1 if a.ndim == 1 else a.shape[1] for a in arrs}) != 1:
        raise _abi.FunasrB200Error("waveforms must be 1-D or [frames, channels] with the same channel count")
    if resampler not in _abi.RESAMPLERS:
        raise _abi.FunasrB200Error("resampler must be one of %s, got %r" % (sorted(_abi.RESAMPLERS), resampler))
    fmt = _SAMPLE_FORMATS[kinds.pop()]
    channels = 1 if arrs[0].ndim == 1 else arrs[0].shape[1]
    if int(fs) == 16000 and fmt in (0, 1) and all(a.ndim == 1 for a in arrs):
        return arrs, fmt, None
    return arrs, fmt, _abi.FaAudioFormat(fmt, channels, int(fs), _abi.RESAMPLERS[resampler])


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data


def _vad_run_options(max_end_silence_time: Optional[int] = None, speech_noise_thres: Optional[float] = None,
                     dynamic_silence: Optional[bool] = None) -> "_abi.FaVadRunOptions":
    """FsmnVADStreamingB200.inference's keywords: an explicit max_end_silence_time switches the dynamic schedule off."""
    if dynamic_silence is None:
        dynamic_silence = max_end_silence_time is None
    return _abi.FaVadRunOptions(1 if dynamic_silence else 0, int(max_end_silence_time or 0),
                                float("nan") if speech_noise_thres is None else float(speech_noise_thres))


class OfflineVad:
    """ctypes binding of fa_vad_init / fa_vad_infer: FSMN-VAD from a model file written by pack.write_vad_model_file."""

    def __init__(self, model_file: str, device: int = 0):
        self.lib = _abi.load()
        self.handle = self.lib.fa_vad_init(model_file.encode(), device)
        if not self.handle:
            raise _abi.FunasrB200Error("fa_vad_init failed: %s" % self.lib.fa_offline_last_error().decode())

    def segments(self, wav: np.ndarray, want_frames: bool = False, fs: int = 16000, resampler: str = "loader", **vad_kwargs):
        """wav: float32 in [-1, 1] or int16 (int32, uint8) PCM, 1-D or [frames, channels], at fs Hz (resampled to 16 kHz on the GPU
        by `resampler`: "loader" or "runtime") -> [[start_ms, end_ms], ...] (and the [2, frames] silence posterior / energy)."""
        (a,), fmt, desc = _pcm_batch([wav], fs, resampler)
        opts = _vad_run_options(**vad_kwargs)
        if desc is None:
            res = self.lib.fa_vad_infer(self.handle, a.ctypes.data, a.shape[0], fmt, C.byref(opts))
        else:
            res = self.lib.fa_vad_infer_audio(self.handle, a.ctypes.data, a.shape[0], C.byref(desc), C.byref(opts))
        if not res:
            raise _abi.FunasrB200Error("fa_vad_infer failed: %s" % self.lib.fa_offline_last_error().decode())
        try:
            n = C.c_int64(0)
            p = self.lib.fa_vad_result_segments(res, C.byref(n))
            segs = [[int(p[2 * i]), int(p[2 * i + 1])] for i in range(n.value)]
            if not want_frames:
                return segs
            f = self.lib.fa_vad_result_frames(res, C.byref(n))
            frames = np.ctypeslib.as_array(f, shape=(2, n.value)).copy() if n.value else np.zeros((2, 0), np.float32)
            return segs, frames
        finally:
            self.lib.fa_vad_free_result(res)

    def close(self):
        if getattr(self, "handle", None):
            self.lib.fa_vad_uninit(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _punc_result(lib, res, n: int) -> List[dict]:
    out = []
    cnt = C.c_int32(0)
    for i in range(n):
        p = lib.fa_punc_result_ids(res, i, C.byref(cnt))
        out.append({"text": lib.fa_punc_result_text(res, i).decode("utf-8"), "punc_array": [int(p[k]) for k in range(cnt.value)]})
    return out


def _c_strings(items: Sequence[str]):
    enc = [s.encode("utf-8") for s in items]
    return (C.c_char_p * max(len(enc), 1))(*enc), enc


class OfflinePunc:
    """ctypes binding of fa_punc_init / fa_punc_infer: CT-Transformer punctuation from a model file written by
    pack.write_punc_model_file.  `infer` punctuates many texts in one call, all of them advancing one window per step."""

    def __init__(self, model_file: str, device: int = 0):
        self.lib = _abi.load()
        self.handle = self.lib.fa_punc_init(model_file.encode(), device)
        if not self.handle:
            raise _abi.FunasrB200Error("fa_punc_init failed: %s" % self.lib.fa_offline_last_error().decode())
        self.last_steps = 0

    def infer(self, texts: Sequence[str]) -> List[dict]:
        """texts -> per text {"text": punctuated text, "punc_array": punctuation id per word} (CTTransformer.inference's result;
        "" and [] for an empty text)."""
        arr, _keep = _c_strings(texts)
        res = self.lib.fa_punc_infer(self.handle, arr, len(texts))
        if not res:
            raise _abi.FunasrB200Error("fa_punc_infer failed: %s" % self.lib.fa_offline_last_error().decode())
        try:
            self.last_steps = int(self.lib.fa_punc_result_steps(res))
            return _punc_result(self.lib, res, len(texts))
        finally:
            self.lib.fa_punc_free_result(res)

    def pool_stats(self):
        """(calls, steps): the calls the handle's pool has admitted since init and the lockstep steps it ran them in; concurrent
        `infer` calls from many threads share steps."""
        c, s = C.c_int64(), C.c_int64()
        _abi.check(self.lib.fa_punc_pool_stats(self.handle, C.byref(c), C.byref(s)), "fa_punc_pool_stats")
        return c.value, s.value

    def close(self):
        if getattr(self, "handle", None):
            self.lib.fa_punc_uninit(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def punc_walk_host(texts: Sequence[str], token_list: Sequence[str], punc_list: Sequence[str], sentence_end_id: int, score,
                   split_size: int = 20, max_window: int = 0) -> List[dict]:
    """fa_punc_walk_host: the punctuation walk of fa_punc_infer with `score` in place of the network.  score(ids [batch, t_max] int32,
    lens [batch] int32) -> punctuation ids [batch, t_max] (only each row's first lens[b] entries are read)."""
    lib = _abi.load()
    err = []

    def cb(_ctx, ids, lens, batch, t_max, out):
        try:
            i = np.ctypeslib.as_array(ids, shape=(batch, t_max)).copy()
            n = np.ctypeslib.as_array(lens, shape=(batch,)).copy()
            np.ctypeslib.as_array(out, shape=(batch, t_max))[:] = np.asarray(score(i, n), dtype=np.int32)
            return 0
        except Exception as e:                                  # an exception must not cross the C frames
            err.append(e)
            return 1

    fn = _abi.PUNC_SCORE_FN(cb)
    ta, _k1 = _c_strings(texts)
    tok, _k2 = _c_strings(token_list)
    pl, _k3 = _c_strings(punc_list)
    res = lib.fa_punc_walk_host(ta, len(texts), tok, len(token_list), pl, len(punc_list), int(sentence_end_id), int(split_size), int(max_window),
                                fn, None)
    if err:
        if res:
            lib.fa_punc_free_result(res)
        raise err[0]
    if not res:
        raise _abi.FunasrB200Error("fa_punc_walk_host failed: %s" % lib.fa_offline_last_error().decode())
    try:
        return _punc_result(lib, res, len(texts))
    finally:
        lib.fa_punc_free_result(res)


def sv_query_ids(n: int, language=None, use_itn=None):
    """SenseVoice queries of n utterances or recordings -> (language ids, textnorm ids) as int32 arrays, through SenseVoiceSmallB200's
    lid_dict / textnorm_dict (an unknown language is "auto", as in SenseVoiceSmall.inference).  language: one name or one per item
    (default "auto"); use_itn: one bool or one per item (default False)."""
    from .modules import SenseVoiceSmallB200
    langs = ["auto" if language is None else language] * n if language is None or isinstance(language, str) else list(language)
    itns = [bool(use_itn)] * n if use_itn is None or isinstance(use_itn, (bool, int, np.bool_)) else [bool(v) for v in use_itn]
    if len(langs) != n or len(itns) != n:
        raise _abi.FunasrB200Error("language / use_itn: one value or one per item (%d items)" % n)
    tn = SenseVoiceSmallB200.textnorm_dict
    lid = np.array([SenseVoiceSmallB200.lid_dict.get(x, 0) for x in langs], dtype=np.int32)
    return lid, np.array([tn["withitn" if v else "woitn"] for v in itns], dtype=np.int32)


class OfflineSpeaker:
    """CAM++ speaker embeddings through the C handle (fa_spk_init / fa_spk_embed) from a pack.write_campplus_model_file file; pass it
    to OfflineRecognizer.infer_long(spk=...) to diarize long audio."""

    def __init__(self, model_file: str, device: int = 0, gemm_mode: str = "fp32"):
        self.lib = _abi.load()
        self.handle = self.lib.fa_spk_init(model_file.encode(), int(device), _abi.GEMM_MODES[gemm_mode])
        if not self.handle:
            raise _abi.FunasrB200Error("fa_spk_init failed: %s" % self.lib.fa_offline_last_error().decode())

    def embed(self, wavs: Sequence[np.ndarray], fs: int = 16000, resampler: str = "loader") -> np.ndarray:
        """Ragged recordings (float32 in [-1, 1] or int16 (int32, uint8) PCM, 1-D or [frames, channels], at fs Hz; `resampler` as in
        OfflineVad.segments) -> [B, 192] float32, CAMPPlusB200.inference's embeddings."""
        arrs, fmt, desc = _pcm_batch(wavs, fs, resampler)
        n = len(arrs)
        ptrs = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
        lens = (C.c_int64 * n)(*[a.shape[0] for a in arrs])
        out = np.empty((n, 192), dtype=np.float32)
        rc = (self.lib.fa_spk_embed(self.handle, ptrs, lens, n, fmt, out.ctypes.data) if desc is None else
              self.lib.fa_spk_embed_audio(self.handle, ptrs, lens, n, C.byref(desc), out.ctypes.data))
        if rc != 0:
            raise _abi.FunasrB200Error("fa_spk_embed failed: %s" % self.lib.fa_offline_last_error().decode())
        return out

    def pool_stats(self):
        """(calls, passes): the embedding and clustering calls the handle's pool has served since init and the passes it ran them in;
        concurrent `embed` calls from many threads share passes."""
        c, p = C.c_int64(), C.c_int64()
        _abi.check(self.lib.fa_spk_pool_stats(self.handle, C.byref(c), C.byref(p)), "fa_spk_pool_stats")
        return c.value, p.value

    def close(self):
        if getattr(self, "handle", None):
            self.lib.fa_spk_uninit(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class OfflineAligner:
    """Forced alignment through the C handle (fa_align_init / fa_align_infer): the MonotonicAligner (fa-zh) from a
    pack.write_aligner_model_file file."""

    def __init__(self, model_file: str, device: int = 0, gemm_mode: str = "fp16x3"):
        self.lib = _abi.load()
        mode = _abi.GEMM_MODES[gemm_mode] if isinstance(gemm_mode, str) else int(gemm_mode)
        self.handle = self.lib.fa_align_init(model_file.encode(), int(device), mode)
        if not self.handle:
            raise _abi.FunasrB200Error("fa_align_init failed: %s" % self.lib.fa_offline_last_error().decode())

    def align(self, wavs: Sequence[np.ndarray], token_ids: Sequence[Sequence[int]], fs: int = 16000,
              resampler: str = "loader") -> List[List[List[int]]]:
        """wavs (float32 in [-1, 1] or int16 (int32, uint8) PCM, 1-D or [frames, channels], at fs Hz; `resampler` as in
        OfflineRecognizer.infer) and one transcript of token ids per wav -> per wav [[start_ms, end_ms], ...], MonotonicAligner.inference's
        "timestamp" for CJK character tokens: one stamp per token (a trailing </s> dropped), fewer when the audio cannot fire for
        them all."""
        arrs, fmt, _ = _pcm_batch(wavs, fs, resampler)
        n = len(arrs)
        if len(token_ids) != n:
            raise _abi.FunasrB200Error("one transcript per waveform: %d waveforms, %d transcripts" % (n, len(token_ids)))
        desc = _abi.FaAudioFormat(fmt, 1 if arrs[0].ndim == 1 else arrs[0].shape[1], int(fs), _abi.RESAMPLERS[resampler])
        toks = [np.ascontiguousarray(t, dtype=np.int32).reshape(-1) for t in token_ids]
        ptrs = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
        lens = (C.c_int64 * n)(*[a.shape[0] for a in arrs])
        id_ptrs = (C.c_void_p * n)(*[t.ctypes.data if t.size else None for t in toks])
        n_ids = (C.c_int32 * n)(*[t.size for t in toks])
        res = self.lib.fa_align_infer(self.handle, ptrs, lens, n, C.byref(desc), id_ptrs, n_ids)
        if not res:
            raise _abi.FunasrB200Error("fa_align_infer failed: %s" % self.lib.fa_offline_last_error().decode())
        try:
            cnt = C.c_int32(0)
            out = []
            for i in range(self.lib.fa_offline_result_count(res)):
                p = self.lib.fa_offline_result_stamps(res, i, C.byref(cnt))
                out.append([[int(p[2 * k]), int(p[2 * k + 1])] for k in range(cnt.value)])
            self.last_audio_seconds = float(self.lib.fa_offline_result_audio_seconds(res))
            return out
        finally:
            self.lib.fa_offline_free_result(res)

    def close(self):
        if getattr(self, "handle", None):
            self.lib.fa_align_uninit(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class OfflineRecognizer:
    def __init__(self, model_file: str, device: int = 0, gemm_mode: str = "fp16x3"):
        self.lib = _abi.load()
        mode = _abi.GEMM_MODES[gemm_mode] if isinstance(gemm_mode, str) else int(gemm_mode)
        self.handle = self.lib.fa_offline_init(model_file.encode(), device, mode)
        if not self.handle:
            raise _abi.FunasrB200Error("fa_offline_init failed: %s" % self.lib.fa_offline_last_error().decode())

    @property
    def has_timestamps(self) -> bool:
        """True for a BiCifParaformer model file: results carry per-token stamps from its upsampled CIF head."""
        return bool(self.lib.fa_offline_has_timestamps(self.handle))

    @property
    def is_sensevoice(self) -> bool:
        """True for a SenseVoiceSmall model file: `infer` / `infer_long` take `language` and `use_itn`."""
        return bool(self.lib.fa_offline_is_sensevoice(self.handle))

    @property
    def is_seaco(self) -> bool:
        """True for a SeacoParaformer model file: `hotword_embeddings` gives the rows `infer` / `infer_long` take."""
        return bool(self.lib.fa_offline_is_seaco(self.handle))

    def hotword_embeddings(self, hw_lists: Sequence[Sequence[int]]) -> np.ndarray:
        """SeACo hotword rows (fa_offline_hotword_embed): token-id lists, the <s> entry [1] last as generate_hotwords_list returns them,
        -> [n, 512] float32, each hotword's bias_encoder output at its last token, computed on the GPU."""
        lens = np.array([len(h) for h in hw_lists], dtype=np.int32)
        ids = np.array([t for h in hw_lists for t in h], dtype=np.int32)
        rows = np.zeros((len(hw_lists), 512), dtype=np.float32)
        rc = self.lib.fa_offline_hotword_embed(self.handle, ids.ctypes.data, lens.ctypes.data, len(hw_lists), rows.ctypes.data)
        if rc != 0:
            raise _abi.FunasrB200Error("fa_offline_hotword_embed failed: %s" % self.lib.fa_offline_last_error().decode())
        return rows

    def _queries(self, n: int, language, use_itn):
        if not self.is_sensevoice:
            if language is not None or use_itn is not None:
                raise _abi.FunasrB200Error("language / use_itn apply to a SenseVoice model file only")
            return None
        return sv_query_ids(n, language, use_itn)

    def _stamps(self, res, i) -> List[List[int]]:
        cnt = C.c_int32(0)
        p = self.lib.fa_offline_result_stamps(res, i, C.byref(cnt))
        return [[int(p[2 * k]), int(p[2 * k + 1])] for k in range(cnt.value)]

    def _infer(self, wavs, stamped: bool, language=None, use_itn=None, hotword_embeddings=None, fs: int = 16000, resampler: str = "loader"):
        arrs, fmt, desc = _pcm_batch(wavs, fs, resampler)
        n = len(arrs)
        ptrs = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
        lens = (C.c_int64 * n)(*[a.shape[0] for a in arrs])
        q = self._queries(n, language, use_itn)
        if desc is not None:
            hw = None if hotword_embeddings is None else np.ascontiguousarray(hotword_embeddings, dtype=np.float32)
            res = self.lib.fa_offline_infer_audio(self.handle, ptrs, lens, n, C.byref(desc), _ptr(hw), 0 if hw is None else hw.shape[0],
                                                  None if q is None else q[0].ctypes.data, None if q is None else q[1].ctypes.data)
        elif hotword_embeddings is not None:
            hw = np.ascontiguousarray(hotword_embeddings, dtype=np.float32)
            res = self.lib.fa_offline_infer_hw(self.handle, ptrs, lens, n, fmt, hw.ctypes.data, hw.shape[0])
        elif q is None:
            res = self.lib.fa_offline_infer(self.handle, ptrs, lens, n, fmt)
        else:
            res = self.lib.fa_offline_infer_sv(self.handle, ptrs, lens, n, fmt, q[0].ctypes.data, q[1].ctypes.data)
        if not res:
            raise _abi.FunasrB200Error("fa_offline_infer failed: %s" % self.lib.fa_offline_last_error().decode())
        try:
            out = []
            cnt = C.c_int32(0)
            for i in range(self.lib.fa_offline_result_count(res)):
                p = self.lib.fa_offline_result_ids(res, i, C.byref(cnt))
                ids = [int(p[k]) for k in range(cnt.value)]
                out.append({"token_int": ids, "timestamp": self._stamps(res, i)} if stamped else ids)
            self.last_audio_seconds = float(self.lib.fa_offline_result_audio_seconds(res))
            return out
        finally:
            self.lib.fa_offline_free_result(res)

    def infer(self, wavs: Sequence[np.ndarray], language=None, use_itn=None, hotword_embeddings: Optional[np.ndarray] = None,
              fs: int = 16000, resampler: str = "loader") -> List[List[int]]:
        """wavs: float32 arrays in [-1, 1] or int16 PCM arrays (all the same dtype; int32 and uint8 PCM too), 1-D or [frames, channels],
        at fs Hz, >= 400 samples each at 16 kHz.  Other rates and layouts are averaged to mono and resampled to 16 kHz on the GPU:
        resampler "loader" as FunASR's Python loader and inference(fs=) (torchaudio's sinc), "runtime" as the C++ runtime (LinearResample).
        SenseVoice model file: language (one name or one per utterance, default "auto") and use_itn (default False) choose each
        utterance's query; the ids include the four tag tokens (SenseVoiceSmall.inference's token_int).  hotword_embeddings: [n, 512]
        float32 rows, the last one the <s> entry (ContextualParaformer's encoder, or `hotword_embeddings()` of a SeACo model file)."""
        return self._infer(wavs, False, language, use_itn, hotword_embeddings, fs, resampler)

    def infer_stamped(self, wavs: Sequence[np.ndarray], hotword_embeddings: Optional[np.ndarray] = None, fs: int = 16000,
                      resampler: str = "loader") -> List[dict]:
        """Like `infer`, per utterance {"token_int": ids, "timestamp": [[start_ms, end_ms], ...]} (BiCifParaformer.inference's result;
        no stamps for a model without the timestamp head)."""
        return self._infer(wavs, True, hotword_embeddings=hotword_embeddings, fs=fs, resampler=resampler)

    def infer_long(self, wavs: Sequence[np.ndarray], vad: OfflineVad, batch_size_s: int = 300, batch_size_threshold_s: int = 60,
                   merge_vad: bool = False, merge_length_s: int = 15, hotword_embeddings: Optional[np.ndarray] = None,
                   language=None, use_itn=None, spk: Optional["OfflineSpeaker"] = None, preset_spk_num: Optional[int] = None,
                   fs: int = 16000, resampler: str = "loader", **vad_kwargs) -> List[dict]:
        """Long recordings through fa_offline_infer_vad, each on its own as LongAudioPipeline.generate treats it -> per recording
        {"token_int": ids in time order, "vad_segments": [[start_ms, end_ms], ...], "n_tokens": tokens per segment}, plus
        "timestamp": [[start_ms, end_ms], ...] in absolute ms when the model has the timestamp head (`has_timestamps`).
        hotword_embeddings: [n, 512] float32 rows (ContextualParaformer or SeACo; last row the <s> entry).  SenseVoice model file
        (fa_offline_infer_vad_sv): language / use_itn as in `infer`, one per recording, applied to all its segments.
        spk (an OfflineSpeaker on the same device): fa_offline_infer_vad_spk also diarizes every recording that decoded a token and adds
        "spk", one speaker per VAD segment (vad_segment mode), with preset_spk_num as LongAudioPipeline.generate takes it.
        fs / resampler and the array layouts as in `infer` (fa_offline_infer_vad_audio); segments and stamps are ms of the recording."""
        arrs, fmt, desc = _pcm_batch(wavs, fs, resampler)
        n = len(arrs)
        ptrs = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
        lens = (C.c_int64 * n)(*[a.shape[0] for a in arrs])
        opts = _abi.FaLongAudioOptions(int(batch_size_s), int(batch_size_threshold_s), 1 if merge_vad else 0, int(merge_length_s),
                                       _vad_run_options(**vad_kwargs))
        hw, n_hw = None, 0
        if hotword_embeddings is not None:
            hw = np.ascontiguousarray(hotword_embeddings, dtype=np.float32)
            n_hw = hw.shape[0]
        q = self._queries(n, language, use_itn)
        if desc is not None:
            res = self.lib.fa_offline_infer_vad_audio(self.handle, vad.handle, None if spk is None else spk.handle, ptrs, lens, n, C.byref(desc),
                                                      _ptr(hw), n_hw, None if q is None else q[0].ctypes.data,
                                                      None if q is None else q[1].ctypes.data, C.byref(opts), int(preset_spk_num or 0))
        elif spk is not None:
            res = self.lib.fa_offline_infer_vad_spk(self.handle, vad.handle, spk.handle, ptrs, lens, n, fmt, None if hw is None else hw.ctypes.data,
                                                    n_hw, None if q is None else q[0].ctypes.data, None if q is None else q[1].ctypes.data,
                                                    C.byref(opts), int(preset_spk_num or 0))
        elif q is None:
            res = self.lib.fa_offline_infer_vad(self.handle, vad.handle, ptrs, lens, n, fmt, None if hw is None else hw.ctypes.data, n_hw,
                                                C.byref(opts))
        else:
            res = self.lib.fa_offline_infer_vad_sv(self.handle, vad.handle, ptrs, lens, n, fmt, q[0].ctypes.data, q[1].ctypes.data, C.byref(opts))
        if not res:
            raise _abi.FunasrB200Error("fa_offline_infer_vad failed: %s" % self.lib.fa_offline_last_error().decode())
        try:
            out = []
            cnt = C.c_int32(0)
            stamped = self.has_timestamps
            for i in range(self.lib.fa_offline_result_count(res)):
                p = self.lib.fa_offline_result_ids(res, i, C.byref(cnt))
                ids = [int(p[k]) for k in range(cnt.value)]
                s = self.lib.fa_offline_result_segments(res, i, C.byref(cnt))
                trip = [[int(s[3 * k]), int(s[3 * k + 1]), int(s[3 * k + 2])] for k in range(cnt.value)]
                out.append({"token_int": ids, "vad_segments": [t[:2] for t in trip], "n_tokens": [t[2] for t in trip]})
                if stamped:
                    out[-1]["timestamp"] = self._stamps(res, i)
                if spk is not None:
                    p = self.lib.fa_offline_result_spk(res, i, C.byref(cnt))
                    out[-1]["spk"] = [int(p[k]) for k in range(cnt.value)]
            self.last_audio_seconds = float(self.lib.fa_offline_result_audio_seconds(res))
            return out
        finally:
            self.lib.fa_offline_free_result(res)

    def close(self):
        if getattr(self, "handle", None):
            self.lib.fa_offline_uninit(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
