"""Long-audio recognition: VAD segmentation -> duration-sorted dynamic batching -> ASR -> re-stitch with segment offsets.

Restates the caller-side loop of `AutoModel.inference_with_vad` (funasr/auto/auto_model.py:852-1035) around this backend's
models: step 1 the FSMN-VAD (`FsmnVADStreamingB200`), optional `merge_vad` (utils/vad_utils.py:57-91); step 2 the segments are
sorted by duration (:918), packed greedily while `max_len_in_batch x count < batch_size_s` and the next segment is shorter than
`batch_size_threshold_s` (:942-954), sliced out of the waveform (utils/vad_utils.py:28-54), decoded as one padded batch per pack,
restored to time order (:996-1000) and merged: timestamps shifted by the segment's start (:1008-1022), texts joined with a
space (:1029-1033), everything else (e.g. token_int) concatenated (:1034-1038).  The waveform stays on the device: slices are
views of one device tensor, so the only host<->device traffic is the waveform in and the results out.

With a speaker model (CAMPPlusB200) the recording is also diarized like the reference's `spk_model` branch (:962-979, :1101-1170) in
its `vad_segment` mode: every VAD segment is cut into 1.5 s chunks (sv_chunk), all chunks of the recording are embedded on the device
in batches, the embeddings are clustered on the host (funasr_b200.diarization) and every segment becomes one sentence
{start, end, sentence, timestamp (absolute), spk}.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _abi
from . import diarization
from .vad import merge_vad as _merge_vad


def pack_segments(segments: Sequence[Sequence[int]], batch_size_s: int = 300, batch_size_threshold_s: int = 60):
    """-> (order: indices sorted by duration, packs: list of [beg, end) ranges into `order`) exactly as auto_model.py:916-989 forms
    its batches on a GPU (on the CPU the reference decodes one segment per call, :929-930)."""
    n = len(segments)
    order = sorted(range(n), key=lambda i: (segments[i][1] - segments[i][0], i))       # sorted() is stable: ties keep time order
    if n == 0:
        return order, []
    batch_size = max(int(batch_size_s) * 1000, 1)
    threshold_ms = int(batch_size_threshold_s) * 1000
    first = segments[order[0]]
    batch_size = max(batch_size, first[1] - first[0])
    packs, beg_idx, end_idx, max_len = [], 0, 1, 0
    for j in range(n):
        length = segments[order[j]][1] - segments[order[j]][0]
        potential = max(max_len, length) * (j + 1 - beg_idx)
        if j < n - 1 and length < threshold_ms and potential < batch_size:
            max_len = max(max_len, length)
            end_idx += 1
            continue
        packs.append((beg_idx, end_idx))
        beg_idx = end_idx
        end_idx += 1
        max_len = length
    return order, packs


def merge_results(per_segment: List[dict], segments: Sequence[Sequence[int]]) -> dict:
    """auto_model.py:1003-1038: per-segment result dicts in TIME order -> one result."""
    result: dict = {}
    for j, res in enumerate(per_segment):
        for k, v in res.items():
            if k.startswith("timestamp"):
                shifted = [[int(t[0]) + int(segments[j][0]), int(t[1]) + int(segments[j][0])] for t in v]
                result.setdefault(k, []).extend(shifted)
            elif "text" in k:
                result[k] = v if k not in result else result[k] + " " + v
            elif k == "key":
                result.setdefault(k, v)
            else:
                result[k] = v if k not in result else result[k] + v
    return result


def speaker_chunks(segments: Sequence[Sequence[int]], n_total: int, fs: int = 16000):
    """VAD segments [[start_ms, end_ms], ...] in time order -> [(chunk_start_s, chunk_end_s, first_sample, n_samples)] of sv_chunk's
    windows over each segment's samples (the slice inference_with_vad decodes, vad_utils.py:44-51)."""
    out = []
    for seg in segments:
        b0 = int(seg[0] * 16)
        b1 = min(int(seg[1] * 16), n_total)
        for st, ed in diarization.chunk_bounds(max(b1 - b0, 0), fs):
            out.append((st / fs + seg[0] / 1000.0, ed / fs + seg[0] / 1000.0, b0 + st, ed - st))
    return out


def diarize(spk_model, wav_dev: torch.Tensor, segments: Sequence[Sequence[int]], device, preset_spk_num: Optional[int] = None,
            return_spk_center: bool = False) -> dict:
    """Speaker turns of one device-resident recording: chunk every segment (zero-padded 1.5 s windows gathered from the device waveform),
    embed all chunks with spk_model (CAMPPlusB200) in batches, cluster and post-process on the host.
    -> {"chunks", "spk_embedding" [n, 192] (device), "labels", "sv_output" [[start_s, end_s, spk], ...] (+ "spk_embedding_center")}."""
    chunk_len = int(diarization.SEG_DUR * 16000)
    n_total = int(wav_dev.numel())
    chunks = speaker_chunks(segments, n_total)
    if not chunks:
        return {"chunks": [], "spk_embedding": torch.zeros((0, 192), device=device), "labels": np.zeros(0, dtype=int), "sv_output": []}
    starts = torch.tensor([c[2] for c in chunks], dtype=torch.int64)
    lens = torch.tensor([c[3] for c in chunks], dtype=torch.int64)
    pos = torch.arange(chunk_len, dtype=torch.int64)
    idx = torch.where(pos[None, :] < lens[:, None], starts[:, None] + pos[None, :], torch.full((1, 1), n_total, dtype=torch.int64))
    src = torch.cat([wav_dev.reshape(-1), torch.zeros(1, dtype=wav_dev.dtype, device=wav_dev.device)])
    batch = src[idx.to(wav_dev.device, non_blocking=True)]                         # [n_chunks, 24000]: windows + zero tails
    eng = spk_model.engine(device)
    n = len(chunks)
    emb = eng.embed_wav(batch, torch.full((n,), chunk_len, dtype=torch.int32, device=wav_dev.device), [chunk_len] * n)
    emb_np = emb.cpu().numpy()
    labels = diarization.ClusterBackend()(emb_np, oracle_num=preset_spk_num)
    segs = [[c[0], c[1]] for c in chunks]
    out = {"chunks": chunks, "spk_embedding": emb, "labels": labels}
    if return_spk_center:
        out["sv_output"], out["spk_embedding_center"] = diarization.postprocess(segs, None, labels, emb_np, return_spk_center=True)
    else:
        out["sv_output"] = diarization.postprocess(segs, None, labels, emb_np)
    return out


class LongAudioPipeline:
    """vad_model / asr_model: this backend's plugin objects (e.g. FsmnVADStreamingB200, ParaformerB200 or BiCif / Seaco / Contextual);
    frontends: WavFrontendOnlineB200 (VAD) and WavFrontendB200 (ASR); spk_model: CAMPPlusB200 or None (no diarization)."""

    def __init__(self, asr_model, asr_frontend, vad_model, vad_frontend, device="cuda", tokenizer=None, spk_model=None):
        self.asr, self.asr_frontend, self.vad, self.vad_frontend = asr_model, asr_frontend, vad_model, vad_frontend
        self.device = torch.device(device)
        self.tokenizer = tokenizer
        self.spk = spk_model
        if self.device.type != "cuda":
            raise _abi.FunasrB200Error("LongAudioPipeline needs a CUDA device; there is no CPU path")

    def generate(self, wav, key: str = "utt", batch_size_s: int = 300, batch_size_threshold_s: int = 60, merge_vad: bool = False,
                 merge_length_s: int = 15, vad_kwargs: Optional[dict] = None, preset_spk_num: Optional[int] = None,
                 return_spk_center: bool = False, **cfg) -> dict:
        if self.spk is not None and "output_timestamp" not in cfg:                # auto_model.py:871-873
            cfg["output_timestamp"] = True
            cfg["return_time_stamps"] = True
        if isinstance(wav, np.ndarray):
            wav = torch.from_numpy(wav)
        wav = wav.to(torch.float32).reshape(-1)
        wav_dev = wav.to(self.device, non_blocking=True).contiguous()
        vres, _ = self.vad.inference(wav_dev, key=[key], frontend=self.vad_frontend, device=self.device, **(vad_kwargs or {}))
        segments = vres[0]["value"]
        if merge_vad:
            segments = _merge_vad(segments, int(merge_length_s) * 1000)
        n_total = int(wav.numel())
        if not segments:
            return {"key": key, "text": "", "timestamp": [], "vad_segments": []}
        order, packs = pack_segments(segments, batch_size_s, batch_size_threshold_s)
        sorted_results: List[Optional[dict]] = []
        for beg, end in packs:
            batch = []
            for i in order[beg:end]:
                b0 = int(segments[i][0] * 16)
                b1 = min(int(segments[i][1] * 16), n_total)                      # slice_padding_audio_samples (vad_utils.py:44-51)
                batch.append(wav_dev[b0:b1])
            res, _ = self.asr.inference(batch, key=["%s_%d" % (key, i) for i in order[beg:end]], tokenizer=self.tokenizer,
                                        frontend=self.asr_frontend, device=self.device, **cfg)
            if len(res) < 1:                                                     # no token in the whole batch (auto_model.py:990-991)
                continue
            sorted_results.extend(res)
        if len(sorted_results) != len(segments):                                 # :996-999
            return {"key": key, "text": "", "timestamp": [], "vad_segments": segments}
        restored: List[Optional[dict]] = [None] * len(segments)
        for j, i in enumerate(order):
            restored[i] = sorted_results[j]
        out = merge_results(restored, segments)
        out["key"] = key
        out["vad_segments"] = segments
        # the reference diarizes recordings with decoded text (:1056-1057); without a tokenizer results carry token ids instead
        decoded = out["text"].strip() if "text" in out else out.get("token_int")
        if self.spk is not None and decoded:
            d = diarize(self.spk, wav_dev, segments, self.device, preset_spk_num, return_spk_center)
            out["spk_embedding"] = d["spk_embedding"]
            if return_spk_center:
                out["spk_embedding_center"] = d["spk_embedding_center"]
            sentences = []
            for res, seg in zip(restored, segments):                              # vad_segment mode (:1150-1170), absolute timestamps
                ts = [[int(t[0]) + int(seg[0]), int(t[1]) + int(seg[0])] for t in res.get("timestamp", [])]
                sentences.append({"start": seg[0], "end": seg[1], "sentence": res.get("text", ""), "timestamp": ts})
            out["sentence_info"] = diarization.distribute_spk(sentences, d["sv_output"])
        return out
