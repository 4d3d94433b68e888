"""Speaker diarization host routines: the reference's chunking, clustering and label post-processing, restated without scikit-learn.

  sv_chunk         <- campplus/utils.py sv_chunk: 1.5 s windows every 0.75 s, the last one pulled back to end at the segment's end,
                      zero-padded when the segment is shorter than 1.5 s
  ClusterBackend   <- campplus/cluster_backend.py ClusterBackend: < 20 chunks -> one speaker; < 2048 -> spectral clustering (cosine
                      similarity, p-pruning, symmetrisation, unnormalised Laplacian, scipy.linalg.eigh, eigengap speaker count unless
                      preset, k-means on the spectral embedding); >= 2048 with a preset count -> k-means on L2-normalised embeddings;
                      then merge_by_cos at 0.78 when no count was preset.  The UMAP + HDBSCAN path (>= 2048 chunks, no preset count) is
                      not provided and raises.
  postprocess, distribute_spk, correct_labels, merge_seque, smooth  <- campplus/utils.py

The reference runs the similarity, the Laplacian and the eigendecomposition in float32 (its input is the float32 embedding tensor); so
does this module.  Its k-means is scikit-learn's; here it is a seeded k-means++ / Lloyd in numpy.  Labels are canonicalised by
correct_labels (order of first appearance), so any k-means that finds the same partition yields identical labels.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import scipy.linalg

SEG_DUR, SEG_SHIFT = 1.5, 0.75
SPECTRAL_MAX_CHUNKS = 2048


def chunk_bounds(n_samples: int, fs: int = 16000):
    """[(start_sample, end_sample)] of sv_chunk's windows over a segment of n_samples (end - start < chunk_len only when the segment
    itself is shorter than one window; that chunk is zero-padded to chunk_len)."""
    chunk_len, chunk_shift = int(SEG_DUR * fs), int(SEG_SHIFT * fs)
    out, last_ed = [], 0
    for st in range(0, n_samples, chunk_shift):
        ed = min(st + chunk_len, n_samples)
        if ed <= last_ed:
            break
        last_ed = ed
        out.append((max(0, ed - chunk_len), ed))
    return out


def sv_chunk(vad_segments: list, fs: int = 16000) -> list:
    """[[start_s, end_s, samples], ...] -> [[chunk_start_s, chunk_end_s, chunk_samples (chunk_len)], ...]."""
    chunk_len = int(SEG_DUR * fs)
    segs = []
    for seg_st, _, data in vad_segments:
        for st, ed in chunk_bounds(int(data.shape[0]), fs):
            c = data[st:ed]
            if c.shape[0] < chunk_len:
                c = np.pad(c, (0, chunk_len - c.shape[0]), "constant")
            segs.append([st / fs + seg_st, ed / fs + seg_st, c])
    return segs


def _normalize_rows(x: np.ndarray) -> np.ndarray:
    n = np.sqrt(np.einsum("ij,ij->i", x, x))
    n[n == 0.0] = 1.0
    return x / n[:, None]


def kmeans(x: np.ndarray, k: int, seed: int = 0, n_init: int = 10, max_iter: int = 300) -> np.ndarray:
    """k-means++ seeding + Lloyd iterations, best inertia of n_init runs (float64, deterministic for a seed) -> labels."""
    x = np.asarray(x, dtype=np.float64)
    n = x.shape[0]
    k = int(k)
    if k < 1 or k > n:
        raise ValueError("k-means needs 1 <= k <= n (k=%d, n=%d)" % (k, n))
    rng = np.random.RandomState(seed)
    best_lab, best_in = None, np.inf
    sq = np.einsum("ij,ij->i", x, x)
    for _ in range(n_init):
        centers = np.empty((k, x.shape[1]))
        centers[0] = x[rng.randint(n)]
        d2 = np.maximum(sq - 2 * x @ centers[0] + centers[0] @ centers[0], 0.0)
        for j in range(1, k):
            tot = d2.sum()
            idx = rng.choice(n, p=d2 / tot) if tot > 0 else rng.randint(n)
            centers[j] = x[idx]
            d2 = np.minimum(d2, np.maximum(sq - 2 * x @ centers[j] + centers[j] @ centers[j], 0.0))
        lab = None
        for _ in range(max_iter):
            dist = sq[:, None] - 2 * x @ centers.T + np.einsum("ij,ij->i", centers, centers)[None, :]
            new = np.argmin(dist, axis=1)
            if lab is not None and np.array_equal(new, lab):
                break
            lab = new
            for j in range(k):
                m = lab == j
                if m.any():
                    centers[j] = x[m].mean(0)
        inertia = float(np.sum((x - centers[lab]) ** 2))
        if inertia < best_in:
            best_in, best_lab = inertia, lab
    return best_lab


class SpectralCluster:
    def __init__(self, min_num_spks: int = 1, max_num_spks: int = 15, pval: float = 0.022):
        self.min_num_spks, self.max_num_spks, self.pval = min_num_spks, max_num_spks, pval

    def __call__(self, x: np.ndarray, oracle_num: Optional[int] = None) -> np.ndarray:
        sim = self.sim_mat(x)
        pruned = self.p_pruning(sim)
        sym = 0.5 * (pruned + pruned.T)
        lap = self.laplacian(sym)
        emb, k = self.spec_embs(lap, oracle_num)
        return kmeans(emb, k)

    @staticmethod
    def sim_mat(x: np.ndarray) -> np.ndarray:
        xn = _normalize_rows(np.asarray(x, dtype=np.float32))
        return xn @ xn.T

    def p_pruning(self, a: np.ndarray) -> np.ndarray:
        n = a.shape[0]
        pval = 6.0 / n if n * self.pval < 6 else self.pval
        n_elems = int((1 - pval) * n)
        for i in range(n):
            a[i, np.argsort(a[i, :])[:n_elems]] = 0
        return a

    @staticmethod
    def laplacian(m: np.ndarray) -> np.ndarray:
        m[np.diag_indices(m.shape[0])] = 0
        return np.diag(np.sum(np.abs(m), axis=1)) - m

    def spec_embs(self, lap: np.ndarray, k_oracle: Optional[int] = None):
        lambdas, vecs = scipy.linalg.eigh(lap)
        if k_oracle is not None:
            k = int(k_oracle)
        else:
            ev = lambdas[self.min_num_spks - 1:self.max_num_spks + 1]
            gaps = [float(ev[i + 1]) - float(ev[i]) for i in range(len(ev) - 1)]
            k = int(np.argmax(gaps)) + self.min_num_spks
        return vecs[:, :k], k


class ClusterBackend:
    """labels = ClusterBackend()(embeddings [N, C], oracle_num=None)."""

    def __init__(self, merge_thr: float = 0.78):
        self.merge_thr = merge_thr
        self.spectral = SpectralCluster()

    def __call__(self, x, oracle_num: Optional[int] = None) -> np.ndarray:
        x = np.asarray(x.detach().cpu().numpy() if hasattr(x, "detach") else x, dtype=np.float32)
        if x.ndim != 2:
            raise ValueError("embeddings must be [N, C]")
        if x.shape[0] < 20:
            return np.zeros(x.shape[0], dtype=int)
        if x.shape[0] < SPECTRAL_MAX_CHUNKS:
            labels = self.spectral(x, oracle_num)
        elif oracle_num is not None:
            labels = kmeans(_normalize_rows(x), oracle_num)
        else:
            raise NotImplementedError("%d speaker chunks without preset_spk_num: the reference clusters %d or more chunks with UMAP + HDBSCAN, "
                                      "which this backend does not provide; pass preset_spk_num or diarize fewer than %d chunks"
                                      % (x.shape[0], SPECTRAL_MAX_CHUNKS, SPECTRAL_MAX_CHUNKS))
        if oracle_num is None:
            labels = self.merge_by_cos(labels, x, self.merge_thr)
        return labels

    @staticmethod
    def merge_by_cos(labels: np.ndarray, embs: np.ndarray, cos_thr: float) -> np.ndarray:
        labels = np.array(labels)
        while True:
            spk_num = labels.max() + 1
            if spk_num == 1:
                break
            center = np.stack([embs[labels == i].mean(0) for i in range(spk_num)], axis=0)
            center = center / np.linalg.norm(center, axis=1, keepdims=True)
            aff = np.triu(center @ center.T, 1)
            a, b = np.unravel_index(np.argmax(aff), aff.shape)
            if aff[a, b] < cos_thr:
                break
            labels[labels == b] = a
            labels[labels > b] -= 1
        return labels


def correct_labels(labels) -> np.ndarray:
    id2id, out = {}, []
    for i in labels:
        if i not in id2id:
            id2id[i] = len(id2id)
        out.append(id2id[i])
    return np.array(out)


def merge_seque(res: list) -> list:
    out = [res[0]]
    for r in res[1:]:
        if r[2] != out[-1][2] or r[0] > out[-1][1]:
            out.append(r)
        else:
            out[-1][1] = r[1]
    return out


def smooth(res: list, mindur: float = 0.7) -> list:
    if len(res) < 2:
        return res
    for i in range(len(res)):
        res[i][0] = round(res[i][0], 2)
        res[i][1] = round(res[i][1], 2)
        if res[i][1] - res[i][0] < mindur:
            if i == 0:
                res[i][2] = res[i + 1][2]
            elif i == len(res) - 1:
                res[i][2] = res[i - 1][2]
            elif res[i][0] - res[i - 1][1] <= res[i + 1][0] - res[i][1]:
                res[i][2] = res[i - 1][2]
            else:
                res[i][2] = res[i + 1][2]
    return merge_seque(res)


def postprocess(segments: list, vad_segments, labels, embeddings: np.ndarray, return_spk_center: bool = False):
    """Chunks [[start_s, end_s, ...], ...] in time order + their labels -> [[start_s, end_s, spk], ...] speaker turns (and the
    per-speaker mean embeddings when return_spk_center)."""
    if len(segments) != len(labels):
        raise ValueError("one label per chunk expected")
    labels = correct_labels(labels)
    res = merge_seque([[segments[i][0], segments[i][1], labels[i]] for i in range(len(segments))])
    for i in range(1, len(res)):
        if res[i - 1][1] > res[i][0] + 1e-4:               # overlapping turns meet at the midpoint
            p = (res[i][0] + res[i - 1][1]) / 2
            res[i][0] = p
            res[i - 1][1] = p
    res = smooth(res)
    if return_spk_center:
        centers = np.stack([embeddings[labels == i].mean(0) for i in range(labels.max() + 1)])
        return res, centers
    return res


def distribute_spk(sentence_list: List[dict], sd_time_list: Sequence) -> List[dict]:
    """Give every sentence {start, end (ms), ...} the speaker whose turns overlap it most (turns in seconds)."""
    sd = [(st * 1000, ed * 1000, spk) for st, ed, spk in sd_time_list]
    for d in sentence_list:
        s0, s1 = d["start"], d["end"]
        spk_best, max_ov = 0, 0
        for st, ed, spk in sd:
            ov = max(min(s1, ed) - max(s0, st), 0)
            if ov > max_ov:
                max_ov = ov
                spk_best = spk
            if ov > 0 and spk_best == spk:
                max_ov += ov
        d["spk"] = int(spk_best)
    return sentence_list
