"""CPU restatement of MonotonicAligner.inference (funasr/models/monotonic_aligner/model.py:182-267) — checker only.

The aligner is the SAN-M encoder (d = 320, 4 x 80 heads for fa-zh) plus CifPredictorV3.get_upsample_timestamp with
token_num = len(tokens) + 1, then ts_prediction_lfr6_standard on the first 3 * enc_len upsampled weights.  Every stage is
the one paraformer_oracle.py already restates for BiCifParaformer; nothing there depends on d = 512.
"""
from typing import Dict, List, Optional

import torch
from torch import Tensor

import paraformer_oracle as O


def aligner_forward(wavs: List[Tensor], token_lists: List[List[int]], p: Dict[str, Tensor], cmvn: Optional[Tensor], enc_layers: int,
                    heads: int = 4, eps: float = 1e-12, smooth2: float = 0.25, noise2: float = 0.01, threshold: float = 1.0):
    """-> {"enc", "enc_lens", "token_num", "us_alphas", "us_peaks"} for a batch of (waveform, token ids) pairs."""
    with torch.no_grad():
        feats, flens = O.frontend(wavs, cmvn)
        enc, elens = O.encoder(feats, flens, p, enc_layers, heads, eps, None)
        tok = torch.tensor([len(t) + 1 for t in token_lists])                 # model.py:226-228
        us_alphas, us_peaks = O.upsample_timestamp(enc, elens, tok, p, smooth2, noise2, threshold)
    return {"enc": enc, "enc_lens": elens, "token_num": tok.to(torch.int32), "us_alphas": us_alphas, "us_peaks": us_peaks}


def fire_margin(us_alphas: Tensor, enc_lens: Tensor, threshold: float = 1.0) -> float:
    """Smallest |integrate - (threshold - 1e-4)| over the valid frames of cif_wo_hidden: how far every fire / no-fire decision of
    the timestamp scan is from flipping."""
    thr = threshold - 1e-4
    m = float("inf")
    for i in range(us_alphas.shape[0]):
        n = int(enc_lens[i]) * 3
        integ = 0.0
        for a in us_alphas[i, :n].tolist():
            integ += a
            m = min(m, abs(integ - thr))
            if integ >= thr:
                integ -= thr
    return m
