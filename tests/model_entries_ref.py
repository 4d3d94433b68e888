"""Float64 restatement of the model-level entry points (csrc/model.cu) and the per-row metric their parity tests use.

The restatement runs oracle/paraformer_oracle.py's own functions (encoder_layer, cif_alphas, cif_tail, sanm_decoder_layers,
sanm_decoder_hidden, contextual_decoder) on float64 copies of the weights and inputs.  Two pieces are restated here:
- the position encoding: the reference (and layernorm.cu) forms the argument pos x inv_timescale in fp32 and only then takes sin
  / cos; the restatement rounds the argument the same way and evaluates sin / cos in the tensor's dtype (a float64 argument
  differs from the reference by up to ~1e-4 at T = 1000);
- integrate-and-fire: cif_v1 / cif_loop round their running sums to fp32, so `cif_fire` restates the same integrate-and-fire in
  the input's dtype (both reference variants compute it; they differ only in fp32 rounding).
Padded rows are produced exactly as the reference defines them (zero-padded input, attention over the valid keys, masked FSMN,
FFN): nothing zeroes them.
"""
import numpy as np
import torch
import torch.nn.functional as F

import paraformer_oracle as O

# Per-row metric: err_r = max_c |got - ref| / max(max_c |ref|, FLOOR).  FLOOR keeps an all-zero reference row (an empty acoustic
# row, a fully masked context) from dividing by zero; every row the tests compare after a LayerNorm has max |ref| well above it.
FLOOR = 1e-2


def row_err(got, ref, floor=FLOOR):
    """[..., C] x [..., C] -> [...] per-row relative error (float64)."""
    g = np.asarray(got, dtype=np.float64)
    r = np.asarray(ref, dtype=np.float64)
    return np.abs(g - r).max(-1) / np.maximum(np.abs(r).max(-1), floor)


def worst(err, valid=None):
    """-> (value, index tuple, valid flag) of the largest entry of err; valid: bool array of err's shape (None: all valid)."""
    err = np.asarray(err, dtype=np.float64)
    if err.size == 0:
        return 0.0, (), True
    i = np.unravel_index(int(np.argmax(err)), err.shape)
    return float(err[i]), tuple(int(v) for v in i), True if valid is None else bool(np.asarray(valid)[i])


def describe(name, w):
    """'name 1.2e-05 at (utt 1, row 7, padded)' for a worst() result over [B, T] rows."""
    v, idx, ok = w
    where = ("utt %d, row %d" % idx[:2]) if len(idx) >= 2 else ("index %s" % (idx,))
    return "%s %.3e at (%s, %s)" % (name, v, where, "valid" if ok else "padded")


def to64(p):
    return {k: v.double() for k, v in p.items()}


def len_mask(lens, T):
    """[B, T] bool: row t of utterance b is valid."""
    return np.arange(T)[None, :] < np.asarray(lens)[:, None]


# ------------------------------------------------------------------------------------------------ encoder
def sinusoid_pe(T, depth, dtype):
    """O.sinusoid_pe with its fp32 argument, sin / cos in `dtype` (== O.sinusoid_pe for float32)."""
    pos = torch.arange(1, T + 1)[None, :].type(torch.float32)
    inc = torch.log(torch.tensor([10000], dtype=torch.float32)) / (depth / 2 - 1)
    inv = torch.exp(torch.arange(depth / 2).type(torch.float32) * (-inc))
    st = (pos.reshape(1, -1, 1) * inv.reshape(1, 1, -1)).to(dtype)
    return torch.cat([torch.sin(st), torch.cos(st)], dim=2)


def encoder(x, lens, p, names, after_norm, heads, eps, embed=True, depths=None):
    """SANMEncoder.forward over the layers `names` (state-dict prefixes without the trailing dot) -> {depth: after_norm(x)} for every
    depth in `depths` (default: all layers).  embed: x * sqrt(D) + PE first (input_layer 'pe'); else a plain stack over x."""
    B, T, _ = x.shape
    lens = torch.as_tensor(lens)
    mask = (torch.arange(T)[None, :] < lens[:, None].long())[:, None, :]
    D = p[after_norm + ".weight"].numel()
    if embed:
        x = x * D ** 0.5
        x = x + sinusoid_pe(T, x.shape[-1], x.dtype)
    depths = set(depths or [len(names)])
    out = {}
    for i, pre in enumerate(names):
        x = O.encoder_layer(x, p, pre + ".", mask, heads, eps)
        if i + 1 in depths:
            out[i + 1] = O.layer_norm(x, p[after_norm + ".weight"], p[after_norm + ".bias"], eps)
    return out


def paraformer_encoder_names(n):
    return ["encoder." + ("encoders0.0" if i == 0 else "encoders.%d" % (i - 1)) for i in range(n)]


# ---------------------------------------------------------------------------------------------- predictor
def cif_fire(hidden, alphas, threshold=1.0):
    """Integrate-and-fire of one utterance in the inputs' dtype: hidden [T, D], alphas [T] (tail included) -> (frames [n, D], peaks
    [T] = the integral before a fire subtracts the threshold, fire frame indices, running integral [T])."""
    h = np.asarray(hidden, dtype=np.float64)
    a = np.asarray(alphas, dtype=np.float64)
    integ, frame = 0.0, np.zeros(h.shape[1])
    frames, peaks, fires = [], np.zeros(a.shape[0]), []
    for t in range(a.shape[0]):
        cur = integ + a[t]
        peaks[t] = cur
        if cur >= threshold:
            c = threshold - integ
            frames.append(frame + c * h[t])
            frame = (a[t] - c) * h[t]
            integ = cur - threshold
            fires.append(t)
        else:
            frame = frame + a[t] * h[t]
            integ = cur
    return (np.stack(frames) if frames else np.zeros((0, h.shape[1]))), peaks, fires, np.cumsum(a)


def predictor(enc, lens, p, tail_threshold, smooth=1.0, noise=0.0):
    """CifPredictorV2 / V3 forward on a [B, T, D] encoder output -> alphas [B, T + 1] (tail added), the alpha sum per utterance
    (token_num = floor of it), and per utterance (frames, peaks, fire frames, running integral) from cif_fire."""
    B, T, _ = enc.shape
    lens = torch.as_tensor(lens)
    mask = (torch.arange(T)[None, :] < lens[:, None].long())[:, None, :]
    al = O.cif_alphas(enc, mask, p, smooth, noise)
    hidden, al2, token_sum = O.cif_tail(enc, al, mask.squeeze(1).to(enc.dtype), tail_threshold)
    fires = [cif_fire(hidden[b].numpy(), al2[b].numpy()) for b in range(B)]
    return al2, al2.sum(-1), fires


# ------------------------------------------------------------------------------------------------ decoder
def decoder_hidden(enc, enc_lens, emb, tok_lens, p, n_layers, heads=4, eps=1e-12):
    """ParaformerSANMDecoder.forward with return_hidden -> (hidden [B, N, D], logits [B, N, V]); == O.decoder's logits."""
    h = O.sanm_decoder_hidden(emb, torch.as_tensor(tok_lens), enc, torch.as_tensor(enc_lens), p, "decoder.", n_layers, heads, eps)
    return h, F.linear(h, p["decoder.output_layer.weight"], p["decoder.output_layer.bias"])


def decision_ok(ids, ref_logits, bound):
    """Arg-max ids [R] against reference rows [R, V]: the reference's arg-max is required where its top-two gap exceeds 2 x bound
    (bound: the row's admitted absolute error), else either of its top two ids is accepted.  -> bool [R]."""
    r = np.asarray(ref_logits, dtype=np.float64)
    top2 = np.argsort(-r, axis=-1)[:, :2]
    gap = r[np.arange(r.shape[0]), top2[:, 0]] - r[np.arange(r.shape[0]), top2[:, 1]]
    ids = np.asarray(ids)
    clear = gap > 2 * np.asarray(bound)
    return np.where(clear, ids == top2[:, 0], (ids == top2[:, 0]) | (ids == top2[:, 1]))
