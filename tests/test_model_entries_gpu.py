"""GPU (-m gpu): the model-level entry points of csrc/model.cu — fa_sanm_encoder_forward, fa_cif_predictor_forward,
fa_paraformer_decoder_forward(_hidden) and fa_sanm_decoder_stack_forward — against the float64 restatement of the same modules
(tests/model_entries_ref.py), row by row, in every GEMM mode.

Metric: err_r = max_c |got - ref| / max(max_c |ref|, FLOOR) per row (model_entries_ref.row_err); every row is compared, valid and
padded.  Alphas, peaks, log-probabilities and attention probabilities are compared by their absolute difference.  Integer outputs
are exact where the float64 result is not within the bound of a decision (token counts: the alpha sum near an integer; arg-max: a
top-two gap under twice the row's bound).  Each split-mode case also reruns its inputs in single-plane fp16 and requires that
output to miss the fp16x3 bar by 10 x or more: a bar that a lost operand plane could pass is too loose.

BARS: at most 4 x the worst error measured over all cases of an entry and mode on an NVIDIA H100 80GB HBM3 (700 W power limit);
MEASURED holds those worst values.  Every case prints its worst row (utterance, row, valid or padded) with -s.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import state_dict_for

import model_entries_ref as R
import paraformer_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MODES = ["fp32", "fp16", "fp16x3", "fp16x6"]
SPLIT = ("fp16x3", "fp16x6")

# Measured worst per entry and mode over every case below, on an NVIDIA H100 80GB HBM3 at its 700 W power limit; each bar is at
# most 4 x its measured worst.  The split-mode bars sit at 2 x where 4 x would let single-plane fp16 come within 10 x of them.
# fp16x6 measures the same as fp16x3 at every entry: the GEMMs' third A plane (gemm_planes: 1 / 2 / 3 for fp16 / fp16x3 / fp16x6)
# sits far below what the attention leaves — its operands and probabilities are at most two fp16 planes in both modes (attn_planes)
# — and below the fp32 accumulation, so no entry-level bar can tell the two apart; the GEMM's own tests do (test_gemm_gpu.py).
MEASURED = {
    "encoder": {"paraformer": {"fp32": 9.26e-6, "fp16": 6.64e-3, "fp16x3": 2.50e-5, "fp16x6": 2.48e-5},
                "aligner": {"fp32": 7.48e-6, "fp16": 7.03e-3, "fp16x3": 2.16e-5, "fp16x6": 2.14e-5},
                "sensevoice_plain": {"fp32": 1.92e-6, "fp16": 1.61e-3, "fp16x3": 4.53e-6, "fp16x6": 4.90e-6},
                "ct_transformer": {"fp32": 9.35e-7},
                "paraformer_large": {"fp32": 6.47e-5, "fp16": 8.66e-2, "fp16x3": 2.05e-4, "fp16x6": 1.75e-4}},
    "alphas": {"fp32": 5.81e-7, "fp16": 1.69e-4, "fp16x3": 1.19e-6, "fp16x6": 1.25e-6},
    "acoustic": {"fp32": 1.10e-5, "fp16": None, "fp16x3": 8.72e-6, "fp16x6": 8.68e-6},
    "peaks": {"fp32": 3.79e-6, "fp16": 7.04e-5, "fp16x3": 9.07e-6, "fp16x6": 9.55e-6},
    "dec_hidden": {"fp32": 3.33e-6, "fp16": 1.21e-3, "fp16x3": 1.09e-5, "fp16x6": 1.12e-5},
    "dec_logits": {"fp32": 2.50e-6, "fp16": 1.30e-3, "fp16x3": 1.11e-5, "fp16x6": 1.17e-5},
    "dec_logp": {"fp32": 2.73e-5, "fp16": 1.33e-2, "fp16x3": 1.09e-4, "fp16x6": 1.13e-4},
    "stack_hidden": {"fp32": 2.22e-6, "fp16": 1.27e-3, "fp16x3": 8.26e-6, "fp16x6": 8.33e-6},
    "stack_probs": {300: {"fp32": 6.56e-7, "fp16": 2.76e-4, "fp16x3": 2.31e-6, "fp16x6": 2.31e-6},
                    3073: {"fp32": 1.18e-7, "fp16": 5.60e-5, "fp16x3": 4.63e-7, "fp16x6": 4.62e-7},
                    6144: {"fp32": 3.49e-8, "fp16": 1.03e-5, "fp16x3": 9.44e-8, "fp16x6": 9.35e-8}},
}
BARS = {
    "encoder": {"paraformer": {"fp32": 3.7e-5, "fp16": 2.6e-2, "fp16x3": 5.0e-5, "fp16x6": 5.0e-5},      # rows after after_norm
                "aligner": {"fp32": 2.9e-5, "fp16": 2.8e-2, "fp16x3": 4.5e-5, "fp16x6": 4.5e-5},
                "sensevoice_plain": {"fp32": 7.6e-6, "fp16": 6.4e-3, "fp16x3": 1.8e-5, "fp16x6": 1.9e-5},
                "ct_transformer": {"fp32": 3.7e-6},
                # 50 layers: the error grows with depth (fp16x3: 2.5e-5 after 3 layers, 2.0e-4 after 50), so the full-depth
                # case has bars of its own
                "paraformer_large": {"fp32": 2.5e-4, "fp16": 3.4e-1, "fp16x3": 8.1e-4, "fp16x6": 7.0e-4}},
    "alphas": {"fp32": 2.3e-6, "fp16": 6.7e-4, "fp16x3": 2.5e-6, "fp16x6": 2.5e-6},                       # |d alpha|
    # token rows of the utterances whose fire decisions all lie outside the alpha bound; fp16: none of those carries a token
    "acoustic": {"fp32": 4.4e-5, "fp16": None, "fp16x3": 3.4e-5, "fp16x6": 3.4e-5},
    "peaks": {"fp32": 1.5e-5, "fp16": 2.8e-4, "fp16x3": 3.6e-5, "fp16x6": 3.8e-5},                        # |d peak|, same utterances
    "dec_hidden": {"fp32": 1.3e-5, "fp16": 4.8e-3, "fp16x3": 4.4e-5, "fp16x6": 4.4e-5},                   # after_norm rows
    "dec_logits": {"fp32": 1.0e-5, "fp16": 5.2e-3, "fp16x3": 4.4e-5, "fp16x6": 4.6e-5},                   # logit rows
    "dec_logp": {"fp32": 1.0e-4, "fp16": 5.3e-2, "fp16x3": 4.3e-4, "fp16x6": 4.5e-4},                     # |d log-prob|
    "stack_hidden": {"fp32": 8.8e-6, "fp16": 5.0e-3, "fp16x3": 3.3e-5, "fp16x6": 3.3e-5},                 # hidden rows
    "stack_probs": {300: {"fp32": 2.6e-6, "fp16": 1.1e-3, "fp16x3": 9.2e-6, "fp16x6": 9.2e-6},            # |d probability|
                    3073: {"fp32": 4.7e-7, "fp16": 2.2e-4, "fp16x3": 1.8e-6, "fp16x6": 1.8e-6},
                    6144: {"fp32": 1.3e-7, "fp16": 4.1e-5, "fp16x3": 3.7e-7, "fp16x6": 3.7e-7}},
}


def _abi():
    from funasr_b200 import _abi as A
    return A, A.load()


def _report(entry, mode, case, err, w=None):
    print("MEASURED %s %s %s %.3e%s" % (entry, mode, case, err, "" if w is None else "  " + R.describe("worst", w)))


def _teeth(entry, case, fp16_err, bar):
    """A split-mode case's inputs in single-plane fp16 must miss the fp16x3 bar by >= 10 x."""
    print("TEETH %s %s fp16 %.3e = %.1f x the fp16x3 bar %.1e" % (entry, case, fp16_err, fp16_err / bar, bar))
    assert fp16_err >= 10 * bar, "fp16 passes within 10 x of the fp16x3 bar: the bar cannot see a lost plane"


# ------------------------------------------------------------------------------------------------ engines and weights
_STATE, _ENG = {}, {}


def _state(kind):
    if kind not in _STATE:
        from funasr_b200 import synth
        T = synth.PARAFORMER_TINY
        _STATE[kind] = {
            "para": lambda: state_dict_for(T, 3),
            "ctx": lambda: synth.make_contextual_state_dict(T, 6),
            "seaco": lambda: synth.make_seaco_state_dict(T, 10),
            "sv": lambda: synth.make_sensevoice_state_dict(synth.SENSEVOICE_TINY, 4),
            "aligner": lambda: synth.make_aligner_state_dict(synth.ALIGNER_TINY, 5),
            "punc": lambda: synth.make_punc_state_dict(0),
            "large": lambda: state_dict_for(synth.PARAFORMER_LARGE, 0),
        }[kind]()
    return _STATE[kind]


def _state64(kind):
    key = kind + "64"
    if key not in _STATE:
        st = _state(kind)
        if kind == "large":                         # the full-depth case needs only the encoder in float64
            st = {k: v for k, v in st.items() if k.startswith("encoder.")}
        _STATE[key] = R.to64(st)
    return _STATE[key]


def _engine(kind, mode):
    key = (kind, mode)
    if key not in _ENG:
        from funasr_b200 import synth
        from funasr_b200.engine import AlignerEngine, ParaformerEngine, SenseVoiceEngine
        from funasr_b200.punc import PuncEngine
        T = synth.PARAFORMER_TINY
        if kind == "para":
            e = ParaformerEngine(_state(kind), T, DEV, gemm_mode=mode)
        elif kind == "large":
            e = ParaformerEngine(_state(kind), synth.PARAFORMER_LARGE, DEV, gemm_mode=mode)
        elif kind == "ctx":
            e = ParaformerEngine(_state(kind), T, DEV, gemm_mode=mode, contextual=True)
        elif kind == "seaco":
            e = ParaformerEngine(_state(kind), T, DEV, gemm_mode=mode, seaco=True, no_bias=synth.seaco_no_bias_id(T))
        elif kind == "sv":
            e = SenseVoiceEngine(_state(kind), synth.SENSEVOICE_TINY, DEV, gemm_mode=mode)
        elif kind == "aligner":
            e = AlignerEngine(_state(kind), synth.ALIGNER_TINY, DEV, gemm_mode=mode)
        else:
            e = PuncEngine(_state(kind), DEV, heads=8)
            e.mode = _abi()[0].GEMM_MODES[mode]       # fp32 packing; a tensor-core mode is refused on the head size alone
        _ENG[key] = e
    return _ENG[key]


def _st(stream=None):
    return (stream or torch.cuda.current_stream()).cuda_stream


# ------------------------------------------------------------------------------------------------ encoder
# name: (engine kind, struct attribute, layer names, after_norm, heads, eps, embedded input, input width, depths)
ENC_CFGS = {
    "paraformer": ("para", "enc", R.paraformer_encoder_names(3), "encoder.after_norm", 4, 1e-12, True, 560, (1, 2, 3)),
    "sensevoice_plain": ("sv", "tp", ["encoder.tp_encoders.0", "encoder.tp_encoders.1"], "encoder.tp_norm", 4, 1e-5, False, 512, (1, 2)),
    "aligner": ("aligner", "enc", R.paraformer_encoder_names(3), "encoder.after_norm", 4, 1e-12, True, 560, (1, 2, 3)),
    "ct_transformer": ("punc", "enc", ["encoder.encoders0.0"] + ["encoder.encoders.%d" % i for i in range(3)], "encoder.after_norm", 8,
                       1e-12, True, 256, (1, 4)),
    "paraformer_large": ("large", "enc", R.paraformer_encoder_names(50), "encoder.after_norm", 4, 1e-12, True, 560, (50,)),
}
FULL_DEPTH_LENS = [300, 217]
T_LIST = [1, 2, 63, 64, 65, 127, 128, 129, 500]


def _lens_for(T):
    out = []
    for n in (T, T - 1, 1, 0, (T + 1) // 2, max(T - 2, 0)):
        if n >= 0 and n not in out:
            out.append(n)
    return out[:6]


_ENC_REF = {}


def _enc_inputs(cfg, T, lens=None, seed=0):
    kind, _, _, _, _, _, embed, din, _ = ENC_CFGS[cfg]
    if lens is None:
        lens = FULL_DEPTH_LENS if cfg == "paraformer_large" else _lens_for(T)
    g = torch.Generator().manual_seed(1000 * T + seed)
    x = torch.randn(len(lens), T, din, generator=g)
    if embed:                                      # the reference pads features with zeros before embedding them
        x = x * torch.from_numpy(R.len_mask(lens, T)).float()[:, :, None]
    return x, torch.tensor(lens, dtype=torch.int32)


def _enc_ref(cfg, T):
    if (cfg, T) not in _ENC_REF:
        kind, _, names, after, heads, eps, embed, _, depths = ENC_CFGS[cfg]
        x, lens = _enc_inputs(cfg, T)
        out = R.encoder(x.double(), lens, _state64(kind), names, after, heads, eps, embed, depths)
        _ENC_REF[(cfg, T)] = {d: v.numpy() for d, v in out.items()}
    return _ENC_REF[(cfg, T)]


def _enc_struct(eng, attr, n_layers, layers=None):
    A, _ = _abi()
    e = getattr(eng, attr)
    return A.FaEncoder(e.layers if layers is None else layers, n_layers, e.heads, e.fsmn_k, 0, e.after_norm, e.pe_inv_timescales)


def _run_encoder(eng, enc, x, lens, stream=None):
    A, lib = _abi()
    B, T, _ = x.shape
    out = torch.full((B, T, enc.after_norm.n), float("nan"), device=DEV)
    ws = torch.empty(lib.fa_sanm_encoder_workspace_bytes(B, T, eng.mode), dtype=torch.uint8, device=DEV)
    xd, ld = x.to(DEV), lens.to(DEV)
    torch.cuda.synchronize()
    rc = lib.fa_sanm_encoder_forward(C.byref(enc), xd.data_ptr(), ld.data_ptr(), B, T, out.data_ptr(), eng.mode, ws.data_ptr(), ws.numel(),
                                     _st(stream))
    torch.cuda.synchronize()
    return rc, out


def _encoder_err(cfg, T, mode):
    kind, attr, _, _, _, _, _, _, depths = ENC_CFGS[cfg]
    eng = _engine(kind, mode)
    x, lens = _enc_inputs(cfg, T)
    ref = _enc_ref(cfg, T)
    valid = R.len_mask(lens.tolist(), T)
    worst = (0.0, (), True)
    for d in depths:
        rc, out = _run_encoder(eng, _enc_struct(eng, attr, d), x, lens)
        assert rc == 0
        w = R.worst(R.row_err(out.cpu().numpy(), ref[d]), valid)
        if w[0] >= worst[0]:
            worst = w + (d,)
    return worst


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("T", T_LIST)
@pytest.mark.parametrize("cfg", ["paraformer", "sensevoice_plain", "aligner", "ct_transformer"])
def test_encoder_rows_vs_float64(cfg, T, mode):
    """Every row of `out`, valid and padded, after 1 ... n layers; t_max straddles the attention query tiles and the FSMN's 64-row
    tile; lens include 0, 1, t_max - 1 and t_max.  CT-Transformer (d 256, 8 x 32 heads, first layer 256 -> 256 keeps the embedded
    rows as its residual) runs on the fp32 path only; the tensor-core modes refuse it."""
    A, lib = _abi()
    if cfg == "ct_transformer" and mode != "fp32":
        eng = _engine("punc", mode)
        x, lens = _enc_inputs(cfg, T)
        n0 = lib.fa_launch_count()
        rc, _ = _run_encoder(eng, _enc_struct(eng, "enc", 4), x, lens)
        assert rc == -4 and lib.fa_launch_count() == n0
        return
    w = _encoder_err(cfg, T, mode)
    _report("encoder", mode, "%s/T%d/depth%d" % (cfg, T, w[3]), w[0], w[:3])
    bars = BARS["encoder"][cfg]
    assert w[0] <= bars[mode], R.describe("encoder", w[:3])
    if mode in SPLIT:
        _teeth("encoder", "%s/T%d" % (cfg, T), _encoder_err(cfg, T, "fp16")[0], bars["fp16x3"])


@pytest.mark.parametrize("mode", MODES)
def test_encoder_full_depth_vs_float64(mode):
    """Paraformer-large's 50-layer encoder at B = 2, t_max 300 (lens 300 and 217): every row against float64, with bars of its own
    measured at this depth, so the per-mode error is shown to stay bounded over the production stack's depth."""
    w = _encoder_err("paraformer_large", 300, mode)
    _report("encoder", mode, "paraformer_large/T300/depth50", w[0], w[:3])
    bars = BARS["encoder"]["paraformer_large"]
    assert w[0] <= bars[mode], R.describe("encoder", w[:3])
    if mode in SPLIT:
        _teeth("encoder", "paraformer_large/T300", _encoder_err("paraformer_large", 300, "fp16")[0], bars["fp16x3"])


# ------------------------------------------------------------------------------------------------ predictor
def _pred_inputs(T, lens, seed=1):
    g = torch.Generator().manual_seed(7 * T + seed)
    return torch.randn(len(lens), T, 512, generator=g), torch.tensor(lens, dtype=torch.int32)   # padded rows: encoder output, not zero


def _run_predictor(eng, variant, enc, lens, stream=None):
    A, lib = _abi()
    pred = A.FaPredictor.from_buffer_copy(eng.pred)
    pred.cif_variant = variant
    B, T, D = enc.shape
    n_cap = T + 1
    acoustic = torch.full((B, n_cap, D), float("nan"), device=DEV)
    tok = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    alphas, peaks = torch.full((B, T + 1), float("nan"), device=DEV), torch.full((B, T + 1), float("nan"), device=DEV)
    ws = torch.empty(lib.fa_cif_predictor_workspace_bytes(B, T, eng.mode), dtype=torch.uint8, device=DEV)
    ed, ld = enc.to(DEV), lens.to(DEV)
    torch.cuda.synchronize()
    rc = lib.fa_cif_predictor_forward(C.byref(pred), ed.data_ptr(), ld.data_ptr(), B, T, acoustic.data_ptr(), n_cap, tok.data_ptr(),
                                      alphas.data_ptr(), peaks.data_ptr(), eng.mode, ws.data_ptr(), ws.numel(), _st(stream))
    torch.cuda.synchronize()
    assert rc == 0
    return acoustic.cpu().numpy(), tok.cpu().numpy(), alphas.cpu().numpy(), peaks.cpu().numpy()


_PRED_REF = {}


def _pred_ref(T, lens):
    key = (T, tuple(lens))
    if key not in _PRED_REF:
        enc, ln = _pred_inputs(T, lens)
        al, asum, fires = R.predictor(enc.double(), ln, _state64("para"), 0.45)
        _PRED_REF[key] = (al.numpy(), asum.numpy(), fires)
    return _PRED_REF[key]


def _acoustic_err(acoustic, tok, fires, utts):
    """Worst token-row error of the utterances `utts` (rows below both the kernel's and the float64 token count)."""
    worst = 0.0
    for b in utts:
        frames = fires[b][0]
        k = min(int(tok[b]), frames.shape[0])
        if k:
            worst = max(worst, float(R.row_err(acoustic[b, :k], frames[:k]).max()))
    return worst


def _check_predictor(T, lens, mode, variant):
    """-> (worst |d alpha|, the utterances whose acoustic rows and peaks were compared); asserts alphas, token_num, acoustic rows and
    peaks."""
    enc, ln = _pred_inputs(T, lens)
    acoustic, tok, alphas, peaks = _run_predictor(_engine("para", mode), variant, enc, ln)
    al, asum, fires = _pred_ref(T, lens)
    d_al = np.abs(alphas - al)
    w = R.worst(d_al, R.len_mask([n + 1 for n in lens], T + 1))
    bar = BARS["alphas"][mode]
    assert w[0] <= bar, R.describe("alphas", w)
    compared, pk_worst = [], 0.0
    for b, (frames, pk, fire_at, integ) in enumerate(fires):
        drift = bar * np.arange(1, T + 2)                     # the running integral's admitted error after t + 1 frames
        near = np.abs(integ - np.round(integ)) <= drift
        if abs(asum[b] - np.round(asum[b])) > drift[-1]:
            assert tok[b] == int(np.floor(asum[b])), (b, tok[b], asum[b])
        if near.any():                                        # a fire decision within the bound: the frames may legitimately move
            print("predictor %s T%d utt %d: a fire decision within the bound, acoustic / peaks not compared" % (mode, T, b))
            continue
        compared.append(b)
        pk_worst = max(pk_worst, float(np.abs(peaks[b] - pk).max()))
    ac_worst = _acoustic_err(acoustic, tok, fires, compared)
    _report("acoustic", mode, "T%d/v%d" % (T, variant), ac_worst)
    _report("peaks", mode, "T%d/v%d (%d of %d utterances compared)" % (T, variant, len(compared), len(lens)), pk_worst)
    assert compared, "every utterance has a fire decision within the bound: nothing compared"
    assert pk_worst <= BARS["peaks"][mode], pk_worst
    if BARS["acoustic"][mode] is not None:
        assert ac_worst <= BARS["acoustic"][mode], ac_worst
    return w, compared


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("T", [1, 2, 64, 65, 129, 300])
def test_predictor_vs_float64(T, variant, mode):
    """Alphas per frame (the frame len - 1 reads the first padded encoder row through the conv window), token_num by the decision
    rule, acoustic per token row and peaks; cif_variant 0 (CifPredictorV2) and 1 (CifPredictorV3's sequential cif)."""
    lens = [n for n in dict.fromkeys([T, max(T - 1, 1), 1, T // 2 + 1])]
    w, compared = _check_predictor(T, lens, mode, variant)
    _report("alphas", mode, "T%d/v%d" % (T, variant), w[0], w)
    if mode in SPLIT and T > 1:     # t_max 1: one alpha per utterance, too few for fp16's error to show (8.8e-6, 3.5 x the bar)
        enc, ln = _pred_inputs(T, lens)
        ac16, tok16, a16, _ = _run_predictor(_engine("para", "fp16"), variant, enc, ln)
        al, _, fires = _pred_ref(T, lens)
        _teeth("predictor", "T%d/v%d" % (T, variant), float(np.abs(a16 - al).max()), BARS["alphas"]["fp16x3"])
        if any(min(int(tok16[b]), fires[b][0].shape[0]) for b in compared):      # utterances with tokens (t_max >= 64)
            _teeth("acoustic", "T%d/v%d" % (T, variant), _acoustic_err(ac16, tok16, fires, compared), BARS["acoustic"]["fp16x3"])


@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_predictor_last_frame_reads_the_padded_row(mode):
    """One utterance of 40 frames run with t_max 40 (the conv's right neighbour of frame 39 is the conv's zero padding) and t_max 45
    (it is the encoder's padded row 40): the reference's alpha at frame 39 differs between the two, and the kernel follows each."""
    enc, _ = _pred_inputs(45, [40])
    p = _state64("para")
    got, ref = {}, {}
    for T in (40, 45):
        e = enc[:, :T].contiguous()
        ln = torch.tensor([40], dtype=torch.int32)
        ref[T] = R.predictor(e.double(), ln, p, 0.45)[0].numpy()[0]
        got[T] = _run_predictor(_engine("para", mode), 0, e, ln)[2][0]
        assert np.abs(got[T][:41] - ref[T][:41]).max() <= BARS["alphas"][mode]
    assert abs(ref[40][39] - ref[45][39]) > 100 * BARS["alphas"][mode]          # the padded row matters to the reference
    assert np.abs(ref[40][:39] - ref[45][:39]).max() <= 1e-12
    assert abs(got[40][39] - got[45][39]) > 50 * BARS["alphas"][mode]


# ------------------------------------------------------------------------------------------------ decoder
def _dec_inputs(n_max, B=4, Tm=80, seed=2):
    g = torch.Generator().manual_seed(11 * n_max + seed)
    enc = torch.randn(B, Tm, 512, generator=g)
    enc_lens = torch.tensor([Tm, 1, 47, Tm][:B], dtype=torch.int32)
    ld_rows = n_max + 3                                        # the acoustic rows' pitch exceeds n_max
    acoustic = torch.randn(B, ld_rows, 512, generator=g)
    tok = torch.tensor([n_max, 0, min(n_max, 5), n_max // 2 + 1][:B], dtype=torch.int32)
    return enc, enc_lens, acoustic, tok


def _run_decoder(eng, dec, enc, enc_lens, acoustic, tok, n_max, log_softmax, want_hidden, n_hw=0, stream=None):
    A, lib = _abi()
    B, Tm, _ = enc.shape
    V = dec.vocab
    ids = torch.full((B, n_max), -7, dtype=torch.int32, device=DEV)
    best = torch.full((B, n_max), float("nan"), device=DEV)
    logits = torch.full((B, n_max, V), float("nan"), device=DEV)
    hidden = torch.full((B, n_max, 512), float("nan"), device=DEV) if want_hidden else None
    ws = torch.empty(lib.fa_paraformer_decoder_workspace_bytes_hw(B, Tm, n_max, V, eng.mode, n_hw), dtype=torch.uint8, device=DEV)
    ed, eld, ad, td = enc.to(DEV), enc_lens.to(DEV), acoustic.to(DEV), tok.to(DEV)
    torch.cuda.synchronize()
    args = (C.byref(dec), ed.data_ptr(), eld.data_ptr(), B, Tm, ad.data_ptr(), acoustic.shape[1], td.data_ptr(), n_max, ids.data_ptr(),
            best.data_ptr(), logits.data_ptr(), log_softmax)
    if want_hidden:
        rc = lib.fa_paraformer_decoder_forward_hidden(*args, hidden.data_ptr(), eng.mode, ws.data_ptr(), ws.numel(), _st(stream))
    else:
        rc = lib.fa_paraformer_decoder_forward(*args, eng.mode, ws.data_ptr(), ws.numel(), _st(stream))
    torch.cuda.synchronize()
    return rc, ids.cpu().numpy(), logits.cpu().numpy(), None if hidden is None else hidden.cpu().numpy()


_DEC_REF = {}


def _dec_ref(n_max):
    if n_max not in _DEC_REF:
        enc, enc_lens, acoustic, tok = _dec_inputs(n_max)
        h, lg = R.decoder_hidden(enc.double(), enc_lens, acoustic[:, :n_max].double(), tok, _state64("para"), 2)
        _DEC_REF[n_max] = (h.numpy(), lg.numpy(), torch.log_softmax(lg, -1).numpy())
    return _DEC_REF[n_max]


def _check_ids(ids, ref_logits, bar):
    r = ref_logits.reshape(-1, ref_logits.shape[-1])
    bound = bar * np.maximum(np.abs(r).max(-1), R.FLOOR)
    ok = R.decision_ok(ids.reshape(-1), r, bound)
    assert ok.all(), np.nonzero(~ok)[0][:5]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n_max", [1, 63, 64, 65, 130])
def test_decoder_vs_float64(n_max, mode):
    """_hidden with raw logits (log_softmax 0) and _forward with log-probabilities: hidden and logit rows, |d log-prob|, arg-max ids by
    the tie rule.  tok_lens hold 0 and n_max, enc_lens hold 1, the acoustic pitch exceeds n_max; n_max picks the FSMN kernel."""
    eng = _engine("para", mode)
    enc, enc_lens, acoustic, tok = _dec_inputs(n_max)
    h_ref, lg_ref, lp_ref = _dec_ref(n_max)
    rc, ids, logits, hidden = _run_decoder(eng, eng.dec, enc, enc_lens, acoustic, tok, n_max, 0, True)
    assert rc == 0
    wh = R.worst(R.row_err(hidden, h_ref), R.len_mask(tok.tolist(), n_max))
    wl = R.worst(R.row_err(logits, lg_ref), R.len_mask(tok.tolist(), n_max))
    _report("dec_hidden", mode, "n%d" % n_max, wh[0], wh)
    _report("dec_logits", mode, "n%d" % n_max, wl[0], wl)
    assert wh[0] <= BARS["dec_hidden"][mode] and wl[0] <= BARS["dec_logits"][mode]
    _check_ids(ids, lg_ref, BARS["dec_logits"][mode])
    rc, ids2, logp, _ = _run_decoder(eng, eng.dec, enc, enc_lens, acoustic, tok, n_max, 1, False)
    assert rc == 0 and (ids2 == ids).all()
    dlp = float(np.abs(logp - lp_ref).max())
    _report("dec_logp", mode, "n%d" % n_max, dlp)
    assert dlp <= BARS["dec_logp"][mode]
    if mode in SPLIT:
        e16 = _engine("para", "fp16")
        _, _, _, h16 = _run_decoder(e16, e16.dec, enc, enc_lens, acoustic, tok, n_max, 0, True)
        _teeth("decoder", "n%d" % n_max, float(R.row_err(h16, h_ref).max()), BARS["dec_hidden"]["fp16x3"])
        _, _, lp16, _ = _run_decoder(e16, e16.dec, enc, enc_lens, acoustic, tok, n_max, 1, False)
        _teeth("dec_logp", "n%d" % n_max, float(np.abs(lp16 - lp_ref).max()), BARS["dec_logp"]["fp16x3"])


_CTX_REF = {}


def _hotwords(nh):
    g = torch.Generator().manual_seed(5 + nh)
    return torch.tanh(torch.randn(nh, 512, generator=g))


def _ctx_dec(eng, hw, B):
    A, _ = _abi()
    dec = A.FaDecoder.from_buffer_copy(eng.dec)
    hwd = hw.to(DEV).contiguous()
    hl = torch.full((B,), hw.shape[0], dtype=torch.int32, device=DEV)
    dec.has_bias, dec.n_hotwords, dec.hw_embed, dec.hw_lens = 1, hw.shape[0], hwd.data_ptr(), hl.data_ptr()
    return dec, (hwd, hl)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n_hw", [1, 5, 300])
def test_contextual_decoder_vs_float64(n_hw, mode):
    """The contextual bias branch ([x_src_attn ; cx] over shared hotword rows) against contextual_decoder."""
    n_max = 65
    eng = _engine("ctx", mode)
    enc, enc_lens, acoustic, tok = _dec_inputs(n_max, seed=3)
    hw = _hotwords(n_hw)
    if n_hw not in _CTX_REF:
        _CTX_REF[n_hw] = O.contextual_decoder(enc.double(), enc_lens, acoustic[:, :n_max].double(), tok, hw.double(), _state64("ctx"),
                                              2).numpy()
    ref = _CTX_REF[n_hw]
    dec, keep = _ctx_dec(eng, hw, enc.shape[0])
    rc, ids, logits, _ = _run_decoder(eng, dec, enc, enc_lens, acoustic, tok, n_max, 0, False, n_hw)
    assert rc == 0
    w = R.worst(R.row_err(logits, ref), R.len_mask(tok.tolist(), n_max))
    _report("dec_logits", mode, "ctx/hw%d" % n_hw, w[0], w)
    assert w[0] <= BARS["dec_logits"][mode]
    _check_ids(ids, ref, BARS["dec_logits"][mode])
    if mode in SPLIT:
        e16 = _engine("ctx", "fp16")
        d16, keep16 = _ctx_dec(e16, hw, enc.shape[0])
        _, _, l16, _ = _run_decoder(e16, d16, enc, enc_lens, acoustic, tok, n_max, 0, False, n_hw)
        _teeth("contextual", "hw%d" % n_hw, float(R.row_err(l16, ref).max()), BARS["dec_logits"]["fp16x3"])


# ------------------------------------------------------------------------------------------------ decoder stack (SeACo)
def _run_stack(eng, memory, mem_lens, mem_shared, B, t_mem, x, tok, n_max, n_run, finish, probs=False, dec=None):
    A, lib = _abi()
    dec = eng.seaco_dec if dec is None else dec
    hidden = None if probs else torch.full((B, n_max, 512), float("nan"), device=DEV)
    ap = torch.full((dec.heads, n_max, t_mem), float("nan"), device=DEV) if probs else None
    ws = torch.empty(lib.fa_sanm_decoder_stack_workspace_bytes(B, t_mem, n_max, eng.mode), dtype=torch.uint8, device=DEV)
    md, mld, xd, td = memory.to(DEV), mem_lens.to(DEV), x.to(DEV), tok.to(DEV)
    torch.cuda.synchronize()
    rc = lib.fa_sanm_decoder_stack_forward(C.byref(dec), md.data_ptr(), mld.data_ptr(), mem_shared, B, t_mem, xd.data_ptr(), x.shape[1],
                                           td.data_ptr(), n_max, n_run, finish, None if hidden is None else hidden.data_ptr(),
                                           None if ap is None else ap.data_ptr(), eng.mode, ws.data_ptr(), ws.numel(), _st())
    torch.cuda.synchronize()
    return rc, (ap if probs else hidden).cpu().numpy()


# name: (mem_shared, t_mem, n_run (None: all layers), finish)
STACK_CASES = {
    "finish1_shared_t6": (1, 6, None, 1),
    "finish1_shared_t1": (1, 1, None, 1),
    "finish1_per_utt_t300": (0, 300, None, 1),
    "finish0_run2_per_utt_t300": (0, 300, 2, 0),
    "finish0_run3_shared_t6": (1, 6, 3, 0),
    "run0_finish1_t6": (1, 6, 0, 1),
    "run0_finish0_t6": (1, 6, 0, 0),
}
_STACK_REF = {}


def _stack_inputs(mem_shared, t_mem, B=3, n_max=7, seed=4):
    g = torch.Generator().manual_seed(13 * t_mem + seed + mem_shared)
    memory = torch.tanh(torch.randn(1 if mem_shared else B, t_mem, 512, generator=g))
    mem_lens = torch.tensor([t_mem] * B if mem_shared else [t_mem, 1, (t_mem + 1) // 2][:B], dtype=torch.int32)
    x = torch.randn(B, n_max + 2, 512, generator=g)
    tok = torch.tensor([n_max, 3, 0][:B], dtype=torch.int32)
    return memory, mem_lens, x, tok


def _stack_run_case(name, mode):
    mem_shared, t_mem, n_run, finish = STACK_CASES[name]
    eng = _engine("seaco", mode)
    L = eng.seaco_dec.n_layers
    n_run = L if n_run is None else n_run
    memory, mem_lens, x, tok = _stack_inputs(mem_shared, t_mem)
    B, n_max = x.shape[0], x.shape[1] - 2
    rc, hidden = _run_stack(eng, memory.reshape(-1, 512), mem_lens, mem_shared, B, t_mem, x, tok, n_max, n_run, finish)
    assert rc == 0
    if name not in _STACK_REF:
        p = _state64("seaco")
        mem = memory.double().expand(B, -1, -1) if mem_shared else memory.double()
        x64 = x[:, :n_max].double()
        if finish:
            ref = O.sanm_decoder_hidden(x64, tok, mem, mem_lens, p, "seaco_decoder.", n_run)
        else:
            ref = O.sanm_decoder_layers(x64, tok, mem, mem_lens, p, "seaco_decoder.", range(n_run))
        _STACK_REF[name] = ref.numpy()
    return hidden, _STACK_REF[name], tok, n_run, finish, x


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(STACK_CASES))
def test_decoder_stack_vs_float64(name, mode):
    """SeACo decoder stack (FFN 1024, FSMN k = 21): finish 1 / 0 with n_run below the layer count, n_run 0, a shared and a
    per-utterance memory of 1, 6 and 300 rows."""
    hidden, ref, tok, n_run, finish, x = _stack_run_case(name, mode)
    n_max = hidden.shape[1]
    if n_run == 0 and not finish:                                 # the stack's input, copied
        assert np.array_equal(hidden, x[:, :n_max].numpy())
        return
    w = R.worst(R.row_err(hidden, ref), R.len_mask(tok.tolist(), n_max))
    _report("stack_hidden", mode, name, w[0], w)
    assert w[0] <= BARS["stack_hidden"][mode]
    if mode in SPLIT:
        h16 = _stack_run_case(name, "fp16")[0]
        _teeth("stack", name, float(R.row_err(h16, ref).max()), BARS["stack_hidden"]["fp16x3"])


_PROBS_REF = {}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("t_mem,key_len,n_runs", [(300, 250, None), (3073, 3000, (1, 6)), (6144, 6144, (1,))])
def test_decoder_stack_attn_probs_vs_float64(t_mem, key_len, n_runs, mode):
    """attn_probs for n_run 1 ... n_layers (utterance 0's cross-attention probabilities of layer n_run - 1): against float64, each row
    sums to 1, columns at or beyond mem_lens[0] are exactly 0.  Above 3 072 memory rows the kernel's scores need the
    large-shared-memory opt-in (4 warps x t_mem fp32 > 48 KB); 6 144 rows fill the 96 KB it allows (more are refused)."""
    eng = _engine("seaco", mode)
    L = eng.seaco_dec.n_layers
    B, n_max = 2, 5
    g = torch.Generator().manual_seed(t_mem)
    memory = torch.tanh(torch.randn(t_mem, 512, generator=g))
    mem_lens = torch.tensor([key_len, t_mem], dtype=torch.int32)
    x = torch.randn(B, n_max, 512, generator=g)
    tok = torch.tensor([n_max, 2], dtype=torch.int32)
    worst, worst16 = 0.0, 0.0
    for n_run in (n_runs or range(1, L + 1)):
        rc, probs = _run_stack(eng, memory, mem_lens, 1, B, t_mem, x, tok, n_max, n_run, 0, probs=True)
        assert rc == 0
        if mode in SPLIT:
            p16 = _run_stack(_engine("seaco", "fp16"), memory, mem_lens, 1, B, t_mem, x, tok, n_max, n_run, 0, probs=True)[1]
        key = (t_mem, n_run)
        if key not in _PROBS_REF:
            mem = memory.double()[None].expand(B, -1, -1)
            _PROBS_REF[key] = O.sanm_decoder_layers(x.double(), tok, mem, mem_lens, _state64("seaco"), "seaco_decoder.", range(n_run),
                                                    attn_of=n_run - 1)[0].numpy()
        ref = _PROBS_REF[key]
        assert (probs[:, :, key_len:] == 0).all()
        assert np.abs(probs.sum(-1) - 1.0).max() <= 1e-5
        worst = max(worst, float(np.abs(probs - ref).max()))
        if mode in SPLIT:
            worst16 = max(worst16, float(np.abs(p16 - ref).max()))
    _report("stack_probs", mode, "t%d" % t_mem, worst)
    bars = BARS["stack_probs"][t_mem]                # probabilities shrink as 1 / t_mem, and so does their error
    assert worst <= bars[mode]
    if mode in SPLIT:
        _teeth("stack_probs", "t%d" % t_mem, worst16, bars["fp16x3"])


# ------------------------------------------------------------------------------------------------ refusals enqueue nothing
def _copy_layers(src, n, cls):
    arr = (cls * n)()
    for i in range(n):
        arr[i] = cls.from_buffer_copy(src[i])
    return arr


@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_refusals_launch_nothing(mode):
    """A malformed LAST layer is refused before the first launch (fa_launch_count unchanged), in the encoder, the decoder and the
    decoder stack; so is an attention probability matrix wider than the kernel's shared memory."""
    A, lib = _abi()
    eng = _engine("para", mode)
    x, lens = _enc_inputs("paraformer", 64)
    layers = _copy_layers(eng.enc.layers, 3, A.FaEncLayer)
    layers[2].w2.in_f += 1                                          # FA_ERR_ARG
    n0 = lib.fa_launch_count()
    rc, _ = _run_encoder(eng, _enc_struct(eng, "enc", 3, layers), x, lens)
    assert rc == -1 and lib.fa_launch_count() == n0
    layers = _copy_layers(eng.enc.layers, 3, A.FaEncLayer)
    layers[2].w1.out_f = layers[2].w2.in_f = 4096                   # FFN wider than the workspace carve: FA_ERR_UNSUPPORTED
    rc, _ = _run_encoder(eng, _enc_struct(eng, "enc", 3, layers), x, lens)
    assert rc == -4 and lib.fa_launch_count() == n0
    if mode != "fp32":
        layers = _copy_layers(eng.enc.layers, 3, A.FaEncLayer)
        layers[2].w2.in_pad += 64                                   # the planes' K pad must equal w1's width on the tensor-core path
        rc, _ = _run_encoder(eng, _enc_struct(eng, "enc", 3, layers), x, lens)
        assert rc == -4 and lib.fa_launch_count() == n0
    # decoder: the last attention layer, then decoders3
    enc, enc_lens, acoustic, tok = _dec_inputs(64)
    for which in ("layer", "last"):
        dec = A.FaDecoder.from_buffer_copy(eng.dec)
        dl = _copy_layers(eng.dec.layers, eng.dec.n_layers, A.FaDecLayer)
        dec.layers = dl
        if which == "layer":
            dl[eng.dec.n_layers - 1].ffn_norm.n += 1
        else:
            dec.last.ffn_w2.in_f += 1
        rc, _, _, _ = _run_decoder(eng, dec, enc, enc_lens, acoustic, tok, 64, 1, False)
        assert rc == -1 and lib.fa_launch_count() == n0
    # decoder stack: the last layer it runs, decoders3 when it finishes, attn_probs over more rows than shared memory holds
    se = _engine("seaco", mode)
    memory, mem_lens, xs, toks = _stack_inputs(1, 6)
    dec = A.FaDecoder.from_buffer_copy(se.seaco_dec)
    dl = _copy_layers(se.seaco_dec.layers, se.seaco_dec.n_layers, A.FaDecLayer)
    dec.layers = dl
    dl[2].ffn_w1.in_f = 256
    rc, _ = _run_stack(se, memory.reshape(-1, 512), mem_lens, 1, 3, 6, xs, toks, 7, 3, 1, dec=dec)
    assert rc == -1 and lib.fa_launch_count() == n0
    dec = A.FaDecoder.from_buffer_copy(se.seaco_dec)
    dec.last.ffn_norm.n += 1
    rc, _ = _run_stack(se, memory.reshape(-1, 512), mem_lens, 1, 3, 6, xs, toks, 7, se.seaco_dec.n_layers, 1, dec=dec)
    assert rc == -1 and lib.fa_launch_count() == n0
    big = 6145                                                      # 4 warps x 6 145 fp32 scores > 96 KB
    mem_big = torch.zeros(big, 512)
    rc, _ = _run_stack(se, mem_big, torch.tensor([big, big], dtype=torch.int32), 1, 2, big, xs[:2], toks[:2], 7, 2, 0, probs=True)
    assert rc == -4 and lib.fa_launch_count() == n0


# ------------------------------------------------------------------------------------------------ bit-exact properties
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_utterances_are_independent_and_runs_repeat(mode):
    """Each utterance run alone with the same t_max gives the rows it gets inside a ragged batch of 64, bit for bit (nothing crosses
    utterances: FSMN halo, CIF conv, attention, cif_pad_planes); the same call on two non-default streams and a second run are
    bit-identical.  Encoder, predictor and decoder."""
    T, B = 129, 64
    g = torch.Generator().manual_seed(64)
    lens = [T, 1, T - 1, 64, 65] + [int(v) for v in torch.randint(1, T + 1, (B - 5,), generator=g)]
    eng = _engine("para", mode)
    enc_s = _enc_struct(eng, "enc", 3)
    x = torch.randn(B, T, 560, generator=g) * torch.from_numpy(R.len_mask(lens, T)).float()[:, :, None]
    ln = torch.tensor(lens, dtype=torch.int32)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    rc, out = _run_encoder(eng, enc_s, x, ln, stream=s1)
    assert rc == 0
    assert torch.equal(_run_encoder(eng, enc_s, x, ln, stream=s2)[1], out)
    assert torch.equal(_run_encoder(eng, enc_s, x, ln, stream=s1)[1], out)
    picks = [0, 1, 2, 3, 4, 37, 63]
    for b in picks:
        assert torch.equal(_run_encoder(eng, enc_s, x[b:b + 1], ln[b:b + 1])[1][0], out[b]), b
    enc = out.cpu()
    pa = _run_predictor(eng, 0, enc, ln, stream=s1)
    pb = _run_predictor(eng, 0, enc, ln, stream=s2)
    assert all(np.array_equal(u, v) for u, v in zip(pa, pb))
    for b in picks:
        one = _run_predictor(eng, 0, enc[b:b + 1], ln[b:b + 1])
        assert all(np.array_equal(u[0], v[b]) for u, v in zip(one, pa)), b
    n_max = 65
    tok = torch.tensor([min(int(t), n_max) for t in pa[1]], dtype=torch.int32)
    acoustic = torch.from_numpy(pa[0])
    da = _run_decoder(eng, eng.dec, enc, ln, acoustic, tok, n_max, 1, True, stream=s1)
    db = _run_decoder(eng, eng.dec, enc, ln, acoustic, tok, n_max, 1, True, stream=s2)
    assert da[0] == 0 and all(np.array_equal(u, v) for u, v in zip(da[1:], db[1:]))
    for b in picks:
        one = _run_decoder(eng, eng.dec, enc[b:b + 1], ln[b:b + 1], acoustic[b:b + 1], tok[b:b + 1], n_max, 1, True)
        assert all(np.array_equal(u[0], v[b]) for u, v in zip(one[1:], da[1:])), b
