"""GPU: the premise of pooling hotword calls, stage by stage.

A row decoded in its own reference pack (the batch the reference decodes it in, with that batch's hotword memory) and the same row in a
pooled pack that holds other groups' rows (a longer row with a larger token count, so a larger n_max and a longer encoder memory, and a
shorter one) over other memories give the same taps, bit for bit.  The reference pack runs the existing entries as the reference's
batch runs them (one shared memory; SeACo's attention-score filter on its utterance 0 over its own n_max query rows); the pooled pack
runs the grouped entries as the handle runs a GPU pack.

Contextual: the decoder's hidden state, log-probs and ids (the bias branch's output is the input of the row-wise decoders3 + after_norm
that give the hidden state).  SeACo: the decoder's hidden state over the reference pack's n_max query rows (padded positions included:
the filter reads them), the filter's probability block [heads, n_max_ref, n_hw] over those rows, cif_att and dec_att, the hotword
arg-max and the merged ids."""
import ctypes as C

import numpy as np
import pytest
import torch

from funasr_b200 import _abi, synth
from funasr_b200.engine import ParaformerEngine

DEV = "cuda:0"
D = 512


def _st():
    return torch.cuda.current_stream().cuda_stream


def _i32(v):
    return (C.c_int32 * len(v))(*v)


def _ws(n):
    return torch.full((int(n),), 255, dtype=torch.uint8, device=DEV)        # NaN-poisoned


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _bits(x):
    return x.contiguous().view(torch.int32).cpu()


class Pack:
    """A padded batch of decoder inputs: encoder output (finite everywhere), encoder lengths, acoustic embeddings (zero past each
    token count, as the CIF predictor leaves them) and token counts."""

    def __init__(self, rows, g):
        self.B = len(rows)
        self.T = max(t for t, _ in rows)
        self.n_max = max(k for _, k in rows)
        self.n_cap = self.T + 1
        enc = torch.randn(self.B, self.T, D, generator=g)
        ac = torch.zeros(self.B, self.n_cap, D)
        for b, (_, k) in enumerate(rows):
            ac[b, :k] = torch.randn(k, D, generator=g)
        self.enc, self.ac = enc.to(DEV), ac.to(DEV)
        self.lens = torch.tensor([t for t, _ in rows], dtype=torch.int32, device=DEV)
        self.tok = torch.tensor([k for _, k in rows], dtype=torch.int32, device=DEV)
        self.tok_h = [k for _, k in rows]

    def rows_from(self, other, at):
        """Copy other's rows into rows at, at.. + other.B (their encoder frames, acoustic rows; lengths and token counts agree)."""
        for j in range(other.B):
            self.enc[at + j].zero_().normal_()
            self.enc[at + j, :other.T] = other.enc[j]
            self.ac[at + j].zero_()
            self.ac[at + j, :other.n_cap] = other.ac[j]


def _make(g, ref_rows, pool_rows, at):
    ref, pool = Pack(ref_rows, g), Pack(pool_rows, g)
    pool.rows_from(ref, at)
    assert pool.n_max > ref.n_max and pool.T > ref.T
    return ref, pool


def _decoder(lib, eng, p, hidden=True, grouped=None):
    """fa_paraformer_decoder_forward_hidden (grouped None) or fa_paraformer_decoder_forward_grouped -> ids, log-probs, hidden."""
    V = eng.cfg.vocab
    ids = torch.full((p.B, p.n_max), -7, dtype=torch.int32, device=DEV)
    best, logp, hid = _nan(p.B, p.n_max), _nan(p.B, p.n_max, V), _nan(p.B, p.n_max, D)
    args = [C.byref(eng.dec), p.enc.data_ptr(), p.lens.data_ptr(), p.B, p.T, p.ac.data_ptr(), p.n_cap, p.tok.data_ptr(), p.n_max, ids.data_ptr(),
            best.data_ptr(), logp.data_ptr(), 1, hid.data_ptr()]
    if grouped is None:
        nh = eng.dec.n_hotwords if eng.dec.has_bias else 0
        ws = _ws(lib.fa_paraformer_decoder_workspace_bytes_hw(p.B, p.T, p.n_max, V, eng.mode, nh))
        _abi.check(lib.fa_paraformer_decoder_forward_hidden(*args, eng.mode, ws.data_ptr(), ws.numel(), _st()), "forward_hidden")
    else:
        mem, lens, group = grouped
        G, nh_max = mem.shape[0], mem.shape[1]
        ws = _ws(lib.fa_paraformer_decoder_grouped_workspace_bytes(p.B, p.T, p.n_max, V, eng.mode, G, nh_max))
        _abi.check(lib.fa_paraformer_decoder_forward_grouped(*args, mem.data_ptr(), _i32(lens), _i32(group), G, nh_max, eng.mode, ws.data_ptr(),
                                                             ws.numel(), _st()), "forward_grouped")
    torch.cuda.synchronize()
    return ids.cpu(), logp, hid


def _padded(sets):
    """Host row sets -> device memories [G, longest, 512] with zero rows past each set, and their lengths."""
    nh = max(s.shape[0] for s in sets)
    mem = torch.zeros(len(sets), nh, D)
    for i, s in enumerate(sets):
        mem[i, :s.shape[0]] = s
    return mem.to(DEV), [s.shape[0] for s in sets]


def _rows(n, g):
    return torch.randn(n, D, generator=g) * 0.5


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_contextual_row_in_pooled_pack_equals_its_reference_pack(mode):
    lib = _abi.load()
    cfg = synth.PARAFORMER_TINY
    eng = ParaformerEngine(synth.make_contextual_state_dict(cfg, 6), cfg, DEV, gemm_mode=mode, contextual=True)
    g = torch.Generator().manual_seed(51)
    ref, pool = _make(g, [(37, 9), (52, 14)], [(90, 20), (37, 9), (52, 14), (11, 3)], 1)
    hw_a, hw_b, hw_c = _rows(25, g), _rows(40, g), _rows(3, g)
    # the reference pack: its memory shared by its rows (fa_paraformer_decoder_forward_hidden, kv_shared)
    mem_a = hw_a.to(DEV).contiguous()
    lens_a = torch.full((ref.B,), 25, dtype=torch.int32, device=DEV)
    eng.dec.has_bias, eng.dec.n_hotwords, eng.dec.hw_embed, eng.dec.hw_lens = 1, 25, mem_a.data_ptr(), lens_a.data_ptr()
    ids_r, logp_r, hid_r = _decoder(lib, eng, ref)
    # the pooled pack: three memories, the reference pack's rows over memory 1
    mem, lens = _padded([hw_b, hw_a, hw_c])
    ids_p, logp_p, hid_p = _decoder(lib, eng, pool, grouped=(mem, lens, [0, 1, 1, 2]))
    for j, k in enumerate(ref.tok_h):
        b = 1 + j
        assert torch.equal(ids_p[b, :k], ids_r[j, :k]), (mode, j)
        assert torch.equal(_bits(logp_p[b, :k]), _bits(logp_r[j, :k])), (mode, j)
        assert torch.equal(_bits(hid_p[b, :k]), _bits(hid_r[j, :k])), (mode, j)


def _stack(lib, eng, memory, x, ld, p, n_max, finish, probs=None, grouped=None, shared_lens=None, batch=None):
    """fa_sanm_decoder_stack_forward (one shared memory) or fa_sanm_decoder_stack_forward_grouped over x -> hidden or probabilities."""
    n_s = eng.seaco_dec.n_layers
    B = batch or p.B
    hid = None if probs is not None else _nan(B, n_max, D)
    n_run = 6 if probs is not None else n_s
    if grouped is None:
        n_hw = memory.shape[0]
        ml = torch.full((B,), n_hw, dtype=torch.int32, device=DEV)
        ws = _ws(lib.fa_sanm_decoder_stack_workspace_bytes(B, n_hw, n_max, eng.mode))
        _abi.check(lib.fa_sanm_decoder_stack_forward(C.byref(eng.seaco_dec), memory.data_ptr(), ml.data_ptr(), 1, B, n_hw, x.data_ptr(), ld,
                                                     p.tok.data_ptr(), n_max, n_run, finish, None if hid is None else hid.data_ptr(),
                                                     None if probs is None else probs.data_ptr(), eng.mode, ws.data_ptr(), ws.numel(), _st()),
                   "stack")
    else:
        lens, group, probe = grouped
        G, t_mem = memory.shape[0], memory.shape[1]
        n_probe = len(probe) if probs is not None else 0
        ws = _ws(lib.fa_sanm_decoder_stack_grouped_workspace_bytes(B, G, t_mem, n_max, n_probe, eng.mode))
        _abi.check(lib.fa_sanm_decoder_stack_forward_grouped(C.byref(eng.seaco_dec), memory.data_ptr(), _i32(lens), _i32(group), G, B, t_mem,
                                                             x.data_ptr(), ld, p.tok.data_ptr(), n_max, n_run, finish,
                                                             None if hid is None else hid.data_ptr(), None if probs is None else probs.data_ptr(),
                                                             _i32(probe) if n_probe else None, n_probe, eng.mode, ws.data_ptr(), ws.numel(),
                                                             _st()), "stack grouped")
    torch.cuda.synchronize()
    return hid


def _select(lib, probs_h, H, n_rows, n_hw, nfilter):
    picked = np.zeros(n_hw, np.int32)
    blk = np.ascontiguousarray(probs_h, np.float32)
    n = lib.fa_seaco_asf_select_host(blk.ctypes.data, H, n_rows, n_hw, nfilter, picked.ctypes.data)
    assert n >= 1
    return picked[:n].tolist()


def _bias(lib, eng, cif, dec, ids, best, B, n_max):
    """hotword_output_layer's arg-max over cif_att + dec_att, then the NO_BIAS merge -> (hotword ids, merged ids)."""
    rows = B * n_max
    V = eng.cfg.vocab
    dha, dbest = torch.full((rows,), -7, dtype=torch.int32, device=DEV), _nan(rows)
    ws = _ws(lib.fa_linear_argmax_workspace_bytes(rows, V, eng.mode))
    _abi.check(lib.fa_linear_argmax(C.byref(eng.hw_out), cif.data_ptr(), dec.data_ptr(), rows, dha.data_ptr(), dbest.data_ptr(), None, eng.mode,
                                    ws.data_ptr(), ws.numel(), _st()), "fa_linear_argmax")
    out, obest = torch.full((rows,), -7, dtype=torch.int32, device=DEV), _nan(rows)
    idd, bd = ids.to(DEV).contiguous(), best.contiguous()
    _abi.check(lib.fa_seaco_merge(idd.data_ptr(), bd.data_ptr(), dha.data_ptr(), dbest.data_ptr(), rows, eng.no_bias, out.data_ptr(), obest.data_ptr(),
                                  None, None, None, V, _st()), "fa_seaco_merge")
    torch.cuda.synchronize()
    return dha.view(B, n_max).cpu(), out.view(B, n_max).cpu()


def _best(logp, ids):
    return torch.gather(logp, 2, ids.to(DEV).long().unsqueeze(-1)).squeeze(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,mode", [("tiny", "fp32"), ("tiny", "fp16x3"), ("large", "fp16x3")])
def test_seaco_row_in_pooled_pack_equals_its_reference_pack(kind, mode):
    """A 25-row list with nfilter 8, as in the seaco_tiny_asf golden: the reference pack's filter runs on its utterance 0 over its own
    n_max = 14 query rows; in the pooled pack the filter probes run together over n_max = 20 query rows (the other reference pack's
    first row, over its own 40-row memory, is the first probe) and the reference pack's block is cut back to 14 rows."""
    lib = _abi.load()
    cfg = synth.PARAFORMER_LARGE if kind == "large" else synth.PARAFORMER_TINY
    nfilter = 8
    eng = ParaformerEngine(synth.make_seaco_state_dict(cfg, 11), cfg, DEV, gemm_mode=mode, seaco=True, no_bias=synth.seaco_no_bias_id(cfg))
    H = eng.seaco_dec.heads
    g = torch.Generator().manual_seed(53)
    ref, pool = _make(g, [(37, 9), (52, 14)], [(90, 20), (37, 9), (52, 14), (11, 3)], 1)
    hw_a, hw_b, hw_c = _rows(25, g), _rows(40, g), _rows(3, g)
    # ---- the reference pack, as the reference decodes it
    ids_r, logp_r, hid_r = _decoder(lib, eng, ref)
    mem_a = hw_a.to(DEV).contiguous()
    probs_r = _nan(H, ref.n_max, 25)
    _stack(lib, eng, mem_a, hid_r, ref.n_max, ref, ref.n_max, 0, probs=probs_r, batch=1)
    pick_r = _select(lib, probs_r.cpu().numpy(), H, ref.n_max, 25, nfilter)
    sel_r = mem_a[torch.tensor(pick_r, device=DEV)].contiguous()
    cif_r = _stack(lib, eng, sel_r, ref.ac, ref.n_cap, ref, ref.n_max, 1)
    dec_r = _stack(lib, eng, sel_r, hid_r, ref.n_max, ref, ref.n_max, 1)
    dha_r, merged_r = _bias(lib, eng, cif_r, dec_r, ids_r, _best(logp_r, ids_r), ref.B, ref.n_max)
    # ---- the pooled pack, as the handle decodes it: rows [other pack (set B), reference pack (set A) x 2, third pack (set C)]
    ids_p, logp_p, hid_p = _decoder(lib, eng, pool)
    mem, lens = _padded([hw_a, hw_b, hw_c])
    group = [1, 0, 0, 2]
    probs_p = _nan(2, H, pool.n_max, 40)
    _stack(lib, eng, mem, hid_p, pool.n_max, pool, pool.n_max, 0, probs=probs_p, grouped=(lens, group, [0, 1]))
    blk = probs_p[1, :, :ref.n_max, :25]                      # the reference pack's block: its first row (pooled row 1), its n_max
    pick_b = _select(lib, probs_p[0].cpu().numpy(), H, pool.n_max, 40, nfilter)
    pick_p = _select(lib, blk.cpu().numpy(), H, ref.n_max, 25, nfilter)
    sel, sel_lens = _padded([hw_b[torch.tensor(pick_b)], hw_a[torch.tensor(pick_p)], hw_c])
    cif_p = _stack(lib, eng, sel, pool.ac, pool.n_cap, pool, pool.n_max, 1, grouped=(sel_lens, [0, 1, 1, 2], []))
    dec_p = _stack(lib, eng, sel, hid_p, pool.n_max, pool, pool.n_max, 1, grouped=(sel_lens, [0, 1, 1, 2], []))
    dha_p, merged_p = _bias(lib, eng, cif_p, dec_p, ids_p, _best(logp_p, ids_p), pool.B, pool.n_max)
    where = (kind, mode)
    assert torch.equal(_bits(blk), _bits(probs_r)), where                  # padded query rows [9, 14) of utterance 0 included
    assert pick_p == pick_r, where
    for j, k in enumerate(ref.tok_h):
        b = 1 + j
        assert torch.equal(_bits(hid_p[b, :ref.n_max]), _bits(hid_r[j])), (where, j)   # padded positions below n_max_ref included
        assert torch.equal(ids_p[b, :k], ids_r[j, :k]), (where, j)
        assert torch.equal(_bits(logp_p[b, :k]), _bits(logp_r[j, :k])), (where, j)
        assert torch.equal(_bits(cif_p[b, :k]), _bits(cif_r[j, :k])), (where, j)
        assert torch.equal(_bits(dec_p[b, :k]), _bits(dec_r[j, :k])), (where, j)
        assert torch.equal(dha_p[b, :k], dha_r[j, :k]), (where, j)
        assert torch.equal(merged_p[b, :k], merged_r[j, :k]), (where, j)
