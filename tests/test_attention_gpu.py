"""GPU (-m gpu): kernel-level parity of the attention path as the models run it.  The models never call fa_attention_tc: the
QKV / q / kv GEMM epilogues write the attention operands as fp16 planes (fa_linear_attn_sinks exposes that epilogue), the
tensor-core kernel reads them (fa_attention_tc_planes) and writes the context as planes for the out-projection.  The fp32 path
runs the tiled kernel for 128-wide heads and the warp-per-query kernel otherwise (fa_attention_f32_ex).

Two kinds of checks.
  * Bit-exact consistency, no tolerance.
      - The sinks against the same GEMM's fp32 epilogue: the tile width depends only on the mode and the main loop is shared, so
        both runs hold the same accumulators, and the sinks must equal the CPU split (hi = RN(x), lo = RN(x - hi), as
        pack_planes2 does) of fl(y * qscale), of y, and of y transposed per utterance.  Every buffer starts as NaN, so a write
        outside the sinks (pad columns of V^T, surplus planes, non-V fp32 columns) shows.
      - fa_attention_tc against the plane entry fed with CPU-made splits of the same operands; the fp32 context against its own
        planes; a shared K/V against the same K/V replicated per utterance; an utterance against a permuted or reduced batch; a
        head against the same head run alone.
  * Against float64.
      - Plane-fed attention against softmax attention in float64 on the RECONSTRUCTED operands (sum of the planes), so only the
        kernel's own arithmetic stands between the two sides: the dropped lo * lo terms of the scores, P rounded to planes, fp32
        accumulation.  The error is max |ctx - ref| / max |V|: the context is a convex combination of V rows.  Expected orders:
        ~2^-22 relative per operand product with two planes, ~2^-12 from the single P plane of fp16 (x1).
      - The whole attention block (planes -> sinks -> attention -> context planes -> out-projection) against a float64
        restatement of MultiHeadedAttentionSANM's attention branch (FSMN excluded).
      - The fp32 kernels against float64 from the same fp32 inputs.
Each float64 bar was measured on an H100 80GB HBM3 (700 W power limit); the comment beside each constant gives the worst case
and where the error comes from.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
HD = 128
NAN = float("nan")
F16 = torch.float16
QSCALE = float(np.float32(1.0 / math.sqrt(128.0)))      # (float)(1 / sqrt(128)), the kernels' d_k^-0.5
NPL = {"fp16": 1, "fp16x3": 2, "fp16x6": 3}             # GEMM A-operand planes
QPL = {"fp16": 1, "fp16x3": 2, "fp16x6": 2}             # attention operand planes: at most two
MODES = list(NPL)

# Bars, each measured on an H100 80GB HBM3 (700 W power limit) and kept at least 3x above the worst case seen.
# Plane-fed attention against float64 (max |d ctx| / max |V|), scores of unit scale (|s| <~ 5: random operands, q = 0, |V| ~ 1e3).
# Worst: 9.2e-7 (x3, H = 8, tq = 128, tk = 65) and 1.6e-4 (x1, |V| ~ 1e3).
F64_TOL = {"fp16x3": 3e-6, "fp16": 5e-4}
# The same with scores in the tens to hundreds (peaked rows, probabilities spanning e^-30, near ties).  Two terms grow there and
# are part of the kernel's arithmetic, not of the planes: the scores are accumulated in fp32 on the tensor cores, which truncate
# at every 16-wide k-step (24 steps over three terms), so |d s| grows with |s| and shifts probability between near-equal keys;
# and the O / l epilogue undoes an expected truncation shrink of 5.3e-8 per P.V k-step (4 per 64-key chunk), which over-corrects
# rows whose P.V steps add only exact zeros (a peaked row): up to 4 * 65 * 5.3e-8 = 1.4e-5 at 4100 keys.
# Worst: 1.3e-5 (x3, near tie, tk = 500; 9.7e-6 peaked at tk = 4100).  x1 keeps F64_TOL (P rounded to one plane dominates).
F64_TOL_LARGE_S = {"fp16x3": 4e-5, "fp16": 5e-4}
LARGE_S = ("peaked", "span_e30", "near_tie")
# Whole attention block against float64 (rel_err of the out-projection output); test_attention_tcgen05_vs_oracle allows 5e-5 and
# 2e-2.  Worst: 3.2e-6 (x3, decoder cross-attention N = 200; x6 3.1e-6) and 5.5e-4 (x1).
BLOCK_TOL = {"fp16x6": 1e-5, "fp16x3": 1e-5, "fp16": 2e-3}
# fp32 kernels against float64 (max |d ctx| / max |V|).  Worst: 2.5e-7.
F32_TOL = 1e-6


def _lib():
    from funasr_b200 import _abi
    return _abi, _abi.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    return t.contiguous().view(torch.int32)


def _split(x, n):
    """fp16 planes [n, *x.shape] of fp32 x as the kernels make them: hi = RN(x), then RN of each fp32 residual."""
    r = x.float().clone()
    out = []
    for _ in range(n):
        h = r.half()
        out.append(h)
        r = r - h.float()
    return torch.stack(out)


def _same(got, want, what):
    """Equal values (fp16 planes compared as values, so -0 == 0), no NaN on either side."""
    g, w = got.float(), want.float()
    bad = ~(g == w)
    n = int(bad.sum())
    if n:
        idx = bad.nonzero()[0].tolist()
        raise AssertionError("%s: %d of %d differ, first at %s: got %r want %r" % (what, n, bad.numel(), idx, float(g[tuple(idx)]),
                                                                                   float(w[tuple(idx)])))


class _Linear:
    """nn.Linear weights on the device with their fp16 planes (fa_split_planes) and the FaLinear describing them."""

    def __init__(self, abi, lib, out_f, in_f, seed):
        g = torch.Generator().manual_seed(seed)
        self.w = torch.randn(out_f, in_f, generator=g) / math.sqrt(in_f)
        self.b = torch.randn(out_f, generator=g) * 0.1
        self.in_pad = (in_f + 63) // 64 * 64
        self.wd, self.bd = self.w.to(DEV), self.b.to(DEV)
        self.wp = torch.empty(3, out_f, self.in_pad, dtype=F16, device=DEV)
        abi.check(lib.fa_split_planes(self.wd.data_ptr(), in_f, out_f, in_f, self.in_pad, self.wp.data_ptr(), _st()), "fa_split_planes")
        self.lin = abi.FaLinear(self.wd.data_ptr(), self.bd.data_ptr(), self.wp.data_ptr(), out_f, in_f, self.in_pad, 0)


def _a_planes(abi, lib, x, npl, in_pad):
    rows, in_f = x.shape
    p = torch.empty(npl, rows, in_pad, dtype=F16, device=DEV)
    abi.check(lib.fa_split_rows(x.data_ptr(), in_f, rows, in_f, in_pad, npl, p.data_ptr(), _st()), "fa_split_rows")
    return p


def _vt(v, B, tk, tkp, npl, pad=NAN):
    """V [B * tk, d] fp32 -> transposed planes [npl][B * d][tkp], columns >= tk filled with `pad`."""
    d = v.shape[1]
    vt = torch.full((npl, B * d, tkp), pad, dtype=F16)
    vt[:, :, :tk] = _split(v.reshape(B, tk, d).transpose(1, 2).reshape(B * d, tk), npl)
    return vt


def _planes_attention(abi, lib, qp, kp, vt, lens, B, H, tq, tk, mode, kv_shared=0):
    """fa_attention_tc_planes on CPU-made planes -> fp32 context [B * tq, H * 128] (NaN-initialised)."""
    d = H * HD
    ctx = torch.full((B * tq, d), NAN, device=DEV)
    qd, kd, vd = qp.to(DEV), kp.to(DEV), vt.to(DEV)
    ld = torch.tensor(lens, dtype=torch.int32, device=DEV)
    st = lib.fa_attention_tc_planes(qd.data_ptr(), kd.data_ptr(), vd.data_ptr(), ld.data_ptr(), B, H, tq, tk, ctx.data_ptr(), d,
                                    None, 0, 0, abi.GEMM_MODES[mode], kv_shared, _st())
    assert st == 0, st
    torch.cuda.synchronize()
    return ctx.cpu()


def _tc_run(abi, lib, q, k, v, lens, B, H, tq, tk, mode, kv_shared=0):
    """Plane-fed tensor-core attention of fp32 operands (q already scaled): planes made on the CPU -> context [B * tq, d]."""
    npl = QPL[mode]
    kb = 1 if kv_shared else B
    tkp = (tk + 63) // 64 * 64
    return _planes_attention(abi, lib, _split(q, npl), _split(k, npl), _vt(v, kb, tk, tkp, npl), lens, B, H, tq, tk, mode, kv_shared)


def _ref64(q, k, v, lens, B, H, tq, tk, hd=HD, kv_shared=False, qh=None, kh=None):
    """float64 masked softmax attention, heads merged: q [B * tq, H * hd] (scaled), k / v [kb * tk, H * hd] -> [B * tq, H * hd].
    With the hi planes qh / kh also returns the largest p' = 2^10 exp(s - m~) (m~: the row maximum of hi . hi, pass A) and the
    number of rows whose hi . hi arg-max is not the exact arg-max."""
    d = H * hd
    out = torch.zeros(B * tq, d, dtype=torch.float64)
    pmax, wrong = 0.0, 0
    for b in range(B):
        n = min(int(lens[b]), tk)
        if n == 0:
            continue
        bk = 0 if kv_shared else b
        qb = q[b * tq:(b + 1) * tq].double().reshape(tq, H, hd).transpose(0, 1)
        kb = k[bk * tk:bk * tk + n].double().reshape(n, H, hd).transpose(0, 1)
        vb = v[bk * tk:bk * tk + n].double().reshape(n, H, hd).transpose(0, 1)
        s = qb @ kb.transpose(1, 2)
        out[b * tq:(b + 1) * tq] = (torch.softmax(s, -1) @ vb).transpose(0, 1).reshape(tq, d)
        if qh is not None:
            sh = qh[b * tq:(b + 1) * tq].double().reshape(tq, H, hd).transpose(0, 1) @ \
                kh[bk * tk:bk * tk + n].double().reshape(n, H, hd).transpose(0, 1).transpose(1, 2)
            m = sh.max(-1, keepdim=True).values
            pmax = max(pmax, float((1024.0 * torch.exp(s - m)).max()))
            wrong += int((sh.argmax(-1) != s.argmax(-1)).sum())
    return out, pmax, wrong


# ============================================================================================ 1. GEMM attention sinks
# (name, batch, t_rows, t_pad, N, q0, k0, v0, in_f, fp32 V copy)
SINK_CASES = [
    ("enc_t100_k560", 3, 100, 128, 1536, 0, 512, 1024, 560, True),   # staged transpose (t_rows % 4 == 0), ragged last row tile
    ("enc_t37", 5, 37, 64, 1536, 0, 512, 1024, 512, True),           # store_vt16 path (t_rows % 4 != 0), ragged
    ("enc_t12", 20, 12, 64, 1536, 0, 512, 1024, 512, False),         # t_rows < 32: a warp's 32 rows span three utterances
    ("enc_t1", 64, 1, 64, 1536, 0, 512, 1024, 512, True),            # t_rows = 1
    ("enc_t256", 2, 256, 256, 1536, 0, 512, 1024, 512, True),        # interior tiles only
    ("enc_pad102", 3, 100, 102, 1536, 0, 512, 1024, 512, False),     # t_pad % 4 != 0 turns the staged path off
    ("dec_q", 3, 13, 64, 512, 0, -1, -1, 512, False),                # decoder cross-attention: q-only sink
    ("dec_kv", 2, 150, 192, 1024, -1, 0, 512, 512, False),           # decoder memory: kv-only sink
    ("dec_kv_t7", 9, 7, 64, 1024, -1, 0, 512, 512, False),           # hotword-sized memory
]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", SINK_CASES, ids=[c[0] for c in SINK_CASES])
def test_attn_sinks_equal_split_of_fp32_epilogue(case, mode):
    name, B, T, t_pad, N, q0, k0, v0, in_f, want_v32 = case
    abi, lib = _lib()
    M, W = B * T, 512
    L = _Linear(abi, lib, N, in_f, seed=N + in_f)
    x = torch.randn(M, in_f, generator=torch.Generator().manual_seed(M))
    ap = _a_planes(abi, lib, x.to(DEV), NPL[mode], L.in_pad)
    gm = abi.GEMM_MODES[mode]
    y = torch.full((M, N), NAN, device=DEV)
    abi.check(lib.fa_linear_planes(ap.data_ptr(), M, C.byref(L.lin), 0, None, 0, None, 0, y.data_ptr(), N, gm, _st()), "fp32 epilogue")
    qp = torch.full((3, M, W), NAN, dtype=F16, device=DEV)
    kp = torch.full((3, M, W), NAN, dtype=F16, device=DEV)
    vt = torch.full((3, B * W, t_pad), NAN, dtype=F16, device=DEV)
    v32 = torch.full((M, N), NAN, device=DEV) if want_v32 else None
    abi.check(lib.fa_linear_attn_sinks(ap.data_ptr(), M, C.byref(L.lin), q0, k0, v0, W, T, t_pad, QSCALE, qp.data_ptr(), kp.data_ptr(),
                                       vt.data_ptr(), v32.data_ptr() if want_v32 else None, N, gm, _st()), "attn sinks")
    torch.cuda.synchronize()
    y, qp, kp, vt = y.cpu(), qp.cpu(), kp.cpu(), vt.cpu()
    assert not torch.isnan(y).any()
    npl = QPL[mode]
    if q0 >= 0:
        _same(qp[:npl], _split(y[:, q0:q0 + W] * torch.tensor(QSCALE), npl), "q planes")
    else:
        assert torch.isnan(qp).all()
    if k0 >= 0:
        _same(kp[:npl], _split(y[:, k0:k0 + W], npl), "k planes")
    else:
        assert torch.isnan(kp).all()
    if v0 >= 0:
        yt = y[:, v0:v0 + W].reshape(B, T, W).transpose(1, 2).reshape(B * W, T)
        _same(vt[:npl, :, :T], _split(yt, npl), "v^T planes")
        assert torch.isnan(vt[:, :, T:]).all(), "pad columns [t_rows, t_pad) of V^T written"
    else:
        assert torch.isnan(vt).all()
    assert torch.isnan(qp[npl:]).all() and torch.isnan(kp[npl:]).all() and torch.isnan(vt[npl:]).all(), "surplus plane written"
    if want_v32:
        v32 = v32.cpu()
        assert torch.equal(v32[:, v0:v0 + W], y[:, v0:v0 + W])
        assert torch.isnan(v32[:, :v0]).all() and torch.isnan(v32[:, v0 + W:]).all(), "fp32 columns outside V written"


# ============================================================================================ 2-5. bit-exact attention
def _rand_qkv(B, H, tq, tk, seed, kb=None):
    g = torch.Generator().manual_seed(seed)
    d = H * HD
    kb = B if kb is None else kb
    return (torch.randn(B * tq, d, generator=g) * 1.5, torch.randn(kb * tk, d, generator=g) * 1.5, torch.randn(kb * tk, d, generator=g))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,H,tq,tk,lens", [(3, 4, 130, 130, [130, 1, 65]), (2, 4, 37, 211, [211, 0]), (1, 1, 1, 1, [1]),
                                            (2, 8, 129, 500, [500, 600])])
def test_attention_tc_equals_plane_entry(B, H, tq, tk, lens, mode):
    """fa_attention_tc (which splits its fp32 operands itself) equals the plane entry fed with the CPU splits of fl(q * 128^-0.5),
    k and V^T.  The plane entry's V^T pad columns hold NaN: they must never be read (the tensor map ends at tk)."""
    abi, lib = _lib()
    q, k, v = _rand_qkv(B, H, tq, tk, seed=tq * 1000 + tk)
    d = H * HD
    gm = abi.GEMM_MODES[mode]
    ld = torch.tensor(lens, dtype=torch.int32, device=DEV)
    ctx = torch.full((B * tq, d), NAN, device=DEV)
    ws = torch.empty(lib.fa_attention_tc_workspace_bytes(B, H, tq, tk, gm), dtype=torch.uint8, device=DEV)
    qd, kd, vd = q.to(DEV), k.to(DEV), v.to(DEV)
    abi.check(lib.fa_attention_tc(qd.data_ptr(), d, kd.data_ptr(), d, vd.data_ptr(), d, ld.data_ptr(), B, H, tq, tk, ctx.data_ptr(), d, gm,
                                  ws.data_ptr(), ws.numel(), _st()), "fa_attention_tc")
    torch.cuda.synchronize()
    got = _tc_run(abi, lib, q * torch.tensor(QSCALE), k, v, lens, B, H, tq, tk, mode)
    assert not torch.isnan(got).any()
    assert torch.equal(_bits(got), _bits(ctx.cpu()))


@pytest.mark.parametrize("mode,opl", [("fp16", 1), ("fp16x3", 2), ("fp16x3", 3), ("fp16x6", 2), ("fp16x6", 3)])
def test_context_planes_are_split_of_fp32_context(mode, opl):
    """One launch writes the fp32 context and its planes: the planes are the exact split of the fp32 values, the fp32 values equal a
    context-only launch, and nothing lands outside [out_nplanes][B * tq][d] (guard columns, surplus planes, a guard row)."""
    abi, lib = _lib()
    B, H, tq, tk, lens = 3, 4, 130, 200, [200, 64, 1]
    d, ldc, ldp = H * HD, H * HD + 4, H * HD + 8
    q, k, v = _rand_qkv(B, H, tq, tk, seed=41)
    npl = QPL[mode]
    qp, kp, vt = _split(q * torch.tensor(QSCALE), npl).to(DEV), _split(k, npl).to(DEV), _vt(v, B, tk, 256, npl).to(DEV)
    ld = torch.tensor(lens, dtype=torch.int32, device=DEV)
    ctx = torch.full((B * tq + 1, ldc), NAN, device=DEV)
    pl = torch.full((4, B * tq, ldp), NAN, dtype=F16, device=DEV)
    gm = abi.GEMM_MODES[mode]
    abi.check(lib.fa_attention_tc_planes(qp.data_ptr(), kp.data_ptr(), vt.data_ptr(), ld.data_ptr(), B, H, tq, tk, ctx.data_ptr(), ldc,
                                         pl.data_ptr(), ldp, opl, gm, 0, _st()), "ctx + planes")
    alone = torch.full((B * tq, d), NAN, device=DEV)
    abi.check(lib.fa_attention_tc_planes(qp.data_ptr(), kp.data_ptr(), vt.data_ptr(), ld.data_ptr(), B, H, tq, tk, alone.data_ptr(), d,
                                         None, 0, 0, gm, 0, _st()), "ctx only")
    torch.cuda.synchronize()
    ctx, pl = ctx.cpu(), pl.cpu()
    assert torch.isnan(ctx[B * tq]).all() and torch.isnan(ctx[:, d:]).all()
    assert not torch.isnan(ctx[:B * tq, :d]).any()
    assert torch.equal(_bits(ctx[:B * tq, :d]), _bits(alone.cpu()))
    _same(pl[:opl, :, :d], _split(ctx[:B * tq, :d], opl), "context planes")
    assert torch.isnan(pl[opl:]).all() and torch.isnan(pl[:, :, d:]).all(), "context planes written outside [out_nplanes][B * tq][d]"


@pytest.mark.parametrize("tk,lens", [(17, [17, 1, 0, 16, 20]), (130, [130, 64, 65, 1, 200])])
def test_kv_shared_equals_replicated_kv(tk, lens):
    """kv_shared (the hotword memory: one K/V for every utterance) against the same K/V replicated per utterance, with per-utterance
    key_lens: the tensor-core kernel in both plane counts and both fp32 kernels."""
    abi, lib = _lib()
    B, tq = len(lens), 9
    for mode in ("fp16", "fp16x3"):
        H = 4
        q, k, v = _rand_qkv(B, H, tq, tk, seed=tk, kb=1)
        q = q * torch.tensor(QSCALE)
        shared = _tc_run(abi, lib, q, k, v, lens, B, H, tq, tk, mode, kv_shared=1)
        rep = _tc_run(abi, lib, q, k.repeat(B, 1), v.repeat(B, 1), lens, B, H, tq, tk, mode)
        assert not torch.isnan(shared).any()
        assert torch.equal(_bits(shared), _bits(rep)), mode
    for hd, H in ((128, 4), (32, 8)):
        g = torch.Generator().manual_seed(hd)
        q, k, v = (torch.randn(n, H * hd, generator=g) for n in (B * tq, tk, tk))
        shared = _f32_run(abi, lib, q, k, v, lens, B, H, hd, tq, tk, kv_shared=1)
        rep = _f32_run(abi, lib, q, k.repeat(B, 1), v.repeat(B, 1), lens, B, H, hd, tq, tk)
        assert torch.equal(_bits(shared), _bits(rep)), hd


def _f32_run(abi, lib, q, k, v, lens, B, H, hd, tq, tk, kv_shared=0, ld=1536):
    """fa_attention_f32_ex over the pitch-1536 views of a QKV buffer: q at column 0, k at 512, v at 1024."""
    d = H * hd
    kb = 1 if kv_shared else B
    qb = torch.full((B * tq, ld), NAN)
    kvb = torch.full((kb * tk, ld), NAN)
    qb[:, :d], kvb[:, 512:512 + d], kvb[:, 1024:1024 + d] = q, k, v
    qb, kvb = qb.to(DEV), kvb.to(DEV)
    ctx = torch.full((B * tq, d), NAN, device=DEV)
    ldev = torch.tensor(lens, dtype=torch.int32, device=DEV)
    st = lib.fa_attention_f32_ex(qb.data_ptr(), ld, kvb.data_ptr() + 512 * 4, ld, kvb.data_ptr() + 1024 * 4, ld, ldev.data_ptr(), B, H, hd,
                                 tq, tk, ctx.data_ptr(), d, kv_shared, _st())
    assert st == 0, st
    torch.cuda.synchronize()
    return ctx.cpu()


def _per_utt(t, rows):
    return list(t.split(rows))


@pytest.mark.parametrize("kind", ["fp16", "fp16x3", "f32_128", "f32_32"])
def test_context_independent_of_batch_and_heads(kind):
    """An utterance's context is bitwise the same in a permuted batch and in a reduced one, and a head's context is the same as that
    head run alone (H = 1 on its column slice of every operand)."""
    abi, lib = _lib()
    B, H, tq, tk, lens = 5, 4, 70, 150, [150, 3, 64, 0, 129]
    hd = 32 if kind == "f32_32" else HD
    g = torch.Generator().manual_seed(7)
    q, k, v = torch.randn(B * tq, H * hd, generator=g), torch.randn(B * tk, H * hd, generator=g), torch.randn(B * tk, H * hd, generator=g)

    def run(qq, kk, vv, ll, hh):
        nb = len(ll)
        if kind.startswith("f32"):
            return _f32_run(abi, lib, qq, kk, vv, ll, nb, hh, hd, tq, tk)
        return _tc_run(abi, lib, qq * torch.tensor(QSCALE), kk, vv, ll, nb, hh, tq, tk, kind)

    full = run(q, k, v, lens, H)
    assert not torch.isnan(full).any()
    qs, ks, vs, outs = _per_utt(q, tq), _per_utt(k, tk), _per_utt(v, tk), _per_utt(full, tq)
    for sel in ([3, 0, 4, 2, 1], [1, 4], [2]):
        got = run(torch.cat([qs[i] for i in sel]), torch.cat([ks[i] for i in sel]), torch.cat([vs[i] for i in sel]), [lens[i] for i in sel], H)
        assert torch.equal(_bits(got), _bits(torch.cat([outs[i] for i in sel]))), sel
    for h in (0, 3):
        c = slice(h * hd, (h + 1) * hd)
        got = run(q[:, c].contiguous(), k[:, c].contiguous(), v[:, c].contiguous(), lens, 1)
        assert torch.equal(_bits(got), _bits(full[:, c].contiguous())), h


# ============================================================================================ 6. plane-fed attention vs float64
F64_SHAPES = [
    (1, 1, 1, 1, [1]),                       # batch 1, tq = 1: the 128-row Q box is larger than the whole tensor
    (1, 4, 1, 7, [7]),
    (2, 4, 4, 63, [63, 0]),                  # an utterance without keys: zero context
    (3, 4, 127, 64, [64, 1, 63]),
    (3, 8, 128, 65, [65, 64, 2]),
    (2, 1, 129, 500, [500, 129]),
    (4, 4, 500, 500, [500, 128, 192, 600]),  # 64-key chunk boundaries; 600 > tk clamps
    (2, 4, 4, 1500, [1500, 1000]),
    (1, 8, 129, 4100, [4100]),               # the K / V ring wraps ~130 times
    (2, 1, 64, 4100, [4097, 4033]),
]
REGIME_SHAPES = [(3, 4, 129, 500, [500, 65, 2]), (1, 4, 4, 4100, [4100])]
REGIMES = ["unit", "q_zero", "peaked", "span_e30", "near_tie", "v_1e3"]


def _regime(name, B, H, tq, tk, lens, seed):
    """(q already scaled, k, v) fp32 for one value regime."""
    g = torch.Generator().manual_seed(seed)
    d = H * HD
    q = torch.randn(B * tq, d, generator=g) * QSCALE
    k = torch.randn(B * tk, d, generator=g)
    v = torch.randn(B * tk, d, generator=g)
    rows = torch.arange(tq)
    if name == "q_zero":                     # uniform weights: the context is the mean of the valid V rows
        q.zero_()
    elif name in ("peaked", "near_tie"):
        if name == "peaked":                 # scores ~256 at one key per row, the rest within ~±80: ahead by far more than 20
            k *= 2.0
        else:                                # key 2i + 1 = key 2i + 1e-4 noise: the pair's scores differ by less than hi . hi resolves
            k = k.reshape(B, tk, d)
            k[:, 1::2] = k[:, 0:tk - tk % 2:2] + 1e-4 * torch.randn(B, tk // 2, d, generator=g)
            k = k.reshape(B * tk, d)
        for b in range(B):
            n = min(lens[b], tk)
            if n < 2:
                continue
            tgt = (rows * 2 % (n - n % 2)) if name == "near_tie" else rows % n
            q[b * tq:(b + 1) * tq] = 0.5 * k[b * tk + tgt] + 0.01 * torch.randn(tq, d, generator=g)
    elif name == "span_e30":                 # scores 30 t_j, t_j in [0, 1), + O(0.01): probabilities from 1 down to ~e^-30
        q = (q / QSCALE * 0.01).reshape(-1, H, HD)
        k = (k * 0.1).reshape(-1, H, HD)
        q[:, :, 0] = 30.0
        k[:, :, 0] = torch.rand(k.shape[0], H, generator=g)
        q, k = q.reshape(-1, d), k.reshape(-1, d)
    elif name == "v_1e3":                    # |V| ~ 1e3 with alternating signs: the context cancels to a small fraction of it
        v = v + 1000.0 * (1 - 2 * (torch.arange(B * tk) % 2)).float()[:, None]
    return q, k, v


def _f64_check(B, H, tq, tk, lens, mode, regime, seed):
    abi, lib = _lib()
    q, k, v = _regime(regime, B, H, tq, tk, lens, seed)
    npl = QPL[mode]
    qp, kp = _split(q, npl), _split(k, npl)
    got = _planes_attention(abi, lib, qp, kp, _vt(v, B, tk, (tk + 63) // 64 * 64, npl), lens, B, H, tq, tk, mode)
    vr = _split(v, npl).double().sum(0)
    ref, pmax, wrong = _ref64(qp.double().sum(0), kp.double().sum(0), vr, lens, B, H, tq, tk, qh=qp[0], kh=kp[0])
    assert not torch.isnan(got).any()
    err = float((got.double() - ref).abs().max() / vr.abs().max())
    bar = (F64_TOL_LARGE_S if regime in LARGE_S else F64_TOL)[mode]
    print("attn f64 %s %-8s B=%d H=%d tq=%d tk=%d lens=%s: err %.2e (bar %.0e), max p' %.1f, hi.hi arg-max misses %d"
          % (mode, regime, B, H, tq, tk, lens, err, bar, pmax, wrong))
    assert err <= bar
    return pmax, wrong


@pytest.mark.parametrize("mode", ["fp16", "fp16x3"])
@pytest.mark.parametrize("B,H,tq,tk,lens", F64_SHAPES)
def test_plane_attention_vs_float64_shapes(B, H, tq, tk, lens, mode):
    pmax, _ = _f64_check(B, H, tq, tk, lens, mode, "unit", seed=tq * 7 + tk)
    assert pmax < 65504.0


@pytest.mark.parametrize("mode", ["fp16", "fp16x3"])
@pytest.mark.parametrize("shape", REGIME_SHAPES, ids=["tq129_tk500", "tq4_tk4100"])
@pytest.mark.parametrize("regime", REGIMES)
def test_plane_attention_vs_float64_regimes(regime, shape, mode):
    B, H, tq, tk, lens = shape
    pmax, wrong = _f64_check(B, H, tq, tk, lens, mode, regime, seed=len(regime) * 31 + tk)
    # p' = 2^10 exp(s - m~) must stay inside fp16 (65504): the pass-A maximum m~ (hi . hi only) lags the exact one by ~2^-11 |s|
    assert pmax < 65504.0
    if regime == "near_tie" and mode == "fp16x3":
        assert wrong > 0, "the construction did not make pass A pick a different key"


# ============================================================================================ 7. whole attention block vs float64
BLOCKS = ["enc_self", "dec_cross_n1", "dec_cross_n200", "hotword_shared"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("arr", BLOCKS)
def test_attention_block_vs_float64(arr, mode):
    """LayerNorm-output planes (fa_split_rows) -> fa_linear_attn_sinks -> fa_attention_tc_planes (context planes) -> fa_linear_planes
    out-projection + bias, as the encoder (one QKV GEMM, ragged lengths, T % 4 != 0), the decoder's cross-attention (q from N tokens,
    k / v from T frames) and the contextual decoder (hotword memory with kv_shared) chain them, against float64 of
    linear_out(softmax(q k^T / sqrt(d_k), key mask) v) on the same fp32 inputs and weights."""
    abi, lib = _lib()
    gm, npl, qpl = abi.GEMM_MODES[mode], NPL[mode], QPL[mode]
    D, H = 512, 4
    g = torch.Generator().manual_seed(BLOCKS.index(arr) + 100)
    if arr == "enc_self":
        B, N, T, lens, shared = 3, 99, 99, [99, 50, 1], 0
    elif arr == "hotword_shared":
        B, N, T, lens, shared = 3, 9, 17, [17, 17, 17], 1
    else:
        B, N, T, lens, shared = 2, (1 if arr == "dec_cross_n1" else 200), 150, [150, 77], 0
    kb = 1 if shared else B
    tkp = (T + 63) // 64 * 64
    qp = torch.full((2, B * N, D), NAN, dtype=F16, device=DEV)
    kp = torch.full((2, kb * T, D), NAN, dtype=F16, device=DEV)
    vt = torch.full((2, kb * D, tkp), NAN, dtype=F16, device=DEV)
    out_lin = _Linear(abi, lib, D, D, seed=9)
    if arr == "enc_self":
        qkv = _Linear(abi, lib, 3 * D, D, seed=8)
        x = torch.randn(B * T, D, generator=g)
        ap = _a_planes(abi, lib, x.to(DEV), npl, D)
        abi.check(lib.fa_linear_attn_sinks(ap.data_ptr(), B * T, C.byref(qkv.lin), 0, D, 2 * D, D, T, tkp, QSCALE, qp.data_ptr(),
                                           kp.data_ptr(), vt.data_ptr(), None, 0, gm, _st()), "qkv sinks")
        wq, bq, wk, bk, wv, bv = qkv.w[:D], qkv.b[:D], qkv.w[D:2 * D], qkv.b[D:2 * D], qkv.w[2 * D:], qkv.b[2 * D:]
        xq = xkv = x
    else:
        ql, kvl = _Linear(abi, lib, D, D, seed=10), _Linear(abi, lib, 2 * D, D, seed=11)
        xq, xkv = torch.randn(B * N, D, generator=g), torch.randn(kb * T, D, generator=g)
        aq, akv = _a_planes(abi, lib, xq.to(DEV), npl, D), _a_planes(abi, lib, xkv.to(DEV), npl, D)
        abi.check(lib.fa_linear_attn_sinks(aq.data_ptr(), B * N, C.byref(ql.lin), 0, -1, -1, D, N, 64, QSCALE, qp.data_ptr(), None, None,
                                           None, 0, gm, _st()), "q sink")
        abi.check(lib.fa_linear_attn_sinks(akv.data_ptr(), kb * T, C.byref(kvl.lin), -1, 0, D, D, T, tkp, 1.0, None, kp.data_ptr(),
                                           vt.data_ptr(), None, 0, gm, _st()), "kv sinks")
        wq, bq, wk, bk, wv, bv = ql.w, ql.b, kvl.w[:D], kvl.b[:D], kvl.w[D:], kvl.b[D:]
    ctxp = torch.full((3, B * N, D), NAN, dtype=F16, device=DEV)
    ld = torch.tensor(lens, dtype=torch.int32, device=DEV)
    abi.check(lib.fa_attention_tc_planes(qp.data_ptr(), kp.data_ptr(), vt.data_ptr(), ld.data_ptr(), B, H, N, T, None, 0, ctxp.data_ptr(), D,
                                         npl, gm, shared, _st()), "attention")
    y = torch.full((B * N, D), NAN, device=DEV)
    abi.check(lib.fa_linear_planes(ctxp.data_ptr(), B * N, C.byref(out_lin.lin), 0, None, 0, None, 0, y.data_ptr(), D, gm, _st()), "out")
    torch.cuda.synchronize()
    f = lambda x_, w_, b_: x_.double() @ w_.double().t() + b_.double()
    ctx, _, _ = _ref64(f(xq, wq, bq) * 128 ** -0.5, f(xkv, wk, bk), f(xkv, wv, bv), lens, B, H, N, T, kv_shared=bool(shared))
    ref = f(ctx, out_lin.w, out_lin.b)
    y = y.cpu()
    assert not torch.isnan(y).any()
    err = rel_err(y.numpy(), ref.numpy())
    print("attention block %s %s: rel err %.2e (bar %.0e)" % (arr, mode, err, BLOCK_TOL[mode]))
    assert err <= BLOCK_TOL[mode]


# ============================================================================================ 8. fp32 kernels vs float64
F32_CASES = [
    # head_dim, heads, batch, tq, tk, key_lens
    (128, 4, 3, 130, 130, [130, 1, 65]),
    (128, 4, 3, 500, 500, [500, 83, 600]),
    (128, 4, 2, 4, 4100, [4100, 64]),
    (128, 1, 2, 1, 1, [1, 0]),
    (32, 8, 3, 37, 63, [63, 64, 0]),          # CT-Transformer heads: 8 x 32 = 256
    (32, 8, 1, 129, 4100, [4100]),
    (64, 4, 3, 65, 500, [500, 65, 1]),
    (96, 2, 2, 128, 200, [200, 129]),
]


@pytest.mark.parametrize("kv_shared", [0, 1])
@pytest.mark.parametrize("hd,H,B,tq,tk,lens", F32_CASES)
def test_f32_attention_vs_float64(hd, H, B, tq, tk, lens, kv_shared):
    """attention_f32_kernel (head_dim 128) and attention_small_kernel (32, 64, 96) on strided views of a QKV buffer."""
    abi, lib = _lib()
    g = torch.Generator().manual_seed(hd * 10 + tk)
    kb = 1 if kv_shared else B
    q, k, v = torch.randn(B * tq, H * hd, generator=g), torch.randn(kb * tk, H * hd, generator=g), torch.randn(kb * tk, H * hd, generator=g)
    got = _f32_run(abi, lib, q, k, v, lens, B, H, hd, tq, tk, kv_shared)
    qs = q * torch.tensor(float(np.float32(1.0 / math.sqrt(hd))))      # __fmul_rn(q, (float)(1 / sqrt(hd)))
    ref, _, _ = _ref64(qs, k, v, lens, B, H, tq, tk, hd=hd, kv_shared=bool(kv_shared))
    assert not torch.isnan(got).any()
    err = float((got.double() - ref).abs().max() / v.abs().max())
    print("f32 attention hd=%d H=%d B=%d tq=%d tk=%d lens=%s shared=%d: err %.2e (bar %.0e)" % (hd, H, B, tq, tk, lens, kv_shared, err, F32_TOL))
    assert err <= F32_TOL


# ============================================================================================ 9. status codes
def test_attention_status_codes():
    """The cases that must answer with a status code rather than a wrong result; a rejected call writes nothing."""
    abi, lib = _lib()
    B, H, tq, tk = 1, 1, 4, 8
    q, k, v = _rand_qkv(B, H, tq, tk, seed=1)
    qp, kp, vt = _split(q, 2).to(DEV), _split(k, 2).to(DEV), _vt(v, B, tk, 64, 2).to(DEV)
    ld = torch.tensor([tk], dtype=torch.int32, device=DEV)
    pl = torch.full((4, tq, HD), NAN, dtype=F16, device=DEV)

    def planes(mode, opl):
        return lib.fa_attention_tc_planes(qp.data_ptr(), kp.data_ptr(), vt.data_ptr(), ld.data_ptr(), B, H, tq, tk, None, 0, pl.data_ptr(), HD,
                                          opl, abi.GEMM_MODES[mode], 0, _st())
    assert planes("fp16", 2) == -4 and planes("fp16", 3) == -4 and planes("fp16x3", 1) == -4
    assert planes("fp16x3", 0) == -1 and planes("fp16x3", 4) == -1 and planes("fp16", 0) == -1 and planes("fp16", 4) == -1
    torch.cuda.synchronize()
    assert torch.isnan(pl.cpu()).all()
    assert planes("fp16", 1) == 0 and planes("fp16x3", 2) == 0 and planes("fp16x6", 3) == 0

    # fa_attention_tc: no fp32 SIMT mode; the workspace query is exact
    qd, kd, vd = q.to(DEV), k.to(DEV), v.to(DEV)
    ctx = torch.full((tq, HD), NAN, device=DEV)
    for mode in ("fp16", "fp16x3"):
        gm = abi.GEMM_MODES[mode]
        ctx.fill_(NAN)
        need = lib.fa_attention_tc_workspace_bytes(B, H, tq, tk, gm)
        ws = torch.empty(need, dtype=torch.uint8, device=DEV)
        call = lambda n, m=gm: lib.fa_attention_tc(qd.data_ptr(), HD, kd.data_ptr(), HD, vd.data_ptr(), HD, ld.data_ptr(), B, H, tq, tk,
                                                   ctx.data_ptr(), HD, m, ws.data_ptr(), n, _st())
        assert call(need - 1) == -3
        torch.cuda.synchronize()
        assert torch.isnan(ctx.cpu()).all()
        assert call(need) == 0
        assert call(need, abi.GEMM_F32_SIMT) == -1

    # attention_small_kernel keeps 4 * tk scores in 160 KB of shared memory
    def small(tk_):
        g = torch.Generator().manual_seed(2)
        qq, kk = torch.randn(1, 64, generator=g).to(DEV), torch.randn(tk_, 64, generator=g).to(DEV)
        out = torch.full((1, 64), NAN, device=DEV)
        lens = torch.tensor([tk_], dtype=torch.int32, device=DEV)
        st = lib.fa_attention_f32_ex(qq.data_ptr(), 64, kk.data_ptr(), 64, kk.data_ptr(), 64, lens.data_ptr(), 1, 1, 64, 1, tk_, out.data_ptr(),
                                     64, 0, _st())
        torch.cuda.synchronize()
        return st, out.cpu()
    st, out = small(10241)
    assert st == -4 and torch.isnan(out).all()
    st, out = small(10240)
    assert st == 0 and not torch.isnan(out).any()

    # fa_linear_attn_sinks argument checks
    L = _Linear(abi, lib, 1536, 512, seed=3)
    M, T = 12, 4
    ap = _a_planes(abi, lib, torch.randn(M, 512).to(DEV), 2, 512)
    sq = torch.full((2, M, 512), NAN, dtype=F16, device=DEV)
    sk = torch.full((2, M, 512), NAN, dtype=F16, device=DEV)
    sv = torch.full((2, 3 * 512, 64), NAN, dtype=F16, device=DEV)

    def sinks(rows=M, q0=0, k0=512, v0=1024, t_rows=T, t_pad=64, mode="fp16x3", width=512):
        return lib.fa_linear_attn_sinks(ap.data_ptr(), rows, C.byref(L.lin), q0, k0, v0, width, t_rows, t_pad, QSCALE, sq.data_ptr(),
                                        sk.data_ptr(), sv.data_ptr(), None, 0, abi.GEMM_MODES[mode], _st())
    assert sinks(t_rows=5) == -1                      # rows % t_rows != 0
    assert sinks(t_pad=3) == -1                       # t_pad < t_rows
    assert sinks(k0=256) == -1                        # q and k overlap
    assert sinks(v0=1280) == -1                       # v leaves [0, N)
    assert sinks(q0=8, k0=-1, v0=-1) == -1            # not a 16-column chunk boundary
    assert sinks(q0=-1, k0=-1, v0=-1) == -1           # nothing to write
    assert sinks(width=48) == -1
    assert sinks(mode="fp32") == -1
    torch.cuda.synchronize()
    assert torch.isnan(sq.cpu()).all() and torch.isnan(sk.cpu()).all() and torch.isnan(sv.cpu()).all()
    assert sinks() == 0 and sinks(v0=-1) == 0
