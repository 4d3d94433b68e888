"""GPU (-m gpu): kernel-level parity of the tensor-core GEMM, its operand splits, the conv-view GEMM and LayerNorm's plane output.

Every tensor-core stage of every model runs through gemm_tc_kernel, and its A operand comes from a split pass (fa_split_rows),
from another GEMM's plane epilogue or from LayerNorm's fused plane epilogue; the weights are split once (fa_split_planes).

Two kinds of checks.
  * Bit-exact, no tolerance (every output buffer starts as NaN, so a write outside the output region shows).
      - The splits equal a CPU emulation of cvt.rn.satfinite.f16x2.f32: hi = RN(x) saturated to +-65504, then RN of each fp32
        residual.  Scalar column tails, pad columns, pitched and overlapping rows, fp16-subnormal inputs, +-0, saturation.
      - Exact-integer GEMM: independent random integers in {-3..3} in EVERY A and W plane.  Each product and partial sum is an
        integer below 2^17, so the tensor cores' truncation never acts and the accumulator equals sum over the mode's terms of
        A_p W_q^T exactly (float64 matmul).  A dropped, duplicated or mis-paired term, a stale or foreign k-block or a wrong tile
        mapping changes the result, however small its share of the sum.  The epilogue is emulated exactly: one rounding of
        acc * acc_scale + b (fmaf), ReLU, then each residual as a float32 add; plane outputs are the split of that value.
      - The conv-view GEMM (fa_linear_planes_view) equals fa_linear on the same rows read with ldx = a_ld < in_f, where the split
        pass materialises the im2col planes.
      - LayerNorm's planes are the split of its own fp32 output, pad columns are zero, plane-only and in-place calls agree.
  * Against float64, with a bar per element instead of a max-normalised error.
      - GEMM on Gaussian operands at the models' scales: |y - y64| <= tau * sum_k |x_k w_k| + ulp(y) / 2, also for the conv view
        against a float64 Conv1d.
      - LayerNorm per row, including rows whose mean is far larger than their spread; the PE prologue against sin / cos in float64.
Each float64 bar was measured on an H100 80GB HBM3 (400 W power limit); the comment beside each constant gives the worst case.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
NAN = float("nan")
F16 = torch.float16
NPL = {"fp16": 1, "fp16x3": 2, "fp16x6": 3}             # A-operand planes per mode
MODES = list(NPL)
TERMS = {"fp16": [(0, 0)], "fp16x3": [(0, 0), (0, 1), (1, 0)], "fp16x6": [(0, 0), (0, 1), (1, 0), (1, 1), (0, 2), (2, 0)]}
BN = {"fp16": 128, "fp16x3": 128, "fp16x6": 64}         # output tile width
F16_MAX = 65504.0
EPS32 = 2.0 ** -24                                      # unit roundoff of fp32

# Float64 bars, each measured on an H100 80GB HBM3 (400 W power limit) and kept at least 3x above the worst case seen.
# GEMM, tau per mode over K = 512 and 2048 (x ~ N(0, 1), W ~ N(0, 1/K), the models' weight scale).  Worst: 9.4e-5 (x1, K = 512),
# 7.3e-7 (x3 and x6 alike, K = 2048).  Split into its two floors (K = 512): the mode's terms on the planes, in float64, are off by
# 1.4e-7 (x3) and 1.35e-7 (x6) - at this weight scale the mid plane is fp16-subnormal and the third is almost all zero, so x6 gains
# nothing - and the kernel against those terms by 4.5e-7 (fp32 accumulation with truncation; 7.1e-7 at K = 2048).
TAU = {"fp16": 3e-4, "fp16x3": 2.5e-6, "fp16x6": 2.5e-6}
# The same with W scaled by 2^8 (mid plane normal): the planes' floor drops to 2.6e-8 (x3) and 4.1e-9 (x6), and what is left is the
# accumulator's own rounding.  Worst: 9.4e-5 (x1: scaling by 2^8 is exact), 4.8e-7 (x3 and x6 alike).
TAU_W256 = {"fp16": 3e-4, "fp16x3": 1.5e-6, "fp16x6": 1.5e-6}
# LayerNorm: |y - y64| <= LN_C * eps32 * (|g| (1 + |z| + |mean| / std) + |b|).  The fp32 two-pass mean is off by ~eps * |mean|,
# which shifts every normalised value by that over std: the |mean| / std term.
# Worst: 2.9 (n = 2048).
LN_C = 9.0
# PE prologue: |emb - fl32(fl32(x * xscale) + pe64)| <= ulp + PE_K * 2^-24: both sides round once, and CUDA sinf / cosf are not
# correctly rounded (arguments up to 4100 rad here).  Worst: 1.38 (n = 512).
PE_K = 4.5


@pytest.fixture(scope="module")
def lib():
    from funasr_b200 import _abi
    return _abi, _abi.load()


@pytest.fixture(scope="module")
def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _st():
    return torch.cuda.current_stream().cuda_stream


def _split(x, n):
    """fp16 planes [n, *x.shape] of fp32 x as cvt.rn.satfinite.f16x2.f32 makes them: hi = RN(x) saturated to +-65504 (torch's
    .half() would give inf), then the same for each fp32 residual."""
    r = x.float().clone()
    out = []
    for _ in range(n):
        h = r.clamp(-F16_MAX, F16_MAX).half()
        out.append(h)
        r = r - h.float()
    return torch.stack(out)


def _same(got, want, what):
    """Equal values (so -0 == 0), no NaN on either side."""
    g, w = got.float(), want.float()
    bad = ~(g == w)
    n = int(bad.sum())
    if n:
        idx = bad.nonzero()[0].tolist()
        raise AssertionError("%s: %d of %d differ, first at %s: got %r want %r" % (what, n, bad.numel(), idx, float(g[tuple(idx)]),
                                                                                   float(w[tuple(idx)])))


def _same_bits(got, want, what):
    g, w = got.contiguous().view(torch.int16), want.contiguous().view(torch.int16)
    bad = g != w
    n = int(bad.sum())
    if n:
        idx = bad.nonzero()[0].tolist()
        raise AssertionError("%s: %d of %d differ, first at %s: got %r want %r" % (what, n, bad.numel(), idx,
                                                                                   float(got[tuple(idx)]), float(want[tuple(idx)])))


def _all_nan(t, what):
    assert bool(torch.isnan(t.float()).all()), "%s: written outside the output (%d non-NaN)" % (what, int((~torch.isnan(t.float())).sum()))


def _lin(abi, w_planes, b, out_f, in_f, in_pad, w=None):
    return abi.FaLinear(w.data_ptr() if w is not None else w_planes.data_ptr(), b.data_ptr() if b is not None else None,
                        w_planes.data_ptr(), out_f, in_f, in_pad, 0)


def _acc_scale(kp, mode):
    """rz_comp_scale of gemm_tc.cu in float32 arithmetic (1 with FA_RZ_COMP=0)."""
    if os.environ.get("FA_RZ_COMP", "")[:1] == "0":
        return 1.0
    c = np.float32(5.3e-8) if len(TERMS[mode]) >= 3 else np.float32(3.4e-8)
    return float(np.float32(1) + np.float32(kp // 16) * c)


def _epilogue(acc, s, b, relu, r1=None, r2=None):
    """fp32 value the epilogue stores: fl32(acc * s + b) rounded ONCE (fmaf), ReLU, + r1, + r2 (float32 adds).  acc is an exact
    integer below 2^17, so acc * s is exact in float64; the sum with b is checked to be exact too (TwoSum error 0)."""
    assert float(acc.abs().max()) < 2.0 ** 17 and bool((acc == acc.round()).all())
    p = acc * s
    b64 = b.double()
    t = p + b64
    bb = t - p
    assert bool((((p - (t - bb)) + (b64 - bb)) == 0).all()), "acc * s + b is not exact in float64"
    v = t.float()
    if relu:
        v = torch.clamp_min(v, 0.0)
    if r1 is not None:
        v = v + r1
    if r2 is not None:
        v = v + r2
    return v


def _int_planes(g, n, rows, cols):
    return torch.randint(-3, 4, (n, rows, cols), generator=g, device=DEV, dtype=torch.int32).to(F16)


def _bias(g, n):
    """fp32 bias on a 2^-10 grid in (-8, 8): acc * s + b stays exact in float64."""
    return (torch.randn(n, generator=g, device=DEV) * 1024 * 3).clamp(-8000, 8000).round() / 1024


# ============================================================================================ 1. operand splits
def _split_source(rows, ldx, cols, seed):
    """Flat fp32 source covering rows of ldx (or, for ldx < cols, overlapping rows): Gaussian values at several scales mixed with
    +-0, fp16-subnormal magnitudes, fp32 subnormals and magnitudes in [65504, 2 * 65504] (saturation)."""
    g = torch.Generator().manual_seed(seed)
    n = (rows - 1) * ldx + max(cols, ldx)
    kind = torch.randint(0, 8, (n,), generator=g)
    x = torch.randn(n, generator=g)
    sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
    x = torch.where(kind == 1, x / math.sqrt(512), x)
    x = torch.where(kind == 2, x * 1e-3, x)
    x = torch.where(kind == 3, sign * torch.rand(n, generator=g) * 6.1e-5, x)                 # fp16 subnormal range
    x = torch.where(kind == 4, sign * (F16_MAX + torch.rand(n, generator=g) * F16_MAX), x)    # saturates
    x = torch.where(kind == 5, sign * 0.0, x)                                                # +-0
    x = torch.where(kind == 6, sign * 1e-40, x)                                              # fp32 subnormal
    x[:4] = torch.tensor([65519.0, 65520.0, -65520.0, 2 * F16_MAX])                          # around the overflow boundary
    return x


def _rows_of(flat, rows, ldx, cols):
    return torch.stack([flat[r * ldx:r * ldx + cols] for r in range(rows)])


SPLIT_ROWS_CASES = [
    # (rows, cols, cols_pad, ldx)
    (37, 130, 192, 136),     # cols % 4 = 2: scalar tail; pad columns; ldx > cols
    (9, 1536, 1536, 512),    # ldx < cols: the overlapping rows of the CIF conv's im2col
    (64, 512, 512, 512),     # dense
    (5, 3, 8, 4),            # scalar tail only
    (3, 560, 576, 560),      # LayerNorm-sized rows padded to the next 64
]


@pytest.mark.parametrize("npl", [1, 2, 3])
@pytest.mark.parametrize("case", SPLIT_ROWS_CASES, ids=["r%d_c%d_p%d_ld%d" % c for c in SPLIT_ROWS_CASES])
def test_split_rows_bit_exact(lib, case, npl):
    abi, L = lib
    rows, cols, cols_pad, ldx = case
    flat = _split_source(rows, ldx, cols, seed=rows * cols + ldx)
    out = torch.full((3, rows, cols_pad), NAN, dtype=F16, device=DEV)
    assert L.fa_split_rows(flat.to(DEV).data_ptr(), ldx, rows, cols, cols_pad, npl, out.data_ptr(), _st()) == 0
    torch.cuda.synchronize()
    got = out.cpu()
    want = _split(_rows_of(flat, rows, ldx, cols), npl)
    _same_bits(got[:npl, :, :cols], want, "split_rows planes")
    assert bool((got[:npl, :, cols:].float() == 0).all()), "pad columns not zero"
    _all_nan(got[npl:], "planes beyond nplanes")


def test_split_planes_bit_exact(lib):
    abi, L = lib
    for rows, cols, cols_pad, ld in ((33, 130, 192, 136), (7, 5, 64, 5), (16, 512, 512, 512)):
        flat = _split_source(rows, ld, cols, seed=cols + ld)
        out = torch.full((4, rows, cols_pad), NAN, dtype=F16, device=DEV)
        assert L.fa_split_planes(flat.to(DEV).data_ptr(), ld, rows, cols, cols_pad, out.data_ptr(), _st()) == 0
        torch.cuda.synchronize()
        got = out.cpu()
        _same_bits(got[:3, :, :cols], _split(_rows_of(flat, rows, ld, cols), 3), "split_planes (%d, %d)" % (rows, cols))
        assert bool((got[:3, :, cols:].float() == 0).all())
        _all_nan(got[3:], "beyond the three planes")


def test_split_rows_status(lib):
    abi, L = lib
    x = torch.zeros(64 * 64 + 8, device=DEV)
    out = torch.full((3, 64, 64), NAN, dtype=F16, device=DEV)
    assert L.fa_split_rows(x.data_ptr(), 62, 64, 60, 64, 2, out.data_ptr(), _st()) == -4          # ldx % 4
    assert L.fa_split_rows(x.data_ptr() + 4, 64, 64, 64, 64, 2, out.data_ptr(), _st()) == -4      # x not 16-byte aligned
    assert L.fa_split_rows(x.data_ptr(), 64, 64, 60, 62, 2, out.data_ptr(), _st()) == -4          # cols_pad % 4
    assert L.fa_split_rows(x.data_ptr(), 64, 64, 64, 64, 4, out.data_ptr(), _st()) == -1          # nplanes
    assert L.fa_split_rows(x.data_ptr(), 64, 0, 64, 64, 2, out.data_ptr(), _st()) == 0            # empty
    torch.cuda.synchronize()
    _all_nan(out, "refused / empty split")


# ============================================================================================ 2. exact-integer GEMM
# (id, M as a function of the SM count, N (None: one column tile of the mode's width), K_pad)
INT_CASES = [
    ("1tile_m100_k64", lambda n: 100, None, 64),                 # one tile: the second consumer idle; one k-block
    ("2tiles_m1_k128", lambda n: 129, None, 128),                # M % 128 = 1
    ("nsm-1_m33_k320", lambda n: (n - 1) * 128 - 95, None, 320),  # 5 k-blocks: tiles start mid-ring at changing phases
    ("nsm_m32_k448", lambda n: n * 128 - 96, None, 448),
    ("nsm+1_m127_k576", lambda n: (n + 1) * 128 - 1, None, 576),
    ("2nsm+1_m31_k320", lambda n: (2 * n + 1) * 128 - 97, None, 320),
    ("3nsm_m96_k2048", lambda n: 3 * n * 128 - 32, None, 2048),
    ("n2080_k128", lambda n: 300, 2080, 128),                    # N % BN != 0, N % 16 == 0 (plane outputs too)
    ("n1000_k64", lambda n: 257, 1000, 64),                      # N % 16 != 0: fp32 only
    ("n8404_k576", lambda n: 130, 8404, 576),
    ("n25055_k512", lambda n: 64, 25055, 512),
    ("m32000_n512_k2048", lambda n: 32000, 512, 2048),           # FFN w_2
    ("m32000_n1536_k512", lambda n: 32000, 1536, 512),           # QKV
]


def _acc(A, W, mode):
    acc = None
    for p, q in TERMS[mode]:
        t = A[p].double() @ W[q].double().T
        acc = t if acc is None else acc + t
    return acc


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", INT_CASES, ids=[c[0] for c in INT_CASES])
def test_int_gemm_bit_exact(lib, n_sm, case, mode):
    abi, L = lib
    name, mfn, N, Kp = case
    M = mfn(n_sm)
    N = N or BN[mode]
    npl = NPL[mode]
    g = torch.Generator(device=DEV).manual_seed(M + N + Kp)
    A = _int_planes(g, npl, M, Kp)
    W = _int_planes(g, 3, N, Kp)
    b = _bias(g, N)
    lin = _lin(abi, W, b, N, Kp, Kp)
    acc = _acc(A, W, mode)
    s = _acc_scale(Kp, mode)
    gm = abi.GEMM_MODES[mode]
    ldr = (N + 3) // 4 * 4 + 8                                  # residual pitches are multiples of 4 floats
    r1 = torch.randn(M, ldr, generator=g, device=DEV)
    r2 = torch.randn(M, ldr, generator=g, device=DEV)

    # fp32 epilogues: (relu, residuals, ldy); ldy = N + 1 takes the scalar interior stores, N + 4 leaves pad columns
    for relu, nres, ldy in ((0, 0, N), (1, 1, N + 4), (0, 2, N + 1), (1, 2, N)):
        y = torch.full((M, ldy), NAN, device=DEV)
        st = L.fa_linear_planes(A.data_ptr(), M, C.byref(lin), relu, r1.data_ptr() if nres >= 1 else None, ldr,
                                r2.data_ptr() if nres >= 2 else None, ldr, y.data_ptr(), ldy, gm, _st())
        assert st == 0, st
        want = _epilogue(acc, s, b, relu, r1[:, :N] if nres >= 1 else None, r2[:, :N] if nres >= 2 else None)
        torch.cuda.synchronize()
        _same(y[:, :N], want, "%s %s fp32 relu=%d residuals=%d ldy=%d" % (name, mode, relu, nres, ldy))
        if ldy > N:
            _all_nan(y[:, N:], "pad columns of y")
    if N % 32:
        return
    # plane epilogue (FFN w_1 with ReLU, and without)
    for relu, ldo in ((1, N + 8), (0, N)):
        out = torch.full((3, M, ldo), NAN, dtype=F16, device=DEV)
        assert L.fa_linear_planes_to_planes(A.data_ptr(), M, C.byref(lin), relu, out.data_ptr(), ldo, gm, _st()) == 0
        v = _epilogue(acc, s, b, relu)
        assert float(v.abs().max()) < F16_MAX
        torch.cuda.synchronize()
        _same(out[:npl, :, :N], _split(v, npl), "%s %s planes relu=%d" % (name, mode, relu))
        if ldo > N:
            _all_nan(out[:npl, :, N:], "pad columns of the output planes")
        _all_nan(out[npl:], "planes beyond the mode's count")


LINEAR_CASES = [
    # (M, N, in_f, in_pad, ldx): split pass + GEMM through fa_linear
    (300, 2080, 560, 576, 600),     # K padding 560 -> 576 with non-zero W pad columns
    (133 * 128 + 5, 512, 512, 512, 516),
]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", LINEAR_CASES, ids=["m%d_n%d_k%d" % c[:3] for c in LINEAR_CASES])
def test_int_linear_split_then_gemm_bit_exact(lib, case, mode):
    abi, L = lib
    M, N, in_f, in_pad, ldx = case
    g = torch.Generator(device=DEV).manual_seed(M + N)
    x = torch.full((M, ldx), NAN, device=DEV)                   # columns beyond in_f must not be read
    x[:, :in_f] = torch.randint(-3, 4, (M, in_f), generator=g, device=DEV).float()
    W = _int_planes(g, 3, N, in_pad)                            # pad columns non-zero: the split must zero A's
    b = _bias(g, N)
    r1 = torch.randn(M, N, generator=g, device=DEV)
    lin = _lin(abi, W, b, N, in_f, in_pad)
    ws = torch.empty(L.fa_linear_workspace_bytes(M, in_f, abi.GEMM_MODES[mode]), dtype=torch.uint8, device=DEV)
    y = torch.full((M, N), NAN, device=DEV)
    assert L.fa_linear(x.data_ptr(), ldx, M, C.byref(lin), 1, r1.data_ptr(), N, None, 0, y.data_ptr(), N, abi.GEMM_MODES[mode],
                       ws.data_ptr(), ws.numel(), _st()) == 0
    xa = torch.zeros(1, M, in_pad, device=DEV, dtype=F16)
    xa[0, :, :in_f] = x[:, :in_f].half()
    acc = None
    for p, q in TERMS[mode]:
        if p == 0:                                              # integer x: the lower A planes are zero
            t = xa[0].double() @ W[q].double().T
            acc = t if acc is None else acc + t
    want = _epilogue(acc, _acc_scale(in_pad, mode), b, 1, r1)
    torch.cuda.synchronize()
    _same(y, want, "fa_linear %s" % mode)


SIMT_CASES = [(300, 200, 16, 20), (129, 1000, 48, 52), (1000, 384, 512, 512), (64, 8404, 64, 64)]


@pytest.mark.parametrize("case", SIMT_CASES, ids=["m%d_n%d_k%d" % c[:3] for c in SIMT_CASES])
def test_int_linear_simt_bit_exact(lib, case):
    abi, L = lib
    M, N, K, ldx = case
    g = torch.Generator(device=DEV).manual_seed(M * N + K)
    x = torch.full((M, ldx), NAN, device=DEV)
    x[:, :K] = torch.randint(-3, 4, (M, K), generator=g, device=DEV).float()
    w = torch.randint(-3, 4, (N, K), generator=g, device=DEV).float()
    b = _bias(g, N)
    r1 = torch.randn(M, N, generator=g, device=DEV)
    r2 = torch.randn(M, N, generator=g, device=DEV)
    lin = abi.FaLinear(w.data_ptr(), b.data_ptr(), None, N, K, K, 0)
    acc = (x[:, :K].double() @ w.double().T).float()            # exact integers
    for relu, nres in ((0, 0), (1, 1), (1, 2)):
        y = torch.full((M, N + 3), NAN, device=DEV)
        assert L.fa_linear(x.data_ptr(), ldx, M, C.byref(lin), relu, r1.data_ptr() if nres >= 1 else None, N,
                           r2.data_ptr() if nres >= 2 else None, N, y.data_ptr(), N + 3, abi.GEMM_F32_SIMT, None, 0, _st()) == 0
        v = acc + b
        if relu:
            v = torch.clamp_min(v, 0.0)
        if nres >= 1:
            v = v + r1
        if nres >= 2:
            v = v + r2
        torch.cuda.synchronize()
        _same(y[:, :N], v, "simt relu=%d residuals=%d" % (relu, nres))
        _all_nan(y[:, N:], "pad columns")


def test_gemm_empty_and_status(lib):
    """rows = 0 writes nothing; every refused call returns before a tensor map is made or a kernel launched."""
    abi, L = lib
    M, N, Kp = 256, 256, 128
    g = torch.Generator(device=DEV).manual_seed(1)
    A = _int_planes(g, 3, M, Kp)
    W = _int_planes(g, 3, N, Kp)
    b = _bias(g, N + 8)
    r = torch.zeros(M, N + 8, device=DEV)
    y = torch.full((M, N + 8), NAN, device=DEV)
    out = torch.full((3, M, N + 8), NAN, dtype=F16, device=DEV)
    lin = _lin(abi, W, b, N, Kp, Kp)
    x3 = abi.GEMM_F16X3
    ws = torch.empty(L.fa_linear_workspace_bytes(M, Kp, x3), dtype=torch.uint8, device=DEV)
    xf = torch.zeros(M, Kp, device=DEV)
    # empty
    assert L.fa_linear_planes(A.data_ptr(), 0, C.byref(lin), 0, None, 0, None, 0, y.data_ptr(), N, x3, _st()) == 0
    assert L.fa_linear_planes_to_planes(A.data_ptr(), 0, C.byref(lin), 0, out.data_ptr(), N, x3, _st()) == 0
    assert L.fa_linear_planes_view(A.data_ptr(), 0, 64, 2, C.byref(lin), 0, y.data_ptr(), N, x3, _st()) == 0
    for mode in (abi.GEMM_F32_SIMT, x3):
        assert L.fa_linear(xf.data_ptr(), Kp, 0, C.byref(lin), 0, None, 0, None, 0, y.data_ptr(), N, mode, ws.data_ptr(), ws.numel(),
                           _st()) == 0
    # alignment the epilogue's vector accesses assume -> FA_ERR_UNSUPPORTED
    bad_b = _lin(abi, W, None, N, Kp, Kp)
    bad_b.b = b.data_ptr() + 4
    assert L.fa_linear_planes(A.data_ptr(), M, C.byref(bad_b), 0, None, 0, None, 0, y.data_ptr(), N, x3, _st()) == -4
    assert L.fa_linear_planes(A.data_ptr(), M, C.byref(lin), 0, r.data_ptr() + 4, N + 8, None, 0, y.data_ptr(), N, x3, _st()) == -4
    assert L.fa_linear_planes(A.data_ptr(), M, C.byref(lin), 0, r.data_ptr(), N + 8, r.data_ptr() + 4, N + 8, y.data_ptr(), N, x3,
                              _st()) == -4
    assert L.fa_linear_planes(A.data_ptr(), M, C.byref(lin), 0, r.data_ptr(), N + 2, None, 0, y.data_ptr(), N, x3, _st()) == -4
    assert L.fa_linear_planes(A.data_ptr(), M, C.byref(lin), 0, None, 0, None, 0, y.data_ptr() + 4, N, x3, _st()) == -4
    assert L.fa_linear_planes_to_planes(A.data_ptr(), M, C.byref(lin), 0, out.data_ptr() + 2, N, x3, _st()) == -4
    assert L.fa_linear_planes_to_planes(A.data_ptr(), M, C.byref(lin), 0, out.data_ptr(), N + 2, x3, _st()) == -4
    # pitches below N -> FA_ERR_ARG
    assert L.fa_linear_planes(A.data_ptr(), M, C.byref(lin), 0, None, 0, None, 0, y.data_ptr(), N - 4, x3, _st()) == -1
    assert L.fa_linear_planes(A.data_ptr(), M, C.byref(lin), 0, r.data_ptr(), N - 4, None, 0, y.data_ptr(), N, x3, _st()) == -1
    assert L.fa_linear_planes(A.data_ptr(), M, C.byref(lin), 0, r.data_ptr(), N, r.data_ptr(), N - 4, y.data_ptr(), N, x3, _st()) == -1
    assert L.fa_linear_planes_to_planes(A.data_ptr(), M, C.byref(lin), 0, out.data_ptr(), N - 32, x3, _st()) == -1
    torch.cuda.synchronize()
    _all_nan(y, "y after empty / refused calls")
    _all_nan(out, "planes after empty / refused calls")


# ============================================================================================ 3. conv-view GEMM
def _conv_weights(g, N, c_in, k):
    """Conv1d weight [N, c_in, k] and its GEMM repack W[n, j * c_in + c] = w[n, c, j]."""
    w = torch.randn(N, c_in, k, generator=g) / math.sqrt(c_in * k)
    return w, w.permute(0, 2, 1).reshape(N, k * c_in).contiguous()


def _split_w(abi, L, Wm):
    N, K = Wm.shape
    kp = (K + 63) // 64 * 64
    wd = Wm.to(DEV)
    wp = torch.empty(3, N, kp, dtype=F16, device=DEV)
    assert L.fa_split_planes(wd.data_ptr(), K, N, K, kp, wp.data_ptr(), _st()) == 0
    return wd, wp, kp


def _f64_bound(y, ref, S, tau):
    """Per-element check |y - ref| <= tau * S + ulp(y) / 2 -> measured tau (max over elements of the excess / S)."""
    y = np.asarray(y, dtype=np.float32)
    err = np.abs(y.astype(np.float64) - ref)
    half_ulp = np.spacing(np.abs(y)).astype(np.float64) / 2
    measured = float((np.clip(err - half_ulp, 0, None) / S).max())
    return measured, bool((err <= tau * S + half_ulp).all())


# (id, kind, B, T)
VIEW_CASES = [("cif_b3_t37", "cif", 3, 37), ("cif_b1_t200", "cif", 1, 200), ("tdnn_b2_t75", "tdnn", 2, 75), ("tdnn_b1_t301", "tdnn", 1, 301)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", VIEW_CASES, ids=[c[0] for c in VIEW_CASES])
def test_conv_view_gemm(lib, case, mode):
    abi, L = lib
    name, kind, B, T = case
    g = torch.Generator().manual_seed(B * 1000 + T)
    if kind == "cif":            # Conv1d(512, 512, 3, pad 1) + ReLU: a zero row either side of every utterance
        c_in, k, stride, a_ld, N = 512, 3, 1, 512, 512
        Pu = T + 2
        rows, pad_rows = B * Pu, B * Pu + 2
        apr = pad_rows
        first = 1
    else:                        # CAM++ TDNN Conv1d(320, 128, 5, stride 2, pad 2) + ReLU: two zero rows either side
        c_in, k, stride, a_ld, N = 320, 5, 2, 640, 128
        Pu = (T + 4 + 1) // 2 * 2
        rows, pad_rows = B * Pu // 2, B * Pu + 4
        apr = pad_rows // 2
        first = 2
    feats = torch.randn(B, T, c_in, generator=g)
    pad = torch.zeros(pad_rows, c_in)
    for bb in range(B):
        pad[bb * Pu + first:bb * Pu + first + T] = feats[bb]
    w, Wm = _conv_weights(g, N, c_in, k)
    b = torch.randn(N, generator=g) * 0.1
    wd, wp, kp = _split_w(abi, L, Wm)
    assert kp == k * c_in
    bd = b.to(DEV)
    lin = _lin(abi, wp, bd, N, k * c_in, kp, w=wd)
    npl = NPL[mode]
    gm = abi.GEMM_MODES[mode]
    padd = pad.to(DEV)
    planes = torch.empty(npl, pad_rows, c_in, dtype=F16, device=DEV)
    assert L.fa_split_rows(padd.data_ptr(), c_in, pad_rows, c_in, c_in, npl, planes.data_ptr(), _st()) == 0
    y = torch.full((rows, N + 4), NAN, device=DEV)
    assert L.fa_linear_planes_view(planes.data_ptr(), rows, a_ld, apr, C.byref(lin), 1, y.data_ptr(), N + 4, gm, _st()) == 0
    # the same rows materialised by the split pass (fa_linear with ldx = a_ld < in_f): same products, same order
    ws = torch.empty(L.fa_linear_workspace_bytes(rows, kp, gm), dtype=torch.uint8, device=DEV)
    y2 = torch.full((rows, N), NAN, device=DEV)
    assert L.fa_linear(padd.data_ptr(), a_ld, rows, C.byref(lin), 1, None, 0, None, 0, y2.data_ptr(), N, gm, ws.data_ptr(), ws.numel(),
                       _st()) == 0
    torch.cuda.synchronize()
    _same(y[:, :N], y2, "%s %s view vs materialised" % (name, mode))
    _all_nan(y[:, N:], "pad columns")
    # float64 Conv1d restatement on the valid output rows
    t_out = (T + 2 * (k // 2) - k) // stride + 1
    got, ref, S = [], [], []
    for bb in range(B):
        x64 = feats[bb].double().T.unsqueeze(0)
        ref.append(torch.relu(torch.nn.functional.conv1d(x64, w.double(), b.double(), stride=stride, padding=k // 2))[0].T)
        S.append(torch.nn.functional.conv1d(x64.abs(), w.double().abs(), None, stride=stride, padding=k // 2)[0].T + 1e-300)
        r0 = bb * Pu // stride
        got.append(y[r0:r0 + t_out, :N].cpu())
    measured, ok = _f64_bound(torch.cat(got).numpy(), torch.cat(ref).numpy(), torch.cat(S).numpy(), TAU[mode])
    print("%s %s: tau %.2e (bar %.0e)" % (name, mode, measured, TAU[mode]))
    assert ok, (name, mode, measured)
    # refused: a_ld % 8, a_plane_rows one short of the bound
    assert L.fa_linear_planes_view(planes.data_ptr(), rows, a_ld - 4, apr, C.byref(lin), 1, y.data_ptr(), N + 4, gm, _st()) == -4
    assert L.fa_linear_planes_view(planes.data_ptr(), rows, a_ld, apr - 1, C.byref(lin), 1, y.data_ptr(), N + 4, gm, _st()) == -1


# ============================================================================================ 4. float64, real-valued data
@pytest.mark.parametrize("K", [512, 2048])
@pytest.mark.parametrize("mode", MODES)
def test_gemm_float64_per_element(lib, mode, K):
    abi, L = lib
    M, N = 1024, 512
    g = torch.Generator().manual_seed(K)
    x = torch.randn(M, K, generator=g)                           # LayerNorm-scale rows
    w0 = torch.randn(N, K, generator=g) / math.sqrt(K)           # the models' weight scale
    b = torch.randn(N, generator=g) * 0.1
    npl = NPL[mode]
    xd = x.to(DEV)
    ap = torch.empty(npl, M, K, dtype=F16, device=DEV)
    assert L.fa_split_rows(xd.data_ptr(), K, M, K, K, npl, ap.data_ptr(), _st()) == 0
    x64 = x.double()
    for wscale, bars in ((1.0, TAU), (256.0, TAU_W256)) if K == 512 else ((1.0, TAU),):
        w = w0 * wscale
        wd, wp, kp = _split_w(abi, L, w)
        bd = b.to(DEV)
        lin = _lin(abi, wp, bd, N, K, kp, w=wd)
        y = torch.full((M, N), NAN, device=DEV)
        assert L.fa_linear_planes(ap.data_ptr(), M, C.byref(lin), 0, None, 0, None, 0, y.data_ptr(), N, abi.GEMM_MODES[mode], _st()) == 0
        torch.cuda.synchronize()
        ref = (x64 @ w.double().T + b.double()).numpy()
        S = (x64.abs() @ w.double().abs().T).numpy()
        measured, ok = _f64_bound(y.cpu().numpy(), ref, S, bars[mode])
        # the two floors apart: the mode's terms on the planes in float64 (representation) and the kernel against them (accumulator)
        terms = _acc(ap, wp, mode).cpu() + b.double()
        repr_tau = float((np.abs(terms.numpy() - ref) / S).max())
        acc_tau = _f64_bound(y.cpu().numpy(), terms.numpy(), S, bars[mode])[0]
        print("float64 %s K=%d W x %g: tau %.2e (bar %.0e); representation %.2e, accumulator %.2e" % (mode, K, wscale, measured, bars[mode],
                                                                                                  repr_tau, acc_tau))
        assert ok, (mode, K, wscale, measured)


# ============================================================================================ 5. LayerNorm
def _norm(abi, n, seed):
    g = torch.Generator().manual_seed(seed)
    gam = 1 + 0.1 * torch.randn(n, generator=g)
    bet = 0.1 * torch.randn(n, generator=g)
    gd, bd = gam.to(DEV), bet.to(DEV)
    return gam, bet, (gd, bd), abi.FaNorm(gd.data_ptr(), bd.data_ptr(), n, 1e-12)


def _ln64(x, gam, bet, eps=1e-12):
    """float64 LayerNorm of fp32 rows -> (y64, bar scale |g| (1 + |z| + |mean| / std) + |b|)."""
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    sd = (var + eps).sqrt()
    z = (x - mu) / sd
    y = z * gam.double() + bet.double()
    return y, gam.double().abs() * (1 + z.abs() + mu.abs() / sd) + bet.double().abs()


def _ln_rows(rows, n, seed):
    """Unit rows, and every fourth row with |mean| >> std (mean 1e3, std 0.1 / mean -50, std 1e-2)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, n, generator=g)
    x[1::4] = 1e3 + 0.1 * x[1::4]
    x[3::4] = -50 + 1e-2 * x[3::4]
    return x


LN_SHAPES = [(256, 256), (512, 512), (560, 576), (1024, 1024), (2048, 2048)]   # NV = 4, 4, 5, 8, 16


@pytest.mark.parametrize("shape", LN_SHAPES, ids=["n%d_pad%d" % s for s in LN_SHAPES])
def test_layernorm_planes(lib, shape):
    abi, L = lib
    n, cols_pad = shape
    gam, bet, keep, nm = _norm(abi, n, n)
    worst = 0.0
    for rows in (1, 7, 8, 9, 1000):
        x = _ln_rows(rows, n, rows + n)
        xd = x.to(DEV)
        y0 = torch.full((rows, n), NAN, device=DEV)
        assert L.fa_layernorm(xd.data_ptr(), rows, C.byref(nm), y0.data_ptr(), None, C.c_float(1.0), 1, _st()) == 0
        for npl in (1, 2, 3):
            y = torch.full((rows, n), NAN, device=DEV)
            pl = torch.full((3, rows, cols_pad), NAN, dtype=F16, device=DEV)
            assert L.fa_layernorm_planes(xd.data_ptr(), rows, C.byref(nm), y.data_ptr(), pl.data_ptr(), npl, cols_pad, None,
                                         C.c_float(1.0), 1, None, _st()) == 0
            pl_only = torch.full((3, rows, cols_pad), NAN, dtype=F16, device=DEV)
            assert L.fa_layernorm_planes(xd.data_ptr(), rows, C.byref(nm), None, pl_only.data_ptr(), npl, cols_pad, None,
                                         C.c_float(1.0), 1, None, _st()) == 0
            xi = xd.clone()
            pl_in = torch.full((3, rows, cols_pad), NAN, dtype=F16, device=DEV)
            assert L.fa_layernorm_planes(xi.data_ptr(), rows, C.byref(nm), xi.data_ptr(), pl_in.data_ptr(), npl, cols_pad, None,
                                         C.c_float(1.0), 1, None, _st()) == 0
            torch.cuda.synchronize()
            what = "LN n=%d rows=%d npl=%d" % (n, rows, npl)
            _same(y, y0, what + ": fp32 output vs fa_layernorm")
            _same_bits(pl[:npl, :, :n], _split(y, npl), what + ": planes vs split of y")
            assert bool((pl[:npl, :, n:].float() == 0).all()), what + ": K padding not zero"
            _all_nan(pl[npl:], what + ": planes beyond nplanes")
            _same_bits(pl_only, pl, what + ": plane-only call")
            _same(xi, y, what + ": in place")
            _same_bits(pl_in, pl, what + ": in-place planes")
        y64, scale = _ln64(x, gam, bet)
        e = ((y0.cpu().double() - y64).abs() / (EPS32 * scale)).max().item()
        worst = max(worst, e)
        assert e <= LN_C, (n, rows, e)
    print("LN n=%d: worst |y - y64| / (eps32 * scale) = %.1f (bar %.0f)" % (n, worst, LN_C))


@pytest.mark.parametrize("n", [512, 560])
def test_layernorm_pe_prologue(lib, n):
    abi, L = lib
    gam, bet, keep, nm = _norm(abi, n, n + 1)
    half = n // 2
    inv = torch.exp(torch.arange(half, dtype=torch.float64) * (-math.log(10000.0) / (half - 1))).float()
    invd = inv.to(DEV)
    xscale = float(np.float32(math.sqrt(512.0)))
    worst_pe, worst_ln = 0.0, 0.0
    for rows, rpb in ((2 * 4100 + 37, 4100), (100, 37), (5, 1)):
        g = torch.Generator().manual_seed(rows + n)
        x = torch.randn(rows, n, generator=g) * 0.3
        xd = x.to(DEV)
        y = torch.full((rows, n), NAN, device=DEV)
        emb = torch.full((rows, n), NAN, device=DEV)
        pl = torch.full((3, rows, n + 64), NAN, dtype=F16, device=DEV)
        assert L.fa_layernorm_planes(xd.data_ptr(), rows, C.byref(nm), y.data_ptr(), pl.data_ptr(), 2, n + 64, invd.data_ptr(),
                                     C.c_float(xscale), rpb, emb.data_ptr(), _st()) == 0
        torch.cuda.synchronize()
        pos = (torch.arange(rows) % rpb + 1).float()
        arg = (pos[:, None] * inv[None, :]).double()                     # fl32(pos * inv), as __fmul_rn
        pe64 = torch.cat([torch.sin(arg), torch.cos(arg)], 1)
        ref = ((x * np.float32(xscale)).double() + pe64).float()          # fl32(fl32(x * xscale) + pe64)
        embc = emb.cpu()
        d = (embc.double() - ref.double()).abs()
        ulp = torch.from_numpy(np.spacing(np.abs(ref.numpy())).astype(np.float64))
        k = float(((d - ulp).clamp_min(0) / 2.0 ** -24).max())
        worst_pe = max(worst_pe, k)
        assert k <= PE_K, (rows, rpb, k)
        # LayerNorm of the embedded rows the kernel itself formed, and the planes of its output
        y64, scale = _ln64(embc, gam, bet)
        e = ((y.cpu().double() - y64).abs() / (EPS32 * scale)).max().item()
        worst_ln = max(worst_ln, e)
        assert e <= LN_C
        _same_bits(pl[:2, :, :n], _split(y, 2), "PE planes")
        assert bool((pl[:2, :, n:].float() == 0).all())
        _all_nan(pl[2:], "third plane")
    print("PE n=%d: worst |emb - ref| beyond one ulp %.2f x 2^-24 (bar %.1f), LN %.1f" % (n, worst_pe, PE_K, worst_ln))


def test_layernorm_planes_status(lib):
    abi, L = lib
    n = 512
    gam, bet, keep, nm = _norm(abi, n, 3)
    x = torch.zeros(8, n, device=DEV)
    y = torch.full((8, n), NAN, device=DEV)
    pl = torch.full((3, 8, n), NAN, dtype=F16, device=DEV)
    inv = torch.ones(n // 2, device=DEV)
    one = C.c_float(1.0)
    assert L.fa_layernorm_planes(x.data_ptr(), 8, C.byref(nm), y.data_ptr(), pl.data_ptr() + 2, 2, n, None, one, 1, None, _st()) == -4
    assert L.fa_layernorm_planes(x.data_ptr(), 8, C.byref(nm), y.data_ptr() + 4, None, 0, 0, None, one, 1, None, _st()) == -4
    assert L.fa_layernorm_planes(x.data_ptr(), 8, C.byref(nm), y.data_ptr(), pl.data_ptr(), 4, n, None, one, 1, None, _st()) == -1
    assert L.fa_layernorm_planes(x.data_ptr(), 8, C.byref(nm), y.data_ptr(), pl.data_ptr(), 2, n - 4, None, one, 1, None, _st()) == -4
    assert L.fa_layernorm_planes(x.data_ptr(), 8, C.byref(nm), y.data_ptr(), None, 0, 0, None, one, 1, y.data_ptr(), _st()) == -1
    assert L.fa_layernorm_planes(x.data_ptr(), 8, C.byref(nm), None, None, 0, 0, None, one, 1, None, _st()) == -1
    assert L.fa_layernorm_planes(x.data_ptr(), 8, C.byref(nm), y.data_ptr(), None, 0, 0, inv.data_ptr(), one, 0, None, _st()) == -1
    assert L.fa_layernorm_planes(x.data_ptr(), 0, C.byref(nm), y.data_ptr(), pl.data_ptr(), 2, n, None, one, 1, None, _st()) == 0
    torch.cuda.synchronize()
    _all_nan(y, "y after refused calls")
    _all_nan(pl, "planes after refused calls")
