"""GPU (-m gpu): the wgmma GEMM's fp32 epilogue with one residual and with none (fa_linear_planes) and its fp16-plane epilogue
with and without ReLU (fa_linear_planes_to_planes, hi + lo (+ lo2) reconstructed) against the CPU fp32 nn.Linear, at the
tolerances of test_linear_tcgen05_vs_oracle.

The shapes cover the encoder's four GEMMs at M = 32000 and the tile counts the persistent ping-pong schedule has to get right:
fewer tiles than SMs, an odd number of tiles per CTA (one consumer warpgroup gets one tile fewer), a single tile (the second
consumer gets none), a ragged last row tile and the ragged vocabulary N (fp32 output only: plane outputs need N % 32 == 0)."""
import ctypes as C

import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TOL = {"fp16x6": 1e-5, "fp16x3": 3e-5, "fp16": 2e-2}
NPL = {"fp16": 1, "fp16x3": 2, "fp16x6": 3}
SHAPES = [
    (32000, 1536, 512),   # encoder QKV
    (32000, 512, 512),    # out-projection
    (32000, 2048, 512),   # FFN w_1
    (32000, 512, 2048),   # FFN w_2
    (300, 384, 512),      # 9 tiles (18 at x6 with 64-wide tiles): fewer tiles than SMs, odd
    (12600, 512, 512),    # 396 tiles on 132 CTAs: three (odd) per CTA; ragged last row tile
    (100, 128, 64),       # a single tile (two at x6); ragged M, one k-block
    (1000, 8404, 512),    # ragged vocabulary N
]


def _lib():
    from funasr_b200 import _abi
    return _abi, _abi.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


@pytest.mark.parametrize("mode", list(TOL))
@pytest.mark.parametrize("rows,out_f,in_f", SHAPES)
def test_linear_planes_epilogues_vs_oracle(rows, out_f, in_f, mode):
    abi, lib = _lib()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(rows, in_f, generator=g)
    w = torch.randn(out_f, in_f, generator=g) / in_f ** 0.5
    b = torch.randn(out_f, generator=g) * 0.1
    r1 = torch.randn(rows, out_f, generator=g)
    xd, wd, bd, r1d = x.to(DEV), w.to(DEV), b.to(DEV), r1.to(DEV)
    in_pad = (in_f + 63) // 64 * 64
    npl = NPL[mode]
    w_planes = torch.empty(3, out_f, in_pad, dtype=torch.float16, device=DEV)
    abi.check(lib.fa_split_planes(wd.data_ptr(), in_f, out_f, in_f, in_pad, w_planes.data_ptr(), _st()), "split w")
    a_planes = torch.empty(npl, rows, in_pad, dtype=torch.float16, device=DEV)
    abi.check(lib.fa_split_rows(xd.data_ptr(), in_f, rows, in_f, in_pad, npl, a_planes.data_ptr(), _st()), "split x")
    lin = abi.FaLinear(wd.data_ptr(), bd.data_ptr(), w_planes.data_ptr(), out_f, in_f, in_pad, 0)
    lin_ref = torch.nn.functional.linear(x, w, b)
    tol = TOL[mode]

    # EPI_F32: one residual, then none (ReLU off, as in the out-projection / w_2 calls)
    for res in (r1d, None):
        y = torch.full((rows, out_f), float("nan"), device=DEV)
        abi.check(lib.fa_linear_planes(a_planes.data_ptr(), rows, C.byref(lin), 0, res.data_ptr() if res is not None else None,
                                       out_f if res is not None else 0, None, 0, y.data_ptr(), out_f, abi.GEMM_MODES[mode], _st()),
                  "linear planes")
        torch.cuda.synchronize()
        ref = lin_ref + r1 if res is not None else lin_ref
        assert not torch.isnan(y).any()
        err = rel_err(y.cpu().numpy(), ref.numpy())
        print("fp32 out %s rows=%d out=%d in=%d residual=%s: rel err %.2e (tol %.0e)" % (mode, rows, out_f, in_f, res is not None, err, tol))
        assert err <= tol

    if out_f % 32:
        return
    # EPI_PLANES: with ReLU (FFN w_1) and without
    for relu in (1, 0):
        out = torch.full((npl, rows, out_f), float("nan"), dtype=torch.float16, device=DEV)
        abi.check(lib.fa_linear_planes_to_planes(a_planes.data_ptr(), rows, C.byref(lin), relu, out.data_ptr(), out_f,
                                                 abi.GEMM_MODES[mode], _st()), "linear planes -> planes")
        torch.cuda.synchronize()
        y = out.float().sum(0)
        ref = torch.relu(lin_ref) if relu else lin_ref
        assert not torch.isnan(y).any()
        err = rel_err(y.cpu().numpy(), ref.numpy())
        print("plane out %s rows=%d out=%d in=%d relu=%d: rel err %.2e (tol %.0e)" % (mode, rows, out_f, in_f, relu, err, tol))
        assert err <= tol
