"""CPU: the host side of audio at any sample rate and PCM layout (FaAudioFormat).  The loader table equals
resample.sinc_resample_table bit for bit; the runtime tables and output counts equal the reference's LinearResample (compiled, or
the committed golden); a numpy restatement of the runtime's sum order equals its outputs; the descriptor's layout and the new
symbols; the table functions' refusals; the Python bindings' input checks."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import linres_ref
from audio_in_ref import RATES, golden, have_oracle, linres_numpy, runtime_tables, sha256
from conftest import ROOT
from funasr_b200 import _abi
from funasr_b200.offline import _pcm_batch
from funasr_b200.resample import sinc_resample_table


def _loader_table(rate):
    lib = _abi.load()
    o, n, w = C.c_int32(), C.c_int32(), C.c_int32()
    need = lib.fa_loader_resample_table_host(rate, 16000, C.byref(o), C.byref(n), C.byref(w), None, 0)
    assert need > 0
    t = np.zeros(need, np.float32)
    assert lib.fa_loader_resample_table_host(rate, 16000, C.byref(o), C.byref(n), C.byref(w), t.ctypes.data, need) == need
    return t.reshape(n.value, -1), o.value, n.value, w.value


def _runtime_table(rate):
    lib = _abi.load()
    iu, ou, mt = C.c_int32(), C.c_int32(), C.c_int32()
    need = lib.fa_runtime_resample_table_host(rate, 16000, C.byref(iu), C.byref(ou), C.byref(mt), None, None, None, 0)
    assert need > 0
    first, n_taps, w = np.zeros(ou.value, np.int32), np.zeros(ou.value, np.int32), np.zeros(need, np.float32)
    assert lib.fa_runtime_resample_table_host(rate, 16000, C.byref(iu), C.byref(ou), C.byref(mt), first.ctypes.data, n_taps.ctypes.data,
                                              w.ctypes.data, need) == need
    return iu.value, ou.value, first, n_taps, w.reshape(ou.value, mt.value)


@pytest.mark.parametrize("rate", RATES + (1000, 17000, 96000, 192000))
def test_loader_table_equals_sinc_resample_table(rate):
    got, orig, new, width = _loader_table(rate)
    want, w_orig, w_new, w_width = sinc_resample_table(rate, 16000)
    assert (orig, new, width) == (w_orig, w_new, w_width)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("rate", RATES)
def test_runtime_tables_equal_the_reference(rate):
    iu, ou, first, n_taps, w = _runtime_table(rate)
    r_iu, r_ou, r_first, r_taps, r_w = runtime_tables(rate)
    assert (iu, ou) == (r_iu, r_ou)
    assert np.array_equal(first, r_first) and np.array_equal(n_taps, r_taps)
    assert w.shape == r_w.shape and np.array_equal(w.view(np.uint32), r_w.view(np.uint32))


@pytest.mark.parametrize("rate", RATES)
def test_runtime_output_counts_equal_the_reference(rate):
    lib = _abi.load()
    if have_oracle():
        lens = np.random.default_rng(rate).integers(1, 3_000_000, 2000)
        lr = linres_ref.LinearResample(rate)
        want = [lr.out_len(int(n)) for n in lens]
    else:
        g = golden()
        lens, want = g["r%d_lens" % rate], g["r%d_out_lens" % rate].tolist()
    got = [lib.fa_runtime_resample_out_len_host(rate, 16000, int(n)) for n in lens]
    assert got == want
    # both resamplers give ceil(16000 n / rate)
    assert got == [-(-16000 * int(n) // rate) for n in lens]
    assert lib.fa_runtime_resample_out_len_host(rate, 16000, 0) == 0


@pytest.mark.parametrize("rate", RATES)
def test_numpy_sum_order_equals_the_reference_outputs(rate):
    iu, _, _, n_taps, _ = runtime_tables(rate)
    edges = linres_ref.edge_lengths(iu, int(n_taps.max()))
    x = linres_ref.noise(rate, 1.0, seed=1)
    got = np.concatenate([linres_numpy(x[:n], rate) for n in edges])
    if have_oracle():
        lr = linres_ref.LinearResample(rate)
        want = np.concatenate([lr.resample(x[:n]) for n in edges])
    else:
        g = golden()
        assert g["r%d_edge_lens" % rate].tolist() == edges
        want = g["r%d_edge_out" % rate]
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # 60 s of seeded noise: against the library's output, and against the digest the golden keeps
    y = linres_numpy(linres_ref.noise(rate), rate)
    assert np.array_equal(sha256(y), golden()["r%d_noise_sha256" % rate])


def test_table_refusals():
    lib = _abi.load()
    for rate in (999, 192001, 0, -8000):
        assert lib.fa_loader_resample_table_host(rate, 16000, None, None, None, None, 0) == -1
        assert lib.fa_runtime_resample_table_host(rate, 16000, None, None, None, None, None, None, 0) == -1
        assert lib.fa_runtime_resample_out_len_host(rate, 16000, 100) == -1
    # 16 001 Hz: a 1 GB loader table (16 000 phases of 16 015 taps) is refused; the runtime's rows are short
    assert lib.fa_loader_resample_table_host(16001, 16000, None, None, None, None, 0) == -4
    assert lib.fa_loader_resample_table_host(7999, 16000, None, None, None, None, 0) == -4
    assert 0 < lib.fa_runtime_resample_table_host(16001, 16000, None, None, None, None, None, None, 0) <= (32 << 20) // 4
    # a cap below the table's size
    assert lib.fa_loader_resample_table_host(8000, 16000, None, None, None, np.zeros(4, np.float32).ctypes.data, 4) == -1


def test_symbols_and_descriptor_layout(tmp_path):
    lib = C.CDLL(_abi.LIB_PATH)
    for s in ("fa_offline_infer_audio", "fa_offline_infer_vad_audio", "fa_vad_infer_audio", "fa_spk_embed_audio", "fa_ingest_pcm",
              "fa_loader_resample_table_host", "fa_runtime_resample_table_host", "fa_runtime_resample_out_len_host"):
        assert hasattr(lib, s) and s in _abi.SIGNATURES
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    src = tmp_path / "sz.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "funasr_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(FaAudioFormat), offsetof(FaAudioFormat, resampler), sizeof(FaIngestTable),\n'
                   '         offsetof(FaIngestTable, weights), offsetof(FaIngestTable, n_taps), (size_t)FA_RESAMPLE_RUNTIME);\n  return 0;\n}\n')
    exe = str(tmp_path / "sz")
    r = subprocess.run(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    got = [int(v) for v in subprocess.run([exe], stdout=subprocess.PIPE, text=True).stdout.split()]
    assert got == [C.sizeof(_abi.FaAudioFormat), _abi.FaAudioFormat.resampler.offset, C.sizeof(_abi.FaIngestTable),
                   _abi.FaIngestTable.weights.offset, _abi.FaIngestTable.n_taps.offset, _abi.RESAMPLE_RUNTIME]


def test_python_input_checks():
    # 16 kHz mono float32 / int16 keep the 16 kHz entries; everything else takes a descriptor
    assert _pcm_batch([np.zeros(400, np.float32)])[2] is None
    assert _pcm_batch([np.zeros(400, np.int16)], 16000, "runtime")[2] is None
    _, fmt, d = _pcm_batch([np.zeros((400, 2), np.int32), np.zeros((10, 2), np.int32)], 44100, "runtime")
    assert (fmt, d.sample_format, d.channels, d.sample_rate, d.resampler) == (3, 3, 2, 44100, 1)
    assert _pcm_batch([np.zeros(400, np.uint8)])[2].sample_format == 4
    with pytest.raises(_abi.FunasrB200Error):
        _pcm_batch([np.zeros(400, np.float64)])
    with pytest.raises(_abi.FunasrB200Error):
        _pcm_batch([np.zeros(400, np.float32), np.zeros(400, np.int16)])
    with pytest.raises(_abi.FunasrB200Error):
        _pcm_batch([np.zeros((400, 2), np.float32), np.zeros((400, 1), np.float32)])
    with pytest.raises(_abi.FunasrB200Error):
        _pcm_batch([np.zeros(400, np.float32)], 8000, "sox")
