"""GPU: hotword calls pooled on one recogniser handle.

Attention with a K/V entry per row (fa_attention_grouped) gives each row exactly what the kv_shared call gives it over its own entry
alone, in every precision.  Concurrent contextual and SeACo calls on one handle (utterance batches and long recordings; distinct hotword
lists, one shared list, the <s> row only, no rows) share GPU packs and each call gets exactly what it gets alone; the SeACo goldens
still come out exactly when decoded among other calls; the RTF client prints the same texts at 8 threads as at 1 on a SeACo model, and
the runtime client on a plain model gets one zero hotword row and decodes."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT, load_seaco_case

from funasr_b200 import _abi, pack, synth
from funasr_b200.offline import OfflineRecognizer, OfflineVad
from test_offline_concurrent_gpu import _threads, _utts, files  # noqa: F401 - the model files fixture
from test_offline_seaco_gpu import _seaco_file
from test_offline_vad_gpu import _s16, _wav_bytes

DEV = "cuda:0"
CFG = synth.PARAFORMER_TINY
MODES = {"fp32": 0, "fp16x1": 1, "fp16x3": 3}


def _st():
    return torch.cuda.current_stream().cuda_stream


def _i32(v):
    return (C.c_int32 * len(v))(*v)


def _grouped(lib, q, kv, key_lens, index, mode, tk, hd=128):
    """fa_attention_grouped over a NaN-filled context and a NaN-poisoned workspace -> CPU context."""
    B, tq, W = q.shape
    G = kv.shape[0]
    m = MODES[mode]
    ctx = torch.full((B, tq, W), float("nan"), device=DEV)
    ws = torch.full((int(lib.fa_attention_grouped_workspace_bytes(B, 4, tq, G, tk, m)),), 255, dtype=torch.uint8, device=DEV)
    kd = kv[:, :tk].contiguous()
    ld = torch.tensor(key_lens, dtype=torch.int32, device=DEV)
    _abi.check(lib.fa_attention_grouped(q.data_ptr(), W, kd.data_ptr(), 2 * W, kd.data_ptr() + 4 * W, 2 * W, ld.data_ptr(), _i32(index), G, B, 4,
                                        hd, tq, tk, ctx.data_ptr(), W, m, ws.data_ptr(), ws.numel(), _st()), "fa_attention_grouped")
    torch.cuda.synchronize()
    return ctx.cpu()


def _split(x, npl):
    """fp32 -> fp16 planes as the library splits them: hi = rn(x), lo = rn(x - hi)."""
    hi = x.half()
    return torch.stack([hi] if npl == 1 else [hi, (x - hi.float()).half()]).contiguous()


def _existing(lib, q, kv, key_lens, mode, kv_shared, hd=128):
    """The existing entries: fa_attention_f32_ex (fp32) or, on the tensor cores, fa_attention_tc_planes_ex over operand planes split here
    (q scaled by d_k^-0.5, k, v transposed per head with zero keys up to the 64-key pitch); kv [E, tk, 2W] with E = 1 (kv_shared) or
    B -> CPU context."""
    B, tq, W = q.shape
    E, tk = kv.shape[0], kv.shape[1]
    ctx = torch.full((B, tq, W), float("nan"), device=DEV)
    ld = torch.tensor(key_lens, dtype=torch.int32, device=DEV)
    kd = kv.contiguous()
    if mode == "fp32":
        _abi.check(lib.fa_attention_f32_ex(q.data_ptr(), W, kd.data_ptr(), 2 * W, kd.data_ptr() + 4 * W, 2 * W, ld.data_ptr(), B, 4, hd, tq, tk,
                                           ctx.data_ptr(), W, kv_shared, _st()), "fa_attention_f32_ex")
    else:
        npl = 1 if mode == "fp16x1" else 2
        qs = q * torch.tensor(np.float32(1.0 / np.sqrt(128.0)), device=DEV)
        tkp = (tk + 63) // 64 * 64
        vt = torch.zeros(E, W, tkp, device=DEV)
        vt[:, :, :tk] = kd[:, :, W:].transpose(1, 2)
        qp, kp, vp = _split(qs.reshape(B * tq, W), npl), _split(kd[:, :, :W].reshape(E * tk, W), npl), _split(vt.reshape(E * W, tkp), npl)
        _abi.check(lib.fa_attention_tc_planes_ex(qp.data_ptr(), kp.data_ptr(), vp.data_ptr(), ld.data_ptr(), B, 4, 128, tq, tk, ctx.data_ptr(), W,
                                                 None, 0, 0, MODES[mode], kv_shared, _st()), "fa_attention_tc_planes_ex")
    torch.cuda.synchronize()
    return ctx.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("mode,hd", [("fp32", 128), ("fp16x1", 128), ("fp16x3", 128), ("fp32", 80)])
def test_attention_grouped_rows_equal_each_entry_alone(mode, hd):
    """Entries of 1, 63, 64, 65 and 300 keys padded to 300 with finite rows past each length; 9 rows mapped to them out of order: each
    row equals the existing kv_shared call over its own entry alone, bit for bit (fp32: the tiled kernel at head_dim 128, the
    warp-per-query kernel at 80; tensor cores: the planes entry).  Index all-zero over one entry equals the kv_shared call, index = b
    over B entries the per-utterance call."""
    lib = _abi.load()
    g = torch.Generator().manual_seed(41)
    lens = [1, 63, 64, 65, 300]
    G, T, tq, W = len(lens), 300, 37, 4 * hd
    kv = torch.randn(G, T, 2 * W, generator=g).to(DEV)
    index = [4, 0, 2, 1, 3, 3, 4, 0, 2]
    B = len(index)
    q = torch.randn(B, tq, W, generator=g).to(DEV)
    got = _grouped(lib, q, kv, [lens[i] for i in index], index, mode, T, hd)
    assert not torch.isnan(got).any()
    for b, e in enumerate(index):
        alone = _existing(lib, q[b:b + 1].contiguous(), kv[e:e + 1, :lens[e]], [lens[e]], mode, 1, hd)
        assert torch.equal(got[b].view(torch.int32), alone[0].view(torch.int32)), (mode, hd, b, e)
    k1 = kv[1:2].contiguous()
    zero = _grouped(lib, q, k1, [65] * B, [0] * B, mode, T, hd)
    assert torch.equal(zero.view(torch.int32), _existing(lib, q, k1, [65] * B, mode, 1, hd).view(torch.int32)), (mode, hd)
    kvb = torch.randn(B, T, 2 * W, generator=g).to(DEV)
    bl = [lens[i] for i in index]
    per = _grouped(lib, q, kvb, bl, list(range(B)), mode, T, hd)
    assert torch.equal(per.view(torch.int32), _existing(lib, q, kvb, bl, mode, 0, hd).view(torch.int32)), (mode, hd)


@pytest.fixture(scope="module")
def ctx_file(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("ctx") / "ctx.fab2")
    pack.write_model_file(path, synth.make_contextual_state_dict(CFG, 6), CFG, synth.make_cmvn(CFG, 1))
    return path


def _rows(n, seed):
    return (np.random.default_rng(seed).standard_normal((n, 512)) * 0.5).astype(np.float32)


def _requests(kind):
    """18 calls: utterance batches and long recordings; hotwords one shared list (each call its own copy of the same bytes), distinct
    lists of 1..30 rows (more than nfilter 8 for most), the <s> row only, and (SeACo) no rows."""
    shared = _rows(20, 5)
    reqs = []
    for k in range(18):
        c = k % 4
        hw = shared.copy() if c == 0 else _rows(1 + (7 * k) % 30, 100 + k) if c == 1 else _rows(1, 7) if c == 2 else None
        if hw is None and kind == "ctx":
            hw = _rows(3 + k, 200 + k)
        long = k % 3 == 2
        wavs = [synth.make_vad_wav(6.0 + k % 5, 70 + k).numpy()] if long else _utts(k)
        reqs.append((long, wavs, hw))
    return reqs


def _call(rec, vad, req):
    long, wavs, hw = req
    if long:
        return rec.infer_long(wavs, vad, batch_size_s=4, hotword_embeddings=hw)
    return rec.infer(wavs, hotword_embeddings=hw)


def _stats(lib, rec):
    c, p = C.c_int64(), C.c_int64()
    _abi.check(lib.fa_offline_pool_stats(rec.handle, C.byref(c), C.byref(p)), "fa_offline_pool_stats")
    return c.value, p.value


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("kind", ["seaco", "ctx"])
def test_pooled_hotword_calls_equal_each_call_alone(files, ctx_file, kind, mode):  # noqa: F811 - the fixture
    lib = _abi.load()
    path = files["seaco"] if kind == "seaco" else ctx_file
    reqs = _requests(kind)
    solo, vad1 = OfflineRecognizer(path, 0, mode), OfflineVad(files["vad"], 0)
    alone = [_call(solo, vad1, r) for r in reqs]
    assert any(t for a in alone for t in (a if isinstance(a[0], list) else [x["token_int"] for x in a]))
    solo.close()
    rec, vad = OfflineRecognizer(path, 0, mode), OfflineVad(files["vad"], 0)
    got = _threads(len(reqs), lambda k: _call(rec, vad, reqs[k]))
    calls, packs = _stats(lib, rec)
    assert got == alone
    assert calls == len(reqs) and packs < calls, (calls, packs)
    rec.close()
    vad1.close()
    vad.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("name", ["seaco_tiny_ragged3", "seaco_tiny_asf"])
def test_seaco_goldens_among_other_calls(tmp_path, name, mode):
    """The golden case decoded while 11 other calls with other hotword lists (and one with none) share its packs: its ids are still
    the unmodified reference's."""
    lib = _abi.load()
    cfg, wseed, wavs, cmvn, hw, nfilter, g = load_seaco_case(name)
    rec = OfflineRecognizer(_seaco_file(str(tmp_path / "m.fab2"), wseed, nfilter, cmvn), 0, mode)
    rows = rec.hotword_embeddings(hw)
    others = [(_utts(k), None if k == 5 else _rows(1 + 3 * k, 300 + k)) for k in range(11)]

    def call(k):
        if k == 0:
            return rec.infer([w.numpy() for w in wavs], hotword_embeddings=rows)
        return rec.infer(others[k - 1][0], hotword_embeddings=others[k - 1][1])
    for _ in range(2):
        got = _threads(12, call)[0]
        assert [t for r in got for t in r] == g["ids_flat"].tolist() and [len(r) for r in got] == g["ids_len"].tolist()
    calls, packs = _stats(lib, rec)
    assert packs < calls, (calls, packs)
    rec.close()


@pytest.mark.gpu
def test_pack_hotword_bound_splits_packs(files):  # noqa: F811 - the fixture
    """A GPU pack holds at most 4096 hotword-memory rows, counted as (distinct sets + filtered reference packs) x the longest set.  12
    SeACo calls with distinct 300-row lists (nfilter 8, so each is filtered: 2 x 300 = 600 rows a call) fit at most 6 to a pack, and a call
    with a 2100-row list (2 x 2100 = 4200 rows on its own) decodes alone: at least 3 packs.  Every call equals the call alone."""
    lib = _abi.load()
    reqs = [(False, _utts(k), _rows(300, 500 + k)) for k in range(12)] + [(False, _utts(12), _rows(2100, 600))]
    solo = OfflineRecognizer(files["seaco"], 0, "fp16x3")
    alone = [_call(solo, None, r) for r in reqs]
    solo.close()
    rec = OfflineRecognizer(files["seaco"], 0, "fp16x3")
    got = _threads(len(reqs), lambda k: _call(rec, None, reqs[k]))
    calls, packs = _stats(lib, rec)
    assert got == alone
    assert calls == len(reqs) and packs >= 3, (calls, packs)
    rec.close()


def _client(name, tmp_path):
    exe = str(tmp_path / name)
    inc = os.path.join(ROOT, "include")
    r = subprocess.run(["g++", "-std=c++17", "-pthread", '-DFUNASR_RUNTIME_HEADER="funasrruntime_b200.h"', "-I" + inc,
                        os.path.join(ROOT, "examples", name + ".cpp"), "-L" + os.path.join(ROOT, "funasr_b200"), "-lfunasr_b200",
                        "-Wl,-rpath," + os.path.join(ROOT, "funasr_b200"), "-o", exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    return exe


def _model_dir(d, path):
    d.mkdir()
    shutil.copy(path, d / "model.fab2")
    (d / "tokens.txt").write_text("\n".join(chr(0x4E00 + i) for i in range(CFG.vocab)) + "\n", encoding="utf-8")
    return str(d)


@pytest.mark.gpu
def test_rtf_client_seaco_eight_threads_equal_one(files, tmp_path):  # noqa: F811 - the fixture
    """examples/offline_rtf_client.cpp on a SeACo model directory (every call carries the <s> row from CompileHotwordEmbedding, so
    every call is a hotword call): 8 threads on one handle print the texts 1 thread prints."""
    exe = _client("offline_rtf_client", tmp_path)
    d = _model_dir(tmp_path / "seaco", files["seaco"])
    lines = []
    for k in range(12):
        p = tmp_path / ("w%d.wav" % k)
        p.write_bytes(_wav_bytes(_s16(synth.make_wav(9000 + 2311 * k, 80 + k, "speechlike").numpy()), "s16"))
        lines.append("u%d %s" % (k, p))
    (tmp_path / "list.txt").write_text("\n".join(lines) + "\n")

    def run(n):
        r = subprocess.run([exe, d, str(tmp_path / "list.txt"), str(n)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:]
        out = r.stdout.strip().splitlines()
        assert out[-1].startswith("threads %d files 12 failed 0" % n), out[-1]
        return out[:-1]
    one = run(1)
    assert len(one) == 12 and sum(len(x.split(" ", 1)) > 1 for x in one) >= 3
    assert run(8) == one


@pytest.mark.gpu
def test_runtime_client_plain_model_gets_one_zero_row(files, tmp_path):  # noqa: F811 - the fixture
    """CompileHotwordEmbedding on a plain Paraformer handle returns one zero row of 512, as the reference's model without a hotword
    branch does, and the runtime client decodes with it."""
    exe = _client("offline_runtime_client", tmp_path)
    d = _model_dir(tmp_path / "asr", files["asr"])
    wav = tmp_path / "a.wav"
    wav.write_bytes(_wav_bytes(_s16(synth.make_wav(48000, 21, "speechlike").numpy()), "s16"))
    r = subprocess.run([exe, d, str(wav)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:]
    out = dict(line.split(" ", 1) if " " in line else (line, "") for line in r.stdout.strip().splitlines())
    assert out["hotword_rows"] == "1"
    rec = OfflineRecognizer(files["asr"], 0, "fp16x3")
    want = rec.infer([_s16(synth.make_wav(48000, 21, "speechlike").numpy())])[0]
    rec.close()
    assert len(want) > 0 and out["file_result"] == "".join(chr(0x4E00 + i) for i in want)
