"""GPU: the punctuation request pool on a real CT-Transformer handle -- the premise (a window's punctuation ids are the same bits whatever
shares its step: batch size, row and padded length), concurrent fa_punc_infer calls against the same calls on a fresh handle, a refused
call among pooled ones, the lone call's launches, and FunOfflineInferBuffer from 16 threads with vad-dir and punc-dir."""
import ctypes as C
import os
import shutil
import subprocess
import threading
import time

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

from funasr_b200 import _abi, pack, synth
from funasr_b200.offline import OfflinePunc
from funasr_b200.punc import PuncEngine, split_words
from test_offline_punc_host import ENC_CONF
from test_offline_stamps_gpu import BICIF_SEED, _bicif_file, _long_wav
from test_offline_vad_gpu import _wav_bytes

DEV = "cuda:0"
CASES = ["punc_short", "punc_long", "punc_english_tail"]
WAIT = 300.0
# kernel launches of one lockstep step of the synthetic CT-Transformer (4 SAN-M layers, d 256): fa_embedding, the encoder and
# fa_linear_argmax, the same as one step of the parent commit's fa_punc_infer
LAUNCHES_PER_STEP = 36


@pytest.fixture(scope="module")
def punc_file(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("punc") / "punc.fab2")
    pack.write_punc_model_file(path, synth.make_punc_state_dict(0), synth.PUNC_LIST, synth.punc_token_list(), 3, ENC_CONF)
    return path


def _step(eng, ids, lens):
    """One padded step through the three entries punc_step runs (fa_embedding, fa_sanm_encoder_forward, fa_linear_argmax) ->
    (punctuation ids, best scores) [B, T] on the host."""
    lib = eng.lib
    B, T = ids.shape
    d_ids = torch.from_numpy(np.ascontiguousarray(ids, np.int32)).to(DEV)
    x = torch.empty((B, T, eng.d_in), dtype=torch.float32, device=DEV)
    st = eng._stream()
    _abi.check(lib.fa_embedding(d_ids.data_ptr(), eng.embed.data_ptr(), eng.d_in, int(eng.embed.shape[0]), B * T, x.data_ptr(), st), "fa_embedding")
    h = eng._encode(eng.enc, x, torch.from_numpy(np.asarray(lens, np.int32)).to(DEV), eng.d_model)
    out = torch.empty(B * T, dtype=torch.int32, device=DEV)
    best = torch.empty(B * T, dtype=torch.float32, device=DEV)
    ws = eng._workspace(lib.fa_linear_argmax_workspace_bytes(B * T, eng.n_punc, eng.mode))
    _abi.check(lib.fa_linear_argmax(C.byref(eng.out), h.data_ptr(), None, B * T, out.data_ptr(), best.data_ptr(), None, eng.mode,
                                    ws.data_ptr(), ws.numel(), st), "fa_linear_argmax")
    return out.cpu().numpy().reshape(B, T), best.cpu().numpy().reshape(B, T)


@pytest.mark.gpu
def test_a_window_scores_the_same_bits_in_any_step():
    """240 seeded windows of 1 to 220 words, each scored alone (batch 1, t_max its length) and again at a random row of a step of 2 to
    64 other windows padded to a longer t_max: punctuation ids and best scores are bit-identical."""
    eng = PuncEngine(synth.make_punc_state_dict(0), DEV, synth.PUNC_HEADS)
    rng = np.random.default_rng(17)
    V = len(synth.punc_token_list())
    lens = [1, 2, 19, 20, 21, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200, 201, 219, 220] + [int(v) for v in rng.integers(1, 221, 222)]
    wins = [rng.integers(0, V, n).astype(np.int32) for n in lens]
    for w in wins:
        ids1, best1 = _step(eng, w[None], [len(w)])
        B = int(rng.integers(2, 65))
        others = [wins[int(k)] for k in rng.integers(0, len(wins), B)]
        row = int(rng.integers(0, B))
        others[row] = w
        T = max(len(o) for o in others) + int(rng.integers(0, 40))
        ids = np.zeros((B, T), np.int32)
        for b, o in enumerate(others):
            ids[b, :len(o)] = o
        idsB, bestB = _step(eng, ids, [len(o) for o in others])
        n = len(w)
        assert np.array_equal(idsB[row, :n], ids1[0, :n]), (n, B, row, T)
        assert bestB[row, :n].tobytes() == best1[0, :n].tobytes(), (n, B, row, T)


def _texts(rng, k):
    """k texts of 0 to 3 000 characters (mixed CJK and English)."""
    out = []
    for _ in range(k):
        n = int(rng.integers(0, 3001))
        out.append(synth.make_punc_text(n, int(rng.integers(0, 1 << 30)))[:n])
    return out


class Call(threading.Thread):
    def __init__(self, p, texts, bar=None):
        super().__init__(daemon=True)
        self.p, self.texts, self.bar, self.out, self.err, self.steps, self.t_end = p, texts, bar, None, None, None, None

    def run(self):
        if self.bar:
            self.bar.wait(WAIT)
        try:
            self.out, self.steps = self.p.infer(self.texts)
        except _abi.FunasrB200Error as e:
            self.err = str(e)
        self.t_end = time.monotonic()


class Handle:
    """OfflinePunc whose infer returns (results, steps) of its own call (OfflinePunc.last_steps is shared by the threads of one
    object)."""

    def __init__(self, path):
        self.p = OfflinePunc(path, 0)
        self.lib = self.p.lib

    def infer(self, texts):
        from funasr_b200.offline import _c_strings, _punc_result
        arr, _k = _c_strings(texts)
        res = self.lib.fa_punc_infer(self.p.handle, arr, len(texts))
        if not res:
            raise _abi.FunasrB200Error("fa_punc_infer failed: %s" % self.lib.fa_offline_last_error().decode())
        try:
            return _punc_result(self.lib, res, len(texts)), int(self.lib.fa_punc_result_steps(res))
        finally:
            self.lib.fa_punc_free_result(res)


def _run(calls):
    for c in calls:
        c.start()
    for c in calls:
        c.join(WAIT)
        assert not c.is_alive()


@pytest.mark.gpu
def test_pooled_calls_equal_each_call_on_a_fresh_handle(punc_file):
    """One thread punctuates 64 texts of 1 600 words while 16 threads post 3 calls each of 1 to 8 texts of 0 to 3 000 characters
    (among them an empty text and the three golden texts).  Every call's texts, ids and steps equal the same call on a fresh handle;
    the pool ran fewer steps than the calls alone; a short call returned before the long one."""
    rng = np.random.default_rng(23)
    long_call = [synth.make_punc_text(1600, 500 + i) for i in range(64)]
    golden = [str(np.load(os.path.join(GOLDEN, n + ".npz"))["text_in"]) for n in CASES]
    reqs = [_texts(rng, int(rng.integers(1, 9))) for _ in range(48)]
    reqs[0] = [""] + golden
    reqs[1] = golden[:1]
    h = Handle(punc_file)
    c0, s0 = h.p.pool_stats()
    bar = threading.Barrier(17)
    lead = Call(h, long_call, bar)

    def post(j):
        bar.wait(WAIT)
        for k in range(j, len(reqs), 16):
            c = Call(h, reqs[k])
            c.run()
            got[k] = c
    got = [None] * len(reqs)
    workers = [threading.Thread(target=post, args=(j,), daemon=True) for j in range(16)]
    _run([lead] + workers)
    c1, s1 = h.p.pool_stats()
    fresh = Handle(punc_file)
    want_long = fresh.infer(long_call)
    assert lead.err is None and (lead.out, lead.steps) == want_long
    alone_steps = want_long[1]
    for r, c in zip(reqs, got):
        w = fresh.infer(r)
        assert c.err is None and (c.out, c.steps) == w, r
        alone_steps += w[1]
    g = {n: np.load(os.path.join(GOLDEN, n + ".npz")) for n in CASES}
    assert got[0].out[1:] == [{"text": str(g[n]["text_out"]), "punc_array": g[n]["punc_array"].tolist()} for n in CASES]
    assert got[0].out[0] == {"text": "", "punc_array": []}
    assert c1 - c0 == 1 + sum(any(split_words(t) for t in r) for r in reqs) and s1 - s0 < alone_steps   # empty calls skip the pool
    assert min(c.t_end for c in got) < lead.t_end
    fresh.p.close()
    h.p.close()


@pytest.mark.gpu
def test_a_refused_call_among_pooled_ones_fails_alone(tmp_path):
    """A model that never predicts a comma or a sentence end, with 2 000-word windows: a call whose second text carries past the fp32
    attention kernel's 10 240 keys fails among concurrent calls with the message it gets alone; the others get what they get alone."""
    st = synth.make_punc_state_dict(0)
    st["decoder.bias"] = st["decoder.bias"].clone()
    st["decoder.bias"][:] = -100.0
    st["decoder.bias"][1] = 100.0                                      # always "_"
    t = pack.punc_model_tensors(st, synth.PUNC_LIST, synth.punc_token_list(), 3, ENC_CONF)
    t["__punc_config__"] = t["__punc_config__"].copy()
    t["__punc_config__"][5] = 2000
    path = str(tmp_path / "blank.fab2")
    pack._write(path, t)
    bad = [synth.make_punc_text(30, 1), "你" * 13000]
    goods = [[synth.make_punc_text(n, 40 + n) for n in (3000, 5000, 700)] for _ in range(6)]
    fresh = Handle(path)
    with pytest.raises(_abi.FunasrB200Error) as e:
        fresh.infer(bad)
    msg = str(e.value)
    assert "text 1: window 5 holds 12000 words" in msg
    want = [fresh.infer(g) for g in goods]
    h = Handle(path)
    bar = threading.Barrier(len(goods) + 1)
    calls = [Call(h, bad, bar)] + [Call(h, g, bar) for g in goods]
    _run(calls)
    assert calls[0].err == msg and calls[0].out is None
    for c, w in zip(calls[1:], want):
        assert c.err is None and (c.out, c.steps) == w
    calls_n, steps = h.p.pool_stats()
    assert calls_n == 1 + len(goods) and steps < sum(w[1] for w in want) + 5      # alone, the refused call runs 5 steps
    assert h.infer(goods[0]) == want[0]
    fresh.p.close()
    h.p.close()


@pytest.mark.gpu
def test_a_lone_call_launches_what_the_parent_launches(punc_file):
    """A lone call launches LAUNCHES_PER_STEP kernels per step, as fa_punc_infer did before calls were pooled, and no more."""
    h = Handle(punc_file)
    lib = h.lib
    h.infer(["你好"])                                                 # buffers grown
    for texts in (["你好"], [synth.make_punc_text(1600, 3)], [synth.make_punc_text(n, n) for n in (5, 300, 1200, 40)]):
        l0 = lib.fa_launch_count()
        _, steps = h.infer(texts)
        launches = lib.fa_launch_count() - l0
        assert launches == steps * LAUNCHES_PER_STEP, (len(texts), steps, launches)
    h.p.close()


RUNTIME_CLIENT = r'''
#include <stdio.h>
#include <stdlib.h>
#include <atomic>
#include <fstream>
#include <sstream>
#include <thread>
#include "funasrruntime_b200.h"
static const char* s(const char* p) { return p ? p : ""; }
int main(int argc, char** argv) {
  std::map<std::string, std::string> mp;
  mp["model-dir"] = argv[1];
  mp["vad-dir"] = argv[2];
  mp["punc-dir"] = argv[3];
  const int T = atoi(argv[4]), reps = 3;
  std::vector<std::string> bufs;
  for (int i = 5; i < argc; ++i) { std::ifstream f(argv[i], std::ios::binary); std::stringstream ss; ss << f.rdbuf(); bufs.push_back(ss.str()); }
  FUNASR_HANDLE h = FunOfflineInit(mp, T);
  if (!h) { printf("init failed %s\n", FunB200LastError()); return 1; }
  const int n = (int)bufs.size();
  std::vector<std::string> out(n * reps);
  std::atomic<int> next(0), failed(0);
  auto run = [&] {
    std::vector<std::vector<float>> hw;
    for (int k; (k = next++) < n * reps;) {
      const std::string& b = bufs[k % n];
      FUNASR_RESULT r = FunOfflineInferBuffer(h, b.data(), (int)b.size(), RASR_NONE, nullptr, hw, 16000, "wav");
      if (!r) { ++failed; continue; }
      out[k] = std::string(s(FunASRGetResult(r, 0))) + "|" + s(FunASRGetStamp(r)) + "|" + s(FunASRGetStampSents(r));
      FunASRFreeResult(r);
    }
  };
  std::vector<std::thread> th;
  for (int t = 0; t < T; ++t) th.emplace_back(run);
  for (auto& t : th) t.join();
  for (int k = 0; k < n * reps; ++k) printf("%d %s\n", k, out[k].c_str());
  FunOfflineUninit(h);
  return failed.load() ? 1 : 0;
}
'''


@pytest.mark.gpu
def test_runtime_punc_dir_from_16_threads(tmp_path, punc_file):
    """FunOfflineInit with model-dir (tiny BiCif), vad-dir and punc-dir: 16 threads of FunOfflineInferBuffer over 8 recordings (3
    times each) give the texts, stamps and stamp sentences of one thread."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    cfg = synth.PARAFORMER_TINY
    d, vd, pd = tmp_path / "asr", tmp_path / "vad", tmp_path / "punc"
    for x in (d, vd, pd):
        x.mkdir()
    _bicif_file(str(d / "model.fab2"), cfg, BICIF_SEED, synth.make_cmvn(cfg, 1))
    cjk = synth.punc_token_list()[3:synth.PUNC_VOCAB - 17]
    (d / "tokens.txt").write_text("\n".join(["<blank>", "<s>", "</s>"] + [cjk[i % len(cjk)] for i in range(3, cfg.vocab)]) + "\n",
                                  encoding="utf-8")
    pack.write_vad_model_file(str(vd / "vad.fab2"), synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    os.symlink(punc_file, str(pd / "punc.fab2"))
    w = _long_wav()
    wavs = []
    for i, (a, b) in enumerate([(0, 40), (0, 12), (5, 40), (10, 30), (3, 21), (20, 40), (8, 16), (1, 35)]):
        path = str(tmp_path / ("r%d.wav" % i))
        open(path, "wb").write(_wav_bytes(w[a * 16000:b * 16000], "f32"))
        wavs.append(path)
    inc, libdir = os.path.join(ROOT, "include"), os.path.join(ROOT, "funasr_b200")
    src, exe = tmp_path / "client.cpp", str(tmp_path / "client")
    src.write_text(RUNTIME_CLIENT)
    r = subprocess.run(["g++", "-std=c++17", "-pthread", "-I" + inc, str(src), "-L" + libdir, "-lfunasr_b200", "-Wl,-rpath," + libdir, "-o", exe],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]

    def run(T):
        p = subprocess.run([exe, str(d), str(vd), str(pd), str(T)] + wavs, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=WAIT)
        out = p.stdout.decode("utf-8")
        assert p.returncode == 0, out[-2000:]
        lines = [ln.split(" ", 1)[1] if " " in ln else "" for ln in out.splitlines()]
        assert len(lines) == 3 * len(wavs)
        return lines
    one, many = run(1), run(16)
    n = len(wavs)
    assert all(one[k] == one[k % n] for k in range(3 * n))
    assert many == one
    texts = [ln.split("|")[0] for ln in one[:n]]
    assert sum(bool(t) for t in texts) >= 6 and all(t[-1] in "。.?？" for t in texts if t)      # the forced sentence end
    assert all('"punc":' in ln for ln in one[:n] if ln.split("|")[0])
