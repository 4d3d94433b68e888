"""CPU: the punctuation request pool through fa_punc_init_host, whose steps call a Python scorer in place of the network.  Concurrent
fa_punc_infer calls on one handle share lockstep steps and each gets what fa_punc_walk_host gives it alone (texts, ids, steps); calls
join at a step boundary; the leader hands off; an over-long window fails only its own call; a failing step fails exactly the calls
that had a window in it.  Every wait has a timeout, so a scheduling bug fails a test instead of hanging it."""
import ctypes as C
import os
import random
import threading
import time

import numpy as np
import pytest

from conftest import ROOT

from funasr_b200 import _abi, synth
from funasr_b200.offline import _c_strings, _punc_result
from punc_scripted import random_text, scripted

NEW = ["fa_punc_init_host", "fa_punc_pool_stats"]
PROBS = (0.0, 0.10, 0.05, 0.02, 0.03)
WAIT = 30.0
CJK = synth.punc_token_list()[3:synth.PUNC_VOCAB - 17]


class Failed(Exception):
    pass


def _callback(score, errors):
    def cb(_ctx, ids, lens, batch, t_max, out):
        try:
            i = np.ctypeslib.as_array(ids, shape=(batch, t_max)).copy()
            n = np.ctypeslib.as_array(lens, shape=(batch,)).copy()
            r = score(i, n)
            if r is None:                                       # the scripted failure of a step
                return 7
            np.ctypeslib.as_array(out, shape=(batch, t_max))[:] = np.asarray(r, dtype=np.int32)
            return 0
        except Exception as e:                                  # an exception must not cross the C frames
            errors.append(e)
            return 1
    return _abi.PUNC_SCORE_FN(cb)


def _vocab():
    tok, k1 = _c_strings(synth.punc_token_list())
    pl, k2 = _c_strings(synth.PUNC_LIST)
    return tok, pl, (k1, k2)


def _take(lib, res, n):
    if not res:
        raise Failed(lib.fa_offline_last_error().decode())
    try:
        return [(r["text"], r["punc_array"]) for r in _punc_result(lib, res, n)], int(lib.fa_punc_result_steps(res))
    finally:
        lib.fa_punc_free_result(res)


def alone(texts, score=None, max_window=0):
    """fa_punc_walk_host over one call -> ([(text, ids)], steps); raises Failed with the call's message."""
    lib = _abi.load()
    errors = []
    fn = _callback(score or (lambda ids, ln: scripted(ids, 1, PROBS)), errors)
    ta, _k = _c_strings(texts)
    tok, pl, _kv = _vocab()
    res = lib.fa_punc_walk_host(ta, len(texts), tok, len(synth.punc_token_list()), pl, len(synth.PUNC_LIST), 3, 20, max_window, fn, None)
    assert not errors, errors
    return _take(lib, res, len(texts))


class HostPunc:
    """A fa_punc_init_host handle with `score(ids, lens)` as its network (None from score fails that step)."""

    def __init__(self, score, max_window=0):
        self.lib = _abi.load()
        self.errors = []
        self.fn = _callback(score, self.errors)
        tok, pl, self._keep = _vocab()
        self.h = self.lib.fa_punc_init_host(tok, len(synth.punc_token_list()), pl, len(synth.PUNC_LIST), 3, 20, max_window, self.fn, None)
        assert self.h, self.lib.fa_offline_last_error()

    def infer(self, texts):
        ta, _k = _c_strings(texts)
        return _take(self.lib, self.lib.fa_punc_infer(self.h, ta, len(texts)), len(texts))

    def stats(self):
        c, s = C.c_int64(), C.c_int64()
        assert self.lib.fa_punc_pool_stats(self.h, C.byref(c), C.byref(s)) == 0
        return c.value, s.value

    def close(self):
        assert not self.errors, self.errors
        self.lib.fa_punc_uninit(self.h)


class Call(threading.Thread):
    """One fa_punc_infer call on its own thread: .out = (results, steps) or .err = the message; .t_end = when it returned."""

    def __init__(self, p, texts):
        super().__init__(daemon=True)
        self.p, self.texts, self.out, self.err, self.t_end = p, texts, None, None, None
        self.returned = threading.Event()

    def run(self):
        try:
            self.out = self.p.infer(self.texts)
        except Failed as e:
            self.err = str(e)
        self.t_end = time.monotonic()
        self.returned.set()


def join_all(calls):
    for c in calls:
        c.join(WAIT)
        assert not c.is_alive(), "a pooled call did not return"


def cjk_text(rng, n):
    return "".join(rng.choice(CJK) for _ in range(n))


class Gated:
    """scripted() as the scorer, recording each step's (batch, lens, thread); hooks[k]() runs inside step k before it is scored (a
    hook that returns False fails that step)."""

    def __init__(self, seed=1):
        self.seed, self.steps, self.hooks = seed, [], {}

    def __call__(self, ids, lens):
        k = len(self.steps)
        self.steps.append((ids.shape[0], lens.tolist(), threading.get_ident()))
        if k in self.hooks and self.hooks[k]() is False:
            return None
        return scripted(ids, self.seed, PROBS)


def block_until(ev):
    def hook():
        assert ev.wait(WAIT), "the test never released the scorer"
    return hook


# ------------------------------------------------------------------------------------------------------------------ interface
def test_new_symbols_exported_and_declared():
    lib = _abi.load()
    with open(os.path.join(ROOT, "include", "funasr_b200.h")) as f:
        header = f.read()
    for name in NEW:
        assert name in _abi.SIGNATURES and hasattr(lib, name) and (name + "(") in header, name


def test_refusals_without_a_device():
    lib = _abi.load()
    c, s = C.c_int64(), C.c_int64()
    assert lib.fa_punc_pool_stats(None, C.byref(c), C.byref(s)) == -1
    p = HostPunc(lambda ids, ln: scripted(ids, 1, PROBS))
    assert lib.fa_punc_pool_stats(p.h, None, C.byref(s)) == -1 and lib.fa_punc_pool_stats(p.h, C.byref(c), None) == -1
    assert p.stats() == (0, 0)
    fn = _callback(lambda ids, ln: ids, [])
    tok, pl, _k = _vocab()
    nt, npl = len(synth.punc_token_list()), len(synth.PUNC_LIST)
    for args in ((None, nt, pl, npl, fn), (tok, 0, pl, npl, fn), (tok, nt, None, npl, fn), (tok, nt, pl, 0, fn), (tok, nt, pl, npl, _abi.PUNC_SCORE_FN())):
        t, n, q, m, f = args
        assert not lib.fa_punc_init_host(t, n, q, m, 3, 20, 0, f, None) and lib.fa_offline_last_error() == b"bad argument"
    bad_tok = (C.c_char_p * 3)(b"<unk>", None, b"a")
    assert not lib.fa_punc_init_host(bad_tok, 3, pl, npl, 3, 20, 0, fn, None) and lib.fa_offline_last_error() == b"token 1 is NULL"
    bad_pl = (C.c_char_p * 2)(b"_", None)
    assert not lib.fa_punc_init_host(tok, nt, bad_pl, 2, 0, 20, 0, fn, None) and lib.fa_offline_last_error() == b"punctuation 1 is NULL"
    dup = (C.c_char_p * 3)(b"<unk>", b"a", b"a")
    assert not lib.fa_punc_init_host(dup, 3, pl, npl, 3, 20, 0, fn, None) and b"duplicated" in lib.fa_offline_last_error()
    assert not lib.fa_punc_init_host(tok, nt, pl, npl, 9, 20, 0, fn, None) and b"sentence_end_id" in lib.fa_offline_last_error()
    assert not lib.fa_punc_init_host(tok, nt, pl, npl, 3, 1, 0, fn, None) and b"split_size" in lib.fa_offline_last_error()
    # argument refusals of fa_punc_infer on a host handle, and a call of empty texts, which never enters the pool
    assert not lib.fa_punc_infer(p.h, None, 2) and lib.fa_offline_last_error() == b"bad argument"
    nul = (C.c_char_p * 2)(b"a", None)
    assert not lib.fa_punc_infer(p.h, nul, 2) and lib.fa_offline_last_error() == b"text 1 is NULL"
    assert p.infer(["", " \t"]) == ([("", []), ("", [])], 0) and p.stats() == (0, 0)
    p.close()
    lib.fa_punc_uninit(None)


# ------------------------------------------------------------------------------------------------------------------ pooling
def test_pooled_calls_equal_each_call_alone():
    """16 threads, 6 seeded calls each of 1-4 random texts (0 to 1 500 words): every call's texts, ids and steps equal
    fa_punc_walk_host on that call alone, and the pool ran fewer steps than the calls' own steps summed."""
    rng = random.Random(11)
    reqs = []
    for _ in range(96):
        n = rng.randint(1, 4)
        reqs.append([random_text(rng, rng.choice([0, rng.randint(1, 60), rng.randint(1, 300), rng.randint(1, 1500)])) for _ in range(n)])
    want = [alone(r) for r in reqs]

    def score(ids, lens):
        time.sleep(0.0005)                                      # long enough for the other threads to queue behind a step
        return scripted(ids, 1, PROBS)
    p = HostPunc(score)
    got = [None] * len(reqs)
    bar = threading.Barrier(16)

    def run(j):
        bar.wait(WAIT)
        for k in range(j, len(reqs), 16):
            got[k] = p.infer(reqs[k])
    ts = [threading.Thread(target=run, args=(j,), daemon=True) for j in range(16)]
    for t in ts:
        t.start()
    join_all(ts)
    for r, w, g in zip(reqs, want, got):
        assert g == w, r
    calls, steps = p.stats()
    pooled = sum(1 for w in want if w[1] > 0)
    assert calls == pooled and steps < sum(w[1] for w in want)
    p.close()


def test_calls_join_at_a_step_boundary():
    """The scorer blocks inside step 3 of a 10-window call while three calls are posted: step 4 holds the long call's window and the
    three calls' first windows, and the one-window call returns while the long call still has windows left."""
    rng = random.Random(3)
    long_t, one, two, three = cjk_text(rng, 200), cjk_text(rng, 10), cjk_text(rng, 30), cjk_text(rng, 50)
    sc = Gated()
    entered, release = threading.Event(), threading.Event()
    sc.hooks[3] = lambda: (entered.set(), block_until(release)())
    p = HostPunc(sc)
    lead = Call(p, [long_t])
    lead.start()
    assert entered.wait(WAIT)
    posted = [Call(p, [t]) for t in (one, two, three)]
    for c in posted:
        c.start()
    time.sleep(0.5)                                             # let the three calls queue behind step 3
    sc.hooks[6] = block_until(posted[0].returned)               # step 6 waits until the one-window call has returned
    release.set()
    join_all([lead] + posted)
    assert sc.steps[4][0] == 4 and sc.steps[4][1][0] >= 20 and sorted(sc.steps[4][1][1:]) == [10, 20, 20]
    assert posted[0].t_end < lead.t_end and len(sc.steps) == 10
    for c, t in zip([lead] + posted, (long_t, one, two, three)):
        assert c.err is None and c.out == alone([t]), t
    assert lead.out[1] == 10 and posted[0].out[1] == 1
    assert p.stats() == (4, 10)
    p.close()


def test_leader_hands_off():
    """The first caller leads; its one-window call ends in the step during which two long calls were posted.  It returns, a waiter
    leads on from the next step, and both long calls complete with what they get alone."""
    rng = random.Random(4)
    short, longs = cjk_text(rng, 15), [cjk_text(rng, 150), cjk_text(rng, 90)]
    sc = Gated()
    entered, release = threading.Event(), threading.Event()
    sc.hooks[0] = lambda: (entered.set(), block_until(release)())
    p = HostPunc(sc)
    lead = Call(p, [short])
    lead.start()
    assert entered.wait(WAIT)
    posted = [Call(p, [t]) for t in longs]
    for c in posted:
        c.start()
    time.sleep(0.5)
    release.set()
    join_all([lead] + posted)
    assert lead.t_end < min(c.t_end for c in posted)
    assert lead.out == alone([short])
    for c, t in zip(posted, longs):
        assert c.err is None and c.out == alone([t])
    leader_thread = sc.steps[0][2]
    assert sc.steps[1][0] == 2 and all(s[2] != leader_thread for s in sc.steps[1:])
    assert p.stats() == (3, 9)
    p.close()


def _no_break(ids, lens):
    """scripted(), except that an unknown word (好 is not in the synthetic vocabulary) never ends a clause, so a window of them
    carries whole into the next one."""
    out = scripted(ids, 1, PROBS)
    out[ids == synth.punc_token_list().index("<unk>")] = 1
    return out


def test_an_over_long_window_fails_only_its_call():
    """With max_window 100, a call whose second text carries past 100 words fails among pooled calls with the message it gets alone
    (naming its own text 1), before the step's scorer runs; the other calls and the next call get what they get alone."""
    bad = ["你好" * 30, "好" * 300]
    with pytest.raises(Failed) as e:
        alone(bad, _no_break, max_window=100)
    msg = str(e.value)
    assert msg.startswith("text 1: window 5 holds 120 words")
    rng = random.Random(5)
    goods = [[cjk_text(rng, 400)], [cjk_text(rng, 37), cjk_text(rng, 120)]]
    entered, release = threading.Event(), threading.Event()

    def score(ids, lens):
        k = len(seen)
        seen.append(lens.tolist())
        if k == 1:
            entered.set()
            assert release.wait(WAIT)
        return _no_break(ids, lens)
    seen = []
    p = HostPunc(score, max_window=100)
    lead = Call(p, goods[0])
    lead.start()
    assert entered.wait(WAIT)
    posted = [Call(p, bad), Call(p, goods[1])]
    for c in posted:
        c.start()
    time.sleep(0.5)
    release.set()
    join_all([lead] + posted)
    assert posted[0].err == msg
    assert max(max(s) for s in seen) <= 100                     # the scorer never saw the refused window
    assert lead.out == alone(goods[0], _no_break, 100) and posted[1].out == alone(goods[1], _no_break, 100)
    assert p.infer(goods[1]) == posted[1].out                  # the handle serves the next call
    p.close()


def test_a_failing_step_fails_exactly_its_calls():
    """Step 3 fails: the three calls with a window in it fail with the scorer's message; a call posted during that step, so not in
    it, and the next call succeed."""
    rng = random.Random(6)
    long_t, a, b, d = cjk_text(rng, 200), cjk_text(rng, 60), cjk_text(rng, 25), cjk_text(rng, 45)
    sc = Gated()
    entered, release = threading.Event(), threading.Event()
    sc.hooks[2] = lambda: (entered.set(), block_until(release)())
    late = []

    def fail_step():
        late.append(Call(p, [d]))
        late[0].start()
        time.sleep(0.5)                                         # the late call queues behind the failing step
        return False
    sc.hooks[3] = fail_step
    p = HostPunc(sc)
    lead = Call(p, [long_t])
    lead.start()
    assert entered.wait(WAIT)
    posted = [Call(p, [a]), Call(p, [b])]
    for c in posted:
        c.start()
    time.sleep(0.5)
    release.set()
    join_all([lead] + posted)
    join_all(late)
    assert sc.steps[3][0] == 3
    for c in [lead] + posted:
        assert c.out is None and c.err == "scorer failed (7)"
    assert late[0].err is None and late[0].out == alone([d])
    assert p.infer([a]) == alone([a])
    calls, steps = p.stats()
    assert calls == 5 and steps == len(sc.steps) - 1           # the failed step is not counted
    p.close()
