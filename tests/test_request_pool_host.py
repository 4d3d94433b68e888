"""CPU: the request pool every pooled handle kind shares (funasr_b200/csrc/request_pool.h), compiled alone with g++ into a small driver
whose admit and round policies are scripted.  Tickets need some rounds each and carry an admission tag; a round appends itself to
every held ticket and ends those that have had their rounds, with a result naming the round.  Each scenario runs in its own process
with a timeout, and every wait inside the driver has one too, so a scheduling bug fails a test instead of hanging it."""
import os
import shutil
import subprocess

import pytest

from conftest import ROOT

DRIVER = r"""
#include "request_pool.h"
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <map>
#include <memory>
#include <stdexcept>
#include <thread>

using fa_handle::PoolTicket;
using fa_handle::RequestPool;

struct Tk : PoolTicket {
  int id = 0, tag = 0, steps = 1;        // the rounds it needs, its admission tag
  bool poison = false;                   // admit throws once, right after moving it
  int result = -1, ends = 0;             // written by the round that ends it
  std::vector<int> rounds;               // the rounds it was held in
};
using Q = std::deque<Tk*>;
using H = std::vector<Tk*>;

[[noreturn]] void fail(const std::string& m) {
  fprintf(stderr, "FAIL: %s\n", m.c_str());
  fflush(stderr);
  std::_Exit(1);
}
#define CHECK(c) do { if (!(c)) fail(std::string(#c) + " (line " + std::to_string(__LINE__) + ")"); } while (0)

void wait_for(const std::function<bool()>& pred, const char* what) {
  for (int i = 0; i < 20000; ++i) {
    if (pred()) return;
    std::this_thread::sleep_for(std::chrono::milliseconds(1));
  }
  fail(std::string("timed out waiting for ") + what);
}

struct Script {
  RequestPool<Tk> pool;
  bool by_tag = false;                   // admission: the head and every later ticket of its tag (the recogniser's); else in order
  size_t cap = 1 << 20;                  // held tickets at most after admission
  std::map<int, std::function<void()>> hooks;   // run at the start of round k; may throw.  Set before any call starts.
  std::atomic<int> started{0};
  int rounds = 0;                        // the rounds below are run by one leader at a time
  std::vector<std::thread::id> leader;   // per round

  size_t queued() {
    std::lock_guard<std::mutex> l(pool.mu);
    return pool.queue.size();
  }
  void admit(Q& q, H& held) {
    for (auto it = q.begin(); it != q.end() && held.size() < cap;) {
      Tk* t = *it;
      if (by_tag && !held.empty() && t->tag != held[0]->tag) { ++it; continue; }
      held.push_back(t);
      it = q.erase(it);
      if (t->poison) {
        t->poison = false;
        throw std::runtime_error("admit failed");
      }
    }
  }
  void run(H& held, H& ended) {
    const int k = rounds++;
    leader.push_back(std::this_thread::get_id());
    ++started;
    auto h = hooks.find(k);
    if (h != hooks.end()) h->second();
    CHECK(!held.empty() && held.size() <= cap);
    for (Tk* t : held) {
      CHECK(!by_tag || t->tag == held[0]->tag);
      t->rounds.push_back(k);
      if ((int)t->rounds.size() < t->steps) continue;
      t->result = t->id * 100000 + k;
      ++t->ends;
      ended.push_back(t);
    }
    held.erase(std::remove_if(held.begin(), held.end(), [](Tk* t) { return t->ends > 0; }), held.end());
    std::this_thread::sleep_for(std::chrono::microseconds(50));
  }
};

struct Call {
  Tk t;
  std::thread th;
  std::thread::id tid;
  std::atomic<bool> returned{false};
};

Call& post(Script& s, std::vector<std::unique_ptr<Call>>& calls, int steps, int tag = 0, bool poison = false) {
  calls.emplace_back(new Call());
  Call& c = *calls.back();
  c.t.id = (int)calls.size() - 1;
  c.t.steps = steps;
  c.t.tag = tag;
  c.t.poison = poison;
  c.th = std::thread([&s, &c] {
    c.tid = std::this_thread::get_id();
    s.pool.call(c.t, [&s](Q& q, H& h) { s.admit(q, h); }, [&s](H& h, H& e) { s.run(h, e); }, "pool-test: ");
    c.returned = true;
  });
  return c;
}

// post in a known order: each call waits in the queue before the next is posted.  Only while the leader is held in a hook, so the
// queue cannot drain; the hook's own wait covers the last call.
Call& post_queued(Script& s, std::vector<std::unique_ptr<Call>>& calls, int steps, int tag = 0, bool poison = false) {
  const size_t n = s.queued();
  Call& c = post(s, calls, steps, tag, poison);
  wait_for([&] { return s.queued() == n + 1; }, "a call to queue");
  return c;
}

void join(std::vector<std::unique_ptr<Call>>& calls) {
  for (auto& c : calls)
    if (c->th.joinable()) c->th.join();
}

// ended once, in its last consecutive round, with that round's result
void served(const Tk& t) {
  if (!t.err.empty()) fail("ticket " + std::to_string(t.id) + " failed: " + t.err);
  CHECK(t.done && t.ends == 1 && (int)t.rounds.size() == t.steps);
  for (size_t i = 1; i < t.rounds.size(); ++i) CHECK(t.rounds[i] == t.rounds[i - 1] + 1);
  CHECK(t.result == t.id * 100000 + t.rounds.back());
}

void idle(Script& s, int64_t calls) {
  std::lock_guard<std::mutex> l(s.pool.mu);
  CHECK(!s.pool.busy && s.pool.queue.empty() && s.pool.held.empty() && (calls < 0 || s.pool.calls == calls));
}

// 16 threads, 30 calls each, posted as fast as they return
void many(bool by_tag) {
  Script s;
  s.by_tag = by_tag;
  s.cap = by_tag ? 6 : 5;
  std::vector<Tk> ts(16 * 30);
  std::vector<std::thread> th;
  for (int j = 0; j < 16; ++j)
    th.emplace_back([&, j] {
      for (int i = j; i < (int)ts.size(); i += 16) {
        ts[i].id = i;
        ts[i].steps = by_tag ? 1 : 1 + i % 4;
        ts[i].tag = i % 3;
        s.pool.call(ts[i], [&s](Q& q, H& h) { s.admit(q, h); }, [&s](H& h, H& e) { s.run(h, e); }, "pool-test: ");
      }
    });
  for (auto& t : th) t.join();
  for (const Tk& t : ts) served(t);
  idle(s, (int64_t)ts.size());
}

int main(int argc, char** argv) {
  const std::string sc = argc > 1 ? argv[1] : "";
  Script s;
  std::vector<std::unique_ptr<Call>> c;
  c.reserve(8);                          // hooks read c[0] while later calls are posted
  if (sc == "many_steps") {
    many(false);
  } else if (sc == "many_passes") {
    many(true);
  } else if (sc == "skip") {
    // round 0 holds A while B (tag 1), C (tag 0), D (tag 1) queue: round 1 takes B and D and skips C, which round 2 takes
    s.by_tag = true;
    s.hooks[0] = [&] { wait_for([&] { return s.queued() == 3; }, "three calls to queue"); };
    post(s, c, 1, 0);
    wait_for([&] { return s.started > 0; }, "round 0");
    post_queued(s, c, 1, 1);
    post_queued(s, c, 1, 0);
    post(s, c, 1, 1);
    join(c);
    for (auto& x : c) served(x->t);
    CHECK(c[1]->t.rounds == std::vector<int>{1} && c[3]->t.rounds == std::vector<int>{1} && c[2]->t.rounds == std::vector<int>{2});
    idle(s, 4);
  } else if (sc == "join") {
    // B posted during round 2 of A's five is held from round 3 on, beside A
    s.hooks[2] = [&] { wait_for([&] { return s.queued() == 1; }, "B to queue"); };
    post(s, c, 5);
    wait_for([&] { return s.started > 2; }, "round 2");
    post(s, c, 2);
    join(c);
    for (auto& x : c) served(x->t);
    CHECK(c[0]->t.rounds == (std::vector<int>{0, 1, 2, 3, 4}) && c[1]->t.rounds == (std::vector<int>{3, 4}));
    idle(s, 2);
  } else if (sc == "handoff") {
    // A's call ends in round 0, while B and C queue: A returns, and round 2 runs only once it has, on another thread
    s.hooks[0] = [&] { wait_for([&] { return s.queued() == 2; }, "B and C to queue"); };
    s.hooks[2] = [&] { wait_for([&] { return c[0]->returned.load(); }, "the first leader to return"); };
    post(s, c, 1);
    wait_for([&] { return s.started > 0; }, "round 0");
    post_queued(s, c, 3);
    post(s, c, 2);
    join(c);
    for (auto& x : c) served(x->t);
    CHECK(s.leader[0] == c[0]->tid);
    for (size_t k = 1; k < s.leader.size(); ++k) CHECK(s.leader[k] != c[0]->tid);
    CHECK(c[1]->t.rounds == (std::vector<int>{1, 2, 3}) && c[2]->t.rounds == (std::vector<int>{1, 2}));
    idle(s, 3);
  } else if (sc == "round_throws") {
    // round 1 holds A and B and throws while C queues: A and B end with the message, C is led on, and the next call is served
    s.hooks[0] = [&] { wait_for([&] { return s.queued() == 1; }, "B to queue"); };
    s.hooks[1] = [&] {
      wait_for([&] { return s.queued() == 1; }, "C to queue");
      throw std::runtime_error("boom");
    };
    post(s, c, 4);
    wait_for([&] { return s.started > 0; }, "round 0");
    post(s, c, 4);
    wait_for([&] { return s.started > 1; }, "round 1");
    post(s, c, 2);
    join(c);
    for (int i = 0; i < 2; ++i) CHECK(c[i]->t.done && c[i]->t.err == "pool-test: boom" && c[i]->t.ends == 0);
    served(c[2]->t);
    CHECK(c[2]->t.rounds == (std::vector<int>{2, 3}));
    post(s, c, 1);
    join(c);
    served(c[3]->t);
    idle(s, 4);
  } else if (sc == "admit_throws") {
    // round 0 holds A while B, C and D queue; the next admission moves B and C, then throws: both end with the message, D is served
    s.hooks[0] = [&] { wait_for([&] { return s.queued() == 3; }, "three calls to queue"); };
    s.cap = 3;
    post(s, c, 1);
    wait_for([&] { return s.started > 0; }, "round 0");
    post_queued(s, c, 2);
    post_queued(s, c, 2, 0, true);
    post(s, c, 1);
    join(c);
    served(c[0]->t);
    for (int i = 1; i < 3; ++i) CHECK(c[i]->t.done && c[i]->t.err == "pool-test: admit failed" && c[i]->t.rounds.empty());
    served(c[3]->t);
    idle(s, -1);
  } else {
    fail("unknown scenario " + sc);
  }
  printf("ok\n");
  return 0;
}
"""

SCENARIOS = {
    "many_steps": "16 threads, admission held across rounds (the punctuation pattern): every ticket ends once with its round's result",
    "many_passes": "16 threads, one pass per round with the head's tag only (the recogniser pattern): every ticket ends once",
    "skip": "a ticket the policy skips stays queued and is led in a later round",
    "join": "a ticket posted during a round joins the held tickets at the next round boundary",
    "handoff": "the leader returns once its own ticket ends, and a waiter leads on",
    "round_throws": "a round that throws ends exactly the held tickets with the message; queued tickets and the next call are served",
    "admit_throws": "an admit that throws after moving tickets ends them with the message; none waits forever",
}


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    d = tmp_path_factory.mktemp("request_pool")
    src, exe = d / "driver.cpp", str(d / "driver")
    src.write_text(DRIVER)
    # hidden visibility, as the header's namespace has: the driver's ticket type derives from PoolTicket
    r = subprocess.run(["g++", "-std=c++17", "-pthread", "-O1", "-Wall", "-Wextra", "-fvisibility=hidden",
                        "-I" + os.path.join(ROOT, "funasr_b200", "csrc"), str(src), "-o", exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and not r.stdout.strip(), r.stdout
    return exe


@pytest.mark.parametrize("scenario", sorted(SCENARIOS))
def test_request_pool(driver, scenario):
    try:
        r = subprocess.run([driver, scenario], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=60)
    except subprocess.TimeoutExpired:
        pytest.fail(scenario + ": the driver hung (" + SCENARIOS[scenario] + ")")
    assert r.returncode == 0 and r.stdout.strip() == "ok", SCENARIOS[scenario] + "\n" + r.stdout
