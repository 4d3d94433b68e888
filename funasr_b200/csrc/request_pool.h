// The request pool of a handle many threads share (the recogniser's, the speaker model's, punctuation's): concurrent calls post
// tickets, and whichever thread finds no leader runs rounds over them for every caller.  Standard headers only, so a host test can
// compile it alone.
//
// A call posts its ticket and waits.  The thread that finds no leader leads: it runs rounds until its own ticket is done, then gives
// up leadership and wakes the waiters, one of which leads on.  In a round the handle's admit policy, under mu, moves queued tickets
// into held; the handle's round, outside mu, runs over held and moves every ticket that ended (a result, or err set) to a list the
// pool marks done under mu, waking their threads.  A ticket is always in the queue, in held, in that list or done, and each move
// pushes it before erasing it, so whatever throws, the pool still reaches it: a round or an admit that throws ends every held ticket
// with its message, and the pool serves the next call.  No thread is created.
#pragma once
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <deque>
#include <exception>
#include <mutex>
#include <string>
#include <vector>

namespace __attribute__((visibility("hidden"))) fa_handle {

// What the pool knows of a call; each handle's ticket derives from it.  Written by the leader, read by the owner once done.
struct PoolTicket {
  std::string err;                                   // set: the call failed with this message
  bool done = false;
};

template <class T>
struct RequestPool {
  std::mutex mu;                                     // guards queue, held, busy and every ticket's done
  std::condition_variable cv;
  std::deque<T*> queue;                              // posted, not admitted, in arrival order
  std::vector<T*> held;                              // admitted by a leader, not yet ended
  bool busy = false;                                 // a thread leads
  std::atomic<int64_t> calls{0};                     // tickets admitted since init

  // t's call: posted, then this thread waits, or leads rounds until t is done.  t failed when t.err is set on return; no exception
  // leaves.
  //   admit(queue, held): under mu, moves tickets from queue into held (at least one when held is empty), each pushed before erased.
  //   run(held, ended): outside mu, one round; every ticket that ended moves from held to ended, pushed before erased.
  //   what: the prefix of the message a ticket gets when a round or an admit throws.
  template <class Admit, class Run>
  void call(T& t, Admit admit, Run run, const char* what) {
    std::unique_lock<std::mutex> q(mu, std::defer_lock);
    bool posted = false;
    try {
      q.lock();
      queue.push_back(&t);
      posted = true;
      while (!t.done) {
        if (busy) {                                  // a leader is running rounds: it may admit t
          cv.wait(q);
          continue;
        }
        busy = true;
        std::vector<T*> ended;
        try {
          while (!t.done) {
            const size_t before = held.size();
            admit(queue, held);
            calls += (int64_t)(held.size() - before);
            q.unlock();
            run(held, ended);
            q.lock();
            for (T* e : ended) e->done = true;
            if (!ended.empty()) cv.notify_all();
            ended.clear();                           // their owners may return and free them once mu is released
          }
        } catch (const std::exception& e) {
          if (!q.owns_lock()) q.lock();
          const std::string msg = std::string(what) + e.what();
          for (T* h : held) {
            if (h->err.empty()) h->err = msg;
            h->done = true;
          }
          for (T* h : ended) h->done = true;
          held.clear();
        }
        busy = false;
        cv.notify_all();
      }
    } catch (const std::exception& e) {
      // this thread's own post failed: its ticket leaves the queue, or, admitted already, is waited for; the call fails either way
      try {
        if (!q.owns_lock()) q.lock();
        auto it = std::find(queue.begin(), queue.end(), &t);
        if (it != queue.end()) queue.erase(it);
        else if (posted) cv.wait(q, [&] { return t.done; });
        t.err = std::string(what) + e.what();
        t.done = true;
      } catch (const std::exception&) {
      }
    }
  }
};

}  // namespace fa_handle
