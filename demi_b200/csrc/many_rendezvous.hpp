// many_rendezvous.hpp — many recursive minimisations side by side, their evaluations served together.
//
// A DDMin driver (ddmin_driver.hpp) asks for one speculative batch at a time and waits for it; a batch of one trace is
// a small fraction of a launch.  Here the drivers of many traces run on host threads with a rendezvous: every driver
// in flight runs until it asks for an evaluation or finishes, then the coordinator (the calling thread) serves the
// union of their requests and each gets its own slice back.  A driver sees exactly the answers it would get alone, so
// its decisions, MCS and counters do not depend on which other drivers share its launches.  demi_ddmin_many (STSSched
// replays) and demi_incremental_ddmin_many (resumable DPOR instances) are run this way.  Host-only.
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstdlib>
#include <functional>
#include <mutex>
#include <new>
#include <string>
#include <system_error>
#include <thread>
#include <vector>
#include "engine.hpp"

namespace demi {

// host threads a call may run at once
constexpr uint32_t MANY_MAX_WINDOW = 4096;

// A driver's request for an evaluation: n tests of trace `trace`, their masks (a slice of the driver's arena, which
// stays put while it waits) and whatever else the serving step reads (`payload`, the driver's own), and once served,
// their results or the launch's error.
template <class Res>
struct ManyRequest {
  uint32_t trace; const uint64_t* masks; size_t n;
  const void* payload = nullptr;
  std::vector<Res> res;
  int32_t rc = DEMI_OK; bool done = false;
};

template <class Res>
struct Rendezvous {
  std::mutex mu;
  std::condition_variable coord, work;
  uint32_t running = 0;            // workers executing driver code; the others wait on a request or have left
  std::vector<ManyRequest<Res>*> queue;

  // called from a driver's evaluate(): queues q and waits until the coordinator has served it
  void submit(ManyRequest<Res>& q) {
    std::unique_lock<std::mutex> lk(mu);
    queue.push_back(&q);
    running--;
    coord.notify_one();
    work.wait(lk, [&] { return q.done; });
  }
};

// A round's requests as one list of tests, in request order: the trace of each test, and its masks of mask_words words
template <class Res>
void flatten_requests(const std::vector<ManyRequest<Res>*>& batch, uint32_t mask_words, std::vector<uint32_t>& tr,
                      std::vector<uint64_t>& masks) {
  tr.clear(); masks.clear();
  for (const ManyRequest<Res>* q : batch) {
    tr.insert(tr.end(), q->n, q->trace);
    masks.insert(masks.end(), q->masks, q->masks + q->n * mask_words);
  }
}

// Hands each request its slice of `res`, the results of the round's tests in request order
template <class Res>
void scatter_results(const std::vector<ManyRequest<Res>*>& batch, const std::vector<Res>& res) {
  size_t k = 0;
  for (ManyRequest<Res>* q : batch) {
    q->res.assign(res.begin() + k, res.begin() + k + q->n);
    k += q->n;
  }
}

// "<who>: trace <t>: <msg>", how a call over many traces reports trace t's failure
inline std::string trace_msg(const char* who, uint32_t t, const std::string& msg) {
  return std::string(who) + ": trace " + std::to_string(t) + ": " + msg;
}

// Drivers in flight: DEMI_DDMIN_MANY_WINDOW, 1..MANY_MAX_WINDOW (default 512), at most n.  It bounds both
// demi_ddmin_many and demi_incremental_ddmin_many.
inline int32_t many_window(demi_handle* h, uint32_t n, uint32_t& window) {
  window = 512;
  if (const char* w = getenv("DEMI_DDMIN_MANY_WINDOW")) {
    char* end = nullptr;
    const long v = strtol(w, &end, 10);
    if (end == w || *end || v < 1 || v > (long)MANY_MAX_WINDOW)
      return fail(h, DEMI_ERR_INVALID, "DEMI_DDMIN_MANY_WINDOW=%s: expected 1..%u", w, MANY_MAX_WINDOW);
    window = (uint32_t)v;
  }
  window = std::min(window, n);
  return DEMI_OK;
}

// Runs drive(t, eh) for every trace t < n on `window` worker threads (a thread that finishes a driver takes the next
// trace); status[t] is what it returns.  fail() records a message on the handle it is given: each worker's drivers get
// a handle of their own (eh) for that, so that the message of each failing trace is kept.  Meanwhile the calling
// thread serves every round's queued requests with serve(batch), which fills each request's res; once a serve fails,
// it is not called again and every request gets its code.  A driver out of host memory fails its trace alone with
// DEMI_ERR_CAPACITY.  Returns the failed serve's code (its message in h->err), else DEMI_OK with the message of the
// lowest failing trace in h->err.
template <class Res>
int32_t run_many(demi_handle* h, const char* who, uint32_t n, uint32_t window,
                 const std::function<int32_t(uint32_t, Rendezvous<Res>&, demi_handle*)>& drive,
                 const std::function<int32_t(std::vector<ManyRequest<Res>*>&)>& serve, int32_t* status) {
  Rendezvous<Res> R;
  std::atomic<uint32_t> next{0};
  std::vector<std::string> msg(n);
  auto worker = [&]() {
    demi_handle eh;
    for (uint32_t t; (t = next.fetch_add(1)) < n;) {
      try {
        eh.err.clear();
        status[t] = drive(t, R, &eh);
        if (status[t] != DEMI_OK) msg[t] = eh.err;
      } catch (const std::bad_alloc&) {
        status[t] = DEMI_ERR_CAPACITY;
        msg[t] = std::string(who) + ": out of host memory";
      }
    }
    std::lock_guard<std::mutex> lk(R.mu);
    R.running--;
    R.coord.notify_one();
  };
  int32_t call_rc = DEMI_OK;
  std::string call_msg;
  std::vector<std::thread> threads;
  {
    std::unique_lock<std::mutex> lk(R.mu);
    // the workers are counted before any of them can take the lock; when the system refuses a thread, the ones already
    // started carry the window (the results do not depend on it)
    try {
      threads.reserve(window);
      for (uint32_t i = 0; i < window; i++) threads.emplace_back(worker);
    } catch (const std::system_error&) {
    } catch (const std::bad_alloc&) {
    }
    R.running = (uint32_t)threads.size();
    if (threads.empty()) return fail(h, DEMI_ERR_CAPACITY, "%s: could not start a worker thread", who);
    for (;;) {
      R.coord.wait(lk, [&] { return R.running == 0; });
      if (R.queue.empty()) break;                  // no driver waits and none runs: every trace is done
      std::vector<ManyRequest<Res>*> batch;
      batch.swap(R.queue);
      lk.unlock();
      int32_t rc = call_rc;
      if (rc == DEMI_OK) {
        rc = serve(batch);
        if (rc != DEMI_OK) { call_rc = rc; call_msg = h->err; }
      }
      for (ManyRequest<Res>* q : batch) q->rc = rc;
      lk.lock();
      for (ManyRequest<Res>* q : batch) q->done = true;
      R.running += (uint32_t)batch.size();
      R.work.notify_all();
    }
  }
  for (std::thread& th : threads) th.join();
  if (call_rc != DEMI_OK) { h->err = call_msg; return call_rc; }
  for (uint32_t t = 0; t < n; t++)
    if (status[t] != DEMI_OK) { h->err = msg[t]; break; }
  return DEMI_OK;
}

}  // namespace demi
