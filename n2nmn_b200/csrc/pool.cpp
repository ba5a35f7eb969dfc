// Native host runtime for keeping several batches in flight: one worker thread per context, and
// dynamic batching of whatever is queued.
//
// A step's host work (layout compile ~10 us, table upload, three launches) is about as long as its
// GPU work at batch 64, and ONE batch of 64 questions is ~4 us of tensor work — far too little to
// fill the SMs per launch. So every context (= stream) has its own worker thread with a job queue;
// n2nmn_pool_submit only copies the token matrix into a job and returns, and a worker takes up to
// n2nmn_max_group(ctx) queued jobs of identical shape at a time and evaluates them with ONE set of
// launches (n2nmn_forward_group): the contraction kernel then walks several tiles per CTA and
// its TMA ring fills for the next tile while an epilogue runs. A worker never waits for more jobs: with one job
// queued it runs one. There is no reference counterpart: the reference's executor is a Python loop
// around session.run (exp_clevr/eval_clevr.py:96-133), one batch at a time.
//
// Uses nothing but the public C ABI of include/n2nmn_b200.h (and the segment limit of common.cuh).
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/n2nmn_b200.h"
#include "common.cuh"

namespace {

struct Job {
  const float* feat;
  const float* wv;
  std::vector<int32_t> tokens;
  int T, N;
  float* scores;
  uint8_t* validity;
  int host_io;
};

struct Worker {
  n2nmn_ctx* ctx = nullptr;
  void* stream = nullptr;
  int max_group = 1;
  std::thread th;
  std::mutex mu;
  std::condition_variable cv;
  std::deque<Job> q;
  std::atomic<int> qsize{0};   // mirrors q.size() so that an idle worker can poll without the lock
  bool stop = false;
};

// An idle worker polls its queue for this long before it sleeps on the condition variable: a
// step is ~10 us of host work, a futex wake-up is 50-100 us, so a sleeping worker turns a short
// burst of submissions (the driver's --steps 20) into a measurement of wake-up latency.
constexpr int kSpinMicros = 300;
constexpr int kMaxGroup = n2nmn::kMaxSeg;   // batches one set of launches may cover

inline void cpu_relax() {
#if defined(__x86_64__) || defined(__i386__)
  __builtin_ia32_pause();
#elif defined(__aarch64__)
  asm volatile("yield" ::: "memory");
#endif
}

}  // namespace

struct n2nmn_pool {
  std::vector<Worker*> workers;
  std::vector<int32_t> vocab;
  uint64_t next = 0;          // cursor of n2nmn_pool_submit_many
  int deal = 1;               // consecutive jobs dealt to one worker before moving to the next
  std::mutex done_mu;
  std::condition_variable done_cv;
  std::atomic<int64_t> pending{0};   // jobs queued or running
  std::atomic<int64_t> groups{0}, grouped_jobs{0};
  int err_code = 0;           // first failure since the last wait
  std::string err_msg;
};

namespace {

thread_local std::string g_pool_err;

void run_group(n2nmn_pool* p, Worker* w, std::vector<Job>& js) {
  const int n = (int)js.size();
  const float* feat[kMaxGroup];
  const float* wv[kMaxGroup];
  const int32_t* tok[kMaxGroup];
  float* scores[kMaxGroup];
  uint8_t* valid[kMaxGroup];
  for (int i = 0; i < n; ++i) {
    feat[i] = js[i].feat; wv[i] = js[i].wv; tok[i] = js[i].tokens.data();
    scores[i] = js[i].scores; valid[i] = js[i].validity;
  }
  const Job& j0 = js[0];
  int rc;
  if (j0.host_io == 2)
    rc = n2nmn_forward_group_host_f16_async(w->ctx, n, reinterpret_cast<const uint16_t* const*>(feat),
                                            wv, tok, j0.T, j0.N, p->vocab.data(),
                                            (int)p->vocab.size(), scores, valid, w->stream);
  else if (j0.host_io)
    rc = n2nmn_forward_group_host_async(w->ctx, n, feat, wv, tok, j0.T, j0.N, p->vocab.data(),
                                        (int)p->vocab.size(), scores, valid, w->stream);
  else
    rc = n2nmn_forward_group(w->ctx, n, feat, wv, tok, j0.T, j0.N, p->vocab.data(),
                             (int)p->vocab.size(), scores, valid, w->stream);
  p->groups.fetch_add(1, std::memory_order_relaxed);
  p->grouped_jobs.fetch_add(n, std::memory_order_relaxed);
  std::lock_guard<std::mutex> lk(p->done_mu);
  if (rc != 0 && p->err_code == 0) {
    p->err_code = rc;
    p->err_msg = n2nmn_last_error();
  }
  if (p->pending.fetch_sub(n) == n) p->done_cv.notify_all();
}

void worker_main(n2nmn_pool* p, Worker* w) {
  std::vector<Job> js;
  for (;;) {
    if (w->qsize.load(std::memory_order_acquire) == 0) {   // stay hot for a while
      const auto t_end = std::chrono::steady_clock::now() + std::chrono::microseconds(kSpinMicros);
      while (w->qsize.load(std::memory_order_acquire) == 0 &&
             std::chrono::steady_clock::now() < t_end)
        for (int i = 0; i < 64; ++i) cpu_relax();
    }
    js.clear();
    {
      std::unique_lock<std::mutex> lk(w->mu);
      w->cv.wait(lk, [&] { return w->stop || !w->q.empty(); });
      if (w->q.empty()) return;   // stop requested and nothing left
      // whatever is queued right now, up to the context's group capacity, same shape only
      js.push_back(std::move(w->q.front()));
      w->q.pop_front();
      while ((int)js.size() < w->max_group && !w->q.empty()) {
        const Job& nx = w->q.front();
        if (nx.T != js[0].T || nx.N != js[0].N || nx.host_io != js[0].host_io) break;
        js.push_back(std::move(w->q.front()));
        w->q.pop_front();
      }
      w->qsize.store((int)w->q.size(), std::memory_order_release);
    }
    run_group(p, w, js);
  }
}

}  // namespace

extern "C" {

const char* n2nmn_pool_last_error(void) { return g_pool_err.c_str(); }

int n2nmn_pool_create(n2nmn_ctx** ctxs, void** streams, int num, const int32_t* vocab_ops,
                      int num_vocab, n2nmn_pool** out) {
  if (!ctxs || !streams || !vocab_ops || !out || num <= 0 || num_vocab <= 0) {
    g_pool_err = "n2nmn_pool_create: bad argument";
    return N2NMN_ERR_ARG;
  }
  n2nmn_pool* p = new n2nmn_pool();
  p->vocab.assign(vocab_ops, vocab_ops + num_vocab);
  int g = kMaxGroup;
  for (int i = 0; i < num; ++i) {
    Worker* w = new Worker();
    w->ctx = ctxs[i];
    w->stream = streams[i];
    w->max_group = std::max(1, std::min(n2nmn_max_group(ctxs[i]), kMaxGroup));
    g = std::min(g, w->max_group);
    p->workers.push_back(w);
  }
  p->deal = g;   // a run of `deal` consecutive jobs lands in one queue -> one full group
  for (Worker* w : p->workers) w->th = std::thread(worker_main, p, w);
  *out = p;
  return 0;
}

int n2nmn_pool_destroy(n2nmn_pool* p) {
  if (!p) return 0;
  for (Worker* w : p->workers) {
    {
      std::lock_guard<std::mutex> lk(w->mu);
      w->stop = true;
    }
    w->cv.notify_all();
  }
  for (Worker* w : p->workers) {
    if (w->th.joinable()) w->th.join();
    delete w;
  }
  delete p;
  return 0;
}

int n2nmn_pool_size(const n2nmn_pool* p) { return p ? (int)p->workers.size() : 0; }

int n2nmn_pool_submit(n2nmn_pool* p, int slot, const float* feat, const float* wv,
                      const int32_t* tokens, int T, int N, float* scores, uint8_t* validity_out,
                      int host_io) {
  if (!p || !feat || !wv || !tokens || !scores || slot < 0 || slot >= (int)p->workers.size() ||
      T <= 0 || N <= 0) {
    g_pool_err = "n2nmn_pool_submit: bad argument";
    return N2NMN_ERR_ARG;
  }
  Job j;
  j.feat = feat; j.wv = wv; j.T = T; j.N = N; j.scores = scores; j.validity = validity_out;
  j.host_io = host_io;
  j.tokens.assign(tokens, tokens + (size_t)T * N);
  p->pending.fetch_add(1);
  Worker* w = p->workers[slot];
  {
    std::lock_guard<std::mutex> lk(w->mu);
    w->q.push_back(std::move(j));
    w->qsize.store((int)w->q.size(), std::memory_order_release);
  }
  w->cv.notify_one();
  return 0;
}

int n2nmn_pool_submit_many(n2nmn_pool* p, int n, const float* const* feat,
                           const float* const* wv, const int32_t* const* tokens, int T, int N,
                           float* const* scores, uint8_t* const* validity_out, int host_io) {
  if (!p || n < 0 || (n > 0 && (!feat || !wv || !tokens || !scores))) {
    g_pool_err = "n2nmn_pool_submit_many: bad argument";
    return N2NMN_ERR_ARG;
  }
  const uint64_t K = p->workers.size();
  for (int i = 0; i < n; ++i) {
    const int slot = (int)((p->next++ / (uint64_t)p->deal) % K);
    if (int rc = n2nmn_pool_submit(p, slot, feat[i], wv[i], tokens[i], T, N, scores[i],
                                   validity_out ? validity_out[i] : nullptr, host_io))
      return rc;
  }
  return 0;
}

int n2nmn_pool_wait(n2nmn_pool* p) {
  if (!p) return 0;
  {   // the workers are usually a few microseconds from done: poll before sleeping
    const auto t_end = std::chrono::steady_clock::now() + std::chrono::microseconds(kSpinMicros);
    while (p->pending.load() != 0 && std::chrono::steady_clock::now() < t_end)
      for (int i = 0; i < 64; ++i) cpu_relax();
  }
  std::unique_lock<std::mutex> lk(p->done_mu);
  p->done_cv.wait(lk, [&] { return p->pending.load() == 0; });
  const int rc = p->err_code;
  if (rc != 0) g_pool_err = p->err_msg;
  p->err_code = 0;
  p->err_msg.clear();
  return rc;
}

int n2nmn_pool_group_stats(const n2nmn_pool* p, int64_t* groups, int64_t* jobs) {
  if (!p) return N2NMN_ERR_ARG;
  if (groups) *groups = p->groups.load();
  if (jobs) *jobs = p->grouped_jobs.load();
  return 0;
}

}  // extern "C"
