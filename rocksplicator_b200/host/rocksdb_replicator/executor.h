// executor.h — a fixed thread pool plus one timer thread (std only).  Stands in for the reference's
// folly CPUThreadPoolExecutor "rptor-worker-" (rocksdb_replicator/rocksdb_replicator.cpp:58-67) and for
// the EventBase::runAfterDelay / futures::sleep calls on the replication path (replicated_db.cpp:412-428,
// non_blocking_condition_variable.h:113-126).
//
// Every worker owns a queue (its own mutex and condition variable); add() deals tasks round-robin and an idle worker
// steals from the others before it sleeps; a sleeping worker is woken only when the awake ones are outnumbered by the
// queued tasks.  With one shared queue the pull loops of a thousand shards — three short
// tasks per ReplicateResponse — serialise on that queue's mutex long before the workers are busy.
#pragma once
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

namespace replicator {

class Executor {
 public:
  explicit Executor(size_t n_threads) : n_(n_threads ? n_threads : 1) {
    for (size_t i = 0; i < n_; i++) q_.emplace_back(new Queue());
    for (size_t i = 0; i < n_; i++) workers_.emplace_back([this, i] { WorkLoop(i); });
    timer_ = std::thread([this] { TimerLoop(); });
  }
  ~Executor() { Stop(); }
  void add(std::function<void()> f) {
    if (stop_.load(std::memory_order_acquire)) return;
    Queue& q = *q_[next_.fetch_add(1, std::memory_order_relaxed) % n_];
    {
      std::lock_guard<std::mutex> g(q.mu);
      q.tasks.push_back(std::move(f));
    }
    const int64_t queued = queued_.fetch_add(1, std::memory_order_acq_rel) + 1;
    // Wake a worker only when the ones already awake will not get to the task soon: a wake-up and the sleep after it
    // cost more CPU time than a short task, and a container's CPU time may be capped.  An awake worker drains its own queue and steals from the others before it sleeps.
    const int64_t awake = (int64_t)n_ - sleepers_.load(std::memory_order_acquire);
    if (awake <= 0 || queued > 2 * awake) {
      if (q.sleeping.load(std::memory_order_acquire)) q.cv.notify_one();
      else WakeOne();
    }
  }
  // run f on the pool after delay_ms
  void addDelayed(std::function<void()> f, uint64_t delay_ms) {
    const auto when = std::chrono::steady_clock::now() + std::chrono::milliseconds(delay_ms);
    {
      std::lock_guard<std::mutex> g(tmu_);
      if (stop_.load()) return;
      timed_.emplace(when, std::move(f));
    }
    tcv_.notify_one();
  }
  void Stop() {
    if (stop_.exchange(true)) return;
    for (auto& q : q_) {
      std::lock_guard<std::mutex> g(q->mu);
      q->cv.notify_all();
    }
    {
      std::lock_guard<std::mutex> g(tmu_);
      tcv_.notify_all();
    }
    for (auto& t : workers_) t.join();
    timer_.join();
  }

 private:
  struct Queue {
    std::mutex mu;
    std::condition_variable cv;
    std::deque<std::function<void()>> tasks;
    std::atomic<bool> sleeping{false};
  };
  bool Pop(Queue& q, std::function<void()>* f, bool try_only) {
    std::unique_lock<std::mutex> l(q.mu, std::defer_lock);
    if (try_only) {
      if (!l.try_lock()) return false;
    } else {
      l.lock();
    }
    if (q.tasks.empty()) return false;
    *f = std::move(q.tasks.front());
    q.tasks.pop_front();
    return true;
  }
  void WakeOne() {
    for (auto& q : q_)
      if (q->sleeping.load(std::memory_order_acquire)) {
        std::lock_guard<std::mutex> g(q->mu);
        q->cv.notify_one();
        return;
      }
  }
  void WorkLoop(size_t me) {
    Queue& mine = *q_[me];
    for (;;) {
      std::function<void()> f;
      bool got = Pop(mine, &f, false);
      for (size_t k = 1; !got && k < n_ && queued_.load(std::memory_order_acquire) > 0; k++) got = Pop(*q_[(me + k) % n_], &f, true);
      if (got) {
        queued_.fetch_sub(1, std::memory_order_acq_rel);
        f();
        continue;
      }
      std::unique_lock<std::mutex> l(mine.mu);
      if (stop_.load(std::memory_order_acquire)) return;
      if (!mine.tasks.empty()) continue;
      mine.sleeping.store(true, std::memory_order_release);
      sleepers_.fetch_add(1, std::memory_order_acq_rel);
      // (a bounded sleep: a task dealt to a busy worker's queue is found by the next idle worker at the latest then)
      if (queued_.load(std::memory_order_acquire) == 0) mine.cv.wait_for(l, std::chrono::milliseconds(2));
      sleepers_.fetch_sub(1, std::memory_order_acq_rel);
      mine.sleeping.store(false, std::memory_order_release);
      if (stop_.load(std::memory_order_acquire) && mine.tasks.empty()) return;
    }
  }
  void TimerLoop() {
    std::unique_lock<std::mutex> l(tmu_);
    for (;;) {
      if (stop_.load()) return;
      if (timed_.empty()) {
        tcv_.wait(l);
        continue;
      }
      const auto when = timed_.begin()->first;
      if (std::chrono::steady_clock::now() < when) {
        tcv_.wait_until(l, when);
        continue;
      }
      auto f = std::move(timed_.begin()->second);
      timed_.erase(timed_.begin());
      l.unlock();
      add(std::move(f));
      l.lock();
    }
  }
  const size_t n_;
  std::vector<std::unique_ptr<Queue>> q_;
  std::atomic<size_t> next_{0};
  std::atomic<int64_t> queued_{0};
  std::atomic<int> sleepers_{0};
  std::atomic<bool> stop_{false};
  std::mutex tmu_;
  std::condition_variable tcv_;
  std::multimap<std::chrono::steady_clock::time_point, std::function<void()>> timed_;
  std::vector<std::thread> workers_;
  std::thread timer_;
};

}  // namespace replicator
