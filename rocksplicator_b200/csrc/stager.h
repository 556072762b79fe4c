// stager.h — multi-buffered staging combiner (std only, no CUDA): many caller threads, one device batch at a time.
//
// Why: the reference calls ApplicationDB::Get / MultiGet from up to 256 thrift worker threads
// (rocksdb_admin/application_db.cpp:85-120, examples/counter_service/counter.cpp:39,81) and applies replicated
// updates from >= 16 executor threads (rocksdb_replicator/rocksdb_replicator.cpp:58-67).  A device batch costs the same
// launch + synchronisation whether it carries 1 request or 100 000, so concurrent callers share batches:
//
//   caller:      begin()  -> a slice of the OPEN batch's pinned staging (items + bytes)
//                copy its own inputs into the slice, in parallel with every other caller
//                commit() -> wait() until the batch has run -> read its own results -> release()
//   dispatcher:  one thread; as soon as it is idle and the open batch is not empty it CLOSES it (another buffer
//                opens for new arrivals), waits for the callers still copying, runs the batch (H2D, kernels, D2H,
//                one synchronisation — the RunFn), fires the asynchronous completions and publishes the batch's epoch.
//
// While the device works on batch k, callers fill batch k+1 and the callers of batch k-1 are still copying their results
// out (four buffers): batches grow with load on their own (no timer).  Requests of one caller thread stay ordered (it
// does not return before its request has run); slices of one batch are ordered by begin() order, which is what
// per-shard FIFO needs.
//
// Synchronisation.  The OPEN batch is one 64-bit word — buffer | class | items reserved | bytes reserved — and a
// reservation is one compare-and-swap on it: hundreds of callers arriving together (every caller of a batch comes back
// at the same moment) do not queue on a lock.  (With the reservation under the spin lock, hundreds of Get callers spent
// most of their CPU time spinning for that lock.)
// Only the transitions of a BUFFER (close, open, free) take the spin lock, and only the dispatcher and the last
// caller out of a batch make them.  The dispatcher knows a closed batch is complete when the items committed equal the
// items reserved, and a buffer is free again when the items released do.
// A caller waits for its batch with a short spin and then sleeps on one of the batch's futex words (sleepers are spread
// over kWakeWords words: the kernel hashes a futex by its address, and hundreds of threads waiting on and waking ONE
// word queue on one hash-bucket lock); the dispatcher wakes a few sleepers per word and every woken caller wakes
// kWakeFan more (a tree: the depth — every level costs the wake-up latency of an idle core, 50-100 us out of a deep
// C-state — stays small; with one word and a fan-out of two the eight levels were the whole 1.5 ms p50 of
// ApplicationDB::Get).  Spins are SHORT (RSP_WAIT_SPINS / RSP_DISPATCH_SPINS pauses): the GPU boxes cap the container's
// CPU time (16 CPUs of 128 visible), and spinning callers spend the budget the dispatcher needs — 64 Get callers: 151 K
// Gets/s with 1500-pause spins, 574 K without.
#pragma once
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#include <linux/futex.h>
#include <sys/syscall.h>
#include <time.h>
#include <unistd.h>

namespace rsp {

class Stager {
 public:
  struct Ticket {
    int buf = -1;
    size_t item0 = 0, byte0 = 0, n_items = 0;
    uint64_t epoch = 0;
  };
  struct BatchInfo {
    int buf;
    size_t n_items, n_bytes;
    uint32_t klass;
    uint64_t epoch;
  };
  using RunFn = std::function<void(const BatchInfo&)>;
  using PostFn = std::function<void()>;  // dispatcher thread, after the asynchronous completions of a batch ran

  static constexpr int kBuffers = 4;  // filling | running | results being read (callers still waking up: two)
  static constexpr int kWakeFan = 4;     // per futex word (kWakeWords of them per batch)
  static constexpr int kWakeWords = 16;

  // cap_items < 2^27, cap_bytes < 2^27 (the open word's fields)
  Stager(size_t cap_items, size_t cap_bytes, RunFn run, PostFn post = nullptr)
      : cap_items_(cap_items < kFieldMax ? cap_items : kFieldMax), cap_bytes_(cap_bytes < kFieldMax ? cap_bytes : kFieldMax),
        run_(std::move(run)), post_(std::move(post)) {
    b_[0].state = OPEN;
    b_[0].epoch = ++epochs_;
    open_word_.store(Pack(0, 0, 0, 0), std::memory_order_release);
    thread_ = std::thread([this] { Loop(); });
  }
  ~Stager() { Stop(); }
  void Stop() {
    if (stop_.exchange(true)) return;
    WakeSleepers();
    if (thread_.joinable()) thread_.join();
  }

  size_t cap_items() const { return cap_items_; }
  size_t cap_bytes() const { return cap_bytes_; }

  // Reserve n_items / n_bytes in a batch of class `klass` (0 or a power of two; requests of different classes never
  // share a batch); max_items bounds the items of a batch of this class (<= cap_items).  Waits while nothing can take the
  // request.  false: the stager is stopping, or the request can never fit (the caller takes its direct path).
  bool begin(size_t n_items, size_t n_bytes, uint32_t klass, size_t max_items, Ticket* t) {
    if (max_items > cap_items_) max_items = cap_items_;
    if (n_items == 0 || n_items > max_items || n_bytes > cap_bytes_ || (klass & (klass - 1))) return false;
    const uint64_t code = KlassCode(klass);
    for (int spins = 0;; spins++) {
      if (stop_.load(std::memory_order_acquire)) return false;
      const uint32_t seen_free = free32_.load(std::memory_order_acquire);
      uint64_t w = open_word_.load(std::memory_order_acquire);
      while (BufOf(w) != kNoBuf) {
        const uint64_t items = ItemsOf(w), bytes = BytesOf(w);
        if ((items != 0 && CodeOf(w) != code) || items + n_items > max_items || bytes + n_bytes > cap_bytes_)
          break;  // full, or of another class: the dispatcher closes it as soon as it can
        if (open_word_.compare_exchange_weak(w, Pack(BufOf(w), code, items + n_items, bytes + n_bytes), std::memory_order_acq_rel,
                                             std::memory_order_acquire)) {
          t->buf = (int)BufOf(w);
          t->item0 = items;
          t->byte0 = bytes;
          t->n_items = n_items;
          t->epoch = b_[t->buf].epoch;  // (written before the word that names this buffer was published)
          work32_.fetch_add(1, std::memory_order_seq_cst);
          if (disp_sleeping_.load(std::memory_order_seq_cst)) FutexWake(&work32_, 1);
          if (buf_waiters_.load(std::memory_order_relaxed)) FutexWake(&free32_, 2);  // (a few at a time: they fit one batch)
          return true;
        }
      }
      // no room right now: a buffer opens within a batch cycle.  Sleep on the word that counts openings (no polling:
      // the box's CPU time is capped); bounded, in case the opening raced the read above
      if (spins < 20) cpu_relax();
      else {
        buf_waiters_.fetch_add(1, std::memory_order_seq_cst);
        FutexWait(&free32_, seen_free, 500000);
        buf_waiters_.fetch_sub(1, std::memory_order_seq_cst);
      }
    }
  }
  // the caller finished writing its slice
  void commit(const Ticket& t) { b_[t.buf].committed.fetch_add(t.n_items, std::memory_order_acq_rel); }
  // completion without a waiting thread: fn runs on the dispatcher thread once the batch has run; the slice is
  // released when fn returns (fn reads its results from the staging buffers itself)
  void commit_async(const Ticket& t, std::function<void()> fn) {
    Batch& b = b_[t.buf];
    {
      SpinGuard g(sl_);
      b.async.push_back(std::move(fn));
      b.async_items += t.n_items;
    }
    b.committed.fetch_add(t.n_items, std::memory_order_acq_rel);
  }
  // until the batch has run
  void wait(const Ticket& t) {
    Batch& b = b_[t.buf];
    static const int kSpins = [] { const char* v = getenv("RSP_WAIT_SPINS"); return v ? atoi(v) : 100; }();
    for (int spins = 0; spins < kSpins; spins++) {  // a batch cycle is often shorter than a sleep + wake-up
      if (b.epoch_done.load(std::memory_order_acquire) >= t.epoch) return;
      cpu_relax();
    }
    WakeWord& ww = b.wake[(uint32_t)((t.item0 * 2654435761u) >> 16) % kWakeWords];
    bool slept = false;
    for (;;) {
      const uint32_t s = ww.seq.load(std::memory_order_acquire);
      if (b.epoch_done.load(std::memory_order_acquire) >= t.epoch) break;
      ww.sleepers.fetch_add(1, std::memory_order_seq_cst);
      FutexWait(&ww.seq, s, 2000000);  // (bounded: 2 ms)
      ww.sleepers.fetch_sub(1, std::memory_order_seq_cst);
      slept = true;
    }
    if (slept && ww.sleepers.load(std::memory_order_seq_cst)) FutexWake(&ww.seq, kWakeFan);  // pass the wake-up on
  }
  void release(const Ticket& t) {
    Batch& b = b_[t.buf];
    const uint64_t r = b.released.fetch_add(t.n_items, std::memory_order_acq_rel) + t.n_items;
    if (r == b.final_items.load(std::memory_order_acquire)) {
      {
        SpinGuard g(sl_);
        MaybeFree(b);
      }
      WakeBufferWaiters();
    }
  }

  uint64_t batches() const { return batches_.load(std::memory_order_relaxed); }
  // diagnostics: batches run, items carried, ns inside the RunFn, ns waiting for callers still copying, ns idle
  void stats(uint64_t out[5]) const {
    out[0] = batches_.load(std::memory_order_relaxed); out[1] = st_items_.load(std::memory_order_relaxed);
    out[2] = st_run_ns_.load(std::memory_order_relaxed); out[3] = st_copy_ns_.load(std::memory_order_relaxed);
    out[4] = st_idle_ns_.load(std::memory_order_relaxed);
  }

 private:
  enum State { FREE, OPEN, CLOSED, DONE };
  struct alignas(64) WakeWord {
    std::atomic<uint32_t> seq{0};
    std::atomic<uint32_t> sleepers{0};  // callers inside FutexWait on seq (a wake-up is a system call: skipped when 0)
  };
  struct Batch {
    State state = FREE;                 // sl_
    uint64_t epoch = 0;                 // written under sl_ before the open word names the buffer
    std::atomic<uint64_t> committed{0};    // items whose slices are written
    std::atomic<uint64_t> released{0};     // items whose callers are done with the buffer
    std::atomic<uint64_t> final_items{~0ull};  // items reserved, known when the batch is closed
    uint64_t async_items = 0;           // sl_
    std::atomic<uint64_t> epoch_done{0};
    WakeWord wake[kWakeWords];          // futex words: bumped when the batch has run
    std::vector<std::function<void()>> async;  // sl_
  };
  // ---- the open word: [63:60] buffer (15 = none) | [59:54] class code | [53:27] items | [26:0] bytes
  static constexpr uint64_t kNoBuf = 15, kFieldMax = (1ull << 27) - 1;
  static uint64_t Pack(uint64_t buf, uint64_t code, uint64_t items, uint64_t bytes) { return (buf << 60) | (code << 54) | (items << 27) | bytes; }
  static uint64_t BufOf(uint64_t w) { return w >> 60; }
  static uint64_t CodeOf(uint64_t w) { return (w >> 54) & 63; }
  static uint64_t ItemsOf(uint64_t w) { return (w >> 27) & kFieldMax; }
  static uint64_t BytesOf(uint64_t w) { return w & kFieldMax; }
  static uint64_t KlassCode(uint32_t klass) { return klass ? 1u + (uint64_t)__builtin_ctz(klass) : 0u; }  // 0 or a power of two
  static uint32_t KlassOf(uint64_t code) { return code ? 1u << (code - 1) : 0u; }

  static inline void cpu_relax() {
#if defined(__x86_64__) || defined(__i386__)
    __builtin_ia32_pause();
#else
    std::this_thread::yield();
#endif
  }
  struct SpinLock {
    std::atomic<bool> f{false};
    void lock() {
      for (;;) {
        if (!f.exchange(true, std::memory_order_acquire)) return;
        for (int n = 0; f.load(std::memory_order_relaxed); n++) {
          if (n < 200) cpu_relax();
          else {  // the holder was descheduled (threads may outnumber cores): get out of its way
            struct timespec ts = {0, 5000};
            nanosleep(&ts, nullptr);
          }
        }
      }
    }
    void unlock() { f.store(false, std::memory_order_release); }
  };
  struct SpinGuard {
    SpinLock& l;
    explicit SpinGuard(SpinLock& x) : l(x) { l.lock(); }
    ~SpinGuard() { l.unlock(); }
  };

  static void FutexWait(std::atomic<uint32_t>* w, uint32_t expected, long timeout_ns) {
    struct timespec ts;
    ts.tv_sec = timeout_ns / 1000000000L;
    ts.tv_nsec = timeout_ns % 1000000000L;
    syscall(SYS_futex, reinterpret_cast<uint32_t*>(w), FUTEX_WAIT_PRIVATE, expected, &ts, nullptr, 0);
  }
  static void FutexWake(std::atomic<uint32_t>* w, int n) {
    syscall(SYS_futex, reinterpret_cast<uint32_t*>(w), FUTEX_WAKE_PRIVATE, n, nullptr, nullptr, 0);
  }
  static int64_t NowNs() {
    return std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
  }
  static void NapUs(long us) {
    struct timespec ts;
    ts.tv_sec = 0;
    ts.tv_nsec = us * 1000L;
    nanosleep(&ts, nullptr);
  }
  void WakeBufferWaiters() {  // after a buffer may have opened (sl_ NOT held: a system call)
    if (buf_waiters_.load(std::memory_order_seq_cst)) FutexWake(&free32_, kWakeFan);
  }
  void WakeSleepers() {  // Stop(): the dispatcher may be asleep, callers may wait for a buffer
    FutexWake(&work32_, 1);
    FutexWake(&free32_, 1 << 20);
  }

  // sl_ held: buffer i becomes an empty batch (not yet named by the open word)
  void ResetBuffer(int i) {
    Batch& b = b_[i];
    b.state = OPEN;
    b.epoch = ++epochs_;
    b.committed.store(0, std::memory_order_relaxed);
    b.released.store(0, std::memory_order_relaxed);
    b.final_items.store(~0ull, std::memory_order_relaxed);
    b.async_items = 0;
  }
  int FindFree() const {
    for (int i = 0; i < kBuffers; i++)
      if (b_[i].state == FREE) return i;
    return -1;
  }
  bool MaybeFree(Batch& b) {  // sl_ held: whoever sees "done and unused" first recycles the buffer
    if (b.state == DONE && b.released.load(std::memory_order_acquire) == b.final_items.load(std::memory_order_acquire)) {
      b.state = FREE;
      if (BufOf(open_word_.load(std::memory_order_acquire)) == kNoBuf) {  // nobody could reserve: open it right away
        const int i = (int)(&b - b_);
        ResetBuffer(i);
        open_word_.store(Pack((uint64_t)i, 0, 0, 0), std::memory_order_release);
        free32_.fetch_add(1, std::memory_order_seq_cst);  // (whoever called wakes the waiters after dropping sl_)
      }
      return true;
    }
    return false;
  }
  void Loop() {
    for (;;) {
      // ---- close the open batch once it holds work; the next free buffer (if any) opens in the same step
      int bi = -1;
      uint64_t closed = 0;
      const int64_t t_idle0 = NowNs();
      for (int spins = 0;; spins++) {
        const uint64_t w = open_word_.load(std::memory_order_acquire);
        if (BufOf(w) != kNoBuf && ItemsOf(w) > 0) {
          SpinGuard g(sl_);
          const int nb = FindFree();
          if (nb >= 0) ResetBuffer(nb);
          closed = open_word_.exchange(nb >= 0 ? Pack((uint64_t)nb, 0, 0, 0) : Pack(kNoBuf, 0, 0, 0), std::memory_order_acq_rel);
          if (nb >= 0) free32_.fetch_add(1, std::memory_order_seq_cst);
          bi = (int)BufOf(closed);
          b_[bi].state = CLOSED;
          b_[bi].final_items.store(ItemsOf(closed), std::memory_order_release);
          break;
        }
        if (stop_.load(std::memory_order_acquire)) return;  // (queued work was taken above: callers wait on it)
        static const int kIdleSpins = [] { const char* v = getenv("RSP_DISPATCH_SPINS"); return v ? atoi(v) : 100; }();
        if (spins < kIdleSpins) cpu_relax();  // stay hot between batches under load
        else {
          disp_sleeping_.store(true, std::memory_order_seq_cst);
          const uint32_t ws = work32_.load(std::memory_order_seq_cst);
          if (ws == seen_work_ && !stop_.load()) FutexWait(&work32_, ws, 2000000);
          disp_sleeping_.store(false, std::memory_order_seq_cst);
        }
      }
      seen_work_ = work32_.load(std::memory_order_seq_cst);
      WakeBufferWaiters();  // (the next buffer opened when this one was closed)
      Batch& b = b_[bi];
      const uint64_t n_items = ItemsOf(closed);
      const int64_t t_copy0 = NowNs();
      st_idle_ns_.fetch_add((uint64_t)(t_copy0 - t_idle0), std::memory_order_relaxed);
      for (int spins = 0; b.committed.load(std::memory_order_acquire) != n_items; spins++) {
        if (spins < 2000) cpu_relax(); else NapUs(10);  // (a copier may have been descheduled)
      }
      const int64_t t_run0 = NowNs();
      st_copy_ns_.fetch_add((uint64_t)(t_run0 - t_copy0), std::memory_order_relaxed);
      BatchInfo info;
      std::vector<std::function<void()>> async;
      uint64_t async_items = 0;
      {
        SpinGuard g(sl_);
        info = BatchInfo{bi, (size_t)n_items, (size_t)BytesOf(closed), KlassOf(CodeOf(closed)), b.epoch};
        async.swap(b.async);
        async_items = b.async_items;
      }
      run_(info);
      st_run_ns_.fetch_add((uint64_t)(NowNs() - t_run0), std::memory_order_relaxed);
      st_items_.fetch_add(info.n_items, std::memory_order_relaxed);
      for (auto& f : async) f();
      if (post_) post_();
      {
        SpinGuard g(sl_);
        b.state = DONE;
      }
      b.epoch_done.store(info.epoch, std::memory_order_release);  // spinning callers go on at once
      for (int w = 0; w < kWakeWords; w++) {  // sleeping ones: a few per word, who wake the others
        b.wake[w].seq.fetch_add(1, std::memory_order_seq_cst);
        if (b.wake[w].sleepers.load(std::memory_order_seq_cst)) FutexWake(&b.wake[w].seq, 2);
      }
      batches_.fetch_add(1, std::memory_order_relaxed);
      // the asynchronous slices are done with the buffer; so may be everybody else already
      const uint64_t r = b.released.fetch_add(async_items, std::memory_order_acq_rel) + async_items;
      if (r == n_items) {
        {
          SpinGuard g(sl_);
          MaybeFree(b);
        }
        WakeBufferWaiters();
      }
    }
  }

  const size_t cap_items_, cap_bytes_;
  RunFn run_;
  PostFn post_;
  SpinLock sl_;
  Batch b_[kBuffers];
  std::atomic<uint64_t> open_word_{Pack(kNoBuf, 0, 0, 0)};
  uint64_t epochs_ = 0;
  std::atomic<bool> stop_{false}, disp_sleeping_{false};
  std::atomic<uint32_t> work32_{0};  // requests ever accepted (futex word): the idle dispatcher sleeps until it moves
  std::atomic<uint32_t> free32_{0};  // buffers ever opened (futex word): callers without a buffer sleep until it moves
  std::atomic<uint32_t> buf_waiters_{0};
  uint32_t seen_work_ = 0;
  std::atomic<uint64_t> batches_{0}, st_items_{0}, st_run_ns_{0}, st_copy_ns_{0}, st_idle_ns_{0};
  std::thread thread_;
};

}  // namespace rsp
