// sjb200_hostpipe.h -- host side of the host-pointer entry points: a small pool of copy threads that moves the caller's
// (pageable) input into a ring of page-locked staging slots, chunk after chunk, ahead of the copy engine.
//
// Why it exists: dom::parser::parse(buf, len) hands the plug-in ordinary pageable memory (a padded_string).  A
// cudaMemcpyAsync from pageable memory is staged by the driver one piece at a time and blocks the calling thread, which
// leaves most of the PCIe link idle; page-locking the caller's buffer per call costs more than the copy, and keeping it
// locked after the call is not safe (the caller may free and re-map the range).  So the library owns a fixed ring of
// page-locked slots and fills it with plain memcpy from several threads (one core cannot fill the link),
// while the copy engine drains the slots and the scan kernels chase the copies (document_stream gets its overlap from a
// worker thread in the same spirit: include/simdjson/dom/document_stream-inl.h L16-85, L321-344).
//
// Host-only C++; no CUDA types (the caller owns events and streams).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#if defined(__x86_64__) || defined(__i386__)
#include <immintrin.h>
#define SJB200_CPU_RELAX() _mm_pause()
#else
#define SJB200_CPU_RELAX() std::this_thread::yield()
#endif

namespace sjb200 {

void copy_to_staging(void *dst, const void *src, size_t n);  // sjb200_hostcopy.cpp: streaming stores

class CopyPool {
 public:
  static constexpr size_t kMaxChunks = 4096;

  CopyPool() : done_(new std::atomic<uint32_t>[kMaxChunks]) {}
  ~CopyPool() { stop(); }
  CopyPool(const CopyPool &) = delete;
  CopyPool &operator=(const CopyPool &) = delete;

  int threads() const { return int(threads_.size()); }

  // (re)start with n worker threads; false when no thread could be created
  bool start(int n) {
    if (n == threads()) return n > 0;
    stop();
    quit_ = false;
    const int s0 = session_;  // no session can begin before start() returns: every worker starts from the same count
    for (int i = 0; i < n; i++) {
      try {
        threads_.emplace_back([this, i, s0] { worker(i, s0); });
      } catch (...) {
        break;
      }
    }
    return !threads_.empty();
  }

  void stop() {
    {
      std::lock_guard<std::mutex> g(mu_);
      quit_ = true;
      session_++;
    }
    cv_.notify_all();
    for (auto &t : threads_) t.join();
    threads_.clear();
  }

  // One session = one document: chunk k (bytes [bounds[k], bounds[k+1])) goes to ring slot k % nslots as soon as allow()
  // has covered it.  nchunks <= kMaxChunks, every chunk <= slot_bytes; `bounds` stays valid until end().
  void begin(const uint8_t *src, const size_t *bounds, size_t nchunks, uint8_t *ring, size_t slot_bytes, int nslots) {
    src_ = src; bounds_ = bounds; ring_ = ring; slot_bytes_ = slot_bytes; nslots_ = nslots;
    nchunks_ = nchunks;
    for (size_t k = 0; k < nchunks_; k++) done_[k].store(0, std::memory_order_relaxed);
    allowed_.store(0, std::memory_order_relaxed);
    abort_.store(false, std::memory_order_relaxed);
    active_.store(threads(), std::memory_order_release);
    {
      std::lock_guard<std::mutex> g(mu_);
      session_++;
    }
    cv_.notify_all();
  }
  // chunks [0, upto) may be copied (their slots are free)
  void allow(size_t upto) { allowed_.store(upto, std::memory_order_release); }
  bool chunk_ready(size_t k) const { return done_[k].load(std::memory_order_acquire) == uint32_t(threads()); }
  // wait until every worker has left the session (abort = true makes them leave early)
  void end(bool abort) {
    if (abort) abort_.store(true, std::memory_order_release);
    uint32_t spins = 0;
    while (active_.load(std::memory_order_acquire) != 0) {
      if (++spins < 256) SJB200_CPU_RELAX();
      else std::this_thread::sleep_for(std::chrono::microseconds(20));
    }
  }

 private:
  void worker(int me, int seen) {
    for (;;) {
      {
        std::unique_lock<std::mutex> l(mu_);
        cv_.wait(l, [&] { return session_ != seen; });
        seen = session_;
        if (quit_) return;
      }
      const int nt = threads();
      for (size_t k = 0; k < nchunks_; k++) {
        uint32_t spins = 0;
        while (allowed_.load(std::memory_order_acquire) <= k && !abort_.load(std::memory_order_acquire)) {
          // a short spin, then sleep: a pool that spins on a machine with a CPU quota (containers) starves its own copies
          if (++spins < 256) SJB200_CPU_RELAX();
          else std::this_thread::sleep_for(std::chrono::microseconds(20));
        }
        if (abort_.load(std::memory_order_acquire)) break;
        const size_t off = bounds_[k];
        const size_t bytes = bounds_[k + 1] - off;
        const size_t per = ((bytes + size_t(nt) - 1) / size_t(nt) + 4095) & ~size_t(4095);  // whole pages per thread
        const size_t lo = size_t(me) * per;
        if (lo < bytes) copy_to_staging(ring_ + size_t(k % size_t(nslots_)) * slot_bytes_ + lo, src_ + off + lo, (bytes - lo < per) ? (bytes - lo) : per);
        done_[k].fetch_add(1, std::memory_order_release);
      }
      active_.fetch_sub(1, std::memory_order_release);
    }
  }

  std::vector<std::thread> threads_;
  std::mutex mu_;
  std::condition_variable cv_;
  int session_ = 0;
  bool quit_ = false;
  const uint8_t *src_ = nullptr;
  uint8_t *ring_ = nullptr;
  const size_t *bounds_ = nullptr;
  size_t slot_bytes_ = 0, nchunks_ = 0;
  int nslots_ = 0;
  std::atomic<size_t> allowed_{0};
  std::atomic<bool> abort_{false};
  std::atomic<int> active_{0};
  std::unique_ptr<std::atomic<uint32_t>[]> done_;
};

}  // namespace sjb200
