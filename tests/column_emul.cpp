// column_emul.cpp -- the size walk and the string copy of sjb200_column_dev (simdjson_b200/csrc/sjb200_column.cuh) under
// the host SIMT emulation: OS threads are the lanes of a warp group or of a CTA group of kCtaWarps warps, the warp
// collectives are rendezvous and __syncthreads a barrier (sjb200_simt.cuh, SJB200_HOST_EMU).  Driven by
// tests/test_column_emul.py against the oracle; no GPU involved.
#define SJB200_HOST_EMU 1
#include <pthread.h>
#include <stdint.h>

#include <vector>

#include "sjb200_column.cuh"

using namespace sjb200;
thread_local simt::ThreadCtx simt::tctx;

namespace {
constexpr unsigned kCtaWarps = 8;  // the sm_90a build's CTA group (sjb200_pointer.h)
constexpr int kCtaItems = 8;

struct Job {
  const uint8_t *type;
  uint32_t n;
  bool obj;
  bool cta;
  uint64_t limit;
  col::SizeAt at;
  bool done;
  ptr::CtaSmem<kCtaWarps> sm;
  simt::CtaShared ctash;
  std::vector<simt::WarpShared> warps;
};
struct ThreadArg { Job *job; unsigned tid; };

void *thread_main(void *vp) {
  ThreadArg *a = static_cast<ThreadArg *>(vp);
  Job &j = *a->job;
  simt::tctx = simt::ThreadCtx();
  simt::tctx.tid = a->tid;
  simt::tctx.nctas = 1;
  simt::tctx.warp = &j.warps[a->tid / 32];
  simt::tctx.ctas = &j.ctash;
  col::SizeAt at = j.at;
  bool done;
  if (j.cta) {
    ptr::CtaGroup<kCtaWarps> g{a->tid, &j.sm};
    done = col::count_children<ptr::CtaGroup<kCtaWarps>, kCtaItems>(g, j.type, j.n, j.obj, &at, j.limit);
  } else {
    ptr::WarpGroup g{a->tid & 31u};
    done = col::count_children<ptr::WarpGroup, 1>(g, j.type, j.n, j.obj, &at, j.limit);
  }
  if (a->tid == 0) {
    j.at = at;
    j.done = done;
  }
  return nullptr;
}

int run(Job &job) {
  const unsigned T = job.cta ? 32 * kCtaWarps : 32;
  job.warps.resize(T / 32);
  for (auto &w : job.warps) pthread_barrier_init(&w.bar, nullptr, 32);
  pthread_barrier_init(&job.ctash.bar, nullptr, T);
  job.ctash.smem = nullptr;
  std::vector<ThreadArg> args(T);
  std::vector<pthread_t> th(T);
  for (unsigned t = 0; t < T; t++) {
    args[t] = ThreadArg{&job, t};
    if (pthread_create(&th[t], nullptr, thread_main, &args[t]) != 0) return -1;
  }
  for (auto &t : th) pthread_join(t, nullptr);
  for (auto &w : job.warps) pthread_barrier_destroy(&w.bar);
  pthread_barrier_destroy(&job.ctash.bar);
  job.warps.clear();
  return 0;
}
}  // namespace

// The children of the container opened at structural `opener` as sjb200_column_dev counts them: a warp over at most
// warp_limit structurals (the warp kernel's kCtaMinStructurals), then -- the walk still open -- a CTA from the warp's
// cursor; warp_limit 0: the CTA from the start.  *handed: whether the CTA took over.  Returns the saturated count, -1 on
// a thread failure.
extern "C" long long emu_size(const uint8_t *type, uint32_t n, uint32_t opener, int obj, uint64_t warp_limit, int *handed) {
  Job job;
  job.type = type;
  job.n = n;
  job.obj = obj != 0;
  job.at = col::SizeAt{opener + 1, 0, 0};
  job.done = false;
  *handed = 0;
  if (warp_limit) {
    job.cta = false;
    job.limit = warp_limit;
    if (run(job) != 0) return -1;
  }
  if (!job.done) {
    *handed = warp_limit != 0;
    job.cta = true;
    job.limit = ~0ull;
    if (run(job) != 0 || !job.done) return -1;
  }
  return job.at.count < col::kCountSat ? job.at.count : col::kCountSat;
}

// group_copy by a group of `width` threads (no collectives: the ranks run one after the other)
extern "C" void emu_copy(unsigned width, uint8_t *dst, const uint8_t *src, uint64_t len) {
  for (unsigned r = 0; r < width; r++) col::group_copy(r, width, dst, src, len);
}
