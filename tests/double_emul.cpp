// double_emul.cpp -- element::get_double of sjb200_column_double_dev (simdjson_b200/csrc/sjb200_double.cuh) on the host:
// the lane routine (summarize by one thread, convert, exact) as the row kernels run it, and the long-number routine
// under the host SIMT emulation, OS threads being the lanes of a warp group or of a CTA group of kCtaWarps warps
// (sjb200_simt.cuh, SJB200_HOST_EMU).  Driven by tests/test_double_emul.py against Python's float(); no GPU involved.
#define SJB200_HOST_EMU 1
#include <pthread.h>
#include <stdint.h>

#include <vector>

#include "sjb200_double.cuh"

using namespace sjb200;
thread_local simt::ThreadCtx simt::tctx;

namespace {
constexpr unsigned kCtaWarps = 8;  // the sm_90a build's CTA group (sjb200_pointer.h)

// The row's error and bits from its summary, as the kernels finish a 'd' row; *slow: exact() decided it.
int32_t finish(const dbl::Num &m, const dbl::SpanSrc &at, uint64_t *bits, int *slow) {
  *bits = 0;
  *slow = 0;
  if (!m.valid) return 24;  // UNEXPECTED_ERROR
  uint64_t fb = 0;
  int32_t e = dbl::convert(m, at, bits, &fb);
  if (e == dbl::kSlow) {
    *slow = 1;
    uint32_t big[2 * dbl::kLimbs];
    e = dbl::finish_exact(m, dbl::exact(m, at, fb, dbl::Big{big, 1, 0}, dbl::Big{big + dbl::kLimbs, 1, 0}), bits);
  }
  if (e) *bits = 0;
  return e;
}

struct Job {
  dbl::SpanSrc at;
  bool cta;
  dbl::Num num;
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
  dbl::Num m;
  if (j.cta) {
    ptr::CtaGroup<kCtaWarps> g{a->tid, &j.sm};
    m = dbl::summarize(g, j.at, j.at.len);
  } else {
    ptr::WarpGroup g{a->tid & 31u};
    m = dbl::summarize(g, j.at, j.at.len);
  }
  if (a->tid == 0) j.num = m;
  return nullptr;
}
}  // namespace

// count numbers, number i being buf[offs[i], offs[i + 1]), each by one lane as dbl_row_kernel / dbl_exact_kernel do:
// err[i], bits[i] and slow[i] (1: decided by the exact comparison)
extern "C" void emu_double_lane(const uint8_t *buf, const uint64_t *offs, uint32_t count, int32_t *err, uint64_t *bits, int32_t *slow) {
  for (uint32_t i = 0; i < count; i++) {
    const dbl::SpanSrc at{buf + offs[i], uint32_t(offs[i + 1] - offs[i])};
    dbl::SerialGroup g;
    const dbl::Num m = dbl::summarize(g, at, at.len);
    int s;
    err[i] = finish(m, at, &bits[i], &s);
    slow[i] = s;
  }
}

// one number of len bytes summarized by a warp (cta = 0) or a CTA of kCtaWarps warps (cta = 1), then converted by the
// group's first thread as dbl_long_kernel does.  Returns the error, -1 on a thread failure.
extern "C" int emu_double_group(const uint8_t *buf, uint32_t len, int cta, uint64_t *bits, int32_t *slow) {
  Job job;
  job.at = dbl::SpanSrc{buf, len};
  job.cta = cta != 0;
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
  int s;
  const int32_t e = finish(job.num, job.at, bits, &s);
  *slow = s;
  return e;
}
