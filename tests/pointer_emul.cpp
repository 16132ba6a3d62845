// pointer_emul.cpp -- the JSON Pointer walk (simdjson_b200/csrc/sjb200_pointer.cuh) and its host compile of the pointers
// under the host SIMT emulation: OS threads are the lanes of a warp group or of a CTA group of kCtaWarps warps, the warp
// collectives are rendezvous and __syncthreads a barrier (sjb200_simt.cuh, SJB200_HOST_EMU).  Driven by
// tests/test_pointer_emul.py against the oracle; no GPU involved.
#define SJB200_HOST_EMU 1
#include <pthread.h>
#include <stdint.h>

#include <vector>

#include "sjb200_pointer.cuh"

using namespace sjb200;
thread_local simt::ThreadCtx simt::tctx;

namespace {
constexpr unsigned kCtaWarps = 8;  // the sm_90a build's CTA group (sjb200_pointer.h)
constexpr int kCtaItems = 8;

struct Job {
  ptr::Walk w;
  const ptr::CompiledPointers *cp;
  uint32_t root, end;
  int32_t *err;
  uint32_t *idx;
  ptr::CtaSmem<kCtaWarps> sm;
  simt::CtaShared cta;
  std::vector<simt::WarpShared> warps;
};
struct ThreadArg { Job *job; unsigned tid; bool cta; };

void *thread_main(void *vp) {
  ThreadArg *a = static_cast<ThreadArg *>(vp);
  Job &j = *a->job;
  simt::tctx = simt::ThreadCtx();
  simt::tctx.tid = a->tid;
  simt::tctx.nctas = 1;
  simt::tctx.warp = &j.warps[a->tid / 32];
  simt::tctx.ctas = &j.cta;
  ptr::WarpGroup wg{a->tid & 31u};
  ptr::CtaGroup<kCtaWarps> cg{a->tid, &j.sm};
  for (size_t p = 0; p < j.cp->headers.size(); p++) {
    int32_t e;
    const uint32_t v = a->cta ? ptr::walk_pointer<ptr::CtaGroup<kCtaWarps>, kCtaItems>(cg, j.w, j.cp->headers[p], j.root, j.end, &e)
                              : ptr::walk_pointer<ptr::WarpGroup, 1>(wg, j.w, j.cp->headers[p], j.root, j.end, &e);
    if (a->tid == 0) {
      j.err[p] = e;
      j.idx[p] = v;
    }
  }
  return nullptr;
}
}  // namespace

// every pointer (pointer k: the next lens[k] bytes of `pointers`) in the document [root, end) of tokens output, walked by a
// warp (cta = 0) or a CTA (cta = 1).  Returns compile_pointers' code.
extern "C" int emu_at_pointer(int cta, const uint8_t *type, const uint64_t *payload, const uint8_t *strbuf, uint64_t string_bytes, uint32_t root,
                              uint32_t end, const char *pointers, const size_t *lens, int np, int32_t *err, uint32_t *idx) {
  std::vector<const char *> ptrs(size_t(np > 0 ? np : 1));
  for (int k = 0; k < np; k++) {
    ptrs[size_t(k)] = pointers;
    pointers += lens[k];
  }
  ptr::CompiledPointers cp;
  const int rc = ptr::compile_pointers(ptrs.data(), lens, np, &cp);
  if (rc != 0) return rc;
  Job job;
  job.w = ptr::Walk{type, payload, strbuf, string_bytes, cp.levels.data(), reinterpret_cast<const uint8_t *>(cp.keys.data())};
  job.cp = &cp;
  job.root = root;
  job.end = end;
  job.err = err;
  job.idx = idx;
  const unsigned T = cta ? 32 * kCtaWarps : 32;
  job.warps.resize(T / 32);
  for (auto &w : job.warps) pthread_barrier_init(&w.bar, nullptr, 32);
  pthread_barrier_init(&job.cta.bar, nullptr, T);
  job.cta.smem = nullptr;
  std::vector<ThreadArg> args(T);
  std::vector<pthread_t> th(T);
  for (unsigned t = 0; t < T; t++) {
    args[t] = ThreadArg{&job, t, cta != 0};
    if (pthread_create(&th[t], nullptr, thread_main, &args[t]) != 0) return -1;
  }
  for (auto &t : th) pthread_join(t, nullptr);
  for (auto &w : job.warps) pthread_barrier_destroy(&w.bar);
  pthread_barrier_destroy(&job.cta.bar);
  return 0;
}
