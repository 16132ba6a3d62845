// sjb200_simt.cuh -- the few hardware primitives the scan4 kernel is written against.
//
// Two implementations of the same small API:
//   * nvcc / sm_90a: warp intrinsics, mbarrier + cp.async.bulk.tensor (TMA) inline PTX, relaxed
//     gpu-scope loads/stores for the look-back descriptors;
//   * SJB200_HOST_EMU (g++, tests/simt_emul.cpp): one OS thread per CUDA thread, warp collectives as
//     32-thread rendezvous, mbarriers with deferred TMA copies.  This exists so that the *actual*
//     kernel source (warp roles, mbarrier protocol, look-back chain, emit) can be run against the
//     oracle on a machine without a GPU.  It is test infrastructure; the product never uses it.
#pragma once
#include <stdint.h>

#if defined(SJB200_HOST_EMU)
// =============================================================================== host emulation
#include <pthread.h>
#include <sched.h>
#include <string.h>
#include <time.h>

#include <atomic>
#include <mutex>
#include <new>

#define SJ_DEV inline
#define SJ_DEV_NOINLINE

namespace sjb200 {
namespace simt {

struct WarpShared {
  pthread_barrier_t bar;
  uint32_t vals[2][32];
};
struct CtaShared {
  pthread_barrier_t bar;
  uint8_t *smem;
};
// Programmatic dependent launch between emulated grids (tests/simt_emul_pdl.cpp): a grid's threads may run while its
// predecessor still runs; sj_griddep_wait blocks until every thread of the predecessor has exited, and the harness
// starts the successor once every CTA of this grid has triggered or exited.  Null: no predecessor, no successor.
struct GridDep {
  GridDep *prev = nullptr;
  std::atomic<unsigned> running{0};   // threads of this grid that have not exited
  std::atomic<unsigned> released{0};  // CTAs that have triggered or exited
  std::atomic<uint8_t> *cta_released = nullptr;
};
struct ThreadCtx {
  unsigned tid = 0, cta = 0, nctas = 0;
  unsigned phase = 0;
  WarpShared *warp = nullptr;
  CtaShared *ctas = nullptr;
  GridDep *dep = nullptr;
};
extern thread_local ThreadCtx tctx;

inline uint32_t exchange(uint32_t v, unsigned &ph) {
  ThreadCtx &t = tctx;
  ph = t.phase;
  t.warp->vals[ph][t.tid & 31u] = v;
  pthread_barrier_wait(&t.warp->bar);
  t.phase ^= 1u;
  return 0;
}

}  // namespace simt

struct alignas(16) sj_u4 { uint32_t x, y, z, w; };
SJ_DEV sj_u4 sj_make_u4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { sj_u4 v; v.x = x; v.y = y; v.z = z; v.w = w; return v; }
SJ_DEV sj_u4 sj_ldg_u4(const void *p) { sj_u4 v; memcpy(&v, p, 16); return v; }
SJ_DEV uint32_t sj_ldg_u32(const void *p) { uint32_t v; memcpy(&v, p, 4); return v; }
SJ_DEV uint32_t sj_ldg_u8(const uint8_t *p) { return *p; }

SJ_DEV unsigned sj_tid() { return simt::tctx.tid; }
SJ_DEV unsigned sj_cta() { return simt::tctx.cta; }
SJ_DEV unsigned sj_nctas() { return simt::tctx.nctas; }
SJ_DEV uint8_t *sj_smem_base() { return simt::tctx.ctas->smem; }

SJ_DEV uint32_t sj_shfl(uint32_t v, int src) {
  unsigned ph;
  simt::exchange(v, ph);
  return simt::tctx.warp->vals[ph][src & 31];
}
SJ_DEV uint32_t sj_shfl_up(uint32_t v, int d) {
  unsigned ph;
  simt::exchange(v, ph);
  const int lane = int(simt::tctx.tid & 31u);
  return lane >= d ? simt::tctx.warp->vals[ph][lane - d] : v;
}
SJ_DEV uint32_t sj_shfl_down(uint32_t v, int d) {
  unsigned ph;
  simt::exchange(v, ph);
  const int lane = int(simt::tctx.tid & 31u);
  return lane + d < 32 ? simt::tctx.warp->vals[ph][lane + d] : v;
}
SJ_DEV uint32_t sj_ballot(bool pred) {
  unsigned ph;
  simt::exchange(pred ? 1u : 0u, ph);
  uint32_t m = 0;
  for (int i = 0; i < 32; i++) m |= (simt::tctx.warp->vals[ph][i] & 1u) << i;
  return m;
}
SJ_DEV bool sj_any(bool pred) { return sj_ballot(pred) != 0; }
SJ_DEV uint32_t sj_reduce_max(uint32_t v) {
  unsigned ph;
  simt::exchange(v, ph);
  uint32_t m = 0;
  for (int i = 0; i < 32; i++) m = simt::tctx.warp->vals[ph][i] > m ? simt::tctx.warp->vals[ph][i] : m;
  return m;
}
SJ_DEV uint32_t sj_reduce_min(uint32_t v) {
  unsigned ph;
  simt::exchange(v, ph);
  uint32_t m = 0xFFFFFFFFu;
  for (int i = 0; i < 32; i++) m = simt::tctx.warp->vals[ph][i] < m ? simt::tctx.warp->vals[ph][i] : m;
  return m;
}
SJ_DEV uint32_t sj_reduce_add(uint32_t v) {
  unsigned ph;
  simt::exchange(v, ph);
  uint32_t m = 0;
  for (int i = 0; i < 32; i++) m += simt::tctx.warp->vals[ph][i];
  return m;
}
SJ_DEV void sj_syncwarp() {
  unsigned ph;
  simt::exchange(0, ph);
}
SJ_DEV void sj_syncthreads() { pthread_barrier_wait(&simt::tctx.ctas->bar); }

SJ_DEV int sj_popc(uint32_t x) { return __builtin_popcount(x); }
SJ_DEV int sj_ffs(uint32_t x) { return __builtin_ffs(int(x)); }
SJ_DEV uint32_t sj_bfind(uint32_t x) { return x ? uint32_t(31 - __builtin_clz(x)) : 0xFFFFFFFFu; }
SJ_DEV uint32_t sj_funnel_l(uint32_t lo, uint32_t hi, int n) { return n ? ((hi << n) | (lo >> (32 - n))) : hi; }
SJ_DEV uint32_t sj_funnel_r(uint32_t lo, uint32_t hi, int n) { return n ? ((lo >> n) | (hi << (32 - n))) : lo; }

SJ_DEV uint32_t sj_atomic_add(uint32_t *p, uint32_t v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
SJ_DEV uint32_t sj_atomic_or(uint32_t *p, uint32_t v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
SJ_DEV uint32_t sj_atomic_exch(uint32_t *p, uint32_t v) { return __atomic_exchange_n(p, v, __ATOMIC_SEQ_CST); }
SJ_DEV unsigned long long sj_ld_relaxed_u64(const unsigned long long *p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
SJ_DEV void sj_st_relaxed_u64(unsigned long long *p, unsigned long long v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
SJ_DEV void sj_threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
SJ_DEV void sj_st_sys_u64(unsigned long long *p, unsigned long long v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
SJ_DEV void sj_fence_gpu_release() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
SJ_DEV uint32_t sj_ld_relaxed_u32(const uint32_t *p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
SJ_DEV void sj_fence_block() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
SJ_DEV void sj_nanosleep(unsigned) {
  struct timespec ts = {0, 20000};
  nanosleep(&ts, nullptr);
}
SJ_DEV unsigned sj_smid() { return simt::tctx.cta; }
SJ_DEV unsigned long long sj_globaltimer() {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (unsigned long long)ts.tv_sec * 1000000000ull + (unsigned long long)ts.tv_nsec;
}
SJ_DEV uint32_t sj_clock32() { return uint32_t(sj_globaltimer()); }

SJ_DEV void sj_griddep_wait() {
  const simt::GridDep *d = simt::tctx.dep;
  if (d == nullptr || d->prev == nullptr) return;
  while (d->prev->running.load(std::memory_order_acquire) != 0) {
    struct timespec ts = {0, 20000};
    nanosleep(&ts, nullptr);
  }
}
SJ_DEV void sj_griddep_launch_dependents() {
  simt::GridDep *d = simt::tctx.dep;
  if (d != nullptr && d->cta_released[simt::tctx.cta].exchange(1) == 0) d->released.fetch_add(1);
}

// ---- mbarrier with deferred TMA copies
struct sj_tensor_map {  // what the emulated TMA needs to know about the 2-D uint8 [rows][128] tensor
  const uint8_t *base;
  uint64_t rows;
  uint32_t box_rows;
};
struct sj_mbar_t {
  std::mutex mu;
  uint32_t count = 0, pending = 0, phase = 0;
  int64_t tx = 0;
  struct Copy { uint8_t *dst; const uint8_t *src; uint32_t rows; uint32_t bytes; } q[4];
  int nq = 0;
};
namespace simt {
inline void mbar_check_complete(sj_mbar_t *b) {
  if (b->pending == 0 && b->tx == 0) {
    b->phase ^= 1u;
    b->pending = b->count;
  }
}
inline void mbar_run_copies(sj_mbar_t *b) {  // caller holds the lock
  for (int i = 0; i < b->nq; i++) {
    const sj_mbar_t::Copy &c = b->q[i];
    for (uint32_t r = 0; r < c.rows; r++)
      for (uint32_t col = 0; col < 128; col++) {
        const uint32_t off = r * 128 + col;
        c.dst[off ^ ((off >> 3) & 0x70u)] = c.src[size_t(r) * 128 + col];  // SWIZZLE_128B
      }
    b->tx -= int64_t(c.bytes);
  }
  b->nq = 0;
  mbar_check_complete(b);
}
}  // namespace simt
SJ_DEV void sj_mbar_init(sj_mbar_t *b, uint32_t count) {
  new (b) sj_mbar_t();
  b->count = b->pending = count;
}
SJ_DEV void sj_fence_mbar_init() {}
SJ_DEV void sj_fence_proxy_async() {}
SJ_DEV void sj_fence_tensormap_acquire(const void *) {}
SJ_DEV void sj_mbar_arrive(sj_mbar_t *b) {
  std::lock_guard<std::mutex> g(b->mu);
  b->pending--;
  simt::mbar_check_complete(b);
}
SJ_DEV void sj_mbar_arrive_expect_tx(sj_mbar_t *b, uint32_t bytes) {
  std::lock_guard<std::mutex> g(b->mu);
  b->tx += int64_t(bytes);
  b->pending--;
  simt::mbar_check_complete(b);
}
SJ_DEV bool sj_mbar_try_wait(sj_mbar_t *b, uint32_t parity) {
  {
    std::lock_guard<std::mutex> g(b->mu);
    if (b->nq) simt::mbar_run_copies(b);  // the "asynchronous" copy lands no earlier than the first wait
    if (b->phase != parity) return true;
  }
  struct timespec ts = {0, 20000};
  nanosleep(&ts, nullptr);
  return false;
}
// one TMA box of box_rows x 128 B starting at tensor row `row`, 128B-swizzled, completing on `bar`
SJ_DEV void sj_tma_load_rows(uint8_t *dst, const sj_tensor_map *map, sj_mbar_t *bar, uint32_t row) {
  std::lock_guard<std::mutex> g(bar->mu);
  sj_mbar_t::Copy &c = bar->q[bar->nq++];
  c.dst = dst;
  c.src = map->base + size_t(row) * 128;
  c.rows = map->box_rows;
  c.bytes = map->box_rows * 128;
}

}  // namespace sjb200

#else
// =============================================================================== sm_90a
#include <cuda.h>
#include <cuda_runtime.h>

#define SJ_DEV __device__ __forceinline__
#define SJ_DEV_NOINLINE static __device__ __noinline__

namespace sjb200 {

constexpr uint32_t kFullMask = 0xFFFFFFFFu;

typedef uint4 sj_u4;
SJ_DEV sj_u4 sj_make_u4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return make_uint4(x, y, z, w); }
SJ_DEV sj_u4 sj_ldg_u4(const void *p) { return __ldg(reinterpret_cast<const uint4 *>(p)); }
SJ_DEV uint32_t sj_ldg_u32(const void *p) { return __ldg(reinterpret_cast<const uint32_t *>(p)); }
SJ_DEV uint32_t sj_ldg_u8(const uint8_t *p) { return __ldg(p); }

SJ_DEV unsigned sj_tid() { return threadIdx.x; }
SJ_DEV unsigned sj_cta() { return blockIdx.x; }
SJ_DEV unsigned sj_nctas() { return gridDim.x; }

SJ_DEV uint32_t sj_shfl(uint32_t v, int src) { return __shfl_sync(kFullMask, v, src); }
SJ_DEV uint32_t sj_shfl_up(uint32_t v, int d) { return __shfl_up_sync(kFullMask, v, d); }
SJ_DEV uint32_t sj_shfl_down(uint32_t v, int d) { return __shfl_down_sync(kFullMask, v, d); }
SJ_DEV uint32_t sj_ballot(bool pred) { return __ballot_sync(kFullMask, pred); }
SJ_DEV bool sj_any(bool pred) { return __any_sync(kFullMask, pred); }
SJ_DEV uint32_t sj_reduce_max(uint32_t v) { return __reduce_max_sync(kFullMask, v); }
SJ_DEV uint32_t sj_reduce_min(uint32_t v) { return __reduce_min_sync(kFullMask, v); }
SJ_DEV uint32_t sj_reduce_add(uint32_t v) { return __reduce_add_sync(kFullMask, v); }
SJ_DEV void sj_syncwarp() { __syncwarp(); }
SJ_DEV void sj_syncthreads() { __syncthreads(); }
SJ_DEV int sj_popc(uint32_t x) { return __popc(x); }
SJ_DEV int sj_ffs(uint32_t x) { return __ffs(int(x)); }
SJ_DEV uint32_t sj_bfind(uint32_t x) {  // index of the highest set bit (0xFFFFFFFF for 0): one FLO
  uint32_t r;
  asm("bfind.u32 %0, %1;" : "=r"(r) : "r"(x));
  return r;
}
SJ_DEV uint32_t sj_funnel_l(uint32_t lo, uint32_t hi, int n) { return __funnelshift_l(lo, hi, n); }
SJ_DEV uint32_t sj_funnel_r(uint32_t lo, uint32_t hi, int n) { return __funnelshift_r(lo, hi, n); }

SJ_DEV uint32_t sj_atomic_add(uint32_t *p, uint32_t v) { return atomicAdd(p, v); }
SJ_DEV uint32_t sj_atomic_or(uint32_t *p, uint32_t v) { return atomicOr(p, v); }
SJ_DEV uint32_t sj_atomic_exch(uint32_t *p, uint32_t v) { return atomicExch(p, v); }
SJ_DEV unsigned long long sj_ld_relaxed_u64(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
SJ_DEV void sj_st_relaxed_u64(unsigned long long *p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
SJ_DEV void sj_threadfence() { __threadfence(); }
// a word of another GPU's memory (peer-mapped over NVLink): system scope
SJ_DEV void sj_st_sys_u64(unsigned long long *p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
SJ_DEV void sj_fence_gpu_release() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
SJ_DEV uint32_t sj_ld_relaxed_u32(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
SJ_DEV void sj_fence_block() { __threadfence_block(); }
SJ_DEV void sj_nanosleep(unsigned ns) { __nanosleep(ns); }
SJ_DEV unsigned sj_smid() {
  unsigned r;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(r));
  return r;
}
SJ_DEV unsigned long long sj_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
SJ_DEV uint32_t sj_clock32() { return uint32_t(clock64()); }  // SM-local cycle counter (cheap; for intervals on one SM)
// Programmatic dependent launch.  wait: until the grids this one depends on have completed and their memory is visible
// (returns at once in a grid launched without the attribute).  launch_dependents: this CTA lets the next grid on the
// stream start (the first call of a CTA counts; a CTA that exits without it counts at its exit).
SJ_DEV void sj_griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
SJ_DEV void sj_griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

typedef CUtensorMap sj_tensor_map;
typedef unsigned long long sj_mbar_t;

SJ_DEV uint32_t sj_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
SJ_DEV void sj_mbar_init(sj_mbar_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sj_smem_u32(bar)), "r"(count) : "memory");
}
SJ_DEV void sj_fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// (MEMBAR.ALL.CTA + FENCE.VIEW.ASYNC: waits for the thread's outstanding loads -- issue it before, not after, a global
// load whose value is not needed yet)
SJ_DEV void sj_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// a tensor map in global memory that the host wrote (cudaMemcpy) is used by this thread's TMA loads only after this fence
SJ_DEV void sj_fence_tensormap_acquire(const void *map) {
  asm volatile("fence.proxy.tensormap::generic.acquire.sys [%0], 128;" ::"l"(map) : "memory");
}
SJ_DEV void sj_mbar_arrive(sj_mbar_t *bar) {
  asm volatile("mbarrier.arrive.release.cta.shared::cta.b64 _, [%0];" ::"r"(sj_smem_u32(bar)) : "memory");
}
SJ_DEV void sj_mbar_arrive_expect_tx(sj_mbar_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sj_smem_u32(bar)), "r"(bytes) : "memory");
}
SJ_DEV bool sj_mbar_try_wait(sj_mbar_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2, 0x1000;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(sj_smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
SJ_DEV void sj_tma_load_rows(uint8_t *dst, const sj_tensor_map *map, sj_mbar_t *bar, uint32_t row) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(sj_smem_u32(dst)),
      "l"(map), "r"(sj_smem_u32(bar)), "r"(0), "r"(int(row))
      : "memory");
}

}  // namespace sjb200
#endif
