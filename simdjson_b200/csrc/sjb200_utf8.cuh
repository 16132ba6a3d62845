// sjb200_utf8.cuh -- validate_utf8 on its own ("utf8v2"): every warp streams its own 4 KiB blocks, nothing is shared.
//
// What it replaces in the reference:  generic_validate_utf8 (src/generic/stage1/utf8_validator.h L18-34) driving
// utf8_checker (src/generic/stage1/utf8_lookup4_algorithm.h L145-202) over 64-byte blocks on one core.
//
// UTF-8 validity needs no scan: byte i is judged from bytes i-3..i (SURVEY.md 8(a) equivalence note).  So this kernel has
// no chain, no tickets and no CTA-wide barrier: warp g of the launch takes blocks g, g + G, g + 2G, ... (neighbouring
// warps read neighbouring 4 KiB blocks), each through its own TMA ring (cp.async.bulk.tensor, 32 rows x 128 B, 128B-swizzled:
// lane L owns row L and reads it with conflict-free LDS.128; kSlotsU slots, kSlotsU - 1 blocks in flight; 24 warps x 2
// slots per SM).  One
// vote per block: without a byte >= 0x80 in any lane a block costs ~50 instructions; otherwise the lane's four 32-byte
// units are transposed into bit planes and checked with the boolean rules of sjb200_bits.cuh, without further votes.
// The three bytes before a lane's row come from the row before it (shared memory), those before a block from global
// memory (one word, loaded one block ahead).  Errors are OR-ed in a register and reach memory once per warp.  In a sharded
// pass (ScanParams::xchg.nranks != 0) the last CTA out also stores the shard's record into every rank's exchange window,
// as scan4 does (sjb200_validate_utf8_sharded*).
//
// Compiles for the host SIMT emulation as well (tests/simt_emul.cpp).
#pragma once
#include "sjb200_bits.cuh"
#include "sjb200_params.h"
#include "sjb200_scan4.cuh"  // block I/O helpers: swz, load_unit, fill_block_guarded, word_before, wait_bar
#include "sjb200_simt.cuh"

namespace sjb200 {
namespace utf8v2 {

#ifndef SJB200_UTF8_WARPS
#define SJB200_UTF8_WARPS 8
#endif
#ifndef SJB200_UTF8_CTAS
#define SJB200_UTF8_CTAS 3
#endif
#ifndef SJB200_UTF8_SLOTS
#define SJB200_UTF8_SLOTS 2
#endif
constexpr int kWarpsU = SJB200_UTF8_WARPS;      // warps per CTA
constexpr int kCtasPerSmU = SJB200_UTF8_CTAS;   // CTAs per SM the launch bounds aim for
constexpr int kSlotsU = SJB200_UTF8_SLOTS;      // ring slots per warp: kSlotsU - 1 blocks in flight while one is checked
constexpr int kThreadsU = 32 * kWarpsU;
constexpr int kBlockBytesU = scan4::kBlockBytes;  // 4 KiB = one TMA box of 32 rows
constexpr int kBlockRowsU = scan4::kBlockRows;

struct SmemU {
  uint8_t ring[kWarpsU][kSlotsU][kBlockBytesU];
  sj_mbar_t full[kWarpsU][kSlotsU];
};
constexpr int kSmemBytesU = int(sizeof(SmemU)) + 1024;

// one block: returns the OR of the error masks of the lane's four units.  One vote per block: a block without a byte
// >= 0x80 in any lane needs only the look at the four bytes before it; any other block is checked unit by unit without
// further votes (on multi-byte text nearly every unit of a warp holds a non-ASCII byte somewhere).
SJ_DEV uint32_t check_block(const uint8_t *T, uint32_t pw0, unsigned lane) {
  const uint32_t lane_off = lane * 128u;
  uint32_t w[32];
#pragma unroll
  for (int c = 0; c < 8; c++) {
    const sj_u4 v = *reinterpret_cast<const sj_u4 *>(T + scan4::swz(lane_off + 16u * c));
    w[4 * c] = v.x; w[4 * c + 1] = v.y; w[4 * c + 2] = v.z; w[4 * c + 3] = v.w;
  }
  uint32_t hi = 0;
#pragma unroll
  for (int i = 0; i < 32; i++) hi |= w[i];
  if (!sj_any((hi & 0x80808080u) != 0)) {
    // only the block before this one can have left a sequence open: it ends in ASCII here, which is an error
    return (lane == 0 && utf8_carry_pending(utf8_carry_from_prev_word(pw0))) ? 1u : 0u;
  }
  const uint32_t pw = (lane == 0) ? pw0 : *reinterpret_cast<const uint32_t *>(T + scan4::swz(lane_off - 4));
  utf8_carry uc = utf8_carry_from_prev_word(pw);
  uint32_t err = 0;
#pragma unroll
  for (int u = 0; u < 4; u++) {
    uint32_t pl[8];
    transpose32(w + 8 * u, pl);
    err |= utf8_check_unit(pl, uc);
  }
  return err;
}

SJ_DEV void utf8_body(const sj_tensor_map *tmap, const ScanParams &p, uint8_t *smem_raw, uint32_t smem_raw_addr) {
  SmemU *S = reinterpret_cast<SmemU *>(smem_raw + ((1024u - (smem_raw_addr & 1023u)) & 1023u));
  const unsigned tid = sj_tid(), lane = tid & 31u, warp = tid >> 5;
  if (lane == 0) {
    for (int r = 0; r < kSlotsU; r++) sj_mbar_init(&S->full[warp][r], 1);
    sj_fence_mbar_init();
  }
  sj_syncwarp();
  const uint64_t launch_start = uint64_t(p.tile_begin) * kTileBytes;
  const uint64_t launch_end_nominal = launch_start + uint64_t(p.ntiles) * kTileBytes;
  const uint64_t scan_limit = p.len < launch_end_nominal ? p.len : launch_end_nominal;
  const uint64_t nblocks = scan_limit > launch_start ? (scan_limit - launch_start + kBlockBytesU - 1) / kBlockBytesU : 0;
  const uint64_t G = uint64_t(sj_nctas()) * kWarpsU;
  const uint64_t g = uint64_t(sj_cta()) * kWarpsU + warp;
  uint32_t err = 0;
  uint32_t phase = 0;  // bit r: parity the next completion of slot r will have been waited with
  // start the load of block b into slot r; returns true when it arrives by TMA; *pw = the 4 bytes before the block
  auto issue = [&](uint64_t b, int r, uint32_t *pw) -> bool {
    const uint64_t bstart = launch_start + b * kBlockBytesU;
    const uint64_t row = bstart / 128;
    const bool full = p.use_tma && (row + kBlockRowsU <= p.len / 128);
    sj_syncwarp();  // every lane is done with the slot
    if (lane == 0) {
      if (full) {
        sj_fence_proxy_async();
        sj_mbar_arrive_expect_tx(&S->full[warp][r], kBlockBytesU);
        sj_tma_load_rows(S->ring[warp][r], tmap, &S->full[warp][r], uint32_t(row));
      }
      *pw = scan4::word_before(p.buf, p.prev_word, bstart);  // after the fence: it would wait for this load
    }
    return full;
  };
  // the loads of the next kSlotsU - 1 blocks are always in flight; q = 0 is the block checked next
  uint32_t pwq[kSlotsU - 1];
  bool tmaq[kSlotsU - 1];
#pragma unroll
  for (int q = 0; q < kSlotsU - 1; q++) {
    pwq[q] = 0x20202020u;
    tmaq[q] = false;
    if (g + uint64_t(q) * G < nblocks) tmaq[q] = issue(g + uint64_t(q) * G, q, &pwq[q]);
  }
  uint32_t r = 0, rn = kSlotsU - 1;  // slot of the block checked next / of the block asked for next
  for (uint64_t b = g; b < nblocks; b += G) {
    const uint64_t bn = b + uint64_t(kSlotsU - 1) * G;
    uint32_t pw_new = 0x20202020u;
    bool tma_new = false;
    if (bn < nblocks) tma_new = issue(bn, int(rn), &pw_new);
    uint8_t *T = S->ring[warp][r];
    if (tmaq[0]) {
      scan4::wait_bar(&S->full[warp][r], (phase >> r) & 1u, p, 32);
      phase ^= 1u << r;
    } else {
      scan4::fill_block_guarded(T, p.buf, p.len, launch_start + b * kBlockBytesU, lane);
      sj_syncwarp();
    }
    err |= check_block(T, sj_shfl(pwq[0], 0), lane);
#pragma unroll
    for (int q = 0; q + 1 < kSlotsU - 1; q++) {
      pwq[q] = pwq[q + 1];
      tmaq[q] = tmaq[q + 1];
    }
    pwq[kSlotsU - 2] = pw_new;
    tmaq[kSlotsU - 2] = tma_new;
    r = (r + 1 == uint32_t(kSlotsU)) ? 0u : r + 1;
    rn = (rn + 1 == uint32_t(kSlotsU)) ? 0u : rn + 1;
  }
  if (p.check_eof && g == 0 && lane == 0) {  // utf8_checker::check_eof (utf8_lookup4_algorithm.h L167-171): input must not end inside a sequence
    if (utf8_carry_pending(utf8_carry_from_prev_word(scan4::word_before(p.buf, p.prev_word, p.len)))) err |= 1u;
  }
  if (sj_any(err != 0) && lane == 0) sj_atomic_or(p.flags, kFlagUtf8);
  // last CTA out hands the flags over and re-arms them (same protocol as the other scans of a context)
  sj_syncthreads();
  if (tid == 0) {
    sj_threadfence();
    const uint32_t done = sj_atomic_add(p.ticket + 1, 1u);
    if (done == sj_nctas() - 1) {
      p.ticket[1] = 0;
      const uint32_t fl = sj_atomic_exch(p.flags, 0u);
      p.carry_out->count = 0;
      p.carry_out->state = 0;
      p.carry_out->ttable = 0;
      p.carry_out->flags = fl;
      if (p.carry_out_host != nullptr) {
        p.carry_out_host->count = 0;
        p.carry_out_host->state = 0;
        p.carry_out_host->ttable = 0;
        p.carry_out_host->flags = fl;
      }
      if (p.xchg.nranks != 0) {
        // sharded validate_utf8: this shard's record goes straight into every rank's window, as scan4 does.  Cuts are at
        // character boundaries, so a shard's verdict needs nothing from its neighbours: count, state and transducer are 0
        // and every rank folds state 0 (no second round); the ranks AND the verdicts (OR the flags).
        const unsigned long long w0 = xchg_word0(p.xchg.seq, 0), w1 = xchg_word1(p.xchg.seq, 0, 0, fl, kUtf8);
        for (uint32_t r = 0; r < p.xchg.nranks; r++) {
          unsigned long long *rec = p.xchg.peer[r] + (size_t(p.xchg.slot) * kMaxRanks + p.xchg.rank) * 2;
          sj_st_sys_u64(rec, w0);
          sj_st_sys_u64(rec + 1, w1);
        }
      }
      sj_threadfence();
    }
  }
}

}  // namespace utf8v2
}  // namespace sjb200
