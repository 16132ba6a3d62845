// sjb200_params.h -- geometry, scan kinds and the launch parameter block shared by the kernels, the C-ABI host
// code and the host SIMT emulation of the scan4 kernel (tests/simt_emul.cpp).  No CUDA types.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "sjb200_common.h"

namespace sjb200 {

// ---- geometry: launch parameters count the document in 32 KiB "tiles" (chunk launches start at tile boundaries);
// the kernels read it in 4 KiB blocks of 32 rows x 128 B
constexpr int kTileBytes = 32 * 1024;
constexpr int kTileRows = kTileBytes / 128;
constexpr int kMaxRanks = 8;                          // GPUs of one node that can share a scan (sjb200_comm)
constexpr int kXchgSteps = 64;                        // sharded passes whose exchange records an exchange window holds (two rounds each)
#ifndef SJB200_SCAN4_MIN_CTAS
#define SJB200_SCAN4_MIN_CTAS 2                       // CTAs per SM of the 8-scan-warp build of scan4
#endif

// ---- scan kinds (kStream: a stage-1 pass of the sharded streaming modes; kDelim: one of the sharded RS / comma-delimited
// modes.  Both scan like kIndex, only their records differ.  kTokens: a sharded stage-2-lite pass, whose record comes
// from tile_scan_kernel, sjb200_tape.cu.  kGrammar: a sharded stage-2 grammar pass, sjb200_grammar.cu.  kPointer: a
// sharded JSON Pointer pass, sjb200_pointer.cu.  kPointer = 7 is the last value the record's 3-bit kind field holds: a
// further kind needs a wider field)
enum : int { kIndex = 0, kMinify = 1, kUtf8 = 2, kStream = 3, kDelim = 4, kTokens = 5, kGrammar = 6, kPointer = 7 };
// a kTokens record's flags: kFlagInternal (the rank could not run its pass), or this rank's string bytes exceed its
// string buffer (it wrote no records)
constexpr uint32_t kTokShortFlag = 8u;

// Scanner state between consecutive launches of one document (chunked streaming,
// multi-GPU shards).  state: bit0 escape, bit1 in_string, bit2 prev_scalar.
struct Carry {
  uint64_t count;     // structurals (kIndex) or kept bytes (kMinify) emitted so far
  uint32_t state;
  uint32_t ttable;    // out only: the 6-bit transducer T(e) of everything this launch scanned
  uint32_t flags;     // out only: kFlag* bits raised by this launch (the launch also clears ScanParams::flags again)
  uint32_t reserved;
};

// One document of a multi-document stage-1 launch (ScanParams::docs).  Its elements are the launch's elements
// [first_elem, first_elem + nelem): tickets and look-back descriptors run over the concatenation of the documents.
// A single-document launch builds the one entry from the scalar fields of ScanParams.
struct DocEntry {
  const uint8_t *buf;
  uint32_t *idx_out;
  Carry *carry_out;
  Carry *carry_out_host;    // optional pinned host mirror of carry_out
  uint32_t *flags;          // kFlag* bits of this document (zero between launches; the last CTA moves them to carry_out)
  const void *tmap;         // null: plain loads.  Else the document's tensor map (4 KiB boxes), 64-byte aligned in global memory
  uint32_t len;             // document length in bytes (>= 1)
  uint32_t scan_end;        // min(len, end of the launch's tile range): blocks at or beyond it are not this launch's
  uint32_t first_elem;
  uint32_t nelem;
};
constexpr int kMaxLaunchDocs = 64;  // documents per multi-document launch (their table is copied into every CTA's shared memory)

// Where a launch of a sharded pass (sjb200_comm) stores its words: into EVERY rank's exchange window over NVLink
// (peer-mapped device memory), each tagged with seq.  nranks == 0: no exchange.
struct Xchg {
  unsigned long long *peer[kMaxRanks];  // [r] = base of rank r's window (layout below)
  uint32_t nranks, rank;
  uint32_t slot;                        // the record slot of (seq, round): [slots][kMaxRanks][2] words
  uint32_t seq;
  uint32_t kind;                        // scan4 stage 1: the kind its record carries (kIndex, kStream or kDelim)
};

struct ScanParams {
  const uint8_t *buf;       // device pointer to byte 0 of the document (or shard)
  uint64_t len;             // document length in bytes (<= 4 GiB - 1); bytes past it read as 0x20
  uint32_t pos_base;        // added to every emitted index (0: positions relative to buf)
  uint32_t prev_word;       // the 4 bytes that precede buf[0] (0x20202020 at start of document)
  uint32_t check_eof;       // 1: this launch scans the last tile -> flag a truncated UTF-8 sequence
  uint32_t use_tma;         // 1: full tiles arrive by cp.async.bulk.tensor (buf 16 B aligned)
  uint32_t tile_begin;      // first document tile of this launch (chunked streaming)
  uint32_t ntiles;          // tiles in this launch: document tiles [tile_begin, tile_begin+ntiles)
  uint32_t epoch;           // tags look-back descriptors so they need no per-launch reset
  uint32_t *idx_out;        // kIndex: device index array
  uint8_t *dst;             // kMinify: device output
  uint32_t write_sentinels; // kIndex: the launch that scans the last tile also stores idx[n]=idx[n+1]=len, idx[n+2]=0
  const Carry *carry_in;    // null: zero state, zero count
  Carry *carry_out;
  Carry *carry_out_host;    // optional second copy of the result in pinned host memory (saves the copy engine a trip between launches)
  uint32_t *flags;          // accumulated with atomicOr; zero between launches (the last CTA moves it to carry_out->flags)
  unsigned long long *count_desc;  // the look-back chain: one descriptor per scan4 element of the launch
  uint32_t *ticket;         // [0] next ticket, [1] CTAs finished, [2] scan4: aggregates published so far (4 words, zero between launches)
  unsigned long long *debug;  // optional [ntiles][8] timeline (globaltimer ns) for tuning; null in production
  // multi-GPU exchange fused into the scan (scan4 and utf8v2): the launch's last CTA stores the shard record {count,
  // state out, transducer, flags, kind} into every rank's exchange window -- the path's one exchange step (SURVEY.md 8e)
  // without a collective launch
  Xchg xchg;
  // scan4 stage 1, several whole documents in one launch: ndocs (1..kMaxLaunchDocs) entries in device memory.  buf, len,
  // use_tma, idx_out, carry_out and carry_out_host are then unused; tile_begin = 0, no carry-in, no exchange, pos_base = 0,
  // prev_word = 0x20202020, check_eof = write_sentinels = 1, and `flags` only collects what concerns the whole launch.
  // ndocs = 0: one document described by the scalar fields above.
  const DocEntry *docs;
  uint32_t ndocs;
  // Programmatic dependent launch (scan4): the launch may start while the previous launch on the stream still runs, and
  // waits for it (griddepcontrol.wait) before its first access that could conflict -- its first index store, carry,
  // sentinel or per-document flags hand-over.  early_input = 1: no input byte lies in memory the previous launch writes,
  // so the input may be read before that wait; 0: everything waits at the top.  ticket, flags and count_desc must not be
  // the previous launch's (the host alternates two sets).
  uint32_t early_input;
  unsigned long long *stamps;  // optional [2]: globaltimer at the first CTA's entry and at the last CTA's exit (tuning)
};

#if defined(__CUDACC__)
#define SJ_PARAMS_HD __host__ __device__
#else
#define SJ_PARAMS_HD
#endif
// one shard record as two independently tagged 64-bit words (8-byte stores are single transactions):
//   w0 = seq[30:0] << 33 | count[32:0]        w1 = seq << 32 | kind << 24 | flags << 16 | ttable << 8 | state_out
// kind (3 bits, 24-26) is the scan kind of the pass (kIndex 0, kMinify 1, kUtf8 2, kStream 3, kDelim 4, kTokens 5,
// kGrammar 6, kPointer 7: the field is full); count is structurals (kIndex, kStream, kDelim, kGrammar: the rank's tokens), kept bytes (kMinify), 0 (kUtf8)
// or string bytes (kTokens, whose state_out
// field carries the state the caller says the shard starts in).  Bit 26 was zero before kDelim existed, so the records of
// the other kinds are unchanged.
SJ_PARAMS_HD inline unsigned long long xchg_word0(uint32_t seq, uint64_t count) {
  return ((unsigned long long)(seq & 0x7FFFFFFFu) << 33) | (count & 0x1FFFFFFFFull);
}
SJ_PARAMS_HD inline unsigned long long xchg_word1(uint32_t seq, uint32_t state, uint32_t ttable, uint32_t flags, int kind) {
  return ((unsigned long long)seq << 32) | ((unsigned long long)(uint32_t(kind) & 7u) << 24) | ((unsigned long long)(flags & 0xFFu) << 16) |
         ((unsigned long long)(ttable & 0x3Fu) << 8) | (state & 7u);
}
SJ_PARAMS_HD inline int xchg_kind(unsigned long long w1) { return int(uint32_t(w1 >> 24) & 7u); }
SJ_PARAMS_HD inline bool xchg_complete(unsigned long long w0, unsigned long long w1, uint32_t seq) {
  return uint32_t(w0 >> 33) == (seq & 0x7FFFFFFFu) && uint32_t(w1 >> 32) == seq;
}
SJ_PARAMS_HD inline uint64_t xchg_count(unsigned long long w0) { return w0 & 0x1FFFFFFFFull; }

// The window: the records of the two rounds, [kXchgSteps][2][kMaxRanks][2] words, then the summary area of the streaming
// passes' extra round, [kXchgSteps][kMaxRanks][kSumWords] words, then the area of the delimited passes' three extra
// rounds, [kXchgSteps][kMaxRanks][kDelimWords] words, then that of the grammar passes' three rounds,
// [kXchgSteps][kMaxRanks][kGramWords] words (layouts below).  A summary is kSumWords words seq << 32 | payload:
//   0 shard length (after the trim)   1 byte of structural 0         2 byte of the last structural (kept or not)
//   3 local index of the last internal document start   4 its byte  5 / 6 object / array bracket net (int32) from that
//   start on, or over every kept structural when there is none
//   7 role of the first kept structural | role of the last << 3 | has an internal start << 6   (roles: kRole*, sjb200_docs.cu)
// (whether byte 0 is a structural is word 1 == 0 with a count > 0; the counts come from the records)
// A tokens pass (kTokens) stores its summary in the same place, from tile_scan_kernel:
//   0 shard length   1 n (tokens)   2 strings   3 local index of the first token in error (0xFFFFFFFF: none)   4 its
//   error code (0: none)   5 / 6 low / high 32 bits of the string bytes   7 zero
constexpr int kSumWords = 8;
constexpr size_t kXchgRecordWords = size_t(kXchgSteps) * 2 * kMaxRanks * 2;
constexpr size_t kXchgSummaryWords = size_t(kXchgSteps) * kMaxRanks * kSumWords;
SJ_PARAMS_HD inline size_t xchg_summary_at(uint32_t seq, uint32_t rank) {
  return kXchgRecordWords + (size_t(seq % uint32_t(kXchgSteps)) * kMaxRanks + rank) * kSumWords;
}
// A delimited pass's block of one rank, kDelimWords words, each seq << 32 | payload:
//   carry round   0 shard length (after the trim)   1 comma: bracket net over the shard's structurals (int32); RS: the
//                 shard ends inside a separator run   2 RS: the shard is whitespace / RS only
//   filter round  4 filtered entries   5 separators   6 last separator (shard-relative)   7 filtered entries before it
//                 8..15 the summary (as above) of the filtered entries   16..23 the same of the entries before the last
//                 separator (comma-delimited partial mode only)
//   tail round    24..26 the words n, n+1, n+2 of the whole call this rank holds (0 for the others)
constexpr int kDelimWords = 32;
enum : int { kDelimCarryAt = 0, kDelimCarryWords = 3, kDelimTotalsAt = 4, kDelimWalkAt = 8, kDelimWalkBelowAt = 16, kDelimTailAt = 24 };
constexpr size_t kXchgDelimWords = size_t(kXchgSteps) * kMaxRanks * kDelimWords;
SJ_PARAMS_HD inline size_t xchg_delim_at(uint32_t seq, uint32_t rank) {
  return kXchgRecordWords + kXchgSummaryWords + (size_t(seq % uint32_t(kXchgSteps)) * kMaxRanks + rank) * kDelimWords;
}
// A grammar pass's block of one rank (sjb200_document_errors_sharded), kGramWords words, each seq << 32 | payload:
//   edge round    0 n   1 ndocs   2 kGramEdge* bits   3 max_depth (saturated to 32 bits)   4 types of structurals 0, 1,
//                 n - 2, n - 1 (a byte each, 0xFF: none)   5 the table's first entry
//   record round  8 .. 8 + 2 + ceil(max_depth / 32): the stack record of the whole shard (the top of its fold tree)
//   result round  138 / 139 low / high half of the first error of the shard's leading continuation segment (global
//                 index << 8 | code, all ones: none)   140 / 141 the same of its last document   142 its other documents
//                 in error   143 the first of them (0xFFFFFFFF: none)   144 / 145 that one's error as 138 / 139
constexpr int kGramWords = 146;
enum : int { kGramEdgeAt = 0, kGramEdgeWords = 6, kGramRecAt = 8, kGramResAt = 138, kGramResWords = 8 };
enum : uint32_t { kGramEdgeFailed = 1, kGramEdgeBadTable = 2, kGramEdgeWhole = 4, kGramEdgeFirstStarts = 8, kGramEdgeLastStarts = 16 };
constexpr size_t kXchgGramWords = size_t(kXchgSteps) * kMaxRanks * kGramWords;
SJ_PARAMS_HD inline size_t xchg_gram_at(uint32_t seq, uint32_t rank) {
  return kXchgRecordWords + kXchgSummaryWords + kXchgDelimWords + (size_t(seq % uint32_t(kXchgSteps)) * kMaxRanks + rank) * kGramWords;
}
// A pointer pass's block (sjb200_at_pointer_sharded), kPtrSlotWords words per slot -- one block per window, not per rank:
// at most one document crosses each rank's end, so a rank receives the walks of at most one document and returns the
// results of at most one (kPtrMaxPointers each).
//   edge round    [kMaxRanks][kPtrEdgeWords], each seq << 32 | payload: 0 n   1 ndocs   2 kPtrEdge* bits   3 npointers
//                 4 / 5 low / high half of the pointer set's hash   6 types of structurals 0 and n - 1 (a byte each, 0xFF:
//                 none)   7 the
//                 table's first entry (n without one)   8 local index of the first token in error before it
//                 (0xFFFFFFFF: none)   9 its error code
//   count rounds  [kMaxRanks][kMaxRanks]: [rank][step] seq << 32 | walks the rank handed over in that step
//   records       [2][kPtrMaxPointers][2]: the walks handed to this rank, by pointer, double-buffered by step parity
//                 (sjb200_pointer.cuh pack_walk)
//   results       [kPtrMaxPointers][2]: seq << 32 | error, global index -- the walks of this rank's document that ended
//                 on later ranks, by pointer
constexpr int kPtrMaxPointers = 1024;  // SJB200_POINTER_SHARDED_MAX_POINTERS
constexpr int kPtrEdgeWords = 10;
enum : int { kPtrCountAt = kMaxRanks * kPtrEdgeWords, kPtrHeadWords = kPtrCountAt + kMaxRanks * kMaxRanks, kPtrRecAt = kPtrHeadWords,
             kPtrResAt = kPtrRecAt + 2 * kPtrMaxPointers * 2, kPtrSlotWords = kPtrResAt + kPtrMaxPointers * 2 };
enum : uint32_t { kPtrEdgeFailed = 1, kPtrEdgeBadTable = 2, kPtrEdgeWhole = 4, kPtrEdgeOver = 8 };
constexpr size_t kXchgPtrWords = size_t(kXchgSteps) * kPtrSlotWords;
constexpr size_t kXchgWindowWords = kXchgRecordWords + kXchgSummaryWords + kXchgDelimWords + kXchgGramWords + kXchgPtrWords;
SJ_PARAMS_HD inline size_t xchg_ptr_at(uint32_t seq) {
  return kXchgRecordWords + kXchgSummaryWords + kXchgDelimWords + kXchgGramWords + size_t(seq % uint32_t(kXchgSteps)) * kPtrSlotWords;
}

}  // namespace sjb200
