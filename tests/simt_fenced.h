// simt_fenced.h -- buffers against inaccessible pages for the fenced passes of the host SIMT emulation
// (tests/simt_emul.cpp, tests/simt_emul_docs.cpp).  Test infrastructure only.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <sys/mman.h>
#include <unistd.h>

// `bytes` usable bytes that end exactly at a PROT_NONE page (at_end) or start right after one; the other side is fenced
// too, a page away at most.  An access outside them kills the process instead of going unnoticed.
struct Fenced {
  uint8_t *map = nullptr;
  size_t map_len = 0;
  uint8_t *p = nullptr;
  Fenced(size_t bytes, bool at_end) {
    const size_t pg = size_t(sysconf(_SC_PAGESIZE));
    const size_t data = ((bytes + pg - 1) / pg) * pg + (bytes == 0 ? pg : 0);
    map_len = data + 2 * pg;
    void *m = mmap(nullptr, map_len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (m == MAP_FAILED) { perror("mmap"); exit(3); }
    map = static_cast<uint8_t *>(m);
    if (mprotect(map, pg, PROT_NONE) != 0 || mprotect(map + pg + data, pg, PROT_NONE) != 0) { perror("mprotect"); exit(3); }
    p = at_end ? map + pg + data - bytes : map + pg;
  }
  ~Fenced() { munmap(map, map_len); }
  Fenced(const Fenced &) = delete;
  Fenced &operator=(const Fenced &) = delete;
};

inline size_t index_words(size_t len) { return ((len + 63) / 64) * 64 + 9; }  // sjb200_index_words
