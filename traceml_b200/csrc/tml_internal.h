// Private glue between the translation units of libtraceml_b200.so (not part of the ABI).
#pragma once

#include "../../include/traceml_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

// sets tml_last_error() for the calling thread and returns `code`
int tml_set_error_(int code, const char* fmt, ...);
// storage for tml_reduce_run's workspace inside the context (owned by tml_summary.cpp)
void** tml_run_ws_slot_(tml_ctx* ctx);
void tml_run_ws_free_(void* ws);

// The dense single-rank build as one device submission (tml_reduce_run's world == 1 branch).
// launch: k_window_fused, then k_bands over `series` with `bands` (the host knows n_window, so the
// band layout, before the pass) and one more row of CTAs that finalises the pass.  finish: one
// device-to-host copy, one stream wait; then reports what tml_win_fused and tml_win_bands would.
// *ok = 0: not dense, drop the bands.  Series row s starts at series + s * ld (ld >= the window's
// rows); paired = 1: rows 2m and 2m+1 share their memory and only the even rows are stored.
int tml_win_fused_chain_launch_(tml_ctx* c, uint32_t window, double* series, uint64_t ld, uint32_t paired,
                                const tml_band_args* bands, void* stream);
int tml_win_fused_chain_finish_(tml_ctx* c, void* stream, tml_win_info* out, tml_align_info* aligned,
                                tml_band_out* band_out, uint32_t* ok);

// tml_reduce_run that also emits tml_sections_json(prev, prev_sections) into prev_json (status in
// *prev_rc): an earlier reduce's sections, from the caller's own copy of its result.  The chained
// single-rank build emits them while its window pass runs, every other path after the reduce.
// Back-to-back builds (SummaryEngine.build) so keep the JSON emitter off the GPU's critical path.
int tml_summary_run_(tml_ctx* c, const tml_comm* comm, const tml_reduce_run_args* args, void* stream,
                     tml_reduce_run_out* out, const tml_reduce_run_out* prev, const tml_sections_args* prev_sections,
                     char* prev_json, size_t prev_cap, int* prev_rc);

// tml_sys_reduce_launch on the native driver's side stream (the one the process aggregates use),
// ordered behind what `stream` holds at the call: SummaryEngine.build runs K6s beside the window pass.
int tml_sys_reduce_beside_(tml_ctx* c, uint32_t max_rows, void* stream);

#ifdef __cplusplus
}
#endif

#ifdef __cplusplus
// ---------------------------------------------------------------------------------------------
// JSON text is built from many short-lived strings (rule engines, section objects: ~10^3 per
// summary).  They all die when the extern "C" entry point returns, so they come from a per-thread
// bump arena that is rewound when the outermost entry point leaves: allocation is a pointer
// increment, deallocation nothing.
#include <cstddef>
#include <cstdlib>
#include <new>
#include <string>

namespace tml_json {

struct Arena {
  static constexpr size_t BLOCK = 1u << 16;
  static constexpr int MAX_BLOCKS = 256;
  char* blocks[MAX_BLOCKS];
  int nblocks = 0, cur = 0, depth = 0;
  size_t off = 0;
  void* big[MAX_BLOCKS];  // requests that do not fit a block
  int nbig = 0;
  void* take(size_t n) {
    n = (n + 15u) & ~(size_t)15u;
    if (n > BLOCK / 4 || depth == 0) {  // oversized, or outside any scope (static initialisers)
      void* p = std::malloc(n);
      if (!p) throw std::bad_alloc();
      if (depth > 0 && nbig < MAX_BLOCKS) big[nbig++] = p;  // else: leaked on purpose (never in practice)
      return p;
    }
    if (nblocks == 0 || off + n > BLOCK) {
      if (nblocks > 0 && cur + 1 < nblocks) { ++cur; }
      else {
        if (nblocks == MAX_BLOCKS) throw std::bad_alloc();
        char* b = (char*)std::malloc(BLOCK);
        if (!b) throw std::bad_alloc();
        blocks[nblocks] = b; cur = nblocks++;
      }
      off = 0;
    }
    void* p = blocks[cur] + off;
    off += n;
    return p;
  }
  void rewind() {
    cur = 0; off = 0;
    for (int i = 0; i < nbig; ++i) std::free(big[i]);
    nbig = 0;
  }
  ~Arena() { rewind(); for (int i = 0; i < nblocks; ++i) std::free(blocks[i]); }
};

inline Arena& arena() {
  static thread_local Arena a;
  return a;
}

struct Scope {  // first statement of every entry point that builds JSON
  Arena& a;
  Scope() : a(arena()) { ++a.depth; }
  ~Scope() { if (--a.depth == 0) a.rewind(); }
  Scope(const Scope&) = delete;
  Scope& operator=(const Scope&) = delete;
};

template <class T>
struct Alloc {
  typedef T value_type;
  Alloc() noexcept {}
  template <class U> Alloc(const Alloc<U>&) noexcept {}
  T* allocate(size_t n) { return (T*)arena().take(n * sizeof(T)); }
  void deallocate(T*, size_t) noexcept {}
  template <class U> bool operator==(const Alloc<U>&) const noexcept { return true; }
  template <class U> bool operator!=(const Alloc<U>&) const noexcept { return false; }
};

typedef std::basic_string<char, std::char_traits<char>, Alloc<char>> Str;

}  // namespace tml_json
#endif
