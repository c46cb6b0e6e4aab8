// Shared host-side plumbing of libplonk_b200: error reporting, per-thread streams, launch counting.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <string>

#include "../../include/plonk_b200.h"
#include "bigint.cuh"

namespace pb {

extern thread_local std::string g_last_error;
extern std::atomic<uint64_t> g_launches;

inline int fail(int code, const char* what, const char* detail = "") {
  g_last_error = std::string(what) + (detail[0] ? ": " : "") + detail;
  return code;
}

#define PB_CUDA(expr)                                                                     \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      char _buf[256];                                                                     \
      snprintf(_buf, sizeof _buf, "%s at %s:%d", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return pb::fail(PB200_ERR_CUDA, #expr, _buf);                                       \
    }                                                                                     \
  } while (0)

#define PB_TRY(expr)          \
  do {                        \
    int _s = (expr);          \
    if (_s != 0) return _s;   \
  } while (0)

// Counted kernel launch: every kernel this library runs goes through here.
#define PB_LAUNCH(kernel, grid, block, smem, stream, ...)            \
  do {                                                               \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);      \
    pb::g_launches.fetch_add(1, std::memory_order_relaxed);          \
  } while (0)

// The calling thread's pb200 stream (created on first use, never destroyed).
cudaStream_t thread_stream();
int ensure_init();
// Host wait for everything enqueued on `st`.  Sleeps on a blocking-sync event instead of spinning in
// cudaStreamSynchronize: a proving process keeps one host thread per proof in flight, and with 8 GPUs
// x 8 proofs per box spinning threads would occupy every core of the host (PB200_SPIN=1 restores
// the spinning wait).
cudaError_t stream_wait(cudaStream_t st);
// Per-thread pinned staging buffer for small device -> host results (an async copy into pageable
// memory would make the driver wait inside the copy call).  Returns nullptr on failure.
void* pinned_scratch(size_t bytes, int slot = 0);  // slot 0: MSM results, slot 1: prover scalars

inline unsigned div_up(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }

// Streaming multiprocessors of the bound device (read by pb200_init / ensure_init before any launch);
// launch shapes aim at a few CTAs per SM.
extern std::atomic<unsigned> g_num_sms;
inline unsigned num_sms() { return g_num_sms.load(std::memory_order_relaxed); }

// Bump allocator over one device allocation.  A proof draws all its scratch from an arena owned by
// the prover (one per in-flight proof), so the steady state makes no allocator calls at all; callers
// without an arena (the stand-alone NTT / MSM entry points) use the stream-ordered pool instead.
// Everything carved from an arena is used on a single stream, so reusing memory after `reset` is
// ordered by the stream itself.
struct Arena {
  char* base = nullptr;
  size_t size = 0, off = 0;
  // Blocks start 256-byte aligned, so a list of blocks fits in the sum of round_up(bytes) over the list.
  static size_t round_up(size_t bytes) { return (bytes + 255) & ~(size_t)255; }
  void* take(size_t bytes) {
    const size_t a = round_up(off);
    if (a + bytes > size) return nullptr;
    off = a + bytes;
    return base + a;
  }
  size_t mark() const { return off; }
  void reset(size_t m) { off = m; }
};

// Scratch of one call: blocks carved from the caller's arena, or stream-ordered pool allocations
// when there is none.  Everything is released when the scope ends, on every exit path (arena: back
// to the mark it started from; pool: cudaFreeAsync, which is ordered behind the work on `st`).
struct ScratchScope {
  Arena* ar;
  cudaStream_t st;
  size_t mark;
  void* blocks[24];
  int n_blocks = 0;
  ScratchScope(Arena* a, cudaStream_t s) : ar(a), st(s), mark(a ? a->mark() : 0) {}
  ~ScratchScope() { release(); }
  ScratchScope(const ScratchScope&) = delete;
  ScratchScope& operator=(const ScratchScope&) = delete;
  void* take(size_t bytes) {
    if (ar) return ar->take(bytes);
    void* p = nullptr;
    if (n_blocks == 24 || cudaMallocAsync(&p, bytes ? bytes : 1, st) != cudaSuccess) return nullptr;
    blocks[n_blocks++] = p;
    return p;
  }
  void release() {
    if (ar) ar->reset(mark);
    for (int i = 0; i < n_blocks; i++) cudaFreeAsync(blocks[i], st);
    n_blocks = 0;
  }
};

#define PB_ALLOC(scope, ptr, bytes)                                                                  \
  do {                                                                                               \
    *(void**)&(ptr) = (scope).take(bytes);                                                           \
    if (!(ptr)) return pb::fail(PB200_ERR_CUDA, (scope).ar ? "workspace arena exhausted" : "device allocation failed", #ptr); \
  } while (0)

}  // namespace pb
