// The reference's debugger check on the device (src/debugger.rs:74-205): every row's 17 gate identities, with the
// rotated wires of the prover's cyclic domain, and the list of failing rows with the first identity each one fails.
//
//   k_unsatisfied_rows     one thread per constraint: the first failing identity (plonk_algebra.cuh) or kSatisfied,
//                          one byte per row, and the failing rows of each block
//   k_unsatisfied_offsets  one block: exclusive prefix sum of the block counts and the total
//   k_unsatisfied_compact  each block places its failing rows at its offset, in row order (ballot + warp prefix),
//                          so the list does not depend on the order in which blocks run
// The entry points (pb200_circuit_unsatisfied, pb200_prover_unsatisfied) build the columns in prover.cu.
#include <string.h>

#include <algorithm>

#include "internal.cuh"
#include "plonk_algebra.cuh"

namespace pb {

namespace {

constexpr unsigned kRowsPerBlock = 256;
constexpr unsigned kScanThreads = 1024;
constexpr uint8_t kSatisfied = 0xFF;

PB_D Fr ld_elem(const uint4* p, size_t i) {
  const uint4 a = __ldg(p + 2 * i), b = __ldg(p + 2 * i + 1);
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}

struct RowArgs {
  const uint4* sel;  // [11][n] selector values (Poly order)
  const uint4* wv;   // [4][n] wire values a, b, c, d, zero from the constraint count up to n
  const uint4* pi;   // [n] dense public inputs, or null when there are none
  size_t n, constraints;
  Fr ed;  // dusk_jubjub::EDWARDS_D
  uint8_t* family;
  unsigned* block_count;
};

__global__ void __launch_bounds__(kRowsPerBlock) k_unsatisfied_rows(RowArgs a) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int f = -1;
  if (i < a.constraints) {
    const size_t n = a.n, iw = (i + 1) & (n - 1);  // shifted_wire_value: row i + 1 of the padded cyclic domain
    WireVals<Fr> v;
    v.a = ld_elem(a.wv, i); v.a_w = ld_elem(a.wv, iw);
    v.b = ld_elem(a.wv, n + i); v.b_w = ld_elem(a.wv, n + iw);
    v.c = ld_elem(a.wv, 2 * n + i);
    v.d = ld_elem(a.wv, 3 * n + i); v.d_w = ld_elem(a.wv, 3 * n + iw);
    const Fr pi = a.pi ? ld_elem(a.pi, i) : Fr::zero();
    f = first_failing_identity([&](int k) { return ld_elem(a.sel, (size_t)k * n + i); }, pi, a.ed, v);
    a.family[i] = f < 0 ? kSatisfied : (uint8_t)f;
  }
  const int failing = __syncthreads_count(f >= 0);
  if (threadIdx.x == 0) a.block_count[blockIdx.x] = failing;
}

// offset[b] = failing rows before block b; *total = all of them.  Thread t scans a contiguous chunk of blocks.
__global__ void __launch_bounds__(kScanThreads) k_unsatisfied_offsets(const unsigned* block_count, size_t nblk,
                                                                      unsigned long long* offset, unsigned long long* total) {
  __shared__ unsigned long long warp_sum[kScanThreads / 32];
  const size_t per = (nblk + kScanThreads - 1) / kScanThreads, lo = threadIdx.x * per, hi = lo + per < nblk ? lo + per : nblk;
  unsigned long long s = 0;
  for (size_t b = lo; b < hi; b++) s += block_count[b];
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long incl = s;
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long y = __shfl_up_sync(~0u, incl, d);
    if (lane >= (unsigned)d) incl += y;
  }
  if (lane == 31) warp_sum[warp] = incl;
  __syncthreads();
  unsigned long long before = incl - s;
  for (unsigned w = 0; w < warp; w++) before += warp_sum[w];
  for (size_t b = lo; b < hi; b++) {
    offset[b] = before;
    before += block_count[b];
  }
  if (threadIdx.x == kScanThreads - 1) *total = before;
}

__global__ void __launch_bounds__(kRowsPerBlock) k_unsatisfied_compact(const uint8_t* family, size_t constraints,
                                                                       const unsigned long long* offset, size_t cap,
                                                                       unsigned long long* rows, int32_t* families) {
  const unsigned long long base = offset[blockIdx.x];
  if (base >= cap) return;  // the whole block: base is the block's
  __shared__ unsigned warp_count[kRowsPerBlock / 32];
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint8_t f = i < constraints ? family[i] : kSatisfied;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned mask = __ballot_sync(~0u, f != kSatisfied);
  if (lane == 0) warp_count[warp] = __popc(mask);
  __syncthreads();
  if (f == kSatisfied) return;
  unsigned long long pos = base + __popc(mask & ((1u << lane) - 1));
  for (unsigned w = 0; w < warp; w++) pos += warp_count[w];
  if (pos < cap) {
    rows[pos] = i;
    families[pos] = f;
  }
}

}  // namespace

int unsatisfied_run(const uint4* sel, const uint4* wv, const uint4* pi, size_t n, size_t constraints, size_t cap, uint64_t* rows,
                    int32_t* families, size_t* n_unsatisfied, cudaStream_t st) {
  const size_t nblk = div_up(constraints, kRowsPerBlock);
  cap = std::min(cap, constraints);
  ScratchScope scope(nullptr, st);
  uint8_t* family = nullptr;
  unsigned* block_count = nullptr;
  unsigned long long *offset = nullptr, *total = nullptr, *d_rows = nullptr;
  int32_t* d_families = nullptr;
  PB_ALLOC(scope, family, constraints);
  PB_ALLOC(scope, block_count, nblk * 4);
  PB_ALLOC(scope, offset, nblk * 8);
  PB_ALLOC(scope, total, 8);
  RowArgs a;
  a.sel = sel;
  a.wv = wv;
  a.pi = pi;
  a.n = n;
  a.constraints = constraints;
  memcpy(a.ed.v, pbh::edwards_d().v, 32);
  a.family = family;
  a.block_count = block_count;
  PB_LAUNCH(k_unsatisfied_rows, (unsigned)nblk, kRowsPerBlock, 0, st, a);
  PB_LAUNCH(k_unsatisfied_offsets, 1, kScanThreads, 0, st, block_count, nblk, offset, total);
  if (cap) {
    PB_ALLOC(scope, d_rows, cap * 8);
    PB_ALLOC(scope, d_families, cap * 4);
    PB_LAUNCH(k_unsatisfied_compact, (unsigned)nblk, kRowsPerBlock, 0, st, family, constraints, offset, cap, d_rows, d_families);
  }
  PB_CUDA(cudaGetLastError());
  unsigned long long h_total = 0;
  PB_CUDA(cudaMemcpyAsync(&h_total, total, 8, cudaMemcpyDeviceToHost, st));
  PB_CUDA(stream_wait(st));
  const size_t k = std::min((size_t)h_total, cap);
  if (k) {
    PB_CUDA(cudaMemcpyAsync(rows, d_rows, k * 8, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaMemcpyAsync(families, d_families, k * 4, cudaMemcpyDeviceToHost, st));
    PB_CUDA(stream_wait(st));
  }
  *n_unsatisfied = (size_t)h_total;
  return 0;
}

}  // namespace pb

extern "C" const char* pb200_identity_family(int k) { return k >= 0 && k < pb::N_IDENTITIES ? pb::kIdentityFamilies[k] : nullptr; }
