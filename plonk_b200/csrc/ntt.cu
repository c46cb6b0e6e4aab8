// Radix-2 NTT / iNTT / coset variants over the BLS12-381 scalar field on sm_90a (H100).
//
// Replaces EvaluationDomain::{fft, ifft, coset_fft, coset_ifft} (reference src/fft/domain.rs:166-232;
// the reference schedule is best_fft/serial_fft :383-463: bit-reversal + log n DIT stages whose
// twiddles are a running product).  The transform is exact field arithmetic, so any schedule that
// computes the same DFT is bit-identical; ours is GPU-first:
//
//   * N = R_0 * R_1 (* R_2): one kernel launch per factor ("pass").  A pass loads a tile of T
//     independent size-R sub-transforms into shared memory (T consecutive elements per row, so
//     every global access is a contiguous T*32-byte segment), runs log R radix-2 DIF stages out
//     of shared memory, multiplies by the inter-pass twiddle w_M^(k*lo) and stores in place.
//     The last pass stores to the digit-reversed position, so input and output are both in
//     natural order and there is no separate bit-reversal sweep.
//   * Twiddles come from per-size tables resident in HBM (w^i, i < M/2; w^(i+M/2) = -w^i), built
//     once per domain size; the sub-transform tables are tiny and stay in L1/L2.
//   * Zero padding (Vec::resize, domain.rs:174), the coset pre-scale g^i (distribute_powers,
//     domain.rs:198-204) and the 1/n and g^-i post-scales (domain.rs:187-196, 229-232) are fused
//     into the first pass' loads and the last pass' stores.
//   * Shared-memory layout is split in two 16-byte planes per element so that a warp reading
//     32 consecutive elements is bank-conflict free.
#include <cuda.h>  // CUtensorMap (types only: the encoder is looked up through the runtime, no libcuda link)

#include <mutex>
#include <vector>

#include "internal.cuh"

namespace pb {

static constexpr int kMaxLogTile = 11;  // 2048 elements = 64 KiB of shared memory per CTA
static constexpr int kNttThreads = 256;

PB_D Fr ld_fr(const uint4* p, size_t i) {
  uint4 a = __ldg(p + 2 * i), b = __ldg(p + 2 * i + 1);
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
PB_D Fr ld_fr_nc(const uint4* p, size_t i) {  // data that other CTAs may have written in this stream: plain load
  uint4 a = p[2 * i], b = p[2 * i + 1];
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
PB_D void st_fr(uint4* p, size_t i, const Fr& r) {
  p[2 * i] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
  p[2 * i + 1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}
PB_D Fr lds_fr(const uint4* s0, const uint4* s1, int i) {
  uint4 a = s0[i], b = s1[i];
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
PB_D void sts_fr(uint4* s0, uint4* s1, int i, const Fr& r) {
  s0[i] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
  s1[i] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}

// Tile accessors.  Two layouts: PLANES - two 16-byte planes per element (a warp reading 32 consecutive
// elements is bank-conflict free), filled by ordinary loads; DENSE - elements as they lie in HBM (32 bytes
// each, rows of T elements), which is what a TMA box writes.
template <bool DENSE>
PB_D Fr tile_ld(const uint4* S, int tile, int e) {
  const uint4 a = DENSE ? S[2 * e] : S[e], b = DENSE ? S[2 * e + 1] : S[tile + e];
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
template <bool DENSE>
PB_D void tile_st(uint4* S, int tile, int e, const Fr& r) {
  const uint4 a = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]), b = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
  if (DENSE) {
    S[2 * e] = a;
    S[2 * e + 1] = b;
  } else {
    S[e] = a;
    S[tile + e] = b;
  }
}

struct PassArgs {
  const uint4* in;
  uint4* out;
  unsigned long long in_len, in_stride, out_stride;  // elements
  int r;         // log2 of this pass' radix R
  int log_lo;    // log2 of the product of the later radices (0 for the last pass)
  int log_h;     // log2 of the product of the earlier radices
  int log_t;     // log2 of the tile width T
  int log_r0;    // log2 of the first pass' radix (last pass only; 0 if single pass)
  int first, last;
  const uint4* w_r;   // w_R^i,   i < R/2
  const uint4* w_m;   // w_M^i,   i < M/2, M = R * Lo  (not last)
  const uint4* pre;   // first pass: element-wise pre-scale table or null
  const uint4* post;  // last pass: element-wise post-scale table or null
  int has_scalar;     // last pass: multiply every output by `scalar`
  Fr scalar;
};

// K consecutive DIF levels l0 .. l0 + K - 1 of the size-R sub-transforms of a tile, in registers.  At level l
// the blocks have B = R >> l rows and row j meets row j + B/2 with twiddle w_R^((j mod B/2) << l).  A thread
// takes the 2^K rows jb + k * s (s = R >> (l0 + K), k < 2^K) of one column: at level l0 + i the partners are
// 2^(K-1-i) apart in k, and the position of row k inside its half-block is p + (k mod 2^(K-1-i)) * s.
template <int K, bool DENSE>
PB_D void ntt_reg_step(uint4* S, const PassArgs& a, int l0, int tid, int tile) {
  constexpr int E = 1 << K;
  const int T = 1 << a.log_t;
  const int log_s = a.r - l0 - K;
  for (int it = tid; it < (tile >> K); it += kNttThreads) {
    const int t = it & (T - 1), jj = it >> a.log_t;
    const int p = jj & ((1 << log_s) - 1), q = jj >> log_s;
    const int jb = (q << (log_s + K)) + p;
    Fr v[E];
#pragma unroll
    for (int k = 0; k < E; k++) v[k] = tile_ld<DENSE>(S, tile, ((jb + (k << log_s)) << a.log_t) + t);
#pragma unroll
    for (int i = 0; i < K; i++) {
      const int hk = 1 << (K - 1 - i);
#pragma unroll
      for (int k = 0; k < E; k++) {
        if (k & hk) continue;
        const int pos = p + ((k & (hk - 1)) << log_s);
        const Fr w = ld_fr(a.w_r, (size_t)pos << (l0 + i));
        const Fr x = v[k], y = v[k + hk];
        v[k] = x + y;
        v[k + hk] = (x - y) * w;
      }
    }
#pragma unroll
    for (int k = 0; k < E; k++) tile_st<DENSE>(S, tile, ((jb + (k << log_s)) << a.log_t) + t, v[k]);
  }
}

// TMA = true: the tile of a non-last pass arrives by cp.async.bulk.tensor (3-D tensor map over
// [batch][rows of lo elements][8 words per element], box = T x 8 words by up to 256 rows) and is signalled
// on an mbarrier; the twiddle loads of the first register step are in flight meanwhile.  Only for passes
// whose input is complete and unscaled (no zero padding, no coset pre-scale), see ntt_run.
// MAXK = 3: the DIF levels run three at a time in registers (full 2048-element tiles: every thread owns 8 rows;
// 128 registers, 2 CTAs per SM); MAXK = 1: one level at a time (smaller tiles, where an 8-row item list would
// leave most of the CTA idle; ~56 registers, so more CTAs per SM hide the shared-memory latency).
template <bool TMA, int MAXK>
__global__ void __launch_bounds__(kNttThreads, MAXK == 3 ? 2 : 1) k_ntt_pass(PassArgs a, const __grid_constant__ CUtensorMap tmap) {
  extern __shared__ __align__(128) uint4 smem[];
  __shared__ __align__(8) unsigned long long tma_bar;
  const int tid = threadIdx.x;
  const int R = 1 << a.r, T = 1 << a.log_t, tile = R << a.log_t;
  const uint4* in = a.in + 2 * (size_t)blockIdx.y * a.in_stride;
  uint4* out = a.out + 2 * (size_t)blockIdx.y * a.out_stride;
  const size_t blk = blockIdx.x;

  size_t base = 0, lo0 = 0, k0b = 0, mid = 0;
  const int log_hmid = a.log_h - a.log_r0;  // rows per first-pass digit (last pass)
  if (!a.last) {
    const int log_lo_tiles = a.log_lo - a.log_t;
    const size_t h = blk >> log_lo_tiles;
    lo0 = (blk & (((size_t)1 << log_lo_tiles) - 1)) << a.log_t;
    base = (h << (a.r + a.log_lo)) + lo0;
    if (TMA) {
      const unsigned bar = (unsigned)__cvta_generic_to_shared(&tma_bar);
      if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      }
      __syncthreads();
      if (tid == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"((unsigned)(tile * 32)) : "memory");
        const int rows_box = R < 256 ? R : 256;
        for (int c = 0; c < R; c += rows_box) {
          const unsigned dst = (unsigned)__cvta_generic_to_shared(smem + 2 * (size_t)c * T);
          asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                       ::"r"(dst), "l"((unsigned long long)&tmap), "r"(bar), "r"((int)(lo0 * 8)), "r"((int)(h * R + c)), "r"((int)blockIdx.y)
                       : "memory");
        }
      }
      asm volatile(
          "{\n\t.reg .pred P1;\n\tLAB_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], 0;\n\t@P1 bra DONE;\n\tbra LAB_WAIT;\n\tDONE:\n\t}" ::"r"(bar)
          : "memory");
    } else
    for (int idx = tid; idx < tile; idx += kNttThreads) {
      const int j = idx >> a.log_t, t = idx & (T - 1);
      const size_t g = base + ((size_t)j << a.log_lo) + t;
      Fr v;
      if (a.first) {
        if (g < a.in_len) {
          v = ld_fr(in, g);
          if (a.pre) v = v * ld_fr(a.pre, g);
        } else {
          v = Fr::zero();
        }
      } else {
        v = ld_fr_nc(in, g);
      }
      tile_st<TMA>(smem, tile, idx, v);
    }
  } else {
    const int log_k0_tiles = a.log_r0 - a.log_t;
    mid = blk >> log_k0_tiles;
    k0b = (blk & (((size_t)1 << log_k0_tiles) - 1)) << a.log_t;
    for (int idx = tid; idx < tile; idx += kNttThreads) {
      const int t = idx >> a.r, j = idx & (R - 1);
      const size_t h = ((k0b + t) << log_hmid) + mid;
      const size_t g = (h << a.r) + j;
      Fr v;
      if (a.first) {
        if (g < a.in_len) {
          v = ld_fr(in, g);
          if (a.pre) v = v * ld_fr(a.pre, g);
        } else {
          v = Fr::zero();
        }
      } else {
        v = ld_fr_nc(in, g);
      }
      tile_st<TMA>(smem, tile, (j << a.log_t) + t, v);
    }
  }
  __syncthreads();

  // log R decimation-in-frequency levels: natural order in, bit-reversed order out.  The last level
  // (twiddle 1: a bare add/sub pair) is fused into the store phase below; the others run in groups of up to
  // three levels held in registers (a thread owns the 8 elements j, j + s, .., j + 7s of one column), so the
  // tile makes one shared-memory round trip per three levels instead of one per level.
  {
    const int m = a.r - 1;
    int l0 = 0;
    if (MAXK == 3) {
      while (m - l0 >= 3) {
        ntt_reg_step<3, TMA>(smem, a, l0, tid, tile);
        __syncthreads();
        l0 += 3;
      }
      if (m - l0 == 2) {
        ntt_reg_step<2, TMA>(smem, a, l0, tid, tile);
        __syncthreads();
        l0 += 2;
      }
    }
    for (; l0 < m; l0++) {
      ntt_reg_step<1, TMA>(smem, a, l0, tid, tile);
      __syncthreads();
    }
  }

  if (a.r == 0) {  // radix 1: nothing to transform (n = 1, or a degenerate plan)
    for (int idx = tid; idx < tile; idx += kNttThreads) {
      Fr v = tile_ld<TMA>(smem, tile, idx);
      size_t o;
      if (!a.last) {
        o = base + idx;
      } else {
        o = (k0b + idx) + (mid << a.log_r0);
        if (a.post) v = v * ld_fr(a.post, o);
        if (a.has_scalar) v = v * a.scalar;
      }
      st_fr(out, o, v);
    }
    return;
  }

  // Store phase with the last butterfly stage fused in: smem rows 2m and 2m+1 hold the operands of
  // outputs k0 = bitrev(2m) (< R/2) and k0 + R/2.
  const int half_r = R >> 1;
  const size_t half_m = a.last ? 0 : ((size_t)1 << (a.r + a.log_lo - 1));
  for (int idx = tid; idx < (tile >> 1); idx += kNttThreads) {
    const int m = idx >> a.log_t, t = idx & (T - 1);
    const Fr x = tile_ld<TMA>(smem, tile, ((2 * m) << a.log_t) + t), y = tile_ld<TMA>(smem, tile, ((2 * m + 1) << a.log_t) + t);
    const int k0 = (int)(__brev((unsigned)(2 * m)) >> (32 - a.r));
    Fr v[2] = {x + y, x - y};
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int k = k0 + u * half_r;
      if (!a.last) {
        const size_t e = (size_t)k * (lo0 + t);
        Fr tw;
        if (e < half_m) {
          tw = ld_fr(a.w_m, e);
        } else {
          tw = ld_fr(a.w_m, e - half_m).neg();
        }
        st_fr(out, base + ((size_t)k << a.log_lo) + t, v[u] * tw);
      } else {
        const size_t o = (k0b + t) + (mid << a.log_r0) + ((size_t)k << a.log_h);
        Fr r = v[u];
        if (a.post) r = r * ld_fr(a.post, o);
        if (a.has_scalar) r = r * a.scalar;
        st_fr(out, o, r);
      }
    }
  }
}

// out[i] = scale * base^i, with base^(2^b) supplied by the host.
struct PowArgs {
  Fr p2[32];
  Fr scale;
};
__global__ void k_powers(uint4* out, size_t n, PowArgs pa) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr acc = pa.scale;
  size_t e = i;
#pragma unroll 1
  for (int b = 0; b < 32 && e; b++, e >>= 1)
    if (e & 1) acc = acc * pa.p2[b];
  st_fr(out, i, acc);
}

// ---------------------------------------------------------------------------------------------
// Host side: domain constants (EvaluationDomain::new, reference src/fft/domain.rs:122-158) and
// the per-size table cache.
// ---------------------------------------------------------------------------------------------
static Fr fr_from_canonical(const uint32_t (&l)[8]) {
  Fr x;
  for (int i = 0; i < 8; i++) x.v[i] = l[i];
  return x.to_mont();
}
static const uint32_t kRootOfUnity[8] = {0x439f0d2bu, 0x3829971fu, 0x8c2280b9u, 0xb6368350u,
                                         0x22c813b4u, 0xd09b6819u, 0xdfe81f20u, 0x16a2a19eu};
static const uint32_t kGenerator[8] = {7, 0, 0, 0, 0, 0, 0, 0};

Fr ntt_group_gen(int log_n, bool inverse) {  // group_gen / group_gen_inv
  Fr g = fr_from_canonical(kRootOfUnity);
  for (int i = log_n; i < 32; i++) g = g.sqr();
  return inverse ? g.inv() : g;
}
static Fr ntt_size_inv_compute(int log_n) {
  uint32_t l[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  l[log_n / 32] = 1u << (log_n % 32);
  Fr x;
  for (int i = 0; i < 8; i++) x.v[i] = l[i];
  return x.to_mont().inv();
}
Fr ntt_size_inv(int log_n) {  // cached: the host-side inversion costs ~0.1 ms
  static Fr cache[32];
  static std::once_flag once;
  std::call_once(once, [] {
    for (int i = 0; i < 32; i++) cache[i] = ntt_size_inv_compute(i);
  });
  return cache[log_n];
}
Fr ntt_coset_gen(bool inverse) {
  Fr g = fr_from_canonical(kGenerator);
  return inverse ? g.inv() : g;
}

struct TableCache {
  std::mutex mu;
  uint4* w[2][33] = {};       // [inverse][log m]: w_m^(+-i), i < max(1, m/2)
  uint4* coset_fwd = nullptr;  // g^i
  size_t coset_fwd_len = 0;
  uint4* coset_inv[33] = {};  // [log n]: g^-i / n
};
static TableCache g_tables;

// out[i] = scale * base^i for i < n, into an existing device buffer.
int fill_powers(uint4* out, size_t n, const Fr& base, const Fr& scale, cudaStream_t st) {
  PowArgs pa;
  Fr p = base;
  for (int b = 0; b < 32; b++) {
    pa.p2[b] = p;
    p = p.sqr();
  }
  pa.scale = scale;
  PB_LAUNCH(k_powers, div_up(n, 256), 256, 0, st, out, n, pa);
  PB_CUDA(cudaGetLastError());
  return 0;
}

static int build_powers(uint4** out, size_t n, const Fr& base, const Fr& scale, cudaStream_t st) {
  PB_CUDA(cudaMalloc((void**)out, n * 32));
  PowArgs pa;
  Fr p = base;
  for (int b = 0; b < 32; b++) {
    pa.p2[b] = p;
    p = p.sqr();
  }
  pa.scale = scale;
  PB_LAUNCH(k_powers, div_up(n, 256), 256, 0, st, *out, n, pa);
  PB_CUDA(cudaGetLastError());
  return 0;
}

// All table builds are issued on the caller's stream under the cache mutex; a consumer on another
// stream must not race with the build, so we synchronise the building stream once per new table.
int get_twiddles(int logm, bool inverse, cudaStream_t st, const uint4** out) {
  std::lock_guard<std::mutex> lk(g_tables.mu);
  uint4*& slot = g_tables.w[inverse ? 1 : 0][logm];
  if (!slot) {
    size_t n = logm >= 1 ? ((size_t)1 << (logm - 1)) : 1;
    PB_TRY(build_powers(&slot, n, ntt_group_gen(logm, inverse), Fr::one(), st));
    PB_CUDA(cudaStreamSynchronize(st));
  }
  *out = slot;
  return 0;
}
static int get_coset_fwd(size_t n, cudaStream_t st, const uint4** out) {
  std::lock_guard<std::mutex> lk(g_tables.mu);
  if (g_tables.coset_fwd_len < n) {
    uint4* fresh = nullptr;
    PB_TRY(build_powers(&fresh, n, ntt_coset_gen(false), Fr::one(), st));
    PB_CUDA(cudaStreamSynchronize(st));
    // the old (shorter) table may still be in use by in-flight kernels: leak it deliberately
    g_tables.coset_fwd = fresh;
    g_tables.coset_fwd_len = n;
  }
  *out = g_tables.coset_fwd;
  return 0;
}
static int get_coset_inv(int log_n, cudaStream_t st, const uint4** out) {
  std::lock_guard<std::mutex> lk(g_tables.mu);
  uint4*& slot = g_tables.coset_inv[log_n];
  if (!slot) {
    PB_TRY(build_powers(&slot, (size_t)1 << log_n, ntt_coset_gen(true), ntt_size_inv(log_n), st));
    PB_CUDA(cudaStreamSynchronize(st));
  }
  *out = slot;
  return 0;
}

static int g_ntt_plan_override[3] = {0, 0, 0};  // PB200_NTT_PLAN="r0,r1[,r2]" for tuning runs

static void ntt_plan(int L, int* radices, int* n_pass) {
  if (g_ntt_plan_override[0] && g_ntt_plan_override[0] + g_ntt_plan_override[1] + g_ntt_plan_override[2] == L) {
    int n = 0;
    for (int i = 0; i < 3; i++)
      if (g_ntt_plan_override[i]) radices[n++] = g_ntt_plan_override[i];
    *n_pass = n;
    return;
  }
  if (L <= kMaxLogTile) {
    radices[0] = L;
    *n_pass = 1;
  } else if (L <= 2 * kMaxLogTile - 2) {
    radices[0] = (L + 1) / 2;
    radices[1] = L - radices[0];
    *n_pass = 2;
  } else {
    radices[0] = (L + 2) / 3;
    radices[1] = (L - radices[0] + 1) / 2;
    radices[2] = L - radices[0] - radices[1];
    *n_pass = 3;
  }
}

// cuTensorMapEncodeTiled through the runtime's driver entry point table (no link-time libcuda dependency)
typedef CUresult (*tmap_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static tmap_encode_fn tmap_encoder() {
  static tmap_encode_fn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
    return (tmap_encode_fn)p;
  }();
  return fn;
}

int ntt_run(const uint64_t* d_in, size_t in_len, uint64_t* d_out, uint32_t log_n, int inverse,
            int coset, uint32_t batch, size_t in_stride, size_t out_stride, cudaStream_t st, Arena* ar) {
  if (log_n >= 32) return fail(PB200_ERR_INVALID_DOMAIN, "log_n >= TWO_ADACITY");
  if (batch == 0) return 0;
  static std::once_flag once;
  static int attr_status = 0;
  std::call_once(once, [] {
    const int smem_max = (2 << kMaxLogTile) * 16;
    attr_status = (int)cudaFuncSetAttribute(k_ntt_pass<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    if (attr_status == 0) attr_status = (int)cudaFuncSetAttribute(k_ntt_pass<false, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    if (attr_status == 0) attr_status = (int)cudaFuncSetAttribute(k_ntt_pass<true, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    if (attr_status == 0) attr_status = (int)cudaFuncSetAttribute(k_ntt_pass<true, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    if (const char* env = getenv("PB200_NTT_PLAN"))
      sscanf(env, "%d,%d,%d", &g_ntt_plan_override[0], &g_ntt_plan_override[1], &g_ntt_plan_override[2]);
  });
  if (attr_status != 0) return fail(PB200_ERR_CUDA, "cudaFuncSetAttribute(k_ntt_pass)");
  const size_t n = (size_t)1 << log_n;
  if (in_len > n) in_len = n;  // Vec::resize truncates (domain.rs:174)
  int radices[3], n_pass;
  ntt_plan((int)log_n, radices, &n_pass);

  const uint4* pre = nullptr;
  const uint4* post = nullptr;
  if (coset && !inverse && in_len > 0) PB_TRY(get_coset_fwd(n, st, &pre));
  if (coset && inverse) PB_TRY(get_coset_inv((int)log_n, st, &post));

  // The last pass scatters to digit-reversed positions, so it cannot run in place: with more
  // than one pass the intermediate passes work in a stream-ordered scratch buffer and the last
  // pass writes the caller's buffer.  (A single pass is one CTA per vector: loads finish before
  // stores begin, so in == out is fine there.)
  uint64_t* d_tmp = nullptr;
  ScratchScope scope(ar, st);  // later users of this memory are ordered behind these kernels by the stream
  if (n_pass > 1) PB_ALLOC(scope, d_tmp, (size_t)batch * n * 32);

  int log_h = 0;
  for (int q = 0; q < n_pass; q++) {
    PassArgs a;
    a.r = radices[q];
    int log_lo = 0;
    for (int i = q + 1; i < n_pass; i++) log_lo += radices[i];
    a.log_lo = log_lo;
    a.log_h = log_h;
    a.first = (q == 0);
    a.last = (q == n_pass - 1);
    a.log_r0 = (n_pass > 1) ? radices[0] : 0;
    // tile width: as wide as shared memory allows, but narrow enough that the launch has a few
    // CTAs per SM (small transforms are otherwise a handful of CTAs on a 132-SM H100)
    int room = kMaxLogTile - a.r;
    {
      int want = 0;  // log2(n * batch / target_ctas) - r
      const size_t per_cta = ((size_t)n * batch) / (4 * num_sms());
      while (((size_t)2 << (want + a.r)) <= per_cta) want++;
      if (want < 1) want = 1;
      if (want < room) room = want;
    }
    a.log_t = a.last ? (a.log_r0 < room ? a.log_r0 : room) : (log_lo < room ? log_lo : room);
    a.in = (const uint4*)(a.first ? d_in : d_tmp);
    a.out = (uint4*)(a.last ? d_out : d_tmp);
    a.in_len = a.first ? in_len : n;
    a.in_stride = a.first ? in_stride : n;
    a.out_stride = a.last ? out_stride : n;
    PB_TRY(get_twiddles(a.r, inverse != 0, st, &a.w_r));
    a.w_m = nullptr;
    if (!a.last) PB_TRY(get_twiddles(a.r + log_lo, inverse != 0, st, &a.w_m));
    a.pre = a.first ? pre : nullptr;
    a.post = a.last ? post : nullptr;
    a.has_scalar = (a.last && inverse && !coset) ? 1 : 0;
    a.scalar = a.has_scalar ? ntt_size_inv((int)log_n) : Fr::zero();
    const size_t tile = (size_t)1 << (a.r + a.log_t);
    dim3 grid((unsigned)(n / tile), batch);
    // TMA staging of the tile: non-last passes whose input is complete (no zero padding) and unscaled, rows of
    // at least 128 bytes.  PB200_NTT_TMA=0 keeps the ordinary loads.
    static const bool tma_env = [] {
      const char* e = getenv("PB200_NTT_TMA");
      return !e || atoi(e) != 0;
    }();
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof tmap);
    bool use_tma = tma_env && !a.last && !a.pre && a.in_len == n && a.log_t >= 2 && a.log_t <= 5 && a.r >= 1 && tmap_encoder() != nullptr;
    if (use_tma) {
      const cuuint64_t gdim[3] = {(cuuint64_t)8 << log_lo, (cuuint64_t)(n >> log_lo), (cuuint64_t)batch};
      const cuuint64_t gstr[2] = {(cuuint64_t)32 << log_lo, (cuuint64_t)a.in_stride * 32};
      const cuuint32_t rows = (cuuint32_t)std::min<size_t>((size_t)1 << a.r, 256);
      const cuuint32_t box[3] = {(cuuint32_t)8 << a.log_t, rows, 1};
      const cuuint32_t estr[3] = {1, 1, 1};
      const CUresult rc = tmap_encoder()(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, (void*)a.in, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (rc != CUDA_SUCCESS) use_tma = false;  // e.g. a stride the descriptor cannot express: ordinary loads
    }
    static const int radix_env = [] {  // PB200_NTT_RADIX8=0: one level per shared-memory round trip everywhere
      const char* e = getenv("PB200_NTT_RADIX8");
      return e ? atoi(e) : 1;
    }();
    const bool k3 = radix_env && tile >= 2048;
    if (use_tma && k3)
      PB_LAUNCH((k_ntt_pass<true, 3>), grid, kNttThreads, tile * 32, st, a, tmap);
    else if (use_tma)
      PB_LAUNCH((k_ntt_pass<true, 1>), grid, kNttThreads, tile * 32, st, a, tmap);
    else if (k3)
      PB_LAUNCH((k_ntt_pass<false, 3>), grid, kNttThreads, tile * 32, st, a, tmap);
    else
      PB_LAUNCH((k_ntt_pass<false, 1>), grid, kNttThreads, tile * 32, st, a, tmap);
    PB_CUDA(cudaGetLastError());
    log_h += a.r;
  }
  return 0;
}

}  // namespace pb
