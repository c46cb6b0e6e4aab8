// Device-resident PLONK prover: Prover::new / Prover::prove (PlonkVersion::V3) of the reference
// (src/compiler/prover.rs:53-115, 415-761; preprocessing as Compiler::preprocess,
// src/compiler.rs:132-461) with every polynomial kept in HBM between rounds.
//
// The two hot kernels (NTT: ntt.cu, G1 MSM: msm.cu) are driven exactly where the reference calls
// domain.{ifft,coset_fft,coset_ifft} and commit_key.commit; the O(n) glue between them
// (SURVEY.md section 8f rows 1-3) runs as small streaming kernels here so that per proof only the
// witnesses go up and 11 x 96 B commitments + 15 x 32 B evaluations come down:
//   round 1  gather wires -> 4 x iNTT(n) -> blind -> 4 commitments            prover.rs:446-479
//   round 2  grand product (batched inversion + prefix-product scan) -> iNTT -> commit  :483-505,
//            composer/permutation.rs:213-294
//   round 3  6 x coset NTT(8n) -> fused gate/permutation quotient kernel -> coset iNTT(8n)
//            -> split + blind -> 4 commitments            quotient_poly.rs:20-310, prover.rs:545-589
//   round 4  15 evaluations (chunked Horner + tree sum)                          prover.rs:593-658
//   round 5  linearisation + both aggregate witnesses as one linear combination per opening,
//            division by (X - z) as a suffix scan, 2 commitments   linearization_poly.rs:168-231,
//            key.rs:394-417, polynomial.rs:345-367
// The Fiat-Shamir transcript (transcript.h) and a handful of scalar formulas run on the host
// between rounds.
#include <algorithm>
#include <mutex>
#include <vector>

#include "compress.h"
#include "internal.cuh"
#include "host_field.h"
#include "plonk_algebra.cuh"
#include "transcript.h"

namespace pb {

// pb200_throughput_mode(1): treat every proof as one of many in flight (a measurement aid: bench.py times the
// dominant kernel with single proofs but wants the launch shape of its timed region)
static std::atomic<int> g_force_throughput{0};

PB_D Fr ldg_fr(const uint4* p, size_t i) {
  uint4 a = __ldg(p + 2 * i), b = __ldg(p + 2 * i + 1);
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
PB_D Fr ld_fr_plain(const uint4* p, size_t i) {
  uint4 a = p[2 * i], b = p[2 * i + 1];
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
PB_D void stg_fr(uint4* p, size_t i, const Fr& r) {
  p[2 * i] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
  p[2 * i + 1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}
PB_D Fr lds_pair(const uint4* s) {  // two consecutive uint4 in shared memory
  uint4 a = s[0], b = s[1];
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
PB_D Fr fr_small(uint32_t x) {  // Montgomery form of a small constant
  Fr r = Fr::zero();
  r.v[0] = x;
  return r.to_mont();
}

// ---------------------------------------------------------------------------------------------
// small streaming kernels
// ---------------------------------------------------------------------------------------------
__global__ void k_gather_wires(const uint4* wit, const uint32_t* wires, size_t constraints, size_t n, uint4* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned k = blockIdx.y;
  Fr v = Fr::zero();
  if (i < constraints) v = ldg_fr(wit, wires[k * constraints + i]);
  stg_fr(out, (size_t)k * n + i, v);
}

// Selector columns of a compressed circuit (Compiler::compile_with_compressed): column k of gate i is
// scalars[polys[11 * gate_poly[i] + k]], zero from the gate count up to n.  cols is [11][n], grid.y = 11.
__global__ void k_expand_selectors(const uint4* __restrict__ scalars, const uint32_t* __restrict__ polys,
                                   const uint32_t* __restrict__ gate_poly, size_t constraints, size_t n, uint4* cols) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned k = blockIdx.y;
  Fr v = Fr::zero();
  if (i < constraints) v = ldg_fr(scalars, __ldg(polys + (size_t)pbz::kSelectors * __ldg(gate_poly + i) + k));
  stg_fr(cols, (size_t)k * n + i, v);
}

// The dense witness table of a compressed circuit's prover: dense[j] = wit[labels[j]] (the circuit's own numbering ->
// the dense ids its wires use).
__global__ void k_gather_witnesses(const uint4* __restrict__ wit, const unsigned long long* __restrict__ labels, size_t n_labels,
                                   uint4* dense) {
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n_labels) stg_fr(dense, j, ldg_fr(wit, __ldg(labels + j)));
}

// coeffs[i] -= b_i ; coeffs[n + i] = b_i  (Prover::blind_poly_with_blinders, prover.rs:139-152)
struct BlindArgs {
  Fr b[4][3];
  int nb;
  int npoly;
};
// Scalars of the blinder terms of a Lagrange-basis wire commitment: blinding adds b_k X^k (X^n - 1), so
// after the n wire values come -b_0, -b_1 (against [1]G, [x]G) and b_0, b_1 (against [x^n]G, [x^(n+1)]G).
__global__ void k_lagrange_tail(uint4* sc, size_t stride, size_t n, BlindArgs a) {
  const int t = threadIdx.x;
  if (t >= 2 * a.npoly) return;
  const int p = t >> 1, k = t & 1;
  stg_fr(sc, (size_t)p * stride + n + k, a.b[p][k].neg());
  stg_fr(sc, (size_t)p * stride + n + 2 + k, a.b[p][k]);
}
__global__ void k_blind(uint4* polys, size_t stride, size_t n, BlindArgs a) {
  const int t = threadIdx.x;
  if (t >= a.npoly * a.nb) return;
  const int p = t / a.nb, i = t % a.nb;
  uint4* c = polys + 2 * (size_t)p * stride;
  stg_fr(c, i, ld_fr_plain(c, i) - a.b[p][i]);
  stg_fr(c, n + i, a.b[p][i]);
}

// BlsScalar::from_bytes for a whole array (canonical little-endian integers -> Montgomery form); a value
// >= r is not canonical and raises `flag` (dusk_bytes::Error::InvalidData in the reference).
__global__ void k_fr_from_canonical(uint4* p, size_t n_elems, unsigned* flag) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_elems) return;
  const Fr x = ld_fr_plain(p, i);
  bool lt = false;
#pragma unroll
  for (int k = 7; k >= 0; k--) {
    const uint32_t m = FrParams::MOD(k);
    if (x.v[k] != m) {
      lt = x.v[k] < m;
      break;
    }
  }
  if (!lt) atomicOr(flag, 1u);
  stg_fr(p, i, x.to_mont());
}

// BlsScalar::to_bytes for a whole array, the inverse of k_fr_from_canonical: one Montgomery product by 1 per
// scalar; the output limbs are little-endian, i.e. the 32 bytes the reference writes.
__global__ void k_fr_to_canonical(const uint4* __restrict__ in, size_t n_elems, uint4* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_elems) stg_fr(out, i, ldg_fr(in, i).from_mont());
}

// Polynomial::from_coefficients_vec drops trailing zero coefficients (polynomial.rs:79-93): len[row] = index of
// the row's last non-zero coefficient + 1, 0 for an all-zero row.  polys is [gridDim.y][n], len starts at zero;
// one atomicMax per block and row.
__global__ void k_poly_trim_len(const uint4* __restrict__ polys, size_t n, unsigned* len) {
  const unsigned row = blockIdx.y;
  const uint4* p = polys + 2 * (size_t)row * n;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned m = 0;
  if (i < n) {
    const uint4 a = __ldg(p + 2 * i), b = __ldg(p + 2 * i + 1);
    if (a.x | a.y | a.z | a.w | b.x | b.y | b.z | b.w) m = (unsigned)i + 1;
  }
  m = __reduce_max_sync(0xffffffffu, m);
  __shared__ unsigned warp_max[32];
  if ((threadIdx.x & 31) == 0) warp_max[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (unsigned w = 1; w < (blockDim.x + 31) / 32; w++) m = max(m, warp_max[w]);
    if (m) atomicMax(len + row, m);
  }
}

__global__ void k_zero(uint4* p, size_t n_elems) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_elems) stg_fr(p, i, Fr::zero());
}

// sigma Lagrange values: K_col * w^idx for the encoded permutation target (col << 40 | idx)
__global__ void k_sigma_lagrange(const unsigned long long* sig, size_t n, const uint4* w_half, uint4* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 4 * n) return;
  const unsigned long long e = sig[i];
  const unsigned col = (unsigned)(e >> 40);
  const size_t idx = (size_t)(e & 0xffffffffffull);
  Fr root = (idx < n / 2 || n == 1) ? ldg_fr(w_half, idx) : ldg_fr(w_half, idx - n / 2).neg();
  const uint32_t ks[4] = {1, 7, 13, 17};
  stg_fr(out, i, root * fr_small(ks[col]));
}

// numerators and denominators of the grand product (permutation.rs:252-294)
__global__ void k_perm_terms(const uint4* wv, const uint4* sigma, const uint4* w_half, size_t n, Fr beta, Fr gamma,
                             uint4* num, uint4* den) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr root = (i < n / 2 || n == 1) ? ldg_fr(w_half, i) : ldg_fr(w_half, i - n / 2).neg();
  Fr br = beta * root;
  Fr a = ldg_fr(wv, i), b = ldg_fr(wv, n + i), c = ldg_fr(wv, 2 * n + i), d = ldg_fr(wv, 3 * n + i);
  Fr nu = (a + br + gamma) * (b + br * fr_small(7) + gamma) * (c + br * fr_small(13) + gamma) * (d + br * fr_small(17) + gamma);
  Fr de = (a + beta * ldg_fr(sigma, i) + gamma) * (b + beta * ldg_fr(sigma, n + i) + gamma) *
          (c + beta * ldg_fr(sigma, 2 * n + i) + gamma) * (d + beta * ldg_fr(sigma, 3 * n + i) + gamma);
  stg_fr(num, i, nu);
  stg_fr(den, i, de);
}

// out[i] = a[i] / b[i] (a may be null: out = 1/b).  Montgomery's trick over chunks of 8 per thread;
// zeros are left as zeros like util::batch_inversion (util.rs:87-118).
__global__ void k_batch_div(const uint4* a, const uint4* b, size_t n, uint4* out) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t base = t * 8;
  if (base >= n) return;
  Fr x[8], p[8];
  Fr acc = Fr::one();
#pragma unroll
  for (int k = 0; k < 8; k++) {
    x[k] = (base + k < n) ? ld_fr_plain(b, base + k) : Fr::one();
    if (!x[k].is_zero()) acc = acc * x[k];
    p[k] = acc;
  }
  Fr inv = acc.inv();
#pragma unroll
  for (int k = 7; k >= 0; k--) {
    if (base + k >= n) continue;
    Fr r;
    if (x[k].is_zero()) {
      r = Fr::zero();
    } else {
      r = (k > 0) ? inv * p[k - 1] : inv;
      inv = inv * x[k];
    }
    if (a) r = r * ld_fr_plain(a, base + k);
    stg_fr(out, base + k, r);
  }
}

// ---------------------------------------------------------------------------------------------
// Scan over Fr (op = multiply or add), exclusive, optional reversed index order.
// Phase 1: 256 threads x 8 elements per CTA; phase 2: scan of the CTA totals; phase 3: fix-up.
// ---------------------------------------------------------------------------------------------
template <bool MUL>
PB_D Fr scan_op(const Fr& a, const Fr& b) {
  return MUL ? a * b : a + b;
}
template <bool MUL>
PB_D Fr scan_id() {
  return MUL ? Fr::one() : Fr::zero();
}

template <bool MUL, bool REV>
__global__ void __launch_bounds__(256) k_scan_local(const uint4* in, size_t n, uint4* out, uint4* totals) {
  __shared__ uint4 sh[2][256][2];
  const int tid = threadIdx.x;
  const size_t base = ((size_t)blockIdx.x * 256 + tid) * 8;
  Fr p[8];
  Fr acc = scan_id<MUL>();
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const size_t i = base + k;
    Fr x = (i < n) ? ld_fr_plain(in, REV ? (n - 1 - i) : i) : scan_id<MUL>();
    acc = scan_op<MUL>(acc, x);
    p[k] = acc;
  }
  int cur = 0;
  sh[0][tid][0] = make_uint4(acc.v[0], acc.v[1], acc.v[2], acc.v[3]);
  sh[0][tid][1] = make_uint4(acc.v[4], acc.v[5], acc.v[6], acc.v[7]);
  __syncthreads();
  for (int d = 1; d < 256; d <<= 1) {
    Fr v = lds_pair(sh[cur][tid]);
    if (tid >= d) v = scan_op<MUL>(lds_pair(sh[cur][tid - d]), v);
    sh[cur ^ 1][tid][0] = make_uint4(v.v[0], v.v[1], v.v[2], v.v[3]);
    sh[cur ^ 1][tid][1] = make_uint4(v.v[4], v.v[5], v.v[6], v.v[7]);
    cur ^= 1;
    __syncthreads();
  }
  Fr prefix = (tid > 0) ? lds_pair(sh[cur][tid - 1]) : scan_id<MUL>();
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const size_t i = base + k;
    if (i < n) {
      Fr v = (k > 0) ? scan_op<MUL>(prefix, p[k - 1]) : prefix;
      stg_fr(out, REV ? (n - 1 - i) : i, v);
    }
  }
  if (tid == 255 && totals) {
    Fr tot = lds_pair(sh[cur][255]);
    stg_fr(totals, blockIdx.x, tot);
  }
}

template <bool MUL, bool REV>
__global__ void k_scan_fixup(uint4* out, size_t n, const uint4* block_prefix) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t blk = i / 2048;
  if (blk == 0) return;
  const size_t j = REV ? (n - 1 - i) : i;
  stg_fr(out, j, scan_op<MUL>(ld_fr_plain(block_prefix, blk), ld_fr_plain(out, j)));
}

// ---------------------------------------------------------------------------------------------
// Quotient numerator on the 8n coset (quotient_poly.rs:160-310 + all widget compute_quotient_i)
// ---------------------------------------------------------------------------------------------
struct QuotArgs {
  const uint4* w8;      // [6][8n]: z, a, b, c, d, pi coset evaluations
  const uint4* key8;    // [15][8n] prover-key coset evaluations (enum order)
  const uint4* linear8; // [8n]
  const uint4* l1_8;    // [8n] L_1 on the coset (without alpha^2)
  uint4* out;           // [8n]
  size_t n8;
  Fr alpha, beta, gamma, alpha_sq;
  // separation challenges with their powers (kappa = ch^2, kappa^2, ...), computed once on the host
  // instead of once per coset point
  SepPowers<Fr> ch_range, ch_logic, ch_fixed, ch_var;
  Fr edwards_d;  // dusk_jubjub::EDWARDS_D, Montgomery form
  Fr vh_inv[8];
  int has_range, has_logic, has_fixed, has_var;
};

// The quotient kernel evaluates ~90 Fr products per coset point.  Fully inlined that is ~23 k
// instructions per thread (~360 KB of SASS), several times what the instruction cache holds: ncu
// showed its warps waiting for instructions (stall no_instruction 2.0 per issue, multiply pipe 29 %
// busy).  Inside this kernel every product therefore goes through one out-of-line routine; `Q` is
// Fr with that product.
__device__ __noinline__ Fr fr_mul_outlined(Fr a, Fr b) { return a * b; }

struct Q {
  Fr v;
  PB_D Q() {}
  PB_D Q(const Fr& f) : v(f) {}
  static PB_D Q one() { return Q(Fr::one()); }
  static PB_D Q zero() { return Q(Fr::zero()); }
  friend PB_D Q operator+(const Q& x, const Q& y) { return Q(x.v + y.v); }
  friend PB_D Q operator-(const Q& x, const Q& y) { return Q(x.v - y.v); }
  friend PB_D Q operator*(const Q& x, const Q& y) { return Q(fr_mul_outlined(x.v, y.v)); }
  PB_D Q sqr() const { return Q(fr_mul_outlined(v, v)); }
  PB_D Q dbl() const { return Q(v.dbl()); }
};

// One point of the quotient.  The six witness rows (z, a, b, c, d, pi) have stride `ws` and are read at
// column i, the "next row" values (X -> omega X) at column iw; the prover-key tables (stride n8),
// the point itself, L_1 and 1/Z_H are read at index ki of the 8n coset; the result goes to out[oi].
//   8n coset (the reference's schedule): ws = 8n, iw = i + 8 mod 8n, ki = oi = i
//   4n coset (its even points):          ws = 4n, iw = i + 4 mod 4n, ki = 2i, oi = i
//   single points (Horner-evaluated):    ws = 16, iw = i + 8,        ki = 1 + n i, oi = i
PB_D void quotient_point(const QuotArgs& q, size_t ws, size_t i, size_t iw, size_t ki, size_t oi) {
  const size_t n8 = q.n8;
  WireVals<Q> v;
  const Q z = ldg_fr(q.w8, i), z_w = ldg_fr(q.w8, iw);
  v.a = ldg_fr(q.w8, ws + i); v.a_w = ldg_fr(q.w8, ws + iw);
  v.b = ldg_fr(q.w8, 2 * ws + i); v.b_w = ldg_fr(q.w8, 2 * ws + iw);
  v.c = ldg_fr(q.w8, 3 * ws + i);
  v.d = ldg_fr(q.w8, 4 * ws + i); v.d_w = ldg_fr(q.w8, 4 * ws + iw);
  const Q pi = ldg_fr(q.w8, 5 * ws + i);
#define KEY(k) ldg_fr(q.key8, (size_t)(k) * n8 + ki)
  const Q q_l = KEY(Q_L), q_r = KEY(Q_R), q_c = KEY(Q_C);
  // arithmetic/proverkey.rs:44-69
  Q t = (v.a * v.b * KEY(Q_M) + v.a * q_l + v.b * q_r + v.c * KEY(Q_O) + v.d * KEY(Q_F) + q_c) * KEY(Q_ARITH);
  if (q.has_range) t = t + widget_range(q.ch_range, v) * KEY(Q_RANGE);
  if (q.has_logic) t = t + widget_logic(q.ch_logic, q_c, v) * KEY(Q_LOGIC);
  if (q.has_fixed) t = t + widget_fixed(q.ch_fixed, Q(q.edwards_d), q_l, q_r, q_c, v) * KEY(Q_FIXED);
  if (q.has_var) t = t + widget_var(q.ch_var, Q(q.edwards_d), v) * KEY(Q_VAR);
  t = t + pi;
  // permutation/proverkey.rs:40-125
  const Q x = ldg_fr(q.linear8, ki);
  const Q alpha = q.alpha, beta = q.beta, gamma = q.gamma;
  const Q bx = beta * x;
  Q ident = perm_ident(v, bx, gamma) * z * alpha;
  Q copy = perm_copy3(v, beta, gamma, [&](int j) { return Q(KEY(S1 + j)); }) * (v.d + beta * KEY(S4) + gamma) * z_w * alpha;
#undef KEY
  Q l1 = Q(ldg_fr(q.l1_8, ki)) * Q(q.alpha_sq);
  t = t + ident - copy + (z - Q::one()) * l1;
  stg_fr(q.out, oi, (t * Q(q.vh_inv[ki & 7])).v);
}

__global__ void __launch_bounds__(128) k_quotient(QuotArgs q) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= q.n8) return;
  quotient_point(q, q.n8, i, (i + 8) & (q.n8 - 1), i, i);
}
// The same on the 4n coset g*H_4n = the even points of the 8n coset (PB200_QUOT4N=1, see prove_dev).
// MINB = resident CTAs per SM the register allocation is made for: 2 -> 240 registers, no spills; 3 -> 168
// registers and ~300 bytes of spills per thread (PB200_QUOT_OCC selects, default 3).
template <int MINB>
__global__ void __launch_bounds__(128, MINB) k_quotient_4n(QuotArgs q) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n4 = q.n8 >> 1;
  if (i >= n4) return;
  quotient_point(q, n4, i, (i + 4) & (n4 - 1), 2 * i, i);
}
// ... and at the eight odd points 1 + n k of the 8n coset, the witness values coming from Horner
// evaluations laid out as [6][16] (columns 0..7: x_k, columns 8..15: omega x_k).
__global__ void __launch_bounds__(128) k_quotient_pts(QuotArgs q) {
  const size_t k = threadIdx.x;
  if (k >= 8) return;
  quotient_point(q, 16, k, k + 8, 1 + (q.n8 >> 3) * k, k);
}

// flag |= any nonzero element in p[lo, hi)
__global__ void k_any_nonzero(const uint4* p, size_t lo, size_t hi, unsigned* flag) {
  size_t i = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hi) return;
  uint4 a = p[2 * i], b = p[2 * i + 1];
  if (a.x | a.y | a.z | a.w | b.x | b.y | b.z | b.w) atomicOr(flag, 1u);
}

// split t(X) into four polynomials of stride `stride` and apply b12..b14 (prover.rs:545-574)
__global__ void k_split_quotient(const uint4* t, size_t n, size_t n8, size_t stride, Fr b12, Fr b13, Fr b14, uint4* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= stride) return;
  const unsigned k = blockIdx.y;
  Fr v = Fr::zero();
  if (k < 3) {
    if (i < n) v = ld_fr_plain(t, (size_t)k * n + i);
    if (i == n) v = (k == 0) ? b12 : (k == 1 ? b13 : b14);
    if (i == 0 && k == 1) v = v - b12;
    if (i == 0 && k == 2) v = v - b13;
  } else {
    if (3 * n + i < n8) v = ld_fr_plain(t, 3 * n + i);
    if (i == 0) v = v - b14;
  }
  stg_fr(out, (size_t)k * stride + i, v);
}

// Polynomial::evaluate (polynomial.rs:120-137) for batches of (polynomial, point) jobs.  A CTA evaluates a
// block of 2048 coefficients: P_blk(x) = sum_{i < 2048} c[2048 blk + i] x^i - every thread runs Horner over
// its 8 coefficients, then a shared-memory tree folds the 256 thread values with the powers x^8, x^16, ...
// (about 27 products per thread; the first version raised x to each thread's offset with a 64-bit
// exponent, ~90 products).  k_sum_rows then runs Horner over the blocks with x^2048.
PB_D void cta_poly_eval(const uint4* poly, unsigned len, const Fr& x, uint4* out_slot) {
  __shared__ uint4 sh[256][2];
  const int tid = threadIdx.x;
  const size_t base = ((size_t)blockIdx.x * 256 + tid) * 8;
  Fr acc = Fr::zero();
  if (base < len) {
#pragma unroll
    for (int k = 7; k >= 0; k--) {
      const Fr c = (base + k < len) ? ld_fr_plain(poly, base + k) : Fr::zero();
      acc = acc * x + c;
    }
  }
  sh[tid][0] = make_uint4(acc.v[0], acc.v[1], acc.v[2], acc.v[3]);
  sh[tid][1] = make_uint4(acc.v[4], acc.v[5], acc.v[6], acc.v[7]);
  Fr pw = x.sqr().sqr().sqr();  // x^8: the weight of the neighbouring thread's value
  __syncthreads();
  for (int d = 1; d < 256; d <<= 1) {
    if ((tid & (2 * d - 1)) == 0) {
      const Fr v = lds_pair(sh[tid]) + lds_pair(sh[tid + d]) * pw;
      sh[tid][0] = make_uint4(v.v[0], v.v[1], v.v[2], v.v[3]);
      sh[tid][1] = make_uint4(v.v[4], v.v[5], v.v[6], v.v[7]);
      pw = pw.sqr();
    }
    __syncthreads();
  }
  if (tid == 0) stg_fr(out_slot, 0, lds_pair(sh[0]));
}

struct EvalJobs {
  const uint4* poly[16];
  unsigned len[16];
  Fr point[16];
  int njobs;
};
__global__ void __launch_bounds__(256) k_poly_eval(EvalJobs jobs, uint4* partial, unsigned nblocks) {
  const int j = blockIdx.y;
  cta_poly_eval(jobs.poly[j], jobs.len[j], jobs.point[j], partial + 2 * ((size_t)j * nblocks + blockIdx.x));
}
// out[j] = sum_blk partial[j][blk] x_j^(2048 blk), x_j = pts.p[j mod npts]: Horner over the blocks
struct EvalPoints {
  Fr p[16];
};
__global__ void k_sum_rows(const uint4* partial, unsigned nblocks, EvalPoints pts, int npts, uint4* out) {
  const int j = blockIdx.x;
  if (threadIdx.x != 0) return;
  Fr step = pts.p[j % npts];
#pragma unroll 1
  for (int k = 0; k < 11; k++) step = step.sqr();  // x^2048
  Fr acc = Fr::zero();
#pragma unroll 1
  for (unsigned b = nblocks; b-- > 0;) acc = acc * step + ld_fr_plain(partial, (size_t)j * nblocks + b);
  stg_fr(out, j, acc);
}

// Step 2 of the 4n-coset quotient evaluates polynomials on whole cosets s*H_8 (s = h: the points x_k; s = omega h:
// omega x_k).  With y = s^8 and F_r(y) = sum_q c_{8q+r} y^q (r < 8),
//   f(s w8^k) = sum_r w8^(rk) s^r F_r(y),
// so a coefficient costs one product (a Horner step of its residue's fold) and the 8-point DFT runs once per
// polynomial and coset.
struct Coset8Consts {
  Fr spow[2][8];   // s^r
  Fr ypow[2][16];  // y^(2^i): lane (i < 5) and warp (5..7) weights, the Horner step y^256, block weights (i >= 10)
  Fr w8pow[8];     // w8^k
};
// Jobs: row z of `rows` (row_len coefficients, stride row_stride) on coset c is job 2z + c, z < nrows; job 2 nrows
// is `tail` (tail_len coefficients) on coset 0.  A job is split into blocks of kC8Block groups of eight
// coefficients (the last block also takes the remainder); flat block index = job * row_blocks + block.
constexpr unsigned kC8Per = 4;               // groups per thread in a full block
constexpr unsigned kC8Block = 256 * kC8Per;  // = 2^10, so the block weight y^kC8Block is ypow[10]
struct Coset8Jobs {
  const uint4* rows;
  size_t row_stride;
  unsigned row_len, row_blocks;
  int nrows;
  const uint4* tail;
  unsigned tail_len, tail_blocks;
};
PB_D Fr shfl_xor_fr(const Fr& a, int m) {
  Fr r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = __shfl_xor_sync(0xffffffffu, a.v[i], m);
  return r;
}
PB_D void sts_pair(uint4* s, const Fr& a) {
  s[0] = make_uint4(a.v[0], a.v[1], a.v[2], a.v[3]);
  s[1] = make_uint4(a.v[4], a.v[5], a.v[6], a.v[7]);
}
// Block b of a job: thread t folds the groups g = b kC8Block + t + 256 i below the block's end,
//   acc_r = sum_i c_{8g+r} (y^256)^i,
// then the CTA forms B_r = sum_t y^t acc_r (weights y^lane per thread, y^(32 warp) per warp) and writes it to
// partial[8 blk + r]; the job's F_r is sum_b (y^kC8Block)^b B_r.
__global__ void __launch_bounds__(256) k_coset8_eval(Coset8Jobs J, Coset8Consts C, uint4* partial) {
  __shared__ uint4 sh[8][8][2];
  const unsigned nrow_blk = 2 * J.nrows * J.row_blocks;
  const uint4* poly;
  unsigned len, b, nb;
  int cs;
  if (blockIdx.x < nrow_blk) {
    const unsigned job = blockIdx.x / J.row_blocks;
    b = blockIdx.x - job * J.row_blocks;
    poly = J.rows + 2 * (size_t)(job >> 1) * J.row_stride;
    len = J.row_len; nb = J.row_blocks; cs = job & 1;
  } else {
    b = blockIdx.x - nrow_blk;
    poly = J.tail; len = J.tail_len; nb = J.tail_blocks; cs = 0;
  }
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t groups = (len + 7) / 8;
  const size_t end = (b + 1 == nb) ? groups : (size_t)(b + 1) * kC8Block;
  const size_t g0 = (size_t)b * kC8Block + tid;
  const int top = g0 < end ? (int)((end - 1 - g0) / 256) : -1;  // this thread's last i
  auto coef = [&](int i, int r) {
    const size_t k = 8 * (g0 + 256 * (size_t)i) + r;
    return k < len ? ld_fr_plain(poly, k) : Fr::zero();
  };
  Fr acc[8];
#pragma unroll
  for (int r = 0; r < 8; r++) acc[r] = top >= 0 ? coef(top, r) : Fr::zero();
  const Fr step = C.ypow[cs][8];
#pragma unroll 1
  for (int i = top - 1; i >= 0; i--)
#pragma unroll
    for (int r = 0; r < 8; r++) acc[r] = acc[r] * step + coef(i, r);
  Fr w = Fr::one();
#pragma unroll
  for (int k = 0; k < 5; k++)
    if (lane >> k & 1) w = w * C.ypow[cs][k];
#pragma unroll
  for (int r = 0; r < 8; r++) {
    Fr v = acc[r] * w;
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v = v + shfl_xor_fr(v, m);
    if (lane == 0) sts_pair(sh[warp][r], v);
  }
  __syncthreads();
  if (tid < 64) {  // warp tid >> 3, residue tid & 7
    Fr v = lds_pair(sh[tid >> 3][tid & 7]);
#pragma unroll
    for (int k = 0; k < 3; k++)
      if (tid >> (3 + k) & 1) v = v * C.ypow[cs][5 + k];
    sts_pair(sh[tid >> 3][tid & 7], v);
  }
  __syncthreads();
  if (tid < 8) {
    Fr s = lds_pair(sh[0][tid]);
#pragma unroll
    for (int k = 1; k < 8; k++) s = s + lds_pair(sh[k][tid]);
    stg_fr(partial, 8 * (size_t)blockIdx.x + tid, s);
  }
}
// One CTA per job: thread (p, r) sums partial B_r of the blocks b = p mod 32 with weights Z^b, Z = y^kC8Block,
// then out_k = sum_r w8^(rk) s^r F_r.  Row job 2z + c writes wpts[16 z + 8 c + k], the tail job ux[k].
__global__ void __launch_bounds__(256) k_coset8_sum(Coset8Jobs J, Coset8Consts C, const uint4* partial, uint4* wpts, uint4* ux) {
  __shared__ uint4 sh[8][8][2];
  const unsigned job = blockIdx.x, nrj = 2 * J.nrows;
  const unsigned nb = job < nrj ? J.row_blocks : J.tail_blocks;
  const int cs = job < nrj ? (job & 1) : 0;
  const unsigned tid = threadIdx.x, r = tid & 7, p = tid >> 3;
  Fr w = Fr::one();
#pragma unroll
  for (int k = 0; k < 5; k++)
    if (p >> k & 1) w = w * C.ypow[cs][10 + k];
  Fr acc = Fr::zero();
#pragma unroll 1
  for (unsigned b = p; b < nb; b += 32) {
    acc = acc + ld_fr_plain(partial, 8 * ((size_t)job * J.row_blocks + b) + r) * w;
    w = w * C.ypow[cs][15];  // Z^32
  }
  acc = acc + shfl_xor_fr(acc, 8);
  acc = acc + shfl_xor_fr(acc, 16);
  if ((tid & 31) < 8) sts_pair(sh[tid >> 5][r], acc);
  __syncthreads();
  if (tid < 8) {  // thread r reads and rewrites column r only
    Fr f = lds_pair(sh[0][r]);
#pragma unroll
    for (int k = 1; k < 8; k++) f = f + lds_pair(sh[k][r]);
    sts_pair(sh[0][r], f * C.spow[cs][r]);
  }
  __syncthreads();
  if (tid < 8) {
    Fr out = lds_pair(sh[0][0]);
#pragma unroll
    for (int j = 1; j < 8; j++) out = out + lds_pair(sh[0][j]) * C.w8pow[(j * tid) & 7];
    if (job < nrj) stg_fr(wpts, 16 * (job >> 1) + 8 * (job & 1) + tid, out);
    else stg_fr(ux, tid, out);
  }
}

// Step 3 + 4 of the 4n-coset quotient (see prove_dev): thread j < 8 computes
//   t_hi[j] = (h^-j / 8) * sum_k e_k w8^(-jk),   e_k = (t(x_k) - u(x_k)) / (-2 g^4n),
// then patches t's coefficients j and 4n + j (j < 7); a non-zero t_hi[7] raises `flag`.
struct Quot4nFix {
  Fr c;             // 1 / (-2 g^4n)
  Fr g4n;
  Fr hinv8[8];      // h^-j / 8
  Fr w8inv_pow[8];  // w8^-m
};
__global__ void k_quot4n_fix(const uint4* tx, const uint4* ux, uint4* tcoef, size_t n4, Quot4nFix f, unsigned* flag) {
  const int j = threadIdx.x;
  if (j >= 8) return;
  Fr acc = Fr::zero();
  for (int k = 0; k < 8; k++) {
    const Fr e = (ld_fr_plain(tx, k) - ld_fr_plain(ux, k)) * f.c;
    acc = acc + e * f.w8inv_pow[(j * k) & 7];
  }
  const Fr t_hi = acc * f.hinv8[j];
  if (j == 7) {
    if (!t_hi.is_zero()) atomicOr(flag, 1u);
    return;
  }
  stg_fr(tcoef, j, ld_fr_plain(tcoef, j) - f.g4n * t_hi);
  stg_fr(tcoef, n4 + j, t_hi);
}

// out[i] = sum_k coef[k] * poly[k][i]
struct LinArgs {
  const uint4* poly[24];
  unsigned len[24];
  Fr coef[24];
  int nterms;
};
__global__ void k_lincomb(LinArgs a, size_t n, uint4* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr acc = Fr::zero();
  for (int k = 0; k < a.nterms; k++)
    if (i < a.len[k]) acc = acc + ld_fr_plain(a.poly[k], i) * a.coef[k];
  stg_fr(out, i, acc);
}

// d[i] = c[i] * pw[i]
__global__ void k_mul_pointwise(const uint4* a, const uint4* b, size_t n, uint4* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) stg_fr(out, i, ld_fr_plain(a, i) * ld_fr_plain(b, i));
}
// out[i] -= 1 ;  out[i] *= c[i & 7]
__global__ void k_sub_one(uint4* p, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) stg_fr(p, i, ld_fr_plain(p, i) - Fr::one());
}
struct Period8 {
  Fr c[8];
};
__global__ void k_scale_period8(uint4* p, size_t n, Period8 c) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) stg_fr(p, i, ld_fr_plain(p, i) * c.c[i & 7]);
}

struct Quot4nConsts {
  Coset8Consts c8;  // the cosets h H_8 (points x_k = h w8^k) and omega h H_8
  Quot4nFix fix;
};

}  // namespace pb

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
using pbh::HFr;

struct pb200_prover {
  std::vector<uint8_t> label;
  size_t constraints = 0, n = 0, n8 = 0;
  int log_n = 0;
  pb200_srs* srs = nullptr;
  // (unless PB200_LAGRANGE=0) [L_0(x)]G .. [L_{n-1}(x)]G, then [1]G, [x]G, [x^n]G, [x^(n+1)]G - the wire polynomials
  // are committed through their values (short scalars) plus the two blinder terms
  pb200_srs* srs_lag = nullptr;
  pb::KeyTables keys;  // owns srs and srs_lag: this prover's alone, or shared through a pb200_pp's cache
  uint32_t* d_wires = nullptr;  // [4][constraints]
  uint4* d_polys = nullptr;     // [15][n]
  uint4* d_key8 = nullptr;      // [15][8n]
  uint4* d_linear8 = nullptr;   // [8n]
  uint4* d_l1_8 = nullptr;      // [8n]
  uint4* d_sigma = nullptr;     // [4][n]
  HFr vh_inv[8];
  pb::Fr edwards_d;       // dusk_jubjub::EDWARDS_D, Montgomery form
  pb::Quot4nConsts q4;    // constants of the 4n-coset quotient (round 3)
  int has_widget[4] = {0, 0, 0, 0};
  uint8_t comm[pb::N_POLY][48];
  size_t n_witnesses = 0;
  // a prover from a compressed circuit: the wires hold dense ids, labels[id] is the circuit's witness index
  unsigned long long* d_labels = nullptr;
  size_t n_labels = 0;
  // scratch arenas, one per proof in flight (allocated on first use, then recycled)
  mutable std::mutex ws_mu;
  mutable std::vector<pb::Arena> ws_free;
  mutable std::vector<char*> ws_all;
  size_t ws_bytes = 0;
  mutable std::atomic<int> active{0};  // proofs in flight on this prover (all host threads)
};

namespace pb {

static Fr to_dev(const HFr& x) {
  Fr r;
  memcpy(r.v, x.v, 32);
  return r;
}
static HFr to_host(const Fr& x) {
  HFr r;
  memcpy(r.v, x.v, 32);
  return r;
}

// Exclusive scan of n elements: CTA-local scans of 2048 elements, the scan of the CTA totals (by the same
// routine, so any length works: 2^22 + 8 elements are 2049 totals, two levels), then the fix-up.
template <bool MUL, bool REV>
static int fr_scan(const uint4* in, size_t n, uint4* out, cudaStream_t st, Arena* ar) {
  const unsigned nblk = div_up(n, 2048);
  uint4 *tot = nullptr, *tot_scan = nullptr;
  ScratchScope scope(ar, st);
  PB_ALLOC(scope, tot, (size_t)nblk * 32);
  PB_ALLOC(scope, tot_scan, (size_t)nblk * 32);
  PB_LAUNCH((k_scan_local<MUL, REV>), nblk, 256, 0, st, in, n, out, tot);
  if (nblk > 1) {
    PB_TRY((fr_scan<MUL, false>((const uint4*)tot, (size_t)nblk, tot_scan, st, ar)));
    PB_LAUNCH((k_scan_fixup<MUL, REV>), div_up(n, 256), 256, 0, st, out, n, (const uint4*)tot_scan);
  }
  PB_CUDA(cudaGetLastError());
  return 0;
}
static size_t fr_scan_bytes(size_t n) {  // the arena bytes fr_scan(n) carves, by the same recursion
  const size_t nblk = div_up(n, 2048);
  return 2 * Arena::round_up(nblk * 32) + (nblk > 1 ? fr_scan_bytes(nblk) : 0);
}

// The buffers prove_dev keeps for a whole proof, in carving order; prover_build sizes the arena from the same list.
enum ProofBuf { kWv, kZp, kNum, kDen, kW8, kQuot, kTcoef, kTq, kAgg, kPw, kScratch, kEvals, kPartial, kFlag, kProofBufs };
static void proof_buffers(size_t n, size_t bytes[kProofBufs]) {
  const size_t stride = n + 8;
  bytes[kWv] = 5 * n * 32;       // wire values a, b, c, d and the dense public-input vector
  bytes[kZp] = 6 * stride * 32;  // [z, a, b, c, d, pi] coefficient form: one coset-NTT batch in round 3
  bytes[kNum] = bytes[kDen] = n * 32;
  bytes[kW8] = 6 * 8 * n * 32;
  bytes[kQuot] = bytes[kTcoef] = 8 * n * 32;
  bytes[kTq] = 4 * stride * 32;
  bytes[kAgg] = bytes[kPw] = bytes[kScratch] = 2 * stride * 32;
  bytes[kEvals] = 16 * 32;
  bytes[kPartial] = (size_t)16 * div_up(stride, 2048) * 32;
  bytes[kFlag] = 4;
}

static void compress_affine(const uint64_t* raw, uint8_t out[48]) { pbh::g1_compress_raw(raw, out); }

void prover_free(pb200_prover* P);

// Stream-ordered scratch that is returned to the pool on every exit path.
struct PoolBlock {
  void* p = nullptr;
  cudaStream_t st;
  explicit PoolBlock(cudaStream_t s) : st(s) {}
  ~PoolBlock() {
    if (p) cudaFreeAsync(p, st);
  }
  cudaError_t alloc(size_t bytes) { return cudaMallocAsync(&p, bytes, st); }
  PoolBlock(const PoolBlock&) = delete;
  PoolBlock& operator=(const PoolBlock&) = delete;
};

// A prover key read from Prover::to_bytes: coefficient-form polynomials (canonical scalars) and commitments,
// both already in this file's enum order.
struct LoadedProverKey {
  const uint8_t* poly[N_POLY];
  size_t poly_len[N_POLY];
  uint8_t comm[N_POLY][48];
};

// The commit-key tables of a circuit of `constraints` gates, whose Prover::new trims the key to next_pow2(constraints +
// 6) + 6 powers (compiler.rs:121-124, srs.rs:188-196): the circuit's own from the host points srs_raw, or the cache's of
// pp.  n_srs is the point count the trimmed key must fit in.
static int circuit_key_tables(size_t constraints, const pb200_pp* pp, const uint8_t* srs_raw, size_t n_srs, cudaStream_t st,
                              KeyTables* out) {
  size_t n_trim = 1;
  while (n_trim < constraints + 6) n_trim <<= 1;
  const size_t keep = n_trim + 6;
  if (keep + 1 > n_srs) return fail(PB200_ERR_DEGREE_TOO_LARGE, "public parameters too small for this circuit (TruncatedDegreeTooLarge)");
  int log_n = 0;
  while (((size_t)1 << log_n) < constraints) log_n++;
  if (log_n + 3 >= 32) return fail(PB200_ERR_INVALID_DOMAIN, "quotient domain too large");
  return pp ? pp_key_tables(pp, keep + 1, log_n, st, out) : key_tables(srs_raw, keep + 1, log_n, st, out);
}

// selectors / wires / n_witnesses: the circuit as pb200_prover_new takes it.  keys: circuit_key_tables' for it.
// loaded: a key read by pb200_prover_from_bytes.  comp: a compressed circuit (selectors unused, wires = comp's dense ids,
// n_witnesses = the circuit's own witness count); its selector columns are expanded on the device.
static int prover_build(pb200_prover* P, const uint8_t* label, size_t label_len, size_t constraints, const uint64_t* selectors,
                        const uint32_t* wires, size_t n_witnesses, const KeyTables& keys, cudaStream_t st,
                        const LoadedProverKey* loaded = nullptr, const pbz::CompressedDescription* comp = nullptr) {
  P->label.assign(label, label + label_len);
  P->constraints = constraints;
  P->n_witnesses = n_witnesses;
  size_t n = 1;
  int log_n = 0;
  while (n < constraints) {
    n <<= 1;
    log_n++;
  }
  P->n = n;
  P->n8 = 8 * n;
  P->log_n = log_n;
  P->keys = keys;
  P->srs = keys.mono.get();
  P->srs_lag = keys.lag.get();
  const size_t n8 = P->n8;
  PB_CUDA(cudaMalloc((void**)&P->d_wires, 4 * constraints * 4));
  PB_CUDA(cudaMalloc((void**)&P->d_polys, (size_t)N_POLY * n * 32));
  PB_CUDA(cudaMalloc((void**)&P->d_key8, (size_t)N_POLY * n8 * 32));
  PB_CUDA(cudaMalloc((void**)&P->d_linear8, n8 * 32));
  PB_CUDA(cudaMalloc((void**)&P->d_l1_8, n8 * 32));
  PB_CUDA(cudaMalloc((void**)&P->d_sigma, 4 * n * 32));
  PB_CUDA(cudaMemcpyAsync(P->d_wires, wires, 4 * constraints * 4, cudaMemcpyHostToDevice, st));

  if (loaded) {
    // Prover::try_from_bytes: the polynomials arrive in coefficient form and the commitments as stored - no
    // interpolation, no MSM
    for (size_t g = 0; g < constraints; g++)
      for (int k = 0; k < 4; k++)
        if (wires[(size_t)k * constraints + g] >= n_witnesses) return fail(PB200_ERR_INVALID_ARG, "wire index out of range");
    PB_CUDA(cudaMemsetAsync(P->d_polys, 0, (size_t)N_POLY * n * 32, st));
    for (int k = 0; k < N_POLY; k++)
      if (loaded->poly_len[k])
        PB_CUDA(cudaMemcpyAsync(P->d_polys + 2 * (size_t)k * n, loaded->poly[k], loaded->poly_len[k] * 32, cudaMemcpyHostToDevice, st));
    PoolBlock flag_block(st);
    PB_CUDA(flag_block.alloc(4));
    unsigned* d_flag = (unsigned*)flag_block.p;
    PB_CUDA(cudaMemsetAsync(d_flag, 0, 4, st));
    PB_LAUNCH(k_fr_from_canonical, div_up((size_t)N_POLY * n, 256), 256, 0, st, P->d_polys, (size_t)N_POLY * n, d_flag);
    unsigned h_flag = 0;
    PB_CUDA(cudaMemcpyAsync(&h_flag, d_flag, 4, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    if (h_flag) return fail(PB200_ERR_POINT_MALFORMED, "InvalidData: a prover-key scalar is not canonical");
    memcpy(P->comm, loaded->comm, sizeof P->comm);
    const int widget_sel[4] = {Q_RANGE, Q_LOGIC, Q_FIXED, Q_VAR};
    for (int w = 0; w < 4; w++) P->has_widget[w] = (P->comm[widget_sel[w]][0] & 0x40) ? 0 : 1;
  } else {
    // selector columns, zero padded to n, then iNTT -> coefficient form (compiler.rs:149-211)
    PoolBlock cols_block(st);
    PB_CUDA(cols_block.alloc((size_t)N_POLY * n * 32));
    uint4* cols = (uint4*)cols_block.p;
    if (!comp) {
      PB_CUDA(cudaMemsetAsync(cols, 0, (size_t)N_POLY * n * 32, st));
      PB_CUDA(cudaMemcpy2DAsync(cols, n * 32, selectors, constraints * 32, constraints * 32, 11, cudaMemcpyHostToDevice, st));
    } else {
      // the scalar table (canonical -> Montgomery on the device), the polynomial table and one index per gate go up;
      // k_expand_selectors writes all 11 x n selector entries and k_sigma_lagrange below the 4 x n sigma ones
      const size_t n_sc = comp->scalars.size() / 32, n_pw = comp->polynomials.size();
      PoolBlock tab_block(st);
      PB_CUDA(tab_block.alloc(Arena::round_up(n_sc * 32) + Arena::round_up(n_pw * 4) + constraints * 4 + 4));
      uint4* d_sc = (uint4*)tab_block.p;
      uint32_t* d_pw = (uint32_t*)((char*)tab_block.p + Arena::round_up(n_sc * 32));
      uint32_t* d_gp = d_pw + Arena::round_up(n_pw * 4) / 4;
      unsigned* d_flag = d_gp + constraints;
      PB_CUDA(cudaMemcpyAsync(d_sc, comp->scalars.data(), n_sc * 32, cudaMemcpyHostToDevice, st));
      PB_CUDA(cudaMemcpyAsync(d_pw, comp->polynomials.data(), n_pw * 4, cudaMemcpyHostToDevice, st));
      PB_CUDA(cudaMemcpyAsync(d_gp, comp->gate_poly.data(), constraints * 4, cudaMemcpyHostToDevice, st));
      PB_CUDA(cudaMemsetAsync(d_flag, 0, 4, st));
      PB_LAUNCH(k_fr_from_canonical, div_up(n_sc, 256), 256, 0, st, d_sc, n_sc, d_flag);
      PB_LAUNCH(k_expand_selectors, dim3(div_up(n, 256), pbz::kSelectors), 256, 0, st, (const uint4*)d_sc, (const uint32_t*)d_pw,
                (const uint32_t*)d_gp, constraints, n, cols);
      unsigned h_flag = 0;
      PB_CUDA(cudaMemcpyAsync(&h_flag, d_flag, 4, cudaMemcpyDeviceToHost, st));
      PB_CUDA(cudaStreamSynchronize(st));  // the host tables must outlive the copies
      if (h_flag) return fail(PB200_ERR_SCALAR_MALFORMED, "BlsScalarMalformed: a compressed circuit's scalar is not canonical");
      PB_CUDA(cudaMalloc((void**)&P->d_labels, comp->labels.size() * 8));
      PB_CUDA(cudaMemcpy(P->d_labels, comp->labels.data(), comp->labels.size() * 8, cudaMemcpyHostToDevice));
      P->n_labels = comp->labels.size();
    }
    // sigma permutation on the host (composer/permutation.rs:106-141), Lagrange values on the device
    {
      const size_t n_ids = comp ? comp->labels.size() : n_witnesses;  // the dense ids of a compressed circuit
      std::vector<std::vector<uint64_t>> wmap(n_ids);
      for (size_t g = 0; g < constraints; g++)
        for (int k = 0; k < 4; k++) {
          const uint32_t w = wires[(size_t)k * constraints + g];
          if (w >= n_ids) {
            return fail(PB200_ERR_INVALID_ARG, "wire index out of range");
          }
          wmap[w].push_back(((uint64_t)k << 40) | g);
        }
      std::vector<unsigned long long> sig(4 * n);
      for (int k = 0; k < 4; k++)
        for (size_t i = 0; i < n; i++) sig[(size_t)k * n + i] = ((uint64_t)k << 40) | i;
      for (auto& lst : wmap)
        for (size_t i = 0; i < lst.size(); i++) {
          const uint64_t cur = lst[i], nxt = lst[(i + 1) % lst.size()];
          sig[(size_t)(cur >> 40) * n + (cur & 0xffffffffffull)] = nxt;
        }
      PoolBlock sig_block(st);
      PB_CUDA(sig_block.alloc(4 * n * 8));
      unsigned long long* d_sig = (unsigned long long*)sig_block.p;
      PB_CUDA(cudaMemcpyAsync(d_sig, sig.data(), 4 * n * 8, cudaMemcpyHostToDevice, st));
      const uint4* w_half = nullptr;
      PB_TRY(get_twiddles(log_n, false, st, &w_half));
      PB_LAUNCH(k_sigma_lagrange, div_up(4 * n, 256), 256, 0, st, d_sig, n, w_half, cols + 2 * (size_t)S1 * n);
      PB_CUDA(cudaStreamSynchronize(st));  // sig (host vector) must outlive the copy
    }
    PB_TRY(ntt_run((const uint64_t*)cols, n, (uint64_t*)P->d_polys, log_n, 1, 0, N_POLY, n, n, st, nullptr));
    // commitments (compiler.rs:213-232): an all-zero selector commits to the identity
    {
      std::vector<uint64_t> aff((size_t)N_POLY * 12);
      PB_TRY(msm_run(P->srs, 0, (const uint64_t*)P->d_polys, n, N_POLY, n, kMsmLatency, aff.data(), st, nullptr));
      for (int k = 0; k < N_POLY; k++) compress_affine(aff.data() + 12 * k, P->comm[k]);
      const int widget_sel[4] = {Q_RANGE, Q_LOGIC, Q_FIXED, Q_VAR};
      for (int w = 0; w < 4; w++) P->has_widget[w] = (P->comm[widget_sel[w]][0] & 0x40) ? 0 : 1;
    }
  }
  // coset evaluations over 8n (compiler.rs:306-377)
  PB_TRY(ntt_run((const uint64_t*)P->d_polys, n, (uint64_t*)P->d_key8, log_n + 3, 0, 1, N_POLY, n, n8, st, nullptr));
  {
    HFr lin[2] = {HFr::zero(), HFr::one()};
    PoolBlock lin_block(st);
    PB_CUDA(lin_block.alloc(64));
    uint4* d_lin = (uint4*)lin_block.p;
    PB_CUDA(cudaMemcpyAsync(d_lin, lin, 64, cudaMemcpyHostToDevice, st));
    PB_TRY(ntt_run((const uint64_t*)d_lin, 2, (uint64_t*)P->d_linear8, log_n + 3, 0, 1, 1, 2, n8, st, nullptr));
    PB_CUDA(cudaStreamSynchronize(st));
  }
  // vanishing polynomial on the coset has period 8 (domain.rs:340-351); its inverses are cached
  // (prover.rs:78-91).  L_1 on the coset: vh[i] * (8 / 8n) / (x_i - 1)  (quotient_poly.rs:265-284).
  {
    const HFr g = to_host(ntt_coset_gen(false)), w8n = to_host(ntt_group_gen(log_n + 3, false));
    HFr point = g.pow_u64(n), step = w8n.pow_u64(n);
    const HFr psi = to_host(ntt_size_inv(log_n + 3)) * HFr::from_u64(8);
    Period8 c;
    for (int i = 0; i < 8; i++) {
      const HFr vh = point - HFr::one();
      P->vh_inv[i] = vh.inv();
      c.c[i] = to_dev(vh * psi);
      point = point * step;
    }
    PB_CUDA(cudaMemcpyAsync(P->d_l1_8, P->d_linear8, n8 * 32, cudaMemcpyDeviceToDevice, st));
    PB_LAUNCH(k_sub_one, div_up(n8, 256), 256, 0, st, P->d_l1_8, n8);
    PB_LAUNCH(k_batch_div, div_up(div_up(n8, 8), 128), 128, 0, st, (const uint4*)nullptr, (const uint4*)P->d_l1_8, n8, P->d_l1_8);
    PB_LAUNCH(k_scale_period8, div_up(n8, 256), 256, 0, st, P->d_l1_8, n8, c);
  }
  {  // per-domain constants of round 3, computed once (each costs a host-side inversion or power)
    P->edwards_d = to_dev(pbh::edwards_d());
    const HFr g = to_host(ntt_coset_gen(false)), w8n = to_host(ntt_group_gen(log_n + 3, false));
    const HFr h = g * w8n, w8r = w8n.pow_u64(n), wn = to_host(ntt_group_gen(log_n, false)), g4n = g.pow_u64(4 * n);
    const HFr shift[2] = {h, h * wn};
    for (int c = 0; c < 2; c++) {
      HFr p = HFr::one();
      for (int r = 0; r < 8; r++, p = p * shift[c]) P->q4.c8.spow[c][r] = to_dev(p);
      for (int i = 0; i < 16; i++, p = p.sqr()) P->q4.c8.ypow[c][i] = to_dev(p);  // p = s^8 first
    }
    HFr w8k = HFr::one();
    for (int k = 0; k < 8; k++, w8k = w8k * w8r) P->q4.c8.w8pow[k] = to_dev(w8k);
    P->q4.fix.c = to_dev((g4n.dbl().neg()).inv());
    P->q4.fix.g4n = to_dev(g4n);
    const HFr h_inv = h.inv(), w8i = w8r.inv();
    HFr hj = HFr::from_u64(8).inv(), wp = HFr::one();
    for (int j = 0; j < 8; j++) {
      P->q4.fix.hinv8[j] = to_dev(hj);
      P->q4.fix.w8inv_pow[j] = to_dev(wp);
      hj = hj * h_inv;
      wp = wp * w8i;
    }
  }
  // sigma evaluations over n (prover.rs:95-100)
  PB_TRY(ntt_run((const uint64_t*)(P->d_polys + 2 * (size_t)S1 * n), n, (uint64_t*)P->d_sigma, log_n, 0, 0, 4, n, n, st, nullptr));
  PB_CUDA(cudaGetLastError());
  PB_CUDA(cudaStreamSynchronize(st));
  {  // arena of one proof: the buffers prove_dev keeps, then the largest scratch of one call it makes (each call
     // releases its scratch before the next one carves)
    const size_t stride = n + 8;
    size_t call = std::max((size_t)6 * n8 * 32, fr_scan_bytes(stride));  // ntt_run (six polynomials on the 8n coset), fr_scan
    call = std::max(call, msm_workspace_bytes(P->srs, std::min(stride, srs_len(P->srs)), 4));  // msm_run
    if (P->srs_lag) call = std::max(call, msm_workspace_bytes(P->srs_lag, n + 4, 4));          // msm_run on the wire values
    size_t bytes[kProofBufs];
    proof_buffers(n, bytes);
    P->ws_bytes = call;
    for (size_t b : bytes) P->ws_bytes += Arena::round_up(b);
    P->ws_bytes += Arena::round_up(P->n_labels * 32);  // the dense witness table of a compressed circuit
  }
  return 0;
}

// circuit_key_tables, then prover_build.  pp: the public parameters the tables come from, or null for tables of the
// prover's own from the host points srs_raw.
static int prover_make(const pb200_pp* pp, const uint8_t* srs_raw, size_t n_srs, const uint8_t* label, size_t label_len,
                       size_t constraints, const uint64_t* selectors, const uint32_t* wires, size_t n_witnesses,
                       const LoadedProverKey* loaded, const pbz::CompressedDescription* comp, pb200_prover** out) {
  cudaStream_t st = thread_stream();
  KeyTables keys;
  PB_TRY(circuit_key_tables(constraints, pp, srs_raw, n_srs, st, &keys));
  pb200_prover* P = new pb200_prover();
  const int rc = prover_build(P, label, label_len, constraints, selectors, wires, n_witnesses, keys, st, loaded, comp);
  if (rc != 0) {
    prover_free(P);  // releases whatever had been allocated; the error message is already set
    return rc;
  }
  *out = P;
  return 0;
}

int prover_new(const pb200_pp* pp, const uint8_t* label, size_t label_len, size_t constraints, const uint64_t* selectors,
               const uint32_t* wires, size_t n_witnesses, const uint8_t* srs_raw, size_t n_srs, pb200_prover** out) {
  if (constraints == 0) return fail(PB200_ERR_INVALID_ARG, "empty circuit");
  return prover_make(pp, srs_raw, n_srs, label, label_len, constraints, selectors, wires, n_witnesses, nullptr, nullptr, out);
}

// Compiler::compile_with_compressed's Prover (compiler.rs:84-112): the description decoded on the host, its selector
// columns expanded on the device.
int prover_from_compressed(const pb200_pp* pp, const uint8_t* label, size_t label_len, const uint8_t* bytes, size_t len,
                           const uint8_t* srs_raw, size_t n_srs, pb200_prover** out) {
  pbz::CompressedDescription d;
  PB_TRY(pbz::decode(bytes, len, n_srs, &d));
  if (d.gates() == 0) return fail(PB200_ERR_INVALID_ARG, "empty circuit");
  return prover_make(pp, srs_raw, n_srs, label, label_len, d.gates(), nullptr, d.wires.data(), (size_t)d.witnesses, nullptr, &d, out);
}

// Prover::try_from_bytes (src/compiler/prover.rs:265-350); the layout is spelled out at pb200_prover_from_bytes
// in include/plonk_b200.h.  With a pp, the serialized commit key must be a prefix of the pp's points, which stands in
// for the per-point validation, and the tables come from the pp's cache.
int prover_from_bytes(const pb200_pp* pp, const uint8_t* bytes, size_t len, const uint32_t* wires, size_t n_witnesses,
                      pb200_prover** out) {
  auto be64 = [](const uint8_t* p) {
    uint64_t v = 0;
    for (int i = 0; i < 8; i++) v = (v << 8) | p[i];
    return v;
  };
  auto le64 = [](const uint8_t* p) {
    uint64_t v = 0;
    for (int i = 7; i >= 0; i--) v = (v << 8) | p[i];
    return v;
  };
  const int short_rc = PB200_ERR_INVALID_ARG, bad_rc = PB200_ERR_POINT_MALFORMED;
  if (len < 48) return fail(short_rc, "NotEnoughBytes: serialized prover shorter than its header");
  const uint64_t label_len = be64(bytes), pk_len = be64(bytes + 8), ck_len = be64(bytes + 16), vk_len = be64(bytes + 24),
                 size = be64(bytes + 32), constraints = be64(bytes + 40);
  const uint8_t* p = bytes + 48;
  size_t left = len - 48;
  if (label_len > left || pk_len > left - label_len || ck_len > left - label_len - pk_len || vk_len > left - label_len - pk_len - ck_len)
    return fail(short_rc, "NotEnoughBytes: serialized prover shorter than its sections");
  size_t pow2 = 1;
  while (pow2 < constraints) pow2 <<= 1;
  if (constraints == 0 || pow2 != size) return fail(bad_rc, "InvalidData: size is not the next power of two of the constraint count");
  const uint8_t* label = p;
  const uint8_t* pk = label + label_len;
  const uint8_t* ck = pk + pk_len;
  const uint8_t* vk = ck + ck_len;
  // ProverKey::to_var_bytes (widget.rs:347-445)
  LoadedProverKey key;
  {
    size_t off = 0;
    auto need = [&](size_t k) { return k <= pk_len - off; };
    if (pk_len < 16) return fail(short_rc, "NotEnoughBytes: prover key");
    const uint64_t n = le64(pk), eval_size = le64(pk + 8);
    off = 16;
    if (n != size) return fail(bad_rc, "InvalidData: prover key domain differs from the prover's size");
    if (eval_size != 8 * n * 32 + 172) return fail(bad_rc, "InvalidData: evaluations are not over the 8n domain");
    for (int i = 0; i < N_POLY; i++) {
      if (!need(8)) return fail(short_rc, "NotEnoughBytes: prover key polynomial header");
      const uint64_t cnt = le64(pk + off);
      off += 8;
      if (cnt > n) return fail(bad_rc, "InvalidData: polynomial longer than the domain");
      if (!need(cnt * 32)) return fail(short_rc, "NotEnoughBytes: prover key polynomial");
      key.poly[kKeyFileOrder[i]] = pk + off;
      key.poly_len[kKeyFileOrder[i]] = (size_t)cnt;
      off += cnt * 32;
      if (!need(eval_size)) return fail(short_rc, "NotEnoughBytes: prover key evaluations");
      off += eval_size;  // recomputed on the device
    }
    if (!need(2 * eval_size)) return fail(short_rc, "NotEnoughBytes: linear / vanishing evaluations");
  }
  // VerifierKey::to_bytes (widget.rs:84-111)
  if (vk_len < 8 + 15 * 48) return fail(short_rc, "NotEnoughBytes: verifier key");
  // VerifierKey::n is the circuit's constraint count (compiler.rs:278-279) and try_from_bytes compares it with
  // nothing (prover.rs:331-348); the transcript takes the prover's own constraint count instead (prove_dev)
  for (int i = 0; i < N_POLY; i++) memcpy(key.comm[kKeyFileOrder[i]], vk + 8 + 48 * i, 48);
  // CommitKey::from_raw_var_bytes: validated points
  size_t n_pts = 0;
  PB_TRY(raw_commit_key_parse(ck, ck_len, 1, &n_pts, nullptr));
  std::vector<uint8_t> raw(n_pts * 96);
  PB_TRY(raw_commit_key_parse(ck, ck_len, 1, &n_pts, raw.data()));
  PB_TRY(pp ? pp_check_prefix(pp, raw.data(), n_pts) : g1_check_raw(raw.data(), n_pts));
  return prover_make(pp, raw.data(), n_pts, label, label_len, constraints, nullptr, wires, n_witnesses, &key, nullptr, out);
}

// Moves key material from HBM into the caller's (pageable) buffer without a second copy of the key on the device:
// chunks of kChunk bytes go through two device scratch blocks and the calling thread's two pinned buffers, so the
// device converts and copies chunk k + 1 while the host moves chunk k from pinned memory to its place in `out`.
struct KeyStreamer {
  static constexpr size_t kChunk = (size_t)8 << 20;
  cudaStream_t st;
  uint4* d_buf[2] = {nullptr, nullptr};
  uint8_t* h_buf[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  struct Pending {
    uint8_t* dst = nullptr;
    size_t count = 0;
    bool points = false;
  } pend[2];
  unsigned issued = 0;

  explicit KeyStreamer(cudaStream_t s) : st(s) {}
  ~KeyStreamer() {
    for (int b = 0; b < 2; b++) {
      if (pend[b].count) cudaEventSynchronize(ev[b]);  // an error path: the pinned buffers outlive this call
      if (d_buf[b]) cudaFreeAsync(d_buf[b], st);
      if (ev[b]) cudaEventDestroy(ev[b]);
    }
  }
  KeyStreamer(const KeyStreamer&) = delete;
  KeyStreamer& operator=(const KeyStreamer&) = delete;

  int init() {
    for (int b = 0; b < 2; b++) {
      PB_CUDA(cudaMallocAsync((void**)&d_buf[b], kChunk, st));
      h_buf[b] = (uint8_t*)pinned_scratch(kChunk, b);
      if (!h_buf[b]) return fail(PB200_ERR_CUDA, "pinned staging buffer allocation failed");
      PB_CUDA(cudaEventCreateWithFlags(&ev[b], cudaEventBlockingSync | cudaEventDisableTiming));
    }
    return 0;
  }
  // `count` Montgomery scalars at d_src -> count x 32 canonical bytes at dst
  int scalars(const uint4* d_src, size_t count, uint8_t* dst) {
    const size_t per = kChunk / 32;
    for (size_t at = 0; at < count; at += per) PB_TRY(issue(d_src + 2 * at, std::min(per, count - at), dst + 32 * at, false));
    return 0;
  }
  // `count` raw points at d_src -> count records of CommitKey::to_raw_var_bytes at dst
  int points(const uint4* d_src, size_t count, uint8_t* dst) {
    const size_t per = kChunk / 96;
    for (size_t at = 0; at < count; at += per)
      PB_TRY(issue(d_src + 6 * at, std::min(per, count - at), dst + (size_t)PB200_G1_RAW_SIZE * at, true));
    return 0;
  }
  int finish() {
    PB_TRY(drain(issued & 1));
    return drain((issued & 1) ^ 1);
  }

 private:
  // On entry at most the previous chunk is still pending, in the other pair of buffers.
  int issue(const uint4* d_src, size_t count, uint8_t* dst, bool points) {
    const int b = issued & 1;
    if (points) {
      PB_CUDA(cudaMemcpyAsync(h_buf[b], d_src, count * 96, cudaMemcpyDeviceToHost, st));
    } else {
      PB_LAUNCH(k_fr_to_canonical, div_up(count, 256), 256, 0, st, d_src, count, d_buf[b]);
      PB_CUDA(cudaGetLastError());
      PB_CUDA(cudaMemcpyAsync(h_buf[b], d_buf[b], count * 32, cudaMemcpyDeviceToHost, st));
    }
    PB_CUDA(cudaEventRecord(ev[b], st));
    pend[b].dst = dst;
    pend[b].count = count;
    pend[b].points = points;
    issued++;
    return drain(b ^ 1);
  }
  int drain(int b) {
    if (!pend[b].count) return 0;
    const size_t count = pend[b].count;
    pend[b].count = 0;
    PB_CUDA(cudaEventSynchronize(ev[b]));
    if (pend[b].points)
      for (size_t i = 0; i < count; i++) raw_commit_key_record(h_buf[b] + 96 * i, pend[b].dst + (size_t)PB200_G1_RAW_SIZE * i);
    else
      memcpy(pend[b].dst, h_buf[b], count * 32);
    return 0;
  }
};

// Prover::to_bytes (src/compiler/prover.rs:212-263); the layout is spelled out at pb200_prover_from_bytes in
// include/plonk_b200.h.  Reads only what the prover never changes after construction, on the caller's stream.
int prover_to_bytes(const pb200_prover* P, uint8_t* out, size_t cap, size_t* len) {
  cudaStream_t st = thread_stream();
  const size_t n = P->n, n8 = P->n8, n_pts = srs_len(P->srs);
  unsigned poly_len[N_POLY];
  {
    PoolBlock len_block(st);
    PB_CUDA(len_block.alloc(sizeof poly_len));
    PB_CUDA(cudaMemsetAsync(len_block.p, 0, sizeof poly_len, st));
    PB_LAUNCH(k_poly_trim_len, dim3(div_up(n, 256), N_POLY), 256, 0, st, (const uint4*)P->d_polys, n, (unsigned*)len_block.p);
    PB_CUDA(cudaGetLastError());
    PB_CUDA(cudaMemcpyAsync(poly_len, len_block.p, sizeof poly_len, cudaMemcpyDeviceToHost, st));
    PB_CUDA(stream_wait(st));
  }
  const size_t eval_size = n8 * 32 + 172, vk_len = 20 * 48 + 8, ck_len = 8 + n_pts * PB200_G1_RAW_SIZE;
  size_t pk_len = 16 + 17 * eval_size;
  for (int k = 0; k < N_POLY; k++) pk_len += 8 + 32 * (size_t)poly_len[k];
  const size_t total = 48 + P->label.size() + pk_len + ck_len + vk_len;
  *len = total;
  if (!out) return 0;
  if (cap < total) return fail(PB200_ERR_INVALID_ARG, "output buffer too small");

  uint8_t* w = out;
  auto be64 = [&](uint64_t v) {
    for (int i = 7; i >= 0; i--) *w++ = (uint8_t)(v >> (8 * i));
  };
  auto le64 = [&](uint64_t v) {
    for (int i = 0; i < 8; i++) *w++ = (uint8_t)(v >> (8 * i));
  };
  auto scalar = [&](const HFr& x) {  // BlsScalar::to_bytes
    const HFr c = x.from_mont();
    memcpy(w, c.v, 32);
    w += 32;
  };
  // EvaluationDomain::to_bytes of the 8n domain (domain.rs:59-80), in front of every Evaluations
  uint8_t domain[172];
  {
    w = domain;
    le64(n8);
    const uint32_t log8 = (uint32_t)P->log_n + 3;
    for (int i = 0; i < 4; i++) *w++ = (uint8_t)(log8 >> (8 * i));
    scalar(HFr::from_u64(n8));
    scalar(to_host(ntt_size_inv(P->log_n + 3)));
    scalar(to_host(ntt_group_gen(P->log_n + 3, false)));
    scalar(to_host(ntt_group_gen(P->log_n + 3, true)));
    scalar(to_host(ntt_coset_gen(true)));
  }
  KeyStreamer stream(st);
  PB_TRY(stream.init());
  auto evaluations = [&](const uint4* d_evals) {  // Evaluations::to_var_bytes (evaluations.rs:52-61)
    memcpy(w, domain, sizeof domain);
    w += sizeof domain;
    uint8_t* at = w;
    w += n8 * 32;
    return stream.scalars(d_evals, n8, at);
  };
  w = out;
  be64(P->label.size());
  be64(pk_len);
  be64(ck_len);
  be64(vk_len);
  be64(n);
  be64(P->constraints);
  memcpy(w, P->label.data(), P->label.size());
  w += P->label.size();
  // ProverKey::to_var_bytes (widget.rs:347-445)
  le64(n);
  le64(eval_size);
  for (int i = 0; i < N_POLY; i++) {
    const int k = kKeyFileOrder[i];
    le64(poly_len[k]);
    PB_TRY(stream.scalars(P->d_polys + 2 * (size_t)k * n, poly_len[k], w));
    w += 32 * (size_t)poly_len[k];
    PB_TRY(evaluations(P->d_key8 + 2 * (size_t)k * n8));
  }
  PB_TRY(evaluations(P->d_linear8));
  {  // v_h_coset_8n (compiler.rs:424-425): (g w_8n^i)^n - 1 has period 8; the prover keeps only the inverses
    memcpy(w, domain, sizeof domain);
    w += sizeof domain;
    uint8_t* base = w;
    const HFr g = to_host(ntt_coset_gen(false)), w8n = to_host(ntt_group_gen(P->log_n + 3, false));
    HFr point = g.pow_u64(n);
    const HFr step = w8n.pow_u64(n);
    for (int i = 0; i < 8; i++) {
      scalar(point - HFr::one());
      point = point * step;
    }
    for (size_t have = 256; have < n8 * 32; have *= 2) memcpy(base + have, base, have);  // n8 is 8 times a power of two
    w = base + n8 * 32;
  }
  // CommitKey::to_raw_var_bytes (key.rs:215-229) of the trimmed key: window 0 of the MSM table holds the points as
  // they were uploaded
  le64(n_pts);
  PB_TRY(stream.points(srs_points(P->srs), n_pts, w));
  w += n_pts * PB200_G1_RAW_SIZE;
  // VerifierKey::to_bytes (widget.rs:84-111)
  le64(P->constraints);
  for (int i = 0; i < N_POLY; i++) {
    memcpy(w, P->comm[kKeyFileOrder[i]], 48);
    w += 48;
  }
  memset(w, 0, vk_len - 8 - 48 * N_POLY);
  return stream.finish();
}

void prover_free(pb200_prover* P) {
  if (!P) return;
  cudaFree(P->d_wires); cudaFree(P->d_polys); cudaFree(P->d_key8); cudaFree(P->d_linear8); cudaFree(P->d_l1_8); cudaFree(P->d_sigma);
  cudaFree(P->d_labels);
  for (char* w : P->ws_all) cudaFree(w);
  delete P;
}

// The public inputs of a proof: positions inside the circuit, strictly increasing (the reference keeps them in a
// BTreeMap keyed by gate index, composer.rs:465-480: ascending, no duplicates).
static int check_public_inputs(const uint64_t* pi_idx, const uint64_t* pi_vals, size_t n_pi, size_t constraints) {
  if (n_pi && (!pi_idx || !pi_vals)) return fail(PB200_ERR_INVALID_ARG, "public inputs announced but not given");
  for (size_t i = 0; i < n_pi; i++) {
    if (pi_idx[i] >= constraints) return fail(PB200_ERR_INVALID_ARG, "public input index out of range");
    if (i && pi_idx[i] <= pi_idx[i - 1]) return fail(PB200_ERR_INVALID_ARG, "public input positions must be strictly increasing");
  }
  return 0;
}

// Prover::prove_inner.  d_wit: n_witnesses Fr on the device; pi_*: host.  version: PB200_PLONK_V3 or V2, which read
// the same except for the transcript seed (Prover::transcript_for_version, prover.rs:404-413).
int prove_dev(const pb200_prover* P, int version, const uint64_t* d_wit, const uint64_t* pi_idx, const uint64_t* pi_vals,
              size_t n_pi, const uint64_t* blinders_host, uint8_t* out_proof, cudaStream_t st) {
  const size_t n = P->n, n8 = P->n8, stride = n + 8;
  const int log_n = P->log_n;
  struct InFlight {
    const pb200_prover* P;
    explicit InFlight(const pb200_prover* p) : P(p) { P->active.fetch_add(1, std::memory_order_relaxed); }
    ~InFlight() { P->active.fetch_sub(1, std::memory_order_relaxed); }
  } in_flight(P);
  static const int hint_at = [] {  // PB200_THROUGHPUT_AT=<k>: proofs in flight from which the prover is busy (0 = never)
    const char* e = getenv("PB200_THROUGHPUT_AT");
    return e ? atoi(e) : 2;
  }();
  // Busy: other proofs keep the GPU filled, so the MSMs take their throughput shape; `active` changes while this proof
  // runs, so it is read at each MSM.  Dense scalars then use one lane per bucket and the wide heavy chunks.
  auto busy = [&] { return hint_at > 0 && (g_force_throughput.load(std::memory_order_relaxed) || P->active.load(std::memory_order_relaxed) >= hint_at); };
  auto dense_shape = [&] { const bool b = busy(); return MsmShape{!b, b}; };
  const HFr* BL = (const HFr*)blinders_host;
  // the prover's own constraint count stands for VerifierKey::n
  pbh::Transcript tr = version == PB200_PLONK_V3
                           ? pbh::seed_transcript(P->label.data(), P->label.size(), P->constraints, P->comm[0], P->constraints)
                           : pbh::seed_transcript_legacy(P->label.data(), P->label.size(), P->constraints, P->comm[0], P->constraints);
  const HFr* PIV = (const HFr*)pi_vals;
  PB_TRY(check_public_inputs(pi_idx, pi_vals, n_pi, P->constraints));
  for (size_t i = 0; i < n_pi; i++) tr.append_scalar("pi", PIV[i]);
  const uint4* w_half = nullptr;
  PB_TRY(get_twiddles(log_n, false, st, &w_half));

  // workspace: one arena per proof in flight
  Arena arena;
  {
    std::lock_guard<std::mutex> lk(P->ws_mu);
    if (!P->ws_free.empty()) {
      arena = P->ws_free.back();
      P->ws_free.pop_back();
    }
  }
  if (!arena.base) {
    char* mem = nullptr;
    PB_CUDA(cudaMalloc((void**)&mem, P->ws_bytes));
    arena.base = mem;
    arena.size = P->ws_bytes;
    std::lock_guard<std::mutex> lk(P->ws_mu);
    P->ws_all.push_back(mem);
  }
  arena.off = 0;
  struct Release {
    const pb200_prover* P;
    Arena* a;
    cudaStream_t st;
    ~Release() {
      stream_wait(st);  // error paths may leave work in flight
      a->off = 0;
      std::lock_guard<std::mutex> lk(P->ws_mu);
      P->ws_free.push_back(*a);
    }
  } release{P, &arena, st};
  Arena* ar = &arena;
  ScratchScope scope(ar, st);
  const unsigned eval_blocks = div_up(stride, 2048);
  size_t bytes[kProofBufs];
  void* kept[kProofBufs];
  proof_buffers(n, bytes);
  for (int i = 0; i < kProofBufs; i++) PB_ALLOC(scope, kept[i], bytes[i]);
  uint4 *wv = (uint4*)kept[kWv], *zp = (uint4*)kept[kZp], *num = (uint4*)kept[kNum], *den = (uint4*)kept[kDen], *w8 = (uint4*)kept[kW8],
        *quot = (uint4*)kept[kQuot], *tcoef = (uint4*)kept[kTcoef], *tq = (uint4*)kept[kTq], *agg = (uint4*)kept[kAgg],
        *pw = (uint4*)kept[kPw], *scratch = (uint4*)kept[kScratch], *evals_d = (uint4*)kept[kEvals], *partial = (uint4*)kept[kPartial];
  unsigned* flag = (unsigned*)kept[kFlag];
  uint4 *wp = zp + 2 * stride, *pi_dense = wv + 2 * 4 * n;

  uint64_t aff[4 * 12];
  uint8_t c48[N_COMM][48];
  Challenges ch;

  if (P->d_labels) {  // a compressed circuit's prover: its wires index the dense table of the labels they use
    uint4* dense = nullptr;
    PB_ALLOC(scope, dense, P->n_labels * 32);
    PB_LAUNCH(k_gather_witnesses, div_up(P->n_labels, 256), 256, 0, st, (const uint4*)d_wit, (const unsigned long long*)P->d_labels,
              P->n_labels, dense);
    d_wit = (const uint64_t*)dense;
  }

  // ---- round 1 -------------------------------------------------------------------------------
  PB_LAUNCH(k_gather_wires, dim3(div_up(n, 256), 4), 256, 0, st, (const uint4*)d_wit, (const uint32_t*)P->d_wires, P->constraints, n, wv);
  // dense public-input vector (prover.rs:434-438) rides along with the wire iNTTs (prover.rs:519-521)
  if (n_pi) {
    PB_CUDA(cudaMemsetAsync(pi_dense, 0, n * 32, st));
    for (size_t i = 0; i < n_pi; i++)
      PB_CUDA(cudaMemcpyAsync(pi_dense + 2 * pi_idx[i], PIV + i, 32, cudaMemcpyHostToDevice, st));
  }
  PB_CUDA(cudaMemsetAsync(zp, 0, 6 * stride * 32, st));
  PB_TRY(ntt_run((const uint64_t*)wv, n, (uint64_t*)wp, log_n, 1, 0, n_pi ? 5 : 4, n, stride, st, ar));
  {
    BlindArgs ba;
    ba.nb = 2;
    ba.npoly = 4;
    for (int p = 0; p < 4; p++)
      for (int i = 0; i < 2; i++) ba.b[p][i] = to_dev(BL[2 * p + i]);
    PB_LAUNCH(k_blind, 1, 32, 0, st, wp, stride, n, ba);
  }
  if (P->srs_lag) {
    // the same four group elements from the wire VALUES: sum_i w_i [L_i(x)]G + b_0 ([x^n]G - [1]G) +
    // b_1 ([x^(n+1)]G - [x]G); w8 is free until round 3 and stages the scalars
    uint4* sc = w8;
    PB_CUDA(cudaMemcpy2DAsync(sc, stride * 32, wv, n * 32, n * 32, 4, cudaMemcpyDeviceToDevice, st));
    BlindArgs ba;
    ba.nb = 2;
    ba.npoly = 4;
    for (int p = 0; p < 4; p++)
      for (int i = 0; i < 2; i++) ba.b[p][i] = to_dev(BL[2 * p + i]);
    PB_LAUNCH(k_lagrange_tail, 1, 32, 0, st, sc, stride, n, ba);
    // sparse scalars: long buckets keep their lanes, only the heavy chunks widen when busy
    PB_TRY(msm_run(P->srs_lag, 0, (const uint64_t*)sc, n + 4, 4, stride, MsmShape{true, busy()}, aff, st, ar));
  } else {
    PB_TRY(msm_run(P->srs, 0, (const uint64_t*)wp, n + 2, 4, stride, dense_shape(), aff, st, ar));
  }
  for (int k = 0; k < 4; k++) compress_affine(aff + 12 * k, c48[C_A + k]);

  // ---- round 2 -------------------------------------------------------------------------------
  pbh::challenge_beta_gamma(tr, c48[0], ch);
  const HFr beta = ch.beta, gamma = ch.gamma;
  PB_LAUNCH(k_perm_terms, div_up(n, 128), 128, 0, st, (const uint4*)wv, (const uint4*)P->d_sigma, w_half, n, to_dev(beta), to_dev(gamma), num, den);
  PB_LAUNCH(k_batch_div, div_up(div_up(n, 8), 128), 128, 0, st, (const uint4*)num, (const uint4*)den, n, num);
  PB_TRY((fr_scan<true, false>(num, n, den, st, ar)));  // den <- permutation vector z[i] = prod_{j<i} num_j/den_j
  PB_TRY(ntt_run((const uint64_t*)den, n, (uint64_t*)zp, log_n, 1, 0, 1, n, stride, st, ar));
  {
    BlindArgs ba;
    ba.nb = 3;
    ba.npoly = 1;
    for (int i = 0; i < 3; i++) ba.b[0][i] = to_dev(BL[8 + i]);
    PB_LAUNCH(k_blind, 1, 32, 0, st, zp, stride, n, ba);
  }
  PB_TRY(msm_run(P->srs, 0, (const uint64_t*)zp, n + 3, 1, stride, dense_shape(), aff, st, ar));
  compress_affine(aff, c48[C_Z]);

  // ---- round 3 -------------------------------------------------------------------------------
  pbh::challenge_alpha(tr, c48[0], ch);
  const HFr alpha = ch.alpha;
  // t(X) has at most 4n + 7 coefficients, so the six coset transforms, the pointwise pass and the
  // inverse transform run on the 4n coset (the even points of the 8n one) and the top seven coefficients
  // are recovered from eight further points; the algebra is validated against the oracle in
  // tests/models/quotient_4n_model.py.  PB200_QUOT4N=0 restores the reference's 8n schedule
  // (quotient_poly.rs:50-137), which the parity suite keeps running as well.
  static const bool quot4n_env = [] {
    const char* e = getenv("PB200_QUOT4N");
    return !e || atoi(e) != 0;
  }();
  const bool quot4n = quot4n_env && n >= 16;  // the small arrays of step 2 live in the upper half of w8
  const size_t n4 = 4 * n;
  size_t t_len = n8;  // coefficients of t(X) present in tcoef
  QuotArgs q;
  {
    q.w8 = w8; q.key8 = P->d_key8; q.linear8 = P->d_linear8; q.l1_8 = P->d_l1_8; q.out = quot; q.n8 = n8;
    q.alpha = to_dev(alpha); q.beta = to_dev(beta); q.gamma = to_dev(gamma); q.alpha_sq = to_dev(alpha.sqr());
    auto powers = [](const HFr& c) {
      const SepPowers<HFr> h = sep_powers(c);
      SepPowers<Fr> s;
      s.ch = to_dev(h.ch); s.k = to_dev(h.k); s.k2 = to_dev(h.k2); s.k3 = to_dev(h.k3); s.k4 = to_dev(h.k4);
      return s;
    };
    q.ch_range = powers(ch.range); q.ch_logic = powers(ch.logic); q.ch_fixed = powers(ch.fixed); q.ch_var = powers(ch.var);
    q.edwards_d = P->edwards_d;
    for (int i = 0; i < 8; i++) q.vh_inv[i] = to_dev(P->vh_inv[i]);
    q.has_range = P->has_widget[0]; q.has_logic = P->has_widget[1]; q.has_fixed = P->has_widget[2]; q.has_var = P->has_widget[3];
  }
  unsigned char* stage = (unsigned char*)pinned_scratch(1024, 1);
  if (!stage) return fail(PB200_ERR_CUDA, "pinned staging buffer");
  volatile unsigned& h_flag = *(volatile unsigned*)(stage + 512);
  if (!quot4n) {
    // coset evaluations of z, a, b, c, d and the public-input polynomial in one batch
    // (quotient_poly.rs:50-59, 177)
    PB_TRY(ntt_run((const uint64_t*)zp, n + 3, (uint64_t*)w8, log_n + 3, 0, 1, n_pi ? 6 : 5, stride, n8, st, ar));
    if (!n_pi) PB_CUDA(cudaMemsetAsync(w8 + 2 * 5 * n8, 0, n8 * 32, st));  // empty PI polynomial: 8n zeros
    PB_LAUNCH(k_quotient, div_up(n8, 128), 128, 0, st, q);
    PB_TRY(ntt_run((const uint64_t*)quot, n8, (uint64_t*)tcoef, log_n + 3, 1, 1, 1, n8, n8, st, ar));
    // quotient_poly.len() > 7n  =>  CircuitUnsatisfied (quotient_poly.rs:132-134); coefficients past
    // 4n+7 cannot be committed with this key either
    PB_CUDA(cudaMemsetAsync(flag, 0, 4, st));
    PB_LAUNCH(k_any_nonzero, div_up(n8 - 7 * n, 256), 256, 0, st, (const uint4*)tcoef, 7 * n, n8, flag);
    PB_CUDA(cudaMemcpyAsync(stage + 512, flag, 4, cudaMemcpyDeviceToHost, st));
  } else {
    // 1. u(X) = t(X) mod (X^4n - g^4n) from the 4n coset
    PB_TRY(ntt_run((const uint64_t*)zp, n + 3, (uint64_t*)w8, log_n + 2, 0, 1, n_pi ? 6 : 5, stride, n4, st, ar));
    if (!n_pi) PB_CUDA(cudaMemsetAsync(w8 + 2 * 5 * n4, 0, n4 * 32, st));
    static const int quot_occ = [] {
      const char* e = getenv("PB200_QUOT_OCC");
      return e ? atoi(e) : 3;
    }();
    if (quot_occ == 3)
      PB_LAUNCH(k_quotient_4n<3>, div_up(n4, 128), 128, 0, st, q);
    else
      PB_LAUNCH(k_quotient_4n<2>, div_up(n4, 128), 128, 0, st, q);
    PB_TRY(ntt_run((const uint64_t*)quot, n4, (uint64_t*)tcoef, log_n + 2, 1, 1, 1, n4, n4, st, ar));
    // 2. t at the eight points x_k = h w8^k, h = g w_8n (indices 1 + n k of the 8n coset): the witness
    //    polynomials on the cosets h H_8 and omega h H_8 and u = tcoef on h H_8 (one fold per polynomial and
    //    coset, k_coset8_eval), the prover key from its 8n tables.  The upper half of w8 is free in this mode and
    //    holds the small arrays.
    uint4* wpts = w8 + 2 * 6 * n4;   // [6][16]
    uint4* tx = wpts + 2 * 96;       // t(x_k)
    uint4* ux = tx + 2 * 8;          // u(x_k)
    uint4* part4 = ux + 2 * 8;       // [jobs][blocks][8] residue sums of the folds
    const Quot4nConsts& qc = P->q4;
    const int rows = n_pi ? 6 : 5;
    {
      Coset8Jobs cj;
      cj.rows = zp; cj.row_stride = stride; cj.row_len = (unsigned)n + 3; cj.nrows = rows;
      cj.row_blocks = (unsigned)std::max<size_t>(1, div_up(n + 3, 8) / kC8Block);
      cj.tail = tcoef; cj.tail_len = (unsigned)n4;
      cj.tail_blocks = (unsigned)std::max<size_t>(1, (n4 / 8) / kC8Block);
      PB_LAUNCH(k_coset8_eval, 2 * rows * cj.row_blocks + cj.tail_blocks, 256, 0, st, cj, qc.c8, part4);
      PB_LAUNCH(k_coset8_sum, 2 * rows + 1, 256, 0, st, cj, qc.c8, (const uint4*)part4, wpts, ux);
    }
    if (!n_pi) PB_CUDA(cudaMemsetAsync(wpts + 2 * 16 * 5, 0, 16 * 32, st));
    QuotArgs qp = q;
    qp.w8 = wpts;
    qp.out = tx;
    PB_LAUNCH(k_quotient_pts, 1, 128, 0, st, qp);
    // 3. t_hi(x_k) = (t(x_k) - u(x_k)) / (x_k^4n - g^4n), and x_k^4n = -g^4n for every k; the 8-point
    //    inverse DFT on h*H_8 gives its coefficients, the eighth of which must vanish (N divisible by Z_H:
    //    replaces the reference's len > 7n test, quotient_poly.rs:132-134);  4. t = (u - g^4n t_hi) + X^4n t_hi.
    //    Both on the device (eight threads), so round 3 has no host synchronisation of its own.
    PB_CUDA(cudaMemsetAsync(flag, 0, 4, st));
    PB_LAUNCH(k_quot4n_fix, 1, 32, 0, st, (const uint4*)tx, (const uint4*)ux, tcoef, n4, qc.fix, flag);
    PB_CUDA(cudaMemcpyAsync(stage + 512, flag, 4, cudaMemcpyDeviceToHost, st));
    t_len = n4 + 7;
  }
  PB_LAUNCH(k_split_quotient, dim3(div_up(stride, 256), 4), 256, 0, st, (const uint4*)tcoef, n, t_len, stride, to_dev(BL[11]), to_dev(BL[12]), to_dev(BL[13]), tq);
  const size_t key_len = srs_len(P->srs);
  const size_t tlen = std::min(stride, key_len);
  PB_TRY(msm_run(P->srs, 0, (const uint64_t*)tq, tlen, 4, stride, dense_shape(), aff, st, ar));  // synchronises the stream
  if (h_flag) return fail(PB200_ERR_UNSATISFIED, "CircuitUnsatisfied");
  for (int k = 0; k < 4; k++) compress_affine(aff + 12 * k, c48[C_T_LOW + k]);

  // ---- round 4 -------------------------------------------------------------------------------
  pbh::challenge_z(tr, c48[0], ch);
  const HFr z_ch = ch.z;
  const HFr zw = z_ch * to_host(ntt_group_gen(log_n, false));
  HFr ev[N_EVAL];  // in Proof::to_bytes order
  {
    EvalJobs jobs;
    jobs.njobs = 15;
    auto poly = [&](int k) { return (const uint4*)(P->d_polys + 2 * (size_t)k * n); };
    const uint4* ps[15] = {wp, wp + 2 * stride, wp + 4 * stride, wp + 6 * stride, wp, wp + 2 * stride, wp + 6 * stride,
                           poly(Q_ARITH), poly(Q_C), poly(Q_L), poly(Q_R), poly(S1), poly(S2), poly(S3), zp};
    const unsigned ls[15] = {(unsigned)n + 2, (unsigned)n + 2, (unsigned)n + 2, (unsigned)n + 2, (unsigned)n + 2, (unsigned)n + 2, (unsigned)n + 2,
                             (unsigned)n, (unsigned)n, (unsigned)n, (unsigned)n, (unsigned)n, (unsigned)n, (unsigned)n, (unsigned)n + 3};
    const bool shifted[15] = {0, 0, 0, 0, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1};
    for (int j = 0; j < 15; j++) {
      jobs.poly[j] = ps[j];
      jobs.len[j] = ls[j];
      jobs.point[j] = to_dev(shifted[j] ? zw : z_ch);
    }
    EvalPoints ep;
    for (int j = 0; j < 15; j++) ep.p[j] = jobs.point[j];
    ep.p[15] = Fr::zero();
    PB_LAUNCH(k_poly_eval, dim3(eval_blocks, 15), 256, 0, st, jobs, partial, eval_blocks);
    PB_LAUNCH(k_sum_rows, 15, 32, 0, st, (const uint4*)partial, eval_blocks, ep, 16, evals_d);
    PB_CUDA(cudaMemcpyAsync(stage, evals_d, 15 * 32, cudaMemcpyDeviceToHost, st));
    PB_CUDA(stream_wait(st));
    memcpy(ev, stage, 15 * 32);
  }
  // ---- round 5 -------------------------------------------------------------------------------
  pbh::challenge_v(tr, ev, ch);
  const HFr v = ch.v, v_w = ch.v_w;
  {
    const HFr z_n = z_ch.pow_u64(n);
    // domain of z_poly.degree() - 2 is the proving domain n (permutation/proverkey.rs:156-163)
    const HFr l1_z = (z_n - HFr::one()) * to_host(ntt_size_inv(log_n)) * (z_ch - HFr::one()).inv();
    const LinScalars ls = linearisation_scalars(ev, ch, z_n, l1_z);
    HFr vp[12];
    vp[0] = HFr::one();
    for (int i = 1; i < 12; i++) vp[i] = vp[i - 1] * v;
    HFr sel[N_POLY];
    for (int k = 0; k < N_POLY; k++) sel[k] = ls.sel[k];
    sel[Q_ARITH] = sel[Q_ARITH] + vp[8];
    sel[Q_C] = sel[Q_C] + vp[9];
    sel[Q_L] = sel[Q_L] + vp[10];
    sel[Q_R] = sel[Q_R] + vp[11];
    auto poly = [&](int k) { return (const uint4*)(P->d_polys + 2 * (size_t)k * n); };
    // W_z numerator: r + v a + v^2 b + v^3 c + v^4 d + v^5 s1 + v^6 s2 + v^7 s3 + v^8 q_arith + v^9 q_c + v^10 q_l + v^11 q_r
    LinArgs la;
    int t = 0;
    auto term = [&](const uint4* p, size_t len, const HFr& coef) { la.poly[t] = p; la.len[t] = (unsigned)len; la.coef[t] = to_dev(coef); t++; };
    for (int k = Q_M; k <= Q_VAR; k++) term(poly(k), n, sel[k]);
    term(zp, n + 3, ls.z);
    term(poly(S4), n, sel[S4]);
    for (int j = 0; j < 4; j++) term(tq + 2 * j * stride, stride, ls.t[j]);
    term(wp, n + 2, vp[1]);
    term(wp + 2 * stride, n + 2, vp[2]);
    term(wp + 4 * stride, n + 2, vp[3]);
    term(wp + 6 * stride, n + 2, vp[4]);
    term(poly(S1), n, vp[5]);
    term(poly(S2), n, vp[6]);
    term(poly(S3), n, vp[7]);
    la.nterms = t;
    PB_LAUNCH(k_lincomb, div_up(stride, 128), 128, 0, st, la, stride, agg);
    // W_zw numerator: z + v_w a + v_w^2 b + v_w^3 d
    LinArgs lb;
    t = 0;
    auto term2 = [&](const uint4* p, size_t len, const HFr& coef) { lb.poly[t] = p; lb.len[t] = (unsigned)len; lb.coef[t] = to_dev(coef); t++; };
    term2(zp, n + 3, HFr::one());
    term2(wp, n + 2, v_w);
    term2(wp + 2 * stride, n + 2, v_w.sqr());
    term2(wp + 6 * stride, n + 2, v_w.sqr() * v_w);
    lb.nterms = t;
    PB_LAUNCH(k_lincomb, div_up(stride, 128), 128, 0, st, lb, stride, agg + 2 * stride);
    // ruffini (polynomial.rs:345-367): q_j = z^-(j+1) * sum_{i>j} c_i z^i
    const HFr pts[2] = {z_ch, zw};
    for (int w = 0; w < 2; w++) {
      uint4* c_w = agg + 2 * (size_t)w * stride;
      uint4* pw_w = pw + 2 * (size_t)w * stride;
      uint4* sc_w = scratch + 2 * (size_t)w * stride;
      PB_TRY(fill_powers(pw_w, stride, to_dev(pts[w]), Fr::one(), st));
      PB_LAUNCH(k_mul_pointwise, div_up(stride, 128), 128, 0, st, (const uint4*)c_w, (const uint4*)pw_w, stride, sc_w);
      PB_TRY((fr_scan<false, true>(sc_w, stride, c_w, st, ar)));  // exclusive suffix sums
      const HFr zi = pts[w].inv();
      PB_TRY(fill_powers(pw_w, stride, to_dev(zi), to_dev(zi), st));
      PB_LAUNCH(k_mul_pointwise, div_up(stride, 128), 128, 0, st, (const uint4*)c_w, (const uint4*)pw_w, stride, c_w);
    }
    const size_t wlen = std::min(stride, key_len);
    PB_TRY(msm_run(P->srs, 0, (const uint64_t*)agg, wlen, 2, stride, dense_shape(), aff, st, ar));
    compress_affine(aff, c48[C_W_Z]);
    compress_affine(aff + 12, c48[C_W_ZW]);
  }
  // Proof::to_bytes (proof.rs:137-162, linearization_poly.rs:98-124)
  memcpy(out_proof, c48, sizeof c48);
  for (int i = 0; i < N_EVAL; i++) {
    HFr cnon = ev[i].from_mont();
    memcpy(out_proof + kProofEvalAt + 32 * i, cnon.v, 32);
  }
  return 0;
}

// The debugger's check (debugger.cu) of a circuit whose selector values sel ([11][n]) are on the device: the wire values
// are gathered from d_wit (the table d_wires indexes) and the dense public-input vector is built as prove_dev builds it.
static int unsatisfied_columns(const uint4* sel, const uint4* d_wit, const uint32_t* d_wires, size_t constraints, size_t n,
                               const uint64_t* pi_idx, const uint64_t* pi_vals, size_t n_pi, size_t cap, uint64_t* rows,
                               int32_t* families, size_t* n_unsatisfied, cudaStream_t st) {
  ScratchScope scope(nullptr, st);
  uint4* wv = nullptr;
  PB_ALLOC(scope, wv, (n_pi ? 5 : 4) * n * 32);
  PB_LAUNCH(k_gather_wires, dim3(div_up(n, 256), 4), 256, 0, st, d_wit, d_wires, constraints, n, wv);
  uint4* pi_dense = nullptr;
  if (n_pi) {
    pi_dense = wv + 2 * 4 * n;
    PB_CUDA(cudaMemsetAsync(pi_dense, 0, n * 32, st));
    for (size_t i = 0; i < n_pi; i++)
      PB_CUDA(cudaMemcpyAsync(pi_dense + 2 * pi_idx[i], pi_vals + 4 * i, 32, cudaMemcpyHostToDevice, st));
  }
  return unsatisfied_run(sel, wv, pi_dense, n, constraints, cap, rows, families, n_unsatisfied, st);
}

}  // namespace pb

using namespace pb;

extern "C" {

int pb200_prover_new(const uint8_t* label, size_t label_len, size_t n_constraints, const uint64_t* selectors,
                     const uint32_t* wires, size_t n_witnesses, const uint8_t* srs_raw, size_t n_srs_points,
                     pb200_prover_t** out) {
  PB_TRY(ensure_init());
  if (!selectors || !wires || !srs_raw || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return prover_new(nullptr, label, label_len, n_constraints, selectors, wires, n_witnesses, srs_raw, n_srs_points, out);
}

int pb200_prover_new_pp(const pb200_pp_t* pp, const uint8_t* label, size_t label_len, size_t n_constraints, const uint64_t* selectors,
                        const uint32_t* wires, size_t n_witnesses, pb200_prover_t** out) {
  PB_TRY(ensure_init());
  if (!pp || !selectors || !wires || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return prover_new(pp, label, label_len, n_constraints, selectors, wires, n_witnesses, nullptr, pp_points(pp), out);
}

int pb200_prover_from_compressed(const uint8_t* label, size_t label_len, const uint8_t* bytes, size_t len,
                                 const uint8_t* srs_raw, size_t n_srs_points, pb200_prover_t** out) {
  if ((!label && label_len) || !bytes || !srs_raw || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  PB_TRY(ensure_init());
  return prover_from_compressed(nullptr, label, label_len, bytes, len, srs_raw, n_srs_points, out);
}

int pb200_prover_from_compressed_pp(const pb200_pp_t* pp, const uint8_t* label, size_t label_len, const uint8_t* bytes, size_t len,
                                    pb200_prover_t** out) {
  if (!pp || (!label && label_len) || !bytes || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  PB_TRY(ensure_init());
  return prover_from_compressed(pp, label, label_len, bytes, len, nullptr, pp_points(pp), out);
}

int pb200_throughput_mode(int on) {
  g_force_throughput.store(on ? 1 : 0, std::memory_order_relaxed);
  return 0;
}

int pb200_prover_from_bytes(const uint8_t* bytes, size_t len, const uint32_t* wires, size_t n_witnesses, pb200_prover_t** out) {
  PB_TRY(ensure_init());
  if (!bytes || !wires || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return prover_from_bytes(nullptr, bytes, len, wires, n_witnesses, out);
}

int pb200_prover_from_bytes_pp(const pb200_pp_t* pp, const uint8_t* bytes, size_t len, const uint32_t* wires, size_t n_witnesses,
                               pb200_prover_t** out) {
  PB_TRY(ensure_init());
  if (!pp || !bytes || !wires || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  return prover_from_bytes(pp, bytes, len, wires, n_witnesses, out);
}

int pb200_prover_to_bytes(const pb200_prover_t* p, uint8_t* out, size_t cap, size_t* len) {
  if (!p || !len) return fail(PB200_ERR_INVALID_ARG, "null argument");
  PB_TRY(ensure_init());
  return prover_to_bytes(p, out, cap, len);
}

void pb200_prover_free(pb200_prover_t* p) {
  if (!p) return;
  ensure_init();  // a thread that has made no other pb200 call yet must free on the library's device
  prover_free(p);
}

int pb200_prover_commitments(const pb200_prover_t* p, uint8_t* out /* 15 x 48 */) {
  if (!p || !out) return fail(PB200_ERR_INVALID_ARG, "null argument");
  memcpy(out, p->comm, sizeof p->comm);
  return 0;
}

// Prover::prove_with_version (prover.rs:364-413) before any work: V1 is UnsupportedProvingVersion.
static int check_proving_version(int version) {
  if (version == PB200_PLONK_V1) return fail(PB200_ERR_UNSUPPORTED_VERSION, "UnsupportedProvingVersion: PlonkVersion::V1 proofs cannot be made");
  if (version != PB200_PLONK_V2 && version != PB200_PLONK_V3) return fail(PB200_ERR_INVALID_ARG, "unknown PlonkVersion");
  return 0;
}

int pb200_prove(const pb200_prover_t* p, const uint64_t* witnesses, size_t n_witnesses, const uint64_t* pi_idx,
                const uint64_t* pi_vals, size_t n_pi, const uint64_t* blinders, uint8_t* out_proof) {
  return pb200_prove_with_version(p, PB200_PLONK_V3, witnesses, n_witnesses, pi_idx, pi_vals, n_pi, blinders, out_proof);
}

int pb200_prove_with_version(const pb200_prover_t* p, int version, const uint64_t* witnesses, size_t n_witnesses,
                             const uint64_t* pi_idx, const uint64_t* pi_vals, size_t n_pi, const uint64_t* blinders,
                             uint8_t* out_proof) {
  PB_TRY(check_proving_version(version));
  PB_TRY(ensure_init());
  if (!p || !witnesses || !blinders || !out_proof) return fail(PB200_ERR_INVALID_ARG, "null argument");
  if (n_witnesses != p->n_witnesses) return fail(PB200_ERR_INVALID_ARG, "witness count differs from the compiled circuit");
  cudaStream_t st = thread_stream();
  uint64_t* d_wit = nullptr;
  PB_CUDA(cudaMallocAsync((void**)&d_wit, n_witnesses * 32, st));
  int rc;
  const cudaError_t e = cudaMemcpyAsync(d_wit, witnesses, n_witnesses * 32, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess)
    rc = fail(PB200_ERR_CUDA, "witness upload", cudaGetErrorString(e));
  else
    rc = prove_dev(p, version, d_wit, pi_idx, pi_vals, n_pi, blinders, out_proof, st);
  cudaFreeAsync(d_wit, st);
  return rc;
}

int pb200_prove_dev(const pb200_prover_t* p, const uint64_t* d_witnesses, size_t n_witnesses, const uint64_t* pi_idx,
                    const uint64_t* pi_vals, size_t n_pi, const uint64_t* blinders, uint8_t* out_proof, void* stream) {
  return pb200_prove_dev_with_version(p, PB200_PLONK_V3, d_witnesses, n_witnesses, pi_idx, pi_vals, n_pi, blinders, out_proof, stream);
}

int pb200_prove_dev_with_version(const pb200_prover_t* p, int version, const uint64_t* d_witnesses, size_t n_witnesses,
                                 const uint64_t* pi_idx, const uint64_t* pi_vals, size_t n_pi, const uint64_t* blinders,
                                 uint8_t* out_proof, void* stream) {
  PB_TRY(check_proving_version(version));
  PB_TRY(ensure_init());
  if (!p || !d_witnesses || !blinders || !out_proof) return fail(PB200_ERR_INVALID_ARG, "null argument");
  if (n_witnesses != p->n_witnesses) return fail(PB200_ERR_INVALID_ARG, "witness count differs from the compiled circuit");
  cudaStream_t st = stream ? (cudaStream_t)stream : thread_stream();
  return prove_dev(p, version, d_witnesses, pi_idx, pi_vals, n_pi, blinders, out_proof, st);
}

int pb200_circuit_unsatisfied(size_t n_constraints, const uint64_t* selectors, const uint32_t* wires, const uint64_t* witnesses,
                              size_t n_witnesses, const uint64_t* pi_idx, const uint64_t* pi_vals, size_t n_pi, size_t cap,
                              uint64_t* rows, int32_t* families, size_t* n_unsatisfied) {
  if (!n_unsatisfied || (cap && (!rows || !families))) return fail(PB200_ERR_INVALID_ARG, "null argument");
  PB_TRY(check_public_inputs(pi_idx, pi_vals, n_pi, n_constraints));
  *n_unsatisfied = 0;
  if (n_constraints == 0) return 0;  // the reference's debugger with no constraints reports nothing
  if (!selectors || !wires || (n_witnesses && !witnesses)) return fail(PB200_ERR_INVALID_ARG, "null argument");
  for (size_t j = 0; j < 4 * n_constraints; j++)
    if (wires[j] >= n_witnesses) return fail(PB200_ERR_INVALID_ARG, "wire index out of range");
  PB_TRY(ensure_init());
  size_t n = 1;
  while (n < n_constraints) n <<= 1;
  cudaStream_t st = thread_stream();
  ScratchScope scope(nullptr, st);
  uint4 *sel = nullptr, *d_wit = nullptr;
  uint32_t* d_wires = nullptr;
  PB_ALLOC(scope, sel, (size_t)11 * n * 32);
  PB_ALLOC(scope, d_wit, n_witnesses * 32);
  PB_ALLOC(scope, d_wires, 4 * n_constraints * 4);
  // only the rows below the constraint count are read, so the columns' padding is left as it is
  PB_CUDA(cudaMemcpy2DAsync(sel, n * 32, selectors, n_constraints * 32, n_constraints * 32, 11, cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(d_wit, witnesses, n_witnesses * 32, cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(d_wires, wires, 4 * n_constraints * 4, cudaMemcpyHostToDevice, st));
  return unsatisfied_columns(sel, d_wit, d_wires, n_constraints, n, pi_idx, pi_vals, n_pi, cap, rows, families, n_unsatisfied, st);
}

int pb200_prover_unsatisfied(const pb200_prover_t* p, const uint64_t* witnesses, size_t n_witnesses, const uint64_t* pi_idx,
                             const uint64_t* pi_vals, size_t n_pi, size_t cap, uint64_t* rows, int32_t* families,
                             size_t* n_unsatisfied) {
  if (!p || !witnesses || !n_unsatisfied || (cap && (!rows || !families))) return fail(PB200_ERR_INVALID_ARG, "null argument");
  if (n_witnesses != p->n_witnesses) return fail(PB200_ERR_INVALID_ARG, "witness count differs from the compiled circuit");
  PB_TRY(check_public_inputs(pi_idx, pi_vals, n_pi, p->constraints));
  PB_TRY(ensure_init());
  const size_t n = p->n;
  cudaStream_t st = thread_stream();
  ScratchScope scope(nullptr, st);
  uint4 *sel = nullptr, *d_wit = nullptr;
  PB_ALLOC(scope, sel, (size_t)11 * n * 32);
  PB_ALLOC(scope, d_wit, n_witnesses * 32);
  // the selector values on the domain: one forward NTT of the key's 11 selector polynomials
  PB_TRY(ntt_run((const uint64_t*)p->d_polys, n, (uint64_t*)sel, p->log_n, 0, 0, 11, n, n, st, nullptr));
  PB_CUDA(cudaMemcpyAsync(d_wit, witnesses, n_witnesses * 32, cudaMemcpyHostToDevice, st));
  if (p->d_labels) {  // a compressed circuit's prover: its wires index the dense table of the labels they use
    uint4* dense = nullptr;
    PB_ALLOC(scope, dense, p->n_labels * 32);
    PB_LAUNCH(k_gather_witnesses, div_up(p->n_labels, 256), 256, 0, st, (const uint4*)d_wit, (const unsigned long long*)p->d_labels,
              p->n_labels, dense);
    d_wit = dense;
  }
  return unsatisfied_columns(sel, d_wit, p->d_wires, p->constraints, n, pi_idx, pi_vals, n_pi, cap, rows, families, n_unsatisfied, st);
}
}
