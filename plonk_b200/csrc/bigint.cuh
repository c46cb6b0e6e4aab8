// Multi-limb (32-bit) Montgomery arithmetic for sm_90a (H100), generic over the limb count.
//
// The GPU arithmetic underneath the two hot kernels of the dusk-plonk prover: BlsScalar (Fr, 8 limbs)
// for EvaluationDomain::{fft,ifft,coset_fft,coset_ifft} (reference src/fft/domain.rs:166-232) and
// Fp (12 limbs) for the G1 MSM behind CommitKey::commit (reference
// src/commitment_scheme/kzg10/key.rs:376-388).  The reference keeps both in dusk-bls12_381 as
// 4x/6x u64 Montgomery limbs; the in-memory little-endian layout is identical, we just address it
// as 32-bit limbs because the Hopper integer pipe is IMAD (32x32+64).
//
// Every carry chain is written with PTX add.cc/addc/mad.lo.cc/madc.hi.cc so ptxas can fuse
// lo/hi pairs into IMAD.WIDE.U32 with predicate carries.  When compiled for the host (g++, used
// only by tests/hosttest to validate the algorithms without a GPU) the same primitives are
// emulated with an explicit carry flag.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define PB_HD __host__ __device__ __forceinline__
#define PB_D __device__ __forceinline__
#else
#define PB_HD inline
#define PB_D inline
#endif

#ifndef PB_SPLIT
#define PB_SPLIT 0
#endif

namespace pb {

#if defined(__CUDA_ARCH__)
#define PB_ASM2(name, ins)                                                         \
  PB_D uint32_t name(uint32_t a, uint32_t b) {                                     \
    uint32_t r;                                                                    \
    asm volatile(ins " %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));                   \
    return r;                                                                      \
  }
#define PB_ASM3(name, ins)                                                         \
  PB_D uint32_t name(uint32_t a, uint32_t b, uint32_t c) {                         \
    uint32_t r;                                                                    \
    asm volatile(ins " %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));       \
    return r;                                                                      \
  }
PB_ASM2(add_cc, "add.cc.u32")
PB_ASM2(addc_cc, "addc.cc.u32")
PB_ASM2(addc, "addc.u32")
PB_ASM2(sub_cc, "sub.cc.u32")
PB_ASM2(subc_cc, "subc.cc.u32")
PB_ASM2(subc, "subc.u32")
PB_ASM2(mul_lo, "mul.lo.u32")
PB_ASM2(mul_hi, "mul.hi.u32")
PB_ASM3(mad_lo_cc, "mad.lo.cc.u32")
PB_ASM3(madc_lo_cc, "madc.lo.cc.u32")
PB_ASM3(mad_hi_cc, "mad.hi.cc.u32")
PB_ASM3(madc_hi_cc, "madc.hi.cc.u32")
PB_ASM3(madc_hi, "madc.hi.u32")
PB_ASM3(madc_lo, "madc.lo.u32")
#undef PB_ASM2
#undef PB_ASM3
// (lo,hi) pair forms: both halves of one 32x32 product in a single asm block, which is the shape
// ptxas fuses into one IMAD.WIDE.U32[.X] with predicate carry-in/out.
//   CIN: consume the carry flag; COUT: leave the carry flag set for the next pair.
template <bool CIN, bool COUT>
PB_D void mad_pair(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
  if (CIN && COUT)
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
  else if (CIN && !COUT)
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.u32 %1, %2, %3, %5;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
  else if (!CIN && COUT)
    asm volatile("mad.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
  else
    asm volatile("mad.lo.cc.u32 %0, %2, %3, %4; madc.hi.u32 %1, %2, %3, %5;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
}
PB_D void mul_pair(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {
  asm volatile("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
// Same contract as mad_pair, but the 64-bit product is formed by a carry-free IMAD.WIDE and added
// with two carry-chained IADD3 on the ALU pipe.  IMAD.WIDE.U32.X (carry in/out) issues at half the
// rate of the carry-free form (tools/mulbench), so moving part of the links of a chain to this
// shape balances the multiply pipe against the otherwise idle ALU pipe.
template <bool CIN, bool COUT>
PB_D void mad_pair_split(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
  uint32_t tl, th;
  asm volatile("{ .reg .u64 t; mul.wide.u32 t, %2, %3; mov.b64 {%0, %1}, t; }" : "=r"(tl), "=r"(th) : "r"(a), "r"(b));
  if (CIN && COUT)
    asm volatile("addc.cc.u32 %0, %2, %3; addc.cc.u32 %1, %4, %5;" : "=r"(lo), "=r"(hi) : "r"(clo), "r"(tl), "r"(chi), "r"(th));
  else if (CIN && !COUT)
    asm volatile("addc.cc.u32 %0, %2, %3; addc.u32 %1, %4, %5;" : "=r"(lo), "=r"(hi) : "r"(clo), "r"(tl), "r"(chi), "r"(th));
  else if (!CIN && COUT)
    asm volatile("add.cc.u32 %0, %2, %3; addc.cc.u32 %1, %4, %5;" : "=r"(lo), "=r"(hi) : "r"(clo), "r"(tl), "r"(chi), "r"(th));
  else
    asm volatile("add.cc.u32 %0, %2, %3; addc.u32 %1, %4, %5;" : "=r"(lo), "=r"(hi) : "r"(clo), "r"(tl), "r"(chi), "r"(th));
}
#else
// Host emulation of the PTX condition-code register (one flag, as in PTX).
static thread_local uint32_t pb_cf = 0;
inline uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t s = (uint64_t)a + b; pb_cf = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { uint64_t s = (uint64_t)a + b + pb_cf; pb_cf = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t addc(uint32_t a, uint32_t b) { return a + b + pb_cf; }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t s = (uint64_t)a - b; pb_cf = (uint32_t)(s >> 63); return (uint32_t)s; }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { uint64_t s = (uint64_t)a - b - pb_cf; pb_cf = (uint32_t)(s >> 63); return (uint32_t)s; }
inline uint32_t subc(uint32_t a, uint32_t b) { return a - b - pb_cf; }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
inline uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return add_cc(a * b, c); }
inline uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return addc_cc(a * b, c); }
inline uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) { return add_cc(mul_hi(a, b), c); }
inline uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { return addc_cc(mul_hi(a, b), c); }
inline uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return addc(mul_hi(a, b), c); }
inline uint32_t madc_lo(uint32_t a, uint32_t b, uint32_t c) { return addc(a * b, c); }
template <bool CIN, bool COUT>
inline void mad_pair(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
  uint32_t l = CIN ? madc_lo_cc(a, b, clo) : mad_lo_cc(a, b, clo);
  uint32_t h = COUT ? madc_hi_cc(a, b, chi) : madc_hi(a, b, chi);
  lo = l;
  hi = h;
}
inline void mul_pair(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { lo = mul_lo(a, b); hi = mul_hi(a, b); }
template <bool CIN, bool COUT>
inline void mad_pair_split(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
  mad_pair<CIN, COUT>(lo, hi, a, b, clo, chi);
}
#endif

// ---------------------------------------------------------------------------------------------
// Double-precision helpers for the two-pipe ("hybrid") Montgomery product, see Field::redc48.
// Host builds emulate fma_rz with fma() under fesetround(FE_TOWARDZERO) (tools/mulbench's check).
// ---------------------------------------------------------------------------------------------
#ifndef PB_FP_HYBRID
#define PB_FP_HYBRID 0
#endif
#ifndef PB_FR_HYBRID
#define PB_FR_HYBRID 0
#endif
}  // namespace pb
#if !defined(__CUDA_ARCH__)
#include <math.h>
#include <string.h>
#endif
namespace pb {
PB_HD double fma_rz(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
  return __fma_rz(a, b, c);
#else
  return fma(a, b, c);  // the caller has set FE_TOWARDZERO
#endif
}
PB_HD uint64_t dbl_bits(double x) {
#if defined(__CUDA_ARCH__)
  return (uint64_t)__double_as_longlong(x);
#else
  uint64_t r;
  memcpy(&r, &x, 8);
  return r;
#endif
}
PB_HD double bits_dbl(uint32_t hi, uint32_t lo) {
#if defined(__CUDA_ARCH__)
  return __hiloint2double((int)hi, (int)lo);
#else
  const uint64_t r = ((uint64_t)hi << 32) | lo;
  double x;
  memcpy(&x, &r, 8);
  return x;
#endif
}

// ---------------------------------------------------------------------------------------------
// Field<P>: P supplies N (even), MOD(i), inv() (= -MOD^-1 mod 2^32), R1 (=2^(32N) mod p), R2.
// Values are always kept fully reduced in [0, p), Montgomery form unless stated otherwise.
// ---------------------------------------------------------------------------------------------
template <class P>
struct Field {
  static constexpr int N = P::N;
  uint32_t v[N];

  static PB_HD Field zero() {
    Field r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = 0;
    return r;
  }
  static PB_HD Field one() {  // Montgomery form of 1
    Field r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = P::R1(i);
    return r;
  }
  static PB_HD Field r2() {
    Field r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = P::R2(i);
    return r;
  }
  PB_HD bool is_zero() const {
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < N; i++) x |= v[i];
    return x == 0;
  }
  PB_HD bool operator==(const Field& o) const {
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < N; i++) x |= v[i] ^ o.v[i];
    return x == 0;
  }
  PB_HD bool operator!=(const Field& o) const { return !(*this == o); }

  // r = (t >= p) ? t - p : t, for t < 2p given with an extra top word `hi` (0 or 1).
  static PB_HD void final_sub(uint32_t* r, const uint32_t* t, uint32_t hi) {
    uint32_t s[N];
    s[0] = sub_cc(t[0], P::MOD(0));
#pragma unroll
    for (int i = 1; i < N; i++) s[i] = subc_cc(t[i], P::MOD(i));
    uint32_t borrow = subc(hi, 0u);  // 0 if t >= p, 0xffffffff (or hi-1) otherwise
    bool ge = (borrow == 0u);
#pragma unroll
    for (int i = 0; i < N; i++) r[i] = ge ? s[i] : t[i];
  }
  // The end of a Montgomery product whose pre-subtraction value t is < 2p: reduced to [0, p) when FULL,
  // left as it is for FpR otherwise.
  template <bool FULL>
  static PB_HD Field finish(const uint32_t* t) {
    Field r;
    if (FULL) {
      final_sub(r.v, t, 0u);
    } else {
#pragma unroll
      for (int i = 0; i < N; i++) r.v[i] = t[i];
    }
    return r;
  }

  friend PB_HD Field operator+(const Field& a, const Field& b) {
    uint32_t t[N];
    t[0] = add_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int i = 1; i < N; i++) t[i] = addc_cc(a.v[i], b.v[i]);
    uint32_t hi = addc(0u, 0u);
    Field r;
    final_sub(r.v, t, hi);
    return r;
  }
  friend PB_HD Field operator-(const Field& a, const Field& b) {
    uint32_t t[N];
    t[0] = sub_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int i = 1; i < N; i++) t[i] = subc_cc(a.v[i], b.v[i]);
    uint32_t borrow = subc(0u, 0u);  // 0xffffffff when a < b
    Field r;
    uint32_t m = borrow;  // add p back under mask
    r.v[0] = add_cc(t[0], P::MOD(0) & m);
#pragma unroll
    for (int i = 1; i < N - 1; i++) r.v[i] = addc_cc(t[i], P::MOD(i) & m);
    r.v[N - 1] = addc(t[N - 1], P::MOD(N - 1) & m);
    return r;
  }
  PB_HD Field neg() const { return zero() - *this; }
  PB_HD Field dbl() const { return *this + *this; }

  // Montgomery product a*b*2^(-32N) mod p (CIOS by rows of b).
  //
  // The running sum T is kept as two N-limb accumulators, T = E + O*2^32: products of the even
  // limbs of the multiplicand land in E as (lo,hi) pairs at even indices, products of the odd limbs
  // land in O the same way, so every pair is an aligned register pair and a whole row is two carry
  // chains of mad.lo.cc/madc.hi.cc (IMAD.WIDE.U32 with predicate carry in SASS).  After the
  // Montgomery step E[0] == 0 and T/2^32 = O + (E >> 32): the accumulators swap roles (new E = O,
  // new O = E >> 64) and the one left-over limb E[1] is folded into the next row's carry chain.
  // The first and last links of a chain are written outside the limb loops, so that no loop body branches
  // on its index: the sm_90a compiler does not fully unroll such loops, and a rolled carry chain ends up
  // in local memory.
  template <bool SPLIT, bool CIN, bool COUT>
  static PB_HD void link(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
    if (SPLIT)
      mad_pair_split<CIN, COUT>(lo, hi, a, b, clo, chi);
    else
      mad_pair<CIN, COUT>(lo, hi, a, b, clo, chi);
  }
  // One row of the product: T += a * bi.  On entry X is the old E (its low limb is zero after the
  // previous Montgomery step, so E >> 64 is what remains) and Y the old O; on exit X is the new O and
  // Y the new E.
  static PB_HD void mul_row(uint32_t* X, uint32_t* Y, const uint32_t* a, uint32_t bi) {
    constexpr bool S0 = (PB_SPLIT & 1) != 0, S1 = (PB_SPLIT & 2) != 0;
    Y[0] = add_cc(Y[0], X[1]);
#pragma unroll
    for (int k = 0; k < N - 2; k += 2) link<S0, true, true>(X[k], X[k + 1], a[k + 1], bi, X[k + 2], X[k + 3]);
    link<S0, true, false>(X[N - 2], X[N - 1], a[N - 1], bi, 0u, 0u);
    link<S1, false, true>(Y[0], Y[1], a[0], bi, Y[0], Y[1]);
#pragma unroll
    for (int j = 2; j < N; j += 2) link<S1, true, true>(Y[j], Y[j + 1], a[j], bi, Y[j], Y[j + 1]);
    X[N - 1] = addc(X[N - 1], 0u);
  }
  // A further product in the same row: T += c * di, with X = O and Y = E already in their new roles.
  static PB_HD void acc_row(uint32_t* X, uint32_t* Y, const uint32_t* c, uint32_t di) {
    constexpr bool S0 = (PB_SPLIT & 1) != 0, S1 = (PB_SPLIT & 2) != 0;
    link<S0, false, true>(X[0], X[1], c[1], di, X[0], X[1]);
#pragma unroll
    for (int k = 2; k < N - 2; k += 2) link<S0, true, true>(X[k], X[k + 1], c[k + 1], di, X[k], X[k + 1]);
    link<S0, true, false>(X[N - 2], X[N - 1], c[N - 1], di, X[N - 2], X[N - 1]);
    link<S1, false, true>(Y[0], Y[1], c[0], di, Y[0], Y[1]);
#pragma unroll
    for (int j = 2; j < N; j += 2) link<S1, true, true>(Y[j], Y[j + 1], c[j], di, Y[j], Y[j + 1]);
    X[N - 1] = addc(X[N - 1], 0u);
  }
  // The Montgomery step of a row: T += m * p with m chosen so that the low limb (Y[0]) vanishes.
  static PB_HD void red_row(uint32_t* X /* O */, uint32_t* Y /* E */) {
    constexpr bool S2 = (PB_SPLIT & 4) != 0, S3 = (PB_SPLIT & 8) != 0;
    const uint32_t m = mul_lo(Y[0], P::inv());
    link<S2, false, true>(X[0], X[1], P::MOD(1), m, X[0], X[1]);
#pragma unroll
    for (int k = 2; k < N - 2; k += 2) link<S2, true, true>(X[k], X[k + 1], P::MOD(k + 1), m, X[k], X[k + 1]);
    link<S2, true, false>(X[N - 2], X[N - 1], P::MOD(N - 1), m, X[N - 2], X[N - 1]);
    link<S3, false, true>(Y[0], Y[1], P::MOD(0), m, Y[0], Y[1]);
#pragma unroll
    for (int j = 2; j < N; j += 2) link<S3, true, true>(Y[j], Y[j + 1], P::MOD(j), m, Y[j], Y[j + 1]);
    X[N - 1] = addc(X[N - 1], 0u);
  }
  template <bool FIRST>
  static PB_HD void mont_row(uint32_t* X /* old E -> new O */, uint32_t* Y /* old O -> new E */,
                             const uint32_t* a, uint32_t bi) {
    if (!FIRST) mul_row(X, Y, a, bi);
    red_row(X, Y);
  }

  friend PB_HD Field operator*(const Field& a, const Field& b) { return mul<true>(a, b); }
  // FULL = false skips the final subtraction (FpR: operands < 2p give a result < 2p, see there).
  template <bool FULL>
  static PB_HD Field mul(const Field& a, const Field& b) {
#if defined(__CUDA_ARCH__)
    if constexpr (P::HYBRID) return mul_hybrid<FULL>(a, b);
#endif
    return mul_imad<FULL>(a, b);
  }
  template <bool FULL = true>
  static PB_HD Field mul_imad(const Field& a, const Field& b) {
    uint32_t A[N], B[N];
    {
      const uint32_t bi = b.v[0];
#pragma unroll
      for (int j = 0; j < N; j += 2) {
        mul_pair(A[j], A[j + 1], a.v[j], bi);
        mul_pair(B[j], B[j + 1], a.v[j + 1], bi);
      }
      mont_row<true>(B, A, a.v, bi);  // E = A, O = B
    }
#pragma unroll
    for (int i = 1; i < N - 1; i += 2) {
      mont_row<false>(A, B, a.v, b.v[i]);      // E = B, O = A
      mont_row<false>(B, A, a.v, b.v[i + 1]);  // E = A, O = B
    }
    mont_row<false>(A, B, a.v, b.v[N - 1]);    // E = B, O = A
    // N is even: E = B (B[0] == 0), O = A.  T/2^32 = A + (B >> 32).
    uint32_t t[N];
    t[0] = add_cc(A[0], B[1]);
#pragma unroll
    for (int k = 1; k < N - 1; k++) t[k] = addc_cc(A[k], B[k + 1]);
    t[N - 1] = addc(A[N - 1], 0u);
    return finish<FULL>(t);
  }
  // Squaring with the symmetric partial products taken once: a^2 = sum_i a_i * B_i with
  // B_i = a_i 2^(32i) + 2 sum_{k>i} a_k 2^(32k), so row i multiplies a_i only by the limbs k >= i of
  // the doubled operand (N(N+1)/2 multiply-adds instead of N^2; the Montgomery steps are unchanged).
  // The skipped links of the shifting accumulator become plain carry-propagating adds.
  // Row 0 adds a_0 * 2a at once, twice what a row of the ordinary product adds, so the running sum
  // needs (2a + p) * 2^32 < 2^(32(N+1)): 3p for a < p, 5p for an FpR operand a < 2p.  Both need two
  // spare bits in the top limb (and 2a must fit N limbs).  Fp has three; Fr (one) keeps the ordinary
  // product.
  template <int I>
  static PB_HD uint32_t sq_limb(const uint32_t* a, const uint32_t* a2, int k) {
    return k == I ? a[k] : (k == I + 1 ? (a[k] << 1) : a2[k]);
  }
  template <int I>
  static PB_HD void sqr_row(uint32_t* X, uint32_t* Y, const uint32_t* a, const uint32_t* a2) {
    constexpr bool S0 = (PB_SPLIT & 1) != 0, S1 = (PB_SPLIT & 2) != 0;
    const uint32_t bi = a[I];
    Y[0] = add_cc(Y[0], X[1]);
    constexpr int K0 = I & ~1;  // first even limb k with a product (k + 1 >= I)
#pragma unroll
    for (int k = 0; k < K0; k += 2) {  // no product at this limb: shift and propagate the carry
      X[k] = addc_cc(X[k + 2], 0u);
      X[k + 1] = addc_cc(X[k + 3], 0u);
    }
#pragma unroll
    for (int k = K0; k < N - 2; k += 2) link<S0, true, true>(X[k], X[k + 1], sq_limb<I>(a, a2, k + 1), bi, X[k + 2], X[k + 3]);
    link<S0, true, false>(X[N - 2], X[N - 1], sq_limb<I>(a, a2, N - 1), bi, 0u, 0u);
    constexpr int J0 = (I + 1) & ~1;  // first even limb >= I
    if (J0 < N) {
      link<S1, false, true>(Y[J0], Y[J0 + 1], sq_limb<I>(a, a2, J0), bi, Y[J0], Y[J0 + 1]);
#pragma unroll
      for (int j = J0 + 2; j < N; j += 2) link<S1, true, true>(Y[j], Y[j + 1], sq_limb<I>(a, a2, j), bi, Y[j], Y[j + 1]);
      X[N - 1] = addc(X[N - 1], 0u);
    }
  }
  template <int I>
  static PB_HD void sqr_rows(uint32_t* A, uint32_t* B, const uint32_t* a, const uint32_t* a2) {
    if constexpr (I < N) {
      sqr_row<I>(A, B, a, a2);  // E = B, O = A
      red_row(A, B);
      if constexpr (I + 1 < N) {
        sqr_row<I + 1>(B, A, a, a2);  // E = A, O = B
        red_row(B, A);
      }
      sqr_rows<I + 2>(A, B, a, a2);
    }
  }
  template <bool FULL = true>
  PB_HD Field sqr() const {
#if defined(__CUDA_ARCH__)
    if constexpr (P::HYBRID && (P::MOD(N - 1) >> 30) == 0) return sqr_hybrid<FULL>();
#endif
    if constexpr ((P::MOD(N - 1) >> 30) != 0) {
      return mul<FULL>(*this, *this);
    } else {
      return sqr_half<FULL>();
    }
  }
  template <bool FULL = true>
  PB_HD Field sqr_half() const {
    static_assert((P::MOD(N - 1) >> 30) == 0, "needs two spare bits in the top limb of the modulus");
    uint32_t a2[N];
    a2[0] = v[0] << 1;
#pragma unroll
    for (int k = 1; k < N; k++) a2[k] = (v[k] << 1) | (v[k - 1] >> 31);
    uint32_t A[N], B[N];
    {
      const uint32_t bi = v[0];
#pragma unroll
      for (int j = 0; j < N; j += 2) {
        mul_pair(A[j], A[j + 1], sq_limb<0>(v, a2, j), bi);
        mul_pair(B[j], B[j + 1], sq_limb<0>(v, a2, j + 1), bi);
      }
      red_row(B, A);  // E = A, O = B
    }
    sqr_rows<1>(A, B, v, a2);
    uint32_t t[N];
    t[0] = add_cc(A[0], B[1]);
#pragma unroll
    for (int k = 1; k < N - 1; k++) t[k] = addc_cc(A[k], B[k + 1]);
    t[N - 1] = addc(A[N - 1], 0u);
    return finish<FULL>(t);
  }

  // a*b + c*d with ONE Montgomery reduction: each row accumulates both partial products before its
  // Montgomery step (3N^2 multiply-adds instead of 4N^2).  Only for moduli with at least two spare
  // bits in the top limb (Fp: 381 of 384 bits), where the running sum keeps fitting the two
  // accumulators and the result stays below 2p; Fr (255 of 256 bits) must not use it.
  // The running sum entering a row is < a + c + p, so a row peaks below (a + c + p) * 2^32: 3p for
  // canonical operands, 5p for FpR operands (all four < 2p), inside 2^(32(N+1)) when 8p < 2^(32N).
  // The result is < p + (ab + cd) / 2^(32N) < p + 8p^2 / 2^(32N) < 2p in both cases.
  template <bool FULL = true>
  static PB_HD Field mul2(const Field& a, const Field& b, const Field& c, const Field& d) {
#if defined(__CUDA_ARCH__)
    if constexpr (P::HYBRID) return mul2_hybrid<FULL>(a, b, c, d);
#endif
    return mul2_imad<FULL>(a, b, c, d);
  }
  template <bool FULL = true>
  static PB_HD Field mul2_imad(const Field& a, const Field& b, const Field& c, const Field& d) {
    static_assert((P::MOD(N - 1) >> 30) == 0, "mul2 needs two spare bits in the top limb of the modulus");
    uint32_t A[N], B[N];
    {
      const uint32_t bi = b.v[0];
#pragma unroll
      for (int j = 0; j < N; j += 2) {
        mul_pair(A[j], A[j + 1], a.v[j], bi);
        mul_pair(B[j], B[j + 1], a.v[j + 1], bi);
      }
      acc_row(B, A, c.v, d.v[0]);
      red_row(B, A);  // E = A, O = B
    }
#pragma unroll
    for (int i = 1; i < N - 1; i += 2) {
      mul_row(A, B, a.v, b.v[i]);
      acc_row(A, B, c.v, d.v[i]);
      red_row(A, B);  // E = B, O = A
      mul_row(B, A, a.v, b.v[i + 1]);
      acc_row(B, A, c.v, d.v[i + 1]);
      red_row(B, A);  // E = A, O = B
    }
    mul_row(A, B, a.v, b.v[N - 1]);
    acc_row(A, B, c.v, d.v[N - 1]);
    red_row(A, B);  // E = B, O = A
    uint32_t t[N];
    t[0] = add_cc(A[0], B[1]);
#pragma unroll
    for (int k = 1; k < N - 1; k++) t[k] = addc_cc(A[k], B[k + 1]);
    t[N - 1] = addc(A[N - 1], 0u);
    return finish<FULL>(t);
  }
  // -------------------------------------------------------------------------------------------
  // Two-pipe ("hybrid") product (Fp: 384 bits = 8 x 48; Fr: 256 bits = 5 x 48 + 16).
  //
  // IMAD.WIDE.U32.X (carry in/out) issues at half the rate of the carry-free form, and the FP64
  // pipe of the H100 idles next to it.  So the 2N-limb product a*b stays on the integer multiply
  // pipe (the same rows as above without their Montgomery steps), and the Montgomery reduction - half
  // of the multiply-adds - moves to DFMA on 48-bit limbs: m * p_j is split exactly into two 48-bit
  // halves by
  //     hi = fma_rz(m, p_j, 2^100)                bits(hi) = bits(2^100) + floor(m p_j / 2^48)
  //     lo = fma_rz(m, p_j, (2^100 + 2^52) - hi)  bits(lo) = bits(2^52)  + (m p_j mod 2^48)
  // and the raw bit patterns are summed into 64-bit integer columns by IADD3 on the ALU pipe.  Both
  // pattern offsets are multiples of 2^48: the low 48 bits of a column are right at all times and
  // the offsets are only taken out where a carry leaves a column.  R stays 2^(32N), so the values
  // are the same Montgomery residues as everywhere else: when 48 does not divide 32N the last step
  // clears only the remaining 32N mod 48 bits and the result is read from the middle of a column.
  // m * p_j < 2^96 and a column sums at most 17 terms below 2^48 plus a carry, far inside 64 bits.
  // -------------------------------------------------------------------------------------------
  static constexpr int L48 = (32 * N + 47) / 48;       // 48-bit limbs of the modulus (Fp 8, Fr 6)
  static constexpr int CUT_COL = (32 * N) / 48;        // the column that holds bit 32N ...
  static constexpr int CUT_SH = (32 * N) % 48;         // ... at this bit (Fp: 8, 0; Fr: 5, 16)
  static constexpr int LAST_BITS = 32 * N - 48 * (L48 - 1);  // width of the last reduction step (Fp 48, Fr 16)
  static PB_HD constexpr int npairs48(int k) { return k < 0 ? 0 : (k < L48 ? k + 1 : (k <= 2 * L48 - 2 ? 2 * L48 - 1 - k : 0)); }
  // what the L48^2 dual products have put into column k by the time it is read (mod 2^64)
  static PB_HD constexpr uint64_t col_off48(int k) {
    return (uint64_t)npairs48(k) * 0x4330000000000000ull + (uint64_t)npairs48(k - 1) * 0x4630000000000000ull;
  }
  static PB_HD uint32_t word_or_zero(const uint32_t* T, int k) { return k < 2 * N ? T[k] : 0u; }
  // T[2N] * 2^(-32N) mod p for T < p * 2^(32N): fully reduced when FULL, else < 2p (FpR).
  template <bool FULL>
  static PB_HD Field redc48(const uint32_t* T) {
    uint64_t c[2 * L48];
    // T[2N-1] has at least two spare bits, so `gate` is zero - but ptxas cannot know, which keeps it
    // from starting the reduction (whose 64-bit adds want carry predicates) inside the carry chains
    // of the product that made T; interleaved, the two spill predicates to registers.
    const uint32_t gate = T[2 * N - 1] >> 30;
#pragma unroll
    for (int q = 0; q < L48; q++) {  // three 32-bit words -> two 48-bit limbs (zero beyond T)
      const uint32_t w0 = word_or_zero(T, 3 * q) | (q == 0 ? gate : 0u), w1 = word_or_zero(T, 3 * q + 1),
                     w2 = word_or_zero(T, 3 * q + 2);
      c[2 * q] = (uint64_t)w0 | ((uint64_t)(w1 & 0xffffu) << 32);
      c[2 * q + 1] = (uint64_t)((w1 >> 16) | (w2 << 16)) | ((uint64_t)(w2 >> 16) << 32);
    }
    const double C1 = 0x1p100, C2 = 0x1p100 + 0x1p52;
#pragma unroll
    for (int i = 0; i < L48; i++) {
      // m = c[i] * (-p^-1) mod 2^48 (one IMAD.WIDE + two IMAD; mod 2^LAST_BITS in the last step),
      // then as a double
      const uint32_t qlo = (uint32_t)c[i], qhi = (uint32_t)(c[i] >> 32);
      const uint64_t r = (uint64_t)qlo * P::inv48_lo();
      uint32_t rlo = (uint32_t)r, rhi = ((uint32_t)(r >> 32) + qlo * P::inv48_hi() + qhi * P::inv48_lo()) & 0xffffu;
      if (i == L48 - 1 && LAST_BITS < 48) {
        static_assert(LAST_BITS == 48 || LAST_BITS <= 32, "last step narrower than a word or a whole limb");
        rhi = 0;
        if (LAST_BITS < 32) rlo &= (1u << (LAST_BITS & 31)) - 1u;
      }
      const double m = bits_dbl(0x43300000u | rhi, rlo) - 0x1p52;
      double hi_prev = 0;
#pragma unroll
      for (int j = 0; j < L48; j++) {
        const double pj = (double)P::MOD48(j);
        const double hi = fma_rz(m, pj, C1);
        const double lo = fma_rz(m, pj, C2 - hi);
        if (j == 0)
          c[i] += dbl_bits(lo);
        else
          c[i + j] += dbl_bits(lo) + dbl_bits(hi_prev);
        hi_prev = hi;
      }
      c[i + L48] += dbl_bits(hi_prev);
      // a column wholly below bit 32N is complete now and is 0 mod 2^48: what is above bit 48 moves
      // to the next column
      if (i < CUT_COL) c[i + 1] += (c[i] - col_off48(i)) >> 48;
    }
    // the result starts at bit CUT_SH of column CUT_COL: offsets out, carries through, 32-bit words
#pragma unroll
    for (int k = CUT_COL; k < 2 * L48; k++) c[k] -= col_off48(k);
#pragma unroll
    for (int k = CUT_COL; k < 2 * L48 - 1; k++) {
      c[k + 1] += c[k] >> 48;
      c[k] &= 0xffffffffffffull;
    }
    uint32_t t[N];
#pragma unroll
    for (int w = 0; w < N; w++) {
      const int s = CUT_SH + 32 * w, k = CUT_COL + s / 48, o = s % 48;  // o is 0, 16 or 32
      if (o == 0)
        t[w] = (uint32_t)c[k];
      else if (o == 16)
        t[w] = (uint32_t)(c[k] >> 16);
      else
        t[w] = (uint32_t)(c[k] >> 32) | ((uint32_t)c[k + 1] << 16);
    }
    return finish<FULL>(t);
  }
  // E = B (low word already out), O = A after the last row: upper half T[N..2N) = A + (B >> 32)
  static PB_HD void wide_top(uint32_t* T, const uint32_t* A, const uint32_t* B) {
    T[N] = add_cc(A[0], B[1]);
#pragma unroll
    for (int k = 1; k < N - 1; k++) T[N + k] = addc_cc(A[k], B[k + 1]);
    T[2 * N - 1] = addc(A[N - 1], 0u);
  }
  // T[2N] = a*b (+ c*d): the rows of the Montgomery product without their reduction steps; the low
  // word of the running sum leaves as an output word after every row.
  template <bool TWO>
  static PB_HD void wide_mul(uint32_t* T, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d) {
    uint32_t A[N], B[N];
#pragma unroll
    for (int j = 0; j < N; j += 2) {
      mul_pair(A[j], A[j + 1], a[j], b[0]);
      mul_pair(B[j], B[j + 1], a[j + 1], b[0]);
    }
    if (TWO) acc_row(B, A, c, d[0]);
    T[0] = A[0];  // E = A, O = B
#pragma unroll
    for (int i = 1; i < N; i += 2) {
      mul_row(A, B, a, b[i]);  // E = B, O = A
      if (TWO) acc_row(A, B, c, d[i]);
      T[i] = B[0];
      if (i + 1 < N) {
        mul_row(B, A, a, b[i + 1]);  // E = A, O = B
        if (TWO) acc_row(B, A, c, d[i + 1]);
        T[i + 1] = A[0];
      }
    }
    wide_top(T, A, B);
  }
  template <int I>
  static PB_HD void wide_sqr_rows(uint32_t* T, uint32_t* A, uint32_t* B, const uint32_t* a, const uint32_t* a2) {
    if constexpr (I < N) {
      sqr_row<I>(A, B, a, a2);  // E = B, O = A
      T[I] = B[0];
      if constexpr (I + 1 < N) {
        sqr_row<I + 1>(B, A, a, a2);  // E = A, O = B
        T[I + 1] = A[0];
      }
      wide_sqr_rows<I + 2>(T, A, B, a, a2);
    }
  }
  static PB_HD void wide_sqr(uint32_t* T, const uint32_t* v) {
    uint32_t a2[N];
    a2[0] = v[0] << 1;
#pragma unroll
    for (int k = 1; k < N; k++) a2[k] = (v[k] << 1) | (v[k - 1] >> 31);
    uint32_t A[N], B[N];
#pragma unroll
    for (int j = 0; j < N; j += 2) {
      mul_pair(A[j], A[j + 1], sq_limb<0>(v, a2, j), v[0]);
      mul_pair(B[j], B[j + 1], sq_limb<0>(v, a2, j + 1), v[0]);
    }
    T[0] = A[0];
    wide_sqr_rows<1>(T, A, B, v, a2);
    wide_top(T, A, B);
  }
  // FpR operands (< 2p) give T < 8p^2 < p * 2^(32N) with three spare bits, and T[2N-1] keeps two
  // zero top bits (8p^2 < 2^765 for Fp), which `gate` relies on.
  template <bool FULL = true>
  static PB_HD Field mul_hybrid(const Field& a, const Field& b) {
    uint32_t T[2 * N];
    wide_mul<false>(T, a.v, b.v, a.v, b.v);
    return redc48<FULL>(T);
  }
  template <bool FULL = true>
  PB_HD Field sqr_hybrid() const {
    static_assert((P::MOD(N - 1) >> 30) == 0, "needs two spare bits in the top limb of the modulus");
    uint32_t T[2 * N];
    wide_sqr(T, v);
    return redc48<FULL>(T);
  }
  // a*b + c*d < 2p^2 < p * 2^(32N) needs one spare bit
  template <bool FULL = true>
  static PB_HD Field mul2_hybrid(const Field& a, const Field& b, const Field& c, const Field& d) {
    static_assert((P::MOD(N - 1) >> 30) == 0, "needs two spare bits in the top limb of the modulus");
    uint32_t T[2 * N];
    wide_mul<true>(T, a.v, b.v, c.v, d.v);
    return redc48<FULL>(T);
  }

  // a*b - c*d
  static PB_HD Field mul_sub(const Field& a, const Field& b, const Field& c, const Field& d) { return mul2(a, b, c.neg(), d); }

  // (Interleaving several independent products in program order was tried for instruction-level
  // parallelism and gives nothing: ptxas keeps at most ~6 carry chains in flight - there are only 7
  // predicate registers - and one product already uses 4.  See DESIGN.md section 4.)

  // out of / into Montgomery form
  PB_HD Field from_mont() const {
    Field o = zero();
    o.v[0] = 1;
    return (*this) * o;
  }
  PB_HD Field to_mont() const { return (*this) * r2(); }

  // this^e for a little-endian multi-word exponent (square and multiply, variable time).
  PB_HD Field pow(const uint32_t* e, int words) const {
    Field acc = one();
    bool started = false;  // skip the leading zero bits of the exponent
    for (int w = words - 1; w >= 0; w--) {
      for (int bit = 31; bit >= 0; bit--) {
        if (started) acc = acc.sqr();
        if ((e[w] >> bit) & 1u) {
          acc = started ? acc * (*this) : *this;
          started = true;
        }
      }
    }
    return acc;
  }
  PB_HD Field pow_u64(uint64_t e) const {
    uint32_t w[2] = {(uint32_t)e, (uint32_t)(e >> 32)};
    return pow(w, 2);
  }
  // Fermat inverse (0 -> 0).
  PB_HD Field inv() const {
    uint32_t e[N];
    e[0] = sub_cc(P::MOD(0), 2u);
#pragma unroll
    for (int i = 1; i < N; i++) e[i] = subc_cc(P::MOD(i), 0u);
    return pow(e, N);
  }
};

// Constants are exposed through constexpr accessor functions with function-local tables so that
// they are usable from device code and fold to immediates once the limb loops are unrolled.
#define PB_LIMB_TABLE(name, n, ...)                     \
  static PB_HD constexpr uint32_t name(int i) {         \
    constexpr uint32_t T[n] = {__VA_ARGS__};            \
    return T[i];                                        \
  }

// Fr's Montgomery constant is -1 mod 2^32.  If ptxas can see that, it rewrites m = -t0 and splits
// every IMAD.WIDE of the reduction rows into IMAD.X + IMAD.HI.X (2x the issue slots, measured in
// SASS).  Reading the constant from __constant__ memory keeps it opaque to the optimiser.
#if defined(__CUDACC__)
static __constant__ uint32_t c_fr_inv = 0xffffffffu;
#endif

struct FrParams {
  static constexpr int N = 8;
  static constexpr bool HYBRID = PB_FR_HYBRID != 0;
  // r in 48-bit limbs and -r^-1 mod 2^48, for Field::redc48
  static PB_HD constexpr uint64_t MOD48(int j) {
    constexpr uint64_t T[6] = {0xffff00000001ull, 0xfffe5bfeffffull, 0xd80553bda402ull, 0x3339d80809a1ull,
                               0xa753299d7d48ull, 0x73edull};
    return T[j];
  }
  static PB_HD constexpr uint32_t inv48_lo() { return 0xffffffffu; }
  static PB_HD constexpr uint32_t inv48_hi() { return 0xfffeu; }
  static PB_HD uint32_t inv() {
#if defined(__CUDA_ARCH__)
    return c_fr_inv;
#else
    return 0xffffffffu;
#endif
  }
  PB_LIMB_TABLE(MOD, 8, 0x00000001u, 0xffffffffu, 0xfffe5bfeu, 0x53bda402u, 0x09a1d805u, 0x3339d808u,
                0x299d7d48u, 0x73eda753u)
  PB_LIMB_TABLE(R1, 8, 0xfffffffeu, 0x00000001u, 0x00034802u, 0x5884b7fau, 0xecbc4ff5u, 0x998c4fefu,
                0xacc5056fu, 0x1824b159u)
  PB_LIMB_TABLE(R2, 8, 0xf3f29c6du, 0xc999e990u, 0x87925c23u, 0x2b6cedcbu, 0x7254398fu, 0x05d31496u,
                0x9f59ff11u, 0x0748d9d9u)
};

struct FpParams {
  static constexpr int N = 12;
  static constexpr bool HYBRID = PB_FP_HYBRID != 0;
  // p in 48-bit limbs and -p^-1 mod 2^48, for Field::redc48
  static PB_HD constexpr uint64_t MOD48(int j) {
    constexpr uint64_t T[8] = {0xffffffffaaabull, 0xb153ffffb9feull, 0xf6241eabfffeull, 0x6730d2a0f6b0ull,
                               0x4b84f38512bfull, 0x434bacd76477ull, 0xe69a4b1ba7b6ull, 0x1a0111ea397full};
    return T[j];
  }
  static PB_HD constexpr uint32_t inv48_lo() { return 0xfffcfffdu; }
  static PB_HD constexpr uint32_t inv48_hi() { return 0xfffcu; }
  static PB_HD uint32_t inv() { return 0xfffcfffdu; }
  PB_LIMB_TABLE(MOD, 12, 0xffffaaabu, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u,
                0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau)
  PB_LIMB_TABLE(R1, 12, 0x0002fffdu, 0x76090000u, 0xc40c0002u, 0xebf4000bu, 0x53c758bau, 0x5f489857u,
                0x70525745u, 0x77ce5853u, 0xa256ec6du, 0x5c071a97u, 0xfa80e493u, 0x15f65ec3u)
  PB_LIMB_TABLE(R2, 12, 0x1c341746u, 0xf4df1f34u, 0x09d104f1u, 0x0a76e6a6u, 0x4c95b6d5u, 0x8de5476cu,
                0x939d83c0u, 0x67eb88a9u, 0xb519952du, 0x9a793e85u, 0x92cae3aau, 0x11988fe5u)
};

typedef Field<FrParams> Fr;
typedef Field<FpParams> Fp;

// ---------------------------------------------------------------------------------------------
// FpR: an Fp residue kept in [0, 2p) instead of [0, p) (Montgomery form, R = 2^384), for the G1
// formulas of the MSM.  p < 2^381, so 8p < R, and a Montgomery product returns
//     (a b + m p) / R < p + a b / R,      m < R,
// which is < 2p whenever a b < p R, i.e. for any two operands below 2p (4p^2 < 8p^2 < p R).  So
// products, squares and mul2 / mul_sub of FpR values need no final subtraction - about 25 of the
// ~1100 instructions of a product.  The running sums of the product rows stay inside the two
// accumulators (each row peaks below (operand bound + p) * 2^32, at most 5p * 2^32 < 2^416; see
// Field::sqr_half and Field::mul2 for the squaring's doubled row 0 and the fused pair).
// Additions and subtractions reduce by 2p and cost what the canonical ones cost.  A residue has up to
// two representations, so equality with zero is is_zero_mod_p(); canonical() is the one way back to Fp.
// Canonical Fp (pairing, decoders, host) is untouched.
// ---------------------------------------------------------------------------------------------
struct FpR {
  static constexpr int N = 12;
  static_assert((FpParams::MOD(N - 1) >> 29) == 0, "FpR needs 8p < 2^384");
  uint32_t v[N];

  static PB_HD constexpr uint32_t MOD2(int i) {  // 2p
    return (FpParams::MOD(i) << 1) | (i > 0 ? FpParams::MOD(i - 1) >> 31 : 0u);
  }
  // limbs < 2p taken as they are: a canonical Fp, or the result of a product routine run without its
  // final subtraction
  static PB_HD FpR from(const Fp& a) {
    FpR r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = a.v[i];
    return r;
  }
  static PB_HD FpR zero() { return from(Fp::zero()); }
  static PB_HD FpR one() { return from(Fp::one()); }
  // [0, 2p) -> [0, p)
  PB_HD Fp canonical() const {
    Fp r;
    Fp::final_sub(r.v, v, 0u);
    return r;
  }
  // the limbs read as an Fp operand of the product routines (which accept operands < 2p, see above)
  PB_HD Fp raw() const {
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = v[i];
    return r;
  }
  // all limbs zero: the representation 0 only (p is the other representation of zero)
  PB_HD bool is_zero_limbs() const {
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < N; i++) x |= v[i];
    return x == 0;
  }
  // == 0 mod p: the value is 0 or p
  PB_HD bool is_zero_mod_p() const {
    uint32_t z = 0, q = 0;
#pragma unroll
    for (int i = 0; i < N; i++) {
      z |= v[i];
      q |= v[i] ^ FpParams::MOD(i);
    }
    return z == 0 || q == 0;
  }

  // a + b < 4p < 2^384 (no carry out of the top limb); one conditional subtraction of 2p -> [0, 2p)
  friend PB_HD FpR operator+(const FpR& a, const FpR& b) {
    uint32_t t[N], s[N];
    t[0] = add_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int i = 1; i < N; i++) t[i] = addc_cc(a.v[i], b.v[i]);
    s[0] = sub_cc(t[0], MOD2(0));
#pragma unroll
    for (int i = 1; i < N; i++) s[i] = subc_cc(t[i], MOD2(i));
    const bool ge = subc(0u, 0u) == 0u;  // no borrow: t >= 2p
    FpR r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = ge ? s[i] : t[i];
    return r;
  }
  // a - b in (-2p, 2p); 2p added back when it borrowed -> [0, 2p)
  friend PB_HD FpR operator-(const FpR& a, const FpR& b) {
    uint32_t t[N];
    t[0] = sub_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int i = 1; i < N; i++) t[i] = subc_cc(a.v[i], b.v[i]);
    const uint32_t m = subc(0u, 0u);  // 0xffffffff when a < b
    FpR r;
    r.v[0] = add_cc(t[0], MOD2(0) & m);
#pragma unroll
    for (int i = 1; i < N - 1; i++) r.v[i] = addc_cc(t[i], MOD2(i) & m);
    r.v[N - 1] = addc(t[N - 1], MOD2(N - 1) & m);
    return r;
  }
  PB_HD FpR neg() const { return zero() - *this; }  // 0 stays 0, else 2p - a
  PB_HD FpR dbl() const { return *this + *this; }

  // products: operands < 2p, result < 2p (no final subtraction)
  friend PB_HD FpR operator*(const FpR& a, const FpR& b) { return from(Fp::mul<false>(a.raw(), b.raw())); }
  PB_HD FpR sqr() const { return from(raw().sqr<false>()); }
  // a*b + c*d and a*b - c*d with one Montgomery reduction (Field::mul2)
  static PB_HD FpR mul2(const FpR& a, const FpR& b, const FpR& c, const FpR& d) {
    return from(Fp::mul2<false>(a.raw(), b.raw(), c.raw(), d.raw()));
  }
  // -c enters the product as 2p - c, in (0, 2p]: no borrow to test, and an operand equal to 2p keeps every
  // bound of Field::mul2 (the row peak is at most 5p * 2^32, the products sum to at most 8p^2 < p R).
  static PB_HD FpR mul_sub(const FpR& a, const FpR& b, const FpR& c, const FpR& d) {
    Fp nc;
    nc.v[0] = sub_cc(MOD2(0), c.v[0]);
#pragma unroll
    for (int i = 1; i < N - 1; i++) nc.v[i] = subc_cc(MOD2(i), c.v[i]);
    nc.v[N - 1] = subc(MOD2(N - 1), c.v[N - 1]);
    return from(Fp::mul2<false>(a.raw(), b.raw(), nc, d.raw()));
  }
};

}  // namespace pb
