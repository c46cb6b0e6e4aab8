// The V3 proof algebra, stated once for the device quotient (prover.cu), the prover's linearisation (prover.cu,
// round 5) and the Verifier (verify.cu): the order of the prover-key polynomials, the proof layout, the gate widgets,
// the permutation products and the linearisation scalars.  The Fiat-Shamir schedule that produces the challenges
// is in transcript.h.
//
// The widgets and the permutation products are templates over the field type.  The quotient kernel instantiates
// them with its out-of-line-product Fr wrapper; the host instantiates them with pbh::HFr.  Their forms are the
// kernel's: delta4 as g (g + 2) and small multiples by additions, which give the same values as the reference's
// f (f - 1)(f - 2)(f - 3) and k * x.  Like bigint.cuh, the header compiles under nvcc and under plain g++.
#pragma once
#include <stddef.h>

#include "bigint.cuh"
#include "host_field.h"

// For the templates below: nvcc checks that a __host__ __device__ function calls no host-only code, but pbh::HFr's
// arithmetic is host code, so its instantiations are exempted.
#if defined(__CUDACC__)
#define PB_HOST_INSTANTIABLE _Pragma("nv_exec_check_disable")
#else
#define PB_HOST_INSTANTIABLE
#endif

namespace pb {

// The 15 prover-key polynomials (11 selectors, then the 4 permutation polynomials) in this library's order: the
// order of pb200_prover_commitments and of every per-polynomial array.
enum Poly { Q_M, Q_L, Q_R, Q_O, Q_F, Q_C, Q_ARITH, Q_RANGE, Q_LOGIC, Q_FIXED, Q_VAR, S1, S2, S3, S4, N_POLY };

// ProverKey::to_var_bytes (widget.rs:347-445) and VerifierKey::to_bytes (widget.rs:84-111) store the polynomials
// and the commitments in this order, with q_logic before q_range.
static const int kKeyFileOrder[N_POLY] = {Q_M, Q_L, Q_R, Q_O, Q_F, Q_C, Q_ARITH, Q_LOGIC, Q_RANGE, Q_FIXED, Q_VAR, S1, S2, S3, S4};

// VerifierKey::seed_transcript (widget.rs:218-257) appends the commitments in this order under these labels.  The
// legacy seed of PlonkVersion::V1 and V2 (seed_transcript_legacy) is the same list with one substitution: the
// commitment of s_sigma_1 goes in under the "s_sigma_4" label, so s_sigma_4 is not bound (transcript.h).
struct SeedEntry {
  const char* label;
  int poly;
};
static const SeedEntry kSeedOrder[N_POLY] = {
    {"q_m", Q_M},         {"q_l", Q_L},         {"q_r", Q_R},
    {"q_o", Q_O},         {"q_c", Q_C},         {"q_f", Q_F},
    {"q_arith", Q_ARITH}, {"q_range", Q_RANGE}, {"q_logic", Q_LOGIC},
    {"q_variable_group_add", Q_VAR}, {"q_fixed_group_add", Q_FIXED}, {"s_sigma_1", S1},
    {"s_sigma_2", S2},    {"s_sigma_3", S3},    {"s_sigma_4", S4}};

// Proof::to_bytes (proof.rs:137-162): 11 compressed commitments, then 15 canonical evaluations.
enum ProofComm { C_A, C_B, C_C, C_D, C_Z, C_T_LOW, C_T_MID, C_T_HIGH, C_T_FOURTH, C_W_Z, C_W_ZW, N_COMM };
enum ProofEval { E_A, E_B, E_C, E_D, E_AW, E_BW, E_DW, E_QARITH, E_QC, E_QL, E_QR, E_S1, E_S2, E_S3, E_Z, N_EVAL };
constexpr size_t kProofEvalAt = 48 * N_COMM;                // 528
constexpr size_t kProofBytes = kProofEvalAt + 32 * N_EVAL;  // 1008

// The challenges of one proof, in transcript order.
struct Challenges {
  pbh::HFr beta, gamma;
  pbh::HFr alpha, range, logic, fixed, var;  // alpha and the four separation challenges
  pbh::HFr z, v, v_w, u;
};

// ---- gate widgets ---------------------------------------------------------------------------------------------
// A separation challenge ch with the powers of kappa = ch^2 its widget uses: k = kappa, k2 = kappa^2, ...
template <class F>
struct SepPowers {
  F ch, k, k2, k3, k4;
};
PB_HOST_INSTANTIABLE
template <class F>
PB_HD SepPowers<F> sep_powers(const F& ch) {
  SepPowers<F> s;
  s.ch = ch;
  s.k = ch.sqr();
  s.k2 = s.k.sqr();
  s.k3 = s.k2 * s.k;
  s.k4 = s.k3 * s.k;
  return s;
}

PB_HOST_INSTANTIABLE
template <class F>
PB_HD F delta4(const F& f) {  // f (f - 1)(f - 2)(f - 3) = g (g + 2) with g = f (f - 3): two products
  const F one = F::one();
  const F g = f * (f - one - one - one);
  return g * (g + one + one);
}
PB_HOST_INSTANTIABLE
template <class F>
PB_HD F mul_small(const F& x, int k) {  // k * x for small positive k by additions
  F acc = F::zero(), p = x;
  while (k) {
    if (k & 1) acc = acc + p;
    p = p.dbl();
    k >>= 1;
  }
  return acc;
}

// The wire values at a point X and at omega X.
template <class F>
struct WireVals {
  F a, b, c, d, a_w, b_w, d_w;
};

// The widgets without their selector.  S is the field type the separation powers are stored in; the kernel keeps
// them as plain Fr and converts them at use.
PB_HOST_INSTANTIABLE
template <class F, class S>
PB_HD F widget_range(const SepPowers<S>& s, const WireVals<F>& v) {  // range/proverkey.rs:32-57
  const F &ch = s.ch, &k = s.k, &k2 = s.k2, &k3 = s.k3;
  F t = delta4(v.c - mul_small(v.d, 4)) + delta4(v.b - mul_small(v.c, 4)) * k + delta4(v.a - mul_small(v.b, 4)) * k2 +
        delta4(v.d_w - mul_small(v.a, 4)) * k3;
  return t * ch;
}
PB_HOST_INSTANTIABLE
template <class F, class S>
PB_HD F widget_logic(const SepPowers<S>& s, const F& q_c, const WireVals<F>& v) {  // logic/proverkey.rs:34-71, 120-144
  const F &ch = s.ch, &k = s.k, &k2 = s.k2, &k3 = s.k3, &k4 = s.k4;
  F A = v.a_w - mul_small(v.a, 4), B = v.b_w - mul_small(v.b, 4), D = v.d_w - mul_small(v.d, 4);
  const F& w = v.c;
  F ab = A + B;
  F Fx = w * (w * (mul_small(w, 4) - mul_small(ab, 18) + mul_small(F::one(), 81)) + mul_small(A.sqr() + B.sqr(), 18) - mul_small(ab, 81) + mul_small(F::one(), 83));
  F E = mul_small(ab + D, 3) - Fx.dbl();
  F Bq = q_c * (mul_small(D, 9) - mul_small(ab, 3));
  F t = delta4(A) + delta4(B) * k + delta4(D) * k2 + (w - A * B) * k3 + (Bq + E) * k4;
  return t * ch;
}
// ed: dusk_jubjub::EDWARDS_D
PB_HOST_INSTANTIABLE
template <class F, class S>
PB_HD F widget_fixed(const SepPowers<S>& s, const F& ed, const F& q_l, const F& q_r, const F& q_c, const WireVals<F>& v) {  // fixed_base/proverkey.rs:39-103
  const F one = F::one();
  const F &ch = s.ch, &k = s.k, &k2 = s.k2, &k3 = s.k3;
  F bit = v.d_w - v.d - v.d;
  F bit_c = bit * (bit - one) * (bit + one);
  F y_alpha = bit.sqr() * (q_r - one) + one, x_alpha = bit * q_l;
  F xy = (bit * q_c - v.c) * k;
  F t = v.c * v.a * v.b * ed;
  F xa = ((v.a_w + v.a_w * t) - (v.a * y_alpha + v.b * x_alpha)) * k2;
  F ya = ((v.b_w - v.b_w * t) - (v.b * y_alpha + v.a * x_alpha)) * k3;
  return (bit_c + xa + ya + xy) * ch;
}
PB_HOST_INSTANTIABLE
template <class F, class S>
PB_HD F widget_var(const SepPowers<S>& s, const F& ed, const WireVals<F>& v) {  // curve_addition/proverkey.rs:33-79
  const F &ch = s.ch, &k = s.k;
  const F &x1 = v.a, &x3 = v.a_w, &y1 = v.b, &y3 = v.b_w, &x2 = v.c, &y2 = v.d, &x1y2 = v.d_w;
  F xy = x1 * y2 - x1y2, y1x2 = y1 * x2, y1y2 = y1 * y2, x1x2 = x1 * x2;
  F t = ed * x1y2 * y1x2;
  F x3c = ((x1y2 + y1x2) - (x3 + x3 * t)) * k;
  F y3c = ((y1y2 + x1x2) - (y3 - y3 * t)) * s.k2;
  return (xy + x3c + y3c) * ch;
}

// ---- gate identities, one per row (debugger.rs:31-49, 95-180) ------------------------------------------------
// The terms the widgets above combine, one by one and without their separation challenge: each widget is ch times
// the kappa-weighted sum of its terms, in the order below (kappa^j weights term j; the fixed-base widget's terms in
// this order are bit, xy kappa, x kappa^2, y kappa^3).  tests/test_debugger_algebra.py checks that relation.  The
// 17 identities of a row are the arithmetic term plus these terms, each times its widget's selector.
enum IdentityFamily { ID_ARITH = 0, ID_RANGE = 1, ID_LOGIC = 5, ID_FIXED = 10, ID_VAR = 14, N_IDENTITIES = 17 };
static const char* const kIdentityFamilies[N_IDENTITIES] = {
    "arithmetic",
    "range delta c/d", "range delta b/c", "range delta a/b", "range accumulator",
    "logic left quad", "logic right quad", "logic output quad", "logic product", "logic relation",
    "fixed-base bit consistency", "fixed-base xy consistency", "fixed-base x accumulator", "fixed-base y accumulator",
    "variable-base xy consistency", "variable-base x accumulator", "variable-base y accumulator"};

template <class F, int K>
struct Terms {
  F t[K];
};
// q(k) returns the selector k (Poly order) of the row
PB_HOST_INSTANTIABLE
template <class F, class Sel>
PB_HD F arith_identity(const Sel& q, const F& pi, const WireVals<F>& v) {  // arithmetic/proverkey.rs:44-69
  return (v.a * v.b * q(Q_M) + v.a * q(Q_L) + v.b * q(Q_R) + v.c * q(Q_O) + v.d * q(Q_F) + q(Q_C)) * q(Q_ARITH) + pi;
}
PB_HOST_INSTANTIABLE
template <class F>
PB_HD Terms<F, 4> range_terms(const WireVals<F>& v) {
  return {{delta4(v.c - mul_small(v.d, 4)), delta4(v.b - mul_small(v.c, 4)), delta4(v.a - mul_small(v.b, 4)), delta4(v.d_w - mul_small(v.a, 4))}};
}
PB_HOST_INSTANTIABLE
template <class F>
PB_HD Terms<F, 5> logic_terms(const F& q_c, const WireVals<F>& v) {
  const F A = v.a_w - mul_small(v.a, 4), B = v.b_w - mul_small(v.b, 4), D = v.d_w - mul_small(v.d, 4);
  const F& w = v.c;
  const F ab = A + B;
  const F Fx = w * (w * (mul_small(w, 4) - mul_small(ab, 18) + mul_small(F::one(), 81)) + mul_small(A.sqr() + B.sqr(), 18) - mul_small(ab, 81) + mul_small(F::one(), 83));
  const F E = mul_small(ab + D, 3) - Fx.dbl();
  const F Bq = q_c * (mul_small(D, 9) - mul_small(ab, 3));
  return {{delta4(A), delta4(B), delta4(D), w - A * B, Bq + E}};
}
PB_HOST_INSTANTIABLE
template <class F>
PB_HD Terms<F, 4> fixed_terms(const F& ed, const F& q_l, const F& q_r, const F& q_c, const WireVals<F>& v) {
  const F one = F::one();
  const F bit = v.d_w - v.d - v.d;
  const F y_alpha = bit.sqr() * (q_r - one) + one, x_alpha = bit * q_l;
  const F t = v.c * v.a * v.b * ed;
  return {{bit * (bit - one) * (bit + one), bit * q_c - v.c, (v.a_w + v.a_w * t) - (v.a * y_alpha + v.b * x_alpha),
           (v.b_w - v.b_w * t) - (v.b * y_alpha + v.a * x_alpha)}};
}
PB_HOST_INSTANTIABLE
template <class F>
PB_HD Terms<F, 3> var_terms(const F& ed, const WireVals<F>& v) {
  const F &x1 = v.a, &x3 = v.a_w, &y1 = v.b, &y3 = v.b_w, &x2 = v.c, &y2 = v.d, &x1y2 = v.d_w;
  const F y1x2 = y1 * x2;
  const F t = ed * x1y2 * y1x2;
  return {{x1 * y2 - x1y2, (x1y2 + y1x2) - (x3 + x3 * t), (y1 * y2 + x1 * x2) - (y3 - y3 * t)}};
}
PB_HOST_INSTANTIABLE
template <class F, int K>
PB_HD int first_nonzero(const Terms<F, K>& t, int family) {
  for (int k = 0; k < K; k++)
    if (!t.t[k].is_zero()) return family + k;
  return -1;
}
// The index (IdentityFamily + term) of the first of the row's 17 identities that is not zero, or -1.  A term times a
// non-zero selector is zero exactly when the term is, so a widget whose selector is zero is skipped and the others are
// tested without the product; the arithmetic identity is skipped only when both q_arith and pi are zero.
PB_HOST_INSTANTIABLE
template <class F, class Sel>
PB_HD int first_failing_identity(const Sel& q, const F& pi, const F& ed, const WireVals<F>& v) {
  int r = -1;
  if ((!q(Q_ARITH).is_zero() || !pi.is_zero()) && !arith_identity(q, pi, v).is_zero()) return ID_ARITH;
  if (!q(Q_RANGE).is_zero() && (r = first_nonzero(range_terms(v), ID_RANGE)) >= 0) return r;
  if (!q(Q_LOGIC).is_zero() && (r = first_nonzero(logic_terms(q(Q_C), v), ID_LOGIC)) >= 0) return r;
  if (!q(Q_FIXED).is_zero() && (r = first_nonzero(fixed_terms(ed, q(Q_L), q(Q_R), q(Q_C), v), ID_FIXED)) >= 0) return r;
  if (!q(Q_VAR).is_zero() && (r = first_nonzero(var_terms(ed, v), ID_VAR)) >= 0) return r;
  return -1;
}

// ---- permutation (permutation/proverkey.rs:40-125) -----------------------------------------------------------
// The identity permutation's product at a point x, with bx = beta x and the coset constants K1..K3 = 7, 13, 17:
// (a + bx + gamma)(b + 7 bx + gamma)(c + 13 bx + gamma)(d + 17 bx + gamma).
PB_HOST_INSTANTIABLE
template <class F>
PB_HD F perm_ident(const WireVals<F>& v, const F& bx, const F& gamma) {
  return (v.a + bx + gamma) * (v.b + mul_small(bx, 7) + gamma) * (v.c + mul_small(bx, 13) + gamma) * (v.d + mul_small(bx, 17) + gamma);
}
// The copy permutation's product up to its sigma_4 factor: (a + beta s1 + gamma)(b + beta s2 + gamma)(c + beta s3 + gamma),
// with s_j = sigma(j - 1).  The quotient multiplies it by (d + beta s4 + gamma); the linearisation keeps s4 as a
// polynomial.  sigma is called where each value is needed, so that the kernel loads each value just before its use.
PB_HOST_INSTANTIABLE
template <class F, class Sigma>
PB_HD F perm_copy3(const WireVals<F>& v, const F& beta, const F& gamma, const Sigma& sigma) {
  return (v.a + beta * sigma(0) + gamma) * (v.b + beta * sigma(1) + gamma) * (v.c + beta * sigma(2) + gamma);
}

// ---- linearisation (host) ------------------------------------------------------------------------------------
inline WireVals<pbh::HFr> eval_wires(const pbh::HFr ev[N_EVAL]) {
  return {ev[E_A], ev[E_B], ev[E_C], ev[E_D], ev[E_AW], ev[E_BW], ev[E_DW]};
}

// The scalars of the linearisation polynomial r(X) (linearization_poly.rs:168-231 with every widget's
// compute_linearization): sel[p] multiplies the prover-key polynomial p and is zero where r(X) has no such term
// (q_arith, s_sigma_1..3); z multiplies z(X); t[j] multiplies t_low .. t_fourth.  z_n = z^n, l1 = L_1(z).
struct LinScalars {
  pbh::HFr sel[N_POLY], z, t[4];
};
inline LinScalars linearisation_scalars(const pbh::HFr ev[N_EVAL], const Challenges& c, const pbh::HFr& z_n, const pbh::HFr& l1) {
  using pbh::HFr;
  const WireVals<HFr> w = eval_wires(ev);
  const HFr qa = ev[E_QARITH];
  LinScalars s;
  for (HFr& x : s.sel) x = HFr::zero();
  s.sel[Q_M] = w.a * w.b * qa;
  s.sel[Q_L] = w.a * qa;
  s.sel[Q_R] = w.b * qa;
  s.sel[Q_O] = w.c * qa;
  s.sel[Q_F] = w.d * qa;
  s.sel[Q_C] = qa;
  s.sel[Q_RANGE] = widget_range(sep_powers(c.range), w);
  s.sel[Q_LOGIC] = widget_logic(sep_powers(c.logic), ev[E_QC], w);
  s.sel[Q_FIXED] = widget_fixed(sep_powers(c.fixed), pbh::edwards_d(), ev[E_QL], ev[E_QR], ev[E_QC], w);
  s.sel[Q_VAR] = widget_var(sep_powers(c.var), pbh::edwards_d(), w);
  s.sel[S4] = (perm_copy3(w, c.beta, c.gamma, [&](int j) { return ev[E_S1 + j]; }) * (c.beta * ev[E_Z]) * c.alpha).neg();
  s.z = perm_ident(w, c.beta * c.z, c.gamma) * c.alpha + l1 * c.alpha.sqr();
  s.t[0] = (z_n - HFr::one()).neg();  // -Z_H(z)
  for (int j = 1; j < 4; j++) s.t[j] = s.t[j - 1] * z_n;
  return s;
}

}  // namespace pb
