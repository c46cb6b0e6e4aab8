// The Verifier's host side for one proof (reference src/proof_system/proof.rs): the transcript replay and the 32
// scalars of k_verify_msm, for each PlonkVersion.  Host code only; it compiles under nvcc (verify.cu) and under
// plain g++ (tests/hosttest/plonk_versions.cpp).
//
// The versions differ in two places:
//   - the seed: V3 starts from Transcript::base_v3, V1 and V2 from Transcript::base (transcript.h);
//   - the opening at z: V2 and V3 open 14 evaluations (Proof::verify, V_MAX_DEGREE = 11 at z, then a_w, b_w, d_w at
//     z omega); V1 opens 10 (Proof::verify_legacy, proof.rs:518-790, V_MAX_DEGREE_LEGACY = 7: a, b, c, d and
//     s_sigma_1..3 at z, then the three shifted ones), so [F] has no q_arith, q_c, q_l, q_r terms and their lanes
//     of k_verify_msm get zero scalars.
// The linearisation terms, r_0, L_1(z), the public-input evaluation and the pairing are shared.  V1 therefore does
// not bind the selector evaluations q_arith, q_c, q_l and q_r to the key: its verdict means something only for proofs
// made under the old rules, as with the reference's verify_legacy.
#pragma once
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../include/plonk_b200.h"
#include "host_field.h"
#include "plonk_algebra.cuh"
#include "transcript.h"

namespace pb {

// What verify_scalars reads of a Verifier.
struct VerifyKeyHost {
  pbh::Transcript base_v3, base_legacy;  // after seeding, before the public inputs
  uint64_t n = 0;                        // the domain size
  pbh::HFr size_fr, size_inv, group_gen;  // |H|, 1/|H|, omega
  std::vector<pbh::HFr> pi_roots;         // group_gen_inv^index for each public-input position
  VerifyKeyHost() : base_v3(nullptr, 0), base_legacy(nullptr, 0) {}
};

#define PB_VERIFY_TERMS 32

inline bool fr_canonical(const uint8_t* b, pbh::HFr* out) {  // BlsScalar::from_bytes: little-endian, below r
  uint64_t w[4];
  memcpy(w, b, 32);
  for (int k = 3; k >= 0; k--) {
    if (w[k] < pbh::kFrMod.p[k]) break;
    if (w[k] > pbh::kFrMod.p[k] || k == 0) return false;
  }
  memcpy(out->v, w, 32);
  *out = out->to_mont();
  return true;
}

// Proof::verify (V2, V3) or Proof::verify_legacy (V1) up to the pairing: the transcript replay and the 32 scalars
// of k_verify_msm (canonical form, in its term order).  version: a pb200_plonk_version.  Returns PB200_OK,
// PB200_ERR_POINT_MALFORMED for a non-canonical evaluation or PB200_ERR_VERIFY.  u_out, when given, receives the
// last challenge u (Montgomery form) of a proof that reaches it.
inline int verify_scalars(const VerifyKeyHost& K, int version, const uint8_t* proof, const pbh::HFr* pi, uint64_t* out,
                          pbh::HFr* u_out = nullptr) {
  using pbh::HFr;
  HFr e[N_EVAL];
  for (int k = 0; k < N_EVAL; k++)
    if (!fr_canonical(proof + kProofEvalAt + 32 * k, &e[k])) return PB200_ERR_POINT_MALFORMED;
  pbh::Transcript tr = version == PB200_PLONK_V3 ? K.base_v3 : K.base_legacy;
  for (size_t k = 0; k < K.pi_roots.size(); k++) tr.append_scalar("pi", pi[k]);
  Challenges c;
  pbh::challenge_beta_gamma(tr, proof, c);
  pbh::challenge_alpha(tr, proof, c);
  pbh::challenge_z(tr, proof, c);
  pbh::challenge_v(tr, e, c);
  pbh::challenge_u(tr, proof, c);
  const HFr &z = c.z, &v = c.v, &v_w = c.v_w, &u = c.u;
  if (u_out) *u_out = u;

  const HFr one = HFr::one();
  const HFr z_n = z.pow_u64(K.n), z_h = z_n - one;
  // compute_lagrange_and_barycentric_evaluations (proof.rs:997-1040): one batch inversion
  std::vector<HFr> den, pref;
  std::vector<size_t> which;
  den.push_back(K.size_fr * (z - one));
  for (size_t k = 0; k < K.pi_roots.size(); k++)
    if (!pi[k].is_zero()) {
      den.push_back(K.pi_roots[k] * z - one);
      which.push_back(k);
    }
  pref.resize(den.size());
  HFr acc = one;
  for (size_t k = 0; k < den.size(); k++) {
    if (den[k].is_zero()) return PB200_ERR_VERIFY;
    pref[k] = acc;
    acc = acc * den[k];
  }
  HFr inv = acc.inv_bingcd();
  for (size_t k = den.size(); k-- > 0;) {
    const HFr d = den[k];
    den[k] = inv * pref[k];
    inv = inv * d;
  }
  const HFr l1 = z_h * den[0];
  HFr pi_eval = HFr::zero();
  for (size_t j = 0; j < which.size(); j++) pi_eval = pi_eval + den[1 + j] * pi[which[j]];
  pi_eval = pi_eval * z_h * K.size_inv;

  const HFr perm = perm_copy3(eval_wires(e), c.beta, c.gamma, [&](int j) { return e[E_S1 + j]; });
  const HFr r0 = pi_eval - l1 * c.alpha.sqr() - c.alpha * perm * (e[E_D] + c.gamma) * e[E_Z];
  // the evaluations opened at z in [E] order, then the three at z omega: V_MAX_DEGREE + 3 (proof.rs:344-375) or
  // V_MAX_DEGREE_LEGACY + 3 (proof.rs:653-689)
  static const int kOpen[14] = {E_A, E_B, E_C, E_D, E_S1, E_S2, E_S3, E_QARITH, E_QC, E_QL, E_QR, E_AW, E_BW, E_DW};
  static const int kOpenLegacy[10] = {E_A, E_B, E_C, E_D, E_S1, E_S2, E_S3, E_AW, E_BW, E_DW};
  const bool legacy = version == PB200_PLONK_V1;
  const int at_z = legacy ? 7 : 11;
  const int* eo = legacy ? kOpenLegacy : kOpen;
  HFr vc[14];
  vc[0] = v;
  for (int k = 1; k < at_z; k++) vc[k] = vc[k - 1] * v;
  vc[at_z] = v_w * u;
  vc[at_z + 1] = vc[at_z] * v_w;
  vc[at_z + 2] = vc[at_z + 1] * v_w;
  HFr E = u * e[E_Z] - r0;
  for (int k = 0; k < at_z + 3; k++) E = E + e[eo[k]] * vc[k];

  const LinScalars ls = linearisation_scalars(e, c, z_n, l1);
  // [F]: a, b, c, d, s_sigma_1..3, then (V2, V3) q_arith, q_c, q_l, q_r; V1 leaves those four zero
  HFr f[11];
  for (int k = 0; k < 11; k++) f[k] = k < at_z ? vc[k] : HFr::zero();
  f[0] = f[0] + vc[at_z];
  f[1] = f[1] + vc[at_z + 1];
  f[3] = f[3] + vc[at_z + 2];
  const HFr s[PB_VERIFY_TERMS] = {ls.sel[Q_M], ls.sel[Q_L], ls.sel[Q_R], ls.sel[Q_O], ls.sel[Q_F], ls.sel[Q_C], ls.sel[Q_RANGE],
                                  ls.sel[Q_LOGIC], ls.sel[Q_FIXED], ls.sel[Q_VAR], ls.z + u, ls.sel[S4], ls.t[0], ls.t[1], ls.t[2],
                                  ls.t[3], f[0], f[1], f[2], f[3], f[4], f[5], f[6], f[7], f[8], f[9], f[10],
                                  E.neg(), z, u * z * K.group_gen, HFr::zero(), u};
  for (int k = 0; k < PB_VERIFY_TERMS; k++) {
    const HFr cn = s[k].from_mont();
    memcpy(out + 4 * k, cn.v, 32);
  }
  return PB200_OK;
}

// The challenge rho of batch verification: w_i = rho^i weighs proof i's pairing check, and the batch passes iff
// e(sum w_i L_i, [x]H) e(sum w_i R_i, H) = 1.  Drawn as the reference's batch_challenge (key.rs:571-591) draws its
// challenge, from a transcript over the whole batch: the version, the length and each proof's u in batch order.  u
// is the last Fiat-Shamir challenge of its proof, so it binds the key, the seed, the public inputs and every proof
// byte, and rho is fixed only once the whole batch is.  us: Montgomery form; returns rho in Montgomery form.
//
// A call over several groups (group g: lens[g] proofs under versions[g], each group under its own verifier) appends
// "version", "batch-len" and the group's u values once per group, in call order, so one group draws exactly the rho
// above.  u binds its proof's verifier key, but not V1 against V2 (both start from the legacy seed), hence the
// per-group version; the per-group lengths make the sequence parse one way only.  us: every group's u in call order.
inline pbh::HFr batch_challenge(const int* versions, const size_t* lens, size_t n_groups, const pbh::HFr* us) {
  pbh::Transcript t((const uint8_t*)"dusk-plonk", 10);
  t.append_message("dom-sep", (const uint8_t*)"plonk-batch-verify-v1", 21);
  for (size_t g = 0; g < n_groups; g++) {
    t.append_u64("version", (uint64_t)versions[g]);
    t.append_u64("batch-len", (uint64_t)lens[g]);
    for (size_t i = 0; i < lens[g]; i++) t.append_scalar("batch-u", *us++);
  }
  return t.challenge_scalar("batch-challenge");
}
inline pbh::HFr batch_challenge(int version, const pbh::HFr* us, size_t n) { return batch_challenge(&version, &n, 1, us); }

// w_i = rho^i for i = 0 .. n-1 (Montgomery form).
inline std::vector<pbh::HFr> batch_weights(const pbh::HFr& rho, size_t n) {
  std::vector<pbh::HFr> w(n);
  pbh::HFr acc = pbh::HFr::one();
  for (size_t i = 0; i < n; i++) {
    w[i] = acc;
    acc = acc * rho;
  }
  return w;
}

}  // namespace pb
