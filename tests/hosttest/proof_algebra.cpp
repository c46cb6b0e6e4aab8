// Host build (g++) of the shared V3 proof algebra (plonk_b200/csrc/plonk_algebra.cuh) and transcript schedule
// (transcript.h), for tests/test_proof_algebra.py.  The widgets and permutation products are instantiated twice:
// with pbh::HFr, as the prover's round 5 and the Verifier use them, and with the host build of pb::Fr, the
// quotient kernel's arithmetic.  All field values cross this interface as 32-byte Montgomery-form integers, the
// in-memory layout of both types.
#include <stddef.h>
#include <string.h>

#include "../../plonk_b200/csrc/host_field.cpp"
#include "../../plonk_b200/csrc/transcript.h"

using namespace pb;
using pbh::HFr;

namespace {

template <class F>
F load(const uint8_t* p) {
  F x;
  memcpy(x.v, p, 32);
  return x;
}
template <class F>
void store(uint8_t* p, const F& x) {
  memcpy(p, x.v, 32);
}

// One point: in = ch_range, ch_logic, ch_fixed, ch_var, q_l, q_r, q_c, a, b, c, d, a_w, b_w, d_w, z, z_w, alpha,
// beta, gamma, x, s1, s2, s3, s4.  out = the four widgets, then the identity and copy terms composed as the
// quotient kernel composes them.
template <class F>
void widgets_at(const uint8_t* in, uint8_t* out) {
  F x[24];
  for (int k = 0; k < 24; k++) x[k] = load<F>(in + 32 * k);
  const F ed = load<F>((const uint8_t*)pbh::edwards_d().v);
  const WireVals<F> v = {x[7], x[8], x[9], x[10], x[11], x[12], x[13]};
  const F &z = x[14], &z_w = x[15], &alpha = x[16], &beta = x[17], &gamma = x[18];
  store(out, widget_range(sep_powers(x[0]), v));
  store(out + 32, widget_logic(sep_powers(x[1]), x[6], v));
  store(out + 64, widget_fixed(sep_powers(x[2]), ed, x[4], x[5], x[6], v));
  store(out + 96, widget_var(sep_powers(x[3]), ed, v));
  store(out + 128, perm_ident(v, beta * x[19], gamma) * z * alpha);
  store(out + 160, perm_copy3(v, beta, gamma, [&](int j) { return x[20 + j]; }) * (v.d + beta * x[23] + gamma) * z_w * alpha);
}

}  // namespace

extern "C" {

// field: 0 = pbh::HFr, 1 = pb::Fr.  in: n x 24 values, out: n x 6 values.
int pa_widgets(int field, const uint8_t* in, size_t n, uint8_t* out) {
  for (size_t i = 0; i < n; i++) {
    if (field == 0)
      widgets_at<HFr>(in + 24 * 32 * i, out + 6 * 32 * i);
    else
      widgets_at<Fr>(in + 24 * 32 * i, out + 6 * 32 * i);
  }
  return 0;
}

// Replays a proof's transcript from its bytes and computes the linearisation scalars.  key_comms: 15 x 48 in
// pb::Poly order; pi: n_pi Montgomery values; n: the domain size.  out: beta, gamma, alpha, the four separation
// challenges, z, v, v_w, u (11 values), then sel[15], z, t[4] of the linearisation (20 values).
int pa_replay(const uint8_t* label, size_t label_len, uint64_t constraints, const uint8_t* key_comms, uint64_t vk_n,
              const uint8_t* pi, size_t n_pi, const uint8_t* proof, uint64_t n, uint8_t* out) {
  HFr ev[N_EVAL];
  for (int k = 0; k < N_EVAL; k++) ev[k] = load<HFr>(proof + kProofEvalAt + 32 * k).to_mont();
  pbh::Transcript tr = pbh::seed_transcript(label, label_len, constraints, key_comms, vk_n);
  for (size_t k = 0; k < n_pi; k++) tr.append_scalar("pi", load<HFr>(pi + 32 * k));
  Challenges c;
  pbh::challenge_beta_gamma(tr, proof, c);
  pbh::challenge_alpha(tr, proof, c);
  pbh::challenge_z(tr, proof, c);
  pbh::challenge_v(tr, ev, c);
  pbh::challenge_u(tr, proof, c);
  const HFr ch[11] = {c.beta, c.gamma, c.alpha, c.range, c.logic, c.fixed, c.var, c.z, c.v, c.v_w, c.u};
  for (int k = 0; k < 11; k++) store(out + 32 * k, ch[k]);
  const HFr z_n = c.z.pow_u64(n);
  const HFr l1 = (z_n - HFr::one()) * (HFr::from_u64(n) * (c.z - HFr::one())).inv();
  const LinScalars ls = linearisation_scalars(ev, c, z_n, l1);
  uint8_t* o = out + 32 * 11;
  for (int k = 0; k < N_POLY; k++) store(o + 32 * k, ls.sel[k]);
  store(o + 32 * N_POLY, ls.z);
  for (int j = 0; j < 4; j++) store(o + 32 * (N_POLY + 1 + j), ls.t[j]);
  return 0;
}
}
