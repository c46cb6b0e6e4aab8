// Host build (g++) of the versioned transcript seeds (plonk_b200/csrc/transcript.h) and of the Verifier's scalars
// (plonk_b200/csrc/verify_scalars.h), for tests/test_plonk_versions.py.  Field values cross this interface as
// 32-byte Montgomery-form integers; the verifier's scalars come back canonical, as k_verify_msm reads them.
#include <stddef.h>
#include <string.h>

#include "../../plonk_b200/csrc/host_field.cpp"
#include "../../plonk_b200/csrc/verify_scalars.h"

using namespace pb;
using pbh::HFr;

namespace {
HFr load(const uint8_t* p) {
  HFr x;
  memcpy(x.v, p, 32);
  return x;
}
}  // namespace

extern "C" {

// The challenges of a proof replayed from its bytes under a seed: legacy = 0 is Transcript::base_v3, 1 is
// Transcript::base.  key_comms: 15 x 48 in pb::Poly order.  out: beta, gamma, alpha, the four separation challenges,
// z, v, v_w, u.
int pv_challenges(const uint8_t* label, size_t label_len, uint64_t constraints, const uint8_t* key_comms, int legacy,
                  const uint8_t* pi, size_t n_pi, const uint8_t* proof, uint8_t* out) {
  HFr ev[N_EVAL];
  for (int k = 0; k < N_EVAL; k++) ev[k] = load(proof + kProofEvalAt + 32 * k).to_mont();
  pbh::Transcript tr = legacy ? pbh::seed_transcript_legacy(label, label_len, constraints, key_comms, constraints)
                              : pbh::seed_transcript(label, label_len, constraints, key_comms, constraints);
  for (size_t k = 0; k < n_pi; k++) tr.append_scalar("pi", load(pi + 32 * k));
  Challenges c;
  pbh::challenge_beta_gamma(tr, proof, c);
  pbh::challenge_alpha(tr, proof, c);
  pbh::challenge_z(tr, proof, c);
  pbh::challenge_v(tr, ev, c);
  pbh::challenge_u(tr, proof, c);
  const HFr ch[11] = {c.beta, c.gamma, c.alpha, c.range, c.logic, c.fixed, c.var, c.z, c.v, c.v_w, c.u};
  for (int k = 0; k < 11; k++) memcpy(out + 32 * k, ch[k].v, 32);
  return 0;
}

// verify_scalars for one proof under `version`.  n: the domain size; group_gen: its generator; pi_roots: n_pi values
// group_gen^-index; pi: the n_pi public inputs.  out: the 32 canonical scalars of k_verify_msm.  Returns the
// status verify_scalars returns.
int pv_scalars(const uint8_t* label, size_t label_len, uint64_t constraints, const uint8_t* key_comms, uint64_t n,
               const uint8_t* group_gen, const uint8_t* pi_roots, const uint8_t* pi, size_t n_pi, const uint8_t* proof,
               int version, uint64_t* out) {
  VerifyKeyHost K;
  K.base_v3 = pbh::seed_transcript(label, label_len, constraints, key_comms, constraints);
  K.base_legacy = pbh::seed_transcript_legacy(label, label_len, constraints, key_comms, constraints);
  K.n = n;
  K.group_gen = load(group_gen);
  K.size_fr = HFr::from_u64(n);
  K.size_inv = K.size_fr.inv();
  for (size_t k = 0; k < n_pi; k++) K.pi_roots.push_back(load(pi_roots + 32 * k));
  std::vector<HFr> pv(n_pi);
  for (size_t k = 0; k < n_pi; k++) pv[k] = load(pi + 32 * k);
  return verify_scalars(K, version, proof, pv.data(), out);
}
}
