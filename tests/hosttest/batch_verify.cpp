// Host build (g++) of batch verification's host side (plonk_b200/csrc/verify_scalars.h): the batch challenge rho,
// its weights and each proof's scalars with its challenge u, for tests/test_batch_verify_model.py.  Field values cross
// this interface as 32-byte Montgomery-form integers; the verifier's scalars come back canonical, as the kernels read
// them.
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

// rho of a batch of n proofs under `version` from their u challenges (us: n x 32 bytes); out: rho, then w_0..w_{n-1}.
int bv_challenge(int version, const uint8_t* us, size_t n, uint8_t* out) {
  std::vector<HFr> u(n);
  for (size_t i = 0; i < n; i++) u[i] = load(us + 32 * i);
  const HFr rho = batch_challenge(version, u.data(), n);
  memcpy(out, rho.v, 32);
  const std::vector<HFr> w = batch_weights(rho, n);
  for (size_t i = 0; i < n; i++) memcpy(out + 32 * (i + 1), w[i].v, 32);
  return 0;
}

// verify_scalars for one proof under `version`, as pv_scalars of plonk_versions.cpp, with its u (u_out, 32 bytes;
// left untouched when the proof stops before u).  Returns the status verify_scalars returns.
int bv_scalars(const uint8_t* label, size_t label_len, uint64_t constraints, const uint8_t* key_comms, uint64_t n,
               const uint8_t* group_gen, const uint8_t* pi_roots, const uint8_t* pi, size_t n_pi, const uint8_t* proof,
               int version, uint64_t* out, uint8_t* u_out) {
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
  HFr u;
  const int st = verify_scalars(K, version, proof, pv.data(), out, &u);
  if (st != PB200_ERR_POINT_MALFORMED) memcpy(u_out, u.v, 32);
  return st;
}
}
