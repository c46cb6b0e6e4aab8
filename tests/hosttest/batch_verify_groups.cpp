// Host build (g++) of the grouped batch challenge of plonk_b200/csrc/verify_scalars.h, for
// tests/test_batch_verify_groups_model.py.  Field values cross this interface as 32-byte Montgomery-form integers.
#include <stddef.h>
#include <string.h>

#include "../../plonk_b200/csrc/host_field.cpp"
#include "../../plonk_b200/csrc/verify_scalars.h"

using namespace pb;
using pbh::HFr;

extern "C" {

// rho of a call over n_groups groups (group g: lens[g] proofs under versions[g]) from every group's u challenges in
// call order (us: N x 32 bytes, N = sum lens); out: rho, then w_0..w_{N-1}.
int bvg_challenge(const int* versions, const size_t* lens, size_t n_groups, const uint8_t* us, uint8_t* out) {
  size_t n = 0;
  for (size_t g = 0; g < n_groups; g++) n += lens[g];
  std::vector<HFr> u(n);
  for (size_t i = 0; i < n; i++) memcpy(u[i].v, us + 32 * i, 32);
  const HFr rho = batch_challenge(versions, lens, n_groups, u.data());
  memcpy(out, rho.v, 32);
  const std::vector<HFr> w = batch_weights(rho, n);
  for (size_t i = 0; i < n; i++) memcpy(out + 32 * (i + 1), w[i].v, 32);
  return 0;
}

// The one-group form, batch_challenge(version, us, n): rho only.
int bvg_challenge_one(int version, const uint8_t* us, size_t n, uint8_t* out) {
  std::vector<HFr> u(n);
  for (size_t i = 0; i < n; i++) memcpy(u[i].v, us + 32 * i, 32);
  const HFr rho = batch_challenge(version, u.data(), n);
  memcpy(out, rho.v, 32);
  return 0;
}
}
