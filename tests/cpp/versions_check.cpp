// include/plonk_b200.hpp's PlonkVersion API end to end: Prover::prove_with_version, Verifier::verify_with_version
// and the versioned verify_batch.  Reads a case file (little-endian u64 fields): label length, constraints, witness
// count, public-input count, commit-key point count, then the label, the 11 selector columns (32-byte Montgomery
// Fr), the 4 wire columns (u32), the witnesses, the public-input positions (u64) and values, the commit key (96-byte
// raw points), the 15 x 48 verifier-key commitments, the 240-byte opening key, two sets of 14 blinders and a V1
// proof of the same witness.  Prints one line per check; the Python side compares them with what the reference
// would return.
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>

#include "../../include/plonk_b200.hpp"

using namespace plonk_b200;

static const char* kind(const Error& e) {
  switch (e.kind) {
    case Error::ProofVerificationError: return "ProofVerificationError";
    case Error::PointMalformed: return "PointMalformed";
    case Error::InvalidArgument: return "InvalidArgument";
    case Error::UnsupportedProvingVersion: return "UnsupportedProvingVersion";
    default: return "other";
  }
}

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  std::ifstream f(argv[1], std::ios::binary);
  std::vector<uint8_t> b((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  size_t at = 0;
  auto u64 = [&]() { uint64_t x; memcpy(&x, b.data() + at, 8); at += 8; return x; };
  auto take = [&](void* dst, size_t n) { memcpy(dst, b.data() + at, n); at += n; };
  const uint64_t label_len = u64(), constraints = u64(), n_witnesses = u64(), n_pi = u64(), n_srs = u64();
  const std::string label((const char*)b.data() + at, label_len);
  at += label_len;
  Circuit c;
  c.n_constraints = constraints;
  c.n_witnesses = n_witnesses;
  c.selectors.resize(11 * constraints);
  take(c.selectors.data(), 32 * c.selectors.size());
  c.wires.resize(4 * constraints);
  take(c.wires.data(), 4 * c.wires.size());
  std::vector<BlsScalar> witnesses(n_witnesses);
  take(witnesses.data(), 32 * n_witnesses);
  std::vector<uint64_t> pi_idx(n_pi);
  take(pi_idx.data(), 8 * n_pi);
  std::vector<BlsScalar> pi(n_pi);
  take(pi.data(), 32 * n_pi);
  std::vector<uint8_t> srs(96 * n_srs);
  take(srs.data(), srs.size());
  std::array<uint8_t, 15 * 48> comms;
  take(comms.data(), comms.size());
  std::array<uint8_t, Verifier::OPENING_KEY_SIZE> okey;
  take(okey.data(), okey.size());
  std::array<BlsScalar, 14> blinders[2];
  take(blinders[0].data(), 14 * 32);
  take(blinders[1].data(), 14 * 32);
  std::array<uint8_t, Verifier::PROOF_SIZE> v1;
  take(v1.data(), v1.size());

  auto attempt = [](const char* what, auto fn) {
    try {
      fn();
      printf("%s ok\n", what);
    } catch (const Error& e) {
      printf("%s %s\n", what, kind(e));
    }
  };
  Prover prover(label, c, srs.data(), n_srs);
  Verifier v(label, constraints, comms, okey, pi_idx);
  attempt("prove_v1", [&] { prover.prove_with_version(PlonkVersion::V1, witnesses, pi_idx, pi, blinders[0]); });
  attempt("prove_v0", [&] { prover.prove_with_version((PlonkVersion)0, witnesses, pi_idx, pi, blinders[0]); });
  const auto v2 = prover.prove_with_version(PlonkVersion::V2, witnesses, pi_idx, pi, blinders[0]);
  const auto v3 = prover.prove_with_version(PlonkVersion::V3, witnesses, pi_idx, pi, blinders[1]);
  attempt("v2_under_v2", [&] { v.verify_with_version(v2, pi, PlonkVersion::V2); });
  attempt("v2_under_v3", [&] { v.verify_with_version(v2, pi, PlonkVersion::V3); });
  attempt("v3_under_v3", [&] { v.verify_with_version(v3, pi, PlonkVersion::V3); });
  attempt("v3_under_v2", [&] { v.verify_with_version(v3, pi, PlonkVersion::V2); });
  attempt("v1_under_v1", [&] { v.verify_with_version(v1, pi, PlonkVersion::V1); });
  attempt("v1_under_v2", [&] { v.verify_with_version(v1, pi, PlonkVersion::V2); });
  attempt("v3_under_v1", [&] { v.verify_with_version(v3, pi, PlonkVersion::V1); });
  const std::vector<std::array<uint8_t, Verifier::PROOF_SIZE>> batch = {v1, v2, v3};
  const std::vector<std::vector<BlsScalar>> pis(3, pi);
  const std::pair<const char*, PlonkVersion> runs[3] = {{"batch_v1", PlonkVersion::V1}, {"batch_v2", PlonkVersion::V2}, {"batch_v3", PlonkVersion::V3}};
  for (const auto& r : runs) {
    printf("%s", r.first);
    for (int32_t s : v.verify_batch(batch, pis, r.second)) printf(" %d", s);
    printf("\n");
  }
  printf("batch_default");
  for (int32_t s : v.verify_batch(batch, pis)) printf(" %d", s);
  printf("\n");
  const std::vector<uint8_t> bytes = v.to_bytes();
  std::unique_ptr<Verifier> w = Verifier::try_from_bytes(bytes.data(), bytes.size());
  attempt("from_bytes_v1", [&] { w->verify_with_version(v1, pi, PlonkVersion::V1); });
  attempt("wrong_pi_count_v1", [&] { v.verify_with_version(v1, std::vector<BlsScalar>(n_pi + 1), PlonkVersion::V1); });
  return 0;
}
