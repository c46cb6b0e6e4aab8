// include/plonk_b200.hpp's batch_verify_groups end to end.  Reads a case file (little-endian u64 fields): the circuit
// count, then per circuit its label length, constraints, public-input count and proof count, the label, 15 x 48
// commitment bytes, the 240-byte opening key, the public-input positions, the proofs (1008 bytes each, valid V3 proofs)
// and their public inputs (32 bytes each, Montgomery).  Every circuit is on one SRS.  Prints one line per check; the
// Python side compares them with what the reference would return.
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
    default: return "other";
  }
}

using Proofs = std::vector<std::array<uint8_t, Verifier::PROOF_SIZE>>;
using Inputs = std::vector<std::vector<BlsScalar>>;

struct Case {
  std::unique_ptr<Verifier> v;
  Proofs proofs;
  Inputs pis;
};

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  std::ifstream f(argv[1], std::ios::binary);
  std::vector<uint8_t> b((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  size_t at = 0;
  auto u64 = [&]() { uint64_t x; memcpy(&x, b.data() + at, 8); at += 8; return x; };
  const uint64_t n_circuits = u64();
  if (n_circuits != 2) return 2;
  std::vector<Case> cs(n_circuits);
  for (Case& c : cs) {
    const uint64_t label_len = u64(), constraints = u64(), n_pi = u64(), n_proofs = u64();
    if (n_proofs != 2) return 2;
    const std::string label((const char*)b.data() + at, label_len);
    at += label_len;
    std::array<uint8_t, 15 * 48> comms;
    memcpy(comms.data(), b.data() + at, comms.size());
    at += comms.size();
    std::array<uint8_t, Verifier::OPENING_KEY_SIZE> okey;
    memcpy(okey.data(), b.data() + at, okey.size());
    at += okey.size();
    std::vector<uint64_t> pi_idx(n_pi);
    for (auto& x : pi_idx) x = u64();
    c.proofs.resize(n_proofs);
    for (auto& p : c.proofs) {
      memcpy(p.data(), b.data() + at, p.size());
      at += p.size();
    }
    c.pis.assign(n_proofs, std::vector<BlsScalar>(n_pi));
    for (auto& v : c.pis)
      for (auto& s : v) {
        memcpy(s.data(), b.data() + at, 32);
        at += 32;
      }
    c.v.reset(new Verifier(label, constraints, comms, okey, pi_idx));
  }
  auto attempt = [](const char* what, auto fn) {
    try {
      fn();
      printf("%s ok\n", what);
    } catch (const Error& e) {
      printf("%s %s\n", what, kind(e));
    }
  };
  const Case &A = cs[0], &B = cs[1];
  Proofs bad = A.proofs, malformed = A.proofs;
  bad[1][528 + 40] ^= 1;                                  // an evaluation moved: still canonical, fails the check
  memset(malformed[0].data() + 528, 0xff, 32);            // an evaluation above r
  attempt("valid", [&] { batch_verify_groups({{*A.v, PlonkVersion::V3, A.proofs, A.pis}, {*B.v, PlonkVersion::V3, B.proofs, B.pis}}); });
  attempt("same_verifier_twice", [&] {
    batch_verify_groups({{*A.v, PlonkVersion::V3, A.proofs, A.pis}, {*B.v, PlonkVersion::V3, B.proofs, B.pis},
                         {*A.v, PlonkVersion::V3, {A.proofs[0]}, {A.pis[0]}}});
  });
  attempt("one_bad", [&] { batch_verify_groups({{*B.v, PlonkVersion::V3, B.proofs, B.pis}, {*A.v, PlonkVersion::V3, bad, A.pis}}); });
  attempt("bad_and_malformed", [&] {
    batch_verify_groups({{*A.v, PlonkVersion::V3, bad, A.pis}, {*B.v, PlonkVersion::V3, B.proofs, B.pis}, {*A.v, PlonkVersion::V3, malformed, A.pis}});
  });
  attempt("under_v2", [&] { batch_verify_groups({{*A.v, PlonkVersion::V3, A.proofs, A.pis}, {*B.v, PlonkVersion::V2, B.proofs, B.pis}}); });
  attempt("no_groups", [&] { batch_verify_groups({}); });
  attempt("all_empty", [&] { batch_verify_groups({{*A.v, PlonkVersion::V3, {}, {}}, {*B.v, PlonkVersion::V2, {}, {}}}); });
  attempt("empty_group", [&] {
    batch_verify_groups({{*A.v, PlonkVersion::V3, A.proofs, A.pis}, {*B.v, PlonkVersion::V1, {}, {}}, {*B.v, PlonkVersion::V3, B.proofs, B.pis}});
  });
  attempt("wrong_pi_count", [&] {
    batch_verify_groups({{*A.v, PlonkVersion::V3, A.proofs, A.pis}, {*B.v, PlonkVersion::V3, B.proofs, A.pis}});
  });
  attempt("unknown_version", [&] { batch_verify_groups({{*A.v, PlonkVersion::V3, A.proofs, A.pis}, {*B.v, (PlonkVersion)4, B.proofs, B.pis}}); });
  const std::vector<uint8_t> bytes = A.v->to_bytes();
  std::unique_ptr<Verifier> w = Verifier::try_from_bytes(bytes.data(), bytes.size());
  attempt("from_bytes_valid", [&] { batch_verify_groups({{*w, PlonkVersion::V3, A.proofs, A.pis}, {*B.v, PlonkVersion::V3, B.proofs, B.pis}}); });
  return 0;
}
