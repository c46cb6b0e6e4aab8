// include/plonk_b200.hpp's Verifier::batch_verify end to end.  Reads the case file of verifier_check.cpp (little-endian
// u64 fields): label length, constraints, public-input count, proof count, then the label, 15 x 48 commitment bytes,
// the 240-byte opening key, the public-input positions, the proofs (1008 bytes each) and their public inputs (32 bytes
// each, Montgomery).  The proofs are two valid V3 proofs, one that fails the check and one that is malformed.  Prints
// one line per check; the Python side compares them with what the reference would return.
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

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  std::ifstream f(argv[1], std::ios::binary);
  std::vector<uint8_t> b((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  size_t at = 0;
  auto u64 = [&]() { uint64_t x; memcpy(&x, b.data() + at, 8); at += 8; return x; };
  const uint64_t label_len = u64(), constraints = u64(), n_pi = u64(), n_proofs = u64();
  if (n_proofs != 4) return 2;
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
  std::vector<std::array<uint8_t, Verifier::PROOF_SIZE>> proofs(n_proofs);
  for (auto& p : proofs) {
    memcpy(p.data(), b.data() + at, p.size());
    at += p.size();
  }
  std::vector<std::vector<BlsScalar>> pis(n_proofs, std::vector<BlsScalar>(n_pi));
  for (auto& v : pis)
    for (auto& s : v) {
      memcpy(s.data(), b.data() + at, 32);
      at += 32;
    }
  auto attempt = [](const char* what, auto fn) {
    try {
      fn();
      printf("%s ok\n", what);
    } catch (const Error& e) {
      printf("%s %s\n", what, kind(e));
    }
  };
  using Proofs = std::vector<std::array<uint8_t, Verifier::PROOF_SIZE>>;
  using Inputs = std::vector<std::vector<BlsScalar>>;
  const Proofs good = {proofs[0], proofs[1]};
  const Inputs good_pi = {pis[0], pis[1]};
  Verifier v(label, constraints, comms, okey, pi_idx);
  attempt("valid", [&] { v.batch_verify(good, good_pi); });
  attempt("valid_v3", [&] { v.batch_verify(good, good_pi, PlonkVersion::V3); });
  attempt("valid_under_v2", [&] { v.batch_verify(good, good_pi, PlonkVersion::V2); });
  attempt("one_bad", [&] { v.batch_verify({proofs[0], proofs[2], proofs[1]}, {pis[0], pis[2], pis[1]}); });
  attempt("bad_and_malformed", [&] { v.batch_verify(proofs, pis); });
  attempt("empty", [&] { v.batch_verify({}, {}); });
  attempt("wrong_pi_count", [&] { v.batch_verify(good, Inputs(2, std::vector<BlsScalar>(n_pi + 1))); });
  attempt("unknown_version", [&] { v.batch_verify(good, good_pi, (PlonkVersion)4); });
  const std::vector<uint8_t> bytes = v.to_bytes();
  std::unique_ptr<Verifier> w = Verifier::try_from_bytes(bytes.data(), bytes.size());
  attempt("from_bytes_valid", [&] { w->batch_verify(good, good_pi); });
  attempt("from_bytes_empty", [&] { w->batch_verify({}, {}); });
  return 0;
}
