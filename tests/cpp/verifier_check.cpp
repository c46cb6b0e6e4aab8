// include/plonk_b200.hpp's Verifier end to end.  Reads a case file (little-endian u64 fields): label length,
// constraints, public-input count, proof count, then the label, 15 x 48 commitment bytes, the 240-byte opening key,
// the public-input positions, the proofs (1008 bytes each) and their public inputs (32 bytes each, Montgomery).
// Prints one line per check; the Python side compares them with what the reference would return.
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
    case Error::InvalidEvalDomainSize: return "InvalidEvalDomainSize";
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
  Verifier v(label, constraints, comms, okey, pi_idx);
  for (size_t i = 0; i < n_proofs; i++) attempt("verify", [&] { v.verify(proofs[i], pis[i]); });
  const std::vector<int32_t> st = v.verify_batch(proofs, pis);
  printf("batch");
  for (int32_t s : st) printf(" %d", s);
  printf("\n");
  const std::vector<uint8_t> bytes = v.to_bytes();
  std::unique_ptr<Verifier> w = Verifier::try_from_bytes(bytes.data(), bytes.size());
  printf("round_trip %s\n", w->to_bytes() == bytes ? "equal" : "differ");
  attempt("from_bytes_verify", [&] { w->verify(proofs[0], pis[0]); });
  attempt("wrong_pi_count", [&] { v.verify(proofs[0], std::vector<BlsScalar>(n_pi + 1)); });
  attempt("truncated", [&] { Verifier::try_from_bytes(bytes.data(), bytes.size() - 1); });
  std::array<uint8_t, Verifier::OPENING_KEY_SIZE> bad = okey;
  memset(bad.data() + 48, 0, 96);
  bad[48] = 0xc0;  // h = the identity (tests/opening_key_validation.rs:61-81)
  attempt("identity_h", [&] { Verifier(label, constraints, comms, bad, pi_idx); });
  return 0;
}
