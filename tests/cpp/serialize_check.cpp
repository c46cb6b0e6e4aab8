// include/plonk_b200.hpp's writers end to end: Prover::to_bytes / serialized_size / try_from_bytes and
// CommitKey::to_var_bytes / to_raw_var_bytes.  Reads a case file (little-endian u64 fields): label length,
// constraints, witness count, commit-key points, public-input count, then the label, 11 selector columns, 4 wire
// columns, the raw commit key, the witnesses, the public-input positions and values and 14 blinders.
// Prints one line per check; the Python side compares them with what its own mirror produces.
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>

#include "../../include/plonk_b200.hpp"

using namespace plonk_b200;

static uint64_t fnv1a(const std::vector<uint8_t>& b) {
  uint64_t h = 0xCBF29CE484222325ull;
  for (uint8_t x : b) h = (h ^ x) * 0x100000001B3ull;
  return h;
}

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  std::ifstream f(argv[1], std::ios::binary);
  std::vector<uint8_t> b((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  size_t at = 0;
  auto u64 = [&]() { uint64_t x; memcpy(&x, b.data() + at, 8); at += 8; return x; };
  auto take = [&](void* dst, size_t bytes) { memcpy(dst, b.data() + at, bytes); at += bytes; };
  const uint64_t label_len = u64(), constraints = u64(), n_witnesses = u64(), n_points = u64(), n_pi = u64();
  const std::string label((const char*)b.data() + at, label_len);
  at += label_len;
  Circuit c;
  c.n_constraints = constraints;
  c.n_witnesses = n_witnesses;
  c.selectors.resize(11 * constraints);
  c.wires.resize(4 * constraints);
  take(c.selectors.data(), 11 * constraints * 32);
  take(c.wires.data(), 4 * constraints * 4);
  std::vector<uint8_t> srs(n_points * 96);
  take(srs.data(), srs.size());
  std::vector<BlsScalar> witnesses(n_witnesses), pi_vals(n_pi);
  std::vector<uint64_t> pi_idx(n_pi);
  take(witnesses.data(), n_witnesses * 32);
  take(pi_idx.data(), n_pi * 8);
  take(pi_vals.data(), n_pi * 32);
  std::array<BlsScalar, 14> blinders;
  take(blinders.data(), 14 * 32);

  Prover p(label, c, srs.data(), n_points);
  const std::vector<uint8_t> bytes = p.to_bytes();
  printf("serialized_size %s\n", p.serialized_size() == bytes.size() ? "equal" : "differ");
  printf("prover %zu %016llx\n", bytes.size(), (unsigned long long)fnv1a(bytes));
  std::unique_ptr<Prover> q = Prover::try_from_bytes(bytes.data(), bytes.size(), c.wires, n_witnesses);
  printf("round_trip %s\n", q->to_bytes() == bytes ? "equal" : "differ");
  printf("proof %s\n", q->prove(witnesses, pi_idx, pi_vals, blinders) == p.prove(witnesses, pi_idx, pi_vals, blinders) ? "equal" : "differ");
  try {
    Prover::try_from_bytes(bytes.data(), bytes.size() - 1, c.wires, n_witnesses);
    printf("truncated ok\n");
  } catch (const Error& e) {
    printf("truncated %s\n", e.kind == Error::InvalidArgument ? "InvalidArgument" : "other");
  }

  CommitKey key(srs.data(), n_points);
  const std::vector<uint8_t> raw_var = key.to_raw_var_bytes(), var = key.to_var_bytes();
  printf("commit_key_raw %zu %016llx\n", raw_var.size(), (unsigned long long)fnv1a(raw_var));
  printf("commit_key_var %zu %016llx\n", var.size(), (unsigned long long)fnv1a(var));
  std::unique_ptr<CommitKey> back = CommitKey::from_raw_var_bytes(raw_var.data(), raw_var.size());
  printf("commit_key_round_trip %s\n", back->to_raw_var_bytes() == raw_var && back->to_var_bytes() == var ? "equal" : "differ");
  return 0;
}
