// include/plonk_b200.hpp's compress and Compiler::compile_with_compressed end to end: the reference's examples/circuit.rs
// compressed, compiled from the bytes and compared with Compiler::compile (keys and proofs byte for byte), and the two
// error kinds.  Prints one line per check; the Python side compares them.
#include <cstdio>

#include "../../include/plonk_b200.hpp"

using namespace plonk_b200;

static const char* kind(const Error& e) {
  switch (e.kind) {
    case Error::ProofVerificationError: return "ProofVerificationError";
    case Error::InvalidCompressedCircuit: return "InvalidCompressedCircuit";
    case Error::BlsScalarMalformed: return "BlsScalarMalformed";
    case Error::InvalidArgument: return "InvalidArgument";
    default: return "other";
  }
}

template <class F>
static void expect(const char* what, F&& f) {
  try {
    f();
    printf("%s ok\n", what);
  } catch (const Error& e) {
    printf("%s %s\n", what, kind(e));
  }
}

// examples/circuit.rs TestCircuit::circuit with main()'s values
static void test_circuit(Composer& composer) {
  const JubJubAffine f = JubJubAffine::generator();
  const Witness a = composer.append_witness(scalar_from_u64(31));
  const Witness b = composer.append_witness(scalar_from_u64(0));
  const Witness d = composer.append_witness(scalar_from_u64(42));
  composer.component_range_bits<6>(a);
  composer.component_range_bits<4>(b);
  Witness result = composer.gate_add(Constraint().left(scalar_from_u64(1)).right(scalar_from_u64(1)).a(a).b(b).constant(scalar_from_u64(42)));
  const Witness c = composer.append_public(scalar_from_u64(73));
  composer.assert_equal(result, c);
  result = composer.gate_mul(Constraint().mult(scalar_from_u64(1)).a(a).b(b).fourth(scalar_from_u64(1)).d(d));
  composer.assert_equal_constant(result, scalar_from_u64(42));
  const Witness e = composer.append_witness(scalar_from_u64(1));
  composer.assert_equal_public_point(composer.component_mul_generator(e, f), f);
}

// One stored (uncompressed) raw-deflate block around `packed`: any inflater reads it.
static std::vector<uint8_t> stored_block(const std::vector<uint8_t>& packed) {
  const uint16_t n = (uint16_t)packed.size();
  std::vector<uint8_t> out = {0x01, (uint8_t)n, (uint8_t)(n >> 8), (uint8_t)~n, (uint8_t)(~n >> 8)};
  out.insert(out.end(), packed.begin(), packed.end());
  return out;
}

int main() {
  const BlsScalar x = scalar_from_u64(0x1234567), gs = scalar_from_u64(0x7654321), hs = scalar_from_u64(0xABCDEF);
  auto pp = PublicParameters::setup(1 << 12, x, gs, hs);
  const std::vector<uint8_t> bytes = compress(test_circuit);
  auto direct = Compiler::compile_with_circuit(*pp, "transcript-arguments", test_circuit);
  auto compiled = Compiler::compile_with_compressed(*pp, "transcript-arguments", bytes);
  printf("prover_bytes %s\n", compiled.first->to_bytes() == direct.first->to_bytes() ? "equal" : "differ");
  printf("verifier_bytes %s\n", compiled.second->to_bytes() == direct.second->to_bytes() ? "equal" : "differ");
  Composer composer;
  test_circuit(composer);
  const Composer::Export w = composer.finish();
  std::array<BlsScalar, 14> blinders;
  for (size_t k = 0; k < blinders.size(); k++) blinders[k] = scalar_from_u64(1000 + k);
  const auto proof = compiled.first->prove(w.witnesses, w.pi_idx, w.pi_vals, blinders);
  printf("proof %s\n", proof == direct.first->prove(w.witnesses, w.pi_idx, w.pi_vals, blinders) ? "equal" : "differ");
  expect("verify", [&] { compiled.second->verify(proof, w.pi_vals); });
  std::vector<BlsScalar> wrong = w.pi_vals;
  wrong[0] = scalar_from_u64(74);
  expect("verify_wrong_pi", [&] { compiled.second->verify(proof, wrong); });

  expect("garbage", [&] { Compiler::compile_with_compressed(*pp, "t", std::vector<uint8_t>{0x00, 0x01, 0x02}); });
  expect("small_parameters", [&] {
    auto small = PublicParameters::setup(1 << 6, x, gs, hs);
    Compiler::compile_with_compressed(*small, "t", bytes);
  });
  // one gate, public input 0, one witness and one serialized scalar of 32 bytes 0xff (above r)
  std::vector<uint8_t> packed = {0xc2, 0x91, 0x00, 0x01, 0x91};
  for (int k = 0; k < 32; k++) packed.insert(packed.end(), {0xcc, 0xff});
  packed.push_back(0x91);
  packed.insert(packed.end(), 11, 0x00);
  packed.push_back(0x91);
  packed.insert(packed.end(), 5, 0x00);
  expect("non_canonical_scalar", [&] { Compiler::compile_with_compressed(*pp, "t", stored_block(packed)); });
  packed.back() = 0x01;  // witness index 1 of 1: index validation comes first
  expect("bad_witness_index", [&] { Compiler::compile_with_compressed(*pp, "t", stored_block(packed)); });
  return 0;
}
