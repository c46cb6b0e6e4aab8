// include/plonk_b200.hpp's PublicParameters and Compiler end to end: the reference's examples/circuit.rs (setup,
// Compiler::compile_with_circuit, prove, verify) and the error kinds of setup, from_slice and compile.  Prints one line
// per check; the Python side compares them with what the reference returns.
#include <cstdio>

#include "../../include/plonk_b200.hpp"

using namespace plonk_b200;

static const char* kind(const Error& e) {
  switch (e.kind) {
    case Error::ProofVerificationError: return "ProofVerificationError";
    case Error::PointMalformed: return "PointMalformed";
    case Error::InvalidArgument: return "InvalidArgument";
    case Error::DegreeIsZero: return "DegreeIsZero";
    case Error::NotEnoughBytes: return "NotEnoughBytes";
    case Error::TruncatedDegreeTooLarge: return "TruncatedDegreeTooLarge";
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

// examples/circuit.rs TestCircuit::circuit with main()'s values (c = 73 is the public input under test)
static void test_circuit(Composer& composer, uint64_t c_value) {
  const JubJubAffine f = JubJubAffine::generator();
  const Witness a = composer.append_witness(scalar_from_u64(31));
  const Witness b = composer.append_witness(scalar_from_u64(0));
  const Witness d = composer.append_witness(scalar_from_u64(42));
  composer.component_range_bits<6>(a);
  composer.component_range_bits<4>(b);
  Witness result = composer.gate_add(Constraint().left(scalar_from_u64(1)).right(scalar_from_u64(1)).a(a).b(b).constant(scalar_from_u64(42)));
  const Witness c = composer.append_public(scalar_from_u64(c_value));
  composer.assert_equal(result, c);
  result = composer.gate_mul(Constraint().mult(scalar_from_u64(1)).a(a).b(b).fourth(scalar_from_u64(1)).d(d));
  composer.assert_equal_constant(result, scalar_from_u64(42));
  const Witness e = composer.append_witness(scalar_from_u64(1));
  composer.assert_equal_public_point(composer.component_mul_generator(e, f), f);
}

int main() {
  const BlsScalar x = scalar_from_u64(0x1234567), gs = scalar_from_u64(0x7654321), hs = scalar_from_u64(0xABCDEF);
  std::unique_ptr<PublicParameters> pp;
  expect("setup", [&] { pp = PublicParameters::setup(1 << 12, x, gs, hs); });
  if (!pp) return 1;
  auto compiled = Compiler::compile_with_circuit(*pp, "transcript-arguments", [](Composer& c) { test_circuit(c, 73); });
  Composer composer;
  test_circuit(composer, 73);
  const Composer::Export w = composer.finish();
  std::array<BlsScalar, 14> blinders;
  for (size_t k = 0; k < blinders.size(); k++) blinders[k] = scalar_from_u64(1000 + k);
  const auto proof = compiled.first->prove(w.witnesses, w.pi_idx, w.pi_vals, blinders);
  expect("verify", [&] { compiled.second->verify(proof, w.pi_vals); });
  std::vector<BlsScalar> wrong = w.pi_vals;
  wrong[0] = scalar_from_u64(74);
  expect("verify_wrong_pi", [&] { compiled.second->verify(proof, wrong); });

  expect("setup_degree_zero", [&] { PublicParameters::setup(0, x, gs, hs); });
  expect("setup_zero_draw", [&] { PublicParameters::setup(4, x, BlsScalar{0, 0, 0, 0}, hs); });
  std::vector<uint8_t> bytes = pp->to_var_bytes();
  expect("from_slice", [&] { PublicParameters::from_slice(bytes.data(), bytes.size()); });
  expect("from_slice_short", [&] { PublicParameters::from_slice(bytes.data(), PublicParameters::OPENING_KEY_SIZE); });
  std::vector<uint8_t> bad = bytes;
  bad[0] = 0xc0;
  for (size_t k = 1; k < 48; k++) bad[k] = 0;
  expect("from_slice_identity_g", [&] { PublicParameters::from_slice(bad.data(), bad.size()); });
  std::vector<uint8_t> raw = pp->to_raw_var_bytes();
  expect("from_slice_unchecked", [&] {
    if (PublicParameters::from_slice_unchecked(raw.data(), raw.size())->raw_points() != pp->raw_points()) throw Error(Error::InvalidArgument, "differs");
  });
  // next_pow2(constraints + 6) = n: max_degree n + 5 is too small, n + 6 compiles
  const size_t n_trim = [&] {
    size_t n = 1;
    while (n < w.n_constraints + 6) n <<= 1;
    return n;
  }();
  expect("compile_small", [&] {
    auto small = PublicParameters::setup(n_trim - 1, x, gs, hs);
    Compiler::compile(*small, "t", composer);
  });
  expect("compile_exact", [&] {
    auto exact = PublicParameters::setup(n_trim, x, gs, hs);
    Compiler::compile(*exact, "t", composer);
  });
  return 0;
}
