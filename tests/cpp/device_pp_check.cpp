// include/plonk_b200.hpp's DevicePublicParameters end to end: setup -> Compiler::compile_with_circuit -> prove ->
// verify through the device parameters, the same prover and verifier bytes as the host PublicParameters give, shared
// tables, Prover::try_from_bytes against the parameters, and the error kinds.  Prints one line per check; the Python
// side compares them.
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

static void require(bool ok, const char* what) {
  if (!ok) throw Error(Error::InvalidArgument, what);
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

int main() {
  const BlsScalar x = scalar_from_u64(0x1234567), gs = scalar_from_u64(0x7654321), hs = scalar_from_u64(0xABCDEF);
  std::unique_ptr<DevicePublicParameters> dpp;
  expect("setup", [&] { dpp = DevicePublicParameters::setup(1 << 12, x, gs, hs); });
  if (!dpp) return 1;
  const auto host = PublicParameters::setup(1 << 12, x, gs, hs);
  expect("to_host", [&] {
    const auto back = dpp->to_host();
    require(back->raw_points() == host->raw_points() && back->opening_key() == host->opening_key(), "setup differs");
  });
  auto compiled = Compiler::compile_with_circuit(*dpp, "transcript-arguments", test_circuit);
  Composer composer;
  test_circuit(composer);
  const Composer::Export w = composer.finish();
  std::array<BlsScalar, 14> blinders;
  for (size_t k = 0; k < blinders.size(); k++) blinders[k] = scalar_from_u64(1000 + k);
  const auto proof = compiled.first->prove(w.witnesses, w.pi_idx, w.pi_vals, blinders);
  expect("verify", [&] { compiled.second->verify(proof, w.pi_vals); });
  expect("same_as_host", [&] {
    auto h = Compiler::compile(*host, "transcript-arguments", composer);
    require(h.first->to_bytes() == compiled.first->to_bytes(), "prover bytes differ");
    require(h.second->to_bytes() == compiled.second->to_bytes(), "verifier bytes differ");
    require(h.first->prove(w.witnesses, w.pi_idx, w.pi_vals, blinders) == proof, "proofs differ");
  });
  expect("shared_tables", [&] {
    const auto before = dpp->tables();
    auto again = Compiler::compile(*dpp, "other-label", composer);
    const auto after = dpp->tables();
    require(before.monomial == 1 && before.lagrange == 1 && after.device_bytes == before.device_bytes, "tables not shared");
  });
  const std::vector<uint8_t> blob = compiled.first->to_bytes();
  expect("try_from_bytes", [&] {
    auto p = Prover::try_from_bytes(*dpp, blob.data(), blob.size(), w.wires, w.witnesses.size());
    require(p->to_bytes() == blob, "reloaded bytes differ");
    compiled.second->verify(p->prove(w.witnesses, w.pi_idx, w.pi_vals, blinders), w.pi_vals);
  });
  expect("try_from_bytes_other_pp", [&] {
    auto other = DevicePublicParameters::setup(1 << 12, gs, x, hs);
    Prover::try_from_bytes(*other, blob.data(), blob.size(), w.wires, w.witnesses.size());
  });
  expect("compressed", [&] {
    const std::vector<uint8_t> data = compress(test_circuit);
    auto c = Compiler::compile_with_compressed(*dpp, "transcript-arguments", data);
    require(c.first->to_bytes() == blob, "compressed prover differs");
  });

  expect("setup_degree_zero", [&] { DevicePublicParameters::setup(0, x, gs, hs); });
  expect("setup_zero_draw", [&] { DevicePublicParameters::setup(4, x, BlsScalar{0, 0, 0, 0}, hs); });
  const std::vector<uint8_t> bytes = host->to_var_bytes();
  expect("from_slice", [&] { require(DevicePublicParameters::from_slice(bytes.data(), bytes.size())->to_host()->raw_points() == host->raw_points(), "differs"); });
  expect("from_slice_short", [&] { DevicePublicParameters::from_slice(bytes.data(), DevicePublicParameters::OPENING_KEY_SIZE); });
  std::vector<uint8_t> bad = bytes;
  bad[0] = 0xc0;
  for (size_t k = 1; k < 48; k++) bad[k] = 0;
  expect("from_slice_identity_g", [&] { DevicePublicParameters::from_slice(bad.data(), bad.size()); });
  const std::vector<uint8_t> raw = host->to_raw_var_bytes();
  expect("from_slice_unchecked", [&] {
    require(DevicePublicParameters::from_slice_unchecked(raw.data(), raw.size())->to_host()->raw_points() == host->raw_points(), "differs");
  });
  const size_t n_trim = [&] {
    size_t n = 1;
    while (n < w.n_constraints + 6) n <<= 1;
    return n;
  }();
  expect("compile_small", [&] {
    auto small = DevicePublicParameters::setup(n_trim - 1, x, gs, hs);
    Compiler::compile(*small, "t", composer);
  });
  expect("compile_exact", [&] {
    auto exact = DevicePublicParameters::setup(n_trim, x, gs, hs);
    Compiler::compile(*exact, "t", composer);
  });
  return 0;
}
