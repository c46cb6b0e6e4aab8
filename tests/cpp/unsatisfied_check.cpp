// include/plonk_b200.hpp's debugger check: the reference's examples/circuit.rs built with a witness that breaks one
// range gate, checked as a Composer (plonk_b200::unsatisfied_constraints / unsatisfied_report) and against the compiled
// Prover (Prover::unsatisfied_constraints / unsatisfied_report), then the honest witness.  Prints one line per check; the
// Python side compares them with the model.
#include <cstdio>

#include "../../include/plonk_b200.hpp"

using namespace plonk_b200;

// examples/circuit.rs TestCircuit::circuit with main()'s values, a = `a_value`
static void test_circuit(Composer& composer, uint64_t a_value) {
  const JubJubAffine f = JubJubAffine::generator();
  const Witness a = composer.append_witness(scalar_from_u64(a_value));
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

static void print(const char* what, const Unsatisfied& u, const std::optional<std::string>& report) {
  printf("%s %zu", what, u.size());
  for (const auto& x : u) printf(" %llu:%s", (unsigned long long)x.first, x.second.c_str());
  printf("\n%s_report %s\n", what, report ? report->c_str() : "none");
}

int main() {
  const BlsScalar x = scalar_from_u64(0x1234567), gs = scalar_from_u64(0x7654321), hs = scalar_from_u64(0xABCDEF);
  auto pp = PublicParameters::setup(1 << 12, x, gs, hs);
  auto compiled = Compiler::compile_with_circuit(*pp, "debugger", [](Composer& c) { test_circuit(c, 31); });
  auto compressed = Compiler::compile_with_compressed(*pp, "debugger", compress([](Composer& c) { test_circuit(c, 31); }));
  for (uint64_t a : {64ull, 31ull}) {  // 64 does not fit in 6 bits
    Composer composer;
    test_circuit(composer, a);
    const Composer::Export w = composer.finish();
    print("composer", unsatisfied_constraints(composer), unsatisfied_report(composer));
    print("prover", compiled.first->unsatisfied_constraints(w.witnesses, w.pi_idx, w.pi_vals),
          compiled.first->unsatisfied_report(w.witnesses, w.pi_idx, w.pi_vals));
    print("compressed", compressed.first->unsatisfied_constraints(w.witnesses, w.pi_idx, w.pi_vals),
          compressed.first->unsatisfied_report(w.witnesses, w.pi_idx, w.pi_vals));
  }
  Composer composer;
  test_circuit(composer, 31);
  const Composer::Export w = composer.finish();
  try {
    std::vector<BlsScalar> short_table(w.witnesses.begin(), w.witnesses.end() - 1);
    compiled.first->unsatisfied_constraints(short_table, w.pi_idx, w.pi_vals);
    printf("short_witness_table ok\n");
  } catch (const Error& e) {
    printf("short_witness_table %s\n", e.kind == Error::InvalidArgument ? "InvalidArgument" : "other");
  }
  return 0;
}
