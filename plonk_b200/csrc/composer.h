// Host-side circuit front end of libplonk_b200: the reference's turbo Composer with the gadget
// library that benches/plonk.rs::BenchCircuit drives.  Circuit construction is CPU work in the
// reference too (O(gates), outside the GPU hot path); it lives here so that a C++ / Python caller of
// the device prover can describe the reference's own benchmark circuit without a Rust toolchain.
//
//   Composer core        src/composer.rs:72-495
//   Constraint           src/composer/constraint_system/constraint.rs:97-230
//   bits / range / logic / truncate / select / point / fixed_base gadgets
//                        src/composer/{bits,range,logic,truncate,select,point,fixed_base}.rs
//   JubJub               dusk-jubjub 0.15 (un-vendored): twisted Edwards -u^2 + v^2 = 1 + d u^2 v^2
//                        over BLS12-381's Fr, d = -(10240/10241); constants pinned by the reference's
//                        gate-layout goldens (tests/test_gadgets.py)
//
// Product code, independent of oracle/.
#pragma once
#include <stdint.h>

#include <array>
#include <map>
#include <string>
#include <vector>

#include "host_field.h"

namespace pbc {

using Fr = pbh::HFr;  // Montgomery form, 4 x u64: the reference's in-memory BlsScalar
typedef uint32_t Witness;

struct ComposerError {
  int code;
  std::string what;
};

enum Selector {
  Q_M = 0, Q_L, Q_R, Q_O, Q_F, Q_C, Q_ARITH, Q_RANGE, Q_LOGIC, Q_FIXED_GROUP_ADD, Q_VARIABLE_GROUP_ADD, N_SELECTORS
};

Fr fr_u64(uint64_t x);
Fr fr_pow2(unsigned k);
void fr_to_bits(const Fr& v, uint8_t bits[256]);  // BlsScalar::to_bits, least significant first
Fr fr_recompose(const uint8_t bits[256], int start, int end);

// ---- JubJub, affine (u, v) ------------------------------------------------------------------
struct JubJubAffine {
  Fr u, v;
  bool operator==(const JubJubAffine& o) const { return u == o.u && v == o.v; }
};
JubJubAffine jj_identity();
JubJubAffine jj_generator();                      // dusk_jubjub::GENERATOR
JubJubAffine jj_add(const JubJubAffine& p, const JubJubAffine& q);
JubJubAffine jj_neg(const JubJubAffine& p);
JubJubAffine jj_mul(const JubJubAffine& p, const uint64_t k[4]);  // canonical little-endian scalar
bool jj_is_on_curve(const JubJubAffine& p);
bool jj_is_torsion_free(const JubJubAffine& p);
using pbh::edwards_d;
extern const uint64_t kJubJubOrder[4];

// One width-4 gate being built: selector coefficients, optional public input, four wires.
struct Constraint {
  Fr q[N_SELECTORS];
  Fr pi;
  bool has_pi = false;
  Witness w[4] = {0, 0, 0, 0};  // a, b, c, d; default Composer::ZERO

  Constraint();
  Constraint& set(Selector s, const Fr& v) { q[s] = v; return *this; }
  Constraint& mult(const Fr& v) { return set(Q_M, v); }
  Constraint& left(const Fr& v) { return set(Q_L, v); }
  Constraint& right(const Fr& v) { return set(Q_R, v); }
  Constraint& output(const Fr& v) { return set(Q_O, v); }
  Constraint& fourth(const Fr& v) { return set(Q_F, v); }
  Constraint& constant(const Fr& v) { return set(Q_C, v); }
  Constraint& pub(const Fr& v) { pi = v; has_pi = true; return *this; }
  Constraint& a(Witness x) { w[0] = x; return *this; }
  Constraint& b(Witness x) { w[1] = x; return *this; }
  Constraint& c(Witness x) { w[2] = x; return *this; }
  Constraint& d(Witness x) { w[3] = x; return *this; }
};

struct Gate {
  Fr q[N_SELECTORS];
  Witness w[4];
};

struct WitnessPoint {
  Witness x, y;
};

class Composer {
 public:
  static constexpr Witness ZERO = 0, ONE = 1;
  static constexpr WitnessPoint IDENTITY = {0, 1};

  Composer();  // Composer::initialized: constants 0, 1 and the two dummy gates

  size_t constraints() const { return n_gates_; }
  // Witness-only mode (the composer of Prover::prove, src/compiler/prover.rs:425: the circuit is re-run for
  // its witness values and public inputs; the gate layout is the one the prover was compiled from): gates
  // are validated and counted but not stored.
  void set_witness_only(bool on);
  bool witness_only() const { return witness_only_; }
  size_t n_witnesses() const { return witnesses_.size(); }
  const Fr& operator[](Witness w) const;
  const std::vector<Gate>& gates() const { return gates_; }
  const std::vector<Fr>& witnesses() const { return witnesses_; }
  const std::map<size_t, Fr>& public_inputs() const { return public_inputs_; }

  // core (composer.rs)
  Witness append_witness(const Fr& v);
  void append_custom_gate(const Constraint& c);
  void append_gate(Constraint c);                       // + q_arith = 1
  bool append_evaluated_output(Constraint c, Witness* out);
  Witness append_constant(const Fr& v);
  Witness append_public(const Fr& v);
  void assert_equal(Witness a, Witness b);
  void assert_equal_constant(Witness a, const Fr& constant, const Fr* pi = nullptr);
  Witness gate_add(Constraint c);
  Witness gate_mul(Constraint c);

  // bits.rs
  void component_boolean(Witness a);
  std::vector<Witness> component_decomposition(Witness scalar, unsigned n);
  // range.rs
  void component_range_bits(Witness w, unsigned bits);
  void component_range(Witness w, unsigned bit_pairs);
  // logic.rs
  Witness append_logic_and(Witness a, Witness b, unsigned bit_pairs);
  Witness append_logic_xor(Witness a, Witness b, unsigned bit_pairs);
  // truncate.rs
  Witness component_truncate(Witness w, unsigned n);
  // select.rs
  Witness component_select(Witness bit, Witness a, Witness b);
  Witness component_select_one(Witness bit, Witness value);
  Witness component_select_zero(Witness bit, Witness value);
  // point.rs
  WitnessPoint append_point(const JubJubAffine& p);
  WitnessPoint append_constant_point(const JubJubAffine& p);
  WitnessPoint append_public_point(const JubJubAffine& p);
  void assert_equal_point(WitnessPoint a, WitnessPoint b);
  void assert_equal_public_point(WitnessPoint p, const JubJubAffine& pub);
  WitnessPoint assert_torsion_free_point(WitnessPoint p);
  WitnessPoint component_neg_point(WitnessPoint p);
  WitnessPoint component_sub_point(WitnessPoint a, WitnessPoint b);
  WitnessPoint component_add_point(WitnessPoint a, WitnessPoint b);
  WitnessPoint component_select_identity(Witness bit, WitnessPoint a);
  WitnessPoint component_select_point(Witness bit, WitnessPoint a, WitnessPoint b);
  WitnessPoint component_mul_point(Witness jubjub, WitnessPoint p);
  // fixed_base.rs
  WitnessPoint component_mul_generator(Witness jubjub, const JubJubAffine& generator);

  // benches/plonk.rs:12-82 with the Default values
  void bench_circuit(size_t degree);

 private:
  std::vector<Gate> gates_;
  size_t n_gates_ = 0;
  bool witness_only_ = false;
  std::vector<Fr> witnesses_;
  std::map<size_t, Fr> public_inputs_;

  void append_gate_inplace(Constraint& c);
  bool evaluated_output_inplace(Constraint& c, Witness* out);
  Witness logic_component(Witness a, Witness b, unsigned bit_pairs, bool is_xor);
  void range_check(Witness value, unsigned num_bits);
  void range_check_even(Witness value, unsigned num_bits);
  void bind_truncation_split(Witness input, Witness low, unsigned num_bits);
  void assert_canonical_truncation(Witness high, Witness low, unsigned num_bits);
  void assert_canonical_jubjub_scalar(Witness scalar);
  WitnessPoint add_point_gates(WitnessPoint a, WitnessPoint b);
  WitnessPoint add_point_gates(WitnessPoint a, WitnessPoint b, const JubJubAffine& sum);
  WitnessPoint select_identity_gates(Witness bit, WitnessPoint a);
  JubJubAffine point_value(WitnessPoint p) const;
};

}  // namespace pbc
