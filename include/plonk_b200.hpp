// C++ mirror of the reference's interface for the hot path, over the C ABI in plonk_b200.h.
//
// The reference is a compiled (Rust) crate; this header is the compiled-language host side a C++
// caller links against, with the reference's names, argument meaning and error behaviour:
//
//   plonk_b200::EvaluationDomain   src/fft/domain.rs:35-232      new / fft / ifft / coset_fft / coset_ifft
//   plonk_b200::CommitKey          src/commitment_scheme/kzg10/key.rs:36-41, 215-308, 362-388   commit, max_degree,
//                                                                                      to_var_bytes, to_raw_var_bytes
//   plonk_b200::Commitment         src/commitment_scheme/kzg10/commitment.rs:77-106    to_bytes (48 B)
//   plonk_b200::Prover             src/compiler/prover.rs:53-115, 212-413              prove, prove_with_version, to_bytes,
//                                                                                      serialized_size, try_from_bytes
//   plonk_b200::Verifier           src/compiler/verifier.rs:32-263                     verify, verify_with_version, to_bytes,
//                                                                                      try_from_bytes
//   plonk_b200::PlonkVersion       src/compiler.rs:22-42
//   plonk_b200::PublicParameters   src/commitment_scheme/kzg10/srs.rs:61-196           setup, from_slice, from_slice_unchecked,
//                                                                                      to_var_bytes, to_raw_var_bytes, max_degree
//   plonk_b200::DevicePublicParameters  the same PublicParameters resident on the GPU, with the MSM tables of the
//                                  provers compiled from it shared between them: setup, from_slice, from_slice_unchecked,
//                                  from_host, to_host, tables
//   plonk_b200::Compiler           src/compiler.rs:47-113, 116-461                     compile, compile_with_circuit,
//                                                                                      compile_with_compressed
//   plonk_b200::compress           src/composer/circuit.rs:28-45, src/composer/compress.rs:136-240   Circuit::compress
//   plonk_b200::unsatisfied_constraints / unsatisfied_report, Prover::unsatisfied_constraints / _report
//                                  src/debugger.rs:95-236 (the report without its "appended at" clause)
//   plonk_b200::Composer           src/composer.rs:72-495 + src/composer/{bits,range,logic,truncate,select,
//                                  point,fixed_base}.rs (host-side circuit front end, plonk_b200_composer.h)
//   plonk_b200::Error              src/error.rs:21-120 (the variants this path can produce)
//
// BlsScalar is the reference's in-memory layout: 4 x u64 little-endian limbs, Montgomery form.
// Infallible reference functions (the NTT family asserts/panics, domain.rs:394) throw
// BackendFailure on a device error - there is no CPU fallback.
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <stdexcept>
#include <memory>
#include <optional>
#include <string>
#include <utility>
#include <vector>

#include "plonk_b200.h"
#include "plonk_b200_composer.h"

namespace plonk_b200 {

using BlsScalar = std::array<uint64_t, 4>;

struct Error : std::runtime_error {
  enum Kind {
    InvalidEvalDomainSize, PolynomialDegreeTooLarge, CircuitUnsatisfied, InvalidArgument, BackendFailure,
    JubJubPointNotTorsionFree, JubJubGeneratorNotPrimeOrder, JubJubScalarMalformed,
    ProofVerificationError,    // Error::ProofVerificationError
    PointMalformed,            // Error::BytesError(dusk_bytes::Error::InvalidData) of the verifier's decoders
    UnsupportedProvingVersion, // Error::UnsupportedProvingVersion
    DegreeIsZero,              // Error::DegreeIsZero: PublicParameters::setup with max_degree = 0
    TruncatedDegreeTooLarge,   // Error::TruncatedDegreeTooLarge: Compiler::compile with too small public parameters
    NotEnoughBytes,            // Error::NotEnoughBytes: PublicParameters::from_slice of at most OpeningKey::SIZE bytes
    InvalidCompressedCircuit,  // Error::InvalidCompressedCircuit: Compiler::compile_with_compressed refuses the description
    BlsScalarMalformed         // Error::BlsScalarMalformed: a compressed circuit's scalar is not canonical
  };
  Kind kind;
  Error(Kind k, const std::string& what) : std::runtime_error(what), kind(k) {}
};

inline void check(int rc) {
  if (rc == PB200_OK) return;
  const std::string msg = pb200_last_error();
  switch (rc) {
    case PB200_ERR_INVALID_DOMAIN: throw Error(Error::InvalidEvalDomainSize, msg);
    case PB200_ERR_DEGREE_TOO_LARGE: throw Error(Error::PolynomialDegreeTooLarge, msg);
    case PB200_ERR_UNSATISFIED: throw Error(Error::CircuitUnsatisfied, msg);
    case PB200_ERR_INVALID_ARG: throw Error(Error::InvalidArgument, msg);
    case PB200_ERR_JUBJUB_POINT: throw Error(Error::JubJubPointNotTorsionFree, msg);
    case PB200_ERR_JUBJUB_GENERATOR: throw Error(Error::JubJubGeneratorNotPrimeOrder, msg);
    case PB200_ERR_JUBJUB_SCALAR: throw Error(Error::JubJubScalarMalformed, msg);
    case PB200_ERR_UNSUPPORTED_VERSION: throw Error(Error::UnsupportedProvingVersion, msg);
    case PB200_ERR_DEGREE_IS_ZERO: throw Error(Error::DegreeIsZero, msg);
    case PB200_ERR_INVALID_COMPRESSED: throw Error(Error::InvalidCompressedCircuit, msg);
    case PB200_ERR_SCALAR_MALFORMED: throw Error(Error::BlsScalarMalformed, msg);
    default: throw Error(Error::BackendFailure, msg);
  }
}

class EvaluationDomain {
 public:
  // EvaluationDomain::new(num_coeffs): size = next power of two; log size must stay below TWO_ADACITY = 32.
  explicit EvaluationDomain(size_t num_coeffs) {
    size_ = 1;
    log_ = 0;
    while (size_ < num_coeffs) {
      size_ <<= 1;
      log_++;
    }
    if (log_ >= 32) throw Error(Error::InvalidEvalDomainSize, "log_size_of_group >= TWO_ADACITY");
  }
  size_t size() const { return size_; }
  std::vector<BlsScalar> fft(const std::vector<BlsScalar>& coeffs) const { return run(coeffs, 0, 0); }
  std::vector<BlsScalar> ifft(const std::vector<BlsScalar>& evals) const { return run(evals, 1, 0); }
  std::vector<BlsScalar> coset_fft(const std::vector<BlsScalar>& coeffs) const { return run(coeffs, 0, 1); }
  std::vector<BlsScalar> coset_ifft(const std::vector<BlsScalar>& evals) const { return run(evals, 1, 1); }

 private:
  size_t size_;
  uint32_t log_;
  std::vector<BlsScalar> run(const std::vector<BlsScalar>& v, int inverse, int coset) const {
    std::vector<BlsScalar> out(size_);
    check(pb200_ntt(v.empty() ? nullptr : v[0].data(), v.size(), out[0].data(), log_, inverse, coset, 1, v.size(), size_));
    return out;
  }
};

struct Commitment {
  std::array<uint64_t, 12> raw{};  // x, y Montgomery limbs; identity = zeros
  std::array<uint8_t, 48> to_bytes() const {
    std::array<uint8_t, 48> b;
    check(pb200_g1_compress(raw.data(), b.data()));
    return b;
  }
  bool operator==(const Commitment& o) const { return raw == o.raw; }
};

class CommitKey {
 public:
  // powers_of_g as 96-byte raw points (CommitKey::to_raw_var_bytes without length prefix / flags)
  CommitKey(const uint8_t* raw_points, size_t n_points) : n_(n_points), raw_(raw_points, raw_points + 96 * n_points) {
    check(pb200_srs_upload(raw_points, n_points, &h_));
  }
  // CommitKey::to_var_bytes (key.rs:303-308): G1Affine::to_bytes per point, encoded on the GPU; what
  // CommitKey::from_slice reads
  std::vector<uint8_t> to_var_bytes() const {
    std::vector<uint8_t> out(48 * n_);
    check(pb200_g1_compress_batch(raw_.data(), n_, out.data()));
    return out;
  }
  // CommitKey::to_raw_var_bytes (key.rs:215-229): what from_raw_var_bytes and from_slice_unchecked read
  std::vector<uint8_t> to_raw_var_bytes() const {
    size_t n = 0;
    check(pb200_commit_key_to_raw_var_bytes(raw_.data(), n_, nullptr, 0, &n));
    std::vector<uint8_t> out(n);
    check(pb200_commit_key_to_raw_var_bytes(raw_.data(), n_, out.data(), out.size(), &n));
    return out;
  }
  // CommitKey::from_raw_var_bytes (key.rs:258-298: every point validated, on the GPU) and
  // CommitKey::from_slice_unchecked (key.rs:242-256: trusted bytes) for CommitKey::to_raw_var_bytes
  static std::unique_ptr<CommitKey> from_raw_var_bytes(const uint8_t* bytes, size_t len) { return from_raw(bytes, len, 1); }
  static std::unique_ptr<CommitKey> from_slice_unchecked(const uint8_t* bytes, size_t len) { return from_raw(bytes, len, 0); }
  ~CommitKey() { pb200_srs_free(h_); }
  CommitKey(const CommitKey&) = delete;
  CommitKey& operator=(const CommitKey&) = delete;
  size_t max_degree() const { return n_ - 1; }
  // CommitKey::commit: trailing zero coefficients are trimmed first (Polynomial::from_coefficients_vec),
  // then Error::PolynomialDegreeTooLarge if degree > max_degree.
  Commitment commit(std::vector<BlsScalar> polynomial) const {
    while (!polynomial.empty() && polynomial.back() == BlsScalar{0, 0, 0, 0}) polynomial.pop_back();
    const size_t degree = polynomial.empty() ? 0 : polynomial.size() - 1;
    if (degree > max_degree()) throw Error(Error::PolynomialDegreeTooLarge, "polynomial degree exceeds the commit key");
    Commitment c;
    check(pb200_msm_g1(h_, polynomial.empty() ? nullptr : polynomial[0].data(), polynomial.size(), 1, polynomial.size(), c.raw.data()));
    return c;
  }

 private:
  pb200_srs_t* h_ = nullptr;
  size_t n_;
  std::vector<uint8_t> raw_;  // the points the key was made from (96 bytes each), kept for the two writers
  static std::unique_ptr<CommitKey> from_raw(const uint8_t* bytes, size_t len, int checked) {
    size_t n = 0;
    check(pb200_raw_commit_key_points(bytes, len, checked, &n));
    std::vector<uint8_t> raw(n * 96 + 1);
    check(pb200_commit_key_from_raw_var_bytes(bytes, len, checked, raw.data()));
    return std::unique_ptr<CommitKey>(new CommitKey(raw.data(), n));
  }
};

// Flat circuit description (what Compiler::preprocess reads out of the Composer, compiler.rs:132-170)
struct Circuit {
  std::vector<BlsScalar> selectors;  // 11 columns x n_constraints, column-major (order of plonk_b200.h)
  std::vector<uint32_t> wires;       // 4 columns x n_constraints witness indices
  size_t n_constraints = 0;
  size_t n_witnesses = 0;
};

// ---- circuit front end ------------------------------------------------------------------------
typedef uint32_t Witness;
struct WitnessPoint {
  Witness x, y;
};
struct JubJubAffine {
  BlsScalar u, v;
  // dusk_jubjub::GENERATOR
  static JubJubAffine generator() {
    uint64_t uv[8];
    check(pb200_jubjub_generator(uv));
    return from_raw(uv);
  }
  // scalar: canonical little-endian limbs of a JubJubScalar
  JubJubAffine mul(const std::array<uint64_t, 4>& scalar) const {
    uint64_t in[8], out[8];
    to_raw(in);
    check(pb200_jubjub_mul(in, scalar.data(), out));
    return from_raw(out);
  }
  void to_raw(uint64_t uv[8]) const {
    for (int i = 0; i < 4; i++) uv[i] = u[i], uv[4 + i] = v[i];
  }
  static JubJubAffine from_raw(const uint64_t uv[8]) {
    JubJubAffine p;
    for (int i = 0; i < 4; i++) p.u[i] = uv[i], p.v[i] = uv[4 + i];
    return p;
  }
};

// One gate under construction (constraint.rs:97-230); coefficients default to zero, wires to
// Composer::ZERO.  Scalars are Montgomery-form BlsScalar values.
struct Constraint {
  std::array<BlsScalar, 11> q{};  // q_m, q_l, q_r, q_o, q_f, q_c, q_arith, q_range, q_logic, q_fixed_group_add, q_variable_group_add
  std::array<Witness, 4> w{};     // a, b, c, d
  BlsScalar pi{};
  bool has_pi = false;
  Constraint& mult(const BlsScalar& s) { q[0] = s; return *this; }
  Constraint& left(const BlsScalar& s) { q[1] = s; return *this; }
  Constraint& right(const BlsScalar& s) { q[2] = s; return *this; }
  Constraint& output(const BlsScalar& s) { q[3] = s; return *this; }
  Constraint& fourth(const BlsScalar& s) { q[4] = s; return *this; }
  Constraint& constant(const BlsScalar& s) { q[5] = s; return *this; }
  Constraint& pub(const BlsScalar& s) { pi = s; has_pi = true; return *this; }
  Constraint& a(Witness x) { w[0] = x; return *this; }
  Constraint& b(Witness x) { w[1] = x; return *this; }
  Constraint& c(Witness x) { w[2] = x; return *this; }
  Constraint& d(Witness x) { w[3] = x; return *this; }
};

// BlsScalar::from(u64), Montgomery form (x * 2^256 mod r computed by 256 modular doublings)
inline BlsScalar scalar_from_u64(uint64_t x) {
  static const uint64_t r[4] = {0xffffffff00000001ull, 0x53bda402fffe5bfeull, 0x3339d80809a1d805ull, 0x73eda753299d7d48ull};
  uint64_t v[4] = {x, 0, 0, 0};
  for (int k = 0; k < 256; k++) {
    const uint64_t top = v[3] >> 63;
    for (int i = 3; i > 0; i--) v[i] = (v[i] << 1) | (v[i - 1] >> 63);
    v[0] <<= 1;
    bool ge = top != 0;
    if (!ge) {
      ge = true;
      for (int i = 3; i >= 0; i--)
        if (v[i] != r[i]) { ge = v[i] > r[i]; break; }
    }
    if (ge) {
      unsigned __int128 borrow = 0;
      for (int i = 0; i < 4; i++) {
        const unsigned __int128 d = (unsigned __int128)v[i] - r[i] - borrow;
        v[i] = (uint64_t)d;
        borrow = (d >> 64) & 1;
      }
    }
  }
  return {v[0], v[1], v[2], v[3]};
}

class Composer {
 public:
  static constexpr Witness ZERO = 0, ONE = 1;
  static constexpr WitnessPoint IDENTITY = {0, 1};

  Composer() { check(pb200_composer_new(&h_)); }  // Composer::initialized()
  ~Composer() { pb200_composer_free(h_); }
  Composer(const Composer&) = delete;
  Composer& operator=(const Composer&) = delete;

  size_t constraints() const { return pb200_composer_constraints(h_); }
  BlsScalar operator[](Witness w) const { BlsScalar v; check(pb200_composer_witness_value(h_, w, v.data())); return v; }

  Witness append_witness(const BlsScalar& v) { Witness w; check(pb200_composer_append_witness(h_, v.data(), &w)); return w; }
  Witness append_witness(uint64_t v) { return append_witness(scalar_from_u64(v)); }
  void append_gate(const Constraint& c) { check(pb200_composer_append_gate(h_, c.q[0].data(), c.w.data(), c.has_pi ? c.pi.data() : nullptr, 0)); }
  void append_custom_gate(const Constraint& c) { check(pb200_composer_append_gate(h_, c.q[0].data(), c.w.data(), c.has_pi ? c.pi.data() : nullptr, 1)); }
  Witness gate_add(const Constraint& c) { Witness w; check(pb200_composer_gate_add(h_, c.q[0].data(), c.w.data(), c.has_pi ? c.pi.data() : nullptr, &w)); return w; }
  Witness gate_mul(const Constraint& c) { return gate_add(c); }
  Witness append_constant(const BlsScalar& v) { Witness w; check(pb200_composer_append_constant(h_, v.data(), &w)); return w; }
  Witness append_constant(uint64_t v) { return append_constant(scalar_from_u64(v)); }
  Witness append_public(const BlsScalar& v) { Witness w; check(pb200_composer_append_public(h_, v.data(), &w)); return w; }
  void assert_equal(Witness a, Witness b) { check(pb200_composer_assert_equal(h_, a, b)); }
  void assert_equal_constant(Witness a, const BlsScalar& constant, const BlsScalar* pi = nullptr) {
    check(pb200_composer_assert_equal_constant(h_, a, constant.data(), pi ? pi->data() : nullptr));
  }
  void component_boolean(Witness a) { check(pb200_composer_component_boolean(h_, a)); }
  template <size_t N>
  std::array<Witness, N> component_decomposition(Witness scalar) {
    std::array<Witness, N> bits;
    check(pb200_composer_component_decomposition(h_, scalar, (uint32_t)N, bits.data()));
    return bits;
  }
  template <size_t BITS>
  void component_range_bits(Witness w) { check(pb200_composer_component_range_bits(h_, w, (uint32_t)BITS)); }
  template <size_t BIT_PAIRS>
  Witness append_logic_and(Witness a, Witness b) { Witness w; check(pb200_composer_append_logic(h_, a, b, (uint32_t)BIT_PAIRS, 0, &w)); return w; }
  template <size_t BIT_PAIRS>
  Witness append_logic_xor(Witness a, Witness b) { Witness w; check(pb200_composer_append_logic(h_, a, b, (uint32_t)BIT_PAIRS, 1, &w)); return w; }
  template <size_t N>
  Witness component_truncate(Witness x) { Witness w; check(pb200_composer_component_truncate(h_, x, (uint32_t)N, &w)); return w; }
  Witness component_select(Witness bit, Witness a, Witness b) { Witness w; check(pb200_composer_component_select(h_, bit, a, b, &w)); return w; }
  Witness component_select_one(Witness bit, Witness v) { Witness w; check(pb200_composer_component_select_one(h_, bit, v, &w)); return w; }
  Witness component_select_zero(Witness bit, Witness v) { Witness w; check(pb200_composer_component_select_zero(h_, bit, v, &w)); return w; }

  WitnessPoint append_point(const JubJubAffine& p) { return point_in(p, 0); }
  WitnessPoint append_constant_point(const JubJubAffine& p) { return point_in(p, 1); }
  WitnessPoint append_public_point(const JubJubAffine& p) { return point_in(p, 2); }
  void assert_equal_point(WitnessPoint a, WitnessPoint b) { check(pb200_composer_assert_equal_point(h_, &a.x, &b.x)); }
  void assert_equal_public_point(WitnessPoint p, const JubJubAffine& pub) {
    uint64_t uv[8];
    pub.to_raw(uv);
    check(pb200_composer_assert_equal_public_point(h_, &p.x, uv));
  }
  WitnessPoint assert_torsion_free_point(WitnessPoint p) { check(pb200_composer_assert_torsion_free_point(h_, &p.x)); return p; }
  WitnessPoint component_add_point(WitnessPoint a, WitnessPoint b) { WitnessPoint r; check(pb200_composer_point_op(h_, PB200_POINT_ADD, &a.x, &b.x, &r.x)); return r; }
  WitnessPoint component_sub_point(WitnessPoint a, WitnessPoint b) { WitnessPoint r; check(pb200_composer_point_op(h_, PB200_POINT_SUB, &a.x, &b.x, &r.x)); return r; }
  WitnessPoint component_neg_point(WitnessPoint a) { WitnessPoint r; check(pb200_composer_point_op(h_, PB200_POINT_NEG, &a.x, nullptr, &r.x)); return r; }
  WitnessPoint component_select_identity(Witness bit, WitnessPoint a) { WitnessPoint r; check(pb200_composer_component_select_identity(h_, bit, &a.x, &r.x)); return r; }
  WitnessPoint component_select_point(Witness bit, WitnessPoint a, WitnessPoint b) { WitnessPoint r; check(pb200_composer_component_select_point(h_, bit, &a.x, &b.x, &r.x)); return r; }
  WitnessPoint component_mul_point(Witness jubjub, WitnessPoint p) { WitnessPoint r; check(pb200_composer_component_mul_point(h_, jubjub, &p.x, &r.x)); return r; }
  WitnessPoint component_mul_generator(Witness jubjub, const JubJubAffine& generator) {
    uint64_t uv[8];
    generator.to_raw(uv);
    WitnessPoint r;
    check(pb200_composer_component_mul_generator(h_, jubjub, uv, &r.x));
    return r;
  }

  // What Compiler::compile and Prover::prove read back from the composer.
  struct Export {
    std::vector<BlsScalar> selectors, witnesses, pi_vals;
    std::vector<uint32_t> wires;
    std::vector<uint64_t> pi_idx;
    size_t n_constraints = 0;
  };
  Export finish() const {
    Export e;
    e.n_constraints = constraints();
    const size_t n_w = pb200_composer_witnesses(h_), n_pi = pb200_composer_public_inputs(h_);
    e.selectors.resize(11 * e.n_constraints);
    e.wires.resize(4 * e.n_constraints);
    e.witnesses.resize(n_w);
    e.pi_idx.resize(n_pi);
    e.pi_vals.resize(n_pi);
    check(pb200_composer_export(h_, e.selectors[0].data(), e.wires.data(), e.witnesses[0].data(), e.pi_idx.data(),
                                n_pi ? e.pi_vals[0].data() : nullptr));
    return e;
  }

 private:
  pb200_composer_t* h_ = nullptr;
  WitnessPoint point_in(const JubJubAffine& p, int kind) {
    uint64_t uv[8];
    p.to_raw(uv);
    WitnessPoint r;
    check(pb200_composer_append_point(h_, uv, kind, &r.x));
    return r;
  }
};

inline Circuit circuit_of(const Composer::Export& e) {
  Circuit c;
  c.selectors = e.selectors;
  c.wires = e.wires;
  c.n_constraints = e.n_constraints;
  c.n_witnesses = e.witnesses.size();
  return c;
}

// ---- which constraint a witness breaks (the reference's debugger, src/debugger.rs:95-236) --------------------------
// A failing constraint and the name of the first of its 17 gate identities that is not zero (IDENTITY_FAMILIES).
using Unsatisfied = std::vector<std::pair<uint64_t, std::string>>;

namespace detail {
// call(cap, rows, families, &n): one of the C entry points with its circuit arguments bound.  Returns the failing count
// and the first min(cap, count) failing constraints.
template <class F>
inline std::pair<size_t, Unsatisfied> unsatisfied_query(F&& call, size_t cap) {
  std::vector<uint64_t> rows(cap);
  std::vector<int32_t> families(cap);
  size_t n = 0;
  check(call(cap, cap ? rows.data() : nullptr, cap ? families.data() : nullptr, &n));
  Unsatisfied out;
  for (size_t i = 0; i < std::min(cap, n); i++) out.emplace_back(rows[i], pb200_identity_family(families[i]));
  return {n, out};
}
// Debugger::unsatisfied_report without its "and was appended at path:line:col" clause (no call sites are recorded)
inline std::optional<std::string> unsatisfied_report(const std::pair<size_t, Unsatisfied>& q, size_t n_constraints) {
  if (q.first == 0) return std::nullopt;
  return "plonk debugger: " + std::to_string(q.first) + " of " + std::to_string(n_constraints) +
         " constraints are unsatisfied; the first, constraint " + std::to_string(q.second[0].first) + ", fails the " +
         q.second[0].second + " identity";
}
inline auto composer_call(const Composer::Export& e) {
  return [&e](size_t cap, uint64_t* rows, int32_t* families, size_t* n) {
    return pb200_circuit_unsatisfied(e.n_constraints, e.selectors.empty() ? nullptr : e.selectors[0].data(), e.wires.data(),
                                     e.witnesses.empty() ? nullptr : e.witnesses[0].data(), e.witnesses.size(), e.pi_idx.data(),
                                     e.pi_vals.empty() ? nullptr : e.pi_vals[0].data(), e.pi_idx.size(), cap, rows, families, n);
  };
}
}  // namespace detail

// The reference debugger's check of a filled composer (its constraints, witnesses and public inputs, as at prove time):
// every failing constraint in ascending order.
inline Unsatisfied unsatisfied_constraints(const Composer& composer) {
  const Composer::Export e = composer.finish();
  return detail::unsatisfied_query(detail::composer_call(e), e.n_constraints).second;
}
// Debugger::unsatisfied_report of a filled composer; nullopt when every constraint holds.
inline std::optional<std::string> unsatisfied_report(const Composer& composer) {
  const Composer::Export e = composer.finish();
  return detail::unsatisfied_report(detail::unsatisfied_query(detail::composer_call(e), 1), e.n_constraints);
}

// PlonkVersion (src/compiler.rs:22-42): V3 is the current profile; V2 is the legacy transcript seed with V3's opening
// checks; V1 is the legacy seed with the legacy opening, which does not bind the q_arith, q_c, q_l and q_r
// evaluations, so a V1 verdict is meaningful only for proofs made under the old rules.
enum class PlonkVersion { V1 = PB200_PLONK_V1, V2 = PB200_PLONK_V2, V3 = PB200_PLONK_V3 };

class DevicePublicParameters;

class Prover {
 public:
  static constexpr size_t PROOF_SIZE = 1008;  // Proof::SIZE
  Prover(const std::string& label, const Circuit& c, const uint8_t* srs_raw, size_t n_srs_points)
      : n_witnesses_(c.n_witnesses), n_constraints_(c.n_constraints) {
    check(pb200_prover_new((const uint8_t*)label.data(), label.size(), c.n_constraints, c.selectors[0].data(), c.wires.data(),
                           c.n_witnesses, srs_raw, n_srs_points, &h_));
  }
  // The same Prover with the commit-key tables of pp, shared with every other prover compiled from it
  inline Prover(const std::string& label, const Circuit& c, const DevicePublicParameters& pp);
  // try_from_bytes against pp: the serialized commit key must be a prefix of pp's points (else InvalidArgument), which
  // stands in for the per-point validation; the tables are pp's
  static inline std::unique_ptr<Prover> try_from_bytes(const DevicePublicParameters& pp, const uint8_t* bytes, size_t len,
                                                       const std::vector<uint32_t>& wires, size_t n_witnesses);
  // from_compressed with pp's points and tables
  static inline std::unique_ptr<Prover> from_compressed(const std::string& label, const std::vector<uint8_t>& compressed,
                                                        const DevicePublicParameters& pp, size_t n_witnesses);
  // Prover::try_from_bytes (prover.rs:265-350) for the bytes of Prover::to_bytes; the wiring of the circuit
  // (4 x constraints witness indices) is not part of that format and comes alongside
  static std::unique_ptr<Prover> try_from_bytes(const uint8_t* bytes, size_t len, const std::vector<uint32_t>& wires, size_t n_witnesses) {
    std::unique_ptr<Prover> p(new Prover());
    p->n_witnesses_ = n_witnesses;
    p->n_constraints_ = wires.size() / 4;
    check(pb200_prover_from_bytes(bytes, len, wires.data(), n_witnesses, &p->h_));
    return p;
  }
  // Compiler::compile_with_compressed's Prover (compiler.rs:84-112): the selector columns are expanded on the device;
  // prove takes the re-run circuit's witness table (n_witnesses entries, the description's count)
  static std::unique_ptr<Prover> from_compressed(const std::string& label, const std::vector<uint8_t>& compressed, const uint8_t* srs_raw,
                                                 size_t n_srs_points, size_t n_witnesses) {
    std::unique_ptr<Prover> p(new Prover());
    p->n_witnesses_ = n_witnesses;
    uint64_t described_witnesses = 0;
    size_t n_labels = 0, n_pi = 0;
    check(pb200_compressed_circuit_info(compressed.data(), compressed.size(), n_srs_points, &p->n_constraints_, &described_witnesses,
                                        &n_labels, &n_pi, nullptr));
    check(pb200_prover_from_compressed((const uint8_t*)label.data(), label.size(), compressed.data(), compressed.size(), srs_raw,
                                       n_srs_points, &p->h_));
    return p;
  }
  // Prover::serialized_size (prover.rs:233-235) and Prover::to_bytes (:238-263): the bytes try_from_bytes reads
  size_t serialized_size() const {
    size_t n = 0;
    check(pb200_prover_to_bytes(h_, nullptr, 0, &n));
    return n;
  }
  std::vector<uint8_t> to_bytes() const {
    size_t n = serialized_size();
    std::vector<uint8_t> out(n);
    check(pb200_prover_to_bytes(h_, out.data(), out.size(), &n));
    return out;
  }
  ~Prover() { pb200_prover_free(h_); }
  const pb200_prover_t* handle() const { return h_; }
  Prover(const Prover&) = delete;
  Prover& operator=(const Prover&) = delete;
  // Prover::prove: `blinders` are the 14 BlsScalar::random draws of prove_inner, in its order.
  std::array<uint8_t, PROOF_SIZE> prove(const std::vector<BlsScalar>& witnesses, const std::vector<uint64_t>& pi_idx,
                                        const std::vector<BlsScalar>& pi_vals, const std::array<BlsScalar, 14>& blinders) const {
    std::array<uint8_t, PROOF_SIZE> proof;
    check(pb200_prove(h_, witnesses[0].data(), witnesses.size(), pi_idx.data(), pi_vals.empty() ? nullptr : pi_vals[0].data(),
                      pi_idx.size(), blinders[0].data(), proof.data()));
    return proof;
  }
  // Prover::prove_with_version: V3 is prove, V2 proves under the legacy transcript seed, V1 throws
  // UnsupportedProvingVersion.
  std::array<uint8_t, PROOF_SIZE> prove_with_version(PlonkVersion version, const std::vector<BlsScalar>& witnesses,
                                                     const std::vector<uint64_t>& pi_idx, const std::vector<BlsScalar>& pi_vals,
                                                     const std::array<BlsScalar, 14>& blinders) const {
    std::array<uint8_t, PROOF_SIZE> proof;
    check(pb200_prove_with_version(h_, (int)version, witnesses[0].data(), witnesses.size(), pi_idx.data(),
                                   pi_vals.empty() ? nullptr : pi_vals[0].data(), pi_idx.size(), blinders[0].data(), proof.data()));
    return proof;
  }
  // The reference debugger's check (debugger.rs:95-205) against this prover's own selectors, with prove's arguments:
  // every failing constraint in ascending order.  Empty means prove makes the proof.  Safe beside proofs on this prover.
  Unsatisfied unsatisfied_constraints(const std::vector<BlsScalar>& witnesses, const std::vector<uint64_t>& pi_idx,
                                      const std::vector<BlsScalar>& pi_vals) const {
    return unsatisfied_query(witnesses, pi_idx, pi_vals, n_constraints_).second;
  }
  // Debugger::unsatisfied_report for unsatisfied_constraints; nullopt when every constraint holds.
  std::optional<std::string> unsatisfied_report(const std::vector<BlsScalar>& witnesses, const std::vector<uint64_t>& pi_idx,
                                                const std::vector<BlsScalar>& pi_vals) const {
    return detail::unsatisfied_report(unsatisfied_query(witnesses, pi_idx, pi_vals, 1), n_constraints_);
  }

 private:
  Prover() : n_witnesses_(0), n_constraints_(0) {}
  std::pair<size_t, Unsatisfied> unsatisfied_query(const std::vector<BlsScalar>& witnesses, const std::vector<uint64_t>& pi_idx,
                                                   const std::vector<BlsScalar>& pi_vals, size_t cap) const {
    return detail::unsatisfied_query(
        [&](size_t c, uint64_t* rows, int32_t* families, size_t* n) {
          return pb200_prover_unsatisfied(h_, witnesses.empty() ? nullptr : witnesses[0].data(), witnesses.size(), pi_idx.data(),
                                          pi_vals.empty() ? nullptr : pi_vals[0].data(), pi_idx.size(), c, rows, families, n);
        },
        cap);
  }
  pb200_prover_t* h_ = nullptr;
  size_t n_witnesses_;
  size_t n_constraints_;
};

class Verifier;
struct BatchGroup;
inline void batch_verify_groups(const std::vector<BatchGroup>& groups);

// Verifier: verify checks PlonkVersion::V3, verify_with_version any version.  Errors as the reference: verify() throws ProofVerificationError for a proof that
// fails the check, PointMalformed for one Proof::from_bytes refuses, InvalidArgument for a public-input count that
// is not the verifier's (InconsistentPublicInputsLen); the constructors throw PointMalformed for a degenerate opening
// key, InvalidArgument for truncated or overflowing bytes (NotEnoughBytes), InvalidEvalDomainSize for a domain of
// 2^32 or more.
class Verifier {
 public:
  static constexpr size_t PROOF_SIZE = 1008;                      // Proof::SIZE
  static constexpr size_t OPENING_KEY_SIZE = PB200_OPENING_KEY_BYTES;  // OpeningKey::SIZE
  // Compiler::compile's Verifier half: the 15 commitments in Prover::commitments order (pb200_prover_commitments)
  Verifier(const std::string& label, size_t n_constraints, const std::array<uint8_t, 15 * 48>& commitments,
           const std::array<uint8_t, OPENING_KEY_SIZE>& opening_key, const std::vector<uint64_t>& pi_idx) {
    check_verifier(pb200_verifier_new((const uint8_t*)label.data(), label.size(), n_constraints, commitments.data(), opening_key.data(),
                                      pi_idx.empty() ? nullptr : pi_idx.data(), pi_idx.size(), &h_));
  }
  static std::unique_ptr<Verifier> try_from_bytes(const uint8_t* bytes, size_t len) {
    std::unique_ptr<Verifier> v(new Verifier());
    check_verifier(pb200_verifier_from_bytes(bytes, len, &v->h_));
    return v;
  }
  ~Verifier() { pb200_verifier_free(h_); }
  Verifier(const Verifier&) = delete;
  Verifier& operator=(const Verifier&) = delete;
  std::vector<uint8_t> to_bytes() const {
    size_t n = 0;
    check(pb200_verifier_to_bytes(h_, nullptr, 0, &n));
    std::vector<uint8_t> out(n);
    check(pb200_verifier_to_bytes(h_, out.data(), out.size(), &n));
    return out;
  }
  // Verifier::verify
  void verify(const std::array<uint8_t, PROOF_SIZE>& proof, const std::vector<BlsScalar>& public_inputs) const {
    verify_with_version(proof, public_inputs, PlonkVersion::V3);
  }
  // Verifier::verify_with_version
  void verify_with_version(const std::array<uint8_t, PROOF_SIZE>& proof, const std::vector<BlsScalar>& public_inputs,
                           PlonkVersion version) const {
    const std::vector<int32_t> st = verify_batch({proof}, {public_inputs}, version);
    if (st[0] == PB200_ERR_POINT_MALFORMED) throw Error(Error::PointMalformed, "InvalidData: malformed proof");
    check_verifier(st[0]);
  }
  // One status per proof (PB200_OK, PB200_ERR_VERIFY or PB200_ERR_POINT_MALFORMED); every proof must come with the
  // same number of public inputs.
  std::vector<int32_t> verify_batch(const std::vector<std::array<uint8_t, PROOF_SIZE>>& proofs,
                                    const std::vector<std::vector<BlsScalar>>& public_inputs) const {
    return verify_batch(proofs, public_inputs, PlonkVersion::V3);
  }
  // The same with every proof checked under `version`.
  std::vector<int32_t> verify_batch(const std::vector<std::array<uint8_t, PROOF_SIZE>>& proofs,
                                    const std::vector<std::vector<BlsScalar>>& public_inputs, PlonkVersion version) const {
    if (proofs.size() != public_inputs.size()) throw Error(Error::InvalidArgument, "one public-input vector per proof");
    const size_t n_pi = public_inputs.empty() ? 0 : public_inputs[0].size();
    std::vector<BlsScalar> pi;
    for (const auto& v : public_inputs) {
      if (v.size() != n_pi) throw Error(Error::InvalidArgument, "every proof needs the same number of public inputs");
      pi.insert(pi.end(), v.begin(), v.end());
    }
    std::vector<int32_t> st(proofs.size());
    check_verifier(pb200_verify_with_version(h_, (int)version, proofs.empty() ? nullptr : proofs[0].data(), proofs.size(),
                                             pi.empty() ? nullptr : pi[0].data(), n_pi, st.data()));
    return st;
  }
  // One verdict for the whole batch with one pairing (pb200_batch_verify): returns when every proof would pass
  // verify_with_version (up to a chance of (n - 1) / r); throws PointMalformed when some proof fails
  // Proof::from_bytes, otherwise ProofVerificationError, also for an empty batch.
  void batch_verify(const std::vector<std::array<uint8_t, PROOF_SIZE>>& proofs, const std::vector<std::vector<BlsScalar>>& public_inputs,
                    PlonkVersion version = PlonkVersion::V3) const {
    if (proofs.size() != public_inputs.size()) throw Error(Error::InvalidArgument, "one public-input vector per proof");
    const size_t n_pi = public_inputs.empty() ? pi_count() : public_inputs[0].size();
    std::vector<BlsScalar> pi;
    for (const auto& v : public_inputs) {
      if (v.size() != n_pi) throw Error(Error::InvalidArgument, "every proof needs the same number of public inputs");
      pi.insert(pi.end(), v.begin(), v.end());
    }
    int32_t verdict = PB200_OK;
    check_verifier(pb200_batch_verify(h_, (int)version, proofs.empty() ? nullptr : proofs[0].data(), proofs.size(),
                                      pi.empty() ? nullptr : pi[0].data(), n_pi, &verdict));
    if (verdict == PB200_ERR_POINT_MALFORMED) throw Error(Error::PointMalformed, "InvalidData: malformed proof");
    check_verifier(verdict);
  }

 private:
  friend void batch_verify_groups(const std::vector<BatchGroup>& groups);
  Verifier() = default;
  // the public-input count, read back from Verifier::to_bytes (its fourth big-endian u64)
  size_t pi_count() const {
    const std::vector<uint8_t> b = to_bytes();
    size_t n = 0;
    for (int k = 24; k < 32; k++) n = (n << 8) | b[k];
    return n;
  }
  static void check_verifier(int rc) {
    if (rc == PB200_ERR_VERIFY) throw Error(Error::ProofVerificationError, "ProofVerificationError");
    if (rc == PB200_ERR_POINT_MALFORMED) throw Error(Error::PointMalformed, std::string("InvalidData: ") + pb200_last_error());
    check(rc);
  }
  pb200_verifier_t* h_ = nullptr;
};

// One group of batch_verify_groups: proofs checked under `verifier` and `version`, with their public inputs.
struct BatchGroup {
  const Verifier& verifier;
  PlonkVersion version;
  std::vector<std::array<uint8_t, Verifier::PROOF_SIZE>> proofs;
  std::vector<std::vector<BlsScalar>> public_inputs;
};

// One verdict for groups of proofs under several verifiers and versions, with one pairing
// (pb200_batch_verify_groups): returns when every proof would pass its group's verify_with_version (up to a chance of
// (N - 1) / r over the N proofs); throws PointMalformed when some proof fails Proof::from_bytes, otherwise
// ProofVerificationError, also when there are no proofs; InvalidArgument for inconsistent public inputs, an unknown
// version or verifiers with different opening keys.  The verifiers must share one SRS; one may serve several groups.
inline void batch_verify_groups(const std::vector<BatchGroup>& groups) {
  std::vector<const pb200_verifier_t*> handles;
  std::vector<int32_t> versions;
  std::vector<size_t> n_proofs, n_pi;
  std::vector<uint8_t> proofs;
  std::vector<BlsScalar> pi;
  for (const BatchGroup& g : groups) {
    if (g.proofs.size() != g.public_inputs.size()) throw Error(Error::InvalidArgument, "one public-input vector per proof");
    const size_t k = g.public_inputs.empty() ? g.verifier.pi_count() : g.public_inputs[0].size();
    for (const auto& v : g.public_inputs) {
      if (v.size() != k) throw Error(Error::InvalidArgument, "every proof needs the same number of public inputs");
      pi.insert(pi.end(), v.begin(), v.end());
    }
    for (const auto& p : g.proofs) proofs.insert(proofs.end(), p.begin(), p.end());
    handles.push_back(g.verifier.h_);
    versions.push_back((int32_t)g.version);
    n_proofs.push_back(g.proofs.size());
    n_pi.push_back(k);
  }
  int32_t verdict = PB200_OK;
  Verifier::check_verifier(pb200_batch_verify_groups(handles.data(), versions.data(), n_proofs.data(), n_pi.data(), groups.size(),
                                                     proofs.empty() ? nullptr : proofs.data(), pi.empty() ? nullptr : pi[0].data(),
                                                     &verdict));
  if (verdict == PB200_ERR_POINT_MALFORMED) throw Error(Error::PointMalformed, "InvalidData: malformed proof");
  Verifier::check_verifier(verdict);
}

// PublicParameters (srs.rs): the commit key as 96-byte raw points and OpeningKey::to_bytes.  setup takes the three
// util::random_nonzero_bls_scalar draws (x, the G1 scalar, the G2 scalar; Montgomery form): the RNG is the caller's.
// Errors: DegreeIsZero (setup), NotEnoughBytes (from_slice of at most OpeningKey::SIZE bytes), PointMalformed (an
// invalid opening key, or a commit-key point from_slice refuses), InvalidArgument (a zero draw).
class PublicParameters {
 public:
  static constexpr size_t ADDED_BLINDING_DEGREE = 6;
  static constexpr size_t OPENING_KEY_SIZE = PB200_OPENING_KEY_BYTES;
  static std::unique_ptr<PublicParameters> setup(size_t max_degree, const BlsScalar& x, const BlsScalar& g_scalar, const BlsScalar& h_scalar) {
    std::unique_ptr<PublicParameters> pp(new PublicParameters());
    pp->raw_.resize(96 * (max_degree + ADDED_BLINDING_DEGREE + 1));
    check(pb200_public_parameters_setup(max_degree, x.data(), g_scalar.data(), h_scalar.data(), pp->raw_.data(), pp->opening_key_.data()));
    return pp;
  }
  // PublicParameters::from_slice (srs.rs:163-178): the opening key and every commit-key point validated
  static std::unique_ptr<PublicParameters> from_slice(const uint8_t* bytes, size_t len) {
    if (len <= OPENING_KEY_SIZE) throw Error(Error::NotEnoughBytes, "NotEnoughBytes");
    if ((len - OPENING_KEY_SIZE) % 48) throw Error(Error::PointMalformed, "InvalidData: the commit key is not whole 48-byte points");
    std::unique_ptr<PublicParameters> pp(new PublicParameters());
    check_points(pb200_opening_key_check(bytes));
    std::copy(bytes, bytes + OPENING_KEY_SIZE, pp->opening_key_.begin());
    const size_t n = (len - OPENING_KEY_SIZE) / 48;
    pp->raw_.resize(96 * n);
    check_points(pb200_g1_decompress(bytes + OPENING_KEY_SIZE, n, 1, pp->raw_.data()));
    return pp;
  }
  // PublicParameters::from_slice_unchecked (srs.rs:121-146) for to_raw_var_bytes: the opening key validated (the
  // reference panics where this throws PointMalformed), the commit-key points not
  static std::unique_ptr<PublicParameters> from_slice_unchecked(const uint8_t* bytes, size_t len) {
    if (len < OPENING_KEY_SIZE) throw Error(Error::NotEnoughBytes, "NotEnoughBytes");
    std::unique_ptr<PublicParameters> pp(new PublicParameters());
    check_points(pb200_opening_key_check(bytes));
    std::copy(bytes, bytes + OPENING_KEY_SIZE, pp->opening_key_.begin());
    size_t n = 0;
    check(pb200_raw_commit_key_points(bytes + OPENING_KEY_SIZE, len - OPENING_KEY_SIZE, 0, &n));
    pp->raw_.resize(96 * n + 1);
    check(pb200_commit_key_from_raw_var_bytes(bytes + OPENING_KEY_SIZE, len - OPENING_KEY_SIZE, 0, pp->raw_.data()));
    pp->raw_.resize(96 * n);
    return pp;
  }
  std::vector<uint8_t> to_var_bytes() const {  // srs.rs:149-153
    std::vector<uint8_t> out(opening_key_.begin(), opening_key_.end());
    out.resize(OPENING_KEY_SIZE + 48 * points());
    check(pb200_g1_compress_batch(raw_.data(), points(), out.data() + OPENING_KEY_SIZE));
    return out;
  }
  std::vector<uint8_t> to_raw_var_bytes() const {  // srs.rs:114-119
    size_t n = 0;
    check(pb200_commit_key_to_raw_var_bytes(raw_.data(), points(), nullptr, 0, &n));
    std::vector<uint8_t> out(opening_key_.begin(), opening_key_.end());
    out.resize(OPENING_KEY_SIZE + n);
    check(pb200_commit_key_to_raw_var_bytes(raw_.data(), points(), out.data() + OPENING_KEY_SIZE, n, &n));
    return out;
  }
  size_t max_degree() const { return points() - 1; }
  std::unique_ptr<CommitKey> commit_key() const { return std::unique_ptr<CommitKey>(new CommitKey(raw_.data(), points())); }
  const std::array<uint8_t, OPENING_KEY_SIZE>& opening_key() const { return opening_key_; }
  const std::vector<uint8_t>& raw_points() const { return raw_; }
  size_t points() const { return raw_.size() / 96; }

 private:
  friend class DevicePublicParameters;
  PublicParameters() = default;
  static void check_points(int rc) {
    if (rc == PB200_ERR_POINT_MALFORMED) throw Error(Error::PointMalformed, std::string("InvalidData: ") + pb200_last_error());
    check(rc);
  }
  std::vector<uint8_t> raw_;
  std::array<uint8_t, OPENING_KEY_SIZE> opening_key_{};
};

// PublicParameters resident on the GPU (pb200_pp_t): the commit key's points in HBM and the opening key.  Compiler
// and Prover take it wherever they take PublicParameters; the provers made from it share the MSM tables derived from the
// key (one per trimmed-key size and one per domain size), built once and kept until it is destroyed.  Those provers may
// outlive it.  RAII and non-copyable.  Errors as PublicParameters'.
class DevicePublicParameters {
 public:
  static constexpr size_t OPENING_KEY_SIZE = PB200_OPENING_KEY_BYTES;
  struct Tables {
    size_t monomial, lagrange, device_bytes;  // trimmed-key tables, Lagrange-form tables, their device bytes
  };
  // PublicParameters::setup with the commit key left on the device
  static std::unique_ptr<DevicePublicParameters> setup(size_t max_degree, const BlsScalar& x, const BlsScalar& g_scalar,
                                                       const BlsScalar& h_scalar) {
    return make([&](pb200_pp_t** h) { return pb200_pp_setup(max_degree, x.data(), g_scalar.data(), h_scalar.data(), h); });
  }
  // PublicParameters::from_slice: every point decoded and validated on the device, straight into place
  static std::unique_ptr<DevicePublicParameters> from_slice(const uint8_t* bytes, size_t len) {
    if (len <= OPENING_KEY_SIZE) throw Error(Error::NotEnoughBytes, "NotEnoughBytes");
    return make([&](pb200_pp_t** h) { return pb200_pp_from_slice(bytes, len, 1, h); });
  }
  // PublicParameters::from_slice_unchecked for to_raw_var_bytes
  static std::unique_ptr<DevicePublicParameters> from_slice_unchecked(const uint8_t* bytes, size_t len) {
    if (len < OPENING_KEY_SIZE) throw Error(Error::NotEnoughBytes, "NotEnoughBytes");
    return make([&](pb200_pp_t** h) { return pb200_pp_from_slice(bytes, len, 0, h); });
  }
  // The same parameters uploaded once; the points are trusted as Prover's constructor trusts them
  static std::unique_ptr<DevicePublicParameters> from_host(const PublicParameters& pp) {
    return make([&](pb200_pp_t** h) { return pb200_pp_new(pp.raw_points().data(), pp.points(), pp.opening_key().data(), h); });
  }
  std::unique_ptr<PublicParameters> to_host() const {
    std::unique_ptr<PublicParameters> pp(new PublicParameters());
    pp->raw_.resize(96 * points());
    check(pb200_pp_raw_points(h_, pp->raw_.data()));
    pp->opening_key_ = opening_key_;
    return pp;
  }
  Tables tables() const {
    Tables t{0, 0, 0};
    check(pb200_pp_tables(h_, &t.monomial, &t.lagrange, &t.device_bytes));
    return t;
  }
  size_t points() const { return pb200_pp_points(h_); }
  size_t max_degree() const { return points() - 1; }
  const std::array<uint8_t, OPENING_KEY_SIZE>& opening_key() const { return opening_key_; }
  const pb200_pp_t* handle() const { return h_; }
  ~DevicePublicParameters() { pb200_pp_free(h_); }
  DevicePublicParameters(const DevicePublicParameters&) = delete;
  DevicePublicParameters& operator=(const DevicePublicParameters&) = delete;

 private:
  DevicePublicParameters() = default;
  template <class F>
  static std::unique_ptr<DevicePublicParameters> make(F&& construct) {
    std::unique_ptr<DevicePublicParameters> pp(new DevicePublicParameters());
    PublicParameters::check_points(construct(&pp->h_));
    check(pb200_pp_opening_key(pp->h_, pp->opening_key_.data()));
    return pp;
  }
  pb200_pp_t* h_ = nullptr;
  std::array<uint8_t, OPENING_KEY_SIZE> opening_key_{};
};

inline Prover::Prover(const std::string& label, const Circuit& c, const DevicePublicParameters& pp)
    : n_witnesses_(c.n_witnesses), n_constraints_(c.n_constraints) {
  check(pb200_prover_new_pp(pp.handle(), (const uint8_t*)label.data(), label.size(), c.n_constraints, c.selectors[0].data(),
                            c.wires.data(), c.n_witnesses, &h_));
}
inline std::unique_ptr<Prover> Prover::try_from_bytes(const DevicePublicParameters& pp, const uint8_t* bytes, size_t len,
                                                      const std::vector<uint32_t>& wires, size_t n_witnesses) {
  std::unique_ptr<Prover> p(new Prover());
  p->n_witnesses_ = n_witnesses;
  p->n_constraints_ = wires.size() / 4;
  check(pb200_prover_from_bytes_pp(pp.handle(), bytes, len, wires.data(), n_witnesses, &p->h_));
  return p;
}
inline std::unique_ptr<Prover> Prover::from_compressed(const std::string& label, const std::vector<uint8_t>& compressed,
                                                       const DevicePublicParameters& pp, size_t n_witnesses) {
  std::unique_ptr<Prover> p(new Prover());
  p->n_witnesses_ = n_witnesses;
  uint64_t described_witnesses = 0;
  size_t n_labels = 0, n_pi = 0;
  check(pb200_compressed_circuit_info(compressed.data(), compressed.size(), pp.points(), &p->n_constraints_, &described_witnesses,
                                      &n_labels, &n_pi, nullptr));
  check(pb200_prover_from_compressed_pp(pp.handle(), (const uint8_t*)label.data(), label.size(), compressed.data(),
                                        compressed.size(), &p->h_));
  return p;
}

namespace detail {
inline Prover* new_prover(const std::string& label, const Circuit& c, const PublicParameters& pp) {
  return new Prover(label, c, pp.raw_points().data(), pp.points());
}
inline Prover* new_prover(const std::string& label, const Circuit& c, const DevicePublicParameters& pp) { return new Prover(label, c, pp); }
inline std::unique_ptr<Prover> compressed_prover(const std::string& label, const std::vector<uint8_t>& compressed,
                                                 const PublicParameters& pp, size_t n_witnesses) {
  return Prover::from_compressed(label, compressed, pp.raw_points().data(), pp.points(), n_witnesses);
}
inline std::unique_ptr<Prover> compressed_prover(const std::string& label, const std::vector<uint8_t>& compressed,
                                                 const DevicePublicParameters& pp, size_t n_witnesses) {
  return Prover::from_compressed(label, compressed, pp, n_witnesses);
}
}  // namespace detail

// Compiler (compiler.rs): Prover::new, the prover's 15 verifier-key commitments and the Verifier over the same opening
// key.  Public parameters too small for the circuit (pp.max_degree() < next_pow2(constraints + 6) + 6) throw
// TruncatedDegreeTooLarge.  Every method takes PublicParameters or DevicePublicParameters; the provers compiled from one
// DevicePublicParameters share its MSM tables.
struct Compiler {
  using Pair = std::pair<std::unique_ptr<Prover>, std::unique_ptr<Verifier>>;
  // Compiler::compile for a filled composer
  static Pair compile(const PublicParameters& pp, const std::string& label, const Composer& composer) {
    return compile_as(pp, label, composer);
  }
  static Pair compile(const DevicePublicParameters& pp, const std::string& label, const Composer& composer) {
    return compile_as(pp, label, composer);
  }
  // Compiler::compile_with_circuit: circuit(composer) fills a fresh Composer::initialized()
  template <class PP, class F>
  static Pair compile_with_circuit(const PP& pp, const std::string& label, F&& circuit) {
    Composer composer;
    circuit(composer);
    return compile(pp, label, composer);
  }
  // Compiler::compile_with_compressed (compiler.rs:84-112) for the bytes of compress(): the public parameters bound
  // the decoding.  Throws InvalidCompressedCircuit or BlsScalarMalformed for a description they refuse.
  template <class PP>
  static Pair compile_with_compressed(const PP& pp, const std::string& label, const std::vector<uint8_t>& compressed) {
    size_t n_constraints = 0, n_labels = 0, n_pi = 0;
    uint64_t n_witnesses = 0;
    check(pb200_compressed_circuit_info(compressed.data(), compressed.size(), pp.points(), &n_constraints, &n_witnesses, &n_labels,
                                        &n_pi, nullptr));
    std::vector<uint64_t> pi_idx(n_pi);
    if (n_pi)
      check(pb200_compressed_circuit_info(compressed.data(), compressed.size(), pp.points(), &n_constraints, &n_witnesses, &n_labels,
                                          &n_pi, pi_idx.data()));
    Pair out;
    out.first = detail::compressed_prover(label, compressed, pp, (size_t)n_witnesses);
    std::array<uint8_t, 15 * 48> comms;
    check(pb200_prover_commitments(out.first->handle(), comms.data()));
    out.second.reset(new Verifier(label, n_constraints, comms, pp.opening_key(), pi_idx));
    return out;
  }

 private:
  template <class PP>
  static Pair compile_as(const PP& pp, const std::string& label, const Composer& composer) {
    const Composer::Export e = composer.finish();
    Pair out;
    try {
      out.first.reset(detail::new_prover(label, circuit_of(e), pp));
    } catch (const Error& err) {
      if (err.kind == Error::PolynomialDegreeTooLarge) throw Error(Error::TruncatedDegreeTooLarge, err.what());
      throw;
    }
    std::array<uint8_t, 15 * 48> comms;
    check(pb200_prover_commitments(out.first->handle(), comms.data()));
    out.second.reset(new Verifier(label, e.n_constraints, comms, pp.opening_key(), e.pi_idx));
    return out;
  }
};

// Circuit::compress (circuit.rs:28-45, CompressedCircuit::from_composer compress.rs:136-240): circuit(composer) fills a
// fresh Composer::initialized(), whose description is returned as MessagePack behind raw deflate.  The reference always
// sets hades_optimization.
template <class F>
std::vector<uint8_t> compress(F&& circuit, bool hades_optimization = true) {
  Composer composer;
  circuit(composer);
  const Composer::Export e = composer.finish();
  size_t n = 0;
  const int hades = hades_optimization ? 1 : 0;
  check(pb200_circuit_compress(e.n_constraints, e.selectors.empty() ? nullptr : e.selectors[0].data(), e.wires.data(),
                               e.witnesses.size(), e.pi_idx.data(), e.pi_idx.size(), hades, nullptr, 0, &n));
  std::vector<uint8_t> out(n);
  check(pb200_circuit_compress(e.n_constraints, e.selectors.empty() ? nullptr : e.selectors[0].data(), e.wires.data(),
                               e.witnesses.size(), e.pi_idx.data(), e.pi_idx.size(), hades, out.data(), n, &n));
  return out;
}

}  // namespace plonk_b200
