// Circuit front end (see composer.h) and its C ABI (include/plonk_b200_composer.h).
#include "composer.h"

#include <string.h>

#include "../../include/plonk_b200_composer.h"

namespace pb {
extern thread_local std::string g_last_error;
}

namespace pbc {

// ---------------------------------------------------------------------------------------------
// Fr helpers
// ---------------------------------------------------------------------------------------------
Fr fr_u64(uint64_t x) {
  static const std::array<Fr, 16> small = [] {  // the gadgets mostly ask for bits, quads and tiny constants
    std::array<Fr, 16> t;
    for (uint64_t i = 0; i < 16; i++) t[i] = Fr::from_u64(i);
    return t;
  }();
  return x < 16 ? small[x] : Fr::from_u64(x);
}

// q * v for a selector coefficient, which is nearly always 0, 1 or -1
static inline void add_term(Fr& acc, const Fr& q, const Fr& v) {
  if (q.is_zero() || v.is_zero()) return;
  if (q == Fr::one())
    acc = acc + v;
  else if (v == Fr::one())  // bits and booleans: half of a gadget circuit's wire values
    acc = acc + q;
  else
    acc = acc + q * v;
}

static Fr fr_from_canonical(const uint64_t limbs[4]) {
  Fr r;
  memcpy(r.v, limbs, 32);
  return r.to_mont();
}

static const Fr& minus_one() {
  static const Fr m = Fr::one().neg();
  return m;
}

Fr fr_pow2(unsigned k) {
  Fr r = Fr::one();
  for (unsigned i = 0; i < k; i++) r = r.dbl();
  return r;
}

void fr_to_bits(const Fr& v, uint8_t bits[256]) {
  const Fr c = v.from_mont();
  for (int i = 0; i < 256; i++) bits[i] = (uint8_t)((c.v[i >> 6] >> (i & 63)) & 1);
}

Fr fr_recompose(const uint8_t bits[256], int start, int end) {
  Fr v = Fr::zero();
  for (int i = end - 1; i >= start; i--) {
    v = v.dbl();
    if (bits[i]) v = v + Fr::one();
  }
  return v;
}

// ---------------------------------------------------------------------------------------------
// JubJub
// ---------------------------------------------------------------------------------------------
const uint64_t kJubJubOrder[4] = {0xd0970e5ed6f72cb7ull, 0xa6682093ccc81082ull, 0x06673b0101343b00ull, 0x0e7db4ea6533afa9ull};

JubJubAffine jj_identity() { return {Fr::zero(), Fr::one()}; }

JubJubAffine jj_generator() {
  static const uint64_t u[4] = {0x4df7b7ffec7beacaull, 0x2e3ebb21fd6c54edull, 0xf1fbf02d0fd6cce6ull, 0x3fd2814c43ac65a6ull};
  static const JubJubAffine g = {fr_from_canonical(u), fr_u64(18)};
  return g;
}

JubJubAffine jj_add(const JubJubAffine& p, const JubJubAffine& q) {
  const Fr x1y2 = p.u * q.v, y1x2 = p.v * q.u;
  const Fr t = edwards_d() * x1y2 * y1x2;
  const Fr dx = Fr::one() + t, dy = Fr::one() - t;
  // a vanishing denominator is the reference's `sum.get_z() == 0` case (point.rs:226-231)
  if (dx.is_zero() || dy.is_zero()) return jj_identity();
  const Fr inv = (dx * dy).inv_bingcd();
  return {(x1y2 + y1x2) * (inv * dy), (p.v * q.v + p.u * q.u) * (inv * dx)};
}

JubJubAffine jj_neg(const JubJubAffine& p) { return {p.u.neg(), p.v}; }

// ---- extended coordinates (X : Y : Z : T), u = X/Z, v = Y/Z, T = XY/Z ---------------------------
// The gadgets below need long chains of curve additions whose every intermediate value becomes a
// witness.  The affine law costs one field inversion (~380 products) per addition; the chains are
// therefore run in extended coordinates (add-2008-hwcd-3 for a = -1, unified: it also doubles) and all
// their points normalised together with ONE inversion (Montgomery's trick).  Affine coordinates are
// unique, so the witness values are exactly those of the affine law; its one special case - a vanishing
// denominator, which jj_add maps to the identity like the reference's `sum.get_z() == 0` branch
// (point.rs:226-231) - is Z3 = (D - C)(D + C) = 0 here and gets the same treatment.
struct JubJubExt {
  Fr x, y, z, t;
};
static JubJubExt ext_identity() { return {Fr::zero(), Fr::one(), Fr::one(), Fr::zero()}; }
static JubJubExt ext_from_affine(const JubJubAffine& p) {
  if (p.u.is_zero()) return {p.u, p.v, Fr::one(), Fr::zero()};
  return {p.u, p.v, Fr::one(), p.u * p.v};
}
static const Fr& edwards_2d() {
  static const Fr d2 = edwards_d().dbl();
  return d2;
}
static JubJubExt ext_add(const JubJubExt& p, const JubJubExt& q) {
  const Fr a = (p.y - p.x) * (q.y - q.x), b = (p.y + p.x) * (q.y + q.x);
  const Fr c = p.t * edwards_2d() * q.t, d = (p.z * q.z).dbl();
  const Fr e = b - a, f = d - c, g = d + c, h = b + a;
  JubJubExt r = {e * f, g * h, f * g, e * h};
  if (r.z.is_zero()) return ext_identity();
  return r;
}
static bool ext_is_identity(const JubJubExt& p) { return p.x.is_zero() && p.y == p.z; }
// all points to affine with one inversion (none of the Z is zero: ext_add never returns such a point)
static void ext_batch_to_affine(const std::vector<JubJubExt>& in, std::vector<JubJubAffine>& out) {
  const size_t n = in.size();
  out.resize(n);
  if (!n) return;
  std::vector<Fr> pre(n);
  Fr acc = Fr::one();
  for (size_t i = 0; i < n; i++) {
    pre[i] = acc;
    acc = acc * in[i].z;
  }
  Fr inv = acc.inv_bingcd();
  for (size_t i = n; i-- > 0;) {
    const Fr zi = inv * pre[i];
    inv = inv * in[i].z;
    out[i] = {in[i].x * zi, in[i].y * zi};
  }
}
static JubJubExt ext_mul(const JubJubAffine& p, const uint64_t k[4]) {
  const JubJubExt pe = ext_from_affine(p);
  JubJubExt acc = ext_identity();
  bool started = false;
  for (int i = 255; i >= 0; i--) {
    if (started) acc = ext_add(acc, acc);
    if ((k[i >> 6] >> (i & 63)) & 1) {
      acc = started ? ext_add(acc, pe) : pe;
      started = true;
    }
  }
  return acc;
}

JubJubAffine jj_mul(const JubJubAffine& p, const uint64_t k[4]) {
  std::vector<JubJubExt> one(1, ext_mul(p, k));
  std::vector<JubJubAffine> out;
  ext_batch_to_affine(one, out);
  return out[0];
}

bool jj_is_on_curve(const JubJubAffine& p) {
  const Fr u2 = p.u.sqr(), v2 = p.v.sqr();
  return v2 - u2 == Fr::one() + edwards_d() * u2 * v2;
}

bool jj_is_torsion_free(const JubJubAffine& p) { return ext_is_identity(ext_mul(p, kJubJubOrder)); }

// on the curve and in the prime-order subgroup; the last point that passed is remembered (a circuit
// appends the same constant point over and over: benches/plonk.rs does so once per loop iteration)
static bool jj_is_valid_subgroup_point(const JubJubAffine& p) {
  static thread_local JubJubAffine last_ok;
  static thread_local bool have = false;
  if (have && last_ok == p) return true;
  if (!jj_is_on_curve(p) || !jj_is_torsion_free(p)) return false;
  last_ok = p;
  have = true;
  return true;
}

static bool lt_order(const uint64_t k[4]) {
  for (int i = 3; i >= 0; i--) {
    if (k[i] < kJubJubOrder[i]) return true;
    if (k[i] > kJubJubOrder[i]) return false;
  }
  return false;
}

// JubJubScalar::compute_windowed_naf(2): digits in {-1, 0, 1}, least significant first
static void wnaf2(const uint64_t scalar[4], int8_t out[256]) {
  uint64_t k[5] = {scalar[0], scalar[1], scalar[2], scalar[3], 0};
  memset(out, 0, 256);
  for (int i = 0; i < 256 && (k[0] | k[1] | k[2] | k[3] | k[4]); i++) {
    if (k[0] & 1) {
      if ((k[0] & 3) == 3) {  // digit -1: k += 1
        out[i] = -1;
        for (int j = 0; j < 5 && ++k[j] == 0; j++) {
        }
      } else {  // digit +1: k -= 1 (k is odd, no borrow)
        out[i] = 1;
        k[0] -= 1;
      }
    }
    for (int j = 0; j < 4; j++) k[j] = (k[j] >> 1) | (k[j + 1] << 63);
    k[4] >>= 1;
  }
}

// ---------------------------------------------------------------------------------------------
// Composer core
// ---------------------------------------------------------------------------------------------
Constraint::Constraint() {
  for (int i = 0; i < N_SELECTORS; i++) q[i] = Fr::zero();
  pi = Fr::zero();
}

static Constraint with(Selector s, const Fr& v) {
  Constraint c;
  c.set(s, v);
  return c;
}

Composer::Composer() {
  const Witness zero = append_witness(Fr::zero());
  const Witness one = append_witness(Fr::one());
  assert_equal_constant(zero, Fr::zero());
  assert_equal_constant(one, Fr::one());
  // append_dummy_gates (composer.rs:206-240)
  const Witness six = append_witness(fr_u64(6));
  const Witness one_ = append_witness(fr_u64(1));
  const Witness seven = append_witness(fr_u64(7));
  const Witness min_twenty = append_witness(fr_u64(20).neg());
  append_gate(Constraint().mult(fr_u64(1)).left(fr_u64(2)).right(fr_u64(3)).fourth(fr_u64(1)).constant(fr_u64(4)).output(fr_u64(4))
                  .a(six).b(seven).d(one_).c(min_twenty));
  append_gate(Constraint().mult(fr_u64(1)).left(fr_u64(1)).right(fr_u64(1)).constant(fr_u64(127)).output(fr_u64(1))
                  .a(min_twenty).b(six).c(seven));
}

const Fr& Composer::operator[](Witness w) const {
  if (w >= witnesses_.size()) throw ComposerError{PB200_ERR_INVALID_ARG, "witness index out of range"};
  return witnesses_[w];
}

Witness Composer::append_witness(const Fr& v) {
  witnesses_.push_back(v);
  return (Witness)(witnesses_.size() - 1);
}

void Composer::append_custom_gate(const Constraint& c) {
  for (int k = 0; k < 4; k++)
    if (c.w[k] >= witnesses_.size()) throw ComposerError{PB200_ERR_INVALID_ARG, "gate wired to an unallocated witness"};
  if (c.has_pi) public_inputs_[n_gates_] = c.pi;
  n_gates_++;
  if (witness_only_) return;
  Gate g;
  memcpy(g.q, c.q, sizeof g.q);
  memcpy(g.w, c.w, sizeof g.w);
  gates_.push_back(g);
}

void Composer::set_witness_only(bool on) {
  if (!on && witness_only_ && n_gates_ != gates_.size())
    throw ComposerError{PB200_ERR_INVALID_ARG, "gates appended in witness-only mode are not stored"};
  witness_only_ = on;
  if (on) {
    gates_.clear();
    gates_.shrink_to_fit();
  }
}

void Composer::append_gate(Constraint c) {
  c.set(Q_ARITH, Fr::one());
  append_custom_gate(c);
}

// append_gate for a constraint the caller no longer needs: q_arith is set in place
void Composer::append_gate_inplace(Constraint& c) {
  c.set(Q_ARITH, Fr::one());
  append_custom_gate(c);
}

// Solves q_M a b + q_L a + q_R b + q_O c + q_F d + q_C + PI = 0 for c (composer.rs:298-352)
bool Composer::append_evaluated_output(Constraint s, Witness* out) { return evaluated_output_inplace(s, out); }

bool Composer::evaluated_output_inplace(Constraint& s, Witness* out) {
  const Fr &a = (*this)[s.w[0]], &b = (*this)[s.w[1]], &d = (*this)[s.w[3]];
  Fr x = s.q[Q_C];
  if (s.has_pi) x = x + s.pi;
  if (!s.q[Q_M].is_zero() && !a.is_zero() && !b.is_zero()) add_term(x, s.q[Q_M], a == Fr::one() ? b : (b == Fr::one() ? a : a * b));
  add_term(x, s.q[Q_L], a);
  add_term(x, s.q[Q_R], b);
  add_term(x, s.q[Q_F], d);
  const Fr& y = s.q[Q_O];
  bool solved = true;
  Fr c;
  if (y == Fr::one())
    c = x.neg();
  else if (y == minus_one())
    c = x;
  else if (y.is_zero())
    solved = false;
  else
    c = x * y.inv_bingcd().neg();
  if (solved) {
    const Witness w = append_witness(c);  // may reallocate the witness table: a, b, d are not used past this point
    s.c(w);
    if (out) *out = w;
  }
  append_gate_inplace(s);
  return solved;
}

Witness Composer::gate_add(Constraint c) {
  c.set(Q_O, minus_one());
  Witness out = 0;
  evaluated_output_inplace(c, &out);
  return out;
}

Witness Composer::gate_mul(Constraint c) { return gate_add(c); }

Witness Composer::append_constant(const Fr& v) {
  const Witness w = append_witness(v);
  assert_equal_constant(w, v);
  return w;
}

Witness Composer::append_public(const Fr& v) {
  const Witness w = append_witness(v);
  append_gate(Constraint().left(minus_one()).a(w).pub(v));
  return w;
}

void Composer::assert_equal(Witness a, Witness b) { append_gate(Constraint().left(Fr::one()).right(minus_one()).a(a).b(b)); }

void Composer::assert_equal_constant(Witness a, const Fr& constant, const Fr* pi) {
  Constraint c = Constraint().left(minus_one()).a(a).constant(constant);
  if (pi) c.pub(*pi);
  append_gate(c);
}

// ---------------------------------------------------------------------------------------------
// bits.rs
// ---------------------------------------------------------------------------------------------
void Composer::component_boolean(Witness a) { append_gate(Constraint().mult(Fr::one()).output(minus_one()).a(a).b(a).c(a).d(ZERO)); }

std::vector<Witness> Composer::component_decomposition(Witness scalar, unsigned n) {
  if (n == 0 || n > 256) throw ComposerError{PB200_ERR_INVALID_ARG, "decomposition width must be in 1..=256"};
  uint8_t bits[256];
  fr_to_bits((*this)[scalar], bits);
  std::vector<Witness> out(n);
  Witness acc = ZERO;
  Fr weight = Fr::one();
  for (unsigned i = 0; i < n; i++) {
    const Witness w_bit = append_witness(fr_u64(bits[i]));
    component_boolean(w_bit);
    acc = gate_add(Constraint().left(weight).right(Fr::one()).a(w_bit).b(acc));
    out[i] = w_bit;
    weight = weight.dbl();
  }
  assert_equal(acc, scalar);
  return out;
}

// ---------------------------------------------------------------------------------------------
// range.rs
// ---------------------------------------------------------------------------------------------
void Composer::component_range_bits(Witness w, unsigned bits) {
  if (bits > 256) throw ComposerError{PB200_ERR_INVALID_ARG, "BITS must be <= 256"};
  range_check(w, bits);
}

void Composer::component_range(Witness w, unsigned bit_pairs) { range_check_even(w, bit_pairs * 2 < 256 ? bit_pairs * 2 : 256); }

void Composer::range_check(Witness value, unsigned num_bits) {
  if (num_bits % 2 == 0) {
    range_check_even(value, num_bits);
    return;
  }
  const unsigned top = num_bits - 1;
  uint8_t bits[256];
  fr_to_bits((*this)[value], bits);
  const Witness lower = append_witness(fr_recompose(bits, 0, (int)top));
  range_check_even(lower, top);
  const Witness top_bit = append_witness(fr_u64(bits[top]));
  component_boolean(top_bit);
  const Witness recomposed = gate_add(Constraint().left(Fr::one()).right(fr_pow2(top)).a(lower).b(top_bit));
  assert_equal(recomposed, value);
}

// Base-4 accumulator chain, four quads per range gate, most significant quad first; the chain ends
// on the d wire of a selector-free closing gate (range.rs:87-169).
void Composer::range_check_even(Witness witness, unsigned num_bits) {
  if (num_bits == 0) {
    append_gate(Constraint().left(Fr::one()).a(witness));
    return;
  }
  uint8_t bits[256];
  fr_to_bits((*this)[witness], bits);
  const unsigned num_gates = (num_bits >> 3) + (num_bits % 8 ? 1 : 0);
  const unsigned num_quads = num_gates * 4;
  const unsigned pad = 1 + (((num_quads << 1) - num_bits) >> 1);
  std::vector<Constraint> rows(num_gates + 1, with(Q_RANGE, Fr::one()));
  static const int wire_of[4] = {3, 2, 1, 0};  // D, C, B, A
  Fr acc = Fr::zero();
  Witness last = ZERO;
  for (unsigned i = pad; i <= num_quads; i++) {
    const unsigned bit_index = (num_quads - i) << 1;
    acc = acc.dbl().dbl() + fr_u64((uint64_t)bits[bit_index] + 2u * bits[bit_index + 1]);
    last = append_witness(acc);
    rows[i / 4].w[wire_of[i % 4]] = last;
  }
  rows.back() = Constraint().d(last);
  for (const Constraint& r : rows) append_custom_gate(r);
  assert_equal(last, witness);
}

// ---------------------------------------------------------------------------------------------
// logic.rs
// ---------------------------------------------------------------------------------------------
Witness Composer::logic_component(Witness a, Witness b, unsigned bit_pairs, bool is_xor) {
  if (bit_pairs > 127) throw ComposerError{PB200_ERR_INVALID_ARG, "BIT_PAIRS must be <= 127"};
  const unsigned num_bits = bit_pairs * 2;
  uint8_t abits[256], bbits[256];
  fr_to_bits((*this)[a], abits);
  fr_to_bits((*this)[b], bbits);
  Constraint row = with(Q_LOGIC, is_xor ? minus_one() : Fr::one());
  row.constant(is_xor ? minus_one() : Fr::one());
  Fr left_acc = Fr::zero(), right_acc = Fr::zero(), out_acc = Fr::zero();
  for (unsigned i = 0; i < bit_pairs; i++) {
    const unsigned hi = num_bits - 1 - 2 * i;  // quads from the most significant pair down
    const unsigned lq = (abits[hi] << 1) | abits[hi - 1];
    const unsigned rq = (bbits[hi] << 1) | bbits[hi - 1];
    const unsigned oq = is_xor ? (lq ^ rq) : (lq & rq);
    left_acc = left_acc.dbl().dbl() + fr_u64(lq);
    right_acc = right_acc.dbl().dbl() + fr_u64(rq);
    out_acc = out_acc.dbl().dbl() + fr_u64(oq);
    const Witness wit_a = append_witness(left_acc);
    const Witness wit_b = append_witness(right_acc);
    const Witness wit_c = append_witness(fr_u64(lq * rq));
    const Witness wit_d = append_witness(out_acc);
    row.c(wit_c);
    append_custom_gate(row);
    row.a(wit_a).b(wit_b).d(wit_d);
  }
  const Witness left_w = row.w[0], right_w = row.w[1], out_w = row.w[3];
  append_custom_gate(Constraint().a(left_w).b(right_w).d(out_w));
  if (bit_pairs) {  // bind_logic_accumulators (logic.rs:155-170)
    bind_truncation_split(a, left_w, num_bits);
    bind_truncation_split(b, right_w, num_bits);
  }
  return out_w;
}

Witness Composer::append_logic_and(Witness a, Witness b, unsigned bit_pairs) { return logic_component(a, b, bit_pairs, false); }
Witness Composer::append_logic_xor(Witness a, Witness b, unsigned bit_pairs) { return logic_component(a, b, bit_pairs, true); }

// ---------------------------------------------------------------------------------------------
// truncate.rs
// ---------------------------------------------------------------------------------------------
void Composer::bind_truncation_split(Witness input, Witness low, unsigned num_bits) {
  const unsigned high_bits = 255 - num_bits;
  uint8_t bits[256];
  fr_to_bits((*this)[input], bits);
  const Witness high = append_witness(fr_recompose(bits, (int)num_bits, 256));
  range_check(high, high_bits);
  const Witness recomposed = gate_add(Constraint().left(fr_pow2(num_bits)).right(Fr::one()).a(high).b(low));
  assert_equal(recomposed, input);
  assert_canonical_truncation(high, low, num_bits);
}

Witness Composer::component_truncate(Witness w, unsigned n) {
  if (n > 254) throw ComposerError{PB200_ERR_INVALID_ARG, "N must be <= 254"};
  uint8_t bits[256];
  fr_to_bits((*this)[w], bits);
  const Witness low = append_witness(fr_recompose(bits, 0, (int)n));
  range_check(low, n);
  bind_truncation_split(w, low, n);
  return low;
}

// (high, low) must be the split of a canonical value: high <= r_high, and low <= r_low whenever
// high == r_high (truncate.rs:65-107)
void Composer::assert_canonical_truncation(Witness high, Witness low, unsigned num_bits) {
  const unsigned high_bits = 255 - num_bits;
  uint8_t mbits[256];
  fr_to_bits(minus_one(), mbits);
  const Fr r_low = fr_recompose(mbits, 0, (int)num_bits);
  const Fr r_high = fr_recompose(mbits, (int)num_bits, 256);
  const Witness diff = gate_add(Constraint().left(minus_one()).a(high).constant(r_high));
  range_check(diff, high_bits);
  const Witness inverse = append_witness((*this)[diff].inv_bingcd());  // inv(0) = 0
  const Witness product = gate_mul(Constraint().mult(Fr::one()).a(diff).b(inverse));
  const Witness is_top = gate_add(Constraint().left(minus_one()).a(product).constant(Fr::one()));
  append_gate(Constraint().mult(Fr::one()).a(diff).b(is_top));
  const Witness r_low_minus_low = gate_add(Constraint().left(minus_one()).a(low).constant(r_low));
  const Witness guard = gate_mul(Constraint().mult(Fr::one()).a(is_top).b(r_low_minus_low));
  range_check(guard, num_bits);
}

// ---------------------------------------------------------------------------------------------
// select.rs
// ---------------------------------------------------------------------------------------------
Witness Composer::component_select(Witness bit, Witness a, Witness b) {
  const Witness bit_times_a = gate_mul(Constraint().mult(Fr::one()).a(bit).b(a));
  const Witness one_min_bit = gate_add(Constraint().left(minus_one()).constant(Fr::one()).a(bit));
  const Witness one_min_bit_b = gate_mul(Constraint().mult(Fr::one()).a(one_min_bit).b(b));
  return gate_add(Constraint().left(Fr::one()).right(Fr::one()).a(one_min_bit_b).b(bit_times_a));
}

Witness Composer::component_select_one(Witness bit, Witness value) {
  const Fr b = (*this)[bit], v = (*this)[value];
  const Witness f_x = append_witness(Fr::one() - b + b * v);
  append_gate(Constraint().mult(Fr::one()).left(minus_one()).output(minus_one()).constant(Fr::one()).a(bit).b(value).c(f_x));
  return f_x;
}

Witness Composer::component_select_zero(Witness bit, Witness value) { return gate_mul(Constraint().mult(Fr::one()).a(bit).b(value)); }

// ---------------------------------------------------------------------------------------------
// point.rs
// ---------------------------------------------------------------------------------------------
JubJubAffine Composer::point_value(WitnessPoint p) const { return {(*this)[p.x], (*this)[p.y]}; }

WitnessPoint Composer::append_point(const JubJubAffine& p) {
  const Witness x = append_witness(p.u);
  const Witness y = append_witness(p.v);
  return {x, y};
}

WitnessPoint Composer::append_constant_point(const JubJubAffine& p) {
  if (!jj_is_valid_subgroup_point(p)) throw ComposerError{PB200_ERR_JUBJUB_POINT, "JubJubPointNotTorsionFree"};
  const Witness x = append_constant(p.u);
  const Witness y = append_constant(p.v);
  return {x, y};
}

WitnessPoint Composer::append_public_point(const JubJubAffine& p) {
  const WitnessPoint w = append_point(p);
  assert_equal_public_point(w, p);
  return w;
}

void Composer::assert_equal_point(WitnessPoint a, WitnessPoint b) {
  assert_equal(a.x, b.x);
  assert_equal(a.y, b.y);
}

void Composer::assert_equal_public_point(WitnessPoint p, const JubJubAffine& pub) {
  assert_equal_constant(p.x, Fr::zero(), &pub.u);
  assert_equal_constant(p.y, Fr::zero(), &pub.v);
}

// P is in the prime-order subgroup iff P = 8 Q for a curve point Q (point.rs:171-221)
WitnessPoint Composer::assert_torsion_free_point(WitnessPoint p) {
  const JubJubAffine value = point_value(p);
  JubJubAffine q = jj_identity();
  if (jj_is_on_curve(value)) {
    // 8^-1 mod the subgroup order = (order + 1) / 8, the order being 7 mod 8
    uint64_t e[4];
    memcpy(e, kJubJubOrder, 32);
    e[0] += 1;  // no carry: the low limb is ...b7
    for (int j = 0; j < 4; j++) e[j] = (e[j] >> 3) | (j < 3 ? e[j + 1] << 61 : 0);
    q = jj_mul(value, e);
  }
  const WitnessPoint qw = append_point(q);
  const Witness u2 = gate_mul(Constraint().mult(Fr::one()).a(qw.x).b(qw.x));
  const Witness v2 = gate_mul(Constraint().mult(Fr::one()).a(qw.y).b(qw.y));
  const Witness u2v2 = gate_mul(Constraint().mult(Fr::one()).a(u2).b(v2));
  append_gate(Constraint().left(minus_one()).a(u2).right(Fr::one()).b(v2).output(edwards_d().neg()).c(u2v2).constant(minus_one()));
  const WitnessPoint q2 = add_point_gates(qw, qw);
  const WitnessPoint q4 = add_point_gates(q2, q2);
  const WitnessPoint q8 = add_point_gates(q4, q4);
  assert_equal_point(p, q8);
  return p;
}

WitnessPoint Composer::component_neg_point(WitnessPoint p) { return {gate_mul(Constraint().left(minus_one()).a(p.x)), p.y}; }

WitnessPoint Composer::component_sub_point(WitnessPoint a, WitnessPoint b) { return component_add_point(a, component_neg_point(b)); }

WitnessPoint Composer::component_add_point(WitnessPoint a, WitnessPoint b) { return add_point_gates(a, b); }

// One curve-addition gate pair: (x1, y1, x2, y2) then (x3, y3, -, x1 y2) (point.rs:266-312)
WitnessPoint Composer::add_point_gates(WitnessPoint a, WitnessPoint b) { return add_point_gates(a, b, jj_add(point_value(a), point_value(b))); }

// ... with the sum already known (chains compute their sums in extended coordinates, one inversion in all)
WitnessPoint Composer::add_point_gates(WitnessPoint a, WitnessPoint b, const JubJubAffine& sum) {
  const JubJubAffine p1 = point_value(a), p2 = point_value(b);
  const Witness x1y2 = append_witness(p1.u * p2.v);
  const Witness x3 = append_witness(sum.u);
  const Witness y3 = append_witness(sum.v);
  append_custom_gate(with(Q_VARIABLE_GROUP_ADD, Fr::one()).a(a.x).b(a.y).c(b.x).d(b.y));
  append_custom_gate(Constraint().a(x3).b(y3).d(x1y2));
  return {x3, y3};
}

WitnessPoint Composer::component_select_identity(Witness bit, WitnessPoint a) {
  component_boolean(bit);
  return select_identity_gates(bit, a);
}

WitnessPoint Composer::select_identity_gates(Witness bit, WitnessPoint a) {
  const Witness x = component_select_zero(bit, a.x);
  const Witness y = component_select_one(bit, a.y);
  return {x, y};
}

WitnessPoint Composer::component_select_point(Witness bit, WitnessPoint a, WitnessPoint b) {
  const Witness x = component_select(bit, a.x, b.x);
  const Witness y = component_select(bit, a.y, b.y);
  return {x, y};
}

// Double-and-add over the 252 scalar bits, most significant first (point.rs:361-378)
WitnessPoint Composer::component_mul_point(Witness jubjub, WitnessPoint p) {
  const std::vector<Witness> bits = component_decomposition(jubjub, 252);
  // the values of the whole chain first (extended coordinates, one inversion), then the gates
  const JubJubExt pe = ext_from_affine(point_value(p));
  std::vector<JubJubExt> chain;
  chain.reserve(2 * bits.size());
  JubJubExt r = ext_identity();
  for (size_t k = bits.size(); k-- > 0;) {
    r = ext_add(r, r);
    chain.push_back(r);
    // select_identity: bit ? P : identity (the bits are boolean-constrained witnesses of a decomposition);
    // adding the identity leaves the point as it is
    if (!(*this)[bits[k]].is_zero()) r = ext_add(r, pe);
    chain.push_back(r);
  }
  std::vector<JubJubAffine> vals;
  ext_batch_to_affine(chain, vals);
  WitnessPoint result = IDENTITY;
  size_t j = 0;
  for (size_t k = bits.size(); k-- > 0;) {
    result = add_point_gates(result, result, vals[j++]);
    const WitnessPoint addend = select_identity_gates(bits[k], p);
    result = add_point_gates(result, addend, vals[j++]);
  }
  return result;
}

// ---------------------------------------------------------------------------------------------
// fixed_base.rs
// ---------------------------------------------------------------------------------------------
void Composer::assert_canonical_jubjub_scalar(Witness scalar) {
  range_check(scalar, 252);
  uint64_t m[4];
  memcpy(m, kJubJubOrder, 32);
  m[0] -= 1;
  const Witness distance = gate_add(Constraint().left(minus_one()).a(scalar).constant(fr_from_canonical(m)));
  range_check(distance, 252);
}

// 256 signed-digit rounds against the precomputed multiples 2^(255-i) G (fixed_base.rs:47-226)
WitnessPoint Composer::component_mul_generator(Witness jubjub, const JubJubAffine& generator) {
  constexpr int kRounds = 256, kLeadingZeroRounds = 256 - (252 + 1);
  // multiples[i] = 2^(255-i) G: a table per generator, validated and built once per thread and generator
  static thread_local JubJubAffine table_gen;
  static thread_local std::vector<JubJubAffine> multiples;
  if (multiples.empty() || !(table_gen == generator)) {
    if (!jj_is_on_curve(generator) || !jj_is_torsion_free(generator) || generator == jj_identity())
      throw ComposerError{PB200_ERR_JUBJUB_GENERATOR, "JubJubGeneratorNotPrimeOrder"};
    std::vector<JubJubExt> dbl(kRounds);
    dbl[kRounds - 1] = ext_from_affine(generator);
    for (int i = kRounds - 2; i >= 0; i--) dbl[i] = ext_add(dbl[i + 1], dbl[i + 1]);
    ext_batch_to_affine(dbl, multiples);
    table_gen = generator;
  }
  const Fr canonical = (*this)[jubjub].from_mont();
  if (!lt_order(canonical.v)) throw ComposerError{PB200_ERR_JUBJUB_SCALAR, "JubJubScalarMalformed"};
  int8_t digits[256];
  wnaf2(canonical.v, digits);

  assert_canonical_jubjub_scalar(jubjub);

  std::vector<Fr> scalar_acc(kRounds + 1), xy_alpha(kRounds);
  std::vector<JubJubExt> point_ext(kRounds + 1);
  scalar_acc[0] = Fr::zero();
  point_ext[0] = ext_identity();
  for (int i = 0; i < kRounds; i++) {
    const int8_t digit = digits[kRounds - 1 - i];
    Fr s_add = Fr::zero();
    JubJubAffine p_add = jj_identity();
    if (digit == 1) {
      s_add = Fr::one();
      p_add = multiples[i];
    } else if (digit == -1) {
      s_add = minus_one();
      p_add = jj_neg(multiples[i]);
    }
    scalar_acc[i + 1] = scalar_acc[i].dbl() + s_add;
    point_ext[i + 1] = digit ? ext_add(point_ext[i], ext_from_affine(p_add)) : point_ext[i];
    xy_alpha[i] = digit ? p_add.u * p_add.v : Fr::zero();
  }
  std::vector<JubJubAffine> point_acc;
  ext_batch_to_affine(point_ext, point_acc);

  Witness leading = ZERO;
  for (int i = 0; i < kRounds; i++) {
    const Witness acc_x = append_witness(point_acc[i].u);
    const Witness acc_y = append_witness(point_acc[i].v);
    const Witness acc_bit = append_witness(scalar_acc[i]);
    if (i == kLeadingZeroRounds) leading = acc_bit;
    if (i == 0) {
      assert_equal_constant(acc_x, Fr::zero());
      assert_equal_constant(acc_y, Fr::one());
      assert_equal_constant(acc_bit, Fr::zero());
    }
    const Witness wxy = append_witness(xy_alpha[i]);
    const JubJubAffine& beta = multiples[i];
    append_custom_gate(with(Q_FIXED_GROUP_ADD, Fr::one()).left(beta.u).right(beta.v).constant(beta.u * beta.v)
                           .a(acc_x).b(acc_y).c(wxy).d(acc_bit));
  }
  const Witness acc_x = append_witness(point_acc[kRounds].u);
  const Witness acc_y = append_witness(point_acc[kRounds].v);
  const Witness last = append_witness(scalar_acc[kRounds]);
  append_gate(Constraint().a(acc_x).b(acc_y).d(last));
  assert_equal_constant(leading, Fr::zero());
  assert_equal(last, jubjub);
  return {acc_x, acc_y};
}

// ---------------------------------------------------------------------------------------------
// benches/plonk.rs BenchCircuit<DEGREE> with its Default values
// ---------------------------------------------------------------------------------------------
void Composer::bench_circuit(size_t degree) {
  const uint64_t seven[4] = {7, 0, 0, 0};
  const JubJubAffine z = jj_mul(jj_generator(), seven);
  const Witness w_a = append_witness(fr_u64(2));
  const Witness w_b = append_witness(fr_u64(3));
  const Witness w_x = append_witness(fr_u64(6));
  const Witness w_y = append_witness(fr_u64(7));
  const WitnessPoint w_z = append_point(z);
  size_t diff = 0, prev = constraints();
  while (prev + diff < degree) {
    const Witness r_w = gate_mul(Constraint().mult(Fr::one()).a(w_a).b(w_b));
    append_constant(fr_u64(15));
    append_constant_point(z);
    assert_equal(w_x, r_w);
    assert_equal_point(w_z, w_z);
    gate_add(Constraint().left(Fr::one()).right(Fr::one()).a(w_a).b(w_b));
    component_add_point(w_z, w_z);
    append_logic_and(w_a, w_b, 127);
    append_logic_xor(w_a, w_b, 127);
    component_boolean(ONE);
    component_decomposition(w_a, 254);
    component_mul_generator(w_y, jj_generator());
    component_mul_point(w_y, w_z);
    component_range_bits(w_a, 256);
    component_select(ONE, w_a, w_b);
    component_select_identity(ONE, w_z);
    component_select_one(ONE, w_a);
    component_select_point(ONE, w_z, w_z);
    component_select_zero(ONE, w_a);
    diff = constraints() - prev;
    prev = constraints();
  }
}

}  // namespace pbc

// =============================================================================================
// C ABI
// =============================================================================================
struct pb200_composer {
  pbc::Composer c;
};

namespace {

using pbc::Fr;

Fr fr_in(const uint64_t* p) {
  Fr r;
  memcpy(r.v, p, 32);
  return r;
}

template <class F>
int guarded(F&& f) {
  try {
    f();
    return PB200_OK;
  } catch (const pbc::ComposerError& e) {
    pb::g_last_error = e.what;
    return e.code;
  } catch (const std::exception& e) {
    pb::g_last_error = e.what();
    return PB200_ERR_INVALID_ARG;
  }
}

pbc::Constraint constraint_in(const uint64_t* selectors, const uint32_t wires[4], const uint64_t* pi) {
  pbc::Constraint c;
  for (int i = 0; i < pbc::N_SELECTORS; i++) c.q[i] = fr_in(selectors + 4 * i);
  for (int k = 0; k < 4; k++) c.w[k] = wires[k];
  if (pi) c.pub(fr_in(pi));
  return c;
}

pbc::JubJubAffine point_in(const uint64_t* uv) { return {fr_in(uv), fr_in(uv + 4)}; }

}  // namespace

#define PBC_REQUIRE(cond)                                  \
  do {                                                     \
    if (!(cond)) {                                         \
      pb::g_last_error = "null argument: " #cond;          \
      return PB200_ERR_INVALID_ARG;                        \
    }                                                      \
  } while (0)

extern "C" {

int pb200_composer_new(pb200_composer_t** out) {
  PBC_REQUIRE(out);
  return guarded([&] { *out = new pb200_composer(); });
}
void pb200_composer_free(pb200_composer_t* c) { delete c; }
size_t pb200_composer_constraints(const pb200_composer_t* c) { return c ? c->c.constraints() : 0; }
size_t pb200_composer_witnesses(const pb200_composer_t* c) { return c ? c->c.n_witnesses() : 0; }
size_t pb200_composer_public_inputs(const pb200_composer_t* c) { return c ? c->c.public_inputs().size() : 0; }

int pb200_composer_witness_value(const pb200_composer_t* c, uint32_t w, uint64_t* out) {
  PBC_REQUIRE(c && out);
  return guarded([&] { memcpy(out, c->c[w].v, 32); });
}
int pb200_composer_append_witness(pb200_composer_t* c, const uint64_t* value, uint32_t* out_w) {
  PBC_REQUIRE(c && value && out_w);
  return guarded([&] { *out_w = c->c.append_witness(fr_in(value)); });
}
int pb200_composer_append_gate(pb200_composer_t* c, const uint64_t* selectors, const uint32_t* wires, const uint64_t* pi, int custom) {
  PBC_REQUIRE(c && selectors && wires);
  return guarded([&] {
    const pbc::Constraint k = constraint_in(selectors, wires, pi);
    if (custom)
      c->c.append_custom_gate(k);
    else
      c->c.append_gate(k);
  });
}
int pb200_composer_append_evaluated_output(pb200_composer_t* c, const uint64_t* selectors, const uint32_t* wires, const uint64_t* pi,
                                           uint32_t* out_w, int* solved) {
  PBC_REQUIRE(c && selectors && wires && out_w);
  return guarded([&] {
    const bool ok = c->c.append_evaluated_output(constraint_in(selectors, wires, pi), out_w);
    if (solved) *solved = ok;
  });
}
int pb200_composer_gate_add(pb200_composer_t* c, const uint64_t* selectors, const uint32_t* wires, const uint64_t* pi, uint32_t* out_w) {
  PBC_REQUIRE(c && selectors && wires && out_w);
  return guarded([&] { *out_w = c->c.gate_add(constraint_in(selectors, wires, pi)); });
}
int pb200_composer_append_constant(pb200_composer_t* c, const uint64_t* value, uint32_t* out_w) {
  PBC_REQUIRE(c && value && out_w);
  return guarded([&] { *out_w = c->c.append_constant(fr_in(value)); });
}
int pb200_composer_append_public(pb200_composer_t* c, const uint64_t* value, uint32_t* out_w) {
  PBC_REQUIRE(c && value && out_w);
  return guarded([&] { *out_w = c->c.append_public(fr_in(value)); });
}
int pb200_composer_assert_equal(pb200_composer_t* c, uint32_t a, uint32_t b) {
  PBC_REQUIRE(c);
  return guarded([&] { c->c.assert_equal(a, b); });
}
int pb200_composer_assert_equal_constant(pb200_composer_t* c, uint32_t a, const uint64_t* constant, const uint64_t* pi) {
  PBC_REQUIRE(c && constant);
  return guarded([&] {
    const Fr p = pi ? fr_in(pi) : Fr::zero();
    c->c.assert_equal_constant(a, fr_in(constant), pi ? &p : nullptr);
  });
}
int pb200_composer_component_boolean(pb200_composer_t* c, uint32_t a) {
  PBC_REQUIRE(c);
  return guarded([&] { c->c.component_boolean(a); });
}
int pb200_composer_component_decomposition(pb200_composer_t* c, uint32_t scalar, uint32_t n_bits, uint32_t* out_bits) {
  PBC_REQUIRE(c && out_bits);
  return guarded([&] {
    const std::vector<pbc::Witness> bits = c->c.component_decomposition(scalar, n_bits);
    memcpy(out_bits, bits.data(), bits.size() * sizeof(uint32_t));
  });
}
int pb200_composer_component_range_bits(pb200_composer_t* c, uint32_t w, uint32_t bits) {
  PBC_REQUIRE(c);
  return guarded([&] { c->c.component_range_bits(w, bits); });
}
int pb200_composer_component_range(pb200_composer_t* c, uint32_t w, uint32_t bit_pairs) {
  PBC_REQUIRE(c);
  return guarded([&] { c->c.component_range(w, bit_pairs); });
}
int pb200_composer_append_logic(pb200_composer_t* c, uint32_t a, uint32_t b, uint32_t bit_pairs, int is_xor, uint32_t* out_w) {
  PBC_REQUIRE(c && out_w);
  return guarded([&] { *out_w = is_xor ? c->c.append_logic_xor(a, b, bit_pairs) : c->c.append_logic_and(a, b, bit_pairs); });
}
int pb200_composer_component_truncate(pb200_composer_t* c, uint32_t w, uint32_t n_bits, uint32_t* out_w) {
  PBC_REQUIRE(c && out_w);
  return guarded([&] { *out_w = c->c.component_truncate(w, n_bits); });
}
int pb200_composer_component_select(pb200_composer_t* c, uint32_t bit, uint32_t a, uint32_t b, uint32_t* out_w) {
  PBC_REQUIRE(c && out_w);
  return guarded([&] { *out_w = c->c.component_select(bit, a, b); });
}
int pb200_composer_component_select_one(pb200_composer_t* c, uint32_t bit, uint32_t value, uint32_t* out_w) {
  PBC_REQUIRE(c && out_w);
  return guarded([&] { *out_w = c->c.component_select_one(bit, value); });
}
int pb200_composer_component_select_zero(pb200_composer_t* c, uint32_t bit, uint32_t value, uint32_t* out_w) {
  PBC_REQUIRE(c && out_w);
  return guarded([&] { *out_w = c->c.component_select_zero(bit, value); });
}
int pb200_composer_append_point(pb200_composer_t* c, const uint64_t* uv, int kind, uint32_t* out_xy) {
  PBC_REQUIRE(c && uv && out_xy);
  return guarded([&] {
    const pbc::JubJubAffine p = point_in(uv);
    const pbc::WitnessPoint w = kind == 1 ? c->c.append_constant_point(p) : kind == 2 ? c->c.append_public_point(p) : c->c.append_point(p);
    out_xy[0] = w.x;
    out_xy[1] = w.y;
  });
}
int pb200_composer_assert_equal_point(pb200_composer_t* c, const uint32_t* a_xy, const uint32_t* b_xy) {
  PBC_REQUIRE(c && a_xy && b_xy);
  return guarded([&] { c->c.assert_equal_point({a_xy[0], a_xy[1]}, {b_xy[0], b_xy[1]}); });
}
int pb200_composer_assert_equal_public_point(pb200_composer_t* c, const uint32_t* p_xy, const uint64_t* uv) {
  PBC_REQUIRE(c && p_xy && uv);
  return guarded([&] { c->c.assert_equal_public_point({p_xy[0], p_xy[1]}, point_in(uv)); });
}
int pb200_composer_assert_torsion_free_point(pb200_composer_t* c, const uint32_t* p_xy) {
  PBC_REQUIRE(c && p_xy);
  return guarded([&] { c->c.assert_torsion_free_point({p_xy[0], p_xy[1]}); });
}
int pb200_composer_point_op(pb200_composer_t* c, int op, const uint32_t* a_xy, const uint32_t* b_xy, uint32_t* out_xy) {
  PBC_REQUIRE(c && a_xy && out_xy);
  return guarded([&] {
    const pbc::WitnessPoint a = {a_xy[0], a_xy[1]};
    pbc::WitnessPoint r;
    if (op == PB200_POINT_NEG) {
      r = c->c.component_neg_point(a);
    } else {
      if (!b_xy) throw pbc::ComposerError{PB200_ERR_INVALID_ARG, "second point missing"};
      const pbc::WitnessPoint b = {b_xy[0], b_xy[1]};
      if (op == PB200_POINT_ADD)
        r = c->c.component_add_point(a, b);
      else if (op == PB200_POINT_SUB)
        r = c->c.component_sub_point(a, b);
      else
        throw pbc::ComposerError{PB200_ERR_INVALID_ARG, "unknown point operation"};
    }
    out_xy[0] = r.x;
    out_xy[1] = r.y;
  });
}
int pb200_composer_component_select_identity(pb200_composer_t* c, uint32_t bit, const uint32_t* a_xy, uint32_t* out_xy) {
  PBC_REQUIRE(c && a_xy && out_xy);
  return guarded([&] {
    const pbc::WitnessPoint r = c->c.component_select_identity(bit, {a_xy[0], a_xy[1]});
    out_xy[0] = r.x;
    out_xy[1] = r.y;
  });
}
int pb200_composer_component_select_point(pb200_composer_t* c, uint32_t bit, const uint32_t* a_xy, const uint32_t* b_xy, uint32_t* out_xy) {
  PBC_REQUIRE(c && a_xy && b_xy && out_xy);
  return guarded([&] {
    const pbc::WitnessPoint r = c->c.component_select_point(bit, {a_xy[0], a_xy[1]}, {b_xy[0], b_xy[1]});
    out_xy[0] = r.x;
    out_xy[1] = r.y;
  });
}
int pb200_composer_component_mul_point(pb200_composer_t* c, uint32_t jubjub, const uint32_t* p_xy, uint32_t* out_xy) {
  PBC_REQUIRE(c && p_xy && out_xy);
  return guarded([&] {
    const pbc::WitnessPoint r = c->c.component_mul_point(jubjub, {p_xy[0], p_xy[1]});
    out_xy[0] = r.x;
    out_xy[1] = r.y;
  });
}
int pb200_composer_component_mul_generator(pb200_composer_t* c, uint32_t jubjub, const uint64_t* generator_uv, uint32_t* out_xy) {
  PBC_REQUIRE(c && out_xy);
  return guarded([&] {
    const pbc::WitnessPoint r = c->c.component_mul_generator(jubjub, generator_uv ? point_in(generator_uv) : pbc::jj_generator());
    out_xy[0] = r.x;
    out_xy[1] = r.y;
  });
}
int pb200_jubjub_generator(uint64_t* out_uv) {
  PBC_REQUIRE(out_uv);
  const pbc::JubJubAffine g = pbc::jj_generator();
  memcpy(out_uv, g.u.v, 32);
  memcpy(out_uv + 4, g.v.v, 32);
  return PB200_OK;
}
int pb200_jubjub_mul(const uint64_t* point_uv, const uint64_t* scalar, uint64_t* out_uv) {
  PBC_REQUIRE(point_uv && scalar && out_uv);
  const pbc::JubJubAffine r = pbc::jj_mul(point_in(point_uv), scalar);
  memcpy(out_uv, r.u.v, 32);
  memcpy(out_uv + 4, r.v.v, 32);
  return PB200_OK;
}
int pb200_composer_set_witness_only(pb200_composer_t* c, int on) {
  PBC_REQUIRE(c);
  return guarded([&] { c->c.set_witness_only(on != 0); });
}
int pb200_composer_bench_circuit(pb200_composer_t* c, size_t degree) {
  PBC_REQUIRE(c);
  return guarded([&] { c->c.bench_circuit(degree); });
}
int pb200_composer_export(const pb200_composer_t* c, uint64_t* selectors, uint32_t* wires, uint64_t* witnesses, uint64_t* pi_idx,
                          uint64_t* pi_vals) {
  PBC_REQUIRE(c);
  if ((selectors || wires) && c->c.witness_only()) {
    pb::g_last_error = "a witness-only composer holds no gate layout (export selectors / wires from the composer the prover was compiled from)";
    return PB200_ERR_INVALID_ARG;
  }
  const std::vector<pbc::Gate>& gates = c->c.gates();
  const size_t n = gates.size();
  for (size_t i = 0; i < n; i++) {
    if (selectors)
      for (int s = 0; s < pbc::N_SELECTORS; s++) memcpy(selectors + 4 * ((size_t)s * n + i), gates[i].q[s].v, 32);
    if (wires)
      for (int k = 0; k < 4; k++) wires[(size_t)k * n + i] = gates[i].w[k];
  }
  if (witnesses) memcpy(witnesses, c->c.witnesses().data(), c->c.n_witnesses() * 32);
  size_t j = 0;
  for (const auto& kv : c->c.public_inputs()) {  // std::map: ascending gate index, as public_input_indexes() sorts
    if (pi_idx) pi_idx[j] = kv.first;
    if (pi_vals) memcpy(pi_vals + 4 * j, kv.second.v, 32);
    j++;
  }
  return PB200_OK;
}

}  // extern "C"
