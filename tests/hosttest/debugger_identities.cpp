// Host build (g++) of the debugger's gate identities (plonk_b200/csrc/plonk_algebra.cuh), for
// tests/test_debugger_algebra.py: the 17 identities and first_failing_identity with pbh::HFr, and the identity terms next
// to the widgets the quotient combines.  Field values cross this interface as 32-byte Montgomery-form integers.
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "../../plonk_b200/csrc/host_field.cpp"
#include "../../plonk_b200/csrc/plonk_algebra.cuh"

using namespace pb;
using pbh::HFr;

namespace {

HFr load(const uint8_t* p) {
  HFr x;
  memcpy(x.v, p, 32);
  return x;
}
void store(uint8_t* p, const HFr& x) { memcpy(p, x.v, 32); }

}  // namespace

extern "C" {

// in: n rows of 11 selectors (Poly order), pi, a, b, c, d, a_w, b_w, d_w.  out: n x 17 identities (each widget term
// times its selector); first: first_failing_identity per row.
int dbg_identities(const uint8_t* in, size_t n, uint8_t* out, int32_t* first) {
  for (size_t r = 0; r < n; r++) {
    HFr x[19];
    for (int k = 0; k < 19; k++) x[k] = load(in + (19 * r + k) * 32);
    auto q = [&](int k) { return x[k]; };
    const HFr& pi = x[11];
    const WireVals<HFr> v = {x[12], x[13], x[14], x[15], x[16], x[17], x[18]};
    const HFr ed = pbh::edwards_d();
    HFr id[N_IDENTITIES];
    id[ID_ARITH] = arith_identity(q, pi, v);
    const Terms<HFr, 4> rt = range_terms(v), ft = fixed_terms(ed, q(Q_L), q(Q_R), q(Q_C), v);
    const Terms<HFr, 5> lt = logic_terms(q(Q_C), v);
    const Terms<HFr, 3> vt = var_terms(ed, v);
    for (int k = 0; k < 4; k++) id[ID_RANGE + k] = rt.t[k] * q(Q_RANGE);
    for (int k = 0; k < 5; k++) id[ID_LOGIC + k] = lt.t[k] * q(Q_LOGIC);
    for (int k = 0; k < 4; k++) id[ID_FIXED + k] = ft.t[k] * q(Q_FIXED);
    for (int k = 0; k < 3; k++) id[ID_VAR + k] = vt.t[k] * q(Q_VAR);
    for (int k = 0; k < N_IDENTITIES; k++) store(out + (N_IDENTITIES * r + k) * 32, id[k]);
    first[r] = first_failing_identity(q, pi, ed, v);
  }
  return 0;
}

// in: n points of ch_range, ch_logic, ch_fixed, ch_var, q_l, q_r, q_c, a, b, c, d, a_w, b_w, d_w.  out: n x (16 terms -
// range 4, logic 5, fixed 4, variable 3 - then widget_range, widget_logic, widget_fixed, widget_var).
int dbg_terms_and_widgets(const uint8_t* in, size_t n, uint8_t* out) {
  for (size_t r = 0; r < n; r++) {
    HFr x[14];
    for (int k = 0; k < 14; k++) x[k] = load(in + (14 * r + k) * 32);
    const WireVals<HFr> v = {x[7], x[8], x[9], x[10], x[11], x[12], x[13]};
    const HFr ed = pbh::edwards_d();
    uint8_t* o = out + 20 * 32 * r;
    const Terms<HFr, 4> rt = range_terms(v), ft = fixed_terms(ed, x[4], x[5], x[6], v);
    const Terms<HFr, 5> lt = logic_terms(x[6], v);
    const Terms<HFr, 3> vt = var_terms(ed, v);
    int j = 0;
    for (int k = 0; k < 4; k++) store(o + 32 * j++, rt.t[k]);
    for (int k = 0; k < 5; k++) store(o + 32 * j++, lt.t[k]);
    for (int k = 0; k < 4; k++) store(o + 32 * j++, ft.t[k]);
    for (int k = 0; k < 3; k++) store(o + 32 * j++, vt.t[k]);
    store(o + 32 * j++, widget_range(sep_powers(x[0]), v));
    store(o + 32 * j++, widget_logic(sep_powers(x[1]), x[6], v));
    store(o + 32 * j++, widget_fixed(sep_powers(x[2]), ed, x[4], x[5], x[6], v));
    store(o + 32 * j++, widget_var(sep_powers(x[3]), ed, v));
  }
  return 0;
}
}
