// Host build (g++) of the redundant Fp type FpR and the G1 formulas built on it (plonk_b200/csrc/bigint.cuh,
// g1.cuh), for tests/test_redundant_fp.py.  TEST INFRASTRUCTURE: the PTX carry chains are emulated by
// bigint.cuh's host primitives; nothing here is reachable from the product library.
#include <fenv.h>
#include <stddef.h>
#include <string.h>

#include "../../plonk_b200/csrc/g1.cuh"

using namespace pb;

static FpR ld(const uint32_t* p, size_t i) {
  FpR r;
  memcpy(r.v, p + 12 * i, 48);
  return r;
}
static void st(uint32_t* p, size_t i, const FpR& a) { memcpy(p + 12 * i, a.v, 48); }

extern "C" {

// op: 0 a*b, 1 a^2, 2 a+b, 3 a-b, 4 -a, 5 2a, 6 a*b + c*d, 7 a*b - c*d, 8 canonical(a), 9 is_zero_mod_p(a)
// (0/1 in limb 0), 10 a*b, 11 a^2 and 12 a*b + c*d by the two-pipe product without its final subtraction.
// Operands are limbs below 2p.
int rf_op(int op, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* out, size_t n) {
  const int old = fegetround();
  if (op >= 10) fesetround(FE_TOWARDZERO);
  for (size_t i = 0; i < n; i++) {
    const FpR x = ld(a, i), y = b ? ld(b, i) : x, z = c ? ld(c, i) : x, w = d ? ld(d, i) : x;
    FpR r = FpR::zero();
    switch (op) {
      case 0: r = x * y; break;
      case 1: r = x.sqr(); break;
      case 2: r = x + y; break;
      case 3: r = x - y; break;
      case 4: r = x.neg(); break;
      case 5: r = x.dbl(); break;
      case 6: r = FpR::mul2(x, y, z, w); break;
      case 7: r = FpR::mul_sub(x, y, z, w); break;
      case 8: r = FpR::from(x.canonical()); break;
      case 9: r.v[0] = x.is_zero_mod_p() ? 1u : 0u; break;
      case 10: r = FpR::from(Fp::mul_hybrid<false>(x.raw(), y.raw())); break;
      case 11: r = FpR::from(x.raw().sqr_hybrid<false>()); break;
      case 12: r = FpR::from(Fp::mul2_hybrid<false>(x.raw(), y.raw(), z.raw(), w.raw())); break;
      default: fesetround(old); return -1;
    }
    st(out, i, r);
  }
  fesetround(old);
  return 0;
}

// One G1 formula on XYZZ operands given as limbs (x, y, zz, zzz; any representation below 2p) or affine
// operands (x, y canonical).  op: 0 xyzz_add(P, Q), 1 xyzz_madd(P, affine Q), 2 xyzz_dbl(P),
// 3 xyzz_dbl_affine(affine Q).  out_xyzz receives the result as the formula left it (48 limbs),
// out_affine its affine normalisation (24 limbs).
int rf_g1(int op, const uint32_t* p, const uint32_t* q, uint32_t* out_xyzz, uint32_t* out_affine) {
  G1Xyzz P, Q, R;
  memcpy(&P, p, sizeof(P));
  G1Affine A;
  if (op == 1 || op == 3)
    memcpy(&A, q, sizeof(A));
  else if (q)
    memcpy(&Q, q, sizeof(Q));
  switch (op) {
    case 0: R = P; xyzz_add(R, Q); break;
    case 1: R = P; xyzz_madd(R, A.x, A.y); break;
    case 2: R = xyzz_dbl(P); break;
    case 3: R = xyzz_dbl_affine(FpR::from(A.x), FpR::from(A.y)); break;
    default: return -1;
  }
  memcpy(out_xyzz, &R, sizeof(R));
  const G1Affine r = xyzz_to_affine(R);
  memcpy(out_affine, &r, sizeof(r));
  return 0;
}
}
