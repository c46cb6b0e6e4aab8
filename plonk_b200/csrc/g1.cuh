// BLS12-381 G1 point arithmetic for the bucket MSM (y^2 = x^3 + 4 over Fp, a = 0).
//
// Replaces the group arithmetic inside dusk_bls12_381::multiscalar_mul::msm_variable_base, the
// callee of CommitKey::commit (reference src/commitment_scheme/kzg10/key.rs:376-388).  The MSM
// result is representation independent once normalised to affine (Commitment::from,
// reference src/commitment_scheme/kzg10/commitment.rs:89-93), so we are free to pick the cheapest
// coordinates: buckets are accumulated in XYZZ (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2), where a mixed
// addition of an affine base costs 8M + 2S and needs no field inversion.
//
// The XYZZ coordinates are FpR values (bigint.cuh: [0, 2p), products without the final subtraction).
// Affine points stay canonical Fp and enter the formulas as they are.  Whatever leaves the formulas
// for other code - affine normalisation, stored points - is made canonical on the way out
// (xyzz_to_affine, G1Xyzz::canonical).
#pragma once
#include "bigint.cuh"

namespace pb {

// Affine base point as stored in HBM: x, y Montgomery limbs; the identity is x = y = 0 (not on the
// curve, so the encoding is unambiguous).
struct G1Affine {
  Fp x, y;
  PB_HD bool is_inf() const { return x.is_zero() && y.is_zero(); }
};

struct G1Xyzz {
  FpR x, y, zz, zzz;
  static PB_HD G1Xyzz identity() {
    G1Xyzz r;
    r.x = FpR::zero();
    r.y = FpR::zero();
    r.zz = FpR::zero();
    r.zzz = FpR::zero();
    return r;
  }
  // The identity is the only point with zz = 0 mod p, and it always has the limbs zero, so a plain test
  // suffices: identity() writes zeros, and every other zz is a product of factors that are nonzero mod p -
  // one (from an affine point), zz * pp with pp = (u2 - u1)^2, where u2 - u1 = 0 mod p is caught by
  // is_zero_mod_p and routed to the doubling or the identity, and zz * (2y)^2, where y = 0 mod p is caught
  // the same way.  A product of nonzero residues is neither 0 nor p.
  PB_HD bool is_inf() const { return zz.is_zero_limbs(); }
  static PB_HD G1Xyzz from_affine(const G1Affine& p) {
    G1Xyzz r;
    if (p.is_inf()) return identity();
    r.x = FpR::from(p.x);
    r.y = FpR::from(p.y);
    r.zz = FpR::one();
    r.zzz = FpR::one();
    return r;
  }
  PB_HD G1Xyzz neg() const {
    G1Xyzz r = *this;
    r.y = y.neg();
    return r;
  }
  // every coordinate in [0, p): the form in which points are stored and handed to other code
  PB_HD G1Xyzz canonical() const {
    G1Xyzz r;
    r.x = FpR::from(x.canonical());
    r.y = FpR::from(y.canonical());
    r.zz = FpR::from(zz.canonical());
    r.zzz = FpR::from(zzz.canonical());
    return r;
  }
};

// 2*P for affine P (mdbl-2008-s-1).  P must not be the identity.
PB_HD G1Xyzz xyzz_dbl_affine(const FpR& x1, const FpR& y1) {
  G1Xyzz r;
  if (y1.is_zero_mod_p()) return G1Xyzz::identity();  // 2-torsion: cannot happen in the prime-order group
  FpR u = y1.dbl();
  FpR v = u.sqr();
  FpR w = u * v;
  FpR s = x1 * v;
  FpR xx = x1.sqr();
  FpR m = xx.dbl() + xx;
  r.x = m.sqr() - s.dbl();
  r.y = FpR::mul_sub(m, s - r.x, w, y1);  // two products, one reduction
  r.zz = v;
  r.zzz = w;
  return r;
}

// 2*P in XYZZ (dbl-2008-s-1).
PB_HD G1Xyzz xyzz_dbl(const G1Xyzz& p) {
  if (p.is_inf()) return p;
  if (p.y.is_zero_mod_p()) return G1Xyzz::identity();
  G1Xyzz r;
  FpR u = p.y.dbl();
  FpR v = u.sqr();
  FpR w = u * v;
  FpR s = p.x * v;
  FpR xx = p.x.sqr();
  FpR m = xx.dbl() + xx;
  r.x = m.sqr() - s.dbl();
  r.y = FpR::mul_sub(m, s - r.x, w, p.y);
  r.zz = v * p.zz;
  r.zzz = w * p.zzz;
  return r;
}

// y or -y (as 2p - y) for a canonical y != 0: the sign of a signed-digit entry, without a borrow test
PB_HD FpR signed_y(const Fp& y, bool neg) {
  FpR n;
  n.v[0] = sub_cc(FpR::MOD2(0), y.v[0]);
#pragma unroll
  for (int i = 1; i < FpR::N - 1; i++) n.v[i] = subc_cc(FpR::MOD2(i), y.v[i]);
  n.v[FpR::N - 1] = subc(FpR::MOD2(FpR::N - 1), y.v[FpR::N - 1]);
#pragma unroll
  for (int i = 0; i < FpR::N; i++) n.v[i] = neg ? n.v[i] : y.v[i];
  return n;
}

// The common case of madd-2008-s, given u2 = x2 * acc.zz and s2 = y2 * acc.zzz: acc += (x2, y2) when
// u2 != acc.x, i.e. acc is neither P, -P nor the identity (whose limbs are all zero, so u2 = acc.x = 0).
// Returns false and leaves acc as it was otherwise.  Split from the two products so that a caller can
// reuse the registers of (x2, y2) once they are read.
PB_HD bool xyzz_madd_distinct(G1Xyzz& acc, const FpR& u2, const FpR& s2) {
  FpR p = u2 - acc.x;
  if (p.is_zero_mod_p()) return false;
  FpR r = s2 - acc.y;
  FpR pp = p.sqr();
  FpR ppp = p * pp;
  FpR q = acc.x * pp;
  FpR x3 = r.sqr() - ppp - q.dbl();
  FpR y3 = FpR::mul_sub(r, q - x3, acc.y, ppp);
  acc.x = x3;
  acc.y = y3;
  acc.zz = acc.zz * pp;
  acc.zzz = acc.zzz * ppp;
  return true;
}

// acc += (x2, y2) for an affine, non-identity point (madd-2008-s), all special cases handled:
// acc = identity, acc == P (doubling), acc == -P (result is the identity).
PB_HD void xyzz_madd(G1Xyzz& acc, const FpR& x2, const FpR& y2) {
  if (acc.is_inf()) {
    acc.x = x2;
    acc.y = y2;
    acc.zz = FpR::one();
    acc.zzz = FpR::one();
    return;
  }
  const FpR s2 = y2 * acc.zzz;
  if (xyzz_madd_distinct(acc, x2 * acc.zz, s2)) return;
  if ((s2 - acc.y).is_zero_mod_p())
    acc = xyzz_dbl_affine(x2, y2);
  else
    acc = G1Xyzz::identity();
}
PB_HD void xyzz_madd(G1Xyzz& acc, const Fp& x2, const Fp& y2) { xyzz_madd(acc, FpR::from(x2), FpR::from(y2)); }

// acc += o, both XYZZ (add-2008-s), all special cases handled.
PB_HD void xyzz_add(G1Xyzz& acc, const G1Xyzz& o) {
  if (o.is_inf()) return;
  if (acc.is_inf()) {
    acc = o;
    return;
  }
  FpR u1 = acc.x * o.zz;
  FpR u2 = o.x * acc.zz;
  FpR s1 = acc.y * o.zzz;
  FpR s2 = o.y * acc.zzz;
  FpR p = u2 - u1;
  FpR r = s2 - s1;
  if (p.is_zero_mod_p()) {
    if (r.is_zero_mod_p())
      acc = xyzz_dbl(acc);
    else
      acc = G1Xyzz::identity();
    return;
  }
  FpR pp = p.sqr();
  FpR ppp = p * pp;
  FpR q = u1 * pp;
  FpR x3 = r.sqr() - ppp - q.dbl();
  FpR y3 = FpR::mul_sub(r, q - x3, s1, ppp);
  acc.x = x3;
  acc.y = y3;
  acc.zz = acc.zz * o.zz * pp;
  acc.zzz = acc.zzz * o.zzz * ppp;
}

// k * P for a canonical (non-Montgomery) little-endian integer k of `words` 32-bit words: plain
// double-and-add, variable time (public data only: twiddle factors of the group-element NTT).
PB_HD G1Xyzz xyzz_mul(const G1Xyzz& p, const uint32_t* k, int words) {
  G1Xyzz acc = G1Xyzz::identity();
  bool started = false;
  for (int w = words - 1; w >= 0; w--) {
    for (int bit = 31; bit >= 0; bit--) {
      if (started) acc = xyzz_dbl(acc);
      if ((k[w] >> bit) & 1u) {
        if (started) {
          xyzz_add(acc, p);
        } else {
          acc = p;
          started = true;
        }
      }
    }
  }
  return acc;
}

// Affine normalisation (one inversion): x = X/ZZ, y = Y/ZZZ, canonical.
PB_HD G1Affine xyzz_to_affine(const G1Xyzz& p) {
  G1Affine r;
  if (p.is_inf()) {
    r.x = Fp::zero();
    r.y = Fp::zero();
    return r;
  }
  const Fp zz = p.zz.canonical(), zzz = p.zzz.canonical();
  Fp i = (zz * zzz).inv();
  Fp izz = i * zzz;
  Fp izzz = i * zz;
  r.x = p.x.canonical() * izz;
  r.y = p.y.canonical() * izzz;
  return r;
}

}  // namespace pb
