// BLS12-381 pairing arithmetic for the verifier: the Fp2 / Fp6 / Fp12 tower, G2 on the M-twist, the prepared
// lines of a G2 point, the multi-Miller loop and the final exponentiation.
//
// The tower and every formula follow zkcrypto's bls12_381 (the crate behind dusk-bls12_381):
//   Fp2 = Fp[u] / (u^2 + 1),  Fp6 = Fp2[v] / (v^3 - (u + 1)),  Fp12 = Fp6[w] / (w^2 - v),
//   G2: y^2 = x^3 + 4(u + 1) over Fp2, embedded in E(Fp12) by (x, y) -> (x / w^2, y / w^3).
// Everything is __host__ __device__ on top of bigint.cuh's Fp, so tests/hosttest can run the same code on the
// CPU.  The Frobenius coefficients are not literals: pairing_consts_init() computes them from p.
#pragma once
#include "bigint.cuh"
#include "g1.cuh"
#if defined(__CUDACC__)
#include "fp_inv.cuh"
#endif

// The tower products are real calls on the device: inlined, one final exponentiation would be hundreds of
// thousands of instructions and minutes of compile time.
#if defined(__CUDACC__)
#define PB_NOINL __host__ __device__ __noinline__
#else
#define PB_NOINL inline
#endif

namespace pb {

PB_HD Fp fp_inverse(const Fp& a) {
#if defined(__CUDA_ARCH__)
  return fp_inv_bingcd(a);
#else
  return a.inv();
#endif
}

// a > p - a as integers, for a canonical Montgomery residue (Fp::lexicographically_largest)
PB_HD bool fp_lex_largest(const Fp& a) {
  const Fp c = a.from_mont(), n = a.neg().from_mont();
  bool larger = false, done = false;
#pragma unroll
  for (int k = 11; k >= 0; k--) {
    if (!done && c.v[k] != n.v[k]) {
      larger = c.v[k] > n.v[k];
      done = true;
    }
  }
  return larger;
}

struct Fp2 {
  Fp c0, c1;
  static PB_HD Fp2 zero() { return {Fp::zero(), Fp::zero()}; }
  static PB_HD Fp2 one() { return {Fp::one(), Fp::zero()}; }
  PB_HD bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
  PB_HD bool operator==(const Fp2& o) const { return c0 == o.c0 && c1 == o.c1; }
  friend PB_HD Fp2 operator+(const Fp2& a, const Fp2& b) { return {a.c0 + b.c0, a.c1 + b.c1}; }
  friend PB_HD Fp2 operator-(const Fp2& a, const Fp2& b) { return {a.c0 - b.c0, a.c1 - b.c1}; }
  PB_HD Fp2 neg() const { return {c0.neg(), c1.neg()}; }
  PB_HD Fp2 dbl() const { return {c0.dbl(), c1.dbl()}; }
  PB_HD Fp2 conj() const { return {c0, c1.neg()}; }
  // (a0 + a1 u)(b0 + b1 u) = (a0 b0 - a1 b1) + (a0 b1 + a1 b0) u: one reduction per coefficient
  friend PB_HD Fp2 operator*(const Fp2& a, const Fp2& b) {
    return {Fp::mul_sub(a.c0, b.c0, a.c1, b.c1), Fp::mul2(a.c0, b.c1, a.c1, b.c0)};
  }
  PB_HD Fp2 sqr() const { return {(c0 + c1) * (c0 - c1), (c0 * c1).dbl()}; }
  PB_HD Fp2 mul_fp(const Fp& s) const { return {c0 * s, c1 * s}; }
  // times the non-residue xi = u + 1
  PB_HD Fp2 mul_xi() const { return {c0 - c1, c0 + c1}; }
  PB_HD Fp2 inv() const {
    const Fp t = fp_inverse(Fp::mul2(c0, c0, c1, c1));
    return {c0 * t, (c1 * t).neg()};
  }
  // this^e for a little-endian exponent of 32-bit words (variable time: public exponents only)
  PB_NOINL Fp2 pow(const uint32_t* e, int words) const {
    Fp2 acc = one();
    bool started = false;
#pragma unroll 1
    for (int w = words - 1; w >= 0; w--) {
#pragma unroll 1
      for (int bit = 31; bit >= 0; bit--) {
        if (started) acc = acc.sqr();
        if ((e[w] >> bit) & 1u) {
          acc = started ? acc * (*this) : *this;
          started = true;
        }
      }
    }
    return acc;
  }
  PB_HD bool lex_largest() const { return fp_lex_largest(c1) || (c1.is_zero() && fp_lex_largest(c0)); }
  // Fp2::sqrt of zkcrypto (Algorithm 9 of eprint 2012/685, p = 3 mod 4); ok = false for a non-square
  PB_NOINL Fp2 sqrt(bool* ok) const {
    uint32_t e[12];  // (p - 3) / 4 = p >> 2, then (p - 1) / 2 = p >> 1
#pragma unroll
    for (int k = 0; k < 12; k++) e[k] = (FpParams::MOD(k) >> 2) | (k < 11 ? FpParams::MOD(k + 1) << 30 : 0u);
    const Fp2 a1 = pow(e, 12);
    const Fp2 alpha = a1.sqr() * (*this);
    const Fp2 x0 = a1 * (*this);
    Fp2 r;
    if (alpha == one().neg()) {
      r = {x0.c1.neg(), x0.c0};
    } else {
#pragma unroll
      for (int k = 0; k < 12; k++) e[k] = (FpParams::MOD(k) >> 1) | (k < 11 ? FpParams::MOD(k + 1) << 31 : 0u);
      r = (alpha + one()).pow(e, 12) * x0;
    }
    *ok = r.sqr() == *this;
    return r;
  }
};

// Frobenius coefficients: xi^((p-1)/3), xi^(2(p-1)/3) for Fp6 and xi^((p-1)/6) for Fp12
struct PairingConsts {
  Fp2 frob_v1, frob_v2, frob_w;
};
#if defined(__CUDACC__)
__constant__ PairingConsts c_pairing;
#endif
static PairingConsts h_pairing;
PB_HD const PairingConsts& pairing_consts() {
#if defined(__CUDA_ARCH__)
  return c_pairing;
#else
  return h_pairing;
#endif
}

struct Fp6 {
  Fp2 c0, c1, c2;
  static PB_HD Fp6 zero() { return {Fp2::zero(), Fp2::zero(), Fp2::zero()}; }
  static PB_HD Fp6 one() { return {Fp2::one(), Fp2::zero(), Fp2::zero()}; }
  friend PB_HD Fp6 operator+(const Fp6& a, const Fp6& b) { return {a.c0 + b.c0, a.c1 + b.c1, a.c2 + b.c2}; }
  friend PB_HD Fp6 operator-(const Fp6& a, const Fp6& b) { return {a.c0 - b.c0, a.c1 - b.c1, a.c2 - b.c2}; }
  PB_HD Fp6 neg() const { return {c0.neg(), c1.neg(), c2.neg()}; }
  PB_HD bool operator==(const Fp6& o) const { return c0 == o.c0 && c1 == o.c1 && c2 == o.c2; }
  // times v: (c0, c1, c2) -> (xi c2, c0, c1)
  PB_HD Fp6 mul_v() const { return {c2.mul_xi(), c0, c1}; }
  friend PB_NOINL Fp6 operator*(const Fp6& a, const Fp6& b) {
    const Fp2 t0 = a.c0 * b.c0, t1 = a.c1 * b.c1, t2 = a.c2 * b.c2;
    return {((a.c1 + a.c2) * (b.c1 + b.c2) - t1 - t2).mul_xi() + t0, (a.c0 + a.c1) * (b.c0 + b.c1) - t0 - t1 + t2.mul_xi(),
            (a.c0 + a.c2) * (b.c0 + b.c2) - t0 - t2 + t1};
  }
  PB_HD Fp6 mul_fp2(const Fp2& s) const { return {c0 * s, c1 * s, c2 * s}; }
  // times (b0 + b1 v)
  PB_NOINL Fp6 mul_01(const Fp2& b0, const Fp2& b1) const {
    const Fp2 aa = c0 * b0, bb = c1 * b1;
    return {(c2 * b1).mul_xi() + aa, (b0 + b1) * (c0 + c1) - aa - bb, c2 * b0 + bb};
  }
  // times b1 v
  PB_NOINL Fp6 mul_1(const Fp2& b1) const { return {(c2 * b1).mul_xi(), c0 * b1, c1 * b1}; }
  PB_HD Fp6 sqr() const { return (*this) * (*this); }
  PB_NOINL Fp6 frob() const {
    const PairingConsts& K = pairing_consts();
    return {c0.conj(), c1.conj() * K.frob_v1, c2.conj() * K.frob_v2};
  }
  PB_NOINL Fp6 inv() const {
    const Fp2 t0 = c0.sqr() - (c1 * c2).mul_xi();
    const Fp2 t1 = c2.sqr().mul_xi() - c0 * c1;
    const Fp2 t2 = c1.sqr() - c0 * c2;
    const Fp2 d = ((c1 * t2) + (c2 * t1)).mul_xi() + c0 * t0;
    const Fp2 di = d.inv();
    return {t0 * di, t1 * di, t2 * di};
  }
};

struct Fp12 {
  Fp6 c0, c1;
  static PB_HD Fp12 one() { return {Fp6::one(), Fp6::zero()}; }
  PB_HD bool is_one() const { return c0 == Fp6::one() && c1 == Fp6::zero(); }
  PB_HD Fp12 conj() const { return {c0, c1.neg()}; }
  friend PB_NOINL Fp12 operator*(const Fp12& a, const Fp12& b) {
    const Fp6 aa = a.c0 * b.c0, bb = a.c1 * b.c1;
    return {bb.mul_v() + aa, (a.c0 + a.c1) * (b.c0 + b.c1) - aa - bb};
  }
  PB_NOINL Fp12 sqr() const {
    const Fp6 ab = c0 * c1;
    return {(c1.mul_v() + c0) * (c0 + c1) - ab - ab.mul_v(), ab + ab};
  }
  // times the sparse line value b0 + b1 v + b4 v w
  PB_NOINL Fp12 mul_014(const Fp2& b0, const Fp2& b1, const Fp2& b4) const {
    const Fp6 aa = c0.mul_01(b0, b1), bb = c1.mul_1(b4);
    return {bb.mul_v() + aa, (c1 + c0).mul_01(b0, b1 + b4) - aa - bb};
  }
  PB_NOINL Fp12 frob() const {
    const Fp6 a = c0.frob(), b = c1.frob();
    return {a, b.mul_fp2(pairing_consts().frob_w)};
  }
  PB_NOINL Fp12 inv() const {
    const Fp6 t = (c0.sqr() - c1.sqr().mul_v()).inv();
    return {c0 * t, (c1 * t).neg()};
  }
};

// Computes the Frobenius coefficients from p into the host copy (the caller uploads it to the device).
inline void pairing_consts_init() {
  const Fp one = Fp::one();
  const Fp2 xi = {one, one};
  uint32_t e[12];  // (p - 1) / 6 from p - 1 by a long division over 32-bit words
  uint64_t rem = 0;
  for (int k = 11; k >= 0; k--) {
    const uint64_t cur = (rem << 32) | (k == 0 ? FpParams::MOD(0) - 1u : FpParams::MOD(k));
    e[k] = (uint32_t)(cur / 6);
    rem = cur % 6;
  }
  h_pairing.frob_w = xi.pow(e, 12);
  h_pairing.frob_v1 = h_pairing.frob_w.sqr();
  h_pairing.frob_v2 = h_pairing.frob_v1.sqr();
}

// ---- G2 -----------------------------------------------------------------------------------------------------
struct G2Affine {
  Fp2 x, y;
  bool inf;
};
struct G2Jac {  // x = X / Z^2, y = Y / Z^3; Z = 0 is the identity
  Fp2 x, y, z;
};

PB_HD Fp2 g2_b() { return Fp2{Fp::one(), Fp::one()}.dbl().dbl(); }  // 4 (u + 1)

PB_NOINL G2Jac g2_dbl(const G2Jac& p) {  // dbl-2009-l
  if (p.z.is_zero()) return p;
  const Fp2 a = p.x.sqr(), b = p.y.sqr(), c = b.sqr();
  const Fp2 d = ((p.x + b).sqr() - a - c).dbl();
  const Fp2 e = a.dbl() + a, f = e.sqr();
  G2Jac r;
  r.x = f - d.dbl();
  r.y = e * (d - r.x) - c.dbl().dbl().dbl();
  r.z = (p.y * p.z).dbl();
  return r;
}
PB_NOINL G2Jac g2_madd(const G2Jac& p, const G2Affine& q) {  // madd-2007-bl, every special case handled
  if (q.inf) return p;
  if (p.z.is_zero()) return {q.x, q.y, Fp2::one()};
  const Fp2 zz = p.z.sqr();
  const Fp2 u2 = q.x * zz, s2 = q.y * p.z * zz;
  const Fp2 h = u2 - p.x, rr = (s2 - p.y).dbl();
  if (h.is_zero()) return rr.is_zero() ? g2_dbl(p) : G2Jac{Fp2::one(), Fp2::one(), Fp2::zero()};
  const Fp2 hh = h.sqr(), i = hh.dbl().dbl(), j = h * i, v = p.x * i;
  G2Jac r;
  r.x = rr.sqr() - j - v.dbl();
  r.y = rr * (v - r.x) - (p.y * j).dbl();
  r.z = (p.z + h).sqr() - zz - hh;
  return r;
}

// G2Affine::from_compressed (zcash encoding: x.c1 || x.c0 big-endian, bit 7 compressed, bit 6 infinity,
// bit 5 "y is the lexicographically larger root") with the on-curve and prime-order subgroup checks of
// from_bytes.  Returns false for an encoding the reference rejects.
PB_NOINL bool g2_decode(const uint8_t* b, G2Affine* out) {
  const unsigned flags = b[0];
  Fp xc[2];
  for (int h = 0; h < 2; h++) {  // h = 0: c1 (first 48 bytes), h = 1: c0
    const uint8_t* s = b + 48 * h;
    for (int k = 0; k < 12; k++) {
      const int o = 44 - 4 * k;
      xc[h].v[k] = ((uint32_t)s[o] << 24) | ((uint32_t)s[o + 1] << 16) | ((uint32_t)s[o + 2] << 8) | (uint32_t)s[o + 3];
    }
  }
  xc[0].v[11] &= 0x1fffffffu;
  out->x = Fp2::zero();
  out->y = Fp2::zero();
  out->inf = true;
  if (!(flags & 0x80u)) return false;
  if (flags & 0x40u) return xc[0].is_zero() && xc[1].is_zero() && !(flags & 0x20u);
  for (int h = 0; h < 2; h++) {
    bool lt = false, done = false;
    for (int k = 11; k >= 0; k--) {
      const uint32_t m = FpParams::MOD(k);
      if (!done && xc[h].v[k] != m) {
        lt = xc[h].v[k] < m;
        done = true;
      }
    }
    if (!lt) return false;
  }
  const Fp2 x = {xc[1].to_mont(), xc[0].to_mont()};
  bool ok;
  Fp2 y = (x.sqr() * x + g2_b()).sqrt(&ok);
  if (!ok) return false;
  if (y.lex_largest() != ((flags & 0x20u) != 0)) y = y.neg();
  out->x = x;
  out->y = y;
  out->inf = false;
  G2Jac acc = {Fp2::one(), Fp2::one(), Fp2::zero()};  // [r] Q = O
#pragma unroll 1
  for (int w = 7; w >= 0; w--) {
    const uint32_t word = FrParams::MOD(w);
#pragma unroll 1
    for (int bit = 31; bit >= 0; bit--) {
      acc = g2_dbl(acc);
      if ((word >> bit) & 1u) acc = g2_madd(acc, *out);
    }
  }
  return acc.z.is_zero();
}

// [k] q for a canonical little-endian scalar of 8 words (double-and-add, variable time: the setup draws are the
// caller's, and this runs once per PublicParameters::setup).
PB_NOINL G2Jac g2_mul(const G2Affine& q, const uint32_t* k) {
  G2Jac acc = {Fp2::one(), Fp2::one(), Fp2::zero()};
#pragma unroll 1
  for (int w = 7; w >= 0; w--) {
#pragma unroll 1
    for (int bit = 31; bit >= 0; bit--) {
      acc = g2_dbl(acc);
      if ((k[w] >> bit) & 1u) acc = g2_madd(acc, q);
    }
  }
  return acc;
}

PB_NOINL G2Affine g2_to_affine(const G2Jac& p) {
  if (p.z.is_zero()) return {Fp2::zero(), Fp2::zero(), true};
  const Fp2 zi = p.z.inv(), zi2 = zi.sqr();
  return {p.x * zi2, p.y * zi2 * zi, false};
}

// G2Affine::to_compressed, the inverse of g2_decode: x.c1 then x.c0 big-endian, bit 7 set, bit 6 for the identity,
// bit 5 when y is the lexicographically larger root (c1 compared first, c0 when c1 = 0).
PB_NOINL void g2_encode(const G2Affine& q, uint8_t* b) {
  for (int k = 0; k < 96; k++) b[k] = 0;
  if (q.inf) {
    b[0] = 0xc0u;
    return;
  }
  const Fp xc[2] = {q.x.c1.from_mont(), q.x.c0.from_mont()};
  for (int h = 0; h < 2; h++)
    for (int k = 0; k < 12; k++) {
      const int o = 48 * h + 44 - 4 * k;
      b[o] = (uint8_t)(xc[h].v[k] >> 24);
      b[o + 1] = (uint8_t)(xc[h].v[k] >> 16);
      b[o + 2] = (uint8_t)(xc[h].v[k] >> 8);
      b[o + 3] = (uint8_t)xc[h].v[k];
    }
  b[0] |= 0x80u | (q.y.lex_largest() ? 0x20u : 0u);
}

// ---- Miller loop --------------------------------------------------------------------------------------------
// |x| of BLS12-381; x itself is negative
#define PB_BLS_X 0xd201000000010000ull
#define PB_G2_LINES 68  // 63 doubling and 5 addition steps

struct LineCoeffs {
  Fp2 c0, c1, c2;  // the line is c2 + (c1 x_P) v + (c0 y_P) v w at a G1 point P
};

// G2Prepared's doubling step (Algorithm 26 of eprint 2010/354) on the Jacobian accumulator r
PB_NOINL LineCoeffs line_dbl(G2Jac& r) {
  const Fp2 t0 = r.x.sqr(), t1 = r.y.sqr(), t2 = t1.sqr();
  const Fp2 t3 = ((t1 + r.x).sqr() - t0 - t2).dbl();
  const Fp2 t4 = t0.dbl() + t0;
  const Fp2 t6 = r.x + t4;
  const Fp2 t5 = t4.sqr();
  const Fp2 zsq = r.z.sqr();
  r.x = t5 - t3.dbl();
  r.z = (r.z + r.y).sqr() - t1 - zsq;
  r.y = (t3 - r.x) * t4 - t2.dbl().dbl().dbl();
  LineCoeffs l;
  l.c0 = (r.z * zsq).dbl();
  l.c1 = (t4 * zsq).dbl().neg();
  l.c2 = (t6.sqr() - t0 - t5) - t1.dbl().dbl();
  return l;
}
// G2Prepared's addition step (Algorithm 27 of eprint 2010/354): r += q
PB_NOINL LineCoeffs line_add(G2Jac& r, const G2Affine& q) {
  const Fp2 zsq = r.z.sqr(), ysq = q.y.sqr();
  const Fp2 t0 = zsq * q.x;
  const Fp2 t1 = ((q.y + r.z).sqr() - ysq - zsq) * zsq;
  const Fp2 t2 = t0 - r.x;
  const Fp2 t3 = t2.sqr();
  const Fp2 t4 = t3.dbl().dbl();
  const Fp2 t5 = t4 * t2;
  const Fp2 t6 = t1 - r.y.dbl();
  const Fp2 t9 = t6 * q.x;
  const Fp2 t7 = t4 * r.x;
  r.x = t6.sqr() - t5 - t7.dbl();
  r.z = (r.z + t2).sqr() - zsq - t3;
  const Fp2 t10 = q.y + r.z;
  const Fp2 t8 = (t7 - r.x) * t6;
  r.y = t8 - (r.y * t5).dbl();
  LineCoeffs l;
  l.c0 = r.z.dbl();
  l.c1 = t6.neg().dbl();
  l.c2 = t9.dbl() - (t10.sqr() - ysq - r.z.sqr());
  return l;
}

// G2Prepared::from: the 68 line coefficient triples of the Miller loop for a non-identity point q
PB_NOINL void g2_prepare(const G2Affine& q, LineCoeffs* out) {
  G2Jac r = {q.x, q.y, Fp2::one()};
  int n = 0;
#pragma unroll 1
  for (int b = 62; b >= 1; b--) {
    out[n++] = line_dbl(r);
    if ((PB_BLS_X >> b) & 1ull) out[n++] = line_add(r, q);
  }
  out[n++] = line_dbl(r);
}

PB_HD Fp12 ell(const Fp12& f, const LineCoeffs& l, const G1Affine& p) {
  return f.mul_014(l.c2, l.c1.mul_fp(p.x), l.c0.mul_fp(p.y));
}

// multi_miller_loop over two pairs (p[k], prepared lines[k]); an identity G1 point contributes 1
PB_NOINL Fp12 miller_loop2(const G1Affine* p, const LineCoeffs* const* lines) {
  const bool use0 = !p[0].is_inf(), use1 = !p[1].is_inf();
  Fp12 f = Fp12::one();
  int n = 0;
#pragma unroll 1
  for (int b = 62; b >= 0; b--) {
    if (use0) f = ell(f, lines[0][n], p[0]);
    if (use1) f = ell(f, lines[1][n], p[1]);
    n++;
    if (b == 0) break;
    if ((PB_BLS_X >> b) & 1ull) {
      if (use0) f = ell(f, lines[0][n], p[0]);
      if (use1) f = ell(f, lines[1][n], p[1]);
      n++;
    }
    f = f.sqr();
  }
  return f.conj();  // x < 0
}

// ---- final exponentiation -----------------------------------------------------------------------------------
PB_HD void fp4_sqr(const Fp2& a, const Fp2& b, Fp2* c0, Fp2* c1) {
  const Fp2 t0 = a.sqr(), t1 = b.sqr();
  *c0 = t1.mul_xi() + t0;
  *c1 = (a + b).sqr() - t0 - t1;
}
// squaring in the cyclotomic subgroup (Granger-Scott, eprint 2009/565)
PB_NOINL Fp12 cyclotomic_sqr(const Fp12& f) {
  Fp2 z0 = f.c0.c0, z4 = f.c0.c1, z3 = f.c0.c2, z2 = f.c1.c0, z1 = f.c1.c1, z5 = f.c1.c2;
  Fp2 t0, t1, t2, t3;
  fp4_sqr(z0, z1, &t0, &t1);
  z0 = t0 - z0;
  z0 = z0.dbl() + t0;
  z1 = t1 + z1;
  z1 = z1.dbl() + t1;
  fp4_sqr(z2, z3, &t0, &t1);
  fp4_sqr(z4, z5, &t2, &t3);
  z4 = t0 - z4;
  z4 = z4.dbl() + t0;
  z5 = t1 + z5;
  z5 = z5.dbl() + t1;
  t0 = t3.mul_xi();
  z2 = t0 + z2;
  z2 = z2.dbl() + t0;
  z3 = t2 - z3;
  z3 = z3.dbl() + t2;
  return {{z0, z4, z3}, {z2, z1, z5}};
}
// f^x (x < 0) for f in the cyclotomic subgroup
PB_NOINL Fp12 cyclotomic_exp_x(const Fp12& f) {
  Fp12 t = f;  // the leading bit of |x|
#pragma unroll 1
  for (int b = 62; b >= 0; b--) {
    t = cyclotomic_sqr(t);
    if ((PB_BLS_X >> b) & 1ull) t = t * f;
  }
  return t.conj();
}
// MillerLoopResult::final_exponentiation: the easy part f^((p^6 - 1)(p^2 + 1)), then the hard part by the
// x-chain.  The chain raises to 3 (p^4 - p^2 + 1) / r, so the result is the cube of f^((p^12 - 1) / r).
PB_NOINL Fp12 final_exponentiation(const Fp12& f) {
  Fp12 t0 = f.conj();  // f^(p^6)
  Fp12 t1 = f.inv();
  Fp12 t2 = t0 * t1;
  t1 = t2;
  t2 = t2.frob().frob() * t1;
  t1 = cyclotomic_sqr(t2).conj();
  Fp12 t3 = cyclotomic_exp_x(t2);
  Fp12 t4 = cyclotomic_sqr(t3);
  Fp12 t5 = t1 * t3;
  t1 = cyclotomic_exp_x(t5);
  t0 = cyclotomic_exp_x(t1);
  Fp12 t6 = cyclotomic_exp_x(t0) * t4;
  t4 = cyclotomic_exp_x(t6);
  t5 = t5.conj();
  t4 = t4 * (t5 * t2);
  t5 = t2.conj();
  t1 = (t1 * t2).frob().frob().frob();
  t6 = (t6 * t5).frob();
  t3 = (t3 * t0).frob().frob();
  t3 = t3 * t1;
  t3 = t3 * t6;
  return t3 * t4;
}

}  // namespace pb
