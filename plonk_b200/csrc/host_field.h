// Host-side (CPU) 64-bit-limb Montgomery arithmetic for the few serial tails the GPU path leaves
// on the host: the last Horner step of the MSM bucket reduction, projective->affine normalisation
// (Commitment::from, reference src/commitment_scheme/kzg10/commitment.rs:89-93), G1 compression
// (commitment.rs:95-101) and the Fiat-Shamir scalars of the prover.  Product code (part of
// libplonk_b200), independent of oracle/.
#pragma once
#include <stdint.h>
#include <string.h>

namespace pbh {

typedef unsigned __int128 u128;

template <int N>
struct Mod64 {
  uint64_t p[N];
  uint64_t inv;    // -p^-1 mod 2^64
  uint64_t r1[N];  // 2^(64N) mod p
  uint64_t r2[N];  // 2^(128N) mod p
};

template <int N, const Mod64<N>& M>
struct HField {
  uint64_t v[N];

  static HField zero() { HField r; memset(r.v, 0, sizeof r.v); return r; }
  static HField one() { HField r; memcpy(r.v, M.r1, sizeof r.v); return r; }
  bool is_zero() const { uint64_t x = 0; for (int i = 0; i < N; i++) x |= v[i]; return x == 0; }
  bool operator==(const HField& o) const { return memcmp(v, o.v, sizeof v) == 0; }
  bool operator!=(const HField& o) const { return !(*this == o); }

  static bool geq_p(const uint64_t* t) {
    for (int i = N - 1; i >= 0; i--) {
      if (t[i] > M.p[i]) return true;
      if (t[i] < M.p[i]) return false;
    }
    return true;
  }
  static void sub_p(uint64_t* t) {
    u128 borrow = 0;
    for (int i = 0; i < N; i++) {
      u128 d = (u128)t[i] - M.p[i] - borrow;
      t[i] = (uint64_t)d;
      borrow = (d >> 64) & 1;
    }
  }
  friend HField operator+(const HField& a, const HField& b) {
    HField r;
    u128 c = 0;
    for (int i = 0; i < N; i++) {
      c += (u128)a.v[i] + b.v[i];
      r.v[i] = (uint64_t)c;
      c >>= 64;
    }
    if (c || geq_p(r.v)) sub_p(r.v);
    return r;
  }
  friend HField operator-(const HField& a, const HField& b) {
    HField r;
    u128 borrow = 0;
    for (int i = 0; i < N; i++) {
      u128 d = (u128)a.v[i] - b.v[i] - borrow;
      r.v[i] = (uint64_t)d;
      borrow = (d >> 64) & 1;
    }
    if (borrow) {
      u128 c = 0;
      for (int i = 0; i < N; i++) {
        c += (u128)r.v[i] + M.p[i];
        r.v[i] = (uint64_t)c;
        c >>= 64;
      }
    }
    return r;
  }
  HField neg() const { return zero() - *this; }
  HField dbl() const { return *this + *this; }
  friend HField operator*(const HField& a, const HField& b) {  // CIOS
    uint64_t t[N + 2];
    memset(t, 0, sizeof t);
    for (int i = 0; i < N; i++) {
      u128 c = 0;
      for (int j = 0; j < N; j++) {
        c += (u128)a.v[j] * b.v[i] + t[j];
        t[j] = (uint64_t)c;
        c >>= 64;
      }
      c += t[N];
      t[N] = (uint64_t)c;
      t[N + 1] = (uint64_t)(c >> 64);
      uint64_t m = t[0] * M.inv;
      c = (u128)m * M.p[0] + t[0];
      c >>= 64;
      for (int j = 1; j < N; j++) {
        c += (u128)m * M.p[j] + t[j];
        t[j - 1] = (uint64_t)c;
        c >>= 64;
      }
      c += t[N];
      t[N - 1] = (uint64_t)c;
      t[N] = t[N + 1] + (uint64_t)(c >> 64);
    }
    HField r;
    memcpy(r.v, t, sizeof r.v);
    if (t[N] || geq_p(r.v)) sub_p(r.v);
    return r;
  }
  HField sqr() const { return (*this) * (*this); }
  HField pow(const uint64_t* e, int words) const {
    HField acc = one();
    for (int w = words - 1; w >= 0; w--)
      for (int bit = 63; bit >= 0; bit--) {
        acc = acc.sqr();
        if ((e[w] >> bit) & 1) acc = acc * (*this);
      }
    return acc;
  }
  HField pow_u64(uint64_t e) const {  // from the low bit: as many squarings as e has bits
    HField acc = one(), b = *this;
    for (; e; e >>= 1, b = b.sqr())
      if (e & 1) acc = acc * b;
    return acc;
  }
  HField inv() const {  // Fermat; 0 -> 0
    uint64_t e[N];
    memcpy(e, M.p, sizeof e);
    e[0] -= 2;  // p is odd and p[0] >= 2 for both moduli
    return pow(e, N);
  }
  // The same inverse by the binary extended Euclidean algorithm (shifts, additions and subtractions only: about
  // five times faster on the host than the Fermat power above; used by the circuit front end, whose gadgets
  // invert a few hundred scalars per run).  0 -> 0.
  HField inv_bingcd() const {
    if (is_zero()) return *this;
    uint64_t u[N], v[N], x1[N], x2[N];
    memcpy(u, this->v, sizeof u);
    memcpy(v, M.p, sizeof v);
    memset(x1, 0, sizeof x1);
    memset(x2, 0, sizeof x2);
    x1[0] = 1;
    auto is_one = [](const uint64_t* t) {
      uint64_t x = t[0] ^ 1;
      for (int i = 1; i < N; i++) x |= t[i];
      return x == 0;
    };
    auto halve = [](uint64_t* t, uint64_t* x) {  // t even: t /= 2, x = x / 2 mod p
      for (int i = 0; i < N - 1; i++) t[i] = (t[i] >> 1) | (t[i + 1] << 63);
      t[N - 1] >>= 1;
      uint64_t carry = 0;
      if (x[0] & 1) {  // x + p < 2^(64N + 1): keep the carry for the shift
        u128 c = 0;
        for (int i = 0; i < N; i++) {
          c += (u128)x[i] + M.p[i];
          x[i] = (uint64_t)c;
          c >>= 64;
        }
        carry = (uint64_t)c;
      }
      for (int i = 0; i < N - 1; i++) x[i] = (x[i] >> 1) | (x[i + 1] << 63);
      x[N - 1] = (x[N - 1] >> 1) | (carry << 63);
    };
    auto sub_mod = [](uint64_t* x, const uint64_t* y) {  // x = x - y mod p, both < p
      u128 borrow = 0;
      for (int i = 0; i < N; i++) {
        u128 d = (u128)x[i] - y[i] - borrow;
        x[i] = (uint64_t)d;
        borrow = (d >> 64) & 1;
      }
      if (borrow) {
        u128 c = 0;
        for (int i = 0; i < N; i++) {
          c += (u128)x[i] + M.p[i];
          x[i] = (uint64_t)c;
          c >>= 64;
        }
      }
    };
    auto geq = [](const uint64_t* a, const uint64_t* b) {
      for (int i = N - 1; i >= 0; i--) {
        if (a[i] > b[i]) return true;
        if (a[i] < b[i]) return false;
      }
      return true;
    };
    auto sub = [](uint64_t* a, const uint64_t* b) {  // a -= b, a >= b
      u128 borrow = 0;
      for (int i = 0; i < N; i++) {
        u128 d = (u128)a[i] - b[i] - borrow;
        a[i] = (uint64_t)d;
        borrow = (d >> 64) & 1;
      }
    };
    while (!is_one(u) && !is_one(v)) {
      while (!(u[0] & 1)) halve(u, x1);
      while (!(v[0] & 1)) halve(v, x2);
      if (geq(u, v)) {
        sub(u, v);
        sub_mod(x1, x2);
      } else {
        sub(v, u);
        sub_mod(x2, x1);
      }
    }
    HField y;  // (aR)^-1 as a plain integer; two Montgomery products by R^2 give a^-1 R
    memcpy(y.v, is_one(u) ? x1 : x2, sizeof y.v);
    HField r2;
    memcpy(r2.v, M.r2, sizeof r2.v);
    return (y * r2) * r2;
  }
  HField to_mont() const { HField r2; memcpy(r2.v, M.r2, sizeof r2.v); return (*this) * r2; }
  HField from_mont() const { HField o = zero(); o.v[0] = 1; return (*this) * o; }
  static HField from_u64(uint64_t x) { HField r = zero(); r.v[0] = x; return r.to_mont(); }
  // canonical integer comparison helper: is (this, canonical form) > (p-1)/2 ?
  bool canonical_gt_half() const {
    HField c = from_mont();
    // compare 2*c with p: c > (p-1)/2  <=>  2c > p - 1  <=>  2c >= p + 1 > p (p odd)
    uint64_t t[N + 1];
    uint64_t carry = 0;
    for (int i = 0; i < N; i++) {
      t[i] = (c.v[i] << 1) | carry;
      carry = c.v[i] >> 63;
    }
    if (carry) return true;
    for (int i = N - 1; i >= 0; i--) {
      if (t[i] > M.p[i]) return true;
      if (t[i] < M.p[i]) return false;
    }
    return false;
  }
};

extern const Mod64<6> kFpMod;
extern const Mod64<4> kFrMod;
typedef HField<6, kFpMod> HFp;
typedef HField<4, kFrMod> HFr;

// dusk_jubjub::EDWARDS_D = -(10240 / 10241), Montgomery form
inline const HFr& edwards_d() {
  static const HFr d = (HFr::from_u64(10240) * HFr::from_u64(10241).inv_bingcd()).neg();
  return d;
}

// G1 in XYZZ coordinates on the host (same formulas as csrc/g1.cuh).
struct HXyzz {
  HFp x, y, zz, zzz;
  static HXyzz identity() { HXyzz r; r.x = r.y = r.zz = r.zzz = HFp::zero(); return r; }
  bool is_inf() const { return zz.is_zero(); }
};
HXyzz hxyzz_dbl(const HXyzz& p);
void hxyzz_add(HXyzz& acc, const HXyzz& o);
// returns false for the identity; out x,y in Montgomery form
bool hxyzz_to_affine(const HXyzz& p, HFp* x, HFp* y);
void g1_compress_raw(const uint64_t* affine_raw /*12 limbs*/, uint8_t out[48]);

}  // namespace pbh
