// Device Fp inversion shared by the MSM (affine batch inversions) and the verifier (pairing tower and affine
// normalisation).
#pragma once
#include "bigint.cuh"

namespace pb {

#if defined(__CUDACC__)
// (aR)^-1 R for a Montgomery residue aR != 0, by the binary extended Euclidean algorithm (shifts, adds and
// subtractions only; data-dependent control flow, meant for ONE lane).  0 -> 0.
static __device__ __noinline__ Fp fp_inv_bingcd(Fp a) {
  if (a.is_zero()) return a;
  uint32_t u[12], v[12], x1[12], x2[12];
#pragma unroll
  for (int i = 0; i < 12; i++) {
    u[i] = a.v[i];
    v[i] = FpParams::MOD(i);
    x1[i] = i == 0 ? 1u : 0u;
    x2[i] = 0u;
  }
  auto is_one = [](const uint32_t* t) {
    uint32_t x = t[0] ^ 1u;
#pragma unroll
    for (int i = 1; i < 12; i++) x |= t[i];
    return x == 0;
  };
  auto halve = [](uint32_t* t, uint32_t* x) {  // t even: t /= 2, x = x / 2 mod p
#pragma unroll
    for (int i = 0; i < 11; i++) t[i] = __funnelshift_r(t[i], t[i + 1], 1);
    t[11] >>= 1;
    const uint32_t m = 0u - (x[0] & 1u);  // odd: add p first (x + p < 2^382)
    x[0] = add_cc(x[0], FpParams::MOD(0) & m);
#pragma unroll
    for (int i = 1; i < 11; i++) x[i] = addc_cc(x[i], FpParams::MOD(i) & m);
    x[11] = addc(x[11], FpParams::MOD(11) & m);
#pragma unroll
    for (int i = 0; i < 11; i++) x[i] = __funnelshift_r(x[i], x[i + 1], 1);
    x[11] >>= 1;
  };
  auto sub_mod = [](uint32_t* x, const uint32_t* y) {  // x = x - y mod p
    x[0] = sub_cc(x[0], y[0]);
#pragma unroll
    for (int i = 1; i < 12; i++) x[i] = subc_cc(x[i], y[i]);
    const uint32_t m = subc(0u, 0u);  // all ones on borrow
    x[0] = add_cc(x[0], FpParams::MOD(0) & m);
#pragma unroll
    for (int i = 1; i < 11; i++) x[i] = addc_cc(x[i], FpParams::MOD(i) & m);
    x[11] = addc(x[11], FpParams::MOD(11) & m);
  };
#pragma unroll 1
  while (!is_one(u) && !is_one(v)) {
#pragma unroll 1
    while (!(u[0] & 1u)) halve(u, x1);
#pragma unroll 1
    while (!(v[0] & 1u)) halve(v, x2);
    uint32_t t[12];
    t[0] = sub_cc(u[0], v[0]);
#pragma unroll
    for (int i = 1; i < 12; i++) t[i] = subc_cc(u[i], v[i]);
    const uint32_t borrow = subc(0u, 0u);
    if (borrow == 0u) {  // u >= v
#pragma unroll
      for (int i = 0; i < 12; i++) u[i] = t[i];
      sub_mod(x1, x2);
    } else {
      v[0] = sub_cc(v[0], u[0]);
#pragma unroll
      for (int i = 1; i < 12; i++) v[i] = subc_cc(v[i], u[i]);
      sub_mod(x2, x1);
    }
  }
  Fp y;
  const bool from_u = is_one(u);
#pragma unroll
  for (int i = 0; i < 12; i++) y.v[i] = from_u ? x1[i] : x2[i];
  return (y * Fp::r2()) * Fp::r2();  // (aR)^-1 -> (aR)^-1 R^2 = a^-1 R
}
#endif

}  // namespace pb
