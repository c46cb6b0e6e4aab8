"""TEST INFRASTRUCTURE - a plain big-integer BLS12-381 pairing, the oracle of the device pairing
(plonk_b200/csrc/pairing.cuh) and of the Verifier's final check.

Written for being obviously correct rather than fast:
- Fp12 is Fp2[w] / (w^6 - xi) with xi = u + 1, stored as six Fp2 coefficients of w^0 .. w^5.  It is the same
  field as the device's tower Fp2[v][w] with v = w^2.
- G2 lives on the M-twist y^2 = x^3 + 4 xi over Fp2 and is carried into E(Fp12) by psi(x, y) = (x / w^2, y / w^3).
- The optimal ate pairing is the textbook Miller loop f_{|x|, psi(Q)}(P) over the bits of |x|, with the chord and
  tangent lines evaluated in Fp12.  The points T run on the twist (psi is a group isomorphism), and the slope of
  psi(T) is taken as psi's image of the twisted slope, lambda = lambda' / w.  Vertical lines lie in a proper
  subfield and are dropped; the final exponentiation removes them.
- The final exponentiation is a direct pow by (p^12 - 1) / r, and x < 0 conjugates the result.

The device follows zkcrypto's final exponentiation, whose hard part raises to 3 (p^4 - p^2 + 1) / r: its value is
the cube of this one (checked by test_pairing_oracle.py).  Neither the reference nor its dependencies hold golden
bytes for a Gt value, the G2 encoding or the G2 generator, so these are restated from the curve's published
parameters and the zcash encoding, not pinned by a reference vector.  The sign convention of Gt (a conjugation)
does not change any verdict: the verifier compares a product of pairings with 1.

Only tests/ may import this file."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

from oracle import pyref as R

P = R.P_MOD
Q_R = R.R_MOD
BLS_X = 0xD201000000010000  # |x|; x is negative

Fp2 = Tuple[int, int]
G2 = Optional[Tuple[Fp2, Fp2]]  # affine; None is the identity

# the standard generator of G2 (x = x0 + x1 u, y = y0 + y1 u)
G2_GEN = (
    (0x024AA2B2F08F0A91260805272DC51051C6E47AD4FA403B02B4510B647AE3D1770BAC0326A805BBEFD48056C8C121BDB8,
     0x13E02B6052719F607DACD3A088274F65596BD0D09920B61AB5DA61BBDC7F5049334CF11213945D57E5AC7D055D042B7E),
    (0x0CE5D527727D6E118CC9CDC6DA2E351AADFD9BAA8CBDD3A76D429A695160D12C923AC9CC3BACA289E193548608B82801,
     0x0606C4A02EA734CC32ACD2B02BC28B99CB3E287E85A763AF267492AB572E99AB3F370D275CEC1DA1AAA9075FF05F79BE),
)


# ---- Fp2 ------------------------------------------------------------------------------------------------------
def f2_add(a: Fp2, b: Fp2) -> Fp2:
    return ((a[0] + b[0]) % P, (a[1] + b[1]) % P)


def f2_sub(a: Fp2, b: Fp2) -> Fp2:
    return ((a[0] - b[0]) % P, (a[1] - b[1]) % P)


def f2_neg(a: Fp2) -> Fp2:
    return (-a[0] % P, -a[1] % P)


def f2_mul(a: Fp2, b: Fp2) -> Fp2:
    return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)


def f2_inv(a: Fp2) -> Fp2:
    t = pow(a[0] * a[0] + a[1] * a[1], P - 2, P)
    return (a[0] * t % P, -a[1] * t % P)


def f2_scale(a: Fp2, k: int) -> Fp2:
    return (a[0] * k % P, a[1] * k % P)


XI = (1, 1)
ZERO2, ONE2 = (0, 0), (1, 0)
B2 = f2_scale(XI, 4)


def _fp_sqrt(a: int) -> Optional[int]:
    s = pow(a, (P + 1) // 4, P)
    return s if s * s % P == a % P else None


def f2_sqrt(a: Fp2) -> Optional[Fp2]:
    """Square root through the norm: (x0 + x1 u)^2 = a gives x0^2 = (a0 + sqrt(a0^2 + a1^2)) / 2, x1 = a1 / (2 x0)."""
    a0, a1 = a
    if a1 == 0:
        s = _fp_sqrt(a0)
        if s is not None:
            return (s, 0)
        s = _fp_sqrt(-a0 % P)
        return None if s is None else (0, s)
    n = _fp_sqrt((a0 * a0 + a1 * a1) % P)
    if n is None:
        return None
    inv2 = pow(2, P - 2, P)
    for cand in ((a0 + n) * inv2 % P, (a0 - n) * inv2 % P):
        x0 = _fp_sqrt(cand)
        if x0:
            x1 = a1 * pow(2 * x0, P - 2, P) % P
            r = (x0, x1)
            if f2_mul(r, r) == (a0 % P, a1 % P):
                return r
    return None


def _lex_largest(a: int) -> bool:
    return a > (P - 1) // 2


def f2_lex_largest(a: Fp2) -> bool:
    return _lex_largest(a[1]) or (a[1] == 0 and _lex_largest(a[0]))


# ---- G2 -------------------------------------------------------------------------------------------------------
def g2_on_curve(q: G2) -> bool:
    if q is None:
        return True
    x, y = q
    return f2_mul(y, y) == f2_add(f2_mul(f2_mul(x, x), x), B2)


def g2_add(p: G2, q: G2) -> G2:
    if p is None:
        return q
    if q is None:
        return p
    if p[0] == q[0]:
        if f2_add(p[1], q[1]) == ZERO2:
            return None
        lam = f2_mul(f2_scale(f2_mul(p[0], p[0]), 3), f2_inv(f2_scale(p[1], 2)))
    else:
        lam = f2_mul(f2_sub(q[1], p[1]), f2_inv(f2_sub(q[0], p[0])))
    x3 = f2_sub(f2_sub(f2_mul(lam, lam), p[0]), q[0])
    return (x3, f2_sub(f2_mul(lam, f2_sub(p[0], x3)), p[1]))


def g2_neg(q: G2) -> G2:
    return None if q is None else (q[0], f2_neg(q[1]))


def g2_mul(q: G2, k: int) -> G2:
    acc: G2 = None
    for bit in bin(k)[2:] if k > 0 else "":
        acc = g2_add(acc, acc)
        if bit == "1":
            acc = g2_add(acc, q)
    return acc


def g2_compress(q: G2) -> bytes:
    if q is None:
        return bytes([0xC0]) + bytes(95)
    x, y = q
    b = bytearray(x[1].to_bytes(48, "big") + x[0].to_bytes(48, "big"))
    b[0] |= 0x80 | (0x20 if f2_lex_largest(y) else 0)
    return bytes(b)


def g2_decompress(b: bytes) -> G2:
    """G2Affine::from_compressed with the on-curve and subgroup checks; ValueError for a rejected encoding."""
    if len(b) != 96:
        raise ValueError("length")
    flags = b[0]
    x1 = int.from_bytes(bytes([b[0] & 0x1F]) + b[1:48], "big")
    x0 = int.from_bytes(b[48:], "big")
    if not flags & 0x80:
        raise ValueError("not compressed")
    if flags & 0x40:
        if x0 or x1 or flags & 0x20:
            raise ValueError("non-canonical identity")
        return None
    if x0 >= P or x1 >= P:
        raise ValueError("non-canonical coordinate")
    x = (x0, x1)
    y = f2_sqrt(f2_add(f2_mul(f2_mul(x, x), x), B2))
    if y is None:
        raise ValueError("not on the curve")
    if f2_lex_largest(y) != bool(flags & 0x20):
        y = f2_neg(y)
    q = (x, y)
    if g2_mul(q, Q_R) is not None:
        raise ValueError("not in the prime-order subgroup")
    return q


# ---- Fp12 = Fp2[w] / (w^6 - xi) -------------------------------------------------------------------------------
Fp12 = List[Fp2]
ONE12: Fp12 = [ONE2] + [ZERO2] * 5


def f12_mul(a: Fp12, b: Fp12) -> Fp12:
    t = [ZERO2] * 11
    for i in range(6):
        if a[i] == ZERO2:
            continue
        for j in range(6):
            t[i + j] = f2_add(t[i + j], f2_mul(a[i], b[j]))
    return [f2_add(t[k], f2_mul(XI, t[k + 6])) if k + 6 < 11 else t[k] for k in range(6)]


def f12_pow(a: Fp12, e: int) -> Fp12:
    r = ONE12
    for bit in bin(e)[2:]:
        r = f12_mul(r, r)
        if bit == "1":
            r = f12_mul(r, a)
    return r


def f12_conj(a: Fp12) -> Fp12:
    """a^(p^6): w^(p^6) = -w."""
    return [c if k % 2 == 0 else f2_neg(c) for k, c in enumerate(a)]


def f12_mono(c: Fp2, k: int) -> Fp12:
    out = [ZERO2] * 6
    out[k] = c
    return out


def f12_from_fp(c: int) -> Fp12:
    return f12_mono((c % P, 0), 0)


def f12_sub(a: Fp12, b: Fp12) -> Fp12:
    return [f2_sub(x, y) for x, y in zip(a, b)]


XI_INV = f2_inv(XI)
W_INV = f12_mono(XI_INV, 5)  # w^-1 = w^5 / xi


def psi(q: Tuple[Fp2, Fp2]) -> Tuple[Fp12, Fp12]:
    x, y = q
    return f12_mono(f2_mul(x, XI_INV), 4), f12_mono(f2_mul(y, XI_INV), 3)  # x w^4 / xi = x / w^2, y w^3 / xi = y / w^3


def _line(t: Tuple[Fp2, Fp2], lam2: Fp2, p: Tuple[int, int]) -> Fp12:
    """l(P) = y_P - y_T - lambda (x_P - x_T) for T = psi(t) and lambda = lam2 / w."""
    xt, yt = psi(t)
    lam = f12_mul(f12_mono(lam2, 0), W_INV)
    return f12_sub(f12_sub(f12_from_fp(p[1]), yt), f12_mul(lam, f12_sub(f12_from_fp(p[0]), xt)))


def miller_loop(p, q: G2) -> Fp12:
    """f_{|x|, psi(Q)}(P) for an affine G1 point p (None: the identity) and G2 point q."""
    if p is None or q is None:
        return ONE12
    f, t = ONE12, q
    for bit in bin(BLS_X)[3:]:
        lam = f2_mul(f2_scale(f2_mul(t[0], t[0]), 3), f2_inv(f2_scale(t[1], 2)))
        f = f12_mul(f12_mul(f, f), _line(t, lam, p))
        t = g2_add(t, t)
        if bit == "1":
            lam = f2_mul(f2_sub(q[1], t[1]), f2_inv(f2_sub(q[0], t[0])))
            f = f12_mul(f, _line(t, lam, p))
            t = g2_add(t, q)
    return f


FINAL_EXP = (P ** 12 - 1) // Q_R


def final_exponentiation(f: Fp12) -> Fp12:
    return f12_conj(f12_pow(f, FINAL_EXP))  # x < 0


def pairing(p, q: G2) -> Fp12:
    return final_exponentiation(miller_loop(p, q))


def pairing_product_is_one(pairs: Sequence[Tuple[object, G2]]) -> bool:
    f = ONE12
    for p, q in pairs:
        f = f12_mul(f, miller_loop(p, q))
    return final_exponentiation(f) == ONE12


def f12_to_tower_mont_words(a: Fp12) -> List[int]:
    """The device layout: c0.c0, c0.c1, c0.c2, c1.c0, c1.c1, c1.c2 (w^0, w^2, w^4, w^1, w^3, w^5), each Fp2 as
    c0 then c1, each Fp as 6 little-endian u64 Montgomery limbs."""
    out: List[int] = []
    for k in (0, 2, 4, 1, 3, 5):
        for c in a[k]:
            m = c * R.FP_MONT_R % P
            out += [(m >> (64 * i)) & ((1 << 64) - 1) for i in range(6)]
    return out


# ---- opening keys ---------------------------------------------------------------------------------------------
def opening_key_bytes(g, h: G2, x_h: G2) -> bytes:
    """OpeningKey::to_bytes (key.rs:560-572): g, h, [x]h compressed."""
    return R.g1_compress(g) + g2_compress(h) + g2_compress(x_h)


def opening_key_from_secret(x: int, g_scalar: int, h_scalar: int) -> bytes:
    g = R.g1_mul(R.G1_GEN, g_scalar)
    h = g2_mul(G2_GEN, h_scalar)
    return opening_key_bytes(g, h, g2_mul(h, x % Q_R))


def srs_setup_with_opening_key(max_degree: int, rng: "R.StdRng", keep: Optional[int] = None):
    """PublicParameters::setup (srs.rs:61-100, util.rs:50-60) replayed, opening key included: the draws are x,
    the G1 scalar, then the G2 scalar.  Returns (powers_of_g, OpeningKey::to_bytes); powers_of_g equals what
    pyref.srs_setup returns for the same RNG."""
    assert max_degree >= 1
    x = R.random_nonzero_bls_scalar(rng)
    gs = R.random_nonzero_bls_scalar(rng)
    hs = R.random_nonzero_bls_scalar(rng)
    n = max_degree + R.ADDED_BLINDING_DEGREE + 1
    pts = R.srs_from_secret(min(n, keep or n), x, gs)
    return pts, opening_key_from_secret(x, gs, hs)


def parse_opening_key(b: bytes):
    return R.g1_decompress(b[:48]), g2_decompress(b[48:144]), g2_decompress(b[144:240])


# ---- the verifier's final check and its byte format ----------------------------------------------------------
def verify_with_pairing(proof: bytes, label: bytes, constraints: int, key_comms, pi_idx, pi_vals, opening_key: bytes) -> bool:
    """Proof::verify ending with the reference's pairing check e(-(W_z + u W_zw), [x]H) e(R, H) == 1
    (proof.rs:498-513) instead of the SRS secret.  The scalars and the two G1 points are those of
    oracle/verify.py, read off its two multi-scalar multiplications."""
    from oracle import verify as V

    g, h, x_h = parse_opening_key(opening_key)
    seen = []
    msm = V._msm

    calls = []

    def spy(points, scalars):
        calls.append(list(points))
        seen.append(msm(points, scalars))
        return seen[-1]

    V._msm = spy
    try:
        V.verify_with_secret(proof, label, constraints, key_comms, pi_idx, pi_vals, g, 1)
    finally:
        V._msm = msm
    if not calls:  # z inside the domain: rejected before the pairing
        return False
    # verify_with_secret forms right_projective, then W_z + u W_zw; fail loudly if that ever changes
    comm, _ = V.parse_proof(proof)
    assert len(calls) == 2 and calls[1] == [comm["w_z"], comm["w_zw"]], "oracle/verify.py no longer forms the two points as expected"
    right, left = seen
    return pairing_product_is_one([(R.g1_neg(left) if left is not None else None, x_h), (right, h)])


FILE_ORDER = ["q_m", "q_l", "q_r", "q_o", "q_f", "q_c", "q_arith", "q_logic", "q_range", "q_fixed_group_add",
              "q_variable_group_add", "s_sigma_1", "s_sigma_2", "s_sigma_3", "s_sigma_4"]


def verifier_to_bytes(label: bytes, n: int, size: int, constraints: int, comms_by_name, opening_key: bytes, pi_idx) -> bytes:
    """Verifier::to_bytes (verifier.rs:62-121) with VerifierKey::to_bytes (widget.rs:84-111); comms_by_name holds
    the compressed commitments by pyref.POLY_NAMES name.  n is VerifierKey::n, which Compiler::compile sets to the
    constraint count (compiler.rs:278-279), and size = constraints.next_power_of_two()."""
    vk = n.to_bytes(8, "little") + b"".join(comms_by_name[k] for k in FILE_ORDER)
    vk += bytes(20 * 48 + 8 - len(vk))
    head = b"".join(v.to_bytes(8, "big") for v in (len(label), len(vk), len(opening_key), len(pi_idx), size, constraints))
    return head + label + vk + opening_key + b"".join(i.to_bytes(8, "big") for i in pi_idx)


def _g2_bytes_for(x: Fp2) -> bytes:
    b = bytearray(x[1].to_bytes(48, "big") + x[0].to_bytes(48, "big"))
    b[0] |= 0x80
    return bytes(b)


def off_curve_g2_bytes() -> bytes:
    """A canonical x for which x^3 + 4 xi has no square root."""
    k = 1
    while f2_sqrt(f2_add(f2_mul(f2_mul((k, 1), (k, 1)), (k, 1)), B2)) is not None:
        k += 1
    return _g2_bytes_for((k, 1))


def non_subgroup_g2_bytes() -> bytes:
    """A point of the twist outside the subgroup of order r (the cofactor is large, so the first x on the curve)."""
    k = 1
    while True:
        x = (k, 2)
        y = f2_sqrt(f2_add(f2_mul(f2_mul(x, x), x), B2))
        if y is not None and g2_mul((x, y), Q_R) is not None:
            return _g2_bytes_for(x)
        k += 1
