"""The redundant Fp type FpR (values in [0, 2p), products without the final subtraction) and the G1 formulas of
plonk_b200/csrc/g1.cuh that run on it, compiled for the host by g++ into tests/hosttest and checked against
Python big integers and the oracle's G1 arithmetic.  Every result is checked both for its value mod p and for
the range FpR promises."""
import ctypes
import itertools
import os
import random
import subprocess

import pytest

from oracle import pyref as R

HERE = os.path.dirname(os.path.abspath(__file__))
P = R.P_MOD
NB = 48
RM = 1 << 384
RINV = pow(RM, -1, P)
EDGE = [0, 1, P - 1, P, P + 1, 2 * P - 1]  # 2p - 1 is the largest allowed operand


@pytest.fixture(scope="module")
def rf():
    so = os.path.join(HERE, "hosttest", "libredundantfp.so")
    src = os.path.join(HERE, "hosttest", "redundant_fp.cpp")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-frounding-math", "-mfma", "-shared", "-fPIC", "-o", so, src])
    return ctypes.CDLL(so)


def _pack(xs):
    return b"".join(x.to_bytes(NB, "little") for x in xs)


def _op(rf, op, a, b=None, c=None, d=None):
    n = len(a)
    out = ctypes.create_string_buffer(n * NB)
    args = [_pack(v) if v is not None else None for v in (a, b, c, d)]
    assert rf.rf_op(op, *args, out, ctypes.c_size_t(n)) == 0
    return [int.from_bytes(out.raw[i * NB : (i + 1) * NB], "little") for i in range(n)]


def _check(got, want, bound=2 * P):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g < bound
        assert g % P == w % P


def _operands():
    rng = random.Random(2024)
    rand = [rng.randrange(2 * P) for _ in range(400)]
    pairs = list(itertools.product(EDGE, EDGE)) + [(rng.choice(rand), rng.choice(rand)) for _ in range(1500)]
    pairs += [(rng.choice(EDGE), x) for x in rand[:200]] + [(x, rng.choice(EDGE)) for x in rand[200:]]
    return [p[0] for p in pairs], [p[1] for p in pairs], rng


def test_unary_and_binary_ops(rf):
    a, b, _ = _operands()
    _check(_op(rf, 0, a, b), [x * y * RINV for x, y in zip(a, b)])
    _check(_op(rf, 1, a), [x * x * RINV for x in a])
    _check(_op(rf, 2, a, b), [x + y for x, y in zip(a, b)])
    _check(_op(rf, 3, a, b), [x - y for x, y in zip(a, b)])
    _check(_op(rf, 4, a), [-x for x in a])
    _check(_op(rf, 5, a), [2 * x for x in a])
    _check(_op(rf, 8, a), a, bound=P)  # canonical(): [0, p)
    assert _op(rf, 9, a) == [int(x % P == 0) for x in a]


def test_squaring_at_the_top_of_the_range(rf):
    """The squaring's row 0 adds a_0 * 2a at once: operands with every lower limb saturated below 2p."""
    top = (2 * P) >> (NB * 8 - 32)
    sq = [((top - k) << (NB * 8 - 32)) | ((1 << (NB * 8 - 32)) - 1) for k in (1, 2, 3)] + [2 * P - 1 - k for k in range(40)]
    _check(_op(rf, 1, sq), [x * x * RINV for x in sq])
    _check(_op(rf, 0, sq, sq[::-1]), [x * y * RINV for x, y in zip(sq, sq[::-1])])


def test_two_products_one_reduction(rf):
    a, b, rng = _operands()
    quads = [q for q in itertools.product(EDGE, repeat=4)] + [tuple(rng.choice(a + b) for _ in range(4)) for _ in range(1500)]
    cols = [[q[k] for q in quads] for k in range(4)]
    _check(_op(rf, 6, *cols), [(x * y + z * w) * RINV for x, y, z, w in quads])
    _check(_op(rf, 7, *cols), [(x * y - z * w) * RINV for x, y, z, w in quads])


def test_two_pipe_product_without_final_subtraction(rf):
    """Field::mul_hybrid / sqr_hybrid / mul2_hybrid<FULL = false> (the PB_FP_HYBRID builds of FpR)."""
    a, b, rng = _operands()
    c = [rng.choice(a) for _ in a]
    d = [rng.choice(b) for _ in b]
    _check(_op(rf, 10, a, b), [x * y * RINV for x, y in zip(a, b)])
    _check(_op(rf, 11, a), [x * x * RINV for x in a])
    _check(_op(rf, 12, a, b, c, d), [(x * y + z * w) * RINV for x, y, z, w in zip(a, b, c, d)])


# ---- G1 formulas -------------------------------------------------------------------------------------------


def _mont(x):
    return x * RM % P


def _xyzz(pt, lam, shift=(0, 0, 0, 0)):
    """XYZZ limbs of an affine point with ZZ = lam^2, ZZZ = lam^3; shift[k] = 1 gives coordinate k as value + p
    (the second representation of the same residue)."""
    if pt is None:
        return [0, 0, 0, 0]
    x, y = pt
    coords = [_mont(x * lam * lam), _mont(y * lam**3), _mont(lam * lam), _mont(lam**3)]
    return [c + P * s for c, s in zip(coords, shift)]


def _g1(rf, op, p_limbs, q):
    out_xyzz = ctypes.create_string_buffer(4 * NB)
    out_aff = ctypes.create_string_buffer(2 * NB)
    if op in (1, 3):
        qb = R.g1_to_raw_bytes(q)
    else:
        qb = _pack(q) if q is not None else None
    assert rf.rf_g1(op, _pack(p_limbs), qb, out_xyzz, out_aff) == 0
    limbs = [int.from_bytes(out_xyzz.raw[k * NB : (k + 1) * NB], "little") for k in range(4)]
    assert all(v < 2 * P for v in limbs)
    if limbs[2] % P == 0:  # only the identity has zz = 0 mod p, and then its limbs are zero
        assert limbs[2] == 0
    aff = out_aff.raw
    assert all(int.from_bytes(aff[k * NB : (k + 1) * NB], "little") < P for k in range(2))
    return R.g1_from_raw_bytes(aff)


SHIFTS = [(0, 0, 0, 0), (1, 1, 1, 1), (1, 0, 1, 0), (0, 1, 0, 1)]


def test_g1_formulas_against_the_oracle(rf):
    rng = random.Random(7)
    g = R.G1_GEN
    pts = [R.g1_mul(g, rng.randrange(1, R.R_MOD)) for _ in range(4)]
    for P1, Q1 in [(pts[0], pts[1]), (pts[2], pts[3])]:
        for s1, s2 in itertools.product(SHIFTS, SHIFTS):
            l1, l2 = rng.randrange(2, P), rng.randrange(2, P)
            a, b = _xyzz(P1, l1, s1), _xyzz(Q1, l2, s2)
            a_same = _xyzz(P1, l2, s2)  # P again, other Z and other representation: a hidden doubling
            a_neg = _xyzz(R.g1_neg(P1), l2, s2)
            # P + Q, P + P, P + (-P), identity on either side
            assert _g1(rf, 0, a, b) == R.g1_add(P1, Q1)
            assert _g1(rf, 0, a, a_same) == R.g1_add(P1, P1)
            assert _g1(rf, 0, a, a_neg) is None
            assert _g1(rf, 0, a, _xyzz(None, 0)) == P1
            assert _g1(rf, 0, _xyzz(None, 0), b) == Q1
            # mixed addition of an affine (canonical) point
            assert _g1(rf, 1, a, Q1) == R.g1_add(P1, Q1)
            assert _g1(rf, 1, a, P1) == R.g1_add(P1, P1)
            assert _g1(rf, 1, a, R.g1_neg(P1)) is None
            assert _g1(rf, 1, _xyzz(None, 0), Q1) == Q1
            # doubling
            assert _g1(rf, 2, a, None) == R.g1_add(P1, P1)
            assert _g1(rf, 2, _xyzz(None, 0), None) is None
        assert _g1(rf, 3, _xyzz(None, 0), P1) == R.g1_add(P1, P1)
