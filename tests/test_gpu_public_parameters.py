"""PublicParameters::setup and Compiler::compile on the GPU (pb200_public_parameters_setup, pb200_opening_key_check,
plonk_b200.PublicParameters / Compiler) against the reference's setup replayed by tests/models/pairing_model.py and
oracle/serialize.py, and the reference's examples/circuit.rs and tests/opening_key_validation.rs."""
import ctypes
import random

import pytest

import plonk_b200
from oracle import cref
from oracle import pyref as R
from oracle import serialize as S
from plonk_b200 import gadgets as native_gadgets
from plonk_b200._lib import PB200_ERR_INVALID_ARG, PB200_ERR_POINT_MALFORMED, Pb200Error, check, lib
from tests.models import pairing_model as M

pytestmark = pytest.mark.gpu


def _draws(rng):
    """The three util::random_nonzero_bls_scalar draws of PublicParameters::setup, in order: x, g_scalar, h_scalar."""
    return [R.random_nonzero_bls_scalar(rng) for _ in range(3)]


def _mont(draws):
    return [R.fr_to_mont_bytes(d) for d in draws]


# every seed at the small degrees; two at 2^10, where the Python replay of the key is the slow part
@pytest.mark.parametrize("seed,max_degree", [(s, d) for d in (1, 5) for s in (0, 7, 0x9235E700)] + [(0, 1 << 10), (0x9235E700, 1 << 10)])
def test_setup_matches_the_reference_rng(seed, max_degree):
    pts, okey = M.srs_setup_with_opening_key(max_degree, R.StdRng.seed_from_u64(seed))
    pp = plonk_b200.PublicParameters.setup(max_degree, _mont(_draws(R.StdRng.seed_from_u64(seed))))
    assert pp.max_degree() == max_degree + 6
    assert pp.opening_key == okey
    assert pp.to_var_bytes() == okey + b"".join(R.g1_compress(p) for p in pts)
    assert pp.to_raw_var_bytes() == okey + S.commit_key_to_raw_var_bytes(pts)
    # and back: both loaders give the same parameters
    assert plonk_b200.PublicParameters.from_slice(pp.to_var_bytes()).raw_points == pp.raw_points
    back = plonk_b200.PublicParameters.from_slice_unchecked(pp.to_raw_var_bytes())
    assert back.raw_points == pp.raw_points and back.opening_key == okey


def test_old_and_new_setup_agree():
    x, gs, hs = _draws(R.StdRng.seed_from_u64(3))
    pp = plonk_b200.PublicParameters.setup(300, _mont([x, gs, hs]))
    n = 300 + 7
    out = ctypes.create_string_buffer(96 * n)
    check(lib().pb200_srs_setup_from_secret(R.fr_to_mont_bytes(x), R.fr_to_mont_bytes(gs), n, out))
    assert out.raw == pp.raw_points
    assert pp.opening_key == M.opening_key_from_secret(x, gs, hs)


def _sample_indices(n, rng):
    """First, last, the boundaries of the kernel's per-thread runs (up to 32 points) and of its 128-thread CTAs, and
    random indices: about 100."""
    idx = {0, 1, n - 1, n - 2}
    for run in (1, 2, 8, 16, 32):
        for k in (1, 127, 128, 129, 1000):
            for d in (-1, 0, 1):
                i = run * k + d
                if 0 <= i < n:
                    idx.add(i)
    idx.update(rng.randrange(n) for _ in range(30))
    return sorted(idx)


@pytest.mark.parametrize("log_n", [20, 24])
def test_large_keys(log_n):
    rng = random.Random(log_n)
    x, gs, hs = (rng.randrange(1, R.R_MOD) for _ in range(3))
    max_degree = 1 << log_n
    n = max_degree + 7
    pp = plonk_b200.PublicParameters.setup(max_degree, _mont([x, gs, hs]))
    raw = pp.raw_points
    assert len(raw) == 96 * n
    for i in _sample_indices(n, rng):
        assert raw[96 * i : 96 * i + 96] == R.g1_to_raw_bytes(R.g1_mul(R.G1_GEN, gs * pow(x, i, R.R_MOD) % R.R_MOD)), i
    # every point takes part in one commitment: sum_i c_i [gs x^i] G = [gs p(x)] G
    key = pp.commit_key()
    if log_n == 20:
        coeffs = [rng.randrange(R.R_MOD) for _ in range(n)]
        px = 0
        for c in reversed(coeffs):
            px = (px * x + c) % R.R_MOD
        poly = R.fr_vec_to_mont_bytes(coeffs)
    else:  # all-ones coefficients: p(x) = (x^n - 1) / (x - 1)
        px = (pow(x, n, R.R_MOD) - 1) * pow(x - 1, R.R_MOD - 2, R.R_MOD) % R.R_MOD
        poly = R.fr_to_mont_bytes(1) * n
    assert key.commit(poly).to_bytes() == R.g1_compress(R.g1_mul(R.G1_GEN, gs * px % R.R_MOD))


def test_setup_errors():
    one = R.fr_to_mont_bytes(1)
    with pytest.raises(plonk_b200.DegreeIsZero):
        plonk_b200.PublicParameters.setup(0, [one, one, one])
    for k in range(3):
        draws = [one, one, one]
        draws[k] = bytes(32)
        with pytest.raises(Pb200Error) as e:
            plonk_b200.PublicParameters.setup(4, draws)
        assert e.value.code == PB200_ERR_INVALID_ARG
    with pytest.raises(plonk_b200.NotEnoughBytes):
        plonk_b200.PublicParameters.from_slice(bytes(240))
    with pytest.raises(plonk_b200.NotEnoughBytes):
        plonk_b200.PublicParameters.from_slice(b"\x01" * 100)


# ---- Compiler.compile --------------------------------------------------------------------------------------------
def example_circuit(c, a=31, b=0, cc=73, d=42, e=1, f=None):
    """examples/circuit.rs TestCircuit::circuit with main()'s values."""
    f = f or native_gadgets.jubjub_generator()
    wa, wb, wd = c.append_witness(a), c.append_witness(b), c.append_witness(d)
    c.component_range_bits(wa, 6)
    c.component_range_bits(wb, 4)
    result = c.gate_add(dict(q_l=1, q_r=1, q_c=42), a=wa, b=wb)
    wc = c.append_public(cc)
    c.assert_equal(result, wc)
    result = c.gate_mul(dict(q_m=1, q_f=1), a=wa, b=wb, d=wd)
    c.assert_equal_constant(result, 42)
    we = c.append_witness(e)
    c.assert_equal_public_point(c.component_mul_generator(we, native_gadgets.jubjub_generator()), f)


def _blinders(seed):
    return cref.draw_blinders(R.StdRng.seed_from_u64(seed))


def test_example_circuit_end_to_end():
    rng = R.StdRng.seed_from_u64(0xC1C)
    x, gs, hs = _draws(rng)
    pp = plonk_b200.PublicParameters.setup(1 << 12, _mont([x, gs, hs]))
    label = b"transcript-arguments"
    prover, verifier = plonk_b200.Compiler.compile_with_circuit(pp, label, example_circuit)
    comp = native_gadgets.Composer.initialized()
    example_circuit(comp)
    a = comp.arrays()
    f = native_gadgets.jubjub_generator()
    assert a.pi_vals == R.fr_vec_to_mont_bytes([73, f[0], f[1]])  # public_inputs = [c, f.u, f.v]
    proof = prover.prove(a.witnesses, a.pi_idx, a.pi_vals, _blinders(1))
    verifier.verify(proof, a.pi_vals)
    with pytest.raises(plonk_b200.ProofVerificationError):
        verifier.verify(proof, R.fr_vec_to_mont_bytes([74, f[0], f[1]]))
    # the same Verifier and Prover as built by hand from the same draws and raw points
    old_v = plonk_b200.Verifier(label, a.constraints, prover.commitments(), M.opening_key_from_secret(x, gs, hs), a.pi_idx)
    assert verifier.to_bytes() == old_v.to_bytes()
    old_p = plonk_b200.Prover(label, a.constraints, a.selectors, a.wires, a.n_witnesses, pp.raw_points)
    assert prover.to_bytes() == old_p.to_bytes()
    # compile with a filled composer gives the same keys
    p2, v2 = plonk_b200.Compiler.compile(pp, label, comp)
    assert v2.to_bytes() == verifier.to_bytes()


def sum_circuit(c, a=2, b=3, claimed=5):
    """tests/opening_key_validation.rs SumCircuit."""
    wa, wb = c.append_public(a), c.append_public(b)
    out = c.gate_add(dict(q_l=1, q_r=1), a=wa, b=wb)
    c.assert_equal(out, c.append_public(claimed))


def _identity_g1():
    return b"\xc0" + bytes(47)


def _identity_g2():
    return b"\xc0" + bytes(95)


def test_opening_key_validation():
    rng = R.StdRng.seed_from_u64(0x1D3E1717)
    pp = plonk_b200.PublicParameters.setup(1 << 5, _mont(_draws(rng)))
    prover, verifier = plonk_b200.Compiler.compile_with_circuit(pp, b"opening-key-validation", sum_circuit)
    comp = native_gadgets.Composer.initialized()
    sum_circuit(comp)
    a = comp.arrays()
    proof = prover.prove(a.witnesses, a.pi_idx, a.pi_vals, cref.draw_blinders(rng))
    verifier.verify(proof, a.pi_vals)
    forged = b"".join(_identity_g1() for _ in range(11)) + bytes(15 * 32)
    with pytest.raises(plonk_b200.ProofVerificationError):
        verifier.verify(forged, R.fr_vec_to_mont_bytes([2, 3, 9]))

    vb = verifier.to_bytes()
    off = 48 + int.from_bytes(vb[0:8], "big") + int.from_bytes(vb[8:16], "big")
    pb = pp.to_var_bytes()
    rb = pp.to_raw_var_bytes()
    bad_keys = [
        _identity_g1() + pp.opening_key[48:],
        pp.opening_key[:48] + _identity_g2() + pp.opening_key[144:],
        pp.opening_key[:144] + _identity_g2(),
        pp.opening_key[:48] + M.non_subgroup_g2_bytes() + pp.opening_key[144:],
        pp.opening_key[:144] + M.off_curve_g2_bytes(),
        _off_curve_g1() + pp.opening_key[48:],
    ]
    for bad in bad_keys:
        with pytest.raises(Pb200Error) as e:  # Verifier::try_from_bytes: InvalidData
            plonk_b200.Verifier.from_bytes(vb[:off] + bad + vb[off + 240 :])
        assert e.value.code == PB200_ERR_POINT_MALFORMED
        with pytest.raises(plonk_b200.PointMalformed):
            plonk_b200.PublicParameters.from_slice(bad + pb[240:])
        with pytest.raises(plonk_b200.PointMalformed):
            plonk_b200.PublicParameters.from_slice_unchecked(bad + rb[240:])
        assert lib().pb200_opening_key_check(bad) == PB200_ERR_POINT_MALFORMED
    assert lib().pb200_opening_key_check(pp.opening_key) == 0
    # a malformed commit-key point: from_slice refuses it, from_slice_unchecked does not look
    with pytest.raises(plonk_b200.PointMalformed):
        plonk_b200.PublicParameters.from_slice(pb[:240 + 48 * 3] + _off_curve_g1() + pb[240 + 48 * 4 :])


def _off_curve_g1():
    """A canonical x for which x^3 + 4 has no square root in Fp."""
    k = 1
    while pow((k ** 3 + 4) % R.P_MOD, (R.P_MOD - 1) // 2, R.P_MOD) == 1:
        k += 1
    b = bytearray(k.to_bytes(48, "big"))
    b[0] |= 0x80
    return bytes(b)


def test_truncated_degree_boundary():
    comp = native_gadgets.Composer.initialized()
    sum_circuit(comp)
    n = 1 << (comp.constraints() + 6 - 1).bit_length()  # next_pow2(constraints + 6)
    draws = _mont([0x1234567, 0x7654321, 0xABCDEF])
    small = plonk_b200.PublicParameters.setup(n - 1, draws)
    assert small.max_degree() == n + 5
    with pytest.raises(plonk_b200.TruncatedDegreeTooLarge):
        plonk_b200.Compiler.compile(small, b"t", comp)
    exact = plonk_b200.PublicParameters.setup(n, draws)
    assert exact.max_degree() == n + 6
    plonk_b200.Compiler.compile(exact, b"t", comp)
