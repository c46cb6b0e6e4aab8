"""Every domain size from 2^4 to 2^17, and every MSM window width, against exact references.

Most launch shapes of the prover follow log n: the window width of the commit-key MSM (max(4, log n) up to 2^16 points)
and of the Lagrange-key MSM (min(12, that)), the NTT pass plan of the 4n-coset transforms, the block counts of the
8-point-coset fold (k_coset8_eval / k_coset8_sum) and of the round-4 evaluations, and the stages of the group-element
iNTT that builds the Lagrange key.  So a kernel that is wrong at one size is wrong for every circuit that lands on it.
These tests run each size with the configuration the library picks by itself and compare with the CPU prover byte for
byte, with closed forms, or with one scalar multiplication of known discrete log: all arithmetic is exact.
"""
import ctypes
import random

import pytest

import plonk_b200
from oracle import cref
from oracle import pyref as R
from plonk_b200._lib import check, lib
from tests.models import pairing_model as M
from tests.util import bases_to_abi, progression_bases, rand_fr, to_abi

LOG_SIZES = list(range(4, 18))  # the prover sweep: domains 2^4 .. 2^17
PP_SIZES = (4, 11, 15)  # also compiled through a DevicePublicParameters (the shared-table path)
BOUNDARY_SIZES = (6, 11, 14)  # n - 5 constraints: the circuit moves to the domain 2n
LAGRANGE_SIZES = list(range(6, 17))
WINDOWS = list(range(2, 21))  # every width pb200_srs_upload_window accepts
X, GS, HS = 0x2F3B8C61D9A0475E16B2C8D4E7F9013A5C6D7E8F9A0B1C2D3E4F5061728394A, 0x51C7E3A9, 0xABCDEF  # SRS secrets
BLINDER_SEED = 0xD0A1


@pytest.fixture(scope="module")
def L():
    check(lib().pb200_init(0))
    return lib()


def _srs(L, n_points):
    """[GS X^i] G for i < n_points, made on the device."""
    out = ctypes.create_string_buffer(96 * n_points)
    check(L.pb200_srs_setup_from_secret(R.fr_to_mont_bytes(X), R.fr_to_mont_bytes(GS), n_points, out))
    return out.raw


def _circuit(constraints, seed):
    """A satisfied circuit of exactly `constraints` gates with public inputs at the first and the last gate.
    Composer::initialized would take gate 0 for its constant gates, so the zero witness is appended by hand and the
    two public-input gates bracket the seeded arithmetic gates (with rows of every widget family where they fit)."""
    rng = random.Random(seed)
    widgets = 0 if constraints < 26 else min(12, constraints.bit_length() - 4)
    comp = R.Composer()
    comp.append_witness(0)  # witness 0: what every unused wire points at
    comp.append_public(rng.randrange(R.R_MOD))
    R.synthetic_arith_circuit(comp, constraints - 1, seed=seed, n_public=0, widgets=widgets)
    comp.append_public(rng.randrange(R.R_MOD))
    assert len(comp.constraints) == constraints and comp.public_input_indexes() == [0, constraints - 1]
    return cref.CircuitArrays(comp)


def _prove_everywhere(L, label, arrays, n_points, with_pp):
    """The CPU prover's commitments and proof, and the GPU prover's in both throughput modes (and through a
    DevicePublicParameters); the GPU proof is then verified with the opening key of the same secrets."""
    srs = _srs(L, n_points)
    okey = M.opening_key_from_secret(X, GS, HS)
    cpu = cref.CrefProver(label, arrays, srs)
    want_comms = cpu.commitments()
    blinders = cref.draw_blinders(R.StdRng.seed_from_u64(BLINDER_SEED + arrays.constraints))
    want = cpu.prove(blinders)
    gpu = plonk_b200.Prover(label, arrays.constraints, arrays.selectors, arrays.wires, arrays.n_witnesses, srs)
    assert gpu.commitments() == want_comms
    prove = lambda p: p.prove(arrays.witnesses, arrays.pi_idx, arrays.pi_vals, blinders)
    try:
        for mode in (0, 1):
            check(L.pb200_throughput_mode(mode))
            assert prove(gpu) == want, "throughput mode %d" % mode
    finally:
        check(L.pb200_throughput_mode(0))
    if with_pp:
        dpp = plonk_b200.DevicePublicParameters.from_host(plonk_b200.PublicParameters(okey, srs))
        shared = plonk_b200.Prover(label, arrays.constraints, arrays.selectors, arrays.wires, arrays.n_witnesses, dpp)
        assert shared.commitments() == want_comms
        assert prove(shared) == want, "DevicePublicParameters"
    verifier = plonk_b200.Verifier(label, arrays.constraints, gpu.commitments(), okey, arrays.pi_idx)
    verifier.verify(want, arrays.pi_vals)


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", LOG_SIZES)
def test_prover_at_every_domain_size(L, log_n):
    """n - 6 constraints, the largest circuit of the domain n, with the n + 7 points of its trimmed key."""
    n = 1 << log_n
    arrays = _circuit(n - 6, seed=log_n)
    assert 1 << (arrays.constraints + 6 - 1).bit_length() == n
    _prove_everywhere(L, b"domain-2^%d" % log_n, arrays, n + 7, log_n in PP_SIZES)


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", BOUNDARY_SIZES)
def test_prover_one_gate_past_the_domain(L, log_n):
    """n - 5 constraints no longer fit with the blinding rows: the circuit is proved on the domain 2n."""
    n = 1 << log_n
    arrays = _circuit(n - 5, seed=100 + log_n)
    assert 1 << (arrays.constraints + 6 - 1).bit_length() == 2 * n
    _prove_everywhere(L, b"boundary-2^%d" % log_n, arrays, 2 * n + 7, False)


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", LAGRANGE_SIZES)
def test_lagrange_key_matches_closed_form(L, log_n):
    """pb200_g1_lagrange_key (the group-element iNTT, csrc/ecntt.cu) of [GS X^i] G, i < n, spot-checked against
    [L_j(X)] [GS] G with L_j(X) = (w^j / n) (X^n - 1) / (X - w^j): one scalar multiplication per entry."""
    n = 1 << log_n
    out = ctypes.create_string_buffer(96 * n)
    check(L.pb200_g1_lagrange_key(_srs(L, n), ctypes.c_size_t(n), out))
    w = R.EvaluationDomain(n).group_gen
    rng = random.Random(log_n)
    vanishing = (pow(X, n, R.R_MOD) - 1) % R.R_MOD
    n_inv = pow(n, -1, R.R_MOD)
    for j in [0, 1, n // 2, n - 1] + [rng.randrange(n) for _ in range(8)]:
        wj = pow(w, j, R.R_MOD)
        lj = wj * n_inv % R.R_MOD * vanishing % R.R_MOD * pow(X - wj, -1, R.R_MOD) % R.R_MOD
        got = R.g1_from_raw_bytes(out.raw[96 * j : 96 * j + 96])
        assert got == R.g1_mul(R.G1_GEN, GS * lj % R.R_MOD), (log_n, j)


def _digit_pattern(c, d):
    """Every c-bit window of the scalar's bits 0..253 holds d (so the value stays below r)."""
    s = 0
    for k in range(0, 254, c):
        s |= d << k
    return s & ((1 << 254) - 1)


def _msm_scalars(c, n, rng):
    """The scalar vectors of the window sweep, each with what it stresses."""
    half = 1 << (c - 1)
    bits = [rng.randrange(2) for _ in range(n)]
    return [
        [R.R_MOD - 1] * n,  # every window full, the top window at its largest value
        [_digit_pattern(c, half)] * n,  # every digit exactly half: kept positive, no carry
        [_digit_pattern(c, half + 1)] * n,  # every digit half + 1: negated, a carry into every next window
        [rng.randrange(R.R_MOD)] * n,  # one scalar: one bucket per window holds every point (heavy buckets)
        [0] * (n - 1) + [rng.randrange(1, R.R_MOD)],  # a single non-zero entry, at the last index
        bits,  # 0/1: only bucket 1 of window 0
        rand_fr(rng, n),
        rand_fr(rng, n),
    ]


@pytest.mark.gpu
@pytest.mark.parametrize("c", WINDOWS)
def test_msm_at_every_window_width(L, c):
    """A key of 3000 points [p0 + i step] G uploaded with window width c; batches of four vectors in one
    pb200_msm_g1 call with a stride past n, each equal to [sum_i s_i (p0 + i step)] G.  pb200_msm_g1 takes the same
    bytes in both throughput modes (the prover's throughput-shaped MSMs run at every width it picks in
    test_prover_at_every_domain_size)."""
    n, stride, batch = 3000, 3000 + 5, 4
    rng = random.Random(c)
    p0, step = rng.randrange(1, R.R_MOD), rng.randrange(1, R.R_MOD)
    pts = progression_bases(n, p0, step)
    vectors = _msm_scalars(c, n, rng)
    h = ctypes.c_void_p()
    check(L.pb200_srs_upload_window(bases_to_abi(pts), n, c, ctypes.byref(h)))
    try:
        assert L.pb200_srs_window(h) == c
        results = {}
        try:
            for mode in (0, 1):
                check(L.pb200_throughput_mode(mode))
                got = []
                for first in range(0, len(vectors), batch):
                    group = vectors[first : first + batch]
                    filler = [rng.randrange(1, R.R_MOD) for _ in range(stride - n)]  # must not be read
                    out = ctypes.create_string_buffer(96 * batch)
                    check(L.pb200_msm_g1(h, to_abi([s for v in group for s in v + filler]), n, batch, stride, out))
                    got += [out.raw[96 * k : 96 * k + 96] for k in range(batch)]
                results[mode] = got
        finally:
            check(L.pb200_throughput_mode(0))
    finally:
        L.pb200_srs_free(h)
    assert results[0] == results[1]
    for k, (v, raw) in enumerate(zip(vectors, results[0])):
        dlog = sum(s * (p0 + i * step) for i, s in enumerate(v)) % R.R_MOD
        assert R.g1_from_raw_bytes(raw) == R.g1_mul(R.G1_GEN, dlog), (c, k)


def test_domain_sweep_reaches_every_window_width():
    """The prover sweep above runs every window width the library picks for a circuit's keys: the trimmed key of
    n + 7 points takes 4..16, the Lagrange key of n + 4 points 4..12.  A change of pick_window that moves a width
    out of the sweep fails here, without a GPU."""
    window = lib().pb200_msm_window_for
    assert {window((1 << k) + 7) for k in LOG_SIZES} >= set(range(4, 17))
    assert {min(12, window((1 << k) + 4)) for k in LOG_SIZES} >= set(range(4, 13))
