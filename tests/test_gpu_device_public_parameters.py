"""DevicePublicParameters on the GPU (pb200_pp_*, pb200_prover_*_pp): one PublicParameters resident in HBM whose
derived MSM tables are shared by every prover compiled from it.  Provers compiled, compressed or reloaded through it are
byte for byte those of the host PublicParameters; setup and the loaders give the host loaders' points and errors; the
cache holds one table per trimmed-key size and per domain size, outlives nothing it should not and is built once under
concurrent compiles."""
import gc
import random
import threading

import pytest

import plonk_b200
from oracle import cref
from oracle import pyref as R
from plonk_b200 import gadgets as N
from plonk_b200._lib import PB200_ERR_INVALID_ARG, Pb200Error, check, lib
from tests.test_gpu_public_parameters import _off_curve_g1, example_circuit, sum_circuit

pytestmark = pytest.mark.gpu

LABEL = b"device-public-parameters"


def _draws(seed):
    rng = R.StdRng.seed_from_u64(seed)
    return [R.fr_to_mont_bytes(R.random_nonzero_bls_scalar(rng)) for _ in range(3)]


@pytest.fixture(scope="module")
def host_pp():
    check(lib().pb200_init(0))
    return plonk_b200.PublicParameters.setup(1 << 14, _draws(0xD0))


def _keep_points(constraints):
    """The trimmed key's point count: next_pow2(constraints + 6) + 7."""
    return (1 << (constraints + 6 - 1).bit_length()) + 7


def arith_circuit(constraints, seed):
    """A seeded circuit of arithmetic gates only, exactly `constraints` gates long."""

    def build(c):
        rng = random.Random(seed)
        acc = c.append_witness(rng.randrange(R.R_MOD))
        while c.constraints() < constraints:
            w = c.append_witness(rng.randrange(R.R_MOD))
            acc = c.gate_add(dict(q_l=rng.randrange(1, 1 << 20), q_r=rng.randrange(1, 1 << 20), q_c=rng.randrange(1 << 20)), a=acc, b=w)

    return build


def _bench(degree):
    return lambda c: c.bench_circuit(degree)


def _arrays(circuit):
    comp = N.Composer.initialized()
    circuit(comp)
    return comp, comp.arrays()


def _compile(pp, circuit, compressed):
    if compressed:
        return plonk_b200.Compiler.compile_with_compressed(pp, LABEL, plonk_b200.compress(circuit))
    return plonk_b200.Compiler.compile_with_circuit(pp, LABEL, circuit)


# n = 1024 with 1021 gates: next_pow2(1027) = 2048, so keep + 1 = 2n + 7
CASES = [("example", example_circuit, False), ("bench_2^12", _bench(1 << 12), False),
         ("arith_2n+7", arith_circuit(1021, 5), False), ("compressed_bench_2^12", _bench(1 << 12), True)]


@pytest.mark.parametrize("name,circuit,compressed", CASES, ids=[c[0] for c in CASES])
def test_device_pp_compiles_what_the_host_pp_compiles(host_pp, name, circuit, compressed):
    comp, a = _arrays(circuit)
    if name == "arith_2n+7":
        assert a.constraints == 1021 and _keep_points(a.constraints) == 2 * 1024 + 7
    dpp = plonk_b200.DevicePublicParameters.from_host(host_pp)
    hp, hv = _compile(host_pp, circuit, compressed)
    dp, dv = _compile(dpp, circuit, compressed)
    assert dp.commitments() == hp.commitments()
    assert dp.to_bytes() == hp.to_bytes()
    assert dv.to_bytes() == hv.to_bytes()
    for seed in (1, 2):
        blinders = cref.draw_blinders(R.StdRng.seed_from_u64(seed))
        proof = dp.prove(a.witnesses, a.pi_idx, a.pi_vals, blinders)
        assert proof == hp.prove(a.witnesses, a.pi_idx, a.pi_vals, blinders)
        dv.verify(proof, a.pi_vals)
        hv.verify(proof, a.pi_vals)


# ---- construction ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("max_degree", [1, 5, 1 << 10])
def test_setup_matches_the_host_setup(max_degree):
    draws = _draws(max_degree)
    host = plonk_b200.PublicParameters.setup(max_degree, draws)
    dpp = plonk_b200.DevicePublicParameters.setup(max_degree, draws)
    assert dpp.max_degree() == host.max_degree() == max_degree + 6
    assert dpp.opening_key == host.opening_key
    back = dpp.to_host()
    assert back.raw_points == host.raw_points and back.opening_key == host.opening_key


def test_loaders_match_the_host_loaders(host_pp):
    checked = plonk_b200.DevicePublicParameters.from_slice(host_pp.to_var_bytes()).to_host()
    assert checked.raw_points == host_pp.raw_points and checked.opening_key == host_pp.opening_key
    unchecked = plonk_b200.DevicePublicParameters.from_slice_unchecked(host_pp.to_raw_var_bytes()).to_host()
    assert unchecked.raw_points == host_pp.raw_points and unchecked.opening_key == host_pp.opening_key


def _non_subgroup_g1():
    """The compressed encoding of the first curve point (smallest x) outside the prime-order subgroup."""
    x = 1
    while True:
        rhs = (x ** 3 + 4) % R.P_MOD
        y = pow(rhs, (R.P_MOD + 1) // 4, R.P_MOD)
        if y * y % R.P_MOD == rhs and R.jac_to_affine(R.jac_mul(R.jac_from_affine((x, y)), R.R_MOD)) is not None:
            return R.g1_compress((x, y))
        x += 1


def test_loader_errors():
    host = plonk_b200.PublicParameters.setup(1 << 4, _draws(9))
    pb, rb = host.to_var_bytes(), host.to_raw_var_bytes()
    at = 240 + 48 * 3
    bad_slices = [pb[:at] + _off_curve_g1() + pb[at + 48 :], pb[:at] + _non_subgroup_g1() + pb[at + 48 :],
                  b"\xc0" + bytes(47) + pb[48:], pb[:-1]]
    for bad in bad_slices:
        with pytest.raises(plonk_b200.PointMalformed):
            plonk_b200.PublicParameters.from_slice(bad)
        with pytest.raises(plonk_b200.PointMalformed):
            plonk_b200.DevicePublicParameters.from_slice(bad)
    with pytest.raises(plonk_b200.PointMalformed):  # the opening key is checked by the unchecked loader too
        plonk_b200.DevicePublicParameters.from_slice_unchecked(b"\xc0" + bytes(47) + rb[48:])
    for short in (b"", pb[:240]):
        with pytest.raises(plonk_b200.NotEnoughBytes):
            plonk_b200.DevicePublicParameters.from_slice(short)
    with pytest.raises(plonk_b200.NotEnoughBytes):
        plonk_b200.DevicePublicParameters.from_slice_unchecked(rb[:239])
    one = R.fr_to_mont_bytes(1)
    with pytest.raises(plonk_b200.DegreeIsZero):
        plonk_b200.DevicePublicParameters.setup(0, [one, one, one])
    with pytest.raises(Pb200Error) as e:
        plonk_b200.DevicePublicParameters.setup(4, [one, bytes(32), one])
    assert e.value.code == PB200_ERR_INVALID_ARG


# ---- sharing -----------------------------------------------------------------------------------------------------
def test_tables_are_shared_per_size(host_pp):
    dpp = plonk_b200.DevicePublicParameters.from_host(host_pp)
    assert dpp.tables() == (0, 0, 0)
    keep = []
    keep.append(_compile(dpp, arith_circuit(600, 1), False))
    one = dpp.tables()
    assert (one.monomial, one.lagrange) == (1, 1) and one.device_bytes > 0
    keep.append(_compile(dpp, arith_circuit(700, 2), False))  # same n = 1024 and keep + 1 = 1031
    assert dpp.tables() == one
    keep.append(_compile(dpp, arith_circuit(300, 3), False))  # n = 512: one more pair
    assert dpp.tables()[:2] == (2, 2)
    keep.append(_compile(dpp, arith_circuit(1021, 4), False))  # n = 1024, keep + 1 = 2055: a monomial table only
    assert dpp.tables()[:2] == (3, 2)
    # freeing and recompiling a size builds nothing new
    keep.clear()
    gc.collect()
    _compile(dpp, arith_circuit(650, 6), False)
    assert dpp.tables()[:2] == (3, 2)


def test_second_compile_allocates_no_tables(host_pp):
    torch = pytest.importorskip("torch")
    first_circuit, second_circuit = arith_circuit(10000, 7), arith_circuit(12000, 8)  # n = 2^14
    _compile(host_pp, first_circuit, False)  # warm-up: the scratch pool grows to this size once
    gc.collect()
    dpp = plonk_b200.DevicePublicParameters.from_host(host_pp)

    def growth(circuit):
        check(lib().pb200_device_sync())
        before = torch.cuda.mem_get_info()[0]
        pair = _compile(dpp, circuit, False)
        check(lib().pb200_device_sync())
        return before - torch.cuda.mem_get_info()[0], pair

    first, p1 = growth(first_circuit)
    shared = dpp.tables().device_bytes
    second, p2 = growth(second_circuit)
    assert dpp.tables().device_bytes == shared
    assert first - second >= shared, (first, second, shared)


# ---- lifetime and concurrency ------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", ["first_then_second", "second_then_first"])
def test_provers_outlive_the_device_pp(host_pp, order):
    circuits = [arith_circuit(500, 11), _bench(1 << 10)]
    dpp = plonk_b200.DevicePublicParameters.from_host(host_pp)
    pairs = [_compile(dpp, c, False) for c in circuits]
    want = [_compile(host_pp, c, False)[0].to_bytes() for c in circuits]
    del dpp
    gc.collect()
    blinders = cref.draw_blinders(R.StdRng.seed_from_u64(3))
    for (prover, verifier), circuit, blob in zip(pairs, circuits, want):
        _, a = _arrays(circuit)
        verifier.verify(prover.prove(a.witnesses, a.pi_idx, a.pi_vals, blinders), a.pi_vals)
        assert prover.to_bytes() == blob
    if order == "second_then_first":
        pairs.reverse()
    while pairs:
        pairs.pop(0)
        gc.collect()


def test_concurrent_compiles_build_one_table_pair(host_pp):
    circuit = _bench(1 << 12)
    comp, _ = _arrays(circuit)
    dpp = plonk_b200.DevicePublicParameters.from_host(host_pp)
    got, errors = [None] * 8, []

    def run(i):
        try:
            got[i] = plonk_b200.Compiler.compile(dpp, LABEL, comp)[0].commitments()
        except Exception as e:  # reported below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors
    assert all(g == got[0] for g in got)
    assert got[0] == plonk_b200.Compiler.compile(host_pp, LABEL, comp)[0].commitments()
    assert dpp.tables()[:2] == (1, 1)


# ---- reloading ---------------------------------------------------------------------------------------------------
def test_from_bytes_with_a_device_pp(host_pp):
    circuit = _bench(1 << 10)
    _, a = _arrays(circuit)
    prover, verifier = _compile(host_pp, circuit, False)
    blob = prover.to_bytes()
    dpp = plonk_b200.DevicePublicParameters.from_host(host_pp)
    plain = plonk_b200.Prover.from_bytes(blob, a.wires, a.n_witnesses)
    shared = plonk_b200.Prover.from_bytes(blob, a.wires, a.n_witnesses, pp=dpp)
    assert shared.commitments() == plain.commitments() == prover.commitments()
    assert shared.to_bytes() == plain.to_bytes() == blob
    blinders = cref.draw_blinders(R.StdRng.seed_from_u64(4))
    proof = shared.prove(a.witnesses, a.pi_idx, a.pi_vals, blinders)
    assert proof == plain.prove(a.witnesses, a.pi_idx, a.pi_vals, blinders)
    verifier.verify(proof, a.pi_vals)
    assert dpp.tables()[:2] == (1, 1)
    # a prover saved under other public parameters
    other = plonk_b200.DevicePublicParameters.setup(1 << 11, _draws(0xD1))
    with pytest.raises(Pb200Error) as e:
        plonk_b200.Prover.from_bytes(blob, a.wires, a.n_witnesses, pp=other)
    assert e.value.code == PB200_ERR_INVALID_ARG and "prefix" in str(e.value)
    # truncated blobs fail as they do without a pp
    for cut in (0, 47, 48 + len(LABEL) + 100, len(blob) - 8 - 15 * 48 - 1, len(blob) - 1):
        codes = []
        for kw in ({}, {"pp": dpp}):
            with pytest.raises(Pb200Error) as e:
                plonk_b200.Prover.from_bytes(blob[:cut], a.wires, a.n_witnesses, **kw)
            codes.append(e.value.code)
        assert codes[0] == codes[1], cut


# ---- bounds ------------------------------------------------------------------------------------------------------
def test_truncated_degree_boundary():
    comp = N.Composer.initialized()
    sum_circuit(comp)
    n = 1 << (comp.constraints() + 6 - 1).bit_length()  # next_pow2(constraints + 6)
    draws = _draws(0xB0)
    small = plonk_b200.DevicePublicParameters.setup(n - 1, draws)
    with pytest.raises(plonk_b200.TruncatedDegreeTooLarge):
        plonk_b200.Compiler.compile(small, b"t", comp)
    assert small.tables() == (0, 0, 0)
    exact = plonk_b200.DevicePublicParameters.setup(n, draws)
    assert exact.max_degree() == n + 6
    plonk_b200.Compiler.compile(exact, b"t", comp)
