"""Compiler.compile_with_compressed on the GPU (pb200_prover_from_compressed): for the reference's DummyCircuit
(tests/composer.rs:19-84), SparseWitnessCircuit (compress.rs), every native gadget circuit and BenchCircuit, the Prover
and Verifier compiled from compress(circuit) are the ones Compiler.compile makes - to_bytes, commitments and proofs byte
for byte - and the sparse-label descriptions of compress.rs compile without allocating per claimed witness."""
import ctypes
import hashlib
import threading

import pytest

import plonk_b200
from oracle import cref
from oracle import pyref as R
from plonk_b200 import gadgets as N
from plonk_b200._lib import PB200_ERR_INVALID_ARG, PB200_ERR_INVALID_COMPRESSED, Pb200Error, PlonkVersion, check, lib
from tests.models import compress_model as M
from tests.test_compressed_circuit_cpu import dummy_circuit, sparse_witness_circuit
from tests.test_gpu_gadget_circuits import CASES

pytestmark = pytest.mark.gpu

LABEL = b"compressed-circuit"


@pytest.fixture(scope="module")
def pp():
    check(lib().pb200_init(0))
    draws = [R.fr_to_mont_bytes(R.random_nonzero_bls_scalar(R.StdRng.seed_from_u64(0xC0C0 + k))) for k in range(3)]
    return plonk_b200.PublicParameters.setup(1 << 17, draws)


def _bench(degree):
    return lambda c: c.bench_circuit(degree)


def _gadget(build, default):
    return lambda c: build(c, *default)


CIRCUITS = ([("dummy", dummy_circuit), ("sparse_witness", sparse_witness_circuit)]
            + [("gadget_" + name, _gadget(build, default)) for name, build, default, _, _ in CASES]
            + [("bench_2^%d" % k, _bench(1 << k)) for k in (5, 13, 16)])


def _digest(b):
    return hashlib.sha256(b).digest()


def _tamper(proof):
    return proof[:-1] + bytes([proof[-1] ^ 1])


@pytest.mark.parametrize("name,circuit", CIRCUITS, ids=[c[0] for c in CIRCUITS])
def test_compressed_compile_matches_compile(pp, name, circuit):
    comp = N.Composer.initialized()
    circuit(comp)
    a = comp.arrays()
    prover, verifier = plonk_b200.Compiler.compile(pp, LABEL, comp)
    data = plonk_b200.compress(circuit)
    cprover, cverifier = plonk_b200.Compiler.compile_with_compressed(pp, LABEL, data)
    assert cprover.commitments() == prover.commitments()
    assert cverifier.to_bytes() == verifier.to_bytes()
    assert _digest(cprover.to_bytes()) == _digest(prover.to_bytes())
    assert cprover.n_witnesses == a.n_witnesses
    for k, version in enumerate((PlonkVersion.V3, PlonkVersion.V2)):
        blinders = cref.draw_blinders(R.StdRng.seed_from_u64(31 + k))
        proof = cprover.prove_with_version(version, a.witnesses, a.pi_idx, a.pi_vals, blinders)
        assert proof == prover.prove_with_version(version, a.witnesses, a.pi_idx, a.pi_vals, blinders)
        cverifier.verify_with_version(proof, a.pi_vals, version)
        if a.n_pi:
            wrong = R.fr_to_mont_bytes((R.fr_from_mont_bytes(a.pi_vals[:32]) + 1) % R.R_MOD) + a.pi_vals[32:]
            with pytest.raises(plonk_b200.ProofVerificationError):
                cverifier.verify_with_version(proof, wrong, version)
        else:
            with pytest.raises((plonk_b200.ProofVerificationError, plonk_b200.PointMalformed)):
                cverifier.verify_with_version(_tamper(proof), a.pi_vals, version)


def test_python_zlib_stream_compiles(pp):
    comp = N.Composer.initialized()
    dummy_circuit(comp)
    prover, _ = plonk_b200.Compiler.compile(pp, LABEL, comp)
    ours = plonk_b200.compress(dummy_circuit)
    theirs = M.deflate(M.inflate(ours), 1)
    assert theirs != ours
    cprover, _ = plonk_b200.Compiler.compile_with_compressed(pp, LABEL, theirs)
    assert _digest(cprover.to_bytes()) == _digest(prover.to_bytes())


def _direct_outcome(prover, *args):
    try:
        return prover.prove(*args)
    except plonk_b200.CircuitUnsatisfied:
        return "CircuitUnsatisfied"


def test_sparse_labels_compile_and_prove():
    """compress.rs compiler_accepts_sparse_witness_labels: one gate whose d wire is label 10^6 - 1 compiles under
    PublicParameters::setup(8), and labels up to 2^40 compile.  Proofs take the circuit's own 10^6-entry table; each
    compressed prover answers as pb200_prover_new on the same circuit does."""
    draws = [R.fr_to_mont_bytes(v) for v in (3, 5, 7)]
    small = plonk_b200.PublicParameters.setup(8, draws)
    witnesses = 10**6
    zero = R.fr_to_mont_bytes(0)
    pi_idx = (0).to_bytes(8, "little")
    table = zero * witnesses
    blinders = cref.draw_blinders(R.StdRng.seed_from_u64(4))
    for gates, pp in ((1, small), (8, plonk_b200.PublicParameters.setup(32, draws))):
        c = M.sample(witnesses=witnesses, constraints=[(0, 0, 0, 0, witnesses - 1)] + [(0, 0, 0, 0, 0)] * (gates - 1))
        prover, verifier = plonk_b200.Compiler.compile_with_compressed(pp, b"bounded-circuit", M.encode(c))
        assert prover.n_witnesses == witnesses and prover.n_constraints == gates
        wires = b"".join(w.to_bytes(4, "little") for w in [0] * (3 * gates) + [witnesses - 1] + [0] * (gates - 1))
        direct = plonk_b200.Prover(b"bounded-circuit", gates, bytes(11 * 32 * gates), wires, witnesses, pp.raw_points)
        assert prover.to_bytes() == direct.to_bytes()
        want = _direct_outcome(direct, table, pi_idx, zero, blinders)
        assert _direct_outcome(prover, table, pi_idx, zero, blinders) == want
        if gates == 8:  # a domain of eight rows holds the blinders; the proof verifies
            verifier.verify(want, zero)
            with pytest.raises(plonk_b200.ProofVerificationError):
                verifier.verify(want, R.fr_to_mont_bytes(1))
            # the table must be the circuit's own length
            rc = lib().pb200_prove(prover._h, zero * 2, 2, pi_idx, zero, 1, blinders, ctypes.create_string_buffer(1008))
            assert rc == PB200_ERR_INVALID_ARG
    # labels up to 2^40: nothing is sized by the claimed count
    data = M.encode(M.sample(witnesses=1 << 40, constraints=[(0, 0, 0, 0, (1 << 40) - 1)]))
    prover, _ = plonk_b200.Compiler.compile_with_compressed(small, b"bounded-circuit", data)
    assert prover.n_witnesses == 1 << 40


def test_public_parameters_too_small(pp):
    data = plonk_b200.compress(dummy_circuit)
    draws = [R.fr_to_mont_bytes(v) for v in (3, 5, 7)]
    small = plonk_b200.PublicParameters.setup(1 << 8, draws)
    with pytest.raises(plonk_b200.InvalidCompressedCircuit):
        plonk_b200.Compiler.compile_with_compressed(small, LABEL, data)
    h = ctypes.c_void_p()
    rc = lib().pb200_prover_from_compressed(LABEL, len(LABEL), data, len(data), small.raw_points, len(small.raw_points) // 96,
                                           ctypes.byref(h))
    assert rc == PB200_ERR_INVALID_COMPRESSED and not h.value


def test_error_kinds(pp):
    with pytest.raises(plonk_b200.BlsScalarMalformed):
        plonk_b200.Compiler.compile_with_compressed(pp, LABEL, M.encode(M.sample(scalars=[R.R_MOD.to_bytes(32, "little")])))
    with pytest.raises(plonk_b200.InvalidCompressedCircuit):
        plonk_b200.Compiler.compile_with_compressed(pp, LABEL, b"\x00garbage")
    # a description without gates fails as an empty circuit does in pb200_prover_new
    with pytest.raises(Pb200Error) as e:
        plonk_b200.Compiler.compile_with_compressed(pp, LABEL, M.encode(M.Compressed()))
    assert e.value.code == PB200_ERR_INVALID_ARG and "empty circuit" in str(e.value)


def test_threads_share_one_compressed_prover(pp):
    comp = N.Composer.initialized()
    dummy_circuit(comp)
    a = comp.arrays()
    prover, verifier = plonk_b200.Compiler.compile_with_compressed(pp, LABEL, plonk_b200.compress(dummy_circuit))
    blinders = cref.draw_blinders(R.StdRng.seed_from_u64(77))
    want = prover.prove(a.witnesses, a.pi_idx, a.pi_vals, blinders)
    verifier.verify(want, a.pi_vals)
    got, errors = [None] * 6, []

    def run(i):
        try:
            got[i] = [prover.prove(a.witnesses, a.pi_idx, a.pi_vals, blinders) for _ in range(3)]
        except Exception as e:  # reported below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(6)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors
    assert all(p == want for ps in got for p in ps)
