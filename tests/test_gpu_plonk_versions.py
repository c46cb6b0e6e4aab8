"""PlonkVersion V1, V2 and V3 on the device: pb200_prove_with_version, pb200_verify_with_version and the Python and
C++ mirrors, against the version-aware oracle of tests/models/plonk_versions_model.py."""
import ctypes
import os
import random
import struct
import subprocess

import pytest

import plonk_b200
from oracle import cref
from oracle import pyref as R
from plonk_b200 import PlonkVersion
from plonk_b200 import gadgets as native_gadgets
from plonk_b200._lib import PB200_ERR_INVALID_ARG, PB200_ERR_UNSUPPORTED_VERSION, PB200_ERR_VERIFY, Pb200Error, lib
from tests.models import pairing_model as M
from tests.models import plonk_versions_model as PV
from tests.test_gpu_verifier import Case, _mutations, _synthetic
from tests.test_host_logic import _build_cpp
from tests.util import bases_to_abi

OK = 0
V1, V2, V3 = PlonkVersion.V1, PlonkVersion.V2, PlonkVersion.V3
X, GS, HS = 0x1234567, 0x7654321, 0xABCDEF  # the secrets of tests/test_gpu_verifier.py's Case


def _idx(arr):
    return [int.from_bytes(arr.pi_idx[8 * i : 8 * i + 8], "little") for i in range(arr.n_pi)]


def _oracle(case, proof, version, arr=None):
    a = arr or case.arrays
    comms = {k: R.g1_decompress(c) for k, c in zip(R.POLY_NAMES, case.comms)}
    return PV.verify_with_secret(proof, case.label, case.arrays.constraints, comms, _idx(a), R.fr_vec_from_mont_bytes(a.pi_vals),
                                 R.g1_mul(R.G1_GEN, GS), X, version)


def _v1(case, v2_proof):
    """The V1 proof of a GPU V2 proof's witness (the library refuses to make V1 proofs, as the reference does)."""
    comms = {k: R.g1_decompress(c) for k, c in zip(R.POLY_NAMES, case.comms)}
    return PV.v1_from_v2_with_secret(v2_proof, case.label, case.arrays.constraints, comms, R.fr_vec_from_mont_bytes(case.arrays.pi_vals),
                                     R.g1_mul(R.G1_GEN, GS), X)


def _prove(case, seed, version):
    a = case.arrays
    return case.prover.prove_with_version(version, a.witnesses, a.pi_idx, a.pi_vals, cref.draw_blinders(R.StdRng.seed_from_u64(seed)))


def _three(case, seed):
    """One proof of each version for the same blinders."""
    v2 = _prove(case, seed, V2)
    return {V1: _v1(case, v2), V2: v2, V3: _prove(case, seed, V3)}


@pytest.fixture(scope="module")
def case():
    return Case(b"gpu-versions", _synthetic(300, 31))


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [5, 8, 10])
def test_v2_proofs_equal_the_oracle_byte_for_byte(log_n):
    comp = R.Composer.initialized()
    R.synthetic_arith_circuit(comp, (1 << log_n) - 12, seed=200 + log_n, n_public=3, widgets=1 if log_n == 5 else 9)
    arr = cref.CircuitArrays(comp)
    c = Case(b"v2-synthetic-%d" % log_n, arr)
    n = 1 << (arr.constraints + 6 - 1).bit_length()
    pd = R.compile_circuit(R.srs_from_secret(n + 7, X, GS), c.label, comp)
    want = PV.prove(pd, R.StdRng.seed_from_u64(7), comp, 2)
    assert _prove(c, 7, V2) == want
    assert c.verifier.verify_batch([want], [arr.pi_vals], V2) == [OK]


@pytest.mark.gpu
def test_v2_proof_of_the_golden_digest_circuit_equals_the_oracle():
    pp = R.srs_setup(1 << 10, R.StdRng.seed_from_u64(0x9235E700), keep=64)
    comp = R.Composer.initialized()
    R.minimal_circuit(comp)
    pd = R.compile_circuit(pp, b"proof-compatibility", comp)
    arr = cref.CircuitArrays(comp)
    prover = plonk_b200.Prover(b"proof-compatibility", arr.constraints, arr.selectors, arr.wires, arr.n_witnesses, bases_to_abi(pp))
    blinders = cref.draw_blinders(R.StdRng.seed_from_u64(0x9235E701))
    got = prover.prove_with_version(V2, arr.witnesses, arr.pi_idx, arr.pi_vals, blinders)
    assert got == PV.prove(pd, R.StdRng.seed_from_u64(0x9235E701), comp, 2)
    assert prover.prove_with_version(V3, arr.witnesses, arr.pi_idx, arr.pi_vals, blinders) == R.kat_proof()


def _mul_circuit(comp):
    """MulCircuit of tests/plonk_versioning.rs."""
    a, b, expected = comp.append_witness(3), comp.append_witness(4), comp.append_witness(12)
    out = comp.gate_evaluated(dict(q_m=1), a=a, b=b)
    comp.assert_equal(out, expected)


@pytest.mark.gpu
def test_plonk_versioning_restated():
    """tests/plonk_versioning.rs with legacy-proving: V1 proving is UnsupportedProvingVersion; V2 and V3 proofs verify
    under their own version only."""
    rng = R.StdRng.seed_from_u64(0xC0FFEE)
    pp, okey = M.srs_setup_with_opening_key(1 << 9, rng)
    comp = R.Composer.initialized()
    _mul_circuit(comp)
    arr = cref.CircuitArrays(comp)
    prover = plonk_b200.Prover(b"versioned", arr.constraints, arr.selectors, arr.wires, arr.n_witnesses, bases_to_abi(pp))
    verifier = plonk_b200.Verifier(b"versioned", arr.constraints, prover.commitments(), okey, arr.pi_idx)
    with pytest.raises(plonk_b200.UnsupportedProvingVersion) as e:
        prover.prove_with_version(V1, arr.witnesses, arr.pi_idx, arr.pi_vals, bytes(14 * 32))
    assert e.value.__cause__.code == PB200_ERR_UNSUPPORTED_VERSION == -12
    for made, other in ((V2, V3), (V3, V2)):
        proof = prover.prove_with_version(made, arr.witnesses, arr.pi_idx, arr.pi_vals, cref.draw_blinders(rng))
        verifier.verify_with_version(proof, arr.pi_vals, made)
        with pytest.raises(plonk_b200.ProofVerificationError):
            verifier.verify_with_version(proof, arr.pi_vals, other)


@pytest.mark.gpu
def test_version_matrix_matches_the_oracle(case):
    proofs = _three(case, 3)
    assert _oracle(case, proofs[V1], V1), "the V1 proof made from the V2 one must be V1-valid"
    for made, proof in proofs.items():
        want = [OK if _oracle(case, proof, v) else PB200_ERR_VERIFY for v in (V1, V2, V3)]
        assert want == [OK if v == made else PB200_ERR_VERIFY for v in (V1, V2, V3)], made
        assert [case.verifier.verify_batch([proof], [case.arrays.pi_vals], v)[0] for v in (V1, V2, V3)] == want, made


@pytest.mark.gpu
def test_version_matrix_on_the_bench_circuit():
    arr = native_gadgets.bench_circuit(1 << 13).arrays()
    c = Case(b"dusk-network", arr)
    proofs = _three(c, 5)
    for made, proof in proofs.items():
        assert [c.verifier.verify_batch([proof], [arr.pi_vals], v)[0] for v in (V1, V2, V3)] == \
            [OK if v == made else PB200_ERR_VERIFY for v in (V1, V2, V3)], made


@pytest.mark.gpu
def test_forged_proof_is_accepted_under_v1_only():
    comp = R.Composer.initialized()
    PV.arith_circuit(comp, 3, 5, 7, 11)
    arr = cref.CircuitArrays(comp)
    n = 1 << (arr.constraints + 6 - 1).bit_length()
    pd = R.compile_circuit(R.srs_from_secret(n + 7, X, GS), b"soundness_test", comp)
    forged = PV.forge_proof(pd, comp, R.StdRng.seed_from_u64(0xDEADBEEF))
    okey = M.opening_key_from_secret(X, GS, HS)
    v = plonk_b200.Verifier(b"soundness_test", arr.constraints, [R.g1_compress(pd.comms[k]) for k in R.POLY_NAMES], okey, arr.pi_idx)
    want = [OK if PV.verify_with_secret(forged, b"soundness_test", arr.constraints, pd.comms, comp.public_input_indexes(), comp.public_inputs_vec(),
                                        pd.commit_key[0], X, ver) else PB200_ERR_VERIFY for ver in (1, 2, 3)]
    assert want == [OK, PB200_ERR_VERIFY, PB200_ERR_VERIFY]
    assert [v.verify_batch([forged], [arr.pi_vals], ver)[0] for ver in (V1, V2, V3)] == want


@pytest.mark.gpu
def test_every_single_mutation_of_v1_and_v2_proofs_is_rejected(case):
    proofs = _three(case, 9)
    for version in (V1, V2):
        muts = _mutations(case, proofs[version])
        got = case.verifier.verify_batch([m[1] for m in muts], [case.arrays.pi_vals] * len(muts), version)
        assert got == [m[2] for m in muts], (version, [(m[0], g) for m, g in zip(muts, got) if g != m[2]])


@pytest.mark.gpu
def test_batches(case):
    proofs = _three(case, 11)
    muts = _mutations(case, proofs[V1])
    rng = random.Random(3)
    batch = [proofs[V1]] + [rng.choice([proofs[V2], proofs[V3], proofs[V1]] + [m[1] for m in muts]) for _ in range(63)]
    pis = [case.arrays.pi_vals] * len(batch)
    mixed = case.verifier.verify_batch(batch, pis, V1)
    assert mixed[0] == OK == case.verifier.verify_batch([proofs[V1]], [case.arrays.pi_vals], V1)[0]
    assert mixed == [case.verifier.verify_batch([b], [p], V1)[0] for b, p in zip(batch, pis)]
    # pb200_verify_with_version(V3) is pb200_verify
    n = len(batch)
    st_a, st_b = (ctypes.c_int32 * n)(), (ctypes.c_int32 * n)()
    assert lib().pb200_verify(case.verifier._h, b"".join(batch), n, b"".join(pis), case.arrays.n_pi, st_a) == 0
    assert lib().pb200_verify_with_version(case.verifier._h, 3, b"".join(batch), n, b"".join(pis), case.arrays.n_pi, st_b) == 0
    assert list(st_a) == list(st_b) and OK in list(st_a) and PB200_ERR_VERIFY in list(st_a)


@pytest.mark.gpu
def test_construction_and_arguments(case):
    proofs = _three(case, 13)
    w = plonk_b200.Verifier.from_bytes(case.verifier.to_bytes())
    assert [w.verify_batch([proofs[v]], [case.arrays.pi_vals], v)[0] for v in (V1, V2, V3)] == [OK] * 3
    a = case.arrays
    st = (ctypes.c_int32 * 1)()
    for bad in (0, 4):
        assert lib().pb200_verify_with_version(case.verifier._h, bad, proofs[V3], 1, a.pi_vals, a.n_pi, st) == PB200_ERR_INVALID_ARG
        with pytest.raises(Pb200Error) as e:
            case.prover.prove_with_version(bad, a.witnesses, a.pi_idx, a.pi_vals, cref.draw_blinders(R.StdRng.seed_from_u64(1)))
        assert e.value.code == PB200_ERR_INVALID_ARG
    for v in (V1, V2, V3):
        assert lib().pb200_verify_with_version(case.verifier._h, int(v), proofs[v], 1, a.pi_vals, a.n_pi - 1, st) == PB200_ERR_INVALID_ARG
        with pytest.raises(ValueError):  # InconsistentPublicInputsLen
            case.verifier.verify_with_version(proofs[v], a.pi_vals[:32], v)


def test_cpp_versions_check_compiles_and_links():
    assert os.path.exists(_build_cpp("versions_check"))


@pytest.mark.gpu
def test_cpp_mirror_versions(case, tmp_path):
    a = case.arrays
    blinders = [cref.draw_blinders(R.StdRng.seed_from_u64(s)) for s in (21, 22)]
    v1 = _v1(case, case.prover.prove_with_version(V2, a.witnesses, a.pi_idx, a.pi_vals, blinders[0]))
    n_srs = (1 << (a.constraints + 6 - 1).bit_length()) + 7
    srs = cref.srs_from_secret(n_srs, X, GS)  # the key Case proves with
    blob = struct.pack("<5Q", len(case.label), a.constraints, a.n_witnesses, a.n_pi, n_srs) + case.label
    blob += a.selectors + a.wires + a.witnesses + a.pi_idx + a.pi_vals + srs + b"".join(case.comms) + case.okey + blinders[0] + blinders[1] + v1
    f = tmp_path / "case.bin"
    f.write_bytes(blob)
    out = subprocess.run([_build_cpp("versions_check"), str(f)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.splitlines() == [
        "prove_v1 UnsupportedProvingVersion", "prove_v0 InvalidArgument",
        "v2_under_v2 ok", "v2_under_v3 ProofVerificationError", "v3_under_v3 ok", "v3_under_v2 ProofVerificationError",
        "v1_under_v1 ok", "v1_under_v2 ProofVerificationError", "v3_under_v1 ProofVerificationError",
        "batch_v1 0 -11 -11", "batch_v2 -11 0 -11", "batch_v3 -11 -11 0", "batch_default -11 -11 0",
        "from_bytes_v1 ok", "wrong_pi_count_v1 InvalidArgument",
    ]
