"""Batch verification on the GPU (pb200_batch_verify, Verifier.batch_verify): one verdict for a batch, against the
per-proof verdicts of pb200_verify_with_version and the folded points of tests/models/batch_verify_model.py."""
import ctypes
import random
import threading

import pytest

import plonk_b200
from oracle import cref
from oracle import gadgets as G
from oracle import pyref as R
from plonk_b200 import gadgets as native_gadgets
from plonk_b200._lib import PB200_ERR_INVALID_ARG, PB200_ERR_POINT_MALFORMED, PB200_ERR_VERIFY, PlonkVersion, lib
from tests.models import batch_verify_model as BV
from tests.models import pairing_model as M
from tests.models import plonk_versions_model as PV
from tests.test_gpu_gadget_circuits import CASES as GADGET_CASES
from tests.test_gpu_plonk_versions import GS, _prove, _v1
from tests.test_gpu_verifier import Case, _mutations, _synthetic

pytestmark = pytest.mark.gpu
OK = 0
SIZES = (1, 2, 31, 32, 33, 257)


def _call(verifier, proofs, pis, version=3, points=False):
    """(return code, verdict, the selftest's 192 point bytes or None)."""
    n_pi = len(pis[0]) // 32 if pis else verifier.n_pi
    verdict = ctypes.c_int32(12345)
    args = (verifier._h, version, b"".join(proofs) or None, len(proofs), b"".join(pis) or None, n_pi, ctypes.byref(verdict))
    if not points:
        return lib().pb200_batch_verify(*args), verdict.value, None
    out = ctypes.create_string_buffer(192)
    rc = lib().pb200_selftest_batch_verify_points(*args, out)
    return rc, verdict.value, out.raw


def verdict(verifier, proofs, pis, version=3):
    rc, v, _ = _call(verifier, proofs, pis, version)
    assert rc == 0
    return v


def _expected(statuses):
    """The batch verdict that the per-proof statuses imply."""
    if all(s == OK for s in statuses):
        return OK
    return PB200_ERR_POINT_MALFORMED if PB200_ERR_POINT_MALFORMED in statuses else PB200_ERR_VERIFY


@pytest.fixture(scope="module")
def case():
    return Case(b"gpu-batch-verify", _synthetic(300, 11))


@pytest.fixture(scope="module")
def valid(case):
    return [case.prove(500 + k) for k in range(40)]


def test_valid_batches_of_every_size_are_accepted(case, valid):
    pi = case.arrays.pi_vals
    for n in SIZES:
        batch = [valid[k % len(valid)] for k in range(n)]
        assert verdict(case.verifier, batch, [pi] * n) == OK, n
    case.verifier.batch_verify(valid[:5], [pi] * 5)
    repeated = [valid[0]] * 64
    assert verdict(case.verifier, repeated, [pi] * 64) == OK


@pytest.mark.parametrize("name,build,default,satisfied,unsatisfied", GADGET_CASES, ids=[c[0] for c in GADGET_CASES])
def test_gadget_circuit_batches_are_accepted(name, build, default, satisfied, unsatisfied):
    comp = G.GadgetComposer.initialized()
    build(comp, *default)
    c = Case(name.encode(), cref.CircuitArrays(comp))
    proofs, pis = [], []
    for k, vals in enumerate([default] + satisfied):
        other = G.GadgetComposer.initialized()
        build(other, *vals)
        arr = cref.CircuitArrays(other)
        proofs.append(c.prove(600 + k, arr))
        pis.append(arr.pi_vals)
    assert verdict(c.verifier, proofs, pis) == OK
    if len(proofs) > 1:  # public inputs moved to another proof of the batch
        rot = pis[1:] + pis[:1]
        if rot != pis:
            assert verdict(c.verifier, proofs, rot) == _expected(c.verifier.verify_batch(proofs, rot))


def test_bench_circuit_and_golden_digest_batches_are_accepted():
    arr = native_gadgets.bench_circuit(1 << 13).arrays()
    c = Case(b"dusk-network", arr)
    assert verdict(c.verifier, [c.prove(1), c.prove(2)], [arr.pi_vals] * 2) == OK
    pp, okey = M.srs_setup_with_opening_key(1 << 10, R.StdRng.seed_from_u64(0x9235E700), keep=64)
    comp = R.Composer.initialized()
    R.minimal_circuit(comp)
    pd = R.compile_circuit(pp, b"proof-compatibility", comp)
    idx = b"".join(i.to_bytes(8, "little") for i in comp.public_input_indexes())
    v = plonk_b200.Verifier(b"proof-compatibility", len(comp.constraints), [R.g1_compress(pd.comms[k]) for k in R.POLY_NAMES], okey, idx)
    pi = R.fr_vec_to_mont_bytes(comp.public_inputs_vec())
    assert verdict(v, [R.kat_proof()], [pi]) == OK
    assert verdict(v, [R.kat_proof()] * 3, [pi] * 3) == OK
    v.batch_verify([R.kat_proof()], [pi])


def test_versions(case):
    pi = case.arrays.pi_vals
    v2 = [_prove(case, 700 + k, PlonkVersion.V2) for k in range(3)]
    v3 = [_prove(case, 710 + k, PlonkVersion.V3) for k in range(3)]
    assert verdict(case.verifier, v2, [pi] * 3, 2) == OK
    case.verifier.batch_verify(v2, [pi] * 3, PlonkVersion.V2)
    assert verdict(case.verifier, v3, [pi] * 3, 2) == PB200_ERR_VERIFY
    assert verdict(case.verifier, v2, [pi] * 3, 3) == PB200_ERR_VERIFY
    with pytest.raises(plonk_b200.ProofVerificationError):
        case.verifier.batch_verify(v3, [pi] * 3, PlonkVersion.V2)
    v1 = [_v1(case, p) for p in v2[:2]]
    for batch in (v1, v1 + v2[:1], v3[:2], v1 + v3[:1]):
        want = _expected(case.verifier.verify_batch(batch, [pi] * len(batch), PlonkVersion.V1))
        assert verdict(case.verifier, batch, [pi] * len(batch), 1) == want
    assert verdict(case.verifier, v1, [pi] * 2, 1) == OK


def _model_pair(case, proof, version=3):
    comms = {k: R.g1_decompress(c) for k, c in zip(R.POLY_NAMES, case.comms)}
    idx = [int.from_bytes(case.arrays.pi_idx[8 * i : 8 * i + 8], "little") for i in range(len(case.arrays.pi_idx) // 8)]
    vals = R.fr_vec_from_mont_bytes(case.arrays.pi_vals)
    right, left = PV.right_and_left(proof, case.label, case.arrays.constraints, comms, idx, vals, R.g1_mul(R.G1_GEN, GS), version)
    u = PV.challenges(proof, case.label, case.arrays.constraints, comms, vals, version)["u"]
    return u, (R.g1_neg(left), right)


def test_selftest_points_equal_the_model(case, valid):
    model = {}
    for n in (1, 3, 40):
        batch = valid[:n]
        for p in batch:
            if p not in model:
                model[p] = _model_pair(case, p)
        us = [model[p][0] for p in batch]
        w = BV.weights(BV.batch_challenge(3, us), n)
        L, Rp = BV.fold([model[p][1] for p in batch], w)
        rc, v, got = _call(case.verifier, batch, [case.arrays.pi_vals] * n, 3, points=True)
        assert rc == 0 and v == OK
        assert got == BV.raw_points(L, Rp), n
        if n == 3:
            assert BV.accepts_with_pairing(L, Rp, case.okey)


def test_each_mutation_at_each_position(case, valid):
    muts = _mutations(case, valid[0])
    kinds = {}
    for name, b, w in muts:
        kinds.setdefault(name.rstrip("0123456789"), (b, w))
    assert set(kinds) == {"eval", "comm", "noncanonical", "off-curve", "non-subgroup"}
    pi = case.arrays.pi_vals
    base = valid[:33]
    for name, (b, w) in kinds.items():
        for pos in (0, 16, 32):
            batch = base[:pos] + [b] + base[pos + 1 :]
            assert verdict(case.verifier, batch, [pi] * 33) == w, (name, pos)
    vals = R.fr_vec_from_mont_bytes(pi)
    wrong = R.fr_vec_to_mont_bytes([vals[0] + 1] + vals[1:])
    permuted = R.fr_vec_to_mont_bytes(vals[1:] + vals[:1])
    for bad in (wrong, permuted):
        for pos in (0, 16, 32):
            pis = [pi] * 33
            pis[pos] = bad
            assert verdict(case.verifier, base, pis) == PB200_ERR_VERIFY, pos
    forged = (bytes([0xC0]) + bytes(47)) * 11 + bytes(15 * 32)
    assert verdict(case.verifier, [forged], [R.fr_vec_to_mont_bytes([2, 3, 9])]) == PB200_ERR_VERIFY
    assert verdict(case.verifier, base[:5] + [forged], [pi] * 6) == PB200_ERR_VERIFY
    other = Case(b"gpu-batch-verify", _synthetic(300, 12))
    assert verdict(other.verifier, [valid[0]], [pi]) == PB200_ERR_VERIFY
    assert verdict(other.verifier, [other.prove(1), valid[0]], [pi, pi]) == PB200_ERR_VERIFY
    # malformed takes precedence over a failed check wherever the two sit
    bad_eval, malformed = kinds["eval"][0], kinds["off-curve"][0]
    assert verdict(case.verifier, [bad_eval, malformed] + base[:3], [pi] * 5) == PB200_ERR_POINT_MALFORMED
    assert verdict(case.verifier, [malformed] + base[:3] + [bad_eval], [pi] * 5) == PB200_ERR_POINT_MALFORMED
    with pytest.raises(plonk_b200.PointMalformed):
        case.verifier.batch_verify([bad_eval, malformed], [pi] * 2)
    with pytest.raises(plonk_b200.ProofVerificationError):
        case.verifier.batch_verify([bad_eval] + base[:2], [pi] * 3)


def test_random_mixed_batches_match_the_per_proof_verdicts(case, valid):
    muts = _mutations(case, valid[1])
    rng = random.Random(0xB47C)
    pi = case.arrays.pi_vals
    outcomes = set()
    for t in range(20):
        n = rng.randrange(1, 48)
        p_bad = rng.choice((0.0, 0.02, 0.1, 0.5))
        batch = [rng.choice(muts)[1] if rng.random() < p_bad else rng.choice(valid) for _ in range(n)]
        want = _expected(case.verifier.verify_batch(batch, [pi] * n))
        outcomes.add(want)
        assert verdict(case.verifier, batch, [pi] * n) == want, t
    assert OK in outcomes and len(outcomes) >= 2


def test_error_cases(case, valid):
    pi = case.arrays.pi_vals
    assert _call(case.verifier, [], []) == (0, PB200_ERR_VERIFY, None)
    with pytest.raises(plonk_b200.ProofVerificationError):
        case.verifier.batch_verify([], [])
    with pytest.raises(ValueError):  # InconsistentPublicInputsLen
        case.verifier.batch_verify([valid[0]], [pi[:32]])
    assert _call(case.verifier, [valid[0]], [pi[:32]])[0] == PB200_ERR_INVALID_ARG
    for version in (0, 4):
        assert _call(case.verifier, [valid[0]], [pi], version)[0] == PB200_ERR_INVALID_ARG
        with pytest.raises(ValueError):
            case.verifier.batch_verify([valid[0]], [pi], version)
    L = lib()
    v = ctypes.c_int32()
    assert L.pb200_batch_verify(None, 3, valid[0], 1, pi, 3, ctypes.byref(v)) == PB200_ERR_INVALID_ARG
    assert L.pb200_batch_verify(case.verifier._h, 3, None, 1, pi, 3, ctypes.byref(v)) == PB200_ERR_INVALID_ARG
    assert L.pb200_batch_verify(case.verifier._h, 3, valid[0], 1, None, 3, ctypes.byref(v)) == PB200_ERR_INVALID_ARG
    assert L.pb200_batch_verify(case.verifier._h, 3, valid[0], 1, pi, 3, None) == PB200_ERR_INVALID_ARG
    assert L.pb200_selftest_batch_verify_points(case.verifier._h, 3, valid[0], 1, pi, 3, ctypes.byref(v), None) == PB200_ERR_INVALID_ARG


def test_concurrent_threads_give_the_same_verdicts(case, valid):
    muts = _mutations(case, valid[2])
    pi = case.arrays.pi_vals
    batches = [valid[:20], valid[:10] + [muts[0][1]] + valid[10:20], [muts[-1][1]] + valid[:5]]
    want = [verdict(case.verifier, b, [pi] * len(b)) for b in batches]
    assert want == [OK, PB200_ERR_VERIFY, PB200_ERR_POINT_MALFORMED]
    got, errs = [None] * 6, []

    def run(k):
        try:
            got[k] = [verdict(case.verifier, b, [pi] * len(b)) for b in batches]
        except Exception as e:  # pragma: no cover - reported below
            errs.append(e)

    th = [threading.Thread(target=run, args=(k,)) for k in range(6)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs and all(g == want for g in got)
