"""Batch verification over groups on the GPU (pb200_batch_verify_groups, plonk_b200.batch_verify_groups): one verdict
for proofs of several circuits and versions on one SRS, against the per-proof verdicts of pb200_verify_with_version,
the one-group call pb200_batch_verify and the folded points of tests/models/batch_verify_groups_model.py."""
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
from tests.models import batch_verify_groups_model as BVG
from tests.models import batch_verify_model as BV
from tests.models import pairing_model as M
from tests.test_gpu_batch_verify import _call as _call_one
from tests.test_gpu_batch_verify import _expected, _model_pair
from tests.test_gpu_gadget_circuits import CASES as GADGET_CASES
from tests.test_gpu_plonk_versions import _prove, _v1
from tests.test_gpu_verifier import Case, _mutations, _synthetic

pytestmark = pytest.mark.gpu
OK = 0


def _args(groups):
    """The ctypes arguments of pb200_batch_verify_groups for groups (verifier, proofs, pis, version), up to the
    verdict."""
    m = len(groups)
    handles = (ctypes.c_void_p * max(1, m))(*[g[0]._h.value if g[0] is not None else None for g in groups])
    versions = (ctypes.c_int32 * max(1, m))(*[int(g[3]) for g in groups])
    counts = (ctypes.c_size_t * max(1, m))(*[len(g[1]) for g in groups])
    n_pi = (ctypes.c_size_t * max(1, m))(*[len(g[2][0]) // 32 if g[2] else g[0].n_pi for g in groups])
    proofs = b"".join(p for g in groups for p in g[1])
    pis = b"".join(v for g in groups for v in g[2])
    return [handles, versions, counts, n_pi, m, proofs or None, pis or None]


def _call(groups, points=False):
    """(return code, verdict, the selftest's 192 point bytes or None)."""
    verdict = ctypes.c_int32(12345)
    args = _args(groups) + [ctypes.byref(verdict)]
    if not points:
        return lib().pb200_batch_verify_groups(*args), verdict.value, None
    out = ctypes.create_string_buffer(192)
    rc = lib().pb200_selftest_batch_verify_groups_points(*args, out)
    return rc, verdict.value, out.raw


def verdict(groups):
    rc, v, _ = _call(groups)
    assert rc == 0
    return v


def _per_proof(groups):
    """The grouped verdict that pb200_verify_with_version's per-proof statuses imply."""
    st = []
    for verifier, proofs, pis, version in groups:
        if proofs:
            st += verifier.verify_batch(proofs, pis, version)
    return _expected(st)


@pytest.fixture(scope="module")
def case():
    return Case(b"gpu-batch-groups-a", _synthetic(300, 11))


@pytest.fixture(scope="module")
def other():
    return Case(b"gpu-batch-groups-b", _synthetic(200, 17, n_public=2))


@pytest.fixture(scope="module")
def valid(case):
    return [case.prove(500 + k) for k in range(40)]


@pytest.fixture(scope="module")
def other_valid(other):
    return [other.prove(800 + k) for k in range(12)]


@pytest.fixture(scope="module")
def circuits():
    """Five circuits on one SRS (the default secrets, so one opening key): synthetic circuits of about 2^9, 2^10 and
    2^12 gates, a gadget circuit and BenchCircuit<2^13>; each with 8 distinct valid V3 proofs and its public inputs."""
    out = []
    for log_n in (9, 10, 12):
        c = Case(b"groups-synthetic-%d" % log_n, _synthetic((1 << log_n) - 12, 300 + log_n))
        out.append(c)
    name, build, default, _, _ = GADGET_CASES[0]
    comp = G.GadgetComposer.initialized()
    build(comp, *default)
    out.append(Case(name.encode(), cref.CircuitArrays(comp)))
    out.append(Case(b"dusk-network", native_gadgets.bench_circuit(1 << 13).arrays()))
    okeys = {c.okey for c in out}
    assert len(okeys) == 1
    return [(c, [c.prove(900 + k) for k in range(8)], c.arrays.pi_vals) for c in out]


def _group(entry, n, version=3, start=0):
    c, proofs, pi = entry
    return (c.verifier, [proofs[(start + k) % len(proofs)] for k in range(n)], [pi] * n, version)


def test_one_group_equals_pb200_batch_verify(case, valid):
    pi = case.arrays.pi_vals
    v2 = [_prove(case, 700 + k, PlonkVersion.V2) for k in range(3)]
    by_version = {3: valid, 2: v2, 1: [_v1(case, p) for p in v2]}
    for version, proofs in by_version.items():
        for n in (1, 3, 40):
            batch = [proofs[k % len(proofs)] for k in range(n)]
            want = _call_one(case.verifier, batch, [pi] * n, version, points=True)
            got = _call([(case.verifier, batch, [pi] * n, version)], points=True)
            assert want[0] == 0 and want[1] == OK, (version, n)
            assert got == want, (version, n)
    # a failing batch and a decided-before-the-pairing batch give the same verdict and points too
    bad = valid[:2] + [_mutations(case, valid[2])[0][1]]
    assert _call([(case.verifier, bad, [pi] * 3, 3)], points=True) == _call_one(case.verifier, bad, [pi] * 3, 3, points=True)
    assert _call([(case.verifier, valid[:3], [pi] * 3, 2)], points=True) == _call_one(case.verifier, valid[:3], [pi] * 3, 2, points=True)


def test_several_circuits_are_accepted(circuits):
    sizes = (1, 7, 8, 9, 33)
    groups = [_group(e, n) for e, n in zip(circuits, sizes)]
    assert verdict(groups) == OK
    assert verdict(groups[::-1]) == OK
    assert verdict([_group(e, n) for e, n in zip(circuits, sizes[::-1])]) == OK
    plonk_b200.batch_verify_groups(groups)
    # the same verifier in several groups, interleaved with others (one key slot per verifier)
    assert verdict([_group(circuits[0], 9), _group(circuits[1], 3), _group(circuits[0], 8, start=3), _group(circuits[4], 1)]) == OK


def test_forty_groups_of_one_proof_are_accepted(circuits):
    groups = [_group(circuits[k % len(circuits)], 1, start=k) for k in range(40)]
    assert verdict(groups) == OK


def test_4096_proofs_over_4_groups_are_accepted(circuits):
    groups = [_group(e, 1024, start=k) for k, e in enumerate(circuits[:4])]
    assert verdict(groups) == OK
    bad = list(groups[3][1])
    bad[1000] = _mutations(None, bad[1000])[3][1]
    assert verdict(groups[:3] + [(groups[3][0], bad, groups[3][2], 3)]) == PB200_ERR_VERIFY


def test_selftest_points_equal_the_model_for_v3_v2_v1(case, other, valid):
    v2 = [_prove(other, 720 + k, PlonkVersion.V2) for k in range(2)]
    v1 = [_v1(case, _prove(case, 730 + k, PlonkVersion.V2)) for k in range(2)]
    spec = [(case, valid[:3], 3), (other, v2, 2), (case, v1, 1)]
    model = []
    for c, proofs, version in spec:
        pairs = [_model_pair(c, p, version) for p in proofs]
        model.append((version, [u for u, _ in pairs], [pr for _, pr in pairs]))
    L, Rp = BVG.fold(model)
    groups = [(c.verifier, proofs, [c.arrays.pi_vals] * len(proofs), version) for c, proofs, version in spec]
    rc, v, got = _call(groups, points=True)
    assert rc == 0 and v == OK
    assert got == BV.raw_points(L, Rp)
    assert BV.accepts_with_pairing(L, Rp, case.okey)


def test_versions_of_one_verifier(case, valid):
    pi = case.arrays.pi_vals
    v2 = [_prove(case, 740 + k, PlonkVersion.V2) for k in range(3)]
    v3 = valid[:3]
    assert verdict([(case.verifier, v2, [pi] * 3, 2), (case.verifier, v3, [pi] * 3, 3)]) == OK
    plonk_b200.batch_verify_groups([(case.verifier, v3, [pi] * 3, PlonkVersion.V3), (case.verifier, v2, [pi] * 3, PlonkVersion.V2)])
    assert verdict([(case.verifier, v2, [pi] * 3, 3), (case.verifier, v3, [pi] * 3, 2)]) == PB200_ERR_VERIFY
    with pytest.raises(plonk_b200.ProofVerificationError):
        plonk_b200.batch_verify_groups([(case.verifier, v2, [pi] * 3, PlonkVersion.V3), (case.verifier, v3, [pi] * 3, PlonkVersion.V2)])
    v1 = [_v1(case, p) for p in v2[:2]]
    for group in (v1, v1 + v2[:1], v3[:2]):
        groups = [(case.verifier, v3, [pi] * 3, 3), (case.verifier, group, [pi] * len(group), 1)]
        assert verdict(groups) == _per_proof(groups)
    assert verdict([(case.verifier, v3, [pi] * 3, 3), (case.verifier, v1, [pi] * 2, 1)]) == OK


def test_each_mutation_at_each_position_of_each_group(case, other, circuits, valid, other_valid):
    entries = [(case, valid[:9]), (other, other_valid[:9]), (circuits[2][0], circuits[2][1] + circuits[2][1][:1])]
    base = [(c.verifier, proofs, [c.arrays.pi_vals] * len(proofs), 3) for c, proofs in entries]
    assert verdict(base) == OK
    for g, (c, proofs) in enumerate(entries):
        kinds = {}
        for name, b, _ in _mutations(c, proofs[0]):
            kinds.setdefault(name.rstrip("0123456789"), b)
        assert set(kinds) == {"eval", "comm", "noncanonical", "off-curve", "non-subgroup"}
        for name, b in kinds.items():
            for pos in (0, 4, 8):
                groups = list(base)
                groups[g] = (c.verifier, proofs[:pos] + [b] + proofs[pos + 1 :], base[g][2], 3)
                want = _per_proof(groups)
                assert want != OK
                assert verdict(groups) == want, (g, name, pos)
    # a proof valid for one circuit in another's group: both have 3 public inputs
    groups = list(base)
    groups[1] = (case.verifier, valid[:2] + [circuits[2][1][0]], [case.arrays.pi_vals] * 3, 3)
    assert verdict(groups) == _per_proof(groups) == PB200_ERR_VERIFY
    # public inputs rotated for one proof of one group
    vals = R.fr_vec_from_mont_bytes(case.arrays.pi_vals)
    pis = [case.arrays.pi_vals] * 9
    pis[4] = R.fr_vec_to_mont_bytes(vals[1:] + vals[:1])
    groups = [base[1], (case.verifier, valid[:9], pis, 3), base[2]]
    assert verdict(groups) == _per_proof(groups) == PB200_ERR_VERIFY
    # malformed takes precedence over a failed check across groups
    kinds_a = {n.rstrip("0123456789"): b for n, b, _ in _mutations(case, valid[0])}
    groups = [(case.verifier, [kinds_a["eval"]], [case.arrays.pi_vals], 3), base[1], (case.verifier, [kinds_a["off-curve"]], [case.arrays.pi_vals], 3)]
    assert verdict(groups) == PB200_ERR_POINT_MALFORMED
    with pytest.raises(plonk_b200.PointMalformed):
        plonk_b200.batch_verify_groups(groups)


def test_random_mixed_calls_match_the_per_proof_verdicts(case, other, valid, other_valid):
    pools = [(case, valid, _mutations(case, valid[1])), (other, other_valid, _mutations(other, other_valid[1]))]
    rng = random.Random(0x6C0B)
    outcomes = set()
    for t in range(20):
        groups = []
        for _ in range(rng.randrange(2, 6)):
            c, good, muts = rng.choice(pools)
            n = rng.randrange(0, 12)
            p_bad = rng.choice((0.0, 0.0, 0.05, 0.3))
            proofs = [rng.choice(muts)[1] if rng.random() < p_bad else rng.choice(good) for _ in range(n)]
            groups.append((c.verifier, proofs, [c.arrays.pi_vals] * n, 3))
        if not any(g[1] for g in groups):
            continue
        want = _per_proof(groups)
        outcomes.add(want)
        assert verdict(groups) == want, t
    assert OK in outcomes and len(outcomes) >= 2


def test_error_cases(case, other, valid, other_valid):
    pi, pi_b = case.arrays.pi_vals, other.arrays.pi_vals
    good = [(case.verifier, valid[:2], [pi] * 2, 3), (other.verifier, other_valid[:1], [pi_b], 3)]
    L = lib()
    v = ctypes.c_int32(12345)
    assert L.pb200_batch_verify_groups(None, None, None, None, 0, None, None, ctypes.byref(v)) == 0 and v.value == PB200_ERR_VERIFY
    assert _call([]) == (0, PB200_ERR_VERIFY, None)
    assert _call([(case.verifier, [], [], 3), (other.verifier, [], [], 2)]) == (0, PB200_ERR_VERIFY, None)
    with pytest.raises(plonk_b200.ProofVerificationError):
        plonk_b200.batch_verify_groups([])
    assert verdict([good[0], (other.verifier, [], [], 3), good[1]]) == OK
    # a NULL verifier, an unknown version, a wrong n_pi in one group
    args = _args(good)
    args[0][1] = None
    assert L.pb200_batch_verify_groups(*args, ctypes.byref(v)) == PB200_ERR_INVALID_ARG
    for version in (0, 4):
        assert _call([good[0], (other.verifier, other_valid[:1], [pi_b], version)])[0] == PB200_ERR_INVALID_ARG
        with pytest.raises(ValueError):
            plonk_b200.batch_verify_groups([good[0], (other.verifier, other_valid[:1], [pi_b], version)])
    args = _args(good)
    args[3][1] = 3
    assert L.pb200_batch_verify_groups(*args, ctypes.byref(v)) == PB200_ERR_INVALID_ARG
    with pytest.raises(ValueError):  # InconsistentPublicInputsLen
        plonk_b200.batch_verify_groups([good[0], (other.verifier, other_valid[:1], [pi], 3)])
    # a verifier on another SRS: the golden-digest circuit's
    pp, okey = M.srs_setup_with_opening_key(1 << 10, R.StdRng.seed_from_u64(0x9235E700), keep=64)
    comp = R.Composer.initialized()
    R.minimal_circuit(comp)
    pd = R.compile_circuit(pp, b"proof-compatibility", comp)
    idx = b"".join(i.to_bytes(8, "little") for i in comp.public_input_indexes())
    golden = plonk_b200.Verifier(b"proof-compatibility", len(comp.constraints), [R.g1_compress(pd.comms[k]) for k in R.POLY_NAMES], okey, idx)
    gpi = R.fr_vec_to_mont_bytes(comp.public_inputs_vec())
    assert verdict([(golden, [R.kat_proof()], [gpi], 3)]) == OK
    assert _call([good[0], (golden, [R.kat_proof()], [gpi], 3)])[0] == PB200_ERR_INVALID_ARG
    with pytest.raises(ValueError, match="opening key"):
        plonk_b200.batch_verify_groups([(golden, [R.kat_proof()], [gpi], 3), good[0]])
    # NULL arrays
    for k in range(4):
        args = _args(good)
        args[k] = None
        assert L.pb200_batch_verify_groups(*args, ctypes.byref(v)) == PB200_ERR_INVALID_ARG, k
    for k in (5, 6):
        args = _args(good)
        args[k] = None
        assert L.pb200_batch_verify_groups(*args, ctypes.byref(v)) == PB200_ERR_INVALID_ARG, k
    assert L.pb200_batch_verify_groups(*_args(good), None) == PB200_ERR_INVALID_ARG
    assert L.pb200_selftest_batch_verify_groups_points(*_args(good), ctypes.byref(v), None) == PB200_ERR_INVALID_ARG


def test_concurrent_threads_give_the_same_verdicts(case, other, valid, other_valid):
    pi, pi_b = case.arrays.pi_vals, other.arrays.pi_vals
    muts = _mutations(case, valid[2])
    calls = [
        [(case.verifier, valid[:10], [pi] * 10, 3), (other.verifier, other_valid[:5], [pi_b] * 5, 3)],
        [(other.verifier, other_valid[:3], [pi_b] * 3, 3), (case.verifier, valid[:5] + [muts[0][1]], [pi] * 6, 3)],
        [(case.verifier, [muts[-1][1]] + valid[:3], [pi] * 4, 3), (other.verifier, other_valid[:2], [pi_b] * 2, 3)],
    ]
    want = [verdict(c) for c in calls]
    assert want == [OK, PB200_ERR_VERIFY, PB200_ERR_POINT_MALFORMED]
    got, errs = [None] * 6, []

    def run(k):
        try:
            got[k] = [verdict(c) for c in calls]
        except Exception as e:  # pragma: no cover - reported below
            errs.append(e)

    th = [threading.Thread(target=run, args=(k,)) for k in range(6)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs and all(g == want for g in got)
