"""The GPU Verifier (pb200_verifier_*, pb200_verify) against the reference's verdicts, restated by
tests/models/pairing_model.py and oracle/verify.py."""
import ctypes
import random
import threading

import pytest

import plonk_b200
from oracle import cref
from oracle import gadgets as G
from oracle import pyref as R
from plonk_b200 import gadgets as native_gadgets
from plonk_b200._lib import PB200_ERR_INVALID_DOMAIN, PB200_ERR_POINT_MALFORMED, PB200_ERR_VERIFY, Pb200Error, lib
from tests.models import pairing_model as M
from tests.test_gpu_gadget_circuits import CASES as GADGET_CASES

pytestmark = pytest.mark.gpu
OK = 0


def test_device_pairing_equals_the_oracle():
    rng = random.Random(0x51)
    pairs = []
    for k in range(6):
        p = None if k == 2 else R.g1_mul(R.G1_GEN, rng.randrange(1, M.Q_R))
        q = None if k == 4 else M.g2_mul(M.G2_GEN, rng.randrange(1, M.Q_R))
        pairs.append((p, q))
    g1 = b"".join(R.g1_to_raw_bytes(p) if p is not None else bytes(96) for p, _ in pairs)
    g2 = b"".join(M.g2_compress(q) for _, q in pairs)
    out = (ctypes.c_uint64 * (72 * len(pairs)))()
    assert lib().pb200_selftest_pairing(g1, g2, len(pairs), out) == 0
    for k, (p, q) in enumerate(pairs):
        # zkcrypto's final exponentiation gives the cube of the textbook value (see pairing_model)
        want = M.f12_to_tower_mont_words(M.f12_pow(M.pairing(p, q), 3))
        assert list(out[72 * k : 72 * k + 72]) == want, k


def _srs(n_points, x, gs):
    out = ctypes.create_string_buffer(96 * n_points)
    assert lib().pb200_srs_setup_from_secret(R.fr_to_mont_bytes(x), R.fr_to_mont_bytes(gs), n_points, out) == 0
    return out.raw


class Case:
    """A compiled circuit, its GPU prover and a GPU verifier over an SRS with known secrets."""

    def __init__(self, label, arrays, x=0x1234567, gs=0x7654321, hs=0xABCDEF):
        n = 1 << (arrays.constraints + 6 - 1).bit_length()
        self.label, self.arrays = label, arrays
        self.prover = plonk_b200.Prover(label, arrays.constraints, arrays.selectors, arrays.wires, arrays.n_witnesses, _srs(n + 7, x, gs))
        self.comms = self.prover.commitments()
        self.okey = M.opening_key_from_secret(x, gs, hs)
        self.verifier = plonk_b200.Verifier(label, arrays.constraints, self.comms, self.okey, arrays.pi_idx)

    def prove(self, seed, arrays=None):
        a = arrays or self.arrays
        return self.prover.prove(a.witnesses, a.pi_idx, a.pi_vals, cref.draw_blinders(R.StdRng.seed_from_u64(seed)))


def _synthetic(n_gates, seed, n_public=3, widgets=9):
    comp = R.Composer.initialized()
    R.synthetic_arith_circuit(comp, n_gates, seed=seed, n_public=n_public, widgets=widgets)
    return cref.CircuitArrays(comp)


@pytest.fixture(scope="module")
def case():
    return Case(b"gpu-verifier", _synthetic(300, 11))


def test_golden_digest_proof_is_accepted():
    pp, okey = M.srs_setup_with_opening_key(1 << 10, R.StdRng.seed_from_u64(0x9235E700), keep=64)
    comp = R.Composer.initialized()
    R.minimal_circuit(comp)
    pd = R.compile_circuit(pp, b"proof-compatibility", comp)
    idx = b"".join(i.to_bytes(8, "little") for i in comp.public_input_indexes())
    v = plonk_b200.Verifier(b"proof-compatibility", len(comp.constraints), [R.g1_compress(pd.comms[k]) for k in R.POLY_NAMES], okey, idx)
    pi = R.fr_vec_to_mont_bytes(comp.public_inputs_vec())
    v.verify(R.kat_proof(), pi)
    other = plonk_b200.Verifier(b"other-label", len(comp.constraints), [R.g1_compress(pd.comms[k]) for k in R.POLY_NAMES], okey, idx)
    with pytest.raises(plonk_b200.ProofVerificationError):
        other.verify(R.kat_proof(), pi)


@pytest.mark.parametrize("log_n", [5, 8, 10, 12])
def test_gpu_proofs_of_synthetic_circuits_are_accepted(log_n):
    arr = _synthetic((1 << log_n) - 12, 100 + log_n, widgets=0 if log_n < 8 else 9)
    c = Case(b"synthetic-%d" % log_n, arr)
    proofs = [c.prove(s) for s in range(3)]
    assert c.verifier.verify_batch(proofs, [arr.pi_vals] * 3) == [OK] * 3


@pytest.mark.parametrize("log_n", [13, 16])
def test_bench_circuit_proofs_are_accepted(log_n):
    arr = native_gadgets.bench_circuit(1 << log_n).arrays()
    c = Case(b"dusk-network", arr)
    assert c.verifier.verify_batch([c.prove(1)], [arr.pi_vals]) == [OK]


def _mutations(case, proof):
    """(name, bytes, expected status) for single changes of a valid proof."""
    out = []
    for k in range(15):  # each evaluation moved by one
        pos = 528 + 32 * k
        v = (int.from_bytes(proof[pos : pos + 32], "little") + 1) % R.R_MOD
        out.append(("eval%d" % k, proof[:pos] + v.to_bytes(32, "little") + proof[pos + 32 :], PB200_ERR_VERIFY))
    other = R.g1_compress(R.g1_mul(R.G1_GEN, 0xC0FFEE))
    for k in range(11):  # each commitment swapped for another valid point
        out.append(("comm%d" % k, proof[: 48 * k] + other + proof[48 * k + 48 :], PB200_ERR_VERIFY))
    out.append(("noncanonical", proof[:528] + R.R_MOD.to_bytes(32, "little") + proof[560:], PB200_ERR_POINT_MALFORMED))
    x = 1
    while R.g1_is_on_curve((x, pow(x ** 3 + 4, (R.P_MOD + 1) // 4, R.P_MOD))):
        x += 1
    off = bytearray(x.to_bytes(48, "big"))
    off[0] |= 0x80
    out.append(("off-curve", bytes(off) + proof[48:], PB200_ERR_POINT_MALFORMED))
    out.append(("non-subgroup", proof[:96] + _non_subgroup_g1() + proof[144:], PB200_ERR_POINT_MALFORMED))
    return out


def _non_subgroup_g1():
    x = 1
    while True:
        y = pow(x ** 3 + 4, (R.P_MOD + 1) // 4, R.P_MOD)
        if y * y % R.P_MOD == (x ** 3 + 4) % R.P_MOD and R.jac_to_affine(R.jac_mul(R.jac_from_affine((x, y)), R.R_MOD)) is not None:
            b = bytearray(x.to_bytes(48, "big"))
            b[0] |= 0x80 | (0x20 if y > (R.P_MOD - 1) // 2 else 0)
            return bytes(b)
        x += 1


def test_tampered_proofs_are_rejected(case):
    proof = case.prove(5)
    muts = _mutations(case, proof)
    got = case.verifier.verify_batch([m[1] for m in muts], [case.arrays.pi_vals] * len(muts))
    assert got == [m[2] for m in muts], [(m[0], g) for m, g in zip(muts, got) if g != m[2]]
    vals = R.fr_vec_from_mont_bytes(case.arrays.pi_vals)
    wrong = R.fr_vec_to_mont_bytes([vals[0] + 1] + vals[1:])
    permuted = R.fr_vec_to_mont_bytes(vals[1:] + vals[:1])
    assert case.verifier.verify_batch([proof] * 3, [case.arrays.pi_vals, wrong, permuted]) == [OK, PB200_ERR_VERIFY, PB200_ERR_VERIFY]
    # the reference's forged all-identity proof (tests/opening_key_validation.rs:89-125)
    forged = (bytes([0xC0]) + bytes(47)) * 11 + bytes(15 * 32)
    imp = R.fr_vec_to_mont_bytes([2, 3, 9])
    assert case.verifier.verify_batch([forged], [imp]) == [PB200_ERR_VERIFY]
    with pytest.raises(ValueError):  # InconsistentPublicInputsLen
        case.verifier.verify(proof, case.arrays.pi_vals[:32])
    # a proof against another circuit of the same shape
    other = Case(b"gpu-verifier", _synthetic(300, 12))
    assert other.verifier.verify_batch([proof], [case.arrays.pi_vals]) == [PB200_ERR_VERIFY]


def test_mixed_batch_matches_the_oracle_and_single_proof_verdicts(case):
    proof = case.prove(6)
    muts = _mutations(case, proof)
    rng = random.Random(7)
    batch, want = [], []
    for _ in range(40):
        if rng.random() < 0.5:
            batch.append(case.prove(rng.randrange(1000)) if len(batch) < 3 else proof)
            want.append(OK)
        else:
            m = rng.choice(muts)
            batch.append(m[1])
            want.append(m[2])
    pis = [case.arrays.pi_vals] * len(batch)
    assert case.verifier.verify_batch(batch, pis) == want
    assert [case.verifier.verify_batch([b], [p])[0] for b, p in zip(batch[:8], pis[:8])] == want[:8]
    # the oracle's verdict (the pairing check of tests/models/pairing_model.py) on a valid proof and on one entry of
    # every mutation kind: a moved evaluation, a swapped commitment, a non-canonical scalar, an off-curve and a
    # non-subgroup commitment (the last three fail Proof::from_bytes, which the oracle's parser asserts)
    comms = {k: R.g1_decompress(c) for k, c in zip(R.POLY_NAMES, case.comms)}
    idx = [int.from_bytes(case.arrays.pi_idx[8 * i : 8 * i + 8], "little") for i in range(len(case.arrays.pi_idx) // 8)]
    vals = R.fr_vec_from_mont_bytes(case.arrays.pi_vals)
    kinds = {"valid": (proof, OK)}
    for name, b, w in muts:
        kinds.setdefault(name.rstrip("0123456789"), (b, w))
    assert set(kinds) == {"valid", "eval", "comm", "noncanonical", "off-curve", "non-subgroup"}
    for name, (b, w) in kinds.items():
        assert case.verifier.verify_batch([b], [case.arrays.pi_vals]) == [w], name
        try:
            ok = M.verify_with_pairing(b, case.label, case.arrays.constraints, comms, idx, vals, case.okey)
            parsed = True
        except AssertionError:
            ok, parsed = False, False
        assert ok == (w == OK), name
        if name in ("noncanonical", "off-curve"):
            assert not parsed, name
        elif name == "non-subgroup":  # pyref's decoder has no subgroup check: the oracle tests torsion itself
            pt = R.g1_decompress(b[96:144])
            assert R.jac_to_affine(R.jac_mul(R.jac_from_affine(pt), R.R_MOD)) is not None
        else:
            assert parsed, name


@pytest.mark.parametrize("name,build,default,satisfied,unsatisfied", GADGET_CASES, ids=[c[0] for c in GADGET_CASES])
def test_gadget_circuit_proofs_are_accepted(name, build, default, satisfied, unsatisfied):
    """Every gadget-circuit family of test_gpu_gadget_circuits.py: the key is compiled from the default values and
    every satisfying assignment's GPU proof is accepted."""
    comp = G.GadgetComposer.initialized()
    build(comp, *default)
    c = Case(name.encode(), cref.CircuitArrays(comp))
    proofs, pis = [], []
    for k, vals in enumerate([default] + satisfied):
        other = G.GadgetComposer.initialized()
        build(other, *vals)
        arr = cref.CircuitArrays(other)
        proofs.append(c.prove(400 + k, arr))
        pis.append(arr.pi_vals)
    assert c.verifier.verify_batch(proofs, pis) == [OK] * len(proofs)


def test_concurrent_threads_give_the_same_verdicts(case):
    proof = case.prove(8)
    muts = _mutations(case, proof)
    batch = [proof] + [m[1] for m in muts[:10]]
    want = case.verifier.verify_batch(batch, [case.arrays.pi_vals] * len(batch))
    got, errs = [None] * 6, []

    def run(k):
        try:
            got[k] = case.verifier.verify_batch(batch, [case.arrays.pi_vals] * len(batch))
        except Exception as e:  # pragma: no cover - reported below
            errs.append(e)

    th = [threading.Thread(target=run, args=(k,)) for k in range(6)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs and all(g == want for g in got)


def test_to_bytes_matches_the_oracle_and_round_trips(case):
    comms = dict(zip(R.POLY_NAMES, case.comms))
    idx = [int.from_bytes(case.arrays.pi_idx[8 * i : 8 * i + 8], "little") for i in range(len(case.arrays.pi_idx) // 8)]
    cons = case.arrays.constraints
    assert cons & (cons - 1), "the case must pin VerifierKey::n = constraints on a non-power-of-two size"
    size = 1 << (cons - 1).bit_length()
    want = M.verifier_to_bytes(case.label, cons, size, cons, comms, case.okey, idx)
    assert case.verifier.to_bytes() == want
    v2 = plonk_b200.Verifier.from_bytes(want)
    assert v2.to_bytes() == want
    proof = case.prove(9)
    assert v2.verify_batch([proof], [case.arrays.pi_vals]) == [OK]
    # an oversized domain (VerifierKey::n = 2^32) is InvalidEvalDomainSize
    big = bytearray(want)
    at = 48 + len(case.label)
    big[at : at + 8] = (1 << 32).to_bytes(8, "little")
    with pytest.raises(Pb200Error) as e:
        plonk_b200.Verifier.from_bytes(bytes(big))
    assert e.value.code == PB200_ERR_INVALID_DOMAIN


def test_degenerate_opening_keys_are_refused(case):
    """tests/opening_key_validation.rs:127-152: an identity g, h or [x]h, by both constructors."""
    ident_g1, ident_g2 = bytes([0xC0]) + bytes(47), bytes([0xC0]) + bytes(95)
    keys = [ident_g1 + case.okey[48:], case.okey[:48] + ident_g2 + case.okey[144:], case.okey[:144] + ident_g2,
            case.okey[:144] + M.non_subgroup_g2_bytes()]
    n = 1 << (case.arrays.constraints - 1).bit_length()
    for k in keys:
        with pytest.raises(Pb200Error) as e:
            plonk_b200.Verifier(case.label, case.arrays.constraints, case.comms, k, case.arrays.pi_idx)
        assert e.value.code == PB200_ERR_POINT_MALFORMED
        b = M.verifier_to_bytes(case.label, case.arrays.constraints, n, case.arrays.constraints, dict(zip(R.POLY_NAMES, case.comms)), k, [])
        with pytest.raises(Pb200Error) as e:
            plonk_b200.Verifier.from_bytes(b)
        assert e.value.code == PB200_ERR_POINT_MALFORMED
