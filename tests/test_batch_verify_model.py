"""Batch verification on the CPU: the batch challenge rho and the weights of plonk_b200/csrc/verify_scalars.h,
compiled by g++ into tests/hosttest, against tests/models/batch_verify_model.py; and the folded check itself, on
proofs of the oracle's prover, with a known SRS secret and with the pairing."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle import pyref as R
from oracle import verify as OV
from tests.models import batch_verify_model as BV
from tests.models import pairing_model as PM
from tests.models import plonk_versions_model as PV
from tests.test_plonk_versions import GS, X, Circuit, _pack, _term_table

HERE = os.path.dirname(os.path.abspath(__file__))
M = R.R_MOD


@pytest.fixture(scope="module")
def bv():
    so = os.path.join(HERE, "hosttest", "libbatchverify.so")
    src = os.path.join(HERE, "hosttest", "batch_verify.cpp")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-frounding-math", "-mfma", "-shared", "-fPIC", "-o", so, src])
    return ctypes.CDLL(so)


def _host_rho(bv, version, us):
    out = ctypes.create_string_buffer(32 * (len(us) + 1))
    assert bv.bv_challenge(version, _pack(us) or None, ctypes.c_size_t(len(us)), out) == 0
    vals = [R.fr_from_mont_bytes(out.raw[32 * i : 32 * i + 32]) for i in range(len(us) + 1)]
    return vals[0], vals[1:]


def test_host_rho_and_weights_equal_the_model_on_random_inputs(bv):
    rng = random.Random(0xBA7C)
    for n in (0, 1, 2, 5, 33):
        for version in PV.VERSIONS:
            us = [rng.randrange(M) for _ in range(n)]
            rho, w = _host_rho(bv, version, us)
            assert rho == BV.batch_challenge(version, us), (n, version)
            assert w == BV.weights(rho, n)


def test_rho_binds_the_complete_batch(bv):
    """batch_challenge_binds_the_complete_batch (key.rs:867-901) for this transcript: rho changes with any u_i,
    the order, the length and the version."""
    rng = random.Random(3)
    us = [rng.randrange(M) for _ in range(4)]
    base = BV.batch_challenge(3, us)
    variants = [us[:k] + [(us[k] + 1) % M] + us[k + 1 :] for k in range(4)]
    variants += [us[1:] + us[:1], us[::-1], us[:3], us + [us[0]], us + us]
    got = [BV.batch_challenge(3, v) for v in variants] + [BV.batch_challenge(v, us) for v in (1, 2)]
    assert base not in got and len(set(got)) == len(got)
    assert [_host_rho(bv, 3, v)[0] for v in variants] == got[: len(variants)]


class Batch:
    """Proofs of one circuit with each proof's (L_i, R_i) formed from the host scalars and the kernels' term table."""

    def __init__(self, bv, circuit, proofs, version=3):
        self.c, self.proofs, self.version = circuit, proofs, version
        dom = R.EvaluationDomain(circuit.pd.size)
        roots = [pow(dom.group_gen_inv, i, M) for i in circuit.idx]
        table = _term_table()
        key_pts = [circuit.pd.comms[k] for k in R.POLY_NAMES] + [circuit.pp[0]]
        self.status, self.us, self.pairs = [], [], []
        for proof in proofs:
            out = (ctypes.c_uint64 * 128)()
            u = ctypes.create_string_buffer(32)
            st = bv.bv_scalars(circuit.label, ctypes.c_size_t(len(circuit.label)), ctypes.c_uint64(circuit.pd.constraints), circuit.key,
                               ctypes.c_uint64(circuit.pd.size), R.fr_to_mont_bytes(dom.group_gen), _pack(roots), _pack(circuit.vals),
                               ctypes.c_size_t(len(circuit.vals)), proof, version, out, u)
            self.status.append(st)
            if st != 0:
                self.us.append(None)
                self.pairs.append(None)
                continue
            s = [sum(out[4 * k + j] << (64 * j) for j in range(4)) for k in range(32)]
            comm, _ = OV.parse_proof(proof)
            proof_pts = [comm[k] for k in OV.COMM_ORDER]
            pts = [None if src < 0 else key_pts[src] if src < 16 else proof_pts[src - 16] for src in table]
            self.us.append(R.fr_from_mont_bytes(u.raw))
            assert s[31] == self.us[-1], "lane 31 carries u"
            self.pairs.append((BV.left(comm["w_z"], comm["w_zw"], s[31]), OV._msm(pts[:31], s[:31])))

    def folded(self):
        rho = BV.batch_challenge(self.version, self.us)
        return BV.fold(self.pairs, BV.weights(rho, len(self.pairs)))


@pytest.fixture(scope="module")
def circuit():
    return Circuit(b"batch-synthetic", lambda c: R.synthetic_arith_circuit(c, 40, seed=9, n_public=3, widgets=2))


@pytest.fixture(scope="module")
def proofs(circuit):
    return [circuit.prove(70 + k, 3) for k in range(3)]


def test_u_is_the_proofs_last_challenge_and_each_pair_satisfies_its_check(bv, circuit, proofs):
    b = Batch(bv, circuit, proofs)
    assert b.status == [0, 0, 0]
    for proof, u, (L, Rp) in zip(proofs, b.us, b.pairs):
        assert u == PV.challenges(proof, circuit.label, circuit.pd.constraints, circuit.pd.comms, circuit.vals, 3)["u"]
        right, left = PV.right_and_left(proof, circuit.label, circuit.pd.constraints, circuit.pd.comms, circuit.idx, circuit.vals,
                                        circuit.pp[0], 3)
        assert (L, Rp) == (R.g1_neg(left), right)
        assert BV.accepts_with_secret(L, Rp, X)


def test_folded_batch_passes_with_the_secret_and_the_pairing(bv, circuit, proofs):
    L, Rp = Batch(bv, circuit, proofs).folded()
    assert BV.accepts_with_secret(L, Rp, X)
    okey = PM.opening_key_from_secret(X, GS, 0xABCDEF)
    assert BV.accepts_with_pairing(L, Rp, okey)
    assert not BV.accepts_with_pairing(L, R.g1_add(Rp, circuit.pp[0]), okey)


def test_folded_batch_with_one_invalid_proof_fails(bv, circuit, proofs):
    bad = bytearray(proofs[1])
    bad[528 + 5] ^= 1  # an evaluation moved: still canonical
    b = Batch(bv, circuit, [proofs[0], bytes(bad), proofs[2]])
    assert b.status == [0, 0, 0]
    assert not BV.accepts_with_secret(*b.pairs[1], X)
    assert not BV.accepts_with_secret(*b.folded(), X)


def test_crafted_pair_passes_unit_weights_and_fails_rho_weights(bv, circuit, proofs):
    """(L_1, R_1 + D) and (L_2, R_2 - D) each fail, their plain sum passes, and the rho-weighted sum fails."""
    b = Batch(bv, circuit, proofs[:2])
    (L1, R1), (L2, R2) = b.pairs
    D = R.g1_mul(R.G1_GEN, 0xD15EA5E)
    crafted = [(L1, R.g1_add(R1, D)), (L2, R.g1_add(R2, R.g1_neg(D)))]
    assert not any(BV.accepts_with_secret(L, Rp, X) for L, Rp in crafted)
    assert BV.accepts_with_secret(*BV.fold(crafted, [1, 1]), X)
    rho = BV.batch_challenge(3, b.us)
    assert not BV.accepts_with_secret(*BV.fold(crafted, BV.weights(rho, 2)), X)
    okey = PM.opening_key_from_secret(X, GS, 0xABCDEF)
    assert BV.accepts_with_pairing(*BV.fold(crafted, [1, 1]), okey)
    assert not BV.accepts_with_pairing(*BV.fold(crafted, BV.weights(rho, 2)), okey)
