"""Batch verification over groups on the CPU: the grouped batch challenge rho and the weights of
plonk_b200/csrc/verify_scalars.h, compiled by g++ into tests/hosttest, against tests/models/batch_verify_groups_model.py;
and the folded check over proofs of two circuits with different keys on one SRS secret, with the secret and with the
pairing."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle import pyref as R
from tests.models import batch_verify_groups_model as BVG
from tests.models import batch_verify_model as BV
from tests.models import pairing_model as PM
from tests.models import plonk_versions_model as PV
from tests.test_batch_verify_model import Batch
from tests.test_plonk_versions import GS, X, Circuit, _pack

HERE = os.path.dirname(os.path.abspath(__file__))
M = R.R_MOD


def _compile(name, so_name):
    so = os.path.join(HERE, "hosttest", so_name)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-frounding-math", "-mfma", "-shared", "-fPIC", "-o", so,
                           os.path.join(HERE, "hosttest", name)])
    return ctypes.CDLL(so)


@pytest.fixture(scope="module")
def bvg():
    return _compile("batch_verify_groups.cpp", "libbatchverifygroups.so")


@pytest.fixture(scope="module")
def bv():
    """The one-group harness (bv_scalars), under a name of its own so as not to replace a library already loaded."""
    return _compile("batch_verify.cpp", "libbatchverify_for_groups.so")


def _host(bvg, groups):
    """(rho, weights) of the host for groups given as (version, us)."""
    n = sum(len(us) for _, us in groups)
    versions = (ctypes.c_int * max(1, len(groups)))(*[v for v, _ in groups])
    lens = (ctypes.c_size_t * max(1, len(groups)))(*[len(us) for _, us in groups])
    out = ctypes.create_string_buffer(32 * (n + 1))
    us = _pack([u for _, g in groups for u in g])
    assert bvg.bvg_challenge(versions, lens, ctypes.c_size_t(len(groups)), us or None, out) == 0
    vals = [R.fr_from_mont_bytes(out.raw[32 * i : 32 * i + 32]) for i in range(n + 1)]
    return vals[0], vals[1:]


def _host_one(bvg, version, us):
    out = ctypes.create_string_buffer(32)
    assert bvg.bvg_challenge_one(version, _pack(us) or None, ctypes.c_size_t(len(us)), out) == 0
    return R.fr_from_mont_bytes(out.raw)


def test_host_rho_and_weights_equal_the_model_on_random_inputs(bvg):
    rng = random.Random(0x6B0F)
    for n_groups in range(6):
        for _ in range(4):
            groups = [(rng.choice(PV.VERSIONS), [rng.randrange(M) for _ in range(rng.choice((0, 1, 2, 5, 9)))]) for _ in range(n_groups)]
            rho, w = _host(bvg, groups)
            assert rho == BVG.batch_challenge(groups), groups
            assert w == BV.weights(rho, sum(len(us) for _, us in groups))


def test_one_group_draws_the_one_group_rho(bvg):
    rng = random.Random(7)
    for n in (0, 1, 3, 33):
        for version in PV.VERSIONS:
            us = [rng.randrange(M) for _ in range(n)]
            want = BV.batch_challenge(version, us)
            assert BVG.batch_challenge([(version, us)]) == want
            assert _host(bvg, [(version, us)])[0] == want
            assert _host_one(bvg, version, us) == want


def test_rho_binds_the_group_structure_versions_and_every_u(bvg):
    rng = random.Random(11)
    u = [rng.randrange(M) for _ in range(5)]
    base = [(3, u[:2]), (2, u[2:3]), (1, u[3:])]
    variants = [
        [(3, u[:1]), (3, u[1:2]), (2, u[2:3]), (1, u[3:])],  # a group split
        [(3, u[:3]), (1, u[3:])],  # two groups merged (same u sequence, the versions aside)
        [(2, u[2:3]), (3, u[:2]), (1, u[3:])],  # groups reordered
        [(3, u[:2]), (1, u[3:]), (2, u[2:3])],
        [(3, u[:2]), (1, u[2:3]), (1, u[3:])],  # V2 -> V1: the u of a V1 and a V2 proof of one witness are equal
        [(3, u[:2]), (2, u[2:3]), (2, u[3:])],  # V1 -> V2
        [(2, u[:2]), (2, u[2:3]), (1, u[3:])],  # V3 -> V2
        [(3, u[:2]), (2, u[2:3]), (1, u[3:]), (3, [])],  # an empty group appended
    ]
    for k in range(5):  # each u_i moved by one
        v = list(u)
        v[k] = (v[k] + 1) % M
        variants.append([(3, v[:2]), (2, v[2:3]), (1, v[3:])])
    want = BVG.batch_challenge(base)
    got = [BVG.batch_challenge(v) for v in variants]
    assert want not in got and len(set(got)) == len(got)
    assert _host(bvg, base)[0] == want
    assert [_host(bvg, v)[0] for v in variants] == got
    assert BVG.batch_challenge([(3, u[:2])]) != BVG.batch_challenge([(3, u[:1]), (3, u[1:2])])


@pytest.fixture(scope="module")
def circuits():
    """Two circuits with different keys and public-input counts on one SRS secret (so one opening key)."""
    a = Circuit(b"groups-a", lambda c: R.synthetic_arith_circuit(c, 40, seed=9, n_public=3, widgets=2))
    b = Circuit(b"groups-b", lambda c: R.synthetic_arith_circuit(c, 90, seed=21, n_public=2, widgets=1))
    assert a.key != b.key and a.pp[0] == b.pp[0]
    return a, b


@pytest.fixture(scope="module")
def groups(bv, circuits):
    """Two V3 proofs of circuit a and two V2 proofs of circuit b, with their (L_i, R_i)."""
    a, b = circuits
    ga = Batch(bv, a, [a.prove(80 + k, 3) for k in range(2)], 3)
    gb = Batch(bv, b, [b.prove(90 + k, 2) for k in range(2)], 2)
    assert ga.status == [0, 0] and gb.status == [0, 0]
    return ga, gb


def _fold(*batches):
    return BVG.fold([(g.version, g.us, g.pairs) for g in batches])


def test_fold_over_two_circuits_passes_with_the_secret_and_the_pairing(groups):
    ga, gb = groups
    L, Rp = _fold(ga, gb)
    assert BV.accepts_with_secret(L, Rp, X)
    okey = PM.opening_key_from_secret(X, GS, 0xABCDEF)
    assert BV.accepts_with_pairing(L, Rp, okey)
    assert not BV.accepts_with_pairing(L, R.g1_add(Rp, ga.c.pp[0]), okey)


def test_proof_swapped_into_the_other_circuits_group_fails(bv, circuits, groups):
    a, b = circuits
    ga, gb = groups
    # proof 0 of circuit a (V3) checked in b's group under b's key; b has 2 public inputs, a's proof carries its own
    swapped = Batch(bv, b, [gb.proofs[0], ga.proofs[0]], 2)
    rest = Batch(bv, a, ga.proofs[1:], 3)
    assert swapped.status == [0, 0]
    assert not BV.accepts_with_secret(*swapped.pairs[1], X)
    assert not BV.accepts_with_secret(*_fold(rest, swapped), X)


def test_crafted_cross_group_pair_passes_unit_weights_and_fails_rho_weights(groups):
    """(L_1, R_1 + D) in group 1 and (L_2, R_2 - D) in group 2 each fail, their plain sum passes, and the rho-weighted
    sum fails."""
    ga, gb = groups
    (L1, R1), (L2, R2) = ga.pairs[0], gb.pairs[0]
    D = R.g1_mul(R.G1_GEN, 0xD15EA5E)
    crafted = [(L1, R.g1_add(R1, D)), (L2, R.g1_add(R2, R.g1_neg(D)))]
    assert not any(BV.accepts_with_secret(L, Rp, X) for L, Rp in crafted)
    assert BV.accepts_with_secret(*BV.fold(crafted, [1, 1]), X)
    folded = BVG.fold([(3, ga.us[:1], crafted[:1]), (2, gb.us[:1], crafted[1:])])
    assert not BV.accepts_with_secret(*folded, X)
    okey = PM.opening_key_from_secret(X, GS, 0xABCDEF)
    assert BV.accepts_with_pairing(*BV.fold(crafted, [1, 1]), okey)
    assert not BV.accepts_with_pairing(*folded, okey)
