"""PlonkVersion V1, V2 and V3 on the CPU: the legacy transcript seed of plonk_b200/csrc/transcript.h and the
Verifier's per-version scalars (plonk_b200/csrc/verify_scalars.h), compiled by g++ into tests/hosttest, against the
version-aware oracle of tests/models/plonk_versions_model.py; and that oracle's own verdict matrix, including the
reference's forged proof (proof.rs:1332-1743)."""
import ctypes
import os
import re
import subprocess

import pytest

from oracle import pyref as R
from oracle import verify as OV
from tests.models import plonk_versions_model as PV

HERE = os.path.dirname(os.path.abspath(__file__))
M = R.R_MOD
X, GS = 0x1234567, 0x7654321  # the test SRS secret and G1 scalar


@pytest.fixture(scope="module")
def pv():
    so = os.path.join(HERE, "hosttest", "libplonkversions.so")
    src = os.path.join(HERE, "hosttest", "plonk_versions.cpp")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-frounding-math", "-mfma", "-shared", "-fPIC", "-o", so, src])
    return ctypes.CDLL(so)


class Circuit:
    """A compiled circuit over a test SRS with a known secret, as the GPU tests build it."""

    def __init__(self, label, build):
        comp = R.Composer.initialized()
        build(comp)
        self.label, self.comp = label, comp
        n = 1 << (len(comp.constraints) + 6 - 1).bit_length()
        self.pp = R.srs_from_secret(n + 7, X, GS)
        self.pd = R.compile_circuit(self.pp, label, comp)
        self.idx, self.vals = comp.public_input_indexes(), comp.public_inputs_vec()
        self.key = b"".join(R.g1_compress(self.pd.comms[k]) for k in R.POLY_NAMES)

    def prove(self, seed, version):
        return PV.prove(self.pd, R.StdRng.seed_from_u64(seed), self.comp, version)

    def verify(self, proof, version):
        return PV.verify_with_secret(proof, self.label, self.pd.constraints, self.pd.comms, self.idx, self.vals, self.pp[0], X, version)


@pytest.fixture(scope="module")
def synthetic():
    return Circuit(b"versions-synthetic", lambda c: R.synthetic_arith_circuit(c, 40, seed=5, n_public=3, widgets=2))


@pytest.fixture(scope="module")
def proofs(synthetic):
    return {v: synthetic.prove(40 + v, v) for v in PV.VERSIONS}


def _pack(xs):
    return b"".join(R.fr_to_mont_bytes(x % M) for x in xs)


def _host_challenges(pv, c, proof, legacy):
    out = ctypes.create_string_buffer(11 * 32)
    assert pv.pv_challenges(c.label, ctypes.c_size_t(len(c.label)), ctypes.c_uint64(c.pd.constraints), c.key, legacy,
                            _pack(c.vals), ctypes.c_size_t(len(c.vals)), proof, out) == 0
    return [R.fr_from_mont_bytes(out.raw[32 * i : 32 * i + 32]) for i in range(11)]


def _model_challenges(c, proof, version):
    ch = PV.challenges(proof, c.label, c.pd.constraints, c.pd.comms, c.vals, version)
    return [ch[k] for k in ("beta", "gamma", "alpha", "range", "logic", "fixed", "var", "z", "v", "v_w", "u")]


def test_legacy_seed_matches_the_oracle_on_the_golden_digest_circuit_and_with_public_inputs(pv, synthetic, proofs):
    pp = R.srs_setup(1 << 10, R.StdRng.seed_from_u64(0x9235E700), keep=64)
    golden = Circuit.__new__(Circuit)
    comp = R.Composer.initialized()
    R.minimal_circuit(comp)
    golden.label, golden.comp, golden.pd = b"proof-compatibility", comp, R.compile_circuit(pp, b"proof-compatibility", comp)
    golden.idx, golden.vals = comp.public_input_indexes(), comp.public_inputs_vec()
    golden.key = b"".join(R.g1_compress(golden.pd.comms[k]) for k in R.POLY_NAMES)
    kat = R.kat_proof()
    assert synthetic.vals, "the synthetic circuit must have public inputs"
    for c, proof in ((golden, kat), (synthetic, proofs[2]), (synthetic, proofs[3])):
        legacy = _host_challenges(pv, c, proof, 1)
        assert legacy == _model_challenges(c, proof, 1) == _model_challenges(c, proof, 2)
        assert _host_challenges(pv, c, proof, 0) == _model_challenges(c, proof, 3)
        assert legacy[0] != _model_challenges(c, proof, 3)[0], "the two seeds must differ"


def _term_table():
    """c_term_point of k_verify_msm, read from plonk_b200/csrc/verify.cu: 0..14 the key commitments in pb::Poly
    order, 15 opening_key.g, 16 + k proof commitment k, -1 none; lane 31 is left's u W_zw."""
    src = open(os.path.join(HERE, "..", "plonk_b200", "csrc", "verify.cu")).read()
    names = re.search(r"enum \{ (P_A = 16[^}]*)\}", src).group(1).replace("P_A = 16", "P_A").split(", ")
    body = re.search(r"c_term_point\[32\] = \{([^}]*)\}", src).group(1)
    sym = {n.strip(): 16 + i for i, n in enumerate(names)}
    return [sym[t.strip()] if t.strip() in sym else int(t) for t in body.split(",")]


def _device_points(pv, c, proof, version):
    """Sum s_k P_k over the 32 host scalars and the kernel's term table: (status, right, left)."""
    n = c.pd.size
    dom = R.EvaluationDomain(n)
    roots = [pow(dom.group_gen_inv, i, M) for i in c.idx]
    out = (ctypes.c_uint64 * 128)()
    st = pv.pv_scalars(c.label, ctypes.c_size_t(len(c.label)), ctypes.c_uint64(c.pd.constraints), c.key, ctypes.c_uint64(n),
                       R.fr_to_mont_bytes(dom.group_gen), _pack(roots), _pack(c.vals), ctypes.c_size_t(len(c.vals)), proof, version, out)
    if st != 0:
        return st, None, None
    s = [sum(out[4 * k + j] << (64 * j) for j in range(4)) for k in range(32)]
    comm, _ = OV.parse_proof(proof)
    key_pts = [c.pd.comms[k] for k in R.POLY_NAMES] + [c.pp[0]]
    proof_pts = [comm[k] for k in OV.COMM_ORDER]
    pts = [None if src < 0 else key_pts[src] if src < 16 else proof_pts[src - 16] for src in _term_table()]
    right = OV._msm(pts[:31], s[:31])
    left = OV._msm([comm["w_z"], pts[31]], [1, s[31]])
    return st, right, left


def test_host_scalars_form_the_oracle_points_for_every_version(pv, synthetic, proofs):
    for pv_version, proof in proofs.items():
        for version in PV.VERSIONS:
            st, right, left = _device_points(pv, synthetic, proof, version)
            assert st == 0
            want = PV.right_and_left(proof, synthetic.label, synthetic.pd.constraints, synthetic.pd.comms, synthetic.idx, synthetic.vals,
                                     synthetic.pp[0], version)
            assert (right, left) == want, (pv_version, version)
    # V3: the same right-hand point as oracle/verify.py, read off its first multi-scalar multiplication
    seen, msm = [], OV._msm
    OV._msm = lambda p, s: seen.append(msm(p, s)) or seen[-1]
    try:
        assert OV.verify_with_secret(proofs[3], synthetic.label, synthetic.pd.constraints, synthetic.pd.comms, synthetic.idx, synthetic.vals,
                                     synthetic.pp[0], X)
    finally:
        OV._msm = msm
    assert _device_points(pv, synthetic, proofs[3], 3)[1:] == (seen[0], seen[1])


def test_v1_leaves_the_selector_opening_lanes_zero(pv, synthetic, proofs):
    out = (ctypes.c_uint64 * 128)()
    dom = R.EvaluationDomain(synthetic.pd.size)
    roots = [pow(dom.group_gen_inv, i, M) for i in synthetic.idx]
    for version in PV.VERSIONS:
        assert pv.pv_scalars(synthetic.label, ctypes.c_size_t(len(synthetic.label)), ctypes.c_uint64(synthetic.pd.constraints), synthetic.key,
                             ctypes.c_uint64(synthetic.pd.size), R.fr_to_mont_bytes(dom.group_gen), _pack(roots), _pack(synthetic.vals),
                             ctypes.c_size_t(len(synthetic.vals)), proofs[1], version, out) == 0
        lanes = [sum(out[4 * k + j] for j in range(4)) for k in range(23, 27)]
        assert (all(x == 0 for x in lanes)) == (version == 1), version


def test_oracle_version_matrix(synthetic, proofs):
    for made, proof in proofs.items():
        for version in PV.VERSIONS:
            assert synthetic.verify(proof, version) == (made == version), (made, version)


def test_v1_proof_from_a_v2_proof_and_the_secret(synthetic, proofs):
    v2 = synthetic.prove(41, 2)  # the seed of proofs[1]
    assert PV.v1_from_v2_with_secret(v2, synthetic.label, synthetic.pd.constraints, synthetic.pd.comms, synthetic.vals, synthetic.pp[0], X) == proofs[1]


def _soundness_circuit():
    a, b, d, public = 3, 5, 7, 11
    return Circuit(b"soundness_test", lambda c: PV.arith_circuit(c, a, b, d, public))


def test_forged_proof_passes_v1_only():
    """forged_selector_eval_proof_must_be_rejected (proof.rs:1690-1743), with the V1 verdict the reference's
    verify_legacy gives: an honest V3 proof fails V1, the forged one passes V1 and fails V2 and V3."""
    c = _soundness_circuit()
    honest = c.prove(0xDEADBEEF, 3)
    assert c.verify(honest, 3) and not c.verify(honest, 1)
    forged = PV.forge_proof(c.pd, c.comp, R.StdRng.seed_from_u64(0xDEADBEEF))
    assert [c.verify(forged, v) for v in PV.VERSIONS] == [True, False, False]
