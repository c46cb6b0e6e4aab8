"""Validates the V3 proof algebra that the prover and the Verifier share (plonk_b200/csrc/plonk_algebra.cuh and the
transcript schedule of transcript.h) on the CPU.

The headers are compiled for the host by g++ into tests/hosttest and compared with the Python oracle: the gate
widgets and the permutation products, instantiated both with the host field (the prover's round 5 and the
Verifier) and with the host build of the kernels' Fr (the quotient kernel); and the transcript schedule and the
linearisation scalars on the reference's known-answer proof."""
import ctypes
import hashlib
import os
import random
import subprocess

import pytest

from oracle import pyref as R

HERE = os.path.dirname(os.path.abspath(__file__))
M = R.R_MOD


@pytest.fixture(scope="module")
def pa():
    so = os.path.join(HERE, "hosttest", "libproofalgebra.so")
    src = os.path.join(HERE, "hosttest", "proof_algebra.cpp")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-frounding-math", "-mfma", "-shared", "-fPIC", "-o", so, src])
    return ctypes.CDLL(so)


def _pack(xs):
    return b"".join(R.fr_to_mont_bytes(x % M) for x in xs)


def _unpack(raw, n):
    return [R.fr_from_mont_bytes(raw[32 * i : 32 * i + 32]) for i in range(n)]


def _ident_copy(alpha, beta, gamma, a, b, c, d, x, s, z, z_w):
    """The identity and copy terms of pyref.quotient_numerator_i: every selector and the public input zero, so
    that the numerator is ident - copy; z_w = 0 leaves ident, z = 0 leaves -copy."""
    q = {k: 0 for k in R.POLY_NAMES}
    q.update(linear=x, s_sigma_1=s[0], s_sigma_2=s[1], s_sigma_3=s[2], s_sigma_4=s[3])
    ch = dict(alpha=alpha, beta=beta, gamma=gamma, range=0, logic=0, fixed=0, var=0)
    ident = R.quotient_numerator_i(q, ch, a, b, c, d, 0, 0, 0, z, 0, 0, 0)
    copy = -R.quotient_numerator_i(q, ch, a, b, c, d, 0, 0, 0, 0, z_w, 0, 0) % M
    return ident, copy


@pytest.mark.parametrize("field", [0, 1], ids=["host_field", "kernel_field"])
def test_widgets_and_permutation_products(pa, field):
    rng = random.Random(2024 + field)
    edge = [0, 1, M - 1]
    points = [[v] * 24 for v in edge]
    points += [[rng.choice(edge) if rng.random() < 0.1 else rng.randrange(M) for _ in range(24)] for _ in range(300)]
    out = ctypes.create_string_buffer(len(points) * 6 * 32)
    assert pa.pa_widgets(field, _pack(v for p in points for v in p), ctypes.c_size_t(len(points)), out) == 0
    got = _unpack(out.raw, 6 * len(points))
    for i, p in enumerate(points):
        ch_r, ch_l, ch_f, ch_v, q_l, q_r, q_c, a, b, c, d, a_w, b_w, d_w, z, z_w, alpha, beta, gamma, x = p[:20]
        want = [
            R.widget_range_scalar(ch_r, a, b, c, d, d_w),
            R.widget_logic_scalar(ch_l, q_c, a, a_w, b, b_w, c, d, d_w),
            R.widget_fixed_base_scalar(ch_f, q_l, q_r, q_c, a, a_w, b, b_w, c, d, d_w),
            R.widget_curve_add_scalar(ch_v, a, a_w, b, b_w, c, d, d_w),
            *_ident_copy(alpha, beta, gamma, a, b, c, d, x, p[20:24], z, z_w),
        ]
        assert got[6 * i : 6 * i + 6] == want, i


def test_transcript_schedule_and_linearisation_on_the_kat_proof(pa):
    trace = R.ProofTrace()
    proof = R.kat_proof(trace)
    assert hashlib.blake2b(proof).digest() == R.KAT_DIGEST
    # the proving key of kat_proof: the same compile_circuit call
    pp = R.srs_setup(1 << 10, R.StdRng.seed_from_u64(0x9235E700), keep=64)
    comp = R.Composer.initialized()
    R.minimal_circuit(comp)
    pd = R.compile_circuit(pp, b"proof-compatibility", comp)
    pis = comp.public_inputs_vec()
    key_comms = b"".join(R.g1_compress(pd.comms[k]) for k in R.POLY_NAMES)
    out = ctypes.create_string_buffer(31 * 32)
    assert pa.pa_replay(pd.label, ctypes.c_size_t(len(pd.label)), ctypes.c_uint64(pd.constraints), key_comms,
                        ctypes.c_uint64(pd.constraints), _pack(pis), ctypes.c_size_t(len(pis)), proof,
                        ctypes.c_uint64(pd.size), out) == 0
    got = _unpack(out.raw, 31)
    t = trace.values
    ch = t["ch"]
    assert got[:10] == [t["beta"], t["gamma"], t["alpha"], ch["range"], ch["logic"], ch["fixed"], ch["var"],
                        t["z_challenge"], t["v_challenge"], t["v_w_challenge"]]

    # the linearisation scalars from pyref's widget functions (pyref.prove, round 5)
    e = t["evals"]
    z, alpha, beta, gamma = t["z_challenge"], t["alpha"], t["beta"], t["gamma"]
    a, b, c, d, a_w, b_w, d_w, qa = e["a"], e["b"], e["c"], e["d"], e["a_w"], e["b_w"], e["d_w"], e["q_arith"]
    bz = beta * z
    s_ident = (a + bz + gamma) * (b + R.K1 * bz + gamma) * (c + R.K2 * bz + gamma) * (d + R.K3 * bz + gamma) * alpha
    s_copy = (a + beta * e["s1"] + gamma) * (b + beta * e["s2"] + gamma) * (c + beta * e["s3"] + gamma) * beta * e["z"] * alpha
    l1 = R.EvaluationDomain(pd.size).first_lagrange_coefficient(z)
    z_n = pow(z, pd.size, M)
    sel = dict.fromkeys(R.POLY_NAMES, 0)
    sel.update(q_m=a * b * qa, q_l=a * qa, q_r=b * qa, q_o=c * qa, q_f=d * qa, q_c=qa, s_sigma_4=-s_copy)
    sel["q_range"] = R.widget_range_scalar(ch["range"], a, b, c, d, d_w)
    sel["q_logic"] = R.widget_logic_scalar(ch["logic"], e["q_c"], a, a_w, b, b_w, c, d, d_w)
    sel["q_fixed_group_add"] = R.widget_fixed_base_scalar(ch["fixed"], e["q_l"], e["q_r"], e["q_c"], a, a_w, b, b_w, c, d, d_w)
    sel["q_variable_group_add"] = R.widget_curve_add_scalar(ch["var"], a, a_w, b, b_w, c, d, d_w)
    want = [sel[k] % M for k in R.POLY_NAMES] + [(s_ident + l1 * alpha * alpha) % M]
    want += [-(z_n - 1) * pow(z_n, j, M) % M for j in range(4)]
    assert got[11:] == want
