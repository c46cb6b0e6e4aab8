"""The debugger's gate identities as the device evaluates them (plonk_b200/csrc/plonk_algebra.cuh), compiled for the
host by g++ with pbh::HFr (tests/hosttest/debugger_identities.cpp), on the CPU:
- they equal the Python restatement of the reference's identity_evaluations (tests/models/debugger_model.py) on every
  fixture row and on random rows, and first_failing_identity names the model's first non-zero identity;
- the terms are exactly what the quotient combines: each widget is its separation challenge ch times the kappa-weighted
  sum of its terms, kappa = ch^2 (widget_range, widget_logic, widget_fixed and widget_var are stated separately)."""
import ctypes
import os
import random
import subprocess

import pytest

from tests.models import debugger_model as D

HERE = os.path.dirname(os.path.abspath(__file__))
M = D.R_MOD


@pytest.fixture(scope="module")
def dbg():
    so = os.path.join(HERE, "hosttest", "libdebuggeridentities.so")
    src = os.path.join(HERE, "hosttest", "debugger_identities.cpp")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    return ctypes.CDLL(so)


def _pack(xs):
    return b"".join((x % M * (1 << 256) % M).to_bytes(32, "little") for x in xs)


def _unpack(raw, n):
    inv = pow(1 << 256, M - 2, M)
    return [int.from_bytes(raw[32 * i : 32 * i + 32], "little") * inv % M for i in range(n)]


def _identities(dbg, points):
    """points: (selectors dict, pi, a, b, c, d, a_w, b_w, d_w) -> (17 identities, first failing index) per point."""
    flat = [v for q, *rest in points for v in [q[k] for k in D.SELECTORS] + rest]
    out = ctypes.create_string_buffer(len(points) * 17 * 32)
    first = (ctypes.c_int32 * len(points))()
    assert dbg.dbg_identities(_pack(flat), ctypes.c_size_t(len(points)), out, first) == 0
    ids = _unpack(out.raw, 17 * len(points))
    return [(ids[17 * i : 17 * i + 17], first[i]) for i in range(len(points))]


def _fixture_points():
    for case in D.load_fixtures():
        rows, witnesses, pi = D.fixture_circuit(case)
        padded = 1 << (len(rows) - 1).bit_length()
        for i, (q, a, b, c, d) in enumerate(rows):
            j = (i + 1) % padded
            nxt = [witnesses[rows[j][k]] for k in (1, 2, 4)] if j < len(rows) else [0, 0, 0]
            yield (q, pi.get(i, 0), witnesses[a], witnesses[b], witnesses[c], witnesses[d], *nxt)


def _random_points(rng, n):
    edge = [0, 1, 2, 3, M - 1]
    for _ in range(n):
        def val():
            return rng.choice(edge) if rng.random() < 0.3 else rng.randrange(M)
        yield ({k: (0 if rng.random() < 0.4 else val()) for k in D.SELECTORS}, 0 if rng.random() < 0.5 else val(), *[val() for _ in range(7)])


def test_identities_equal_the_model(dbg):
    points = list(_fixture_points()) + list(_random_points(random.Random(7), 400))
    for p, (ids, first) in zip(points, _identities(dbg, points)):
        want = D.identity_evaluations(*p)
        assert ids == want, p
        assert first == next((k for k, x in enumerate(want) if x), -1), p


def test_widgets_are_kappa_weighted_sums_of_the_terms(dbg):
    rng = random.Random(11)
    edge = [0, 1, M - 1]
    points = [[rng.choice(edge) if rng.random() < 0.1 else rng.randrange(M) for _ in range(14)] for _ in range(300)]
    points += [[v] * 14 for v in edge]
    out = ctypes.create_string_buffer(len(points) * 20 * 32)
    assert dbg.dbg_terms_and_widgets(_pack(v for p in points for v in p), ctypes.c_size_t(len(points)), out) == 0
    got = _unpack(out.raw, 20 * len(points))
    for i, p in enumerate(points):
        terms, widgets = got[20 * i : 20 * i + 16], got[20 * i + 16 : 20 * i + 20]
        groups = [terms[0:4], terms[4:9], terms[9:13], terms[13:16]]
        for ch, ts, widget in zip(p[:4], groups, widgets):
            kappa = ch * ch % M
            assert widget == ch * sum(t * pow(kappa, j, M) for j, t in enumerate(ts)) % M, (i, p)
