"""The reference debugger's check on the GPU (pb200_circuit_unsatisfied, pb200_prover_unsatisfied and their Python
mirrors), against the Python restatement of src/debugger.rs (tests/models/debugger_model.py):
- the reference's unit-test fixtures at both levels, both directions of the rotated wires' wrap included;
- every gadget circuit: satisfying witnesses report nothing and prove, failing ones give the model's list;
- BenchCircuit<2^16> (and one case of <2^20>) with one witness of each gate family corrupted: exactly the rows that
  read it, as the model names them;
- provers from to_bytes and from a compressed description report what the compiled prover reports;
- an assignment that sets a selector the compiled circuit leaves at zero (the reference's debugger.rs:216-220 case);
- cap, the argument checks, and a check running beside proofs on the same prover."""
import ctypes
import threading

import pytest

import plonk_b200
from oracle import cref
from oracle import pyref as R
from plonk_b200 import gadgets as N
from plonk_b200._lib import PB200_ERR_INVALID_ARG, check, lib
from tests.models import debugger_model as D
from tests.test_gpu_gadget_circuits import CASES

pytestmark = pytest.mark.gpu

M = D.R_MOD
FIXTURES = D.load_fixtures()


@pytest.fixture(scope="module", autouse=True)
def init():
    check(lib().pb200_init(0))


def _srs_small(constraints, secret=0x5EED):
    n = 1 << (constraints + 6 - 1).bit_length()  # pp.trim(next_pow2(constraints + 6))
    return cref.srs_from_secret(n + 7, secret, 0xACE)


def _srs_device(constraints):  # the same points as cref.srs_from_secret, computed on the GPU
    n = (1 << (constraints + 6 - 1).bit_length()) + 7
    raw = ctypes.create_string_buffer(96 * n)
    check(lib().pb200_srs_setup_from_secret(R.fr_to_mont_bytes(0xABCDEF), R.fr_to_mont_bytes(0x13579), n, raw))
    return raw.raw


def _prover(arrays, srs, label=b"debugger"):
    return plonk_b200.Prover(label, arrays.constraints, arrays.selectors, arrays.wires, arrays.n_witnesses, srs)


def _both(prover, arrays):
    return (plonk_b200.unsatisfied_constraints(arrays),
            prover.unsatisfied_constraints(arrays.witnesses, arrays.pi_idx, arrays.pi_vals))


def _model(arrays, only=None):
    return D.unsatisfied_constraints(*D.from_arrays(arrays), only=only)


def _with_witness(arrays, w, delta=1):
    """arrays with witness w increased by delta (Montgomery bytes)."""
    v = (D._fr(arrays.witnesses, w) + delta) % M
    wit = arrays.witnesses[: 32 * w] + (v * (1 << 256) % M).to_bytes(32, "little") + arrays.witnesses[32 * w + 32 :]
    return type(arrays)(arrays.constraints, arrays.selectors, arrays.wires, wit, arrays.pi_idx, arrays.pi_vals)


def _readers(arrays, w):
    """The rows that read witness w: as a, b, c or d, or through the next row's a, b or d (cyclic over next_pow2)."""
    n = arrays.constraints
    padded = 1 << (n - 1).bit_length()
    wires = memoryview(arrays.wires).cast("I")
    rows = set()
    for k in range(4):
        col = wires[k * n : (k + 1) * n]
        for i in (i for i, x in enumerate(col) if x == w):
            rows.add(i)
            if k != 2:
                prev = (i - 1) % padded
                if prev < n:
                    rows.add(prev)
    return sorted(rows)


# ---- 1. the reference's fixtures --------------------------------------------------------------------------------
@pytest.mark.parametrize("case", FIXTURES, ids=[c["name"] for c in FIXTURES])
def test_reference_fixtures_at_both_levels(case):
    arrays = D.to_arrays(*D.fixture_circuit(case))
    want = [tuple(x) for x in case["unsatisfied"]]
    prover = _prover(arrays, _srs_small(arrays.constraints))
    assert _both(prover, arrays) == (want, want)
    for report in (plonk_b200.unsatisfied_report(arrays), prover.unsatisfied_report(arrays.witnesses, arrays.pi_idx, arrays.pi_vals)):
        if case["report"] is None:
            assert report is None
        else:
            assert report == D.report(want, arrays.constraints)
            for fragment in case["report"]["contains"]:
                assert fragment in report


# ---- 2. gadget circuits ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,build,default,satisfied,unsatisfied", CASES, ids=[c[0] for c in CASES])
def test_gadget_circuits(name, build, default, satisfied, unsatisfied):
    def arrays_of(vals):
        c = N.Composer.initialized()
        build(c, *vals)
        return c.arrays()

    compiled = arrays_of(default)
    prover = _prover(compiled, _srs_small(compiled.constraints, 0x5EED + len(name)), name.encode())
    for k, vals in enumerate([default] + satisfied):
        a = arrays_of(vals)
        assert _both(prover, a) == ([], []), vals
        prover.prove(a.witnesses, a.pi_idx, a.pi_vals, cref.draw_blinders(R.StdRng.seed_from_u64(100 + k)))
    for vals in unsatisfied:
        a = arrays_of(vals)
        want = _model(a)
        assert want
        assert _both(prover, a) == (want, want), vals


# ---- 3. BenchCircuit ---------------------------------------------------------------------------------------------
FAMILY_SELECTOR = {"arithmetic": 6, "range": 7, "logic": 8, "fixed-base": 9, "variable-base": 10}


def _witness_of_family(arrays, sel_index):
    """A witness other than the constants 0 and 1 read by the first row whose selector sel_index is set."""
    n = arrays.constraints
    wires = memoryview(arrays.wires).cast("I")
    zero = bytes(32)
    for i in range(n):
        if arrays.selectors[32 * (sel_index * n + i) : 32 * (sel_index * n + i) + 32] != zero:
            for k in range(4):
                if wires[k * n + i] > 1:
                    return wires[k * n + i]
    raise AssertionError("no such row")


@pytest.fixture(scope="module")
def bench16():
    arrays = N.bench_circuit(1 << 16).arrays()
    return arrays, _prover(arrays, _srs_device(arrays.constraints))


def test_bench_circuit_honest_witness_reports_nothing(bench16):
    arrays, prover = bench16
    assert _both(prover, arrays) == ([], [])
    assert plonk_b200.unsatisfied_report(arrays) is None


@pytest.mark.parametrize("family", list(FAMILY_SELECTOR))
def test_bench_circuit_corrupted_witness(bench16, family):
    arrays, prover = bench16
    w = _witness_of_family(arrays, FAMILY_SELECTOR[family])
    bad = _with_witness(arrays, w)
    want = _model(bad, only=_readers(bad, w))
    assert want
    assert _both(prover, bad) == (want, want)


def test_bench_circuit_2_20_last_constraint():
    arrays = N.bench_circuit(1 << 20).arrays()
    n = arrays.constraints
    wires = memoryview(arrays.wires).cast("I")
    w = max(wires[k * n + n - 1] for k in range(4))
    bad = _with_witness(arrays, w, 5)
    readers = _readers(bad, w)
    assert n - 1 in readers
    want = _model(bad, only=readers)
    assert want
    prover = _prover(arrays, _srs_device(n))
    assert _both(prover, arrays) == ([], [])
    assert _both(prover, bad) == (want, want)


# ---- 4. every prover kind ----------------------------------------------------------------------------------------
def test_loaded_and_compressed_provers_report_the_same():
    arrays = N.bench_circuit(1 << 13).arrays()
    draws = [R.fr_to_mont_bytes(R.random_nonzero_bls_scalar(R.StdRng.seed_from_u64(0xD0 + k))) for k in range(3)]
    pp = plonk_b200.PublicParameters.setup(1 << 14, draws)
    prover = plonk_b200.Prover(b"kinds", arrays.constraints, arrays.selectors, arrays.wires, arrays.n_witnesses, pp.raw_points)
    loaded = plonk_b200.Prover.from_bytes(prover.to_bytes(), arrays.wires, arrays.n_witnesses)
    compressed, _ = plonk_b200.Compiler.compile_with_compressed(pp, b"kinds", plonk_b200.compress_arrays(arrays))
    for family, sel in FAMILY_SELECTOR.items():
        bad = _with_witness(arrays, _witness_of_family(arrays, sel))
        args = (bad.witnesses, bad.pi_idx, bad.pi_vals)
        want = prover.unsatisfied_constraints(*args)
        assert want, family
        assert loaded.unsatisfied_constraints(*args) == want
        assert compressed.unsatisfied_constraints(*args) == want
        assert compressed.unsatisfied_report(*args) == prover.unsatisfied_report(*args)


# ---- 5. description and assignment disagree (debugger.rs:216-220) ------------------------------------------------
def test_selector_live_only_in_the_assignment():
    zero = {k: 0 for k in D.SELECTORS}
    gate = dict(zero, q_l=1, q_r=1, q_o=M - 1, q_arith=1)  # a + b - c = 0
    rows = [(gate, 1, 2, 3, 0)] * 6 + [(dict(zero), 4, 4, 4, 4)]  # the last row is vacuous in the description
    witnesses, pi = [0, 2, 3, 5, 9], {}
    described = D.to_arrays(rows, witnesses, pi)
    live = D.to_arrays(rows[:-1] + [(dict(zero, q_c=1, q_arith=1), 4, 4, 4, 4)], witnesses, pi)
    prover = _prover(described, _srs_small(described.constraints))
    assert plonk_b200.unsatisfied_constraints(live) == [(6, "arithmetic")]
    assert prover.unsatisfied_constraints(live.witnesses, live.pi_idx, live.pi_vals) == []
    prover.prove(live.witnesses, live.pi_idx, live.pi_vals, cref.draw_blinders(R.StdRng.seed_from_u64(5)))


# ---- 6. outputs and argument checks ------------------------------------------------------------------------------
def _raw_circuit(a, cap, rows=True, **over):
    args = dict(n=a.constraints, sel=a.selectors, wires=a.wires, wit=a.witnesses, n_wit=a.n_witnesses, pi_idx=a.pi_idx or None,
                pi_vals=a.pi_vals or None, n_pi=a.n_pi)
    args.update(over)
    r, f, n = (ctypes.c_uint64 * max(cap, 1))(), (ctypes.c_int32 * max(cap, 1))(), ctypes.c_size_t(12345)
    rc = lib().pb200_circuit_unsatisfied(args["n"], args["sel"], args["wires"], args["wit"], args["n_wit"], args["pi_idx"], args["pi_vals"],
                                         args["n_pi"], cap, r if rows else None, f if rows else None, ctypes.byref(n))
    return rc, n.value, [(r[i], D.IDENTITY_FAMILIES[f[i]]) for i in range(min(cap, n.value))] if rc == 0 else None


def _raw_prover(p, a, cap, rows=True, **over):
    args = dict(wit=a.witnesses, n_wit=a.n_witnesses, pi_idx=a.pi_idx or None, pi_vals=a.pi_vals or None, n_pi=a.n_pi)
    args.update(over)
    r, f, n = (ctypes.c_uint64 * max(cap, 1))(), (ctypes.c_int32 * max(cap, 1))(), ctypes.c_size_t(12345)
    rc = lib().pb200_prover_unsatisfied(p._h, args["wit"], args["n_wit"], args["pi_idx"], args["pi_vals"], args["n_pi"], cap,
                                        r if rows else None, f if rows else None, ctypes.byref(n))
    return rc, n.value, [(r[i], D.IDENTITY_FAMILIES[f[i]]) for i in range(min(cap, n.value))] if rc == 0 else None


def test_cap_and_counts(bench16):
    arrays, prover = bench16
    bad = _with_witness(_with_witness(arrays, _witness_of_family(arrays, 6)), _witness_of_family(arrays, 8))
    full = plonk_b200.unsatisfied_constraints(bad)
    total = len(full)
    assert total >= 2
    for cap in (0, 1, total - 1, total, total + 5, arrays.constraints + 100):
        for call in (_raw_circuit, lambda a, c, **kw: _raw_prover(prover, a, c, **kw)):
            rc, n, got = call(bad, cap)
            assert (rc, n, got) == (0, total, full[: min(cap, total)])
    assert _raw_circuit(bad, 0, rows=False)[:2] == (0, total)
    assert _raw_prover(prover, bad, 0, rows=False)[:2] == (0, total)
    assert plonk_b200.unsatisfied_report(bad) == D.report(full, arrays.constraints)


def test_argument_checks():
    case = next(c for c in FIXTURES if c["name"] == "satisfied arithmetic")
    rows, witnesses, _ = D.fixture_circuit(case)
    a = D.to_arrays(rows * 4, witnesses, {0: 7, 3: 1, 5: 2})
    prover = _prover(a, _srs_small(a.constraints))
    u64 = lambda *xs: b"".join(x.to_bytes(8, "little") for x in xs)  # noqa: E731
    vals3 = a.pi_vals
    for call in (_raw_circuit, lambda x, c, **kw: _raw_prover(prover, x, c, **kw)):
        assert call(a, 4)[0] == 0
        assert call(a, 4, rows=False)[0] == PB200_ERR_INVALID_ARG  # NULL arrays with cap > 0
        assert call(a, 4, pi_idx=u64(3, 0, 5), pi_vals=vals3)[0] == PB200_ERR_INVALID_ARG  # not increasing
        assert call(a, 4, pi_idx=u64(0, 3, 3), pi_vals=vals3)[0] == PB200_ERR_INVALID_ARG  # duplicate
        assert call(a, 4, pi_idx=u64(0, 3, a.constraints), pi_vals=vals3)[0] == PB200_ERR_INVALID_ARG  # outside the circuit
        assert call(a, 4, pi_idx=None)[0] == PB200_ERR_INVALID_ARG  # announced but not given
    assert _raw_prover(prover, a, 4, n_wit=a.n_witnesses - 1, wit=a.witnesses[:-32])[0] == PB200_ERR_INVALID_ARG
    wires = bytearray(a.wires)
    wires[4 * 5 : 4 * 6] = a.n_witnesses.to_bytes(4, "little")
    assert _raw_circuit(a, 4, wires=bytes(wires))[0] == PB200_ERR_INVALID_ARG  # a wire index >= n_witnesses
    # no constraints: nothing to report, as the reference's empty debugger
    assert _raw_circuit(a, 4, n=0, sel=None, wires=None, pi_idx=None, pi_vals=None, n_pi=0) == (0, 0, [])
    for k in range(17):
        assert plonk_b200.identity_family(k) == D.IDENTITY_FAMILIES[k]
    assert lib().pb200_identity_family(17) is None and lib().pb200_identity_family(-1) is None


# ---- 7. beside proofs on the same prover -------------------------------------------------------------------------
def test_check_runs_beside_proofs(bench16):
    arrays, prover = bench16
    bad = _with_witness(arrays, _witness_of_family(arrays, 7))
    want = prover.unsatisfied_constraints(bad.witnesses, bad.pi_idx, bad.pi_vals)
    blinders = [cref.draw_blinders(R.StdRng.seed_from_u64(300 + k)) for k in range(4)]
    quiet = [prover.prove(arrays.witnesses, arrays.pi_idx, arrays.pi_vals, b) for b in blinders]
    stop, seen = threading.Event(), []

    def checker():
        while not stop.is_set():
            seen.append(prover.unsatisfied_constraints(bad.witnesses, bad.pi_idx, bad.pi_vals))

    t = threading.Thread(target=checker)
    t.start()
    try:
        busy = [prover.prove(arrays.witnesses, arrays.pi_idx, arrays.pi_vals, b) for b in blinders * 2]
    finally:
        stop.set()
        t.join()
    assert busy == quiet * 2
    assert seen and all(s == want for s in seen)
