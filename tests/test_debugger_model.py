"""The Python restatement of the reference's debugger check (tests/models/debugger_model.py), on the CPU: it reproduces
the reference's own unit-test expectations (tests/golden/debugger_fixtures.json), and it agrees with the oracle's
row checker (oracle/gadgets.py::unsatisfied_rows) on which rows of the gadget circuits fail, except where the two
checkers are known to differ: the oracle's checker gates the public input under q_arith, the reference does not."""
import pytest

from oracle import gadgets as G
from tests.models import debugger_model as D
from tests.test_gpu_gadget_circuits import CASES

FIXTURES = D.load_fixtures()


def test_fixture_set_is_complete():
    names = [c["name"] for c in FIXTURES]
    assert len(names) == len(set(names)) == 29
    assert sum(n.startswith("satisfied ") for n in names) == 6
    failing = [c for c in FIXTURES if c["name"].startswith("fails ")]
    assert len(failing) == 18
    # every identity family is the expected one of some single-identity fixture; logic relation twice (AND and XOR)
    assert sorted({c["unsatisfied"][0][1] for c in failing}) == sorted(D.IDENTITY_FAMILIES)


@pytest.mark.parametrize("case", FIXTURES, ids=[c["name"] for c in FIXTURES])
def test_model_reproduces_the_reference_fixtures(case):
    rows, witnesses, pi = D.fixture_circuit(case)
    got = D.unsatisfied_constraints(rows, witnesses, pi)
    assert got == [tuple(x) for x in case["unsatisfied"]]
    report = D.report(got, len(rows))
    if case["report"] is None:
        assert report is None
    else:
        for fragment in case["report"]["contains"]:
            assert fragment in report
    if case["name"].startswith("fails "):  # the failing identity itself is non-zero, not only the first one reported
        k = D.IDENTITY_FAMILIES.index(case["unsatisfied"][0][1])
        assert D.row_identities(rows, witnesses, pi, 0)[k] != 0


def test_report_wording():
    assert D.report([(0, "arithmetic"), (1, "arithmetic")], 2) == (
        "plonk debugger: 2 of 2 constraints are unsatisfied; the first, constraint 0, fails the arithmetic identity")


def _gadget_circuits():
    for name, build, default, satisfied, unsatisfied in CASES:
        for kind, vals in [("default", default)] + [("satisfied", v) for v in satisfied] + [("unsatisfied", v) for v in unsatisfied]:
            yield name, kind, build, vals


@pytest.mark.parametrize("name,kind,build,vals", list(_gadget_circuits()))
def test_model_agrees_with_the_oracle_checker_on_gadget_circuits(name, kind, build, vals):
    comp = G.GadgetComposer.initialized()
    build(comp, *vals)
    rows, witnesses, pi = D.from_composer(comp)
    model_rows = {i for i, _ in D.unsatisfied_constraints(rows, witnesses, pi)}
    oracle_rows = {i for i, _ in G.unsatisfied_rows(comp, limit=len(rows) * 5 + 1)}
    for i in model_rows ^ oracle_rows:  # only the public input outside q_arith may tell them apart
        assert pi.get(i, 0) and rows[i][0]["q_arith"] == 0, (i, rows[i])
    assert bool(model_rows) == (kind == "unsatisfied")


def test_public_input_outside_q_arith_fails_arithmetic():
    zero = {k: 0 for k in D.SELECTORS}
    rows, witnesses, pi = [(zero, 0, 0, 0, 0)], [0], {0: 5}
    assert D.unsatisfied_constraints(rows, witnesses, pi) == [(0, "arithmetic")]

    class Gate:  # the same row through the oracle's checker, which gates pi under q_arith and so passes it
        sel, a, b, c, d = dict(zero), 0, 0, 0, 0

    class Comp:
        constraints, witnesses, public_inputs = [Gate()], [0], {0: 5}

    assert G.unsatisfied_rows(Comp()) == []
