"""The reference's debugger check (src/debugger.rs:74-236) restated in plain Python integers mod r: the 17 gate identities
of a row (identity_evaluations, :95-180), the rotated wires of the padded cyclic domain (shifted_wire_value, :74-93),
the list of failing rows (unsatisfied_constraints, :192-205) and the report (unsatisfied_report, :221-236, here without
its call-site clause).

A circuit is given as rows of (selectors, a, b, c, d): selectors maps the 11 names of SELECTORS to canonical ints, the
wires are indices into the witness table; pi maps a row to its public input."""
from __future__ import annotations

import json
import os
from typing import Dict, List, Optional, Sequence, Tuple

R_MOD = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
EDWARDS_D = (-10240 * pow(10241, R_MOD - 2, R_MOD)) % R_MOD  # dusk_jubjub::EDWARDS_D
SELECTORS = ["q_m", "q_l", "q_r", "q_o", "q_f", "q_c", "q_arith", "q_range", "q_logic", "q_fixed_group_add", "q_variable_group_add"]
IDENTITY_FAMILIES = [
    "arithmetic",
    "range delta c/d", "range delta b/c", "range delta a/b", "range accumulator",
    "logic left quad", "logic right quad", "logic output quad", "logic product", "logic relation",
    "fixed-base bit consistency", "fixed-base xy consistency", "fixed-base x accumulator", "fixed-base y accumulator",
    "variable-base xy consistency", "variable-base x accumulator", "variable-base y accumulator",
]
_MONT_R_INV = pow(1 << 256, R_MOD - 2, R_MOD)

Row = Tuple[Dict[str, int], int, int, int, int]


def delta(f: int) -> int:  # range and logic proverkey.rs: f (f - 1)(f - 2)(f - 3)
    return f * (f - 1) * (f - 2) * (f - 3) % R_MOD


def delta_xor_and(a: int, b: int, w: int, c: int, q_c: int) -> int:  # logic/proverkey.rs
    f = w * (w * (4 * w - 18 * (a + b) + 81) + 18 * (a * a + b * b) - 81 * (a + b) + 83)
    e = 3 * (a + b + c) - 2 * f
    return (q_c * (9 * c - 3 * (a + b)) + e) % R_MOD


def identity_evaluations(q: Dict[str, int], pi: int, a: int, b: int, c: int, d: int, a_w: int, b_w: int, d_w: int) -> List[int]:
    arithmetic = (q["q_m"] * a * b + q["q_l"] * a + q["q_r"] * b + q["q_o"] * c + q["q_f"] * d + q["q_c"]) * q["q_arith"] + pi
    rng = [delta(c - 4 * d), delta(b - 4 * c), delta(a - 4 * b), delta(d_w - 4 * a)]
    left, right, out = a_w - 4 * a, b_w - 4 * b, d_w - 4 * d
    logic = [delta(left), delta(right), delta(out), c - left * right, delta_xor_and(left, right, c, out, q["q_c"])]
    bit = d_w - 2 * d  # fixed_base extract_bit
    y_alpha, x_alpha = bit * bit * (q["q_r"] - 1) + 1, q["q_l"] * bit
    t = c * a * b * EDWARDS_D
    fixed = [bit * (bit - 1) * (bit + 1), bit * q["q_c"] - c, a_w + a_w * t - (a * y_alpha + b * x_alpha),
             b_w - b_w * t - (b * y_alpha + a * x_alpha)]
    x1_y2, y1_x2 = d_w, b * c
    var = [a * d - x1_y2, x1_y2 + y1_x2 - (a_w + a_w * EDWARDS_D * x1_y2 * y1_x2), b * d + a * c - (b_w - b_w * EDWARDS_D * x1_y2 * y1_x2)]
    terms = ([arithmetic] + [x * q["q_range"] for x in rng] + [x * q["q_logic"] for x in logic] +
             [x * q["q_fixed_group_add"] for x in fixed] + [x * q["q_variable_group_add"] for x in var])
    return [x % R_MOD for x in terms]


def row_identities(rows: Sequence[Row], witnesses: Sequence[int], pi: Dict[int, int], i: int) -> List[int]:
    """identity_evaluations of row i, with the wires rotated over next_pow2(len(rows)) rows and zero padding."""
    padded = 1
    while padded < len(rows):
        padded <<= 1

    def value(w: int) -> int:
        return witnesses[w] if w < len(witnesses) else 0  # witness_value: a missing witness reads zero

    q, a, b, c, d = rows[i]
    j = (i + 1) % padded
    a_w, b_w, d_w = (value(rows[j][1]), value(rows[j][2]), value(rows[j][4])) if j < len(rows) else (0, 0, 0)
    return identity_evaluations(q, pi.get(i, 0), value(a), value(b), value(c), value(d), a_w, b_w, d_w)


def first_failing(identities: Sequence[int]) -> Optional[str]:
    return next((IDENTITY_FAMILIES[k] for k, x in enumerate(identities) if x), None)


def unsatisfied_constraints(rows: Sequence[Row], witnesses: Sequence[int], pi: Dict[int, int],
                            only: Optional[Sequence[int]] = None) -> List[Tuple[int, str]]:
    """Every failing row (or every failing row of `only`), ascending, with the first identity it fails."""
    out = []
    for i in sorted(only) if only is not None else range(len(rows)):
        family = first_failing(row_identities(rows, witnesses, pi, i))
        if family is not None:
            out.append((i, family))
    return out


def report(unsatisfied: List[Tuple[int, str]], n_constraints: int) -> Optional[str]:
    """Debugger::unsatisfied_report without its "and was appended at path:line:col" clause."""
    if not unsatisfied:
        return None
    row, family = unsatisfied[0]
    return (f"plonk debugger: {len(unsatisfied)} of {n_constraints} constraints are unsatisfied; the first, constraint {row}, "
            f"fails the {family} identity")


def from_composer(comp) -> Tuple[List[Row], List[int], Dict[int, int]]:
    """The rows, witness table and public inputs of an oracle composer (oracle/pyref.py, oracle/gadgets.py)."""
    rows = [({k: g.sel[k] % R_MOD for k in SELECTORS}, g.a, g.b, g.c, g.d) for g in comp.constraints]
    return rows, [w % R_MOD for w in comp.witnesses], {i: v % R_MOD for i, v in comp.public_inputs.items()}


def _fr(raw: bytes, i: int) -> int:
    return int.from_bytes(raw[32 * i : 32 * i + 32], "little") * _MONT_R_INV % R_MOD


class _Lazy:
    """A column read from CircuitArrays bytes on demand, so that a check of a few rows of a large circuit decodes only
    those rows."""

    def __init__(self, n: int, get):
        self.n, self.get = n, get

    def __len__(self) -> int:
        return self.n

    def __getitem__(self, i: int):
        if not 0 <= i < self.n:
            raise IndexError(i)
        return self.get(i)


def from_arrays(arrays) -> Tuple[Sequence[Row], Sequence[int], Dict[int, int]]:
    """The same from the CircuitArrays of either composer (Montgomery bytes)."""
    n = arrays.constraints

    def wire(k: int, i: int) -> int:
        return int.from_bytes(arrays.wires[4 * (k * n + i) : 4 * (k * n + i) + 4], "little")

    rows = _Lazy(n, lambda i: ({k: _fr(arrays.selectors, s * n + i) for s, k in enumerate(SELECTORS)},) + tuple(wire(k, i) for k in range(4)))
    witnesses = _Lazy(arrays.n_witnesses, lambda i: _fr(arrays.witnesses, i))
    pi = {int.from_bytes(arrays.pi_idx[8 * k : 8 * k + 8], "little"): _fr(arrays.pi_vals, k) for k in range(arrays.n_pi)}
    return rows, witnesses, pi


# ---- the reference's unit-test fixtures (tests/golden/debugger_fixtures.json) --------------------------------------
FIXTURES = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "golden", "debugger_fixtures.json")


def load_fixtures() -> List[dict]:
    with open(FIXTURES) as f:
        return json.load(f)["cases"]


def fixture_circuit(case: dict) -> Tuple[List[Row], List[int], Dict[int, int]]:
    rows = [({k: int(r["selectors"][k], 16) for k in SELECTORS},) + tuple(r["wires"]) for r in case["rows"]]
    pi = {i: int(r["pi"], 16) for i, r in enumerate(case["rows"]) if int(r["pi"], 16)}
    return rows, [int(w, 16) for w in case["witnesses"]], pi


def to_arrays(rows: Sequence[Row], witnesses: Sequence[int], pi: Dict[int, int]):
    """CircuitArrays (plonk_b200.composer) of a circuit in this module's form."""
    from plonk_b200.composer import CircuitArrays

    def mont(vals) -> bytes:
        return b"".join((v * (1 << 256) % R_MOD).to_bytes(32, "little") for v in vals)

    n = len(rows)
    selectors = b"".join(mont(r[0][k] for r in rows) for k in SELECTORS)
    wires = b"".join(r[1 + k].to_bytes(4, "little") for k in range(4) for r in rows)
    idx = sorted(pi)
    return CircuitArrays(n, selectors, wires, mont(witnesses), b"".join(i.to_bytes(8, "little") for i in idx), mont(pi[i] for i in idx))
