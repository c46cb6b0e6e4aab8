"""Which constraint a witness breaks: the reference's debugger check (src/debugger.rs:95-236) on the GPU.

`unsatisfied_constraints(arrays)` checks a circuit as the composer holds it at prove time (its selectors, wires,
witness table and public inputs), which is what the reference's debugger checks; `Prover.unsatisfied_constraints`
checks the same witnesses against the compiled prover's own selectors, which is what a proof enforces.  Both return
every failing row with the first of the 17 gate identities it fails, by the reference's names (IDENTITY_FAMILIES,
debugger.rs:31-49).  The report is the reference's sentence without its "and was appended at path:line:col" clause:
no call sites are recorded here."""
from __future__ import annotations

import ctypes
from typing import Callable, List, Optional, Tuple

from ._lib import check, lib

N_IDENTITIES = 17


def identity_family(k: int) -> str:
    """IDENTITY_FAMILIES[k] of the reference, k = 0..16."""
    name = lib().pb200_identity_family(k)
    if name is None:
        raise IndexError(k)
    return name.decode()


def query(call: Callable, cap: int) -> Tuple[int, List[Tuple[int, str]]]:
    """Runs call(cap, rows, families, n) - one of the C entry points with its circuit arguments bound - and returns the
    number of failing constraints and the first min(cap, that number) of them as (row, family name)."""
    n = ctypes.c_size_t()
    rows = (ctypes.c_uint64 * max(cap, 1))()
    fams = (ctypes.c_int32 * max(cap, 1))()
    check(call(cap, rows if cap else None, fams if cap else None, ctypes.byref(n)))
    return n.value, [(rows[i], identity_family(fams[i])) for i in range(min(cap, n.value))]


def report(n_unsatisfied: int, n_constraints: int, first: List[Tuple[int, str]]) -> Optional[str]:
    """Debugger::unsatisfied_report (debugger.rs:221-236) without the call-site clause; None when nothing fails."""
    if not n_unsatisfied:
        return None
    row, family = first[0]
    return (f"plonk debugger: {n_unsatisfied} of {n_constraints} constraints are unsatisfied; the first, constraint {row}, "
            f"fails the {family} identity")


def _circuit_call(arrays) -> Callable:
    return lambda cap, rows, fams, n: lib().pb200_circuit_unsatisfied(
        arrays.constraints, arrays.selectors or None, arrays.wires or None, arrays.witnesses or None, arrays.n_witnesses,
        arrays.pi_idx or None, arrays.pi_vals or None, arrays.n_pi, cap, rows, fams, n)


def unsatisfied_constraints(arrays) -> List[Tuple[int, str]]:
    """Debugger::unsatisfied_constraints for the CircuitArrays of a composer (`.arrays()` of either composer): every
    failing row, ascending, with the first identity it fails."""
    return query(_circuit_call(arrays), arrays.constraints)[1]


def unsatisfied_report(arrays) -> Optional[str]:
    """Debugger::unsatisfied_report for the CircuitArrays of a composer, without the call-site clause."""
    n, first = query(_circuit_call(arrays), 1)
    return report(n, arrays.constraints, first)
