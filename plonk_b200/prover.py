"""Prover mirror (reference src/compiler/prover.rs: Prover::new :53-115, Prover::prove :352-362,
Prover::prove_with_version :364-413) over the device-resident CUDA prover.

A circuit crosses the boundary as flat arrays, i.e. what Compiler::preprocess reads out of the
Composer (reference src/compiler.rs:132-170): 11 selector columns, 4 wire columns, the witness
table and the sparse public inputs."""
from __future__ import annotations

import ctypes

from . import debugger
from ._lib import PB200_ERR_UNSATISFIED, PB200_ERR_UNSUPPORTED_VERSION, Pb200Error, PlonkVersion, check, lib
from .srs import DevicePublicParameters

PROOF_BYTES = 1008


class CircuitUnsatisfied(ValueError):
    """Error::CircuitUnsatisfied (reference src/proof_system/quotient_poly.rs:132-134)."""


class UnsupportedProvingVersion(ValueError):
    """Error::UnsupportedProvingVersion: PlonkVersion::V1 proofs cannot be made (reference prover.rs:376)."""


def compressed_circuit_info(compressed: bytes, n_srs_points: int):
    """pb200_compressed_circuit_info: (constraints, witnesses, labels, public-input count, public-input positions as
    little-endian u64) of a compressed circuit, decoded within the bounds of public parameters of n_srs_points points.
    Raises Pb200Error (PB200_ERR_INVALID_COMPRESSED or PB200_ERR_SCALAR_MALFORMED) for a description they reject."""
    n, nw, nl, npi = ctypes.c_size_t(), ctypes.c_uint64(), ctypes.c_size_t(), ctypes.c_size_t()
    args = (compressed, len(compressed), n_srs_points, ctypes.byref(n), ctypes.byref(nw), ctypes.byref(nl), ctypes.byref(npi))
    check(lib().pb200_compressed_circuit_info(*args, None))
    idx = ctypes.create_string_buffer(max(1, npi.value) * 8)
    if npi.value:
        check(lib().pb200_compressed_circuit_info(*args, idx))
    return n.value, nw.value, nl.value, npi.value, idx.raw[: 8 * npi.value]


class Prover:
    def __init__(self, label: bytes, n_constraints: int, selectors: bytes, wires: bytes, n_witnesses: int, srs_raw):
        """srs_raw: the commit key as 96-byte raw points, or a DevicePublicParameters whose tables the prover shares."""
        assert len(selectors) == 11 * n_constraints * 32 and len(wires) == 4 * n_constraints * 4
        h = ctypes.c_void_p()
        if isinstance(srs_raw, DevicePublicParameters):
            check(lib().pb200_prover_new_pp(srs_raw._h, label, len(label), n_constraints, selectors, wires, n_witnesses, ctypes.byref(h)))
        else:
            check(lib().pb200_prover_new(label, len(label), n_constraints, selectors, wires, n_witnesses, srs_raw,
                                         len(srs_raw) // 96, ctypes.byref(h)))
        self._h = h
        self.n_constraints = n_constraints
        self.n_witnesses = n_witnesses

    @classmethod
    def from_bytes(cls, prover_bytes: bytes, wires: bytes, n_witnesses: int, pp: "DevicePublicParameters" = None) -> "Prover":
        """Prover::try_from_bytes (prover.rs:265-350) for the output of Prover::to_bytes; the circuit's wiring
        (4 x constraints u32) is not part of that format and comes alongside.  With pp, the serialized commit key must
        be a prefix of pp's points (else a Pb200Error with PB200_ERR_INVALID_ARG) and the prover shares pp's tables."""
        self = cls.__new__(cls)
        h = ctypes.c_void_p()
        if pp is None:
            check(lib().pb200_prover_from_bytes(prover_bytes, len(prover_bytes), wires, n_witnesses, ctypes.byref(h)))
        else:
            check(lib().pb200_prover_from_bytes_pp(pp._h, prover_bytes, len(prover_bytes), wires, n_witnesses, ctypes.byref(h)))
        self._h = h
        self.n_constraints = len(wires) // 16
        self.n_witnesses = n_witnesses
        return self

    @classmethod
    def from_compressed(cls, label: bytes, compressed: bytes, srs_raw, info=None) -> "Prover":
        """The Prover of Compiler::compile_with_compressed (compiler.rs:84-112): the selector columns are expanded on the
        GPU from the description's tables.  prove takes the re-run circuit's witness table, as for any Prover.  srs_raw:
        raw points or a DevicePublicParameters, as for Prover().  info: what compressed_circuit_info returned for these
        bytes and keys, if the caller has it already."""
        device = isinstance(srs_raw, DevicePublicParameters)
        n_points = srs_raw.points() if device else len(srs_raw) // 96
        n_constraints, n_witnesses, _, _, _ = info or compressed_circuit_info(compressed, n_points)
        self = cls.__new__(cls)
        h = ctypes.c_void_p()
        if device:
            check(lib().pb200_prover_from_compressed_pp(srs_raw._h, label, len(label), compressed, len(compressed), ctypes.byref(h)))
        else:
            check(lib().pb200_prover_from_compressed(label, len(label), compressed, len(compressed), srs_raw, n_points,
                                                     ctypes.byref(h)))
        self._h = h
        self.n_constraints = n_constraints
        self.n_witnesses = n_witnesses
        return self

    def serialized_size(self) -> int:
        """Prover::serialized_size (prover.rs:233-235)."""
        n = ctypes.c_size_t()
        check(lib().pb200_prover_to_bytes(self._h, None, 0, ctypes.byref(n)))
        return n.value

    def to_bytes(self) -> bytes:
        """Prover::to_bytes (prover.rs:238-263): what from_bytes reads, here or in another process; the scalars are
        converted to canonical form on the GPU.  Safe beside proofs running on this prover."""
        n = ctypes.c_size_t(self.serialized_size())
        out = ctypes.create_string_buffer(n.value)
        check(lib().pb200_prover_to_bytes(self._h, out, n.value, ctypes.byref(n)))
        return out.raw

    def commitments(self):
        out = ctypes.create_string_buffer(15 * 48)
        check(lib().pb200_prover_commitments(self._h, out))
        return [out.raw[48 * i : 48 * i + 48] for i in range(15)]

    def prove(self, witnesses: bytes, pi_idx: bytes, pi_vals: bytes, blinders: bytes) -> bytes:
        """Prover::prove (PlonkVersion::V3).  witnesses: n_witnesses x 32 B; pi_idx: u64 LE positions; pi_vals: 32 B
        each; blinders: 14 x 32 B."""
        return self.prove_with_version(PlonkVersion.V3, witnesses, pi_idx, pi_vals, blinders)

    def prove_with_version(self, version: PlonkVersion, witnesses: bytes, pi_idx: bytes, pi_vals: bytes, blinders: bytes) -> bytes:
        """Prover::prove_with_version: as prove, under `version`.  V3 is prove; V2 uses the legacy transcript seed;
        V1 raises UnsupportedProvingVersion; any other value is a Pb200Error with PB200_ERR_INVALID_ARG."""
        assert len(blinders) == 14 * 32 and len(witnesses) == self.n_witnesses * 32
        n_pi = len(pi_idx) // 8
        out = ctypes.create_string_buffer(PROOF_BYTES)
        try:
            check(lib().pb200_prove_with_version(self._h, int(version), witnesses, self.n_witnesses, pi_idx or None, pi_vals or None,
                                                 n_pi, blinders, out))
        except Pb200Error as e:
            if e.code == PB200_ERR_UNSATISFIED:
                raise CircuitUnsatisfied() from e
            if e.code == PB200_ERR_UNSUPPORTED_VERSION:
                raise UnsupportedProvingVersion("UnsupportedProvingVersion") from e
            raise
        return out.raw

    def _unsatisfied_call(self, witnesses: bytes, pi_idx: bytes, pi_vals: bytes):
        assert len(witnesses) == self.n_witnesses * 32
        return lambda cap, rows, fams, n: lib().pb200_prover_unsatisfied(self._h, witnesses, self.n_witnesses, pi_idx or None,
                                                                        pi_vals or None, len(pi_idx) // 8, cap, rows, fams, n)

    def unsatisfied_constraints(self, witnesses: bytes, pi_idx: bytes, pi_vals: bytes):
        """The reference debugger's check (debugger.rs:95-205) against this prover's own selectors, with prove's
        arguments: every failing row, ascending, as (row, identity family).  Empty means prove makes the proof.  Safe
        beside proofs running on this prover."""
        return debugger.query(self._unsatisfied_call(witnesses, pi_idx, pi_vals), self.n_constraints)[1]

    def unsatisfied_report(self, witnesses: bytes, pi_idx: bytes, pi_vals: bytes):
        """Debugger::unsatisfied_report (debugger.rs:221-236) for unsatisfied_constraints, without the call-site
        clause; None when every constraint holds."""
        n, first = debugger.query(self._unsatisfied_call(witnesses, pi_idx, pi_vals), 1)
        return debugger.report(n, self.n_constraints, first)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().pb200_prover_free(self._h)
                self._h = None
        except Exception:
            pass
