"""Compiler mirror (reference src/compiler.rs: Compiler::compile, compile_with_circuit, compile_with_compressed and
preprocess :84-461): Prover::new on the GPU, its 15 verifier-key commitments, and the Verifier for the same circuit and
opening key.  Circuit::compress (src/composer/circuit.rs:28-45) writes the description compile_with_compressed reads."""
from __future__ import annotations

import ctypes
from typing import Callable, Tuple, Union

from ._lib import PB200_ERR_DEGREE_TOO_LARGE, PB200_ERR_INVALID_ARG, PB200_ERR_INVALID_COMPRESSED, PB200_ERR_SCALAR_MALFORMED, Pb200Error, check, lib
from .prover import Prover, compressed_circuit_info
from .srs import DevicePublicParameters, PublicParameters
from .verifier import Verifier


class TruncatedDegreeTooLarge(ValueError):
    """Error::TruncatedDegreeTooLarge: the public parameters are too small for the circuit.  PublicParameters::trim
    needs next_pow2(constraints + 6) + 6 <= pp.max_degree() (compiler.rs:121-124, srs.rs:188-196)."""


class InvalidCompressedCircuit(ValueError):
    """Error::InvalidCompressedCircuit: a compressed circuit that does not inflate, unpack or validate within the bounds
    of the public parameters (compress.rs:242-334)."""


class BlsScalarMalformed(ValueError):
    """Error::BlsScalarMalformed: a scalar of a compressed circuit is not canonical (compress.rs:329-335)."""


def _compressed_errors(call):
    try:
        return call()
    except Pb200Error as e:
        if e.code == PB200_ERR_INVALID_COMPRESSED:
            raise InvalidCompressedCircuit("InvalidCompressedCircuit") from e
        if e.code == PB200_ERR_SCALAR_MALFORMED:
            raise BlsScalarMalformed("BlsScalarMalformed") from e
        raise


def compress_arrays(a, hades_optimization: bool = True) -> bytes:
    """CompressedCircuit::from_composer (compress.rs:136-240) for a circuit's arrays (anything with constraints,
    selectors, wires, n_witnesses and pi_idx, as Composer.arrays() returns them): MessagePack behind raw deflate."""
    n = ctypes.c_size_t()
    args = (a.constraints, a.selectors, a.wires, a.n_witnesses, a.pi_idx or None, len(a.pi_idx) // 8, int(bool(hades_optimization)))
    # one pass with a generous buffer; a second one only when the description is larger than that
    cap = 4096 + 64 * a.constraints
    out = ctypes.create_string_buffer(cap)
    rc = lib().pb200_circuit_compress(*args, out, cap, ctypes.byref(n))
    if rc == PB200_ERR_INVALID_ARG and n.value > cap:
        out = ctypes.create_string_buffer(n.value)
        rc = lib().pb200_circuit_compress(*args, out, n.value, ctypes.byref(n))
    check(rc)
    return out.raw[: n.value]


def compress(circuit: Callable, hades_optimization: bool = True) -> bytes:
    """Circuit::compress (circuit.rs:28-45): circuit(composer) fills a fresh native Composer.initialized(), whose
    description is returned compressed.  The reference always compresses with hades_optimization = true."""
    from .gadgets import Composer

    composer = Composer.initialized()
    circuit(composer)
    return compress_arrays(composer.arrays(), hades_optimization)


Parameters = Union[PublicParameters, DevicePublicParameters]


def _keys(pp: Parameters):
    """What Prover takes for the commit key: the raw points of host parameters, or the device parameters themselves."""
    return pp if isinstance(pp, DevicePublicParameters) else pp.raw_points


def _points(pp: Parameters) -> int:
    return pp.points() if isinstance(pp, DevicePublicParameters) else len(pp.raw_points) // 96


class Compiler:
    """Each method takes PublicParameters or DevicePublicParameters; the provers compiled from one
    DevicePublicParameters share its MSM tables instead of building their own."""

    @staticmethod
    def compile(pp: Parameters, label: bytes, composer) -> Tuple[Prover, Verifier]:
        """Compiler::compile for a filled composer: anything with .arrays() (the Python Composer or the native gadget
        Composer).  Returns (Prover, Verifier)."""
        a = composer.arrays()
        try:
            prover = Prover(label, a.constraints, a.selectors, a.wires, a.n_witnesses, _keys(pp))
        except Pb200Error as e:
            if e.code == PB200_ERR_DEGREE_TOO_LARGE:
                raise TruncatedDegreeTooLarge("TruncatedDegreeTooLarge") from e
            raise
        verifier = Verifier(label, a.constraints, prover.commitments(), pp.opening_key, a.pi_idx)
        return prover, verifier

    @staticmethod
    def compile_with_circuit(pp: Parameters, label: bytes, circuit: Callable) -> Tuple[Prover, Verifier]:
        """Compiler::compile_with_circuit: circuit(composer) fills a fresh native Composer.initialized()."""
        from .gadgets import Composer

        composer = Composer.initialized()
        circuit(composer)
        return Compiler.compile(pp, label, composer)

    @staticmethod
    def compile_with_compressed(pp: Parameters, label: bytes, compressed: bytes) -> Tuple[Prover, Verifier]:
        """Compiler::compile_with_compressed (compiler.rs:84-112): the Prover and Verifier of a description written by
        compress.  The public parameters bound the decoding; raises InvalidCompressedCircuit or BlsScalarMalformed for a
        description they reject.  The Prover's prove takes the re-run circuit's witness table."""
        info = _compressed_errors(lambda: compressed_circuit_info(compressed, _points(pp)))
        prover = _compressed_errors(lambda: Prover.from_compressed(label, compressed, _keys(pp), info))
        n_constraints, _, _, _, pi_idx = info
        verifier = Verifier(label, n_constraints, prover.commitments(), pp.opening_key, pi_idx)
        return prover, verifier
