"""Compiler mirror (reference src/compiler.rs: Compiler::compile, compile_with_circuit and preprocess :116-461):
Prover::new on the GPU, its 15 verifier-key commitments, and the Verifier for the same circuit and opening key."""
from __future__ import annotations

from typing import Callable, Tuple

from ._lib import PB200_ERR_DEGREE_TOO_LARGE, Pb200Error
from .prover import Prover
from .srs import PublicParameters
from .verifier import Verifier


class TruncatedDegreeTooLarge(ValueError):
    """Error::TruncatedDegreeTooLarge: the public parameters are too small for the circuit.  PublicParameters::trim
    needs next_pow2(constraints + 6) + 6 <= pp.max_degree() (compiler.rs:121-124, srs.rs:188-196)."""


class Compiler:
    @staticmethod
    def compile(pp: PublicParameters, label: bytes, composer) -> Tuple[Prover, Verifier]:
        """Compiler::compile for a filled composer: anything with .arrays() (the Python Composer or the native gadget
        Composer).  Returns (Prover, Verifier)."""
        a = composer.arrays()
        try:
            prover = Prover(label, a.constraints, a.selectors, a.wires, a.n_witnesses, pp.raw_points)
        except Pb200Error as e:
            if e.code == PB200_ERR_DEGREE_TOO_LARGE:
                raise TruncatedDegreeTooLarge("TruncatedDegreeTooLarge") from e
            raise
        verifier = Verifier(label, a.constraints, prover.commitments(), pp.opening_key, a.pi_idx)
        return prover, verifier

    @staticmethod
    def compile_with_circuit(pp: PublicParameters, label: bytes, circuit: Callable) -> Tuple[Prover, Verifier]:
        """Compiler::compile_with_circuit: circuit(composer) fills a fresh native Composer.initialized()."""
        from .gadgets import Composer

        composer = Composer.initialized()
        circuit(composer)
        return Compiler.compile(pp, label, composer)
