"""include/plonk_b200.hpp's compress and Compiler::compile_with_compressed (tests/cpp/compressed_check.cpp): the
reference's examples/circuit.rs compiled from its compressed bytes gives Compiler::compile's keys and proofs, and the
InvalidCompressedCircuit and BlsScalarMalformed kinds reach the C++ caller."""
import subprocess

import pytest

from tests.test_host_logic import _build_cpp


@pytest.mark.gpu
def test_cpp_mirror_compiles_compressed_circuits():
    out = subprocess.run([_build_cpp("compressed_check")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.splitlines() == [
        "prover_bytes equal", "verifier_bytes equal", "proof equal", "verify ok", "verify_wrong_pi ProofVerificationError",
        "garbage InvalidCompressedCircuit", "small_parameters InvalidCompressedCircuit",
        "non_canonical_scalar BlsScalarMalformed", "bad_witness_index InvalidCompressedCircuit",
    ]
