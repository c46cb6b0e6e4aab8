"""include/plonk_b200.hpp's PublicParameters and Compiler end to end (tests/cpp/compile_check.cpp): the reference's
examples/circuit.rs and the error kinds of setup, from_slice and compile through the C++ mirror."""
import subprocess

import pytest

from tests.test_host_logic import _build_cpp


@pytest.mark.gpu
def test_cpp_mirror_compiles_and_runs_the_reference_example():
    out = subprocess.run([_build_cpp("compile_check")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.splitlines() == [
        "setup ok", "verify ok", "verify_wrong_pi ProofVerificationError",
        "setup_degree_zero DegreeIsZero", "setup_zero_draw InvalidArgument",
        "from_slice ok", "from_slice_short NotEnoughBytes", "from_slice_identity_g PointMalformed", "from_slice_unchecked ok",
        "compile_small TruncatedDegreeTooLarge", "compile_exact ok",
    ]
