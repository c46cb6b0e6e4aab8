"""include/plonk_b200.hpp's DevicePublicParameters end to end (tests/cpp/device_pp_check.cpp): setup, compile, prove
and verify through the device parameters, equality with the host parameters' compile, try_from_bytes against them and
the error kinds, through the C++ mirror."""
import subprocess

import pytest

from tests.test_host_logic import _build_cpp


@pytest.mark.gpu
def test_cpp_mirror_device_public_parameters():
    out = subprocess.run([_build_cpp("device_pp_check")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.splitlines() == [
        "setup ok", "to_host ok", "verify ok", "same_as_host ok", "shared_tables ok", "try_from_bytes ok",
        "try_from_bytes_other_pp InvalidArgument", "compressed ok",
        "setup_degree_zero DegreeIsZero", "setup_zero_draw InvalidArgument",
        "from_slice ok", "from_slice_short NotEnoughBytes", "from_slice_identity_g PointMalformed", "from_slice_unchecked ok",
        "compile_small TruncatedDegreeTooLarge", "compile_exact ok",
    ]
