"""pb200_public_parameters_setup / pb200_opening_key_check argument checks that need no device, the errors of the
Python mirror that are decided on the host, and the C++ mirror of PublicParameters / Compiler (compile and link)."""
import ctypes
import os

import pytest

from oracle import pyref as R
from plonk_b200._lib import PB200_ERR_CUDA, PB200_ERR_DEGREE_IS_ZERO, PB200_ERR_INVALID_ARG, lib

ONE = R.fr_to_mont_bytes(1)
R_LIMBS = R.R_MOD.to_bytes(32, "little")  # r itself: zero mod r, not a canonical draw


def _setup(max_degree, draws, pts=True, okey=True):
    n = max(max_degree + 7, 1)
    p = ctypes.create_string_buffer(96 * min(n, 64)) if pts else None
    k = ctypes.create_string_buffer(240) if okey else None
    return lib().pb200_public_parameters_setup(max_degree, *draws, p, k)


def test_setup_argument_errors_come_before_the_device():
    assert _setup(0, [ONE, ONE, ONE]) == PB200_ERR_DEGREE_IS_ZERO
    for k in range(3):
        for bad in (bytes(32), R_LIMBS, b"\xff" * 32):
            draws = [ONE, ONE, ONE]
            draws[k] = bad
            assert _setup(4, draws) == PB200_ERR_INVALID_ARG, (k, bad)
        draws = [ONE, ONE, ONE]
        draws[k] = None
        assert _setup(4, draws) == PB200_ERR_INVALID_ARG
    assert _setup(4, [ONE, ONE, ONE], pts=False) == PB200_ERR_INVALID_ARG
    assert _setup(4, [ONE, ONE, ONE], okey=False) == PB200_ERR_INVALID_ARG
    assert lib().pb200_opening_key_check(None) == PB200_ERR_INVALID_ARG


def test_no_cuda_device_fails_loudly():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a device is present")
    assert _setup(4, [ONE, ONE, ONE]) == PB200_ERR_CUDA
    assert lib().pb200_opening_key_check(bytes(240)) == PB200_ERR_CUDA


def test_python_mirror_host_errors():
    import plonk_b200

    with pytest.raises(plonk_b200.DegreeIsZero):
        plonk_b200.PublicParameters.setup(0, [ONE, ONE, ONE])
    for n in (0, 100, 240):
        with pytest.raises(plonk_b200.NotEnoughBytes):
            plonk_b200.PublicParameters.from_slice(bytes(n))
    with pytest.raises(plonk_b200.NotEnoughBytes):
        plonk_b200.PublicParameters.from_slice_unchecked(bytes(239))


def test_cpp_mirror_compile_check_builds():
    from tests.test_host_logic import _build_cpp

    assert os.path.exists(_build_cpp("compile_check"))
