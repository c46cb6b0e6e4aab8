"""include/plonk_b200.hpp's batch_verify_groups end to end (tests/cpp/batch_verify_groups_check.cpp): grouped verdicts
over two circuits on one SRS and the reference's error kinds through the C++ mirror."""
import os
import struct
import subprocess

import pytest

from tests.test_host_logic import _build_cpp


def test_cpp_batch_verify_groups_check_compiles_and_links():
    assert os.path.exists(_build_cpp("batch_verify_groups_check"))


@pytest.mark.gpu
def test_cpp_mirror_batch_verifies_groups_like_the_reference(tmp_path):
    from tests.test_gpu_verifier import Case, _synthetic

    blob = struct.pack("<Q", 2)
    for label, arr in ((b"cpp-groups-a", _synthetic(200, 22)), (b"cpp-groups-b", _synthetic(400, 23, n_public=2))):
        c = Case(label, arr)
        proofs = [c.prove(1), c.prove(2)]
        idx = [int.from_bytes(arr.pi_idx[8 * i : 8 * i + 8], "little") for i in range(len(arr.pi_idx) // 8)]
        blob += struct.pack("<4Q", len(label), arr.constraints, len(idx), len(proofs)) + label + b"".join(c.comms) + c.okey
        blob += b"".join(struct.pack("<Q", i) for i in idx) + b"".join(proofs) + arr.pi_vals * len(proofs)
    f = tmp_path / "case.bin"
    f.write_bytes(blob)
    out = subprocess.run([_build_cpp("batch_verify_groups_check"), str(f)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.splitlines() == [
        "valid ok", "same_verifier_twice ok", "one_bad ProofVerificationError", "bad_and_malformed PointMalformed",
        "under_v2 ProofVerificationError", "no_groups ProofVerificationError", "all_empty ProofVerificationError", "empty_group ok",
        "wrong_pi_count InvalidArgument", "unknown_version InvalidArgument", "from_bytes_valid ok",
    ]
