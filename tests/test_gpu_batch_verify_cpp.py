"""include/plonk_b200.hpp's Verifier::batch_verify end to end (tests/cpp/batch_verify_check.cpp): batch verdicts and
the reference's error kinds through the C++ mirror."""
import os
import struct
import subprocess

import pytest

from oracle import pyref as R
from tests.test_host_logic import _build_cpp


def test_cpp_batch_verify_check_compiles_and_links():
    assert os.path.exists(_build_cpp("batch_verify_check"))


@pytest.mark.gpu
def test_cpp_mirror_batch_verifies_like_the_reference(tmp_path):
    from tests.test_gpu_verifier import Case, _synthetic

    c = Case(b"cpp-batch-verify", _synthetic(200, 22))
    a = c.arrays
    good = [c.prove(1), c.prove(2)]
    bad = bytearray(good[0])
    bad[528 + 40] ^= 1  # an evaluation moved: still canonical, fails the check
    malformed = good[1][:528] + R.R_MOD.to_bytes(32, "little") + good[1][560:]
    proofs = good + [bytes(bad), malformed]
    idx = [int.from_bytes(a.pi_idx[8 * i : 8 * i + 8], "little") for i in range(len(a.pi_idx) // 8)]
    blob = struct.pack("<4Q", len(c.label), a.constraints, len(idx), len(proofs)) + c.label + b"".join(c.comms) + c.okey
    blob += b"".join(struct.pack("<Q", i) for i in idx) + b"".join(proofs) + a.pi_vals * len(proofs)
    f = tmp_path / "case.bin"
    f.write_bytes(blob)
    out = subprocess.run([_build_cpp("batch_verify_check"), str(f)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.splitlines() == [
        "valid ok", "valid_v3 ok", "valid_under_v2 ProofVerificationError", "one_bad ProofVerificationError",
        "bad_and_malformed PointMalformed", "empty ProofVerificationError", "wrong_pi_count InvalidArgument",
        "unknown_version InvalidArgument", "from_bytes_valid ok", "from_bytes_empty ProofVerificationError",
    ]
