"""include/plonk_b200.hpp's Verifier end to end (tests/cpp/verifier_check.cpp): verdicts, the byte round trip and the
reference's error kinds through the C++ mirror."""
import os
import struct
import subprocess

import pytest

from oracle import pyref as R
from tests.models import pairing_model as M
from tests.test_host_logic import _build_cpp


def test_cpp_verifier_check_compiles_and_links():
    assert os.path.exists(_build_cpp("verifier_check"))


@pytest.mark.gpu
def test_cpp_mirror_verifies_like_the_reference(tmp_path):
    from tests.test_gpu_verifier import Case, _synthetic

    c = Case(b"cpp-verifier", _synthetic(200, 21))
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
    out = subprocess.run([_build_cpp("verifier_check"), str(f)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.splitlines() == [
        "verify ok", "verify ok", "verify ProofVerificationError", "verify PointMalformed",
        "batch 0 0 -11 -10", "round_trip equal", "from_bytes_verify ok", "wrong_pi_count InvalidArgument",
        "truncated InvalidArgument", "identity_h PointMalformed",
    ]
    assert M.verify_with_pairing(good[0], c.label, a.constraints, {k: R.g1_decompress(x) for k, x in zip(R.POLY_NAMES, c.comms)},
                                 idx, R.fr_vec_from_mont_bytes(a.pi_vals), c.okey)
