"""include/plonk_b200.hpp's Prover::to_bytes / serialized_size and CommitKey::to_var_bytes / to_raw_var_bytes end to
end (tests/cpp/serialize_check.cpp): the C++ mirror writes the bytes the Python mirror writes."""
import os
import random
import struct
import subprocess

import pytest

from oracle import cref
from oracle import pyref as R
from tests.test_host_logic import _build_cpp
from tests.util import bases_to_abi


def _fnv1a(blob):
    h = 0xCBF29CE484222325
    for byte in blob:
        h = ((h ^ byte) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return "%016x" % h


def test_cpp_serialize_check_compiles_and_links():
    assert os.path.exists(_build_cpp("serialize_check"))


@pytest.mark.gpu
def test_cpp_mirror_serializes_like_the_python_mirror(tmp_path):
    import plonk_b200
    from plonk_b200 import kzg
    from plonk_b200._lib import check, lib

    check(lib().pb200_init(0))
    rng = random.Random(21)
    pp = R.srs_from_secret(256 + 7, rng.randrange(1, R.R_MOD), rng.randrange(1, R.R_MOD))
    comp = R.Composer.initialized()
    R.synthetic_arith_circuit(comp, 200, seed=22, n_public=2, widgets=4)
    a = cref.CircuitArrays(comp)
    srs_raw = bases_to_abi(pp)
    label = b"cpp-serialize"
    blob = struct.pack("<5Q", len(label), a.constraints, a.n_witnesses, len(pp), a.n_pi) + label + a.selectors + a.wires + srs_raw
    blob += a.witnesses + a.pi_idx + a.pi_vals + cref.draw_blinders(R.StdRng.seed_from_u64(5))
    f = tmp_path / "case.bin"
    f.write_bytes(blob)
    out = subprocess.run([_build_cpp("serialize_check"), str(f)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    want = plonk_b200.Prover(label, a.constraints, a.selectors, a.wires, a.n_witnesses, srs_raw).to_bytes()
    raw_var, var = kzg.commit_key_to_raw_var_bytes(srs_raw), kzg.commit_key_to_var_bytes(srs_raw)
    assert out.stdout.splitlines() == [
        "serialized_size equal", "prover %d %s" % (len(want), _fnv1a(want)), "round_trip equal", "proof equal",
        "truncated InvalidArgument", "commit_key_raw %d %s" % (len(raw_var), _fnv1a(raw_var)),
        "commit_key_var %d %s" % (len(var), _fnv1a(var)), "commit_key_round_trip equal",
    ]
