"""The host-only key writer (pb200_commit_key_to_raw_var_bytes = CommitKey::to_raw_var_bytes, key.rs:215-229) and
the ABI surface of the three serialization entry points.  No device needed."""
import ctypes
import os
import re

from oracle import serialize as S
from tests.util import bases_to_abi, progression_bases


def _to_raw_var_bytes(raw, n, cap=None):
    from plonk_b200._lib import lib

    ln = ctypes.c_size_t()
    assert lib().pb200_commit_key_to_raw_var_bytes(raw, n, None, 0, ctypes.byref(ln)) == 0  # out = NULL: length only
    cap = ln.value if cap is None else cap
    guard = 16
    buf = ctypes.create_string_buffer(b"\xa5" * (cap + guard), cap + guard)
    rc = lib().pb200_commit_key_to_raw_var_bytes(raw, n, buf, cap, ctypes.byref(ln))
    assert buf.raw[cap:] == b"\xa5" * guard
    return rc, ln.value, buf.raw[:cap]


def test_commit_key_to_raw_var_bytes_writes_what_the_loader_reads():
    from plonk_b200._lib import check, lib

    pts = progression_bases(9, 3, 5)
    pts[0] = None
    pts[4] = None
    raw = b"".join(bytes(96) if p is None else bases_to_abi([p]) for p in pts)  # this library's identity: zeros
    want = S.commit_key_to_raw_var_bytes(pts)
    rc, ln, blob = _to_raw_var_bytes(raw, 9)
    assert (rc, ln) == (0, 8 + 9 * 97) and blob == want
    # the identity leaves as the reference's G1Affine::identity(): x = 0, y = Montgomery one, flag 1
    assert blob[8:8 + 97] == S.g1_to_raw_bytes_97(None) and blob[8 + 96] == 1 and blob[8 + 97 + 96] == 0
    back = ctypes.create_string_buffer(96 * 9)
    check(lib().pb200_commit_key_from_raw_var_bytes(blob, len(blob), 0, back))
    assert back.raw == raw
    # a buffer one byte short: PB200_ERR_INVALID_ARG, nothing written, the length still reported
    rc, ln, untouched = _to_raw_var_bytes(raw, 9, cap=8 + 9 * 97 - 1)
    assert (rc, ln) == (-4, 8 + 9 * 97) and untouched == b"\xa5" * (8 + 9 * 97 - 1)
    # an empty key is its 8-byte zero count
    assert _to_raw_var_bytes(None, 0) == (0, 8, bytes(8))
    assert lib().pb200_commit_key_to_raw_var_bytes(raw, 9, None, 0, None) == -4
    assert lib().pb200_commit_key_to_raw_var_bytes(None, 9, None, 0, ctypes.byref(ctypes.c_size_t())) == -4


def test_public_parameters_raw_form_is_the_opening_key_then_the_commit_key():
    from plonk_b200 import kzg

    pts = progression_bases(5, 2, 9)
    raw = bases_to_abi(pts)
    okey = bytes(range(240))
    blob = kzg.public_parameters_to_raw_var_bytes(okey, raw)
    assert blob == okey + S.commit_key_to_raw_var_bytes(pts)
    assert kzg.commit_key_bytes_of_public_parameters(blob) == kzg.commit_key_to_raw_var_bytes(raw)


def test_serialization_entry_points_are_declared_and_exported():
    from plonk_b200._lib import EXPORTS, LIB_PATH

    header = open(os.path.join(os.path.dirname(LIB_PATH), "..", "include", "plonk_b200.h")).read()
    header = " ".join(re.sub(r"/\*.*?\*/", "", header, flags=re.S).split())
    L = ctypes.CDLL(LIB_PATH)
    for proto in (
        "int pb200_prover_to_bytes(const pb200_prover_t* prover, uint8_t* out, size_t cap, size_t* len);",
        "int pb200_g1_compress_batch(const uint8_t* raw_points, size_t n_points, uint8_t* out_48);",
        "int pb200_commit_key_to_raw_var_bytes(const uint8_t* raw_points, size_t n_points, uint8_t* out, size_t cap, size_t* len);",
    ):
        assert proto in header, proto
        name = re.search(r"pb200_[a-z0-9_]+", proto).group(0)
        assert name in EXPORTS and hasattr(L, name), name
