"""The pairing oracle (tests/models/pairing_model.py) against the pairing's defining properties, the G2 codec, the
verifier's final check against the secret-based one of oracle/verify.py, and the Verifier byte format.  CPU only."""
import ctypes
import random

import pytest

from oracle import pyref as R
from oracle import verify as V
from tests.models import pairing_model as M

rng = random.Random(0x9A1)


def test_g2_generator_is_on_the_curve_and_of_order_r():
    assert M.g2_on_curve(M.G2_GEN)
    assert M.g2_mul(M.G2_GEN, M.Q_R) is None


def test_pairing_is_bilinear_and_non_degenerate():
    p, q = R.g1_mul(R.G1_GEN, rng.randrange(1, M.Q_R)), M.g2_mul(M.G2_GEN, rng.randrange(1, M.Q_R))
    a, b = rng.randrange(1, M.Q_R), rng.randrange(1, M.Q_R)
    e = M.pairing(p, q)
    assert e != M.ONE12
    assert M.pairing(R.g1_mul(p, a), M.g2_mul(q, b)) == M.f12_pow(e, a * b % M.Q_R)
    assert M.f12_pow(e, M.Q_R) == M.ONE12
    assert M.f12_mul(M.pairing(R.g1_neg(p), q), e) == M.ONE12
    assert M.pairing(None, q) == M.ONE12 and M.pairing(p, None) == M.ONE12


def test_final_exponentiation_chain_raises_to_three_times_the_textbook_exponent():
    """pairing.cuh's hard part (zkcrypto's x-chain) is f^(l0 + l1 p + l2 p^2 + l3 p^3) with these l."""
    x, p = -M.BLS_X, M.P
    l3 = (x - 1) ** 2
    l2 = l3 * x
    l1 = l2 * x - l3
    l0 = l1 * x + 3
    assert l0 + l1 * p + l2 * p * p + l3 * p ** 3 == 3 * (p ** 4 - p ** 2 + 1) // M.Q_R


def test_g2_codec_round_trip_and_rejections():
    for k in (1, 2, 12345, M.Q_R - 1):
        q = M.g2_mul(M.G2_GEN, k)
        assert M.g2_decompress(M.g2_compress(q)) == q
    identity = bytes([0xC0]) + bytes(95)  # the reference's identity_g2_bytes (tests/opening_key_validation.rs:61-65)
    assert M.g2_decompress(identity) is None
    good = M.g2_compress(M.G2_GEN)
    with pytest.raises(ValueError):  # x.c1 >= p
        M.g2_decompress(bytes([0x80 | (M.P >> 376)]) + (M.P % (1 << 376)).to_bytes(47, "big") + good[48:])
    with pytest.raises(ValueError):  # compression flag cleared
        M.g2_decompress(bytes([good[0] & 0x7F]) + good[1:])
    with pytest.raises(ValueError):  # identity with a sort flag
        M.g2_decompress(bytes([0xE0]) + bytes(95))
    off, twist = M.off_curve_g2_bytes(), M.non_subgroup_g2_bytes()
    with pytest.raises(ValueError):
        M.g2_decompress(off)
    with pytest.raises(ValueError):
        M.g2_decompress(twist)


def _golden():
    pp, okey = M.srs_setup_with_opening_key(1 << 10, R.StdRng.seed_from_u64(0x9235E700), keep=64)
    assert pp == R.srs_setup(1 << 10, R.StdRng.seed_from_u64(0x9235E700), keep=64)
    comp = R.Composer.initialized()
    R.minimal_circuit(comp)
    pd = R.compile_circuit(pp, b"proof-compatibility", comp)
    args = (b"proof-compatibility", len(comp.constraints), pd.comms, comp.public_input_indexes(), comp.public_inputs_vec())
    return R.kat_proof(), args, okey, pd, comp


def test_verify_with_pairing_agrees_with_the_secret_on_the_golden_proof():
    proof, args, okey, _, _ = _golden()
    x = R.random_nonzero_bls_scalar(R.StdRng.seed_from_u64(0x9235E700))
    g = M.parse_opening_key(okey)[0]
    assert V.verify_with_secret(proof, *args, g, x)
    assert M.verify_with_pairing(proof, *args, okey)
    for pos in (528 + 3, 528 + 32 * 14 + 1):  # evaluations
        bad = bytearray(proof)
        bad[pos] ^= 1
        assert not V.verify_with_secret(bytes(bad), *args, g, x)
        assert not M.verify_with_pairing(bytes(bad), *args, okey)
    swapped = proof[48:96] + proof[:48] + proof[96:]  # a and b commitments exchanged: valid points, wrong proof
    assert not V.verify_with_secret(swapped, *args, g, x)
    assert not M.verify_with_pairing(swapped, *args, okey)


def test_verifier_bytes_layout():
    proof, args, okey, pd, comp = _golden()
    comms = {k: R.g1_compress(pd.comms[k]) for k in R.POLY_NAMES}
    b = M.verifier_to_bytes(b"lbl", 5, 8, 5, comms, okey, [1, 3])  # VerifierKey::n = constraints, not the size
    assert [int.from_bytes(b[8 * i : 8 * i + 8], "big") for i in range(6)] == [3, 968, 240, 2, 8, 5]
    assert b[48:51] == b"lbl" and int.from_bytes(b[51:59], "little") == 5
    assert b[59 + 7 * 48 : 59 + 8 * 48] == comms["q_logic"] and b[59 + 8 * 48 : 59 + 9 * 48] == comms["q_range"]
    assert b[51 + 968 : 51 + 968 + 240] == okey and b[-16:] == (1).to_bytes(8, "big") + (3).to_bytes(8, "big")
    assert len(b) == 48 + 3 + 968 + 240 + 16


def test_verifier_from_bytes_overflowing_lengths_is_not_enough_bytes():
    """verifier.rs's `try_from_bytes` tests: lengths whose sum overflows, or that exceed the bytes, are
    NotEnoughBytes (PB200_ERR_INVALID_ARG) without a crash.  These checks run before any device work."""
    from plonk_b200._lib import PB200_ERR_INVALID_ARG, lib

    L = lib()
    h = ctypes.c_void_p()
    big = (1 << 64) - 1
    for head in ((big, 1, 1, 0, 8, 5), (1, big, 1, 0, 8, 5), (0, 0, 0, (1 << 61) + 1, 8, 5), (1 << 62, 1 << 62, 1 << 62, 1 << 62, 8, 5),
                 (3, 968, 240, 0, 8, 5)):
        b = b"".join(v.to_bytes(8, "big") for v in head) + bytes(16)
        assert L.pb200_verifier_from_bytes(b, len(b), ctypes.byref(h)) == PB200_ERR_INVALID_ARG, head
    assert L.pb200_verifier_from_bytes(bytes(47), 47, ctypes.byref(h)) == PB200_ERR_INVALID_ARG
