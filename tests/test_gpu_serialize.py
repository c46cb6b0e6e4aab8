"""The writers of the reference's key formats on the GPU: Prover::to_bytes (prover.rs:212-263) through
pb200_prover_to_bytes and CommitKey::to_var_bytes (key.rs:303-308) through pb200_g1_compress_batch, against the
byte strings oracle/serialize.py builds from the oracle's own keys.

oracle/serialize.py writes the domain size into VerifierKey::n; the reference writes the constraint count
(compiler.rs:278-279).  `reference_prover_bytes` below is the oracle's string with that one field as the reference
has it, and is what the product must write."""
import ctypes
import random
import threading

import pytest

from oracle import cref
from oracle import pyref as R
from oracle import serialize as S
from tests.util import bases_to_abi, progression_bases


@pytest.fixture(scope="module")
def pb():
    import plonk_b200
    from plonk_b200._lib import check, lib

    check(lib().pb200_init(0))
    return plonk_b200


def _sections(blob):
    """Offsets of the prover key, the commit key and the verifier key in a serialized prover."""
    label_len, pk_len, ck_len, vk_len = (int.from_bytes(blob[8 * i : 8 * i + 8], "big") for i in range(4))
    pk = 48 + label_len
    return pk, pk + pk_len, pk + pk_len + ck_len, vk_len


def with_verifier_key_n(blob, value):
    vk = _sections(blob)[2]
    return blob[:vk] + value.to_bytes(8, "little") + blob[vk + 8 :]


def reference_prover_bytes(pd):
    return with_verifier_key_n(S.prover_to_bytes(pd), pd.constraints)


def commit_key_to_var_bytes(points):
    """CommitKey::to_var_bytes (key.rs:303-308): G1Affine::to_bytes per point."""
    return b"".join(R.g1_compress(p) for p in points)


def expected_bytes_by_cref(label, comp, arrays, srs_raw):
    """Prover::to_bytes assembled from the C++ oracle's transforms and commitments: the same string as
    reference_prover_bytes(R.compile_circuit(...)), for circuits too large for the Python oracle."""
    c = arrays.constraints
    size = 1 << (c - 1).bit_length() if c > 1 else 1
    log_n = size.bit_length() - 1
    n_trim = 1 << (c + R.CIRCUIT_SIZE_PADDING - 1).bit_length()
    polys = {}
    for j, k in enumerate(R.SELECTORS):
        polys[k] = R.poly_trim(R.fr_vec_from_mont_bytes(cref.ntt(arrays.selectors[32 * c * j : 32 * c * (j + 1)], log_n, 1, 0)))
    roots = R.EvaluationDomain(size).elements()
    kk = [1, R.K1, R.K2, R.K3]
    for j, sigma in enumerate(R.compute_sigma_permutations(comp, size)):
        lag = R.fr_vec_to_mont_bytes([kk[col] * roots[idx] % R.R_MOD for (col, idx) in sigma])
        polys[f"s_sigma_{j + 1}"] = R.poly_trim(R.fr_vec_from_mont_bytes(cref.ntt(lag, log_n, 1, 0)))
    domain = S.domain_to_bytes(8 * size)

    def evaluations(coeffs):
        data = R.fr_vec_to_mont_bytes(coeffs) if coeffs else bytes(32)
        return domain + b"".join(v.to_bytes(32, "little") for v in R.fr_vec_from_mont_bytes(cref.ntt(data, log_n + 3, 0, 1)))

    pk = size.to_bytes(8, "little") + (8 * size * 32 + 172).to_bytes(8, "little")
    for k in S.FILE_ORDER:
        pk += len(polys[k]).to_bytes(8, "little") + b"".join(v.to_bytes(32, "little") for v in polys[k]) + evaluations(polys[k])
    pk += evaluations([0, 1])
    w8n = R.EvaluationDomain(8 * size).group_gen
    v_h = [(pow(R.GENERATOR * pow(w8n, i, R.R_MOD) % R.R_MOD, size, R.R_MOD) - 1) % R.R_MOD for i in range(8)]
    pk += domain + b"".join(v.to_bytes(32, "little") for v in v_h) * size
    n_pts = n_trim + 7
    ck = n_pts.to_bytes(8, "little") + b"".join(srs_raw[96 * i : 96 * i + 96] + b"\0" for i in range(n_pts))
    comms = dict(zip(R.POLY_NAMES, cref.CrefProver(label, arrays, srs_raw).commitments()))
    vk = c.to_bytes(8, "little") + b"".join(comms[k] for k in S.FILE_ORDER)
    vk += bytes(20 * 48 + 8 - len(vk))
    head = b"".join(v.to_bytes(8, "big") for v in (len(label), len(pk), len(ck), len(vk), size, c))
    return head + label + pk + ck + vk


def test_cref_assembly_equals_the_oracle_serializer():
    """The two ways this file builds the expected bytes agree (no device involved)."""
    rng = random.Random(4)
    pp = R.srs_from_secret(64 + 7, rng.randrange(1, R.R_MOD), rng.randrange(1, R.R_MOD))
    comp = R.Composer.initialized()
    R.synthetic_arith_circuit(comp, 37, seed=3, n_public=1)
    arrays = cref.CircuitArrays(comp)
    assert expected_bytes_by_cref(b"two-ways", comp, arrays, bases_to_abi(pp)) == reference_prover_bytes(R.compile_circuit(pp, b"two-ways", comp))


def _poly_lengths(blob):
    pk = _sections(blob)[0]
    n = int.from_bytes(blob[pk : pk + 8], "little")
    at, out = pk + 16, []
    for _ in range(15):
        out.append(int.from_bytes(blob[at : at + 8], "little"))
        at += 8 + 32 * out[-1] + 8 * n * 32 + 172
    return out


def _synthetic(rows, seed, widgets, srs_points):
    rng = random.Random(seed)
    pp = R.srs_from_secret(srs_points, rng.randrange(1, R.R_MOD), rng.randrange(1, R.R_MOD))
    comp = R.Composer.initialized()
    R.synthetic_arith_circuit(comp, rows, seed=seed, n_public=2, widgets=widgets)
    return pp, comp, cref.CircuitArrays(comp)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,widgets,srs_points", [(300, 5, 512 + 7), (100, 0, 128 + 7), (128, 3, 256 + 7)],
                         ids=["every-gate-family", "arithmetic-only", "constraints-a-power-of-two"])
def test_to_bytes_equals_the_oracle_serializer(pb, rows, widgets, srs_points):
    pp, comp, arrays = _synthetic(rows, 77 if rows == 300 else rows, widgets, srs_points)
    assert arrays.constraints == rows
    want = reference_prover_bytes(R.compile_circuit(pp, b"serialized", comp))
    prover = pb.Prover(b"serialized", arrays.constraints, arrays.selectors, arrays.wires, arrays.n_witnesses, bases_to_abi(pp))
    got = prover.to_bytes()
    assert prover.serialized_size() == len(want) == len(got)
    assert got == want
    if widgets == 0:  # the four widget selectors are never used: Polynomial length 0
        lengths = dict(zip(S.FILE_ORDER, _poly_lengths(got)))
        assert [lengths[k] for k in ("q_logic", "q_range", "q_fixed_group_add", "q_variable_group_add")] == [0, 0, 0, 0]


@pytest.mark.gpu
def test_to_bytes_of_the_bench_circuit(pb):
    from oracle import gadgets

    comp = gadgets.GadgetComposer.initialized()
    gadgets.bench_circuit(comp, 1 << 13)
    arrays = cref.CircuitArrays(comp)
    srs_raw = cref.srs_from_secret((1 << 13) + 7, 0x1234567, 0x7654321)
    prover = pb.Prover(b"dusk-network", arrays.constraints, arrays.selectors, arrays.wires, arrays.n_witnesses, srs_raw)
    want = expected_bytes_by_cref(b"dusk-network", comp, arrays, srs_raw)
    assert prover.serialized_size() == len(want)
    assert prover.to_bytes() == want


@pytest.mark.gpu
def test_round_trip_and_the_loader_fix(pb):
    """to_bytes -> from_bytes gives the same prover; a blob with VerifierKey::n = constraints (what the reference
    writes; constraints not a power of two) loads, and so does one with the domain size there."""
    pp, comp, arrays = _synthetic(300, 77, 5, 512 + 7)
    compiled = pb.Prover(b"serialized", arrays.constraints, arrays.selectors, arrays.wires, arrays.n_witnesses, bases_to_abi(pp))
    blob = compiled.to_bytes()
    vk = _sections(blob)[2]
    assert int.from_bytes(blob[vk : vk + 8], "little") == 300
    bl = cref.draw_blinders(R.StdRng.seed_from_u64(3))
    want = cref.CrefProver(b"serialized", arrays, bases_to_abi(pp)).prove(bl)
    assert compiled.prove(arrays.witnesses, arrays.pi_idx, arrays.pi_vals, bl) == want
    for b in (blob, with_verifier_key_n(blob, 512)):
        loaded = pb.Prover.from_bytes(b, arrays.wires, arrays.n_witnesses)
        assert loaded.commitments() == compiled.commitments()
        assert loaded.prove(arrays.witnesses, arrays.pi_idx, arrays.pi_vals, bl) == want
        assert loaded.to_bytes() == blob  # the writer takes VerifierKey::n from the constraint count


@pytest.mark.gpu
def test_g1_compress_batch(pb):
    from plonk_b200 import kzg
    from plonk_b200._lib import lib

    n = (1 << 16) + 7
    pts = progression_bases(n, 11, 13)
    for i in (0, 5, 4097, n - 1):
        pts[i] = None
    raw = b"".join(bytes(96) if p is None else R.g1_to_raw_bytes(p) for p in pts)
    out = ctypes.create_string_buffer(48 * n)
    assert lib().pb200_g1_compress_batch(raw, n, out) == 0
    got = out.raw
    signs = {got[48 * i] & 0xE0 for i in range(n)}
    assert signs == {0x80, 0xA0, 0xC0}  # both y signs and the identity occur
    one = ctypes.create_string_buffer(48)
    for i in range(n):
        assert lib().pb200_g1_compress(raw[96 * i : 96 * i + 96], one) == 0
        assert one.raw == got[48 * i : 48 * i + 48], i
    step = 97
    assert b"".join(got[48 * i : 48 * i + 48] for i in range(0, n, step)) == commit_key_to_var_bytes(pts[::step])
    assert kzg.g1_decompress(got) == raw
    assert kzg.g1_compress(raw) == got and kzg.commit_key_to_var_bytes(raw) == got
    assert kzg.g1_compress(raw[: 3 * 96]) == got[: 3 * 48]  # a handful of points: the host path, same bytes
    assert lib().pb200_g1_compress_batch(raw, 0, out) == 0
    assert lib().pb200_g1_compress_batch(None, 3, out) == -4
    okey = bytes(range(240))
    assert kzg.public_parameters_to_var_bytes(okey, raw[: 96 * 50]) == okey + got[: 48 * 50]


@pytest.mark.gpu
def test_prover_to_bytes_argument_checks(pb):
    from plonk_b200._lib import lib

    pp, comp, arrays = _synthetic(100, 100, 0, 128 + 7)
    prover = pb.Prover(b"args", arrays.constraints, arrays.selectors, arrays.wires, arrays.n_witnesses, bases_to_abi(pp))
    L = lib()
    ln = ctypes.c_size_t()
    assert L.pb200_prover_to_bytes(prover._h, None, 0, None) == -4
    assert L.pb200_prover_to_bytes(None, None, 0, ctypes.byref(ln)) == -4
    assert L.pb200_prover_to_bytes(prover._h, None, 0, ctypes.byref(ln)) == 0  # out = NULL: the length only
    size = ln.value
    assert size == prover.serialized_size() == len(prover.to_bytes())
    guard = 64
    buf = ctypes.create_string_buffer(b"\x5a" * (size - 1 + guard), size - 1 + guard)
    ln.value = 0
    assert L.pb200_prover_to_bytes(prover._h, buf, size - 1, ctypes.byref(ln)) == -4
    assert ln.value == size and buf.raw == b"\x5a" * (size - 1 + guard)  # nothing written, guard bytes included
    buf = ctypes.create_string_buffer(b"\x5a" * (size + guard), size + guard)
    assert L.pb200_prover_to_bytes(prover._h, buf, size, ctypes.byref(ln)) == 0
    assert buf.raw[:size] == prover.to_bytes() and buf.raw[size:] == b"\x5a" * guard


@pytest.mark.gpu
def test_to_bytes_beside_proofs_on_the_same_prover(pb):
    """One thread serializes while two others prove on the same prover: same blob, same proofs as when quiet."""
    pp, comp, arrays = _synthetic(300, 77, 5, 512 + 7)
    prover = pb.Prover(b"busy", arrays.constraints, arrays.selectors, arrays.wires, arrays.n_witnesses, bases_to_abi(pp))
    blinders = [cref.draw_blinders(R.StdRng.seed_from_u64(s)) for s in (1, 2)]
    quiet_blob = prover.to_bytes()
    quiet_proofs = [prover.prove(arrays.witnesses, arrays.pi_idx, arrays.pi_vals, b) for b in blinders]
    start = threading.Barrier(3)
    result = {}

    def prove(i):
        start.wait()
        result[i] = [prover.prove(arrays.witnesses, arrays.pi_idx, arrays.pi_vals, blinders[i]) for _ in range(4)]

    def serialize():
        start.wait()
        result["blob"] = prover.to_bytes()

    threads = [threading.Thread(target=prove, args=(0,)), threading.Thread(target=prove, args=(1,)), threading.Thread(target=serialize)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert result["blob"] == quiet_blob
    assert result[0] == [quiet_proofs[0]] * 4 and result[1] == [quiet_proofs[1]] * 4


@pytest.mark.gpu
def test_bench_circuit_2_16_reloads_from_its_own_bytes(pb):
    from plonk_b200 import gadgets

    arr = gadgets.bench_circuit(1 << 16).arrays()
    srs_raw = cref.srs_from_secret((1 << 16) + 7, 0x1234567, 0x7654321)
    label = b"dusk-network"
    compiled = pb.Prover(label, arr.constraints, arr.selectors, arr.wires, arr.n_witnesses, srs_raw)
    blob = compiled.to_bytes()
    n = 1 << 16
    points = (1 << (arr.constraints + 6 - 1).bit_length()) + 7
    assert len(blob) == 48 + len(label) + 16 + sum(8 + 32 * k for k in _poly_lengths(blob)) + 17 * (8 * n * 32 + 172) + 8 + 97 * points + 968
    loaded = pb.Prover.from_bytes(blob, arr.wires, arr.n_witnesses)
    del blob
    assert loaded.commitments() == compiled.commitments()
    bl = cref.draw_blinders(R.StdRng.seed_from_u64(12))
    assert loaded.prove(arr.witnesses, arr.pi_idx, arr.pi_vals, bl) == compiled.prove(arr.witnesses, arr.pi_idx, arr.pi_vals, bl)
