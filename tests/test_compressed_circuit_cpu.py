"""Circuit::compress and the decoding half of Compiler::compile_with_compressed on the host (pb200_circuit_compress,
pb200_compressed_circuit_info) against tests/models/compress_model.py: the payload of every circuit is the model's
packing, and every unit test of the reference's src/composer/compress.rs (lines 526-763) runs through the library's
bounded decoder.  No GPU involved."""
import random
import zlib

import pytest

from oracle import cref
from oracle import gadgets as G
from oracle import pyref as R
from plonk_b200 import compress_arrays
from plonk_b200 import gadgets as N
from plonk_b200._lib import PB200_ERR_INVALID_ARG, PB200_ERR_INVALID_COMPRESSED, PB200_ERR_SCALAR_MALFORMED, Pb200Error
from plonk_b200.prover import compressed_circuit_info
from tests.models import compress_model as M
from tests.test_gpu_gadget_circuits import CASES

# public parameters with Compiler::max_constraints = 2, the MAX_CONSTRAINTS of the reference's unit tests: max_degree 14,
# available 8, domain 8
SRS_2 = 15
assert M.max_constraints(SRS_2) == 2


# ---- circuits --------------------------------------------------------------------------------------------------------
def dummy_circuit(c):
    """tests/composer.rs:19-84 DummyCircuit::circuit with its Default values, every gadget family once."""
    z = N.jubjub_mul(N.jubjub_generator(), 7)
    w_a, w_b, w_x, w_y = (c.append_witness(v) for v in (2, 3, 6, 7))
    w_z = c.append_point(z)
    r_w = c.gate_mul(dict(q_m=1), a=w_a, b=w_b)
    c.append_constant(15)
    c.append_constant_point(z)
    c.append_public_point(z)
    c.append_public(7)
    c.assert_equal(w_x, r_w)
    c.assert_equal_constant(w_x, 0, 6)
    c.assert_equal_point(w_z, w_z)
    c.assert_equal_public_point(w_z, z)
    c.gate_add(dict(q_l=1, q_r=1), a=w_a, b=w_b)
    c.component_add_point(w_z, w_z)
    c.append_logic_and(w_a, w_b, 127)
    c.component_boolean(c.ONE)
    c.component_decomposition(w_a, 254)
    c.component_mul_generator(w_y, N.jubjub_generator())
    c.component_mul_point(w_y, w_z)
    c.component_range_bits(w_a, 256)
    c.component_select(c.ONE, w_a, w_b)
    c.component_select_identity(c.ONE, w_z)
    c.component_select_one(c.ONE, w_a)
    c.component_select_point(c.ONE, w_z, w_z)
    c.component_select_zero(c.ONE, w_a)
    c.append_logic_xor(w_a, w_b, 127)


def sparse_witness_circuit(c):
    """compress.rs SparseWitnessCircuit: 37 witnesses no gate uses."""
    for _ in range(37):
        c.append_witness(0)


def native_arrays(circuit):
    comp = N.Composer.initialized()
    circuit(comp)
    return comp.arrays()


def bench_arrays(degree):
    return N.bench_circuit(degree).arrays()


class Arrays:
    """A circuit's arrays built by hand: selectors[k][g] as field elements, wires[k][g]."""

    def __init__(self, selectors, wires, n_witnesses, pi_idx=()):
        self.constraints = len(wires[0])
        self.selectors = b"".join(R.fr_vec_to_mont_bytes(col) for col in selectors)
        self.wires = b"".join(w.to_bytes(4, "little") for col in wires for w in col)
        self.n_witnesses = n_witnesses
        self.pi_idx = b"".join(i.to_bytes(8, "little") for i in pi_idx)


def _code(f):
    with pytest.raises(Pb200Error) as e:
        f()
    return e.value.code


def info(data, n_srs=SRS_2):
    return compressed_circuit_info(data, n_srs)


def model_code(data, n_srs=SRS_2):
    try:
        M.decode(data, n_srs)
    except M.DecodeError as e:
        return e.code
    return 0


def check_info(data, n_srs=SRS_2):
    """The library's decoding agrees with the model's: counts, labels and public inputs, or the same error."""
    try:
        got = info(data, n_srs)
    except Pb200Error as e:
        assert model_code(data, n_srs) == e.code
        raise
    d = M.decode(data, n_srs)
    pis = b"".join(i.to_bytes(8, "little") for i in d.circuit.public_inputs)
    assert got == (len(d.circuit.constraints), d.circuit.witnesses, len(d.labels), len(d.circuit.public_inputs), pis)
    return got


# ---- the encoder against the model -----------------------------------------------------------------------------------
def _gadget_arrays():
    for name, build, default, _, _ in CASES:
        o = G.GadgetComposer.initialized()
        build(o, *default)
        yield name, cref.CircuitArrays(o)


@pytest.mark.parametrize("hades", [True, False])
def test_payload_is_the_models_packing(hades):
    circuits = list(_gadget_arrays()) + [("dummy", native_arrays(dummy_circuit)), ("sparse", native_arrays(sparse_witness_circuit)),
                                         ("bench_2^13", bench_arrays(1 << 13))]
    for name, a in circuits:
        data = compress_arrays(a, hades)
        expect = M.from_arrays(a, hades)
        assert M.inflate(data) == M.pack(expect), name
        # and it decodes to the same circuit: the selector columns it stands for are the circuit's
        n_srs = (1 << (a.constraints + 6 - 1).bit_length()) + 7
        d = M.decode(data, n_srs)
        assert d.circuit == expect, name
        sel = R.fr_vec_from_mont_bytes(a.selectors)
        assert M.expand_selectors(d.circuit) == [sel[k * a.constraints : (k + 1) * a.constraints] for k in range(11)], name
        check_info(data, n_srs)


def test_hades_constants_are_never_serialized():
    """A circuit whose q_c takes every Hades round constant and MDS entry writes no scalar with the optimization on,
    and all of them without it."""
    extra = M.hades_scalars()
    assert len(extra) == 335 + 9  # the 25 MDS entries (i + j + 5)^-1 hold 9 values
    n = len(extra)
    zero = [0] * n
    sel = [zero, zero, zero, zero, zero, extra, [1] * n, zero, zero, zero, zero]
    a = Arrays(sel, [[0] * n] * 4, 1)
    on = M.unpack_bounded(M.inflate(compress_arrays(a, True)), n)
    off = M.unpack_bounded(M.inflate(compress_arrays(a, False)), n)
    assert on.scalars == [] and [p[5] for p in on.polynomials] == list(range(3, 3 + n))
    assert off.scalars == [R.fr_to_bytes(s) for s in extra]


def test_encoder_argument_errors():
    a = Arrays([[0]] * 11, [[0], [0], [0], [5]], 5)
    assert _code(lambda: compress_arrays(a)) == PB200_ERR_INVALID_ARG  # wire 5 of 5 witnesses
    a = Arrays([[0]] * 11, [[0]] * 4, 1, pi_idx=(1,))
    assert _code(lambda: compress_arrays(a)) == PB200_ERR_INVALID_ARG  # public input past the last gate
    a = Arrays([[0, 0]] * 11, [[0, 0]] * 4, 1, pi_idx=(1, 1))
    assert _code(lambda: compress_arrays(a)) == PB200_ERR_INVALID_ARG
    # public inputs are written sorted, as from_composer sorts the composer's keys
    a = Arrays([[0, 0]] * 11, [[0, 0]] * 4, 1, pi_idx=(1, 0))
    assert M.unpack_bounded(M.inflate(compress_arrays(a)), 2).public_inputs == [0, 1]


# ---- compress.rs unit tests through pb200_compressed_circuit_info ------------------------------------------------------
def test_valid_indices_are_accepted():
    assert check_info(M.encode(M.sample())) == (1, 1, 1, 1, bytes(8))


def test_capacity_limits_are_inclusive():
    c = M.sample(public_inputs=[0, 1], constraints=[(0, 0, 0, 0, 0)] * 2)
    assert check_info(M.encode(c))[:4] == (2, 1, 1, 2)


@pytest.mark.parametrize("which", ["public_inputs", "scalars", "polynomials", "constraints"])
def test_excessive_collection_counts_are_rejected(which):
    c = M.sample()
    c.public_inputs = [0] * 3 if which == "public_inputs" else c.public_inputs
    c.scalars = [bytes(32)] * (2 * 11 + 1) if which == "scalars" else c.scalars
    c.polynomials = [(0,) * 11] * 3 if which == "polynomials" else c.polynomials
    c.constraints = [(0,) * 5] * 3 if which == "constraints" else c.constraints
    assert _code(lambda: check_info(M.encode(c))) == PB200_ERR_INVALID_COMPRESSED


def _packed_exactly(size):
    """A valid packed circuit of exactly `size` bytes, at most the largest one the limit allows: two gates, two
    polynomials, 22 serialized scalars whose bytes use the 0xcc form, array headers in the 0xdd form and integers
    widened (any unsigned width is read) until the size is reached."""
    c = M.sample(public_inputs=[0, 1], constraints=[(0, 0, 0, 0, 0), (1, 0, 0, 0, 0)], polynomials=[(0,) * 11, (1,) * 11],
                 scalars=[bytes([i]) * 32 for i in range(22)])
    ints = list(c.public_inputs) + [c.witnesses] + [x for p in c.polynomials for x in p] + [x for k in c.constraints for x in k]

    def u(v, w):
        return M.pack_uint(v) if w == 0 else bytes([{1: 0xCC, 2: 0xCD, 4: 0xCE, 8: 0xCF}[w]]) + v.to_bytes(w, "big")

    def arr(n):
        return b"\xdd" + n.to_bytes(4, "big")

    def build(widths):
        it = iter(zip(ints, widths))
        out = [b"\xc2", arr(2)] + [u(*next(it)) for _ in range(2)] + [u(*next(it)), arr(22)]
        out += [b"".join(b"\xcc" + bytes([b]) for b in s) for s in c.scalars]
        out += [arr(2)] + [u(*next(it)) for _ in range(22)] + [arr(2)] + [u(*next(it)) for _ in range(10)]
        return b"".join(out)

    grow = size - len(build([0] * len(ints)))
    assert 0 <= grow <= 8 * len(ints)
    widths = []
    for _ in ints:
        w = next(s for s in (8, 4, 2, 1, 0) if s <= grow)
        widths.append(w)
        grow -= w
    packed = build(widths)
    assert len(packed) == size and M.unpack_bounded(packed, 2) == c
    return packed


def test_inflated_size_limit():
    limit = M.packed_size_limit(2)
    assert limit == 2 * 857 + 30
    assert check_info(M.deflate(_packed_exactly(limit)))[:4] == (2, 1, 1, 2)  # an inflated size equal to the limit passes
    assert _code(lambda: check_info(M.deflate(bytes(limit + 1)))) == PB200_ERR_INVALID_COMPRESSED
    assert _code(lambda: check_info(M.deflate(_packed_exactly(limit) + b"\x00"))) == PB200_ERR_INVALID_COMPRESSED


@pytest.mark.parametrize("k", range(1, 5))
def test_invalid_witness_indices_are_rejected(k):
    c = M.sample()
    g = list(c.constraints[0])
    g[k] = c.witnesses
    c.constraints = [tuple(g)]
    assert not M.validate_indices(c, 3)
    assert _code(lambda: check_info(M.encode(c))) == PB200_ERR_INVALID_COMPRESSED


def test_invalid_polynomial_index_is_rejected():
    c = M.sample(constraints=[(1, 0, 0, 0, 0)])
    assert _code(lambda: check_info(M.encode(c))) == PB200_ERR_INVALID_COMPRESSED


@pytest.mark.parametrize("k", range(11))
def test_invalid_scalar_indices_are_rejected(k):
    p = [0] * 11
    p[k] = len(M.scalar_map(False))
    c = M.sample(polynomials=[tuple(p)])
    assert _code(lambda: check_info(M.encode(c))) == PB200_ERR_INVALID_COMPRESSED
    # the same index is in range once one scalar is serialized, and in range of the larger Hades table
    assert check_info(M.encode(M.sample(polynomials=[tuple(p)], scalars=[bytes(32)])))[0] == 1
    assert check_info(M.encode(M.sample(polynomials=[tuple(p)], hades_optimization=True)))[0] == 1


@pytest.mark.parametrize("pis,gates", [([1], 1), ([0, 0], 2), ([1, 0], 2)])
def test_invalid_public_input_indices_are_rejected(pis, gates):
    c = M.sample(public_inputs=pis, constraints=[(0, 0, 0, 0, 0)] * gates)
    assert _code(lambda: check_info(M.encode(c))) == PB200_ERR_INVALID_COMPRESSED


@pytest.mark.parametrize("witnesses", [10**6, 1 << 40])
def test_sparse_witness_labels_do_not_drive_allocation(witnesses):
    c = M.sample(witnesses=witnesses, constraints=[(0, 0, 0, 0, witnesses - 1)])
    assert check_info(M.encode(c)) == (1, witnesses, 2, 1, bytes(8))


# ---- the byte stream ---------------------------------------------------------------------------------------------------
def test_trailing_packed_data_is_rejected():
    """tests/composer.rs:93-105: a msgpack nil after the payload."""
    data = compress_arrays(native_arrays(dummy_circuit))
    n_srs = (1 << 12) + 7
    check_info(data, n_srs)
    assert _code(lambda: check_info(M.deflate(M.inflate(data) + b"\xc0"), n_srs)) == PB200_ERR_INVALID_COMPRESSED


def test_non_canonical_scalars_fail_after_index_validation():
    for bad in (R.R_MOD, (1 << 256) - 1):
        c = M.sample(scalars=[bad.to_bytes(32, "little")])
        assert _code(lambda: check_info(M.encode(c))) == PB200_ERR_SCALAR_MALFORMED
        c.constraints = [(0, 0, 0, 0, 1)]  # an invalid witness index is reported first
        assert _code(lambda: check_info(M.encode(c))) == PB200_ERR_INVALID_COMPRESSED
    c = M.sample(scalars=[(R.R_MOD - 1).to_bytes(32, "little")])
    assert check_info(M.encode(c))[0] == 1


def test_any_deflate_stream_decodes_alike():
    a = bench_arrays(1 << 13)
    n_srs = (1 << 14) + 7
    ours = compress_arrays(a)
    packed = M.inflate(ours)
    want = check_info(ours, n_srs)
    for level in (0, 1, 9):
        assert check_info(M.deflate(packed, level), n_srs) == want
    z = zlib.compressobj(6, zlib.DEFLATED, -15, 9, zlib.Z_FILTERED)  # another strategy, window and memory level
    assert check_info(z.compress(packed) + z.flush(), n_srs) == want


def test_truncated_streams_and_garbage_are_rejected():
    data = compress_arrays(native_arrays(dummy_circuit))
    n_srs = (1 << 12) + 7
    for cut in (0, 1, len(data) // 2, len(data) - 1):
        assert _code(lambda: check_info(data[:cut], n_srs)) == PB200_ERR_INVALID_COMPRESSED, cut
    rng = random.Random(5)
    for size in (1, 7, 100, 5000):
        junk = bytes(rng.randrange(256) for _ in range(size))
        assert _code(lambda: info(junk, n_srs)) in (PB200_ERR_INVALID_COMPRESSED, PB200_ERR_SCALAR_MALFORMED)
    # a zlib-wrapped stream is not raw deflate
    assert _code(lambda: info(zlib.compress(M.inflate(data)), n_srs)) == PB200_ERR_INVALID_COMPRESSED


def test_public_parameters_too_small_for_the_description():
    data = compress_arrays(native_arrays(dummy_circuit))
    need = len(M.decode(data, 1 << 14).circuit.constraints)
    fits = next(p for p in range(need, 1 << 14) if M.max_constraints(p) >= need)  # the smallest parameters that fit
    assert check_info(data, fits)[0] == need
    assert _code(lambda: check_info(data, fits - 1)) == PB200_ERR_INVALID_COMPRESSED
    # without public parameters only a description without gates fits
    assert check_info(M.encode(M.Compressed()), 0)[:4] == (0, 0, 0, 0)
    assert _code(lambda: check_info(M.encode(M.sample()), 0)) == PB200_ERR_INVALID_COMPRESSED
