"""Python restatement of the reference's CompressedCircuit (src/composer/compress.rs, compress/hades.rs) and of
Compiler::max_constraints (src/compiler.rs:101-112): from_composer on a circuit's arrays, the MessagePack layout
(msgpacker 0.4: shortest unsigned integers, array headers, no struct headers, [u8; 32] as 32 bare u8), the bounded
reader, validate_indices and scalar_map.  Independent of plonk_b200/csrc/compress.cpp: Python ints, hashlib SHA-512 and
Python's zlib (raw deflate, wbits -15)."""
from __future__ import annotations

import hashlib
import zlib
from dataclasses import dataclass, field
from typing import List, Tuple

from oracle import pyref as R

SELECTORS = 11
PACKED_FIXED_BYTES = 30
PACKED_BYTES_PER_CONSTRAINT = 857

INVALID = -14  # Error::InvalidCompressedCircuit
MALFORMED = -15  # Error::BlsScalarMalformed


class DecodeError(Exception):
    def __init__(self, code: int, why: str):
        super().__init__(why)
        self.code = code


# ---- scalar_map (compress.rs:63-87, compress/hades.rs) ---------------------------------------------------------------
def hades_constants() -> List[int]:
    out, p, b = [], 1, b"poseidon-for-plonk"
    for _ in range(67 * 5):
        b = hashlib.sha512(b).digest()
        p = (R.fr_from_bytes_wide(b) + p) % R.R_MOD
        out.append(p)
    return out


def hades_mds() -> List[List[int]]:
    return [[R.fr_inv(i + j + 5) for j in range(5)] for i in range(5)]


_BASE = {}


def scalar_map(hades: bool) -> List[int]:
    """The base table: 0, 1, -1, then (hades) every round constant and MDS entry not already present."""
    if hades not in _BASE:
        t = [0, 1, R.R_MOD - 1]
        if hades:
            for s in hades_constants() + [x for row in hades_mds() for x in row]:
                if s not in t:
                    t.append(s)
        _BASE[hades] = t
    return _BASE[hades]


# ---- the circuit ------------------------------------------------------------------------------------------------------
@dataclass
class Compressed:
    hades_optimization: bool = False
    public_inputs: List[int] = field(default_factory=list)
    witnesses: int = 0
    scalars: List[bytes] = field(default_factory=list)  # 32 bytes each (any values: the encoder does not check)
    polynomials: List[Tuple[int, ...]] = field(default_factory=list)  # 11 scalar indices each
    constraints: List[Tuple[int, int, int, int, int]] = field(default_factory=list)  # polynomial, a, b, c, d


def from_arrays(a, hades: bool) -> Compressed:
    """CompressedCircuit::from_composer for a circuit's arrays (selectors in Montgomery form, column-major)."""
    n = a.constraints
    sel = R.fr_vec_from_mont_bytes(a.selectors)
    wires = [int.from_bytes(a.wires[4 * i : 4 * i + 4], "little") for i in range(4 * n)]
    base = scalar_map(hades)
    index = {s: i for i, s in enumerate(base)}
    extra: List[int] = []
    polys = {}
    constraints = []
    for g in range(n):
        p = []
        for k in range(SELECTORS):
            s = sel[k * n + g]
            if s not in index:
                index[s] = len(base) + len(extra)
                extra.append(s)
            p.append(index[s])
        p = tuple(p)
        if p not in polys:
            polys[p] = len(polys)
        constraints.append((polys[p],) + tuple(wires[k * n + g] for k in range(4)))
    pis = sorted(int.from_bytes(a.pi_idx[i : i + 8], "little") for i in range(0, len(a.pi_idx), 8))
    return Compressed(hades, pis, a.n_witnesses, [R.fr_to_bytes(s) for s in extra], list(polys), constraints)


# ---- MessagePack ------------------------------------------------------------------------------------------------------
def pack_uint(v: int) -> bytes:
    if v < 0x80:
        return bytes([v])
    for tag, width in ((0xCC, 1), (0xCD, 2), (0xCE, 4), (0xCF, 8)):
        if v < 1 << (8 * width):
            return bytes([tag]) + v.to_bytes(width, "big")
    raise ValueError(v)


def pack_array(n: int) -> bytes:
    if n <= 15:
        return bytes([0x90 | n])
    if n <= 0xFFFF:
        return b"\xdc" + n.to_bytes(2, "big")
    return b"\xdd" + n.to_bytes(4, "big")


def pack(c: Compressed) -> bytes:
    out = [b"\xc3" if c.hades_optimization else b"\xc2", pack_array(len(c.public_inputs))]
    out += [pack_uint(i) for i in c.public_inputs]
    out += [pack_uint(c.witnesses), pack_array(len(c.scalars))]
    out += [b"".join(pack_uint(b) for b in s) for s in c.scalars]
    out.append(pack_array(len(c.polynomials)))
    out += [b"".join(pack_uint(i) for i in p) for p in c.polynomials]
    out.append(pack_array(len(c.constraints)))
    out += [b"".join(pack_uint(i) for i in k) for k in c.constraints]
    return b"".join(out)


def deflate(data: bytes, level: int = 9) -> bytes:
    z = zlib.compressobj(level, zlib.DEFLATED, -15)
    return z.compress(data) + z.flush()


def inflate(data: bytes) -> bytes:
    return zlib.decompress(data, -15)


def encode(c: Compressed, level: int = 9) -> bytes:
    return deflate(pack(c), level)


class _Reader:
    def __init__(self, b: bytes):
        self.b, self.at = b, 0

    def take(self, k: int) -> bytes:
        if self.at + k > len(self.b):
            raise DecodeError(INVALID, "short")
        self.at += k
        return self.b[self.at - k : self.at]

    def boolean(self) -> bool:
        t = self.take(1)[0]
        if t not in (0xC2, 0xC3):
            raise DecodeError(INVALID, "bool")
        return t == 0xC3

    def uint(self, u8: bool = False) -> int:
        t = self.take(1)[0]
        if t < 0x80:
            return t
        widths = {0xCC: 1} if u8 else {0xCC: 1, 0xCD: 2, 0xCE: 4, 0xCF: 8}
        if t not in widths:
            raise DecodeError(INVALID, "uint")
        return int.from_bytes(self.take(widths[t]), "big")

    def array(self, max_len: int) -> int:
        t = self.take(1)[0]
        if 0x90 <= t <= 0x9F:
            n = t & 0x0F
        elif t == 0xDC:
            n = int.from_bytes(self.take(2), "big")
        elif t == 0xDD:
            n = int.from_bytes(self.take(4), "big")
        else:
            raise DecodeError(INVALID, "array")
        if n > max_len:
            raise DecodeError(INVALID, "array too long")
        return n


def unpack_bounded(packed: bytes, max_constraints: int) -> Compressed:
    r = _Reader(packed)
    c = Compressed()
    c.hades_optimization = r.boolean()
    c.public_inputs = [r.uint() for _ in range(r.array(max_constraints))]
    c.witnesses = r.uint()
    c.scalars = [bytes(r.uint(u8=True) for _ in range(32)) for _ in range(r.array(max_constraints * SELECTORS))]
    c.polynomials = [tuple(r.uint() for _ in range(SELECTORS)) for _ in range(r.array(max_constraints))]
    c.constraints = [tuple(r.uint() for _ in range(5)) for _ in range(r.array(max_constraints))]
    if r.at != len(packed):
        raise DecodeError(INVALID, "trailing bytes")
    return c


def validate_indices(c: Compressed, base_scalars: int) -> bool:
    count = base_scalars + len(c.scalars)
    pis = c.public_inputs
    return not (
        any(i >= len(c.constraints) for i in pis)
        or any(pis[k] >= pis[k + 1] for k in range(len(pis) - 1))
        or any(i >= count for p in c.polynomials for i in p)
        or any(k[0] >= len(c.polynomials) or any(w >= c.witnesses for w in k[1:]) for k in c.constraints)
    )


def max_constraints(n_srs_points: int) -> int:
    available = max(0, max(0, n_srs_points - 1) - 6)
    domain = 1 << (available.bit_length() - 1) if available else 0
    return max(0, domain - 6)


def packed_size_limit(max_c: int) -> int:
    return max_c * PACKED_BYTES_PER_CONSTRAINT + PACKED_FIXED_BYTES


@dataclass
class Decoded:
    circuit: Compressed
    labels: List[int]  # dense id -> label, first appearance in gate order, a b c d


def decode(data: bytes, n_srs_points: int) -> Decoded:
    """CompressedCircuit::from_bytes with compile_with_compressed's bounds; raises DecodeError(code)."""
    max_c = max_constraints(n_srs_points)
    limit = packed_size_limit(max_c)
    d = zlib.decompressobj(-15)
    try:
        packed = d.decompress(data, limit + 1)
    except zlib.error:
        raise DecodeError(INVALID, "deflate")
    if len(packed) > limit:
        raise DecodeError(INVALID, "too large")
    if not d.eof:
        raise DecodeError(INVALID, "truncated")
    c = unpack_bounded(packed, max_c)
    if not validate_indices(c, len(scalar_map(c.hades_optimization))):
        raise DecodeError(INVALID, "indices")
    if any(int.from_bytes(s, "little") >= R.R_MOD for s in c.scalars):
        raise DecodeError(MALFORMED, "scalar")
    seen, labels = {}, []
    for k in c.constraints:
        for w in k[1:]:
            if w not in seen:
                seen[w] = len(labels)
                labels.append(w)
    return Decoded(c, labels)


def expand_selectors(c: Compressed) -> List[List[int]]:
    """The 11 selector columns the description stands for (gate order)."""
    table = scalar_map(c.hades_optimization) + [int.from_bytes(s, "little") for s in c.scalars]
    return [[table[c.polynomials[k[0]][j]] for k in c.constraints] for j in range(SELECTORS)]


def sample(witnesses: int = 1, **kw) -> Compressed:
    """The reference unit tests' circuit(): one default constraint and polynomial, public input 0 (compress.rs:532-541)."""
    c = Compressed(False, [0], witnesses, [], [(0,) * SELECTORS], [(0, 0, 0, 0, 0)])
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def hades_scalars() -> List[int]:
    """Every Hades round constant and distinct MDS entry: the base entries beyond 0, 1 and -1."""
    return scalar_map(True)[3:]
