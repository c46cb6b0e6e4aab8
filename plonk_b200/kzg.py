"""CommitKey / Commitment mirror (reference src/commitment_scheme/kzg10/key.rs:36-41, 362-388,
commitment.rs:77-106) over the CUDA MSM."""
from __future__ import annotations

import ctypes

from ._lib import PB200_ERR_DEGREE_TOO_LARGE, PB200_ERR_POINT_MALFORMED, Pb200Error, check, lib

G1_RAW_BYTES = 96
FR_BYTES = 32


class PolynomialDegreeTooLarge(ValueError):
    """Error::PolynomialDegreeTooLarge (reference key.rs:362-370)."""


class PointMalformed(ValueError):
    """dusk_bytes::Error::InvalidData / Error::PointMalformed: a G1 encoding that is not canonical, not on
    the curve or not in the prime-order subgroup (G1Affine::from_bytes)."""


def g1_decompress(compressed: bytes, check_subgroup: bool = True) -> bytes:
    """N x 48-byte compressed points -> N x 96-byte raw points (square roots and subgroup checks on the GPU)."""
    if len(compressed) % 48:
        raise PointMalformed("length is not a multiple of 48")  # chunks(G1Affine::SIZE) then from_slice fails
    n = len(compressed) // 48
    out = ctypes.create_string_buffer(max(n, 1) * G1_RAW_BYTES)
    try:
        check(lib().pb200_g1_decompress(compressed, n, 1 if check_subgroup else 0, out))
    except Pb200Error as e:
        if e.code == PB200_ERR_POINT_MALFORMED:
            raise PointMalformed(str(e)) from e
        raise
    return out.raw[: n * G1_RAW_BYTES]


def _raw_key_points(blob: bytes, checked: bool) -> bytes:
    n = ctypes.c_size_t()
    try:
        check(lib().pb200_raw_commit_key_points(blob, len(blob), 1 if checked else 0, ctypes.byref(n)))
        out = ctypes.create_string_buffer(max(n.value, 1) * G1_RAW_BYTES)
        check(lib().pb200_commit_key_from_raw_var_bytes(blob, len(blob), 1 if checked else 0, out))
    except Pb200Error as e:
        if e.code == PB200_ERR_POINT_MALFORMED:
            raise PointMalformed(str(e)) from e
        raise
    return out.raw[: n.value * G1_RAW_BYTES]


def commit_key_bytes_of_public_parameters(raw_var_bytes: bytes) -> bytes:
    """PublicParameters::to_raw_var_bytes (srs.rs:114-119) = OpeningKey::to_bytes (240 bytes: a compressed G1 and
    two compressed G2 points, verifier material) followed by CommitKey::to_raw_var_bytes: returns the latter."""
    return raw_var_bytes[240:]


_HOST_COMPRESS_MAX = 8  # up to this many points the per-point host encoder is quicker than a trip to the GPU


def g1_compress(raw_points: bytes) -> bytes:
    """N x 96-byte raw points -> N x 48-byte compressed points (G1Affine::to_bytes): one pb200_g1_compress_batch
    call on the GPU, or the host encoder for a handful of points; the bytes are the same."""
    n = len(raw_points) // G1_RAW_BYTES
    if n > _HOST_COMPRESS_MAX:
        out = ctypes.create_string_buffer(48 * n)
        check(lib().pb200_g1_compress_batch(raw_points, n, out))
        return out.raw
    out = ctypes.create_string_buffer(48)
    res = bytearray()
    for i in range(0, n * G1_RAW_BYTES, G1_RAW_BYTES):
        check(lib().pb200_g1_compress(raw_points[i : i + G1_RAW_BYTES], out))
        res += out.raw
    return bytes(res)


def commit_key_to_var_bytes(raw_points: bytes) -> bytes:
    """CommitKey::to_var_bytes (key.rs:303-308) of a key given as 96-byte raw points: the input of
    CommitKey.from_slice."""
    return g1_compress(raw_points)


def commit_key_to_raw_var_bytes(raw_points: bytes) -> bytes:
    """CommitKey::to_raw_var_bytes (key.rs:215-229): the input of CommitKey.from_raw_var_bytes and
    from_slice_unchecked.  Host only."""
    n = len(raw_points) // G1_RAW_BYTES
    size = ctypes.c_size_t()
    check(lib().pb200_commit_key_to_raw_var_bytes(raw_points or None, n, None, 0, ctypes.byref(size)))
    out = ctypes.create_string_buffer(size.value)
    check(lib().pb200_commit_key_to_raw_var_bytes(raw_points or None, n, out, size.value, ctypes.byref(size)))
    return out.raw


def public_parameters_to_var_bytes(opening_key: bytes, raw_points: bytes) -> bytes:
    """PublicParameters::to_var_bytes (srs.rs:149-153): OpeningKey::to_bytes, then CommitKey::to_var_bytes."""
    assert len(opening_key) == 240
    return opening_key + commit_key_to_var_bytes(raw_points)


def public_parameters_to_raw_var_bytes(opening_key: bytes, raw_points: bytes) -> bytes:
    """PublicParameters::to_raw_var_bytes (srs.rs:114-119): OpeningKey::to_bytes, then
    CommitKey::to_raw_var_bytes - what commit_key_bytes_of_public_parameters splits."""
    assert len(opening_key) == 240
    return opening_key + commit_key_to_raw_var_bytes(raw_points)


class Commitment:
    """Commitment(G1Affine): ``raw`` is x||y Montgomery limbs (identity = zeros)."""

    def __init__(self, raw: bytes):
        assert len(raw) == G1_RAW_BYTES
        self.raw = raw

    def to_bytes(self) -> bytes:
        """48-byte compressed encoding (reference commitment.rs:95-101)."""
        out = ctypes.create_string_buffer(48)
        check(lib().pb200_g1_compress(self.raw, out))
        return out.raw

    def __eq__(self, other):
        return isinstance(other, Commitment) and self.raw == other.raw


class CommitKey:
    """powers_of_g resident in HBM (uploaded once, like the immutable CommitKey of a Prover)."""

    def __init__(self, raw_points: bytes):
        assert len(raw_points) % G1_RAW_BYTES == 0 and raw_points
        self.n_points = len(raw_points) // G1_RAW_BYTES
        h = ctypes.c_void_p()
        check(lib().pb200_srs_upload(raw_points, self.n_points, ctypes.byref(h)))
        self._h = h
        self._raw = bytes(raw_points)  # the writers below re-encode the points the key was made from

    def to_var_bytes(self) -> bytes:
        """CommitKey::to_var_bytes (key.rs:303-308): 48 compressed bytes per point, encoded on the GPU."""
        return commit_key_to_var_bytes(self._raw)

    def to_raw_var_bytes(self) -> bytes:
        """CommitKey::to_raw_var_bytes (key.rs:215-229)."""
        return commit_key_to_raw_var_bytes(self._raw)

    @classmethod
    def from_slice(cls, compressed: bytes) -> "CommitKey":
        """CommitKey::from_slice (key.rs:319-326): 48-byte compressed powers, validated like the reference."""
        return cls(g1_decompress(compressed))

    @classmethod
    def from_raw_var_bytes(cls, raw_var_bytes: bytes) -> "CommitKey":
        """CommitKey::from_raw_var_bytes (key.rs:258-298): the raw format with every point validated (on the GPU)."""
        return cls(_raw_key_points(raw_var_bytes, True))

    @classmethod
    def from_slice_unchecked(cls, raw_var_bytes: bytes) -> "CommitKey":
        """CommitKey::from_slice_unchecked (key.rs:242-256): the raw format from a trusted source, no validation."""
        return cls(_raw_key_points(raw_var_bytes, False))

    def max_degree(self) -> int:
        return self.n_points - 1

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().pb200_srs_free(self._h)
                self._h = None
        except Exception:
            pass

    @staticmethod
    def _trim(poly: bytes) -> bytes:
        """Polynomial::from_coefficients_vec drops trailing zero coefficients (polynomial.rs:79-93)."""
        n = len(poly) // FR_BYTES
        zero = bytes(FR_BYTES)
        while n and poly[(n - 1) * FR_BYTES : n * FR_BYTES] == zero:
            n -= 1
        return poly[: n * FR_BYTES]

    def commit(self, polynomial: bytes) -> Commitment:
        return self.commit_batch([polynomial])[0]

    def commit_batch(self, polynomials) -> list:
        polys = [self._trim(p) for p in polynomials]
        for p in polys:
            degree = max(len(p) // FR_BYTES - 1, 0)
            if degree > self.max_degree():
                raise PolynomialDegreeTooLarge()
        n = max(len(p) for p in polys) // FR_BYTES
        stride = max(n, 1)
        buf = bytearray(stride * FR_BYTES * len(polys))
        for i, p in enumerate(polys):
            buf[i * stride * FR_BYTES : i * stride * FR_BYTES + len(p)] = p
        out = ctypes.create_string_buffer(G1_RAW_BYTES * len(polys))
        src = (ctypes.c_char * len(buf)).from_buffer(buf)
        try:
            check(lib().pb200_msm_g1(self._h, src, n, len(polys), stride, out))
        except Pb200Error as e:
            if e.code == PB200_ERR_DEGREE_TOO_LARGE:
                raise PolynomialDegreeTooLarge() from e
            raise
        return [Commitment(out.raw[i * G1_RAW_BYTES : (i + 1) * G1_RAW_BYTES]) for i in range(len(polys))]
