"""PublicParameters mirror (reference src/commitment_scheme/kzg10/srs.rs): the commit key (CommitKey::powers_of_g) and
the opening key (OpeningKey::to_bytes) of one SRS, made by PublicParameters::setup on the GPU or read back from the
reference's byte formats.

The mirror has no RNG, as Prover.prove takes its blinders as bytes: setup takes the three draws of
util::random_nonzero_bls_scalar that the reference makes (x, the G1 scalar, then the G2 scalar)."""
from __future__ import annotations

import ctypes
from typing import NamedTuple, Sequence

from ._lib import PB200_ERR_DEGREE_IS_ZERO, PB200_ERR_POINT_MALFORMED, Pb200Error, check, lib
from . import kzg
from .verifier import OPENING_KEY_BYTES, PointMalformed

ADDED_BLINDING_DEGREE = 6  # PublicParameters::ADDED_BLINDING_DEGREE (srs.rs:54)


class DegreeIsZero(ValueError):
    """Error::DegreeIsZero: PublicParameters::setup with max_degree = 0 (srs.rs:65-68)."""


class NotEnoughBytes(ValueError):
    """Error::NotEnoughBytes: PublicParameters::from_slice of at most OpeningKey::SIZE bytes (srs.rs:166-168)."""


def opening_key_check(opening_key: bytes) -> None:
    """OpeningKey::from_bytes (key.rs:609-648): raises PointMalformed unless g, h and [x]h decode, lie on their curves
    and in the prime-order subgroups, and none is the identity."""
    if len(opening_key) != OPENING_KEY_BYTES:
        raise NotEnoughBytes("NotEnoughBytes")
    try:
        check(lib().pb200_opening_key_check(opening_key))
    except Pb200Error as e:
        if e.code == PB200_ERR_POINT_MALFORMED:
            raise PointMalformed("InvalidData") from e
        raise


class PublicParameters:
    """opening_key: OpeningKey::to_bytes (240 bytes); raw_points: CommitKey::powers_of_g as 96-byte raw points."""

    def __init__(self, opening_key: bytes, raw_points: bytes):
        assert len(opening_key) == OPENING_KEY_BYTES and len(raw_points) % kzg.G1_RAW_BYTES == 0
        self.opening_key = bytes(opening_key)
        self.raw_points = bytes(raw_points)

    @classmethod
    def setup(cls, max_degree: int, draws: Sequence[bytes]) -> "PublicParameters":
        """PublicParameters::setup (srs.rs:61-100) on the GPU: max_degree + 7 powers [g_scalar x^i]G and the opening
        key.  draws: the three nonzero scalars x, g_scalar, h_scalar in the reference's draw order, 32 bytes each in
        Montgomery form.  Raises DegreeIsZero for max_degree = 0; a zero draw is a Pb200Error (PB200_ERR_INVALID_ARG)."""
        x, gs, hs = draws
        assert len(x) == len(gs) == len(hs) == 32
        n = max_degree + ADDED_BLINDING_DEGREE + 1
        pts = ctypes.create_string_buffer(max(n, 1) * kzg.G1_RAW_BYTES)
        okey = ctypes.create_string_buffer(OPENING_KEY_BYTES)
        try:
            check(lib().pb200_public_parameters_setup(max_degree, x, gs, hs, pts, okey))
        except Pb200Error as e:
            if e.code == PB200_ERR_DEGREE_IS_ZERO:
                raise DegreeIsZero("DegreeIsZero") from e
            raise
        return cls(okey.raw, pts.raw[: n * kzg.G1_RAW_BYTES])

    @classmethod
    def from_slice(cls, data: bytes) -> "PublicParameters":
        """PublicParameters::from_slice (srs.rs:163-178): the opening key and every commit-key point checked."""
        if len(data) <= OPENING_KEY_BYTES:
            raise NotEnoughBytes("NotEnoughBytes")
        opening_key_check(data[:OPENING_KEY_BYTES])
        try:
            return cls(data[:OPENING_KEY_BYTES], kzg.g1_decompress(data[OPENING_KEY_BYTES:]))
        except kzg.PointMalformed as e:
            raise PointMalformed(str(e)) from e

    @classmethod
    def from_slice_unchecked(cls, data: bytes) -> "PublicParameters":
        """PublicParameters::from_slice_unchecked (srs.rs:121-146) for the bytes of to_raw_var_bytes: the opening key is
        checked (the reference panics where this raises PointMalformed), the commit-key points are not."""
        if len(data) < OPENING_KEY_BYTES:
            raise NotEnoughBytes("NotEnoughBytes")
        opening_key_check(data[:OPENING_KEY_BYTES])
        return cls(data[:OPENING_KEY_BYTES], kzg._raw_key_points(data[OPENING_KEY_BYTES:], False))

    def to_var_bytes(self) -> bytes:
        """PublicParameters::to_var_bytes (srs.rs:149-153)."""
        return kzg.public_parameters_to_var_bytes(self.opening_key, self.raw_points)

    def to_raw_var_bytes(self) -> bytes:
        """PublicParameters::to_raw_var_bytes (srs.rs:114-119)."""
        return kzg.public_parameters_to_raw_var_bytes(self.opening_key, self.raw_points)

    def max_degree(self) -> int:
        """PublicParameters::max_degree: the commit key's, one less than its point count."""
        return len(self.raw_points) // kzg.G1_RAW_BYTES - 1

    def commit_key(self) -> kzg.CommitKey:
        """The commit key, uploaded to the GPU."""
        return kzg.CommitKey(self.raw_points)


class PublicParameterTables(NamedTuple):
    """The derived MSM tables a DevicePublicParameters holds: trimmed-key tables (one per trimmed point count),
    Lagrange-form tables (one per domain size) and their device bytes."""

    monomial: int
    lagrange: int
    device_bytes: int


def _pp_call(call):
    """A pb200_pp_* constructor: call(out) fills a handle; the errors PublicParameters raises are raised as such."""
    h = ctypes.c_void_p()
    try:
        check(call(ctypes.byref(h)))
    except Pb200Error as e:
        if e.code == PB200_ERR_DEGREE_IS_ZERO:
            raise DegreeIsZero("DegreeIsZero") from e
        if e.code == PB200_ERR_POINT_MALFORMED:
            raise PointMalformed(str(e)) from e
        raise
    return DevicePublicParameters(h)


class DevicePublicParameters:
    """One PublicParameters resident on the GPU (pb200_pp_t): the commit key's points in HBM and the opening key.  The
    Compiler and Prover.from_bytes take it wherever they take a PublicParameters; the provers compiled from it share the
    MSM tables derived from the key (one per trimmed-key size and one per domain size), built once and kept until this
    object is freed.  Those provers may outlive it."""

    def __init__(self, handle: ctypes.c_void_p):
        self._h = handle
        okey = ctypes.create_string_buffer(OPENING_KEY_BYTES)
        check(lib().pb200_pp_opening_key(self._h, okey))
        self.opening_key = okey.raw

    @classmethod
    def setup(cls, max_degree: int, draws: Sequence[bytes]) -> "DevicePublicParameters":
        """PublicParameters.setup with the commit key left on the GPU: the same draws, points and errors."""
        x, gs, hs = draws
        assert len(x) == len(gs) == len(hs) == 32
        return _pp_call(lambda out: lib().pb200_pp_setup(max_degree, x, gs, hs, out))

    @classmethod
    def from_slice(cls, data: bytes) -> "DevicePublicParameters":
        """PublicParameters.from_slice, decoding and checking every point on the GPU straight into its place."""
        if len(data) <= OPENING_KEY_BYTES:
            raise NotEnoughBytes("NotEnoughBytes")
        return _pp_call(lambda out: lib().pb200_pp_from_slice(data, len(data), 1, out))

    @classmethod
    def from_slice_unchecked(cls, data: bytes) -> "DevicePublicParameters":
        """PublicParameters.from_slice_unchecked: the opening key checked, the raw commit-key records not."""
        if len(data) < OPENING_KEY_BYTES:
            raise NotEnoughBytes("NotEnoughBytes")
        return _pp_call(lambda out: lib().pb200_pp_from_slice(data, len(data), 0, out))

    @classmethod
    def from_host(cls, pp: PublicParameters) -> "DevicePublicParameters":
        """The same parameters uploaded once; the points are trusted as pb200_prover_new trusts them."""
        n = len(pp.raw_points) // kzg.G1_RAW_BYTES
        return _pp_call(lambda out: lib().pb200_pp_new(pp.raw_points, n, pp.opening_key, out))

    def points(self) -> int:
        return lib().pb200_pp_points(self._h)

    def max_degree(self) -> int:
        """PublicParameters::max_degree: one less than the commit key's point count."""
        return self.points() - 1

    def to_host(self) -> PublicParameters:
        raw = ctypes.create_string_buffer(max(1, self.points()) * kzg.G1_RAW_BYTES)
        check(lib().pb200_pp_raw_points(self._h, raw))
        return PublicParameters(self.opening_key, raw.raw[: self.points() * kzg.G1_RAW_BYTES])

    def tables(self) -> PublicParameterTables:
        mono, lag, nbytes = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
        check(lib().pb200_pp_tables(self._h, ctypes.byref(mono), ctypes.byref(lag), ctypes.byref(nbytes)))
        return PublicParameterTables(mono.value, lag.value, nbytes.value)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().pb200_pp_free(self._h)
                self._h = None
        except Exception:
            pass
