"""Verifier (reference src/compiler/verifier.rs) on the GPU, through pb200_verifier_*, pb200_verify_with_version,
pb200_batch_verify and pb200_batch_verify_groups of include/plonk_b200.h.  Every PlonkVersion is verified on the
device; V3 is the default."""
from __future__ import annotations

import ctypes
from typing import List, Sequence, Tuple

from ._lib import PB200_ERR_INVALID_ARG, PB200_ERR_POINT_MALFORMED, PB200_ERR_VERIFY, Pb200Error, PlonkVersion, check, lib

PROOF_BYTES = 1008
OPENING_KEY_BYTES = 240


class ProofVerificationError(Exception):
    """Error::ProofVerificationError: the proof does not satisfy the verifier's equation."""


class PointMalformed(Exception):
    """dusk_bytes InvalidData from Proof::from_bytes: a malformed commitment or a non-canonical scalar."""


class Verifier:
    def __init__(self, label: bytes, n_constraints: int, commitments: Sequence[bytes], opening_key: bytes, pi_idx: bytes = b""):
        """commitments: the 15 compressed verifier-key commitments in Prover.commitments() order; opening_key:
        OpeningKey::to_bytes; pi_idx: public-input positions as little-endian u64 (as Prover.prove takes them)."""
        assert len(commitments) == 15 and len(opening_key) == OPENING_KEY_BYTES and len(pi_idx) % 8 == 0
        h = ctypes.c_void_p()
        check(lib().pb200_verifier_new(label, len(label), n_constraints, b"".join(commitments), opening_key, pi_idx or None,
                                       len(pi_idx) // 8, ctypes.byref(h)))
        self._h = h
        self.n_pi = len(pi_idx) // 8

    @classmethod
    def from_bytes(cls, data: bytes) -> "Verifier":
        """Verifier::try_from_bytes."""
        self = cls.__new__(cls)
        h = ctypes.c_void_p()
        check(lib().pb200_verifier_from_bytes(data, len(data), ctypes.byref(h)))
        self._h = h
        self.n_pi = int.from_bytes(data[24:32], "big")
        return self

    def to_bytes(self) -> bytes:
        """Verifier::to_bytes."""
        n = ctypes.c_size_t()
        check(lib().pb200_verifier_to_bytes(self._h, None, 0, ctypes.byref(n)))
        out = ctypes.create_string_buffer(n.value)
        check(lib().pb200_verifier_to_bytes(self._h, out, n.value, ctypes.byref(n)))
        return out.raw

    def verify_batch(self, proofs: Sequence[bytes], pi_vals: Sequence[bytes], version: PlonkVersion = PlonkVersion.V3) -> List[int]:
        """One status per proof (PB200_OK, PB200_ERR_VERIFY or PB200_ERR_POINT_MALFORMED); pi_vals[i]: the public
        inputs of proof i, 32 bytes (Montgomery form) each.  Every proof is checked under `version`."""
        assert len(proofs) == len(pi_vals) and all(len(p) == PROOF_BYTES for p in proofs)
        n_pi = len(pi_vals[0]) // 32 if pi_vals else self.n_pi
        if any(len(v) != 32 * n_pi for v in pi_vals):
            raise ValueError("every proof needs the same number of public inputs")
        status = (ctypes.c_int32 * max(1, len(proofs)))()
        vals = b"".join(pi_vals)
        check(lib().pb200_verify_with_version(self._h, int(version), b"".join(proofs), len(proofs), vals or None, n_pi, status))
        return list(status[: len(proofs)])

    def batch_verify(self, proofs: Sequence[bytes], pi_vals: Sequence[bytes], version: PlonkVersion = PlonkVersion.V3) -> None:
        """One verdict for the whole batch at the cost of one pairing (pb200_batch_verify): returns when every proof
        would pass verify_with_version (up to a chance of (len(proofs) - 1) / r), raises PointMalformed when some
        proof fails Proof::from_bytes, otherwise ProofVerificationError, also for an empty batch; ValueError for
        inconsistent public inputs or an unknown version."""
        assert len(proofs) == len(pi_vals) and all(len(p) == PROOF_BYTES for p in proofs)
        n_pi = len(pi_vals[0]) // 32 if pi_vals else self.n_pi
        if any(len(v) != 32 * n_pi for v in pi_vals):
            raise ValueError("every proof needs the same number of public inputs")
        verdict = ctypes.c_int32()
        vals = b"".join(pi_vals)
        _raise_verdict(lambda: lib().pb200_batch_verify(self._h, int(version), b"".join(proofs) or None, len(proofs), vals or None,
                                                        n_pi, ctypes.byref(verdict)), verdict)

    def verify(self, proof: bytes, pi_vals: bytes) -> None:
        """Verifier::verify: returns on success, raises ProofVerificationError, PointMalformed or ValueError."""
        self.verify_with_version(proof, pi_vals, PlonkVersion.V3)

    def verify_with_version(self, proof: bytes, pi_vals: bytes, version: PlonkVersion) -> None:
        """Verifier::verify_with_version: as verify, under `version`.  A V1 verdict does not bind the selector
        evaluations; it is meaningful only for proofs made under the old rules."""
        try:
            (st,) = self.verify_batch([proof], [pi_vals], version)
        except Pb200Error as e:
            if e.code == PB200_ERR_INVALID_ARG:
                raise ValueError(str(e)) from e
            raise
        if st == PB200_ERR_VERIFY:
            raise ProofVerificationError("ProofVerificationError")
        if st == PB200_ERR_POINT_MALFORMED:
            raise PointMalformed("InvalidData")

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().pb200_verifier_free(self._h)
                self._h = None
        except Exception:
            pass


def _raise_verdict(call, verdict: ctypes.c_int32) -> None:
    """Runs a batch call and turns its return code and verdict into the errors of Verifier.batch_verify."""
    try:
        check(call())
    except Pb200Error as e:
        if e.code == PB200_ERR_INVALID_ARG:
            raise ValueError(str(e)) from e
        raise
    if verdict.value == PB200_ERR_VERIFY:
        raise ProofVerificationError("ProofVerificationError")
    if verdict.value == PB200_ERR_POINT_MALFORMED:
        raise PointMalformed("InvalidData")


def batch_verify_groups(groups: Sequence[Tuple[Verifier, Sequence[bytes], Sequence[bytes], PlonkVersion]]) -> None:
    """One verdict for groups of proofs under several verifiers and versions, at the cost of one pairing
    (pb200_batch_verify_groups).  groups: (verifier, proofs, pi_vals, version) each, as Verifier.batch_verify takes
    them; the verifiers must share one opening key (one SRS), and one verifier may appear in several groups.  Returns
    when every proof would pass its group's verify_with_version (up to a chance of (N - 1) / r over the N proofs),
    raises PointMalformed when some proof fails Proof::from_bytes, otherwise ProofVerificationError, also when there
    are no proofs at all; ValueError for inconsistent public inputs, an unknown version or verifiers with different
    opening keys."""
    n_pi, n_proofs, proofs, vals = [], [], [], []
    for verifier, ps, pis, _ in groups:
        assert len(ps) == len(pis) and all(len(p) == PROOF_BYTES for p in ps)
        k = len(pis[0]) // 32 if pis else verifier.n_pi
        if any(len(v) != 32 * k for v in pis):
            raise ValueError("every proof needs the same number of public inputs")
        n_pi.append(k)
        n_proofs.append(len(ps))
        proofs += ps
        vals += pis
    m = len(groups)
    handles = (ctypes.c_void_p * max(1, m))(*[g[0]._h.value for g in groups])
    versions = (ctypes.c_int32 * max(1, m))(*[int(g[3]) for g in groups])
    counts = (ctypes.c_size_t * max(1, m))(*n_proofs)
    pi_counts = (ctypes.c_size_t * max(1, m))(*n_pi)
    verdict = ctypes.c_int32()
    _raise_verdict(lambda: lib().pb200_batch_verify_groups(handles, versions, counts, pi_counts, m, b"".join(proofs) or None,
                                                           b"".join(vals) or None, ctypes.byref(verdict)), verdict)
