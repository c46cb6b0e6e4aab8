"""TEST INFRASTRUCTURE - batch verification (pb200_batch_verify) restated on top of oracle/pyref.py.

Proof i's pairing check is e(L_i, [x]H) e(R_i, H) = 1 with L_i = -(W_z + u_i W_zw) and R_i the right-hand point of
Proof::verify (tests/models/plonk_versions_model.right_and_left).  A batch passes iff
e(sum w_i L_i, [x]H) e(sum w_i R_i, H) = 1, w_i = rho^i, with rho drawn from a merlin transcript over the batch in
the style of the reference's batch_challenge (key.rs:571-591):

    T = Transcript::new(b"dusk-plonk")
    T.append_message(b"dom-sep", b"plonk-batch-verify-v1")
    T.append_u64(b"version", version); T.append_u64(b"batch-len", n)
    for each proof: T.append_scalar(b"batch-u", u_i)
    rho = T.challenge_scalar(b"batch-challenge")

Only tests/ may import this file."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

from oracle import pyref as P

from . import pairing_model as PM

R_MOD = P.R_MOD


def batch_challenge(version: int, us: Sequence[int]) -> int:
    t = P.Transcript(b"dusk-plonk")
    t.append_message(b"dom-sep", b"plonk-batch-verify-v1")
    t.append_u64(b"version", version)
    t.append_u64(b"batch-len", len(us))
    for u in us:
        t.append_scalar(b"batch-u", u % R_MOD)
    return t.challenge_scalar(b"batch-challenge")


def weights(rho: int, n: int) -> List[int]:
    return [pow(rho, i, R_MOD) for i in range(n)]


def _lin(points: Sequence[Optional[tuple]], scalars: Sequence[int]):
    acc = None
    for p, s in zip(points, scalars):
        if p is None or s % R_MOD == 0:
            continue
        t = P.jac_mul(P.jac_from_affine(p), s % R_MOD)
        acc = t if acc is None else P.jac_add(acc, t)
    return None if acc is None else P.jac_to_affine(acc)


def left(w_z, w_zw, u: int):
    """L = -(W_z + u W_zw)."""
    s = _lin([w_z, w_zw], [1, u])
    return None if s is None else P.g1_neg(s)


def fold(pairs: Sequence[Tuple[object, object]], w: Sequence[int]):
    """(sum w_i L_i, sum w_i R_i) for pairs (L_i, R_i)."""
    return _lin([p[0] for p in pairs], w), _lin([p[1] for p in pairs], w)


def accepts_with_secret(L, R, x: int) -> bool:
    """e(L, [x]H) e(R, H) = 1 iff R = -[x] L."""
    want = None if L is None else P.g1_neg(P.g1_mul(L, x % R_MOD))
    return R == want


def accepts_with_pairing(L, R, opening_key: bytes) -> bool:
    _, h, x_h = PM.parse_opening_key(opening_key)
    return PM.pairing_product_is_one([(L, x_h), (R, h)])


def raw_points(L, R) -> bytes:
    """The selftest's layout: L then R, 96-byte raw affine each, zeros for the identity."""
    return b"".join(P.g1_to_raw_bytes(p) if p is not None else bytes(96) for p in (L, R))
