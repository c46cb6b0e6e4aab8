"""TEST INFRASTRUCTURE - batch verification over groups (pb200_batch_verify_groups) on top of
tests/models/batch_verify_model.py.

Group g is a list of proofs checked under its own verifier and version; every verifier shares one opening key.  The
call passes iff e(sum w_i L_i, [x]H) e(sum w_i R_i, H) = 1 over all proofs in call order, w_i = rho^i, with rho drawn
from one merlin transcript over the whole call:

    T = Transcript::new(b"dusk-plonk")
    T.append_message(b"dom-sep", b"plonk-batch-verify-v1")
    for each group: T.append_u64(b"version", version); T.append_u64(b"batch-len", n_g)
                    for each proof of the group: T.append_scalar(b"batch-u", u_i)
    rho = T.challenge_scalar(b"batch-challenge")

One group gives batch_verify_model.batch_challenge(version, us).

Only tests/ may import this file."""
from __future__ import annotations

from typing import Sequence, Tuple

from oracle import pyref as P

from . import batch_verify_model as BV

R_MOD = P.R_MOD


def batch_challenge(groups: Sequence[Tuple[int, Sequence[int]]]) -> int:
    """rho for groups given as (version, [u_i of the group's proofs])."""
    t = P.Transcript(b"dusk-plonk")
    t.append_message(b"dom-sep", b"plonk-batch-verify-v1")
    for version, us in groups:
        t.append_u64(b"version", version)
        t.append_u64(b"batch-len", len(us))
        for u in us:
            t.append_scalar(b"batch-u", u % R_MOD)
    return t.challenge_scalar(b"batch-challenge")


def fold(groups: Sequence[Tuple[int, Sequence[int], Sequence[Tuple[object, object]]]]):
    """(sum w_i L_i, sum w_i R_i) over groups given as (version, us, pairs (L_i, R_i)), weights over the call order."""
    rho = batch_challenge([(v, us) for v, us, _ in groups])
    pairs = [p for _, _, ps in groups for p in ps]
    return BV.fold(pairs, BV.weights(rho, len(pairs)))
