"""GPU tests of the bucket walk's rare steps: a bucket whose first two entries are P and P (doubling) or P and -P
(cancellation), reached from the entry that starts the sum, and commit keys that hold the identity, whose
entries the MSM leaves out before the walk."""
import random

import pytest

from oracle import pyref as R
from tests.util import bases_to_abi, progression_bases, rand_fr, to_abi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pb():
    import plonk_b200
    from plonk_b200._lib import check, lib

    check(lib().pb200_init(0))
    return plonk_b200


def _check(pb, pts, scalars_list):
    key = pb.CommitKey(bases_to_abi(pts))
    got = key.commit_batch([to_abi(s) for s in scalars_list])
    for g, s in zip(got, scalars_list):
        assert R.g1_from_raw_bytes(g.raw) == R.jac_to_affine(R.msm_pippenger(pts, s))


def test_bucket_starting_with_equal_or_opposite_points(pb):
    """Equal scalars on two bases put both into the same bucket of every window, as its only two entries: the
    first starts the sum and the second is the rare step.  A third base makes the step after it meet the
    identity (P + (-P)) or a doubled point, in whichever order the entries land."""
    rng = random.Random(71)
    P, Q = progression_bases(2, rng.randrange(1, R.R_MOD), rng.randrange(1, R.R_MOD))
    s = rng.randrange(1, R.R_MOD)
    cases = [
        ([P, P], [[s, s], [1, 1], [R.R_MOD - 1, R.R_MOD - 1]]),  # doubling
        ([P, R.g1_neg(P)], [[s, s], [3, 3]]),  # cancellation by the base
        ([P, P], [[s, R.R_MOD - s], [5, R.R_MOD - 5]]),  # cancellation by the digit signs
        ([P, R.g1_neg(P), Q], [[s, s, s], [7, 7, 7]]),
        ([P, P, Q], [[s, s, s], [s, s, R.R_MOD - s]]),
    ]
    for pts, scalars in cases:
        _check(pb, pts, scalars)


def test_commit_key_holding_the_identity(pb):
    """Identity bases at the ends and inside a key, and a key of identities only: the commitment is that of
    the other bases, with all-equal scalars (every entry in one bucket per window) and random ones."""
    rng = random.Random(72)
    n = 300
    pts = progression_bases(n, rng.randrange(1, R.R_MOD), rng.randrange(1, R.R_MOD))
    for i in (0, 1, 150, 151, 152, n - 1):
        pts[i] = None
    big = rng.randrange(R.R_MOD)
    _check(pb, pts, [[big] * n, [1] * n, rand_fr(rng, n), [rng.randrange(1 << 16) for _ in range(n)]])
    _check(pb, [None] * 5, [[big] * 5, rand_fr(rng, 5)])
