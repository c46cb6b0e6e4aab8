"""tests/models/coset8_eval_model.py: the 4n-coset quotient's evaluations on h*H_8 and omega*h*H_8, computed as
k_coset8_eval + k_coset8_sum split them (one fold per polynomial, an 8-point DFT), equal Horner at all 16 points
for random polynomials of n + 3 and 4n coefficients."""
import importlib.util
import os

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _model():
    spec = importlib.util.spec_from_file_location("coset8_eval_model", os.path.join(HERE, "models", "coset8_eval_model.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.mark.parametrize("log_n", range(4, 11))
def test_coset8_fold_matches_horner_kernel_geometry(log_n):
    _model().check(log_n, 100 + log_n)


@pytest.mark.parametrize("log_n", range(4, 11))
def test_coset8_fold_matches_horner_many_blocks(log_n):
    """Blocks of 4 threads x 2 groups: at n = 2^10 the 4n polynomial has 64 blocks, so the sum's block lanes
    take several blocks each and every job's last block takes a remainder."""
    _model().check(log_n, 200 + log_n, dict(thread_bits=2, per=2, lane_bits=1, sum_lane_bits=5))
