"""tests/models/bucket_reduction_model.py: the row/column bucket reduction of the MSM (csrc/msm.cu, k_msm_rows_cols ..
k_msm_final plus the host Horner) yields sum_b (b + 1) B_b for every window width the library uses, within its
work and depth budget."""
import importlib.util
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def _model():
    spec = importlib.util.spec_from_file_location("bucket_reduction_model", os.path.join(HERE, "models", "bucket_reduction_model.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_bucket_reduction_equals_weighted_bucket_sum():
    m = _model()
    for c in (2, 3, 4, 5, 8, 12, 13):
        m.check(c, seed=c)
    m.check(12, seed=1, density=0.05)  # mostly empty buckets (sparse scalars)


def test_bucket_reduction_work_and_depth_at_c16():
    m = _model()
    adds, depth = m.check(16, seed=16)
    nb = 1 << 15
    assert adds <= 2.3 * nb, adds / nb  # full additions on the device
    assert depth <= 28, depth           # longest chain of dependent ones


def test_bucket_reduction_c20_folds_chunk_sums():
    m = _model()
    adds, depth = m.check(20, seed=20)
    assert adds <= 2.5 * (1 << 19), adds / (1 << 19)
    assert depth <= 34, depth


def test_bucket_reduction_on_curve_points():
    _model().check_curve(5, seed=3)
