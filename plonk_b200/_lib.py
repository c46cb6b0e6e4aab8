"""ctypes loader for libplonk_b200.so (the C ABI declared in include/plonk_b200.h).

Fails loudly when the CUDA library is missing: there is no CPU fallback in the product path."""
from __future__ import annotations

import ctypes
import enum
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# PB200_LIB selects another build of the same library (A/B measurements of compile-time variants)
LIB_PATH = os.environ.get("PB200_LIB") or os.path.join(_HERE, "libplonk_b200.so")

PB200_OK = 0
PB200_ERR_CUDA = -1
PB200_ERR_INVALID_DOMAIN = -2
PB200_ERR_DEGREE_TOO_LARGE = -3
PB200_ERR_INVALID_ARG = -4
PB200_ERR_UNSATISFIED = -5
PB200_ERR_POINT_MALFORMED = -10
PB200_ERR_VERIFY = -11
PB200_ERR_UNSUPPORTED_VERSION = -12
PB200_ERR_DEGREE_IS_ZERO = -13
PB200_ERR_INVALID_COMPRESSED = -14
PB200_ERR_SCALAR_MALFORMED = -15


class PlonkVersion(enum.IntEnum):
    """PlonkVersion (reference src/compiler.rs:22-42), pb200_plonk_version of the C ABI.  V3 is the current
    profile.  V2 is the legacy transcript seed with V3's opening checks.  V1 is the legacy seed with the legacy
    opening, which does not bind the q_arith, q_c, q_l and q_r evaluations: its verdict is meaningful only for
    proofs made under the old rules."""

    V1 = 1
    V2 = 2
    V3 = 3

_lib = None

# every symbol include/plonk_b200.h declares (tests/test_host_logic.py checks the list against the header)
EXPORTS = [
    "pb200_init", "pb200_last_error", "pb200_device_sync", "pb200_launch_count",
    "pb200_ntt", "pb200_ntt_dev",
    "pb200_srs_upload", "pb200_srs_upload_window", "pb200_msm_window_for", "pb200_srs_window", "pb200_srs_free", "pb200_srs_len",
    "pb200_msm_g1", "pb200_msm_g1_dev", "pb200_msm_g1_range", "pb200_msm_g1_allgather", "pb200_msm_g1_allgather_dev", "pb200_msm_combine_parts",
    "pb200_g1_compress", "pb200_g1_compress_batch", "pb200_g1_decompress", "pb200_raw_commit_key_points", "pb200_commit_key_from_raw_var_bytes",
    "pb200_commit_key_to_raw_var_bytes", "pb200_prover_to_bytes", "pb200_g1_add_affine", "pb200_srs_setup_from_secret", "pb200_g1_lagrange_key",
    "pb200_public_parameters_setup", "pb200_opening_key_check",
    "pb200_pp_new", "pb200_pp_setup", "pb200_pp_from_slice", "pb200_pp_points", "pb200_pp_opening_key", "pb200_pp_raw_points",
    "pb200_pp_tables", "pb200_pp_free", "pb200_prover_new_pp", "pb200_prover_from_compressed_pp", "pb200_prover_from_bytes_pp",
    "pb200_circuit_compress", "pb200_compressed_circuit_info", "pb200_prover_from_compressed",
    "pb200_identity_family", "pb200_circuit_unsatisfied", "pb200_prover_unsatisfied",
    "pb200_profile_enable", "pb200_throughput_mode", "pb200_profile_read", "pb200_profile_read_sparse",
    "pb200_prover_new", "pb200_prover_from_bytes", "pb200_prover_free", "pb200_prover_commitments", "pb200_prove", "pb200_prove_dev",
    "pb200_prove_with_version", "pb200_prove_dev_with_version",
    "pb200_verifier_new", "pb200_verifier_from_bytes", "pb200_verifier_to_bytes", "pb200_verifier_free", "pb200_verify", "pb200_verify_with_version",
    "pb200_batch_verify", "pb200_selftest_batch_verify_points", "pb200_batch_verify_groups", "pb200_selftest_batch_verify_groups_points",
    "pb200_imad_peak", "pb200_fp_product_peak", "pb200_selftest_pairing", "pb200_selftest_fr_mul", "pb200_selftest_fp_mul", "pb200_selftest_fp_ops",
]


# every symbol include/plonk_b200_composer.h declares (host-side circuit front end)
COMPOSER_EXPORTS = [
    "pb200_composer_new", "pb200_composer_set_witness_only", "pb200_composer_free", "pb200_composer_constraints", "pb200_composer_witnesses",
    "pb200_composer_public_inputs", "pb200_composer_witness_value", "pb200_composer_append_witness",
    "pb200_composer_append_gate", "pb200_composer_append_evaluated_output", "pb200_composer_gate_add",
    "pb200_composer_append_constant", "pb200_composer_append_public", "pb200_composer_assert_equal",
    "pb200_composer_assert_equal_constant", "pb200_composer_component_boolean", "pb200_composer_component_decomposition",
    "pb200_composer_component_range_bits", "pb200_composer_component_range", "pb200_composer_append_logic",
    "pb200_composer_component_truncate", "pb200_composer_component_select", "pb200_composer_component_select_one",
    "pb200_composer_component_select_zero", "pb200_composer_append_point", "pb200_composer_assert_equal_point",
    "pb200_composer_assert_equal_public_point", "pb200_composer_assert_torsion_free_point", "pb200_composer_point_op",
    "pb200_composer_component_select_identity", "pb200_composer_component_select_point", "pb200_composer_component_mul_point",
    "pb200_composer_component_mul_generator", "pb200_jubjub_generator", "pb200_jubjub_mul",
    "pb200_composer_bench_circuit", "pb200_composer_export",
]


class Pb200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"plonk_b200 error {code}: {msg}")
        self.code = code


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with ./build.sh (or __graft_entry__.build()); "
                "plonk_b200 has no CPU fallback"
            )
        L = ctypes.CDLL(LIB_PATH)
        c = ctypes
        L.pb200_last_error.restype = c.c_char_p
        L.pb200_launch_count.restype = c.c_uint64
        L.pb200_srs_len.restype = c.c_size_t
        L.pb200_srs_len.argtypes = [c.c_void_p]
        L.pb200_srs_free.argtypes = [c.c_void_p]
        L.pb200_srs_free.restype = None
        L.pb200_init.argtypes = [c.c_int]
        L.pb200_ntt.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p, c.c_uint32, c.c_int, c.c_int, c.c_uint32, c.c_size_t, c.c_size_t]
        L.pb200_ntt_dev.argtypes = L.pb200_ntt.argtypes + [c.c_void_p]
        L.pb200_srs_upload.argtypes = [c.c_void_p, c.c_size_t, c.POINTER(c.c_void_p)]
        L.pb200_msm_g1.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_uint32, c.c_size_t, c.c_void_p]
        L.pb200_msm_g1_dev.argtypes = L.pb200_msm_g1.argtypes + [c.c_void_p]
        L.pb200_msm_g1_range.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t, c.c_void_p]
        L.pb200_msm_g1_allgather.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_uint32, c.c_size_t, c.c_void_p, c.c_int, c.c_void_p]
        L.pb200_msm_g1_allgather_dev.argtypes = L.pb200_msm_g1_allgather.argtypes + [c.c_void_p]
        L.pb200_msm_combine_parts.argtypes = [c.c_void_p, c.c_int, c.c_int, c.c_uint32, c.c_void_p, c.POINTER(c.c_size_t)]
        L.pb200_srs_upload_window.argtypes = [c.c_void_p, c.c_size_t, c.c_int, c.POINTER(c.c_void_p)]
        L.pb200_msm_window_for.argtypes = [c.c_size_t]
        L.pb200_srs_window.argtypes = [c.c_void_p]
        L.pb200_g1_lagrange_key.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p]
        L.pb200_selftest_fp_ops.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
        L.pb200_device_sync.argtypes = []
        L.pb200_g1_compress.argtypes = [c.c_void_p, c.c_void_p]
        L.pb200_g1_decompress.argtypes = [c.c_void_p, c.c_size_t, c.c_int, c.c_void_p]
        L.pb200_raw_commit_key_points.argtypes = [c.c_void_p, c.c_size_t, c.c_int, c.POINTER(c.c_size_t)]
        L.pb200_commit_key_from_raw_var_bytes.argtypes = [c.c_void_p, c.c_size_t, c.c_int, c.c_void_p]
        L.pb200_prover_from_bytes.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t, c.POINTER(c.c_void_p)]
        L.pb200_prover_to_bytes.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.POINTER(c.c_size_t)]
        L.pb200_g1_compress_batch.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p]
        L.pb200_commit_key_to_raw_var_bytes.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t, c.POINTER(c.c_size_t)]
        L.pb200_g1_add_affine.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p]
        L.pb200_prover_new.argtypes = [c.c_void_p, c.c_size_t, c.c_size_t, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t, c.POINTER(c.c_void_p)]
        L.pb200_prover_free.argtypes = [c.c_void_p]
        L.pb200_prover_free.restype = None
        L.pb200_prover_commitments.argtypes = [c.c_void_p, c.c_void_p]
        L.pb200_prove.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p]
        L.pb200_prove_dev.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p]
        L.pb200_prove_with_version.argtypes = L.pb200_prove.argtypes[:1] + [c.c_int] + L.pb200_prove.argtypes[1:]
        L.pb200_prove_dev_with_version.argtypes = L.pb200_prove_dev.argtypes[:1] + [c.c_int] + L.pb200_prove_dev.argtypes[1:]
        L.pb200_srs_setup_from_secret.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p]
        L.pb200_public_parameters_setup.argtypes = [c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p]
        L.pb200_opening_key_check.argtypes = [c.c_void_p]
        L.pb200_pp_new.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p, c.POINTER(c.c_void_p)]
        L.pb200_pp_setup.argtypes = [c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p, c.POINTER(c.c_void_p)]
        L.pb200_pp_from_slice.argtypes = [c.c_void_p, c.c_size_t, c.c_int, c.POINTER(c.c_void_p)]
        L.pb200_pp_points.argtypes = [c.c_void_p]
        L.pb200_pp_points.restype = c.c_size_t
        L.pb200_pp_opening_key.argtypes = [c.c_void_p, c.c_void_p]
        L.pb200_pp_raw_points.argtypes = [c.c_void_p, c.c_void_p]
        L.pb200_pp_tables.argtypes = [c.c_void_p, c.POINTER(c.c_size_t), c.POINTER(c.c_size_t), c.POINTER(c.c_size_t)]
        L.pb200_pp_free.argtypes = [c.c_void_p]
        L.pb200_pp_free.restype = None
        L.pb200_prover_new_pp.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_size_t, c.c_void_p, c.c_void_p, c.c_size_t, c.POINTER(c.c_void_p)]
        L.pb200_prover_from_compressed_pp.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t, c.POINTER(c.c_void_p)]
        L.pb200_prover_from_bytes_pp.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t, c.POINTER(c.c_void_p)]
        L.pb200_circuit_compress.argtypes = [c.c_size_t, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t, c.c_int, c.c_void_p,
                                             c.c_size_t, c.POINTER(c.c_size_t)]
        L.pb200_compressed_circuit_info.argtypes = [c.c_void_p, c.c_size_t, c.c_size_t, c.POINTER(c.c_size_t), c.POINTER(c.c_uint64),
                                                    c.POINTER(c.c_size_t), c.POINTER(c.c_size_t), c.c_void_p]
        L.pb200_prover_from_compressed.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t, c.POINTER(c.c_void_p)]
        L.pb200_identity_family.argtypes = [c.c_int]
        L.pb200_identity_family.restype = c.c_char_p
        L.pb200_circuit_unsatisfied.argtypes = [c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p,
                                                c.c_size_t, c.c_size_t, c.c_void_p, c.c_void_p, c.POINTER(c.c_size_t)]
        L.pb200_prover_unsatisfied.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_size_t, c.c_size_t,
                                               c.c_void_p, c.c_void_p, c.POINTER(c.c_size_t)]
        L.pb200_profile_enable.argtypes = [c.c_int]
        L.pb200_throughput_mode.argtypes = [c.c_int]
        L.pb200_profile_read.argtypes = [c.POINTER(c.c_double), c.POINTER(c.c_uint64), c.POINTER(c.c_uint64), c.POINTER(c.c_uint64)]
        L.pb200_profile_read_sparse.argtypes = L.pb200_profile_read.argtypes
        L.pb200_imad_peak.argtypes = [c.POINTER(c.c_double)]
        L.pb200_fp_product_peak.argtypes = [c.POINTER(c.c_double)]
        L.pb200_selftest_fr_mul.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
        L.pb200_selftest_fp_mul.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t]
        L.pb200_verifier_new.argtypes = [c.c_void_p, c.c_size_t, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t, c.POINTER(c.c_void_p)]
        L.pb200_verifier_from_bytes.argtypes = [c.c_void_p, c.c_size_t, c.POINTER(c.c_void_p)]
        L.pb200_verifier_to_bytes.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.POINTER(c.c_size_t)]
        L.pb200_verifier_free.argtypes = [c.c_void_p]
        L.pb200_verifier_free.restype = None
        L.pb200_verify.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t, c.c_void_p]
        L.pb200_verify_with_version.argtypes = [c.c_void_p, c.c_int] + L.pb200_verify.argtypes[1:]
        L.pb200_batch_verify.argtypes = L.pb200_verify_with_version.argtypes
        L.pb200_selftest_batch_verify_points.argtypes = L.pb200_batch_verify.argtypes + [c.c_void_p]
        L.pb200_batch_verify_groups.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p]
        L.pb200_selftest_batch_verify_groups_points.argtypes = L.pb200_batch_verify_groups.argtypes + [c.c_void_p]
        L.pb200_selftest_pairing.argtypes = [c.c_void_p, c.c_void_p, c.c_size_t, c.c_void_p]
        _bind_composer(L)
        _lib = L
    return _lib


def _bind_composer(L) -> None:
    c = ctypes
    H, W, P, I = c.c_void_p, c.c_uint32, c.c_void_p, c.c_int
    sig = {
        "pb200_composer_new": [c.POINTER(c.c_void_p)],
        "pb200_composer_set_witness_only": [H, I],
        "pb200_composer_witness_value": [H, W, P],
        "pb200_composer_append_witness": [H, P, P],
        "pb200_composer_append_gate": [H, P, P, P, I],
        "pb200_composer_append_evaluated_output": [H, P, P, P, P, P],
        "pb200_composer_gate_add": [H, P, P, P, P],
        "pb200_composer_append_constant": [H, P, P],
        "pb200_composer_append_public": [H, P, P],
        "pb200_composer_assert_equal": [H, W, W],
        "pb200_composer_assert_equal_constant": [H, W, P, P],
        "pb200_composer_component_boolean": [H, W],
        "pb200_composer_component_decomposition": [H, W, W, P],
        "pb200_composer_component_range_bits": [H, W, W],
        "pb200_composer_component_range": [H, W, W],
        "pb200_composer_append_logic": [H, W, W, W, I, P],
        "pb200_composer_component_truncate": [H, W, W, P],
        "pb200_composer_component_select": [H, W, W, W, P],
        "pb200_composer_component_select_one": [H, W, W, P],
        "pb200_composer_component_select_zero": [H, W, W, P],
        "pb200_composer_append_point": [H, P, I, P],
        "pb200_composer_assert_equal_point": [H, P, P],
        "pb200_composer_assert_equal_public_point": [H, P, P],
        "pb200_composer_assert_torsion_free_point": [H, P],
        "pb200_composer_point_op": [H, I, P, P, P],
        "pb200_composer_component_select_identity": [H, W, P, P],
        "pb200_composer_component_select_point": [H, W, P, P, P],
        "pb200_composer_component_mul_point": [H, W, P, P],
        "pb200_composer_component_mul_generator": [H, W, P, P],
        "pb200_jubjub_generator": [P],
        "pb200_jubjub_mul": [P, P, P],
        "pb200_composer_bench_circuit": [H, c.c_size_t],
        "pb200_composer_export": [H, P, P, P, P, P],
    }
    for name, args in sig.items():
        getattr(L, name).argtypes = args
    L.pb200_composer_free.argtypes = [H]
    L.pb200_composer_free.restype = None
    for name in ("pb200_composer_constraints", "pb200_composer_witnesses", "pb200_composer_public_inputs"):
        getattr(L, name).argtypes = [H]
        getattr(L, name).restype = c.c_size_t


def check(rc: int) -> None:
    if rc != 0:
        raise Pb200Error(rc, lib().pb200_last_error().decode())
