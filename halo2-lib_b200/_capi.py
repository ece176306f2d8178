"""ctypes binding of libh2b200.so: the symbols include/h2b200.h declares (SIGNATURES), and the private calls through
which prover.py drives the compiled resident prover (PROVER_SIGNATURES, halo2-lib_b200/csrc/prover_binding.cu).

There is no fallback: if the shared library is missing the import fails, and if no CUDA device is present
`Context()` raises (h2b_ctx_create returns H2B_ERR_CUDA)."""
from __future__ import annotations
import ctypes as C
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libh2b200.so")
HEADER_PATH = os.path.join(os.path.dirname(HERE), "include", "h2b200.h")

H2B_OK, H2B_ERR_ARG, H2B_ERR_CUDA, H2B_ERR_OOM, H2B_ERR_LAYOUT, H2B_ERR_UNSATISFIED = 0, -1, -2, -3, -4, -5
BASIS_MONOMIAL, BASIS_LAGRANGE = 0, 1
CHECK_MAX_REPORT = 65536  # H2B_CHECK_MAX_REPORT

_vp, _sz, _u32, _int = C.c_void_p, C.c_size_t, C.c_uint32, C.c_int
_u64p = C.POINTER(C.c_uint64)



class Graph(C.Structure):
    """h2b_graph (include/h2b200.h): a GraphEvaluator program plus its column tables and challenges."""
    _fields_ = [
        ("program", C.POINTER(C.c_uint32)), ("program_words", C.c_size_t),
        ("n_calculations", C.c_uint32), ("result", C.c_uint32),
        ("constants", C.c_void_p), ("n_constants", C.c_size_t),
        ("rotations", C.POINTER(C.c_int32)), ("n_rotations", C.c_size_t),
        ("fixed", C.POINTER(C.c_void_p)), ("n_fixed", C.c_size_t),
        ("advice", C.POINTER(C.c_void_p)), ("n_advice", C.c_size_t),
        ("instance", C.POINTER(C.c_void_p)), ("n_instance", C.c_size_t),
        ("challenges", C.c_void_p), ("n_challenges", C.c_size_t),
        ("beta", C.c_uint64 * 4), ("gamma", C.c_uint64 * 4), ("theta", C.c_uint64 * 4), ("y", C.c_uint64 * 4),
    ]


_gp = C.POINTER(Graph)
_vpp = C.POINTER(C.c_void_p)

# name -> (restype, argtypes)
SIGNATURES = {
    "h2b_version": (C.c_char_p, []),
    "h2b_ctx_create": (_int, [_int, C.POINTER(_vp)]),
    "h2b_ctx_create_multi": (_int, [C.POINTER(_int), _int, C.POINTER(_vp)]),
    "h2b_ctx_device_count": (_int, [_vp]),
    "h2b_ctx_destroy": (None, [_vp]),
    "h2b_ctx_set_stream": (_int, [_vp, _vp]),
    "h2b_ctx_synchronize": (_int, [_vp]),
    "h2b_ctx_side_begin": (_int, [_vp]),
    "h2b_ctx_side_end": (_int, [_vp]),
    "h2b_ctx_side_join": (_int, [_vp]),
    "h2b_ctx_set_option": (_int, [_vp, C.c_char_p, C.c_int64]),
    "h2b_last_error": (C.c_char_p, [_vp]),
    "h2b_kernel_launches": (C.c_uint64, [_vp]),
    "h2b_profile_enable": (_int, [_vp, C.c_char_p]),
    "h2b_profile_reset": (_int, [_vp]),
    "h2b_profile_read": (_int, [_vp, C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    "h2b_profile_dump": (_int, [_vp, _vp, C.c_char_p]),
    "h2b_srs_upload": (_int, [_vp, _vp, _vp, _u32, _sz, _sz, C.POINTER(_vp)]),
    "h2b_srs_upload_dev": (_int, [_vp, _vp, _vp, _u32, _sz, _sz, C.POINTER(_vp)]),
    "h2b_srs_info": (_int, [_vp, C.POINTER(_int), C.POINTER(_int)]),
    "h2b_srs_destroy": (None, [_vp, _vp]),
    "h2b_msm_g1": (_int, [_vp, _vp, _int, _vp, _sz, _vp]),
    "h2b_msm_g1_batch": (_int, [_vp, _vp, C.POINTER(_int), C.POINTER(_vp), _sz, _sz, _vp]),
    "h2b_msm_g1_batch_reduced": (_int, [_vp, _vp, C.POINTER(_int), C.POINTER(_vp), _sz, _sz, _vp]),
    "h2b_msm_g1_batch_dev": (_int, [_vp, _vp, C.POINTER(_int), C.POINTER(_vp), _sz, _sz, _vp]),
    "h2b_msm_g1_bases": (_int, [_vp, _vp, _vp, _sz, _vp]),
    "h2b_msm_g1_dev": (_int, [_vp, _vp, _int, _vp, _sz, _vp]),
    "h2b_msm_g1_bases_dev": (_int, [_vp, _vp, _vp, _sz, _vp]),
    "h2b_g1_sum": (_int, [_vp, _vp, _sz, _vp]),
    "h2b_g1_sum_dev": (_int, [_vp, _vp, _sz, _vp]),
    "h2b_g1_normalize": (_int, [_vp, _vp, _sz]),
    "h2b_g1_fixed_base_mul": (_int, [_vp, _vp, _vp, _sz, _vp]),
    "h2b_g1_fixed_base_mul_dev": (_int, [_vp, _vp, _vp, _sz, _vp]),
    "h2b_peer_create": (_int, [_vp, _int, _int, _vp]),
    "h2b_peer_connect": (_int, [_vp, _vp]),
    "h2b_g1_allreduce_dev": (_int, [_vp, _vp, _sz]),
    "h2b_ntt_fr": (_int, [_vp, _vp, _u32, _vp, _int]),
    "h2b_ntt_fr_dev": (_int, [_vp, _vp, _u32, _vp, _int]),
    "h2b_domain_omega": (_int, [_u32, _vp]),
    "h2b_lagrange_to_coeff": (_int, [_vp, _vp, _u32]),
    "h2b_coeff_to_lagrange": (_int, [_vp, _vp, _u32]),
    "h2b_lagrange_to_coeff_dev": (_int, [_vp, _vp, _u32]),
    "h2b_coeff_to_lagrange_dev": (_int, [_vp, _vp, _u32]),
    "h2b_lagrange_to_coeff_batch": (_int, [_vp, C.POINTER(_vp), _sz, _u32]),
    "h2b_coeff_to_lagrange_batch": (_int, [_vp, C.POINTER(_vp), _sz, _u32]),
    "h2b_lagrange_to_coeff_and_extended_batch": (_int, [_vp, C.POINTER(_vp), _sz, _u32, _u32, C.POINTER(_vp)]),
    "h2b_coeff_to_extended_batch": (_int, [_vp, C.POINTER(_vp), _sz, _sz, _u32, C.POINTER(_vp)]),
    "h2b_coeff_to_extended": (_int, [_vp, _vp, _sz, _u32, _vp]),
    "h2b_coeff_to_extended_dev": (_int, [_vp, _vp, _sz, _u32, _vp]),
    "h2b_extended_to_coeff": (_int, [_vp, _vp, _u32]),
    "h2b_extended_to_coeff_dev": (_int, [_vp, _vp, _u32]),
    "h2b_assign_columns": (_int, [_vp, _vp, _sz, _vp, _sz, _u32, _sz, _vp]),
    "h2b_assign_columns_dev": (_int, [_vp, _vp, _sz, _vp, _sz, _u32, _sz, _vp]),
    "h2b_assign_columns_assigned": (_int, [_vp, _vp, _sz, _vp, _sz, _u32, _sz, _vp]),
    "h2b_assign_columns_assigned_dev": (_int, [_vp, _vp, _sz, _vp, _sz, _u32, _sz, _vp]),
    "h2b_assign_lookups": (_int, [_vp, _vp, _sz, _u32, _sz, _vp]),
    "h2b_assign_lookups_dev": (_int, [_vp, _vp, _sz, _u32, _sz, _vp]),
    "h2b_eval_rational": (_int, [_vp, _vp, _vp, _sz, _vp]),
    "h2b_eval_rational_dev": (_int, [_vp, _vp, _vp, _sz, _vp]),
    "h2b_apply_rational_dev": (_int, [_vp, _vp, _sz, _vp, _vp, _sz, _vp]),
    "h2b_assign_lookups_indexed_dev": (_int, [_vp, _vp, _sz, _vp, _sz, _u32, _sz, _vp, _vp]),
    "h2b_batch_invert_fr": (_int, [_vp, _vp, _sz]),
    "h2b_batch_invert_fr_dev": (_int, [_vp, _vp, _sz]),
    "h2b_grand_product_fr": (_int, [_vp, _vp, _vp, _sz, _vp]),
    "h2b_grand_product_fr_dev": (_int, [_vp, _vp, _vp, _sz, _vp]),
    "h2b_flex_gate_fold": (_int, [_vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "h2b_flex_gate_fold_dev": (_int, [_vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "h2b_g_to_lagrange": (_int, [_vp, _vp, _u32, _vp]),
    "h2b_g_to_lagrange_dev": (_int, [_vp, _vp, _u32, _vp]),
    "h2b_srs_setup": (_int, [_vp, _vp, _vp, _u32, _vp, _vp]),
    "h2b_srs_setup_dev": (_int, [_vp, _vp, _vp, _u32, _vp, _vp]),
    "h2b_g1_check_on_curve": (_int, [_vp, _vp, _sz, C.POINTER(_sz)]),
    "h2b_g1_check_on_curve_dev": (_int, [_vp, _vp, _sz, C.POINTER(_sz)]),
    "h2b_g1_decompress": (_int, [_vp, _vp, _sz, _vp, C.POINTER(_sz)]),
    "h2b_g1_decompress_dev": (_int, [_vp, _vp, _sz, _vp, C.POINTER(_sz)]),
    "h2b_params_processed_view": (_int, [_vp, _sz, C.POINTER(_u32), C.POINTER(_sz), C.POINTER(_sz), C.POINTER(_sz), C.POINTER(_sz)]),
    "h2b_srs_read_processed": (_int, [_vp, _vp, _sz, _sz, _sz, C.POINTER(_vp)]),
    "h2b_params_raw_view": (_int, [_vp, _sz, C.POINTER(_u32), C.POINTER(_sz), C.POINTER(_sz), C.POINTER(_sz), C.POINTER(_sz)]),
    "h2b_g1_compress": (_int, [_vp, _vp, _sz, _vp]),
    "h2b_g1_compress_dev": (_int, [_vp, _vp, _sz, _vp]),
    "h2b_srs_seeded_tau": (_int, [_vp, _vp]),
    "h2b_g2_generator_mul": (_int, [_vp, _vp, _vp]),
    "h2b_params_write_processed": (_int, [_vp, _vp, _vp, _u32, _vp, _vp, C.POINTER(_sz)]),
    "h2b_params_write_raw": (_int, [_vp, _vp, _vp, _u32, _vp, _vp, C.POINTER(_sz)]),
    "h2b_permute_expression_pair": (_int, [_vp, _vp, _vp, _u32, _u32, _vp, _vp]),
    "h2b_permute_expression_pair_dev": (_int, [_vp, _vp, _vp, _u32, _u32, _vp, _vp]),
    "h2b_permute_expression_pair_async_dev": (_int, [_vp, _vp, _vp, _u32, _u32, _vp, _vp, _vp]),
    "h2b_quotient_graph": (_int, [_vp, _gp, _u32, _u32, _vp]),
    "h2b_quotient_graph_dev": (_int, [_vp, _gp, _u32, _u32, _vp]),
    "h2b_permutation_fold": (_int, [_vp, _vpp, _sz, _vpp, _vpp, _sz, _sz, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _u32, _vp]),
    "h2b_permutation_fold_dev": (_int, [_vp, _vpp, _sz, _vpp, _vpp, _sz, _sz, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _u32, _vp]),
    "h2b_lookup_fold": (_int, [_vp, _gp, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "h2b_lookup_fold_dev": (_int, [_vp, _gp, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "h2b_check_graph_dev": (_int, [_vp, _gp, _u32, _sz, _sz, _vp]),
    "h2b_check_lookup_dev": (_int, [_vp, _vp, _vp, _u32, _sz, _sz, _vp]),
    "h2b_permutation_decode_dev": (_int, [_vp, _vpp, _sz, _u32, _vp, _sz, _vp]),
    "h2b_check_copies_dev": (_int, [_vp, _vpp, _vp, _sz, _u32, _sz, _vp]),
    "h2b_mock_selectors_dev": (_int, [_vp, _vp, _sz, _vp, _sz, _u32, _sz, _vp]),
    "h2b_mock_lookup_selector_dev": (_int, [_vp, _vp, _sz, _sz, _sz, _u32, _vp, _vp]),
    "h2b_check_equalities_dev": (_int, [_vp, _vp, _sz, _vp, _sz, _sz, _vp, _vp]),
    "h2b_check_constants_dev": (_int, [_vp, _vp, _sz, _vp, _vp, _sz, _sz, _vp, _vp]),
    "h2b_count_distinct_dev": (_int, [_vp, _vp, _sz, _vp]),
    "h2b_keygen_copies_dev": (_int, [_vp, _sz, _vp, _sz, _u32, _sz, _sz, _vp, _sz, _vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp]),
    "h2b_keygen_instance_edges_dev": (_int, [_vp, _sz, _vp, _sz, _u32, _sz, _sz, _sz, _sz, _vp, _vp, _vp, _vp]),
    "h2b_keygen_copies_nf_dev": (_int, [_vp, _sz, _vp, _sz, _u32, _sz, _sz, _sz, _vp, _sz, _vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp]),
    "h2b_keygen_instance_edges_nf_dev": (_int, [_vp, _sz, _vp, _sz, _u32, _sz, _sz, _sz, _sz, _sz, _vp, _vp, _vp, _vp]),
    "h2b_keygen_sigma_map_dev": (_int, [_vp, _vp, _sz, _sz, _u32, _vp]),
    "h2b_keygen_sigma_values_dev": (_int, [_vp, _vp, _sz, _u32, _vp]),
    "h2b_divide_by_vanishing_poly": (_int, [_vp, _vp, _u32, _u32]),
    "h2b_divide_by_vanishing_poly_dev": (_int, [_vp, _vp, _u32, _u32]),
    "h2b_eval_polynomial": (_int, [_vp, _vp, _sz, _vp, _vp]),
    "h2b_eval_polynomial_dev": (_int, [_vp, _vp, _sz, _vp, _vp]),
    "h2b_kate_division": (_int, [_vp, _vp, _sz, _vp, _vp]),
    "h2b_kate_division_dev": (_int, [_vp, _vp, _sz, _vp, _vp]),
    "h2b_kate_division_multi": (_int, [_vp, _vp, _sz, _vp, _sz, _vp, _vp]),
    "h2b_kate_division_multi_dev": (_int, [_vp, _vp, _sz, _vp, _sz, _vp, _vp]),
    "h2b_selector_conflicts": (_int, [_vp, _vpp, _sz, _u32, _vp]),
    "h2b_selector_conflicts_dev": (_int, [_vp, _vpp, _sz, _u32, _vp]),
    "h2b_poly_lincomb": (_int, [_vp, _vpp, _vp, _sz, _sz, _vp]),
    "h2b_poly_lincomb_dev": (_int, [_vp, _vpp, _vp, _sz, _sz, _vp]),
    "h2b_poly_alloc": (_int, [_vp, _sz, C.POINTER(_vp)]),
    "h2b_poly_free": (None, [_vp, _vp]),
    "h2b_poly_device_ptr": (_vp, [_vp]),
    "h2b_poly_len": (_sz, [_vp]),
    "h2b_poly_zero": (_int, [_vp, _vp]),
    "h2b_poly_upload_async": (_int, [_vp, _vp, _sz, _vp, _sz]),
    "h2b_poly_copy_dev": (_int, [_vp, _vp, _vp, _sz]),
    "h2b_poly_upload": (_int, [_vp, _vp, _sz, _vp, _sz]),
    "h2b_poly_download": (_int, [_vp, _vp, _sz, _vp, _sz]),
    "h2b_permutation_product_dev": (_int, [_vp, _vpp, _vpp, _sz, _sz, _vp, _vp, _u32, _u32, _vp, _vp]),
    "h2b_lookup_product_dev": (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "h2b_fr_mul_elementwise_dev": (_int, [_vp, _vp, _vp, _sz, _vp]),
    "h2b_eval_polynomial_batch_dev": (_int, [_vp, _vpp, _vp, _sz, _sz, _vp]),
    "h2b_test_field_op": (_int, [_vp, _int, _int, _vp, _vp, _sz, _vp]),
}


class Witness(C.Structure):
    """h2b::WitnessView (include/h2b200_prover.hpp): the witness of one proof or check, host pointers + counts"""
    _fields_ = [
        ("cells", _vp), ("n_cells", _sz), ("break_points", _vp), ("n_break_points", _sz),
        ("lookup_cells", _vp), ("lookup_index", _vp), ("n_lookup", _sz),
        ("rational_index", _vp), ("rational_den", _vp), ("n_rational", _sz),
        ("instance", _vp), ("n_instance", _vp), ("n_instance_columns", _sz),
    ]


class BuilderView(C.Structure):
    """h2b::BuilderView (include/h2b200_mock.hpp): a halo2-base builder in its keygen form, host pointers + counts"""
    _fields_ = [
        ("cells", _vp), ("n_cells", _sz), ("rational_index", _vp), ("rational_den", _vp), ("n_rational", _sz),
        ("selectors", _vp), ("advice_equalities", _vp), ("n_advice_equalities", _sz),
        ("constants", _vp), ("constant_index", _vp), ("n_constant_equalities", _sz), ("lookup_index", _vp), ("n_lookup", _sz),
        ("instance_index", _vp), ("instance_values", _vp), ("n_instance", _vp), ("n_instance_columns", _sz),
    ]


# callbacks of the compiled prover (first argument: the `user` pointer); 0 = success, anything else stops the proof
BLIND_FN = C.CFUNCTYPE(_int, _vp, _sz, _vp)             # (rows, out: rows x 4 limbs)
ALLREDUCE_FN = C.CFUNCTYPE(_int, _vp, _vp, _sz)         # (device pointer of the m partial commitments, m)
COMMIT_FN = C.CFUNCTYPE(_int, _vp, _int, _vp, _sz)      # (basis, host rows of the committed polynomial, n)
_witp = C.POINTER(Witness)
_u64s = C.POINTER(C.c_uint64)

PROVER_SIGNATURES = {
    "h2bp_circuit_create": (_int, [_vp, _u32, _sz, _sz, _int, _sz, _sz, C.POINTER(C.c_char_p), _vpp, _sz, _vpp, _sz, C.POINTER(_vp), _int]),
    "h2bp_circuit_free": (None, [_vp]),
    "h2bp_circuit_info": (_int, [_vp, _u64s, C.c_char_p, _sz]),
    "h2bp_circuit_column": (_int, [_vp, C.c_char_p, C.c_char_p, C.POINTER(_vp), C.POINTER(_sz), C.POINTER(_sz)]),
    "h2bp_session_create": (_int, [_vp, _vp, _u32, _sz, _vp, C.POINTER(_vp)]),
    "h2bp_session_free": (None, [_vp]),
    "h2bp_session_info": (_int, [_vp, _u64s, C.c_char_p, _sz]),
    "h2bp_session_column": (_int, [_vp, C.c_char_p, C.c_char_p, C.POINTER(_vp), C.POINTER(_sz), C.POINTER(_sz)]),
    "h2bp_session_shard": (_int, [_vp, _sz, _sz, ALLREDUCE_FN, _vp]),
    "h2bp_prove": (_int, [_vp, _witp, _vp, BLIND_FN, _vp, COMMIT_FN, _vp, _vp, _vp, _vp, _vp]),
    "h2bp_prove_halo2": (_int, [_vp, _witp, _vp, BLIND_FN, _vp, _vp, _vp, _sz, C.POINTER(_sz)]),
    "h2bp_check": (_int, [_vp, _witp, _sz, _vp]),
    "h2bp_mock_create": (_int, [_vp, _u32, _sz, _sz, _int, _u32, _sz, _sz, _sz, C.POINTER(_vp), _u64s]),
    "h2bp_mock_free": (None, [_vp]),
    "h2bp_mock_column": (_int, [_vp, C.c_char_p, C.POINTER(_vp), C.POINTER(_sz), C.POINTER(_sz)]),
    "h2bp_mock_run": (_int, [_vp, C.POINTER(BuilderView), _sz, _vp, _u64s, _vp, _vp, _u64s]),
    "h2bp_keygen": (_int, [_vp, _vp, _u32, _sz, _sz, _sz, _int, _u32, _sz, _sz, C.POINTER(BuilderView), C.POINTER(_vp), _vp, _u64s, _vp, _vp, _int]),
}


def header_symbols() -> list[str]:
    """Function names declared in include/h2b200.h (used by the CPU test that every symbol is exported)."""
    txt = open(HEADER_PATH).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(h2b_[a-z0-9_]+)\s*\(", txt)))


def load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in {**SIGNATURES, **PROVER_SIGNATURES}.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


lib = load()
