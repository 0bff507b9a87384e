"""Dry run of GPU test bodies on the CPU: the CUDA engine is replaced by the oracle-backed stand-in of
tests/oracle_engine.py and the functions of tests/test_gpu_parity.py, tests/test_gpu_float32.py and
tests/test_gpu_scale_edges.py, tests/test_gpu_infeasibility.py, tests/test_gpu_projection_jacobian.py and
tests/test_gpu_ruiz.py and tests/test_gpu_anderson.py are called directly.  What this checks is the
Python side of those tests (imports, helpers, fixtures, the host glue they drive) -- a NameError in a GPU test would
otherwise only show up on the next GPU run.  Assertion failures are tolerated where the stand-in legitimately differs
from the engine (it ignores the D/E unscaling of the termination test); every other exception fails the test."""
import importlib
import inspect

import pytest

from cosmo_b200 import engine as E, model as M
from tests.oracle_engine import OracleEngine

CASES = ["test_engine_matches_committed_golden_iterates", "test_g6_chordal_sdp_through_the_clique_batch",
         "test_g4_g5_g11_literal_problems", "test_g15_g16_exp_pow_cone_problems", "test_project_exp_pow_cones",
         "test_accelerated_iterates_match_oracle", "test_accelerator_rho_adaption_limits", "test_g1_simple_qp",
         "test_g2_box_statuses", "test_g3_hs21_with_soc_and_merging", "test_g14_model_updates_and_warm_start",
         "test_project_composite_matches_oracle", "test_soc_branches", "test_complex_psd_cone_projection_and_least_eigenvalue",
         "test_project_psd_tensor_core_path_n150",
         "test_gpu_float32::test_clamp_cones_bit_exact_float32", "test_gpu_float32::test_soc_float32",
         "test_gpu_float32::test_project_exp_pow_cones_float32", "test_gpu_float32::test_project_psd_small_batch_float32",
         "test_gpu_float32::test_project_psd_tensor_core_path_float32_kinds", "test_gpu_float32::test_complex_psd_float32",
         "test_gpu_float32::test_g1_float32", "test_gpu_float32::test_g2_statuses_float32",
         "test_gpu_float32::test_g15_g16_float32", "test_gpu_float32::test_g14_model_updates_float32",
         "test_gpu_float32::test_closest_correlation_float32",
         "test_gpu_scale_edges::test_homogeneity_ladder", "test_gpu_scale_edges::test_mixed_large_cone_shapes_share_the_workspace",
         "test_gpu_scale_edges::test_small_kernel_tensor_core_boundary",
         "test_gpu_infeasibility::test_gate_quantities_match_the_reference",
         "test_gpu_infeasibility::test_gates_reached_on_either_side_pin_E_D_and_c",
         "test_gpu_infeasibility::test_rows_at_the_tolerance_edge",
         "test_gpu_infeasibility::test_soc_exact_boundary_points_are_certified",
         "test_gpu_infeasibility::test_psd_verdicts_at_the_tolerance",
         "test_gpu_infeasibility::test_nonsymmetric_square_psd_certificate_reads_the_upper_triangle",
         "test_gpu_infeasibility::test_exp_pow_verdicts_near_the_boundary",
         "test_gpu_infeasibility::test_composite_bitmask_names_exactly_the_failing_family",
         "test_gpu_infeasibility::test_soc_margins_dimensions_and_scale",
         "test_gpu_infeasibility::test_psd_lambda_max_small_and_large_paths",
         "test_gpu_infeasibility::test_psd_lambda_max_homogeneity_ladder",
         "test_gpu_infeasibility::test_unconverged_eigensolver_is_not_certified",
         "test_gpu_infeasibility::test_reference_infeasible_problems_status_and_iterations",
         "test_gpu_infeasibility::test_reference_infeasible_problems_float32",
         "test_gpu_projection_jacobian::test_psd_size_and_spectrum_sweep",
         "test_gpu_projection_jacobian::test_psd_sweep_float32", "test_gpu_projection_jacobian::test_soc_sweep",
         "test_gpu_projection_jacobian::test_rows_bit_exact", "test_gpu_projection_jacobian::test_properties_per_path",
         "test_gpu_projection_jacobian::test_scale_ladder", "test_gpu_projection_jacobian::test_path_boundary_96_97",
         "test_gpu_projection_jacobian::test_kink_counts",
         "test_gpu_ruiz::test_clip_edges_at_the_first_pass", "test_gpu_ruiz::test_zero_rows_and_columns_keep_the_scale_one",
         "test_gpu_ruiz::test_cost_scaling_guard", "test_gpu_ruiz::test_dynamic_range_clips_in_every_pass",
         "test_gpu_ruiz::test_every_rectified_family", "test_gpu_ruiz::test_box_bounds_and_row_classes",
         "test_gpu_ruiz::test_long_rows_and_n_above_1024", "test_gpu_ruiz::test_wide_qp_slabs_hold_the_scaled_values",
         "test_gpu_ruiz::test_scaled_P_is_symmetric", "test_gpu_ruiz::test_update_matrices_reproduces_a_fresh_engine",
         "test_gpu_anderson::test_windows_and_dimensions", "test_gpu_anderson::test_prescribed_condition",
         "test_gpu_anderson::test_grid_stride_wrap", "test_gpu_anderson::test_min_mem_above_the_window",
         "test_gpu_anderson::test_exact_duplicate_differences", "test_gpu_anderson::test_eta_norm_rule",
         "test_gpu_anderson::test_non_finite_inputs", "test_gpu_anderson::test_pivot_ties_of_opposite_sign",
         "test_gpu_anderson::test_safeguard_norms_over_the_whole_range",
         "test_gpu_anderson::test_overflowing_squares_never_accept_non_finite",
         "test_gpu_anderson::test_power_of_two_ladder_and_determinism",
         "test_gpu_anderson::test_probe_leaves_the_solve_state_untouched", "test_gpu_anderson::test_report_worst_ratios"]
MUST_PASS = {"test_engine_matches_committed_golden_iterates", "test_g6_chordal_sdp_through_the_clique_batch",
             "test_project_exp_pow_cones", "test_soc_branches", "test_complex_psd_cone_projection_and_least_eigenvalue",
             "test_gpu_float32::test_clamp_cones_bit_exact_float32", "test_gpu_float32::test_project_psd_small_batch_float32",
             "test_gpu_infeasibility::test_gate_quantities_match_the_reference",
             "test_gpu_infeasibility::test_gates_reached_on_either_side_pin_E_D_and_c",
             "test_gpu_infeasibility::test_rows_at_the_tolerance_edge",
             "test_gpu_infeasibility::test_soc_exact_boundary_points_are_certified",
             "test_gpu_infeasibility::test_composite_bitmask_names_exactly_the_failing_family",
             "test_gpu_projection_jacobian::test_psd_size_and_spectrum_sweep",
             "test_gpu_projection_jacobian::test_soc_sweep", "test_gpu_projection_jacobian::test_rows_bit_exact",
             "test_gpu_projection_jacobian::test_kink_counts",
             "test_gpu_ruiz::test_clip_edges_at_the_first_pass", "test_gpu_ruiz::test_zero_rows_and_columns_keep_the_scale_one",
             "test_gpu_ruiz::test_cost_scaling_guard", "test_gpu_ruiz::test_scaled_P_is_symmetric",
             "test_gpu_ruiz::test_every_rectified_family",
             "test_gpu_ruiz::test_update_matrices_reproduces_a_fresh_engine",
             "test_gpu_anderson::test_windows_and_dimensions", "test_gpu_anderson::test_min_mem_above_the_window",
             "test_gpu_anderson::test_exact_duplicate_differences", "test_gpu_anderson::test_eta_norm_rule",
             "test_gpu_anderson::test_non_finite_inputs", "test_gpu_anderson::test_pivot_ties_of_opposite_sign"}


def _calls(fn):
    """argument tuples of a (possibly multiply) parametrized test function: first value of every parameter"""
    marks = [m for m in getattr(fn, "pytestmark", []) if m.name == "parametrize"]
    kwargs = {}
    for m in marks:
        names = [a.strip() for a in m.args[0].split(",")]
        first = m.args[1][0]
        first = first if isinstance(first, (tuple, list)) and len(names) > 1 else (first,)
        kwargs.update(dict(zip(names, first)))
    return kwargs


@pytest.mark.parametrize("name", CASES)
def test_gpu_test_body_runs_against_the_oracle_stand_in(name, monkeypatch):
    monkeypatch.setattr(M._eng, "Engine", OracleEngine)
    monkeypatch.setattr(E, "Engine", OracleEngine)
    module, _, func = name.rpartition("::")      # "module::test" for the other GPU modules, a bare name for the parity module
    T = importlib.import_module("tests." + (module or "test_gpu_parity"))
    fn = getattr(T, func)
    kwargs = _calls(fn)
    if "monkeypatch" in inspect.signature(fn).parameters:
        kwargs["monkeypatch"] = monkeypatch
    try:
        fn(**kwargs)
    except AssertionError:
        if name in MUST_PASS:
            raise
