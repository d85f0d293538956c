"""The velocity-aware IK GPU tests (tests/test_gpu_velocity_ik.py) on the emulated device of test_emulated_gpu_suite_cpu.py, at
small sizes: the per-operator kernel and every fused family against the reference-source golden, fused equals composed with self,
scene and pose terms active, the edge cases and the refusal.  CUDA-graph replay and the L-BFGS solves need a real GPU and are
not re-run."""
import pytest

from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)

import test_gpu_velocity_ik as g


@pytest.mark.parametrize("case", g.GOLDEN_CASES)
def test_per_operator_golden_emulated(run, case):  # noqa: F811
    run("test_gpu_velocity_ik", "test_per_operator_kernel_matches_reference_source", case)


@pytest.mark.parametrize("variant", ["arm", "pairs", "big", "traj", "cost_arm", "cost_big"])
@pytest.mark.parametrize("case", ["vel_acc", "mixed_dt", "empty_window", "with_target"])
def test_fused_golden_emulated(run, monkeypatch, case, variant):  # noqa: F811
    run("test_gpu_velocity_ik", "test_fused_kernels_match_reference_source", monkeypatch, case, variant)


@pytest.mark.parametrize("robot,variant,kind,n,H", [("franka", "arm", "cuboid", 12, 1), ("franka", "pairs", "cuboid", 13, 1),
                                                    ("franka", "arm", "esdf", 10, 1), ("g1_29", "standard", "cuboid", 6, 1),
                                                    ("g1_29", "big", "esdf", 6, 1),
                                                    ("franka", "traj", "cuboid", 4, 4)])
def test_fused_equals_composed_emulated(run, monkeypatch, robot, variant, kind, n, H):  # noqa: F811
    run("test_gpu_velocity_ik", "test_fused_equals_composed", monkeypatch, robot, variant, kind, n, H)


@pytest.mark.parametrize("edge", ["empty_window", "no_velocity", "many_rows", "multi_env"])
def test_edge_cases_emulated(run, monkeypatch, edge):  # noqa: F811
    run("test_gpu_velocity_ik", "test_edge_cases", monkeypatch, edge)


def test_refusal_emulated(run):  # noqa: F811
    run("test_gpu_velocity_ik", "test_null_fields_and_refusal")


def test_update_params_current_js_emulated(run):  # noqa: F811
    run("test_gpu_velocity_ik", "test_robot_rollout_update_params_current_js")
