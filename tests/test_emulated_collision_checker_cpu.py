"""Validity rows (tests/test_gpu_collision_checker.py) on the emulated device of test_emulated_gpu_suite_cpu.py, at small sizes:
the float64 oracle, the single-check masks against the cost kernels, and early exit against static striding and a buried
robot."""
import pytest

from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)


@pytest.mark.parametrize("robot,kind,n", [("franka", "cuboid", 48), ("franka", "esdf", 32), ("franka", "mesh", 12),
                                          ("g1_29", "esdf", 6), ("g1_43", "esdf", 4)])
def test_validate_vs_float64_oracle_emulated(run, robot, kind, n):  # noqa: F811
    run("test_gpu_collision_checker", "test_validate_vs_float64_oracle", robot, kind, n)


def test_validate_environments_and_link_spheres_emulated(run):  # noqa: F811
    run("test_gpu_collision_checker", "test_validate_two_environments_and_sphere_configurations", 40)
    run("test_gpu_collision_checker", "test_validate_attached_object_and_disabled_link", 48)


@pytest.mark.parametrize("robot,kind,n", [("franka", "cuboid", 40), ("franka", "esdf", 24), ("franka", "mesh", 12),
                                          ("g1_29", "esdf", 8), ("g1_43", "esdf", 4), ("franka", "two_env", 24)])
def test_single_checks_equal_cost_kernels_emulated(run, robot, kind, n):  # noqa: F811
    run("test_gpu_collision_checker", "test_single_checks_equal_cost_kernels", robot, kind, n)


@pytest.mark.parametrize("robot,kind,n", [("franka", "cuboid", 64), ("franka", "buried", 48)])
def test_early_exit_changes_nothing_emulated(run, monkeypatch, robot, kind, n):  # noqa: F811
    run("test_gpu_collision_checker", "test_early_exit_changes_nothing", monkeypatch, robot, kind, n)


def test_checker_api_emulated(run):  # noqa: F811
    run("test_gpu_collision_checker", "test_abi_refusals")
    run("test_gpu_collision_checker", "test_distance_methods_equal_composition_and_oracle", 64)
