"""The cost-only fused rollout (tests/test_gpu_cost_only.py) on the emulated device of test_emulated_gpu_suite_cpu.py, at small
sizes: every kernel variant against the gradient launch (also without a link-pair list), multi-environment rows, the refusals
and the B200RobotRollout routing."""
import pytest

from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)


@pytest.mark.parametrize("robot,variant,kind,n", [("franka", "arm", "cuboid", 20), ("franka", "pairs", "cuboid", 21),
                                                   ("franka", "standard", "mesh", 12), ("franka", "big", "esdf", 10),
                                                   ("franka", "team", "esdf", 6), ("g1_29", "standard", "cuboid", 16),
                                                   ("g1_29", "team", "esdf", 4), ("g1_43", "big", "all", 3),
                                                   ("franka-pairlist", "pairs", "cuboid", 21),
                                                   ("g1_29-pairlist", "standard", "cuboid", 16)])
def test_cost_only_equals_gradient_launch_emulated(run, monkeypatch, robot, variant, kind, n):  # noqa: F811
    run("test_gpu_cost_only", "test_cost_only_equals_gradient_launch", monkeypatch, robot, variant, kind, n)


def test_cost_only_misc_emulated(run, monkeypatch):  # noqa: F811
    run("test_gpu_cost_only", "test_cost_only_multi_env_and_cost_without_terms", monkeypatch, "arm")
    run("test_gpu_cost_only", "test_cost_only_refusals")
    run("test_gpu_cost_only", "test_robot_rollout_takes_cost_only_without_grad")
