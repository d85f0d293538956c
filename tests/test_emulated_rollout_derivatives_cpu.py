"""The derivative tests of the fused rollout (tests/test_gpu_rollout_derivatives.py) on the emulated device of
test_emulated_gpu_suite_cpu.py: every case and kernel family, the gradient against float64 central differences of the oracle's
cost.  The batch larger than the persistent grid is sized from the emulated device's two SMs."""
import pytest

from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)

import test_gpu_rollout_derivatives as g


@pytest.mark.parametrize("name,family", g.RUNS)
def test_gradient_is_derivative_of_cost_emulated(run, monkeypatch, name, family):  # noqa: F811
    run("test_gpu_rollout_derivatives", "test_gradient_is_derivative_of_cost", monkeypatch, name, family)


@pytest.mark.parametrize("name,family", g.AXIS_ANGLE_RUNS)
def test_axis_angle_gradient_is_half_the_derivative_emulated(run, monkeypatch, name, family):  # noqa: F811
    run("test_gpu_rollout_derivatives", "test_axis_angle_gradient_is_half_the_derivative", monkeypatch, name, family)
