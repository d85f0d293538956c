"""The trajectory-gradient derivative tests (tests/test_gpu_trajectory_derivatives.py) on the emulated device of
test_emulated_gpu_suite_cpu.py: every run, at the same sizes, against float64 central differences of the composed cost."""
import pytest

from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)

import test_gpu_trajectory_derivatives as g


@pytest.mark.parametrize("name,family", g.STATE_RUNS)
def test_state_gradients_are_derivatives_emulated(run, monkeypatch, name, family):  # noqa: F811
    run("test_gpu_trajectory_derivatives", "test_state_gradients_are_derivatives", monkeypatch, name, family)


@pytest.mark.parametrize("name,family", g.KNOTS_RUNS)
def test_knots_gradient_is_derivative_emulated(run, monkeypatch, name, family):  # noqa: F811
    run("test_gpu_trajectory_derivatives", "test_knots_gradient_is_derivative", monkeypatch, name, family)


@pytest.mark.parametrize("name,family", g.CLIQUE_RUNS)
def test_position_clique_gradient_is_derivative_emulated(run, monkeypatch, name, family):  # noqa: F811
    run("test_gpu_trajectory_derivatives", "test_position_clique_gradient_is_derivative", monkeypatch, name, family)


@pytest.mark.parametrize("name,family", g.DYNAMICS_RUNS)
def test_dynamics_aware_gradients_are_derivatives_emulated(run, monkeypatch, name, family):  # noqa: F811
    run("test_gpu_trajectory_derivatives", "test_dynamics_aware_gradients_are_derivatives", monkeypatch, name, family)


@pytest.mark.parametrize("name,family", g.PROTOCOL_RUNS)
def test_protocol_autograd_gradient_is_derivative_emulated(run, monkeypatch, name, family):  # noqa: F811
    run("test_gpu_trajectory_derivatives", "test_protocol_autograd_gradient_is_derivative", monkeypatch, name, family)
