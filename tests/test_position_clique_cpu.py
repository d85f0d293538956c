"""Position (clique) and acceleration control spaces without a GPU:
  * properties of the oracle (oracle/clique_oracle.py) the reference's arithmetic must have;
  * the backend launchers' signatures against the reference's (tests/golden/reference_legacy_trajectory_signatures.json);
  * argument errors raised before any launch;
  * the kernels, the host mirrors, RolloutEngine.evaluate_positions and the position_clique Rollout on the emulated device of
    test_emulated_gpu_suite_cpu.py (the test functions of tests/test_gpu_position_clique.py at small sizes)."""
import inspect
import json
import os

import numpy as np
import pytest
import torch

from clique_cases import make_case
from oracle import clique_oracle as co
from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)

HERE = os.path.dirname(os.path.abspath(__file__))
F64 = np.float64


def _fwd64(c, u, implicit=None):
    imp = c["implicit"] if implicit is None else implicit
    return co.clique_forward(u, *c["start"], c["goal"][0], c["start_idx"], c["goal_idx"], c["traj_dt"], imp, c["H"], dtype=F64)


# ------------------------------------------------------------------------------------------------ oracle properties
def test_constant_positions_with_matching_start_have_zero_derivatives():
    c = make_case(seed=1, B=4, H=14, D=7, n_start=4, n_goal=4, implicit="mixed")
    q = np.random.default_rng(0).normal(size=(4, 7)).astype(np.float32)
    c["start"] = (q, np.zeros_like(q), np.zeros_like(q))
    c["start_idx"] = np.arange(4, dtype=np.int32)
    c["goal"] = (q.copy(), np.zeros_like(q), np.zeros_like(q))
    c["goal_idx"] = np.arange(4, dtype=np.int32)
    u = np.repeat(q[:, None], c["n"], axis=1)
    for dtype in (np.float32, F64):
        p, v, a, j, _ = co.clique_forward(u, *c["start"], c["goal"][0], c["start_idx"], c["goal_idx"], c["traj_dt"],
                                          c["implicit"], c["H"], dtype=dtype)
        np.testing.assert_array_equal(p, np.repeat(q[:, None], c["H"], axis=1).astype(dtype))
        dt = c["traj_dt"][c["goal_idx"]][:, None, None]
        tol = 1e-6 if dtype == np.float32 else 1e-14
        assert (np.abs(v) * dt <= tol * 4).all() and (np.abs(a) * dt ** 2 <= tol * 8).all() and (np.abs(j) * dt ** 3 <= tol * 4).all()


def test_linear_ramp_has_constant_velocity_and_zero_interior_acceleration_and_jerk():
    B, H, D = 3, 20, 5
    c = make_case(seed=2, B=B, H=H, D=D, n_start=B, n_goal=B, implicit=False)
    rng = np.random.default_rng(3)
    x0, r = rng.normal(size=(B, D)), rng.normal(size=(B, D))
    c["start_idx"] = c["goal_idx"] = np.arange(B, dtype=np.int32)
    dt = c["traj_dt"].astype(F64)[:, None]
    x = lambda w: x0 + r * w * dt  # noqa: E731  waypoint w of the ramp
    c["start"] = (x(1), r, np.zeros((B, D)))
    u = np.stack([x(i + 2) for i in range(H - 4)], axis=1)
    p, v, a, j, _ = co.clique_forward(u, *c["start"], c["goal"][0], c["start_idx"], c["goal_idx"], c["traj_dt"], c["implicit"], H,
                                      dtype=F64)
    rows = slice(0, H - 4)                 # rows whose five stencil waypoints all lie on the ramp
    np.testing.assert_allclose(p[:, rows], np.stack([x(h) for h in range(H - 4)], axis=1), atol=1e-12)
    np.testing.assert_allclose(v[:, rows], np.repeat(r[:, None], H - 4, axis=1), rtol=1e-8, atol=1e-8)
    assert np.abs(a[:, rows]).max() < 1e-6 and np.abs(j[:, rows]).max() < 1e-4


def test_integrator_matches_constant_acceleration_closed_form():
    B, H, D = 3, 25, 4
    rng = np.random.default_rng(4)
    p0, v0, acc = (rng.normal(size=(B, D)) for _ in range(3))
    dt = 0.03
    u = np.repeat(acc[:, None], H, axis=1)
    p, v, a, j = co.integrate_acceleration(u, p0, v0, acc, np.arange(B), np.full(H, dt), dtype=F64)
    h = np.arange(H, dtype=F64)[None, :, None]
    np.testing.assert_allclose(v, v0[:, None] + acc[:, None] * h * dt, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(p, p0[:, None] + v0[:, None] * h * dt + acc[:, None] * dt * dt * h * (h + 1) / 2, rtol=1e-12,
                               atol=1e-12)
    np.testing.assert_allclose(a, u, atol=0)
    assert np.abs(j).max() < 1e-9


def _transpose64(c, implicit):
    """Exact J^T g of the float64 forward (an affine map of u), column by column."""
    B, n, D = c["u"].shape
    base = _fwd64(c, np.zeros((B, n, D)), implicit)
    out = np.zeros((B, n, D))
    for i in range(n):
        for d in range(D):
            e = np.zeros((B, n, D))
            e[:, i, d] = 1.0
            col = _fwd64(c, e, implicit)
            out[:, i, d] = sum(((col[k] - base[k]) * c["grads"][k].astype(F64)).sum(axis=(1, 2)) for k in range(4))
    return out


@pytest.mark.parametrize("H", [9, 10, 14, 30])
@pytest.mark.parametrize("implicit", [False, True])
def test_backward_is_the_transpose_of_the_forward(H, implicit):
    c = make_case(seed=10 + H, B=3, H=H, D=3, implicit=implicit)
    want = _transpose64(c, c["implicit"])
    got = co.clique_backward(*c["grads"], c["traj_dt"], c["goal_idx"], c["implicit"], dtype=F64)
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-9 * np.abs(want).max())


def test_h8_implicit_goal_differs_from_the_transpose_at_row3_last_action_only():
    """At H = 8 the forward's row 3 takes the `h == 3` branch before `h == H-5`, so with the implicit goal it reads the raw last
    action where the adjoint treats it as replaced by the goal: the adjoint lacks exactly row 3's stencil weight on it."""
    c = make_case(seed=8, B=3, H=8, D=3, implicit=True)
    want = _transpose64(c, c["implicit"])
    got = co.clique_backward(*c["grads"], c["traj_dt"], c["goal_idx"], c["implicit"], dtype=F64)
    np.testing.assert_allclose(got[:, :3], want[:, :3], rtol=1e-9, atol=1e-9 * np.abs(want).max())
    assert np.all(got[:, 3] == 0.0)
    dti = 1.0 / c["traj_dt"][c["goal_idx"]].astype(F64)[:, None]
    gv, ga, gj = (g[:, 3].astype(F64) for g in c["grads"][1:])
    row3 = -0.083333333 * gv * dti - 0.083333333 * ga * dti ** 2 + 0.5 * gj * dti ** 3
    np.testing.assert_allclose(want[:, 3], row3, rtol=1e-9, atol=1e-9 * np.abs(row3).max())
    # without the implicit goal H = 8 is an exact transpose too
    c = make_case(seed=8, B=3, H=8, D=3, implicit=False)
    np.testing.assert_allclose(co.clique_backward(*c["grads"], c["traj_dt"], c["goal_idx"], c["implicit"], dtype=F64),
                               _transpose64(c, c["implicit"]), rtol=1e-9, atol=1e-9)


# ------------------------------------------------------------------------------------------------ backend boundary
SIGS = json.load(open(os.path.join(HERE, "golden", "reference_legacy_trajectory_signatures.json")))


@pytest.mark.parametrize("key", sorted(SIGS))
def test_launcher_signature_matches_the_reference(key):
    from curobo_b200.backends import trajectory
    mod, name = key.split(".")
    params = inspect.signature(getattr(trajectory, name)).parameters
    assert list(params) == SIGS[key]["params"], f"{key} ({SIGS[key]['file']}:{SIGS[key]['line']})"
    assert {k: repr(p.default) for k, p in params.items() if p.default is not inspect.Parameter.empty} == SIGS[key]["defaults"]


def test_backend_argument_errors_before_launch():
    from curobo_b200.backends import trajectory as trajectory_cu
    z = lambda *s: torch.zeros(s)  # noqa: E731
    i = torch.zeros(2, dtype=torch.int32)
    imp = torch.zeros(2, dtype=torch.uint8)
    with pytest.raises(ValueError, match="horizon >= 8"):
        trajectory_cu.launch_differentiation_position_forward_kernel(*[z(2, 7, 3)] * 4, z(2), z(2, 3, 3), *[z(2, 3)] * 6, i, i,
                                                                     z(2), imp, 2, 7, 3)
    with pytest.raises(ValueError, match="horizon >= 8"):
        trajectory_cu.launch_differentiation_position_backward_kernel(z(2, 1, 3), *[z(2, 5, 3)] * 4, z(2), i, imp, 2, 5, 3)
    with pytest.raises(ValueError, match="CUDA-only"):      # no CPU path
        trajectory_cu.launch_differentiation_position_forward_kernel(*[z(2, 9, 3)] * 4, z(2), z(2, 5, 3), *[z(2, 3)] * 6, i, i,
                                                                     z(2), imp, 2, 9, 3)
    with pytest.raises(ValueError, match="CUDA-only"):
        trajectory_cu.launch_integration_acceleration_kernel(*[z(2, 9, 3)] * 5, *[z(2, 3)] * 3, i, z(9), 2, 9, 3)


# ------------------------------------------------------------------------------------------------ emulated device
@pytest.mark.parametrize("kw", [dict(seed=1, B=5, H=8, D=7, implicit="mixed"), dict(seed=3, B=7, H=9, D=7, implicit="mixed"),
                                dict(seed=5, B=3, H=14, D=35, implicit="mixed"), dict(seed=7, B=2, H=34, D=7, implicit=True)])
def test_kernels_emulated(run, kw):  # noqa: F811
    run("test_gpu_position_clique", "test_clique_forward_vs_oracle_and_reference", kw)
    run("test_gpu_position_clique", "test_clique_backward_vs_oracle_and_reference", kw)
    run("test_gpu_position_clique", "test_acceleration_integration_vs_oracle_and_reference", kw)


def test_errors_and_state_transitions_emulated(run):  # noqa: F811
    run("test_gpu_position_clique", "test_error_behaviour")
    run("test_gpu_position_clique", "test_state_transitions", False)
    run("test_gpu_position_clique", "test_state_transitions", True)


def test_evaluate_positions_emulated(run):  # noqa: F811
    run("test_gpu_position_clique", "test_evaluate_positions_vs_composition_and_oracle_chain", "trajopt_swept", 2, 9)
    run("test_gpu_position_clique", "test_rollout_protocol_position_clique", 2, 9)
