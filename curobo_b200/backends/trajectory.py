"""`trajectory` kernel-backend module: same function names and argument order as
curobo/_src/curobolib/backends/cuda_core_backend/trajectory.py:25-560 (pybind twin:
backends/pybind/trajectory_kernel_launch.cu:26-683), for the three B-spline launches the trajopt / MPC path
uses (SURVEY.md section 8f rank 1) and the three legacy launches of the POSITION (clique) and ACCELERATION control
spaces.  Tensors are validated like the reference's cuda_ops/trajectory.py:334-357
(device, contiguity, dtype) BEFORE launch; errors raise.  Launches go to `torch.cuda.current_stream()`.
"""
from __future__ import annotations

import torch

from .. import lib as _lib
from .tensor_checks import check_tensors, stream_ptr


def _check_degree(bspline_degree: int) -> None:
    if bspline_degree not in (3, 4, 5):
        # trajectory_kernel_launch.cu:562,614
        raise RuntimeError(f"Unsupported B-spline degree: {bspline_degree}")


def launch_bspline_interpolation_forward_kernel(
    out_position: torch.Tensor,
    out_velocity: torch.Tensor,
    out_acceleration: torch.Tensor,
    out_jerk: torch.Tensor,
    out_dt: torch.Tensor,
    u_position: torch.Tensor,
    start_position: torch.Tensor,
    start_velocity: torch.Tensor,
    start_acceleration: torch.Tensor,
    start_jerk: torch.Tensor,
    goal_position: torch.Tensor,
    goal_velocity: torch.Tensor,
    goal_acceleration: torch.Tensor,
    goal_jerk: torch.Tensor,
    start_idx: torch.Tensor,
    goal_idx: torch.Tensor,
    traj_dt: torch.Tensor,
    use_implicit_goal_state: torch.Tensor,
    batch_size: int,
    horizon: int,
    dof: int,
    n_knots: int,
    bspline_degree: int,
) -> None:
    """u_position = knots [B,n_knots,D] -> position / velocity / acceleration / jerk [B,horizon,D] (in place); `horizon` is the
    padded horizon.  Parameter names are the reference's (cuda_core_backend/trajectory.py:28-52)."""
    _check_degree(bspline_degree)
    dev = u_position.device
    check_tensors(dev, torch.float32, out_position=out_position, out_velocity=out_velocity,
                  out_acceleration=out_acceleration, out_jerk=out_jerk, out_dt=out_dt, u_position=u_position,
                  start_position=start_position, start_velocity=start_velocity, start_acceleration=start_acceleration,
                  start_jerk=start_jerk, goal_position=goal_position, goal_velocity=goal_velocity,
                  goal_acceleration=goal_acceleration, goal_jerk=goal_jerk, traj_dt=traj_dt)
    check_tensors(dev, torch.int32, start_idx=start_idx, goal_idx=goal_idx)
    check_tensors(dev, torch.uint8, use_implicit_goal_state=use_implicit_goal_state)
    L = _lib.load()
    err = L.cb200_bspline_forward(
        out_position.data_ptr(), out_velocity.data_ptr(), out_acceleration.data_ptr(), out_jerk.data_ptr(),
        out_dt.data_ptr(), u_position.data_ptr(), start_position.data_ptr(), start_velocity.data_ptr(),
        start_acceleration.data_ptr(), start_jerk.data_ptr(), goal_position.data_ptr(), goal_velocity.data_ptr(),
        goal_acceleration.data_ptr(), goal_jerk.data_ptr(), start_idx.data_ptr(), goal_idx.data_ptr(),
        traj_dt.data_ptr(), use_implicit_goal_state.data_ptr(), int(batch_size), int(horizon), int(dof),
        int(n_knots), int(bspline_degree), stream_ptr(dev))
    _lib.check(err, "launch_bspline_interpolation_forward_kernel")


def launch_bspline_interpolation_single_dt_kernel(
    out_position: torch.Tensor,
    out_velocity: torch.Tensor,
    out_acceleration: torch.Tensor,
    out_jerk: torch.Tensor,
    out_dt: torch.Tensor,
    knots: torch.Tensor,
    knot_dt: torch.Tensor,
    start_position: torch.Tensor,
    start_velocity: torch.Tensor,
    start_acceleration: torch.Tensor,
    start_jerk: torch.Tensor,
    goal_position: torch.Tensor,
    goal_velocity: torch.Tensor,
    goal_acceleration: torch.Tensor,
    goal_jerk: torch.Tensor,
    start_idx: torch.Tensor,
    goal_idx: torch.Tensor,
    interpolation_dt: torch.Tensor,
    use_implicit_goal_state: torch.Tensor,
    interpolation_horizon: torch.Tensor,
    batch_size: int,
    max_out_tsteps: int,
    dof: int,
    n_knots: int,
    bspline_degree: int,
) -> None:
    """Re-sample every trajectory at one common dt with its own horizon (final-trajectory interpolation)."""
    _check_degree(bspline_degree)
    dev = knots.device
    check_tensors(dev, torch.float32, out_position=out_position, out_velocity=out_velocity,
                  out_acceleration=out_acceleration, out_jerk=out_jerk, out_dt=out_dt, knots=knots,
                  start_position=start_position, start_velocity=start_velocity, start_acceleration=start_acceleration,
                  start_jerk=start_jerk, goal_position=goal_position, goal_velocity=goal_velocity,
                  goal_acceleration=goal_acceleration, goal_jerk=goal_jerk, interpolation_dt=interpolation_dt)
    check_tensors(dev, torch.int32, start_idx=start_idx, goal_idx=goal_idx, interpolation_horizon=interpolation_horizon)
    check_tensors(dev, torch.uint8, use_implicit_goal_state=use_implicit_goal_state)
    L = _lib.load()
    err = L.cb200_bspline_single_dt(
        out_position.data_ptr(), out_velocity.data_ptr(), out_acceleration.data_ptr(), out_jerk.data_ptr(),
        out_dt.data_ptr(), knots.data_ptr(), knot_dt.data_ptr() if knot_dt is not None else None,
        start_position.data_ptr(), start_velocity.data_ptr(), start_acceleration.data_ptr(), start_jerk.data_ptr(),
        goal_position.data_ptr(), goal_velocity.data_ptr(), goal_acceleration.data_ptr(), goal_jerk.data_ptr(),
        start_idx.data_ptr(), goal_idx.data_ptr(), interpolation_dt.data_ptr(), use_implicit_goal_state.data_ptr(),
        interpolation_horizon.data_ptr(), int(batch_size), int(max_out_tsteps), int(dof), int(n_knots),
        int(bspline_degree), stream_ptr(dev))
    _lib.check(err, "launch_bspline_interpolation_single_dt_kernel")


def launch_bspline_interpolation_backward_kernel(
    out_grad_position: torch.Tensor,
    grad_position: torch.Tensor,
    grad_velocity: torch.Tensor,
    grad_acceleration: torch.Tensor,
    grad_jerk: torch.Tensor,
    traj_dt: torch.Tensor,
    dt_idx: torch.Tensor,
    use_implicit_goal_state: torch.Tensor,
    batch_size: int,
    padded_horizon: int,
    dof: int,
    n_knots: int,
    bspline_degree: int,
    use_direct_polynomial: bool = False,
) -> None:
    """Adjoint: the four row gradients [B,padded_horizon,D] -> out_grad_position [B,n_knots,D] (overwritten)."""
    _check_degree(bspline_degree)
    horizon = padded_horizon - 1
    if horizon < 5:
        raise RuntimeError("horizon must be greater than 5")  # trajectory_kernel_launch.cu:594-597
    steps = horizon // (n_knots + bspline_degree + 1)
    if steps <= 0:
        raise RuntimeError(f"interpolation_steps is 0: horizon ({horizon}) too small for n_knots ({n_knots}) "
                           f"and degree ({bspline_degree})")  # :617-621
    if steps > 32:
        raise RuntimeError("interpolation_steps > 32 is not supported")  # :623-625
    dev = grad_position.device
    check_tensors(dev, torch.float32, out_grad_position=out_grad_position, grad_position=grad_position,
                  grad_velocity=grad_velocity, grad_acceleration=grad_acceleration, grad_jerk=grad_jerk, traj_dt=traj_dt)
    check_tensors(dev, torch.int32, dt_idx=dt_idx)
    check_tensors(dev, torch.uint8, use_implicit_goal_state=use_implicit_goal_state)
    L = _lib.load()
    err = L.cb200_bspline_backward(
        out_grad_position.data_ptr(), grad_position.data_ptr(), grad_velocity.data_ptr(), grad_acceleration.data_ptr(),
        grad_jerk.data_ptr(), traj_dt.data_ptr(), dt_idx.data_ptr(), use_implicit_goal_state.data_ptr(), int(batch_size),
        int(padded_horizon), int(dof), int(n_knots), int(bspline_degree), stream_ptr(dev))
    _lib.check(err, "launch_bspline_interpolation_backward_kernel")


# ------------------------------------------------------------------------------------------------
# position (clique) and acceleration control spaces: cuda_core_backend/trajectory.py:309-560
# ------------------------------------------------------------------------------------------------
def _check_clique_horizon(horizon: int) -> None:
    if horizon < 8:
        # the reference's first four rows read actions 0..3 whatever the horizon: below 8 that is past the row's actions
        raise ValueError(f"position clique needs horizon >= 8 (horizon - 4 >= 4 actions), got {horizon}")


def _check_rows(what: str, rows: int, **tensors: torch.Tensor) -> None:
    for name, t in tensors.items():
        if t.numel() < rows:
            raise ValueError(f"{name}: {what} needs at least {rows} elements, got shape {tuple(t.shape)}")


def launch_differentiation_position_forward_kernel(
    out_position: torch.Tensor,
    out_velocity: torch.Tensor,
    out_acceleration: torch.Tensor,
    out_jerk: torch.Tensor,
    out_dt: torch.Tensor,
    u_position: torch.Tensor,
    start_position: torch.Tensor,
    start_velocity: torch.Tensor,
    start_acceleration: torch.Tensor,
    goal_position: torch.Tensor,
    goal_velocity: torch.Tensor,
    goal_acceleration: torch.Tensor,
    start_idx: torch.Tensor,
    goal_idx: torch.Tensor,
    traj_dt: torch.Tensor,
    use_implicit_goal_state: torch.Tensor,
    batch_size: int,
    horizon: int,
    dof: int,
) -> None:
    """u_position = waypoints [B, horizon-4, D] -> position / velocity / acceleration / jerk [B, horizon, D] by the
    5-point stencil with start-state and (implicit) goal padding, out_dt [B] (in place)."""
    _check_clique_horizon(horizon)
    dev = u_position.device
    check_tensors(dev, torch.float32, out_position=out_position, out_velocity=out_velocity,
                  out_acceleration=out_acceleration, out_jerk=out_jerk, out_dt=out_dt, u_position=u_position,
                  start_position=start_position, start_velocity=start_velocity, start_acceleration=start_acceleration,
                  goal_position=goal_position, goal_velocity=goal_velocity, goal_acceleration=goal_acceleration,
                  traj_dt=traj_dt)
    check_tensors(dev, torch.int32, start_idx=start_idx, goal_idx=goal_idx)
    check_tensors(dev, torch.uint8, use_implicit_goal_state=use_implicit_goal_state)
    B, H, D = int(batch_size), int(horizon), int(dof)
    _check_rows("[B, horizon, dof]", B * H * D, out_position=out_position, out_velocity=out_velocity,
                out_acceleration=out_acceleration, out_jerk=out_jerk)
    _check_rows("[B, horizon - 4, dof]", B * (H - 4) * D, u_position=u_position)
    _check_rows("[B]", B, out_dt=out_dt, start_idx=start_idx, goal_idx=goal_idx)
    L = _lib.load()
    err = L.cb200_position_clique_forward(
        out_position.data_ptr(), out_velocity.data_ptr(), out_acceleration.data_ptr(), out_jerk.data_ptr(),
        out_dt.data_ptr(), u_position.data_ptr(), start_position.data_ptr(), start_velocity.data_ptr(),
        start_acceleration.data_ptr(), goal_position.data_ptr(), goal_velocity.data_ptr(), goal_acceleration.data_ptr(),
        start_idx.data_ptr(), goal_idx.data_ptr(), traj_dt.data_ptr(), use_implicit_goal_state.data_ptr(), B, H, D,
        stream_ptr(dev))
    _lib.check(err, "launch_differentiation_position_forward_kernel")


def launch_differentiation_position_backward_kernel(
    out_grad_position: torch.Tensor,
    grad_position: torch.Tensor,
    grad_velocity: torch.Tensor,
    grad_acceleration: torch.Tensor,
    grad_jerk: torch.Tensor,
    traj_dt: torch.Tensor,
    dt_idx: torch.Tensor,
    use_implicit_goal_state: torch.Tensor,
    batch_size: int,
    horizon: int,
    dof: int,
) -> None:
    """Adjoint: the four row gradients [B, horizon, D] -> out_grad_position [B, horizon-4, D] (overwritten)."""
    _check_clique_horizon(horizon)
    dev = grad_position.device
    check_tensors(dev, torch.float32, out_grad_position=out_grad_position, grad_position=grad_position,
                  grad_velocity=grad_velocity, grad_acceleration=grad_acceleration, grad_jerk=grad_jerk, traj_dt=traj_dt)
    check_tensors(dev, torch.int32, dt_idx=dt_idx)
    check_tensors(dev, torch.uint8, use_implicit_goal_state=use_implicit_goal_state)
    B, H, D = int(batch_size), int(horizon), int(dof)
    _check_rows("[B, horizon, dof]", B * H * D, grad_position=grad_position, grad_velocity=grad_velocity,
                grad_acceleration=grad_acceleration, grad_jerk=grad_jerk)
    _check_rows("[B, horizon - 4, dof]", B * (H - 4) * D, out_grad_position=out_grad_position)
    _check_rows("[B]", B, dt_idx=dt_idx)
    L = _lib.load()
    err = L.cb200_position_clique_backward(
        out_grad_position.data_ptr(), grad_position.data_ptr(), grad_velocity.data_ptr(), grad_acceleration.data_ptr(),
        grad_jerk.data_ptr(), traj_dt.data_ptr(), dt_idx.data_ptr(), use_implicit_goal_state.data_ptr(), B, H, D,
        stream_ptr(dev))
    _lib.check(err, "launch_differentiation_position_backward_kernel")


def launch_integration_acceleration_kernel(
    out_position: torch.Tensor,
    out_velocity: torch.Tensor,
    out_acceleration: torch.Tensor,
    out_jerk: torch.Tensor,
    u_acc: torch.Tensor,
    start_position: torch.Tensor,
    start_velocity: torch.Tensor,
    start_acceleration: torch.Tensor,
    start_idx: torch.Tensor,
    traj_dt: torch.Tensor,
    batch_size: int,
    horizon: int,
    dof: int,
    use_rk2: bool = True,
) -> None:
    """u_acc [B, horizon, D] -> position / velocity / acceleration / jerk [B, horizon, D] by semi-implicit Euler with
    dt[h] = traj_dt[h] ([horizon]).  `use_rk2` is accepted for either value: the reference's two kernels compute the same."""
    dev = u_acc.device
    check_tensors(dev, torch.float32, out_position=out_position, out_velocity=out_velocity,
                  out_acceleration=out_acceleration, out_jerk=out_jerk, u_acc=u_acc, start_position=start_position,
                  start_velocity=start_velocity, start_acceleration=start_acceleration, traj_dt=traj_dt)
    check_tensors(dev, torch.int32, start_idx=start_idx)
    B, H, D = int(batch_size), int(horizon), int(dof)
    if H < 1:
        raise ValueError(f"horizon must be >= 1, got {H}")
    _check_rows("[B, horizon, dof]", B * H * D, out_position=out_position, out_velocity=out_velocity,
                out_acceleration=out_acceleration, out_jerk=out_jerk, u_acc=u_acc)
    _check_rows("[horizon]", H, traj_dt=traj_dt)
    _check_rows("[B]", B, start_idx=start_idx)
    L = _lib.load()
    err = L.cb200_acceleration_integrate(
        out_position.data_ptr(), out_velocity.data_ptr(), out_acceleration.data_ptr(), out_jerk.data_ptr(),
        u_acc.data_ptr(), start_position.data_ptr(), start_velocity.data_ptr(), start_acceleration.data_ptr(),
        start_idx.data_ptr(), traj_dt.data_ptr(), B, H, D, int(bool(use_rk2)), stream_ptr(dev))
    _lib.check(err, "launch_integration_acceleration_kernel")
