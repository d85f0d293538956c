"""Host mirror of the reference's B-spline control space (SURVEY.md section 8f rank 1).

  ControlSpace / spline helpers  <- curobo/_src/types/control_space.py:18-53
  BSplineIdxKernel               <- curobo/_src/curobolib/cuda_ops/trajectory.py:299-441 (torch.autograd.Function,
                                    same positional arguments)
  get_bspline_interpolation      <- cuda_ops/trajectory.py:21-96 (single-dt resampling of the final trajectory)
  StateFromBSplineKnot           <- curobo/_src/transition/fns_state_transition.py:309-463
and of its legacy POSITION (clique, non-teleport) and ACCELERATION control spaces:
  CliqueTensorStepIdxKernel / AccelerationTensorStepIdxKernel <- cuda_ops/trajectory.py:95-296
  StateFromPositionClique / StateFromAcceleration             <- transition/fns_state_transition.py:90-308

CUDA only, float32 only, like the reference (fns_state_transition.py:323).  No CPU fallback.
"""
from __future__ import annotations

from dataclasses import dataclass
from enum import Enum
from typing import Optional

import torch

from .backends import trajectory as trajectory_cu


class ControlSpace(Enum):
    """types/control_space.py:18-53 (same member values)."""
    POSITION = 0
    VELOCITY = 1
    ACCELERATION = 2
    BSPLINE_3 = 3
    BSPLINE_4 = 4
    BSPLINE_5 = 5

    @staticmethod
    def bspline_types():
        return [ControlSpace.BSPLINE_3, ControlSpace.BSPLINE_4, ControlSpace.BSPLINE_5]

    @staticmethod
    def spline_degree(control_space: "ControlSpace") -> int:
        return {ControlSpace.BSPLINE_3: 3, ControlSpace.BSPLINE_4: 4, ControlSpace.BSPLINE_5: 5}.get(control_space, 0)

    @staticmethod
    def spline_total_knots(control_space: "ControlSpace", action_knots: int) -> int:
        if control_space not in ControlSpace.bspline_types():
            return action_knots
        return action_knots + ControlSpace.spline_degree(control_space) + 1  # control_space.py:41

    @staticmethod
    def spline_total_interpolation_steps(control_space: "ControlSpace", action_knots: int, interpolation_steps: int) -> int:
        return ControlSpace.spline_total_knots(control_space, action_knots) * interpolation_steps + 1  # :44-49


@dataclass
class JointState:
    """The five tensors of curobo's JointState that the spline kernels touch."""
    position: torch.Tensor
    velocity: torch.Tensor
    acceleration: torch.Tensor
    jerk: torch.Tensor
    dt: Optional[torch.Tensor] = None

    @property
    def shape(self):
        return self.position.shape

    @staticmethod
    def zeros(shape, device, dt_shape=None) -> "JointState":
        z = lambda: torch.zeros(shape, device=device, dtype=torch.float32)  # noqa: E731
        dt = torch.zeros(dt_shape if dt_shape is not None else shape[:1], device=device, dtype=torch.float32)
        return JointState(z(), z(), z(), z(), dt)


class BSplineIdxKernel(torch.autograd.Function):
    """knots -> (position, velocity, acceleration, jerk); backward returns d loss / d knots into `out_grad_position`."""

    @staticmethod
    def forward(ctx, u_act, start_position, start_velocity, start_acceleration, start_jerk, goal_position, goal_velocity,
                goal_acceleration, goal_jerk, start_idx, goal_idx, out_position, out_velocity, out_acceleration,
                out_jerk, out_dt, traj_dt, use_implicit_goal_state, out_grad_position, bspline_degree,
                use_flat_gradient=False):
        n_knots = u_act.shape[-2]
        trajectory_cu.launch_bspline_interpolation_forward_kernel(
            out_position, out_velocity, out_acceleration, out_jerk, out_dt, u_act, start_position, start_velocity,
            start_acceleration, start_jerk, goal_position, goal_velocity, goal_acceleration, goal_jerk, start_idx,
            goal_idx, traj_dt, use_implicit_goal_state, out_position.shape[0], out_position.shape[1],
            out_position.shape[-1], n_knots, bspline_degree)
        ctx.use_flat_gradient = use_flat_gradient
        ctx.save_for_backward(traj_dt, out_grad_position, goal_idx, use_implicit_goal_state)
        ctx.n_knots = n_knots
        ctx.bspline_degree = bspline_degree
        ctx.mark_non_differentiable(out_dt)
        return out_position, out_velocity, out_acceleration, out_jerk

    @staticmethod
    def backward(ctx, grad_out_p, grad_out_v, grad_out_a, grad_out_j):
        u_grad = None
        if ctx.needs_input_grad[0]:
            traj_dt, out_grad_position, dt_idx, use_implicit_goal_state = ctx.saved_tensors
            padded_horizon = grad_out_p.shape[1]
            if (grad_out_v.shape[1] != padded_horizon or grad_out_a.shape[1] != padded_horizon
                    or grad_out_j.shape[1] != padded_horizon):
                raise ValueError(f"BSpline backward: grad tensor dim-1 mismatch: p={padded_horizon}, "
                                 f"v={grad_out_v.shape[1]}, a={grad_out_a.shape[1]}, j={grad_out_j.shape[1]}")
            trajectory_cu.launch_bspline_interpolation_backward_kernel(
                out_grad_position, grad_out_p.contiguous(), grad_out_v.contiguous(), grad_out_a.contiguous(),
                grad_out_j.contiguous(), traj_dt, dt_idx, use_implicit_goal_state, grad_out_p.shape[0],
                grad_out_p.shape[1], grad_out_p.shape[2], ctx.n_knots, ctx.bspline_degree, ctx.use_flat_gradient)
            u_grad = out_grad_position
        return (u_grad,) + (None,) * 20


def get_bspline_interpolation(knots, knot_dt, start: JointState, goal: JointState, start_idx, goal_idx, interpolation_dt,
                              use_implicit_goal_state, interpolation_horizon, out: JointState, bspline_degree: int = 4):
    """Resample every spline at one common `interpolation_dt` with its own horizon (cuda_ops/trajectory.py:21-96)."""
    trajectory_cu.launch_bspline_interpolation_single_dt_kernel(
        out.position, out.velocity, out.acceleration, out.jerk, out.dt, knots, knot_dt, start.position, start.velocity,
        start.acceleration, start.jerk, goal.position, goal.velocity, goal.acceleration, goal.jerk, start_idx, goal_idx,
        interpolation_dt, use_implicit_goal_state, interpolation_horizon, out.position.shape[0], out.position.shape[1],
        out.position.shape[-1], knots.shape[-2], bspline_degree)
    return out


class StateFromBSplineKnot:
    """Action (knots) -> state sequence.  horizon = (n_knots + degree + 1) * interpolation_steps + 1."""

    def __init__(self, device: torch.device, dof: int, batch_size: int = 1, n_knots: int = 6, interpolation_steps: int = 1,
                 use_implicit_goal_state: bool = False, control_space: ControlSpace = ControlSpace.BSPLINE_4) -> None:
        self.device = torch.device(device)
        self.dof = dof
        self.n_knots = n_knots
        self.use_implicit_goal_state = use_implicit_goal_state
        self.control_space = control_space
        self.bspline_degree = ControlSpace.spline_degree(control_space)
        self.interpolation_steps = interpolation_steps
        self.padded_horizon = ControlSpace.spline_total_interpolation_steps(control_space, n_knots, interpolation_steps)
        self.batch_size = -1
        self._u_grad = None
        self.update_batch_size(batch_size)

    def update_batch_size(self, batch_size: int) -> None:
        if batch_size != self.batch_size:
            self.batch_size = batch_size
            self.action_horizon = self.n_knots
            self._u_grad = torch.zeros((batch_size, self.n_knots, self.dof), device=self.device, dtype=torch.float32)

    def forward(self, start_state: JointState, u_act: torch.Tensor, out_state_seq: JointState,
                start_state_idx: Optional[torch.Tensor] = None, goal_state: Optional[JointState] = None,
                goal_state_idx: Optional[torch.Tensor] = None,
                use_implicit_goal_state: Optional[torch.Tensor] = None) -> JointState:
        # argument checks of fns_state_transition.py:404-441
        if self.use_implicit_goal_state:
            if goal_state is None:
                raise ValueError("Goal state is not provided for implicit goal state")
            if start_state_idx is not None and goal_state_idx is None:
                raise ValueError("Goal state index is not provided for implicit goal state")
        else:
            if goal_state is None:
                goal_state = start_state
            if goal_state_idx is None:
                goal_state_idx = start_state_idx
        if start_state_idx is None:
            raise ValueError("Start state index is required for BSpline kernel")
        if goal_state_idx is None:
            raise ValueError("idx is None")
        if goal_state.dt is None:
            raise ValueError("dt is None")
        if use_implicit_goal_state is None:
            raise ValueError("use_implicit_goal_state is None")
        if goal_state_idx.shape[0] != u_act.shape[0]:
            raise ValueError(f"Shape mismatch: goal_state_idx.shape[0] != u_act.shape[0]: "
                             f"{goal_state_idx.shape[0]} != {u_act.shape[0]}")
        if use_implicit_goal_state.shape[0] != goal_state.shape[0]:
            raise ValueError(f"Shape mismatch: use_implicit_goal_state.shape[0] != goal_state.shape[0]: "
                             f"{use_implicit_goal_state.shape[0]} != {goal_state.shape[0]}")
        if out_state_seq.dt is None:
            raise ValueError("out dt is None")
        if u_act.shape[1] != self.n_knots:
            raise ValueError(f"u_act.shape[1] != self.n_knots: {u_act.shape[1]} != {self.n_knots}")
        if self.padded_horizon != out_state_seq.shape[1]:
            raise ValueError(f"padded_horizon != out_state_seq.shape[1]: {self.padded_horizon} != {out_state_seq.shape[1]}")
        self.update_batch_size(u_act.shape[0])
        (out_state_seq.position, out_state_seq.velocity, out_state_seq.acceleration, out_state_seq.jerk) = \
            BSplineIdxKernel.apply(u_act, start_state.position, start_state.velocity, start_state.acceleration,
                                   start_state.jerk, goal_state.position, goal_state.velocity, goal_state.acceleration,
                                   goal_state.jerk, start_state_idx, goal_state_idx, out_state_seq.position,
                                   out_state_seq.velocity, out_state_seq.acceleration, out_state_seq.jerk,
                                   out_state_seq.dt, goal_state.dt, use_implicit_goal_state, self._u_grad,
                                   self.bspline_degree)
        return out_state_seq


# ------------------------------------------------------------------------------------------------
# POSITION (clique) and ACCELERATION control spaces
#   CliqueTensorStepIdxKernel        <- cuda_ops/trajectory.py:95-235
#   AccelerationTensorStepIdxKernel  <- cuda_ops/trajectory.py:237-296
#   StateFromPositionClique          <- transition/fns_state_transition.py:159-308
#   StateFromAcceleration            <- transition/fns_state_transition.py:90-157
# ------------------------------------------------------------------------------------------------
class CliqueTensorStepIdxKernel(torch.autograd.Function):
    """Waypoints u [B, H-4, D] -> (position, velocity, acceleration, jerk) [B, H, D]; backward returns d loss / d u into
    `out_grad_position`."""

    @staticmethod
    def forward(ctx, u_act, start_position, start_velocity, start_acceleration, goal_position, goal_velocity,
                goal_acceleration, start_idx, goal_idx, out_position, out_velocity, out_acceleration, out_jerk, out_dt,
                traj_dt, use_implicit_goal_state, out_grad_position):
        horizon = out_position.shape[1]
        if u_act.shape[-2] != horizon - 4:
            raise ValueError("Action shape is not compatible with horizon: " + str(u_act.shape))
        trajectory_cu.launch_differentiation_position_forward_kernel(
            out_position, out_velocity, out_acceleration, out_jerk, out_dt, u_act, start_position, start_velocity,
            start_acceleration, goal_position, goal_velocity, goal_acceleration, start_idx, goal_idx, traj_dt,
            use_implicit_goal_state, out_position.shape[0], out_position.shape[1], out_position.shape[-1])
        if ctx.needs_input_grad[0]:
            ctx.save_for_backward(traj_dt, out_grad_position, goal_idx, use_implicit_goal_state)
        return out_position, out_velocity, out_acceleration, out_jerk

    @staticmethod
    def backward(ctx, grad_out_p, grad_out_v, grad_out_a, grad_out_j):
        u_grad = None
        if ctx.needs_input_grad[0]:
            traj_dt, out_grad_position, goal_idx, use_implicit_goal_state = ctx.saved_tensors
            for name, g in (("grad_out_p", grad_out_p), ("grad_out_v", grad_out_v), ("grad_out_a", grad_out_a),
                            ("grad_out_j", grad_out_j)):
                if g is None:
                    raise ValueError(f"{name} is None")
            trajectory_cu.launch_differentiation_position_backward_kernel(
                out_grad_position, grad_out_p.contiguous(), grad_out_v.contiguous(), grad_out_a.contiguous(),
                grad_out_j.contiguous(), traj_dt, goal_idx, use_implicit_goal_state, grad_out_p.shape[0],
                grad_out_p.shape[1], grad_out_p.shape[2])
            u_grad = out_grad_position
        return (u_grad,) + (None,) * 16


class AccelerationTensorStepIdxKernel(torch.autograd.Function):
    """Accelerations u [B, H, D] -> (position, velocity, acceleration, jerk) [B, H, D]; no backward, like the reference."""

    @staticmethod
    def forward(ctx, u_act, start_position, start_velocity, start_acceleration, start_idx, out_position, out_velocity,
                out_acceleration, out_jerk, traj_dt, out_grad_position):
        trajectory_cu.launch_integration_acceleration_kernel(
            out_position, out_velocity, out_acceleration, out_jerk, u_act, start_position, start_velocity,
            start_acceleration, start_idx, traj_dt, out_position.shape[0], out_position.shape[1], out_position.shape[-1],
            True)
        ctx.save_for_backward(traj_dt, out_grad_position)
        return out_position, out_velocity, out_acceleration, out_jerk

    @staticmethod
    def backward(ctx, grad_out_p, grad_out_v, grad_out_a, grad_out_j):
        if ctx.needs_input_grad[0]:
            raise NotImplementedError()
        return (None,) * 11


def _no_filters(filter_velocity: bool, filter_acceleration: bool, filter_jerk: bool) -> None:
    if filter_velocity or filter_acceleration or filter_jerk:
        raise ValueError("the moving-average filters of the clique state (filter_velocity / filter_acceleration / "
                         "filter_jerk) are not supported")


class StateFromPositionClique:
    """Action (waypoints [B, H-4, D]) -> state sequence [B, H, D] by the 5-point stencil (position control space without
    teleport).  `dt_h` is kept for update_dt like the reference's; the stencil reads dt from goal_state.dt."""

    def __init__(self, device: torch.device, dt_h: torch.Tensor, dof: int, filter_velocity: bool = False,
                 filter_acceleration: bool = False, filter_jerk: bool = False, batch_size: int = 1,
                 horizon: int = 1) -> None:
        _no_filters(filter_velocity, filter_acceleration, filter_jerk)
        self.device = torch.device(device)
        self.dof = dof
        self._dt_h = dt_h
        self._inv_dt_h = 1.0 / dt_h
        self._u_grad = None
        self.batch_size = self.horizon = -1
        self.update_batch_size(batch_size, horizon)

    def update_dt(self, dt: float) -> None:
        self._dt_h[:] = dt
        self._inv_dt_h[:] = 1.0 / dt

    def update_batch_size(self, batch_size: Optional[int] = None, horizon: Optional[int] = None,
                          force_update: bool = False) -> None:
        if batch_size != self.batch_size or horizon != self.horizon or self._u_grad is None:
            self.action_horizon = horizon - 4
            self._u_grad = torch.zeros((batch_size, self.action_horizon, self.dof), device=self.device, dtype=torch.float32)
        if force_update:
            self._u_grad = self._u_grad.detach()
        self.batch_size, self.horizon = batch_size, horizon

    def forward(self, start_state: JointState, u_act: torch.Tensor, out_state_seq: JointState,
                start_state_idx: Optional[torch.Tensor] = None, goal_state: Optional[JointState] = None,
                goal_state_idx: Optional[torch.Tensor] = None, use_implicit_goal_state: Optional[torch.Tensor] = None,
                **kwargs) -> JointState:
        # argument checks of fns_state_transition.py:260-277
        if start_state_idx is None:
            raise ValueError("Start state index is required for Clique kernel")
        if goal_state is None:
            goal_state = start_state
        if goal_state_idx is None:
            goal_state_idx = start_state_idx
        if goal_state.dt.shape != goal_state.position.shape[0:2]:
            raise ValueError(f"Shape mismatch: goal_state.dt.shape[0] != goal_state.position.shape[0:2]: "
                             f"{goal_state.dt.shape} != {goal_state.position.shape[0:2]}")
        if use_implicit_goal_state.shape != goal_state.position.shape[0:2]:
            raise ValueError(f"Shape mismatch: use_implicit_goal_state.shape[0] != goal_state.position.shape[0]: "
                             f"{use_implicit_goal_state.shape[0]} != "
                             f"{goal_state.position.view(-1, goal_state.position.shape[-1]).shape[0]}")
        (out_state_seq.position, out_state_seq.velocity, out_state_seq.acceleration, out_state_seq.jerk) = \
            CliqueTensorStepIdxKernel.apply(u_act, start_state.position, start_state.velocity, start_state.acceleration,
                                            goal_state.position, goal_state.velocity, goal_state.acceleration,
                                            start_state_idx, goal_state_idx, out_state_seq.position,
                                            out_state_seq.velocity, out_state_seq.acceleration, out_state_seq.jerk,
                                            out_state_seq.dt, goal_state.dt, use_implicit_goal_state, self._u_grad)
        return out_state_seq


class StateFromAcceleration:
    """Action (accelerations [B, H, D]) -> state sequence [B, H, D] by semi-implicit Euler with dt[h] = dt_h[h]."""

    def __init__(self, device: torch.device, dt_h: torch.Tensor, dof: int, batch_size: int = 1, horizon: int = 1) -> None:
        self.device = torch.device(device)
        self.dof = dof
        self._dt_h = dt_h
        self._inv_dt_h = None
        self.batch_size = self.horizon = -1
        self.action_horizon = horizon
        self._u_grad = torch.zeros((batch_size, horizon, dof), device=self.device, dtype=torch.float32)
        self.batch_size, self.horizon = batch_size, horizon

    def update_dt(self, dt: float) -> None:
        self._dt_h[:] = dt

    def update_batch_size(self, batch_size: Optional[int] = None, horizon: Optional[int] = None,
                          force_update: bool = False) -> None:
        if batch_size != self.batch_size or horizon != self.horizon:
            self._u_grad = torch.zeros((batch_size, horizon, self.dof), device=self.device, dtype=torch.float32)
        if force_update:
            self._u_grad = self._u_grad.detach()
        self.batch_size, self.horizon = batch_size, horizon

    def forward(self, start_state: JointState, u_act: torch.Tensor, out_state_seq: JointState,
                start_state_idx: Optional[torch.Tensor] = None, **kwargs) -> JointState:
        if start_state_idx is None:
            raise ValueError("Start state index is required for Acceleration kernel")
        (out_state_seq.position, out_state_seq.velocity, out_state_seq.acceleration, out_state_seq.jerk) = \
            AccelerationTensorStepIdxKernel.apply(u_act, start_state.position, start_state.velocity,
                                                  start_state.acceleration, start_state_idx, out_state_seq.position,
                                                  out_state_seq.velocity, out_state_seq.acceleration, out_state_seq.jerk,
                                                  self._dt_h, self._u_grad)
        return out_state_seq
