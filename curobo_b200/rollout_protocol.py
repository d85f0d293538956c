"""`B200RobotRollout`: the fused rollout behind the reference's `Rollout` Protocol, so that the reference's optimizers
and solvers (GradientOptCore / LBFGSOpt -> IKSolver / TrajOptSolver / MPCSolver) can be pointed at it unchanged.

  Rollout (runtime_checkable Protocol)      <- curobo/_src/rollout/rollout_protocol.py:35-176
  RobotRollout.evaluate_action              <- curobo/_src/rollout/rollout_robot.py:252-263
  RobotRollout.compute_metrics_from_*       <- rollout_robot.py:267-318
  RolloutResult / RolloutMetrics /
  CostsAndConstraints / CostCollection      <- curobo/_src/rollout/metrics.py:56-420 (the members optimizers call)
  how the optimizer consumes the result     <- optim/components/gradient_opt_core.py:445-480:
        r = rollout.evaluate_action(x_in); c = r.costs_and_constraints.get_sum_cost_and_constraint(sum_horizon=True)
        c.backward(gradient=ones); g = x.grad

The returned term tensors are outputs of ONE autograd node (`FusedTermsFunction`): forward = one fused launch (two more
with the B-spline and position-clique action spaces), backward hands out the gradient that launch already wrote -- the
reference's own contract for its cost Functions with use_grad_input=False (cuda_ops/geometry.py:95-104,
wp_autograd.py:103-110), so the reference's `cat + sum + backward(ones)` yields exactly `grad_q` / `grad_knots` / `grad_u`.  Term classification follows the shipped task files
(content/configs/task/*/lbfgs_*.yml): tool pose and c-space are costs, scene and self collision are constraints.

CUDA only; buffers are allocated once per batch size (update_batch_size), never inside evaluate_action.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, List, Optional, Union

import torch

from .robot_model import RobotModel
from .rollout import RolloutConfig, RolloutEngine
from .trajectory import JointState


def _cat_sum(values: List[torch.Tensor], dims) -> torch.Tensor:
    """Sum of [B,H,k_i] term tensors over the term axis (and the horizon): what util/tensor_util.cat_sum does."""
    return torch.cat(values, dim=-1).sum(dim=dims)


@dataclass
class CostCollection:
    """metrics.py:56-148: parallel lists of term tensors [B,H,k] and their names."""
    values: List[torch.Tensor] = field(default_factory=list)
    names: List[str] = field(default_factory=list)
    weights: List[torch.Tensor] = field(default_factory=list)
    sq_weights: List[torch.Tensor] = field(default_factory=list)

    def add(self, value, name, weight=None, sq_weight=None) -> None:
        self.values.append(value)
        self.names.append(name)
        if weight is not None:
            self.weights.append(weight)
        if sq_weight is not None:
            self.sq_weights.append(sq_weight)

    def is_empty(self) -> bool:
        return not self.values

    def get_sum(self, sum_horizon: bool = True) -> torch.Tensor:
        if not self.values:
            raise ValueError("empty CostCollection")
        return _cat_sum(self.values, (1, 2) if sum_horizon else 2)

    def clone(self) -> "CostCollection":
        return CostCollection([v.clone() for v in self.values], list(self.names), [w.clone() for w in self.weights],
                              [w.clone() for w in self.sq_weights])


@dataclass
class CostsAndConstraints:
    """metrics.py:151-330."""
    costs: CostCollection = field(default_factory=CostCollection)
    constraints: CostCollection = field(default_factory=CostCollection)
    hybrid_costs_constraints: CostCollection = field(default_factory=CostCollection)

    def _pick(self, base: CostCollection, include_all_hybrid, include_from_hybrid):
        vals = list(base.values)
        hy = self.hybrid_costs_constraints
        if include_all_hybrid:
            vals += hy.values
        else:
            vals += [hy.values[hy.names.index(n)] for n in include_from_hybrid if n in hy.names]
        return vals

    def get_sum_cost(self, sum_horizon=False, include_all_hybrid=True, include_from_hybrid=()):
        vals = self._pick(self.costs, include_all_hybrid, include_from_hybrid)
        return _cat_sum(vals, (1, 2) if sum_horizon else 2) if vals else None

    def get_sum_constraint(self, sum_horizon=False, include_all_hybrid=True, include_from_hybrid=()):
        vals = self._pick(self.constraints, include_all_hybrid, include_from_hybrid)
        return _cat_sum(vals, (1, 2) if sum_horizon else 2) if vals else None

    def get_sum_cost_and_constraint(self, sum_horizon=False, include_all_hybrid=True):
        vals = list(self.costs.values) + list(self.constraints.values)
        if include_all_hybrid:
            vals += self.hybrid_costs_constraints.values
        return _cat_sum(vals, (1, 2) if sum_horizon else 2)

    def get_list_costs_and_constraints(self):
        return list(self.costs.values) + list(self.constraints.values) + list(self.hybrid_costs_constraints.values)

    def get_feasible(self, sum_horizon=False, include_all_hybrid=True, include_from_hybrid=()):
        s = self.get_sum_constraint(sum_horizon, include_all_hybrid, include_from_hybrid)
        return True if s is None else s <= 0.0

    def clone(self) -> "CostsAndConstraints":
        return CostsAndConstraints(self.costs.clone(), self.constraints.clone(), self.hybrid_costs_constraints.clone())


@dataclass
class RolloutResult:
    """metrics.py:333-380."""
    actions: Optional[torch.Tensor] = None
    costs_and_constraints: Optional[CostsAndConstraints] = None
    state: Optional[JointState] = None
    debug: Optional[Any] = None

    def __len__(self):
        return self.actions.shape[0] if self.actions is not None else -1


@dataclass
class RolloutMetrics(RolloutResult):
    """metrics.py:383-420."""
    feasible: Optional[Union[torch.Tensor, bool]] = None
    convergence: CostCollection = field(default_factory=CostCollection)


class FusedTermsFunction(torch.autograd.Function):
    """act_seq -> (self [B,H,1], scene [B,H,S], pose [B,H,2L], cspace [B,H,D]); d(sum of all)/d act_seq in backward."""

    @staticmethod
    def forward(ctx, act_seq: torch.Tensor, rollout: "B200RobotRollout"):
        out = rollout._launch(act_seq.detach())
        ctx.save_for_backward(out.grad_knots if rollout.is_bspline else out.grad_u if rollout.is_clique else out.grad_q)
        # fresh aliases of the engine's persistent output buffers: autograd attaches this node to the alias objects
        return (out.self_cost.detach().unsqueeze(-1), out.scene_cost.detach(), out.pose_cost.detach(),
                out.cspace_cost.detach())

    @staticmethod
    def backward(ctx, *grads):
        (g,) = ctx.saved_tensors
        return g, None


class B200RobotRollout:
    """The fused cost+gradient evaluation as a `Rollout`.

    action space "position": act_seq [B, H, D] are joint positions of the H waypoints (H = 1: IK).  vel / acc / jerk
    of the STATE c-space cost come from the optional `state` given to update_params (else zeros, like a transition model
    that only integrates positions).
    action space "bspline": act_seq [B, n_knots, D] are B-spline knots; waypoints, their derivatives and d/d knots are
    evaluated by the spline kernels in front of / behind the rollout kernel (RolloutEngine.evaluate_knots;
    transition/fns_state_transition.py:309-463).
    action space "position_clique": act_seq [B, horizon - 4, D] are waypoints; the state [B, horizon, D] and d/d act_seq come
    from the 5-point stencil with start-state and implicit-goal padding in front of / behind the rollout kernel
    (RolloutEngine.evaluate_positions; the reference's POSITION control space without teleport,
    transition/fns_state_transition.py:159-308).  Like "bspline" it needs update_params(start_state=..., goal_state=...).

    When a call cannot be differentiated -- grad mode off, or `act_seq` does not require grad, as in a particle optimizer or
    compute_metrics_from_action -- evaluate_action launches the cost-only kernels (RolloutEngine.evaluate_cost) where they
    cover the rollout (position action space, discrete collision, no dynamics-aware cost attached).  The returned term tensors
    are the same buffers with the same shapes; `engine.out.grad_q` is not refreshed by such calls."""

    def __init__(self, robot: RobotModel, cfg: RolloutConfig, device="cuda:0", cuboid=None, voxel=None, horizon: int = 1,
                 dt: float = 0.05, action_space: str = "position", n_knots: int = 0, bspline_degree: int = 4,
                 interpolation_steps: int = 4, sum_horizon: bool = True, use_voxel_mip: bool = False, mesh=None):
        if action_space not in ("position", "bspline", "position_clique"):
            raise ValueError("action_space must be 'position', 'bspline' or 'position_clique'")
        self.robot, self.cfg, self.device = robot, cfg, torch.device(device)
        self.engine = RolloutEngine(robot, cfg, device, cuboid, voxel, store_fk_outputs=True, use_voxel_mip=use_voxel_mip,
                                    mesh=mesh)
        self.is_bspline = action_space == "bspline"
        self.is_clique = action_space == "position_clique"
        self._degree, self._steps = bspline_degree, interpolation_steps
        if self.is_bspline:
            if n_knots < 1:
                raise ValueError("bspline action space needs n_knots >= 1")
            self._action_horizon = n_knots
            self._horizon = (n_knots + bspline_degree + 1) * interpolation_steps + 1
        elif self.is_clique:
            if horizon < 8:
                raise ValueError(f"position_clique action space needs horizon >= 8, got {horizon}")
            self._action_horizon, self._horizon = horizon - 4, horizon
        else:
            self._action_horizon = self._horizon = horizon
        self._dt = float(dt)
        self._sum_horizon = sum_horizon
        self._batch_size = -1
        lim = torch.as_tensor(robot.position_limits, dtype=torch.float32, device=self.device)
        self._lows, self._highs = lim[0].contiguous(), lim[1].contiguous()
        self._state: Optional[JointState] = None
        self._env_query_idx = None
        self._spline_args = None
        self._dt_tensor = None
        self._zeros_idx = None

    # -- properties of the Protocol (rollout_protocol.py:46-74) --------------------------------------------------
    @property
    def action_dim(self) -> int:
        return self.robot.num_dof

    @property
    def action_horizon(self) -> int:
        return self._action_horizon

    @property
    def horizon(self) -> int:
        return self._horizon

    @property
    def action_bound_lows(self) -> torch.Tensor:
        return self._lows

    @property
    def action_bound_highs(self) -> torch.Tensor:
        return self._highs

    @property
    def dt(self) -> float:
        return self._dt

    @property
    def sum_horizon(self) -> bool:
        return self._sum_horizon

    @sum_horizon.setter
    def sum_horizon(self, value: bool) -> None:
        # the reference's optimizer core sets this on the rollout it drives (gradient_opt_core.py:113)
        self._sum_horizon = bool(value)

    @property
    def batch_size(self) -> int:
        return self._batch_size

    # -- core ----------------------------------------------------------------------------------------------------
    def _cost_only_covers(self) -> bool:
        """Whether RolloutEngine.evaluate_cost evaluates this rollout's rows: position action space, discrete collision, no
        dynamics-aware cost attached."""
        e = self.engine
        return not (self.is_bspline or self.is_clique or self.cfg.use_sweep or e._effort_cost is not None or
                    e._dyn_params is not None)

    def _launch(self, act_seq: torch.Tensor, grad: bool = True):
        B = act_seq.shape[0]
        if B != self._batch_size:
            self.update_batch_size(B)
        if self.is_bspline:
            s = self._spline_args
            if s is None:
                raise ValueError("bspline action space: call update_params(start_state=..., goal_state=...) first")
            return self.engine.evaluate_knots(act_seq, s["start"], s["start_idx"], s["goal"], s["goal_idx"], s["implicit"],
                                              bspline_degree=self._degree, interpolation_steps=self._steps,
                                              env_query_idx=self._env_query_idx)
        if self.is_clique:
            s = self._spline_args
            if s is None:
                raise ValueError("position_clique action space: call update_params(start_state=..., goal_state=...) first")
            return self.engine.evaluate_positions(act_seq, s["start"], s["start_idx"], s["goal"], s["goal_idx"], s["implicit"],
                                                  env_query_idx=self._env_query_idx)
        evaluate = self.engine.evaluate_action if grad else self.engine.evaluate_cost
        st = self._state
        if st is not None:
            return evaluate(act_seq, vel=st.velocity, acc=st.acceleration, jerk=st.jerk, dt=st.dt,
                            env_query_idx=self._env_query_idx)
        dt = self._dt_tensor if (self.cfg.cspace_type == "state" or self.cfg.use_speed_metric) else None
        return evaluate(act_seq, dt=dt, env_query_idx=self._env_query_idx)

    def _terms(self, act_seq: torch.Tensor) -> CostsAndConstraints:
        if act_seq.ndim != 3 or act_seq.shape[1] != self._action_horizon or act_seq.shape[2] != self.action_dim:
            raise ValueError(f"act_seq must be [B, {self._action_horizon}, {self.action_dim}], got {tuple(act_seq.shape)}")
        if self._cost_only_covers() and not (torch.is_grad_enabled() and act_seq.requires_grad):
            # no gradient can be asked for: the cost-only kernels (engine.out.grad_q is not refreshed)
            out = self._launch(act_seq, grad=False)
            self_c, scene_c, pose_c, cs_c = (out.self_cost.detach().unsqueeze(-1), out.scene_cost.detach(), out.pose_cost.detach(),
                                             out.cspace_cost.detach())
        else:
            self_c, scene_c, pose_c, cs_c = FusedTermsFunction.apply(act_seq, self)
        cc = CostsAndConstraints()
        if self.cfg.pose_weight is not None:
            cc.costs.add(pose_c, "tool_pose")
        if self.cfg.cspace_type is not None:
            cc.costs.add(cs_c, "cspace")
        if self.cfg.scene_weight > 0.0:
            cc.constraints.add(scene_c, "scene_collision")
        if self.cfg.self_weight > 0.0:
            cc.constraints.add(self_c, "self_collision")
        if cc.costs.is_empty() and cc.constraints.is_empty():
            cc.costs.add(cs_c, "cspace")            # all weights zero: keep the graph connected (zeros)
        return cc

    def _state_of(self, act_seq: torch.Tensor) -> JointState:
        if self.is_bspline or self.is_clique:
            p, v, a, j = self.engine._state
            return JointState(p, v, a, j, self.engine._state_dt)
        st = self._state
        if st is not None:
            return JointState(act_seq, st.velocity, st.acceleration, st.jerk, st.dt)
        return JointState(act_seq, None, None, None, self._dt_tensor)

    def evaluate_action(self, act_seq: torch.Tensor, **kwargs) -> RolloutResult:
        cc = self._terms(act_seq)
        return RolloutResult(actions=act_seq, state=self._state_of(act_seq), costs_and_constraints=cc)

    def compute_metrics_from_action(self, act_seq: torch.Tensor, **kwargs) -> RolloutMetrics:
        """Costs, feasibility (constraints <= 0) and the convergence terms solvers read (position / rotation error of
        every tool frame against its goal, rollout_robot.py:267-318)."""
        with torch.no_grad():
            cc = self._terms(act_seq)
            out = self.engine.out
            conv = CostCollection()
            if self.engine._goal is not None and self.cfg.pose_weight is not None:
                pe, re = self._pose_errors(out)
                conv.add(pe, "position_tolerance")
                conv.add(re, "orientation_tolerance")
            feas = cc.get_feasible(sum_horizon=self._sum_horizon)
        return RolloutMetrics(actions=act_seq, state=self._state_of(act_seq), costs_and_constraints=cc, feasible=feas,
                              convergence=conv)

    def compute_metrics_from_state(self, state: JointState, **kwargs) -> RolloutMetrics:
        """Metrics of a given joint-state trajectory [B, H, D] (position action space semantics)."""
        if self.is_bspline:
            raise ValueError("compute_metrics_from_state: pass knots to compute_metrics_from_action in the bspline action space")
        if self.is_clique:
            raise ValueError("compute_metrics_from_state: pass waypoints to compute_metrics_from_action in the position_clique "
                             "action space")
        prev = self._state
        try:
            if state.velocity is not None and state.acceleration is not None and state.jerk is not None and state.dt is not None:
                self._state = state
            return self.compute_metrics_from_action(state.position)
        finally:
            self._state = prev

    def _pose_errors(self, out):
        from .cost import tool_pose_distance
        gp, gq, ig, extra = self.engine._goal
        B, H, L = out.link_pos.shape[:3]
        dev = self.device
        b = self._pose_buf
        ones6 = b["ones6"]
        tol0 = b["tol0"]
        tool_pose_distance(out.link_pos, out.link_quat, gp, gq, ig.view(B, 1), b["w"],
                           extra["terminal_axes"] if extra["terminal_axes"] is not None else ones6,
                           extra["non_terminal_axes"] if extra["non_terminal_axes"] is not None else ones6,
                           tol0, tol0, None, b["dist"], b["pe"], b["re"], b["gp"], b["gq"], b["gi"],
                           use_lie_group=self.cfg.pose_lie)
        return b["pe"], b["re"]

    # -- lifecycle -----------------------------------------------------------------------------------------------
    def update_batch_size(self, batch_size: int) -> None:
        if batch_size == self._batch_size:
            return
        dev, L = self.device, self.robot.num_tool_frames
        H = self._horizon
        self.engine.setup_batch_tensors(batch_size, H)
        z = lambda *s, dt=torch.float32: torch.zeros(s, dtype=dt, device=dev)  # noqa: E731
        pw = self.cfg.pose_weight if self.cfg.pose_weight is not None else (0.0, 0.0)
        self._pose_buf = dict(w=torch.tensor([float(pw[0]), float(pw[1])], dtype=torch.float32, device=dev),
                              ones6=torch.ones((L, 6), dtype=torch.float32, device=dev), tol0=z(L, 2),
                              dist=z(batch_size, H, 2 * L), pe=z(batch_size, H, L), re=z(batch_size, H, L),
                              gp=z(batch_size, H, L, 3), gq=z(batch_size, H, L, 4), gi=z(batch_size, H, L, dt=torch.int32))
        self._dt_tensor = torch.full((batch_size,), self._dt, dtype=torch.float32, device=dev)
        self._batch_size = batch_size
        if self._state is not None and self._state.position.shape[0] != batch_size:
            self._state = None

    def update_params(self, goal_position: Optional[torch.Tensor] = None, goal_quat: Optional[torch.Tensor] = None,
                      idxs_goal: Optional[torch.Tensor] = None, cspace_target: Optional[torch.Tensor] = None,
                      idxs_cspace_target: Optional[torch.Tensor] = None, cspace_target_dof_weight: Optional[torch.Tensor] = None,
                      env_query_idx: Optional[torch.Tensor] = None, state: Optional[JointState] = None,
                      start_state: Optional[JointState] = None, goal_state: Optional[JointState] = None,
                      start_state_idx: Optional[torch.Tensor] = None, goal_state_idx: Optional[torch.Tensor] = None,
                      use_implicit_goal_state: Optional[torch.Tensor] = None, current_js: Optional[JointState] = None,
                      idxs_current_js: Optional[torch.Tensor] = None, current_state_dt: Optional[torch.Tensor] = None,
                      **pose_extra) -> bool:
        """Targets of the next solve: tool-pose goals (GoalRegistry rows: goal_* [G, L, n_goalset, 3|4], idxs_goal [B]),
        the c-space target, the world index per seed, and -- bspline and position_clique action spaces -- the boundary
        states of the trajectory.  `current_js` (position [n, D], optional velocity), `idxs_current_js` [B] and
        `current_state_dt` [n] (GoalRegistry's fields) are the current state of the POSITION c-space cost
        (RolloutEngine.update_current_state); `current_state_dt` defaults to `current_js.dt`, as in the reference.  A dt of one
        element (a float, a 0-d or [1] tensor) applies to every row; it is expanded into a tensor of this rollout, so later
        in-place writes to the caller's scalar need another update_params.  `idxs_current_js` has one entry per evaluated row
        (the line-search-expanded batch, like `idxs_goal`), int32 (other integer types are converted, a copy) and every entry
        in [0, n)."""
        if current_js is not None:
            dt = current_state_dt if current_state_dt is not None else current_js.dt
            if dt is None:
                raise ValueError("current_js needs current_state_dt (or current_js.dt)")
            pos = current_js.position
            pos = pos.view(1, -1) if pos.ndim == 1 else pos
            vel = current_js.velocity
            if vel is not None and vel.ndim == 1:
                vel = vel.view(1, -1)
            n = pos.shape[0]
            if not isinstance(dt, torch.Tensor):
                dt = torch.full((n,), float(dt), dtype=torch.float32, device=self.device)
            elif dt.numel() == 1 and n != 1:
                dt = dt.reshape(1).to(torch.float32).expand(n).contiguous()
            else:
                dt = dt.reshape(-1)
            idx = idxs_current_js
            if idx is not None and idx.dtype != torch.int32 and not idx.is_floating_point():
                idx = idx.to(torch.int32)
            self.engine.update_current_state(pos, vel, dt, idx)
        if goal_position is not None:
            self.engine.update_goal(goal_position, goal_quat, idxs_goal, **pose_extra)
        if cspace_target is not None:
            self.engine.update_cspace_target(cspace_target, idxs_cspace_target, cspace_target_dof_weight)
        if env_query_idx is not None:
            self._env_query_idx = env_query_idx
        if state is not None:
            self._state = state
        if start_state is not None or goal_state is not None:
            if start_state is None or goal_state is None or start_state_idx is None or goal_state_idx is None:
                raise ValueError("start_state, goal_state, start_state_idx and goal_state_idx go together")
            if use_implicit_goal_state is None:
                use_implicit_goal_state = torch.zeros(goal_state.position.shape[0], dtype=torch.uint8, device=self.device)
            self._spline_args = dict(start=start_state, goal=goal_state, start_idx=start_state_idx, goal_idx=goal_state_idx,
                                     implicit=use_implicit_goal_state)
        return True

    def update_dt(self, dt: Union[float, torch.Tensor], **kwargs) -> bool:
        if isinstance(dt, torch.Tensor):
            self._dt = float(dt.reshape(-1)[0]) if not torch.cuda.is_current_stream_capturing() else self._dt
            if self._dt_tensor is not None:
                self._dt_tensor.copy_(dt.reshape(-1).expand_as(self._dt_tensor) if dt.numel() == 1 else dt.reshape(-1))
        else:
            self._dt = float(dt)
            if self._dt_tensor is not None:
                self._dt_tensor.fill_(self._dt)
        return True

    def reset(self, reset_problem_ids: Optional[torch.Tensor] = None, **kwargs) -> bool:
        return True          # the fused kernel keeps no per-problem state between calls

    def reset_shape(self) -> bool:
        self._batch_size = -1
        return True

    def reset_seed(self) -> None:
        return None

    def reset_cuda_graph(self) -> None:
        return None

    def refresh_world(self) -> None:
        self.engine.refresh_world()

    # -- link spheres: RolloutEngine's calls (the reference's KinematicsParams / AttachmentManager); graphs captured on this
    # rollout see an update on their next replay without recapture (the packed robot constants keep their address) -------------
    @property
    def link_spheres(self) -> torch.Tensor:
        """[n_cfg, S, 4] link-frame spheres (see RolloutEngine.refresh_link_spheres for in-place writes)."""
        return self.engine.link_spheres

    def update_link_spheres(self, link_name: str, spheres: torch.Tensor, start_sph_idx: int = 0,
                            config_idx: Optional[int] = None) -> None:
        self.engine.update_link_spheres(link_name, spheres, start_sph_idx, config_idx)

    def get_link_spheres(self, link_name: str, config_idx: int = 0) -> torch.Tensor:
        return self.engine.get_link_spheres(link_name, config_idx)

    def disable_link_spheres(self, link_name: str) -> None:
        self.engine.disable_link_spheres(link_name)

    def enable_link_spheres(self, link_name: str) -> None:
        self.engine.enable_link_spheres(link_name)

    def reset_link_spheres(self, link_name: str) -> None:
        self.engine.reset_link_spheres(link_name)

    def refresh_link_spheres(self) -> None:
        self.engine.refresh_link_spheres()

    def attach_object_spheres(self, spheres: torch.Tensor, link_name: str = "attached_object",
                              joint_position: Optional[torch.Tensor] = None, object_pose: Optional[torch.Tensor] = None) -> None:
        self.engine.attach_object_spheres(spheres, link_name, joint_position, object_pose)

    def detach_object_spheres(self, link_name: str = "attached_object") -> None:
        self.engine.detach_object_spheres(link_name)
