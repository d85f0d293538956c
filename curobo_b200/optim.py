"""Host mirror of the reference's L-BFGS optimizer iteration (SURVEY.md section 8f rank 2), built on the fused
rollout: one optimizer iteration = 3 kernel launches

    cb200_lbfgs_step (+ search points)  ->  cb200_rollout_cost_grad on [B * n_linesearch] rows  ->  cb200_line_search

where the reference runs ~30 (gradient_opt_core.py:334-400: line search strategy -> rollout 15-25 launches ->
wolfe kernel -> LBFGS kernel + torch glue).

  LBFGScu                 <- curobo/_src/curobolib/cuda_ops/optimization.py:192-252 (same positional arguments)
  wolfe_line_search       <- cuda_ops/optimization.py:22-189 (flat-tensor form of the same launch)
  QuasiNewtonBuffers      <- optim/components/quasi_newton_buffers.py:20-130
  LBFGSOpt.optimize       <- optim/gradient/lbfgs.py:157-240 + optim/components/gradient_opt_core.py:290-400 with
                             line_search_type approx_wolfe, CUDA-kernel step direction and line search
                             (content/configs/task/ik/lbfgs_ik.yml)
  MPPIOpt.optimize        <- optim/particle/mppi.py + optim/components/particle_opt_core.py:283-441 (DIAG_A, CLAMP,
                             content/configs/task/ik/particle_ik.yml): per inner iteration cb200_mppi_sample -> cost-only
                             rollout -> cb200_mppi_update, where the reference runs ~20 torch launches around its rollout
  MultiStageOpt           <- optim/multi_stage_optimizer.py:96-180 (MPPI then L-BFGS: the reference's default IK)

CUDA only; no CPU path.
"""
from __future__ import annotations

from dataclasses import dataclass, field, replace
from typing import Callable, List, Optional, Tuple

import torch

from .backends import optimization as optimization_cu
from .backends import tensor_checks as _tc


class LBFGScu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, step_vec, rho_buffer, y_buffer, s_buffer, q, grad_q, x_0, grad_0, epsilon=0.1, stable_mode=False,
                use_shared_buffers=True):
        m, b, v_dim, _ = y_buffer.shape
        R = optimization_cu.launch_lbfgs_step(step_vec, rho_buffer, y_buffer, s_buffer, q, grad_q, x_0, grad_0, epsilon, b, m,
                                              v_dim, stable_mode, use_shared_buffers)
        return R[0].view(step_vec.shape)

    @staticmethod
    def backward(ctx, grad_output):
        return (None,) * 11


@dataclass
class QuasiNewtonBuffers:
    """(s, y, rho) history + reference point, shapes as in the reference ([m,B,V,1], [m,B,1,1], [B,V,1])."""
    history: int
    device: torch.device
    s: Optional[torch.Tensor] = None
    y: Optional[torch.Tensor] = None
    rho: Optional[torch.Tensor] = None
    x_0: Optional[torch.Tensor] = None
    grad_0: Optional[torch.Tensor] = None
    step_q_buffer: Optional[torch.Tensor] = None

    def resize(self, num_problems: int, opt_dim: int) -> None:
        z = lambda *s: torch.zeros(s, device=self.device, dtype=torch.float32)  # noqa: E731
        b = num_problems
        self.x_0, self.grad_0 = z(b, opt_dim, 1), z(b, opt_dim, 1)
        self.y, self.s = z(self.history, b, opt_dim, 1), z(self.history, b, opt_dim, 1)
        self.rho = z(self.history, b, 1, 1)
        self.step_q_buffer = z(b, opt_dim)

    def clear(self) -> None:
        for t in (self.s, self.y, self.rho, self.step_q_buffer):
            t.fill_(0.0)

    def set_reference(self, x: torch.Tensor, grad: torch.Tensor) -> None:
        self.x_0.copy_(x.view_as(self.x_0))
        self.grad_0.copy_(grad.view_as(self.grad_0))


@dataclass
class LBFGSOptCfg:
    """The fields of optim/gradient/lbfgs.py:38-86 this loop uses (defaults = content/configs/task/ik/lbfgs_ik.yml)."""
    num_iters: int = 100
    history: int = 7
    epsilon: float = 0.01
    stable_mode: bool = True
    line_search_scale: List[float] = field(default_factory=lambda: [0.0, 0.1, 0.5, 1.0])
    line_search_wolfe_c_1: float = 1e-5
    line_search_wolfe_c_2: float = 0.9
    strong_wolfe: bool = False
    approx_wolfe: bool = True
    step_scale: float = 0.98
    fix_terminal_action: bool = False
    cost_delta_threshold: float = 0.0
    cost_relative_threshold: float = 0.0
    convergence_iteration: int = 10
    initial_step_scale: float = 0.001


class LBFGSOpt:
    """Batched L-BFGS over `num_problems` independent problems of dimension action_horizon * action_dim.

    `cost_grad_fn(x_set)` evaluates x_set [B * n_linesearch, opt_dim] and returns (cost [B * n], grad [B * n, opt_dim])
    -- with the fused rollout that is one kernel launch (see IKSolver below)."""

    def __init__(self, cfg: LBFGSOptCfg, num_problems: int, action_horizon: int, action_dim: int,
                 action_bound_lows: torch.Tensor, action_bound_highs: torch.Tensor,
                 cost_grad_fn: Callable[[torch.Tensor], Tuple[torch.Tensor, torch.Tensor]], device="cuda:0"):
        cfg = replace(cfg, line_search_scale=list(cfg.line_search_scale))   # never mutate the caller's config
        self.cfg, self.device = cfg, torch.device(device)
        _tc.require_cuda(self.device, "LBFGSOpt is CUDA-only")
        self.B, self.H, self.D = num_problems, action_horizon, action_dim
        self.V = action_horizon * action_dim
        if cfg.history > self.V:
            cfg.history = self.V  # lbfgs.py:186-188
        if self.V > 1024 or cfg.history > 31:
            raise ValueError("opt_dim > 1024 or history > 31 is not supported by the step kernel")
        self.n = len(cfg.line_search_scale)
        dev, B, V, n = self.device, self.B, self.V, self.n
        z = lambda *s, dt=torch.float32: torch.zeros(s, device=dev, dtype=dt)  # noqa: E731
        self.qn = QuasiNewtonBuffers(cfg.history, dev)
        self.qn.resize(B, V)
        self.magnitudes = torch.tensor(cfg.line_search_scale, device=dev, dtype=torch.float32)
        # optim/components/action_bounds.py:31: step_max = step_scale * |high - low|
        self.step_max = (cfg.step_scale * (action_bound_highs - action_bound_lows).abs()).to(dev, torch.float32).contiguous()
        self.clamp_step = cfg.step_scale not in (0.0, 1.0)
        self.cost_grad_fn = cost_grad_fn
        self.x_set, self.step_scaled = z(B, n, V), z(B, V)
        self.best_cost, self.best_action = z(B), z(B, V)
        self.best_iteration, self.current_iteration = z(B, dt=torch.int16), z(B, dt=torch.int16)
        self.converged = z(B, dt=torch.uint8)
        self.exploration_cost, self.exploration_action, self.exploration_gradient = z(B), z(B, V), z(B, V)
        self.cost, self.action, self.gradient = z(B), z(B, V), z(B, V)
        self.exploration_idx, self.selected_idx = z(B, n, dt=torch.int32), z(B, n, dt=torch.int32)

    def reset(self, x0: torch.Tensor) -> None:
        """Initial evaluation (gradient_opt_core.py:400-470): cost/grad at x0, best = x0, first step = -initial_step_scale * grad."""
        B, V, n = self.B, self.V, self.n
        self.qn.clear()
        self.current_iteration.zero_()
        self.best_iteration.zero_()
        self.converged.zero_()
        x0 = x0.reshape(B, V).contiguous()
        self.x_set.copy_(x0[:, None, :].expand(B, n, V))
        c, g = self.cost_grad_fn(self.x_set.view(B * n, V))
        c, g = c.view(B, n), g.view(B, n, V)
        self.exploration_action.copy_(x0)
        self.exploration_gradient.copy_(g[:, 0])
        self.exploration_cost.copy_(c[:, 0])
        self.action.copy_(x0)
        self.gradient.copy_(g[:, 0])
        self.cost.copy_(c[:, 0])
        self.best_cost.copy_(c[:, 0])
        self.best_action.copy_(x0)
        self.qn.set_reference(x0, g[:, 0])
        self._first = True

    def _step_direction(self) -> None:
        cfg, qn = self.cfg, self.qn
        if self._first:
            # no curvature pair yet: steepest descent scaled by initial_step_scale, through the same search-point set-up
            self._first = False
            step = (-cfg.initial_step_scale * self.exploration_gradient)
            if self.clamp_step:
                ratio = (step.view(self.B, self.H, self.D).abs() / self.step_max.view(1, 1, -1)).reshape(self.B, -1).amax(dim=1)
                step = step / ratio.clamp(min=1.0)[:, None]
            if cfg.fix_terminal_action and self.H > 1:
                step.view(self.B, self.H, self.D)[:, -1] = 0.0
            self.step_scaled.copy_(step)
            self.x_set.copy_(self.exploration_action[:, None, :] + self.magnitudes.view(1, -1, 1) * step[:, None, :])
            return
        optimization_cu.launch_lbfgs_step(
            qn.step_q_buffer, qn.rho, qn.y, qn.s, self.exploration_action, self.exploration_gradient, qn.x_0, qn.grad_0,
            cfg.epsilon, self.B, cfg.history, self.V, cfg.stable_mode, True, x_set=self.x_set, step_scaled=self.step_scaled,
            search_magnitudes=self.magnitudes, action_step_max=self.step_max if self.clamp_step else None,
            fix_terminal_action=cfg.fix_terminal_action, action_dim=self.D)

    def step(self) -> None:
        """One optimizer iteration: step direction + search points, rollout, line search."""
        cfg, B, V, n = self.cfg, self.B, self.V, self.n
        self._step_direction()
        c, g = self.cost_grad_fn(self.x_set.view(B * n, V))
        optimization_cu.launch_line_search(
            self.best_cost, self.best_action, self.best_iteration, self.current_iteration, self.converged,
            cfg.convergence_iteration, cfg.cost_delta_threshold, cfg.cost_relative_threshold, self.exploration_cost,
            self.exploration_action, self.exploration_gradient, self.exploration_idx.view(-1), self.cost, self.action,
            self.gradient, self.selected_idx.view(-1), c.view(B, n).contiguous(), self.x_set, g.view(B, n, V).contiguous(),
            self.step_scaled, self.magnitudes, cfg.line_search_wolfe_c_1, cfg.line_search_wolfe_c_2, cfg.strong_wolfe,
            cfg.approx_wolfe, n, V, B)

    def optimize(self, x0: torch.Tensor, num_iters: Optional[int] = None) -> torch.Tensor:
        self.reset(x0)
        for _ in range(num_iters if num_iters is not None else self.cfg.num_iters):
            self.step()
        return self.best_action.view(self.B, self.H, self.D)

    def optimize_graphed(self, x0: torch.Tensor, num_iters: Optional[int] = None) -> torch.Tensor:
        """The whole solve -- initial evaluation + `num_iters` x (step direction, rollout, line search) -- as ONE CUDA-graph
        launch (SURVEY.md 8f rank 2: "whole _opt_iters as one launch", gradient_opt_core.py:334-400, which the reference
        also replays from a graph, one graph per iteration block).  The first call runs one eager solve (allocations, launch-plan
        caches), captures the loop on a side stream and replays it; later calls copy x0 into the captured input and replay.
        Every buffer the loop touches is owned by this object or by the cost function's engine, so the replay is allocation
        free; `cost_grad_fn` must launch on the current stream and must not synchronise (RolloutEngine does neither)."""
        n_it = num_iters if num_iters is not None else self.cfg.num_iters
        g = getattr(self, "_graph", None)
        if g is None or self._graph_iters != n_it:
            self._graph_x0 = torch.empty((self.B, self.V), device=self.device, dtype=torch.float32)
            self._graph_x0.copy_(x0.reshape(self.B, self.V))
            self.optimize(self._graph_x0, n_it)                          # eager warm-up, same buffers
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.device(self.device), torch.cuda.graph(g):
                self.optimize(self._graph_x0, n_it)
            self._graph, self._graph_iters = g, n_it
        self._graph_x0.copy_(x0.reshape(self.B, self.V))
        self._graph.replay()
        return self.best_action.view(self.B, self.H, self.D)


def _capture_solve(owner, x0: torch.Tensor, shape: Tuple[int, ...]) -> torch.Tensor:
    """`owner.optimize` as one CUDA graph, replayed on every call with x0 copied into the captured input (the scheme of
    LBFGSOpt.optimize_graphed: one eager warm-up solve on the same buffers, then the capture).  Every buffer the solve
    touches is owned by `owner`'s stages or their cost functions' engines, so the replay allocates nothing."""
    if getattr(owner, "_graph", None) is None:
        owner._graph_x0 = torch.empty(shape, device=owner.device, dtype=torch.float32)
        owner._graph_x0.copy_(x0.reshape(shape))
        owner._graph_out = owner.optimize(owner._graph_x0)            # eager warm-up, same buffers
        torch.cuda.synchronize(owner.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.device(owner.device), torch.cuda.graph(g):
            owner._graph_out = owner.optimize(owner._graph_x0)
        owner._graph = g
    owner._graph_x0.copy_(x0.reshape(shape))
    owner._graph.replay()
    return owner._graph_out


@dataclass
class MPPIOptCfg:
    """The fields of MPPICfg (optim/particle/mppi.py:64-127) this loop uses; defaults = content/configs/task/ik/particle_ik.yml.
    Supported: DIAG_A covariance, CLAMP squash, BEST or MEAN sample mode, fixed or cycling sample sets."""
    num_iters: int = 4
    inner_iters: int = 4
    num_particles: int = 25
    init_cov: float = 1.0
    beta: float = 1.0
    kappa: float = 0.01
    step_size_mean: float = 0.9
    step_size_cov: float = 0.2
    gamma: float = 1.0
    null_act_frac: float = 0.0
    sample_mode: str = "BEST"
    update_cov: bool = True
    fixed_samples: bool = True
    sample_per_problem: bool = True
    seed: int = 0
    cov_type: str = "DIAG_A"
    squash_fn: str = "CLAMP"
    random_mean: bool = False


def mppi_particle_counts(num_particles: int, null_act_frac: float) -> Tuple[int, int, int]:
    """(sampled, negated-mean, zero) particles per problem, ParticleOptCore._init_particle_counts (particle_opt_core.py:190-203)."""
    n_null = round(int(null_act_frac * num_particles * 0.5))
    n_neg = round(int(null_act_frac * num_particles)) - n_null
    return num_particles - n_null - n_neg, n_neg, n_null


class MPPIOpt:
    """Batched MPPI over `num_problems` independent problems, three launches per inner iteration:

        cb200_mppi_sample  ->  cost_fn (the cost-only fused rollout)  ->  cb200_mppi_update

    `cost_fn(actions [P * Np, H, D]) -> cost [P * Np, H]`: rows are problem-major, particle-minor.  `noise`
    [n_sets, P or 1, Ns, H, D] (n_sets = 1 with fixed samples, else num_iters; 1 problem = one set shared by every problem)
    is copied into this object's buffer and the last sampled particle of every set is zeroed, as
    GaussianDistribution.initialize_samples does; the default is seeded torch normal noise (the reference's scrambled-Halton
    sample library is not reproduced).  Noise set k mod n_sets is used at global inner iteration k.

    In BEST mode the result is the best particle of the LAST inner iteration of the last outer iteration -- the reference's
    rule (mppi.py:214-218, particle_opt_core.py:464-465) -- not the best particle seen during the solve."""

    def __init__(self, cfg: MPPIOptCfg, num_problems: int, action_horizon: int, action_dim: int,
                 lows: torch.Tensor, highs: torch.Tensor, cost_fn: Callable[[torch.Tensor], torch.Tensor],
                 noise: Optional[torch.Tensor] = None, device="cuda:0"):
        if cfg.cov_type != "DIAG_A":
            raise ValueError(f"MPPIOpt supports cov_type DIAG_A only, got {cfg.cov_type}")
        if cfg.sample_mode not in ("BEST", "MEAN"):
            raise ValueError(f"MPPIOpt supports sample_mode BEST or MEAN, got {cfg.sample_mode}")
        if cfg.random_mean:
            raise ValueError("MPPIOpt does not support random_mean; the mean is updated from the weighted samples")
        if cfg.squash_fn != "CLAMP":
            raise ValueError(f"MPPIOpt supports squash_fn CLAMP only, got {cfg.squash_fn}")
        if cfg.num_iters < 1 or cfg.inner_iters < 1 or not cfg.beta > 0.0:
            raise ValueError("num_iters and inner_iters must be >= 1 and beta > 0")
        self.cfg, self.device = replace(cfg), torch.device(device)
        _tc.require_cuda(self.device, "MPPIOpt is CUDA-only")
        self.P, self.H, self.D, self.Np = num_problems, action_horizon, action_dim, cfg.num_particles
        self.Ns, self.n_neg, self.n_null = mppi_particle_counts(cfg.num_particles, cfg.null_act_frac)
        if self.Ns < 1:
            raise ValueError("null_act_frac leaves no sampled particle")
        P, H, D, dev = self.P, self.H, self.D, self.device
        self.n_sets = 1 if cfg.fixed_samples else cfg.num_iters
        shape = (self.n_sets, P if cfg.sample_per_problem else 1, self.Ns, H, D)
        if noise is None:
            gen = torch.Generator().manual_seed(cfg.seed)
            noise = torch.randn(shape, generator=gen, dtype=torch.float32)
        if tuple(noise.shape) != shape:
            raise ValueError(f"noise must be {shape}, got {tuple(noise.shape)}")
        self.noise = noise.to(dev, torch.float32).clone().contiguous()
        self.noise[:, :, -1] = 0.0
        self.lows = lows.to(dev, torch.float32).reshape(-1).contiguous()
        self.highs = highs.to(dev, torch.float32).reshape(-1).contiguous()
        if self.lows.numel() != D or self.highs.numel() != D:
            raise ValueError(f"lows / highs must have {D} entries")
        gamma_seq = torch.cumprod(torch.tensor([1.0] + [cfg.gamma] * (H - 1), dtype=torch.float32), 0)
        self.discount = float(gamma_seq.sum() / gamma_seq[0])
        self.cost_fn = cost_fn
        z = lambda *s: torch.zeros(s, device=dev, dtype=torch.float32)  # noqa: E731
        self.mean, self.best, self.action = z(P, H, D), z(P, H, D), z(P, H, D)
        self.cov, self.scale = z(P, D), z(P, D)
        self.actions = z(P, self.Np, H, D)
        self.outer_iters = -(-cfg.num_iters // cfg.inner_iters)

    def step(self, k: int) -> None:
        """One inner iteration with noise set k mod n_sets: sample, evaluate, update."""
        cfg, P, Np, H, D = self.cfg, self.P, self.Np, self.H, self.D
        optimization_cu.launch_mppi_sample(self.actions, self.mean, self.scale, self.noise[k % self.n_sets], self.lows,
                                           self.highs, self.n_neg)
        cost = self.cost_fn(self.actions.view(P * Np, H, D))
        upd = cfg.update_cov
        optimization_cu.launch_mppi_update(self.actions, cost, self.mean, self.cov if upd else None, self.scale if upd else None,
                                           self.best if cfg.sample_mode == "BEST" else None, cfg.beta, cfg.step_size_mean,
                                           cfg.step_size_cov, cfg.kappa, self.discount)

    def optimize(self, x0: torch.Tensor) -> torch.Tensor:
        """ParticleOptCore.optimize / _opt_iters (particle_opt_core.py:283-388) after reinitialize: the covariance is reset to
        init_cov and the sample index to 0; each outer iteration seeds mean and best with the current action, runs
        inner_iters x (sample, cost_fn, update) and takes best (BEST) or mean (MEAN) as the action.  Returns [P, H, D]."""
        cfg = self.cfg
        self.cov.fill_(cfg.init_cov)
        torch.sqrt(self.cov, out=self.scale)
        self.action.copy_(x0.reshape(self.P, self.H, self.D))
        k = 0
        for _ in range(self.outer_iters):
            self.mean.copy_(self.action)
            self.best.copy_(self.action)
            for _ in range(cfg.inner_iters):
                self.step(k)
                k += 1
            self.action.copy_(self.best if cfg.sample_mode == "BEST" else self.mean)
        return self.action

    def optimize_graphed(self, x0: torch.Tensor) -> torch.Tensor:
        """The whole stage as ONE CUDA-graph launch, as LBFGSOpt.optimize_graphed; `cost_fn` must launch on the current
        stream and must not synchronise (RolloutEngine.evaluate_cost does neither)."""
        return _capture_solve(self, x0, (self.P, self.H, self.D))


class MultiStageOpt:
    """Stages run in sequence, each seeded with the previous stage's best action (MultiStageOptimizer._opt_iters,
    optim/multi_stage_optimizer.py:96-180): MultiStageOpt([MPPIOpt(...), LBFGSOpt(...)]) is the reference's default two-stage
    IK.  Every stage must solve the same number of problems over the same action shape."""

    def __init__(self, stages: List):
        if not stages:
            raise ValueError("MultiStageOpt needs at least one stage")
        shapes = {(getattr(s, "P", getattr(s, "B", None)), s.H, s.D) for s in stages}
        if len(shapes) != 1:
            raise ValueError(f"stages disagree on (problems, horizon, action_dim): {sorted(shapes)}")
        self.stages = list(stages)
        self.shape = shapes.pop()
        self.device = stages[0].device

    def optimize(self, x0: torch.Tensor) -> torch.Tensor:
        x = x0.reshape(self.shape)
        for s in self.stages:
            x = s.optimize(x).view(self.shape)
        return x

    def optimize_graphed(self, x0: torch.Tensor) -> torch.Tensor:
        """Every stage in ONE CUDA graph: MPPI followed by L-BFGS is one launch."""
        return _capture_solve(self, x0, self.shape)
