"""`optimization` kernel-backend module: same function names and argument order as
curobo/_src/curobolib/backends/cuda_core_backend/optimization.py:26-246 (pybind twins:
backends/pybind/line_search_kernel_launch.cu, lbfgs_step_kernel_launch.cu), SURVEY.md section 8f rank 2.
Tensors are validated (device, contiguity, dtype) BEFORE launch; errors raise; launches go to the current stream.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from .. import lib as _lib
from .tensor_checks import check_tensors, stream_ptr


def launch_line_search(
    best_cost: torch.Tensor,
    best_action: torch.Tensor,
    best_iteration: torch.Tensor,
    current_iteration: torch.Tensor,
    converged_global: torch.Tensor,
    convergence_iteration: int,
    cost_delta_threshold: float,
    cost_relative_threshold: float,
    exploration_cost: torch.Tensor,
    exploration_action: torch.Tensor,
    exploration_gradient: torch.Tensor,
    exploration_idx: torch.Tensor,
    selected_cost: torch.Tensor,
    selected_action: torch.Tensor,
    selected_gradient: torch.Tensor,
    selected_idx: torch.Tensor,
    search_cost: torch.Tensor,
    search_action: torch.Tensor,
    search_gradient: torch.Tensor,
    step_direction: torch.Tensor,
    search_magnitudes: torch.Tensor,
    armijo_threshold_c_1: float,
    curvature_threshold_c_2: float,
    strong_wolfe: bool,
    approx_wolfe: bool,
    n_linesearch: int,
    opt_dim: int,
    batchsize: int,
) -> None:
    """Parallel Wolfe line search + best / convergence bookkeeping; every output is written in place."""
    if n_linesearch > 32:
        raise RuntimeError("n_linesearch greater than 32 is not supported")
    if opt_dim > 1024:
        raise RuntimeError("opt_dim greater than 1024 is not supported")
    dev = search_cost.device
    check_tensors(dev, torch.float32, best_cost=best_cost, best_action=best_action, exploration_cost=exploration_cost,
                  exploration_action=exploration_action, exploration_gradient=exploration_gradient,
                  selected_cost=selected_cost, selected_action=selected_action, selected_gradient=selected_gradient,
                  search_cost=search_cost, search_action=search_action, search_gradient=search_gradient,
                  step_direction=step_direction, search_magnitudes=search_magnitudes)
    check_tensors(dev, torch.int16, best_iteration=best_iteration, current_iteration=current_iteration)
    check_tensors(dev, torch.uint8, converged_global=converged_global)
    check_tensors(dev, torch.int32, exploration_idx=exploration_idx, selected_idx=selected_idx)
    L = _lib.load()
    err = L.cb200_line_search(
        best_cost.data_ptr(), best_action.data_ptr(), best_iteration.data_ptr(), current_iteration.data_ptr(),
        converged_global.data_ptr(), int(convergence_iteration), float(cost_delta_threshold),
        float(cost_relative_threshold), exploration_cost.data_ptr(), exploration_action.data_ptr(),
        exploration_gradient.data_ptr(), exploration_idx.data_ptr(), selected_cost.data_ptr(),
        selected_action.data_ptr(), selected_gradient.data_ptr(), selected_idx.data_ptr(), search_cost.data_ptr(),
        search_action.data_ptr(), search_gradient.data_ptr(), step_direction.data_ptr(), search_magnitudes.data_ptr(),
        float(armijo_threshold_c_1), float(curvature_threshold_c_2), int(bool(strong_wolfe)), int(bool(approx_wolfe)),
        int(n_linesearch), int(opt_dim), int(batchsize), stream_ptr(dev))
    _lib.check(err, "launch_line_search")


def launch_lbfgs_step(
    step_vec: torch.Tensor,
    rho_buffer: torch.Tensor,
    y_buffer: torch.Tensor,
    s_buffer: torch.Tensor,
    q: torch.Tensor,
    grad_q: torch.Tensor,
    x_0: torch.Tensor,
    grad_0: torch.Tensor,
    epsilon: float,
    batch_size: int,
    history_m: int,
    v_dim: int,
    stable_mode: bool,
    use_shared_buffers: bool = True,
    x_set: Optional[torch.Tensor] = None,
    step_scaled: Optional[torch.Tensor] = None,
    search_magnitudes: Optional[torch.Tensor] = None,
    action_step_max: Optional[torch.Tensor] = None,
    fix_terminal_action: bool = False,
    action_dim: int = 0,
) -> List[torch.Tensor]:
    """L-BFGS two-loop step + history roll, in place.  Returns [step_vec, rho_buffer, y_buffer, s_buffer, x_0, grad_0]
    like the reference.  `use_shared_buffers` is accepted for signature parity (the history is always staged on
    chip for v_dim <= 32).  The five keyword arguments after it are this library's optional fused line-search
    set-up (include/curobo_b200.h): x_set [B,n,V] = q + magnitudes * scale_action(step)."""
    if history_m > 31:
        raise RuntimeError("History_m greater than 31 is not supported")  # optimization.py:173-174
    if history_m < 0:
        raise RuntimeError("History_m less than 0 is not supported")
    dev = step_vec.device
    check_tensors(dev, torch.float32, step_vec=step_vec, rho_buffer=rho_buffer, y_buffer=y_buffer, s_buffer=s_buffer, q=q,
                  grad_q=grad_q, x_0=x_0, grad_0=grad_0)
    n_ls, adim = 0, 0
    if x_set is not None:
        check_tensors(dev, torch.float32, x_set=x_set, search_magnitudes=search_magnitudes)
        n_ls = int(search_magnitudes.numel())
        if step_scaled is not None:
            check_tensors(dev, torch.float32, step_scaled=step_scaled)
        if action_step_max is not None:
            check_tensors(dev, torch.float32, action_step_max=action_step_max)
            adim = int(action_step_max.numel())
        if action_dim > 0:   # explicit: the terminal action is frozen whether or not the step is clamped
            if action_step_max is not None and int(action_step_max.numel()) != int(action_dim):
                raise ValueError("action_step_max must have action_dim entries")
            adim = int(action_dim)
    L = _lib.load()
    p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    err = L.cb200_lbfgs_step(
        step_vec.data_ptr(), rho_buffer.data_ptr(), y_buffer.data_ptr(), s_buffer.data_ptr(), q.data_ptr(),
        grad_q.data_ptr(), x_0.data_ptr(), grad_0.data_ptr(), float(epsilon), int(batch_size), int(history_m), int(v_dim),
        int(bool(stable_mode)), p(x_set), p(step_scaled), p(search_magnitudes), n_ls, p(action_step_max), adim,
        int(bool(fix_terminal_action)), stream_ptr(dev))
    _lib.check(err, "launch_lbfgs_step")
    return [step_vec, rho_buffer, y_buffer, s_buffer, x_0, grad_0]


def launch_mppi_sample(actions: torch.Tensor, mean: torch.Tensor, scale: torch.Tensor, noise: torch.Tensor,
                       lows: torch.Tensor, highs: torch.Tensor, num_neg: int = 0) -> torch.Tensor:
    """MPPI particles (ParticleOptCore.sample_actions, DIAG_A + CLAMP) into actions [P, Np, H, D]: per problem the
    Ns = noise.shape[1] sampled particles mean + noise * scale, then `num_neg` copies of -mean, then zeros, clamped to
    [lows, highs].  mean [P, H, D], scale [P, D], noise [P or 1, Ns, H, D] (1: one sample set for every problem),
    lows / highs [D].  This library's extension of the reference's kernel set (the reference builds particles in torch)."""
    dev = actions.device
    check_tensors(dev, torch.float32, actions=actions, mean=mean, scale=scale, noise=noise, lows=lows, highs=highs)
    if actions.ndim != 4:
        raise ValueError(f"actions must be [P, Np, H, D], got {tuple(actions.shape)}")
    P, Np, H, D = actions.shape
    if noise.ndim != 4 or noise.shape[0] not in (1, P) or tuple(noise.shape[2:]) != (H, D):
        raise ValueError(f"noise must be [{P} or 1, Ns, {H}, {D}], got {tuple(noise.shape)}")
    Ns = int(noise.shape[1])
    if tuple(mean.shape) != (P, H, D) or tuple(scale.shape) != (P, D) or lows.numel() != D or highs.numel() != D:
        raise ValueError("mean must be [P, H, D], scale [P, D], lows / highs [D]")
    if Ns < 1 or num_neg < 0 or Ns + num_neg > Np:
        raise ValueError(f"{Ns} sampled + {num_neg} negated particles do not fit {Np} particles")
    if P == 0:
        return actions                        # empty tensors have no storage to hand the kernel
    err = _lib.load().cb200_mppi_sample(actions.data_ptr(), mean.data_ptr(), scale.data_ptr(), noise.data_ptr(), lows.data_ptr(),
                                        highs.data_ptr(), P, Np, Ns, int(num_neg), H, D, int(noise.shape[0] == P and P > 1),
                                        stream_ptr(dev))
    _lib.check(err, "launch_mppi_sample")
    return actions


def launch_mppi_update(actions: torch.Tensor, cost: torch.Tensor, mean: torch.Tensor, cov: Optional[torch.Tensor],
                       scale: Optional[torch.Tensor], best: Optional[torch.Tensor], beta: float, step_size_mean: float,
                       step_size_cov: float, kappa: float, discount: float = 1.0) -> None:
    """MPPI distribution update (MPPI._update_distribution with jit_mean_cov_diag_a) from actions [P, Np, H, D] and their
    row costs [P * Np, H], in place: mean [P, H, D]; cov / scale [P, D] when both are given (update_cov); best [P, H, D]
    = the particle of largest weight when given (BEST mode).  `discount` = sum_h gamma^h / gamma^0."""
    dev = mean.device
    check_tensors(dev, torch.float32, actions=actions, cost=cost, mean=mean)
    if actions.ndim != 4:
        raise ValueError(f"actions must be [P, Np, H, D], got {tuple(actions.shape)}")
    P, Np, H, D = actions.shape
    if cost.numel() != P * Np * H or cost.shape[0] != P * Np or tuple(mean.shape) != (P, H, D):
        raise ValueError(f"cost must be [{P * Np}, {H}] and mean [{P}, {H}, {D}]")
    if (cov is None) != (scale is None):
        raise ValueError("cov and scale are updated together: pass both or neither")
    if cov is not None:
        check_tensors(dev, torch.float32, cov=cov, scale=scale)
        if tuple(cov.shape) != (P, D) or tuple(scale.shape) != (P, D):
            raise ValueError(f"cov / scale must be [{P}, {D}]")
    if best is not None:
        check_tensors(dev, torch.float32, best=best)
        if tuple(best.shape) != (P, H, D):
            raise ValueError(f"best must be [{P}, {H}, {D}]")
    if not beta > 0.0:
        raise ValueError("beta must be positive")
    if P == 0:
        return
    p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    err = _lib.load().cb200_mppi_update(actions.data_ptr(), cost.data_ptr(), mean.data_ptr(), p(cov), p(scale), p(best), P, Np, H, D,
                                        float(beta), float(step_size_mean), float(step_size_cov), float(kappa), float(discount),
                                        int(cov is not None), int(best is not None), stream_ptr(dev))
    _lib.check(err, "launch_mppi_update")
