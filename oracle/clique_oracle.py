"""CPU ORACLE for the position (clique) and acceleration control-space transitions  --  TEST INFRASTRUCTURE, NOT PRODUCT.

Only tests/ and scripts/ may import this module; curobo_b200/ never does.

Numpy restatement of the reference's legacy kernels (paths relative to curobo/_src/curobolib/kernels/trajectory/legacy/):
  clique_forward    <- differentiation_position_kernel.cuh:18-231 (row logic), :406-466 (kernel)
  clique_backward   <- differentiation_position_kernel.cuh:236-401
  integrate_acc     <- integration_acceleration_kernel.cuh:13-139

`dtype=np.float32` follows the kernels' precision: float32 everywhere except where the reference writes double literals
(`1.0 / dt`, `2.0 * dt * v` in the start padding, the unsuffixed stencil coefficients of the adjoint), which are
evaluated in float64 and rounded where the kernel assigns to a float.  numpy neither contracts a * b + c into an FMA
nor approximates division, so against the GPU (--fmad=true --prec-div=false) the float32 variant agrees to float
rounding, not bit for bit.  `dtype=np.float64` evaluates the same formulas in float64 throughout: the forward is then
an affine map of u and the adjoint checks compare the backward with its exact transpose.
"""
from __future__ import annotations

import numpy as np

F = np.float32

# 5-point stencil coefficients as the kernels write them (:201-220 forward, :349-389 backward)
_V = (0.083333333, -0.666666667, 0.666666667, -0.083333333)                     # rows 0, 1, 3, 4
_A = (-0.083333333, 1.333333333, -2.5, 1.333333333, -0.083333333)
_J = (-0.5, 1.0, -1.0, 0.5)                                                     # rows 0, 1, 3, 4


def _c(x, dt):
    return np.asarray(x, dtype=dt)


def _start_padding(p, v, a, dt, dtype):
    """Waypoints -2, -1, 0 extrapolated back from the start state at zero jerk (:83-91)."""
    f64 = dtype == np.float64
    one_half, seven_sixths, four_thirds = _c(1.5, dtype), _c(7.0 / 6.0, dtype), _c(4.0 / 3.0, dtype)
    if f64:
        w0 = -one_half * a * dt * dt - seven_sixths * dt * dt * dt * 0.0 - dt * v + p
        wm1 = -2.0 * a * dt * dt - four_thirds * dt * dt * dt * 0.0 - 2.0 * dt * v + p
        wm2 = one_half * (-1 * a * (dt * dt) - (dt * dt * dt) * 0.0) - 3.0 * dt * v + p
        return wm2, wm1, w0
    z = F(0)
    w0 = (-F(1.5) * a * dt * dt - F(7.0 / 6.0) * dt * dt * dt * z - dt * v + p).astype(F)
    head = (-F(2.0) * a * dt * dt - F(4.0 / 3.0) * dt * dt * dt * z).astype(F)
    wm1 = (head.astype(np.float64) - 2.0 * dt.astype(np.float64) * v.astype(np.float64) + p.astype(np.float64)).astype(F)
    wm2 = (F(1.5) * (-a * (dt * dt) - (dt * dt * dt) * z) - F(3.0) * dt * v + p).astype(F)
    return wm2, wm1, w0


def clique_forward(u, start_position, start_velocity, start_acceleration, goal_position, start_idx, goal_idx, traj_dt,
                   implicit, horizon, dtype=F):
    """u [B, H-4, D] -> (position, velocity, acceleration, jerk [B, H, D], out_dt [B]).  start_* / goal_position are
    gathered at flat offsets start_idx[b] * D / goal_idx[b] * D; traj_dt / implicit are indexed through goal_idx."""
    H = int(horizon)
    u = np.asarray(u, dtype)
    B, n, D = u.shape
    assert n == H - 4 and H >= 8
    sp, sv, sa = (np.asarray(x, dtype).reshape(-1, D)[np.asarray(start_idx)] for x in
                  (start_position, start_velocity, start_acceleration))
    gp = np.asarray(goal_position, dtype).reshape(-1, D)[np.asarray(goal_idx)]
    dt32 = np.asarray(traj_dt, F).reshape(-1)[np.asarray(goal_idx)]
    dt = dt32.astype(dtype)[:, None]
    use_goal = np.asarray(implicit).reshape(-1)[np.asarray(goal_idx)] != 0
    dt_inv = (1.0 / dt.astype(np.float64)).astype(dtype)
    wm2, wm1, w0 = _start_padding(sp, sv, sa, dt, dtype)
    # waypoints w = -2 .. H+1 at index w + 2; past the last action they repeat it
    W = np.concatenate([wm2[:, None], wm1[:, None], w0[:, None], sp[:, None], u, np.repeat(u[:, -1:], 4, axis=1)], axis=1)
    Wg = W.copy()                              # rows >= 4: the implicit goal replaces the last action and what repeats it
    Wg[use_goal, n + 3:] = gp[use_goal][:, None]
    pos, vel, acc, jerk = (np.zeros((B, H, D), dtype) for _ in range(4))
    c = lambda x: _c(x, dtype)  # noqa: E731
    for h in range(H):
        src = W if h <= 3 else Wg              # the reference tests h == 0..3 before h == H-5 .. H-1 (matters at H = 8)
        i0, i1, i2, i3, i4 = (src[:, h + k] for k in range(5))
        pos[:, h] = i2
        vel[:, h] = (c(_V[0]) * i0 - c(-_V[1]) * i1 + c(_V[2]) * i3 + c(_V[3]) * i4) * dt_inv
        acc[:, h] = (c(_A[0]) * i0 + c(_A[1]) * i1 + c(_A[2]) * i2 + c(_A[3]) * i3 + c(_A[4]) * i4) * dt_inv * dt_inv
        jerk[:, h] = (c(_J[0]) * i0 + i1 - i3 + c(_J[3]) * i4) * (dt_inv * dt_inv * dt_inv)
    return pos, vel, acc, jerk, dt32.copy()


def clique_backward(grad_position, grad_velocity, grad_acceleration, grad_jerk, traj_dt, dt_idx, implicit, dtype=F):
    """The four gradients [B, H, D] -> d loss / d u [B, H-4, D], as the reference's adjoint computes it (:236-401)."""
    gp, gv, ga, gj = (np.asarray(g, dtype) for g in (grad_position, grad_velocity, grad_acceleration, grad_jerk))
    B, H, D = gp.shape
    n = H - 4
    dt = np.asarray(traj_dt, F).reshape(-1)[np.asarray(dt_idx)].astype(dtype)[:, None]
    use_goal = np.asarray(implicit).reshape(-1)[np.asarray(dt_idx)] != 0
    dt_inv = (dtype(1.0) / dt).astype(dtype)
    d2 = (dt_inv * dt_inv).astype(dtype)
    d3 = (d2 * dt_inv).astype(dtype)
    f64 = lambda x: np.asarray(x, np.float64)  # noqa: E731
    out = np.zeros((B, n, D), dtype)
    for i in range(n):
        V, A, J = (gv[:, i + k] for k in range(5)), (ga[:, i + k] for k in range(5)), [gj[:, i + k] for k in range(5)]
        V, A = [f64(x) for x in V], [f64(x) for x in A]
        o = gp[:, i + 2].copy()
        if i < n - 1:
            sv = -0.0833333330000000 * V[0] + 0.666666667000000 * V[1] + 0 * V[2] - 0.666666667000000 * V[3] + \
                0.0833333330000000 * V[4]
            o = (f64(o) + sv * f64(dt_inv)).astype(dtype)
            sa = -0.0833333330000000 * A[0] + 1.33333333300000 * A[1] + (-2.5) * A[2] + 1.33333333300000 * A[3] + \
                (-0.0833333330000000) * A[4]
            o = (f64(o) + sa * f64(d2)).astype(dtype)
            sj = (dtype(0.5) * J[0] - dtype(1.0) * J[1] + dtype(1.0) * J[3] - dtype(0.5) * J[4]) * d3
            o = (o + sj).astype(dtype)
        else:
            o = (o + (gp[:, i + 3] + gp[:, i + 4])).astype(dtype)
            sv = -0.0833333330000000 * V[0] + 0.583333334000000 * V[1] + 0.583333334000000 * V[2] - \
                0.0833333330000000 * V[3] + 0.0 * V[4]
            o = (f64(o) + sv * f64(dt_inv)).astype(dtype)
            sa = -0.0833333330000000 * A[0] + 1.25 * A[1] + (-1.25) * A[2] + 0.0833333330000000 * A[3]
            o = (f64(o) + sa * f64(d2)).astype(dtype)
            sj = (0.5 * f64(J[0]) - 0.5 * f64(J[1]) - 0.5 * f64(J[2]) + 0.5 * f64(J[3])) * f64(d3)
            o = (f64(o) + sj).astype(dtype)
            o[use_goal] = 0.0
        out[:, i] = o
    return out


def integrate_acceleration(u_acc, start_position, start_velocity, start_acceleration, start_idx, traj_dt, dtype=F):
    """u_acc [B, H, D] -> (position, velocity, acceleration, jerk [B, H, D]) by semi-implicit Euler with dt[h] = traj_dt[h]
    (integration_acceleration_kernel.cuh:49-61)."""
    u = np.asarray(u_acc, dtype)
    B, H, D = u.shape
    dt = np.asarray(traj_dt, dtype).reshape(-1)
    sidx = np.asarray(start_idx)
    pos, vel, acc, jerk = (np.zeros((B, H, D), dtype) for _ in range(4))
    pos[:, 0] = np.asarray(start_position, dtype).reshape(-1, D)[sidx]
    vel[:, 0] = np.asarray(start_velocity, dtype).reshape(-1, D)[sidx]
    acc[:, 0] = np.asarray(start_acceleration, dtype).reshape(-1, D)[sidx]
    for h in range(1, H):
        acc[:, h] = u[:, h - 1]
        vel[:, h] = vel[:, h - 1] + acc[:, h] * dt[h]
        pos[:, h] = pos[:, h - 1] + vel[:, h] * dt[h]
        jerk[:, h] = (acc[:, h] - acc[:, h - 1]) / dt[h]
    return pos, vel, acc, jerk
