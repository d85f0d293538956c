"""CPU ORACLE for the current-state block of the POSITION c-space cost (velocity-aware IK)  --  TEST INFRASTRUCTURE.

A float32 numpy restatement of cost/wp_cspace_position.py:299-356: when the seed's current state has dt > 0 the position
bounds, already shrunk by the activation distance, are intersected with the window one step of dt reaches from the current
position, and the implied velocity and acceleration are regularized.  `rollout_cost_grad` is rollout_oracle.rollout_cost_grad
with that block: the functions of rollout_oracle.py are left as they are, so their callers see no change, and the block is
added in the order rollout_oracle.rollout_cost_grad adds its c-space term.
Pinned on the reference's own source by tests/golden/cspace_position_current_state_golden.npz
(tests/golden/make_current_state_golden.py)."""
from __future__ import annotations

import numpy as np

from . import rollout_oracle as O

F = np.float32


def cspace_position_cost(pos, limits_p, weight, activation, target=None, idxs_target=None, target_weight=0.0,
                         target_dof_weight=None, current_position=None, current_velocity=None, idxs_current=None,
                         state_dt=None, limits_v=None, reg_weight=(0.0, 0.0)):
    """O.cspace_position_cost plus the current-state block (off when current_position is None: then it is O's function).

    pos [B,H,D]; limits_p / limits_v [2,D]; weight, activation (2,); current_position / current_velocity [n,D] (velocity
    None = 0); idxs_current [B] (None = row 0); state_dt [n]; reg_weight (2,) = squared_l2_regularization_weight (velocity,
    acceleration).  Returns cost [B,H,D], grad_p."""
    if current_position is None:
        return O.cspace_position_cost(pos, limits_p, weight, activation, target=target, idxs_target=idxs_target,
                                      target_weight=target_weight, target_dof_weight=target_dof_weight)
    x = np.asarray(pos, F)
    B, H, D = x.shape
    lp, lv = np.asarray(limits_p, F), np.asarray(limits_v, F)
    ci = np.zeros(B, np.int64) if idxs_current is None else np.asarray(idxs_current).astype(np.int64)
    dt = np.asarray(state_dt, F)[ci].reshape(B, 1, 1)
    cur_p = np.asarray(current_position, F)[ci][:, None, :]
    cur_v = np.zeros_like(cur_p) if current_velocity is None else np.asarray(current_velocity, F)[ci][:, None, :]
    on = dt > 0
    # :290-304 -- shrink, then the velocity window
    lo, hi = O._shrink(lp[0], lp[1], F(activation[0]))
    lo = np.where(on, np.maximum(lo[None, None], (cur_p + lv[0] * dt).astype(F)), lo[None, None]).astype(F)
    hi = np.where(on, np.minimum(hi[None, None], (cur_p + lv[1] * dt).astype(F)), hi[None, None]).astype(F)
    c, g = O._bound(x, lo, hi, F(weight[0]))                     # :312-320 (an empty window hinges on both sides)
    tw = F(target_weight) * (np.ones(D, F) if target_dof_weight is None else np.asarray(target_dof_weight, F))
    if target is not None and np.any(tw > 0):                    # :331-340
        tgt = np.asarray(target, F)[np.asarray(idxs_target).astype(np.int64)][:, None, :]
        e = (x - tgt).astype(F)
        t_on = tw > 0
        c = (c + np.where(t_on, tw * e * e, F(0))).astype(F)
        g = (g + np.where(t_on, F(2.0) * tw * e, F(0))).astype(F)
    # :345-356 -- weights retimed by dt and dt^2
    vw = (F(reg_weight[0]) * dt).astype(F)
    aw = (F(reg_weight[1]) * dt * dt).astype(F)
    sdt = np.where(on, dt, F(1)).astype(F)
    vi = ((x - cur_p) / sdt).astype(F)
    ai = ((vi - cur_v) / sdt).astype(F)
    v_on, a_on = on & (vw > 0), on & (aw > 0)
    c = (c + np.where(v_on, F(0.5) * vw * vi * vi, F(0))).astype(F)
    g = (g + np.where(v_on, vw * vi / sdt, F(0))).astype(F)
    c = (c + np.where(a_on, F(0.5) * aw * ai * ai, F(0))).astype(F)
    g = (g + np.where(a_on, aw * ai / (sdt * sdt), F(0))).astype(F)
    return c, g


def rollout_cost_grad(rm, q, cfg, current_position=None, current_velocity=None, idxs_current=None, state_dt=None, **kw):
    """O.rollout_cost_grad (same arguments in **kw) with the current-state block in the POSITION c-space term; the
    regularization weights are cfg["cspace_reg"][0:2], the velocity limits rm.velocity_limits.  The other terms come from
    O.rollout_cost_grad without a c-space term; the c-space term is then added in the order O.rollout_cost_grad adds it, so with
    current_position None (or dt <= 0 on every row) the result is O.rollout_cost_grad's to the bit."""
    if current_position is None or cfg.get("cspace_type") != "position":
        return O.rollout_cost_grad(rm, q, cfg, **kw)
    out = O.rollout_cost_grad(rm, q, dict(cfg, cspace_type=None), **kw)
    q = np.asarray(q, F)
    B = q.shape[0]
    tgt = kw.get("cspace_target")
    tgt_w = float(cfg.get("cspace_target_weight", 0.0)) if tgt is not None else 0.0
    tidx = kw.get("idxs_cspace_target")
    c, gp = cspace_position_cost(q, rm.position_limits, cfg["cspace_weight"], cfg["cspace_activation"],
                                 target=tgt if tgt_w > 0 else None, idxs_target=np.zeros(B, np.int64) if tidx is None else tidx,
                                 target_weight=tgt_w, target_dof_weight=kw.get("cspace_target_dof_weight"),
                                 current_position=current_position, current_velocity=current_velocity,
                                 idxs_current=idxs_current, state_dt=state_dt, limits_v=rm.velocity_limits,
                                 reg_weight=list(cfg.get("cspace_reg", (0.0, 0.0)))[:2])
    out["cspace_cost"], out["cspace_grad_p"] = c, gp
    out["cost_bh"] += np.sum(c, axis=-1)
    out["grad_q"] = (out["grad_q"] + gp).astype(F)
    out["cost"] = np.sum(out["cost_bh"], axis=1).astype(F)
    return out
