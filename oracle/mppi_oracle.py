"""CPU ORACLE for the MPPI particle stage  --  TEST INFRASTRUCTURE, NOT PRODUCT.

Numpy restatement of the reference's MPPI for DIAG_A covariance and CLAMP squash (paths relative to curobo/_src/):
  sample    optim/components/particle_opt_core.py:409-441 (sample_actions) + optim/particle/particle_opt_utils.py:20-28
  update    optim/particle/mppi.py:200-248 (_update_distribution) + mppi.py:630-757 (jit_* helpers)
  optimize  optim/components/particle_opt_core.py:283-388 (optimize / _opt_iters) after reinitialize
in float32 (`dtype=np.float32`: every sum in the order of cb200_mppi_update -- per particle serial over the horizon, serial
over the particles -- so the kernel and this oracle agree to rounding of exp) or float64.  Only tests/ and bench scripts
may import this module.
"""
from __future__ import annotations

import math

import numpy as np


def particle_counts(num_particles: int, null_act_frac: float):
    """(sampled, negated-mean, zero) particles per problem (particle_opt_core.py:190-203)."""
    n_null = round(int(null_act_frac * num_particles * 0.5))
    n_neg = round(int(null_act_frac * num_particles)) - n_null
    return num_particles - n_null - n_neg, n_neg, n_null


def discount_factor(gamma: float, horizon: int, dtype=np.float32):
    """sum_h gamma^h / gamma^0 of the reference's gamma_seq (particle_opt_core.py:149-154)."""
    seq = np.cumprod(np.array([1.0] + [gamma] * (horizon - 1), dtype))
    return dtype(seq.sum(dtype=dtype) / seq[0])


def sample(mean, scale, noise, lows, highs, num_particles: int, num_neg: int, dtype=np.float32):
    """actions [P, Np, H, D]: noise [P or 1, Ns, H, D] -> mean + noise * scale; then -mean x num_neg; then zeros; clamped."""
    mean, scale, noise = (np.asarray(x, dtype) for x in (mean, scale, noise))
    P, H, D = mean.shape
    Ns = noise.shape[1]
    out = np.zeros((P, num_particles, H, D), dtype)
    out[:, :Ns] = mean[:, None] + (noise * scale[:, None, None, :]).astype(dtype)
    out[:, Ns:Ns + num_neg] = -mean[:, None]
    return np.maximum(np.minimum(out, np.asarray(highs, dtype)), np.asarray(lows, dtype))


def weights(cost, P: int, Np: int, beta: float, discount, dtype=np.float32):
    """softmax(-discount * sum_h cost / beta) per problem: cost [P * Np, H] -> w [P, Np]."""
    c = np.asarray(cost, dtype).reshape(P, Np, -1)
    s = np.zeros((P, Np), dtype)
    for h in range(c.shape[2]):
        s = (s + c[:, :, h]).astype(dtype)
    x = (dtype(-1.0 / beta) * (dtype(discount) * s).astype(dtype)).astype(dtype)
    e = np.exp((x - x.max(axis=1, keepdims=True)).astype(dtype)).astype(dtype)
    se = np.zeros(P, dtype)
    for j in range(Np):
        se = (se + e[:, j]).astype(dtype)
    return (e / se[:, None]).astype(dtype)


def update(actions, cost, mean, cov, beta, step_size_mean, step_size_cov, kappa, discount, update_cov=True, best_mode=True,
           dtype=np.float32):
    """One MPPI distribution update.  Returns dict(mean, cov, scale, best, w, best_idx); cov / scale unchanged when not
    update_cov (scale then None), best None when not best_mode."""
    a = np.asarray(actions, dtype)
    P, Np, H, D = a.shape
    mo, cv = np.asarray(mean, dtype), np.asarray(cov, dtype)
    w = weights(cost, P, Np, beta, discount, dtype)
    m = np.zeros((P, H, D), dtype)
    c = np.zeros((P, H, D), dtype)
    for j in range(Np):
        wj = w[:, j, None, None]
        dl = (a[:, j] - mo).astype(dtype)
        m = (m + (wj * a[:, j]).astype(dtype)).astype(dtype)
        c = (c + (wj * (dl * dl).astype(dtype)).astype(dtype)).astype(dtype)
    out = dict(w=w, best_idx=np.argmax(w, axis=1), best=None, scale=None, cov=cv)
    out["mean"] = ((dtype(1.0 - step_size_mean) * mo).astype(dtype) + (dtype(step_size_mean) * m).astype(dtype)).astype(dtype)
    if update_cov:
        s = np.zeros((P, D), dtype)
        for h in range(H):
            s = (s + c[:, h]).astype(dtype)
        upd = (s / dtype(H)).astype(dtype)
        new = ((dtype(1.0 - step_size_cov) * cv).astype(dtype) + (dtype(step_size_cov) * upd).astype(dtype)).astype(dtype)
        out["cov"] = (new + dtype(kappa)).astype(dtype)
        out["scale"] = np.sqrt(out["cov"]).astype(dtype)
    if best_mode:
        out["best"] = a[np.arange(P), out["best_idx"]].copy()
    return out


def optimize(x0, noise_sets, lows, highs, cost_fn, num_iters=4, inner_iters=4, num_particles=25, init_cov=1.0, beta=1.0,
             kappa=0.01, step_size_mean=0.9, step_size_cov=0.2, gamma=1.0, null_act_frac=0.0, sample_mode="BEST",
             update_cov=True, dtype=np.float32):
    """The particle stage: noise_sets [n_sets, P or 1, Ns, H, D] (the last sampled particle already zeroed); set k mod n_sets
    at global inner iteration k.  cost_fn(actions [P * Np, H, D]) -> [P * Np, H].  Returns (action [P, H, D], records) with one
    record per inner iteration: actions, cost, and mean / cov / scale / best after the update."""
    x0 = np.asarray(x0, dtype)
    P, H, D = x0.shape
    Ns, n_neg, _ = particle_counts(num_particles, null_act_frac)
    g = discount_factor(gamma, H, dtype)
    cov = np.full((P, D), init_cov, dtype)
    scale = np.sqrt(cov).astype(dtype)
    action, records, k = x0.copy(), [], 0
    for _ in range(math.ceil(num_iters / inner_iters)):
        mean, best = action.copy(), action.copy()
        for _ in range(inner_iters):
            acts = sample(mean, scale, noise_sets[k % len(noise_sets)], lows, highs, num_particles, n_neg, dtype)
            k += 1
            cost = np.asarray(cost_fn(acts.reshape(P * num_particles, H, D)), dtype)
            o = update(acts, cost, mean, cov, beta, step_size_mean, step_size_cov, kappa, g, update_cov, sample_mode == "BEST", dtype)
            mean, cov = o["mean"], o["cov"]
            if update_cov:
                scale = o["scale"]
            if sample_mode == "BEST":
                best = o["best"]
            records.append(dict(actions=acts, cost=cost, mean=mean, cov=cov, scale=scale, best=best))
        action = (best if sample_mode == "BEST" else mean).copy()
    return action, records
