#!/usr/bin/env python
"""Golden iterates of the reference's own MPPI (curobo/_src/optim/particle/mppi.py over ParticleOptCore), imported from
/root/reference in the build container and run on the CPU through `_core._opt_iters` (`optimize` needs a CUDA timer).

    python tests/golden/make_mppi_golden.py        # rewrites tests/golden/mppi_reference_torch.npz

The rollout is a synthetic quadratic defined here: cost[b, h] = sum_d w_d (a[b, h, d] - target[problem(b), h, d])^2 on
problem-major, particle-minor rows.  Stored per case: the configuration, the reference's sample set (the last sampled
particle zeroed), the seed, the bounds, the target, and per inner iteration the actions, the row costs and the
distribution after the update (mean, cov, scale, best), plus the action the stage returns.
"""
import json
import math
import os
import sys
import zlib
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [HERE, ROOT, os.environ.get("CUROBO_REFERENCE", "/root/reference")]

CASES = {
    # name: (P, H, D, MPPICfg overrides)
    "ik": (6, 1, 7, dict()),
    "horizon": (4, 4, 3, dict(gamma=0.98, null_act_frac=0.2, num_particles=20)),
    "mean_nocov": (5, 2, 4, dict(sample_mode="MEAN", update_cov=False, num_particles=16)),
    "cycling": (3, 2, 5, dict(fixed_samples=False, num_iters=3, inner_iters=2, num_particles=12)),
}
BASE = dict(num_iters=4, inner_iters=4, num_particles=25, init_cov=1.0, beta=1.0, kappa=0.01, step_size_mean=0.9,
            step_size_cov=0.2, gamma=1.0, null_act_frac=0.0, sample_mode="BEST", update_cov=True, fixed_samples=True)


class QuadraticRollout:
    """The pieces of the Rollout protocol ParticleOptCore reads, over a batched quadratic cost."""

    def __init__(self, P, H, D, Np, target, weight, lows, highs):
        self.P, self.horizon, self.action_horizon, self.action_dim, self.Np = P, H, H, D, Np
        self.target, self.weight = target, weight
        self.action_bound_lows, self.action_bound_highs = lows, highs
        self.log = []

    def get_initial_action(self):
        return torch.zeros(self.action_horizon, self.action_dim)

    def update_batch_size(self, batch_size=None, **kw):
        pass

    def cost(self, acts):
        a = acts.view(self.P, self.Np, self.horizon, self.action_dim)
        return (self.weight * (a - self.target[:, None]) ** 2).sum(-1).reshape(self.P * self.Np, self.horizon)

    def evaluate_action(self, act_seq):
        c = self.cost(act_seq)
        self.log.append((act_seq.clone(), c.clone()))

        def total(sum_horizon=False):
            return c.sum(-1, keepdim=True) if sum_horizon else c
        return SimpleNamespace(actions=act_seq, costs_and_constraints=SimpleNamespace(get_sum_cost_and_constraint=total),
                               state=None)


def run_case(name, P, H, D, over):
    from curobo._src.optim.particle.mppi import MPPI, MPPICfg
    from curobo._src.types.device_cfg import DeviceCfg
    cfg = dict(BASE, **over)
    torch.manual_seed(zlib.crc32(name.encode()) % 1000)
    dev = DeviceCfg(device=torch.device("cpu"))
    lows, highs = -torch.rand(D) - 0.5, torch.rand(D) + 0.5
    target = (torch.rand(P, H, D) * 2.0 - 1.0) * 0.8
    weight = torch.rand(D) + 0.5
    roll = QuadraticRollout(P, H, D, cfg["num_particles"], target, weight, lows, highs)
    seed = 23
    mcfg = MPPICfg(num_iters=cfg["num_iters"], inner_iters=cfg["inner_iters"], num_particles=cfg["num_particles"],
                   init_cov=cfg["init_cov"], beta=cfg["beta"], kappa=cfg["kappa"], step_size_mean=cfg["step_size_mean"],
                   step_size_cov=cfg["step_size_cov"], gamma=cfg["gamma"], null_act_frac=cfg["null_act_frac"],
                   sample_mode=cfg["sample_mode"], update_cov=cfg["update_cov"], num_problems=P, device_cfg=dev,
                   sample_params=dict(fixed_samples=cfg["fixed_samples"], seed=seed,
                                      sample_ratio={"halton": 1.0, "halton-knot": 0.0, "random": 0.0, "random-knot": 0.0,
                                                    "stomp": 0.0}),
                   sample_per_problem=True, squash_fn="CLAMP", cov_type="DIAG_A")
    opt = MPPI(mcfg, [roll])
    core = opt._core
    core.reinitialize(torch.zeros(P, H, D))
    sample_set = core._dist._sample_set.clone()
    x0 = (torch.rand(P, H, D) * 2.0 - 1.0) * 0.5
    from curobo._src.optim.components.particle_opt_core import OptimizationIterationState
    state = OptimizationIterationState(action=x0.clone(), exploration_action=x0.clone())
    rec = {k: [] for k in ("mean", "cov", "scale", "best")}
    orig_update = core._update_distribution_fn

    def recording_update(traj):
        orig_update(traj)
        d = core._dist
        rec["mean"].append(d.mean.clone())
        rec["cov"].append(d.cov.reshape(P, D).clone())
        rec["scale"].append(d.scale_tril.reshape(P, D).clone())
        rec["best"].append(d.best_traj.clone())
    core._update_distribution_fn = recording_update
    for _ in range(math.ceil(cfg["num_iters"] / cfg["inner_iters"])):
        state = core._opt_iters(state)
    out = {"config": np.array(json.dumps(dict(cfg, P=P, H=H, D=D, seed=seed))), "noise": sample_set.numpy(),
           "x0": x0.numpy(), "lows": lows.numpy(), "highs": highs.numpy(), "target": target.numpy(), "weight": weight.numpy(),
           "actions": torch.stack([a for a, _ in roll.log]).numpy(), "cost": torch.stack([c for _, c in roll.log]).numpy(),
           "result": state.best_action.reshape(P, H, D).numpy()}
    for k, v in rec.items():
        out[k] = torch.stack(v).numpy()
    return out


def main():
    import _reference_under_shim as shim
    shim.prepare()
    out = {}
    for name, (P, H, D, over) in CASES.items():
        for k, v in run_case(name, P, H, D, over).items():
            out[f"{name}/{k}"] = np.asarray(v, np.float32) if v.dtype.kind == "f" else v
    path = os.path.join(HERE, "mppi_reference_torch.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items() if k.endswith("/actions")})


if __name__ == "__main__":
    main()
