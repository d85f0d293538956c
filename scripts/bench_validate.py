"""Validity of joint configurations: the early-exit kernel (RolloutEngine.validate) against the cost-only fused rollout followed by
`cost == 0` (evaluate_cost(with_terms=False) with weight 1 and activation 0 on the bound, self and scene terms), on the same rows.

Workloads: Franka 1,048,576 rows in the benchmark cuboid world and against the 256^3 box ESDF, G1-29 and G1-43 65,536 rows against
the ESDF.  Rows are uniform draws from the position limits widened by 5 % on each side, so some rows fail on bounds alone; the
humanoids' floating-base joints are drawn where bench.py puts them (the robot standing in the world).  The two arms give the
same mask (checked).  Also printed: the fraction of invalid rows, split by the first check that fails in the kernel's order
(bounds, scene, self), and the fractions of rows in scene contact and in self contact whatever their other checks.

Timing: CUDA events around every launch, L2 flushed (256 MiB write) before each, the two arms alternating launch by launch;
median of `--iters` launches per arm after `--warmup`.  The card name, power limit and maximum SM clock are read first.
    python scripts/bench_validate.py [--iters 50] [--warmup 5]"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
from helpers import humanoid_q  # noqa: E402

WORKLOADS = (("franka_cuboid", "franka_ik_512x32_cuboid", 1 << 20), ("franka_esdf", "franka_16384_esdf", 1 << 20),
             ("g1_29_esdf", "g1_29_8192_esdf", 1 << 16), ("g1_43_esdf", "g1_43_8192_esdf", 1 << 16))


def draws(rm, humanoid, n, seed):
    lo, hi = np.asarray(rm.position_limits, np.float32)
    u = np.random.default_rng(seed).uniform(-0.05, 1.05, (n, rm.num_dof)).astype(np.float32)
    q = lo + (hi - lo) * u
    if humanoid:   # the floating base where bench.py's humanoid rows put it
        base = humanoid_q(rm, n, seed=seed)
        for d, name in enumerate(rm.joint_names):
            if name.startswith("base_j_"):
                q[:, d] = base[:, d]
    return np.ascontiguousarray(q[:, None, :])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    dev = "cuda:0"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    from curobo_b200 import lib as cblib
    from curobo_b200.rollout import RolloutConfig
    cfg = RolloutConfig(self_weight=1.0, scene_weight=1.0, scene_activation=0.0, cspace_type="position",
                        cspace_weight=(1.0, 0, 0, 0, 0), cspace_activation=(0.0,) * 5)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    for label, name, n in WORKLOADS:
        wl = bench.make_workload(name)
        rm = wl["robot"]
        eng = bench.build_engine(dict(wl, cfg=cfg, goal=None, cs_target=None), dev)
        q = torch.as_tensor(draws(rm, name.startswith("g1"), n, seed=11)).to(dev)
        arms = {"validate": lambda: eng.validate(q), "cost": lambda: eng.evaluate_cost(q, with_terms=False).cost == 0}
        variants = {}
        for a, f in arms.items():
            for _ in range(args.warmup):
                f()
            variants[a] = int(cblib.load().cb200_last_rollout_variant())
        torch.cuda.synchronize()
        ev = {a: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
              for a in arms}
        for i in range(args.iters):
            for a, f in arms.items():
                flush.fill_(i & 0xFF)
                ev[a][i][0].record()
                f()
                ev[a][i][1].record()
        torch.cuda.synchronize()
        med = {a: float(np.median([s.elapsed_time(e) for s, e in ev[a]])) for a in arms}
        v = eng.validate(q).clone()
        same = bool(torch.equal(v, eng.evaluate_cost(q, with_terms=False).cost == 0))
        vb, vs, vp = (eng.validate(q, None, *f).clone() for f in ((True, False, False), (False, False, True), (False, True, False)))
        frac = lambda m: float(m.float().mean())  # noqa: E731
        print(f"{label} ({n} rows): validate {n / med['validate'] * 1e3:.4g} cfg/s ({med['validate']:.3f} ms) [variant "
              f"{variants['validate']:#x}]  cost==0 {n / med['cost'] * 1e3:.4g} cfg/s ({med['cost']:.3f} ms) [variant "
              f"{variants['cost']:#x}]  speed-up {med['cost'] / med['validate']:.2f}x  same mask {same}  invalid {frac(~v):.3f}: "
              f"bounds {frac(~vb):.3f} scene {frac(vb & ~vs):.3f} self {frac(vb & vs & ~vp):.3f}  (any order: scene {frac(~vs):.3f} "
              f"self {frac(~vp):.3f})", flush=True)
        del eng, q
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
