"""Cost-only against cost + gradient fused rollout on the same rows (RolloutEngine.evaluate_cost vs evaluate_action), the
batches a particle optimizer evaluates: Franka IK at 16,384 and 409,600 rows (512 goals x 32 seeds x 25 particles) in the
benchmark cuboid world, Franka 16,384 rows against the 256^3 ESDF, G1-29 and G1-43 at 8,192 x 25 rows against the ESDF.

Timing: CUDA events around every launch, L2 flushed (256 MiB write) before each, the three modes alternating launch by launch;
median of `--iters` launches per mode after `--warmup`.  Prints the card name and power limit first, then one line per workload.
    python scripts/bench_cost_only.py [--iters 200] [--warmup 20]"""
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
from helpers import humanoid_q, random_q  # noqa: E402

WORKLOADS = (("franka_ik_512x32_cuboid", 1), ("franka_ik_512x32_cuboid", 25), ("franka_16384_esdf", 1),
             ("g1_29_8192_esdf", 25), ("g1_43_8192_esdf", 25))


def scaled(name, k):
    """The bench workload with k times its rows (particles per seed): fresh random rows, the same goals and world."""
    wl = bench.make_workload(name)
    if k == 1:
        return wl
    rm, B = wl["robot"], wl["B"] * k
    q = humanoid_q(rm, B, seed=400) if name.startswith("g1") else random_q(rm, B, seed=400)
    wl = dict(wl, B=B, q=q[:, None, :])
    if wl["goal"] is not None:
        gp, gq, idx = wl["goal"]
        wl["goal"] = (gp, gq, np.repeat(idx, k).astype(np.int32))
    return wl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    dev = "cuda:0"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    from curobo_b200 import lib as cblib
    for name, k in WORKLOADS:
        wl = scaled(name, k)
        eng = bench.build_engine(wl, dev)
        q = torch.as_tensor(wl["q"]).to(dev)
        modes = {"grad": lambda: eng.evaluate_action(q), "cost": lambda: eng.evaluate_cost(q),
                 "cost_no_terms": lambda: eng.evaluate_cost(q, with_terms=False)}
        variants = {}
        for m, f in modes.items():
            for _ in range(args.warmup):
                f()
            variants[m] = int(cblib.load().cb200_last_rollout_variant())
        torch.cuda.synchronize()
        ev = {m: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
              for m in modes}
        for i in range(args.iters):
            for m, f in modes.items():
                flush.fill_(i & 0xFF)
                ev[m][i][0].record()
                f()
                ev[m][i][1].record()
        torch.cuda.synchronize()
        med = {m: float(np.median([a.elapsed_time(b) for a, b in ev[m]])) for m in modes}
        # the outputs agree (same rows, one after the other)
        c_grad = eng.evaluate_action(q).cost.clone()
        c_cost = eng.evaluate_cost(q).cost.clone()
        rel = float((c_cost - c_grad).abs().max() / c_grad.abs().max().clamp_min(1e-30))
        print(f"{name} x{k} ({wl['B'] * wl['H']} rows): grad {med['grad']:.4f} ms [variant {variants['grad']}]  "
              f"cost-only {med['cost']:.4f} ms [variant {variants['cost']:#x}]  cost-only without terms "
              f"{med['cost_no_terms']:.4f} ms  -> cost-only / grad {med['cost'] / med['grad']:.3f}  (max rel cost diff {rel:.1e})",
              flush=True)
        del eng, q
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
