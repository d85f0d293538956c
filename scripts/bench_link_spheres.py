"""Run-time link-sphere updates (RolloutEngine.update_link_spheres & co. -> cb200_refresh_robot_spheres).

(1) Refresh latency: one launch copies configuration 0 into the device blob and rebuilds the broad-phase bounds of every collision
    link over all configurations; Franka, G1-29 and G1-43 at 1 and 8 sphere configurations.  CUDA events around `--iters`
    back-to-back refreshes after `--warmup`, mean per launch.
(2) The headline IK batch (bench.py's franka_ik_512x32_cuboid) as a captured evaluate_action graph: replayed right after an attach
    (4 spheres on `attached_object`) on the engine the graph was captured on, against the same graph captured on a fresh engine
    built from the modified model.  Both run the same kernel on the same rows; the replays alternate, median of `--iters` each.
Prints the card name and power limit first, then one JSON line per measurement.
    python scripts/bench_link_spheres.py [--iters 500] [--warmup 50]"""
import argparse
import dataclasses
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from curobo_b200.robot_model import load_robot  # noqa: E402
from curobo_b200.rollout import RolloutConfig, RolloutEngine  # noqa: E402

ATTACHED = np.array([[0.0, 0.0, 0.08, 0.05], [0.0, 0.0, 0.12, 0.05], [0.03, 0.0, 0.1, 0.04], [-0.03, 0.0, 0.1, 0.04]], np.float32)


def refresh_latency(robot, n_cfg, iters, warmup, dev):
    rm = load_robot(robot)
    if n_cfg > 1:
        rm = dataclasses.replace(rm, link_spheres=np.stack([rm.link_spheres] * n_cfg))
    eng = RolloutEngine(rm, RolloutConfig.ik(), dev)
    for _ in range(warmup):
        eng.refresh_link_spheres()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        eng.refresh_link_spheres()
    b.record()
    torch.cuda.synchronize()
    h = np.frombuffer(eng._blob_host[:192].tobytes(), np.int32)
    return {"bench": "refresh", "robot": robot, "n_cfg": n_cfg, "collision_links": int(h[27]), "spheres": rm.num_spheres,
            "us_per_refresh": 1000.0 * a.elapsed_time(b) / iters}


def ik_replay_after_attach(iters, warmup, dev):
    wl = bench.make_workload("franka_ik_512x32_cuboid")
    q = torch.as_tensor(wl["q"]).to(dev)
    rm = wl["robot"]
    ls = np.array(rm.link_spheres, np.float32)
    ls[np.nonzero(rm.link_sphere_idx_map == rm.link_names.index("attached_object"))[0]] = ATTACHED
    engines = {"attached": bench.build_engine(wl, dev), "fresh": bench.build_engine(dict(wl, robot=dataclasses.replace(rm, link_spheres=ls)), dev)}
    graphs = {}
    for k, e in engines.items():
        for _ in range(3):
            e.evaluate_action(q)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            e.evaluate_action(q)
        graphs[k] = g
    engines["attached"].update_link_spheres("attached_object", torch.as_tensor(ATTACHED).to(dev))
    for _ in range(warmup):
        for g in graphs.values():
            g.replay()
    times = {k: [] for k in graphs}
    for _ in range(iters):
        for k, g in graphs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            g.replay()
            b.record()
            torch.cuda.synchronize()
            times[k].append(a.elapsed_time(b))
    same = all(torch.equal(getattr(engines["attached"].out, t), getattr(engines["fresh"].out, t)) for t in ("cost", "grad_q"))
    return {"bench": "ik_graph_replay_after_attach", "workload": "franka_ik_512x32_cuboid", "rows": int(q.shape[0]),
            "ms_median": {k: float(np.median(v)) for k, v in times.items()}, "outputs_bit_identical": bool(same)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()
    dev = "cuda:0"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    for robot in ("franka", "g1_29", "g1_43"):
        for n_cfg in (1, 8):
            print(json.dumps(refresh_latency(robot, n_cfg, args.iters, args.warmup, dev)), flush=True)
    print(json.dumps(ik_replay_after_attach(args.iters, args.warmup, dev)), flush=True)


if __name__ == "__main__":
    main()
