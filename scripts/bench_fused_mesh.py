"""Mesh obstacles inside the fused rollout kernels vs the per-operator composition (FK -> self collision + sphere/mesh collision
launches -> autograd backward), on the workloads of DESIGN.md section 8:
  Franka IK 16,384 rows against the benchmark table + pillar as cuboids, the same two boxes as meshes, and the table plus an
  icosphere of 1,280 and 20,480 triangles; 1024 x 30 MPC (swept, speed metric) and G1-29 8,192 rows against the table + icosphere.
Each mesh workload is timed fused and composed (CUDA events after warm-up) and the two must give the same outputs.  Prints one
JSON line with the card's name and power limit read in the same run.

    python scripts/bench_fused_mesh.py [--iters 50] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from helpers import humanoid_q, random_q  # noqa: E402
from curobo_b200.kinematics import Kinematics, SelfCollisionCost  # noqa: E402
from curobo_b200.mesh import MeshData, MeshWorld, box_mesh, icosphere  # noqa: E402
from curobo_b200.robot_model import load_robot  # noqa: E402
from curobo_b200.rollout import RolloutConfig, RolloutEngine  # noqa: E402
from curobo_b200.scene import (CollisionBuffer, CuboidData, SceneData, SphereObstacleCollision,  # noqa: E402
                               SweptSphereObstacleCollision)
from curobo_b200.world import make_benchmark_cuboid_world  # noqa: E402

DEV = "cuda:0"
TABLE = {"dims": [2.2, 2.2, 0.2], "pose": [0.0, 0.0, -0.1, 1, 0, 0, 0]}
PILLAR = {"dims": [0.1, 0.1, 1.5], "pose": [0.45, 0.0, 0.3, 1, 0, 0, 0]}


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def box(c):
    v, f = box_mesh(c["dims"])
    return {"vertices": v, "faces": f, "pose": c["pose"]}


def ball(subdiv, pose):
    v, f = icosphere(0.2, subdiv)
    return {"vertices": v, "faces": f, "pose": pose}


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def workload(name, robot, B, H, world, args):
    rm = load_robot(robot)
    traj = H > 1
    cfg = RolloutConfig(self_weight=5000.0, scene_weight=5000.0, scene_activation=0.02, use_sweep=traj, use_speed_metric=traj)
    rng = np.random.default_rng(1)
    base = (random_q(rm, B, seed=2) if robot == "franka" else humanoid_q(rm, B, seed=2, scale=0.5))[:, None, :]
    qn = base + (np.cumsum(rng.normal(0, 0.03, (B, H, rm.num_dof)), axis=1) if traj else 0.0)
    lim = np.asarray(rm.position_limits, np.float32)
    q = torch.as_tensor(np.ascontiguousarray(np.clip(qn, lim[0], lim[1]), np.float32)).to(DEV)
    dt = torch.full((B,), 0.05, dtype=torch.float32, device=DEV)
    kw = dict(dt=dt) if traj else {}
    cub = mesh = None
    if world == "cuboids":
        cub = CuboidData.from_world(make_benchmark_cuboid_world(), DEV)
    elif world == "box_meshes":
        mesh = MeshData.from_world(MeshWorld.create([box(TABLE), box(PILLAR)]), DEV)
    else:
        pose = [0.35, 0.25, 0.45, 1, 0, 0, 0] if robot == "franka" else [0.25, 0.0, 0.8, 1, 0, 0, 0]
        mesh = MeshData.from_world(MeshWorld.create([box(TABLE), ball(int(world[-1]), pose)]), DEV)
    eng = RolloutEngine(rm, cfg, DEV, cub, mesh=mesh)
    fused_ms = timed(lambda: eng.evaluate_action(q, **kw), args.iters, args.warmup)
    o = eng.evaluate_action(q, **kw)
    torch.cuda.synchronize()
    from curobo_b200 import lib as cblib
    r = {"rows": B * H, "fused_ms": round(fused_ms, 4), "variant": int(cblib.load().cb200_last_rollout_variant()),
         "colliding_spheres": int((o.scene_cost > 0).sum())}
    if mesh is None:
        return r
    kin, selfc = Kinematics(rm, DEV), SelfCollisionCost(rm, cfg.self_weight, DEV)
    buf = CollisionBuffer.from_shape((B, H, rm.num_spheres, 4), DEV)
    w, eta = torch.tensor([cfg.scene_weight], device=DEV), torch.tensor([cfg.scene_activation], device=DEV)
    env = torch.zeros(B, dtype=torch.int32, device=DEV)
    scene = SceneData(None, None, mesh)
    sdt = torch.tensor([0.05], device=DEV)
    res = {}

    def composed():
        qg = q.clone().requires_grad_(True)
        st = kin.compute_kinematics(qg)
        d_self = selfc.forward(st.robot_spheres)
        if traj:
            d_scene = SweptSphereObstacleCollision.apply(st.robot_spheres, buf, scene, w, eta, None, sdt, True, env, False, False)
        else:
            d_scene = SphereObstacleCollision.apply(st.robot_spheres, buf, scene, w, eta, None, env, False, False)
        (d_self.sum() + d_scene.sum()).backward()
        res["scene"], res["grad"] = d_scene, qg.grad
    r["composed_ms"] = round(timed(composed, args.iters, args.warmup), 4)
    composed()
    torch.cuda.synchronize()
    torch.testing.assert_close(o.scene_cost, res["scene"], rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(o.grad_q, res["grad"], rtol=2e-3, atol=2e-5 * float(res["grad"].abs().max()))
    r["outputs_agree"] = True
    r["speedup"] = round(r["composed_ms"] / fused_ms, 2)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_fused_mesh.py needs a GPU"
    out = {"gpu": gpu_info()}
    for name, robot, B, H, world in (("franka_ik_16384_cuboids", "franka", 16384, 1, "cuboids"),
                                     ("franka_ik_16384_box_meshes", "franka", 16384, 1, "box_meshes"),
                                     ("franka_ik_16384_table_ico1280", "franka", 16384, 1, "ico3"),
                                     ("franka_ik_16384_table_ico20480", "franka", 16384, 1, "ico5"),
                                     ("franka_mpc_1024x30_table_ico1280", "franka", 1024, 30, "ico3"),
                                     ("g1_29_8192_table_ico1280", "g1_29", 8192, 1, "ico3")):
        out[name] = workload(name, robot, B, H, world, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
