"""Position (clique) and acceleration control spaces on the H100: the three transition kernels alone, and
RolloutEngine.evaluate_positions (clique forward -> fused rollout -> clique adjoint) against evaluate_action on the same,
precomputed states, on
  Franka 1024 x 30 MPC (swept, speed metric) against the 256^3 box ESDF,
  Franka 128 x 34 trajopt against the benchmark cuboids,
  G1-29 512 x 34 trajopt against the benchmark cuboids.
Times are CUDA events over `--iters` launches after `--warmup`: `call_ms` / `*_ms` launched from Python one by one (what
an eager caller pays, host overhead included), `kernel_ms` / `*_graphed_ms` replayed from a CUDA graph of 50 calls (the
GPU time).  Every kernel's output is checked against the numpy oracle
(oracle/clique_oracle.py) in the same run, and evaluate_positions against the hand-composed three steps.  Kernel rates are
the bytes each kernel must move (computed from the shapes below) over its time, with the H100 SXM data-sheet 3.35 TB/s as the
bound.  Prints one JSON line with the card's name and power limit read in the same run.

    python scripts/bench_position_clique.py [--iters 200] [--warmup 20]
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

from helpers import humanoid_q, make_box_esdf, random_walk_q  # noqa: E402
from curobo_b200.backends import trajectory as trajectory_cu  # noqa: E402
from curobo_b200.robot_model import load_robot  # noqa: E402
from curobo_b200.rollout import RolloutConfig, RolloutEngine  # noqa: E402
from curobo_b200.scene import CuboidData, VoxelData  # noqa: E402
from curobo_b200.trajectory import JointState  # noqa: E402
from curobo_b200.world import make_benchmark_cuboid_world  # noqa: E402
from oracle import clique_oracle as co  # noqa: E402

DEV = "cuda:0"
HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


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


def graphed(fn, iters, warmup, per_graph=50):
    """Time of one `fn` with the host out of the way: `per_graph` calls captured in one CUDA graph, replayed."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()                                    # warm launch-plan caches outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(per_graph):
                fn()
    torch.cuda.current_stream().wait_stream(s)
    reps = max(1, iters // per_graph)
    return timed(g.replay, reps, max(1, warmup // per_graph)) / per_graph


def T(a):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV)


def workload(robot, B, H, world, args):
    rm = load_robot(robot)
    D, n = rm.num_dof, H - 4
    rng = np.random.default_rng(1)
    if robot == "franka":
        u = random_walk_q(rm, B, n, seed=2).astype(np.float32)
    else:
        base = humanoid_q(rm, B, seed=2, scale=0.5)[:, None, :]
        lim = np.asarray(rm.position_limits, np.float32)
        u = np.clip(base + np.cumsum(rng.normal(0, 0.02, (B, n, D)), axis=1), lim[0], lim[1]).astype(np.float32)
    z = np.zeros((B, D), np.float32)
    start = (u[:, 0].copy(), rng.normal(0, 0.1, (B, D)).astype(np.float32), z)
    goal = (u[:, -1].copy(), z, z)
    idx = np.arange(B, dtype=np.int32)
    traj_dt = np.full(B, 0.05, np.float32)
    imp = (np.arange(B) % 2).astype(np.uint8)
    u_t, idx_t, dt_t, imp_t = T(u), T(idx), T(traj_dt), T(imp)
    st = JointState(*[T(x) for x in start], jerk=None)
    gl = JointState(*[T(x) for x in goal], jerk=None, dt=dt_t)
    if world == "esdf":
        cfg = RolloutConfig.mpc()
        cfg.pose_weight = None          # no goal registry needed: collision, c-space state, target and bound terms
        sdf = make_box_esdf(n=256, voxel_size=0.01, num_boxes=12, seed=0, xp=torch)
        vox = VoxelData(T(np.array([[[256, 256, 256, 0.01]]], np.float32)), T(np.array([[[0, 0, 0, 1, 0, 0, 0, 0]]], np.float32)),
                        torch.ones((1, 1), dtype=torch.uint8, device=DEV), torch.ones(1, dtype=torch.int32, device=DEV),
                        sdf.reshape(1, 1, -1).contiguous(), 1, 1, 100.0)
        eng = RolloutEngine(rm, cfg, DEV, voxel=vox)
        eng2 = RolloutEngine(rm, cfg, DEV, voxel=vox)
        if cfg.cspace_target_weight > 0:
            for e in (eng, eng2):
                e.update_cspace_target(T(goal[0]), idx_t)
    else:
        cfg = RolloutConfig.trajopt()
        cfg.pose_weight = None          # no goal registry needed: collision, c-space state and bound terms
        cub = CuboidData.from_world(make_benchmark_cuboid_world(), DEV)
        eng, eng2 = RolloutEngine(rm, cfg, DEV, cub), RolloutEngine(rm, cfg, DEV, cub)

    r = {"rows": B * H, "dof": D}
    # the three transition kernels alone
    seq = [torch.zeros((B, H, D), device=DEV) for _ in range(4)]
    odt, gu = torch.zeros(B, device=DEV), torch.zeros((B, n, D), device=DEV)
    grads = [T(rng.normal(size=(B, H, D)).astype(np.float32)) for _ in range(4)]
    dt_h = T(np.full(H, 0.05, np.float32))
    u_acc = T(rng.normal(size=(B, H, D)).astype(np.float32))

    def fwd():
        trajectory_cu.launch_differentiation_position_forward_kernel(*seq, odt, u_t, st.position, st.velocity, st.acceleration,
                                                                     gl.position, gl.velocity, gl.acceleration, idx_t, idx_t,
                                                                     dt_t, imp_t, B, H, D)

    def bwd():
        trajectory_cu.launch_differentiation_position_backward_kernel(gu, *grads, dt_t, idx_t, imp_t, B, H, D)

    def acc():
        trajectory_cu.launch_integration_acceleration_kernel(*seq, u_acc, st.position, st.velocity, st.acceleration, idx_t, dt_h,
                                                             B, H, D)
    f4 = 4
    # bytes each kernel must move: forward reads u and writes four states; adjoint reads four gradients, writes u; integrator
    # reads u_acc and writes four states (index / start-state reads are O(B*D) and counted too)
    need = {"clique_forward": f4 * (B * n * D + 4 * B * H * D + 3 * B * D),
            "clique_backward": f4 * (4 * B * H * D + B * n * D),
            "acceleration_integrate": f4 * (5 * B * H * D + 3 * B * D)}
    for name, fn in (("clique_forward", fwd), ("clique_backward", bwd), ("acceleration_integrate", acc)):
        ms = graphed(fn, args.iters, args.warmup)
        r[name] = {"kernel_ms": round(ms, 5), "call_ms": round(timed(fn, args.iters, args.warmup), 5),
                   "GB_per_s": round(need[name] / (ms * 1e-3) / 1e9, 1),
                   "share_of_hbm_peak": round(need[name] / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}
    # check the kernels against the oracle on these inputs
    fwd()
    want = co.clique_forward(u, *start, goal[0], idx, idx, traj_dt, imp, H)
    for g, w in zip(seq, want[:4]):
        np.testing.assert_allclose(g.cpu().numpy(), w, rtol=2e-5, atol=2e-5 * max(1.0, float(np.abs(w).max())))
    bwd()
    wb = co.clique_backward(*[g.cpu().numpy() for g in grads], traj_dt, idx, imp)
    np.testing.assert_allclose(gu.cpu().numpy(), wb, rtol=1e-5, atol=1e-5 * float(np.abs(wb).max()))
    acc()
    wa = co.integrate_acceleration(u_acc.cpu().numpy(), *start, idx, np.full(H, 0.05, np.float32))
    for g, w in zip(seq, wa):
        np.testing.assert_allclose(g.cpu().numpy(), w, rtol=2e-5, atol=2e-5 * max(1.0, float(np.abs(w).max())))
    r["kernels_match_oracle"] = True

    # evaluate_positions vs evaluate_action on the precomputed states
    fwd()
    pre = [t.clone() for t in seq]
    pre_dt = odt.clone()
    r["evaluate_positions_ms"] = round(timed(lambda: eng.evaluate_positions(u_t, st, idx_t, gl, idx_t, imp_t), args.iters,
                                             args.warmup), 4)
    r["evaluate_action_ms"] = round(timed(lambda: eng2.evaluate_action(pre[0], vel=pre[1], acc=pre[2], jerk=pre[3], dt=pre_dt),
                                          args.iters, args.warmup), 4)
    r["transition_overhead_ms"] = round(r["evaluate_positions_ms"] - r["evaluate_action_ms"], 4)
    # the same two with the host out of the way (CUDA-graph replay): what a graphed optimizer loop pays
    r["evaluate_positions_graphed_ms"] = round(graphed(lambda: eng.evaluate_positions(u_t, st, idx_t, gl, idx_t, imp_t),
                                                       args.iters, args.warmup), 4)
    r["evaluate_action_graphed_ms"] = round(graphed(lambda: eng2.evaluate_action(pre[0], vel=pre[1], acc=pre[2], jerk=pre[3],
                                                                                 dt=pre_dt), args.iters, args.warmup), 4)
    o = eng.evaluate_positions(u_t, st, idx_t, gl, idx_t, imp_t)
    o2 = eng2.evaluate_action(pre[0], vel=pre[1], acc=pre[2], jerk=pre[3], dt=pre_dt)
    gu2 = torch.zeros_like(gu)
    trajectory_cu.launch_differentiation_position_backward_kernel(gu2, o2.grad_q, o2.grad_vel, o2.grad_acc, o2.grad_jerk, dt_t, idx_t,
                                                                  imp_t, B, H, D)
    torch.cuda.synchronize()
    assert torch.equal(o.cost, o2.cost) and torch.equal(o.grad_u, gu2)
    r["evaluate_positions_equals_composition"] = True
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_position_clique.py needs a GPU"
    out = {"gpu": gpu_info()}
    for name, robot, B, H, world in (("franka_mpc_1024x30_esdf", "franka", 1024, 30, "esdf"),
                                     ("franka_trajopt_128x34_cuboids", "franka", 128, 34, "cuboids"),
                                     ("g1_29_trajopt_512x34_cuboids", "g1_29", 512, 34, "cuboids")):
        out[name] = workload(robot, B, H, world, args)
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
