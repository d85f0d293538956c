"""Velocity-aware IK (the current-state block of the POSITION c-space cost) on the GPU, in three parts:

(a) cost of the block on the rollout: the bench.py rows of Franka IK (16,384 rows, benchmark cuboid world) and G1-29 (8,192 rows,
    256^3 ESDF), evaluate_action without a current state and with one (dt = 0.05 on every row).  CUDA events around every
    launch, L2 flushed (256 MiB write) before each, the two arms alternating launch by launch; medians.
(b) fused against composed at retargeting sizes: G1-29 local-IK rows (1 / 64 / 1,024 clips x 4 line-search candidates,
    lbfgs_retarget_ik.yml weights, no world): one fused launch against FK, self collision, tool pose, cb200_cspace_position_cost and
    the FK backward chained as separate launches (the reference's compiled FK / self-collision / backward kernels from oracle/_ref,
    this library's tool-pose and c-space operators, the torch gradient sum), both captured as CUDA graphs; the outputs of both
    are compared in the same run.
(c) retargeting a synthetic clip: tool-frame poses from FK of a seeded smooth G1-29 joint trajectory, 120 frames at dt = 0.05,
    1 and 256 clips in parallel.  Frame 0: global IK with 64 seeds per clip (RolloutConfig.retarget_ik(), L-BFGS 100 iterations),
    best seed kept.  Frames 1..: one seed, LBFGSOptCfg(num_iters=200, history=15, cost_relative_threshold=0.01,
    convergence_iteration=10), current state = the previous solution with velocity (q_t - q_{t-1}) / dt, each frame one replay of
    one captured CUDA graph with the goal and the current state rewritten in place.  Reports ms per frame, the median tool-frame
    position / rotation error and max over joints and frames of |q_t - q_{t-1}| / (v_lim dt); the same run without the current
    state for contrast.

    python scripts/bench_velocity_ik.py [--iters 200] [--frames 120] [--parts abc]
Prints the card name and power limit first, then one line per measurement."""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import bench  # noqa: E402
from helpers import humanoid_q  # noqa: E402
from curobo_b200 import cost as cb_cost  # noqa: E402
from curobo_b200.optim import LBFGSOpt, LBFGSOptCfg  # noqa: E402
from curobo_b200.robot_model import load_robot  # noqa: E402
from curobo_b200.rollout import RolloutConfig, RolloutEngine  # noqa: E402
from oracle import rollout_oracle as O  # noqa: E402

DEV = "cuda:0"
DT = 0.05
N_LS = 4                   # line-search candidates per problem (LBFGSOptCfg.line_search_scale)


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def alternate(fns, iters, warmup):
    """Median ms of each fn over `iters` launches, alternating, L2 flushed before each."""
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=DEV)
    for f in fns.values():
        for _ in range(warmup):
            f()
    torch.cuda.synchronize()
    ev = {k: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)] for k in fns}
    for i in range(iters):
        for k, f in fns.items():
            flush.fill_(i & 0xFF)
            ev[k][i][0].record()
            f()
            ev[k][i][1].record()
    torch.cuda.synchronize()
    return {k: float(np.median([a.elapsed_time(b) for a, b in ev[k]])) for k in fns}


# ------------------------------------------------------------------------------------------------ (a)
def part_a(iters, warmup):
    for name in ("franka_ik_512x32_cuboid", "g1_29_8192_esdf"):
        wl = bench.make_workload(name)
        rm, B = wl["robot"], wl["B"]
        plain_eng, state_eng = bench.build_engine(wl, DEV), bench.build_engine(wl, DEV)
        q = T(wl["q"])
        rng = np.random.default_rng(5)
        lim_v = np.asarray(rm.velocity_limits, np.float32)[1]
        cur = T((wl["q"][:, 0] + rng.normal(0, 1, wl["q"][:, 0].shape) * lim_v * DT).astype(np.float32))
        vel, dt, idx = T(rng.normal(0, 0.3, cur.shape).astype(np.float32)), T(np.full(B, DT, np.float32)), T(np.arange(B, dtype=np.int32))
        state_eng.update_current_state(cur, vel, dt, idx)

        def plain():
            plain_eng.evaluate_action(q)

        def with_state():
            state_eng.evaluate_action(q)
        med = alternate({"plain": plain, "state": with_state}, iters, warmup)
        print(f"(a) {name} ({B} rows): no current state {med['plain']:.4f} ms, current state dt=0.05 {med['state']:.4f} ms "
              f"(x{med['state'] / med['plain']:.3f})", flush=True)
        del plain_eng, state_eng
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ (b)
def part_b(iters, warmup):
    import ref_kernels
    from curobo_b200.kinematics import KinematicsParams
    if not os.path.exists(ref_kernels.PATH):
        print("(b) skipped: oracle/_ref/libcurobo_ref.so (the reference's compiled kernels) not built", flush=True)
        return
    lib = ref_kernels.lib()
    rm = load_robot("g1_29")
    cfg = RolloutConfig.retarget_ik()
    D, S, L, nl = rm.num_dof, rm.num_spheres, rm.num_tool_frames, rm.num_links
    kp = KinematicsParams.from_robot_model(rm, DEV)
    p_ = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    for clips in (1, 64, 1024):
        B, H = clips * N_LS, 1
        N = B
        z = lambda *s, dt=torch.float32: torch.zeros(s, dtype=dt, device=DEV)  # noqa: E731
        q_np = humanoid_q(rm, B, seed=40 + clips, scale=0.5).astype(np.float32)
        q = T(q_np).view(B, 1, D)
        _, _, gpn, gqn = O.fk_forward(rm, humanoid_q(rm, clips, seed=41, scale=0.5))
        gp, gq = T(gpn[:, :, None, :].copy()), T(gqn[:, :, None, :].copy())
        gidx = T(np.repeat(np.arange(clips), N_LS).astype(np.int32))
        cur_np = (q_np + np.random.default_rng(3).normal(0, 0.05, q_np.shape)).astype(np.float32)
        cur, cvel = T(cur_np), T(np.zeros_like(cur_np))
        cdt = T(np.full(B, DT, np.float32))
        cidx = T(np.arange(B, dtype=np.int32))
        eng = RolloutEngine(rm, cfg, DEV)
        eng.update_goal(gp, gq, gidx)
        eng.update_current_state(cur, cvel, cdt, cidx)
        # composed chain buffers
        pos, quat, sph, com, cum = z(N, L, 3), z(N, L, 4), z(N, S, 4), z(N, 4), z(N, nl, 3, 4)
        eq = z(1, dt=torch.int32)
        sc_dist, sc_vec, sc_sparse = z(B, H), z(B, H, S, 4), z(B, H, S, dt=torch.uint8)
        nb = rm.num_blocks_per_batch
        sc_pd, sc_bv, sc_bi = z(1), z(B, H, nb), z(B, H, nb, 2, dt=torch.int16)
        w_self = torch.tensor([cfg.self_weight], device=DEV)
        padding, pairs = T(rm.sphere_padding), T(rm.collision_pairs)
        pw = torch.tensor(list(cfg.pose_weight), device=DEV)
        ones6, zeros2, proj = torch.ones((L, 6), device=DEV), z(L, 2), z(L, 1, dt=torch.uint8)
        p_cost, p_pd, p_rd = z(B, H, 2 * L), z(B, H, L), z(B, H, L)
        p_gp, p_gq, p_gi = z(B, H, L, 3), z(B, H, L, 4), z(B, H, L, dt=torch.int32)
        lim, efl, vlim = T(rm.position_limits), T(rm.effort_limits), T(rm.velocity_limits)
        cs_w = torch.tensor(list(cfg.cspace_weight[:2]), device=DEV)
        cs_a = torch.tensor(list(cfg.cspace_activation[:2]), device=DEV)
        cs_reg = torch.tensor(list(cfg.cspace_reg[:2]), device=DEV)
        cs_cost, cs_gp, cs_gt = z(B, H, D), z(B, H, D), z(B, H, D)
        zeros_bhd, zi, zd, tw0, tdw = z(B, H, D), z(B, dt=torch.int32), z(1, D), z(1), torch.ones(D, device=DEV)
        g_q, g_com, total, grad = z(N, D), z(N, 4), z(B, H), z(B, H, D)

        def composed():
            st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            assert lib.ref_kinematics_forward_spheres(
                p_(pos), p_(quat), p_(sph), p_(com), p_(cum), p_(q), p_(kp.fixed_transforms), p_(kp.link_spheres),
                p_(kp.link_masses_com), p_(kp.joint_map_type), p_(kp.joint_map), p_(kp.link_map), p_(kp.tool_frame_map),
                p_(kp.link_sphere_idx_map), p_(kp.joint_offset_map), p_(eq), kp.num_envs, N, 1, kp.num_dof, kp.num_spheres,
                kp.num_links, kp.num_pose_links, st) == 0
            assert lib.ref_self_collision_distance(p_(sc_dist), p_(sc_vec), p_(sc_pd), p_(sc_sparse), p_(sph.view(B, H, S, 4)),
                                                   p_(padding), p_(w_self), p_(pairs), p_(sc_bv), p_(sc_bi), nb,
                                                   rm.max_threads_per_block, B, H, S, pairs.shape[0], 1, st) == 0
            cb_cost.tool_pose_distance(pos.view(B, H, L, 3), quat.view(B, H, L, 4), gp, gq, gidx.view(B, 1), pw, ones6, ones6,
                                       zeros2, zeros2, proj, p_cost, p_pd, p_rd, p_gp, p_gq, p_gi, cfg.pose_lie)
            cb_cost.cspace_position_cost(q, zeros_bhd, zd, zi, lim, efl, cs_w, cs_a, tw0, tdw, cs_reg, cur, cvel, cidx, vlim, cdt,
                                         cs_cost, cs_gp, cs_gt)
            assert lib.ref_kinematics_backward(
                p_(g_q), p_(p_gp.view(N, L, 3)), p_(p_gq.view(N, L, 4)), p_(sc_vec.view(N, S, 4)), p_(g_com), p_(g_com), None,
                p_(cum), p_(kp.link_spheres), p_(kp.link_masses_com), p_(kp.link_map), p_(kp.joint_map), p_(kp.joint_map_type),
                p_(kp.tool_frame_map), p_(kp.link_sphere_idx_map), p_(kp.link_chain_data), p_(kp.link_chain_offsets),
                p_(kp.joint_links_data), p_(kp.joint_links_offsets), p_(kp.joint_affects_endeffector), p_(kp.joint_offset_map),
                p_(eq), kp.num_envs, N, 1, kp.num_dof, kp.num_spheres, kp.num_links, kp.num_pose_links, st) == 0
            torch.add(g_q.view(B, H, D), cs_gp, out=grad)
            total.copy_(sc_dist + p_cost.sum(-1) + cs_cost.sum(-1))

        def fused():
            eng.evaluate_action(q)

        graphs = {}
        for k, f in (("fused", fused), ("composed", composed)):
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(3):
                    f()
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                f()
            graphs[k] = g
        med = alternate({k: g.replay for k, g in graphs.items()}, iters, warmup)
        torch.cuda.synchronize()
        o = eng.out
        dc = float((o.cost - total).abs().max() / total.abs().max().clamp_min(1e-30))
        dg = float((o.grad_q - grad).abs().max() / grad.abs().max().clamp_min(1e-30))
        print(f"(b) G1-29 {clips} clips x {N_LS} rows: fused {med['fused']:.4f} ms, composed {med['composed']:.4f} ms "
              f"(composed / fused {med['composed'] / med['fused']:.2f}); max rel diff cost {dc:.1e}, grad_q {dg:.1e}", flush=True)
        del eng, graphs
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ (c)
def clip_trajectory(rm, clips, frames, seed):
    """[clips, frames, D]: smooth joint trajectories (sums of sines) inside the joint limits, peak speed ~0.6 v_lim."""
    rng = np.random.default_rng(seed)
    lim = np.asarray(rm.position_limits, np.float32)
    v = np.asarray(rm.velocity_limits, np.float32)[1]
    D = rm.num_dof
    mid, half = (lim[0] + lim[1]) / 2, (lim[1] - lim[0]) / 2
    t = np.arange(frames, dtype=np.float64)[None, :, None] * DT
    q = np.broadcast_to(mid + rng.uniform(-0.2, 0.2, (clips, 1, D)) * half, (clips, frames, D)).copy()
    for _ in range(2):
        w = rng.uniform(0.5, 2.0, (clips, 1, D))
        amp = np.minimum(0.25 * half, 0.3 * v / w)
        q = q + amp * np.sin(w * t + rng.uniform(0, 2 * np.pi, (clips, 1, D)))
    return np.clip(q, lim[0] + 0.02, lim[1] - 0.02).astype(np.float32)


def pose_errors(rm, q, gp, gq):
    """Tool-frame position (m) and rotation (rad) errors of q [N, D] against goals [N, L, 3|4]."""
    _, _, p, qt = O.fk_forward(rm, q)
    pe = np.linalg.norm(p - gp, axis=-1)
    re = 2 * np.arccos(np.clip(np.abs(np.sum(qt * gq, axis=-1)), 0, 1))
    return pe, re


def retarget(rm, traj, use_state, seeds=64):
    clips, frames, D = traj.shape
    L = rm.num_tool_frames
    _, _, gp_all, gq_all = O.fk_forward(rm, traj.reshape(-1, D))
    gp_all, gq_all = gp_all.reshape(clips, frames, L, 3), gq_all.reshape(clips, frames, L, 4)
    lo, hi = T(rm.position_limits[0]), T(rm.position_limits[1])
    tol = T(np.full((L, 2), 1e-8, np.float32))
    # frame 0: global IK, 64 seeds per clip, best seed kept
    P0 = clips * seeds
    e0 = RolloutEngine(rm, RolloutConfig.retarget_ik(), DEV)
    e0.update_goal(T(gp_all[:, 0, :, None, :].copy()), T(gq_all[:, 0, :, None, :].copy()),
                   T(np.repeat(np.arange(clips), seeds * N_LS).astype(np.int32)), terminal_tol=tol)

    def f0(x):
        o = e0.evaluate_action(x.view(-1, 1, D))
        return o.cost.view(-1), o.grad_q.view(-1, D)
    opt0 = LBFGSOpt(LBFGSOptCfg(num_iters=100), P0, 1, D, lo, hi, f0, DEV)
    x = opt0.optimize(T(humanoid_q(rm, P0, seed=9, scale=0.5).astype(np.float32)).view(P0, 1, D)).view(clips, seeds, D)
    best = opt0.best_cost.view(clips, seeds).argmin(dim=1)
    q0 = x[torch.arange(clips, device=DEV), best].clone()
    # frames 1..: one seed, one graph replay per frame
    gpos, gquat = T(gp_all[:, 1, :, None, :].copy()), T(gq_all[:, 1, :, None, :].copy())
    eng = RolloutEngine(rm, RolloutConfig.retarget_ik(), DEV)
    eng.update_goal(gpos, gquat, T(np.repeat(np.arange(clips), N_LS).astype(np.int32)), terminal_tol=tol)
    cur_p, cur_v = q0.clone(), torch.zeros_like(q0)
    if use_state:
        eng.update_current_state(cur_p, cur_v, T(np.full(clips, DT, np.float32)),
                                 T(np.repeat(np.arange(clips), N_LS).astype(np.int32)))

    def f1(xx):
        o = eng.evaluate_action(xx.view(-1, 1, D))
        return o.cost.view(-1), o.grad_q.view(-1, D)
    opt = LBFGSOpt(LBFGSOptCfg(num_iters=200, history=15, cost_relative_threshold=0.01, convergence_iteration=10), clips, 1, D, lo,
                   hi, f1, DEV)
    sol = torch.zeros((clips, frames, D), device=DEV)
    sol[:, 0] = q0
    prev, ms = q0.clone(), []
    for t in range(1, frames):
        gpos.copy_(T(gp_all[:, t, :, None, :].copy()))
        gquat.copy_(T(gq_all[:, t, :, None, :].copy()))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        qt = opt.optimize_graphed(prev.view(clips, 1, D)).view(clips, D)
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
        sol[:, t] = qt
        cur_v.copy_((qt - prev) / DT)
        cur_p.copy_(qt)
        prev.copy_(qt)
    s = sol.cpu().numpy()
    pe, re = pose_errors(rm, s.reshape(-1, D), gp_all.reshape(-1, L, 3), gq_all.reshape(-1, L, 4))
    v = np.asarray(rm.velocity_limits, np.float32)[1]
    ratio = float(np.max(np.abs(np.diff(s, axis=1)) / (v * DT)))
    ratio_ref = float(np.max(np.abs(np.diff(traj, axis=1)) / (v * DT)))
    # the first replay includes the eager warm-up and the capture
    return float(np.median(ms[1:])), float(np.median(pe)), float(np.median(re)), ratio, ratio_ref


def part_c(frames):
    rm = load_robot("g1_29")
    for clips in (1, 256):
        traj = clip_trajectory(rm, clips, frames, seed=7)
        for use_state in (True, False):
            ms, pe, re, ratio, ratio_ref = retarget(rm, traj, use_state)
            print(f"(c) G1-29 {clips} clip(s) x {frames} frames, {'with' if use_state else 'without'} current state: "
                  f"{ms:.2f} ms per frame, median tool-frame error {pe * 1e3:.2f} mm / {re:.4f} rad, "
                  f"max |dq| / (v_lim dt) {ratio:.2f} (source clip {ratio_ref:.2f})", flush=True)
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--parts", default="abc")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    if "a" in args.parts:
        part_a(args.iters, args.warmup)
    if "b" in args.parts:
        part_b(args.iters, args.warmup)
    if "c" in args.parts:
        part_c(args.frames)


if __name__ == "__main__":
    main()
