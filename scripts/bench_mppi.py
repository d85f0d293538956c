"""The MPPI particle stage on the GPU.

1. One inner iteration: cb200_mppi_sample -> cost-only rollout without terms -> cb200_mppi_update (3 launches), against a torch
   restatement of the reference's glue (particle_opt_core.py:409-441, get_sum_cost_and_constraint, mppi.py:200-248, 722-757)
   over the same rollout with its per-term tensors written.  Franka IK 16,384 x 25 rows on the benchmark cuboid world, G1-29
   8,192 x 25 rows on the 256^3 ESDF.
2. The sample and update kernels alone: bytes each must move (from the shapes) over its time, as a share of the 3.35 TB/s HBM3
   bound of the H100 SXM data sheet.
3. IK solve, 512 goals x 32 seeds: MPPI (particle_ik.yml: 4 iterations, 25 particles) then L-BFGS (100 iterations) as one CUDA
   graph, against L-BFGS alone; time per solve and success (best seed within 5 mm and 0.05 rad).

Timing: CUDA events, L2 flushed (256 MiB write) before each timed call, arms alternating call by call, median of `--iters`.
Prints the card name and power limit first.
    python scripts/bench_mppi.py [--iters 100] [--warmup 10]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]
import bench  # noqa: E402
from bench_cost_only import scaled  # noqa: E402
from curobo_b200.backends import optimization as optimization_cu  # noqa: E402
from curobo_b200.optim import LBFGSOpt, LBFGSOptCfg, MPPIOpt, MPPIOptCfg, MultiStageOpt  # noqa: E402
from curobo_b200.rollout import RolloutConfig  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
NP = 25


def timed(arms, iters, warmup, flush):
    """{name: fn} -> {name: median ms}, arms alternating, L2 flushed before every call."""
    for f in arms.values():
        for _ in range(warmup):
            f()
    torch.cuda.synchronize()
    ev = {m: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)] for m in arms}
    for i in range(iters):
        for m, f in arms.items():
            flush.fill_(i & 0xFF)
            ev[m][i][0].record()
            f()
            ev[m][i][1].record()
    torch.cuda.synchronize()
    return {m: float(np.median([a.elapsed_time(b) for a, b in ev[m]])) for m in arms}


def inner_iteration(name, iters, warmup, flush, dev):
    wl = scaled(name, NP)
    rm, H, D = wl["robot"], wl["H"], wl["robot"].num_dof
    P = wl["B"] // NP
    eng = bench.build_engine(wl, dev)
    lows = torch.as_tensor(rm.position_limits[0], dtype=torch.float32).to(dev)
    highs = torch.as_tensor(rm.position_limits[1], dtype=torch.float32).to(dev)
    gen = torch.Generator().manual_seed(0)
    noise = torch.randn((P, NP, H, D), generator=gen).to(dev)
    noise[:, -1] = 0.0
    x0 = torch.as_tensor(wl["q"]).to(dev).view(P, NP, H, D)[:, 0].contiguous()
    mean, scale, cov, best = x0.clone(), torch.ones(P, D, device=dev), torch.ones(P, D, device=dev), x0.clone()
    acts = torch.empty(P, NP, H, D, device=dev)

    def ours():
        optimization_cu.launch_mppi_sample(acts, mean, scale, noise, lows, highs)
        c = eng.evaluate_cost(acts.view(P * NP, H, D), with_terms=False).cost
        optimization_cu.launch_mppi_update(acts, c, mean, cov, scale, best, 1.0, 0.9, 0.2, 0.01, 1.0)

    gamma_seq = torch.ones(1, H, device=dev)
    t_mean, t_cov, t_scale, t_best = mean.clone(), cov.clone().view(P, 1, D), scale.clone().view(P, 1, D), best.clone()
    problem_col = torch.arange(P, device=dev)

    def torch_glue():
        # particle_opt_core.py:409-441 (no neg / null particles at null_act_frac 0)
        a = t_mean.unsqueeze(-3) + noise * t_scale.unsqueeze(-2).expand(-1, -1, H, -1)
        a = torch.max(torch.min(a.reshape(P * NP, H * D), highs.repeat(H)), lows.repeat(H)).reshape(P * NP, H, D)
        out = eng.evaluate_cost(a, with_terms=True)
        # get_sum_cost_and_constraint(sum_horizon=True): concatenate the term tensors, sum terms, then the horizon
        terms = [out.pose_cost, out.cspace_cost, out.scene_cost, out.self_cost.unsqueeze(-1)]
        costs = torch.cat(terms, dim=-1).sum(-1).sum(-1, keepdim=True).view(P, NP, 1)
        actions = a.view(P, NP, H, D)
        w = torch.softmax((-1.0 / 1.0) * (gamma_seq * costs).sum(-1) / gamma_seq[..., 0], dim=-1)      # BEST
        t_best.copy_(actions[problem_col, torch.argmax(w, dim=-1)])
        cost_seq = (gamma_seq * costs).sum(-1) / gamma_seq[..., 0]                                      # jit_mean_cov_diag_a
        w = torch.softmax((-1.0 / 1.0) * cost_seq, dim=-1)[..., None, None]
        new_mean = 0.1 * t_mean + 0.9 * torch.sum(w * actions, dim=-3)
        cov_upd = torch.mean(torch.sum(w * (actions - t_mean.unsqueeze(-3)) ** 2, dim=-3), dim=-2).unsqueeze(-2)
        t_cov.copy_(0.8 * t_cov + 0.2 * cov_upd + 0.01)
        t_scale.copy_(torch.sqrt(t_cov))
        t_mean.copy_(new_mean)

    med = timed({"ours_3_launches": ours, "torch_glue": torch_glue}, iters, warmup, flush)
    print(f"[inner iteration] {name} {P} x {NP} particles ({P * NP} rows, V = {H * D}): ours {med['ours_3_launches']:.4f} ms, "
          f"torch glue over the rollout with terms {med['torch_glue']:.4f} ms -> {med['torch_glue'] / med['ours_3_launches']:.2f}x",
          flush=True)

    # the two kernels alone
    c = eng.evaluate_cost(acts.view(P * NP, H, D), with_terms=False).cost
    kmed = timed({"sample": lambda: optimization_cu.launch_mppi_sample(acts, mean, scale, noise, lows, highs),
                  "update": lambda: optimization_cu.launch_mppi_update(acts, c, mean, cov, scale, best, 1.0, 0.9, 0.2, 0.01, 1.0)},
                 iters, warmup, flush)
    V = H * D
    nbytes = {"sample": 4 * (P * NP * V + P * NP * V + P * V + P * D),            # noise in, actions out, mean + scale in
              "update": 4 * (P * NP * V + P * NP * H + 2 * P * V + 2 * P * D + P * D + P * V)}  # actions, cost, mean rw, cov rw, scale, best
    for k in ("sample", "update"):
        t = kmed[k] * 1e-3
        print(f"[kernel] {name} {k}: {kmed[k] * 1e3:.1f} us, {nbytes[k] / 1e6:.2f} MB -> {nbytes[k] / t / 1e12:.2f} TB/s = "
              f"{100 * nbytes[k] / t / HBM_BYTES_PER_S:.0f} % of 3.35 TB/s", flush=True)
    del eng
    torch.cuda.empty_cache()


def ik_solve(dev, problems=512, seeds=32, repeats=5):
    from helpers import random_q
    from curobo_b200.kinematics import Kinematics
    from oracle import rollout_oracle as O
    wl = bench.make_workload("franka_ik_512x32_cuboid")
    rm, n = wl["robot"], 4
    B, D = problems * seeds, rm.num_dof
    q_goal = random_q(rm, problems, seed=11) * 0.8
    _, _, gp, gq = O.fk_forward(rm, q_goal)
    goal = lambda k: (gp[:, :, None, :].copy(), gq[:, :, None, :].copy(), np.repeat(np.arange(B) // seeds, k).astype(np.int32))  # noqa: E731
    e_lbfgs = bench.build_engine(dict(wl, goal=goal(n)), dev)
    e_mppi = bench.build_engine(dict(wl, goal=goal(NP), cfg=RolloutConfig.particle_ik()), dev)
    td = lambda a: torch.as_tensor(a).to(dev)  # noqa: E731
    lows, highs = td(rm.position_limits[0]), td(rm.position_limits[1])

    def cost_grad(x):
        out = e_lbfgs.evaluate_action(x.view(B * n, 1, D))
        return out.cost.view(-1), out.grad_q.view(B * n, D)

    def make(two_stage):
        lb = LBFGSOpt(LBFGSOptCfg(num_iters=100), B, 1, D, lows, highs, cost_grad, dev)
        if not two_stage:
            return lb
        mp = MPPIOpt(MPPIOptCfg(), B, 1, D, lows, highs, lambda a: e_mppi.evaluate_cost(a, with_terms=False).cost, device=dev)
        return MultiStageOpt([mp, lb])
    x0 = td(random_q(rm, B, seed=12)).view(B, 1, D)
    res = {}
    for name, two in (("lbfgs_only", False), ("mppi_then_lbfgs", True)):
        opt = make(two)
        opt.optimize_graphed(x0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(repeats):
            q_sol = opt.optimize_graphed(x0)
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / repeats
        q_sol = q_sol.reshape(B, D)
        st = Kinematics(rm, dev).compute_kinematics(q_sol.view(B, 1, D))
        pos = st.tool_pose_position.reshape(B, -1, 3)[:, 0].cpu().numpy().reshape(problems, seeds, 3)
        quat = st.tool_pose_quaternion.reshape(B, -1, 4)[:, 0].cpu().numpy().reshape(problems, seeds, 4)
        perr = np.linalg.norm(pos - gp[:, 0][:, None, :], axis=-1)
        rerr = 2.0 * np.arccos(np.abs(np.sum(quat * gq[:, 0][:, None, :], axis=-1)).clip(0, 1))
        ok = ((perr < 5e-3) & (rerr < 0.05)).any(axis=1)
        res[name] = (dt * 1e3, float(ok.mean()))
        print(f"[ik solve] {problems} x {seeds} {name}: {dt * 1e3:.3f} ms per solve (one CUDA graph, wall clock over {repeats}), "
              f"success {100 * ok.mean():.1f} %", flush=True)
        del opt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mppi.py measures on a GPU; none is visible")
    dev = "cuda:0"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    for name in ("franka_ik_512x32_cuboid", "g1_29_8192_esdf"):
        inner_iteration(name, args.iters, args.warmup, flush, dev)
    del flush
    ik_solve(dev)


if __name__ == "__main__":
    main()
