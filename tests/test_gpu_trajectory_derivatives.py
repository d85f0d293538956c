"""The fused rollout's trajectory gradients against float64 derivatives of the composed cost they belong to.

tests/test_gpu_rollout_derivatives.py checks grad_q.  Here the other gradient outputs are checked the same way, each against the
float64 central differences of the cost it is the gradient of (the chains are pinned on the CPU by
tests/test_trajectory_derivatives_cpu.py):
  * evaluate_action with the STATE c-space cost: grad_q, grad_vel, grad_acc and grad_jerk jointly (directions perturb q, v, a and
    j), on the trajectory kernel (swept, scene off) and every discrete family (cuboids);
  * evaluate_knots: grad_knots through bspline_forward -> rollout -> bspline_backward, expanded and in-kernel spline schedules;
  * evaluate_positions: grad_u through clique_forward -> rollout -> clique_backward;
  * attach_dynamics: the STATE cost plus the effort channel on tau = RNEA(q, qd, qdd), host composition (CTA and row RNEA
    kernels) and inside the trajectory kernel across its 32-waypoint dynamics chunk, also under evaluate_knots;
  * B200RobotRollout in the bspline and position_clique action spaces: torch.autograd.grad of the summed cost terms.
Trajectory horizons fall below, at and across the trajectory kernel's tile (one waypoint per warp, 8 warps per CTA) and the
dynamics kernel's chunk.  Start and goal rows are gathered by index (fewer rows than trajectories), with a dt per goal row and
implicit and replicate (or explicit) goal rows mixed.

Per run, as in test_gpu_rollout_derivatives.py: the variant asserted, each row's cost and term costs against the float64 oracle,
sum(grad * d) against the central difference for N_DIR directions per row within TOL of sum|grad * d| (for the STATE front end
also along directions that perturb q, v, a or j alone: each gradient output on its own), at least 90 % of the row/directions
past the kink guard, every term under test active in most counted rows.  The float64 reference of a case does not
depend on the family, so it is computed once per case.  Dynamics runs use Franka only: the RNEA adjoint is the derivative for
revolute trees (G1's floating base is prismatic, and the reference's prismatic motion_cross_S is reproduced on purpose)."""
import dataclasses
import functools

import numpy as np
import pytest
import torch

import test_gpu_rollout_derivatives as G
from test_gpu_rollout_derivatives import check_costs, colliding_rows, derivative_errors, goalset, walk
from dynamics_cases import make_case, model_args
from curobo_b200.robot_model import load_robot
from curobo_b200.rollout import RolloutConfig, RolloutEngine
from curobo_b200.scene import CuboidData
from curobo_b200.world import CuboidWorld
from oracle import bspline_oracle as bo
from oracle import clique_oracle as co
from oracle import dynamics_oracle as do
from oracle import rollout_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VARIANT_ENV = dict(G.VARIANT_ENV, expanded={"CB200_BIG": "0", "CB200_ARM_PAIRS": "0"}, in_kernel={"CB200_BIG": "0"},
                   host={"CB200_BIG": "0"}, host_rows={"CB200_BIG": "0", "CB200_RNEA_ROWS": "1"}, fused={"CB200_BIG": "0"},
                   protocol={"CB200_BIG": "0"})
GRAD_VARIANT = G.GRAD_VARIANT                              # arm 2, pairs 2, standard 1, big 4, team 5, team4 6, traj 7
TRAJ, TRAJ_DYN, STANDARD, ARM = 7, 8, 1, 2               # include/curobo_b200.h
last_variant = G.last_variant
N_DIR = 4
# |an - fd| / sum|grad * d|, the tolerance of test_gpu_rollout_derivatives.py.  Worst measured over every run and direction set:
# 1.4e-6 on an H100 80GB HBM3 (700 W power limit).  One term scaled by 1.001 measured 7.6e-4 to 1.0e-3 (jerk gradient, on the
# "jerk" set), 5.2e-4 (the spline adjoint's jerk coefficient) and 4.6e-4 (the RNEA adjoint's qdd gradient, on the "acc" set).
TOL = 2e-5
G1_BOX = {"dims": [0.6, 0.6, 0.3], "pose": [0.25, 0.0, 0.9] + G.ROT}


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def sync():
    if DEV != "cpu":
        torch.cuda.synchronize()


def float64_oracle(monkeypatch):
    for m in (O, G.CS, bo, do):
        monkeypatch.setattr(m, "F", np.float64)


# ------------------------------------------------------------------------------------------------ the float64 chains
def effort_cost(dyn, q, qd, qdd, jerk, dt, cfg):
    """The effort channel of the STATE cost (bound hinge, squared-L2, energy) on tau = RNEA(q, qd, qdd): cost [B,H,D] and the
    gradients with respect to (q, qd, qdd) through the RNEA adjoint, in the precision of the oracle modules."""
    c, elim = dyn
    B, H, D = q.shape
    rm, m = c["rm"], model_args(c)
    tau, cache = do.rnea_forward(q.reshape(-1, D), qd.reshape(-1, D), qdd.reshape(-1, D), *m)
    lim = dict(p=rm.position_limits, v=rm.velocity_limits, a=rm.acceleration_limits, j=rm.jerk_limits, tau=elim)
    w = [0, 0, 0, 0, cfg.cspace_weight[4]]
    r = [0, 0, 0, cfg.cspace_reg[3], cfg.cspace_reg[4]]
    cost, g = O.cspace_state_cost(q, qd, qdd, jerk, dt, lim, w, cfg.cspace_activation, r, cfg.retime_weights, cfg.retime_reg,
                                  effort=tau.reshape(B, H, D))
    bq, bqd, bqdd = do.rnea_backward(g[4].reshape(-1, D), q.reshape(-1, D), qd.reshape(-1, D), cache, *m)
    s = lambda x: np.asarray(x).reshape(B, H, D)  # noqa: E731
    return cost, (g[0] + s(bq), g[1] + s(bqd), g[2] + s(bqdd)), s(tau)


def rollout64(c, p, v, a, j, dt):
    """The rollout oracle (precision of the oracle modules) at states p, v, a, j [B,H,D], dt [B], plus the effort channel when the
    case attaches dynamics."""
    kw = dict(world_cuboid=c["cub"], goal_pos=c["goal"][0], goal_quat=c["goal"][1], idxs_goal=c["goal"][2],
              cspace_target=c["target"][0], idxs_cspace_target=c["target"][1], cspace_target_dof_weight=c["target"][2])
    w = O.rollout_cost_grad(c["rm"], p, c["cfg"].to_oracle_cfg(c["rm"].num_tool_frames), vel=v, acc=a, jerk=j, dt=dt, **kw)
    if c["dyn"] is not None:
        ec = effort_cost(c["dyn"], p, v, a, j, dt, c["cfg"])[0]
        w["cspace_cost"] = w["cspace_cost"] + ec
        w["cost"] = w["cost"] + ec.reshape(p.shape[0], -1).sum(-1)
    w["_state"] = (v, a, j)
    return w


def live_hinges(rm, cfg, v, a, j):
    """Whether the velocity, acceleration and jerk bound hinges of the STATE cost are live somewhere."""
    out = []
    for i, (x, lim) in enumerate(((v, rm.velocity_limits), (a, rm.acceleration_limits), (j, rm.jerk_limits)), start=1):
        lim = np.asarray(lim, np.float64)
        lo, hi = lim[0] + cfg.cspace_activation[i] * (lim[1] - lim[0]), lim[1] - cfg.cspace_activation[i] * (lim[1] - lim[0])
        out.append(bool(((x < lo) | (x > hi)).any()))
    return out


# ------------------------------------------------------------------------------------------------ cases
def state_cfg(swept, robot):
    """MPC weights (lbfgs_mpc.yml) with self collision, cuboids in discrete mode, the Lie-group pose and no speed metric; bound
    weights retimed for Franka and not for G1-29."""
    cfg = RolloutConfig.mpc()
    cfg.self_weight, cfg.scene_weight, cfg.scene_activation = 1000.0, 0.0 if swept else 1000.0, 0.05
    cfg.use_sweep, cfg.use_speed_metric, cfg.pose_lie, cfg.pose_weight = swept, False, True, (1000.0, 100.0)
    cfg.cspace_reg = (0.5, 10.0, 0.01, 0.0, 0.0)
    cfg.retime_weights = robot == "franka"
    return cfg


def boundary(rm, first, last, seed):
    """Two start and two goal rows (float32 values), gathered by index for B trajectories; a dt per goal row; goal 0 implicit."""
    D = rm.num_dof
    B = first.shape[0]
    rng = np.random.default_rng(seed)
    f = lambda x: np.ascontiguousarray(x, np.float32)  # noqa: E731
    start = tuple(f(x) for x in (first[[1, 0]] + rng.normal(0, 0.02, (2, D)), rng.normal(0, 0.3, (2, D)),
                                 rng.normal(0, 1.0, (2, D)), rng.normal(0, 5.0, (2, D))))
    goal = tuple(f(x) for x in (last[[0, 1]] + rng.normal(0, 0.02, (2, D)), rng.normal(0, 0.3, (2, D)),
                                rng.normal(0, 1.0, (2, D)), np.zeros((2, D))))
    sidx = (np.arange(B) % 2 ^ 1).astype(np.int32)
    gidx = (np.arange(B) // 2 % 2).astype(np.int32)
    return start, goal, sidx, gidx, np.array([0.05, 0.08], np.float32), np.array([1, 0], np.uint8)


def _case(name, dev):
    """Case dict: robot, rm, cfg, x (the variables the gradient is taken with respect to, float32 [B,K,D]), f64 (x -> the float64
    oracle's outputs at x), worlds, goals, target, dynamics and the terms that must be active."""
    seed = sum(map(ord, name))
    robot, kind = name.split("-", 1)
    rm = load_robot(robot)
    D = rm.num_dof
    swept = "discrete" not in kind
    cfg = state_cfg(swept, robot)
    cub = None if swept else CuboidWorld.create([G.TABLE, G.PILLAR, G.TILTED_BOX] if robot == "franka" else [G1_BOX], max_n=3)
    c = dict(robot=robot, rm=rm, cfg=cfg, cub=cub, vox=None, current=None, env=None, dyn=None, kind=kind.split("_")[0],
             terms=("self_cost", "pose_cost", "cspace_cost") + (() if swept else ("scene_cost",)))
    B = {"franka": 4, "g1_29": 3}[robot]
    if kind.startswith("dyn"):
        B = 2
        c["dyn_case"] = make_case("franka", 1, seed)       # Franka with random inertial parameters
        cfg.cspace_weight = tuple(cfg.cspace_weight[:4]) + (20.0,)
        cfg.cspace_activation = (0.01, 0.01, 0.01, 0.01, 0.05)
        cfg.cspace_reg = (0.5, 10.0, 0.01, 0.05, 0.3)
    rng = np.random.default_rng(seed)
    if kind.startswith(("state", "dyn_")):
        H = int(kind.rsplit("_h", 1)[1])
        q = walk(colliding_rows(rm, robot, B, seed, cub=cub), H, seed)
        v, a, j = [rng.normal(0, s, size=q.shape).astype(np.float32) for s in (2.0, 12.0, 400.0)]
        dt = rng.uniform(0.02, 0.1, size=B).astype(np.float32)
        c.update(x=np.concatenate([q, v, a, j], axis=1), H=H, dt=dt)
        c["f64"] = lambda x: rollout64(c, x[:, :H], x[:, H:2 * H], x[:, 2 * H:3 * H], x[:, 3 * H:], dt.astype(np.float64))
    elif kind.startswith(("knots", "protocol_bspline", "dynknots")):
        nk, degree, steps = 6, 4, 4
        if kind.startswith("knots"):
            degree, steps = int(kind.rsplit("_d", 1)[1][0]), int(kind.rsplit("_s", 1)[1][0])
        elif kind.startswith("dynknots"):
            nk = 8                                     # H = 53: two dynamics chunks
        knots = walk(colliding_rows(rm, robot, B, seed, cub=cub), nk, seed, sigma=0.08)
        start, goal, sidx, gidx, traj_dt, imp = boundary(rm, knots[:, 0], knots[:, -1], seed + 1)
        H = bo.padded_horizon_for(nk, degree, steps)
        c.update(x=knots, H=H, degree=degree, steps=steps, spline=(start, goal, sidx, gidx, traj_dt, imp))
        f64 = lambda t: tuple(np.asarray(x, np.float64) for x in t)  # noqa: E731

        def spline64(x):
            p, v, a, j, odt = bo.bspline_forward(x, f64(start), f64(goal), sidx, gidx, traj_dt.astype(np.float64), imp, H, degree)
            return rollout64(c, p, v, a, j, odt)
        c["f64"] = spline64
    elif kind.startswith(("clique", "protocol_clique")):
        H = int(kind.rsplit("_h", 1)[1]) if "_h" in kind else 14
        u = walk(colliding_rows(rm, robot, B, seed, cub=cub), H - 4, seed, sigma=0.03)
        start, goal, sidx, gidx, traj_dt, imp = boundary(rm, u[:, 0], u[:, -1], seed + 1)
        c.update(x=u, H=H, spline=(start, goal, sidx, gidx, traj_dt, imp))

        def clique64(x):
            p, v, a, j, odt = co.clique_forward(x, *start[:3], goal[0], sidx, gidx, traj_dt, imp, H, dtype=np.float64)
            return rollout64(c, p, v, a, j, odt.astype(np.float64))
        c["f64"] = clique64
    else:
        raise KeyError(name)
    gp, gq = goalset(rm, robot, 2, seed + 2)
    c["goal"] = (gp, gq, (np.arange(B) % 2).astype(np.int32))
    c["target"] = (G.configurations(rm, robot, 2, seed + 3), (np.arange(B) % 2).astype(np.int32),
                   np.linspace(0.5, 1.5, D).astype(np.float32))
    c["spline_kind"] = kind
    if "dyn_case" in c:                                 # effort limits at the quartiles of the case's torques: the hinge is live
        dc = c["dyn_case"]
        p, v, a = _dyn_states(c)
        tau = do.rnea_forward(p.reshape(-1, D), v.reshape(-1, D), a.reshape(-1, D), *model_args(dc))[0]
        elim = np.stack([np.quantile(tau, 0.25, axis=0), np.quantile(tau, 0.75, axis=0)]).astype(np.float32)
        c["dyn"] = (dc, elim)
    return c


def _dyn_states(c):
    """float32 positions, velocities and accelerations of a dynamics case (the spline's for the knots case)."""
    H = c["H"]
    if c["kind"] == "dynknots":
        start, goal, sidx, gidx, traj_dt, imp = c["spline"]
        p, v, a, _, _ = bo.bspline_forward(c["x"], start, goal, sidx, gidx, traj_dt, imp, H, c["degree"])
        return p, v, a
    x = c["x"]
    return x[:, :H], x[:, H:2 * H], x[:, 2 * H:3 * H]


_cases = functools.lru_cache(maxsize=None)(_case)


def case(name):
    return _cases(name, DEV)


def reference(name):
    return _reference(name, DEV)


def blocks(c):
    """The direction sets of a case: "all" perturbs every variable; with the STATE front end also "q", "vel", "acc" and "jerk",
    each perturbing one block of x alone, so that every gradient output is checked against its own part of the derivative (the
    jerk gradient is small beside the others: a jerk gradient scaled by 1.001 moves the joint check by only ~3e-6)."""
    out = {"all": slice(None)}
    if c["kind"] in ("state", "dyn"):
        H = c["H"]
        out.update((k, slice(i * H, (i + 1) * H)) for i, k in enumerate(("q", "vel", "acc", "jerk")))
    return out


@functools.lru_cache(maxsize=None)
def _reference(name, dev):
    """float64: the oracle at x and, per direction set of blocks(c), the directions [N_DIR, B, K, D] and the central differences
    [2, N_DIR, B]."""
    assert O.F is np.float64 and bo.F is np.float64 and do.F is np.float64
    c = case(name)
    x = c["x"].astype(np.float64)
    w = c["f64"](x)
    full = np.random.default_rng(7).standard_normal((N_DIR,) + x.shape)
    sets = {}
    for label, sl in blocks(c).items():
        d = np.zeros_like(full)
        d[:, :, sl] = full[:, :, sl] * (1.0 if label == "all" else max(float(x[:, sl].std()), 1.0))  # (v, a, j: their own scale)
        sets[label] = (d, np.stack([np.stack([(c["f64"](x + e * dk)["cost"] - c["f64"](x - e * dk)["cost"]) / (2 * e) for dk in d])
                                    for e in G.EPS]))
    return w, sets


# ------------------------------------------------------------------------------------------------ runs
def engine(c, family):
    from curobo_b200.dynamics import Dynamics
    rm = c["rm"]
    if family == "fused":                              # the in-kernel effort limits are the robot blob's
        rm = dataclasses.replace(rm, effort_limits=c["dyn"][1])
    mesh = None
    if family == "standard" and c["robot"] == "franka":    # Franka reaches the standard kernel only with mesh obstacles
        from curobo_b200.mesh import MeshData, MeshWorld, box_mesh
        v, f = box_mesh([0.1, 0.1, 0.1])
        mesh = MeshData.from_world(MeshWorld.create([{"vertices": v, "faces": f, "pose": [10.0, 10.0, 10.0, 1, 0, 0, 0]}], max_n=2),
                                   DEV)
    eng = RolloutEngine(rm, c["cfg"], DEV, CuboidData.from_world(c["cub"], DEV) if c["cub"] is not None else None, mesh=mesh)
    eng.update_goal(T(c["goal"][0]), T(c["goal"][1]), T(c["goal"][2]))
    eng.update_cspace_target(T(c["target"][0]), T(c["target"][1]), T(c["target"][2]))
    if c["dyn"] is not None:
        dc, elim = c["dyn"]
        dyn = Dynamics(rm, dc["mc"], dc["inn"], gravity=(0.0, 0.0, -9.81), device=DEV)
        eng.attach_dynamics(dyn, fused=True) if family == "fused" else eng.attach_dynamics(dyn, effort_limits=elim)
        assert (eng._dyn_params is not None) == (family == "fused")
    return eng


def want_variant(c, family):
    if family == "fused":
        return TRAJ_DYN
    if c["cfg"].use_sweep:
        return TRAJ
    if family in GRAD_VARIANT:
        return GRAD_VARIANT[family]
    if family == "in_kernel":
        return STANDARD                                # the spline build of the standard kernel
    return ARM if c["robot"] == "franka" else STANDARD


def spline_args(c):
    start, goal, sidx, gidx, traj_dt, imp = c["spline"]
    from curobo_b200.trajectory import JointState
    st = JointState(*[T(x) for x in start])
    gl = JointState(*[T(x) for x in goal], dt=T(traj_dt))
    return st, T(sidx), gl, T(gidx), T(imp)


def launch(c, family):
    """(the engine's output, the kernel's gradient with respect to x, numpy float64 [B,K,D])."""
    H, kind = c["H"], c["kind"]
    if kind == "protocol":
        from curobo_b200.rollout_protocol import B200RobotRollout
        bspline = "bspline" in c["spline_kind"]
        ro = B200RobotRollout(c["rm"], c["cfg"], DEV, horizon=H, action_space="bspline" if bspline else "position_clique",
                              n_knots=c["x"].shape[1], bspline_degree=4, interpolation_steps=4)
        st, sidx, gl, gidx, imp = spline_args(c)
        ro.update_params(goal_position=T(c["goal"][0]), goal_quat=T(c["goal"][1]), idxs_goal=T(c["goal"][2]),
                         cspace_target=T(c["target"][0]), idxs_cspace_target=T(c["target"][1]),
                         cspace_target_dof_weight=T(c["target"][2]), start_state=st, goal_state=gl, start_state_idx=sidx,
                         goal_state_idx=gidx, use_implicit_goal_state=imp)
        x = T(c["x"]).requires_grad_(True)
        r = ro.evaluate_action(x)
        total = r.costs_and_constraints.get_sum_cost_and_constraint(sum_horizon=True)
        (g,) = torch.autograd.grad(total.sum(), x)
        sync()
        return ro.engine.out, g.double().cpu().numpy()
    eng = engine(c, family)
    if kind in ("state", "dyn"):
        x = T(c["x"])
        o = eng.evaluate_action(x[:, :H].contiguous(), vel=x[:, H:2 * H].contiguous(), acc=x[:, 2 * H:3 * H].contiguous(),
                                jerk=x[:, 3 * H:].contiguous(), dt=T(c["dt"]))
        sync()
        g = torch.cat([o.grad_q, o.grad_vel, o.grad_acc, o.grad_jerk], dim=1)
    elif kind in ("knots", "dynknots"):
        o = eng.evaluate_knots(T(c["x"]), *spline_args(c), bspline_degree=c["degree"], interpolation_steps=c["steps"],
                               in_kernel_spline=family == "in_kernel")
        sync()
        g = o.grad_knots
    else:
        o = eng.evaluate_positions(T(c["x"]), *spline_args(c))
        sync()
        g = o.grad_u
    return o, g.double().cpu().numpy()


def run_case(monkeypatch, name, family):
    float64_oracle(monkeypatch)
    c = case(name)
    w, sets = reference(name)
    for k, v in VARIANT_ENV[family].items():
        monkeypatch.setenv(k, v)
    o, grad = launch(c, family)
    assert last_variant() == want_variant(c, family), (last_variant(), want_variant(c, family))
    B = c["x"].shape[0]
    sel = np.arange(B)
    want = G.want_terms(w)
    check_costs(G.row_terms(o, sel), want, f"{name} {family}")
    worst, rows = {}, np.ones(B, bool)
    for label, (d, fd) in sets.items():
        err, counted = derivative_errors(grad, d, fd, 1.0)
        frac = float(counted.mean())
        worst[label] = float(err[counted].max())
        print(f"DERIV {name} {family} {label}: worst {worst[label]:.3g}, kink guard dropped {1 - frac:.1%} of {counted.size}")
        assert frac >= 0.9, f"{label}: the kink guard dropped {1 - frac:.1%} of the row/directions"
        rows &= counted.any(0)
    for k in c["terms"]:
        active = float((want[k][rows] > 0).mean())
        assert active > 0.5, f"{k} active in only {active:.0%} of the counted rows"
    live = live_hinges(c["rm"], c["cfg"], *w["_state"])
    assert all(live) if c["kind"] in ("state", "dyn") else any(live), f"velocity / acceleration / jerk hinges live: {live}"
    if c["dyn"] is not None:
        p, v, a = (np.asarray(t, np.float64) for t in _dyn_states(c))
        tau = effort_cost(c["dyn"], p, v, a, np.zeros_like(p), np.full(B, 0.05), c["cfg"])[2]
        elim = c["dyn"][1]
        assert ((tau < elim[0]) | (tau > elim[1])).mean() > 0.2, "the effort hinge must be live"
    for label, e in worst.items():
        assert e <= TOL, f"{name} {family} {label}: sum(grad * d) vs the float64 derivative: worst {e:.3g} of sum|grad * d|"
    return max(worst.values())


STATE_RUNS = [(f"franka-state_h{H}", "traj") for H in (7, 8, 9, 17)] + [("g1_29-state_h9", "traj")] + \
             [("franka-state_discrete_h3", f) for f in ("arm", "pairs", "standard", "big", "team", "team4")] + \
             [("g1_29-state_discrete_h2", f) for f in ("standard", "big", "team", "team4")]
KNOTS_RUNS = [("franka-knots_d3_s2", s) for s in ("expanded", "in_kernel")] + \
             [("franka-knots_discrete_d4_s1", s) for s in ("expanded", "in_kernel")] + \
             [("franka-knots_d5_s4", "expanded"), ("franka-knots_discrete_d5_s2", "in_kernel")] + \
             [("g1_29-knots_d4_s2", s) for s in ("expanded", "in_kernel")] + [("g1_29-knots_discrete_d3_s1", "expanded")]
CLIQUE_RUNS = [(f"franka-clique_h{H}", "traj") for H in (9, 14, 30, 37)] + [("franka-clique_discrete_h10", "expanded")] + \
              [("g1_29-clique_h14", "traj"), ("g1_29-clique_discrete_h9", "expanded")]
DYNAMICS_RUNS = [("franka-dyn_h32", "host"), ("franka-dyn_h32", "host_rows")] + \
                [(f"franka-dyn_h{H}", "fused") for H in (31, 32, 33)] + [("franka-dynknots", "fused")]
PROTOCOL_RUNS = [("franka-protocol_bspline", "protocol"), ("franka-protocol_clique_h14", "protocol")]


@pytest.mark.parametrize("name,family", STATE_RUNS)
def test_state_gradients_are_derivatives(monkeypatch, name, family):
    """grad_q, grad_vel, grad_acc and grad_jerk of evaluate_action with the STATE cost, jointly."""
    run_case(monkeypatch, name, family)


@pytest.mark.parametrize("name,family", KNOTS_RUNS)
def test_knots_gradient_is_derivative(monkeypatch, name, family):
    """grad_knots of evaluate_knots, expanded and in-kernel spline schedules."""
    run_case(monkeypatch, name, family)


@pytest.mark.parametrize("name,family", CLIQUE_RUNS)
def test_position_clique_gradient_is_derivative(monkeypatch, name, family):
    """grad_u of evaluate_positions."""
    run_case(monkeypatch, name, family)


@pytest.mark.parametrize("name,family", DYNAMICS_RUNS)
def test_dynamics_aware_gradients_are_derivatives(monkeypatch, name, family):
    """attach_dynamics: host composition (CTA and row RNEA kernels) and the fused trajectory-dynamics kernel at H = 31, 32, 33;
    evaluate_knots with the fused kernel behind the expanded spline schedule (H = 53)."""
    run_case(monkeypatch, name, family)


@pytest.mark.parametrize("name,family", PROTOCOL_RUNS)
def test_protocol_autograd_gradient_is_derivative(monkeypatch, name, family):
    """B200RobotRollout(action_space="bspline" / "position_clique"): torch.autograd.grad of the summed cost terms with respect to
    act_seq."""
    run_case(monkeypatch, name, family)
