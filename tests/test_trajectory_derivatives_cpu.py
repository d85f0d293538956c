"""The float64 trajectory chains against central differences of their own composed cost (CPU, no device).

tests/test_gpu_trajectory_derivatives.py takes these chains, run in float64, as the costs whose derivatives the trajectory gradients
of the fused rollout must be (grad_vel / grad_acc / grad_jerk, grad_knots, grad_u and the dynamics-aware STATE cost).  Here each
chain's composed gradient is shown to be the derivative of its composed cost:
  * the STATE c-space cost with respect to position, velocity, acceleration and jerk jointly: bound hinges on all four, the
    squared-L2 regularization with either retime flag off, the energy term (a given torque), the target and its non-terminal
    factor;
  * knots -> bspline_forward -> rollout -> bspline_backward, degrees 3 / 4 / 5, 1 / 2 / 4 interpolation steps, start and goal
    rows gathered by index, a dt per goal row and implicit / replicate goal rows mixed;
  * u -> clique_forward -> rollout -> clique_backward, H in {9, 10, 14, 30}, implicit and explicit goals (H = 8 with the implicit
    goal is not a transpose by the reference's design: tests/test_position_clique_cpu.py);
  * q, qd, qdd -> RNEA -> effort channel of the STATE cost -> RNEA adjoint, on Franka (revolute joints only: the reference's
    prismatic motion_cross_S is reproduced on purpose, so the adjoint is the derivative only for revolute trees).
The rollout in the chains carries self collision, the Lie-group pose, rotated cuboids (eta > 0) and the STATE c-space cost.
bspline_oracle keeps its basis and boundary tables as float32-rounded constants (the values the kernels use); everything else
follows the patched float64 `F`.  A row/direction counts only where the central differences at eps 1e-5 and 1e-6 agree."""
import numpy as np
import pytest

import test_gpu_rollout_derivatives as G
from dynamics_cases import make_case, model_args
from curobo_b200.robot_model import load_robot
from curobo_b200.rollout import RolloutConfig
from curobo_b200.world import CuboidWorld
from oracle import bspline_oracle as bo
from oracle import clique_oracle as co
from oracle import current_state_oracle as CS
from oracle import dynamics_oracle as do
from oracle import rollout_oracle as O

N_DIR = 3
EXACT = 1e-6


@pytest.fixture
def f64(monkeypatch):
    for m in (O, CS, bo, do):
        monkeypatch.setattr(m, "F", np.float64)


def check_chain(fn, x, seed=1, tol=EXACT):
    """fn(x [B,K,D] float64) -> (cost [B], grad [B,K,D], extra).  Asserts sum(grad * d) == the central difference of cost along
    N_DIR random directions per row, to tol of sum|grad * d|; returns the extra output at x."""
    cost, grad, extra = fn(x)
    assert grad.dtype == np.float64 and cost.dtype == np.float64
    d = np.random.default_rng(seed).standard_normal((N_DIR,) + x.shape)
    fd = np.stack([np.stack([(fn(x + e * dk)[0] - fn(x - e * dk)[0]) / (2 * e) for dk in d]) for e in G.EPS])
    err, counted = G.derivative_errors(grad, d, fd, 1.0)
    assert counted.mean() >= 0.9, counted.mean()
    assert float(err[counted].max()) <= tol, float(err[counted].max())
    return extra


def state_cfg(retime_weights=True, retime_reg=True):
    cfg = RolloutConfig.mpc()
    cfg.scene_weight, cfg.scene_activation, cfg.use_sweep, cfg.use_speed_metric, cfg.pose_lie = 1000.0, 0.05, False, False, True
    cfg.self_weight = 1000.0
    cfg.cspace_reg = (0.5, 10.0, 0.01, 0.0, 0.0)
    cfg.retime_weights, cfg.retime_reg = retime_weights, retime_reg
    return cfg


def live_hinges(rm, cfg, v, a, j):
    """Whether the velocity, acceleration and jerk bound hinges are live somewhere."""
    out = []
    for i, (x, lim) in enumerate(((v, rm.velocity_limits), (a, rm.acceleration_limits), (j, rm.jerk_limits)), start=1):
        lo, hi = O._shrink(np.asarray(lim[0], np.float64), np.asarray(lim[1], np.float64), cfg.cspace_activation[i])
        out.append(bool(((x < lo) | (x > hi)).any()))
    return out


@pytest.mark.parametrize("retime_weights,retime_reg", [(True, True), (False, True), (True, False)])
@pytest.mark.parametrize("H", [1, 9])
def test_state_cost_position_velocity_acceleration_jerk(f64, retime_weights, retime_reg, H):
    """cspace_state_cost's four gradients are the derivative of its cost with respect to (p, v, a, j): bound hinges, squared-L2
    regularization (retimed or not), the energy term (tau v dt)^2 with a given torque, the target and its non-terminal factor."""
    rm = load_robot("franka")
    B, D = 4, rm.num_dof
    rng = np.random.default_rng(H + 2 * retime_weights + retime_reg)
    p = G.walk(G.configurations(rm, "franka", B, 5) * 1.2, H, 5).astype(np.float64)
    v, a, j = [rng.normal(0, s, size=p.shape) for s in (2.0, 12.0, 400.0)]
    tau = rng.normal(0, 20.0, size=p.shape)
    dt = rng.uniform(0.02, 0.1, size=B)
    lim = dict(p=rm.position_limits, v=rm.velocity_limits, a=rm.acceleration_limits, j=rm.jerk_limits, tau=rm.effort_limits)
    cfg = state_cfg(retime_weights, retime_reg)
    reg = (0.5, 10.0, 0.01, 0.0, 0.3)                        # velocity, acceleration, jerk, torque, energy
    tgt, tidx, dofw = G.configurations(rm, "franka", 2, 6), np.arange(B) % 2, np.linspace(0.5, 1.5, D)

    def fn(x):
        c, g = O.cspace_state_cost(x[:, :H], x[:, H:2 * H], x[:, 2 * H:3 * H], x[:, 3 * H:], dt, lim, cfg.cspace_weight,
                                   cfg.cspace_activation, reg, retime_weights, retime_reg, effort=tau, target=tgt, idxs_target=tidx,
                                   target_weight=1000.0, non_terminal_factor=0.05, target_dof_weight=dofw)
        return c.reshape(B, -1).sum(-1), np.concatenate(g[:4], axis=1), c
    c = check_chain(fn, np.concatenate([p, v, a, j], axis=1))
    assert (c.reshape(B, -1).sum(-1) > 0).all()
    assert all(live_hinges(rm, cfg, v, a, j))


def boundary_rows(rm, robot, knots, seed):
    """Two start and two goal rows for B trajectories (gathered by index), a dt per goal row, goal 0 implicit."""
    D = rm.num_dof
    rng = np.random.default_rng(seed)
    q0 = knots[[1, 0], 0] + rng.normal(0, 0.02, size=(2, D))
    start = (q0, rng.normal(0, 0.3, (2, D)), rng.normal(0, 1.0, (2, D)), rng.normal(0, 5.0, (2, D)))
    goal = (knots[[0, 1], -1] + rng.normal(0, 0.02, size=(2, D)), rng.normal(0, 0.3, (2, D)), rng.normal(0, 1.0, (2, D)),
            np.zeros((2, D)))
    B = knots.shape[0]
    return start, goal, np.arange(B) % 2 ^ 1, np.arange(B) // 2 % 2, np.array([0.05, 0.08]), np.array([1, 0], np.uint8)


def chain_world(robot):
    return CuboidWorld.create([G.TABLE, G.PILLAR, G.TILTED_BOX], max_n=3) if robot == "franka" else None


def rollout_kw(rm, robot, B, seed, cub):
    gp, gq = G.goalset(rm, robot, 2, seed)
    return dict(world_cuboid=cub, goal_pos=gp, goal_quat=gq, idxs_goal=np.arange(B) % 2,
                cspace_target=G.configurations(rm, robot, 2, seed + 1), idxs_cspace_target=np.arange(B) % 2)


@pytest.mark.parametrize("degree,steps", [(3, 1), (3, 2), (4, 2), (4, 4), (5, 4), (5, 1)])
def test_knots_chain(f64, degree, steps):
    """knots -> spline -> rollout (self, Lie pose, cuboids, STATE) -> spline adjoint: grad_knots is the derivative."""
    robot = "franka"
    rm = load_robot(robot)
    B, nk = 4, 6
    cub = chain_world(robot)
    knots = G.walk(G.colliding_rows(rm, robot, B, 40 + degree, cub=cub), nk, 40 + degree, sigma=0.08).astype(np.float64)
    start, goal, sidx, gidx, traj_dt, imp = boundary_rows(rm, robot, knots, 41 + steps)
    T = bo.padded_horizon_for(nk, degree, steps)
    cfg = state_cfg().to_oracle_cfg(rm.num_tool_frames)
    kw = rollout_kw(rm, robot, B, 43, cub)

    def fn(x):
        p, v, a, j, odt = bo.bspline_forward(x, start, goal, sidx, gidx, traj_dt, imp, T, degree)
        w = CS.rollout_cost_grad(rm, p, cfg, vel=v, acc=a, jerk=j, dt=odt, **kw)
        gs = w["cspace_grads"]
        gk = bo.bspline_backward(w["grad_q"], gs[1], gs[2], gs[3], traj_dt, gidx, imp, nk, degree)
        return w["cost"], gk, (w, v, a, j)
    w, v, a, j = check_chain(fn, knots)
    for k in ("self_cost", "scene_cost", "pose_cost", "cspace_cost"):
        assert (w[k].reshape(B, -1).sum(-1) > 0).all(), k
    assert any(live_hinges(rm, state_cfg(), v, a, j))


@pytest.mark.parametrize("H", [9, 10, 14, 30])
@pytest.mark.parametrize("implicit", [0, 1])
def test_clique_chain(f64, H, implicit):
    """u -> clique stencil -> rollout (self, Lie pose, cuboids, STATE) -> clique adjoint, in float64: grad_u is the derivative."""
    robot = "franka"
    rm = load_robot(robot)
    B, D = 3, rm.num_dof
    u = G.walk(G.colliding_rows(rm, robot, B, 50 + H), H - 4, 50 + H, sigma=0.03).astype(np.float64)
    start, goal, sidx, gidx, traj_dt, _ = boundary_rows(rm, robot, u, 51 + H)
    imp = np.array([implicit, implicit], np.uint8)
    cfg = state_cfg().to_oracle_cfg(rm.num_tool_frames)
    kw = rollout_kw(rm, robot, B, 53, chain_world(robot))

    def fn(x):
        p, v, a, j, odt = co.clique_forward(x, *start[:3], goal[0], sidx, gidx, traj_dt, imp, H, dtype=np.float64)
        w = CS.rollout_cost_grad(rm, p, cfg, vel=v, acc=a, jerk=j, dt=odt, **kw)
        gs = w["cspace_grads"]
        return w["cost"], co.clique_backward(w["grad_q"], gs[1], gs[2], gs[3], traj_dt, gidx, imp, dtype=np.float64), w
    w = check_chain(fn, u)
    for k in ("self_cost", "pose_cost", "cspace_cost"):
        assert (w[k].reshape(B, -1).sum(-1) > 0).mean() > 0.5, k


def effort_setup(B, H, seed):
    """Franka with random inertial parameters, effort limits inside the torques of the case (the hinge is live)."""
    c = make_case("franka", B * H, seed)
    D = c["D"]
    rng = np.random.default_rng(seed)
    q = G.walk(G.configurations(c["rm"], "franka", B, seed), H, seed, sigma=0.05).astype(np.float64)
    qd = rng.uniform(-1.5, 1.5, size=q.shape)
    qdd = rng.uniform(-3.0, 3.0, size=q.shape)
    tau = do.rnea_forward(q.reshape(-1, D).astype(np.float32), qd.reshape(-1, D).astype(np.float32),
                          qdd.reshape(-1, D).astype(np.float32), *model_args(c))[0]
    elim = np.stack([np.quantile(tau, 0.25, axis=0), np.quantile(tau, 0.75, axis=0)])
    return c, q, qd, qdd, elim


def effort_cost(c, q, qd, qdd, jerk, dt, elim, weight, act, reg, retime=True):
    """The effort channel of the STATE cost on tau = RNEA(q, qd, qdd): cost [B,H,D], gradients (q, qd, qdd) through the RNEA
    adjoint, tau."""
    B, H, D = q.shape
    rm, m = c["rm"], model_args(c)
    tau, cache = do.rnea_forward(q.reshape(-1, D), qd.reshape(-1, D), qdd.reshape(-1, D), *m)
    lim = dict(p=rm.position_limits, v=rm.velocity_limits, a=rm.acceleration_limits, j=rm.jerk_limits, tau=elim)
    w_eff = np.array([0, 0, 0, 0, weight[4]], np.float64)
    r_eff = np.array([0, 0, 0, reg[3], reg[4]], np.float64)
    cost, g = O.cspace_state_cost(q, qd, qdd, jerk, dt, lim, w_eff, act, r_eff, retime, retime, effort=tau.reshape(B, H, D))
    bq, bqd, bqdd = do.rnea_backward(g[4].reshape(-1, D), q.reshape(-1, D), qd.reshape(-1, D), cache, *m)
    r = lambda x: np.asarray(x).reshape(B, H, D)  # noqa: E731
    return cost, (g[0] + r(bq), g[1] + r(bqd), g[2] + r(bqdd)), r(tau)


@pytest.mark.parametrize("B,H,retime", [(3, 4, True), (2, 9, False)])
def test_rnea_effort_chain(f64, B, H, retime):
    """q, qd, qdd -> RNEA -> effort hinge, squared-L2 and energy terms -> RNEA adjoint (Franka, float64): the gradients with
    respect to q, qd and qdd are the derivative."""
    c, q, qd, qdd, elim = effort_setup(B, H, 61 + H)
    rng = np.random.default_rng(H)
    jerk = rng.normal(0, 50.0, size=q.shape)
    dt = rng.uniform(0.02, 0.1, size=B)
    weight, act, reg = (0, 0, 0, 0, 20.0), np.array([0.01, 0.01, 0.01, 0.01, 0.05]), (0, 0, 0, 0.05, 0.3)
    assert do.F is np.float64

    def fn(x):
        cost, g, tau = effort_cost(c, x[:, :H], x[:, H:2 * H], x[:, 2 * H:], jerk, dt, elim, weight, act, reg, retime)
        return cost.reshape(B, -1).sum(-1), np.concatenate(g, axis=1), (cost, tau)
    cost, tau = check_chain(fn, np.concatenate([q, qd, qdd], axis=1))
    assert tau.dtype == np.float64 and (cost.reshape(B, -1).sum(-1) > 0).all()
    assert ((tau < elim[0]) | (tau > elim[1])).mean() > 0.2, "the effort hinge must be live"
