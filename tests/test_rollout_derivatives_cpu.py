"""The float64 oracle's gradient against central differences of its own cost, term by term (CPU, no device).

tests/test_gpu_rollout_derivatives.py takes the oracle, run in float64, as the cost whose derivative the fused kernels' `grad_q`
must be.  These tests pin which terms of that cost have a gradient that is its derivative, on Franka and G1-29, at H = 1 and
H > 1:
  * exact: tool position, Lie-group rotation with unit axis weights, self collision, rotated cuboids (eta > 0), a planar ESDF
    (unit slope), the POSITION c-space bound and target, its current-state block (velocity window that clips, both
    regularizers, rows with dt = 0) and the STATE c-space position bound and target;
  * by the reference's design: the axis-angle rotation's gradient is exactly 0.5 x the derivative (the hand-defined scale factor
    of compute_rotation_error_axis_angle, wp_tool_pose.py, carried through the quaternion-rate map);
  * not derivatives, so not covered by the derivative tests: the ESDF on a field without unit slope (the gradient is normalised,
    compute_local_sdf_with_grad), swept collision and the speed metric.  Those are pinned here as measured, so that a change to
    them shows up.
A row/direction counts only where the central differences at eps 1e-5 and 1e-6 agree (kinks: hinges, worst pair, cuboid ridges)."""
import numpy as np
import pytest

import test_gpu_rollout_derivatives as G
from helpers import small_voxel_world
from curobo_b200.robot_model import load_robot
from curobo_b200.rollout import RolloutConfig
from curobo_b200.world import CuboidWorld
from oracle import current_state_oracle as CS
from oracle import rollout_oracle as O

N_DIR = 3
EXACT = 1e-6


@pytest.fixture
def f64(monkeypatch):
    monkeypatch.setattr(O, "F", np.float64)
    monkeypatch.setattr(CS, "F", np.float64)


def rows(robot, n, H, seed, **kw):
    rm = load_robot(robot)
    q = G.colliding_rows(rm, robot, n, seed, **kw)
    return rm, (G.walk(q, H, seed) if H > 1 else q[:, None, :]).astype(np.float64)


def probe(rm, q, cfg, seed=1, **kw):
    """(an [N_DIR,B], fd [N_DIR,B], scale [N_DIR,B], counted [N_DIR,B], oracle output at q)."""
    w = CS.rollout_cost_grad(rm, q, cfg, **kw)
    assert w["grad_q"].dtype == np.float64
    d = np.random.default_rng(seed).standard_normal((N_DIR,) + q.shape)
    fd = np.stack([np.stack([(CS.rollout_cost_grad(rm, q + e * dk, cfg, **kw)["cost"] -
                              CS.rollout_cost_grad(rm, q - e * dk, cfg, **kw)["cost"]) / (2 * e) for dk in d]) for e in G.EPS])
    an = np.einsum("bhk,rbhk->rb", w["grad_q"], d)
    scale = np.einsum("bhk,rbhk->rb", np.abs(w["grad_q"]), np.abs(d))
    counted = np.abs(fd[0] - fd[1]) <= G.KINK * np.maximum(np.abs(fd[1]), scale)
    return an, fd[1], scale, counted, w


def assert_relation(res, relation=1.0, tol=EXACT, term=None):
    an, fd, scale, counted, w = res
    assert counted.mean() >= 0.9, counted.mean()
    err = np.abs(an - relation * fd) / np.maximum(scale, 1e-30)
    assert float(err[counted].max()) <= tol, float(err[counted].max())
    if term is not None:
        B = w["cost"].shape[0]
        assert (w[term].reshape(B, -1).sum(-1) > 0).mean() > 0.5, f"{term} inactive"


def goal_kw(rm, robot, B, seed=3):
    gp, gq = G.goalset(rm, robot, 3, seed)
    return dict(goal_pos=gp, goal_quat=gq, idxs_goal=np.arange(B) % 3)


ROBOTS = [("franka", 6, 1), ("franka", 3, 7), ("g1_29", 3, 1), ("g1_29", 2, 4)]


@pytest.mark.parametrize("robot,B,H", ROBOTS)
@pytest.mark.parametrize("term", ["position", "lie", "self", "cuboid", "planar_esdf", "cspace_position"])
def test_exact_terms(f64, robot, B, H, term):
    seed = 11 + H
    cub = CuboidWorld.create([G.TABLE, G.PILLAR, G.TILTED_BOX], max_n=3) if term == "cuboid" else None
    vox = G.planar_esdf(0.0) if term == "planar_esdf" else None
    rm, q = rows(robot, B, H, seed, cub=cub, vox=vox, need_self=term == "self")
    cfg, kw, name = {}, {}, None
    if term in ("position", "lie"):
        cfg = dict(pose_weight=[100.0, 0.0] if term == "position" else [0.0, 100.0], pose_lie=term == "lie")
        kw, name = goal_kw(rm, robot, B), "pose_cost"
    elif term == "self":
        cfg, name = dict(self_weight=100.0), "self_cost"
    elif term in ("cuboid", "planar_esdf"):
        cfg, kw, name = dict(scene_weight=100.0, scene_eta=0.05), dict(world_cuboid=cub, world_voxel=vox), "scene_cost"
    else:
        cfg = RolloutConfig(cspace_type="position", cspace_weight=(100.0, 0, 0, 0, 0), cspace_activation=(0.01, 0, 0, 0, 0),
                            cspace_target_weight=3.0).to_oracle_cfg(rm.num_tool_frames)
        dofw = np.linspace(0.5, 1.5, rm.num_dof)
        kw, name = dict(cspace_target=G.configurations(rm, robot, 2, 5), idxs_cspace_target=np.arange(B) % 2,
                        cspace_target_dof_weight=dofw), "cspace_cost"
    assert_relation(probe(rm, q, cfg, **kw), term=name)


@pytest.mark.parametrize("robot,B,H", ROBOTS)
def test_axis_angle_is_half_the_derivative(f64, robot, B, H):
    rm, q = rows(robot, B, H, 21 + H, need_self=False)
    assert_relation(probe(rm, q, dict(pose_weight=[0.0, 100.0]), **goal_kw(rm, robot, B)), relation=0.5, term="pose_cost")


@pytest.mark.parametrize("robot,B,H", [("franka", 6, 1), ("franka", 3, 8), ("g1_29", 3, 1)])
def test_current_state_block(f64, robot, B, H):
    """Velocity window (clipping on the rows far from their current state), both regularizers, a current-state row with dt = 0,
    and the target term, on the POSITION c-space cost."""
    rm, q = rows(robot, B, H, 31 + H, need_self=False)
    D = rm.num_dof
    rng = np.random.default_rng(3)
    cur_p = G.configurations(rm, robot, 3, 4).astype(np.float64)
    idx = np.arange(B) % 3
    lim_v = np.asarray(rm.velocity_limits, np.float64)
    q[0::2] = cur_p[idx[0::2]][:, None, :] + rng.normal(0, 1.0, size=q[0::2].shape) * lim_v[1] * 0.05
    cfg = RolloutConfig(cspace_type="position", cspace_weight=(100.0, 0, 0, 0, 0), cspace_activation=(0.01, 0, 0, 0, 0),
                        cspace_reg=(0.5, 0.05, 0, 0, 0), cspace_target_weight=3.0).to_oracle_cfg(rm.num_tool_frames)
    kw = dict(current_position=cur_p, current_velocity=rng.normal(0, 0.4, size=(3, D)), idxs_current=idx,
              state_dt=np.array([0.05, 0.0, 0.08]), cspace_target=G.configurations(rm, robot, 2, 5),
              idxs_cspace_target=np.arange(B) % 2)
    res = probe(rm, q, cfg, **kw)
    assert_relation(res, term="cspace_cost")
    # the window clips: on some rows the bound of the window is tighter than the joint limits and violated
    lo = np.maximum(rm.position_limits[0][None] + 0.01 * np.ptp(rm.position_limits, 0)[None], cur_p + lim_v[0] * 0.05)
    assert (q[idx == 0] < lo[0][None, None, :]).any()
    # and the block is live: without it the cost differs on the rows with dt > 0 only
    plain = O.rollout_cost_grad(rm, q, cfg, cspace_target=kw["cspace_target"], idxs_cspace_target=kw["idxs_cspace_target"])
    on = np.array([0.05, 0.0, 0.08])[idx] > 0
    assert np.all(res[4]["cost"][on] != plain["cost"][on]) and np.array_equal(res[4]["cost"][~on], plain["cost"][~on])


@pytest.mark.parametrize("H", [1, 9])
def test_state_cspace_position_part(f64, H):
    """STATE c-space cost with velocity / acceleration / jerk given (their bound and regularization terms are constants in q):
    the position bound, the target term and its non-terminal factor are exact."""
    rm = load_robot("franka")
    B = 4
    q = G.walk(G.configurations(rm, "franka", B, 5) * 1.2, H, 5).astype(np.float64)
    rng = np.random.default_rng(H)
    v, a, j = [rng.normal(0, s, size=q.shape) for s in (2.0, 12.0, 400.0)]
    cfg = RolloutConfig.mpc()
    cfg.scene_weight = 0.0
    kw = dict(vel=v, acc=a, jerk=j, dt=rng.uniform(0.02, 0.1, size=B), cspace_target=G.configurations(rm, "franka", 2, 6),
              idxs_cspace_target=np.arange(B) % 2, cspace_target_dof_weight=np.linspace(0.5, 1.5, 7))
    assert_relation(probe(rm, q, cfg.to_oracle_cfg(1), **kw), term="cspace_cost")


def test_not_derivatives_as_measured(f64):
    """Terms outside the derivative tests, as measured on Franka: the ESDF of boxes (normalised gradient of an fp16 field),
    swept collision and the speed metric.  Each gradient differs from the derivative by more than 100 x the tolerance of the exact terms."""
    rm = load_robot("franka")
    _, q1 = rows("franka", 4, 1, 41, need_self=False, vox=small_voxel_world())
    res = probe(rm, q1, dict(scene_weight=100.0, scene_eta=0.02), world_voxel=small_voxel_world())
    err = np.abs(res[0] - res[1]) / res[2]
    assert err[res[3]].max() > 100 * EXACT
    cub = CuboidWorld.create([G.TABLE, G.PILLAR, G.TILTED_BOX], max_n=3)
    _, qH = rows("franka", 3, 9, 42, need_self=False, cub=cub)
    for speed in (False, True):
        res = probe(rm, qH, dict(scene_weight=100.0, scene_eta=0.05, sweep=True, speed_metric=speed), world_cuboid=cub,
                    dt=np.full(3, 0.05))
        err = np.abs(res[0] - res[1]) / res[2]
        assert err.max() > 100 * EXACT, (speed, err.max())
