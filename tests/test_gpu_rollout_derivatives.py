"""The fused rollout's gradient against float64 derivatives of its own cost, on every kernel family.

Every other test of `grad_q` compares it with something built the same way (the float32 oracle restates the kernel's backward
formulas; the variant tests compare one kernel with another).  Here the float64 oracle (oracle/rollout_oracle.py and
oracle/current_state_oracle.py with their `F` set to float64) is the cost, and its central differences are the derivative.
tests/test_rollout_derivatives_cpu.py pins which terms of that cost have a gradient that is their true derivative; these cases use
only those terms, plus the axis-angle rotation, whose gradient is exactly half the derivative by the reference's design.

Per case and kernel family (forced with CB200_BIG / CB200_ARM_PAIRS / CB200_TEAM, asserted with cb200_last_rollout_variant()):
(1) cost: each row's cost and each term's row cost equal the float64 oracle's (float32 rounding);
(2) gradient: for N_DIR random directions d_b [H, D] per row b, sum(grad_q[b] * d_b) equals the float64 central difference of
    cost[b] (all rows perturbed at once, rows are independent), within TOL of sum(|grad_q[b] * d_b|);
(3) kink guard: a row/direction counts only if the central differences at eps 1e-5 and 1e-6 agree to 1e-6 (hinges, the goalset
    argmin, the worst self-collision pair and cuboid ridges are kinks); at least 90 % count, and every term under test is active
    in most counted rows;
(4) the cost-only twins give the float64 cost as well.
The float64 reference of a case (cost and central differences) does not depend on the family, so it is computed once per case.

The ESDF's gradient is the normalised gradient of the trilinear field (compute_local_sdf_with_grad), the derivative only where the
interpolated field has unit slope: the ESDF cases use a tilted planar field, stored exactly in fp16, which has that slope
everywhere.  Franka reaches the standard kernel only with mesh obstacles in the scene; its "standard" runs add one mesh box far
out of reach, which adds no cost.  Swept collision and the speed metric are not derivatives and are left to the parity tests."""
import functools

import numpy as np
import pytest
import torch

from test_gpu_cost_only import COST_VARIANT, GRAD_VARIANT, VARIANT_ENV, last_variant
from helpers import humanoid_q, random_q
from curobo_b200 import lib as cblib
from curobo_b200.robot_model import load_robot
from curobo_b200.rollout import RolloutConfig, RolloutEngine
from curobo_b200.scene import CuboidData, VoxelData
from curobo_b200.world import CuboidWorld, VoxelWorld
from oracle import current_state_oracle as CS
from oracle import rollout_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VARIANT_ENV = dict(VARIANT_ENV, team4={"CB200_BIG": "1", "CB200_TEAM": "4"}, traj={"CB200_BIG": "0"})
GRAD_VARIANT = dict(GRAD_VARIANT, team4=6, traj=7)          # include/curobo_b200.h: CB200_VARIANT_TEAM4 6, TRAJ 7
N_DIR = 4
EPS = (1e-5, 1e-6)
KINK = 1e-6
# |an - fd| / sum|grad_q * d|.  Worst measured over every case: 2.3e-6 on the emulated device, 3.1e-6 on an H100 80GB HBM3
# (700 W power limit).  A gradient scaled by 1.001 in one place measured 7e-4 to 9e-4.
TOL = 2e-5
COST_RTOL = 2e-5
ROT = [0.9238795, 0.0, 0.3826834, 0.0]                    # 45 degrees about y
TABLE = {"dims": [2.2, 2.2, 0.2], "pose": [0.0, 0.0, -0.1, 1, 0, 0, 0]}
PILLAR = {"dims": [0.1, 0.1, 1.5], "pose": [0.45, 0.0, 0.3, 1, 0, 0, 0]}
TILTED_BOX = {"dims": [0.3, 0.25, 0.4], "pose": [0.35, 0.25, 0.45] + ROT}


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def sync():
    if DEV != "cpu":
        torch.cuda.synchronize()


def float64_oracle(monkeypatch):
    monkeypatch.setattr(O, "F", np.float64)
    monkeypatch.setattr(CS, "F", np.float64)


# ------------------------------------------------------------------------------------------------ scenes
def planar_esdf(height, buried=False):
    """A 64^3 grid of 1/16 m voxels holding z - height in its own frame (multiples of 1/32, exact in fp16), tilted 30 degrees
    about x: the trilinear field is linear with unit slope everywhere.  `buried`: the plane lies above the whole robot."""
    k = (np.arange(64, dtype=np.float64) - 31.5) * 0.0625
    sdf = np.broadcast_to(k[None, None, :] - height, (64, 64, 64))
    pose = (0, 0, 0.0, 1, 0, 0, 0) if buried else (0, 0, 0.3, 0.9659258, 0.2588190, 0, 0)
    return VoxelWorld.from_grid(sdf, 0.0625, pose=pose)


def two_env_cuboids():
    """env 0: table + pillar + the tilted box; env 1: a wall rotated about z and a box on the other side."""
    c0 = CuboidWorld.create([TABLE, PILLAR, TILTED_BOX], max_n=3)
    c1 = CuboidWorld.create([{"dims": [0.05, 1.5, 1.5], "pose": [0.35, 0.0, 0.5, 0.9659258, 0, 0, 0.2588190]},
                             {"dims": [0.3, 0.3, 0.3], "pose": [0.0, 0.5, 0.4, 1, 0, 0, 0]}], max_n=3)
    return CuboidWorld(np.concatenate([c0.dims, c1.dims]), np.concatenate([c0.inv_pose, c1.inv_pose]),
                       np.concatenate([c0.enable, c1.enable]), np.concatenate([c0.count, c1.count]))


def far_mesh():
    from curobo_b200.mesh import MeshData, MeshWorld, box_mesh
    v, f = box_mesh([0.1, 0.1, 0.1])
    return MeshData.from_world(MeshWorld.create([{"vertices": v, "faces": f, "pose": [10.0, 10.0, 10.0, 1, 0, 0, 0]}], max_n=2), DEV)


# ------------------------------------------------------------------------------------------------ cases
def configurations(rm, robot, n, seed):
    return (random_q(rm, n, seed=seed) if robot == "franka" else humanoid_q(rm, n, seed=seed, scale=0.5)).astype(np.float32)


def colliding_rows(rm, robot, n, seed, cub=None, vox=None, need_self=True):
    """n configurations with self collision (and scene collision when a world is given), one joint per row pushed beyond the
    activation band of its limit so the c-space hinge is live on every row."""
    cand = configurations(rm, robot, 40 * n if robot == "franka" else 12 * n, seed)
    lim = np.asarray(rm.position_limits, np.float32)
    j = np.random.default_rng(seed).integers(0, rm.num_dof, size=cand.shape[0])
    side = np.arange(cand.shape[0]) % 2
    r = np.arange(cand.shape[0])
    cand[r, j] = np.where(side == 1, lim[1, j] - 0.004 * (lim[1, j] - lim[0, j]), lim[0, j] + 0.004 * (lim[1, j] - lim[0, j]))
    w = O.rollout_cost_grad(rm, cand[:, None], dict(self_weight=1.0, scene_weight=1.0, scene_eta=0.05), world_cuboid=cub,
                            world_voxel=vox)
    ok = np.ones(cand.shape[0], bool)
    if need_self:
        ok &= w["self_cost"][:, 0] > 0
    if cub is not None or vox is not None:
        ok &= w["scene_cost"][:, 0].sum(-1) > 0
    idx = np.nonzero(ok)[0]
    assert idx.size >= n, (robot, idx.size, n)
    return np.ascontiguousarray(cand[idx[:n]])


def goalset(rm, robot, n_goals, seed):
    """[G, L, 2, 3|4]: two goals per tool frame, from two configurations (the argmin picks either)."""
    _, _, gp, gq = O.fk_forward(rm, configurations(rm, robot, 2 * n_goals, seed))
    L = rm.num_tool_frames
    gp = np.ascontiguousarray(gp.reshape(2, n_goals, L, 3).transpose(1, 2, 0, 3), np.float32)
    gq = np.ascontiguousarray(gq.reshape(2, n_goals, L, 4).transpose(1, 2, 0, 3), np.float32)
    return gp, gq


def walk(q0, H, seed, sigma=0.01):
    steps = np.random.default_rng(seed).normal(0, sigma, size=(q0.shape[0], H, q0.shape[1])).astype(np.float32)
    steps[:, 0] = 0
    return np.ascontiguousarray(q0[:, None, :] + np.cumsum(steps, axis=1), np.float32)


def _case(name, dev):
    """Case dict: robot, cfg (RolloutConfig), q [B,H,D] f32, sel (rows the derivative check runs on), worlds, goals, per-row
    inputs, the terms that must be active and the relation (an = relation * fd)."""
    seed = sum(map(ord, name))
    robot = name.split("-")[0]
    rm = load_robot(robot)
    D = rm.num_dof
    c = dict(robot=robot, rm=rm, cub=None, vox=None, goal=None, target=None, current=None, state=None, env=None, relation=1.0)
    ik = RolloutConfig(self_weight=1000.0, scene_weight=1000.0, scene_activation=0.05, pose_weight=(1000.0, 100.0), pose_lie=True,
                       cspace_type="position", cspace_weight=(5000.0, 0, 0, 0, 0), cspace_activation=(0.01, 0, 0, 0, 0),
                       cspace_target_weight=10.0)
    dofw = np.linspace(0.5, 1.5, D).astype(np.float32)
    dofw[2] = 0.0
    if name in ("franka-ik", "franka-many_rows"):
        c["cub"] = CuboidWorld.create([TABLE, PILLAR, TILTED_BOX], max_n=3)
        n = 33 if name == "franka-ik" else None
        if n is None:
            sms = 2 if dev == "cpu" else torch.cuda.get_device_properties(dev).multi_processor_count
            n = sms * 4 * 8 * 2 + 7          # more warps than the arm build keeps resident (3 CTAs x 8 warps per SM)
        q = colliding_rows(rm, robot, min(n, 40), seed, cub=c["cub"])
        if n > q.shape[0]:                   # the rest: plain random rows, the checked ones spread over the batch
            rest = configurations(rm, robot, n, seed + 1)
            sel = np.linspace(0, n - 1, q.shape[0]).round().astype(np.int64)
            rest[sel] = q
            q, c["sel"] = rest, sel
        c.update(cfg=ik, q=q[:, None, :], terms=("self_cost", "scene_cost", "pose_cost", "cspace_cost"))
    elif name == "franka-velocity":        # H = 1 rows: current state with dt, both regularizers, dt = 0 rows, two environments
        cub = two_env_cuboids()
        n = 33
        q = colliding_rows(rm, robot, n, seed, cub=CuboidWorld(cub.dims[:1], cub.inv_pose[:1], cub.enable[:1], cub.count[:1]))
        c.update(cub=cub, env=(np.arange(n) % 2).astype(np.int32))
        cfg = RolloutConfig.retarget_ik()
        cfg.pose_lie, cfg.scene_activation, cfg.cspace_reg = True, 0.05, (0.5, 0.05, 0, 0, 0)
        c.update(cfg=cfg, q=q[:, None, :], terms=("pose_cost", "cspace_cost"))
    elif name == "franka-velocity_traj":   # H = 8 rows of the trajectory kernel (no scene: its collision term is swept)
        n, H = 7, 8
        q = walk(colliding_rows(rm, robot, n, seed), H, seed)
        cfg = RolloutConfig.retarget_ik()
        cfg.pose_lie, cfg.use_sweep, cfg.scene_weight, cfg.cspace_reg = True, True, 0.0, (0.5, 0.05, 0, 0, 0)
        c.update(cfg=cfg, q=q, terms=("pose_cost", "cspace_cost"))
    elif name.startswith("franka-state"):  # trajectory kernel, STATE c-space cost (bounds, target, non-terminal factor)
        H = int(name.rsplit("_h", 1)[1])
        n = {1: 6, 9: 4, 30: 3}[H]
        q = walk(colliding_rows(rm, robot, n, seed), H, seed)
        rng = np.random.default_rng(seed)
        v, a, j = [rng.normal(0, s, size=q.shape).astype(np.float32) for s in (2.0, 12.0, 400.0)]
        cfg = RolloutConfig.mpc()
        cfg.scene_weight, cfg.use_speed_metric, cfg.pose_lie, cfg.retime_weights = 0.0, False, True, True
        c.update(cfg=cfg, q=q, state=(v, a, j, rng.uniform(0.02, 0.1, size=n).astype(np.float32)),
                 terms=("self_cost", "pose_cost", "cspace_cost"))
    elif name in ("g1_29-esdf", "g1_43-esdf", "g1_43-buried"):
        buried = name.endswith("buried")
        c["vox"] = planar_esdf(1.875 if buried else 0.0, buried)
        n = {"g1_29-esdf": 12, "g1_43-esdf": 8, "g1_43-buried": 8}[name]
        q = colliding_rows(rm, robot, n, seed, vox=c["vox"])
        c.update(cfg=ik, q=q[:, None, :], terms=("self_cost", "scene_cost", "pose_cost", "cspace_cost"))
    elif name.endswith("axis_angle"):      # rotation only, the reference's axis-angle error: an = 0.5 fd
        H = 9 if name.endswith("traj_axis_angle") else 1
        n = 9 if robot == "franka" else 6
        q = walk(configurations(rm, robot, n, seed), H, seed, sigma=0.03) if H > 1 else configurations(rm, robot, n, seed)[:, None]
        cfg = RolloutConfig(pose_weight=(0.0, 100.0), use_sweep=H > 1)
        c.update(cfg=cfg, q=np.ascontiguousarray(q), terms=("pose_cost",), relation=0.5)
    else:
        raise KeyError(name)
    B = c["q"].shape[0]
    c.setdefault("sel", np.arange(B))
    if c["cfg"].pose_weight is not None:
        gp, gq = goalset(rm, robot, 3, seed + 2)
        c["goal"] = (gp, gq, (np.arange(B) % 3).astype(np.int32))
    if c["cfg"].cspace_target_weight > 0:
        c["target"] = (configurations(rm, robot, 2, seed + 3), (np.arange(B) % 2).astype(np.int32), dofw)
    if name.startswith("franka-velocity"):
        # current-state rows: dt 0.05 and 0.08 (even rows start within a few steps of theirs, odd rows are far outside the
        # window), a row with dt = 0 (no current state)
        rng = np.random.default_rng(seed + 4)
        cur_p = configurations(rm, robot, 3, seed + 5)
        cur_v = rng.normal(0, 0.4, size=(3, D)).astype(np.float32)
        idx = (np.arange(B) % 3).astype(np.int32)
        dt = np.array([0.05, 0.0, 0.08], np.float32)
        lim_v = np.asarray(rm.velocity_limits, np.float32)
        q = c["q"].copy()
        q[0::2] = cur_p[idx[0::2]][:, None, :] + rng.normal(0, 1.0, size=q[0::2].shape).astype(np.float32) * lim_v[1] * 0.05
        c["q"] = np.ascontiguousarray(q, np.float32)
        c["current"] = (cur_p, cur_v, idx, dt)
    return c


_cases = functools.lru_cache(maxsize=None)(_case)


def case(name):
    return _cases(name, DEV)


def oracle(c, q, sel):
    """The oracle's outputs for rows `sel` at q [len(sel), H, D] (the precision is the oracle modules' F)."""
    kw = dict(world_cuboid=c["cub"], world_voxel=c["vox"])
    if c["goal"] is not None:
        kw.update(goal_pos=c["goal"][0], goal_quat=c["goal"][1], idxs_goal=c["goal"][2][sel])
    if c["target"] is not None:
        kw.update(cspace_target=c["target"][0], idxs_cspace_target=c["target"][1][sel], cspace_target_dof_weight=c["target"][2])
    if c["env"] is not None:
        kw["env_query_idx"] = c["env"][sel]
    if c["state"] is not None:
        v, a, j, dt = c["state"]
        kw.update(vel=v[sel], acc=a[sel], jerk=j[sel], dt=dt[sel])
    if c["current"] is not None:
        p, v, idx, dt = c["current"]
        kw.update(current_position=p, current_velocity=v, idxs_current=idx[sel], state_dt=dt)
    return CS.rollout_cost_grad(c["rm"], q, c["cfg"].to_oracle_cfg(c["rm"].num_tool_frames), **kw)


def reference(name):
    return _reference(name, DEV)


@functools.lru_cache(maxsize=None)
def _reference(name, dev):
    """float64: the oracle at the case's rows, the directions [N_DIR, n, H, D] and the central differences [2, N_DIR, n]."""
    assert O.F is np.float64 and CS.F is np.float64
    c = case(name)
    sel = c["sel"]
    q = c["q"][sel].astype(np.float64)
    w = oracle(c, q, sel)
    d = np.random.default_rng(7).standard_normal((N_DIR,) + q.shape)
    fd = np.stack([np.stack([(oracle(c, q + e * dk, sel)["cost"] - oracle(c, q - e * dk, sel)["cost"]) / (2 * e) for dk in d])
                   for e in EPS])
    return w, d, fd


def engine(c, family):
    cub = CuboidData.from_world(c["cub"], DEV) if c["cub"] is not None else None
    vox = VoxelData.from_world(c["vox"], DEV) if c["vox"] is not None else None
    mesh = far_mesh() if family == "standard" and c["robot"] == "franka" else None
    eng = RolloutEngine(c["rm"], c["cfg"], DEV, cub, vox, mesh=mesh)
    if c["goal"] is not None:
        eng.update_goal(T(c["goal"][0]), T(c["goal"][1]), T(c["goal"][2]))
    if c["target"] is not None:
        eng.update_cspace_target(T(c["target"][0]), T(c["target"][1]), T(c["target"][2]))
    if c["current"] is not None:
        p, v, idx, dt = c["current"]
        eng.update_current_state(T(p), T(v), T(dt), T(idx))
    return eng


def launch_kw(c):
    kw = {}
    if c["env"] is not None:
        kw["env_query_idx"] = T(c["env"])
    if c["state"] is not None:
        kw.update(zip(("vel", "acc", "jerk", "dt"), (T(x) for x in c["state"])))
    return kw


def row_terms(o, sel):
    """Per-row sums of cost and each term, numpy [n]."""
    s = torch.as_tensor(sel, device=o.cost.device)
    return {k: getattr(o, k)[s].reshape(len(sel), -1).double().sum(-1).cpu().numpy()
            for k in ("cost", "self_cost", "scene_cost", "pose_cost", "cspace_cost")}


def want_terms(w):
    B = w["cost"].shape[0]
    return {k: (w[k].reshape(B, -1).sum(-1) if k in w else np.zeros(B)) for k in ("cost", "self_cost", "scene_cost", "pose_cost",
                                                                               "cspace_cost")}


def check_costs(got, want, label):
    for k, v in want.items():
        tol = COST_RTOL * np.abs(v) + 1e-6 * max(float(np.abs(v).max()), 1e-6)
        err = np.abs(got[k] - v)
        assert np.all(err <= tol), f"{label} {k}: worst {float((err / np.maximum(np.abs(v), 1e-30)).max()):.3g} relative"


def derivative_errors(grad, d, fd, relation):
    """grad [n,H,D] (kernel, f64), d [N_DIR,n,H,D], fd [2,N_DIR,n] -> (error [N_DIR,n], counted [N_DIR,n])."""
    an = np.einsum("bhk,rbhk->rb", grad, d)
    scale = np.einsum("bhk,rbhk->rb", np.abs(grad), np.abs(d))
    counted = np.abs(fd[0] - fd[1]) <= KINK * np.maximum(np.abs(fd[1]), scale)
    err = np.abs(an - relation * fd[1]) / np.maximum(scale, 1e-30)
    return err, counted


def run_case(monkeypatch, name, family):
    float64_oracle(monkeypatch)
    c = case(name)
    w, d, fd = reference(name)
    cost_only = family.startswith("cost_")
    base = family.replace("cost_", "")
    for k, v in VARIANT_ENV[base].items():
        monkeypatch.setenv(k, v)
    eng = engine(c, base)
    q = T(c["q"])
    o = eng.evaluate_cost(q, **launch_kw(c)) if cost_only else eng.evaluate_action(q, **launch_kw(c))
    sync()
    want_variant = COST_VARIANT[base] | cblib.VARIANT_COST_ONLY if cost_only else GRAD_VARIANT[base]
    assert last_variant() == want_variant, (last_variant(), want_variant)
    sel = c["sel"]
    check_costs(row_terms(o, sel), want_terms(w), f"{name} {family}")
    if cost_only:
        return None
    if name == "franka-many_rows":
        assert int(eng._work_counter.abs().sum()) == 0, "the ticket counter was not re-armed"
    grad = o.grad_q[torch.as_tensor(sel, device=o.grad_q.device)].double().cpu().numpy()
    err, counted = derivative_errors(grad, d, fd, c["relation"])
    frac = float(counted.mean())
    worst = float(err[counted].max())
    print(f"DERIV {name} {family}: worst {worst:.3g}, kink guard dropped {1 - frac:.1%} of {counted.size}")
    assert frac >= 0.9, f"the kink guard dropped {1 - frac:.1%} of the row/directions"
    rows = counted.any(0)
    if name.endswith("buried"):
        assert int((w["scene_cost"] > 0).reshape(len(sel), -1).sum(-1).min()) > 96, "every row must overflow the gradient list"
    for k in c["terms"]:
        active = float((want_terms(w)[k][rows] > 0).mean())
        assert active > 0.5, f"{k} active in only {active:.0%} of the counted rows"
    assert worst <= TOL, f"{name} {family}: sum(grad_q * d) vs the float64 derivative: worst {worst:.3g} of sum|grad_q * d|"
    return worst


RUNS = [("franka-ik", f) for f in ("arm", "pairs", "standard", "big", "cost_arm", "cost_big")] + \
       [("franka-velocity", f) for f in ("arm", "pairs", "big", "cost_arm", "cost_big")] + \
       [("franka-velocity_traj", "traj")] + \
       [(f"franka-state_h{H}", "traj") for H in (1, 9, 30)] + \
       [("g1_29-esdf", f) for f in ("standard", "big", "team", "team4", "cost_standard", "cost_big")] + \
       [(c, f) for c in ("g1_43-esdf", "g1_43-buried") for f in ("big", "team")] + \
       [("franka-many_rows", "arm")]
AXIS_ANGLE_RUNS = [("franka-axis_angle", f) for f in ("arm", "pairs", "big")] + [("franka-traj_axis_angle", "traj")] + \
                  [("g1_29-axis_angle", f) for f in ("standard", "big", "team", "team4")]


@pytest.mark.parametrize("name,family", RUNS)
def test_gradient_is_derivative_of_cost(monkeypatch, name, family):
    run_case(monkeypatch, name, family)


@pytest.mark.parametrize("name,family", AXIS_ANGLE_RUNS)
def test_axis_angle_gradient_is_half_the_derivative(monkeypatch, name, family):
    """The reference's axis-angle rotation error (compute_rotation_error_axis_angle, wp_tool_pose.py) hand-defines its gradient
    with a scale factor that makes it exactly half the derivative of its cost; every family reproduces that factor."""
    run_case(monkeypatch, name, family)
