"""Mesh obstacles inside the fused rollout kernels (RolloutEngine(..., mesh=MeshData)).

Pins: (1) the fused kernels equal the per-operator composition FK -> self collision + SphereObstacleCollision(SceneData(cuboid,
voxel, mesh)) -> autograd backward on every kernel family that has a mesh build (standard, big, trajectory), bit for bit on the
scene cost of a mesh-only discrete world; (2) the brute-force mesh oracle (tests/mesh_rollout_oracle.py); (3) a box mesh costs what
the analytic cuboid costs (the reference's regression, tests/_src/collision/test_mesh_collision_sdf.py:17-60); (4) scene
combinations, environments, disabled slots, empty environments; (5) scene_weight = 0 ignores the meshes; (6) CUDA-graph replay and
in-place pose updates; (7) the schedules without a mesh build refuse mesh scenes; (8) full-size determinism.
Variants are forced with CB200_BIG / CB200_TEAM and checked through cb200_last_rollout_variant()."""
import numpy as np
import pytest
import torch

import mesh_rollout_oracle as MRO
from helpers import humanoid_q, random_q, random_walk_q, small_voxel_world
from curobo_b200.kinematics import Kinematics, SelfCollisionCost
from curobo_b200.mesh import MeshData, MeshWorld, box_mesh, icosphere
from curobo_b200.robot_model import load_robot
from curobo_b200.rollout import RolloutConfig, RolloutEngine
from curobo_b200.scene import (CollisionBuffer, CuboidData, SceneData, SphereObstacleCollision, SweptSphereObstacleCollision,
                               VoxelData)
from curobo_b200.world import CuboidWorld, make_benchmark_cuboid_world
from oracle import rollout_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
V_STANDARD, V_BIG, V_TRAJ = 1, 4, 7  # include/curobo_b200.h: CB200_VARIANT_*

TABLE = {"dims": [2.2, 2.2, 0.2], "pose": [0.0, 0.0, -0.1, 1, 0, 0, 0]}
PILLAR = {"dims": [0.1, 0.1, 1.5], "pose": [0.45, 0.0, 0.3, 1, 0, 0, 0]}
ROT = [0.9238795, 0.0, 0.3826834, 0.0]


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def last_variant():
    from curobo_b200 import lib as cblib
    return int(cblib.load().cb200_last_rollout_variant())


def sync():
    if DEV != "cpu":
        torch.cuda.synchronize()


def box(c):
    v, f = box_mesh(c["dims"])
    return {"vertices": v, "faces": f, "pose": c["pose"]}


def ball(r, pose, subdiv=2):
    v, f = icosphere(r, subdiv)
    return {"vertices": v, "faces": f, "pose": pose}


def mesh_world(robot):
    """A table and a rotated, translated icosphere where the robot's spheres reach them."""
    if robot == "franka":
        return MeshWorld.create([box(TABLE), ball(0.2, [0.35, 0.25, 0.45] + ROT)], max_n=3)
    return MeshWorld.create([ball(0.25, [0.25, 0.0, 0.8] + ROT), box({"dims": [0.3, 0.2, 0.4], "pose": [0.0, 0.3, 0.5] + ROT})],
                            max_n=3)


def scene_of(robot, kind):
    """(CuboidData, VoxelData, MeshData, MeshWorld): kind "mesh" = meshes only, "all" = pillar cuboid + ESDF + meshes."""
    mw = mesh_world(robot)
    cub = vox = None
    if kind == "all":
        cub = CuboidData.from_world(CuboidWorld.create([PILLAR], max_n=2), DEV)
        vox = VoxelData.from_world(small_voxel_world(), DEV)
    return cub, vox, MeshData.from_world(mw, DEV), mw


def rows(rm, robot, n, H=1, seed=0):
    """[n, H, D]: random configurations (H = 1) or short joint-space walks from them, inside the joint limits."""
    q = (random_q(rm, n, seed=seed) if robot == "franka" else humanoid_q(rm, n, seed=seed, scale=0.5))[:, None, :]
    if H > 1:
        walk = np.cumsum(np.random.default_rng(seed).normal(0, 0.03, (n, H, q.shape[-1])), axis=1)
        lim = np.asarray(rm.position_limits, np.float32)
        q = np.clip(q + walk, lim[0], lim[1])
    return np.ascontiguousarray(q, np.float32)


def composition(rm, q, cfg, scene, env=None, dt=None):
    """FK -> self collision + scene collision (per-operator launches) -> autograd backward."""
    B, H, _ = q.shape
    kin = Kinematics(rm, DEV)
    selfc = SelfCollisionCost(rm, cfg.self_weight, DEV)
    buf = CollisionBuffer.from_shape((B, H, rm.num_spheres, 4), DEV)
    qg = q.clone().requires_grad_(True)
    st = kin.compute_kinematics(qg)
    d_self = selfc.forward(st.robot_spheres)
    w, eta = T(np.array([cfg.scene_weight], np.float32)), T(np.array([cfg.scene_activation], np.float32))
    if env is None:
        env = torch.zeros(B, dtype=torch.int32, device=DEV)
    multi = bool(env.abs().sum() > 0)
    if not cfg.use_sweep:
        d_scene = SphereObstacleCollision.apply(st.robot_spheres, buf, scene, w, eta, None, env, multi, False)
    else:
        d_scene = SweptSphereObstacleCollision.apply(st.robot_spheres, buf, scene, w, eta, None, T(np.array([dt], np.float32)),
                                                     cfg.use_speed_metric, env, multi, False)
    (d_self.sum() + d_scene.sum()).backward()
    sync()
    return d_self.detach(), d_scene.detach(), qg.grad


def _variant_env(monkeypatch, variant):
    monkeypatch.setenv("CB200_BIG", "1" if variant == "big" else "0")
    monkeypatch.setenv("CB200_TEAM", "2")            # the team kernel has no mesh build: mesh scenes must stay on the big kernel


CASES = [("franka", "standard", "all", 257, 1), ("franka", "standard", "mesh", 300, 1), ("franka", "big", "mesh", 100, 1),
         ("g1_29", "standard", "all", 64, 1), ("g1_29", "big", "all", 200, 1), ("g1_43", "big", "mesh", 64, 1),
         ("franka", "traj", "all", 8, 12), ("g1_29", "traj", "all", 4, 9)]


@pytest.mark.parametrize("robot,variant,kind,n,H", CASES)
def test_fused_matches_per_operator_composition(monkeypatch, robot, variant, kind, n, H):
    rm = load_robot(robot)
    _variant_env(monkeypatch, variant)
    traj = variant == "traj"
    cfg = RolloutConfig(self_weight=5000.0, scene_weight=5000.0, scene_activation=0.02, use_sweep=traj, use_speed_metric=traj)
    cub, vox, mesh, _ = scene_of(robot, kind)
    q = T(rows(rm, robot, n, H, seed=11))
    dt = 0.05
    eng = RolloutEngine(rm, cfg, DEV, cub, vox, mesh=mesh)
    o = eng.evaluate_action(q, dt=T(np.full(n, dt, np.float32)) if traj else None)
    sync()
    assert last_variant() == {"standard": V_STANDARD, "big": V_BIG, "traj": V_TRAJ}[variant]
    d_self, d_scene, g = composition(rm, q, cfg, SceneData(cub, vox, mesh), dt=dt)
    assert int((o.scene_cost > 0).sum()) > 2, "no sphere collides"
    torch.testing.assert_close(o.self_cost.view(-1), d_self.view(-1), rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(o.scene_cost, d_scene, rtol=1e-5, atol=1e-4)
    if kind == "mesh" and not traj:
        assert torch.equal(o.scene_cost, d_scene)
    torch.testing.assert_close(o.grad_q, g, rtol=2e-3, atol=2e-5 * float(g.abs().max()))


@pytest.mark.parametrize("n", [48])
def test_fused_vs_mesh_oracle(n):
    """Rotated, translated icosphere and box, self + pose + c-space terms on: the oracle's tolerances (SURVEY.md 8c)."""
    rm = load_robot("franka")
    mw = MeshWorld.create([ball(0.2, [0.35, 0.25, 0.45] + ROT, 1),
                           box({"dims": [0.3, 0.25, 0.4], "pose": [0.3, -0.3, 0.3, 0.8660254, 0.0, 0.0, 0.5]})], max_n=2)
    cfg = RolloutConfig.ik()
    cfg.scene_activation = 0.02
    q = random_q(rm, n, seed=21)[:, None, :]
    _, _, gp, gq = O.fk_forward(rm, random_q(rm, 4, seed=22))
    gp, gq = gp[:, :, None, :].copy(), gq[:, :, None, :].copy()
    idx = (np.arange(n) % 4).astype(np.int32)
    eng = RolloutEngine(rm, cfg, DEV, mesh=MeshData.from_world(mw, DEV))
    eng.update_goal(T(gp), T(gq), T(idx))
    o = eng.evaluate_action(T(q))
    sync()
    want = MRO.rollout_cost_grad(rm, q, cfg.to_oracle_cfg(1), world_mesh=mw, goal_pos=gp, goal_quat=gq, idxs_goal=idx)
    assert (want["scene_cost"] > 0).sum() > 20
    np.testing.assert_allclose(o.scene_cost.cpu().numpy(), want["scene_cost"], rtol=1e-4, atol=1e-6 * want["scene_cost"].max())
    np.testing.assert_allclose(o.cost.cpu().numpy(), want["cost_bh"], rtol=1e-4, atol=1e-6 * want["cost_bh"].max())
    g = want["grad_q"]
    np.testing.assert_allclose(o.grad_q.cpu().numpy(), g, rtol=1e-3, atol=1e-5 * np.abs(g).max())


@pytest.mark.parametrize("robot,variant,n,H", [("franka", "standard", 200, 1), ("franka", "big", 100, 1), ("g1_29", "big", 64, 1),
                                                ("franka", "traj", 6, 10)])
def test_box_mesh_costs_what_the_cuboid_costs(monkeypatch, robot, variant, n, H):
    """Same box as a mesh and as a cuboid: same row and sphere costs (gradients are not compared: outside the surface the mesh
    gradient has the opposite sign, data_mesh.py:694-698, as in the per-operator path)."""
    rm = load_robot(robot)
    _variant_env(monkeypatch, variant)
    traj = variant == "traj"
    b = {"dims": [0.5, 0.4, 0.6], "pose": [0.3, 0.1, 0.3] + ROT} if robot == "franka" else \
        {"dims": [0.4, 0.5, 0.6], "pose": [0.15, 0.0, 0.6] + ROT}
    cfg = RolloutConfig(self_weight=5000.0, scene_weight=5000.0, scene_activation=0.02, use_sweep=traj, use_speed_metric=traj)
    q = T(rows(rm, robot, n, H, seed=31))
    kw = dict(dt=T(np.full(n, 0.05, np.float32))) if traj else {}
    om = RolloutEngine(rm, cfg, DEV, mesh=MeshData.from_world(MeshWorld.create([box(b)]), DEV)).evaluate_action(q, **kw)
    sync()
    assert last_variant() == {"standard": V_STANDARD, "big": V_BIG, "traj": V_TRAJ}[variant]
    oc = RolloutEngine(rm, cfg, DEV, CuboidData.from_world(CuboidWorld.create([b]), DEV)).evaluate_action(q, **kw)
    sync()
    dc = oc.scene_cost.cpu().numpy()
    assert (dc > 0).sum() > 20 and (dc == 0).sum() > 20
    np.testing.assert_allclose(om.scene_cost.cpu().numpy(), dc, rtol=2e-4, atol=2e-6 * dc.max())
    c = oc.cost.cpu().numpy()
    np.testing.assert_allclose(om.cost.cpu().numpy(), c, rtol=2e-4, atol=2e-6 * c.max())


def test_scene_combinations_envs_disabled_and_empty(n=90):
    """Cuboids + ESDF + meshes together; three environments picked by env_query_idx (env 2 has no mesh: count = 0); a disabled
    mesh slot equals the world without that mesh."""
    rm = load_robot("franka")
    cfg = RolloutConfig(self_weight=5000.0, scene_weight=5000.0, scene_activation=0.02)
    tbl, bl = box(TABLE), ball(0.2, [0.35, 0.25, 0.45] + ROT)
    mw = MeshWorld([[tbl, bl], [ball(0.25, [0.3, -0.2, 0.3] + ROT)], []], max_n=2)
    mesh = MeshData.from_world(mw, DEV)
    cub = CuboidData.from_world(CuboidWorld.create([PILLAR], max_n=2), DEV)
    vox = VoxelData.from_world(small_voxel_world(), DEV)
    q = T(rows(rm, "franka", n, seed=41))
    env = T((np.arange(n) % 3).astype(np.int32))
    o = RolloutEngine(rm, cfg, DEV, cub, vox, mesh=mesh).evaluate_action(q, env_query_idx=env)
    sync()
    d_self, d_scene, g = composition(rm, q, cfg, SceneData(cub, vox, mesh), env=env)
    torch.testing.assert_close(o.scene_cost, d_scene, rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(o.grad_q, g, rtol=2e-3, atol=2e-5 * float(g.abs().max()))
    # meshes only: env 2 (count = 0) sees nothing, env 1 sees its own mesh
    om = RolloutEngine(rm, cfg, DEV, mesh=mesh).evaluate_action(q, env_query_idx=env)
    sync()
    sc = om.scene_cost.clone()
    assert float(sc[2::3].abs().sum()) == 0.0 and float(sc[0::3].sum()) > 0 and float(sc[1::3].sum()) > 0
    single = MeshData.from_world(MeshWorld.create([mw.envs[1][0]]), DEV)
    o1 = RolloutEngine(rm, cfg, DEV, mesh=single).evaluate_action(q[1::3].contiguous())
    sync()
    assert torch.equal(o1.scene_cost, sc[1::3]) and torch.equal(o1.grad_q, om.grad_q[1::3])
    # disabled slot (the icosphere of env 0), updated in place: no refresh_world needed
    eng = RolloutEngine(rm, cfg, DEV, mesh=mesh)
    mesh.enable[0, 1] = 0
    od = eng.evaluate_action(q[0::3].contiguous())
    sync()
    ot = RolloutEngine(rm, cfg, DEV, mesh=MeshData.from_world(MeshWorld.create([tbl]), DEV)).evaluate_action(q[0::3].contiguous())
    sync()
    assert torch.equal(od.scene_cost, ot.scene_cost) and torch.equal(od.grad_q, ot.grad_q)
    assert not torch.equal(od.scene_cost, sc[0::3])


def test_zero_scene_weight_ignores_meshes(n=64):
    rm = load_robot("franka")
    cfg = RolloutConfig.ik()
    cfg.scene_weight = 0.0
    q = T(rows(rm, "franka", n, seed=51))
    _, _, gp, gq = O.fk_forward(rm, random_q(rm, 2, seed=52))
    outs = []
    for mesh in (MeshData.from_world(mesh_world("franka"), DEV), None):
        eng = RolloutEngine(rm, cfg, DEV, CuboidData.from_world(make_benchmark_cuboid_world(), DEV), mesh=mesh)
        eng.update_goal(T(gp[:, :, None, :].copy()), T(gq[:, :, None, :].copy()), T((np.arange(n) % 2).astype(np.int32)))
        o = eng.evaluate_action(q)
        sync()
        outs.append({k: getattr(o, k).clone() for k in ("cost", "grad_q", "self_cost", "scene_cost", "pose_cost", "cspace_cost")})
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k


def test_graph_replay_and_in_place_pose_update(n=512):
    """The mesh pose tensor updated in place between calls (and between graph replays) is picked up without refresh_world()."""
    rm = load_robot("franka")
    cfg = RolloutConfig(self_weight=5000.0, scene_weight=5000.0, scene_activation=0.02)
    mw = mesh_world("franka")
    mesh = MeshData.from_world(mw, DEV)
    q = T(rows(rm, "franka", n, seed=61))
    eng = RolloutEngine(rm, cfg, DEV, mesh=mesh)
    o = eng.evaluate_action(q)
    sync()
    ref = (o.cost.clone(), o.grad_q.clone())
    moved = MeshWorld.create([mw.envs[0][0], dict(mw.envs[0][1], pose=[0.3, -0.25, 0.4] + ROT)], max_n=3)
    want = RolloutEngine(rm, cfg, DEV, mesh=MeshData.from_world(moved, DEV)).evaluate_action(q)
    sync()
    want = (want.cost.clone(), want.grad_q.clone())
    assert not torch.equal(want[0], ref[0])
    new_pose = MeshData.from_world(moved, DEV).inv_pose
    old_pose = mesh.inv_pose.clone()
    if DEV == "cpu":          # (no CUDA graphs on the emulated device: the in-place update between eager calls)
        mesh.inv_pose.copy_(new_pose)
        o = eng.evaluate_action(q)
        assert torch.equal(o.cost, want[0]) and torch.equal(o.grad_q, want[1])
        return
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        eng.evaluate_action(q)
    for pose, expect in ((old_pose, ref), (new_pose, want), (old_pose, ref)):
        mesh.inv_pose.copy_(pose)
        eng.out.cost.zero_()
        eng.out.grad_q.zero_()
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(eng.out.cost, expect[0]) and torch.equal(eng.out.grad_q, expect[1])


def test_schedules_without_mesh_build_refuse_mesh_scenes():
    """In-kernel spline and the fused-dynamics kernel raise ValueError with a mesh; the expanded spline schedule works and equals
    evaluate_action on the states it expanded."""
    from dynamics_cases import effort_cost_setup
    from curobo_b200.dynamics import Dynamics
    from curobo_b200.trajectory import JointState
    c = effort_cost_setup("franka", 2, 3)[0]
    rm = c["rm"]
    B, nk, D = 3, 6, rm.num_dof
    mesh = MeshData.from_world(mesh_world("franka"), DEV)
    cfg = RolloutConfig.trajopt()
    knots = random_walk_q(rm, B, nk, seed=71).astype(np.float32)
    z = np.zeros((B, D), np.float32)
    start = JointState(T(knots[:, 0].copy()), T(z), T(z), T(z))
    goal = JointState(T(knots[:, -1].copy()), T(z), T(z), T(z), dt=T(np.full(B, 0.05, np.float32)))
    sidx = T(np.arange(B, dtype=np.int32))
    imp = T(np.zeros(B, np.uint8))
    eng = RolloutEngine(rm, cfg, DEV, mesh=mesh)
    with pytest.raises(ValueError, match="in_kernel_spline=False"):
        eng.evaluate_knots(T(knots), start, sidx, goal, sidx, imp, in_kernel_spline=True)
    o = eng.evaluate_knots(T(knots), start, sidx, goal, sidx, imp)
    sync()
    assert last_variant() == V_TRAJ
    cost = o.cost.clone()
    assert torch.isfinite(cost).all() and torch.isfinite(o.grad_knots).all() and float(o.scene_cost.sum()) > 0
    st = [t.clone() for t in eng._state]
    o2 = RolloutEngine(rm, cfg, DEV, mesh=mesh).evaluate_action(st[0], vel=st[1], acc=st[2], jerk=st[3], dt=eng._state_dt.clone())
    sync()
    assert torch.equal(o2.cost, cost)
    H = 5
    q = T(random_walk_q(rm, B, H, seed=72))
    v = torch.zeros_like(q)
    eng_d = RolloutEngine(rm, cfg, DEV, mesh=mesh)
    eng_d.attach_dynamics(Dynamics(rm, c["mc"], c["inn"], gravity=(0.0, 0.0, -9.81), device=DEV), fused=True)
    with pytest.raises(ValueError, match="fused=False"):
        eng_d.evaluate_action(q, vel=v, acc=v, jerk=v, dt=T(np.full(B, 0.05, np.float32)))


def test_full_size_ik_and_mpc_against_meshes():
    """16,384 Franka IK rows and 1024 x 30 MPC trajectories against the table + icosphere: run-to-run identical, finite."""
    rm = load_robot("franka")
    mesh = MeshData.from_world(mesh_world("franka"), DEV)
    q = T(rows(rm, "franka", 16384, seed=81))
    eng = RolloutEngine(rm, RolloutConfig.ik(), DEV, mesh=mesh)
    _, _, gp, gq = O.fk_forward(rm, random_q(rm, 512, seed=82))
    eng.update_goal(T(gp[:, :, None, :].copy()), T(gq[:, :, None, :].copy()), T((np.arange(16384) // 32).astype(np.int32)))
    runs = [tuple(t.clone() for t in (o.cost, o.grad_q)) for o in (eng.evaluate_action(q), eng.evaluate_action(q))]
    sync()
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert torch.isfinite(runs[0][0]).all() and torch.isfinite(runs[0][1]).all() and float(eng.out.scene_cost.sum()) > 0
    B, H = 1024, 30
    qm = T(random_walk_q(rm, B, H, seed=83))
    z = torch.zeros_like(qm)
    dt = T(np.full(B, 0.05, np.float32))
    cfg = RolloutConfig.mpc()
    eng = RolloutEngine(rm, cfg, DEV, mesh=mesh)
    eng.update_goal(T(gp[:, :, None, :].copy()), T(gq[:, :, None, :].copy()), T((np.arange(B) % 512).astype(np.int32)))
    eng.update_cspace_target(T(random_q(rm, B, seed=84)), T(np.arange(B, dtype=np.int32)))
    runs = [tuple(t.clone() for t in (o.cost, o.grad_q)) for o in (eng.evaluate_action(qm, vel=z, acc=z, jerk=z, dt=dt),
                                                                  eng.evaluate_action(qm, vel=z, acc=z, jerk=z, dt=dt))]
    sync()
    assert last_variant() == V_TRAJ
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert torch.isfinite(runs[0][0]).all() and torch.isfinite(runs[0][1]).all() and float(eng.out.scene_cost.sum()) > 0
