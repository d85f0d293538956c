"""Link spheres changed at run time (RolloutEngine.update_link_spheres / disable / enable / reset / attach_object_spheres ->
cb200_refresh_robot_spheres): the engine then computes, bit for bit, what an engine built from the modified model computes, and
its device blob is byte for byte the packer's for that model.

Pins, on every kernel variant (forced with CB200_BIG / CB200_ARM_PAIRS / CB200_TEAM and checked through
cb200_last_rollout_variant()) and the trajectory kernel, in cuboid, ESDF and mesh worlds and for a robot whose pair list is not a
union of link blocks (no broad-phase bounds in the blob): (1) update == fresh engine, gradient and cost-only launches, for an
attached object, a sphere grown past its packed bound, the hand disabled as a grasp does, and a reset back to the model;
(2) per-environment configurations; (3) CUDA graphs captured before an update, and a refresh captured in a graph;
(4) the B200RobotRollout forwarding and in-place writes; (5) attach_object_spheres against a float64 restatement of
AttachmentManager.update; (6) refusals."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from helpers import small_voxel_world
from test_gpu_cost_only import GRAD_VARIANT, COST_VARIANT, VARIANT_ENV
from test_gpu_fused_mesh import PILLAR, TABLE, mesh_world, rows
from curobo_b200 import lib as cblib
from curobo_b200.mesh import MeshData
from curobo_b200.robot_model import load_robot
from curobo_b200.rollout import RolloutConfig, RolloutEngine, pack_robot_blob
from curobo_b200.scene import CuboidData, VoxelData
from curobo_b200.world import CuboidWorld
from oracle import rollout_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
INVALID = 1  # cudaErrorInvalidValue
TERMS = ("cost", "grad_q", "self_cost", "scene_cost", "pose_cost", "cspace_cost")
COST_TERMS = ("cost", "self_cost", "scene_cost", "pose_cost", "cspace_cost")
VARIANT_ENV = dict(VARIANT_ENV, traj={"CB200_BIG": "0"})
GRAD_VARIANT = dict(GRAD_VARIANT, traj=7)   # CB200_VARIANT_TRAJ


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def sync():
    if DEV != "cpu":
        torch.cuda.synchronize()


def last_variant():
    return int(cblib.load().cb200_last_rollout_variant())


def robot_of(name):
    """"<robot>" or "<robot>-pairlist" (without its first collision pair: no link-pair list, no bounds in the blob)."""
    robot, _, tag = name.partition("-")
    rm = load_robot(robot)
    if tag == "pairlist":
        rm = dataclasses.replace(rm, collision_pairs=np.ascontiguousarray(rm.collision_pairs[1:]))
    return robot, rm


def world(robot, kind, n_env=1):
    cub = vox = mesh = None
    if kind == "cuboid":
        w = CuboidWorld.create([TABLE, PILLAR], max_n=3)
        if n_env > 1:
            w = CuboidWorld(*(np.concatenate([a] * n_env) for a in (w.dims, w.inv_pose, w.enable, w.count)))
        cub = CuboidData.from_world(w, DEV)
    elif kind == "esdf":
        vox = VoxelData.from_world(small_voxel_world(), DEV)
    else:
        mesh = MeshData.from_world(mesh_world(robot), DEV)
    return cub, vox, mesh


def make_engine(rm, robot, kind, n, traj=False, n_env=1):
    """IK cost (self, scene, pose, c-space bound) or, with traj, swept collision over H = 30 waypoints."""
    if traj:
        cfg = RolloutConfig(self_weight=5000.0, scene_weight=5000.0, scene_activation=0.02, use_sweep=True,
                            pose_weight=(1000.0, 100.0), cspace_type="position", cspace_weight=(5000.0, 0, 0, 0, 0),
                            cspace_activation=(0.01, 0, 0, 0, 0))
    else:
        cfg = RolloutConfig.ik()
        cfg.scene_activation = 0.02
    cub, vox, mesh = world(robot, kind, n_env)
    eng = RolloutEngine(rm, cfg, DEV, cub, vox, mesh=mesh)
    _, _, gp, gq = O.fk_forward(rm, rows(rm, robot, 4, seed=21)[:, 0], env_query_idx=np.zeros(4, np.int32))
    eng.update_goal(T(gp[:, :, None, :].copy()), T(gq[:, :, None, :].copy()), T((np.arange(n) % 4).astype(np.int32)))
    return eng


def sphere_slots(rm, link):
    return np.nonzero(rm.link_sphere_idx_map == rm.link_names.index(link))[0]


def attach_link(rm):
    return "attached_object" if "attached_object" in rm.link_names else rm.collision_link_names[-1]


def object_spheres(k):
    """k spheres big enough to reach the table / pillar and the forearm from the hand."""
    s = np.array([[0.0, 0.0, 0.08, 0.12], [0.0, 0.0, -0.12, 0.1], [0.08, 0.0, 0.12, 0.1], [-0.08, 0.0, 0.12, 0.1]], np.float32)
    return s[:k]


def scenario_ops(rm, name):
    """[(method, args)] applied through the API and their effect on a copy of the model's link_spheres [n_cfg, S, 4]."""
    link = attach_link(rm)
    k = min(4, len(sphere_slots(rm, link)))
    grow = next(l for l in rm.collision_link_names if len(sphere_slots(rm, l)) >= 2)
    g = rm.link_spheres.reshape(-1, rm.num_spheres, 4)[0, sphere_slots(rm, grow)[:1]].copy()
    g[0, :3] += np.array([0.06, -0.04, 0.05], np.float32)
    g[0, 3] += 0.08
    hand = ["panda_hand", "panda_leftfinger", "panda_rightfinger"] if rm.name == "franka" or "panda_hand" in rm.link_names \
        else list(rm.collision_link_names[-3:])
    ops = {"attach": [("update_link_spheres", (link, object_spheres(k)))],
           "grow": [("update_link_spheres", (grow, g))],
           "grasp": [("disable_link_spheres", (h,)) for h in hand],
           "reset": [("update_link_spheres", (link, object_spheres(k))), ("update_link_spheres", (grow, g)),
                     ("disable_link_spheres", (hand[0],)), ("reset_link_spheres", (link,)), ("reset_link_spheres", (grow,)),
                     ("enable_link_spheres", (hand[0],))]}[name]
    ls = np.array(rm.link_spheres.reshape(-1, rm.num_spheres, 4), np.float32)
    ref = ls.copy()
    for meth, args in ops:
        idx = sphere_slots(rm, args[0])
        if meth == "update_link_spheres":
            ls[:, idx[:len(args[1])]] = args[1]
        elif meth == "disable_link_spheres":
            ls[:, idx, 3] = -100.0
        elif meth == "enable_link_spheres":
            ls[:, idx, 3] = ref[:, idx, 3]
        else:
            ls[:, idx] = ref[:, idx]
    return ops, ls


def apply_ops(target, ops):
    for meth, args in ops:
        args = tuple(T(a) if isinstance(a, np.ndarray) else a for a in args)
        getattr(target, meth)(*args)


def with_spheres(rm, ls):
    return dataclasses.replace(rm, link_spheres=ls if ls.shape[0] > 1 or rm.link_spheres.ndim == 3 else ls[0])


def snapshot(o, names):
    return {k: getattr(o, k).clone() for k in names}


def assert_bitwise(got, want, what):
    for k in want:
        assert torch.equal(got[k], want[k]), f"{what}: {k} differs (max {float((got[k] - want[k]).abs().max())})"


CASES = [("franka", "arm", "cuboid", 300), ("franka", "pairs", "cuboid", 301), ("franka", "arm", "esdf", 200),
         ("franka", "standard", "mesh", 200), ("franka", "big", "esdf", 150), ("g1_29", "team", "esdf", 40),
         ("g1_29", "standard", "cuboid", 64), ("franka-pairlist", "arm", "cuboid", 300), ("franka", "traj", "esdf", 8)]
SCENARIOS = ["attach", "grow", "grasp", "reset"]


@pytest.mark.parametrize("scenario", SCENARIOS)
@pytest.mark.parametrize("robot,variant,kind,n", CASES)
def test_update_equals_fresh_engine(monkeypatch, robot, variant, kind, n, scenario):
    name = robot
    robot, rm = robot_of(name)
    for k, v in VARIANT_ENV[variant].items():
        monkeypatch.setenv(k, v)
    traj = variant == "traj"
    H = 30 if traj else 1
    q = T(rows(rm, robot, n, H=H, seed=11))
    eng = make_engine(rm, robot, kind, n, traj)
    before = snapshot(eng.evaluate_action(q), TERMS)
    ops, ls = scenario_ops(rm, scenario)
    apply_ops(eng, ops)
    got = snapshot(eng.evaluate_action(q), TERMS)
    sync()
    assert last_variant() == GRAD_VARIANT[variant]
    rm2 = with_spheres(rm, ls)
    assert np.array_equal(eng.link_spheres.cpu().numpy(), ls)
    assert np.array_equal(eng._blob.cpu().numpy(), pack_robot_blob(rm2)), "device blob != packer's blob"
    fresh = make_engine(rm2, robot, kind, n, traj)
    assert_bitwise(got, snapshot(fresh.evaluate_action(q), TERMS), f"{name} {variant} {kind} {scenario}")
    if scenario == "reset":
        assert_bitwise(got, before, "reset vs original engine")
        assert np.array_equal(eng._blob.cpu().numpy(), pack_robot_blob(rm))
    if scenario == "attach" and robot == "franka" and kind == "cuboid" and n >= 200:   # rows enough to reach table and forearm
        idx = torch.as_tensor(sphere_slots(rm, "attached_object"), device=q.device)
        assert float(before["scene_cost"][..., idx].abs().sum()) == 0.0
        assert float(got["scene_cost"][..., idx].sum()) > 0.0, "the attached spheres touch no obstacle"
        assert bool((got["self_cost"] > before["self_cost"]).any()), "the attached spheres touch no robot sphere"
    if not traj:                                                    # the cost-only twin on the same blob
        got_c = snapshot(eng.evaluate_cost(q), COST_TERMS)
        assert last_variant() == COST_VARIANT[variant] | cblib.VARIANT_COST_ONLY
        assert_bitwise(got_c, snapshot(fresh.evaluate_cost(q), COST_TERMS), f"cost-only {name} {variant} {kind} {scenario}")


def test_per_environment_configuration(monkeypatch, n=90):
    """n_cfg = 3: configuration 1 gets an attached object; rows of environment 1 change to what a fresh engine computes, rows of
    environments 0 and 2 stay bit for bit."""
    monkeypatch.setenv("CB200_BIG", "0")
    rm = load_robot("franka")
    rm3 = dataclasses.replace(rm, link_spheres=np.stack([rm.link_spheres] * 3))
    q = T(rows(rm, "franka", n, seed=12))
    env = T((np.arange(n) % 3).astype(np.int32))
    eng = make_engine(rm3, "franka", "cuboid", n, n_env=3)
    before = snapshot(eng.evaluate_action(q, env_query_idx=env), TERMS)
    sph = object_spheres(4)
    eng.update_link_spheres("attached_object", T(sph), config_idx=1)
    got = snapshot(eng.evaluate_action(q, env_query_idx=env), TERMS)
    ls = rm3.link_spheres.copy()
    ls[1, sphere_slots(rm, "attached_object")] = sph
    fresh = make_engine(dataclasses.replace(rm, link_spheres=ls), "franka", "cuboid", n, n_env=3)
    want = snapshot(fresh.evaluate_action(q, env_query_idx=env), TERMS)
    assert_bitwise(got, want, "per-environment update")
    assert np.array_equal(eng._blob.cpu().numpy(), pack_robot_blob(dataclasses.replace(rm, link_spheres=ls)))
    keep = (np.arange(n) % 3) != 1
    for k in TERMS:
        assert torch.equal(got[k][keep], before[k][keep]), k
    assert not torch.equal(got["cost"][~keep], before["cost"][~keep])


def test_graphs_see_updates_without_recapture():
    """evaluate_action and an L-BFGS IK solve captured before an attach replay with the attached object; a refresh captured in a
    graph takes effect on replay."""
    from curobo_b200.optim import LBFGSOpt
    rm = load_robot("franka")
    n = 64
    q = T(rows(rm, "franka", n, seed=13))
    eng = make_engine(rm, "franka", "cuboid", n)
    eng.evaluate_action(q)
    sync()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eng.evaluate_action(q)
    ops, ls = scenario_ops(rm, "attach")
    apply_ops(eng, ops)
    eng.out.cost.zero_()
    g.replay()
    sync()
    fresh = make_engine(with_spheres(rm, ls), "franka", "cuboid", n)
    assert_bitwise(snapshot(eng.out, TERMS), snapshot(fresh.evaluate_action(q), TERMS), "graph replay after attach")
    # a refresh inside the graph: write the tensor, replay, the capture re-reads it
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2):
        eng.refresh_link_spheres()
        eng.evaluate_action(q)
    with torch.no_grad():
        eng.link_spheres.copy_(eng.reference_link_spheres)
    eng._link_spheres_version = eng.link_spheres._version       # as if the caller relied on the captured refresh alone
    g2.replay()
    sync()
    base = make_engine(rm, "franka", "cuboid", n)
    assert_bitwise(snapshot(eng.out, TERMS), snapshot(base.evaluate_action(q), TERMS), "refresh captured in a graph")
    assert np.array_equal(eng._blob.cpu().numpy(), pack_robot_blob(rm))
    # an L-BFGS IK solve captured before the attach
    from curobo_b200.optim import LBFGSOptCfg
    B, nls, D = 16, 4, rm.num_dof

    def solver(e):
        e.update_goal(*eng._goal[:2], T((np.arange(B * nls) // nls % 4).astype(np.int32)))

        def cost_grad(x):
            out = e.evaluate_action(x.view(B * nls, 1, D))
            return out.cost.view(-1), out.grad_q.view(B * nls, D)
        lim = T(rm.position_limits)
        return LBFGSOpt(LBFGSOptCfg(num_iters=8), B, 1, D, lim[0], lim[1], cost_grad, DEV)
    e1 = make_engine(rm, "franka", "cuboid", B * nls)
    opt = solver(e1)
    x0 = T(rows(rm, "franka", B, seed=32)).view(B, 1, D)
    opt.optimize_graphed(x0)
    apply_ops(e1, ops)
    got = opt.optimize_graphed(x0).clone()
    want = solver(make_engine(with_spheres(rm, ls), "franka", "cuboid", B * nls)).optimize_graphed(x0)
    sync()
    assert torch.equal(got, want)


def test_robot_rollout_forwarding_and_in_place_writes():
    from curobo_b200.rollout_protocol import B200RobotRollout
    rm = load_robot("franka")
    n = 48
    ro = B200RobotRollout(rm, RolloutConfig.ik(), DEV, cuboid=world("franka", "cuboid")[0])
    assert ro.link_spheres is ro.engine.link_spheres
    ops, ls = scenario_ops(rm, "attach")
    apply_ops(ro, ops)
    idx = sphere_slots(rm, "attached_object")
    assert np.array_equal(ro.get_link_spheres("attached_object").cpu().numpy(), ls[0, idx])
    assert np.array_equal(ro.engine._blob.cpu().numpy(), pack_robot_blob(with_spheres(rm, ls)))
    ro.detach_object_spheres()
    assert np.array_equal(ro.engine._blob.cpu().numpy(), pack_robot_blob(rm))
    ro.disable_link_spheres("panda_hand")
    ro.enable_link_spheres("panda_hand")
    ro.reset_link_spheres("panda_hand")
    assert np.array_equal(ro.engine._blob.cpu().numpy(), pack_robot_blob(rm))
    # an in-place write, picked up by the next eager call
    q = T(rows(rm, "franka", n, seed=14))
    with torch.no_grad():
        ro.link_spheres[:, torch.as_tensor(idx, device=q.device)] = T(object_spheres(4))
    ro.engine.evaluate_action(q)
    assert np.array_equal(ro.engine._blob.cpu().numpy(), pack_robot_blob(with_spheres(rm, ls)))
    ro.attach_object_spheres(T(object_spheres(2)))
    ro.refresh_link_spheres()
    assert float(ro.get_link_spheres("attached_object")[2:, 3].max()) == -100.0


def attach_oracle(rm, spheres, q, object_pose, n_cfg):
    """AttachmentManager.update in float64 numpy: obj_to_link = ee^-1 * object_pose per environment, centres mapped, the rest of
    the link's slots at radius -100, environment i into configuration i."""
    def qmul(a, b):
        aw, ax, ay, az = a
        bw, bx, by, bz = b
        return np.array([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                         aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw])

    def rot(qq, v):
        return qmul(qmul(qq, np.concatenate([[0.0], v])), qq * np.array([1, -1, -1, -1]))[1:]
    _, _, ee_p, ee_q = O.fk_forward(rm, q.astype(np.float32))
    ls = np.array(rm.link_spheres.reshape(-1, rm.num_spheres, 4), np.float64)
    ls = np.repeat(ls, n_cfg, 0) if ls.shape[0] == 1 else ls
    idx = sphere_slots(rm, "attached_object")
    for i in range(q.shape[0]):
        op = object_pose[min(i, object_pose.shape[0] - 1)].astype(np.float64)
        ei = np.asarray(ee_q[i, 0], np.float64) * np.array([1, -1, -1, -1])
        rq, rp = qmul(ei, op[3:]), rot(ei, op[:3] - ee_p[i, 0])
        env = np.zeros((len(idx), 4))
        env[:, 3] = -100.0
        for j, s in enumerate(spheres.astype(np.float64)):
            env[j, :3] = rot(rq, s[:3]) + rp
            env[j, 3] = s[3]
        ls[i, idx] = env
    return ls


def test_attach_object_spheres_vs_float64_restatement(n=40):
    rm = load_robot("franka")
    rm2 = dataclasses.replace(rm, link_spheres=np.stack([rm.link_spheres] * 2))
    eng = make_engine(rm2, "franka", "cuboid", n, n_env=2)
    qg = rows(rm, "franka", 2, seed=15)[:, 0]
    ang = 0.4
    pose = np.array([[0.45, 0.1, 0.35, np.cos(ang), 0.0, np.sin(ang), 0.0], [0.3, -0.2, 0.5, 1.0, 0.0, 0.0, 0.0]], np.float32)
    sph = object_spheres(3)
    eng.attach_object_spheres(T(sph), joint_position=T(qg), object_pose=T(pose))
    want = attach_oracle(rm, sph, qg, pose, 2)
    got = eng.link_spheres.cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=0, atol=2e-6)
    assert (got[:, sphere_slots(rm, "attached_object")[3:], 3] == -100.0).all()
    # the rollout equals a fresh engine built with the written spheres
    q = T(rows(rm, "franka", n, seed=16))
    env = T((np.arange(n) % 2).astype(np.int32))
    got_o = snapshot(eng.evaluate_action(q, env_query_idx=env), TERMS)
    fresh = make_engine(dataclasses.replace(rm, link_spheres=got.copy()), "franka", "cuboid", n, n_env=2)
    assert_bitwise(got_o, snapshot(fresh.evaluate_action(q, env_query_idx=env), TERMS), "attach_object_spheres")
    # one pose broadcast to both environments; no pose: link-frame centres
    eng.attach_object_spheres(T(sph), joint_position=T(qg), object_pose=T(pose[:1]))
    np.testing.assert_allclose(eng.link_spheres.cpu().numpy(), attach_oracle(rm, sph, qg, pose[:1], 2), rtol=0, atol=2e-6)
    eng.attach_object_spheres(T(sph))
    assert np.array_equal(eng.get_link_spheres("attached_object")[:3].cpu().numpy(), sph)
    eng.detach_object_spheres()
    assert np.array_equal(eng.link_spheres.cpu().numpy(), eng.reference_link_spheres.cpu().numpy())


def test_refusals():
    rm = load_robot("franka")
    eng = make_engine(rm, "franka", "cuboid", 8)
    blob = eng._blob.clone()
    ls = eng.link_spheres.clone()
    sph = T(object_spheres(4))
    bad = [lambda: eng.update_link_spheres("no_such_link", sph),
           lambda: eng.update_link_spheres("attached_object", T(np.zeros((5, 4), np.float32))),
           lambda: eng.update_link_spheres("attached_object", sph, start_sph_idx=1),
           lambda: eng.update_link_spheres("attached_object", T(np.zeros((4, 3), np.float32))),
           lambda: eng.update_link_spheres("attached_object", sph.double()),
           lambda: eng.update_link_spheres("attached_object", sph.cpu() if DEV != "cpu" else sph.to("meta")),
           lambda: eng.update_link_spheres("attached_object", sph, config_idx=1),
           lambda: eng.get_link_spheres("attached_object", config_idx=-1),
           lambda: eng.disable_link_spheres("nope"), lambda: eng.enable_link_spheres("nope"),
           lambda: eng.reset_link_spheres("nope"),
           lambda: eng.attach_object_spheres(T(np.zeros((5, 4), np.float32))),
           lambda: eng.attach_object_spheres(sph, joint_position=T(rows(rm, "franka", 2)[:, 0])),      # 2 envs, 1 configuration
           lambda: eng.attach_object_spheres(sph, object_pose=T(np.array([[0, 0, 0, 1, 0, 0, 0]], np.float32))),
           lambda: eng.attach_object_spheres(sph, joint_position=T(rows(rm, "franka", 1)[:, 0]),
                                             object_pose=T(np.zeros((1, 6), np.float32)))]
    for f in bad:
        with pytest.raises(ValueError):
            f()
    sync()
    assert torch.equal(eng._blob, blob) and torch.equal(eng.link_spheres, ls)
    L = cblib.load()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream if DEV != "cpu" else None)
    host = eng._blob_host
    nb = int(host.shape[0])
    args = lambda **kw: [kw.get("blob", eng._blob.data_ptr()), kw.get("host", host.ctypes.data), kw.get("nb", nb),  # noqa: E731
                         kw.get("ls", eng.link_spheres.data_ptr()), kw.get("n_cfg", 1), stream]
    assert L.cb200_refresh_robot_spheres(*args()) == 0
    assert L.cb200_refresh_robot_spheres(*args(n_cfg=2)) == INVALID
    assert L.cb200_refresh_robot_spheres(*args(nb=nb - 16)) == INVALID
    assert L.cb200_refresh_robot_spheres(*args(blob=None)) == INVALID
    assert L.cb200_refresh_robot_spheres(*args(host=None)) == INVALID
    assert L.cb200_refresh_robot_spheres(*args(ls=None)) == INVALID
    junk = np.zeros(nb, np.uint8)
    assert L.cb200_refresh_robot_spheres(*args(host=junk.ctypes.data)) == INVALID       # no blob magic
    sync()
    assert torch.equal(eng._blob, blob)
