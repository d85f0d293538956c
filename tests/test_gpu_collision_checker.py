"""Validity of joint configurations (RolloutEngine.validate -> cb200_rollout_validate) and RobotCollisionChecker.

(1) `validate` equals a float64 mask from the oracle (bounds, self-collision pairs, scene SDFs; the brute-force mesh oracle for
meshes) for Franka in cuboid, ESDF and mesh worlds, G1-29 and G1-43 against an ESDF, two environments, per-environment sphere
configurations, an attached object and a disabled link -- rows whose smallest margin is within 1e-5 of zero are left out, and
they must be under 1 %; (2) each single-check mask equals "that term's cost from evaluate_cost at activation 0 is 0", row for
row; (3) early exit changes nothing: the same masks with and without the ticket counter, and on a batch where nearly every row
collides; (4) graph capture; (5) the ABI's refusals and variant bit; (6) the checker's distance methods, sampling and
trajectory sampling."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from helpers import small_voxel_world
from test_gpu_fused_mesh import PILLAR, TABLE, mesh_world, rows
from curobo_b200 import lib as cblib
from curobo_b200.collision import RobotCollisionChecker
from curobo_b200.mesh import MeshData
from curobo_b200.robot_model import load_robot
from curobo_b200.rollout import RolloutConfig, RolloutEngine
from curobo_b200.scene import CuboidData, VoxelData
from curobo_b200.world import CuboidWorld
from oracle import mesh_oracle as MO
from oracle import rollout_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
INVALID = 1  # cudaErrorInvalidValue
EPS = 1e-5
COST_CFG = RolloutConfig(self_weight=1.0, scene_weight=1.0, scene_activation=0.0, cspace_type="position",
                         cspace_weight=(1.0, 0, 0, 0, 0), cspace_activation=(0.0,) * 5)


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def sync():
    if DEV != "cpu":
        torch.cuda.synchronize()


def draws(rm, robot, n, seed):
    """[n, 1, D]: half plausible configurations (test_gpu_fused_mesh.rows), half uniform in the limits widened by 5 %."""
    lo, hi = np.asarray(rm.position_limits, np.float32)
    u = np.random.default_rng(seed).uniform(-0.05, 1.05, (n - n // 2, rm.num_dof)).astype(np.float32)
    wide = lo + (hi - lo) * u
    return np.ascontiguousarray(np.concatenate([rows(rm, robot, n // 2, seed=seed), wide[:, None]]), np.float32)


def world(robot, kind):
    """(CuboidWorld | None, VoxelWorld | None, MeshWorld | None)."""
    if kind == "cuboid":
        return CuboidWorld.create([TABLE, PILLAR], max_n=3), None, None
    if kind == "esdf":
        return None, small_voxel_world(), None
    if kind == "mesh":
        return None, None, mesh_world(robot)
    if kind == "two_env":
        from test_gpu_rollout import _two_env_worlds
        cub, vox = _two_env_worlds()
        return cub, vox, None
    raise ValueError(kind)


def checker_of(rm, cw, vw, mw, **kw):
    return RobotCollisionChecker(rm, DEV, CuboidData.from_world(cw, DEV) if cw is not None else None,
                                 VoxelData.from_world(vw, DEV) if vw is not None else None,
                                 MeshData.from_world(mw, DEV) if mw is not None else None, **kw)


# ------------------------------------------------------------------------------------------------ float64 oracle margins
def margins(rm, q, cw, vw, mw, env=None, link_spheres=None):
    """Per row [N]: (bound margin: min over dofs of min(q - lo, hi - q), >= 0 when inside; scene margin: max over enabled spheres
    and obstacles of r - sdf, > 0 in contact; self margin: max over pairs with padded radii >= 0 of r_i + r_j - |p_i - p_j|,
    > 0 in contact), all in float64."""
    q = np.asarray(q, np.float64).reshape(-1, rm.num_dof)
    N = q.shape[0]
    env = np.zeros(N, np.int64) if env is None else np.asarray(env, np.int64)
    lo, hi = np.asarray(rm.position_limits, np.float64)
    bound = np.minimum(q - lo, hi - q).min(1)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(O, "F", np.float64)
        rmx = rm if link_spheres is None else dataclasses.replace(rm, link_spheres=link_spheres)
        _, sph, _, _ = O.fk_forward(rmx, q, env_query_idx=env)
        scene = np.full(N, -np.inf)
        for e in np.unique(env):
            sel = np.nonzero(env == e)[0]
            sp = sph[sel]
            active = sp[..., 3] >= 0
            for inv_row, sdf_fn in O._obstacles(cw, vw, int(e)):
                ip, iq = O._load_inv_transform(inv_row)
                loc = O._quat_rotate(np.broadcast_to(iq, sp.shape[:-1] + (4,)), sp[..., :3]) + ip
                sdf, _ = sdf_fn(loc)
                scene[sel] = np.maximum(scene[sel], np.where(active, sp[..., 3] - sdf, -np.inf).max(1))
            if mw is not None:
                from curobo_b200.world import _inv_pose_from_pose
                for m in mw.envs[int(e)][:mw.max_n]:
                    ip, iq = O._load_inv_transform(_inv_pose_from_pose(m.get("pose", (0, 0, 0, 1, 0, 0, 0))))
                    loc = O._quat_rotate(np.broadcast_to(iq, sp.shape[:-1] + (4,)), sp[..., :3]) + ip
                    sdf, _ = MO.mesh_sdf_grad(m["vertices"], m["faces"], loc.reshape(-1, 3),
                                              query_distance=float(sp[..., 3].max()))
                    scene[sel] = np.maximum(scene[sel], np.where(active, sp[..., 3] - sdf.reshape(sp.shape[:2]), -np.inf).max(1))
        pairs = np.asarray(rm.collision_pairs, np.int64)
        pad = np.asarray(rm.sphere_padding, np.float64)
        selfm = np.full(N, -np.inf)
        for n0 in range(0, N, 8):
            s = sph[n0:n0 + 8]
            r = s[..., 3] + pad
            ri, rj = r[:, pairs[:, 0]], r[:, pairs[:, 1]]
            d = np.linalg.norm(s[:, pairs[:, 0], :3] - s[:, pairs[:, 1], :3], axis=-1)
            selfm[n0:n0 + 8] = np.where((ri >= 0) & (rj >= 0), ri + rj - d, -np.inf).max(1) if len(pairs) else -np.inf
    return bound, scene, selfm


def check_against_oracle(got, rm, q, cw, vw, mw, env=None, link_spheres=None):
    b, s, p = margins(rm, q, cw, vw, mw, env, link_spheres)
    want = (b >= 0) & (s <= 0) & (p <= 0)
    near = (np.abs(b) < EPS) | (np.abs(s) < EPS) | (np.abs(p) < EPS)
    got = got.reshape(-1)
    assert near.mean() < 0.01, f"{near.mean():.3%} of rows within {EPS} of a contact"
    bad = np.nonzero((got != want) & ~near)[0]
    assert bad.size == 0, f"{bad.size} rows differ from the oracle, e.g. {bad[:5]}: b {b[bad[:5]]} s {s[bad[:5]]} p {p[bad[:5]]}"
    return want, (b < 0).mean(), (s > 0).mean(), (p > 0).mean()


CASES = [("franka", "cuboid", 512), ("franka", "esdf", 512), ("franka", "mesh", 128), ("g1_29", "esdf", 96), ("g1_43", "esdf", 64)]


@pytest.mark.parametrize("robot,kind,n", CASES)
def test_validate_vs_float64_oracle(robot, kind, n):
    rm = load_robot(robot)
    cw, vw, mw = world(robot, kind)
    ck = checker_of(rm, cw, vw, mw)
    q = draws(rm, robot, n, seed=5)
    got = ck.validate(T(q)).cpu().numpy()
    sync()
    assert int(cblib.load().cb200_last_rollout_variant()) == cblib.VARIANT_VALIDATE
    want, fb, fs, fp = check_against_oracle(got, rm, q, cw, vw, mw)
    print(f"{robot} {kind}: valid {want.mean():.3f} bounds {fb:.3f} scene {fs:.3f} self {fp:.3f}")
    assert 0 < want.sum() < n or robot != "franka"          # Franka draws hold both kinds of rows


def test_validate_two_environments_and_sphere_configurations(n=256):
    """Rows pick their obstacles through env_query_idx and, with two sphere configurations, their spheres: configuration 1 has
    a ball attached to the hand and the first link's spheres disabled."""
    rm = load_robot("franka")
    cw, vw, _ = world("franka", "two_env")
    ls = np.stack([rm.link_spheres, rm.link_spheres]).astype(np.float32)
    att = np.nonzero(rm.link_sphere_idx_map == rm.link_names.index("attached_object"))[0]
    ls[1, att[0]] = [0.0, 0.0, 0.12, 0.08]
    first = np.nonzero(rm.link_sphere_idx_map == rm.link_sphere_idx_map[0])[0]
    ls[1, first, 3] = -100.0
    rm2 = dataclasses.replace(rm, link_spheres=ls)
    ck = checker_of(rm2, cw, vw, None)
    q = draws(rm, "franka", n, seed=9)
    env = (np.arange(n) % 2).astype(np.int32)
    got = ck.validate(T(q), T(env)).cpu().numpy()
    check_against_oracle(got, rm2, q, cw, vw, None, env, ls)


def test_validate_attached_object_and_disabled_link(n=384):
    """Engine-side updates (attach_object_spheres, disable_link_spheres) reach validate."""
    rm = load_robot("franka")
    cw, vw, mw = world("franka", "cuboid")
    ck = checker_of(rm, cw, vw, mw)
    q = draws(rm, "franka", n, seed=13)
    before = ck.validate(T(q)).cpu().numpy().copy()
    ck.engine.attach_object_spheres(T(np.array([[0.0, 0.0, 0.1, 0.1], [0.0, 0.05, 0.15, 0.06]], np.float32)))
    link = rm.link_names[int(rm.link_sphere_idx_map[-10])]
    ck.engine.disable_link_spheres(link)
    ls = ck.engine.link_spheres.cpu().numpy()
    got = ck.validate(T(q)).cpu().numpy()
    check_against_oracle(got, rm, q, cw, vw, mw, None, ls)
    assert not np.array_equal(before, got)


# ------------------------------------------------------------------------------------------------ against the cost kernels
def single_check_masks(rm, robot, kind, n, seed, monkeypatch=None, queue=True):
    cw, vw, mw = world(robot, kind)
    ck = checker_of(rm, cw, vw, mw)
    q = T(draws(rm, robot, n, seed))
    env = T((np.arange(n) % 2).astype(np.int32)) if kind == "two_env" else None
    if monkeypatch is not None:
        monkeypatch.setenv("CB200_QUEUE", "1" if queue else "0")
    out = [ck.validate(q, env).clone()]
    for flags in ((True, False, False), (False, True, False), (False, False, True)):
        out.append(ck.engine.validate(q, env, *flags).clone())
    return ck, q, env, out


@pytest.mark.parametrize("robot,kind,n", CASES + [("franka", "two_env", 256)])
def test_single_checks_equal_cost_kernels(robot, kind, n):
    rm = load_robot(robot)
    ck, q, env, (full, vb, vp, vs) = single_check_masks(rm, robot, kind, n, seed=21)
    eng = RolloutEngine(rm, COST_CFG, DEV, ck.engine.cuboid, ck.engine.voxel, mesh=ck.engine.mesh)
    o = eng.evaluate_cost(q, env_query_idx=env)
    sync()
    assert torch.equal(vb, o.cspace_cost.sum(-1) == 0)
    assert torch.equal(vp, o.self_cost == 0)
    assert torch.equal(vs, o.scene_cost.sum(-1) == 0)
    assert torch.equal(full, vb & vs & vp)
    if n >= 64:                                              # (the emulated runs use a few rows)
        assert int((~vb).sum()) > 0 and int((~vs).sum()) > 0 and int((~vp).sum()) > 0, "a check never fails"


@pytest.mark.parametrize("robot,kind,n", [("franka", "cuboid", 4096), ("g1_29", "esdf", 512), ("franka", "buried", 2048)])
def test_early_exit_changes_nothing(monkeypatch, robot, kind, n):
    """Static striding against the ticket counter, and a world box that buries the robot so nearly every row leaves early."""
    rm = load_robot(robot)
    if kind == "buried":
        cw = CuboidWorld.create([{"dims": [3.0, 3.0, 3.0], "pose": [0.0, 0.0, 0.5, 1, 0, 0, 0]}], max_n=2)
        ck = checker_of(rm, cw, None, None)
        q = T(draws(rm, robot, n, seed=2))
        masks = []
        for queue in ("1", "0"):
            monkeypatch.setenv("CB200_QUEUE", queue)
            masks.append([ck.engine.validate(q, None, *f).clone() for f in
                          ((True, True, True), (True, False, False), (False, True, False), (False, False, True))])
        assert int(masks[0][3].sum()) <= n // 100
        eng = RolloutEngine(rm, COST_CFG, DEV, ck.engine.cuboid)
        o = eng.evaluate_cost(q)
        sync()
        assert torch.equal(masks[0][3], o.scene_cost.sum(-1) == 0) and torch.equal(masks[0][2], o.self_cost == 0)
    else:
        masks = [single_check_masks(rm, robot, kind, n, seed=4, monkeypatch=monkeypatch, queue=qu)[3] for qu in (True, False)]
    for a, b in zip(*masks):
        assert torch.equal(a, b)


def test_graph_capture_and_replay(n=1024):
    rm = load_robot("franka")
    cw, vw, mw = world("franka", "cuboid")
    ck = checker_of(rm, cw, vw, mw)
    q = T(draws(rm, "franka", n, seed=1))
    ck.validate(q)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ck.validate(q)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ck.validate(q)
    q.copy_(T(draws(rm, "franka", n, seed=2)))
    g.replay()
    sync()
    got = out.clone()
    want = ck.validate(q).clone()
    assert torch.equal(got, want) and not torch.equal(want, ck.validate(T(draws(rm, "franka", n, seed=1))))


def test_abi_refusals():
    rm = load_robot("franka")
    eng = RolloutEngine(rm, RolloutConfig(), DEV)
    n = 8
    q = T(draws(rm, "franka", n, seed=0))
    valid = torch.zeros((n, 1), dtype=torch.uint8, device=DEV)
    L = cblib.load()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream if DEV != "cpu" else None)

    def io_of(**kw):
        io = cblib.RolloutIO()
        io.q = q.data_ptr()
        io.robot_blob, io.robot_blob_host = eng._blob.data_ptr(), eng._blob_host.ctypes.data
        io.robot_blob_bytes = int(eng._blob_host.shape[0])
        io.batch_size, io.horizon = n, 1
        for k, v in kw.items():
            setattr(io, k, v)
        return io
    assert L.cb200_rollout_validate(C.byref(io_of()), valid.data_ptr(), 1, 1, 1, stream) == 0
    sync()
    assert L.cb200_last_rollout_variant() == cblib.VARIANT_VALIDATE
    assert L.cb200_rollout_validate(C.byref(io_of()), None, 1, 1, 1, stream) == INVALID
    assert L.cb200_rollout_validate(None, valid.data_ptr(), 1, 1, 1, stream) == INVALID
    assert L.cb200_rollout_validate(C.byref(io_of(q=None)), valid.data_ptr(), 1, 1, 1, stream) == INVALID
    assert L.cb200_rollout_validate(C.byref(io_of(robot_blob=None)), valid.data_ptr(), 1, 1, 1, stream) == INVALID
    assert L.cb200_rollout_validate(C.byref(io_of(spline=C.pointer(cblib.SplineInput()))), valid.data_ptr(), 1, 1, 1, stream) == INVALID
    dp = cblib.DynamicsParams()
    assert L.cb200_rollout_validate(C.byref(io_of(dynamics=C.pointer(dp))), valid.data_ptr(), 1, 1, 1, stream) == INVALID
    assert L.cb200_rollout_validate(C.byref(io_of(current_position=q.data_ptr())), valid.data_ptr(), 1, 1, 1, stream) == INVALID
    # cost and gradient fields are ignored
    assert L.cb200_rollout_validate(C.byref(io_of(cost=None, grad_q=None)), valid.data_ptr(), 1, 1, 1, stream) == 0


# ------------------------------------------------------------------------------------------------ checker API
def test_distance_methods_equal_composition_and_oracle(n=64):
    from curobo_b200.kinematics import Kinematics
    from curobo_b200.scene import CollisionBuffer, SceneData, SphereObstacleCollision
    rm = load_robot("franka")
    cw, vw, _ = world("franka", "cuboid")
    ck = checker_of(rm, cw, vw, None)
    q = draws(rm, "franka", n, seed=3)
    d_scene, d_self = ck.get_scene_self_collision_distance_from_joints(T(q))
    st = Kinematics(rm, DEV).compute_kinematics(T(q))
    buf = CollisionBuffer.from_shape(tuple(st.robot_spheres.shape), DEV)
    want_scene = SphereObstacleCollision.apply(st.robot_spheres, buf, SceneData(ck.engine.cuboid), T(np.array([1.0], np.float32)),
                                               T(np.array([0.2], np.float32)), None, None, False)
    assert torch.equal(d_scene, want_scene)
    cost, _ = O.scene_collision(O.fk_forward(rm, q[:, 0])[1][:, None], 1.0, 0.2, cw)
    np.testing.assert_allclose(d_scene.cpu().numpy(), cost, rtol=1e-4, atol=1e-5)
    scost, _, _ = O.self_collision(O.fk_forward(rm, q[:, 0])[1], rm.sphere_padding, rm.collision_pairs, 1.0)
    np.testing.assert_allclose(d_self.cpu().numpy()[:, 0, 0], scost, rtol=1e-4, atol=1e-6)
    assert (cost > 0).any() and (scost > 0).any()
    b = ck.get_bound(T(q))
    bc, _ = O.cspace_position_cost(q, rm.position_limits, [1.0, 0.0], [0.0, 0.0])
    np.testing.assert_allclose(b.cpu().numpy(), bc, rtol=1e-5, atol=1e-9)
    assert (bc > 0).any()
    # gradients: self and bound apply the upstream gradient, scene does not (the reference's use_grad_input)
    x = T(q).requires_grad_(True)
    (2.0 * ck.get_bound(x)).sum().backward()
    _, gb = O.cspace_position_cost(q, rm.position_limits, [1.0, 0.0], [0.0, 0.0])
    np.testing.assert_allclose(x.grad.cpu().numpy(), 2.0 * gb, rtol=1e-5, atol=1e-7)
    x.grad = None
    ds, dp = ck.get_scene_self_collision_distance_from_joints(x)
    (ds.sum() + dp.sum()).backward()
    assert torch.isfinite(x.grad).all() and float(x.grad.abs().sum()) > 0


def test_sample_and_sample_trajectory():
    rm = load_robot("franka")
    cw, _, _ = world("franka", "cuboid")
    ck = checker_of(rm, cw, None, None)
    g = torch.Generator(device=DEV).manual_seed(7)
    s = ck.sample(200, generator=g)
    assert 0 < s.shape[0] <= 200 and s.shape[1] == rm.num_dof
    assert bool(ck.validate(s[:, None]).all())
    lo, hi = T(rm.position_limits[0]), T(rm.position_limits[1])
    assert bool(((s >= lo) & (s <= hi)).all())
    s2 = ck.sample(200, generator=torch.Generator(device=DEV).manual_seed(7))
    assert torch.equal(s, s2)
    # draw order: the first valid draws of the same generator stream
    q = lo + (hi - lo) * torch.rand((2000, rm.num_dof), generator=torch.Generator(device=DEV).manual_seed(7), device=DEV)
    v = ck.validate(q[:, None])[:, 0]
    assert torch.equal(s, q[v][:200])
    assert ck.sample(30, mask_valid=False, generator=g).shape == (30, rm.num_dof)
    tr = ck.sample_trajectory(4, 10, generator=g)
    assert tr.shape == (4, 10, rm.num_dof) and bool(ck.validate_trajectory(tr.contiguous()).all())
    # a box over the whole workspace: fewer than n samples, and sample_trajectory raises
    box = checker_of(rm, CuboidWorld.create([{"dims": [3.0, 3.0, 3.0], "pose": [0.0, 0.0, 0.5, 1, 0, 0, 0]}], max_n=2), None, None)
    assert box.sample(50, generator=g).shape[0] < 50
    with pytest.raises(ValueError):
        box.sample_trajectory(2, 5, generator=g)
