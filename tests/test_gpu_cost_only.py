"""Cost-only fused rollout (RolloutEngine.evaluate_cost -> cb200_rollout_cost): the rollout a particle optimizer (MPPI) evaluates.

Pins, on every kernel variant (forced with CB200_BIG / CB200_ARM_PAIRS / CB200_TEAM and checked through
cb200_last_rollout_variant()), for Franka, G1-29 and G1-43 in cuboid, ESDF and mesh worlds, with goalsets and the c-space target:
(1) `cost`, every term cost and the FK outputs equal the gradient launch's -- bit for bit, accepted at 2e-6 relative where the
compiler contracts an FMA differently; (2) the gradient outputs are not written (a NaN-filled grad_q stays NaN); (3) the variant
is the gradient launch's with CB200_VARIANT_COST_ONLY set, and the big kernel where the gradient launch takes the team kernel;
(4) robots whose pair list is not a union of link blocks (no link-pair list in the blob: the pair scan reads the padded
sphere copy the cost-only row keeps for them); (5) multi-environment rows; (6) `with_terms=False` writes the cost only;
(7) CUDA-graph replay; (8) refusals; (9) the B200RobotRollout routing: calls that cannot be differentiated take the
cost-only kernels and return the same terms."""
import ctypes as C
import dataclasses
import struct

import numpy as np
import pytest
import torch

from helpers import small_voxel_world
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

VARIANT_ENV = {"arm": {"CB200_BIG": "0", "CB200_ARM_PAIRS": "0"}, "pairs": {"CB200_BIG": "0", "CB200_ARM_PAIRS": "1"},
               "standard": {"CB200_BIG": "0"}, "big": {"CB200_BIG": "1", "CB200_TEAM": "0"},
               "team": {"CB200_BIG": "1", "CB200_TEAM": "2"}}
# include/curobo_b200.h: CB200_VARIANT_STANDARD 1, ARM 2, BIG 4, TEAM2 5
GRAD_VARIANT = {"arm": 2, "pairs": 2, "standard": 1, "big": 4, "team": 5}
COST_VARIANT = {"arm": 2, "pairs": 2, "standard": 1, "big": 4, "team": 4}
TERMS = ("cost", "self_cost", "scene_cost", "pose_cost", "cspace_cost", "link_pos", "link_quat", "robot_spheres",
         "pose_goalset_idx")


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def last_variant():
    return int(cblib.load().cb200_last_rollout_variant())


def sync():
    if DEV != "cpu":
        torch.cuda.synchronize()


def world(robot, kind):
    """(CuboidData, VoxelData, MeshData): "cuboid", "esdf", "mesh" or "all" (cuboids + ESDF + meshes)."""
    cub = vox = mesh = None
    if kind in ("cuboid", "all"):
        cub = CuboidData.from_world(CuboidWorld.create([TABLE, PILLAR], max_n=3), DEV)
    if kind in ("esdf", "all"):
        vox = VoxelData.from_world(small_voxel_world(), DEV)
    if kind in ("mesh", "all"):
        mesh = MeshData.from_world(mesh_world(robot), DEV)
    return cub, vox, mesh


def engine(rm, robot, kind, n, seed=3):
    """IK cost (self, scene, pose with a goalset of 2, c-space bound + target) on the given world."""
    cfg = RolloutConfig.ik()
    cfg.scene_activation = 0.02
    cfg.cspace_target_weight = 100.0
    cub, vox, mesh = world(robot, kind)
    eng = RolloutEngine(rm, cfg, DEV, cub, vox, store_fk_outputs=True, mesh=mesh)
    G = 4
    _, _, gp, gq = O.fk_forward(rm, rows(rm, robot, 2 * G, seed=seed + 1)[:, 0])
    Lt = rm.num_tool_frames
    gp = np.ascontiguousarray(gp.reshape(2, G, Lt, 3).transpose(1, 2, 0, 3))       # [G, L, 2, 3]
    gq = np.ascontiguousarray(gq.reshape(2, G, Lt, 4).transpose(1, 2, 0, 3))
    eng.update_goal(T(gp), T(gq), T((np.arange(n) % G).astype(np.int32)))
    target = rows(rm, robot, 2, seed=seed + 2)[:, 0]
    eng.update_cspace_target(T(target), T((np.arange(n) % 2).astype(np.int32)))
    return eng


def snapshot(o):
    return {k: getattr(o, k).clone() for k in TERMS}


def poison(o):
    for k in TERMS:
        t = getattr(o, k)
        t.fill_(-1 if k == "pose_goalset_idx" else float("nan"))
    o.grad_q.fill_(float("nan"))


def assert_same(got, want, name):
    """Bit for bit, or within 2e-6 relative (an FMA contracted differently); returns whether it was bit for bit."""
    if torch.equal(got, want):
        return True
    if not got.is_floating_point():
        raise AssertionError(f"{name}: integer output differs")
    torch.testing.assert_close(got, want, rtol=2e-6, atol=2e-6 * float(want.abs().max()), msg=name)
    return False


def robot_of(name):
    """"<robot>" or "<robot>-pairlist": the stock robot without its first collision pair, so the pair list is no longer a union
    of link x link blocks and the blob carries no link-pair list (the self-collision scan walks the pair list)."""
    robot, _, tag = name.partition("-")
    rm = load_robot(robot)
    if tag == "pairlist":
        rm = dataclasses.replace(rm, collision_pairs=np.ascontiguousarray(rm.collision_pairs[1:]))
        assert struct.unpack("<48i", pack_robot_blob(rm)[:192].tobytes())[28] == 0   # n_lp
    return robot, rm


CASES = [("franka", "arm", "cuboid", 300), ("franka", "pairs", "cuboid", 301), ("franka", "arm", "esdf", 200),
         ("franka", "standard", "mesh", 200), ("franka", "big", "esdf", 150), ("franka", "big", "mesh", 150),
         ("franka", "team", "esdf", 40), ("g1_29", "standard", "cuboid", 64), ("g1_29", "big", "esdf", 100),
         ("g1_29", "team", "esdf", 40), ("g1_43", "big", "all", 64), ("g1_43", "team", "cuboid", 30),
         ("franka-pairlist", "arm", "cuboid", 300), ("franka-pairlist", "pairs", "cuboid", 301),
         ("franka-pairlist", "standard", "mesh", 200), ("g1_29-pairlist", "standard", "cuboid", 64)]


@pytest.mark.parametrize("robot,variant,kind,n", CASES)
def test_cost_only_equals_gradient_launch(monkeypatch, robot, variant, kind, n):
    robot, rm = robot_of(robot)
    for k, v in VARIANT_ENV[variant].items():
        monkeypatch.setenv(k, v)
    eng = engine(rm, robot, kind, n)
    q = T(rows(rm, robot, n, seed=11))
    eng.evaluate_action(q)
    sync()
    assert last_variant() == GRAD_VARIANT[variant]
    if variant == "team":          # the team kernel reduces a row in another order: compare with the big kernel it twins
        monkeypatch.setenv("CB200_TEAM", "0")
        eng.evaluate_action(q)
        monkeypatch.setenv("CB200_TEAM", "2")
    want = snapshot(eng.out)
    poison(eng.out)
    o = eng.evaluate_cost(q)
    sync()
    assert last_variant() == COST_VARIANT[variant] | cblib.VARIANT_COST_ONLY
    assert torch.isnan(o.grad_q).all(), "the cost-only launch wrote grad_q"
    assert int((want["scene_cost"] > 0).sum()) > 2 and int((want["self_cost"] > 0).sum()) > 0, "collision terms inactive"
    bitwise = {k: assert_same(getattr(o, k), want[k], k) for k in TERMS}
    print(f"{robot} {variant} {kind}: not bit for bit: {[k for k, b in bitwise.items() if not b]}")


@pytest.mark.parametrize("variant", ["arm", "big"])
def test_cost_only_multi_env_and_cost_without_terms(monkeypatch, variant):
    """Rows pick their world through env_query_idx; with_terms=False writes `cost` and nothing else."""
    from test_gpu_rollout import _two_env_worlds
    rm = load_robot("franka")
    for k, v in VARIANT_ENV[variant].items():
        monkeypatch.setenv(k, v)
    cub, vox = _two_env_worlds()
    cfg = RolloutConfig(self_weight=5000.0, scene_weight=5000.0, scene_activation=0.02, cspace_type="position",
                        cspace_weight=(5000.0, 0, 0, 0, 0), cspace_activation=(0.01, 0, 0, 0, 0))
    eng = RolloutEngine(rm, cfg, DEV, CuboidData.from_world(cub, DEV), VoxelData.from_world(vox, DEV))
    B = 64
    q, env = T(rows(rm, "franka", B, seed=77)), T((np.arange(B) % 2).astype(np.int32))
    og = eng.evaluate_action(q, env_query_idx=env)
    cost, scene = og.cost.clone(), og.scene_cost.clone()
    assert scene[0::2].sum() > 0 and scene[1::2].sum() > 0
    og.cost.fill_(float("nan"))
    og.scene_cost.fill_(-7.0)
    o = eng.evaluate_cost(q, env_query_idx=env)
    sync()
    assert_same(o.scene_cost, scene, "scene_cost")
    assert_same(o.cost, cost, "cost")
    o.scene_cost.fill_(-7.0)
    o.cost.fill_(float("nan"))
    eng.evaluate_cost(q, env_query_idx=env, with_terms=False)
    sync()
    assert_same(o.cost, cost, "cost")
    assert (o.scene_cost == -7.0).all()


def test_cost_only_graph_replay():
    rm = load_robot("franka")
    n = 512
    eng = engine(rm, "franka", "cuboid", n)
    q = T(rows(rm, "franka", n, seed=5))
    want = eng.evaluate_cost(q, with_terms=False).cost.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.evaluate_cost(q, with_terms=False)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eng.evaluate_cost(q, with_terms=False)
    q.copy_(T(rows(rm, "franka", n, seed=6)))
    g.replay()
    sync()
    other = eng.evaluate_cost(q, with_terms=False).cost.clone()
    assert not torch.equal(other, want)
    eng.out.cost.zero_()
    g.replay()
    sync()
    assert torch.equal(eng.out.cost, other)


def test_cost_only_refusals():
    """cb200_rollout_cost refuses what it does not cover (swept rows, the spline front end, fused dynamics) and null inputs;
    cb200_rollout_cost_grad keeps refusing a null grad_q."""
    rm = load_robot("franka")
    eng = RolloutEngine(rm, RolloutConfig(self_weight=1.0), DEV)
    n = 8
    q = T(rows(rm, "franka", n))
    eng.setup_batch_tensors(n, 1)
    L = cblib.load()

    def io_of(**kw):
        io = cblib.RolloutIO()
        io.q, io.cost = q.data_ptr(), eng.out.cost.data_ptr()
        io.robot_blob, io.robot_blob_host = eng._blob.data_ptr(), eng._blob_host.ctypes.data
        io.robot_blob_bytes = int(eng._blob_host.shape[0])
        io.batch_size, io.horizon = n, 1
        for k, v in kw.items():
            setattr(io, k, v)
        return io
    cfg = eng._ccfg
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream if DEV != "cpu" else None)
    assert L.cb200_rollout_cost(C.byref(cfg), C.byref(io_of()), stream) == 0
    assert L.cb200_rollout_cost(C.byref(cfg), C.byref(io_of(q=None)), stream) == INVALID
    assert L.cb200_rollout_cost(C.byref(cfg), C.byref(io_of(cost=None)), stream) == INVALID
    assert L.cb200_rollout_cost(C.byref(cfg), C.byref(io_of(robot_blob=None)), stream) == INVALID
    sp = cblib.SplineInput()
    assert L.cb200_rollout_cost(C.byref(cfg), C.byref(io_of(spline=C.pointer(sp))), stream) == INVALID
    dp = cblib.DynamicsParams()
    assert L.cb200_rollout_cost(C.byref(cfg), C.byref(io_of(dynamics=C.pointer(dp))), stream) == INVALID
    swept = eng._make_ccfg(1)
    swept.use_sweep = 1
    assert L.cb200_rollout_cost(C.byref(swept), C.byref(io_of()), stream) == INVALID
    assert L.cb200_rollout_cost_grad(C.byref(cfg), C.byref(io_of()), stream) == INVALID    # grad_q is null
    assert L.cb200_rollout_cost(None, None, stream) == INVALID
    with pytest.raises(ValueError):
        RolloutEngine(rm, RolloutConfig(self_weight=1.0, use_sweep=True), DEV).evaluate_cost(T(rows(rm, "franka", 2, H=4)))


def test_robot_rollout_takes_cost_only_without_grad():
    """B200RobotRollout: evaluate_action under no_grad (or on an act_seq without requires_grad) and compute_metrics_from_action
    run the cost-only kernels -- same term values and buffers as the differentiable call, grad_q untouched."""
    from curobo_b200.rollout_protocol import B200RobotRollout
    rm = load_robot("franka")
    n = 96
    cub = CuboidData.from_world(CuboidWorld.create([TABLE, PILLAR], max_n=3), DEV)
    ro = B200RobotRollout(rm, RolloutConfig.ik(), DEV, cuboid=cub, horizon=1)
    _, _, gp, gq = O.fk_forward(rm, rows(rm, "franka", 4, seed=2)[:, 0])
    ro.update_params(goal_position=T(gp[:, :, None, :].copy()), goal_quat=T(gq[:, :, None, :].copy()),
                     idxs_goal=T((np.arange(n) % 4).astype(np.int32)))
    q = T(rows(rm, "franka", n, seed=9))
    x = q.clone().requires_grad_(True)
    res = ro.evaluate_action(x)
    assert last_variant() & cblib.VARIANT_COST_ONLY == 0
    want = [t.clone() for t in res.costs_and_constraints.costs.values + res.costs_and_constraints.constraints.values]
    ro.engine.out.grad_q.fill_(float("nan"))
    with torch.no_grad():
        r2 = ro.evaluate_action(x)
    assert last_variant() & cblib.VARIANT_COST_ONLY
    got = r2.costs_and_constraints.costs.values + r2.costs_and_constraints.constraints.values
    for a, b in zip(got, want):
        assert a.shape == b.shape
        assert_same(a, b, "term")
    assert got[0].data_ptr() == ro.engine.out.pose_cost.data_ptr()
    ro.evaluate_action(q)                                     # q does not require grad
    assert last_variant() & cblib.VARIANT_COST_ONLY
    m = ro.compute_metrics_from_action(q)
    assert last_variant() & cblib.VARIANT_COST_ONLY and m.feasible.shape == (n,)
    assert torch.isnan(ro.engine.out.grad_q).all()
