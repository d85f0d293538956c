"""Velocity-aware IK in the fused rollout: the current-state block of the POSITION c-space cost (RolloutEngine.update_current_state
-> cb200_rollout_io.current_position / current_velocity / idxs_current_state / current_state_dt; cost/wp_cspace_position.py:299-356).

Pins:
(1) the per-operator cb200_cspace_position_cost and the fused kernels (every family, gradient and cost-only) against the output of
    the reference's own forward_cspace_position_warp (tests/golden/cspace_position_current_state_golden.npz);
(2) fused equals composed on every kernel variant with self, scene and pose terms active: the self / scene / pose outputs are
    bit-identical to the launch without a current state, and the c-space term and its gradient are those of the per-operator
    kernel; both agree with the oracle (oracle/current_state_oracle.py);
(3) rows without a current state (NULL fields, or dt = 0) are bit-identical to the launch without one;
(4) empty windows, velocity absent, several current-state rows, multi-environment rows;
(5) CUDA-graph replay with the current state rewritten in place;
(6) the step-limiting property of L-BFGS with the retargeting weights."""
import os

import numpy as np
import pytest
import torch

from test_gpu_cost_only import COST_VARIANT, GRAD_VARIANT, VARIANT_ENV, assert_same, last_variant
from test_gpu_fused_mesh import PILLAR, TABLE, rows
from helpers import small_voxel_world
from curobo_b200 import cost as cb_cost
from curobo_b200 import lib as cblib
from curobo_b200.robot_model import load_robot
from curobo_b200.rollout import RolloutConfig, RolloutEngine
from curobo_b200.scene import CuboidData, VoxelData
from curobo_b200.world import CuboidWorld
from oracle import current_state_oracle as CS
from oracle import rollout_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cspace_position_current_state_golden.npz")
GOLDEN_CASES = ("vel_acc", "no_velocity", "mixed_dt", "empty_window", "with_target")
VARIANT_ENV = dict(VARIANT_ENV, traj={"CB200_BIG": "0"})
GRAD_VARIANT = dict(GRAD_VARIANT, traj=7)
TERMS = ("self_cost", "scene_cost", "pose_cost", "link_pos", "link_quat", "robot_spheres")


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def sync():
    if DEV != "cpu":
        torch.cuda.synchronize()


def golden(name):
    G = np.load(GOLDEN)
    pre = name + "/"
    return {k[len(pre):]: G[k] for k in G.files if k.startswith(pre)}


def close(got, want, name, rtol=1e-4, atol_rel=1e-6):
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    want = np.asarray(want)
    atol = atol_rel * max(float(np.abs(want).max()), 1e-6)
    err = np.abs(got - want)
    assert np.all(err <= atol + rtol * np.abs(want)), f"{name}: max err {float(err.max()):.3g} (atol {atol:.3g})"


# ------------------------------------------------------------------------------------------------ per-operator kernel
def per_operator(q, lim_p, lim_v, weight, act, reg, cur_p, cur_v, idxs_cur, dt, target=None, idxs_target=None, target_weight=0.0,
                 dof_weight=None):
    """cb200_cspace_position_cost (the composed path's c-space operator); returns cost, grad_p [B,H,D]."""
    B, H, D = q.shape
    oc, gp, gt = (torch.zeros((B, H, D), device=DEV) for _ in range(3))
    f = lambda x: T(np.asarray(x, np.float32))  # noqa: E731
    cb_cost.cspace_position_cost(f(q), torch.zeros((B, H, D), device=DEV), f(np.zeros((1, D)) if target is None else target),
                                 T(np.zeros(B, np.int32) if idxs_target is None else np.asarray(idxs_target, np.int32)), f(lim_p),
                                 f(np.ones((2, D))), f(weight), f(act), f([target_weight]), f(np.ones(D) if dof_weight is None else dof_weight),
                                 f(reg), f(cur_p), f(np.zeros_like(cur_p) if cur_v is None else cur_v), T(np.asarray(idxs_cur, np.int32)),
                                 f(lim_v), f(dt), oc, gp, gt)
    sync()
    return oc, gp


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_per_operator_kernel_matches_reference_source(case):
    c = golden(case)
    oc, gp = per_operator(c["q"], c["lim_p"], c["lim_v"], c["weight"], c["act"], c["reg"], c["cur_p"], c["cur_v"], c["idxs_cur"],
                          c["dt"], c["target"], c["idxs_target"], float(c["target_weight"][0]), c["dof_weight"])
    close(oc, c["cost"], "cost")
    close(gp, c["grad_p"], "grad_p")


def golden_engine(c, use_sweep=False):
    """Franka, POSITION c-space cost only, with the fixture's weights and current state."""
    rm = load_robot("franka")
    cfg = RolloutConfig(cspace_type="position", cspace_weight=(float(c["weight"][0]), 0, 0, 0, 0),
                        cspace_activation=(float(c["act"][0]), 0, 0, 0, 0), cspace_reg=(float(c["reg"][0]), float(c["reg"][1]), 0, 0, 0),
                        cspace_target_weight=float(c["target_weight"][0]), use_sweep=use_sweep)
    eng = RolloutEngine(rm, cfg, DEV)
    if cfg.cspace_target_weight > 0:
        eng.update_cspace_target(T(c["target"]), T(c["idxs_target"]), T(c["dof_weight"]))
    eng.update_current_state(T(c["cur_p"]), T(c["cur_v"]) if int(c["has_velocity"]) else None, T(c["dt"]), T(c["idxs_cur"]))
    return eng


@pytest.mark.parametrize("variant", ["arm", "pairs", "big", "traj", "cost_arm", "cost_big"])
@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_fused_kernels_match_reference_source(monkeypatch, case, variant):
    c = golden(case)
    rm = load_robot("franka")
    assert np.array_equal(np.asarray(rm.velocity_limits, np.float32), c["lim_v"]) and np.array_equal(
        np.asarray(rm.position_limits, np.float32), c["lim_p"])
    base = variant.replace("cost_", "")
    for k, v in VARIANT_ENV[base].items():
        monkeypatch.setenv(k, v)
    eng = golden_engine(c, use_sweep=base == "traj")
    q = T(c["q"])
    o = eng.evaluate_cost(q) if variant.startswith("cost_") else eng.evaluate_action(q)
    sync()
    want = {"arm": 2, "pairs": 2, "big": 4, "traj": 7}[base] | (cblib.VARIANT_COST_ONLY if variant.startswith("cost_") else 0)
    assert last_variant() == want, (last_variant(), want)
    close(o.cspace_cost, c["cost"], "cspace_cost")
    close(o.cost, c["cost"].sum(-1), "cost", atol_rel=2e-6)
    if not variant.startswith("cost_"):
        close(o.grad_q, c["grad_p"], "grad_q")


# ------------------------------------------------------------------------------------------------ fused equals composed
def worlds(kind, two_env=False):
    """(CuboidData, VoxelData, CuboidWorld, VoxelWorld) for "cuboid" / "esdf"."""
    if two_env:
        from test_gpu_rollout import _two_env_worlds
        cw, vw = _two_env_worlds()
        return CuboidData.from_world(cw, DEV), VoxelData.from_world(vw, DEV), cw, vw
    cw = CuboidWorld.create([TABLE, PILLAR], max_n=3) if kind == "cuboid" else None
    vw = small_voxel_world() if kind == "esdf" else None
    return (CuboidData.from_world(cw, DEV) if cw is not None else None, VoxelData.from_world(vw, DEV) if vw is not None else None,
            cw, vw)


def current_state(rm, robot, q, n_cur, dts, seed, velocity=True, outside=False):
    """n_cur current-state rows, one per seed through idxs; even seeds start within a step or two of their current state."""
    rng = np.random.default_rng(seed)
    B, H, D = q.shape
    idx = (np.arange(B) % n_cur).astype(np.int32)
    cur_p = rows(rm, robot, n_cur, seed=seed)[:, 0].astype(np.float32)
    lim_p, lim_v = np.asarray(rm.position_limits, np.float32), np.asarray(rm.velocity_limits, np.float32)
    if outside:
        cur_p[:, 0] = lim_p[1, 0] + 0.4
        cur_p[:, 1] = lim_p[0, 1] - 0.4
    cur_v = rng.normal(0, 0.4, size=(n_cur, D)).astype(np.float32) if velocity else None
    q = q.copy()
    step = rng.normal(0, 1.0, size=(B, H, D)).astype(np.float32) * lim_v[1] * np.float32(0.05)
    q[0::2] = np.clip(cur_p[idx[0::2]][:, None, :] + step[0::2], lim_p[0] - 0.05, lim_p[1] + 0.05)
    return q, cur_p, cur_v, idx, np.asarray(dts, np.float32)


def pose_goal(rm, robot, n, seed):
    G = 4
    _, _, gp, gq = O.fk_forward(rm, rows(rm, robot, G, seed=seed)[:, 0])
    return gp[:, :, None, :].copy(), gq[:, :, None, :].copy(), (np.arange(n) % G).astype(np.int32)


FC_CASES = [("franka", "arm", "cuboid", 300, 1), ("franka", "pairs", "cuboid", 301, 1), ("franka", "arm", "esdf", 200, 1),
            ("g1_29", "standard", "cuboid", 64, 1),
            ("g1_29", "big", "esdf", 100, 1), ("g1_43", "team", "cuboid", 30, 1), ("franka", "traj", "cuboid", 24, 4)]


def composed_case(monkeypatch, robot, variant, kind, n, H, seed=17, n_cur=3, dts=(0.05, 0.0, 0.08), velocity=True, outside=False,
                  two_env=False):
    rm = load_robot(robot)
    for k, v in VARIANT_ENV[variant].items():
        monkeypatch.setenv(k, v)
    cfg = RolloutConfig.retarget_ik()
    cfg.scene_activation = 0.02
    cfg.cspace_reg = (0.5, 0.05, 0, 0, 0)
    cfg.use_sweep = variant == "traj"
    cub, vox, cw, vw = worlds(kind, two_env)
    eng = RolloutEngine(rm, cfg, DEV, cub, vox, store_fk_outputs=True)
    gp, gq, ig = pose_goal(rm, robot, n, seed + 1)
    eng.update_goal(T(gp), T(gq), T(ig))
    q, cur_p, cur_v, idx, dt = current_state(rm, robot, rows(rm, robot, n, H=H, seed=seed), n_cur, dts, seed + 2, velocity, outside)
    env = T((np.arange(n) % 2).astype(np.int32)) if two_env else None
    return rm, cfg, eng, q, (cur_p, cur_v, idx, dt), (gp, gq, ig), (cw, vw), env


def check_composed(rm, cfg, eng, q, cs, goal, world, env, variant, cost_only=False):
    cur_p, cur_v, idx, dt = cs
    qt = T(q)
    B = q.shape[0]
    eng.clear_current_state()
    plain = eng.evaluate_action(qt, env_query_idx=env)
    sync()
    want_variant = GRAD_VARIANT[variant]
    assert last_variant() == want_variant
    base = {k: getattr(plain, k).clone() for k in TERMS + ("cost", "cspace_cost", "grad_q")}
    eng.update_current_state(T(cur_p), T(cur_v) if cur_v is not None else None, T(dt), T(idx))
    o = eng.evaluate_action(qt, env_query_idx=env)
    sync()
    assert last_variant() == want_variant
    assert int((base["scene_cost"] > 0).sum()) > 2 and int((base["self_cost"] > 0).sum()) > 0, "collision terms inactive"
    for k in TERMS:                                   # FK, self, scene and pose do not see the current state
        assert torch.equal(getattr(o, k), base[k]), k
    # the c-space term and its gradient are the per-operator kernel's
    lim_p, lim_v = np.asarray(rm.position_limits, np.float32), np.asarray(rm.velocity_limits, np.float32)
    args = (lim_p, lim_v, [cfg.cspace_weight[0], 0.0], [cfg.cspace_activation[0], 0.0], list(cfg.cspace_reg[:2]))
    pc, pg = per_operator(q, *args, cur_p, cur_v, idx, dt)
    pc0, pg0 = per_operator(q, *args, cur_p, cur_v, idx, np.zeros_like(dt))
    close(o.cspace_cost, pc.cpu().numpy(), "cspace_cost vs per-operator", rtol=2e-6, atol_rel=1e-7)
    close(base["cspace_cost"], pc0.cpu().numpy(), "plain cspace_cost vs per-operator", rtol=2e-6, atol_rel=1e-7)
    dg = (pg - pg0).cpu().numpy()
    close((o.grad_q - base["grad_q"]).cpu().numpy(), dg, "grad_q - plain grad_q vs per-operator", rtol=1e-5,
          atol_rel=1e-6 * float(np.abs(base["grad_q"].cpu().numpy()).max()) / max(float(np.abs(dg).max()), 1e-9))
    close((o.cost - base["cost"]).cpu().numpy(), (pc - pc0).sum(-1).cpu().numpy(), "cost - plain cost", rtol=1e-5,
          atol_rel=1e-6 * float(base["cost"].abs().max()) / max(float((pc - pc0).sum(-1).abs().max()), 1e-9))
    # rows whose current state has dt = 0 take the plain arithmetic, bit for bit
    off = np.asarray(dt)[idx] <= 0
    if off.any():
        sel = torch.as_tensor(np.nonzero(off)[0], device=o.cost.device)
        for k in ("cost", "cspace_cost", "grad_q"):
            assert torch.equal(getattr(o, k)[sel], base[k][sel]), f"dt = 0 rows differ in {k}"
    assert (np.asarray(dt)[idx] > 0).any() and not torch.equal(o.cspace_cost, base["cspace_cost"])
    # both against the oracle
    gp, gq, ig = goal
    w = CS.rollout_cost_grad(rm, q, cfg.to_oracle_cfg(1), current_position=cur_p, current_velocity=cur_v, idxs_current=idx,
                             state_dt=dt, world_cuboid=world[0], world_voxel=world[1], goal_pos=gp, goal_quat=gq, idxs_goal=ig,
                             env_query_idx=None if env is None else env.cpu().numpy(), dt=np.full(B, 0.05, np.float32))
    np.testing.assert_allclose(o.cost.cpu().numpy(), w["cost_bh"], rtol=2e-4, atol=1e-5 * float(np.abs(w["cost_bh"]).max()))
    np.testing.assert_allclose(o.cspace_cost.cpu().numpy(), w["cspace_cost"], rtol=2e-4,
                               atol=1e-5 * float(np.abs(w["cspace_cost"]).max()))
    g = w["grad_q"]
    np.testing.assert_allclose(o.grad_q.cpu().numpy(), g, rtol=2e-3, atol=2e-5 * float(np.abs(g).max()))
    if cost_only:
        want = {k: getattr(o, k).clone() for k in ("cost", "cspace_cost", "self_cost", "scene_cost", "pose_cost")}
        o.grad_q.fill_(float("nan"))
        oc = eng.evaluate_cost(qt, env_query_idx=env)
        sync()
        assert last_variant() == COST_VARIANT[variant] | cblib.VARIANT_COST_ONLY
        for k, v in want.items():
            assert_same(getattr(oc, k), v, k)
        assert torch.isnan(oc.grad_q).all()


@pytest.mark.parametrize("robot,variant,kind,n,H", FC_CASES)
def test_fused_equals_composed(monkeypatch, robot, variant, kind, n, H):
    """The cost-only twins are checked against the gradient launch of the same family: not for the team kernel, which reduces a
    row in another order than the big kernel its cost-only launch takes, nor for trajectory rows, which have no cost-only twin."""
    r = composed_case(monkeypatch, robot, variant, kind, n, H)
    check_composed(*r, variant, cost_only=variant not in ("traj", "team"))


@pytest.mark.parametrize("edge", ["empty_window", "no_velocity", "many_rows", "multi_env"])
def test_edge_cases(monkeypatch, edge):
    kw = dict(empty_window=dict(outside=True), no_velocity=dict(velocity=False),
              many_rows=dict(n_cur=7, dts=(0.05, 0.02, 0.0, 0.1, 0.05, 0.0, 0.07)), multi_env=dict(two_env=True))[edge]
    r = composed_case(monkeypatch, "franka", "arm", "cuboid", 64, 1, seed=31, **kw)
    check_composed(*r, "arm", cost_only=True)


def test_null_fields_and_refusal():
    """Without a current state the POSITION rows equal the oracle without the block; current_position without current_state_dt is
    refused by both C entry points, while the same call without current_position succeeds."""
    import ctypes as C
    rm = load_robot("franka")
    cfg = RolloutConfig.retarget_ik()
    eng = RolloutEngine(rm, cfg, DEV)
    n = 16
    q_np = rows(rm, "franka", n, seed=3)
    q_np[::3, 0, 0] = rm.position_limits[1][0] + 0.1                      # some rows beyond the limits: the hinge is live
    q = T(q_np)
    out = eng.evaluate_action(q)
    sync()
    w = O.rollout_cost_grad(rm, q_np, cfg.to_oracle_cfg(1))
    np.testing.assert_allclose(out.cspace_cost.cpu().numpy(), w["cspace_cost"], rtol=2e-5, atol=1e-6 * float(np.abs(w["cspace_cost"]).max()))
    np.testing.assert_allclose(out.grad_q.cpu().numpy(), w["grad_q"], rtol=2e-3, atol=2e-5 * float(np.abs(w["grad_q"]).max()))
    assert float(np.abs(w["cspace_cost"]).max()) > 0
    cur = T(rows(rm, "franka", 1, seed=4)[:, 0])
    io = cblib.RolloutIO()
    io.q, io.cost, io.grad_q = q.data_ptr(), eng.out.cost.data_ptr(), eng.out.grad_q.data_ptr()
    io.robot_blob, io.robot_blob_host = eng._blob.data_ptr(), eng._blob_host.ctypes.data
    io.robot_blob_bytes = int(eng._blob_host.shape[0])
    io.batch_size, io.horizon = n, 1
    L = cblib.load()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream if DEV != "cpu" else None)
    assert L.cb200_rollout_cost_grad(C.byref(eng._ccfg), C.byref(io), stream) == 0      # control: the same call, no current state
    assert L.cb200_rollout_cost(C.byref(eng._ccfg), C.byref(io), stream) == 0
    io.current_position = cur.data_ptr()
    assert L.cb200_rollout_cost_grad(C.byref(eng._ccfg), C.byref(io), stream) == 1
    assert L.cb200_rollout_cost(C.byref(eng._ccfg), C.byref(io), stream) == 1
    sync()
    with pytest.raises(ValueError):
        eng.update_current_state(cur, dt=None)
    with pytest.raises(ValueError):
        eng.update_current_state(cur, dt=T(np.zeros(2, np.float32)))


def test_robot_rollout_update_params_current_js():
    """B200RobotRollout.update_params(current_js=..., idxs_current_js=..., current_state_dt=...) (GoalRegistry's names) feeds the
    engine's current state: the terms equal those of RolloutEngine.update_current_state with the same tensors; dt falls back to
    current_js.dt; a dt of one element (float, 0-d, [1]) applies to every row; int64 indices are accepted; no dt is refused."""
    from curobo_b200.rollout_protocol import B200RobotRollout
    from curobo_b200.trajectory import JointState
    rm = load_robot("franka")
    P, n = 6, 4                                                   # problems x line-search rows, problem-major
    B = P * n
    ro = B200RobotRollout(rm, RolloutConfig.retarget_ik(), DEV, horizon=1)
    gp, gq, _ = pose_goal(rm, "franka", B, 8)
    idx_goal = T(np.repeat(np.arange(P) % gp.shape[0], n).astype(np.int32))
    ro.update_params(goal_position=T(gp), goal_quat=T(gq), idxs_goal=idx_goal)
    cur_np = rows(rm, "franka", P, seed=9)[:, 0]
    q_np = np.repeat(cur_np, n, axis=0)[:, None, :] + np.random.default_rng(1).normal(0, 0.15, (B, 1, 7)).astype(np.float32)
    q = T(q_np.astype(np.float32))
    cur, vel = T(cur_np), T(np.random.default_rng(2).normal(0, 0.3, cur_np.shape).astype(np.float32))
    idx = np.repeat(np.arange(P), n).astype(np.int32)
    dt = np.full(P, 0.05, np.float32)
    dt[1] = 0.0

    def terms():
        r = ro.evaluate_action(q.clone().requires_grad_(True))
        sync()
        return r.costs_and_constraints.costs.values[1].clone(), ro.engine.out.grad_q.clone()

    ref = RolloutEngine(rm, RolloutConfig.retarget_ik(), DEV)
    ref.update_goal(T(gp), T(gq), idx_goal)
    ref.update_current_state(cur, vel, T(dt), T(idx))
    want = ref.evaluate_action(q)
    sync()
    want_c, want_g = want.cspace_cost.clone(), want.grad_q.clone()
    ro.update_params(current_js=JointState(cur, vel, None, None, T(dt)), idxs_current_js=T(idx))       # dt from current_js.dt
    c, g = terms()
    assert torch.equal(c, want_c) and torch.equal(g, want_g)
    ro.update_params(current_js=JointState(cur, vel, None, None, None), idxs_current_js=T(idx.astype(np.int64)),
                     current_state_dt=T(dt))
    c, g = terms()
    assert torch.equal(c, want_c) and torch.equal(g, want_g)
    ref.update_current_state(cur, vel, T(np.full(P, 0.05, np.float32)), T(idx))
    want = ref.evaluate_action(q)
    sync()
    want_c = want.cspace_cost.clone()
    for one in (0.05, T(np.float32(0.05)), T(np.array([0.05], np.float32))):
        ro.update_params(current_js=JointState(cur, vel, None, None, None), idxs_current_js=T(idx), current_state_dt=one)
        c, _ = terms()
        assert torch.equal(c, want_c)
    with pytest.raises(ValueError):
        ro.update_params(current_js=JointState(cur, vel, None, None, None), idxs_current_js=T(idx))
    ro.engine.clear_current_state()
    c, _ = terms()
    assert not torch.equal(c, want_c)


def test_reference_lbfgs_with_current_js():
    """The reference's own LBFGSOpt over two B200RobotRollout instances, the current state given through
    update_params(current_js=..., idxs_current_js=..., current_state_dt=...): warm-started IK toward a goal ten velocity windows
    away moves no joint more than 2.5 windows (the bound of test_step_limiting_property), and gets closer to the goal than the
    seed.  Skipped when the reference's byte code (oracle/_ref/pyref) was not built."""
    import test_gpu_reference_callsites as rc
    if not os.path.exists(os.path.join(rc.PYREF, "MANIFEST.json")):
        pytest.skip("oracle/_ref/pyref not built")
    ref = rc.load_reference()
    from curobo_b200.rollout_protocol import B200RobotRollout
    from curobo_b200.trajectory import JointState
    rm = load_robot("franka")
    P, n, D, dt = 8, 4, 7, 0.05
    lim_p, lim_v = np.asarray(rm.position_limits, np.float32), np.asarray(rm.velocity_limits, np.float32)
    rng = np.random.default_rng(2)
    q0 = ((lim_p[0] + lim_p[1]) / 2 + rng.uniform(-0.2, 0.2, size=(P, D))).astype(np.float32)
    sign = np.where(rng.random((P, D)) < 0.5, -1.0, 1.0).astype(np.float32)
    q_goal = np.clip(q0 + sign * 10 * lim_v[1] * dt, lim_p[0] + 0.05, lim_p[1] - 0.05).astype(np.float32)
    _, _, gp, gq = O.fk_forward(rm, q_goal)
    scales = [0.0, 0.1, 0.5, 1.0]
    rollouts = [B200RobotRollout(rm, RolloutConfig.retarget_ik(), DEV, horizon=1) for _ in range(2)]
    dc = ref.device_cfg.DeviceCfg(device=torch.device(DEV))
    cfg = ref.lbfgs.LBFGSOptCfg(num_iters=200, inner_iters=25, num_problems=P, device_cfg=dc, line_search_scale=scales,
                                step_scale=0.98, history=15, epsilon=0.01, initial_step_scale=0.001)
    opt = ref.lbfgs.LBFGSOpt(cfg, rollouts, use_cuda_graph=False)
    idx = T(np.repeat(np.arange(P), n).astype(np.int32))
    for ro in rollouts:
        ro.update_params(goal_position=T(gp[:, :, None, :].copy()), goal_quat=T(gq[:, :, None, :].copy()), idxs_goal=idx,
                         current_js=JointState(T(q0), T(np.zeros_like(q0)), None, None, None), idxs_current_js=idx,
                         current_state_dt=T(np.full(P, dt, np.float32)))
    x0 = T(q0).view(P, 1, D)
    q = (opt.optimize(x0) if DEV != "cpu" else opt._core._optimize_impl(x0)).reshape(P, D).detach().cpu().numpy()
    ratio = float(np.max(np.abs(q - q0) / (lim_v[1] * dt)))
    print(f"reference LBFGSOpt with current_js: max step / (v_lim dt) {ratio:.2f}")
    assert ratio <= 2.5
    _, _, p_sol, _ = O.fk_forward(rm, q)
    _, _, p_0, _ = O.fk_forward(rm, q0)
    assert np.median(np.linalg.norm(p_sol[:, 0] - gp[:, 0], axis=-1)) < np.median(np.linalg.norm(p_0[:, 0] - gp[:, 0], axis=-1))


def test_graph_replay_with_current_state_updated_in_place():
    rm = load_robot("franka")
    n = 256
    cfg = RolloutConfig.retarget_ik()
    eng = RolloutEngine(rm, cfg, DEV, CuboidData.from_world(CuboidWorld.create([TABLE, PILLAR], max_n=3), DEV))
    gp, gq, ig = pose_goal(rm, "franka", n, 5)
    eng.update_goal(T(gp), T(gq), T(ig))
    q = T(rows(rm, "franka", n, seed=6))
    cur_p, cur_v = T(rows(rm, "franka", 2, seed=7)[:, 0]), T(np.zeros((2, 7), np.float32))
    dt, idx = T(np.array([0.05, 0.05], np.float32)), T((np.arange(n) % 2).astype(np.int32))
    eng.update_current_state(cur_p, cur_v, dt, idx)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.evaluate_action(q)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eng.evaluate_action(q)
    for k in range(3):                                # a retargeting loop: new current state every frame, same graph
        cur_p.copy_(T(rows(rm, "franka", 2, seed=20 + k)[:, 0]))
        cur_v.normal_(0, 0.3)
        dt.copy_(T(np.array([0.05, 0.02 * k], np.float32)))
        g.replay()
        sync()
        got = (eng.out.cost.clone(), eng.out.grad_q.clone())
        eng.evaluate_action(q)
        sync()
        assert torch.equal(got[0], eng.out.cost) and torch.equal(got[1], eng.out.grad_q)


def test_step_limiting_property():
    """L-BFGS with the retargeting weights, dt = 0.05, from q0 to a goal whose IK solution lies about ten velocity windows
    away on every joint.  Bound with the current state: outside the window [q0 + v_l dt, q0 + v_u dt] the hinge's gradient
    w_b * d (w_b = 10000) must balance the pose gradient, which for the pose weights (1000, 100) and an arm of about one metre
    is at most ~1000 + 100 per radian of joint motion, so the overshoot d stays below ~0.11 rad -- about one window
    (v_lim * dt = 0.109 rad on Franka's first four joints) -- and the step below ~2 windows; 2.5 windows is asserted.
    Without the current state nothing limits the step: it is several windows (4 or more asserted)."""
    from curobo_b200.optim import LBFGSOpt, LBFGSOptCfg
    rm = load_robot("franka")
    dt = 0.05
    lim_p, lim_v = np.asarray(rm.position_limits, np.float32), np.asarray(rm.velocity_limits, np.float32)
    n = 8
    rng = np.random.default_rng(2)
    mid = (lim_p[0] + lim_p[1]) / 2
    q0 = (mid + rng.uniform(-0.2, 0.2, size=(n, 7))).astype(np.float32)
    sign = np.where(rng.random((n, 7)) < 0.5, -1.0, 1.0).astype(np.float32)
    q_goal = np.clip(q0 + sign * 10 * lim_v[1] * dt, lim_p[0] + 0.05, lim_p[1] - 0.05).astype(np.float32)
    _, _, gp, gq = O.fk_forward(rm, q_goal)
    cfg = LBFGSOptCfg(num_iters=200, history=15, cost_relative_threshold=0.01, convergence_iteration=10)
    # the line search evaluates len(line_search_scale) rows per problem, problem-major
    problem = np.repeat(np.arange(n, dtype=np.int32), len(cfg.line_search_scale))
    ratios = {}
    for with_state in (True, False):
        eng = RolloutEngine(rm, RolloutConfig.retarget_ik(), DEV)
        eng.update_goal(T(gp[:, :, None, :].copy()), T(gq[:, :, None, :].copy()), T(problem))
        if with_state:
            eng.update_current_state(T(q0), T(np.zeros_like(q0)), T(np.full(n, dt, np.float32)), T(problem))

        def fn(x, e=eng):
            o = e.evaluate_action(x.view(-1, 1, 7))
            return o.cost.view(-1), o.grad_q.view(-1, 7)
        opt = LBFGSOpt(cfg, n, 1, 7, T(lim_p[0]), T(lim_p[1]), fn, DEV)
        x = opt.optimize(T(q0).view(n, 1, 7)).view(n, 7).cpu().numpy()
        ratios[with_state] = float(np.max(np.abs(x - q0) / (lim_v[1] * dt)))
    print(f"max step / (v_lim dt): with current state {ratios[True]:.2f}, without {ratios[False]:.2f}")
    assert ratios[True] <= 2.5
    assert ratios[False] >= 4.0
