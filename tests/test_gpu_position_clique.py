"""GPU parity of the position (clique) and acceleration control-space transitions, called through the C ABI
(curobo_b200.backends.trajectory), against
  * the numpy oracle (oracle/clique_oracle.py), and
  * the REFERENCE's own legacy kernels compiled into oracle/_ref (stored outputs, tests/ref_legacy_kernels.py): positions bit for
    bit, velocity / acceleration / jerk / gradients within 1e-6 of each batch row's largest magnitude.
Then the front ends: the host mirrors (StateFromPositionClique, StateFromAcceleration), the reference's own autograd Functions
over our backend, RolloutEngine.evaluate_positions and B200RobotRollout(action_space="position_clique").
Tolerances vs the float32 oracle (numpy neither contracts FMAs nor approximates division): 2e-5 of the output scale.
"""
import os

import numpy as np
import pytest
import torch

import ref_kernels
import ref_legacy_kernels
from clique_cases import CASES, case_id, make_case
from curobo_b200.backends import trajectory as trajectory_cu
from curobo_b200.trajectory import (AccelerationTensorStepIdxKernel, CliqueTensorStepIdxKernel, JointState,
                                    StateFromAcceleration, StateFromPositionClique)
from oracle import clique_oracle as co

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def dev_case(c):
    d = dict(c)
    d["u_t"], d["u_acc_t"], d["dt_h_t"] = T(c["u"]), T(c["u_acc"]), T(c["dt_h"])
    d["start_t"] = tuple(T(x) for x in c["start"])
    d["goal_t"] = tuple(T(x) for x in c["goal"])
    d["sidx_t"], d["gidx_t"] = T(c["start_idx"]), T(c["goal_idx"])
    d["dt_t"], d["imp_t"] = T(c["traj_dt"]), T(c["implicit"])
    d["grads_t"] = tuple(T(g) for g in c["grads"])
    return d


def nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def ours_forward(c):
    B, H, D = c["B"], c["H"], c["D"]
    outs = [nan(B, H, D) for _ in range(4)] + [nan(B)]
    trajectory_cu.launch_differentiation_position_forward_kernel(*outs, c["u_t"], *c["start_t"], *c["goal_t"], c["sidx_t"],
                                                                 c["gidx_t"], c["dt_t"], c["imp_t"], B, H, D)
    return outs


def ours_backward(c):
    out = nan(c["B"], c["n"], c["D"])
    trajectory_cu.launch_differentiation_position_backward_kernel(out, *c["grads_t"], c["dt_t"], c["gidx_t"], c["imp_t"],
                                                                  c["B"], c["H"], c["D"])
    return out


def ours_integrate(c):
    B, H, D = c["B"], c["H"], c["D"]
    outs = [nan(B, H, D) for _ in range(4)]
    trajectory_cu.launch_integration_acceleration_kernel(*outs, c["u_acc_t"], *c["start_t"], c["sidx_t"], c["dt_h_t"], B, H, D)
    return outs


def close_to_oracle(got, want, rtol=2e-5):
    g = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    assert np.isfinite(g).all()
    np.testing.assert_allclose(g, want, rtol=rtol, atol=rtol * max(1.0, float(np.abs(want).max())))


def close_per_row(got, ref, rel=1e-6):
    """|got - ref| <= rel * max |ref| of the same batch row."""
    g, r = got.cpu().numpy(), ref.cpu().numpy()
    scale = np.abs(r).reshape(r.shape[0], -1).max(1).reshape((-1,) + (1,) * (r.ndim - 1))
    assert (np.abs(g - r) <= rel * scale).all(), float((np.abs(g - r) / np.maximum(scale, 1e-30)).max())


@pytest.mark.parametrize("kw", CASES, ids=case_id)
def test_clique_forward_vs_oracle_and_reference(kw):
    c = dev_case(make_case(**kw))
    got = ours_forward(c)
    want = co.clique_forward(c["u"], *c["start"], c["goal"][0], c["start_idx"], c["goal_idx"], c["traj_dt"], c["implicit"], c["H"])
    for k in range(4):
        close_to_oracle(got[k], want[k])
    assert np.array_equal(got[4].cpu().numpy(), want[4])
    if ref_kernels.available():
        ref = ref_legacy_kernels.clique_forward(c["u_t"], c["start_t"], c["goal_t"], c["sidx_t"], c["gidx_t"], c["dt_t"], c["imp_t"], c["H"])
        assert torch.equal(got[0], ref[0]), "positions vs reference"
        for k in (1, 2, 3):
            close_per_row(got[k], ref[k])
        assert torch.equal(got[4], ref[4])


@pytest.mark.parametrize("kw", CASES, ids=case_id)
def test_clique_backward_vs_oracle_and_reference(kw):
    c = dev_case(make_case(**kw))
    got = ours_backward(c)
    want = co.clique_backward(*c["grads"], c["traj_dt"], c["goal_idx"], c["implicit"])
    close_to_oracle(got, want, rtol=1e-5)
    if ref_kernels.available():
        ref = ref_legacy_kernels.clique_backward(c["grads_t"], c["dt_t"], c["gidx_t"], c["imp_t"])
        close_per_row(got, ref)


@pytest.mark.parametrize("kw", CASES, ids=case_id)
def test_acceleration_integration_vs_oracle_and_reference(kw):
    c = dev_case(make_case(**kw))
    got = ours_integrate(c)
    want = co.integrate_acceleration(c["u_acc"], *c["start"], c["start_idx"], c["dt_h"])
    for k in range(4):
        close_to_oracle(got[k], want[k])
    if ref_kernels.available():
        ref = ref_legacy_kernels.integrate_acceleration(c["u_acc_t"], c["start_t"], c["sidx_t"], c["dt_h_t"])
        assert torch.equal(got[0], ref[0]), "positions vs reference"
        for k in (1, 2, 3):
            close_per_row(got[k], ref[k])


def test_error_behaviour():
    c = dev_case(make_case(seed=41, B=2, H=9, D=7))
    B, H, D = c["B"], c["H"], c["D"]
    outs = [torch.zeros((B, H, D), device=DEV) for _ in range(4)] + [torch.zeros(B, device=DEV)]
    fwd = lambda *o, u=c["u_t"], H=H: trajectory_cu.launch_differentiation_position_forward_kernel(  # noqa: E731
        *o, u, *c["start_t"], *c["goal_t"], c["sidx_t"], c["gidx_t"], c["dt_t"], c["imp_t"], B, H, D)
    with pytest.raises(ValueError, match="horizon >= 8"):
        fwd(*outs, H=7)
    with pytest.raises(ValueError, match="horizon >= 8"):
        trajectory_cu.launch_differentiation_position_backward_kernel(torch.zeros((B, 3, D), device=DEV), *c["grads_t"], c["dt_t"],
                                                                      c["gidx_t"], c["imp_t"], B, 7, D)
    with pytest.raises(ValueError, match="dtype"):
        fwd(*outs, u=c["u_t"].double())
    if DEV != "cpu":             # (the emulated run of this test has no other device to refuse)
        with pytest.raises(ValueError, match="CUDA-only|device"):
            fwd(*outs, u=c["u_t"].cpu())
    with pytest.raises(ValueError, match="elements"):
        fwd(*outs, u=c["u_t"][:1].contiguous())
    with pytest.raises(ValueError, match="elements"):
        trajectory_cu.launch_integration_acceleration_kernel(*outs[:4], c["u_acc_t"], *c["start_t"], c["sidx_t"], c["dt_h_t"][:3],
                                                             B, H, D)
    # batch_size == 0: nothing is launched, nothing is written
    fwd0 = [torch.full((1, H, D), 5.0, device=DEV) for _ in range(4)] + [torch.full((1,), 5.0, device=DEV)]
    trajectory_cu.launch_differentiation_position_forward_kernel(*fwd0, c["u_t"], *c["start_t"], *c["goal_t"], c["sidx_t"],
                                                                 c["gidx_t"], c["dt_t"], c["imp_t"], 0, H, D)
    torch.cuda.synchronize()
    assert all(bool((t == 5.0).all()) for t in fwd0)
    # the autograd Functions' own checks
    with pytest.raises(ValueError, match="Action shape is not compatible with horizon"):
        CliqueTensorStepIdxKernel.apply(c["u_t"][:, 1:].contiguous(), *c["start_t"], *c["goal_t"], c["sidx_t"], c["gidx_t"],
                                        *outs, c["dt_t"], c["imp_t"], torch.zeros((B, H - 4, D), device=DEV))
    u = c["u_acc_t"].clone().requires_grad_(True)
    p, _, _, _ = AccelerationTensorStepIdxKernel.apply(u, *c["start_t"], c["sidx_t"], *[torch.zeros((B, H, D), device=DEV)
                                                                                         for _ in range(4)],
                                                       c["dt_h_t"], torch.zeros((B, H, D), device=DEV))
    with pytest.raises(NotImplementedError):
        p.sum().backward()
    with pytest.raises(ValueError, match="filter"):
        StateFromPositionClique(DEV, torch.full((B,), 0.05, device=DEV), D, filter_velocity=True, batch_size=B, horizon=H)
    # after the rejected calls the library and torch are still healthy
    torch.cuda.synchronize()
    assert torch.isfinite(ours_forward(c)[0]).all()


@pytest.mark.parametrize("implicit", [False, True])
def test_state_transitions(implicit):
    """StateFromPositionClique.forward + loss.backward(): u.grad equals the oracle's adjoint; StateFromAcceleration.forward
    equals the oracle's integration (the reference's transition classes, fns_state_transition.py:90-308)."""
    B, H, D, n_goal = 6, 14, 7, 3
    c = dev_case(make_case(seed=31, B=B, H=H, D=D, n_goal=n_goal, implicit=implicit))
    fn = StateFromPositionClique(DEV, torch.full((B,), 0.05, device=DEV), D, batch_size=B, horizon=H)
    assert fn.action_horizon == H - 4
    start = JointState(*c["start_t"], jerk=None)
    # goal rows [n_goal, 1, D] with dt / use_implicit_goal_state [n_goal, 1]: the shapes the reference's checks require
    goal = JointState(*[g.view(n_goal, 1, D) for g in c["goal_t"]], jerk=None, dt=c["dt_t"].view(n_goal, 1))
    out = JointState.zeros((B, H, D), DEV)
    u = c["u_t"].clone().requires_grad_(True)
    seq = fn.forward(start, u, out, start_state_idx=c["sidx_t"], goal_state=goal, goal_state_idx=c["gidx_t"],
                     use_implicit_goal_state=c["imp_t"].view(n_goal, 1))
    want = co.clique_forward(c["u"], *c["start"], c["goal"][0], c["start_idx"], c["goal_idx"], c["traj_dt"], c["implicit"], H)
    for g, w in zip((seq.position, seq.velocity, seq.acceleration, seq.jerk), want):
        close_to_oracle(g.detach(), w)
    w = c["grads_t"]
    ((seq.position * w[0]).sum() + (seq.velocity * w[1]).sum() + (seq.acceleration * w[2]).sum() + (seq.jerk * w[3]).sum()).backward()
    close_to_oracle(u.grad, co.clique_backward(*c["grads"], c["traj_dt"], c["goal_idx"], c["implicit"]), rtol=1e-5)
    with pytest.raises(ValueError, match="Shape mismatch"):
        fn.forward(start, u, out, start_state_idx=c["sidx_t"], goal_state=JointState(*c["goal_t"], jerk=None, dt=c["dt_t"]),
                   goal_state_idx=c["gidx_t"], use_implicit_goal_state=c["imp_t"])

    fa = StateFromAcceleration(DEV, c["dt_h_t"], D, batch_size=B, horizon=H)
    sa = fa.forward(start, c["u_acc_t"], JointState.zeros((B, H, D), DEV), start_state_idx=c["sidx_t"])
    want = co.integrate_acceleration(c["u_acc"], *c["start"], c["start_idx"], c["dt_h"])
    for g, w_ in zip((sa.position, sa.velocity, sa.acceleration, sa.jerk), want):
        close_to_oracle(g, w_)


def test_reference_functions_over_b200_backend():
    """The reference's own CliqueTensorStepIdxKernel.apply (forward + backward) and AccelerationTensorStepIdxKernel.apply
    (cuda_ops/trajectory.py:95-296) with trajectory_cu = curobo_b200.backends.trajectory (INTEGRATION.md section 4)."""
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "pyref", "MANIFEST.json")):
        pytest.skip("oracle/_ref/pyref not built (python oracle/build_pyref.py where the reference tree exists)")
    from test_gpu_reference_callsites import load_reference
    ref = load_reference()
    B, H, D = 6, 30, 7
    c = dev_case(make_case(seed=17, B=B, H=H, D=D))
    u = c["u_t"].clone().requires_grad_(True)
    outs = [torch.zeros((B, H, D), device=DEV) for _ in range(4)]
    out_dt, gu = torch.zeros(B, device=DEV), torch.zeros((B, H - 4, D), device=DEV)
    p, v, a, j = ref.trajectory.CliqueTensorStepIdxKernel.apply(u, *c["start_t"], *c["goal_t"], c["sidx_t"], c["gidx_t"], *outs,
                                                                out_dt, c["dt_t"], c["imp_t"], gu)
    g = c["grads_t"]
    ((p * g[0]).sum() + (v * g[1]).sum() + (a * g[2]).sum() + (j * g[3]).sum()).backward()
    want = co.clique_forward(c["u"], *c["start"], c["goal"][0], c["start_idx"], c["goal_idx"], c["traj_dt"], c["implicit"], H)
    for got, w in zip((p, v, a, j), want):
        close_to_oracle(got.detach(), w)
    close_to_oracle(u.grad, co.clique_backward(*c["grads"], c["traj_dt"], c["goal_idx"], c["implicit"]), rtol=1e-5)
    acc_outs = [torch.zeros((B, H, D), device=DEV) for _ in range(4)]
    ap, av, aa, aj = ref.trajectory.AccelerationTensorStepIdxKernel.apply(c["u_acc_t"], *c["start_t"], c["sidx_t"], *acc_outs,
                                                                          c["dt_h_t"], torch.zeros((B, H, D), device=DEV))
    want_acc = co.integrate_acceleration(c["u_acc"], *c["start"], c["start_idx"], c["dt_h"])
    for got, w in zip((ap, av, aa, aj), want_acc):
        close_to_oracle(got, w)
    if ref_kernels.available():   # and against the reference's own compiled kernels on the same inputs
        rf = ref_legacy_kernels.clique_forward(c["u_t"], c["start_t"], c["goal_t"], c["sidx_t"], c["gidx_t"], c["dt_t"], c["imp_t"], H)
        assert torch.equal(p.detach(), rf[0])
        for got, r in zip((v, a, j), rf[1:4]):
            close_per_row(got.detach(), r)
        close_per_row(u.grad, ref_legacy_kernels.clique_backward(c["grads_t"], c["dt_t"], c["gidx_t"], c["imp_t"]))
        ra = ref_legacy_kernels.integrate_acceleration(c["u_acc_t"], c["start_t"], c["sidx_t"], c["dt_h_t"])
        assert torch.equal(ap, ra[0])
        for got, r in zip((av, aa, aj), ra[1:]):
            close_per_row(got, r)


# ------------------------------------------------------------------------------------------------
# front end on the fused rollout: RolloutEngine.evaluate_positions
# ------------------------------------------------------------------------------------------------
def _trajopt_problem(B, H, seed, mode="trajopt_swept"):
    """Franka trajopt rows: waypoints around a joint-space random walk, start near the first, goal = the last."""
    from helpers import random_q, random_walk_q, small_voxel_world
    from curobo_b200.robot_model import load_robot
    from curobo_b200.rollout import RolloutConfig, RolloutEngine
    from curobo_b200.scene import CuboidData, VoxelData
    from curobo_b200.world import make_benchmark_cuboid_world
    from oracle import rollout_oracle as O
    rm = load_robot("franka")
    D = rm.num_dof
    rng = np.random.default_rng(seed)
    u = random_walk_q(rm, B, H - 4, seed=seed).astype(np.float32)
    z = np.zeros((B, D), np.float32)
    start = (u[:, 0] + rng.normal(0, 0.02, (B, D)).astype(np.float32), rng.normal(0, 0.1, (B, D)).astype(np.float32), z)
    goal = (u[:, -1].copy(), z, z)
    idx = np.arange(B, dtype=np.int32)
    traj_dt = np.full(B, 0.05, np.float32)
    imp = (np.arange(B) % 2).astype(np.uint8)
    cfg = RolloutConfig.trajopt()
    if mode == "discrete":
        cfg.use_sweep = False
        cfg.use_speed_metric = False
    cub, vox = make_benchmark_cuboid_world(), small_voxel_world()
    _, _, gp, gq = O.fk_forward(rm, random_q(rm, B, seed=seed + 1))
    gp, gq = gp[:, :, None, :].copy(), gq[:, :, None, :].copy()

    def engine():
        e = RolloutEngine(rm, cfg, DEV, CuboidData.from_world(cub, DEV), VoxelData.from_world(vox, DEV))
        e.update_goal(T(gp), T(gq), T(idx), non_terminal_axes=torch.zeros((1, 6), dtype=torch.float32, device=DEV))
        return e
    return dict(rm=rm, B=B, H=H, D=D, u=u, start=start, goal=goal, idx=idx, traj_dt=traj_dt, imp=imp, cfg=cfg, cub=cub,
                vox=vox, gp=gp, gq=gq, engine=engine,
                start_t=JointState(*[T(x) for x in start], jerk=None),
                goal_t=JointState(*[T(x) for x in goal], jerk=None, dt=T(traj_dt)))


@pytest.mark.parametrize("mode", ["trajopt_swept", "discrete"])
def test_evaluate_positions_vs_composition_and_oracle_chain(mode, B=4, H=14):
    """evaluate_positions == clique forward -> evaluate_action -> clique adjoint composed by hand (bit for bit), and
    == the oracle chain clique oracle -> rollout oracle -> clique-adjoint oracle."""
    from oracle import rollout_oracle as O
    P = _trajopt_problem(B, H, seed=71, mode=mode)
    D, idx_t = P["D"], T(P["idx"])
    eng = P["engine"]()
    out = eng.evaluate_positions(T(P["u"]), P["start_t"], idx_t, P["goal_t"], idx_t, T(P["imp"]))
    torch.cuda.synchronize()
    cost, gu = out.cost.clone(), out.grad_u.clone()
    state = [t.clone() for t in eng._state]
    assert tuple(gu.shape) == (B, H - 4, D) and torch.isfinite(gu).all() and float(gu.abs().max()) > 0

    # by hand, on a second engine
    seq = [torch.zeros((B, H, D), device=DEV) for _ in range(4)]
    odt = torch.zeros(B, device=DEV)
    st, gl = P["start_t"], P["goal_t"]
    trajectory_cu.launch_differentiation_position_forward_kernel(*seq, odt, T(P["u"]), st.position, st.velocity, st.acceleration,
                                                                 gl.position, gl.velocity, gl.acceleration, idx_t, idx_t, gl.dt,
                                                                 T(P["imp"]), B, H, D)
    o2 = P["engine"]().evaluate_action(seq[0], vel=seq[1], acc=seq[2], jerk=seq[3], dt=odt)
    gu2 = torch.zeros_like(gu)
    trajectory_cu.launch_differentiation_position_backward_kernel(gu2, o2.grad_q, o2.grad_vel, o2.grad_acc, o2.grad_jerk, gl.dt,
                                                                  idx_t, T(P["imp"]), B, H, D)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(state, seq))
    assert torch.equal(o2.cost, cost) and torch.equal(gu2, gu)

    # oracle chain (the rollout oracle is fed the GPU's states, already checked against the clique oracle: swept-collision
    # sample counts are a discontinuous function of waypoint distances)
    p, v, a, j, odt_w = co.clique_forward(P["u"], *P["start"], P["goal"][0], P["idx"], P["idx"], P["traj_dt"], P["imp"], H)
    for g, w in zip(state, (p, v, a, j)):
        close_to_oracle(g, w)
    ocfg = P["cfg"].to_oracle_cfg(1)
    ocfg["pose_non_terminal_axes"] = np.zeros((1, 6), np.float32)
    sp, sv, sa, sj = (t.cpu().numpy() for t in state)
    want = O.rollout_cost_grad(P["rm"], sp, ocfg, world_cuboid=P["cub"], world_voxel=P["vox"], goal_pos=P["gp"], goal_quat=P["gq"],
                               idxs_goal=P["idx"], vel=sv, acc=sa, jerk=sj, dt=odt_w)
    np.testing.assert_allclose(cost.cpu().numpy(), want["cost_bh"], rtol=5e-4, atol=2e-5 * want["cost_bh"].max())
    gs = want["cspace_grads"]
    want_gu = co.clique_backward(want["grad_q"], gs[1], gs[2], gs[3], P["traj_dt"], P["idx"], P["imp"])
    np.testing.assert_allclose(gu.cpu().numpy(), want_gu, rtol=5e-3, atol=5e-5 * np.abs(want_gu).max())


def test_evaluate_positions_graph_replay(B=128, H=34):
    """Trajopt size: a captured evaluate_positions replays to the eager result."""
    P = _trajopt_problem(B, H, seed=81)
    idx_t, u_t, imp_t = T(P["idx"]), T(P["u"]), T(P["imp"])
    eng = P["engine"]()
    out = eng.evaluate_positions(u_t, P["start_t"], idx_t, P["goal_t"], idx_t, imp_t)
    torch.cuda.synchronize()
    cost, gu = out.cost.clone(), out.grad_u.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            eng.evaluate_positions(u_t, P["start_t"], idx_t, P["goal_t"], idx_t, imp_t)
        eng.out.cost.zero_()
        eng.out.grad_u.zero_()
        graph.replay()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert torch.equal(eng.out.cost, cost) and torch.equal(eng.out.grad_u, gu)


def test_rollout_protocol_position_clique(B=4, H=14):
    """B200RobotRollout(action_space="position_clique"): the reference's `cat + sum + backward(ones)` through
    FusedTermsFunction yields the engine's grad_u, and the state returned is the stencil's."""
    from curobo_b200.rollout_protocol import B200RobotRollout
    from curobo_b200.scene import CuboidData
    P = _trajopt_problem(B, H, seed=91)
    D, idx_t = P["D"], T(P["idx"])
    ro = B200RobotRollout(P["rm"], P["cfg"], DEV, cuboid=CuboidData.from_world(P["cub"], DEV), horizon=H,
                          action_space="position_clique")
    assert ro.action_horizon == H - 4 and ro.horizon == H
    with pytest.raises(ValueError, match="update_params"):
        ro.evaluate_action(T(P["u"]))
    ro.update_params(goal_position=T(P["gp"]), goal_quat=T(P["gq"]), idxs_goal=idx_t, start_state=P["start_t"],
                     goal_state=P["goal_t"], start_state_idx=idx_t, goal_state_idx=idx_t, use_implicit_goal_state=T(P["imp"]))
    x = T(P["u"]).requires_grad_(True)
    r = ro.evaluate_action(x)
    c = r.costs_and_constraints.get_sum_cost_and_constraint(sum_horizon=True)
    c.backward(gradient=torch.ones_like(c))
    torch.cuda.synchronize()
    assert torch.equal(x.grad, ro.engine.out.grad_u)
    assert float(x.grad.abs().max()) > 0
    want = co.clique_forward(P["u"], *P["start"], P["goal"][0], P["idx"], P["idx"], P["traj_dt"], P["imp"], H)
    for g, w in zip((r.state.position, r.state.velocity, r.state.acceleration, r.state.jerk), want):
        close_to_oracle(g, w)
    with pytest.raises(ValueError, match="horizon >= 8"):
        B200RobotRollout(P["rm"], P["cfg"], DEV, horizon=7, action_space="position_clique")


def test_lbfgs_lowers_trajopt_cost_in_position_space(P_=8, H=34, iters=40):
    """This repository's LBFGSOpt drives evaluate_positions from a seeded straight-line start on a Franka trajopt problem
    and lowers the cost of every problem."""
    from curobo_b200.optim import LBFGSOpt, LBFGSOptCfg
    P = _trajopt_problem(P_, H, seed=101)
    rm, D, n = P["rm"], P["D"], H - 4
    cfg = LBFGSOptCfg(num_iters=iters, line_search_scale=[0.0, 0.1, 0.5, 1.0], initial_step_scale=0.001)
    n_ls = len(cfg.line_search_scale)
    rows = P_ * n_ls
    rep = lambda a: np.repeat(a, n_ls, axis=0)  # noqa: E731  rows: problem-major, line-search-minor
    idx = np.arange(rows, dtype=np.int32)
    st = JointState(*[T(rep(x)) for x in P["start"]], jerk=None)
    gl = JointState(*[T(rep(x)) for x in P["goal"]], jerk=None, dt=T(rep(P["traj_dt"])))
    imp = T(rep(P["imp"]))
    eng = P["engine"]()
    eng.update_goal(T(P["gp"]), T(P["gq"]), T(rep(P["idx"])), non_terminal_axes=torch.zeros((1, 6), device=DEV))
    idx_t = T(idx)

    def cost_grad(x):
        out = eng.evaluate_positions(x.view(rows, n, D), st, idx_t, gl, idx_t, imp)
        return out.cost.sum(-1), out.grad_u.view(rows, n * D)
    lo, hi = T(rm.position_limits[0]), T(rm.position_limits[1])
    opt = LBFGSOpt(cfg, P_, n, D, lo, hi, cost_grad, DEV)
    # seed: the straight line from the start to the goal position
    s = np.linspace(0.0, 1.0, n, dtype=np.float32)[None, :, None]
    x0 = T(P["start"][0][:, None] * (1 - s) + P["goal"][0][:, None] * s).reshape(P_, n * D)
    c0 = cost_grad(x0.repeat_interleave(n_ls, 0))[0].view(P_, n_ls)[:, 0].clone()
    x = opt.optimize(x0).reshape(P_, n * D)
    c1 = cost_grad(x.repeat_interleave(n_ls, 0))[0].view(P_, n_ls)[:, 0].clone()
    torch.cuda.synchronize()
    assert torch.isfinite(c1).all()
    assert (c1 < c0).all(), (c0, c1)
    assert float(c1.sum()) < 0.5 * float(c0.sum()), (c0, c1)
