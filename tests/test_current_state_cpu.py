"""The current-state block of the POSITION c-space cost on the CPU: oracle/current_state_oracle.py against the output of the
reference's own forward_cspace_position_warp (tests/golden/cspace_position_current_state_golden.npz), and the host-side
plumbing (RolloutConfig.retarget_ik, the RolloutIO fields)."""
import os

import numpy as np
import pytest

from oracle import current_state_oracle as CS
from oracle import rollout_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cspace_position_current_state_golden.npz")
CASES = ("vel_acc", "no_velocity", "mixed_dt", "empty_window", "with_target")


def golden(name):
    G = np.load(GOLDEN)
    pre = name + "/"
    return {k[len(pre):]: G[k] for k in G.files if k.startswith(pre)}


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference_source(case):
    c = golden(case)
    cost, g = CS.cspace_position_cost(c["q"], c["lim_p"], c["weight"], c["act"], target=c["target"], idxs_target=c["idxs_target"],
                                      target_weight=float(c["target_weight"][0]), target_dof_weight=c["dof_weight"],
                                      current_position=c["cur_p"], current_velocity=c["cur_v"] if int(c["has_velocity"]) else None,
                                      idxs_current=c["idxs_cur"], state_dt=c["dt"], limits_v=c["lim_v"], reg_weight=c["reg"])
    for got, want in ((cost, c["cost"]), (g, c["grad_p"])):
        assert np.allclose(got, want, rtol=1e-5, atol=1e-7 * np.abs(want).max()), float(np.abs(got - want).max())


def test_golden_exercises_the_block():
    """The fixture reaches every branch: rows with dt = 0, dofs hinged against the velocity window, empty windows, and
    regularizer-only dofs (inside the window, off the limits)."""
    c = golden("mixed_dt")
    assert (c["dt"][c["idxs_cur"]] == 0).any() and (c["dt"][c["idxs_cur"]] > 0).any()
    e = golden("empty_window")
    lo = np.maximum(e["lim_p"][0] + 0.01 * (e["lim_p"][1] - e["lim_p"][0]), e["cur_p"] + e["lim_v"][0] * e["dt"][:, None])
    hi = np.minimum(e["lim_p"][1] - 0.01 * (e["lim_p"][1] - e["lim_p"][0]), e["cur_p"] + e["lim_v"][1] * e["dt"][:, None])
    assert (lo > hi).any()
    v = golden("vel_acc")
    plain, _ = O.cspace_position_cost(v["q"], v["lim_p"], v["weight"], v["act"])
    assert ((plain == 0) & (v["cost"] > 0)).any() and ((plain == 0) & (v["cost"] > 1e3 * np.abs(v["cost"][plain == 0]).min())).any()


def test_without_current_state_is_the_plain_oracle():
    c = golden("vel_acc")
    a = CS.cspace_position_cost(c["q"], c["lim_p"], c["weight"], c["act"])
    b = O.cspace_position_cost(c["q"], c["lim_p"], c["weight"], c["act"])
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    z = CS.cspace_position_cost(c["q"], c["lim_p"], c["weight"], c["act"], current_position=c["cur_p"], idxs_current=c["idxs_cur"],
                                state_dt=np.zeros_like(c["dt"]), limits_v=c["lim_v"], reg_weight=c["reg"])
    assert all(np.array_equal(x, y) for x, y in zip(z, b))


def test_retarget_ik_weights_and_io_fields():
    import ctypes as C
    from curobo_b200 import lib as cblib
    from curobo_b200.rollout import RolloutConfig
    cfg = RolloutConfig.retarget_ik()
    assert cfg.cspace_type == "position" and tuple(cfg.cspace_weight[:2]) == (10000.0, 0.0)
    assert tuple(cfg.cspace_activation[:2]) == (0.01, 0.01) and tuple(cfg.cspace_reg[:2]) == (0.01, 0.01)
    assert tuple(cfg.pose_weight) == (1000.0, 100.0) and cfg.scene_weight == 10000.0 and cfg.scene_activation == 0.0
    assert cfg.self_weight == 10000.0
    names = [f[0] for f in cblib.RolloutIO._fields_]
    assert names[-5:] == ["meshes", "current_position", "current_velocity", "idxs_current_state", "current_state_dt"]
    assert cblib.RolloutIO.current_state_dt.offset == C.sizeof(cblib.RolloutIO) - C.sizeof(C.c_void_p)


def test_rollout_oracle_with_inactive_current_state_is_bit_identical():
    """oracle/current_state_oracle.rollout_cost_grad adds the c-space term in rollout_oracle's order: with dt = 0 on every row it
    returns rollout_oracle.rollout_cost_grad's arrays to the bit."""
    from curobo_b200.robot_model import load_robot
    from curobo_b200.rollout import RolloutConfig
    from helpers import random_q
    rm = load_robot("franka")
    q = random_q(rm, 6, seed=2)[:, None, :]
    q[0, 0, 0] = rm.position_limits[1][0] + 0.1
    cfg = RolloutConfig.retarget_ik().to_oracle_cfg(1)
    a = O.rollout_cost_grad(rm, q, cfg)
    b = CS.rollout_cost_grad(rm, q, cfg, current_position=q[:2, 0], idxs_current=np.arange(6) % 2, state_dt=np.zeros(2, np.float32))
    for k in ("cost", "cost_bh", "grad_q", "cspace_cost"):
        assert np.array_equal(a[k], b[k]), k
