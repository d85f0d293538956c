"""The paired arm build of the fused rollout kernel (rollout_fused_kernel<SCENE, false, 3, 2>: two rows per warp, one per
half-warp; scenes without an ESDF) against the one-warp arm build on the same rows.  A row's result must not depend on its
partner row or on the half that ran it: per-term costs and grad_q bit for bit, the row cost up to the order of the lane sum.
CB200_ARM_PAIRS forces one (0) or two (1) rows per warp."""
import numpy as np
import pytest
import torch

from helpers import random_q
from curobo_b200.robot_model import load_robot
from curobo_b200.rollout import RolloutConfig, RolloutEngine
from curobo_b200.scene import CuboidData
from curobo_b200.world import CuboidWorld, make_benchmark_cuboid_world
from oracle import rollout_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VARIANT_ARM = 2  # include/curobo_b200.h: CB200_VARIANT_ARM


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def last_variant():
    from curobo_b200 import lib as cblib
    return int(cblib.load().cb200_last_rollout_variant())


def _buried_env_world():
    """env 0: the benchmark table + pillar; env 1: a 5 m box around the robot, so every sphere of a row in env 1 collides."""
    c0 = make_benchmark_cuboid_world(max_n=4)
    c1 = CuboidWorld.create([{"dims": [5.0, 5.0, 5.0], "pose": [0.0, 0.0, 0.0, 1, 0, 0, 0]}], max_n=4)
    return CuboidWorld(np.concatenate([c0.dims, c1.dims]), np.concatenate([c0.inv_pose, c1.inv_pose]),
                       np.concatenate([c0.enable, c1.enable]), np.concatenate([c0.count, c1.count]))


def _engine(rm, scene, n):
    cfg = RolloutConfig(self_weight=5000.0, scene_weight=5000.0, scene_activation=0.02, cspace_type="position",
                        cspace_weight=(5000.0, 0, 0, 0, 0), cspace_activation=(0.01, 0, 0, 0, 0), pose_weight=(2000.0, 100.0))
    cub = _buried_env_world() if scene == "buried" else make_benchmark_cuboid_world() if scene == "cuboid" else None
    eng = RolloutEngine(rm, cfg, DEV, CuboidData.from_world(cub, DEV) if cub is not None else None)
    _, _, gp, gq = O.fk_forward(rm, random_q(rm, 2, seed=82))
    eng.update_goal(T(gp[:, :, None, :].copy()), T(gq[:, :, None, :].copy()), T((np.arange(n) % 2).astype(np.int32)))
    return eng


def _outputs(o):
    return {k: getattr(o, k).clone() for k in ("cost", "grad_q", "self_cost", "scene_cost", "pose_cost", "cspace_cost")}


@pytest.mark.parametrize("scene,n", [("cuboid", 33), ("cuboid", 8), ("none", 21), ("buried", 22)])
def test_paired_arm_build_matches_one_warp_build(monkeypatch, scene, n):
    """Odd N (the last warp's second half has no row), N below the warp-slot count, cuboids and no obstacles, pairs of a
    colliding and a free row, and (`buried`) pairs where only one row's gradient is dense enough for the dense J^T."""
    rm = load_robot("franka")
    q = random_q(rm, n, seed=81)[:, None, :]
    env = ((np.arange(n) % 4) == 0).astype(np.int32) if scene == "buried" else np.zeros(n, np.int32)
    outs = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("CB200_ARM_PAIRS", flag)
        eng = _engine(rm, scene, n)
        outs[flag] = _outputs(eng.evaluate_action(T(q), env_query_idx=T(env)))
        assert last_variant() == VARIANT_ARM
    a, b = outs["0"], outs["1"]
    for k in ("self_cost", "scene_cost", "pose_cost", "cspace_cost", "grad_q"):
        assert torch.equal(a[k], b[k]), k
    assert torch.allclose(a["cost"], b["cost"], rtol=1e-6, atol=0.0)
    if scene == "none":
        return
    hit = (a["scene_cost"] > 0).sum(-1).view(-1).cpu().numpy()
    pairs = hit[: n - n % 2].reshape(-1, 2)
    assert ((pairs[:, 0] > 0) != (pairs[:, 1] > 0)).any(), "no pair of a colliding and a free row"
    if scene == "buried":
        dense = hit + 2 > 2 * rm.num_links          # the sparse J^T's limit (row_phase_b1 counts the self-collision pair too)
        assert dense[0::4].all() and not dense[1::4].any()


def test_paired_arm_build_graph_replay_and_counter(monkeypatch):
    """Paired rows through the ticket counter (more pairs than warps in the grid), captured in a CUDA graph: replays give the
    eager result and leave the counter re-armed."""
    rm = load_robot("franka")
    n = 20001
    q = T(random_q(rm, n, seed=83)[:, None, :])
    monkeypatch.setenv("CB200_ARM_PAIRS", "1")
    eng = _engine(rm, "cuboid", n)
    ref = _outputs(eng.evaluate_action(q))
    assert last_variant() == VARIANT_ARM
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        eng.evaluate_action(q)
    for _ in range(2):
        eng.out.cost.zero_()
        eng.out.grad_q.zero_()
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(eng.out.cost, ref["cost"]) and torch.equal(eng.out.grad_q, ref["grad_q"])
    assert int(eng._work_counter.abs().sum()) == 0
    monkeypatch.setenv("CB200_ARM_PAIRS", "0")
    one = _outputs(_engine(rm, "cuboid", n).evaluate_action(q))
    for k in ("self_cost", "scene_cost", "pose_cost", "cspace_cost", "grad_q"):
        assert torch.equal(one[k], ref[k]), k
    assert torch.allclose(one["cost"], ref["cost"], rtol=1e-6, atol=0.0)


def test_default_selection_pairs_full_batches(monkeypatch):
    """Without an override, a batch of two rows per resident warp slot of the arm build runs paired and one of half a row per
    slot runs a warp per row; both report the arm build and agree with each other bit for bit on the shared rows."""
    rm = load_robot("franka")
    monkeypatch.delenv("CB200_ARM_PAIRS", raising=False)
    props = torch.cuda.get_device_properties(0)
    slots = props.multi_processor_count * 24
    outs = []
    for n in (slots // 2, 2 * slots + 1):
        q = T(random_q(rm, n, seed=84)[:, None, :])
        outs.append(_outputs(_engine(rm, "cuboid", n).evaluate_action(q)))
        assert last_variant() == VARIANT_ARM
    m = slots // 2
    assert torch.equal(outs[0]["grad_q"], outs[1]["grad_q"][:m]) and torch.equal(outs[0]["scene_cost"], outs[1]["scene_cost"][:m])
