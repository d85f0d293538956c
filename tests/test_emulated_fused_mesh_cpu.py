"""Mesh obstacles inside the fused rollout kernels (tests/test_gpu_fused_mesh.py) on the emulated device of
test_emulated_gpu_suite_cpu.py, at small sizes, plus a CPU-only check of the mesh-aware oracle."""
import numpy as np
import pytest

from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)


@pytest.mark.parametrize("robot,variant,kind,n,H", [("franka", "standard", "all", 21, 1), ("franka", "standard", "mesh", 24, 1),
                                                    ("franka", "big", "mesh", 9, 1), ("g1_29", "standard", "all", 4, 1),
                                                    ("g1_29", "big", "all", 5, 1), ("franka", "traj", "all", 3, 7),
                                                    ("g1_29", "traj", "all", 2, 5)])
def test_fused_mesh_matches_composition_emulated(run, monkeypatch, robot, variant, kind, n, H):  # noqa: F811
    run("test_gpu_fused_mesh", "test_fused_matches_per_operator_composition", monkeypatch, robot, variant, kind, n, H)


def test_fused_mesh_vs_oracle_emulated(run):  # noqa: F811
    run("test_gpu_fused_mesh", "test_fused_vs_mesh_oracle", 24)


@pytest.mark.parametrize("robot,variant,n,H", [("franka", "standard", 40, 1), ("franka", "big", 40, 1), ("g1_29", "big", 6, 1),
                                                ("franka", "traj", 4, 8)])
def test_fused_box_mesh_equals_cuboid_emulated(run, monkeypatch, robot, variant, n, H):  # noqa: F811
    run("test_gpu_fused_mesh", "test_box_mesh_costs_what_the_cuboid_costs", monkeypatch, robot, variant, n, H)


def test_fused_mesh_scene_misc_emulated(run):  # noqa: F811
    run("test_gpu_fused_mesh", "test_scene_combinations_envs_disabled_and_empty", 30)
    run("test_gpu_fused_mesh", "test_zero_scene_weight_ignores_meshes", 12)
    run("test_gpu_fused_mesh", "test_graph_replay_and_in_place_pose_update", 24)
    run("test_gpu_fused_mesh", "test_schedules_without_mesh_build_refuse_mesh_scenes")


def test_oracle_box_mesh_equals_cuboid():
    """The mesh-aware oracle (tests/mesh_rollout_oracle.py) on the reference's regression: a box mesh costs what the analytic
    cuboid costs through rollout_oracle.rollout_cost_grad."""
    import mesh_rollout_oracle as MRO
    from helpers import random_q
    from curobo_b200.mesh import MeshWorld, box_mesh
    from curobo_b200.robot_model import load_robot
    from curobo_b200.rollout import RolloutConfig
    from curobo_b200.world import CuboidWorld
    from oracle import rollout_oracle as O
    rm = load_robot("franka")
    b = {"dims": [0.5, 0.4, 0.6], "pose": [0.3, 0.1, 0.3, 0.9238795, 0.0, 0.3826834, 0.0]}
    v, f = box_mesh(b["dims"])
    cfg = RolloutConfig(self_weight=5000.0, scene_weight=5000.0, scene_activation=0.02).to_oracle_cfg(1)
    q = random_q(rm, 64, seed=5)[:, None, :]
    wm = MRO.rollout_cost_grad(rm, q, cfg, world_mesh=MeshWorld.create([{"vertices": v, "faces": f, "pose": b["pose"]}]))
    wc = O.rollout_cost_grad(rm, q, cfg, world_cuboid=CuboidWorld.create([b]))
    assert (wc["scene_cost"] > 0).sum() > 20 and (wc["scene_cost"] == 0).sum() > 20
    np.testing.assert_allclose(wm["scene_cost"], wc["scene_cost"], rtol=2e-4, atol=2e-6 * wc["scene_cost"].max())
    np.testing.assert_allclose(wm["cost_bh"], wc["cost_bh"], rtol=2e-4, atol=2e-6 * wc["cost_bh"].max())
