"""The fused rollout's default kernel selection (no CB200_BIG / CB200_TEAM / CB200_ARM_PAIRS / CB200_QUEUE override), pinned through
cb200_last_rollout_variant() on both sides of each measured threshold, for the gradient and the cost-only launch.  The emulated
device of test_emulated_gpu_suite_cpu.py has 2 SMs with 3 resident CTAs each, so the thresholds lie at a few dozen rows: 32 warp
slots of the big kernel.  Paired arm rows report the arm variant, so this test does not tell them apart from one row per warp."""
import pytest
import torch

from dynamics_cases import make_case
from helpers import small_voxel_world
from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)
from test_gpu_cost_only import robot_of
from test_gpu_fused_mesh import PILLAR, TABLE, mesh_world, rows
from curobo_b200 import lib as cblib
from curobo_b200.dynamics import Dynamics
from curobo_b200.mesh import MeshData
from curobo_b200.rollout import RolloutConfig, RolloutEngine
from curobo_b200.scene import CuboidData, VoxelData
from curobo_b200.world import CuboidWorld

DEV = "cpu"
# include/curobo_b200.h: CB200_VARIANT_*
STANDARD, ARM, BIG, TEAM2, TEAM4, TRAJ, TRAJ_DYN = 1, 2, 4, 5, 6, 7, 8
OVERRIDES = ("CB200_BIG", "CB200_TEAM", "CB200_ARM_PAIRS", "CB200_QUEUE")

CASES = [  # robot, world, batch, horizon, gradient launch, cost-only launch (None: not covered by the cost-only kernels)
    ("franka", "esdf", 16, 1, TEAM2, BIG),           # a row per two warp slots: the team kernel (its cost-only twin is big)
    ("franka", "esdf", 17, 1, ARM, ARM),             # more rows: the arm build
    ("franka", "cuboid", 16, 1, ARM, ARM),
    ("franka", "mesh", 16, 1, STANDARD, STANDARD),   # arm-sized, but the arm build has no mesh build
    ("g1_29", "cuboid", 8, 1, TEAM4, BIG),           # humanoid: four warps per row while a row has four warp slots
    ("g1_29", "cuboid", 9, 1, TEAM2, BIG),
    ("g1_29", "cuboid", 64, 1, TEAM2, BIG),          # two warps per row up to two rows per warp slot
    ("g1_29", "cuboid", 65, 1, BIG, BIG),
    ("g1_29", "mesh", 8, 1, BIG, BIG),               # the team kernel has no mesh build
    ("g1_29-pairlist", "cuboid", 8, 1, STANDARD, STANDARD),   # no link-pair list: no big kernel
    ("franka", "swept", 2, 4, TRAJ, None),
    ("g1_29", "swept", 2, 4, TRAJ, None),
    ("franka", "dynamics", 2, 4, TRAJ_DYN, None),
]


def engine(rm, robot, world):
    cub = vox = mesh = None
    if world in ("cuboid", "swept", "dynamics"):
        cub = CuboidData.from_world(CuboidWorld.create([TABLE, PILLAR], max_n=3), DEV)
    if world == "esdf":
        vox = VoxelData.from_world(small_voxel_world(), DEV)
    if world == "mesh":
        mesh = MeshData.from_world(mesh_world(robot), DEV)
    swept = world in ("swept", "dynamics")
    cfg = RolloutConfig(self_weight=5000.0, scene_weight=5000.0, scene_activation=0.02, use_sweep=swept, use_speed_metric=swept,
                        cspace_type="state" if swept else "position", cspace_weight=(5000.0, 0, 0, 0, 0),
                        cspace_activation=(0.01, 0, 0, 0, 0))
    eng = RolloutEngine(rm, cfg, DEV, cub, vox, mesh=mesh)
    if world == "dynamics":
        c = make_case(robot, 1, 31)
        eng.attach_dynamics(Dynamics(rm, c["mc"], c["inn"], gravity=(0.0, 0.0, -9.81), device=DEV), fused=True)
    return eng


@pytest.mark.parametrize("robot,world,B,H,grad_variant,cost_variant", CASES)
def test_default_selection(run, monkeypatch, robot, world, B, H, grad_variant, cost_variant):  # noqa: F811
    for k in OVERRIDES:
        monkeypatch.delenv(k, raising=False)
    robot, rm = robot_of(robot)
    eng = engine(rm, robot, world)
    L = cblib.load()
    q = torch.as_tensor(rows(rm, robot, B, H=H, seed=5))
    state = {}
    if H > 1:
        D = rm.num_dof
        state = dict(vel=torch.zeros(B, H, D), acc=torch.zeros(B, H, D), jerk=torch.zeros(B, H, D),
                     dt=torch.full((B,), 0.05, dtype=torch.float32))
    eng.evaluate_action(q, **state)
    assert int(L.cb200_last_rollout_variant()) == grad_variant
    if cost_variant is not None:
        eng.evaluate_cost(q)
        assert int(L.cb200_last_rollout_variant()) == cost_variant | cblib.VARIANT_COST_ONLY
