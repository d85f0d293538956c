"""Launch plans of the fused rollout kernels under several host threads.

A launch plan (warps per CTA, resident CTAs per SM) is cached per thread, while a kernel's dynamic shared-memory cap is one
setting per device.  Threads that run different robots on the same kernel must not invalidate each other's cached plans."""
import threading

import numpy as np
import pytest
import torch

from curobo_b200 import lib as cblib
from curobo_b200.robot_model import load_robot
from curobo_b200.rollout import RolloutConfig, RolloutEngine
from curobo_b200.scene import CuboidData
from curobo_b200.trajectory import JointState
from curobo_b200.world import make_benchmark_cuboid_world
from helpers import random_walk_q

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VARIANT_STANDARD = 1  # include/curobo_b200.h: CB200_VARIANT_STANDARD


def _knots_runner(name, cfg, cub, seed):
    """A closure that evaluates one robot's knots through the in-kernel spline schedule and returns (cost, grad_knots, variant)."""
    rm = load_robot(name)
    B, nk, D, degree, steps = 64, 8, rm.num_dof, 4, 2
    knots = torch.as_tensor(random_walk_q(rm, B, nk, seed=seed).astype(np.float32)).to(DEV)
    z = torch.zeros((1, D), device=DEV)
    start = JointState(knots[:1, 0].contiguous(), z, z, z)
    goal = JointState(knots[:1, -1].contiguous(), z, z, z, dt=torch.full((1,), 0.05, device=DEV))
    zi = torch.zeros(B, dtype=torch.int32, device=DEV)
    imp = torch.zeros(1, dtype=torch.uint8, device=DEV)
    eng = RolloutEngine(rm, cfg, DEV, cub)

    def run():
        out = eng.evaluate_knots(knots, start, zi, goal, zi, imp, degree, steps, in_kernel_spline=True)
        torch.cuda.synchronize()
        return out.cost.clone(), out.grad_knots.clone(), int(cblib.load().cb200_last_rollout_variant())
    return run


def test_two_threads_two_robots_one_kernel():
    """Franka on one thread and G1-29 on another, both on the same kernel: the in-kernel spline schedule of rollout_fused_kernel,
    discrete mode, cuboids.  G1 plans, then Franka plans, then G1 launches again from its cached plan.  Every result equals that
    robot's single-threaded result bit for bit."""
    cfg = RolloutConfig.trajopt()
    cfg.use_sweep = False
    cfg.use_speed_metric = False
    cub = CuboidData.from_world(make_benchmark_cuboid_world(), DEV)
    franka, g1 = _knots_runner("franka", cfg, cub, 93), _knots_runner("g1_29", cfg, cub, 94)
    want = {"franka": franka(), "g1": g1()}
    got, errors = {}, []
    g1_planned, franka_planned = threading.Event(), threading.Event()

    def g1_thread():
        try:
            got["g1_first"] = g1()
            g1_planned.set()
            franka_planned.wait(timeout=300)
            got["g1"] = g1()
        except Exception as e:  # reported by the main thread
            errors.append(e)
        finally:
            g1_planned.set()

    def franka_thread():
        try:
            g1_planned.wait(timeout=300)
            got["franka"] = franka()
        except Exception as e:
            errors.append(e)
        finally:
            franka_planned.set()

    threads = [threading.Thread(target=g1_thread), threading.Thread(target=franka_thread)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    assert not errors, errors
    for key, name in (("g1_first", "g1"), ("g1", "g1"), ("franka", "franka")):
        cost, gk, variant = got[key]
        assert variant == want[name][2] == VARIANT_STANDARD  # both robots on rollout_fused_kernel<1, true>
        assert torch.equal(cost, want[name][0]) and torch.equal(gk, want[name][1]), key
