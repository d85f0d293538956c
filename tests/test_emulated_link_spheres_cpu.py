"""Run-time link-sphere updates (tests/test_gpu_link_spheres.py) on the emulated device of test_emulated_gpu_suite_cpu.py, at small
sizes, plus the refresh kernel against the host packer for the three shipped robots: the one bounds routine both call gives the
packer's bytes when it runs on the device."""
import dataclasses

import numpy as np
import pytest
import torch

from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)


@pytest.mark.parametrize("scenario", ["attach", "grow", "grasp", "reset"])
@pytest.mark.parametrize("robot,variant,kind,n", [("franka", "arm", "cuboid", 12), ("franka", "pairs", "esdf", 9),
                                                   ("franka", "standard", "mesh", 6), ("g1_29", "team", "esdf", 3),
                                                   ("franka-pairlist", "arm", "cuboid", 8), ("franka", "traj", "cuboid", 2)])
def test_update_equals_fresh_engine_emulated(run, monkeypatch, robot, variant, kind, n, scenario):  # noqa: F811
    run("test_gpu_link_spheres", "test_update_equals_fresh_engine", monkeypatch, robot, variant, kind, n, scenario)


def test_link_spheres_misc_emulated(run, monkeypatch):  # noqa: F811
    run("test_gpu_link_spheres", "test_per_environment_configuration", monkeypatch, 12)
    run("test_gpu_link_spheres", "test_robot_rollout_forwarding_and_in_place_writes")
    run("test_gpu_link_spheres", "test_attach_object_spheres_vs_float64_restatement", 8)
    run("test_gpu_link_spheres", "test_refusals")


@pytest.mark.parametrize("robot", ["franka", "g1_29", "g1_43"])
def test_refresh_kernel_gives_the_packer_bytes(run, robot):  # noqa: F811
    """Spheres moved, grown and disabled in three configurations: cb200_refresh_robot_spheres on a blob packed from the model gives
    the bytes cb200_pack_robot_blob packs from the modified spheres -- both bounds of every collision link bit for bit."""
    from curobo_b200.robot_model import load_robot
    from curobo_b200.rollout import pack_robot_blob
    from curobo_b200 import lib as cblib
    rm = load_robot(robot)
    rng = np.random.default_rng(7)
    ls = np.repeat(rm.link_spheres[None], 3, 0).astype(np.float32)
    ls[1, :, :3] += rng.normal(0, 0.02, ls[1, :, :3].shape).astype(np.float32)
    ls[1, :, 3] = np.where(ls[1, :, 3] >= 0, ls[1, :, 3] + rng.uniform(0, 0.05, ls.shape[1]), ls[1, :, 3]).astype(np.float32)
    ls[2, :, 3] = np.where(rng.random(ls.shape[1]) < 0.3, -100.0, ls[2, :, 3]).astype(np.float32)
    ls[0, ::7, 3] = -100.0
    rm3 = dataclasses.replace(rm, link_spheres=np.stack([rm.link_spheres] * 3))
    host = pack_robot_blob(rm3)
    dev = torch.from_numpy(host.copy())
    sph = torch.from_numpy(ls)
    L = cblib.load()
    assert L.cb200_refresh_robot_spheres(dev.data_ptr(), host.ctypes.data, int(host.shape[0]), sph.data_ptr(), 3, None) == 0
    want = pack_robot_blob(dataclasses.replace(rm, link_spheres=ls))
    assert not np.array_equal(host, want)
    assert np.array_equal(dev.numpy(), want)
