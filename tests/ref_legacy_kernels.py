"""The REFERENCE's legacy trajectory kernels -- POSITION (clique) and ACCELERATION control spaces -- as a test oracle.

Same contract as tests/ref_kernels.py, whose record / replay machinery this module uses: each function runs one reference
kernel (oracle/ref_legacy_trajectory_launcher.cu, compiled from the reference's sources into
oracle/_ref/libcurobo_ref_legacy.so) when CB200_REF_RECORD is set, and otherwise replays its stored outputs from
tests/golden/ref_kernels_<test module>.npz.  Tests guard the comparison with `ref_kernels.available()`."""
import ctypes as C
import os

import torch

from ref_kernels import RECORD, ROOT, _io, _p, _stream

PATH = os.path.join(ROOT, "oracle", "_ref", "libcurobo_ref_legacy.so")

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(PATH)
    return _lib


def clique_forward(u, start, goal, start_idx, goal_idx, traj_dt, implicit, horizon):
    """start = (position, velocity, acceleration), goal = (position, velocity, acceleration)."""
    dev = u.device
    B, _, D = u.shape
    outs = [torch.zeros((B, horizon, D), dtype=torch.float32, device=dev) for _ in range(4)]
    odt = torch.zeros((B,), dtype=torch.float32, device=dev)
    if RECORD:
        err = lib().ref_clique_forward(*[_p(o) for o in outs], _p(odt), _p(u), *[_p(x) for x in start], *[_p(x) for x in goal],
                                       _p(start_idx), _p(goal_idx), _p(traj_dt), _p(implicit), B, horizon, D, _stream(dev))
        assert err == 0, err
    return _io("clique_forward", outs + [odt])


def clique_backward(grads, traj_dt, dt_idx, implicit):
    dev = grads[0].device
    B, H, D = grads[0].shape
    out = torch.zeros((B, H - 4, D), dtype=torch.float32, device=dev)
    if RECORD:
        err = lib().ref_clique_backward(_p(out), *[_p(g) for g in grads], _p(traj_dt), _p(dt_idx), _p(implicit), B, H, D,
                                        _stream(dev))
        assert err == 0, err
    return _io("clique_backward", [out])[0]


def integrate_acceleration(u, start, start_idx, traj_dt):
    """acceleration_loop_idx_rk2_kernel<float, H> for the horizons oracle/ref_legacy_trajectory_launcher.cu instantiates."""
    dev = u.device
    B, H, D = u.shape
    outs = [torch.zeros((B, H, D), dtype=torch.float32, device=dev) for _ in range(4)]
    if RECORD:
        err = lib().ref_integrate_acceleration(*[_p(o) for o in outs], _p(u), *[_p(x) for x in start], _p(start_idx),
                                               _p(traj_dt), B, H, D, _stream(dev))
        assert err == 0, err
    return _io("integrate_acceleration", outs)
