"""Argument checks of cb200_rollout_cost, the cost-only fused rollout, without a GPU: they run before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

from curobo_b200 import build, lib as cblib

INVALID = 1  # cudaErrorInvalidValue


@pytest.fixture(scope="module")
def L():
    build.build_product()
    return cblib.load()


def test_cost_only_entry_point_refuses_what_it_does_not_cover(L):
    buf = np.zeros(256, np.float32)
    p = buf.ctypes.data

    def io_of(**kw):
        io = cblib.RolloutIO()
        io.q = io.cost = io.robot_blob = io.robot_blob_host = p
        io.batch_size, io.horizon = 4, 1
        for k, v in kw.items():
            setattr(io, k, v)
        return io
    cfg = cblib.RolloutCfg()
    assert L.cb200_rollout_cost(None, None, None) == INVALID
    assert L.cb200_rollout_cost(C.byref(cfg), C.byref(io_of(q=None)), None) == INVALID
    assert L.cb200_rollout_cost(C.byref(cfg), C.byref(io_of(cost=None)), None) == INVALID
    assert L.cb200_rollout_cost(C.byref(cfg), C.byref(io_of(robot_blob=None)), None) == INVALID
    sp = cblib.SplineInput()
    assert L.cb200_rollout_cost(C.byref(cfg), C.byref(io_of(spline=C.pointer(sp))), None) == INVALID
    dp = cblib.DynamicsParams()
    assert L.cb200_rollout_cost(C.byref(cfg), C.byref(io_of(dynamics=C.pointer(dp))), None) == INVALID
    swept = cblib.RolloutCfg()
    swept.use_sweep = 1
    assert L.cb200_rollout_cost(C.byref(swept), C.byref(io_of()), None) == INVALID
    # the gradient entry point keeps refusing a null grad_q
    assert L.cb200_rollout_cost_grad(C.byref(cfg), C.byref(io_of()), None) == INVALID
