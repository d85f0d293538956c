"""Generate tests/golden/cspace_position_current_state_golden.npz: outputs of the REFERENCE's own forward_cspace_position_warp
(cost/wp_cspace_position.py:232-362) with its current-state block live (state_dt > 0), executed on the CPU thread by thread
under the pure-Python Warp stand-in (oracle/warp_shim), on seeded inputs.  The fixture stores inputs and outputs;
tests/test_current_state_golden_cpu.py replays them through oracle/current_state_oracle.py, the per-operator kernel and the
fused kernels on the emulated device.  Needs the reference tree (authoring container only):

    python tests/golden/make_current_state_golden.py

Cases (Franka, D = 7):
  vel_acc        dt > 0, both regularizers, current velocity given, several current-state rows picked by idxs_current_state
  no_velocity    the same with a zero velocity buffer (what the reference passes when current_js.velocity is None)
  mixed_dt       rows with dt = 0 (plain bound) next to rows with dt > 0, horizon 3
  empty_window   current positions outside the limits: the velocity window and the limits do not intersect
  with_target    the c-space target term on at the same time
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]
import _reference_under_shim as R  # noqa: E402

R.prepare()
import warp as wp  # noqa: E402  (the stand-in)

from curobo_b200.robot_model import load_robot  # noqa: E402

OUT = {}


def A(x):
    x = np.ascontiguousarray(x)
    dtype = {np.dtype(np.float32): wp.float32, np.dtype(np.int32): wp.int32}[x.dtype]
    return wp.from_numpy(x.reshape(-1), dtype=dtype)


def case(name, rng, B, H, n_cur, dt, vel=True, outside=False, target=False, reg=(0.01, 0.01), weight=10000.0):
    m = R.ref("curobo._src.cost.wp_cspace_position")
    rm = load_robot("franka")
    D = rm.num_dof
    lim_p, lim_tau, lim_v = (np.asarray(x, np.float32) for x in (rm.position_limits, rm.effort_limits, rm.velocity_limits))
    cur_p = rng.uniform(lim_p[0] + 0.05, lim_p[1] - 0.05, size=(n_cur, D)).astype(np.float32)
    if outside:                       # beyond the limits by more than one step: empty windows on those dofs
        cur_p[:, ::2] = lim_p[1, ::2] + rng.uniform(0.3, 0.6, size=(n_cur, (D + 1) // 2)).astype(np.float32)
        cur_p[:, 1::2] = lim_p[0, 1::2] - rng.uniform(0.3, 0.6, size=(n_cur, D // 2)).astype(np.float32)
    cur_v = (rng.normal(0, 0.5, size=(n_cur, D)) if vel else np.zeros((n_cur, D))).astype(np.float32)
    idx = rng.integers(0, n_cur, size=B).astype(np.int32)
    dtv = np.asarray(dt, np.float32)
    # seeds near their current state (inside and outside the window) and across the limits
    step = rng.normal(0, 1.0, size=(B, H, D)).astype(np.float32) * lim_v[1][None, None] * np.float32(0.08)
    q = (cur_p[idx][:, None, :] + step).astype(np.float32)
    q[-1] = rng.uniform(lim_p[0] - 0.2, lim_p[1] + 0.2, size=(H, D)).astype(np.float32)
    w, act = np.array([weight, 0.0], np.float32), np.array([0.01, 0.01], np.float32)
    tgt = rng.uniform(-1, 1, size=(2, D)).astype(np.float32)
    it = (np.arange(B) % 2).astype(np.int32)
    tw = np.array([3.0 if target else 0.0], np.float32)
    dofw = rng.uniform(0.0, 1.5, D).astype(np.float32)
    regw = np.asarray(reg, np.float32)
    z = np.zeros((B, H, D), np.float32)
    outs = [A(np.zeros(B * H * D, np.float32)) for _ in range(3)]
    args = [A(q), A(z), A(tgt), A(it), A(lim_p), A(lim_tau), A(w), A(act), A(tw), A(dofw), A(regw), A(cur_p), A(cur_v), A(idx),
            A(lim_v), A(dtv)] + outs + [1, B, H, D]
    wp.launch(m.forward_cspace_position_warp, dim=B * H * D, inputs=args)
    arrays = dict(q=q, lim_p=lim_p, lim_v=lim_v, weight=w, act=act, target=tgt, idxs_target=it, target_weight=tw,
                  dof_weight=dofw, reg=regw, cur_p=cur_p, cur_v=cur_v, idxs_cur=idx, dt=dtv, has_velocity=np.uint8(vel),
                  cost=outs[0].data.reshape(B, H, D).copy(), grad_p=outs[1].data.reshape(B, H, D).copy())
    for k, v in arrays.items():
        OUT[f"{name}/{k}"] = np.asarray(v)


if __name__ == "__main__":
    rng = np.random.default_rng(21)
    case("vel_acc", rng, B=12, H=1, n_cur=3, dt=[0.05, 0.02, 0.1])
    case("no_velocity", rng, B=10, H=1, n_cur=2, dt=[0.05, 0.05], vel=False)
    case("mixed_dt", rng, B=8, H=3, n_cur=4, dt=[0.05, 0.0, 0.03, 0.0])
    case("empty_window", rng, B=8, H=1, n_cur=2, dt=[0.05, 0.08], outside=True)
    case("with_target", rng, B=10, H=2, n_cur=3, dt=[0.05, 0.0, 0.04], target=True, reg=(0.5, 0.2))
    path = os.path.join(HERE, "cspace_position_current_state_golden.npz")
    np.savez_compressed(path, **OUT)
    print(f"wrote {path}: {len(OUT)} arrays, {os.path.getsize(path) / 1024:.0f} KiB")
