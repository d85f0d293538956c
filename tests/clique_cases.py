"""Shared seeded inputs for the position (clique) and acceleration control-space tests."""
import numpy as np


def make_case(seed, B, H, D, n_start=2, n_goal=3, implicit="mixed"):
    """implicit: False / True for every goal row, "mixed" for alternating rows (goal_idx then picks both modes)."""
    rng = np.random.default_rng(seed)
    c = dict(B=B, H=H, D=D, n=H - 4)
    c["u"] = rng.normal(size=(B, H - 4, D)).astype(np.float32)
    c["start"] = tuple((rng.normal(size=(n_start, D)) * s).astype(np.float32) for s in (1.0, 0.5, 0.3))
    c["goal"] = tuple((rng.normal(size=(n_goal, D)) * s).astype(np.float32) for s in (1.0, 0.5, 0.3))
    c["start_idx"] = rng.integers(0, n_start, B).astype(np.int32)
    c["goal_idx"] = (np.arange(B) % n_goal).astype(np.int32)
    c["traj_dt"] = rng.uniform(0.02, 0.2, n_goal).astype(np.float32)
    if implicit == "mixed":
        c["implicit"] = (np.arange(n_goal) % 2).astype(np.uint8)
    else:
        c["implicit"] = np.full(n_goal, int(implicit), np.uint8)
    c["grads"] = tuple(rng.normal(size=(B, H, D)).astype(np.float32) for _ in range(4))
    c["u_acc"] = rng.normal(size=(B, H, D)).astype(np.float32)
    c["dt_h"] = rng.uniform(0.02, 0.1, H).astype(np.float32)
    return c


# H in {8, 9, 14, 30, 34}, D in {7, 35}, batch sizes that fill no whole warp or CTA, several start / goal rows, mixed modes
CASES = [
    dict(seed=1, B=5, H=8, D=7, implicit="mixed"),
    dict(seed=2, B=3, H=8, D=7, implicit=True),
    dict(seed=3, B=7, H=9, D=7, implicit="mixed"),
    dict(seed=4, B=13, H=14, D=7, implicit=False),
    dict(seed=5, B=6, H=14, D=35, implicit="mixed"),
    dict(seed=6, B=11, H=30, D=7, implicit="mixed"),
    dict(seed=7, B=3, H=34, D=35, implicit=True),
    dict(seed=8, B=37, H=34, D=7, implicit="mixed"),
]


def case_id(kw):
    return f"H{kw['H']}-D{kw['D']}-B{kw['B']}-{kw['implicit'] if isinstance(kw['implicit'], str) else ('imp' if kw['implicit'] else 'rep')}"
