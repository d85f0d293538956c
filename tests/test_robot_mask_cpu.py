"""The float64 robot-mask oracle (oracle/robot_mask_oracle.py) against the reference's own segmentation steps
(tests/golden/robot_mask_reference_golden.npz, made by tests/golden/make_robot_mask_golden.py): robot batch 1 and B, thresholds
0.05 and 0, a disabled link, zero / NaN / inf pixels and a camera that sees no robot.  Masks may differ only at pixels whose
margin is within 1e-5 m of the threshold; the filtered depth is where(mask, 0, depth) in both."""
import os

import numpy as np
import pytest

from oracle import robot_mask_oracle as M

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "robot_mask_reference_golden.npz")
G = np.load(GOLDEN)
CASES = sorted({k.split("/")[0] for k in G.files})


@pytest.mark.parametrize("name", CASES)
def test_oracle_vs_reference(name):
    c = {k.split("/", 1)[1]: G[k] for k in G.files if k.startswith(name + "/")}
    mask, filt, margin = M.robot_mask(c["depth"], c["K"], c["pos"], c["quat"], c["spheres"], float(c["threshold"]))
    near = np.abs(np.nan_to_num(margin, nan=1.0, posinf=1.0, neginf=-1.0)) <= 1e-5
    assert near.mean() < 1e-3
    assert not ((mask != c["mask"]) & ~near).any()
    assert np.array_equal(np.where(c["mask"], np.float32(0), c["depth"]).view(np.uint32), c["filtered"].view(np.uint32))
    if name == "no_robot":
        assert not c["mask"].any()
    else:
        assert c["mask"].sum() > 50
    if name == "invalid_pixels":
        d = c["depth"]
        assert np.isnan(d).any() and np.isinf(d).any() and (d == 0).any() and not c["mask"][~(np.isfinite(d) & (d > 0))].any()


def test_disabled_link_unmasks_its_pixels():
    on = {k.split("/", 1)[1]: G[k] for k in G.files if k.startswith("batch1_thr005/")}
    off = {k.split("/", 1)[1]: G[k] for k in G.files if k.startswith("disabled_hand/")}
    assert (off["spheres"][..., 3] == -100).sum() > (on["spheres"][..., 3] == -100).sum()
    assert M.robot_mask(off["depth"], off["K"], off["pos"], off["quat"], on["spheres"], 0.05)[0].sum() > off["mask"].sum()
