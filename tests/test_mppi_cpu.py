"""The MPPI particle stage without a GPU: the numpy oracle (oracle/mppi_oracle.py) against the reference's own MPPI iterates
(tests/golden/mppi_reference_torch.npz, written by tests/golden/make_mppi_golden.py), the C ABI table of the two kernels, and
the refusals of MPPIOpt / MultiStageOpt that need no device."""
import json
import os
import re

import numpy as np
import pytest
import torch

from oracle import mppi_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mppi_reference_torch.npz")
CASES = ("ik", "horizon", "mean_nocov", "cycling")


def golden(case):
    z = np.load(GOLDEN)
    g = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(case + "/")}
    g["config"] = json.loads(str(g["config"]))
    return g


def test_golden_covers_the_issue_cases():
    shapes = {c: golden(c)["config"] for c in CASES}
    assert shapes["ik"]["H"] == 1 and shapes["ik"]["D"] == 7 and shapes["ik"]["num_particles"] == 25
    assert shapes["horizon"]["H"] == 4 and shapes["horizon"]["gamma"] == 0.98 and shapes["horizon"]["null_act_frac"] == 0.2
    assert shapes["mean_nocov"]["sample_mode"] == "MEAN" and not shapes["mean_nocov"]["update_cov"]
    cy = golden("cycling")
    assert not cy["config"]["fixed_samples"] and cy["noise"].shape[0] == 3 and cy["actions"].shape[0] == 4  # 2 outer x 2 inner
    for c in CASES:
        assert not golden(c)["noise"][:, :, -1].any()                   # the last sampled particle is zeroed


@pytest.mark.parametrize("dtype,rtol", [(np.float32, 1e-5), (np.float64, 1e-4)])
@pytest.mark.parametrize("case", CASES)
def test_oracle_equals_reference_golden(case, dtype, rtol):
    """The oracle's outer / inner loop, sample rule and update rule reproduce every iterate of the reference's MPPI; the row
    costs of the golden run are fed back so that only the optimizer is compared."""
    g = golden(case)
    c = g["config"]
    P, H, D, Np = c["P"], c["H"], c["D"], c["num_particles"]
    k = [0]

    def cost_fn(acts):
        want = g["actions"][k[0]].reshape(P * Np, H, D)
        assert np.allclose(acts, want, rtol=rtol, atol=rtol), (k[0], np.abs(acts - want).max())
        out = g["cost"][k[0]]
        k[0] += 1
        return out
    kw = {n: c[n] for n in ("num_iters", "inner_iters", "num_particles", "init_cov", "beta", "kappa", "step_size_mean",
                            "step_size_cov", "gamma", "null_act_frac", "sample_mode", "update_cov")}
    action, recs = mo.optimize(g["x0"], g["noise"], g["lows"], g["highs"], cost_fn, dtype=dtype, **kw)
    assert len(recs) == g["actions"].shape[0]
    for i, r in enumerate(recs):
        for name in ("mean", "cov", "scale"):
            np.testing.assert_allclose(r[name], g[name][i], rtol=rtol, atol=rtol, err_msg=f"{name} at {i}")
        if c["sample_mode"] == "BEST":
            np.testing.assert_allclose(r["best"], g["best"][i], rtol=rtol, atol=rtol)
    np.testing.assert_allclose(action, g["result"], rtol=rtol, atol=rtol)
    if dtype == np.float32:       # the sample rule is the reference's to the bit
        assert np.array_equal(recs[0]["actions"].reshape(g["actions"][0].shape), g["actions"][0])


def test_particle_counts():
    assert mo.particle_counts(25, 0.0) == (25, 0, 0)
    assert mo.particle_counts(20, 0.2) == (16, 2, 2)
    assert mo.particle_counts(25, 0.3) == (18, 4, 3)
    from curobo_b200.optim import mppi_particle_counts
    for n, f in ((25, 0.0), (20, 0.2), (25, 0.3), (100, 0.05)):
        assert mppi_particle_counts(n, f) == mo.particle_counts(n, f)


def test_abi_table():
    from curobo_b200 import lib
    header = open(os.path.join(ROOT, "include", "curobo_b200.h")).read()
    for name, n_args in (("cb200_mppi_sample", 14), ("cb200_mppi_update", 18)):
        assert name in lib.EXPORTED_SYMBOLS
        m = re.search(r"int %s\(([^)]*)\);" % name, header)
        assert m, name
        assert len(m.group(1).split(",")) == n_args == len(lib._SIGS[name][0])
    assert "#define CB200_ABI_VERSION 6" in header


def test_mppi_opt_refusals():
    from curobo_b200.optim import MPPIOpt, MPPIOptCfg, MultiStageOpt
    lows, highs = -torch.ones(3), torch.ones(3)
    f = lambda a: a.sum(-1)  # noqa: E731
    for bad, what in ((dict(cov_type="SIGMA_I"), "DIAG_A"), (dict(sample_mode="SAMPLE"), "BEST or MEAN"),
                      (dict(random_mean=True), "random_mean"), (dict(squash_fn="TANH"), "CLAMP"),
                      (dict(beta=0.0), "beta"), (dict(num_particles=2, null_act_frac=1.0), "no sampled particle")):
        with pytest.raises(ValueError, match=what):
            MPPIOpt(MPPIOptCfg(**bad), 4, 1, 3, lows, highs, f, device="cuda:0")
    with pytest.raises(ValueError, match="CUDA-only"):
        MPPIOpt(MPPIOptCfg(), 4, 1, 3, lows, highs, f, device="cpu")
    with pytest.raises(ValueError, match="at least one stage"):
        MultiStageOpt([])


def test_particle_ik_preset():
    from curobo_b200.rollout import RolloutConfig
    c = RolloutConfig.particle_ik()
    assert (c.self_weight, c.scene_weight, c.scene_activation) == (50.0, 500.0, 0.01)
    assert tuple(c.pose_weight) == (1000.0, 10.0) and c.cspace_type == "position"
    assert tuple(c.cspace_weight[:2]) == (50.0, 1.0) and tuple(c.cspace_activation[:2]) == (0.001, 0.001)
    assert not c.use_sweep
