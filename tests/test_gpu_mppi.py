"""The MPPI particle stage on the GPU: cb200_mppi_sample / cb200_mppi_update against the numpy oracle (oracle/mppi_oracle.py)
on every thread mapping, MPPIOpt against the reference's own MPPI iterates (tests/golden/mppi_reference_torch.npz, and the
reference's MPPI class itself over B200RobotRollout when oracle/_ref/pyref is built), determinism of eager and graphed runs,
and the two-stage IK (MPPI then L-BFGS) as one CUDA graph."""
import json
import os

import numpy as np
import pytest
import torch

from curobo_b200.backends import optimization as optimization_cu
from curobo_b200.optim import LBFGSOpt, LBFGSOptCfg, MPPIOpt, MPPIOptCfg, MultiStageOpt
from oracle import mppi_oracle as mo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mppi_reference_torch.npz")
GOLDEN_CASES = ("ik", "horizon", "mean_nocov", "cycling")


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def close(a, b, rtol=1e-5):
    a, b = np.asarray(a), np.asarray(b)
    assert np.allclose(a, b, rtol=rtol, atol=rtol * max(float(np.abs(b).max()), 1e-30)), float(np.abs(a - b).max())


def near_tie(w, i, j):
    """Whether particles i and j of one problem carry weights within one float32 ulp of each other."""
    a, b = np.float32(w[i]), np.float32(w[j])
    return abs(float(a) - float(b)) <= float(np.spacing(max(a, b)))


def particle_index(best, actions):
    """[P] index of the particle equal to best[p] (the first such), -1 where none is."""
    hit = (actions == best[:, None]).reshape(actions.shape[0], actions.shape[1], -1).all(-1)
    return np.where(hit.any(1), hit.argmax(1), -1)


def assert_best(got, got_actions, want, want_actions, w):
    """best [P, H, D] is the particle the reference picks, or -- on a near-tie of the top two weights -- the other tied one."""
    jg, jw = particle_index(got, got_actions), particle_index(want, want_actions)
    assert (jg >= 0).all() and (jw >= 0).all()
    for p in np.nonzero(jg != jw)[0]:
        assert near_tie(w[p], jg[p], jw[p]), (p, jg[p], jw[p], w[p][[jg[p], jw[p]]])
    close(got, want)


# ------------------------------------------------------------------------------------------------ kernels
SAMPLE_CASES = [dict(P=7, Np=25, neg=0, H=1, D=7, shared=False), dict(P=5, Np=20, neg=2, H=4, D=3, shared=False),
                dict(P=6, Np=12, neg=3, H=2, D=5, shared=True), dict(P=3, Np=64, neg=0, H=30, D=7, shared=True),
                dict(P=1, Np=9, neg=1, H=3, D=2, shared=False)]


def sample_case(P, Np, neg, H, D, shared, null=None, seed=0):
    rng = np.random.default_rng(seed)
    null = Np // 10 if null is None else null
    Ns = Np - neg - null
    mean = rng.uniform(-1.5, 1.5, (P, H, D)).astype(np.float32)
    scale = rng.uniform(0.1, 1.2, (P, D)).astype(np.float32)
    noise = rng.standard_normal((1 if shared else P, Ns, H, D)).astype(np.float32)
    lows = -rng.uniform(0.5, 1.5, D).astype(np.float32)
    highs = rng.uniform(0.2, 1.5, D).astype(np.float32)
    return mean, scale, noise, lows, highs


@pytest.mark.parametrize("kw", SAMPLE_CASES, ids=lambda k: "P{P}_Np{Np}_neg{neg}_H{H}_D{D}_{s}".format(s="shared" if k["shared"] else "own", **k))
def test_sample_kernel_bit_exact(kw):
    mean, scale, noise, lows, highs = sample_case(**kw)
    P, Np, H, D = kw["P"], kw["Np"], kw["H"], kw["D"]
    lows_shift = lows.copy()
    lows_shift[0] = 0.25                                      # zero particles of dimension 0 are clamped up to the low bound
    highs_shift = np.maximum(highs, lows_shift + 0.1).astype(np.float32)
    acts = torch.full((P, Np, H, D), float("nan"), device=DEV)
    optimization_cu.launch_mppi_sample(acts, T(mean), T(scale), T(noise), T(lows_shift), T(highs_shift), kw["neg"])
    want = mo.sample(mean, scale, noise, lows_shift, highs_shift, Np, kw["neg"])
    got = acts.cpu().numpy()
    assert np.array_equal(got, want)
    clamped = (want == highs_shift) | (want == lows_shift)
    assert clamped.any() and (~clamped).any()


UPDATE_CASES = [  # (P, Np, H, D): group of 8 / 16 / 32 lanes, both sides of the group threshold (Np * V <= 2048), CTA per problem
    (37, 25, 1, 7), (20, 25, 2, 6), (11, 25, 5, 7), (9, 64, 4, 8), (5, 64, 3, 11), (3, 300, 30, 7), (2, 1024, 30, 7)]


@pytest.mark.parametrize("P,Np,H,D", UPDATE_CASES)
@pytest.mark.parametrize("update_cov,best_mode", [(True, True), (False, False)])
def test_update_kernel_vs_oracle(P, Np, H, D, update_cov, best_mode):
    rng = np.random.default_rng(P * 1000 + Np)
    acts = rng.uniform(-1.0, 1.0, (P, Np, H, D)).astype(np.float32)
    cost = rng.uniform(0.0, 3.0, (P * Np, H)).astype(np.float32)
    cost.reshape(P, Np, H)[:, 1] = cost.reshape(P, Np, H)[:, 0]      # exact ties: the lower index must win
    mean = rng.uniform(-0.5, 0.5, (P, H, D)).astype(np.float32)
    cov = rng.uniform(0.2, 1.0, (P, D)).astype(np.float32)
    g = mo.discount_factor(0.98, H)
    m, c, s, b = T(mean), T(cov), torch.zeros((P, D), device=DEV), torch.zeros((P, H, D), device=DEV)
    optimization_cu.launch_mppi_update(T(acts), T(cost), m, c if update_cov else None, s if update_cov else None,
                                       b if best_mode else None, 1.0, 0.9, 0.2, 0.01, float(g))
    o = mo.update(acts, cost, mean, cov, 1.0, 0.9, 0.2, 0.01, g, update_cov, best_mode)
    close(m.cpu().numpy(), o["mean"])
    close(c.cpu().numpy(), o["cov"])
    if update_cov:
        close(s.cpu().numpy(), o["scale"])
    else:
        assert not s.any()
    if best_mode:
        assert_best(b.cpu().numpy(), acts, o["best"], acts, o["w"])


def test_update_refusals():
    z = lambda *s: torch.zeros(s, device=DEV)  # noqa: E731
    with pytest.raises(ValueError, match="beta"):
        optimization_cu.launch_mppi_update(z(2, 3, 1, 2), z(6, 1), z(2, 1, 2), None, None, None, 0.0, 0.9, 0.2, 0.01)
    with pytest.raises(ValueError, match="cost"):
        optimization_cu.launch_mppi_update(z(2, 3, 1, 2), z(5, 1), z(2, 1, 2), None, None, None, 1.0, 0.9, 0.2, 0.01)
    with pytest.raises(ValueError, match="both"):
        optimization_cu.launch_mppi_update(z(2, 3, 1, 2), z(6, 1), z(2, 1, 2), z(2, 2), None, None, 1.0, 0.9, 0.2, 0.01)
    with pytest.raises(ValueError, match="do not fit"):
        optimization_cu.launch_mppi_sample(z(2, 3, 1, 2), z(2, 1, 2), z(2, 2), z(2, 3, 1, 2), z(2), z(2), num_neg=1)
    # no problems: nothing is launched, nothing fails
    optimization_cu.launch_mppi_sample(z(0, 3, 1, 2), z(0, 1, 2), z(0, 2), z(1, 3, 1, 2), z(2), z(2))
    optimization_cu.launch_mppi_update(z(0, 3, 1, 2), z(0, 1), z(0, 1, 2), z(0, 2), z(0, 2), z(0, 1, 2), 1.0, 0.9, 0.2, 0.01)


# ------------------------------------------------------------------------------------------------ MPPIOpt
def golden(case):
    z = np.load(GOLDEN)
    g = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(case + "/")}
    g["config"] = json.loads(str(g["config"]))
    return g


def quadratic_cost(g, P, Np, H, D):
    target, weight = T(g["target"]), T(g["weight"])

    def cost(acts):
        a = acts.view(P, Np, H, D)
        return (weight * (a - target[:, None]) ** 2).sum(-1).reshape(P * Np, H)
    return cost


def mppi_cfg(c):
    return MPPIOptCfg(**{k: c[k] for k in ("num_iters", "inner_iters", "num_particles", "init_cov", "beta", "kappa",
                                           "step_size_mean", "step_size_cov", "gamma", "null_act_frac", "sample_mode",
                                           "update_cov", "fixed_samples")})


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_mppi_opt_vs_reference_golden(case):
    """Each case of the reference's own MPPI run (sample set fed in) through MPPIOpt with a torch cost: every inner iterate
    (actions, mean, cov, scale, best) and the returned action."""
    g = golden(case)
    c = g["config"]
    P, H, D, Np = c["P"], c["H"], c["D"], c["num_particles"]
    log = []
    cost = quadratic_cost(g, P, Np, H, D)

    def cost_fn(acts):
        out = cost(acts)
        log.append((acts.clone(), out.clone()))
        return out
    opt = MPPIOpt(mppi_cfg(c), P, H, D, T(g["lows"]), T(g["highs"]), cost_fn, noise=T(g["noise"]), device=DEV)
    mean_log, cov_log, scale_log, best_log = [], [], [], []
    step = opt.step

    def recording_step(k):
        step(k)
        mean_log.append(opt.mean.clone())
        cov_log.append(opt.cov.clone())
        scale_log.append(opt.scale.clone())
        best_log.append(opt.best.clone())
    opt.step = recording_step
    res = opt.optimize(T(g["x0"])).cpu().numpy()
    assert len(log) == g["actions"].shape[0]
    for k, (acts, cst) in enumerate(log):
        a = acts.view(P, Np, H, D).cpu().numpy()
        close(a, g["actions"][k].reshape(P, Np, H, D), 1e-5)
        close(cst.cpu().numpy(), g["cost"][k], 1e-4)
        close(mean_log[k].cpu().numpy(), g["mean"][k], 1e-5)
        close(cov_log[k].cpu().numpy(), g["cov"][k], 1e-5)
        close(scale_log[k].cpu().numpy(), g["scale"][k], 1e-5)
        if c["sample_mode"] == "BEST":
            w = mo.weights(g["cost"][k], P, Np, c["beta"], mo.discount_factor(c["gamma"], H, np.float64), np.float64)
            assert_best(best_log[k].cpu().numpy(), a, g["best"][k], g["actions"][k].reshape(P, Np, H, D), w)
    close(res, g["result"], 1e-5)


def test_mppi_opt_refusals_and_defaults():
    lows, highs = -torch.ones(3, device=DEV), torch.ones(3, device=DEV)
    f = lambda a: a.sum(-1)  # noqa: E731
    for bad, what in ((dict(cov_type="SIGMA_I"), "DIAG_A"), (dict(sample_mode="SAMPLE"), "BEST or MEAN"),
                      (dict(random_mean=True), "random_mean"), (dict(squash_fn="TANH"), "CLAMP")):
        with pytest.raises(ValueError, match=what):
            MPPIOpt(MPPIOptCfg(**bad), 4, 1, 3, lows, highs, f, device=DEV)
    with pytest.raises(ValueError, match="noise must be"):
        MPPIOpt(MPPIOptCfg(), 4, 1, 3, lows, highs, f, noise=torch.zeros(1, 4, 24, 1, 2), device=DEV)
    opt = MPPIOpt(MPPIOptCfg(), 4, 1, 3, lows, highs, f, device=DEV)
    assert tuple(opt.noise.shape) == (1, 4, 25, 1, 3) and not opt.noise[:, :, -1].any() and opt.noise[:, :, :-1].abs().sum() > 0
    opt2 = MPPIOpt(MPPIOptCfg(), 4, 1, 3, lows, highs, f, device=DEV)
    assert torch.equal(opt.noise, opt2.noise)                 # seeded


def _quadratic_problem(P=64, H=2, D=7, seed=3):
    gen = torch.Generator().manual_seed(seed)
    target = (torch.rand(P, H, D, generator=gen) * 2 - 1).to(DEV)
    lows, highs = -torch.ones(D, device=DEV), torch.ones(D, device=DEV)
    x0 = (torch.rand(P, H, D, generator=gen) * 2 - 1).to(DEV) * 0.5
    return target, lows, highs, x0


def test_mppi_opt_deterministic_eager_and_graphed():
    P, H, D = 64, 2, 7
    target, lows, highs, x0 = _quadratic_problem(P, H, D)
    cfg = MPPIOptCfg(num_iters=6, inner_iters=3, fixed_samples=False, gamma=0.95, null_act_frac=0.2)
    out = torch.empty(cfg.num_particles * P, H, device=DEV)

    def cost(acts):
        a = acts.view(P, -1, H, D)
        torch.sum((a - target[:, None]) ** 2, dim=-1, out=out.view(P, -1, H))
        return out
    opt = MPPIOpt(cfg, P, H, D, lows, highs, cost, device=DEV)
    e1 = opt.optimize(x0).clone()
    e2 = opt.optimize(x0).clone()
    g1 = opt.optimize_graphed(x0).clone()
    g2 = opt.optimize_graphed(x0).clone()
    torch.cuda.synchronize()
    assert torch.equal(e1, e2) and torch.equal(e1, g1) and torch.equal(g1, g2)
    c0 = ((x0 - target) ** 2).sum((-1, -2))
    c1 = ((e1 - target) ** 2).sum((-1, -2))
    assert float((c1 < c0).float().mean()) > 0.9


# ------------------------------------------------------------------------------------------------ robot: reference MPPI, two-stage IK
def _franka_ik(P, seeds, Np, cfg, seed=5):
    from helpers import random_q
    from curobo_b200.robot_model import load_robot
    from curobo_b200.scene import CuboidData
    from curobo_b200.world import make_benchmark_cuboid_world
    from oracle import rollout_oracle as O
    rm = load_robot("franka")
    q_goal = random_q(rm, P, seed=seed) * 0.7
    _, _, gp, gq = O.fk_forward(rm, q_goal)
    cub = CuboidData.from_world(make_benchmark_cuboid_world(), DEV)
    return rm, (T(gp[:, :, None, :]), T(gq[:, :, None, :])), cub


def test_two_stage_ik_graphed_equals_eager():
    """MPPI (particle_ik weights, 25 particles) then L-BFGS (lbfgs_ik weights) on Franka against the cuboid world, problem-major
    rows: the graphed solve equals the eager one bit for bit, and L-BFGS never ends above the MPPI stage's cost."""
    from helpers import random_q
    from curobo_b200.rollout import RolloutConfig, RolloutEngine
    P, seeds, Np, n = 8, 4, 25, 4
    B, D = P * seeds, 7
    rm, (gp, gq), cub = _franka_ik(P, seeds, Np, None)
    e_mppi = RolloutEngine(rm, RolloutConfig.particle_ik(), DEV, cub)
    e_mppi.update_goal(gp, gq, torch.arange(B * Np, device=DEV, dtype=torch.int32).div(seeds * Np, rounding_mode="floor").int())
    e_lbfgs = RolloutEngine(rm, RolloutConfig.ik(), DEV, cub)
    e_lbfgs.update_goal(gp, gq, torch.arange(B * n, device=DEV, dtype=torch.int32).div(seeds * n, rounding_mode="floor").int())
    lows, highs = T(rm.position_limits[0]), T(rm.position_limits[1])

    def cost_fn(acts):
        return e_mppi.evaluate_cost(acts, with_terms=False).cost

    def cost_grad(x):
        out = e_lbfgs.evaluate_action(x.view(B * n, 1, D))
        return out.cost.view(-1), out.grad_q.view(B * n, D)
    mppi = MPPIOpt(MPPIOptCfg(), B, 1, D, lows, highs, cost_fn, device=DEV)
    lbfgs = LBFGSOpt(LBFGSOptCfg(num_iters=30), B, 1, D, lows, highs, cost_grad, DEV)
    two = MultiStageOpt([mppi, lbfgs])
    x0 = T(random_q(rm, B, seed=6)).view(B, 1, D)
    eager = two.optimize(x0).clone()
    stage1 = mppi.action.clone()
    graphed = two.optimize_graphed(x0).clone()
    graphed2 = two.optimize_graphed(x0).clone()
    torch.cuda.synchronize()
    assert torch.equal(eager, graphed) and torch.equal(graphed, graphed2)
    assert torch.equal(stage1, mppi.action)
    # both costs under the L-BFGS stage's weights: the line search only accepts improvements over its seed
    c1 = e_lbfgs.evaluate_action(stage1.view(B, 1, D).repeat_interleave(n, 0)).cost.view(B, n)[:, 0].clone()
    c2 = e_lbfgs.evaluate_action(eager.view(B, 1, D).repeat_interleave(n, 0)).cost.view(B, n)[:, 0].clone()
    assert bool((c2 <= c1).all()), (c1 - c2).min()


PYREF = os.path.join(ROOT, "oracle", "_ref", "pyref")


def _pyref_has_mppi():
    path = os.path.join(PYREF, "MANIFEST.json")
    return os.path.exists(path) and "curobo._src.optim.particle.mppi" in json.load(open(path))["modules"]


@pytest.mark.skipif(not _pyref_has_mppi(), reason="oracle/_ref/pyref without the reference's MPPI "
                    "(python oracle/build_pyref_particle.py where /root/reference exists)")
def test_mppi_opt_vs_reference_mppi_on_robot_rollout():
    """The reference's MPPI class (byte code from oracle/_ref/pyref) drives B200RobotRollout on the Franka cuboid world; MPPIOpt
    runs over the same rollout's engine (cost-only rows, no terms) with the reference's sample set.  Same best particles."""
    from test_gpu_reference_callsites import load_reference
    from helpers import random_q
    from curobo_b200.rollout import RolloutConfig
    from curobo_b200.rollout_protocol import B200RobotRollout
    load_reference()
    from curobo._src.optim.particle.mppi import MPPI, MPPICfg
    from curobo._src.optim.components.particle_opt_core import OptimizationIterationState
    from curobo._src.types.device_cfg import DeviceCfg
    P, seeds, Np = 6, 4, 25
    B, D = P * seeds, 7
    rm, (gp, gq), cub = _franka_ik(P, seeds, Np, None, seed=9)
    roll = B200RobotRollout(rm, RolloutConfig.particle_ik(), DEV, cuboid=cub)
    idx = torch.arange(B * Np, device=DEV, dtype=torch.int32).div(seeds * Np, rounding_mode="floor").int()
    roll.update_params(goal_position=gp, goal_quat=gq, idxs_goal=idx)
    mcfg = MPPICfg(num_iters=4, inner_iters=4, num_particles=Np, init_cov=1.0, beta=1.0, kappa=0.01, step_size_mean=0.9,
                   step_size_cov=0.2, gamma=1.0, null_act_frac=0.0, sample_mode="BEST", update_cov=True, num_problems=B,
                   device_cfg=DeviceCfg(device=torch.device(DEV)), sample_params=dict(fixed_samples=True, seed=23),
                   sample_per_problem=True, squash_fn="CLAMP", cov_type="DIAG_A", init_mean=torch.zeros(1, D))
    ref = MPPI(mcfg, [roll])
    core = ref._core
    core.reinitialize(torch.zeros(B, 1, D, device=DEV))
    noise = core._dist._sample_set.clone()
    x0 = T(random_q(rm, B, seed=10)).view(B, 1, D)
    with torch.no_grad():
        st = core._opt_iters(OptimizationIterationState(action=x0.clone(), exploration_action=x0.clone()))
    want = st.best_action.view(B, 1, D).clone()

    def cost_fn(acts):
        return roll.engine.evaluate_cost(acts, with_terms=False).cost
    opt = MPPIOpt(MPPIOptCfg(), B, 1, D, roll.action_bound_lows, roll.action_bound_highs, cost_fn, noise=noise, device=DEV)
    got = opt.optimize(x0)
    torch.cuda.synchronize()
    err = (got - want).abs().amax(dim=(-1, -2))
    # the reference sums the term tensors in torch, the kernel sums its terms itself: the costs, and from the second inner
    # iteration on the means, differ in the last bits, so a particle pick may flip on a near-tie of two weights; the rest agree
    same = err <= 1e-4
    assert float(same.float().mean()) >= 0.9, err.tolist()
