"""The MPPI GPU tests (tests/test_gpu_mppi.py) on the emulated device of test_emulated_gpu_suite_cpu.py, at small sizes: the
sample kernel to the bit, the update kernel on every thread mapping, MPPIOpt against the reference's golden iterates and the
refusals.  CUDA-graph captures and the robot solves need a real GPU and are not re-run."""
import pytest

from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)

import test_gpu_mppi as g


@pytest.mark.parametrize("kw", g.SAMPLE_CASES[:3] + g.SAMPLE_CASES[4:])
def test_sample_kernel_emulated(run, kw):  # noqa: F811
    run("test_gpu_mppi", "test_sample_kernel_bit_exact", kw)


@pytest.mark.parametrize("P,Np,H,D", [(5, 25, 1, 7), (3, 25, 2, 6), (2, 25, 5, 7), (2, 64, 3, 11)])
def test_update_kernel_emulated(run, P, Np, H, D):  # noqa: F811
    run("test_gpu_mppi", "test_update_kernel_vs_oracle", P, Np, H, D, True, True)
    run("test_gpu_mppi", "test_update_kernel_vs_oracle", P, Np, H, D, False, False)


@pytest.mark.parametrize("case", g.GOLDEN_CASES)
def test_mppi_opt_golden_emulated(run, case):  # noqa: F811
    run("test_gpu_mppi", "test_mppi_opt_vs_reference_golden", case)


def test_refusals_emulated(run):  # noqa: F811
    run("test_gpu_mppi", "test_update_refusals")
