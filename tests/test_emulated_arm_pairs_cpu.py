"""The paired arm build's A/B tests (tests/test_gpu_arm_pairs.py) on the emulated device of test_emulated_gpu_suite_cpu.py: the
two halves of a warp run different rows and meet on per-half barriers, so a collective that named the whole warp on a path
where the halves diverge would deadlock here, and a race between the halves' shared-memory slices is a real race."""
import pytest

from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)


@pytest.mark.parametrize("scene,n", [("cuboid", 33), ("cuboid", 8), ("none", 21), ("buried", 22)])
def test_paired_arm_build_emulated(run, monkeypatch, scene, n):  # noqa: F811
    run("test_gpu_arm_pairs", "test_paired_arm_build_matches_one_warp_build", monkeypatch, scene, n)
