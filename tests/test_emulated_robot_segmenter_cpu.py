"""Robot segmentation (tests/test_gpu_robot_segmenter.py) on the emulated device of test_emulated_gpu_suite_cpu.py, at small
image sizes: the kernel and RobotSegmenter against the float64 oracle, the reference's outputs, the cull on adversarial tiles,
attached and disabled link spheres, and the refusals.  Graph capture needs a real GPU."""
import pytest

from test_emulated_gpu_suite_cpu import emulated_library, run  # noqa: F401  (fixtures)


@pytest.mark.parametrize("robot", ["franka", "g1_29", "g1_43"])
@pytest.mark.parametrize("per_image", [False, True])
def test_kernel_vs_oracle_emulated(run, robot, per_image):  # noqa: F811
    run("test_gpu_robot_segmenter", "test_kernel_vs_oracle", robot, per_image, 2, (40, 72))


def test_segmenter_and_reference_emulated(run):  # noqa: F811
    run("test_gpu_robot_segmenter", "test_segmenter_vs_oracle", "franka", 2, (24, 40))
    run("test_gpu_robot_segmenter", "test_reference_golden")


def test_cull_exact_on_adversarial_tiles_emulated(run):  # noqa: F811
    run("test_gpu_robot_segmenter", "test_cull_exact_on_adversarial_tiles")
    run("test_gpu_robot_segmenter", "test_cull_exact_at_one_ulp")
    run("test_gpu_robot_segmenter", "test_subnormal_depth_is_a_candidate")


def test_link_spheres_and_refusals_emulated(run):  # noqa: F811
    run("test_gpu_robot_segmenter", "test_attached_object_and_disabled_link", (72, 96))
    run("test_gpu_robot_segmenter", "test_refusals")


def test_segmented_depth_to_esdf_and_collision_checker_emulated(run):  # noqa: F811
    run("test_gpu_robot_segmenter", "test_segmented_depth_to_esdf_and_collision_checker", 0.03, (120, 160))
