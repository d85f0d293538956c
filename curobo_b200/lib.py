"""ctypes binding of libcurobo_b200.so (the C ABI in include/curobo_b200.h).

There is NO fallback: if the library is missing it is built with nvcc; if that fails, import of any
op raises.  Nothing here computes anything on the CPU.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_LIB: Optional[C.CDLL] = None

c_f = C.c_void_p      # device float*
c_p = C.c_void_p


class CuboidSet(C.Structure):
    _fields_ = [("dims", C.c_void_p), ("inv_pose", C.c_void_p), ("enable", C.c_void_p), ("count", C.c_void_p),
                ("max_n", C.c_int32), ("num_envs", C.c_int32)]


class VoxelSet(C.Structure):
    _fields_ = [("params", C.c_void_p), ("inv_pose", C.c_void_p), ("enable", C.c_void_p), ("count", C.c_void_p),
                ("features", C.c_void_p), ("n_voxels_per_layer", C.c_int32), ("max_n", C.c_int32),
                ("num_envs", C.c_int32), ("max_dist", C.c_float), ("mip", C.c_void_p), ("mip_stride", C.c_int32)]


class MeshSet(C.Structure):
    _fields_ = [("nodes", C.c_void_p), ("triangles", C.c_void_p), ("node_offset", C.c_void_p), ("triangle_offset", C.c_void_p),
                ("dims", C.c_void_p), ("inv_pose", C.c_void_p), ("enable", C.c_void_p), ("count", C.c_void_p),
                ("max_n", C.c_int32), ("num_envs", C.c_int32)]


class RobotSizes(C.Structure):
    _fields_ = [("num_links", C.c_int32), ("num_dof", C.c_int32), ("num_spheres", C.c_int32),
                ("num_tool_frames", C.c_int32), ("num_pairs", C.c_int32), ("num_sphere_configs", C.c_int32)]


class RolloutCfg(C.Structure):
    _fields_ = [("self_weight", C.c_float), ("scene_weight", C.c_float), ("scene_activation", C.c_float),
                ("use_sweep", C.c_int32), ("use_speed_metric", C.c_int32), ("pose_weight", C.c_float * 2),
                ("pose_rotation_method", C.c_int32), ("cspace_type", C.c_int32), ("cspace_weight", C.c_float * 5),
                ("cspace_activation", C.c_float * 5), ("cspace_reg", C.c_float * 5), ("retime_weights", C.c_int32),
                ("retime_regularization_weights", C.c_int32), ("num_goalset", C.c_int32),
                ("cspace_target_weight", C.c_float), ("cspace_non_terminal_weight_factor", C.c_float)]


class SplineInput(C.Structure):
    _fields_ = [("knots", c_p), ("start_position", c_p), ("start_velocity", c_p), ("start_acceleration", c_p),
                ("start_jerk", c_p), ("goal_position", c_p), ("goal_velocity", c_p), ("goal_acceleration", c_p),
                ("goal_jerk", c_p), ("start_idx", c_p), ("goal_idx", c_p), ("traj_dt", c_p),
                ("use_implicit_goal_state", c_p), ("n_knots", C.c_int32), ("degree", C.c_int32), ("grad_knots", c_p),
                ("out_position", c_p), ("out_velocity", c_p), ("out_acceleration", c_p), ("out_jerk", c_p),
                ("out_dt", c_p)]


class DynamicsParams(C.Structure):
    _fields_ = [("link_masses_com", c_p), ("link_inertias", c_p), ("gravity", c_p)]


class RolloutIO(C.Structure):
    _fields_ = [("q", c_p), ("vel", c_p), ("acc", c_p), ("jerk", c_p), ("dt", c_p),
                ("robot_blob", c_p), ("robot_blob_host", c_p), ("robot_blob_bytes", C.c_int32),
                ("cuboids", C.POINTER(CuboidSet)), ("voxels", C.POINTER(VoxelSet)), ("env_query_idx", c_p),
                ("goal_position", c_p), ("goal_quat", c_p), ("idxs_goal", c_p),
                ("pose_axes_terminal", c_p), ("pose_axes_non_terminal", c_p),
                ("pose_tol_terminal", c_p), ("pose_tol_non_terminal", c_p),
                ("cost", c_p), ("grad_q", c_p), ("self_cost", c_p), ("scene_cost", c_p), ("pose_cost", c_p),
                ("cspace_cost", c_p), ("grad_vel", c_p), ("grad_acc", c_p), ("grad_jerk", c_p),
                ("link_pos", c_p), ("link_quat", c_p), ("robot_spheres", c_p), ("pose_goalset_idx", c_p),
                ("batch_size", C.c_int32), ("horizon", C.c_int32), ("spline", C.POINTER(SplineInput)),
                ("dynamics", C.POINTER(DynamicsParams)),
                ("cspace_target", c_p), ("idxs_cspace_target", c_p), ("cspace_target_dof_weight", c_p),
                ("sphere_configs", c_p), ("num_sphere_configs", C.c_int32), ("work_counter", c_p),
                ("meshes", C.POINTER(MeshSet)),
                ("current_position", c_p), ("current_velocity", c_p), ("idxs_current_state", c_p), ("current_state_dt", c_p)]


_I = C.c_int
_SIGS = {
    "cb200_abi_version": ([], _I),
    "cb200_last_rollout_variant": ([], _I),
    "cb200_sm_arch": ([], _I),
    "cb200_error_string": ([_I], C.c_char_p),
    "cb200_device_info": ([_I, C.POINTER(_I), C.POINTER(_I)], _I),
    "cb200_kinematics_forward_spheres": ([c_p] * 16 + [_I] * 9 + [c_p], _I),
    "cb200_kinematics_backward": ([c_p] * 22 + [_I] * 9 + [c_p], _I),
    "cb200_self_collision_distance": ([c_p] * 10 + [_I] * 8 + [c_p], _I),
    "cb200_sphere_obstacle_collision": ([c_p] * 3 + [C.POINTER(CuboidSet), C.POINTER(VoxelSet)] + [c_p] * 3 + [_I] * 4 + [c_p], _I),
    "cb200_swept_sphere_obstacle_collision": ([c_p] * 3 + [C.POINTER(CuboidSet), C.POINTER(VoxelSet)] + [c_p] * 3 + [_I, c_p] + [_I] * 4 + [c_p], _I),
    "cb200_tool_pose_distance": ([c_p] * 16 + [_I] * 5 + [c_p], _I),
    "cb200_cspace_state_cost": ([c_p] * 25 + [_I] * 6 + [c_p], _I),
    "cb200_cspace_position_cost": ([c_p] * 19 + [_I] * 4 + [c_p], _I),
    "cb200_bspline_forward": ([c_p] * 18 + [_I] * 5 + [c_p], _I),
    "cb200_bspline_single_dt": ([c_p] * 20 + [_I] * 5 + [c_p], _I),
    "cb200_bspline_backward": ([c_p] * 8 + [_I] * 5 + [c_p], _I),
    "cb200_position_clique_forward": ([c_p] * 16 + [_I] * 3 + [c_p], _I),
    "cb200_position_clique_backward": ([c_p] * 8 + [_I] * 3 + [c_p], _I),
    "cb200_acceleration_integrate": ([c_p] * 10 + [_I] * 4 + [c_p], _I),
    "cb200_lbfgs_step": ([c_p] * 8 + [C.c_float] + [_I] * 4 + [c_p] * 3 + [_I, c_p, _I, _I, c_p], _I),
    "cb200_line_search": ([c_p] * 5 + [_I, C.c_float, C.c_float] + [c_p] * 13 + [C.c_float, C.c_float] + [_I] * 5 + [c_p], _I),
    "cb200_mppi_sample": ([c_p] * 6 + [_I] * 7 + [c_p], _I),
    "cb200_mppi_update": ([c_p] * 6 + [_I] * 4 + [C.c_float] * 5 + [_I] * 2 + [c_p], _I),
    "cb200_voxel_mip_block": ([], _I),
    "cb200_voxel_mip_stride": ([c_p, _I], C.c_int64),
    "cb200_voxel_build_mip": ([C.POINTER(VoxelSet), c_p], _I),
    "cb200_rnea_forward": ([c_p] * 15 + [_I] * 4 + [c_p, c_p], _I),
    "cb200_rnea_backward": ([c_p] * 17 + [_I] * 4 + [c_p, c_p], _I),
    "cb200_pba3d": ([c_p, c_p, _I, _I, _I, _I, c_p], _I),
    "cb200_sphere_mesh_collision": ([c_p, c_p, c_p, C.POINTER(MeshSet), c_p, c_p, c_p, _I, c_p, _I, _I, _I, _I, _I, _I, c_p], _I),
    "cb200_edt_unsigned_distance": ([c_p, c_p, _I, _I, _I, C.c_float, C.c_float, c_p], _I),
    "cb200_esdf_seed_sites": ([c_p, c_p, _I, _I, _I, C.c_float, C.c_float, c_p], _I),
    "cb200_esdf_signed_distance": ([c_p, c_p, c_p, c_p, _I, _I, _I, C.c_float, C.c_float, c_p], _I),
    "cb200_esdf_seed_sites_gather": ([c_p, c_p, _I, _I, _I, C.c_float, C.c_float, C.POINTER(C.c_float), c_p], _I),
    "cb200_tsdf_integrate_depth": ([c_p, _I, _I, _I, C.c_float, C.POINTER(C.c_float), _I, c_p, c_p, c_p, c_p, _I, _I, C.c_float,
                                    C.c_float, C.c_float, c_p], _I),
    "cb200_tsdf_combined_sdf": ([c_p, c_p, c_p, C.c_longlong, C.c_float, c_p], _I),
    "cb200_segment_robot_depth": ([c_p, _I, _I, _I, c_p, c_p, c_p, c_p, _I, _I, C.c_float, c_p, c_p, c_p], _I),
    "cb200_tsdf_stamp_cuboids": ([c_p, _I, _I, _I, C.c_float, C.POINTER(C.c_float), C.c_float, C.POINTER(CuboidSet), _I, c_p], _I),
    "cb200_robot_blob_bytes": ([C.POINTER(RobotSizes)], C.c_int64),
    "cb200_pack_robot_blob": ([c_p, C.c_int64, C.POINTER(RobotSizes)] + [c_p] * 15, C.c_int64),
    "cb200_refresh_robot_spheres": ([c_p, c_p, C.c_int32, c_p, C.c_int32, c_p], _I),
    "cb200_rollout_cost_grad": ([C.POINTER(RolloutCfg), C.POINTER(RolloutIO), c_p], _I),
    "cb200_rollout_cost": ([C.POINTER(RolloutCfg), C.POINTER(RolloutIO), c_p], _I),
    "cb200_rollout_validate": ([C.POINTER(RolloutIO), c_p, C.c_int32, C.c_int32, C.c_int32, c_p], _I),
}

VARIANT_COST_ONLY = 0x10    # include/curobo_b200.h: CB200_VARIANT_COST_ONLY, or'd into cb200_last_rollout_variant()
VARIANT_VALIDATE = 0x20     # include/curobo_b200.h: CB200_VARIANT_VALIDATE

EXPORTED_SYMBOLS = tuple(_SIGS.keys())


def lib_path() -> str:
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libcurobo_b200.so")


def load() -> C.CDLL:
    """Load (building first if absent) the native library and attach argtypes."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    # rebuild when a source is newer than the library (cheap mtime check); a box without nvcc -- the GPU box
    # receives the prebuilt library -- uses what is there and fails loudly below if nothing is
    from . import build
    try:
        build.build_product()
    except RuntimeError:
        if not os.path.exists(path):
            raise
    lib = C.CDLL(path)
    for name, (args, res) in _SIGS.items():
        fn = getattr(lib, name)       # AttributeError if the symbol is missing: fail loudly
        fn.argtypes = args
        fn.restype = res
    if lib.cb200_abi_version() != 6:
        raise RuntimeError("libcurobo_b200.so ABI version mismatch")
    _LIB = lib
    return lib


class CudaCallError(RuntimeError):
    pass


def check(err: int, what: str) -> None:
    """Error convention of the reference's launch_helper (cudaGetLastError -> log_and_raise,
    curobo/_src/curobolib/backends/cuda_core_backend/launch_helper.py:13-19)."""
    if err != 0:
        msg = load().cb200_error_string(err)
        raise CudaCallError(f"{what} failed: cudaError {err} ({msg.decode() if msg else '?'})")
