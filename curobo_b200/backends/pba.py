"""Drop-in for curobo._src.curobolib.backends.cuda_core_backend.pba (SURVEY.md section 8f rank 4): same function name and
argument order as `launch_pba3d` (pba.py:60-124), forwarding to the C ABI on the current stream."""
from __future__ import annotations

import torch

from .. import lib as _lib
from .tensor_checks import check_tensors, stream_ptr


def launch_pba3d(site_index: torch.Tensor, buffer: torch.Tensor, nx: int, ny: int, nz: int, m3: int = 2) -> None:
    """Exact 3-D nearest-site transform of `site_index` in place ((nx*ny*nz,) or (nx, ny, nz) int32; sites >= 0 hold
    their packed coordinates, non-sites < 0).  `buffer` (same size, int32) is the reference's scratch: checked like the
    reference checks it, not used.  `m3` is accepted for signature parity."""
    dev = site_index.device
    check_tensors(dev, torch.int32, site_index=site_index, buffer=buffer)
    n = int(nx) * int(ny) * int(nz)
    if site_index.numel() != n or buffer.numel() != n:
        raise ValueError(f"site_index / buffer must hold nx*ny*nz = {n} elements, got {site_index.numel()} / {buffer.numel()}")
    err = _lib.load().cb200_pba3d(site_index.data_ptr(), buffer.data_ptr(), int(nx), int(ny), int(nz), int(m3), stream_ptr(dev))
    _lib.check(err, "pba3d")


def launch_edt_unsigned_distance(site_index: torch.Tensor, distance: torch.Tensor, nx: int, ny: int, nz: int,
                                 voxel_size: float, empty_value: float = 1e4) -> None:
    """distance (float16, nx*ny*nz) = |voxel - nearest site| * voxel_size; `empty_value` where the grid has no site."""
    dev = site_index.device
    check_tensors(dev, torch.int32, site_index=site_index)
    check_tensors(dev, torch.float16, distance=distance)
    n = int(nx) * int(ny) * int(nz)
    if site_index.numel() != n or distance.numel() != n:
        raise ValueError(f"site_index / distance must hold nx*ny*nz = {n} elements")
    err = _lib.load().cb200_edt_unsigned_distance(site_index.data_ptr(), distance.data_ptr(), int(nx), int(ny), int(nz),
                                                  float(voxel_size), float(empty_value), stream_ptr(dev))
    _lib.check(err, "edt_unsigned_distance")


def launch_esdf_seed_sites(combined_sdf: torch.Tensor, site_index: torch.Tensor, nx: int, ny: int, nz: int, voxel_size: float,
                           truncation_distance: float) -> None:
    """site_index (int32, nx*ny*nz) from a dense SDF (float32; > 1e9 = unobserved): surface / truncation-boundary voxels become
    sites (builder_esdf.py:255-261), everything else -1."""
    dev = site_index.device
    check_tensors(dev, torch.float32, combined_sdf=combined_sdf)
    check_tensors(dev, torch.int32, site_index=site_index)
    n = int(nx) * int(ny) * int(nz)
    if site_index.numel() != n or combined_sdf.numel() != n:
        raise ValueError(f"combined_sdf / site_index must hold nx*ny*nz = {n} elements")
    err = _lib.load().cb200_esdf_seed_sites(combined_sdf.data_ptr(), site_index.data_ptr(), int(nx), int(ny), int(nz),
                                            float(voxel_size), float(truncation_distance), stream_ptr(dev))
    _lib.check(err, "esdf_seed_sites")


def launch_esdf_signed_distance(site_index: torch.Tensor, static_sdf, combined_sdf, distance: torch.Tensor, nx: int, ny: int,
                                nz: int, voxel_size: float, adjacent_skip_steps: float = 1.0) -> None:
    """distance (float16) = +-|voxel - nearest site| * voxel_size, signed like compute_esdf_from_min_tsdf_kernel
    (builder_esdf.py:410-503) from dense static / combined SDFs (float32, > 1e9 = unobserved; either may be None)."""
    dev = site_index.device
    check_tensors(dev, torch.int32, site_index=site_index)
    check_tensors(dev, torch.float16, distance=distance)
    n = int(nx) * int(ny) * int(nz)
    ptrs = []
    for name, t in (("static_sdf", static_sdf), ("combined_sdf", combined_sdf)):
        if t is not None:
            check_tensors(dev, torch.float32, **{name: t})
            if t.numel() != n:
                raise ValueError(f"{name} must hold nx*ny*nz = {n} elements")
        ptrs.append(t.data_ptr() if t is not None else None)
    if site_index.numel() != n or distance.numel() != n:
        raise ValueError(f"site_index / distance must hold nx*ny*nz = {n} elements")
    err = _lib.load().cb200_esdf_signed_distance(site_index.data_ptr(), ptrs[0], ptrs[1], distance.data_ptr(), int(nx), int(ny),
                                                 int(nz), float(voxel_size), float(adjacent_skip_steps), stream_ptr(dev))
    _lib.check(err, "esdf_signed_distance")


def launch_tsdf_integrate_depth(block_data: torch.Tensor, nx: int, ny: int, nz: int, voxel_size: float, origin,
                                intrinsics: torch.Tensor, cam_positions: torch.Tensor, cam_quaternions: torch.Tensor,
                                depth_images: torch.Tensor, depth_min: float, depth_max: float, truncation_distance: float) -> None:
    """Dense form of integrate_voxels_kernel (builder_camera_integrate.py:399-489): block_data [nx*ny*nz, 2] float16 holds
    (sum sdf * w, sum w) per voxel and is updated in place from depth_images [C, H, W] (float32, metres), intrinsics [C, 3, 3],
    cam_positions [C, 3], cam_quaternions [C, 4] (wxyz, camera -> world).  `origin` = grid centre (3 floats, host)."""
    import ctypes as C
    dev = block_data.device
    check_tensors(dev, torch.float16, block_data=block_data)
    check_tensors(dev, torch.float32, intrinsics=intrinsics, cam_positions=cam_positions, cam_quaternions=cam_quaternions,
                  depth_images=depth_images)
    n = int(nx) * int(ny) * int(nz)
    if block_data.numel() != 2 * n:
        raise ValueError(f"block_data must hold 2 * nx*ny*nz = {2 * n} elements")
    if depth_images.dim() != 3:
        raise ValueError("depth_images must be [num_cameras, height, width]")
    c, h, w = (int(v) for v in depth_images.shape)
    if intrinsics.numel() != 9 * c or cam_positions.numel() != 3 * c or cam_quaternions.numel() != 4 * c:
        raise ValueError("intrinsics / cam_positions / cam_quaternions must be [C,3,3] / [C,3] / [C,4] for C = depth_images.shape[0]")
    org = (C.c_float * 3)(*[float(v) for v in origin])
    err = _lib.load().cb200_tsdf_integrate_depth(block_data.data_ptr(), int(nx), int(ny), int(nz), float(voxel_size), org, c,
                                                 intrinsics.data_ptr(), cam_positions.data_ptr(), cam_quaternions.data_ptr(),
                                                 depth_images.data_ptr(), h, w, float(depth_min), float(depth_max),
                                                 float(truncation_distance), stream_ptr(dev))
    _lib.check(err, "tsdf_integrate_depth")



def launch_segment_robot_depth(depth_images: torch.Tensor, intrinsics: torch.Tensor, cam_positions: torch.Tensor,
                               cam_quaternions: torch.Tensor, robot_spheres: torch.Tensor, distance_threshold: float,
                               mask: torch.Tensor, filtered: torch.Tensor) -> None:
    """The robot's own pixels of depth_images [B, H, W] (float32, metres): mask (bool or uint8 [B, H, W]) = depth > 0 and the
    pixel's point within distance_threshold of a sphere of robot_spheres [1 or B, S, 4] (robot base frame); filtered (float32
    [B, H, W]) = depth with the masked pixels set to 0.  intrinsics [B, 3, 3], cam_positions [B, 3], cam_quaternions [B, 4]
    (wxyz, camera -> robot base): the tensors launch_tsdf_integrate_depth takes.  RobotSegmenter._mask_op
    (robot_segmenter.py:267-366) in one launch."""
    dev = depth_images.device
    check_tensors(dev, torch.float32, depth_images=depth_images, intrinsics=intrinsics, cam_positions=cam_positions,
                  cam_quaternions=cam_quaternions, robot_spheres=robot_spheres, filtered=filtered)
    if mask.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"mask: expected dtype torch.bool or torch.uint8, got {mask.dtype}")
    check_tensors(dev, mask.dtype, mask=mask)
    if depth_images.dim() != 3:
        raise ValueError("depth_images must be [batch, height, width]")
    b, h, w = (int(v) for v in depth_images.shape)
    if intrinsics.numel() != 9 * b or cam_positions.numel() != 3 * b or cam_quaternions.numel() != 4 * b:
        raise ValueError("intrinsics / cam_positions / cam_quaternions must be [B,3,3] / [B,3] / [B,4] for B = depth_images.shape[0]")
    if robot_spheres.dim() != 3 or robot_spheres.shape[-1] != 4 or robot_spheres.shape[0] not in (1, b):
        raise ValueError(f"robot_spheres must be [1 or {b}, num_spheres, 4], got {tuple(robot_spheres.shape)}")
    if tuple(mask.shape) != (b, h, w) or tuple(filtered.shape) != (b, h, w):
        raise ValueError(f"mask / filtered must be [{b}, {h}, {w}]")
    err = _lib.load().cb200_segment_robot_depth(depth_images.data_ptr(), b, h, w, intrinsics.data_ptr(), cam_positions.data_ptr(),
                                                cam_quaternions.data_ptr(), robot_spheres.data_ptr(), int(robot_spheres.shape[0]),
                                                int(robot_spheres.shape[1]), float(distance_threshold), mask.data_ptr(),
                                                filtered.data_ptr(), stream_ptr(dev))
    _lib.check(err, "segment_robot_depth")

def launch_tsdf_combined_sdf(block_data: torch.Tensor, static_sdf, combined_sdf: torch.Tensor, min_weight: float) -> None:
    """combined_sdf (float32) = min(sum_sdf_w / sum_w where sum_w > min_weight else 1e10, static_sdf): sample_combined_sdf
    (wp_tsdf_sample.py:22-97) for the dense grid."""
    dev = block_data.device
    check_tensors(dev, torch.float16, block_data=block_data)
    check_tensors(dev, torch.float32, combined_sdf=combined_sdf)
    n = combined_sdf.numel()
    if block_data.numel() != 2 * n:
        raise ValueError("block_data must hold two float16 per voxel of combined_sdf")
    if static_sdf is not None:
        check_tensors(dev, torch.float32, static_sdf=static_sdf)
        if static_sdf.numel() != n:
            raise ValueError("static_sdf must match combined_sdf")
    err = _lib.load().cb200_tsdf_combined_sdf(block_data.data_ptr(), None if static_sdf is None else static_sdf.data_ptr(),
                                              combined_sdf.data_ptr(), n, float(min_weight), stream_ptr(dev))
    _lib.check(err, "tsdf_combined_sdf")


def launch_esdf_seed_sites_gather(combined_sdf: torch.Tensor, site_index: torch.Tensor, nx: int, ny: int, nz: int, voxel_size: float,
                                  truncation_distance: float, origin) -> None:
    """The reference's default seeding (seed_esdf_sites_gather_kernel, builder_esdf.py:308-404) for a dense SDF on the ESDF's own
    grid: the seed rule probed at the voxel centre and half a voxel away along each axis.  Every voxel is written (-1 = no site)."""
    import ctypes as C
    dev = site_index.device
    check_tensors(dev, torch.float32, combined_sdf=combined_sdf)
    check_tensors(dev, torch.int32, site_index=site_index)
    n = int(nx) * int(ny) * int(nz)
    if combined_sdf.numel() != n or site_index.numel() != n:
        raise ValueError(f"combined_sdf / site_index must hold nx*ny*nz = {n} elements")
    org = (C.c_float * 3)(*[float(v) for v in origin])
    err = _lib.load().cb200_esdf_seed_sites_gather(combined_sdf.data_ptr(), site_index.data_ptr(), int(nx), int(ny), int(nz),
                                                   float(voxel_size), float(truncation_distance), org, stream_ptr(dev))
    _lib.check(err, "esdf_seed_sites_gather")


def launch_tsdf_stamp_cuboids(static_sdf: torch.Tensor, nx: int, ny: int, nz: int, voxel_size: float, origin,
                              truncation_distance: float, cuboids, env_idx: int = 0) -> None:
    """Dense form of stamp_sdf_kernel (builder_stamp.py:263-315) for cuboids: static_sdf (float32 [nx*ny*nz], > 1e9 = nothing
    stamped) is updated in place from `cuboids` (curobo_b200.scene.CuboidData) of environment `env_idx`."""
    import ctypes as C
    from ..scene import c_cuboid_set
    dev = static_sdf.device
    check_tensors(dev, torch.float32, static_sdf=static_sdf)
    n = int(nx) * int(ny) * int(nz)
    if static_sdf.numel() != n:
        raise ValueError(f"static_sdf must hold nx*ny*nz = {n} elements")
    cs = c_cuboid_set(cuboids, dev)
    if cs is None:
        raise ValueError("cuboids must be given")
    org = (C.c_float * 3)(*[float(v) for v in origin])
    err = _lib.load().cb200_tsdf_stamp_cuboids(static_sdf.data_ptr(), int(nx), int(ny), int(nz), float(voxel_size), org,
                                               float(truncation_distance), C.byref(cs), int(env_idx), stream_ptr(dev))
    _lib.check(err, "tsdf_stamp_cuboids")
