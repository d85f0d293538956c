"""`RobotSegmenter`: the reference's curobo.perception.RobotSegmenter (curobo/_src/perception/robot_segmenter.py:35-366) on this
backend.  It masks the pixels of depth images that see the robot itself, so that `DenseTSDF.integrate` does not map the robot
as an obstacle: FK (the `Kinematics` drop-in) gives the robot's spheres, then one launch (cb200_segment_robot_depth) deprojects
every pixel, moves it into the robot base frame and masks it when it lies within `distance_threshold` of a sphere.

Differences from the reference: everything runs in float32 (the reference's default `ops_dtype` is bfloat16); depth is float32
metres, the integrator's input, so there is no `depth_to_meter` and no uint16 input; plain tensors take the place of
`CameraObservation`; there is no `from_robot_file`.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from .backends import pba as pba_cu
from .kinematics import Kinematics
from .robot_model import RobotModel


class RobotSegmenter:
    """`robot`: RobotModel; `distance_threshold`: metres beyond a sphere's surface that still count as robot;
    `link_spheres`: the [n_cfg, S, 4] link-sphere tensor to read, e.g. a RolloutEngine's `link_spheres`, so that its attached
    objects are masked and its disabled links are not (configuration 0 is used).  Default: the robot model's spheres."""

    def __init__(self, robot: RobotModel, device="cuda:0", distance_threshold: float = 0.05,
                 link_spheres: Optional[torch.Tensor] = None):
        self.robot, self.device = robot, torch.device(device)
        self.distance_threshold = float(distance_threshold)
        self.kinematics = Kinematics(robot, self.device)
        if link_spheres is not None:
            self.kinematics.params.link_spheres = link_spheres
        self._shape = None

    def get_robot_mask(self, depth: torch.Tensor, intrinsics: torch.Tensor, cam_positions: torch.Tensor,
                       cam_quaternions: torch.Tensor, q: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """depth [B, H, W] float32 metres; intrinsics [B, 3, 3], cam_positions [B, 3], cam_quaternions [B, 4] (wxyz, camera ->
        robot base), the tensors `DenseTSDF.integrate` takes; q [dof] or [1 or B, dof] -> (mask bool [B, H, W], filtered float32
        [B, H, W]).  Both are buffers that the next call with the same image shape overwrites; after the first call at a shape
        a call allocates nothing and never synchronises, so it can be captured in a CUDA graph."""
        if depth.ndim != 3:
            raise ValueError(f"depth must be [batch, height, width], got {tuple(depth.shape)}")
        if q.ndim == 1:
            q = q.unsqueeze(0)
        if q.ndim != 2 or q.shape[0] not in (1, depth.shape[0]):
            raise ValueError(f"q must be [dof] or [1 or {depth.shape[0]}, dof], got {tuple(q.shape)}")
        with torch.no_grad():
            spheres = self.kinematics.compute_kinematics(q).robot_spheres      # [1 or B, 1, S, 4]
        shape = tuple(depth.shape)
        if self._shape != shape:
            self._mask = torch.empty(shape, dtype=torch.bool, device=self.device)
            self._filtered = torch.empty(shape, dtype=torch.float32, device=self.device)
            self._shape = shape
        pba_cu.launch_segment_robot_depth(depth, intrinsics, cam_positions, cam_quaternions, spheres.view(q.shape[0], -1, 4),
                                          self.distance_threshold, self._mask, self._filtered)
        return self._mask, self._filtered
