"""Host side of the fused rollout cost+gradient evaluation.

`RolloutEngine.evaluate_action(q)` is what one optimizer iteration calls: it stands where the
reference has  RobotRollout.evaluate_action -> RobotCostManager.compute_costs -> sum -> backward
(curobo/_src/rollout/rollout_robot.py:252-263; rollout/cost_manager/cost_manager_robot.py:195-286;
optim/components/gradient_opt_core.py:445-480) and returns the per-row cost and d(cost)/dq from ONE
kernel launch.  All buffers are allocated once per (B, H) (reference ownership contract,
cuda_ops/kinematics.py:27-90) so the call is CUDA-graph capturable.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np
import torch

from . import lib as _lib
from .backends.tensor_checks import check_tensors, stream_ptr
from .backends import tensor_checks as _tc
from .backends import trajectory as trajectory_cu
from .robot_model import RobotModel
from .mesh import c_mesh_set
from .scene import CuboidData, VoxelData, c_cuboid_set, c_voxel_set


@dataclass
class RolloutConfig:
    """Weights/switches of the cost terms (value semantics; a zero weight disables the term)."""
    self_weight: float = 0.0
    scene_weight: float = 0.0
    scene_activation: float = 0.0
    use_sweep: bool = False
    use_speed_metric: bool = False
    pose_weight: Optional[Sequence[float]] = None        # (position, rotation)
    pose_lie: bool = False
    cspace_type: Optional[str] = None                    # None | "position" | "state"
    cspace_weight: Sequence[float] = (0.0,) * 5
    cspace_activation: Sequence[float] = (0.0,) * 5
    cspace_reg: Sequence[float] = (0.0,) * 5
    retime_weights: bool = True
    retime_reg: bool = True
    cspace_target_weight: float = 0.0                    # needs RolloutEngine.update_cspace_target
    cspace_non_terminal_weight_factor: float = 1.0       # STATE cost only (waypoints h < H-1)

    # shipped task configs of the reference -------------------------------------------------
    @classmethod
    def ik(cls) -> "RolloutConfig":
        """content/configs/task/ik/lbfgs_ik.yml:4-37."""
        return cls(self_weight=5000.0, scene_weight=5000.0, scene_activation=0.0, pose_weight=(10000.0, 500.0),
                   cspace_type="position", cspace_weight=(5000.0, 1000.0, 0, 0, 0),
                   cspace_activation=(0.01, 0.01, 0, 0, 0))

    @classmethod
    def particle_ik(cls) -> "RolloutConfig":
        """content/configs/task/ik/particle_ik.yml:3-32, the weights of the MPPI stage of the reference's two-stage IK.
        Fields of that file RolloutConfig cannot express, at their values there: tool_pose_cfg._project_distance_to_goal
        (false), tool_pose_cfg._terminal_pose_convergence_tolerance ([1e-8, 1e-8]), tool_pose_cfg.use_grad_input (false);
        scene_collision_cfg.use_sweep (false) is `use_sweep`."""
        return cls(self_weight=50.0, scene_weight=500.0, scene_activation=0.01, pose_weight=(1000.0, 10.0),
                   cspace_type="position", cspace_weight=(50.0, 1.0, 0, 0, 0), cspace_activation=(0.001, 0.001, 0, 0, 0))

    @classmethod
    def retarget_ik(cls) -> "RolloutConfig":
        """content/configs/task/ik/lbfgs_retarget_ik.yml:3-38, the local IK of motion retargeting: with a current state
        (RolloutEngine.update_current_state) the POSITION cost limits each step to the velocity window and regularizes the
        implied velocity and acceleration with `cspace_reg[0]` / `cspace_reg[1]`.  The file's pose convergence tolerance
        (1e-8, 1e-8) is update_goal(terminal_tol=...)."""
        return cls(self_weight=10000.0, scene_weight=10000.0, scene_activation=0.0, pose_weight=(1000.0, 100.0),
                   cspace_type="position", cspace_weight=(10000.0, 0.0, 0, 0, 0), cspace_activation=(0.01, 0.01, 0, 0, 0),
                   cspace_reg=(0.01, 0.01, 0, 0, 0))

    @classmethod
    def trajopt(cls) -> "RolloutConfig":
        """content/configs/task/trajopt/lbfgs_bspline_trajopt.yml:40-90."""
        return cls(self_weight=10000.0, scene_weight=100000.0, scene_activation=0.0025, use_sweep=True,
                   use_speed_metric=True, pose_weight=(1000000.0, 100000.0), cspace_type="state",
                   cspace_weight=(10000.0, 10000.0, 100.0, 50.0, 100.0), cspace_activation=(0.01,) * 5,
                   cspace_reg=(1000.0, 10000.0, 5.0, 0.0, 10000.0))

    @classmethod
    def mpc(cls) -> "RolloutConfig":
        """content/configs/task/mpc/lbfgs_mpc.yml:4-52 (c-space target term at weight 1000, 0.05 on non-terminal
        waypoints; bound weights not retimed, regularisation weights retimed)."""
        return cls(self_weight=100000.0, scene_weight=10000.0, scene_activation=0.01, use_sweep=True,
                   use_speed_metric=True, pose_weight=(5000.0, 200.0), cspace_type="state",
                   cspace_weight=(1000.0, 1000.0, 1000.0, 100.0, 0.0), cspace_activation=(0.01,) * 5,
                   cspace_reg=(0.01, 10000.0, 10.0, 0.0, 0.0), retime_weights=False, retime_reg=True,
                   cspace_target_weight=1000.0, cspace_non_terminal_weight_factor=0.05)

    def to_oracle_cfg(self, num_tool_frames: int) -> dict:
        d = dict(self_weight=self.self_weight, scene_weight=self.scene_weight, scene_eta=self.scene_activation,
                 sweep=self.use_sweep, speed_metric=self.use_speed_metric, pose_lie=self.pose_lie,
                 cspace_type=self.cspace_type, cspace_weight=list(self.cspace_weight),
                 cspace_activation=list(self.cspace_activation), cspace_reg=list(self.cspace_reg),
                 retime_weights=self.retime_weights, retime_reg=self.retime_reg,
                 cspace_target_weight=self.cspace_target_weight,
                 cspace_non_terminal_weight_factor=self.cspace_non_terminal_weight_factor)
        if self.pose_weight is not None:
            d["pose_weight"] = list(self.pose_weight)
        return d


@dataclass
class RolloutOutput:
    cost: torch.Tensor                 # [B,H] sum of all terms per row
    grad_q: torch.Tensor               # [B,H,D]
    self_cost: torch.Tensor            # [B,H]
    scene_cost: torch.Tensor           # [B,H,S]
    pose_cost: torch.Tensor            # [B,H,2L]
    cspace_cost: torch.Tensor          # [B,H,D]
    grad_vel: Optional[torch.Tensor] = None
    grad_acc: Optional[torch.Tensor] = None
    grad_jerk: Optional[torch.Tensor] = None
    link_pos: Optional[torch.Tensor] = None
    link_quat: Optional[torch.Tensor] = None
    robot_spheres: Optional[torch.Tensor] = None
    pose_goalset_idx: Optional[torch.Tensor] = None
    grad_knots: Optional[torch.Tensor] = None   # [B,n_knots,D] (evaluate_knots only)
    grad_u: Optional[torch.Tensor] = None       # [B,H-4,D] (evaluate_positions only)


def pack_robot_blob(rm: RobotModel) -> np.ndarray:
    """Robot constants -> one byte blob (layout: curobo_b200/csrc/cb200_blob.h), packed by the C helper."""
    L = _lib.load()
    ls = rm.link_spheres if rm.link_spheres.ndim == 3 else rm.link_spheres[None]     # [n_cfg, S, 4]
    sz = _lib.RobotSizes(rm.num_links, rm.num_dof, rm.num_spheres, rm.num_tool_frames, int(rm.collision_pairs.shape[0]),
                         int(ls.shape[0]))
    nbytes = L.cb200_robot_blob_bytes(C.byref(sz))
    if nbytes <= 0:
        raise ValueError(f"robot does not fit the blob format (code {nbytes}); links <= 64 required")
    out = np.zeros(nbytes, np.uint8)

    def p(a, dt):
        a = np.ascontiguousarray(a, dtype=dt)
        keep.append(a)
        return a.ctypes.data
    keep = []
    n = L.cb200_pack_robot_blob(
        out.ctypes.data, nbytes, C.byref(sz), p(rm.fixed_transforms, np.float32), p(rm.link_map, np.int16),
        p(rm.joint_map, np.int16), p(rm.joint_map_type, np.int8), p(rm.joint_offset_map, np.float32),
        p(rm.tool_frame_map, np.int16), p(ls, np.float32), p(rm.link_sphere_idx_map, np.int16),
        p(rm.sphere_padding, np.float32), p(rm.collision_pairs, np.int16), p(rm.position_limits, np.float32),
        p(rm.velocity_limits, np.float32), p(rm.acceleration_limits, np.float32), p(rm.jerk_limits, np.float32),
        p(rm.effort_limits, np.float32))
    if n <= 0:
        raise ValueError(f"cb200_pack_robot_blob rejected the robot model (code {n})")
    return out[:n]


def _quat_mul(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Hamilton product of wxyz quaternions [..., 4]."""
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack((aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw), -1)


def _quat_rotate(q: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """Rotate points v [..., 3] by unit wxyz quaternions q [..., 4]: v + 2 w (u x v) + 2 u x (u x v)."""
    w, u = q[..., :1], q[..., 1:]
    t = 2.0 * torch.linalg.cross(u, v, dim=-1)
    return v + w * t + torch.linalg.cross(u, t, dim=-1)


class RolloutEngine:
    """`mesh` (curobo_b200.mesh.MeshData): triangle-mesh obstacles, evaluated inside the fused kernels next to the cuboids and
    the ESDF grids.  In-place updates of its `inv_pose` / `enable` tensors take effect on the next call; a replaced MeshData
    needs refresh_world().  Mesh scenes support every schedule except `evaluate_knots(in_kernel_spline=True)` and
    `attach_dynamics(fused=True)`, which raise ValueError.

    `link_spheres` [n_cfg, S, 4] (device, float32) are the robot's collision spheres in their link frames, one set per sphere
    configuration (rows pick theirs through env_query_idx when n_cfg > 1); `reference_link_spheres` keeps the model's.  The
    update_link_spheres / disable_link_spheres / enable_link_spheres / reset_link_spheres / attach_object_spheres calls (the
    reference's KinematicsParams and AttachmentManager calls) write `link_spheres` and refresh the packed robot constants on the
    device in one launch (cb200_refresh_robot_spheres): the broad-phase bounds are rebuilt over the new spheres, so the next
    evaluation equals, bit for bit, that of an engine built from the modified model.  The device blob keeps its address, so CUDA
    graphs captured before an update see it on their next replay without recapture."""

    def __init__(self, robot: RobotModel, cfg: RolloutConfig, device="cuda:0",
                 cuboid: Optional[CuboidData] = None, voxel: Optional[VoxelData] = None,
                 store_fk_outputs: bool = False, use_voxel_mip: bool = False, mesh=None):
        self.robot, self.cfg, self.device = robot, cfg, torch.device(device)
        _tc.require_cuda(self.device, "RolloutEngine is CUDA-only (sm_90a); there is no CPU path")
        self._lib = _lib.load()
        self._blob_host = pack_robot_blob(robot)
        self._blob = torch.from_numpy(self._blob_host.copy()).to(self.device)
        # link-sphere configurations (attached objects per environment): rows pick theirs through env_query_idx when n_cfg > 1;
        # configuration 0 is also the blob's staged set
        ls = robot.link_spheres if robot.link_spheres.ndim == 3 else robot.link_spheres[None]
        self.link_spheres = torch.from_numpy(np.ascontiguousarray(ls, np.float32)).to(self.device)
        self.reference_link_spheres = self.link_spheres.clone()
        self._link_spheres_version = self.link_spheres._version
        self._cs_target = None
        self._current_state = None
        self.cuboid, self.voxel, self.mesh = cuboid, voxel, mesh
        self.use_voxel_mip = use_voxel_mip
        self.refresh_world()
        self.store_fk_outputs = store_fk_outputs
        self._B = self._H = -1
        self._goal = None
        self._ccfg = self._make_ccfg(1)
        self._effort_cost = None
        self._dyn_params = None
        # row ticket counter of the humanoid kernel (zero between launches; this engine's launches are stream ordered)
        self._work_counter = torch.zeros(2, dtype=torch.int32, device=self.device)

    def attach_dynamics(self, dynamics, effort_limits=None, fused: bool = False) -> None:
        """Make the STATE c-space cost dynamics-aware (SURVEY.md 8f rank 3): after the fused launch, tau = RNEA(q, qd, qdd) is
        evaluated for every row and the effort channel of the STATE cost -- bound hinge (cspace_weight[4], cspace_activation[4]),
        squared-L2 (cspace_reg[3]) and the energy term (cspace_reg[4]) -- is added to cost / cspace_cost, its gradient to
        grad_q / grad_vel / grad_acc through the RNEA adjoint (curobo_b200.dynamics.DynamicsStateCost: three more launches).
        The fused kernel evaluates those terms with tau = 0, where they vanish (what the reference does without
        `compute_inverse_dynamics`, transition/robot_state_transition.py:380-396), so nothing is counted twice.
        Applies to evaluate_action with vel / acc / jerk / dt given; `dynamics` is a curobo_b200.dynamics.Dynamics."""
        from .dynamics import DynamicsStateCost
        if self.cfg.cspace_type != "state":
            raise ValueError("attach_dynamics needs the STATE c-space cost")
        rm = self.robot
        # fused = the trajectory kernel evaluates RNEA, the effort terms and the RNEA adjoint for its own rows (swept mode;
        # effort limits = the robot's, which are part of the packed robot blob); otherwise -- and for custom limits or
        # discrete mode -- the same terms are added by three more launches after the fused one.  Default: the host
        # composition, measured faster on an H100 (MPC 1024 x 30: 0.53 ms vs 0.55 ms in-kernel, plain kernel 0.34 ms).
        self._dyn_params = None
        if fused and effort_limits is None and self.cfg.use_sweep:
            m = dynamics._model       # (fixed, masses_com, inertias, joint types, joint map, link map, offsets, gravity, ...)
            self._dyn_keepalive = (m[1], m[2], m[7])
            self._dyn_params = _lib.DynamicsParams(m[1].data_ptr(), m[2].data_ptr(), m[7].data_ptr())
            self._effort_cost = None
            return
        w = [0.0, 0.0, 0.0, 0.0, float(self.cfg.cspace_weight[4])]
        reg = [0.0, 0.0, 0.0, float(self.cfg.cspace_reg[3]), float(self.cfg.cspace_reg[4])]
        lim = dict(p=rm.position_limits, v=rm.velocity_limits, a=rm.acceleration_limits, j=rm.jerk_limits,
                   tau=rm.effort_limits if effort_limits is None else effort_limits)
        self._effort_cost = DynamicsStateCost(dynamics, lim, w, list(self.cfg.cspace_activation), reg,
                                              retime_weights=self.cfg.retime_weights,
                                              retime_regularization_weights=self.cfg.retime_reg)

    def refresh_world(self) -> None:
        """Re-read the obstacle holders (cuboids, ESDF grids, meshes); call after the ESDF values (or obstacle tensors) were
        replaced or updated in place.  With `use_voxel_mip=True` (opt-in) it rebuilds the ESDF lower-bound pyramid level (one tiny launch) that
        lets discrete collision skip the corner fetches of samples that are provably inactive.  Exact while the level
        matches the grid: torch-side updates of `features` are detected (version stamp; the level is rebuilt on the next
        call), updates through raw pointers by foreign kernels are not -- call this after each of those."""
        if self.voxel is not None and self.use_voxel_mip:
            from .scene import build_voxel_mip
            build_voxel_mip(self.voxel)
        self._cs = c_cuboid_set(self.cuboid, self.device)
        self._vs = c_voxel_set(self.voxel, self.device)
        self._ms = c_mesh_set(self.mesh, self.device)
        if self.voxel is not None and not self.use_voxel_mip and self._vs is not None:
            self._vs.mip, self._vs.mip_stride = None, 0

    # -- link spheres (KinematicsParams.update_link_spheres & co., kinematics_params.py:493-595) -----------------------------
    def refresh_link_spheres(self) -> None:
        """Re-read `link_spheres` into the packed robot constants on the device (one launch on the current stream: configuration
        0 into the blob's sphere section, broad-phase bounds of every collision link rebuilt over all configurations).  The
        methods below call it.  Eager evaluations also pick up in-place writes to `link_spheres` by themselves (version
        stamp); a CUDA graph does not -- after writing the tensor yourself, call this before replaying, or capture this call
        in the graph."""
        ls = self.link_spheres
        err = self._lib.cb200_refresh_robot_spheres(self._blob.data_ptr(), self._blob_host.ctypes.data,
                                                    int(self._blob_host.shape[0]), ls.data_ptr(), int(ls.shape[0]),
                                                    stream_ptr(self.device))
        _lib.check(err, "refresh_robot_spheres")
        self._link_spheres_version = ls._version

    def _sphere_index(self, link_name: str) -> torch.Tensor:
        """Sphere slots of `link_name` (KinematicsParams.get_sphere_index_from_link_name)."""
        rm = self.robot
        if link_name not in rm.link_names:
            raise ValueError(f"unknown link {link_name!r}")
        idx = np.nonzero(rm.link_sphere_idx_map == rm.link_names.index(link_name))[0]
        if idx.size == 0:
            raise ValueError(f"link {link_name!r} has no collision spheres")
        return torch.as_tensor(idx, dtype=torch.long, device=self.device)

    def _config_index(self, config_idx: int) -> int:
        n = int(self.link_spheres.shape[0])
        if not 0 <= int(config_idx) < n:
            raise ValueError(f"config_idx {config_idx} out of range: the engine has {n} sphere configuration(s)")
        return int(config_idx)

    def update_link_spheres(self, link_name: str, spheres: torch.Tensor, start_sph_idx: int = 0,
                            config_idx: Optional[int] = None) -> None:
        """Write spheres [k, 4] (x, y, z, r in the link frame; r < 0 disables a sphere) into slots start_sph_idx ..
        start_sph_idx + k - 1 of `link_name`, in configuration `config_idx` (None: every configuration), then refresh."""
        idx = self._sphere_index(link_name)
        check_tensors(self.device, torch.float32, spheres=spheres)
        if spheres.ndim != 2 or spheres.shape[1] != 4:
            raise ValueError(f"spheres must be [k, 4], got {tuple(spheres.shape)}")
        k = int(spheres.shape[0])
        if start_sph_idx < 0 or start_sph_idx + k > idx.numel():
            raise ValueError(f"link {link_name!r} has {idx.numel()} sphere slots; cannot write {k} from slot {start_sph_idx}")
        idx = idx[start_sph_idx:start_sph_idx + k]
        if config_idx is None:
            self.link_spheres[:, idx, :] = spheres
        else:
            self.link_spheres[self._config_index(config_idx), idx, :] = spheres
        self.refresh_link_spheres()

    def get_link_spheres(self, link_name: str, config_idx: int = 0) -> torch.Tensor:
        """Spheres [n, 4] of `link_name` in configuration `config_idx` (a copy)."""
        return self.link_spheres[self._config_index(config_idx), self._sphere_index(link_name), :]

    def disable_link_spheres(self, link_name: str) -> None:
        """Radius -100 for every sphere of `link_name` in every configuration (MotionPlanner.disable_link_collision)."""
        self.link_spheres[:, self._sphere_index(link_name), 3] = -100.0
        self.refresh_link_spheres()

    def enable_link_spheres(self, link_name: str) -> None:
        """Radii of `link_name` back to the model's in every configuration; centres are left as they are."""
        idx = self._sphere_index(link_name)
        self.link_spheres[:, idx, 3] = self.reference_link_spheres[:, idx, 3]
        self.refresh_link_spheres()

    def reset_link_spheres(self, link_name: str) -> None:
        """Spheres (centres and radii) of `link_name` back to the model's in every configuration."""
        idx = self._sphere_index(link_name)
        self.link_spheres[:, idx, :] = self.reference_link_spheres[:, idx, :]
        self.refresh_link_spheres()

    def attach_object_spheres(self, spheres: torch.Tensor, link_name: str = "attached_object",
                              joint_position: Optional[torch.Tensor] = None, object_pose: Optional[torch.Tensor] = None) -> None:
        """AttachmentManager.update (collision/attachment_manager.py:102-179) as one call: spheres [k, 4] fitted to the object,
        in the object frame, become the spheres of `link_name`, one environment per sphere configuration.

        joint_position [n_env, D]: the grasp configuration of each environment; object_pose [n_env or 1, 7] (x, y, z, qw, qx, qy,
        qz): the object's pose in the robot base frame.  With object_pose, environment i gets the centres mapped by
        obj_to_link = ee_pose(joint_position[i])^-1 * object_pose[i], ee_pose being the first tool frame's pose from the
        forward kinematics (joint_position is then required); without it the centres are taken as link-frame centres.  The
        link's slots past k get radius -100 (disabled).  Environment i is written into configuration i, then the blob is
        refreshed once.  Per-environment attachment needs an engine built with at least n_env sphere configurations (a model
        whose link_spheres is [n_cfg, S, 4]); rows pick theirs through env_query_idx.  Sphere fitting stays with the caller."""
        idx = self._sphere_index(link_name)
        dev = self.device
        check_tensors(dev, torch.float32, spheres=spheres)
        if spheres.ndim != 2 or spheres.shape[1] != 4:
            raise ValueError(f"spheres must be [k, 4], got {tuple(spheres.shape)}")
        k, n_slots = int(spheres.shape[0]), int(idx.numel())
        if k > n_slots:
            raise ValueError(f"{k} spheres but link {link_name!r} only has {n_slots} sphere slots")
        n_env = 1
        if joint_position is not None:
            check_tensors(dev, torch.float32, joint_position=joint_position)
            if joint_position.ndim != 2 or joint_position.shape[1] != self.robot.num_dof:
                raise ValueError(f"joint_position must be [n_env, {self.robot.num_dof}], got {tuple(joint_position.shape)}")
            n_env = int(joint_position.shape[0])
        if n_env > int(self.link_spheres.shape[0]):
            raise ValueError(f"{n_env} environments but the engine has {int(self.link_spheres.shape[0])} sphere configuration(s)")
        centres = spheres[:, :3].expand(n_env, k, 3)
        if object_pose is not None:
            if joint_position is None:
                raise ValueError("object_pose needs joint_position (the grasp configuration the end-effector pose comes from)")
            check_tensors(dev, torch.float32, object_pose=object_pose)
            if object_pose.ndim != 2 or object_pose.shape[1] != 7 or object_pose.shape[0] not in (1, n_env):
                raise ValueError(f"object_pose must be [{n_env} or 1, 7], got {tuple(object_pose.shape)}")
            from .kinematics import Kinematics
            # one sphere configuration index per row: with several configurations the FK kernel reads env_query_idx[row]
            st = Kinematics(self.robot, dev).compute_kinematics(joint_position,
                                                                torch.zeros(n_env, dtype=torch.int32, device=dev))
            ee_p, ee_q = st.tool_pose_position[:, 0, 0], st.tool_pose_quaternion[:, 0, 0]       # [n_env, 3], [n_env, 4]
            ee_qi = ee_q * torch.tensor([1.0, -1.0, -1.0, -1.0], device=dev)
            op, oq = object_pose[:, :3].expand(n_env, 3), object_pose[:, 3:].expand(n_env, 4)
            rel_q = _quat_mul(ee_qi, oq)
            rel_p = _quat_rotate(ee_qi, op - ee_p)
            centres = _quat_rotate(rel_q[:, None, :].expand(n_env, k, 4), centres) + rel_p[:, None, :]
        env = torch.zeros((n_env, n_slots, 4), dtype=torch.float32, device=dev)
        env[:, :, 3] = -100.0
        env[:, :k, :3] = centres
        env[:, :k, 3] = spheres[:, 3]
        self.link_spheres[:n_env, idx, :] = env
        self.refresh_link_spheres()

    def detach_object_spheres(self, link_name: str = "attached_object") -> None:
        """The attached object's spheres off again: reset_link_spheres(link_name)."""
        self.reset_link_spheres(link_name)

    # -- configuration ------------------------------------------------------------------------
    def _make_ccfg(self, num_goalset: int) -> _lib.RolloutCfg:
        c = self.cfg
        cc = _lib.RolloutCfg()
        cc.self_weight, cc.scene_weight, cc.scene_activation = c.self_weight, c.scene_weight, c.scene_activation
        cc.use_sweep, cc.use_speed_metric = int(c.use_sweep), int(c.use_speed_metric)
        pw = c.pose_weight if c.pose_weight is not None else (0.0, 0.0)
        cc.pose_weight[0], cc.pose_weight[1] = float(pw[0]), float(pw[1])
        cc.pose_rotation_method = 1 if c.pose_lie else 0
        cc.cspace_type = {None: 0, "position": 1, "state": 2}[c.cspace_type]
        for i in range(5):
            cc.cspace_weight[i] = float(c.cspace_weight[i]) if i < len(c.cspace_weight) else 0.0
            cc.cspace_activation[i] = float(c.cspace_activation[i]) if i < len(c.cspace_activation) else 0.0
            cc.cspace_reg[i] = float(c.cspace_reg[i]) if i < len(c.cspace_reg) else 0.0
        cc.retime_weights, cc.retime_regularization_weights = int(c.retime_weights), int(c.retime_reg)
        cc.num_goalset = num_goalset
        cc.cspace_target_weight = float(c.cspace_target_weight)
        cc.cspace_non_terminal_weight_factor = float(c.cspace_non_terminal_weight_factor)
        return cc

    def update_cspace_target(self, target: torch.Tensor, idxs_target: Optional[torch.Tensor] = None,
                             dof_weight: Optional[torch.Tensor] = None) -> None:
        """C-space target of the cost (`target_joint_position [n, D]`, `idxs_target_joint_position [B]` int32,
        `cspace_target_dof_weight [D]`; cost/cost_cspace_state.py, wp_cspace_state.py:84-89,220-226).  Read when
        cfg.cspace_target_weight > 0."""
        dev, D = self.device, self.robot.num_dof
        check_tensors(dev, torch.float32, cspace_target=target)
        if target.ndim != 2 or target.shape[1] != D:
            raise ValueError(f"cspace target must be [n, {D}], got {tuple(target.shape)}")
        if idxs_target is not None:
            check_tensors(dev, torch.int32, idxs_cspace_target=idxs_target)
        if dof_weight is not None:
            check_tensors(dev, torch.float32, cspace_target_dof_weight=dof_weight)
            if tuple(dof_weight.shape) != (D,):
                raise ValueError(f"cspace_target_dof_weight must be [{D}]")
        self._cs_target = (target, idxs_target, dof_weight)

    def update_current_state(self, position: torch.Tensor, velocity: Optional[torch.Tensor] = None,
                             dt: Optional[torch.Tensor] = None, idxs: Optional[torch.Tensor] = None) -> None:
        """Current state of the POSITION c-space cost (velocity-aware IK; GoalRegistry.current_js / idxs_current_js /
        current_state_dt, cost/wp_cspace_position.py:299-356): `position` [n, D], `velocity` [n, D] (None = zero), `dt` [n]
        (required), `idxs` [B] int32 rows per seed (None = row 0), every entry in [0, n): like idxs_cspace_target, the indices are not
        range-checked on the device (reading them back would synchronise), and an index outside the rows reads past the buffers.  Rows with dt > 0 bound every waypoint of their seeds to
        the window one step of dt reaches from `position` and add the implied velocity / acceleration regularizers
        (cfg.cspace_reg[0], cfg.cspace_reg[1]); rows with dt <= 0 get the plain bound.  The tensors are read at every call,
        so updating them in place needs no CUDA-graph recapture.  Other c-space types ignore the current state."""
        dev, D = self.device, self.robot.num_dof
        if dt is None:
            raise ValueError("update_current_state needs dt [n] (current_state_dt)")
        check_tensors(dev, torch.float32, current_position=position, current_state_dt=dt)
        if position.ndim != 2 or position.shape[1] != D:
            raise ValueError(f"current position must be [n, {D}], got {tuple(position.shape)}")
        n = position.shape[0]
        if tuple(dt.shape) != (n,):
            raise ValueError(f"current_state_dt must be [{n}], got {tuple(dt.shape)}")
        if velocity is not None:
            check_tensors(dev, torch.float32, current_velocity=velocity)
            if tuple(velocity.shape) != (n, D):
                raise ValueError(f"current velocity must be [{n}, {D}], got {tuple(velocity.shape)}")
        if idxs is not None:
            check_tensors(dev, torch.int32, idxs_current_state=idxs)
            if idxs.ndim != 1:
                raise ValueError("idxs_current_state must be [B]")
        self._current_state = (position, velocity, dt, idxs)

    def clear_current_state(self) -> None:
        """Back to the plain POSITION cost (no velocity window, no regularizers)."""
        self._current_state = None

    def setup_batch_tensors(self, batch: int, horizon: int) -> None:
        """Allocate every output once per (B, H) -- never inside evaluate_action."""
        rm, dev = self.robot, self.device
        z = lambda *s, dt=torch.float32: torch.zeros(s, dtype=dt, device=dev)  # noqa: E731
        D, S, Lt = rm.num_dof, rm.num_spheres, rm.num_tool_frames
        self.out = RolloutOutput(cost=z(batch, horizon), grad_q=z(batch, horizon, D), self_cost=z(batch, horizon),
                                 scene_cost=z(batch, horizon, S), pose_cost=z(batch, horizon, 2 * Lt),
                                 cspace_cost=z(batch, horizon, D))
        if self.cfg.cspace_type == "state":
            self.out.grad_vel, self.out.grad_acc, self.out.grad_jerk = (z(batch, horizon, D) for _ in range(3))
        if self.store_fk_outputs:
            self.out.link_pos, self.out.link_quat = z(batch, horizon, Lt, 3), z(batch, horizon, Lt, 4)
            self.out.robot_spheres = z(batch, horizon, S, 4)
            self.out.pose_goalset_idx = z(batch, horizon, Lt, dt=torch.int32)
        self._B, self._H = batch, horizon

    def update_goal(self, goal_position: torch.Tensor, goal_quat: torch.Tensor, idxs_goal: torch.Tensor,
                    terminal_axes=None, non_terminal_axes=None, terminal_tol=None, non_terminal_tol=None) -> None:
        """goal_* [G, L, n_goalset, 3|4] (quat wxyz), idxs_goal [B] int32 (GoalRegistry rows)."""
        dev = self.device
        check_tensors(dev, torch.float32, goal_position=goal_position, goal_quat=goal_quat)
        check_tensors(dev, torch.int32, idxs_goal=idxs_goal)
        Lt = self.robot.num_tool_frames
        if goal_position.ndim != 4 or goal_position.shape[1] != Lt or goal_quat.shape[:3] != goal_position.shape[:3]:
            raise ValueError("goal tensors must be [G, num_tool_frames, n_goalset, 3|4]")
        extra = {}
        for name, t, shape in (("terminal_axes", terminal_axes, (Lt, 6)), ("non_terminal_axes", non_terminal_axes, (Lt, 6)),
                               ("terminal_tol", terminal_tol, (Lt, 2)), ("non_terminal_tol", non_terminal_tol, (Lt, 2))):
            if t is not None:
                check_tensors(dev, torch.float32, **{name: t})
                if tuple(t.shape) != shape:
                    raise ValueError(f"{name} must have shape {shape}")
            extra[name] = t
        self._goal = (goal_position, goal_quat, idxs_goal, extra)
        self._ccfg = self._make_ccfg(int(goal_position.shape[2]))

    # -- the hot call --------------------------------------------------------------------------
    def evaluate_action(self, q: torch.Tensor, vel=None, acc=None, jerk=None, dt=None,
                        env_query_idx: Optional[torch.Tensor] = None) -> RolloutOutput:
        io, B, H = self._state_io(q, vel, acc, jerk, dt)
        out = self._launch(io, B, H, env_query_idx)
        if self._effort_cost is not None and vel is not None and acc is not None and jerk is not None and dt is not None:
            c, gp, gv, ga, _, _ = self._effort_cost.evaluate(q, vel, acc, jerk, dt)
            out.cspace_cost.add_(c)
            out.cost.add_(c.sum(-1))
            out.grad_q.add_(gp)
            out.grad_vel.add_(gv)
            out.grad_acc.add_(ga)
        return out

    def evaluate_cost(self, q: torch.Tensor, vel=None, acc=None, jerk=None, dt=None,
                      env_query_idx: Optional[torch.Tensor] = None, with_terms: bool = True) -> RolloutOutput:
        """Cost without gradient (what a sampling-based optimizer such as MPPI evaluates): the rows and cost outputs of
        evaluate_action from the cost-only kernels, which skip the J^T backward and every other piece of work only the
        gradient reads.  `grad_q` (and grad_vel / grad_acc / grad_jerk) are left untouched.  `with_terms=False` writes `cost`
        only -- the per-term tensors keep their previous contents; at particle batch sizes the per-sphere scene_cost alone is
        ~100 MB of writes.  Discrete rows only (cfg.use_sweep raises ValueError), and the dynamics-aware cost of
        attach_dynamics is not evaluated here (ValueError).  Buffers are allocated once per (B, H), so the call is CUDA-graph
        capturable."""
        if self.cfg.use_sweep:
            raise ValueError("evaluate_cost covers discrete rows only (cfg.use_sweep = False)")
        if self._effort_cost is not None or self._dyn_params is not None:
            raise ValueError("evaluate_cost does not evaluate the dynamics-aware cost of attach_dynamics")
        io, B, H = self._state_io(q, vel, acc, jerk, dt)
        return self._launch(io, B, H, env_query_idx, grad=False, with_terms=with_terms)

    def _state_io(self, q, vel, acc, jerk, dt):
        """Checks the row states of evaluate_action / evaluate_cost, (re)allocates the outputs for their (B, H) and returns the
        RolloutIO holding them, with B and H."""
        if q.ndim != 3 or q.shape[2] != self.robot.num_dof:
            raise ValueError(f"q must be [B, H, {self.robot.num_dof}], got {tuple(q.shape)}")
        B, H, _ = q.shape
        if (B, H) != (self._B, self._H):
            self.setup_batch_tensors(B, H)
        dev = self.device
        check_tensors(dev, torch.float32, q=q)
        io = _lib.RolloutIO()
        io.q = q.data_ptr()
        for name, t in (("vel", vel), ("acc", acc), ("jerk", jerk), ("dt", dt)):
            if t is not None:
                check_tensors(dev, torch.float32, **{name: t})
                setattr(io, name, t.data_ptr())
        return io, B, H

    def evaluate_knots(self, knots: torch.Tensor, start_state, start_state_idx: torch.Tensor, goal_state,
                       goal_state_idx: torch.Tensor, use_implicit_goal_state: torch.Tensor, bspline_degree: int = 4,
                       interpolation_steps: int = 4, env_query_idx: Optional[torch.Tensor] = None,
                       store_state: bool = False, in_kernel_spline: bool = False) -> RolloutOutput:
        """B-spline action space (SURVEY.md 8f rank 1): knots [B,n_knots,D] -> row costs and d cost / d knots in ONE C
        call.  Default schedule: spline kernel -> rollout kernel -> adjoint kernel on the same stream (3 launches, the
        state makes one round trip through L2).  `in_kernel_spline=True`: the rollout kernel evaluates its rows from the
        knots itself (2 launches; the state never leaves the SM unless `store_state`); identical results, currently
        slower at MPC scale.  start_state / goal_state
        carry position, velocity, acceleration, jerk [n, D]; goal_state.dt [n_goal] is the trajectory dt
        (same contract as curobo_b200.trajectory.StateFromBSplineKnot.forward)."""
        D = self.robot.num_dof
        if knots.ndim != 3 or knots.shape[2] != D:
            raise ValueError(f"knots must be [B, n_knots, {D}], got {tuple(knots.shape)}")
        if bspline_degree not in (3, 4, 5):
            raise RuntimeError(f"Unsupported B-spline degree: {bspline_degree}")
        if self.cfg.cspace_type != "state":
            raise ValueError("evaluate_knots needs the STATE c-space cost (velocity / acceleration / jerk gradients)")
        if goal_state.dt is None:
            raise ValueError("dt is None")
        B, nk, _ = knots.shape
        H = (nk + bspline_degree + 1) * interpolation_steps + 1
        if not 1 <= interpolation_steps <= 32:
            raise RuntimeError("interpolation_steps must be in [1, 32]")
        dev = self.device
        if (B, H) != (self._B, self._H):
            self.setup_batch_tensors(B, H)
        o = self.out
        if o.grad_knots is None or tuple(o.grad_knots.shape) != (B, nk, D):
            o.grad_knots = torch.zeros((B, nk, D), dtype=torch.float32, device=dev)
        f32 = dict(knots=knots, traj_dt=goal_state.dt)
        for pre, st in (("start", start_state), ("goal", goal_state)):
            for fld in ("position", "velocity", "acceleration", "jerk"):
                f32[f"{pre}_{fld}"] = getattr(st, fld)
        check_tensors(dev, torch.float32, **f32)
        check_tensors(dev, torch.int32, start_state_idx=start_state_idx, goal_state_idx=goal_state_idx)
        check_tensors(dev, torch.uint8, use_implicit_goal_state=use_implicit_goal_state)
        if goal_state_idx.shape[0] != B or start_state_idx.shape[0] != B:
            raise ValueError("start_state_idx / goal_state_idx need one entry per batch row")
        sp = _lib.SplineInput()
        sp.knots = knots.data_ptr()
        for pre, st in (("start", start_state), ("goal", goal_state)):
            for fld in ("position", "velocity", "acceleration", "jerk"):
                setattr(sp, f"{pre}_{fld}", getattr(st, fld).data_ptr())
        sp.start_idx, sp.goal_idx = start_state_idx.data_ptr(), goal_state_idx.data_ptr()
        sp.traj_dt, sp.use_implicit_goal_state = goal_state.dt.data_ptr(), use_implicit_goal_state.data_ptr()
        sp.n_knots, sp.degree = nk, bspline_degree
        sp.grad_knots = o.grad_knots.data_ptr()
        if store_state or not in_kernel_spline:
            if getattr(self, "_state", None) is None or tuple(self._state[0].shape) != (B, H, D):
                self._state = tuple(torch.zeros((B, H, D), dtype=torch.float32, device=dev) for _ in range(4))
                self._state_dt = torch.zeros((B,), dtype=torch.float32, device=dev)
            sp.out_position, sp.out_velocity, sp.out_acceleration, sp.out_jerk = (t.data_ptr() for t in self._state)
            if not in_kernel_spline:
                sp.out_dt = self._state_dt.data_ptr()
        io = _lib.RolloutIO()
        io.spline = C.pointer(sp)
        # dynamics-aware cost with the expanded schedule: the trajectory kernel reads the spline states like caller-provided
        # ones, its RNEA-adjoint gradients flow into grad_knots through the spline adjoint behind it
        if self._dyn_params is not None and not in_kernel_spline:
            io.dynamics = C.pointer(self._dyn_params)
        if self._effort_cost is not None:
            raise ValueError("evaluate_knots supports the dynamics-aware cost only inside the kernel (attach_dynamics(fused=True), "
                             "swept mode, in_kernel_spline=False)")
        if self._dyn_params is not None and in_kernel_spline:
            raise ValueError("the dynamics-aware cost needs the expanded spline schedule (in_kernel_spline=False)")
        return self._launch(io, B, H, env_query_idx)

    def evaluate_positions(self, u: torch.Tensor, start_state, start_state_idx: torch.Tensor, goal_state,
                           goal_state_idx: torch.Tensor, use_implicit_goal_state: torch.Tensor,
                           env_query_idx: Optional[torch.Tensor] = None) -> RolloutOutput:
        """Position action space without teleport (the reference's POSITION control space, StateFromPositionClique):
        waypoints u [B, H-4, D] -> row costs and d cost / d u (`grad_u`).  Three launches on the current stream: the clique
        stencil (u -> position / velocity / acceleration / jerk [B, H, D] with start-state and implicit-goal padding), the
        fused rollout in trajectory mode (evaluate_action with those states), the clique adjoint of grad_q / grad_vel /
        grad_acc / grad_jerk.  start_state / goal_state carry position, velocity, acceleration; goal_state.dt [n_goal] is
        the trajectory dt; start / goal rows are gathered through start_state_idx / goal_state_idx [B] (same contract as
        curobo_b200.trajectory.StateFromPositionClique.forward).  The states are kept in `_state` / `_state_dt`; every
        buffer is allocated once per (B, H), so the call is CUDA-graph capturable."""
        D = self.robot.num_dof
        if u.ndim != 3 or u.shape[2] != D:
            raise ValueError(f"u must be [B, horizon - 4, {D}], got {tuple(u.shape)}")
        if self.cfg.cspace_type != "state":
            raise ValueError("evaluate_positions needs the STATE c-space cost (velocity / acceleration / jerk gradients)")
        if goal_state.dt is None:
            raise ValueError("dt is None")
        B, n, _ = u.shape
        H = n + 4
        if start_state_idx.shape[0] != B or goal_state_idx.shape[0] != B:
            raise ValueError("start_state_idx / goal_state_idx need one entry per batch row")
        dev = self.device
        if getattr(self, "_state", None) is None or tuple(self._state[0].shape) != (B, H, D):
            self._state = tuple(torch.zeros((B, H, D), dtype=torch.float32, device=dev) for _ in range(4))
            self._state_dt = torch.zeros((B,), dtype=torch.float32, device=dev)
        if (B, H) != (self._B, self._H):
            self.setup_batch_tensors(B, H)
        o = self.out
        if o.grad_u is None or tuple(o.grad_u.shape) != (B, n, D):
            o.grad_u = torch.zeros((B, n, D), dtype=torch.float32, device=dev)
        p, v, a, j = self._state
        trajectory_cu.launch_differentiation_position_forward_kernel(
            p, v, a, j, self._state_dt, u, start_state.position, start_state.velocity, start_state.acceleration,
            goal_state.position, goal_state.velocity, goal_state.acceleration, start_state_idx, goal_state_idx, goal_state.dt,
            use_implicit_goal_state, B, H, D)
        out = self.evaluate_action(p, vel=v, acc=a, jerk=j, dt=self._state_dt, env_query_idx=env_query_idx)
        trajectory_cu.launch_differentiation_position_backward_kernel(
            out.grad_u, out.grad_q, out.grad_vel, out.grad_acc, out.grad_jerk, goal_state.dt, goal_state_idx,
            use_implicit_goal_state, B, H, D)
        return out

    def validate(self, q: torch.Tensor, env_query_idx: Optional[torch.Tensor] = None, check_bounds: bool = True,
                 check_self: bool = True, check_scene: bool = True) -> torch.Tensor:
        """Validity of joint configurations q [B, H, D] -> torch.bool [B, H] (cb200_rollout_validate; the reference's
        RobotSceneCollision.validate): a row is valid iff it is inside the position limits (check_bounds), no pair of the
        self-collision pair list overlaps with padded radii (check_self), and no enabled sphere touches an enabled obstacle of
        the row's environment, r - sdf > 0 (check_scene).  Independent of `cfg`: the terms are tested at activation 0.  H > 1
        rows are independent discrete rows.  The output buffer is allocated once per (B, H) and returned as a bool view of it,
        so the call is CUDA-graph capturable; a later call with the same (B, H) overwrites it."""
        if q.ndim != 3 or q.shape[2] != self.robot.num_dof:
            raise ValueError(f"q must be [B, H, {self.robot.num_dof}], got {tuple(q.shape)}")
        check_tensors(self.device, torch.float32, q=q)
        B, H, _ = q.shape
        if getattr(self, "_valid", None) is None or tuple(self._valid.shape) != (B, H):
            self._valid = torch.zeros((B, H), dtype=torch.uint8, device=self.device)
        io = _lib.RolloutIO()
        io.q = q.data_ptr()
        io.batch_size, io.horizon = B, H
        self._world_io(io, env_query_idx)
        err = self._lib.cb200_rollout_validate(C.byref(io), self._valid.data_ptr(), int(bool(check_bounds)), int(bool(check_self)),
                                               int(bool(check_scene)), stream_ptr(self.device))
        _lib.check(err, "rollout_validate")
        return self._valid.view(torch.bool)

    def _world_io(self, io, env_query_idx) -> None:
        """The robot blob, the obstacle sets, env_query_idx, the sphere configurations and the ticket counter into io."""
        dev = self.device
        io.robot_blob, io.robot_blob_host = self._blob.data_ptr(), self._blob_host.ctypes.data
        io.robot_blob_bytes = int(self._blob_host.shape[0])
        if self._cs is not None:
            io.cuboids = C.pointer(self._cs)
        if self._vs is not None:
            io.voxels = C.pointer(self._vs)
        if self._ms is not None:
            io.meshes = C.pointer(self._ms)
        if self.voxel is not None and self.use_voxel_mip:
            from .scene import voxel_mip_is_fresh
            if not voxel_mip_is_fresh(self.voxel):      # the ESDF tensor was updated or replaced since the level was built
                if torch.cuda.is_current_stream_capturing():
                    raise RuntimeError("the ESDF changed since refresh_world(); call it before capturing a graph")
                self.refresh_world()
                io.voxels = C.pointer(self._vs)
        if env_query_idx is not None:
            check_tensors(dev, torch.int32, env_query_idx=env_query_idx)
            io.env_query_idx = env_query_idx.data_ptr()
        if self.link_spheres._version != self._link_spheres_version:   # written in place since the last refresh
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("link_spheres changed since the last refresh; call refresh_link_spheres() before capturing")
            self.refresh_link_spheres()
        if self.link_spheres.shape[0] > 1:
            io.sphere_configs, io.num_sphere_configs = self.link_spheres.data_ptr(), int(self.link_spheres.shape[0])
        io.work_counter = self._work_counter.data_ptr()

    def _launch(self, io, B: int, H: int, env_query_idx, grad: bool = True, with_terms: bool = True) -> RolloutOutput:
        dev = self.device
        o = self.out
        self._world_io(io, env_query_idx)
        if self._goal is not None and self.cfg.pose_weight is not None:
            gp, gq, ig, extra = self._goal
            if ig.shape[0] != B:
                raise ValueError("idxs_goal must have one entry per batch row")
            io.goal_position, io.goal_quat, io.idxs_goal = gp.data_ptr(), gq.data_ptr(), ig.data_ptr()
            for cname, key in (("pose_axes_terminal", "terminal_axes"), ("pose_axes_non_terminal", "non_terminal_axes"),
                               ("pose_tol_terminal", "terminal_tol"), ("pose_tol_non_terminal", "non_terminal_tol")):
                if extra[key] is not None:
                    setattr(io, cname, extra[key].data_ptr())
        if self.cfg.cspace_target_weight > 0.0 and self.cfg.cspace_type is not None:
            if self._cs_target is None:
                raise ValueError("cspace_target_weight > 0 needs update_cspace_target(...) first")
            tgt, tidx, tdw = self._cs_target
            if tidx is not None and tidx.shape[0] != B:
                raise ValueError("idxs_cspace_target must have one entry per batch row")
            io.cspace_target = tgt.data_ptr()
            if tidx is not None:
                io.idxs_cspace_target = tidx.data_ptr()
            if tdw is not None:
                io.cspace_target_dof_weight = tdw.data_ptr()
        if self._current_state is not None and self.cfg.cspace_type == "position":
            cp, cv, cdt, cidx = self._current_state
            if cidx is not None and cidx.shape[0] != B:
                raise ValueError("idxs_current_state must have one entry per batch row")
            io.current_position, io.current_state_dt = cp.data_ptr(), cdt.data_ptr()
            if cv is not None:
                io.current_velocity = cv.data_ptr()
            if cidx is not None:
                io.idxs_current_state = cidx.data_ptr()
        io.cost = o.cost.data_ptr()
        if grad:
            io.grad_q = o.grad_q.data_ptr()
        outs = ("grad_vel", "grad_acc", "grad_jerk") if grad else ()
        if with_terms:
            io.self_cost, io.scene_cost = o.self_cost.data_ptr(), o.scene_cost.data_ptr()
            io.pose_cost, io.cspace_cost = o.pose_cost.data_ptr(), o.cspace_cost.data_ptr()
            outs += ("link_pos", "link_quat", "robot_spheres", "pose_goalset_idx")
        for name in outs:
            t = getattr(o, name)
            if t is not None:
                setattr(io, name, t.data_ptr())
        io.batch_size, io.horizon = B, H
        if self._dyn_params is not None and io.vel and io.acc and not bool(io.spline):
            io.dynamics = C.pointer(self._dyn_params)
        if self._ms is not None and self.cfg.scene_weight > 0.0:
            if io.dynamics:
                raise ValueError("mesh obstacles are not supported by the dynamics-aware cost inside the kernel "
                                 "(attach_dynamics(fused=True)); use attach_dynamics(fused=False), which adds the same terms "
                                 "with separate launches")
            if io.spline and not io.spline.contents.out_dt:
                raise ValueError("mesh obstacles are not supported by the in-kernel spline schedule; use "
                                 "evaluate_knots(in_kernel_spline=False), the expanded schedule")
        if grad:
            err = self._lib.cb200_rollout_cost_grad(C.byref(self._ccfg), C.byref(io), stream_ptr(dev))
            _lib.check(err, "rollout_cost_grad")
        else:
            err = self._lib.cb200_rollout_cost(C.byref(self._ccfg), C.byref(io), stream_ptr(dev))
            _lib.check(err, "rollout_cost")
        return o


class FusedRolloutFunction(torch.autograd.Function):
    """cost[B] = sum_h rollout cost; backward returns the gradient computed in the same launch
    (the reference's own pattern: forward writes the gradient buffer, backward hands it out,
    cuda_ops/geometry.py:95-104, wp_autograd.py:103-110; the optimizer's upstream gradient is all-ones,
    gradient_opt_core.py:478).  Unlike the reference's Functions with use_grad_input=False the upstream gradient IS
    applied (per seed), so `cost.mean()` or a weighted sum differentiates correctly, and the gradient is saved as a
    copy: a second forward before backward does not disturb the first one's gradient."""

    @staticmethod
    def forward(ctx, q: torch.Tensor, engine: RolloutEngine):
        out = engine.evaluate_action(q.detach())
        ctx.save_for_backward(out.grad_q.clone())
        return out.cost.sum(dim=1)

    @staticmethod
    def backward(ctx, grad_cost):
        (g,) = ctx.saved_tensors
        return g * grad_cost.reshape(-1, 1, 1), None


class HostRolloutPipeline:
    """`evaluate_action` for HOST-resident inputs, the way an optimizer that keeps its iterate on the host (or another
    process feeding joint batches) drives the kernel: per step  pinned q -> H2D -> fused rollout -> D2H of cost + grad_q.

    Each slot owns an engine (= one set of output buffers), pinned host buffers and ONE captured CUDA graph holding the
    three stages, replayed on the slot's own stream: a step costs the host a single graph launch, and with two slots the
    upload of step i+1 overlaps the kernel of step i (stream order inside a slot makes buffer reuse safe).

        pipe = HostRolloutPipeline([eng_a, eng_b], B, H, dt=dt)
        pipe.slots[k].q_host[...] = ...      # fill the pinned input of slot k
        pipe.submit(k)                       # H2D + kernel + D2H, asynchronous
        cost, grad = pipe.result(k)          # waits for slot k; pinned host tensors
    """

    class Slot:
        def __init__(self, engine, B, H, D, device):
            self.engine = engine
            self.stream = torch.cuda.Stream(device)
            self.q_host = torch.empty((B, H, D), dtype=torch.float32).pin_memory()
            self.cost_host = torch.empty((B, H), dtype=torch.float32).pin_memory()
            self.grad_host = torch.empty((B, H, D), dtype=torch.float32).pin_memory()
            self.q_dev = torch.empty((B, H, D), dtype=torch.float32, device=device)
            self.graph = None

    def __init__(self, engines: Sequence[RolloutEngine], batch: int, horizon: int, **eval_kwargs):
        if not engines:
            raise ValueError("at least one engine")
        self.device = engines[0].device
        D = engines[0].robot.num_dof
        self._kw = eval_kwargs
        self.slots = [HostRolloutPipeline.Slot(e, batch, horizon, D, self.device) for e in engines]
        self.h2d_bytes = int(self.slots[0].q_host.numel() * 4)
        self.d2h_bytes = int((self.slots[0].cost_host.numel() + self.slots[0].grad_host.numel()) * 4)
        for s in self.slots:
            s.q_host.zero_()
            self._stages(s)                                    # eager once: output allocation, launch-plan caches
        torch.cuda.synchronize(self.device)
        for s in self.slots:
            s.graph = torch.cuda.CUDAGraph()
            with torch.cuda.device(self.device), torch.cuda.graph(s.graph, stream=s.stream):
                self._stages(s)

    def _stages(self, s) -> None:
        s.q_dev.copy_(s.q_host, non_blocking=True)
        out = s.engine.evaluate_action(s.q_dev, **self._kw)
        s.cost_host.copy_(out.cost, non_blocking=True)
        s.grad_host.copy_(out.grad_q, non_blocking=True)

    def submit(self, k: int) -> None:
        s = self.slots[k]
        with torch.cuda.stream(s.stream):
            s.graph.replay()

    def result(self, k: int):
        s = self.slots[k]
        s.stream.synchronize()
        return s.cost_host, s.grad_host

    def wait_all(self) -> None:
        for s in self.slots:
            s.stream.synchronize()
