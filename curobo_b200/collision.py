"""`RobotCollisionChecker`: the reference's curobo.collision_checking.RobotCollisionChecker (RobotSceneCollision,
curobo/_src/collision/collision_robot_scene.py) on this backend.

`validate` / `validate_trajectory` and the rejection sampling behind `sample` / `sample_trajectory` run on one early-exit launch
(RolloutEngine.validate -> cb200_rollout_validate).  The distance methods are composed from the per-operator drop-ins
(Kinematics, SphereObstacleCollision, SelfCollisionDistance, the POSITION c-space cost) with the reference's weights,
activation distances and `use_grad_input` settings (collision_robot_scene_cfg.py:147-186).

Differences from the reference: samples are uniform draws from a torch generator, not its Halton sequence, so the sampled
configurations differ from the reference's; `pose_distance`, `get_point_robot_distance` and the AttachmentManager wiring are
not provided (attached objects go through `checker.engine.attach_object_spheres`, which the distance methods see too).
"""
from __future__ import annotations

from typing import Optional, Tuple, Union

import torch

from .backends.tensor_checks import check_tensors
from .cost import cspace_position_cost
from .kinematics import Kinematics, KinematicsState, SelfCollisionCost, SelfCollisionDistance
from .robot_model import RobotModel
from .rollout import RolloutConfig, RolloutEngine
from .scene import CollisionBuffer, CuboidData, SceneData, SphereObstacleCollision, VoxelData


class _PositionBoundCost(torch.autograd.Function):
    """Bound cost of the POSITION c-space cost at weight [1, 0], activation 0 ([B, H, D]); backward applies the upstream
    gradient to the per-dof gradient written by the same launch (use_grad_input=True)."""

    @staticmethod
    def forward(ctx, q, checker):
        bufs = checker._bound_buffers(q.shape)
        cost, grad = bufs["cost"], bufs["grad_p"]
        cspace_position_cost(q.detach(), bufs["effort"], bufs["zd"], bufs["zi"], checker._p_lim, checker._tau_lim,
                             checker._bound_w, checker._bound_act, bufs["f0"], bufs["dofw"], bufs["reg"], bufs["zd"],
                             bufs["zd"], bufs["zi"], checker._v_lim, bufs["f0"], cost, grad, bufs["grad_tau"])
        ctx.save_for_backward(grad)
        return cost

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * g, None


class RobotCollisionChecker:
    """Collision checks of a robot against a scene (cuboids, ESDF grids, meshes), per joint configuration.

    `robot`: RobotModel; `cuboid` / `voxel` / `mesh`: the obstacle holders of RolloutEngine; `collision_activation_distance`:
    the activation distance of get_collision_distance (validity uses 0); `rejection_ratio`: draws per requested sample."""

    def __init__(self, robot: RobotModel, device="cuda:0", cuboid: Optional[CuboidData] = None, voxel: Optional[VoxelData] = None,
                 mesh=None, collision_activation_distance: float = 0.2, rejection_ratio: int = 10):
        self.robot, self.device = robot, torch.device(device)
        self.rejection_ratio = int(rejection_ratio)
        self.collision_activation_distance = float(collision_activation_distance)
        self.engine = RolloutEngine(robot, RolloutConfig(), self.device, cuboid, voxel, mesh=mesh)
        self.kinematics = Kinematics(robot, self.device)
        self.kinematics.params.link_spheres = self.engine.link_spheres   # attached / disabled spheres reach the drop-ins too
        self.scene = SceneData(cuboid, voxel, mesh)
        self.has_scene = cuboid is not None or voxel is not None or mesh is not None
        self.self_collision_cost = SelfCollisionCost(robot, 1.0, self.device)
        t = lambda a: torch.as_tensor(a, dtype=torch.float32).to(self.device).contiguous()  # noqa: E731
        self._p_lim, self._v_lim, self._tau_lim = t(robot.position_limits), t(robot.velocity_limits), t(robot.effort_limits)
        self._scene_w, self._scene_act = t([1.0]), t([self.collision_activation_distance])
        self._bound_w, self._bound_act = t([1.0, 0.0]), t([0.0, 0.0])
        self._scene_buf = None
        self._bound_bufs = None

    # -- validity (cb200_rollout_validate) ----------------------------------------------------------------------------------
    def validate(self, q: torch.Tensor, env_query_idx: Optional[torch.Tensor] = None) -> torch.Tensor:
        """q [batch, horizon, dof] -> bool [batch, horizon]: inside the position limits, no self contact, no scene contact
        (RobotSceneCollision.validate).  The result is a view of a buffer the next call with the same shape overwrites."""
        if q.ndim != 3:
            raise ValueError(f"q must have shape [batch, horizon, dof], got {tuple(q.shape)}")
        return self.engine.validate(q, env_query_idx)

    def validate_trajectory(self, q: torch.Tensor, env_query_idx: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Every waypoint of q [batch, horizon, dof] as an independent configuration (no sweep between waypoints)."""
        return self.validate(q, env_query_idx)

    # -- sampling -----------------------------------------------------------------------------------------------------------
    def _uniform(self, shape, generator) -> torch.Tensor:
        lo, hi = self._p_lim[0], self._p_lim[1]
        u = torch.rand(shape + (self.robot.num_dof,), generator=generator, dtype=torch.float32, device=self.device)
        return lo + (hi - lo) * u

    def sample(self, n: int, mask_valid: bool = True, env_query_idx: Optional[torch.Tensor] = None,
               generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """Up to n valid configurations [<= n, dof]: n * rejection_ratio uniform draws inside the limits, validated, the
        first n valid ones kept in draw order (the reference's q[q_mask][:n]).  With mask_valid=False: n draws, unchecked.
        The only synchronisation is the read of the number of rows kept."""
        if not mask_valid:
            return self._uniform((int(n),), generator)
        m = int(n) * self.rejection_ratio
        q = self._uniform((m,), generator)
        valid = self.validate(q[:, None, :], env_query_idx)[:, 0]
        rank = torch.cumsum(valid.to(torch.int32), 0)
        keep = valid & (rank <= n)
        dst = torch.where(keep, rank - 1, torch.full_like(rank, n)).to(torch.int64)   # row n collects the rest
        out = torch.zeros((int(n) + 1, self.robot.num_dof), dtype=torch.float32, device=self.device)
        out.index_copy_(0, dst, q)
        count = min(int(rank[-1]), int(n)) if m > 0 else 0
        return out[:count]

    def sample_trajectory(self, batch: int, horizon: int, mask_valid: bool = True, env_query_idx: Optional[torch.Tensor] = None,
                          generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """[batch, horizon, dof]: per batch row, the first `horizon` valid configurations of horizon * rejection_ratio draws.
        Raises ValueError when a row has fewer than `horizon` valid draws."""
        if not mask_valid:
            return self._uniform((int(batch), int(horizon)), generator)
        m = int(horizon) * self.rejection_ratio
        q = self._uniform((int(batch), m), generator)
        valid = self.validate_trajectory(q, env_query_idx)
        rank = torch.cumsum(valid.to(torch.int32), 1)
        if batch > 0 and int(rank[:, -1].min()) < horizon:
            raise ValueError(f"a batch row has fewer than {horizon} valid samples among {m} draws; raise rejection_ratio")
        keep = valid & (rank <= horizon)
        dst = torch.where(keep, rank - 1, torch.full_like(rank, horizon)).to(torch.int64)
        out = torch.zeros((int(batch), int(horizon) + 1, self.robot.num_dof), dtype=torch.float32, device=self.device)
        out.scatter_(1, dst[..., None].expand(-1, -1, self.robot.num_dof), q)
        return out[:, :horizon]

    # -- distances (per-operator drop-ins) ----------------------------------------------------------------------------------
    def get_kinematics(self, q: torch.Tensor, env_query_idx: Optional[torch.Tensor] = None) -> KinematicsState:
        """Forward kinematics of q [batch, (horizon,) dof] with the engine's current link spheres (sphere configuration
        env_query_idx[b] when the engine has several)."""
        eq = env_query_idx if self.engine.link_spheres.shape[0] > 1 else None
        return self.kinematics.compute_kinematics(q, eq)

    def get_collision_distance(self, x_sph: Union[torch.Tensor, KinematicsState],
                               env_query_idx: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Scene collision cost per sphere [batch, horizon, spheres] at weight 1 and `collision_activation_distance`; its
        gradient is the sphere gradient of the same launch, not scaled by the upstream gradient (use_grad_input=False)."""
        sph = x_sph.robot_spheres if isinstance(x_sph, KinematicsState) else x_sph
        if not self.has_scene:
            return torch.zeros(sph.shape[:-1], dtype=sph.dtype, device=sph.device)
        if self._scene_buf is None or tuple(self._scene_buf.gradient.shape) != tuple(sph.shape):
            self._scene_buf = CollisionBuffer.from_shape(tuple(sph.shape), self.device)
        if env_query_idx is not None:
            check_tensors(self.device, torch.int32, env_query_idx=env_query_idx)
        return SphereObstacleCollision.apply(sph, self._scene_buf, self.scene, self._scene_w, self._scene_act, None,
                                             env_query_idx, env_query_idx is not None, False)

    def get_self_collision_distance(self, x_sph: torch.Tensor) -> torch.Tensor:
        """Self-collision cost [batch, horizon, 1] (0.5 f of the worst pair, weight 1); the upstream gradient is applied
        (use_grad_input=True)."""
        c = self.self_collision_cost
        b, h = int(x_sph.shape[0]), int(x_sph.shape[1])
        if c._shape != (b, h):
            c.setup_batch_tensors(b, h)
        return SelfCollisionDistance.apply(x_sph, c._out_distance, c._out_vec, c._pair_distance, c._sparse, c.weight,
                                           c.sphere_padding, c.pairs, c._bbmv, c._bbmi, self.robot.num_blocks_per_batch,
                                           self.robot.max_threads_per_block, False, True)

    def get_scene_self_collision_distance_from_joints(self, q: torch.Tensor, env_query_idx: Optional[torch.Tensor] = None
                                                      ) -> Tuple[torch.Tensor, torch.Tensor]:
        """(scene distance [batch, horizon, spheres], self distance [batch, horizon, 1]) of q [batch, horizon, dof];
        differentiable in q through the forward kinematics."""
        state = self.get_kinematics(q, env_query_idx)
        return self.get_collision_distance(state, env_query_idx), self.get_self_collision_distance(state.robot_spheres)

    def get_scene_self_collision_distance_from_joint_trajectory(self, q: torch.Tensor,
                                                                env_query_idx: Optional[torch.Tensor] = None
                                                                ) -> Tuple[torch.Tensor, torch.Tensor]:
        return self.get_scene_self_collision_distance_from_joints(q, env_query_idx)

    def get_bound(self, q: torch.Tensor) -> torch.Tensor:
        """Joint-bound cost [batch, horizon, dof]: 0.5 d^2 with d the distance outside the position limits (weight [1, 0],
        activation 0); the upstream gradient is applied (use_grad_input=True)."""
        if q.ndim != 3:
            raise ValueError(f"q must have shape [batch, horizon, dof], got {tuple(q.shape)}")
        return _PositionBoundCost.apply(q, self)

    def _bound_buffers(self, shape) -> dict:
        if self._bound_bufs is None or self._bound_bufs["shape"] != tuple(shape):
            B, H, D = shape
            dev = self.device
            z = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)  # noqa: E731
            self._bound_bufs = dict(shape=tuple(shape), cost=z(B, H, D), grad_p=z(B, H, D), grad_tau=z(B, H, D), effort=z(B, H, D),
                                    zd=z(1, D), zi=torch.zeros(B, dtype=torch.int32, device=dev), f0=z(1),
                                    dofw=torch.ones(D, dtype=torch.float32, device=dev), reg=z(2))
        return self._bound_bufs
