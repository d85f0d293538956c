/*
 * curobo_b200.h  --  C ABI of libcurobo_b200.so: the sm_90a rollout cost+gradient hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  Every entry point takes raw DEVICE pointers,
 * plain ints/floats and the CUDA stream to launch on, returns a cudaError_t (0 = success) and
 * never allocates, synchronises or touches the default stream -- exactly what the reference's
 * `cuda_core` backend passes to its NVRTC kernels (`tensor.data_ptr()` ints + scalars on
 * `torch.cuda.current_stream`, curobo/_src/curobolib/backends/cuda_core_backend/kinematics.py:130-176),
 * so the calls are CUDA-graph capturable like the reference's (util/cuda_graph_util.py:101-175).
 *
 * Each function names the reference interface it replaces (file:line, relative to the reference
 * root).  Argument ORDER follows the reference launcher so a binding is a 1:1 forward
 * (see INTEGRATION.md for the ctypes stub a curobo maintainer would add).
 *
 * All tensors are contiguous, float = IEEE fp32, layouts as in the reference:
 *   q [B*H, D]; link_pos [B*H, L, 3]; link_quat [B*H, L, 4] (w,x,y,z; w >= 0);
 *   robot_spheres [B*H, S, 4] (x,y,z,r); cumul_mat [B*H, nl, 3, 4] row-major.
 */
#ifndef CUROBO_B200_H
#define CUROBO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st *cb200_stream_t; /* == cudaStream_t */

#define CB200_ABI_VERSION 6

/* Library / build identity.  cb200_abi_version() == CB200_ABI_VERSION; cb200_sm_arch() == 90. */
int cb200_abi_version(void);
int cb200_sm_arch(void);
/* Human-readable string for the last non-zero return code of this thread (cudaGetErrorString). */
const char *cb200_error_string(int err);
/* Which kernel the last cb200_rollout_cost_grad / cb200_rollout_cost call of this thread launched (introspection for tests and the
   bench line; the choice is made by the launcher from the robot, the scene content and the row count -- see DESIGN.md "Row
   scheduling").  A cost-only launch reports the variant it twins with CB200_VARIANT_COST_ONLY set. */
#define CB200_VARIANT_NONE 0
#define CB200_VARIANT_STANDARD 1 /* rollout_fused_kernel: one warp per row */
#define CB200_VARIANT_ARM 2      /* ... its 80-register build for arms (one row per warp, or two: one per half-warp) */
#define CB200_VARIANT_BIG 4      /* rollout_fused_big_kernel: humanoids / ESDF scenes, gradient list */
#define CB200_VARIANT_TEAM2 5    /* rollout_fused_team_kernel: two warps per row */
#define CB200_VARIANT_TEAM4 6    /* ... four warps per row */
#define CB200_VARIANT_TRAJ 7     /* rollout_traj_kernel: trajectory mode (swept collision, state costs) */
#define CB200_VARIANT_TRAJ_DYN 8 /* rollout_traj_dyn_kernel: trajectory mode + inverse dynamics */
#define CB200_VARIANT_COST_ONLY 0x10 /* bit: cb200_rollout_cost (rollout_cost_kernel / rollout_cost_big_kernel) */
#define CB200_VARIANT_VALIDATE 0x20  /* bit: cb200_rollout_validate (rollout_validate_kernel) */
int cb200_last_rollout_variant(void);

/* -------------------------------------------------------------------------------------------
 * (a2) FK + robot spheres + tool poses.
 * Replaces launch_kinematics_forward_spheres
 *   curobo/_src/curobolib/backends/cuda_core_backend/kinematics.py:90-177
 *   (kernel kinematics_forward_spheres_kernel, kernels/kinematics/kinematics_forward_kernel.cuh:131-261).
 * batch_size is B*H (cuda_ops/kinematics.py:115).  env_query_idx [B] selects the sphere set
 * robot_spheres[num_envs, S, 4] for batch row n via env_query_idx[n / horizon] when num_envs > 1.
 * compute_com != 0: batch_center_of_mass [B*H, 4] = mass-weighted mean of the links' world centres of mass (xyz) and the total mass
 * (w), from link_masses_com [nl, 4] = local CoM xyz, mass; links with mass <= 0 are skipped (kinematics_forward_helper.cuh:538-601).
 * global_cumul_mat is written iff write_global_cumul != 0.
 * ------------------------------------------------------------------------------------------- */
int cb200_kinematics_forward_spheres(
    float *link_pos, float *link_quat, float *batch_robot_spheres, float *batch_center_of_mass,
    float *global_cumul_mat, const float *joint_vec, const float *fixed_transform,
    const float *robot_spheres, const float *link_masses_com, const int8_t *joint_map_type,
    const int16_t *joint_map, const int16_t *link_map, const int16_t *tool_frame_map,
    const int16_t *link_sphere_map, const float *joint_offset_map, const int32_t *env_query_idx,
    int num_envs, int batch_size, int horizon, int n_joints, int num_spheres, int num_links,
    int n_tool_frames, int write_global_cumul, int compute_com, cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * (a4) FK backward: grad_out[B*H, D] = sum_spheres J^T g + sum_tool_frames J^T (g_pos, omega(g_quat)).
 * Replaces launch_kinematics_backward
 *   curobo/_src/curobolib/backends/cuda_core_backend/kinematics.py:282-379
 *   (kernel kinematics_backward_kernel, kernels/kinematics/kinematics_backward_kernel.cuh:34-160).
 * link_chain_*, joint_links_*, joint_affects_endeffector are accepted for signature parity (the tree
 * is re-derived from link_map).  compute_com != 0 adds the gradient of the centre of mass (grad_center_of_mass [B*H, 4], w ignored;
 * batch_center_of_mass carries the total mass): the force g m_k / M at each link's world CoM, walked down the chain like a sphere
 * gradient (kinematics_backward_helper.cuh:187-260).  compute_jacobian_grad must be 0.
 * ------------------------------------------------------------------------------------------- */
int cb200_kinematics_backward(
    float *grad_out, const float *grad_nlinks_pos, const float *grad_nlinks_quat,
    const float *grad_spheres, const float *grad_center_of_mass, const float *batch_center_of_mass,
    const float *grad_jacobian, const float *global_cumul_mat, const float *robot_spheres,
    const float *link_masses_com, const int16_t *link_map, const int16_t *joint_map,
    const int8_t *joint_map_type, const int16_t *tool_frame_map, const int16_t *link_sphere_map,
    const int16_t *link_chain_data, const int16_t *link_chain_offsets, const int16_t *joint_links_data,
    const int16_t *joint_links_offsets, const uint8_t *joint_affects_endeffector,
    const float *joint_offset_map, const int32_t *env_query_idx, int num_envs, int batch_size,
    int horizon, int n_joints, int num_spheres, int num_links, int n_tool_frames, int compute_com,
    int compute_jacobian_grad, cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * (a7) Self-collision: worst sphere pair, cost 0.5*w*f_max, gradient on the two spheres of that pair.
 * Replaces self_collision_distance
 *   curobo/_src/curobolib/backends/cuda_core_backend/geometry.py:63-227
 *   (kernels self_collision_max_distance_kernel / max_block / max_reduce,
 *    kernels/geometry/self_collision/self_collision_kernel.cuh:20-303).
 * One launch for any pair count (the 2-kernel map-reduce of the reference collapses into one kernel;
 * block_batch_max_* are accepted and left untouched).  out_vec rows are lazily zeroed through
 * sparse_index exactly like the reference (self_collision_helper.cuh:151-192).
 * ------------------------------------------------------------------------------------------- */
int cb200_self_collision_distance(
    float *out_distance, float *out_vec, float *pair_distance, uint8_t *sparse_index,
    const float *robot_spheres, const float *sphere_padding, const float *weight,
    const int16_t *pair_locations, float *block_batch_max_value, int16_t *block_batch_max_index,
    int num_blocks_per_batch, int max_threads_per_block, int batch_size, int horizon, int nspheres,
    int num_collision_pairs, int store_pair_distance, int compute_grad, cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * Obstacle sets, passed by value.  Tensor layouts are the reference's CuboidData / VoxelData
 * (geom/data/data_cuboid.py:43-110, geom/data/data_voxel.py:41-92); a null `inv_pose` = absent.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  const float *dims;       /* [n_env, max_n, 4] full extents */
  const float *inv_pose;   /* [n_env, max_n, 8] x,y,z,qw,qx,qy,qz,pad (world -> obstacle) */
  const uint8_t *enable;   /* [n_env, max_n] */
  const int32_t *count;    /* [n_env] */
  int32_t max_n;
  int32_t num_envs;
} cb200_cuboid_set;

typedef struct {
  const float *params;     /* [n_env, max_n, 4] nx,ny,nz,voxel_size */
  const float *inv_pose;   /* [n_env, max_n, 8] */
  const uint8_t *enable;   /* [n_env, max_n] */
  const int32_t *count;    /* [n_env] */
  const uint16_t *features; /* [n_env, max_n, n_voxels_per_layer] IEEE fp16, C order (z fastest) */
  int32_t n_voxels_per_layer;
  int32_t max_n;
  int32_t num_envs;
  float max_dist;
  /* Optional acceleration structure owned by the caller (NULL = none; results are identical either way): one fp16
   * per block of cb200_voxel_mip_block()^3 trilinear base corners holding the minimum ESDF value any sample based in that block can read,
   * filled by cb200_voxel_build_mip after every ESDF update.  Discrete collision skips the eight corner fetches of a
   * sample whose block bound already proves sdf >= r + eta.  Layer k starts at mip + k * mip_stride. */
  const uint16_t *mip;
  int32_t mip_stride;
} cb200_voxel_set;

/* Block edge B of the pyramid level (base corners per block and axis). */
int cb200_voxel_mip_block(void);
/* mip_stride needed for a grid set: max over layers of ceil(nx/B)*ceil(ny/B)*ceil(nz/B) (HOST params pointer). */
int64_t cb200_voxel_mip_stride(const float *host_params, int num_layers);
/* Mesh obstacles (curobo/_src/geom/data/data_mesh.py:40-520 MeshData; the Warp mesh handles are replaced by BVHs built on the
 * host by curobo_b200/mesh.py).  Node = 2 float4 (box min, skip link) (box max, leaf word); triangle = 8 float4 (a, b, c, face
 * normal, edge pseudo-normals ab / bc / ca, vertex pseudo-normals in the w lanes): curobo_b200/csrc/cb200_mesh.cuh. */
typedef struct cb200_mesh_set {
  const float *nodes;             /* all meshes' BVH nodes, 8 floats each */
  const float *triangles;         /* all meshes' triangles, 32 floats each */
  const int32_t *node_offset;     /* [num_envs * max_n] first node of mesh k */
  const int32_t *triangle_offset; /* [num_envs * max_n] first triangle of mesh k */
  const float *dims;              /* [num_envs * max_n, 4] bounding-box extents */
  const float *inv_pose;          /* [num_envs * max_n, 8] x y z qw qx qy qz pad */
  const uint8_t *enable;          /* [num_envs * max_n] */
  const int32_t *count;           /* [num_envs] */
  int32_t max_n, num_envs;
} cb200_mesh_set;

/* Sphere / swept-sphere collision against mesh obstacles: the reference's generic collision kernels instantiated for MeshData
 * (geom/collision/wp_collision_kernel.py:70-166, wp_sweep_collision_kernel.py:83-260 with data_mesh.py:643-700 as the SDF).
 * accumulate = 1 adds to distance / gradient (after the cuboid / ESDF launch), 0 overwrites. */
int cb200_sphere_mesh_collision(float *distance, float *gradient, const float *spheres, const cb200_mesh_set *meshes,
                                const float *weight, const float *activation_distance, const float *speed_dt,
                                int enable_speed_metric, const int32_t *env_query_idx, int batch_size, int horizon,
                                int num_spheres, int use_multi_env, int sweep, int accumulate, cb200_stream_t stream);

/* Fill vs->mip (device, num_envs*max_n*mip_stride uint16) from vs->features / vs->params on `stream`. */
int cb200_voxel_build_mip(const cb200_voxel_set *vs, cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * (a8-a11) sphere vs scene, discrete.  distance [B,H,S], gradient [B,H,S,4] are OVERWRITTEN
 * (the reference zeroes the buffer and atomically accumulates one launch per obstacle type;
 * here one thread owns a sphere and loops over every obstacle of every type: same sum, no atomics).
 * Replaces SphereObstacleCollision.forward  curobo/_src/geom/collision/wp_autograd.py:37-121
 *   (Warp kernel sphere_obstacle_collision_kernel, geom/collision/wp_collision_kernel.py:70-166).
 * weight / activation_distance are 1-element device arrays, like the reference.
 * ------------------------------------------------------------------------------------------- */
int cb200_sphere_obstacle_collision(
    float *distance, float *gradient, const float *spheres, const cb200_cuboid_set *cuboids,
    const cb200_voxel_set *voxels, const float *weight, const float *activation_distance,
    const int32_t *env_query_idx, int batch_size, int horizon, int num_spheres, int use_multi_env,
    cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * (a12) swept sphere vs scene + optional speed metric (one launch).
 * Replaces SweptSphereObstacleCollision.forward  curobo/_src/geom/collision/wp_autograd.py:124-247
 *   (Warp kernels swept_sphere_obstacle_collision_kernel wp_sweep_collision_kernel.py:83-260 and
 *    apply_speed_metric wp_speed_metric.py:10-93).  speed_dt is a 1-element device array.
 * ------------------------------------------------------------------------------------------- */
int cb200_swept_sphere_obstacle_collision(
    float *distance, float *gradient, const float *spheres, const cb200_cuboid_set *cuboids,
    const cb200_voxel_set *voxels, const float *weight, const float *activation_distance,
    const float *speed_dt, int enable_speed_metric, const int32_t *env_query_idx, int batch_size,
    int horizon, int num_spheres, int use_multi_env, cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * (a13) goal-set tool-pose cost.  Replaces ToolPoseDistance.forward
 *   curobo/_src/cost/wp_tool_pose.py:698-855 (Warp kernel goalset_pose_distance_* :457-692).
 * rotation_method: 0 axis-angle, 1 Lie group.  project_distance_to_goal must be all zero.
 * ------------------------------------------------------------------------------------------- */
int cb200_tool_pose_distance(
    float *out_distance, float *out_position_distance, float *out_rotation_distance,
    float *out_position_gradient, float *out_rotation_gradient, int32_t *out_goalset_idx,
    const float *current_position, const float *current_quat, const float *goal_position,
    const float *goal_quat, const int32_t *idxs_goal, const float *position_orientation_weight,
    const float *terminal_pose_axes_weight_factor, const float *non_terminal_pose_axes_weight_factor,
    const float *terminal_pose_convergence_tolerance,
    const float *non_terminal_pose_convergence_tolerance, int batch_size, int horizon,
    int num_links, int num_goalset, int rotation_method, cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * (a14) c-space costs.
 * cb200_cspace_state_cost replaces StateCSpaceFunction.forward's kernel launch
 *   curobo/_src/cost/wp_cspace_state.py:21-285 (forward_cspace_state_warp).
 * cb200_cspace_position_cost replaces forward_cspace_position_warp
 *   curobo/_src/cost/wp_cspace_position.py:232-362.
 * Limits are [2, D] (lower row, upper row); weight/activation/regularisation arrays as in the
 * reference (5 / 5 / 5 entries for STATE; 2 / 2 / 2 for POSITION).
 * ------------------------------------------------------------------------------------------- */
int cb200_cspace_state_cost(
    float *out_cost, float *out_grad_p, float *out_grad_v, float *out_grad_a, float *out_grad_j,
    float *out_grad_tau, const float *pos, const float *vel, const float *acc, const float *jerk,
    const float *effort, const float *state_dt, const float *target_joint_position,
    const int32_t *idxs_target_joint_position, const float *p_b, const float *v_b, const float *a_b,
    const float *j_b, const float *effort_b, const float *weight, const float *activation_distance,
    const float *squared_l2_regularization_weights, const float *cspace_target_weight,
    const float *cspace_non_terminal_weight_factor, const float *cspace_target_dof_weight,
    int write_grad, int batch_size, int horizon, int dof, int retime_weights,
    int retime_regularization_weights, cb200_stream_t stream);

int cb200_cspace_position_cost(
    float *out_cost, float *out_grad_p, float *out_grad_tau, const float *pos, const float *effort,
    const float *cspace_target, const int32_t *cspace_target_idx, const float *p_b,
    const float *effort_b, const float *weight, const float *activation_distance,
    const float *cspace_target_weight, const float *cspace_target_dof_weight,
    const float *squared_l2_reg_weight, const float *current_position, const float *current_velocity,
    const int32_t *idxs_current_state, const float *v_b, const float *state_dt, int write_grad,
    int batch_size, int horizon, int dof, cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * (a16/a17) THE FUSED HOT PATH: one launch = FK -> spheres -> {self, scene, tool-pose, c-space}
 * cost -> J^T gradient, for every (seed x waypoint) row of q [B, H, D].
 * Replaces the whole of  RobotRollout.evaluate_action + cost.backward()
 *   curobo/_src/rollout/rollout_robot.py:252-263, rollout/cost_manager/cost_manager_robot.py:195-286,
 *   optim/components/gradient_opt_core.py:445-480
 * (15-25 launches + 4 streams in the reference).  Robot constants live in one packed device blob
 * (cb200_robot_blob_*), staged into shared memory by a single bulk async copy per CTA.
 * ------------------------------------------------------------------------------------------- */

/* Size in bytes of the packed robot blob for the given sizes (host helper; 16-byte multiple). */
typedef struct {
  int32_t num_links, num_dof, num_spheres, num_tool_frames, num_pairs;
  int32_t num_sphere_configs; /* 0 or 1: link_spheres is [S,4]; n > 1: [n,S,4] (config 0 is staged, bounds cover all) */
} cb200_robot_sizes;

typedef struct {
  /* weights / switches (value semantics: 0 weight disables a term) */
  float self_weight;
  float scene_weight, scene_activation;
  int32_t use_sweep, use_speed_metric;
  float pose_weight[2];
  int32_t pose_rotation_method;        /* 0 axis-angle, 1 Lie */
  int32_t cspace_type;                 /* 0 off, 1 POSITION, 2 STATE */
  float cspace_weight[5], cspace_activation[5], cspace_reg[5];
  int32_t retime_weights, retime_regularization_weights;
  int32_t num_goalset;
  /* c-space target term (cost/wp_cspace_state.py:84-89,220-226; cost/wp_cspace_position.py target block): adds
   * w_d * (q_d - target[idxs_cspace_target[b], d])^2 with w_d = cspace_target_weight * cspace_target_dof_weight[d];
   * STATE cost: non-terminal waypoints (h < H-1) scale the weight by cspace_non_terminal_weight_factor
   * (content/configs/task/mpc/lbfgs_mpc.yml:28-29).  Needs io->cspace_target; 0 disables. */
  float cspace_target_weight, cspace_non_terminal_weight_factor;
} cb200_rollout_cfg;

/* Optional B-spline front end of the fused rollout (SURVEY.md 8f rank 1): the rows of the rollout are the
 * spline states of `knots`, evaluated inside the kernel (q, qd, qdd, qddd never touch HBM), and the adjoint runs
 * right behind it on the same stream, so one C call maps  knots -> cost, grad_knots.
 * Semantics of every field = cb200_bspline_forward / cb200_bspline_backward below; io->horizon is the padded
 * horizon (n_knots + degree + 1) * interpolation_steps + 1 and io->q/vel/acc/jerk/dt are ignored. */
typedef struct {
  const float *knots;                                          /* [B, n_knots, D] */
  const float *start_position, *start_velocity, *start_acceleration, *start_jerk; /* [n_start, D] */
  const float *goal_position, *goal_velocity, *goal_acceleration, *goal_jerk;     /* [n_goal, D] */
  const int32_t *start_idx, *goal_idx;                         /* [B] */
  const float *traj_dt;                                        /* [n_goal] */
  const uint8_t *use_implicit_goal_state;                      /* [n_goal] */
  int32_t n_knots, degree;
  float *grad_knots;                                           /* out [B, n_knots, D]; needs io->grad_vel/acc/jerk */
  float *out_position, *out_velocity, *out_acceleration, *out_jerk; /* optional state buffers [B,H,D] */
  float *out_dt;                                               /* optional [B] */
  /* Two schedules, same results to float rounding (tests/test_gpu_bspline.py):
   *   all five out_* given  -> "expanded": spline kernel -> rollout kernel -> adjoint kernel (3 launches; the state
   *                            makes one 4*B*H*D*4-byte round trip through L2) -- the faster one at every measured size;
   *   otherwise             -> "in-kernel": the rollout kernel evaluates each row from the knots (2 launches; state
   *                            never leaves the SM; out_position.. are then optional dumps). */
} cb200_spline_input;

/* Optional inverse dynamics inside the trajectory kernel (SURVEY.md 8f rank 3; reference: joint_torque =
 * robot_dynamics.compute_inverse_dynamics(state), transition/robot_state_transition.py:380-389, consumed by the effort
 * channel of the STATE c-space cost, cost/wp_cspace_state.py:209-275).  When io->dynamics is given (swept / trajectory mode,
 * STATE c-space cost, io->vel and io->acc present) every row evaluates tau = RNEA(q, qd, qdd) on chip, adds the effort terms
 * (bound hinge with the blob's effort limits, cspace_weight[4] / cspace_activation[4]; squared-L2 cspace_reg[3]; energy
 * cspace_reg[4]) to cost / cspace_cost and their gradients -- through the RNEA adjoint -- to grad_q / grad_vel / grad_acc.
 * DEVICE pointers; layouts as in cb200_rnea_forward. */
typedef struct {
  const float *link_masses_com;   /* [nl,4] cx,cy,cz,m */
  const float *link_inertias;     /* [nl,8] ixx,iyy,izz,ixy,ixz,iyz,pad,pad */
  const float *gravity;           /* [6] spatial */
} cb200_dynamics_params;

typedef struct {
  /* inputs */
  const float *q;                 /* [B,H,D] */
  const float *vel, *acc, *jerk;  /* [B,H,D] or null (STATE c-space only) */
  const float *dt;                /* [B] or null */
  const void *robot_blob;         /* DEVICE copy of the blob packed by cb200_pack_robot_blob */
  const void *robot_blob_host;    /* HOST copy of the same blob (its 192-byte header is read on the host) */
  int32_t robot_blob_bytes;
  const cb200_cuboid_set *cuboids; /* host pointers to structs holding device pointers; may be null */
  const cb200_voxel_set *voxels;
  const int32_t *env_query_idx;   /* [B] or null */
  const float *goal_position;     /* [G, L, n_goalset, 3] or null */
  const float *goal_quat;         /* [G, L, n_goalset, 4] wxyz */
  const int32_t *idxs_goal;       /* [B] */
  const float *pose_axes_terminal, *pose_axes_non_terminal; /* [L,6] or null (=1) */
  const float *pose_tol_terminal, *pose_tol_non_terminal;   /* [L,2] or null (=0) */
  /* outputs (any may be null except grad_q and cost) */
  float *cost;          /* [B,H]  sum of all terms for the row */
  float *grad_q;        /* [B,H,D] */
  float *self_cost;     /* [B,H] */
  float *scene_cost;    /* [B,H,S] */
  float *pose_cost;     /* [B,H,2L] */
  float *cspace_cost;   /* [B,H,D] */
  float *grad_vel, *grad_acc, *grad_jerk; /* [B,H,D] (STATE c-space) */
  float *link_pos, *link_quat;            /* optional FK outputs [B,H,L,3/4] */
  float *robot_spheres;                   /* optional [B,H,S,4] */
  int32_t *pose_goalset_idx;              /* optional [B,H,L] */
  int32_t batch_size, horizon;
  const cb200_spline_input *spline;       /* optional B-spline front end (host pointer); NULL = rows come from q */
  const cb200_dynamics_params *dynamics;  /* optional (host pointer): dynamics-aware STATE cost, see cb200_dynamics_params */
  /* c-space target (retract / MPC reference configuration), read when cfg->cspace_target_weight > 0 */
  const float *cspace_target;             /* [n_target, D] or null */
  const int32_t *idxs_cspace_target;      /* [B] rows of cspace_target; null = row 0 */
  const float *cspace_target_dof_weight;  /* [D] or null (= 1) */
  /* link-sphere configurations (attached objects per environment; kinematics_forward_helper.cuh:232-233): row b uses
   * sphere_configs[env_query_idx[b]] instead of the blob's set when num_sphere_configs > 1.  The blob must have been
   * packed with the same configurations (cb200_robot_sizes.num_sphere_configs) so its broad-phase bounds cover all. */
  const float *sphere_configs;            /* [num_sphere_configs, S, 4] or null */
  int32_t num_sphere_configs;
  /* Row ticket counter of the big-robot (humanoid) kernel: int32[2], zero on entry, zero again when the launch has finished
   * (the kernel re-arms it), owned by ONE stream at a time -- concurrent launches need one counter each.  Null: rows are
   * strided statically over the resident warps. */
  int32_t *work_counter;
  /* Mesh obstacles, next to `cuboids` / `voxels` (host pointer to a struct of device pointers); NULL = none.  Read when
   * cfg->scene_weight > 0 and meshes->inv_pose is set; discrete and swept collision against them run inside the fused kernels
   * with the arithmetic of cb200_sphere_mesh_collision.  The in-kernel B-spline schedule and `dynamics` have no mesh support:
   * with meshes present they return cudaErrorInvalidValue (the expanded spline schedule supports meshes). */
  const cb200_mesh_set *meshes;
  /* Current state of the POSITION c-space cost (velocity-aware IK, the local IK of motion retargeting;
   * cost/wp_cspace_position.py:299-356, fed from GoalRegistry.current_js / idxs_current_js / current_state_dt).  Seed b reads
   * row c = idxs_current_state[b]; when current_state_dt[c] > 0 every waypoint of the seed gets
   *   - position bounds shrunk by cspace_activation[0], then intersected with what one step reaches:
   *     [max(p_l, current_position[c] + v_l*dt), min(p_u, current_position[c] + v_u*dt)] (v_l, v_u: the blob's velocity limits),
   *     hinged with activation 0 (an empty window hinges on both sides, as the reference does);
   *   - 0.5*cspace_reg[0]*dt*v^2 with v = (q - current_position[c]) / dt, and
   *   - 0.5*cspace_reg[1]*dt^2*a^2 with a = (v - current_velocity[c]) / dt.
   * Rows whose dt <= 0, and every row when current_position is NULL, get the plain bound hinge, bit for bit.  Read by
   * cb200_rollout_cost_grad and cb200_rollout_cost when cfg->cspace_type == 1 (POSITION); the STATE cost ignores them. */
  const float *current_position;          /* [n_cur, D] or null (= off) */
  const float *current_velocity;          /* [n_cur, D] or null (= 0) */
  const int32_t *idxs_current_state;      /* [B] rows of current_position; null = row 0 */
  const float *current_state_dt;          /* [n_cur]; required with current_position (else cudaErrorInvalidValue) */
} cb200_rollout_io;

int cb200_rollout_cost_grad(const cb200_rollout_cfg *cfg, const cb200_rollout_io *io,
                            cb200_stream_t stream);

/* Cost without gradient: the rows and every cost output of cb200_rollout_cost_grad (cost required; the term costs and the FK
 * outputs optional), from kernels that skip the J^T backward and everything else only the gradient reads -- what a
 * sampling-based optimizer (MPPI) evaluates.  grad_q, grad_vel, grad_acc and grad_jerk are ignored and may be NULL.
 * Covers discrete rows from io->q: use_sweep, a spline front end or dynamics return cudaErrorInvalidValue, as do a NULL
 * cost, robot_blob or q.  cb200_last_rollout_variant() reports the variant of the kernel it twins | CB200_VARIANT_COST_ONLY. */
int cb200_rollout_cost(const cb200_rollout_cfg *cfg, const cb200_rollout_io *io, cb200_stream_t stream);

/* Validity of joint configurations (the reference's RobotSceneCollision.validate, collision_robot_scene.py:341-372): valid[b,h] = 1
 * iff every check asked for holds, else 0.
 *   check_bounds: position limits of the blob, lower[d] <= q[d] <= upper[d] (the POSITION c-space bound cost at weight 1 and
 *                 activation 0 is exactly 0);
 *   check_self:   no pair of the self-collision pair list with both padded radii >= 0 overlaps, (r_i + r_j)^2 - |p_i - p_j|^2 > 0;
 *   check_scene:  no sphere with r >= 0 touches an enabled obstacle of the row's environment, r - sdf > 0 (cuboids, ESDF grids
 *                 and meshes with the SDF arithmetic of the fused kernels; env_query_idx and sphere_configs apply as there).
 * H > 1 rows are independent discrete rows (no sweep).  One persistent warp per row; a row stops at its first failed check
 * (bounds before FK, then scene, then self), which changes the time it takes, never its verdict.
 * Reads only q, robot_blob, robot_blob_host, robot_blob_bytes, cuboids, voxels, meshes, env_query_idx, sphere_configs,
 * num_sphere_configs, work_counter, batch_size and horizon; every cost and gradient field is ignored.  Returns
 * cudaErrorInvalidValue for a NULL valid, io, q or robot_blob, and when spline, dynamics or current_position is set.
 * cb200_last_rollout_variant() reports CB200_VARIANT_VALIDATE.  Allocates nothing and never synchronises (graph-capturable). */
int cb200_rollout_validate(const cb200_rollout_io *io, uint8_t *valid /* [B,H] */, int32_t check_bounds, int32_t check_self,
                           int32_t check_scene, cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * (8f-1) B-spline knot -> state kernels and their adjoint: the step in front of / behind the rollout
 * on the trajopt / MPC path.  Argument order and meaning are the reference launchers':
 *   cb200_bspline_forward    <- launch_bspline_interpolation_forward_kernel
 *       curobo/_src/curobolib/backends/cuda_core_backend/trajectory.py:25-137
 *       (pybind twin: backends/pybind/trajectory_kernel_launch.cu:263-404)
 *   cb200_bspline_single_dt  <- launch_bspline_interpolation_single_dt_kernel  trajectory.py:213-330
 *   cb200_bspline_backward   <- launch_bspline_interpolation_backward_kernel   trajectory.py:140-210
 * u_position [B, n_knots, D]; start_* / goal_* [n_start|n_goal, D] gathered through start_idx / goal_idx [B];
 * traj_dt and use_implicit_goal_state are [n_goal] and indexed through goal_idx (dt_idx in the adjoint);
 * outputs [B, padded_horizon, D] with padded_horizon = (n_knots + degree + 1) * interpolation_steps + 1.
 * degree in {3,4,5} (MATRIX basis).  The adjoint returns cudaErrorInvalidValue where the reference launcher
 * throws (horizon < 5, interpolation_steps == 0 or > 32, unsupported degree).
 * ------------------------------------------------------------------------------------------- */
int cb200_bspline_forward(
    float *out_position, float *out_velocity, float *out_acceleration, float *out_jerk, float *out_dt,
    const float *u_position, const float *start_position, const float *start_velocity,
    const float *start_acceleration, const float *start_jerk, const float *goal_position,
    const float *goal_velocity, const float *goal_acceleration, const float *goal_jerk,
    const int32_t *start_idx, const int32_t *goal_idx, const float *traj_dt,
    const uint8_t *use_implicit_goal_state, int batch_size, int padded_horizon, int dof, int n_knots,
    int bspline_degree, cb200_stream_t stream);

int cb200_bspline_single_dt(
    float *out_position, float *out_velocity, float *out_acceleration, float *out_jerk, float *out_dt,
    const float *u_position, const float *knot_dt, const float *start_position,
    const float *start_velocity, const float *start_acceleration, const float *start_jerk,
    const float *goal_position, const float *goal_velocity, const float *goal_acceleration,
    const float *goal_jerk, const int32_t *start_idx, const int32_t *goal_idx,
    const float *interpolation_dt, const uint8_t *use_implicit_goal_state,
    const int32_t *interpolation_horizon, int batch_size, int max_out_tsteps, int dof, int n_knots,
    int bspline_degree, cb200_stream_t stream);

int cb200_bspline_backward(
    float *out_grad_knots, const float *grad_position, const float *grad_velocity,
    const float *grad_acceleration, const float *grad_jerk, const float *traj_dt,
    const int32_t *dt_idx, const uint8_t *use_implicit_goal_state, int batch_size, int padded_horizon,
    int dof, int n_knots, int bspline_degree, cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * Position (clique) and acceleration control spaces: the reference's legacy state transitions
 * (kernels/trajectory/legacy/).  Argument order and meaning are the reference launchers':
 *   cb200_position_clique_forward  <- launch_differentiation_position_forward_kernel
 *       curobo/_src/curobolib/backends/cuda_core_backend/trajectory.py:309-393
 *       (pybind twin: backends/pybind/trajectory_kernel_launch.cu:26-107)
 *   cb200_position_clique_backward <- launch_differentiation_position_backward_kernel  trajectory.py:396-465
 *   cb200_acceleration_integrate   <- launch_integration_acceleration_kernel           trajectory.py:468-560
 * Clique: u_position [B, H-4, D] -> position / velocity / acceleration / jerk [B, H, D] by the 5-point stencil,
 * padded with the start state before the first action and with the last action (or, where
 * use_implicit_goal_state[goal_idx[b]], the goal position) after it; out_dt [B] = traj_dt[goal_idx[b]].
 * start_* / goal_* are gathered at flat offsets start_idx[b] * D / goal_idx[b] * D.  The adjoint maps the four
 * [B, H, D] gradients to out_grad_position [B, H-4, D]; dt and the goal mode come through dt_idx[b].
 * Both return cudaErrorInvalidValue for horizon < 8 (the reference's first rows read actions 0..3 whatever the
 * horizon).
 * Acceleration: u_acc [B, H, D] -> the four state tensors [B, H, D] by semi-implicit Euler with dt[h] = traj_dt[h]
 * ([H], indexed by waypoint); the start state comes through start_idx.  use_rk2 selects a kernel with identical
 * arithmetic in the reference and is accepted for either value.  No horizon limit.
 * batch_size == 0 returns cudaSuccess without launching.
 * ------------------------------------------------------------------------------------------- */
int cb200_position_clique_forward(
    float *out_position, float *out_velocity, float *out_acceleration, float *out_jerk, float *out_dt,
    const float *u_position, const float *start_position, const float *start_velocity,
    const float *start_acceleration, const float *goal_position, const float *goal_velocity,
    const float *goal_acceleration, const int32_t *start_idx, const int32_t *goal_idx, const float *traj_dt,
    const uint8_t *use_implicit_goal_state, int batch_size, int horizon, int dof, cb200_stream_t stream);

int cb200_position_clique_backward(
    float *out_grad_position, const float *grad_position, const float *grad_velocity,
    const float *grad_acceleration, const float *grad_jerk, const float *traj_dt, const int32_t *dt_idx,
    const uint8_t *use_implicit_goal_state, int batch_size, int horizon, int dof, cb200_stream_t stream);

int cb200_acceleration_integrate(
    float *out_position, float *out_velocity, float *out_acceleration, float *out_jerk, const float *u_acc,
    const float *start_position, const float *start_velocity, const float *start_acceleration,
    const int32_t *start_idx, const float *traj_dt, int batch_size, int horizon, int dof, int use_rk2,
    cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * (8f-2) Optimizer-side kernels of the solve loop: the L-BFGS step and the parallel Wolfe line search
 * that sit either side of the rollout in every optimizer iteration.
 *   cb200_lbfgs_step   <- launch_lbfgs_step
 *       curobo/_src/curobolib/backends/cuda_core_backend/optimization.py:136-246
 *       (kernels/optimization/lbfgs/lbfgs_step_kernel.cuh:39-199)
 *   cb200_line_search  <- launch_line_search  cuda_core_backend/optimization.py:26-133
 *       (kernels/optimization/line_search/line_search_kernel.cuh:60-199)
 * Buffers and meaning as in the reference: rho [m,B], y/s [m,B,V] (rolled in place, newest pair in slot m-1),
 * q / grad_q / x_0 / grad_0 / step_vec [B,V]; search_* [B,n,(V)], idx outputs [B,n], iterations int16, converged u8.
 * 1 <= history_m <= 31, v_dim <= 1024, n_linesearch <= 32 (cudaErrorInvalidValue otherwise, where the reference raises).
 * Extension (all optional, pass NULL/0 to get the reference kernel's behaviour exactly): the step kernel also
 * prepares the line search the way LineSearchStrategy._prepare_search_points does
 * (optim/gradient/line_search_strategy.py:136-240): step_scaled = scale_action(step) with per-dimension
 * action_step_max [action_dim] (and the terminal action frozen when fix_terminal_action), and
 * x_set[b,j,:] = q[b,:] + search_magnitudes[j] * step_scaled[b,:].
 * ------------------------------------------------------------------------------------------- */
int cb200_lbfgs_step(
    float *step_vec, float *rho_buffer, float *y_buffer, float *s_buffer, const float *q,
    const float *grad_q, float *x_0, float *grad_0, float epsilon, int batch_size, int history_m,
    int v_dim, int stable_mode, float *x_set, float *step_scaled, const float *search_magnitudes,
    int n_linesearch, const float *action_step_max, int action_dim, int fix_terminal_action,
    cb200_stream_t stream);

int cb200_line_search(
    float *best_cost, float *best_action, int16_t *best_iteration, int16_t *current_iteration,
    uint8_t *converged_global, int convergence_iteration, float cost_delta_threshold,
    float cost_relative_threshold, float *exploration_cost, float *exploration_action,
    float *exploration_gradient, int32_t *exploration_idx, float *selected_cost,
    float *selected_action, float *selected_gradient, int32_t *selected_idx, const float *search_cost,
    const float *search_action, const float *search_gradient, const float *step_direction,
    const float *search_magnitudes, float armijo_threshold_c_1, float curvature_threshold_c_2,
    int strong_wolfe, int approx_wolfe, int n_linesearch, int opt_dim, int batchsize,
    cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * MPPI particle stage (DIAG_A covariance, CLAMP squash): the two launches either side of the cost-only rollout in
 * every inner iteration of the reference's MPPI (optim/particle/mppi.py, optim/components/particle_opt_core.py).
 *   cb200_mppi_sample  <- ParticleOptCore.sample_actions (particle_opt_core.py:409-441)
 *       actions [P, Np, H, D]: per problem num_sampled particles mean + noise * scale, then num_neg copies of -mean, then
 *       zeros; every element clamped to max(min(a, highs[d]), lows[d]).  mean [P, H, D], scale [P, D] (the DIAG_A
 *       scale_tril), noise [P, num_sampled, H, D], or [1, num_sampled, H, D] shared by every problem when
 *       noise_per_problem == 0; lows / highs [D].  Bit-equal to the reference's torch (mul, then add).
 *   cb200_mppi_update  <- MPPI._update_distribution + jit_mean_cov_diag_a (mppi.py:200-248, 722-757), in place
 *       cost [P * Np, H] (the cost-only rollout's per-row cost); total = discount * sum_h cost, discount =
 *       sum_h gamma^h / gamma^0 (the reference broadcasts gamma_seq over the horizon-summed cost);
 *       w = softmax(-total / beta); when best_mode, best [P, H, D] = the particle of largest w (lowest index on ties);
 *       when update_cov, cov [P, D] = (1 - step_size_cov) cov + step_size_cov mean_h sum_p w (a - mean_old)^2 + kappa
 *       and scale = sqrt(cov); mean = (1 - step_size_mean) mean + step_size_mean sum_p w a.
 *       Np + H * D <= 12288.  Sums run in a fixed order: repeated calls are bit-identical.
 * num_problems == 0 launches nothing; bad sizes or null pointers return cudaErrorInvalidValue.
 * ------------------------------------------------------------------------------------------- */
int cb200_mppi_sample(
    float *actions, const float *mean, const float *scale, const float *noise, const float *lows,
    const float *highs, int num_problems, int num_particles, int num_sampled, int num_neg, int horizon,
    int action_dim, int noise_per_problem, cb200_stream_t stream);

int cb200_mppi_update(
    const float *actions, const float *cost, float *mean, float *cov, float *scale, float *best,
    int num_problems, int num_particles, int horizon, int action_dim, float beta, float step_size_mean,
    float step_size_cov, float kappa, float discount, int update_cov, int best_mode, cb200_stream_t stream);

/* -------------------------------------------------------------------------------------------
 * (8f-3) RNEA inverse dynamics and its adjoint: tau = RNEA(q, qd, qdd [, f_ext]) feeds the effort terms of the STATE
 * c-space cost; the adjoint maps d loss / d tau back to (q, qd, qdd).
 *   cb200_rnea_forward   <- launch_rnea_forward   curobo/_src/curobolib/backends/cuda_core_backend/dynamics.py:24-131
 *                           (kernels/dynamics/rnea_forward_kernel.cuh:54-285)
 *   cb200_rnea_backward  <- launch_rnea_backward  cuda_core_backend/dynamics.py:134-250
 *                           (kernels/dynamics/rnea_backward_kernel.cuh:60-460)
 * Same tensors and meaning: q/qd/qdd/tau/grads [B, num_dof]; fixed_transforms [nl,3,4]; link_masses_com [nl,4]
 * (cx,cy,cz,m); link_inertias [nl,8] (ixx,iyy,izz,ixy,ixz,iyz,pad,pad at the CoM); gravity [6] spatial; level_starts
 * [n_levels+1] / level_links [nl] = CSR of links by tree depth; forward_cache [B, nl, 20] (v, a, f per link; the same
 * layout as the reference's, so either side can consume the other's).  The reference's threads_per_batch knob has no
 * equivalent (the launcher picks rows / workers per CTA itself; sums keep the reference's serial order).  Gradients are
 * overwritten.  level arrays must be depth levels (children of a level-l link are level-(l+1) links).
 * ------------------------------------------------------------------------------------------- */
int cb200_rnea_forward(
    float *tau, const float *q, const float *qd, const float *qdd, const float *fixed_transforms,
    const float *link_masses_com, const float *link_inertias, const int8_t *joint_map_type,
    const int16_t *joint_map, const int16_t *link_map, const float *joint_offset_map,
    const float *gravity, const int16_t *level_starts, const int16_t *level_links,
    float *forward_cache, int batch_size, int num_links, int num_dof, int n_levels,
    const float *f_ext, cb200_stream_t stream);

int cb200_rnea_backward(
    float *grad_q, float *grad_qd, float *grad_qdd, const float *grad_tau, const float *q,
    const float *qd, const float *fixed_transforms, const float *link_masses_com,
    const float *link_inertias, const int8_t *joint_map_type, const int16_t *joint_map,
    const int16_t *link_map, const float *joint_offset_map, const float *gravity,
    const int16_t *level_starts, const int16_t *level_links, const float *forward_cache,
    int batch_size, int num_links, int num_dof, int n_levels, float *grad_f_ext,
    cb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * (8f-4) Exact 3-D nearest-site transform (Euclidean distance transform), the producer side of the ESDF wire format.
 *   cb200_pba3d  <- launch_pba3d  cuda_core_backend/pba.py:60-124  (kernels/parallel_banding/pba3d_kernel.cuh,
 *                   driven by perception/mapper/esdf/edt_parallel_banding.py:63-80)
 * site_index [nx, ny, nz] int32, z contiguous: a site holds its own packed coordinates (z << 20) | (y << 10) | x
 * (perception/mapper/util/utils_quantization.py:40-54), anything negative is "no site".  In place: afterwards every
 * voxel holds the packed coordinates of a nearest site (exact; which of several equidistant sites is unspecified, as in
 * the reference where it depends on the sweep order), or 0x80000000 when the grid holds no site.  nx, ny, nz <= 1023.
 * `buffer` (the reference's ping-pong scratch) and `m3` (its colour-kernel block height) are accepted and unused.
 *   cb200_edt_unsigned_distance: fp16(|voxel - site| * voxel_size) per voxel, fp16(empty_value) where no site exists --
 *   the distance step of compute_esdf_from_min_tsdf (kernel/builder/builder_esdf.py:434-446) without the TSDF sign.
 * ------------------------------------------------------------------------------------------- */
int cb200_pba3d(int32_t *site_index, int32_t *buffer, int nx, int ny, int nz, int m3, cb200_stream_t stream);

int cb200_edt_unsigned_distance(const int32_t *site_index, uint16_t *distance_fp16, int nx, int ny, int nz,
                                float voxel_size, float empty_value, cb200_stream_t stream);
/* The stages either side of the transform in BlockSparseESDFIntegrator._compute_esdf_impl (perception/mapper/integrator_esdf.py:
 * 640-704) for a DENSE signed-distance source at the ESDF's own resolution ([nx, ny, nz] f32, z contiguous, > 1e9 = unobserved;
 * the reference reads its block-sparse TSDF through a hash table at the same places):
 *   cb200_esdf_seed_sites       <- seed_esdf_sites_gather_kernel  kernel/builder/builder_esdf.py:308-404 (seed rule :255-261):
 *                                  site = own packed coordinates where |sdf| <= 0.9 voxel or sdf < -(truncation - 1.1 voxel),
 *                                  -1 elsewhere (every voxel is written: no pre-clear).
 *   cb200_esdf_signed_distance  <- compute_esdf_from_min_tsdf_kernel  builder_esdf.py:410-503: fp16(+-|voxel - site| * voxel),
 *                                  sign from the static SDF one `adjacent_skip_steps` step from the site towards the voxel
 *                                  (dist > 1 voxel), else from the combined SDF at the voxel, unsigned when both are
 *                                  unobserved; fp16(1e4) where the grid has no site.  Either SDF pointer may be NULL. */
int cb200_esdf_seed_sites(const float *combined_sdf, int32_t *site_index, int nx, int ny, int nz, float voxel_size,
                          float truncation_distance, cb200_stream_t stream);
/*   cb200_esdf_seed_sites_gather <- seed_esdf_sites_gather_kernel  builder_esdf.py:308-404 (the reference's default,
 *                                  mapper_cfg.py:103): the same rule probed at the voxel centre and half a voxel away along each
 *                                  axis (7 probes, _check_seed_at_world_pos :267-306), world -> voxel by int((w - origin) / voxel +
 *                                  n / 2) in IEEE float32 in the reference's order, so the dilated band is the reference's band.
 *                                  `origin` = grid centre (3 floats, host).  ESDF grid == TSDF grid (the dense case). */
int cb200_esdf_seed_sites_gather(const float *combined_sdf, int32_t *site_index, int nx, int ny, int nz, float voxel_size,
                                 float truncation_distance, const float *origin, cb200_stream_t stream);
int cb200_esdf_signed_distance(const int32_t *site_index, const float *static_sdf, const float *combined_sdf,
                               uint16_t *distance_fp16, int nx, int ny, int nz, float voxel_size, float adjacent_skip_steps,
                               cb200_stream_t stream);
/* Depth images -> TSDF -> combined SDF, the stage in front of the seeding, for the same DENSE grid:
 *   cb200_tsdf_integrate_depth  <- integrate_voxels_kernel  kernel/builder/builder_camera_integrate.py:399-489 (phase 4 of
 *                                  CameraProjectIntegrator, kernel/wp_integrate_camera_project.py:27-41): one thread per voxel,
 *                                  serial camera loop: voxel centre ((idx + 0.5 - n / 2) voxel + origin, builder_coord.py:57-66)
 *                                  into the camera frame (quaternion wxyz = camera -> world), pinhole projection, pixel index by
 *                                  truncation, depth within [depth_min, depth_max], sdf = depth - z_cam kept when >= -truncation
 *                                  and clamped to +truncation, weight = max((fx voxel / z)(fy voxel / z), 1)
 *                                  (compute_tsdf_weight == 1, kernel/wp_integrate_common.py:57-105);
 *                                  block_data[voxel] = fp16 pair (sum sdf * w, sum w), accumulated in fp32, rounded once per call.
 *                                  The block discovery / allocation phases of the block-sparse store are out of scope.
 *   cb200_tsdf_combined_sdf     <- sample_combined_sdf  kernel/wp_tsdf_sample.py:22-97: sum_sdf_w / sum_w where the weight exceeds
 *                                  min_weight, else 1e10; min with static_sdf (may be NULL).  Output feeds cb200_esdf_seed_sites. */
int cb200_tsdf_integrate_depth(uint16_t *block_data_fp16, int nx, int ny, int nz, float voxel_size, const float *origin /* host [3] */,
                               int num_cameras, const float *intrinsics /* [C,3,3] */, const float *cam_positions /* [C,3] */,
                               const float *cam_quaternions /* [C,4] wxyz */, const float *depth_images /* [C,H,W] */,
                               int image_height, int image_width, float depth_min, float depth_max, float truncation_distance,
                               cb200_stream_t stream);
int cb200_tsdf_combined_sdf(const uint16_t *block_data_fp16, const float *static_sdf, float *combined_sdf, long long num_voxels,
                            float min_weight, cb200_stream_t stream);
/* Robot pixels of depth images, masked in front of cb200_tsdf_integrate_depth (same camera model, quaternion convention and
 * depth layout):
 *   cb200_segment_robot_depth   <- RobotSegmenter._mask_op  perception/robot_segmenter.py:267-366 with get_projection_rays /
 *                                  project_depth_using_rays  geom/cv.py:47-157 and _mask_spheres_image_cdist.  Pixel (u, v) at
 *                                  integer coordinates: p_cam = ((u - cx) / fx d, (v - cy) / fy d, d) (IEEE divisions),
 *                                  p = R(q) p_cam + t.  mask = d > 0 and |p - c_s| < r_s + distance_threshold for some sphere s
 *                                  (the reference's max_s(r_s - |p - c_s|) > -distance_threshold); a sphere with
 *                                  r_s + distance_threshold <= 0 (a disabled sphere at radius -100) never masks, nor does a pixel
 *                                  with non-finite depth.  d > 0 is decided on the bits, so a subnormal positive depth counts
 *                                  although the library flushes subnormals to zero (its point is then the camera position).
 *                                  filtered = mask ? 0 : depth, every other pixel copied bit for bit.
 *                                  robot_spheres [robot_batch, S, 4], robot_batch 1 (one state for every image) or B.  Refused
 *                                  (nothing launched): a NULL pointer, robot_batch neither 1 nor B, S spheres beyond the shared-
 *                                  memory opt-in (16 bytes each), more than 2^31 - 1 tiles of 32 x 8 pixels in all. */
int cb200_segment_robot_depth(const float *depth /* [B,H,W] metres */, int batch, int height, int width,
                              const float *intrinsics /* [B,3,3] */, const float *cam_positions /* [B,3] */,
                              const float *cam_quaternions /* [B,4] wxyz, camera -> robot base */,
                              const float *robot_spheres /* [Bs,S,4], Bs == 1 or B */, int robot_batch, int num_spheres,
                              float distance_threshold, uint8_t *mask /* [B,H,W] */, float *filtered /* [B,H,W] */,
                              cb200_stream_t stream);
/*   cb200_tsdf_stamp_cuboids   <- stamp_sdf_kernel  kernel/builder/builder_stamp.py:263-315 with the cuboid overloads of
 *                                  geom/data/data_cuboid.py:461-545 (the per-voxel step of BlockSparseTSDFIntegrator's obstacle
 *                                  stamping; block enumeration / allocation out of scope): static_sdf (f32, > 1e9 = nothing
 *                                  stamped, updated in place) takes clamp(min(existing, min over enabled cuboids of the box SDF
 *                                  at the voxel centre), +-truncation), rounded through fp16, where |min| <= truncation. */
int cb200_tsdf_stamp_cuboids(float *static_sdf, int nx, int ny, int nz, float voxel_size, const float *origin /* host [3] */,
                             float truncation_distance, const cb200_cuboid_set *cuboids, int env_idx, cb200_stream_t stream);

/* Host helper: pack robot constants (HOST pointers) into `out` (host buffer of
 * cb200_robot_blob_bytes(...) bytes) that the caller then copies to the device once.
 * Returns bytes written or a negative number on invalid input. */
int64_t cb200_robot_blob_bytes(const cb200_robot_sizes *sz);
int64_t cb200_pack_robot_blob(
    void *out, int64_t out_bytes, const cb200_robot_sizes *sz, const float *fixed_transforms,
    const int16_t *link_map, const int16_t *joint_map, const int8_t *joint_map_type,
    const float *joint_offset_map, const int16_t *tool_frame_map, const float *link_spheres,
    const int16_t *link_sphere_map, const float *sphere_padding, const int16_t *collision_pairs,
    const float *position_limits, const float *velocity_limits, const float *acceleration_limits,
    const float *jerk_limits, const float *effort_limits);

/* Link spheres changed after packing (KinematicsParams.update_link_spheres / disable_link_spheres / AttachmentManager.update,
 * curobo/_src/robot/types/kinematics_params.py:493-595, collision/attachment_manager.py:102-315): one launch on `stream` copies
 * configuration 0 of link_spheres into the DEVICE blob's sphere section and rebuilds the broad-phase bounds of every collision link
 * (padded radii for self collision, raw radii for the scene) over the enabled spheres (r >= 0) of all configurations, with the
 * packer's own arithmetic: the blob becomes, byte for byte, what cb200_pack_robot_blob packs from the same spheres.  Every other
 * byte is left alone; a blob without a link-pair list (n_lp == 0) has no bounds, and only the spheres are copied.
 * robot_blob: DEVICE blob; robot_blob_host: HOST copy (its header is read on the host, its bytes are not updated);
 * link_spheres: DEVICE [num_sphere_configs, S, 4], num_sphere_configs equal to the configurations the blob was packed with.
 * A null pointer, a header that is not a blob of robot_blob_bytes bytes or another configuration count return
 * cudaErrorInvalidValue before any device work.  No allocation, no synchronisation: the call can be captured in a CUDA graph. */
int cb200_refresh_robot_spheres(void *robot_blob, const void *robot_blob_host, int32_t robot_blob_bytes,
                                const float *link_spheres /*[n_cfg, S, 4]*/, int32_t num_sphere_configs,
                                cb200_stream_t stream);

/* Device properties the host side sizes persistent grids with (SM count, max dynamic smem). */
int cb200_device_info(int device, int *sm_count, int *max_smem_optin);

#ifdef __cplusplus
}
#endif
#endif /* CUROBO_B200_H */
