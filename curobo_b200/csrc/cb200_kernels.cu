// cb200_kernels.cu -- sm_90a kernels + the C ABI of include/curobo_b200.h.
//
// Kernels (all fp32 SIMT; there is no dense contraction on this path, so no tensor cores):
//   rollout_fused_kernel, rollout_fused_big_kernel, rollout_fused_team_kernel, rollout_traj_kernel, rollout_traj_dyn_kernel and
//   the cost-only rollout_cost_kernel, rollout_cost_big_kernel (select_rollout picks one): persistent CTAs, robot constants staged
//   by one cp.async.bulk (TMA) per CTA; FK -> spheres -> self/scene/pose/c-space cost -> J^T gradient in ONE launch
//   kin_forward_kernel          drop-in for kinematics_forward_spheres_kernel
//   kin_backward_kernel         drop-in for kinematics_backward_kernel
//   self_collision_kernel       drop-in for self_collision_max_* kernels (single launch)
//   scene_collision_kernel      drop-in for the Warp sphere/swept obstacle kernels + speed metric
//   tool_pose_kernel, cspace_state_kernel, cspace_position_kernel   drop-ins for the Warp cost kernels
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <type_traits>
#include <vector>

#include "../../include/curobo_b200.h"
#include "cb200_blob.h"
#include "cb200_bspline.cuh"
#include "cb200_dynamics.cuh"
#include "cb200_dynamics_tile.cuh"
#include "cb200_launch.h"
#include "cb200_math.cuh"
#include "cb200_mesh.cuh"
#include "cb200_warp.cuh"

using namespace cb200;

namespace {

constexpr int kWarpsPerCta = 8;
constexpr int kMinCtas = 2;  // CTAs/SM the register allocator must leave room for at 256 threads (the arm builds use 3)

struct FusedArgs {
  cb200_rollout_cfg cfg;
  const float *q, *vel, *acc, *jerk, *dt;
  const unsigned char *blob;
  CuboidSet cuboids;
  VoxelSet voxels;
  const int32_t *env_query_idx;
  const float *goal_position, *goal_quat;
  const int32_t *idxs_goal;
  const float *pose_axes_t, *pose_axes_nt, *pose_tol_t, *pose_tol_nt;
  float *cost, *grad_q, *self_cost, *scene_cost, *pose_cost, *cspace_cost;
  float *grad_vel, *grad_acc, *grad_jerk;
  float *link_pos, *link_quat, *robot_spheres;
  int32_t *pose_goalset_idx;
  int32_t B, H;
  int32_t blob_smem_bytes, eval_floats;
  // B-spline front end (8f-1): when spl.knots != nullptr the rows are the spline states of the knots and
  // q / vel / acc / jerk / dt above are not read
  struct Spline {
    const float *knots, *sp, *sv, *sa, *sj, *gp, *gv, *ga, *gj, *traj_dt;
    const int32_t *start_idx, *goal_idx;
    const uint8_t *implicit;
    float *out_p, *out_v, *out_a, *out_j;
    int32_t n_knots, degree, steps;
  } spl;
  // Inverse dynamics inside the trajectory kernel (8f-3): inertial parameters of the links (the kinematic tree is the blob's).
  // Only read by rollout_traj_dyn_kernel.
  struct Dyn {
    const float *masses_com, *inertias, *gravity;
  } dyn;
  // c-space target term (a14): target rows [n, D], row index per seed (null = row 0), per-dof weight (null = 1)
  const float *cs_target;
  const int32_t *cs_target_idx;
  const float *cs_target_dofw;
  // link-sphere configurations (a2, num_envs > 1): [n_cfg, S] float4 in global memory; null = the blob's set
  const float4 *sphere_cfgs;
  int32_t n_sphere_cfgs;
  // big-robot kernel: row ticket counter [2] (zero between launches; null = static striding)
  int32_t *work_counter;
  // mesh obstacles (read by the SCENE & 4 builds only).  Last member, so the parameter offsets of the members above -- and the
  // code of the builds without meshes -- do not depend on it.
  MeshSet meshes;
  // current state of the POSITION c-space cost (velocity-aware IK): rows [n_cur, D], row index per seed (null = row 0), dt per
  // row; cur_pos == null turns the block off, cur_vel == null reads as zero velocity
  const float *cur_pos, *cur_vel, *cur_dt;
  const int32_t *cur_idx;
};

// link-frame sphere set of seed b: the blob's (shared memory) unless the caller passed several configurations
__device__ __forceinline__ const float4 *row_sphere_cfg(const FusedArgs &a, int b, int S) {
  if (a.sphere_cfgs == nullptr) return nullptr;
  int cfg = a.env_query_idx != nullptr ? __ldg(a.env_query_idx + b) : 0;
  if (cfg < 0 || cfg >= a.n_sphere_cfgs) cfg = 0;
  return a.sphere_cfgs + (size_t)cfg * S;
}

// c-space target term for one dof (wp_cspace_state.py:84-89,220-226; wp_cspace_position.py target block).
// STATE: the weight is tested before the per-dof factor is applied and non-terminal waypoints scale it;
// POSITION: the product weight * dof weight is tested.
__device__ __forceinline__ void cspace_target_term(const FusedArgs &a, int b, int h, int d, int D, float x, float &cost,
                                                   float &gp) {
  const cb200_rollout_cfg &c = a.cfg;
  if (a.cs_target == nullptr) return;
  float tw = c.cspace_target_weight;
  const float dofw = a.cs_target_dofw != nullptr ? __ldg(a.cs_target_dofw + d) : 1.0f;
  if (c.cspace_type == 2) {
    if (h < a.H - 1) tw *= c.cspace_non_terminal_weight_factor;
    if (!(tw > 0.0f)) return;
    tw *= dofw;
  } else {
    tw *= dofw;
    if (!(tw > 0.0f)) return;
  }
  const int row = a.cs_target_idx != nullptr ? __ldg(a.cs_target_idx + b) : 0;
  const float err = x - __ldg(a.cs_target + (size_t)row * D + d);
  cost += tw * err * err;
  gp += 2.0f * tw * err;
}

// State (q, qd, qdd, qddd) of row (b, h), dof d.  Spline mode evaluates the knots in place (one out-of-line copy
// for the three degrees); otherwise the caller's [B,H,D] arrays are read.
__device__ __noinline__ bspline::State4 spline_row_state(const FusedArgs::Spline &s, int b, int h, int d, int D) {
  const int srow = __ldg(s.start_idx + b), grow = __ldg(s.goal_idx + b);
  const float dt = __ldg(s.traj_dt + grow);
  const bool implicit = s.implicit[grow] != 0;
  bspline::State4 st;
  if (s.degree == 3) {
    st = bspline::evaluate<3>(bspline::make_polygon<3>(s.knots, b, d, D, s.n_knots, dt, s.steps, implicit, s.sp, s.sv, s.sa, s.sj, srow, s.gp, s.gv, s.ga, s.gj, grow), h, s.steps);
  } else if (s.degree == 5) {
    st = bspline::evaluate<5>(bspline::make_polygon<5>(s.knots, b, d, D, s.n_knots, dt, s.steps, implicit, s.sp, s.sv, s.sa, s.sj, srow, s.gp, s.gv, s.ga, s.gj, grow), h, s.steps);
  } else {
    st = bspline::evaluate<4>(bspline::make_polygon<4>(s.knots, b, d, D, s.n_knots, dt, s.steps, implicit, s.sp, s.sv, s.sa, s.sj, srow, s.gp, s.gv, s.ga, s.gj, grow), h, s.steps);
  }
  return st;
}

template <bool SPLINE>
__device__ __forceinline__ bspline::State4 load_row_state(const FusedArgs &a, int e, int b, int h, int d, int D) {
  if (SPLINE) {
    const bspline::State4 st = spline_row_state(a.spl, b, h, d, D);
    const size_t idx = (size_t)e * D + d;
    if (a.spl.out_p) a.spl.out_p[idx] = st.p;
    if (a.spl.out_v) a.spl.out_v[idx] = st.v;
    if (a.spl.out_a) a.spl.out_a[idx] = st.a;
    if (a.spl.out_j) a.spl.out_j[idx] = st.j;
    return st;
  }
  const size_t idx = (size_t)e * D + d;
  bspline::State4 st;
  st.p = __ldg(a.q + idx);
  st.v = a.vel ? __ldg(a.vel + idx) : 0.0f;
  st.a = a.acc ? __ldg(a.acc + idx) : 0.0f;
  st.j = a.jerk ? __ldg(a.jerk + idx) : 0.0f;
  return st;
}

// trajectory dt of seed b (STATE c-space retiming): the spline's own dt in spline mode
__device__ __forceinline__ float seed_dt(const FusedArgs &a, int b) {
  if (a.spl.knots != nullptr) return __ldg(a.spl.traj_dt + __ldg(a.spl.goal_idx + b));
  return a.dt ? __ldg(a.dt + b) : 1.0f;
}

// POSITION c-space cost of one dof with the current-state block (wp_cspace_position.py:299-356), in the order of
// cspace_position_kernel: shrink the bounds by the activation distance, intersect them with the window one step of dt reaches
// from the current position, hinge with activation 0, target term, then the implied velocity / acceleration regularizers with
// weights retimed by dt and dt^2.  Every waypoint of seed b reads the same current state.  A row whose dt <= 0 takes the plain
// hinge of cspace_dof.  Returns the cost and d cost / d q.  Out of line: the builds that run without a current state keep their
// register allocation.
struct CostGrad {
  float cost, grad;
};
__device__ __noinline__ CostGrad cspace_position_current(const FusedArgs &a, const float *lim, int b, int h, int d, int D,
                                                       float qd) {
  const cb200_rollout_cfg &c = a.cfg;
  float cost = 0.0f, gp = 0.0f;
  const int cur = a.cur_idx != nullptr ? __ldg(a.cur_idx + b) : 0;
  const float dt = __ldg(a.cur_dt + cur);
  if (!(dt > 0.0f)) {
    bound_cost(qd, lim[d], lim[D + d], c.cspace_activation[0], c.cspace_weight[0], cost, gp);
    cspace_target_term(a, b, h, d, D, qd, cost, gp);
    return CostGrad{cost, gp};
  }
  float lo = lim[d], hi = lim[D + d];
  {
    const float eta = c.cspace_activation[0], r = hi - lo;
    lo = lo + eta * r;
    hi = hi - eta * r;
  }
  const float cur_p = __ldg(a.cur_pos + (size_t)cur * D + d);
  lo = fmaxf(lo, cur_p + lim[2 * D + d] * dt);
  hi = fminf(hi, cur_p + lim[3 * D + d] * dt);
  bound_cost(qd, lo, hi, 0.0f, c.cspace_weight[0], cost, gp);  // an empty window (lo > hi) hinges on both sides
  cspace_target_term(a, b, h, d, D, qd, cost, gp);
  const float vw = c.cspace_reg[0] * dt, aw = c.cspace_reg[1] * dt * dt;
  if (vw > 0.0f || aw > 0.0f) {
    const float vi = (qd - cur_p) / dt;
    if (vw > 0.0f) {
      cost += 0.5f * vw * vi * vi;
      gp += vw * vi / dt;
    }
    if (aw > 0.0f) {
      const float cur_v = a.cur_vel != nullptr ? __ldg(a.cur_vel + (size_t)cur * D + d) : 0.0f;
      const float ai = (vi - cur_v) / dt;
      cost += 0.5f * aw * ai * ai;
      gp += aw * ai / (dt * dt);
    }
  }
  return CostGrad{cost, gp};
}

// c-space cost for one dof; returns cost, writes gradient wrt position into gp (and v/a/j grads to global unless !GRAD)
template <bool GRAD = true>
__device__ __forceinline__ float cspace_dof(const FusedArgs &a, const RobotView &rv, int e, int b, int h, int d,
                                            const bspline::State4 &st, float &gp) {
  const float qd = st.p;
  const cb200_rollout_cfg &c = a.cfg;
  const int D = rv.D;
  const float *lim = rv.limits;
  float cost = 0.0f;
  gp = 0.0f;
  if (c.cspace_type == 1) {
    if (a.cur_pos != nullptr) {
      const CostGrad r = cspace_position_current(a, lim, b, h, d, D, qd);
      cost = r.cost;
      gp = r.grad;
    } else {
      bound_cost(qd, lim[d], lim[D + d], c.cspace_activation[0], c.cspace_weight[0], cost, gp);
      cspace_target_term(a, b, h, d, D, qd, cost, gp);
    }
  } else if (c.cspace_type == 2) {
    const size_t idx = (size_t)e * D + d;
    const float dt = seed_dt(a, b);
    float wb[5], wr[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      wb[i] = c.cspace_weight[i];
      wr[i] = c.cspace_reg[i];
    }
    // dt^2, dt^3 by multiplication: correctly rounded products are at least as close to the reference's
    // wp.pow(dt, n) (wp_cspace_state.py) as powf, which costs ~100 instructions per call
    const float dt2 = dt * dt, dt3 = dt2 * dt;
    if (c.retime_weights) {
      wb[1] = dt * wb[1];
      wb[2] = dt2 * wb[2];
      wb[3] = dt3 * wb[3];
    }
    if (c.retime_regularization_weights) {
      wr[0] = dt * wr[0];
      wr[1] = dt2 * wr[1];
      wr[2] = dt3 * wr[2];
      wr[4] = dt * wr[4];
    }
    const float v = st.v, ac = st.a, jk = st.j;
    float gv = 0.0f, ga = 0.0f, gj = 0.0f;
    bound_cost(qd, lim[d], lim[D + d], c.cspace_activation[0], wb[0], cost, gp);
    bound_cost(v, lim[2 * D + d], lim[3 * D + d], c.cspace_activation[1], wb[1], cost, gv);
    bound_cost(ac, lim[4 * D + d], lim[5 * D + d], c.cspace_activation[2], wb[2], cost, ga);
    bound_cost(jk, lim[6 * D + d], lim[7 * D + d], c.cspace_activation[3], wb[3], cost, gj);
    // effort = 0 in this path: bound/regularisation/energy terms on torque vanish
    cspace_target_term(a, b, h, d, D, qd, cost, gp);
    l2_reg(v, wr[0], cost, gv);
    l2_reg(ac, wr[1], cost, ga);
    l2_reg(jk, wr[2], cost, gj);
    if (GRAD) {
      if (a.grad_vel) a.grad_vel[idx] = gv;
      if (a.grad_acc) a.grad_acc[idx] = ga;
      if (a.grad_jerk) a.grad_jerk[idx] = gj;
    }
  }
  return cost;
}

// ------------------------------------------------------------------------------------------------
// Row phases shared by the fused kernels.
//   phase A: q load + c-space cost, FK, spheres (+ padded copy), tool poses + tool-pose cost
//   phase B: self collision, scene collision (discrete | swept + speed metric), J^T backward, row cost
// The helpers are inlined: out-of-line phases needed fewer registers and ran slower (DESIGN.md section 4).
// GRAD = false (the cost-only kernels): the same costs, minus everything whose only consumer is the gradient -- the c-space and
// pose gradients, the sphere gradients and their count, the self-collision pair gradient, the J^T backward.
// ------------------------------------------------------------------------------------------------

// c-space phase of row (b, h): loads the row state into es.qv, the position gradient into es.gqv; returns the lane's cost sum
template <bool SPLINE, int W = 32, bool GRAD = true>
__device__ __forceinline__ float row_cspace(const FusedArgs &a, const RobotView &rv, const EvalSmem &es, int lane, int e, int b,
                                            int h) {
  const int D = rv.D;
  float cs_cost = 0.0f;
  #pragma unroll 1
  for (int d = lane; d < D; d += W) {
    const bspline::State4 st = load_row_state<SPLINE>(a, e, b, h, d, D);
    es.qv[d] = st.p;
    float gp;
    const float c = cspace_dof<GRAD>(a, rv, e, b, h, d, st, gp);
    if (GRAD) es.gqv[d] = gp;
    cs_cost += c;
    if (a.cspace_cost) a.cspace_cost[(size_t)e * D + d] = c;
  }
  return cs_cost;
}

// tool poses of row (b, h) (link_pos / link_quat) and the tool-pose cost: its gradient goes to es.pose_g; returns the lane's
// cost sum
template <int W = 32, bool GRAD = true>
__device__ __forceinline__ float row_tool_poses(const FusedArgs &a, const RobotView &rv, const EvalSmem &es, int lane, int e, int b,
                                                int h) {
  const cb200_rollout_cfg &cfg = a.cfg;
  const int L = rv.L;
  float pose_c = 0.0f;
  const bool do_pose = (a.goal_position != nullptr);
  #pragma unroll 1
  for (int t = lane; t < L; t += W) {
    const float *T = es.cumul + 12 * rv.tool_map[t];
    const V3 p = mk3(T[3], T[7], T[11]);
    const Q4 qt = quat_from_transform(T);
    if (a.link_pos) {
      float *o = a.link_pos + ((size_t)e * L + t) * 3;
      o[0] = p.x;
      o[1] = p.y;
      o[2] = p.z;
    }
    if (a.link_quat) *reinterpret_cast<float4 *>(a.link_quat + ((size_t)e * L + t) * 4) = make_float4(qt.w, qt.x, qt.y, qt.z);
    float *pg = GRAD ? es.pose_g + 8 * t : nullptr;
    if (GRAD) pg[0] = pg[1] = pg[2] = pg[4] = pg[5] = pg[6] = 0.0f;
    if (do_pose) {
      const int gi = a.idxs_goal ? __ldg(a.idxs_goal + b) : 0;
      const bool term = !(h < a.H - 1 && a.H > 1);
      const float *axes = term ? a.pose_axes_t : a.pose_axes_nt;
      const float *tol = term ? a.pose_tol_t : a.pose_tol_nt;
      const size_t go = ((size_t)gi * L + t) * cfg.num_goalset;
      const PoseOut po = tool_pose_cost(p, qt, a.goal_position + go * 3, a.goal_quat + go * 4, cfg.num_goalset,
                                        cfg.pose_weight[0], cfg.pose_weight[1], axes, t,
                                        tol != nullptr ? __ldg(tol + 2 * t) : 0.0f,
                                        tol != nullptr ? __ldg(tol + 2 * t + 1) : 0.0f, cfg.pose_rotation_method);
      if (GRAD) {
        const V3 om = quat_grad_to_omega(qt, po.gq_w, po.gq_x, po.gq_y, po.gq_z);
        pg[0] = po.g_pos.x;
        pg[1] = po.g_pos.y;
        pg[2] = po.g_pos.z;
        pg[4] = om.x;
        pg[5] = om.y;
        pg[6] = om.z;
      }
      pose_c += po.pos_cost + po.rot_cost;
      if (a.pose_cost) {
        a.pose_cost[((size_t)e * L + t) * 2] = po.pos_cost;
        a.pose_cost[((size_t)e * L + t) * 2 + 1] = po.rot_cost;
      }
      if (a.pose_goalset_idx) a.pose_goalset_idx[(size_t)e * L + t] = po.goal_idx;
    }
  }
  return pose_c;
}

template <bool SPLINE, int W = 32, bool GRAD = true>
__device__ __forceinline__ void row_phase_a(const FusedArgs &a, const RobotView &rv, const EvalSmem &es, int lane, int e,
                                            int b, int h, float &cs_cost, float &pose_c) {
  const int S = rv.S;
  cs_cost = row_cspace<SPLINE, W, GRAD>(a, rv, es, lane, e, b, h);
  row_sync<W>();
  warp_fk<W>(rv, es, lane);
  warp_spheres<W>(rv, es, lane, a.robot_spheres ? reinterpret_cast<float4 *>(a.robot_spheres) + (size_t)e * S : nullptr,
                  row_sphere_cfg(a, b, S));
  pose_c = row_tool_poses<W, GRAD>(a, rv, es, lane, e, b, h);
  row_sync<W>();
}

// phase B1: self collision + scene collision.  Leaves the scene sphere-gradients in es.gsph and returns the
// pieces phase B2 needs in registers.
struct RowB1 {
  float self_c, fmax, scene_c;
  int bi, bj, nnz;
};

// Cuboids of the row's environment (ce, ncub clamped to the set's capacity) and whether the broad phase culls them.
struct CuboidCull {
  int ce, ncub;
  bool cull;
};
// Whether the row has cuboid terms.  The mesh build, SCENE = 7, runs with or without cuboids and ESDF grids: it checks at run
// time which sets are present.
template <int SCENE>
__device__ __forceinline__ bool has_cuboids(const FusedArgs &a, bool do_scene) {
  return (SCENE & 1) && do_scene && (!(SCENE & 4) || a.cuboids.inv_pose != nullptr);
}
// Fills cc when has_cuboids; returns cc.cull.  The callers keep this split from has_cuboids, with the mask fill nested inside
// it: folding the two into one helper changed the register allocation of kernels that have no cuboid terms at all.
__device__ __forceinline__ bool cuboid_cull_state(const FusedArgs &a, const RobotView &rv, int env, bool discrete, CuboidCull &cc) {
  cc.ce = env < a.cuboids.num_envs ? env : 0;
  cc.ncub = a.cuboids.count[cc.ce];
  if (cc.ncub > a.cuboids.max_n) cc.ncub = a.cuboids.max_n;
  cc.cull = discrete && rv.n_lp > 0 && cc.ncub <= 32;  // (one mask bit per cuboid)
  return cc.cull;
}

// Cuboid broad phase (discrete mode): es.cmask[ca] = the cuboids collision link ca may touch, for ca = first, first + stride, ...
// A box SDF is 1-Lipschitz, so sdf(link bound centre) >= R_link + eta means no sphere of the link has pen = r + eta - sdf > 0
// against that cuboid: skipping it is exact.  The caller synchronises its lanes before the masks are read.
__device__ __forceinline__ void cuboid_cull_masks(const FusedArgs &a, const RobotView &rv, const EvalSmem &es, int ce, int ncub,
                                                  int first, int stride) {
#pragma unroll 1
  for (int ca = first; ca < rv.n_cl; ca += stride) {
    const float4 cb = rv.cl_bound_scene[ca];
    uint32_t mask = 0u;
    if (cb.w >= 0.0f) {
      const float *Tk = es.cumul + 12 * rv.cl_link[ca];
      const V3 cw = mk3(Tk[0] * cb.x + Tk[1] * cb.y + Tk[2] * cb.z + Tk[3], Tk[4] * cb.x + Tk[5] * cb.y + Tk[6] * cb.z + Tk[7],
                        Tk[8] * cb.x + Tk[9] * cb.y + Tk[10] * cb.z + Tk[11]);
#pragma unroll 1
      for (int i = 0; i < ncub; ++i) {
        const int kk = ce * a.cuboids.max_n + i;
        if (a.cuboids.enable[kk] != 1) continue;
        const ObsFrame f = load_obs_frame(a.cuboids.inv_pose + 8 * kk);
        const SdfGrad sg = cuboid_sdf_grad(to_obstacle(f, cw), ldgf(a.cuboids.dims + 4 * kk), ldgf(a.cuboids.dims + 4 * kk + 1),
                                           ldgf(a.cuboids.dims + 4 * kk + 2));
        if (sg.sdf < cb.w + a.cfg.scene_activation) mask |= (1u << i);
      }
    }
    es.cmask[ca] = mask;
  }
}

// Mesh terms of one sphere (the SCENE & 4 builds): weighted world-frame gradient in xyz, weighted cost in w.  The caller adds them
// to the cuboid + ESDF sum: the order of the per-operator composition, where one launch writes the cuboid + ESDF terms and the
// mesh launch adds to them (cb200_sphere_mesh_collision with accumulate = 1).  Inlined: an out-of-line call spilled more than the
// inlined traversal in every family (the registers live across the call are saved around it; DESIGN.md section 4).
__device__ __forceinline__ float4 mesh_terms(const MeshSet *ms, float eta, float w, V3 c, float r, int env, bool sweep, bool has_prev,
                                          V3 prev, bool has_next, V3 next) {
  const CuboidSet no_cuboids{};
  const VoxelSet no_voxels{};
  V3 g = mk3(0, 0, 0);
  const float cost = sweep ? sphere_scene_swept<4>(c, r, eta, w, has_prev, prev, has_next, next, no_cuboids, no_voxels, env, g, ms)
                           : sphere_scene_discrete<4>(c, r, eta, w, no_cuboids, no_voxels, env, g, ms);
  return make_float4(g.x, g.y, g.z, cost);
}

// Discrete scene terms of sphere s: the cuboids the broad phase kept, the ESDF grids, the meshes.  Returns the weighted cost and
// adds the weighted world-frame gradient to g.
template <int SCENE>
__device__ __forceinline__ float sphere_discrete_terms(const FusedArgs &a, const RobotView &rv, const EvalSmem &es,
                                                       const CuboidCull &cc, int env, int s, V3 &g) {
  const cb200_rollout_cfg &cfg = a.cfg;
  const float4 sp = es.sph[s];
  const V3 cen = mk3(sp.x, sp.y, sp.z);
  float c = 0.0f;
  if (sp.w >= 0.0f) {
    if (SCENE & 1) {
      uint32_t m = cc.cull ? es.cmask[rv.sph_cl[s]] : 0xffffffffu;
      const float radj = sp.w + cfg.scene_activation;
#pragma unroll 1
      for (int i = 0; i < cc.ncub && m != 0u; ++i) {
        if (cc.cull && !((m >> i) & 1u)) continue;
        if (cc.cull) m &= ~(1u << i);
        const int kk = cc.ce * a.cuboids.max_n + i;
        if (a.cuboids.enable[kk] != 1) continue;
        const ObsFrame f = load_obs_frame(a.cuboids.inv_pose + 8 * kk);
        const SdfGrad sg = cuboid_sdf_grad(to_obstacle(f, cen), ldgf(a.cuboids.dims + 4 * kk), ldgf(a.cuboids.dims + 4 * kk + 1),
                                           ldgf(a.cuboids.dims + 4 * kk + 2));
        const float pen = radj - sg.sdf;
        if (pen > 0.0f) {
          float ac, as;
          collision_activation(pen, cfg.scene_activation, ac, as);
          c += cfg.scene_weight * ac;
          g = g + (cfg.scene_weight * as) * from_obstacle(f, sg.n);
        }
      }
    }
    if (SCENE & 2) {
      const CuboidSet none{};
      c += sphere_scene_discrete<2>(cen, sp.w, cfg.scene_activation, cfg.scene_weight, none, a.voxels, env, g);
    }
    if (SCENE & 4) {
      const float4 m = mesh_terms(&a.meshes, cfg.scene_activation, cfg.scene_weight, cen, sp.w, env, false, false, cen, false, cen);
      c += m.w;
      g = g + mk3(m.x, m.y, m.z);
    }
  }
  return c;
}

template <bool SWEEP, int SCENE, bool CULL2 = true, int W = 32, bool GRAD = true>
__device__ __forceinline__ RowB1 row_phase_b1(const FusedArgs &a, const RobotView &rv, const EvalSmem &es, int lane, int e,
                                              int b, const float4 *prev_sph, const float4 *next_sph) {
  const cb200_rollout_cfg &cfg = a.cfg;
  const int S = rv.S;
  RowB1 r{0.0f, 0.0f, 0.0f, 0, 0, 0};
  // ---- self collision (reads padded spheres in gsph; the cost-only layout keeps that copy only for the pair scan)
  if (cfg.self_weight > 0.0f && rv.P > 0) {
    r.fmax = (rv.n_lp > 0) ? warp_self_collision_tiles<GRAD, CULL2, W>(rv, es, lane, r.bi, r.bj)
                           : warp_self_collision_pairs<W>(es.gsph, rv.pairs, rv.P, lane, r.bi, r.bj);
    r.self_c = (r.fmax > 0.0f) ? 0.5f * cfg.self_weight * r.fmax : 0.0f;
  }
  if (a.self_cost && lane == 0) a.self_cost[e] = r.self_c;
  row_sync<W>();
  // ---- scene collision (lane per sphere) -> gsph = gradient
  const bool do_scene = SCENE != 0 && cfg.scene_weight > 0.0f;
  const int env = (a.env_query_idx != nullptr) ? __ldg(a.env_query_idx + b) : 0;
  const float sdt = (SWEEP && cfg.use_speed_metric && (a.dt != nullptr || a.spl.knots != nullptr))
                        ? (a.spl.knots != nullptr ? __ldg(a.spl.traj_dt + __ldg(a.spl.goal_idx)) : __ldg(a.dt))
                        : 0.0f;
  CuboidCull cc{0, 0, false};
  if (has_cuboids<SCENE>(a, do_scene)) {
    if (cuboid_cull_state(a, rv, env, !SWEEP, cc)) {
      cuboid_cull_masks(a, rv, es, cc.ce, cc.ncub, lane, W);
      row_sync<W>();
    }
  }
#pragma unroll 1
  for (int s = lane; s < S; s += W) {
    V3 g = mk3(0, 0, 0);
    float c = 0.0f;
    if (do_scene) {
      if (!SWEEP) {
        c = sphere_discrete_terms<SCENE>(a, rv, es, cc, env, s, g);
      } else {
        const float4 sp = es.sph[s];
        const V3 cen = mk3(sp.x, sp.y, sp.z);
        V3 pv = cen, nx = cen;
        if (prev_sph != nullptr) {
          const float4 t = prev_sph[s];
          pv = mk3(t.x, t.y, t.z);
        }
        if (next_sph != nullptr) {
          const float4 t = next_sph[s];
          nx = mk3(t.x, t.y, t.z);
        }
        c = sphere_scene_swept<SCENE & 3>(cen, sp.w, cfg.scene_activation, cfg.scene_weight, prev_sph != nullptr, pv,
                                          next_sph != nullptr, nx, a.cuboids, a.voxels, env, g);
        if (SCENE & 4) {
          const float4 m = mesh_terms(&a.meshes, cfg.scene_activation, cfg.scene_weight, cen, sp.w, env, true, prev_sph != nullptr,
                                      pv, next_sph != nullptr, nx);
          c += m.w;
          g = g + mk3(m.x, m.y, m.z);
        }
        if (cfg.use_speed_metric && prev_sph != nullptr && next_sph != nullptr) speed_metric(pv, cen, nx, sdt, c, g);
      }
    }
    if (GRAD) {
      es.gsph[s] = make_float4(g.x, g.y, g.z, 0.0f);
      r.nnz += (g.x != 0.0f || g.y != 0.0f || g.z != 0.0f) ? 1 : 0;
    }
    r.scene_c += c;
    if (a.scene_cost) a.scene_cost[(size_t)e * S + s] = c;
  }
  row_sync<W>();
  if (GRAD) r.nnz = (int)row_reduce<W, 0>((unsigned)r.nnz) + 2;  // + the two self-collision spheres
  return r;
}

// phase B2: add the self-collision gradient to the two spheres of the worst pair, J^T backward, row cost.
template <bool SMALL = false, int W = 32, bool GRAD = true>
__device__ __forceinline__ void row_phase_b2(const FusedArgs &a, const RobotView &rv, const EvalSmem &es,
                                             const unsigned char *smem_blob, int lane, int e, const RowB1 &r,
                                             float cs_cost, float pose_c) {
  if (GRAD) {
    if (r.fmax > 0.0f && lane == 0) {
      const float4 pi = es.sph[r.bi], pj = es.sph[r.bj];
      const float w = a.cfg.self_weight;
      float4 gi = es.gsph[r.bi], gj = es.gsph[r.bj];
      const float gx = w * (pj.x - pi.x), gy = w * (pj.y - pi.y), gz = w * (pj.z - pi.z);
      gi.x += gx;
      gi.y += gy;
      gi.z += gz;
      gj.x -= gx;
      gj.y -= gy;
      gj.z -= gz;
      es.gsph[r.bi] = gi;
      es.gsph[r.bj] = gj;
    }
    row_sync<W>();
    float *gq = a.grad_q + (size_t)e * rv.D;
    if (!warp_fk_backward_sparse<SMALL, W>(rv, es, lane, gq, r.nnz)) warp_fk_backward_cold<W>(smem_blob, a.blob, es.cumul, lane, gq);
  }
  const float tot = warp_sum<W>(cs_cost + pose_c + r.scene_c) + r.self_c;
  if (lane == 0) a.cost[e] = tot;
  row_sync<W>();
}

// Ticket counter [2] of the persistent kernels (FusedArgs::work_counter): [0] hands out work units after each worker's first,
// [1] counts the workers (warps, teams or CTAs) that have left.  It is zero between launches.
// Next work unit of a warp that just finished unit u: a ticket when the caller passed a counter, else static striding.
__device__ __forceinline__ int next_warp_unit(int32_t *counter, int u, int stride, bool leader) {
  if (counter == nullptr) return u + stride;
  int nxt = 0;
  if (leader) nxt = stride + atomicAdd(counter, 1);
  return __shfl_sync(kFull, nxt, 0);
}
// Called once per worker on its way out: the last of `workers` to leave re-arms the counter for the next launch on the stream.
__device__ __forceinline__ void rearm_ticket_counter(int32_t *counter, int workers) {
  __threadfence();
  if (atomicAdd(counter + 1, 1) == workers - 1) {
    counter[0] = 0;
    counter[1] = 0;
  }
}

// ------------------------------------------------------------------------------------------------
// THE fused kernel, discrete scene collision: rows are independent, one persistent warp per row, phases
// inlined (measured best: out-of-line phases needed fewer registers and ran slower).
// ------------------------------------------------------------------------------------------------
// ROWS = 2 (arm build only, robots of <= 16 links): two rows per warp, half h = lane >> 4 owns row 2 u + h of the warp's work
// unit u, with the row helpers at width 16.  The halves run the same code on different rows and may diverge inside a row; they
// meet again at the end of it, where the next unit is fetched.  A row's result does not depend on its partner.
template <int SCENE, bool SPLINE, int MINB = kMinCtas, int ROWS = 1>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB) rollout_fused_kernel(const __grid_constant__ FusedArgs a) {
  static_assert(ROWS == 1 || (ROWS == 2 && MINB == 3 && !SPLINE), "paired rows: arm build only");
  constexpr int W = 32 / ROWS;
  CB200_EXTERN_SHARED __align__(128) unsigned char smem[];
  __shared__ unsigned long long mbar;
  stage_blob_to_smem(smem, a.blob, (uint32_t)a.blob_smem_bytes, &mbar);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & (W - 1), nwarps = blockDim.x >> 5;
  const int half = ROWS == 1 ? 0 : (int)(threadIdx.x >> 4) & 1;
  const bool leader = (threadIdx.x & 31) == 0;
  float *base = reinterpret_cast<float *>(smem + a.blob_smem_bytes) + (size_t)(warp * ROWS + half) * a.eval_floats;
  const int N = a.B * a.H;
  const int stride = gridDim.x * nwarps;
  // work units (one row per warp, or one pair of rows): the first one statically, the rest from the ticket counter when the
  // caller provides one (rows differ in cost and 16,384 rows over 3,168 resident warps -- 132 SMs x 24 on an H100 -- is 5.2
  // rounds: with static striding the last round is partly empty)
  int u = blockIdx.x * nwarps + warp;
  while (u * ROWS < N) {
    const int e = u * ROWS + half;
    if (ROWS == 1 || e < N) {  // (odd N: the last unit's second half has no row)
      int b = e, h = 0;
      if (a.H != 1) {  // integer division is ~60 instructions: skip it for H == 1 (IK)
        b = e / a.H;
        h = e - b * a.H;
      }
      const RobotView rv = make_robot_view(smem, a.blob);
      const EvalSmem es = carve_eval_smem(base, rv.nl, rv.D, rv.S, rv.L, rv.n_cl);
      float cs_cost = 0.0f, pose_c = 0.0f;
      row_phase_a<SPLINE, W>(a, rv, es, lane, e, b, h, cs_cost, pose_c);
      const RowB1 r = row_phase_b1<false, SCENE, MINB != 3, W>(a, rv, es, lane, e, b, nullptr, nullptr);
      row_phase_b2<MINB == 3, W>(a, rv, es, smem, lane, e, r, cs_cost, pose_c);
    }
    u = next_warp_unit(a.work_counter, u, stride, leader);
  }
  if (a.work_counter != nullptr && leader) rearm_ticket_counter(a.work_counter, stride);
}

// Cost-only twin of rollout_fused_kernel (cb200_rollout_cost): the same rows and costs through the same phases at GRAD = false,
// no gradient, a smaller row state (carve_cost_smem).  Discrete rows from caller-provided positions only.  (A body shared with
// rollout_fused_kernel through one inlined template changed that kernel's register allocation, so the two are kept apart.)
template <int SCENE, int MINB = kMinCtas, int ROWS = 1>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB) rollout_cost_kernel(const __grid_constant__ FusedArgs a) {
  static_assert(ROWS == 1 || (ROWS == 2 && MINB == 3), "paired rows: arm build only");
  constexpr int W = 32 / ROWS;
  CB200_EXTERN_SHARED __align__(128) unsigned char smem[];
  __shared__ unsigned long long mbar;
  stage_blob_to_smem(smem, a.blob, (uint32_t)a.blob_smem_bytes, &mbar);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & (W - 1), nwarps = blockDim.x >> 5;
  const int half = ROWS == 1 ? 0 : (int)(threadIdx.x >> 4) & 1;
  const bool leader = (threadIdx.x & 31) == 0;
  float *base = reinterpret_cast<float *>(smem + a.blob_smem_bytes) + (size_t)(warp * ROWS + half) * a.eval_floats;
  const int N = a.B * a.H;
  const int stride = gridDim.x * nwarps;
  int u = blockIdx.x * nwarps + warp;
  while (u * ROWS < N) {
    const int e = u * ROWS + half;
    if (ROWS == 1 || e < N) {
      int b = e, h = 0;
      if (a.H != 1) {
        b = e / a.H;
        h = e - b * a.H;
      }
      const RobotView rv = make_robot_view(smem, a.blob);
      const EvalSmem es = carve_cost_smem(base, rv.nl, rv.D, rv.S, rv.n_cl, rv.n_lp == 0);
      float cs_cost = 0.0f, pose_c = 0.0f;
      row_phase_a<false, W, false>(a, rv, es, lane, e, b, h, cs_cost, pose_c);
      const RowB1 r = row_phase_b1<false, SCENE, MINB != 3, W, false>(a, rv, es, lane, e, b, nullptr, nullptr);
      row_phase_b2<MINB == 3, W, false>(a, rv, es, smem, lane, e, r, cs_cost, pose_c);
    }
    u = next_warp_unit(a.work_counter, u, stride, leader);
  }
  if (a.work_counter != nullptr && leader) rearm_ticket_counter(a.work_counter, stride);
}

// ------------------------------------------------------------------------------------------------
// Validity rows (cb200_rollout_validate): is row (b, h) inside the position limits, free of scene contact and free of self
// contact?  The reference's RobotSceneCollision.validate sums non-negative terms and tests the sum against 0, so each check is
// "its term is exactly 0", asked in the order of cost: bounds (before FK), scene, self.  A row leaves at the first check that
// fails; every exit is a warp vote (__ballot_sync) at a chunk boundary -- 32 dofs, 32 spheres, one link-pair block of the
// self-collision scan -- so an exit changes when the row ends, never its verdict.  The row state is the cost-only layout
// (carve_cost_smem: cumulative transforms, world spheres, broad-phase bounds and masks), one persistent warp per row for every
// robot; rows are handed out by the ticket counter.  a.cfg holds weight 1 and activation 0 for the scene and self terms.
enum : int { kCheckBounds = 1, kCheckSelf = 2, kCheckScene = 4 };

template <int SCENE>
__device__ __forceinline__ bool validate_row(const FusedArgs &a, const RobotView &rv, const EvalSmem &es, int lane, int e, int b,
                                             int checks) {
  const int D = rv.D, S = rv.S;
#pragma unroll 1
  for (int d0 = 0; d0 < D; d0 += 32) {
    const int d = d0 + lane;
    bool out = false;
    if (d < D) {
      const float x = __ldg(a.q + (size_t)e * D + d);
      es.qv[d] = x;
      float c = 0.0f, g;
      bound_cost(x, rv.limits[d], rv.limits[D + d], 0.0f, 1.0f, c, g);
      out = (checks & kCheckBounds) && c != 0.0f;
    }
    if (__ballot_sync(kFull, out) != 0u) return false;
  }
  if (!(checks & (kCheckScene | kCheckSelf))) return true;
  __syncwarp();
  warp_fk<32>(rv, es, lane);
  warp_spheres<32>(rv, es, lane, nullptr, row_sphere_cfg(a, b, S));
  __syncwarp();
  if (SCENE != 0 && (checks & kCheckScene)) {
    const int env = a.env_query_idx != nullptr ? __ldg(a.env_query_idx + b) : 0;
    CuboidCull cc{0, 0, false};
    if (has_cuboids<SCENE>(a, true)) {
      if (cuboid_cull_state(a, rv, env, true, cc)) {
        cuboid_cull_masks(a, rv, es, cc.ce, cc.ncub, lane, 32);
        __syncwarp();
      }
    }
#pragma unroll 1
    for (int s0 = 0; s0 < S; s0 += 32) {
      const int s = s0 + lane;
      V3 g = mk3(0, 0, 0);
      const bool hit = s < S && sphere_discrete_terms<SCENE>(a, rv, es, cc, env, s, g) != 0.0f;
      if (__ballot_sync(kFull, hit) != 0u) return false;
    }
  }
  if ((checks & kCheckSelf) && rv.P > 0) {
    int bi, bj;
    const float f = rv.n_lp > 0 ? warp_self_collision_tiles<false, true, 32, true>(rv, es, lane, bi, bj)
                                : warp_self_collision_pairs<32>(es.gsph, rv.pairs, rv.P, lane, bi, bj);
    if (f > 0.0f) return false;
  }
  return true;
}

template <int SCENE>
__global__ void __launch_bounds__(kWarpsPerCta * 32, kMinCtas) rollout_validate_kernel(const __grid_constant__ FusedArgs a,
                                                                                       uint8_t *valid, const int checks) {
  CB200_EXTERN_SHARED __align__(128) unsigned char smem[];
  __shared__ unsigned long long mbar;
  stage_blob_to_smem(smem, a.blob, (uint32_t)a.blob_smem_bytes, &mbar);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const bool leader = lane == 0;
  float *base = reinterpret_cast<float *>(smem + a.blob_smem_bytes) + (size_t)warp * a.eval_floats;
  const int N = a.B * a.H;
  const int stride = gridDim.x * nwarps;
  int e = blockIdx.x * nwarps + warp;
  while (e < N) {
    const int b = a.H != 1 ? e / a.H : e;
    const RobotView rv = make_robot_view(smem, a.blob);
    const EvalSmem es = carve_cost_smem(base, rv.nl, rv.D, rv.S, rv.n_cl, rv.n_lp == 0);
    const bool ok = validate_row<SCENE>(a, rv, es, lane, e, b, checks);
    if (leader) valid[e] = ok ? 1 : 0;
    __syncwarp();  // the next row rewrites the row state
    e = next_warp_unit(a.work_counter, e, stride, leader);
  }
  if (a.work_counter != nullptr && leader) rearm_ticket_counter(a.work_counter, stride);
}

// ------------------------------------------------------------------------------------------------
// THE fused kernel for big robots (humanoids), discrete scene collision.  Same phases and arithmetic as rollout_fused_kernel;
// what changes is how many rows an SM keeps in flight.  The kernel is latency bound and shared memory caps the resident warps: a G1-29 row is 17.3 KB, of which 12.8 KB
// are two [S] float4 arrays -- the padded copy of the spheres for the pair phase and the dense sphere gradients.  Here
//   * the pair phase rebuilds padded radii from the padding table (one extra shared load per sphere read),
//   * sphere gradients go to a short list (the spheres that collide are a handful) that feeds the sparse J^T directly; a row
//     that overflows the list drains it into per-link force / torque accumulators and finishes with the dense up-sweep,
//   * one CTA of up to 16 warps per SM (the robot blob is staged once), rows handed out by a ticket counter instead of
//     static striding (rows differ in cost; 8192 rows over 2112 warps -- 132 SMs x 16 -- is 3.9 rounds: the last one is partly empty otherwise).
// Row: 10.9 KB (G1-29), 16.4 KB (G1-43) -> 16 / 11 rows in flight per SM instead of 10 / 7.
// ------------------------------------------------------------------------------------------------
constexpr int kBigWarps = 16;

template <int SCENE, bool SMALL = false, bool GRAD = true>
__device__ __forceinline__ RowB1 row_phase_b1_list(const FusedArgs &a, const RobotView &rv, const EvalSmem &es, int lane, int e,
                                                   int b, int &n_list, bool &dense) {
  const cb200_rollout_cfg &cfg = a.cfg;
  const int S = rv.S;
  RowB1 r{0.0f, 0.0f, 0.0f, 0, 0, 0};
  n_list = 0;
  dense = false;
  if (cfg.self_weight > 0.0f && rv.P > 0) {
    r.fmax = warp_self_collision_tiles<false, !SMALL>(rv, es, lane, r.bi, r.bj);
    r.self_c = (r.fmax > 0.0f) ? 0.5f * cfg.self_weight * r.fmax : 0.0f;
  }
  if (a.self_cost && lane == 0) a.self_cost[e] = r.self_c;
  __syncwarp();
  const bool do_scene = SCENE != 0 && cfg.scene_weight > 0.0f;
  const int env = (a.env_query_idx != nullptr) ? __ldg(a.env_query_idx + b) : 0;
  CuboidCull cc{0, 0, false};
  if (has_cuboids<SCENE>(a, do_scene)) {
    if (cuboid_cull_state(a, rv, env, true, cc)) {
      cuboid_cull_masks(a, rv, es, cc.ce, cc.ncub, lane, 32);
      __syncwarp();
    }
  }
  bool ft_live = false;
  const unsigned lt = (1u << lane) - 1u;
#pragma unroll 1
  for (int base = 0; base < S; base += 32) {  // uniform trip count: the list append below is a warp collective
    const int s = base + lane;
    V3 g = mk3(0, 0, 0);
    float c = 0.0f;
    if (s < S && do_scene) c = sphere_discrete_terms<SCENE>(a, rv, es, cc, env, s, g);
    if (GRAD) {
      const bool nz = (g.x != 0.0f) || (g.y != 0.0f) || (g.z != 0.0f);
      const unsigned m = __ballot_sync(kFull, nz);
      if (m) {
        const int cnt = __popc(m);
        if (n_list + cnt > kGradListCap - 2) {  // (two slots stay free for the self-collision pair)
          if (!ft_live) {
            warp_zero_ft(rv, es, lane);
            ft_live = true;
          }
          warp_drain_list_to_ft(rv, es, lane, n_list);
          n_list = 0;
          dense = true;
        }
        if (nz) es.glist[n_list + __popc(m & lt)] = make_float4(g.x, g.y, g.z, __int_as_float(s));
        n_list += cnt;
        __syncwarp();
      }
    }
    r.scene_c += c;
    if (a.scene_cost && s < S) a.scene_cost[(size_t)e * S + s] = c;
  }
  if (GRAD && dense && !ft_live) warp_zero_ft(rv, es, lane);
  return r;
}

// the worst self-collision pair's gradient: two more entries of a gradient list (lane 0 writes them, the caller synchronises)
__device__ __forceinline__ void append_self_pair(const FusedArgs &a, const EvalSmem &es, int lane, int bi, int bj, float4 *list,
                                                 int &n_list) {
  if (lane == 0) {
    const float4 pi = es.sph[bi], pj = es.sph[bj];
    const float w = a.cfg.self_weight;
    const float gx = w * (pj.x - pi.x), gy = w * (pj.y - pi.y), gz = w * (pj.z - pi.z);
    list[n_list] = make_float4(gx, gy, gz, __int_as_float(bi));
    list[n_list + 1] = make_float4(-gx, -gy, -gz, __int_as_float(bj));
  }
  n_list += 2;
}

template <bool SMALL = false, bool GRAD = true>
__device__ __forceinline__ void row_phase_b2_list(const FusedArgs &a, const RobotView &rv, const EvalSmem &es, int lane, int e,
                                                  const RowB1 &r, float cs_cost, float pose_c, int n_list, bool dense) {
  if (GRAD) {
    if (r.fmax > 0.0f) {
      append_self_pair(a, es, lane, r.bi, r.bj, es.glist, n_list);
      __syncwarp();
    }
    float *gq = a.grad_q + (size_t)e * rv.D;
    if (!dense) {
      warp_fk_backward_list<SMALL>(rv, es, lane, gq, n_list);
    } else {
      warp_drain_list_to_ft(rv, es, lane, n_list);
      warp_fk_backward_from_ft(rv, es, lane, gq);
    }
  }
  const float tot = warp_sum(cs_cost + pose_c + r.scene_c) + r.self_c;
  if (lane == 0) a.cost[e] = tot;
  __syncwarp();
}

// SMALL: arms (<= 24 links, <= 128 spheres) that come here because of an ESDF scene -- the trims of the IK kernel's arm build
// (whole-block self-collision scan, one-slot J^T with the tool frames in the list loop): less code to fetch per row.
template <int SCENE, bool SMALL = false>
__global__ void __launch_bounds__(kBigWarps * 32, 1) rollout_fused_big_kernel(const __grid_constant__ FusedArgs a) {
  CB200_EXTERN_SHARED __align__(128) unsigned char smem[];
  __shared__ unsigned long long mbar;
  stage_blob_to_smem(smem, a.blob, (uint32_t)a.blob_smem_bytes, &mbar);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  float *base = reinterpret_cast<float *>(smem + a.blob_smem_bytes) + (size_t)warp * a.eval_floats;
  const RobotView rv = make_robot_view(smem, a.blob);
  const EvalSmem es = carve_big_smem(base, rv.nl, rv.D, rv.S, rv.L, rv.n_cl);
  const int N = a.B * a.H;
  const int total_warps = gridDim.x * nwarps;
  int e = blockIdx.x * nwarps + warp;  // first row: static; afterwards rows come from the ticket counter
  while (e < N) {
    int b = e, h = 0;
    if (a.H != 1) {
      b = e / a.H;
      h = e - b * a.H;
    }
    float cs_cost = 0.0f, pose_c = 0.0f;
    row_phase_a<false>(a, rv, es, lane, e, b, h, cs_cost, pose_c);
    int n_list;
    bool dense;
    const RowB1 r = row_phase_b1_list<SCENE, SMALL>(a, rv, es, lane, e, b, n_list, dense);
    row_phase_b2_list<SMALL>(a, rv, es, lane, e, r, cs_cost, pose_c, n_list, dense);
    e = next_warp_unit(a.work_counter, e, total_warps, lane == 0);
  }
  if (a.work_counter != nullptr && lane == 0) rearm_ticket_counter(a.work_counter, total_warps);
}

// Cost-only twin of rollout_fused_big_kernel (cb200_rollout_cost).  Also where cost-only batches go whose gradient launch would
// take the team kernel: particle batches are large, so there is no cost-only team build.
template <int SCENE, bool SMALL = false>
__global__ void __launch_bounds__(kBigWarps * 32, 1) rollout_cost_big_kernel(const __grid_constant__ FusedArgs a) {
  CB200_EXTERN_SHARED __align__(128) unsigned char smem[];
  __shared__ unsigned long long mbar;
  stage_blob_to_smem(smem, a.blob, (uint32_t)a.blob_smem_bytes, &mbar);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  float *base = reinterpret_cast<float *>(smem + a.blob_smem_bytes) + (size_t)warp * a.eval_floats;
  const RobotView rv = make_robot_view(smem, a.blob);
  const EvalSmem es = carve_cost_smem(base, rv.nl, rv.D, rv.S, rv.n_cl, rv.n_lp == 0);
  const int N = a.B * a.H;
  const int total_warps = gridDim.x * nwarps;
  int e = blockIdx.x * nwarps + warp;
  while (e < N) {
    int b = e, h = 0;
    if (a.H != 1) {
      b = e / a.H;
      h = e - b * a.H;
    }
    float cs_cost = 0.0f, pose_c = 0.0f;
    row_phase_a<false, 32, false>(a, rv, es, lane, e, b, h, cs_cost, pose_c);
    int n_list;
    bool dense;
    const RowB1 r = row_phase_b1_list<SCENE, SMALL, false>(a, rv, es, lane, e, b, n_list, dense);
    row_phase_b2_list<SMALL, false>(a, rv, es, lane, e, r, cs_cost, pose_c, n_list, dense);
    e = next_warp_unit(a.work_counter, e, total_warps, lane == 0);
  }
  if (a.work_counter != nullptr && lane == 0) rearm_ticket_counter(a.work_counter, total_warps);
}

// ------------------------------------------------------------------------------------------------
// Small-batch variant of the big-robot kernel: a TEAM of warps per row.
//
// When a GPU holds fewer rows than resident warps -- BASELINE config 5 on eight H100s is 1,024 humanoid rows for 2,112 warp
// slots -- the launch takes one row's latency however idle the SMs are.  Here TEAM (2 or 4) warps share one
// row's state and split its parallel phases: local link transforms, spheres, link bounds, the link-pair scan, the ESDF sphere
// loop and the list-based J^T are strided over TEAM x 32 lanes; the serial parts (c-space, the level-scheduled FK compose) run
// on the team's first warp, the tool-pose cost on its last; teams meet at named barriers (one id per team), every team has its
// own gradient-list segment (a full segment is folded into the warp's partial sums and restarted: no overflow case;
// deterministic) and partial J^T accumulators.  The host picks the variant from rows vs resident warp slots (see the launcher).
// ------------------------------------------------------------------------------------------------
template <int TEAM>
struct TeamScratch {  // per team, behind the row state
  unsigned long long key[TEAM];
  float scene_c[TEAM];
  float cs_cost, pose_c;
  int next_row, pad;
};
// Every warp of a team has its own kGradListCap-entry list segment (the first warp uses the row's own list).  A warp whose segment
// fills up -- a row deep in collision -- folds the segment into its J^T partial sums on the spot and starts it again
// (team_flush_list: out of line, cold), so a segment never overflows and no row is ever redone.
__host__ __device__ inline int team_extra_floats(int team, int nl) {
  return team * nl + 28 + 4 * team + (team - 1) * kGradListCap * 4;
}
static __device__ __noinline__ void team_flush_list(const unsigned char *smem_blob, const unsigned char *gmem_blob, float *base,
                                                    int lane, const float4 *list, int n, float *acc0, float *acc1) {
  const RobotView rv = make_robot_view(smem_blob, gmem_blob);
  const EvalSmem es = carve_big_smem(base, rv.nl, rv.D, rv.S, rv.L, rv.n_cl);
  float t[2];
  warp_list_accumulate(rv, es, lane, list, n, false, t);
  *acc0 += t[0];
  *acc1 += t[1];
}

template <int SCENE, int TEAM>
__global__ void __launch_bounds__(kBigWarps * 32, 1) rollout_fused_team_kernel(const __grid_constant__ FusedArgs a) {
  CB200_EXTERN_SHARED __align__(128) unsigned char smem[];
  __shared__ unsigned long long mbar;
  stage_blob_to_smem(smem, a.blob, (uint32_t)a.blob_smem_bytes, &mbar);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int team = warp / TEAM, tw = warp - team * TEAM, nteams = nwarps / TEAM;
  const int tlane = tw * 32 + lane, tsize = TEAM * 32;  // lane index / lane count inside the team
  if (team >= nteams) return;                             // (blockDim is a multiple of TEAM * 32; kept for safety)
  float *base = reinterpret_cast<float *>(smem + a.blob_smem_bytes) + (size_t)team * a.eval_floats;
  const RobotView rv = make_robot_view(smem, a.blob);
  const EvalSmem es = carve_big_smem(base, rv.nl, rv.D, rv.S, rv.L, rv.n_cl);
  float *extra = base + big_smem_floats(rv.nl, rv.D, rv.S, rv.L, rv.n_cl);
  float *partial = extra;                                   // [TEAM][nl] J^T accumulators
  TeamScratch<TEAM> *ts = reinterpret_cast<TeamScratch<TEAM> *>(extra + ((TEAM * rv.nl + 1) & ~1));
  float4 *my_list =
      tw == 0 ? es.glist : reinterpret_cast<float4 *>(extra + ((TEAM * rv.nl + 24 + 4 * TEAM + 3) & ~3)) + (tw - 1) * kGradListCap;
  const int bar_id = 1 + team;
  const cb200_rollout_cfg &cfg = a.cfg;
  const int N = a.B * a.H, S = rv.S, D = rv.D;
  const int total_teams = gridDim.x * nteams;
  int e = blockIdx.x * nteams + team;
  while (e < N) {
    int b = e, h = 0;
    if (a.H != 1) {
      b = e / a.H;
      h = e - b * a.H;
    }
    // ---------------- phase A
    if (tw == 0) {
      const float cs = warp_sum(row_cspace<false>(a, rv, es, lane, e, b, h));
      if (lane == 0) ts->cs_cost = cs;
    }
    CB200_NAMED_BARRIER(bar_id, tsize);
    {  // local link transforms over the whole team (scratch = the not-yet-written sphere area, as warp_fk)
      const bool scratch = rv.S * 4 >= rv.nl * 12;
      float *loc = scratch ? reinterpret_cast<float *>(es.sph) : es.cumul;
      if (scratch || tw == 0) {
#pragma unroll 1
        for (int l = scratch ? tlane : lane; l < rv.nl; l += scratch ? tsize : 32) {
          const int jt = rv.joint_type[l];
          float th = 0.0f;
          if (jt >= 0) th = rv.joff[2 * l] * es.qv[rv.joint_map[l]] + rv.joff[2 * l + 1];
          local_link_transform(rv.fixed + 12 * l, jt, th, (l == 0 ? es.cumul : loc) + 12 * l);
        }
      }
    }
    CB200_NAMED_BARRIER(bar_id, tsize);
    if (tw == 0) warp_fk_compose(rv, es, lane);
    CB200_NAMED_BARRIER(bar_id, tsize);
    {  // spheres over the whole team: warp_spheres' vector loads of the link transform took the 2-warp build from 126 to 128 registers
      const float4 *cfg_sph = row_sphere_cfg(a, b, S);
      float4 *out_global = a.robot_spheres ? reinterpret_cast<float4 *>(a.robot_spheres) + (size_t)e * S : nullptr;
#pragma unroll 1
      for (int s = tlane; s < S; s += tsize) {
        const float *T = es.cumul + 12 * rv.sph_link[s];
        const float4 p = cfg_sph != nullptr ? __ldg(cfg_sph + s) : rv.spheres[s];
        const float4 w = make_float4(T[0] * p.x + T[1] * p.y + T[2] * p.z + T[3], T[4] * p.x + T[5] * p.y + T[6] * p.z + T[7],
                                     T[8] * p.x + T[9] * p.y + T[10] * p.z + T[11], p.w);
        es.sph[s] = w;
        if (out_global != nullptr) out_global[s] = w;
      }
    }
    link_bounds<TEAM * 32>(rv, es, tlane);
    if (tw == TEAM - 1) {
      const float pose_c = warp_sum(row_tool_poses(a, rv, es, lane, e, b, h));
      if (lane == 0) ts->pose_c = pose_c;
    }
    CB200_NAMED_BARRIER(bar_id, tsize);
    // ---------------- phase B1: self collision (interleaved slices of the link-pair list), then scene collision
    float self_c = 0.0f, fmax = 0.0f;
    int bi = 0, bj = 0;
    if (cfg.self_weight > 0.0f && rv.P > 0) {
      unsigned long long key = 0ull;
      int di, dj;
      warp_self_collision_tiles<false>(rv, es, lane, di, dj, tw * 32, tsize, reinterpret_cast<unsigned char *>(es.ft) + 64 * tw, &key,
                                       false);
      if (lane == 0) ts->key[tw] = key;
      CB200_NAMED_BARRIER(bar_id, tsize);
      unsigned long long best = 0ull;
#pragma unroll
      for (int w = 0; w < TEAM; ++w) best = ts->key[w] > best ? ts->key[w] : best;
      if (best != 0ull) {
        bi = 0xffff - (int)((best >> 16) & 0xffffu);
        bj = 0xffff - (int)(best & 0xffffu);
        fmax = __uint_as_float((uint32_t)(best >> 32));
        self_c = 0.5f * cfg.self_weight * fmax;
      }
    }
    if (a.self_cost && tlane == 0) a.self_cost[e] = self_c;
    const bool do_scene = SCENE != 0 && cfg.scene_weight > 0.0f;
    const int env = (a.env_query_idx != nullptr) ? __ldg(a.env_query_idx + b) : 0;
    CuboidCull cc{0, 0, false};
    if (has_cuboids<SCENE>(a, do_scene)) {
      if (cuboid_cull_state(a, rv, env, true, cc)) {
        cuboid_cull_masks(a, rv, es, cc.ce, cc.ncub, tlane, tsize);
        CB200_NAMED_BARRIER(bar_id, tsize);
      }
    }
    int n_list = 0;
    float scene_c = 0.0f, flushed0 = 0.0f, flushed1 = 0.0f;
    const unsigned lt = (1u << lane) - 1u;
#pragma unroll 1
    for (int sb = tw * 32; sb < S; sb += tsize) {  // this warp's passes; uniform trip count inside the warp
      const int s = sb + lane;
      V3 g = mk3(0, 0, 0);
      float c = 0.0f;
      if (s < S && do_scene) c = sphere_discrete_terms<SCENE>(a, rv, es, cc, env, s, g);
      const bool nz = (g.x != 0.0f) || (g.y != 0.0f) || (g.z != 0.0f);
      const unsigned m = __ballot_sync(kFull, nz);
      if (m) {
        if (n_list + __popc(m) > kGradListCap - 2) {  // (two slots stay free for the self-collision pair)
          __syncwarp();
          team_flush_list(smem, a.blob, base, lane, my_list, n_list, &flushed0, &flushed1);
          __syncwarp();
          n_list = 0;
        }
        if (nz) my_list[n_list + __popc(m & lt)] = make_float4(g.x, g.y, g.z, __int_as_float(s));
        n_list += __popc(m);
      }
      scene_c += c;
      if (a.scene_cost && s < S) a.scene_cost[(size_t)e * S + s] = c;
    }
    scene_c = warp_sum(scene_c);
    if (lane == 0) ts->scene_c[tw] = scene_c;
    {
      // ---------------- phase B2: J^T over the team's list segments
      if (tw == 0 && fmax > 0.0f) append_self_pair(a, es, lane, bi, bj, my_list, n_list);
      __syncwarp();  // the warp's list entries are visible to all of its lanes
      float acc[2];
      warp_list_accumulate(rv, es, lane, my_list, n_list, tw == 0, acc);
      acc[0] += flushed0;
      acc[1] += flushed1;
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int j = lane + 32 * u;
        if (j < rv.nl) partial[tw * rv.nl + j] = acc[u];
      }
      CB200_NAMED_BARRIER(bar_id, tsize);
      if (tw == 0) {
        for (int j = lane; j < rv.nl; j += 32) {
          float c = 0.0f;
#pragma unroll
          for (int w = 0; w < TEAM; ++w) c += partial[w * rv.nl + j];
          es.contrib[j] = c;
        }
        __syncwarp();
        float *gq = a.grad_q + (size_t)e * D;
        for (int d = lane; d < D; d += 32) {
          float g = es.gqv[d];
          for (int i = rv.jl_off[d]; i < rv.jl_off[d + 1]; ++i) g += es.contrib[rv.jl_idx[i]];
          gq[d] = g;
        }
        if (lane == 0) {
          float tot = ts->cs_cost + ts->pose_c + self_c;
#pragma unroll
          for (int w = 0; w < TEAM; ++w) tot += ts->scene_c[w];
          a.cost[e] = tot;
        }
      }
    }
    // ---------------- next row
    if (tw == 0 && lane == 0) ts->next_row = a.work_counter != nullptr ? total_teams + atomicAdd(a.work_counter, 1) : e + total_teams;
    CB200_NAMED_BARRIER(bar_id, tsize);
    e = ts->next_row;
    CB200_NAMED_BARRIER(bar_id, tsize);  // every warp has read next_row / the row state before the next row rewrites them
  }
  if (a.work_counter != nullptr && tw == 0 && lane == 0) rearm_ticket_counter(a.work_counter, total_teams);
}

// ------------------------------------------------------------------------------------------------
// THE fused kernel, trajectory mode (swept scene collision + speed metric couple row h to h-1, h+1).
// A CTA walks tiles of `nwarps` consecutive waypoints of one seed: every warp runs phase A for its
// waypoint (warp 0 / the last warp also compute the halo waypoints' spheres), the CTA synchronises, then
// every warp runs phase B reading its neighbours' sphere positions from shared memory.
// ------------------------------------------------------------------------------------------------
// Halo waypoints of the tile h0 .. h0 + nwarps - 1 of seed b, spheres only: warp 0 writes those of h0 - 1 to halo_prev, the last
// warp those of h0 + nwarps to halo_next (when the trajectory has them).  Uses the warp's row state as scratch.
template <bool SPLINE>
__device__ __forceinline__ void tile_halo(const FusedArgs &a, const RobotView &rv, const EvalSmem &es, int lane, int warp, int nwarps,
                                          int b, int h0, float4 *halo_prev, float4 *halo_next) {
  const int D = rv.D, S = rv.S;
  int hh = -1;
  float4 *hdst = nullptr;
  if (warp == 0 && h0 > 0) {
    hh = h0 - 1;
    hdst = halo_prev;
  } else if (warp == nwarps - 1 && h0 + nwarps < a.H) {
    hh = h0 + nwarps;
    hdst = halo_next;
  }
  if (hh >= 0) {
    const size_t eh = (size_t)b * a.H + hh;
    for (int d = lane; d < D; d += 32)
      es.qv[d] = SPLINE ? spline_row_state(a.spl, b, hh, d, D).p : __ldg(a.q + eh * D + d);
    __syncwarp();
    warp_fk(rv, es, lane);
    const float4 *cfg_sph = row_sphere_cfg(a, b, S);
    for (int s = lane; s < S; s += 32) {
      const float *T = es.cumul + 12 * rv.sph_link[s];
      const float4 p = cfg_sph != nullptr ? __ldg(cfg_sph + s) : rv.spheres[s];
      hdst[s] = make_float4(T[0] * p.x + T[1] * p.y + T[2] * p.z + T[3], T[4] * p.x + T[5] * p.y + T[6] * p.z + T[7],
                            T[8] * p.x + T[9] * p.y + T[10] * p.z + T[11], p.w);
    }
    __syncwarp();
  }
}

// Spheres of a neighbouring waypoint for the swept terms: those of warp nb's row when nb is in the tile (`all` holds the warps'
// eval_floats slices), else the halo
__device__ __forceinline__ const float4 *neighbour_spheres(const FusedArgs &a, const RobotView &rv, const float *all, int nb, bool in_tile,
                                                          const float4 *halo) {
  return in_tile ? reinterpret_cast<const float4 *>(all + (size_t)nb * a.eval_floats + rv.nl * 12) : halo;
}

// SMALL: arms (<= 24 links, <= 128 spheres): whole-block self-collision scan and the one-slot sparse J^T (see the IK arm build).
template <int SCENE, bool SPLINE, bool SMALL = false>
__global__ void __launch_bounds__(kWarpsPerCta * 32, kMinCtas) rollout_traj_kernel(const __grid_constant__ FusedArgs a) {
  CB200_EXTERN_SHARED __align__(128) unsigned char smem[];
  __shared__ unsigned long long mbar;
  stage_blob_to_smem(smem, a.blob, (uint32_t)a.blob_smem_bytes, &mbar);
  const RobotView rv = make_robot_view(smem, a.blob);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  float *all = reinterpret_cast<float *>(smem + a.blob_smem_bytes);
  const EvalSmem es = carve_eval_smem(all + (size_t)warp * a.eval_floats, rv.nl, rv.D, rv.S, rv.L, rv.n_cl);
  float4 *halo_prev = reinterpret_cast<float4 *>(all + (size_t)nwarps * a.eval_floats);
  float4 *halo_next = halo_prev + rv.S;
  const int tiles_per_seed = (a.H + nwarps - 1) / nwarps;
  const long long n_tiles = (long long)a.B * tiles_per_seed;
  __shared__ int next_tile;  // tiles after a CTA's first come from the ticket counter (tiles differ in cost: see rollout_fused_kernel)
  for (long long tile = blockIdx.x; tile < n_tiles;) {
    const int b = (int)(tile / tiles_per_seed);
    const int h0 = (int)(tile - (long long)b * tiles_per_seed) * nwarps;
    const int h = h0 + warp;
    const bool active = h < a.H;
    tile_halo<SPLINE>(a, rv, es, lane, warp, nwarps, b, h0, halo_prev, halo_next);
    const int e = b * a.H + h;
    float cs_cost = 0.0f, pose_c = 0.0f;
    RowB1 r{0.0f, 0.0f, 0.0f, 0, 0, 0};
    if (active) row_phase_a<SPLINE>(a, rv, es, lane, e, b, h, cs_cost, pose_c);
    __syncthreads();
    if (active) {
      const float4 *prev = nullptr, *next = nullptr;
      if (h > 0) prev = neighbour_spheres(a, rv, all, warp - 1, warp > 0, halo_prev);
      if (h < a.H - 1) next = neighbour_spheres(a, rv, all, warp + 1, warp < nwarps - 1, halo_next);
      r = row_phase_b1<true, SCENE, !SMALL>(a, rv, es, lane, e, b, prev, next);
    }
    if (threadIdx.x == 0 && a.work_counter != nullptr) next_tile = (int)gridDim.x + atomicAdd(a.work_counter, 1);
    __syncthreads();
    if (active) row_phase_b2<SMALL>(a, rv, es, smem, lane, e, r, cs_cost, pose_c);
    // (next_tile is rewritten only after the next iteration's first __syncthreads, which every thread passes after this read)
    tile = a.work_counter != nullptr ? (long long)next_tile : tile + gridDim.x;
  }
  if (a.work_counter != nullptr && threadIdx.x == 0) rearm_ticket_counter(a.work_counter, (int)gridDim.x);
}

// ------------------------------------------------------------------------------------------------
// Trajectory mode with the dynamics-aware STATE cost (SURVEY.md 8f rank 3): tau = RNEA(q, qd, qdd) of every row, the
// effort channel of the STATE cost on it (bound hinge, squared-L2, energy (tau qd dt)^2: wp_cspace_state.py:209-275) and
// the RNEA adjoint of d cost / d tau onto the position / velocity / acceleration gradients -- tau never leaves the SM.
//
// A CTA owns a CHUNK of R consecutive waypoints of one seed (R = 32 / 16 / 8, a multiple of the warp count) and alternates
// between two mappings:
//   dynamics phase   thread = (row r = tid % R, worker w = tid / R): the lanes of a warp are different rows walking the same
//                    link (cb200_dynamics_tile.cuh: level-synchronous recursions, everything else over (link, row) pairs,
//                    the row state in a transposed shared-memory tile); results stay in the tile's IO rows
//   tile phase       the chunk's waypoints, nwarps at a time, exactly as rollout_traj_kernel (warp per waypoint, halo
//                    waypoints either side), each row adding its dynamics terms from the IO rows.
// Measured on the MPC workload (1024 x 30, H100): plain trajectory kernel 0.34 ms; this kernel 0.55 ms; the host composition
// (three more launches, HBM round trip of the 80 B / link cache) 0.53 ms -- which is why RolloutEngine.attach_dynamics defaults
// to the host composition.  Running the recursion on lane 0 of every row's warp inside phase A was slower.  A warp-specialised
// pipeline (one dynamics warp producing chunk c + 1 while the row warps roll out chunk c) was built and was slower too: the
// dynamics of a chunk is ~32 k warp-instructions, which a single warp issues more slowly than eight warps roll the chunk out.
// ------------------------------------------------------------------------------------------------
template <int SCENE>
__global__ void __launch_bounds__(kWarpsPerCta * 32, kMinCtas) rollout_traj_dyn_kernel(const __grid_constant__ FusedArgs a,
                                                                                         const int R) {
  CB200_EXTERN_SHARED __align__(128) unsigned char smem[];
  __shared__ unsigned long long mbar;
  stage_blob_to_smem(smem, a.blob, (uint32_t)a.blob_smem_bytes, &mbar);
  const RobotView rv = make_robot_view(smem, a.blob);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  float *all = reinterpret_cast<float *>(smem + a.blob_smem_bytes);
  const EvalSmem es = carve_eval_smem(all + (size_t)warp * a.eval_floats, rv.nl, rv.D, rv.S, rv.L, rv.n_cl);
  float4 *halo_prev = reinterpret_cast<float4 *>(all + (size_t)nwarps * a.eval_floats);
  float4 *halo_next = halo_prev + rv.S;
  const int D = rv.D, S = rv.S, nl = rv.nl, RS = R + 1;
  float *dynbase = reinterpret_cast<float *>(halo_next + S);
  // the tree part of the model points into the shared-memory copy of the robot blob (plain loads: the read-only global path
  // must not be used on shared addresses); the inertial parameters are the caller's arrays in global memory
  const dyn::Model M{rv.fixed, a.dyn.masses_com, a.dyn.inertias, rv.joint_type, rv.joint_map, rv.link_map, rv.joff,
                     a.dyn.gravity, rv.level_off, rv.level_links, nl, D, rv.n_levels};
  const dyn::Tile<dyn::LdPlain> T{dynbase, dynbase + 5 * nl * 6 * RS, dynbase + (5 * 6 + 2) * nl * RS, nl, D, RS,
                                  (int)threadIdx.x % R, (int)threadIdx.x / R, (int)blockDim.x / R, M};
  const cb200_rollout_cfg &cfg = a.cfg;
  const int chunks_per_seed = (a.H + R - 1) / R;
  const long long n_chunks = (long long)a.B * chunks_per_seed;
  for (long long chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
    const int b = (int)(chunk / chunks_per_seed);
    const int c0 = (int)(chunk - (long long)b * chunks_per_seed) * R;
    const int rows = (a.H - c0) < R ? (a.H - c0) : R;
    const size_t e0 = (size_t)b * a.H + c0;
    // ---------------- dynamics phase
    for (int i = threadIdx.x; i < R * D; i += blockDim.x) {  // coalesced: the chunk's rows are contiguous in q / vel / acc
      const int rr = i / D, d = i - rr * D;
      const bool ok = rr < rows;
      const size_t gi = e0 * D + i;
      T.IO[(0 * D + d) * RS + rr] = ok ? __ldg(a.q + gi) : 0.0f;
      T.IO[(1 * D + d) * RS + rr] = ok ? __ldg(a.vel + gi) : 0.0f;
      T.IO[(2 * D + d) * RS + rr] = ok ? __ldg(a.acc + gi) : 0.0f;
      T.IO[(3 * D + d) * RS + rr] = 0.0f;
    }
    __syncthreads();
    dyn::tile_rnea_forward<dyn::SyncCta>(T);
    {
      const float dt = seed_dt(a, b);
      float w_b = cfg.cspace_weight[4], w_l2 = cfg.cspace_reg[3], w_en = cfg.cspace_reg[4];
      if (cfg.retime_regularization_weights) w_en = dt * w_en;
      const float *lim = rv.limits;
      for (int i = threadIdx.x; i < R * D; i += blockDim.x) {  // effort terms per (row, dof)
        const int rr = i / D, d = i - rr * D;
        const float tau = T.IO[(3 * D + d) * RS + rr], v = T.IO[(1 * D + d) * RS + rr];
        float c = 0.0f, gt = 0.0f, gve = 0.0f;
        bound_cost(tau, lim[8 * D + d], lim[9 * D + d], cfg.cspace_activation[4], w_b, c, gt);
        l2_reg(tau, w_l2, c, gt);
        if (w_en > 0.0f) {
          const float ce = tau * v * dt;
          c += w_en * ce * ce;
          gt += 2.0f * w_en * ce * v * dt;
          gve = 2.0f * w_en * ce * tau * dt;
        }
        T.IO[(3 * D + d) * RS + rr] = gt;
        T.IO[(4 * D + d) * RS + rr] = 0.0f;
        T.IO[(5 * D + d) * RS + rr] = gve;
        T.IO[(6 * D + d) * RS + rr] = 0.0f;
        T.IO[(7 * D + d) * RS + rr] = c;
      }
    }
    __syncthreads();
    dyn::tile_rnea_backward<dyn::SyncCta>(T);
    // ---------------- tile phase: the chunk's waypoints, nwarps at a time
    for (int t0 = 0; t0 < rows; t0 += nwarps) {
      const int h0 = c0 + t0;
      const int h = h0 + warp;
      const bool active = h < a.H;
      tile_halo<false>(a, rv, es, lane, warp, nwarps, b, h0, halo_prev, halo_next);
      const int e = b * a.H + h;
      float cs_cost = 0.0f, pose_c = 0.0f;
      RowB1 r{0.0f, 0.0f, 0.0f, 0, 0, 0};
      if (active) {
        row_phase_a<false>(a, rv, es, lane, e, b, h, cs_cost, pose_c);
        const int rr = t0 + warp;  // this row's column of the dynamics tile; lane d owns dof d here and in cspace_dof
#pragma unroll 1
        for (int d = lane; d < D; d += 32) {
          es.gqv[d] += T.IO[(4 * D + d) * RS + rr];
          const float c = T.IO[(7 * D + d) * RS + rr];
          cs_cost += c;
          const size_t gi = (size_t)e * D + d;
          if (a.cspace_cost) a.cspace_cost[gi] += c;
          if (a.grad_vel) a.grad_vel[gi] += T.IO[(5 * D + d) * RS + rr];
          if (a.grad_acc) a.grad_acc[gi] += T.IO[(6 * D + d) * RS + rr];
        }
        __syncwarp();
      }
      __syncthreads();
      if (active) {
        const float4 *prev = nullptr, *next = nullptr;
        if (h > 0) prev = neighbour_spheres(a, rv, all, warp - 1, warp > 0, halo_prev);
        if (h < a.H - 1) next = neighbour_spheres(a, rv, all, warp + 1, warp < nwarps - 1, halo_next);
        r = row_phase_b1<true, SCENE>(a, rv, es, lane, e, b, prev, next);
      }
      __syncthreads();
      if (active) row_phase_b2(a, rv, es, smem, lane, e, r, cs_cost, pose_c);
    }
    __syncthreads();  // the next chunk's dynamics phase rewrites the tile the last rows just read
  }
}

// ------------------------------------------------------------------------------------------------
// Drop-in FK forward: warp per row, parameters read from global memory (L1-resident, a few KB).
// ------------------------------------------------------------------------------------------------
struct KinFwdArgs {
  float *link_pos, *link_quat, *spheres_out, *cumul_out;
  const float *q, *fixed, *robot_spheres, *joff;
  const int8_t *jtype;
  const int16_t *jmap, *lmap, *tool_map, *sph_link;
  const int32_t *env_query_idx;
  int num_envs, N, horizon, D, S, nl, L, write_cumul;
  // centre of mass (COM instantiation only): link_masses_com [nl,4] = local CoM xyz, mass; com_out [N,4] = world CoM xyz, total mass
  const float *masses_com;
  float *com_out;
};

template <bool COM = false>
__global__ void __launch_bounds__(kWarpsPerCta * 32) kin_forward_kernel(const __grid_constant__ KinFwdArgs a) {
  CB200_EXTERN_SHARED __align__(16) float fsm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float *cumul = fsm + (size_t)warp * a.nl * 12;
  for (int e = blockIdx.x * kWarpsPerCta + warp; e < a.N; e += gridDim.x * kWarpsPerCta) {
    for (int l = lane; l < a.nl; l += 32) {
      const int jt = a.jtype[l];
      float th = 0.0f;
      if (jt >= 0) th = __ldg(a.joff + 2 * l) * __ldg(a.q + (size_t)e * a.D + a.jmap[l]) + __ldg(a.joff + 2 * l + 1);
      local_link_transform(a.fixed + 12 * l, jt, th, cumul + 12 * l);
    }
    __syncwarp();
    const int k = lane, r = k >> 2, c = k & 3;
    for (int l = 1; l < a.nl; ++l) {  // parents precede children: index order is a valid schedule
      float out = 0.0f;
      if (k < 12) {
        const float *P = cumul + 12 * a.lmap[l];
        const float *Lm = cumul + 12 * l;
        const float4 pr = *reinterpret_cast<const float4 *>(P + 4 * r);
        out = pr.x * Lm[c] + pr.y * Lm[4 + c] + pr.z * Lm[8 + c] + (c == 3 ? pr.w : 0.0f);
      }
      __syncwarp();
      if (k < 12) cumul[12 * l + k] = out;
      __syncwarp();
    }
    if (a.write_cumul) {
      float4 *dst = reinterpret_cast<float4 *>(a.cumul_out + (size_t)e * a.nl * 12);
      const float4 *src = reinterpret_cast<const float4 *>(cumul);
      for (int i = lane; i < a.nl * 3; i += 32) dst[i] = src[i];
    }
    const int cfg = (a.num_envs > 1) ? __ldg(a.env_query_idx + e / a.horizon) : 0;
    const float4 *ls = reinterpret_cast<const float4 *>(a.robot_spheres) + (size_t)cfg * a.S;
    float4 *so = reinterpret_cast<float4 *>(a.spheres_out) + (size_t)e * a.S;
    for (int s = lane; s < a.S; s += 32) {
      const float *T = cumul + 12 * a.sph_link[s];
      const float4 p = __ldg(ls + s);
      float4 w;
      w.x = T[0] * p.x + T[1] * p.y + T[2] * p.z + T[3];
      w.y = T[4] * p.x + T[5] * p.y + T[6] * p.z + T[7];
      w.z = T[8] * p.x + T[9] * p.y + T[10] * p.z + T[11];
      w.w = p.w;
      so[s] = w;
    }
    for (int t = lane; t < a.L; t += 32) {
      const float *T = cumul + 12 * a.tool_map[t];
      const Q4 qt = quat_from_transform(T);
      float *o = a.link_pos + ((size_t)e * a.L + t) * 3;
      o[0] = T[3];
      o[1] = T[7];
      o[2] = T[11];
      *reinterpret_cast<float4 *>(a.link_quat + ((size_t)e * a.L + t) * 4) = make_float4(qt.w, qt.x, qt.y, qt.z);
    }
    if constexpr (COM) {  // mass-weighted mean of the links' centres of mass (kinematics_forward_helper.cuh:538-601)
      float sx = 0.0f, sy = 0.0f, sz = 0.0f, sm = 0.0f;
      for (int l = lane; l < a.nl; l += 32) {
        const float4 mc = __ldg(reinterpret_cast<const float4 *>(a.masses_com) + l);
        if (mc.w > 0.0f) {
          const float *T = cumul + 12 * l;
          sx += mc.w * (T[0] * mc.x + T[1] * mc.y + T[2] * mc.z + T[3]);
          sy += mc.w * (T[4] * mc.x + T[5] * mc.y + T[6] * mc.z + T[7]);
          sz += mc.w * (T[8] * mc.x + T[9] * mc.y + T[10] * mc.z + T[11]);
          sm += mc.w;
        }
      }
      sx = warp_sum(sx), sy = warp_sum(sy), sz = warp_sum(sz), sm = warp_sum(sm);
      if (lane == 0) {
        float4 o = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (sm > 0.0f) o = make_float4(sx / sm, sy / sm, sz / sm, sm);
        *reinterpret_cast<float4 *>(a.com_out + (size_t)e * 4) = o;
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// Drop-in FK backward: warp per row; cumul re-read from global; link force/torque accumulators.
// ------------------------------------------------------------------------------------------------
struct KinBwdArgs {
  float *grad_out;
  const float *g_pos, *g_quat, *g_sph, *cumul, *robot_spheres, *joff;
  const int16_t *lmap, *jmap, *tool_map, *sph_link;
  const int8_t *jtype;
  const int32_t *env_query_idx;
  int num_envs, N, horizon, D, S, nl, L;
  // centre-of-mass gradient (COM instantiation only): g_com [N,4] (w ignored), com [N,4] (w = total mass), masses_com [nl,4]
  const float *g_com, *com, *masses_com;
};

template <bool COM = false>
__global__ void __launch_bounds__(kWarpsPerCta * 32) kin_backward_kernel(const __grid_constant__ KinBwdArgs a) {
  CB200_EXTERN_SHARED __align__(16) float fsm[];
  // CTA-shared: ancestor masks [nl] (uint64)
  unsigned long long *anc = reinterpret_cast<unsigned long long *>(fsm);
  const int anc_floats = (2 * a.nl + 3) & ~3, per_warp = (a.nl * 12 + a.nl * 8 + a.nl + a.D + 3) & ~3;  // keep float4 alignment
  float *wbase = fsm + anc_floats + (size_t)(threadIdx.x >> 5) * per_warp;
  float *cumul = wbase, *ft = wbase + a.nl * 12, *contrib = ft + a.nl * 8, *gq = contrib + a.nl;
  if (threadIdx.x == 0) {
    anc[0] = 1ull;
    for (int l = 1; l < a.nl; ++l) anc[l] = anc[a.lmap[l]] | (1ull << l);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int e = blockIdx.x * kWarpsPerCta + warp; e < a.N; e += gridDim.x * kWarpsPerCta) {
    {
      const float4 *src = reinterpret_cast<const float4 *>(a.cumul + (size_t)e * a.nl * 12);
      float4 *dst = reinterpret_cast<float4 *>(cumul);
      for (int i = lane; i < a.nl * 3; i += 32) dst[i] = __ldg(src + i);
    }
    for (int i = lane; i < a.nl * 8; i += 32) ft[i] = 0.0f;
    for (int d = lane; d < a.D; d += 32) gq[d] = 0.0f;
    __syncwarp();
    const int cfg = (a.num_envs > 1) ? __ldg(a.env_query_idx + e / a.horizon) : 0;
    // lane per link gathers its spheres (deterministic order)
    for (int k = lane; k < a.nl; k += 32) {
      const float *Tk = cumul + 12 * k;
      const V3 o = mk3(Tk[3], Tk[7], Tk[11]);
      V3 F = mk3(0, 0, 0), T = mk3(0, 0, 0);
      if (a.g_sph != nullptr) {
        for (int s = 0; s < a.S; ++s) {
          if (a.sph_link[s] != k) continue;
          const float4 g4 = __ldg(reinterpret_cast<const float4 *>(a.g_sph) + (size_t)e * a.S + s);
          if (g4.x == 0.0f && g4.y == 0.0f && g4.z == 0.0f) continue;
          const float4 p = __ldg(reinterpret_cast<const float4 *>(a.robot_spheres) + (size_t)cfg * a.S + s);
          const V3 rel = mk3(Tk[0] * p.x + Tk[1] * p.y + Tk[2] * p.z, Tk[4] * p.x + Tk[5] * p.y + Tk[6] * p.z,
                             Tk[8] * p.x + Tk[9] * p.y + Tk[10] * p.z);  // p_world - o_k
          const V3 g = mk3(g4.x, g4.y, g4.z);
          F = F + g;
          T = T + cross(rel, g);
        }
      }
      if (a.g_pos != nullptr) {
        for (int t = 0; t < a.L; ++t) {
          if (a.tool_map[t] != k) continue;
          const float *gp = a.g_pos + ((size_t)e * a.L + t) * 3;
          const float4 gqv = __ldg(reinterpret_cast<const float4 *>(a.g_quat) + (size_t)e * a.L + t);
          const V3 g = mk3(__ldg(gp), __ldg(gp + 1), __ldg(gp + 2));
          if (g.x == 0.0f && g.y == 0.0f && g.z == 0.0f && gqv.x == 0.0f && gqv.y == 0.0f && gqv.z == 0.0f && gqv.w == 0.0f)
            continue;
          const Q4 qt = quat_from_transform(Tk);
          F = F + g;
          T = T + quat_grad_to_omega(qt, gqv.x, gqv.y, gqv.z, gqv.w);
        }
      }
      if constexpr (COM) {
        // d loss / d CoM acts on link k as the force g * m_k / M applied at the link's world centre of mass
        // (kinematics_backward_helper.cuh:187-260: compute_center_of_mass_gradients walks the same chain as a sphere)
        const float4 mc = __ldg(reinterpret_cast<const float4 *>(a.masses_com) + k);
        const float M = __ldg(a.com + (size_t)e * 4 + 3);
        const V3 gc = mk3(__ldg(a.g_com + (size_t)e * 4), __ldg(a.g_com + (size_t)e * 4 + 1), __ldg(a.g_com + (size_t)e * 4 + 2));
        if (mc.w > 0.0f && M > 0.0f && !(gc.x == 0.0f && gc.y == 0.0f && gc.z == 0.0f)) {
          const float sc = mc.w / M;
          const V3 g = mk3(gc.x * sc, gc.y * sc, gc.z * sc);
          const V3 rel = mk3(Tk[0] * mc.x + Tk[1] * mc.y + Tk[2] * mc.z, Tk[4] * mc.x + Tk[5] * mc.y + Tk[6] * mc.z,
                             Tk[8] * mc.x + Tk[9] * mc.y + Tk[10] * mc.z);
          F = F + g;
          T = T + cross(rel, g);
        }
      }
      ft[8 * k + 0] = F.x;
      ft[8 * k + 1] = F.y;
      ft[8 * k + 2] = F.z;
      ft[8 * k + 4] = T.x;
      ft[8 * k + 5] = T.y;
      ft[8 * k + 6] = T.z;
    }
    __syncwarp();
    for (int j = lane; j < a.nl; j += 32) {
      const int jt = a.jtype[j];
      float res = 0.0f;
      if (jt >= 0) {
        const float *Tj = cumul + 12 * j;
        const V3 oj = mk3(Tj[3], Tj[7], Tj[11]);
        V3 F = mk3(0, 0, 0), T = mk3(0, 0, 0);
        for (int k = j; k < a.nl; ++k) {
          if (!((anc[k] >> j) & 1ull)) continue;
          const V3 Fk = mk3(ft[8 * k], ft[8 * k + 1], ft[8 * k + 2]);
          const float *Tk = cumul + 12 * k;
          F = F + Fk;
          T = T + mk3(ft[8 * k + 4], ft[8 * k + 5], ft[8 * k + 6]) + cross(mk3(Tk[3], Tk[7], Tk[11]) - oj, Fk);
        }
        const int ax = (jt >= JT_XR) ? jt - JT_XR : jt;
        const V3 av = mk3(Tj[ax], Tj[4 + ax], Tj[8 + ax]);
        res = __ldg(a.joff + 2 * j) * ((jt >= JT_XR) ? dot(av, T) : dot(av, F));
      }
      contrib[j] = res;
    }
    __syncwarp();
    for (int d = lane; d < a.D; d += 32) {
      float g = 0.0f;
      for (int j = 0; j < a.nl; ++j)
        if (a.jmap[j] == d && a.jtype[j] >= 0) g += contrib[j];
      a.grad_out[(size_t)e * a.D + d] = g;
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// Drop-in self collision.  TPE threads per eval: 32 (warp) for short pair lists, 256 (CTA) otherwise.
// ------------------------------------------------------------------------------------------------
struct SelfArgs {
  float *out_distance, *out_vec, *pair_distance;
  uint8_t *sparse_index;
  const float *spheres, *padding, *weight;
  const uint32_t *pairs;
  int N, S, P, store_pair, compute_grad;
};

template <int TPE>
__global__ void __launch_bounds__(256) self_collision_kernel(const __grid_constant__ SelfArgs a) {
  CB200_EXTERN_SHARED __align__(16) float fsm[];
  __shared__ unsigned long long red[8];
  constexpr int EPB = 256 / TPE;  // evals per block
  const int sub = threadIdx.x / TPE, t = threadIdx.x % TPE;
  float4 *psph = reinterpret_cast<float4 *>(fsm) + (size_t)sub * a.S;
  const float w = __ldg(a.weight);
  for (int e0 = blockIdx.x * EPB; e0 < a.N; e0 += gridDim.x * EPB) {
    const int e = e0 + sub;
    const bool valid = e < a.N;
    if (valid) {
      for (int s = t; s < a.S; s += TPE) {
        float4 v = __ldg(reinterpret_cast<const float4 *>(a.spheres) + (size_t)e * a.S + s);
        v.w += __ldg(a.padding + s);
        psph[s] = v;
        const size_t gi = (size_t)e * a.S + s;
        if (a.sparse_index[gi] == 1) {  // lazy zeroing of last call's two rows
          *reinterpret_cast<float4 *>(a.out_vec + gi * 4) = make_float4(0, 0, 0, 0);
          a.sparse_index[gi] = 0;
        }
      }
    }
    if (TPE == 32) __syncwarp(); else __syncthreads();
    unsigned long long key = 0ull;  // (float bits << 32) | ~pair index  -> max = largest f, first pair on ties
    if (valid) {
      for (int p = t; p < a.P; p += TPE) {
        const uint32_t pr = __ldg(a.pairs + p);
        const float4 x = psph[pr & 0xffffu], y = psph[pr >> 16];
        const float rs = x.w + y.w;
        const float dx = x.x - y.x, dy = x.y - y.y, dz = x.z - y.z;
        float f = rs * rs - (dx * dx + dy * dy + dz * dz);
        if (!(x.w >= 0.0f && y.w >= 0.0f)) f = 0.0f;
        if (a.store_pair) a.pair_distance[(size_t)e * a.P + p] = f;
        if (f > 0.0f) {
          const unsigned long long kk = ((unsigned long long)__float_as_uint(f) << 32) | (0xffffffffu - (uint32_t)p);
          key = kk > key ? kk : key;
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(kFull, key, o);
      key = other > key ? other : key;
    }
    if (TPE > 32) {
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = key;
      __syncthreads();
      key = red[0];
#pragma unroll
      for (int i = 1; i < 8; ++i) key = red[i] > key ? red[i] : key;
    }
    if (valid && t == 0) {
      if (key == 0ull) {
        a.out_distance[e] = 0.0f;
      } else {
        const float f = __uint_as_float((uint32_t)(key >> 32));
        const uint32_t p = 0xffffffffu - (uint32_t)(key & 0xffffffffu);
        const uint32_t pr = __ldg(a.pairs + p);
        const int i = pr & 0xffffu, j = pr >> 16;
        a.out_distance[e] = 0.5f * w * f;
        if (a.compute_grad) {
          const float4 x = psph[i], y = psph[j];
          float4 g = make_float4(w * (y.x - x.x), w * (y.y - x.y), w * (y.z - x.z), -w);
          *reinterpret_cast<float4 *>(a.out_vec + ((size_t)e * a.S + i) * 4) = g;
          g = make_float4(-g.x, -g.y, -g.z, -w);
          *reinterpret_cast<float4 *>(a.out_vec + ((size_t)e * a.S + j) * 4) = g;
          a.sparse_index[(size_t)e * a.S + i] = 1;
          a.sparse_index[(size_t)e * a.S + j] = 1;
        }
      }
    }
    if (TPE == 32) __syncwarp(); else __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// Drop-in scene collision: thread per (b,h,s); discrete or swept(+speed metric).
// ------------------------------------------------------------------------------------------------
struct SceneArgs {
  float *distance, *gradient;
  const float *spheres, *weight, *eta, *speed_dt;
  CuboidSet cuboids;
  VoxelSet voxels;
  const int32_t *env_query_idx;
  int B, H, S, use_multi_env, sweep, speed_metric;
};

__global__ void __launch_bounds__(128) scene_collision_kernel(const __grid_constant__ SceneArgs a) {
  const long long total = (long long)a.B * a.H * a.S;
  const float w = __ldg(a.weight), eta = __ldg(a.eta);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / ((long long)a.H * a.S));
    const int h = (int)((i - (long long)b * a.H * a.S) / a.S);
    const int env = a.use_multi_env ? __ldg(a.env_query_idx + b) : 0;
    const float4 sp = __ldg(reinterpret_cast<const float4 *>(a.spheres) + i);
    const V3 c = mk3(sp.x, sp.y, sp.z);
    V3 g = mk3(0, 0, 0);
    float cost;
    if (!a.sweep) {
      cost = sphere_scene_discrete(c, sp.w, eta, w, a.cuboids, a.voxels, env, g);
    } else {
      const bool hp = h > 0, hn = h < a.H - 1;
      V3 pv = c, nx = c;
      if (hp) {
        const float4 t = __ldg(reinterpret_cast<const float4 *>(a.spheres) + i - a.S);
        pv = mk3(t.x, t.y, t.z);
      }
      if (hn) {
        const float4 t = __ldg(reinterpret_cast<const float4 *>(a.spheres) + i + a.S);
        nx = mk3(t.x, t.y, t.z);
      }
      cost = sphere_scene_swept(c, sp.w, eta, w, hp, pv, hn, nx, a.cuboids, a.voxels, env, g);
      if (a.speed_metric && hp && hn) speed_metric(pv, c, nx, __ldg(a.speed_dt), cost, g);
    }
    a.distance[i] = cost;
    *reinterpret_cast<float4 *>(a.gradient + 4 * i) = make_float4(g.x, g.y, g.z, 0.0f);
  }
}

// ------------------------------------------------------------------------------------------------
// Mesh obstacles (SURVEY.md 8f rank 4): the same sphere / swept-sphere collision against triangle meshes through the BVH of
// cb200_mesh.cuh.  The reference launches its generic collision kernel once per obstacle TYPE and accumulates with atomics
// (checker_collision.py:76-184); here the mesh type is one more launch that ADDS to the buffers the cuboid / ESDF launch
// wrote (accumulate = 1) or overwrites them when meshes are the only obstacles.  The speed metric is linear in (cost, gradient),
// so applying it per obstacle type and summing equals applying it to the sum.
// ------------------------------------------------------------------------------------------------
struct MeshSceneArgs {
  float *distance, *gradient;
  const float *spheres, *weight, *eta, *speed_dt;
  MeshSet meshes;
  const int32_t *env_query_idx;
  int B, H, S, use_multi_env, sweep, speed_metric, accumulate;
};

__global__ void __launch_bounds__(128) mesh_collision_kernel(const __grid_constant__ MeshSceneArgs a) {
  const long long total = (long long)a.B * a.H * a.S;
  const float w = __ldg(a.weight), eta = __ldg(a.eta);
  const CuboidSet no_cuboids{};
  const VoxelSet no_voxels{};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / ((long long)a.H * a.S));
    const int h = (int)((i - (long long)b * a.H * a.S) / a.S);
    const int env = a.use_multi_env ? __ldg(a.env_query_idx + b) : 0;
    const float4 sp = __ldg(reinterpret_cast<const float4 *>(a.spheres) + i);
    const V3 c = mk3(sp.x, sp.y, sp.z);
    V3 g = mk3(0, 0, 0);
    float cost;
    if (!a.sweep) {
      cost = sphere_scene_discrete<4>(c, sp.w, eta, w, no_cuboids, no_voxels, env, g, &a.meshes);
    } else {
      const bool hp = h > 0, hn = h < a.H - 1;
      V3 pv = c, nx = c;
      if (hp) {
        const float4 t = __ldg(reinterpret_cast<const float4 *>(a.spheres) + i - a.S);
        pv = mk3(t.x, t.y, t.z);
      }
      if (hn) {
        const float4 t = __ldg(reinterpret_cast<const float4 *>(a.spheres) + i + a.S);
        nx = mk3(t.x, t.y, t.z);
      }
      cost = sphere_scene_swept<4>(c, sp.w, eta, w, hp, pv, hn, nx, no_cuboids, no_voxels, env, g, &a.meshes);
      if (a.speed_metric && hp && hn) speed_metric(pv, c, nx, __ldg(a.speed_dt), cost, g);
    }
    float4 *gp = reinterpret_cast<float4 *>(a.gradient + 4 * i);
    if (a.accumulate) {
      const float4 g0 = *gp;
      a.distance[i] += cost;
      *gp = make_float4(g0.x + g.x, g0.y + g.y, g0.z + g.z, 0.0f);
    } else {
      a.distance[i] = cost;
      *gp = make_float4(g.x, g.y, g.z, 0.0f);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Drop-in tool pose cost: thread per (b,h,l)
// ------------------------------------------------------------------------------------------------
struct PoseArgs {
  float *out_distance, *out_pos_dist, *out_rot_dist, *out_pos_grad, *out_rot_grad;
  int32_t *out_goalset_idx;
  const float *cur_pos, *cur_quat, *goal_pos, *goal_quat, *weight, *axes_t, *axes_nt, *tol_t, *tol_nt;
  const int32_t *idxs_goal;
  int B, H, L, G, method;
};

__global__ void __launch_bounds__(128) tool_pose_kernel(const __grid_constant__ PoseArgs a) {
  const int total = a.B * a.H * a.L;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int b = i / (a.H * a.L);
    const int h = (i - b * a.H * a.L) / a.L;
    const int l = i - b * a.H * a.L - h * a.L;
    const bool term = !(h < a.H - 1 && a.H > 1);
    const float *axes = term ? a.axes_t : a.axes_nt;
    const float *tol = (term ? a.tol_t : a.tol_nt) + 2 * l;
    const int gi = __ldg(a.idxs_goal + b);
    const V3 p = mk3(__ldg(a.cur_pos + 3 * i), __ldg(a.cur_pos + 3 * i + 1), __ldg(a.cur_pos + 3 * i + 2));
    const float4 qw = __ldg(reinterpret_cast<const float4 *>(a.cur_quat) + i);
    const size_t go = ((size_t)gi * a.L + l) * a.G;
    const PoseOut po = tool_pose_cost(p, Q4{qw.y, qw.z, qw.w, qw.x}, a.goal_pos + go * 3, a.goal_quat + go * 4, a.G,
                                      __ldg(a.weight), __ldg(a.weight + 1), axes, l, __ldg(tol), __ldg(tol + 1), a.method);
    a.out_distance[2 * i] = po.pos_cost;
    a.out_distance[2 * i + 1] = po.rot_cost;
    a.out_goalset_idx[i] = po.goal_idx;
    a.out_pos_dist[i] = po.pos_err;
    a.out_rot_dist[i] = po.rot_err;
    a.out_pos_grad[3 * i] = po.g_pos.x;
    a.out_pos_grad[3 * i + 1] = po.g_pos.y;
    a.out_pos_grad[3 * i + 2] = po.g_pos.z;
    *reinterpret_cast<float4 *>(a.out_rot_grad + 4 * i) = make_float4(po.gq_w, po.gq_x, po.gq_y, po.gq_z);
  }
}

// ------------------------------------------------------------------------------------------------
// Drop-in c-space kernels: thread per (b,h,d)
// ------------------------------------------------------------------------------------------------
struct CsStateArgs {
  float *out_cost, *gp, *gv, *ga, *gj, *gtau;
  const float *pos, *vel, *acc, *jerk, *effort, *dt, *target, *p_b, *v_b, *a_b, *j_b, *e_b, *weight, *act, *reg, *tw,
      *ntf, *tdw;
  const int32_t *idxs_target;
  int write_grad, B, H, D, retime_w, retime_r;
};

__global__ void __launch_bounds__(128) cspace_state_kernel(const __grid_constant__ CsStateArgs a) {
  const int total = a.B * a.H * a.D;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int b = i / (a.H * a.D);
    const int h = (i - b * a.H * a.D) / a.D;
    const int d = i - b * a.H * a.D - h * a.D;
    const int D = a.D;
    const float dt = __ldg(a.dt + b);
    float tw = __ldg(a.tw);
    if (h < a.H - 1) tw *= __ldg(a.ntf);
    float wb[5], wr[5], act[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      wb[k] = __ldg(a.weight + k);
      wr[k] = __ldg(a.reg + k);
      act[k] = __ldg(a.act + k);
    }
    if (a.retime_w) {
      wb[1] = dt * wb[1];
      wb[2] = powf(dt, 2.0f) * wb[2];
      wb[3] = powf(dt, 3.0f) * wb[3];
    }
    if (a.retime_r) {
      wr[0] = dt * wr[0];
      wr[1] = powf(dt, 2.0f) * wr[1];
      wr[2] = powf(dt, 3.0f) * wr[2];
      wr[4] = dt * wr[4];
    }
    const float p = __ldg(a.pos + i), v = __ldg(a.vel + i), ac = __ldg(a.acc + i), jk = __ldg(a.jerk + i),
                tau = __ldg(a.effort + i);
    float cost = 0.0f, gp = 0.0f, gv = 0.0f, ga = 0.0f, gj = 0.0f, gt = 0.0f;
    bound_cost(p, __ldg(a.p_b + d), __ldg(a.p_b + D + d), act[0], wb[0], cost, gp);
    bound_cost(v, __ldg(a.v_b + d), __ldg(a.v_b + D + d), act[1], wb[1], cost, gv);
    bound_cost(ac, __ldg(a.a_b + d), __ldg(a.a_b + D + d), act[2], wb[2], cost, ga);
    bound_cost(jk, __ldg(a.j_b + d), __ldg(a.j_b + D + d), act[3], wb[3], cost, gj);
    bound_cost(tau, __ldg(a.e_b + d), __ldg(a.e_b + D + d), act[4], wb[4], cost, gt);
    if (tw > 0.0f) {
      tw *= __ldg(a.tdw + d);
      const float err = p - __ldg(a.target + (size_t)__ldg(a.idxs_target + b) * D + d);
      cost += tw * err * err;
      gp += 2.0f * tw * err;
    }
    l2_reg(v, wr[0], cost, gv);
    l2_reg(ac, wr[1], cost, ga);
    l2_reg(jk, wr[2], cost, gj);
    l2_reg(tau, wr[3], cost, gt);
    if (wr[4] > 0.0f) {
      const float ce = tau * v * dt;
      cost += wr[4] * ce * ce;
      gt += 2.0f * wr[4] * ce * v * dt;
      gv += 2.0f * wr[4] * ce * tau * dt;
    }
    a.out_cost[i] = cost;
    if (a.write_grad) {
      a.gp[i] = gp;
      a.gv[i] = gv;
      a.ga[i] = ga;
      a.gj[i] = gj;
      a.gtau[i] = gt;
    }
  }
}

struct CsPosArgs {
  float *out_cost, *gp, *gtau;
  const float *pos, *effort, *target, *p_b, *e_b, *weight, *act, *tw, *tdw, *reg, *cur_p, *cur_v, *v_b, *dt;
  const int32_t *target_idx, *idxs_cur;
  int write_grad, B, H, D;
};

__global__ void __launch_bounds__(128) cspace_position_kernel(const __grid_constant__ CsPosArgs a) {
  const int total = a.B * a.H * a.D;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int b = i / (a.H * a.D);
    const int d = i % a.D;
    const int D = a.D;
    const float eta_p = __ldg(a.act), eta_t = __ldg(a.act + 1), w = __ldg(a.weight), tau_w = __ldg(a.weight + 1);
    float pl = __ldg(a.p_b + d), pu = __ldg(a.p_b + D + d);
    {
      const float r = pu - pl;
      pl = pl + eta_p * r;
      pu = pu - eta_p * r;
    }
    const int cur = __ldg(a.idxs_cur + b);
    const float dt = __ldg(a.dt + cur);
    float cur_p = 0.0f;
    if (dt > 0.0f) {
      cur_p = __ldg(a.cur_p + (size_t)cur * D + d);
      pl = fmaxf(pl, cur_p + __ldg(a.v_b + d) * dt);
      pu = fminf(pu, cur_p + __ldg(a.v_b + D + d) * dt);
    }
    const float p = __ldg(a.pos + i), tau = __ldg(a.effort + i);
    float cost = 0.0f, gp = 0.0f, gt = 0.0f;
    bound_cost(p, pl, pu, 0.0f, w, cost, gp);
    if (tau_w > 0.0f) bound_cost(tau, __ldg(a.e_b + d), __ldg(a.e_b + D + d), eta_t, tau_w, cost, gt);
    const float tw = __ldg(a.tw) * __ldg(a.tdw + d);
    if (tw > 0.0f) {
      const float err = p - __ldg(a.target + (size_t)__ldg(a.target_idx + b) * D + d);
      cost += tw * err * err;
      gp += 2.0f * tw * err;
    }
    const float vw = __ldg(a.reg) * dt, aw = __ldg(a.reg + 1) * dt * dt;
    if (dt > 0.0f && (vw > 0.0f || aw > 0.0f)) {
      const float vi = (p - cur_p) / dt;
      if (vw > 0.0f) {
        cost += 0.5f * vw * vi * vi;
        gp += vw * vi / dt;
      }
      if (aw > 0.0f) {
        const float ai = (vi - __ldg(a.cur_v + (size_t)cur * D + d)) / dt;
        cost += 0.5f * aw * ai * ai;
        gp += aw * ai / (dt * dt);
      }
    }
    a.out_cost[i] = cost;
    if (a.write_grad) {
      a.gp[i] = gp;
      a.gtau[i] = gt;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host helpers
// ------------------------------------------------------------------------------------------------
// Launch plan of a fused rollout kernel: its CTA shape for one robot geometry on one device.  The key holds everything the plan
// depends on and is compared field by field.
struct PlanKey {
  const void *kernel;
  int device;
  size_t fixed_bytes;  // shared memory per CTA besides the rows: the staged robot blob, plus the trajectory kernels' halo
  int unit_floats;     // shared floats per unit of work: a warp's row (or pair of rows), or a team's row
  int horizon;         // trajectory and fused-dynamics kernels: waypoints per seed, which their scores use (0 elsewhere)
  int nl, dof;         // fused-dynamics kernel: links and dofs, which size its dynamics tile (0 elsewhere)
  bool operator==(const PlanKey &o) const {
    return kernel == o.kernel && device == o.device && fixed_bytes == o.fixed_bytes && unit_floats == o.unit_floats &&
           horizon == o.horizon && nl == o.nl && dof == o.dof;
  }
};
struct Plan {
  int nw = 0;       // warps per CTA; 0: no CTA of this kernel fits the geometry
  int per_sm = 0;   // resident CTAs per SM (not queried for team kernels, which run one CTA per SM)
  int R = 0;        // fused-dynamics kernel: rows per dynamics chunk
  size_t smem = 0;  // dynamic shared memory per CTA
};

// Standard, arm, trajectory and big kernels: the warps per CTA (max_nw down to 1) that keep the most warps resident per SM --
// shared memory is the limiter for big robots; ties go to the larger CTA so the blob is staged fewer times.
Plan plan_warps(const PlanKey &k, size_t limit, int max_nw) {
  Plan p;
  double best = 0.0;
  for (int nw = max_nw; nw >= 1; --nw) {
    const size_t need = k.fixed_bytes + (size_t)nw * k.unit_floats * sizeof(float);
    if (need > limit) continue;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k.kernel, nw * 32, need) != cudaSuccess) continue;
    double score = (double)per_sm * nw;
    if (k.horizon > 0) {  // trajectory: rows of the last tile of a trajectory idle, and halo waypoints cost 2 extra FK per tile
      const int tiles = (k.horizon + nw - 1) / nw;
      score *= (double)k.horizon / ((double)tiles * nw + 0.3 * 2.0 * (tiles - 1));
    }
    if (score > best) {
      best = score;
      p = Plan{nw, per_sm, 0, need};
    }
  }
  return p;
}

// Team kernels: the largest multiple of the team size, up to kBigWarps warps, whose teams fit.  No occupancy query: the grid is
// one CTA per SM.
Plan plan_team(const PlanKey &k, size_t limit, int team) {
  for (int w = kBigWarps; w >= team; w -= team) {
    const size_t need = k.fixed_bytes + (size_t)(w / team) * k.unit_floats * sizeof(float);
    if (need <= limit) return Plan{w, 0, 0, need};
  }
  return Plan{};
}

// Fused-dynamics kernel: (warps per CTA, rows per dynamics chunk) that keeps the most warps resident; R is a multiple of the warp
// count so a chunk is a whole number of waypoint tiles.
Plan plan_dyn(const PlanKey &k, size_t limit) {
  Plan p;
  double best = 0.0;
  for (int nw = kWarpsPerCta; nw >= 1; nw >>= 1) {
    for (int R = 32; R >= 8 && R >= nw; R >>= 1) {
      const size_t need = k.fixed_bytes + (size_t)nw * k.unit_floats * sizeof(float) +
                          (size_t)dyn::tile_floats(k.nl, k.dof, R) * sizeof(float);
      if (need > limit) continue;
      int per_sm = 0;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k.kernel, nw * 32, need) != cudaSuccess || per_sm < 1) continue;
      // resident warps, discounted for idle rows of the last tile / chunk of a trajectory and for short dynamics chunks
      // (the recursion's serial depth is paid once per chunk whatever its width)
      const int chunks = (k.horizon + R - 1) / R;
      const double score = (double)per_sm * nw * ((double)k.horizon / ((double)chunks * R)) * (0.75 + 0.25 * R / 32.0);
      if (score > best) {
        best = score;
        p = Plan{nw, per_sm, R, need};
      }
    }
  }
  return p;
}

// This thread's plans, replaced round-robin.
struct PlanEntry {
  PlanKey key;
  Plan plan;
};
constexpr int kPlanSlots = 16;
thread_local PlanEntry g_plans[kPlanSlots];
thread_local int g_plans_used = 0, g_plans_next = 0;

// The plan of key k: cached, or made by make(k, limit).  Before planning, the kernel's dynamic shared-memory cap (a device-wide
// setting) is set to the opt-in limit less the kernel's static shared memory.  That value depends only on (kernel, device), so
// no thread planning another geometry can lower it under a plan this thread cached.
template <typename F>
cudaError_t cached_plan(const PlanKey &k, const DevInfo &d, F make, Plan &out) {
  for (int i = 0; i < g_plans_used; ++i) {
    if (g_plans[i].key == k) {
      out = g_plans[i].plan;
      return cudaSuccess;
    }
  }
  cudaFuncAttributes fa;
  cudaError_t e = cudaFuncGetAttributes(&fa, k.kernel);
  if (e != cudaSuccess) return e;
  const size_t limit = (size_t)d.max_smem - fa.sharedSizeBytes;
  e = cudaFuncSetAttribute(k.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit);
  if (e != cudaSuccess) return e;
  out = make(k, limit);
  g_plans[g_plans_next] = PlanEntry{k, out};
  g_plans_next = (g_plans_next + 1) % kPlanSlots;
  if (g_plans_used < kPlanSlots) ++g_plans_used;
  return cudaSuccess;
}

// A per-call override from the environment (tests switch these inside one process); dflt when unset.
int env_int(const char *name, int dflt) {
  const char *s = getenv(name);
  return s ? atoi(s) : dflt;
}

inline CuboidSet to_dev(const cb200_cuboid_set *c) {
  CuboidSet o{};
  if (c != nullptr && c->inv_pose != nullptr && c->max_n > 0)
    o = CuboidSet{c->dims, c->inv_pose, c->enable, c->count, c->max_n, c->num_envs};
  return o;
}
inline VoxelSet to_dev(const cb200_voxel_set *v) {
  VoxelSet o{};
  if (v != nullptr && v->inv_pose != nullptr && v->max_n > 0)
    o = VoxelSet{v->params, v->inv_pose, v->enable, v->count, v->features, v->n_voxels_per_layer,
                 v->max_n,  v->num_envs, v->max_dist, v->mip, v->mip_stride};
  return o;
}
// No meshes (o empty) when there is no set or it has no poses; a set with poses must give every array the kernels read.
inline cudaError_t to_dev(const cb200_mesh_set *m, MeshSet &o) {
  o = {};
  if (m == nullptr || m->inv_pose == nullptr) return cudaSuccess;
  if (m->nodes == nullptr || m->triangles == nullptr || m->node_offset == nullptr || m->triangle_offset == nullptr ||
      m->dims == nullptr || m->enable == nullptr || m->count == nullptr)
    return cudaErrorInvalidValue;
  o = MeshSet{reinterpret_cast<const float4 *>(m->nodes), reinterpret_cast<const float4 *>(m->triangles), m->node_offset,
              m->triangle_offset, m->dims, m->inv_pose, m->enable, m->count, m->max_n, m->num_envs};
  return cudaSuccess;
}

// The header of the robot blob from its host copy; false unless that copy is a packed blob of exactly `bytes` bytes.
bool read_blob_header(const void *host, int32_t bytes, BlobHeader &h) {
  if (host == nullptr || bytes < (int32_t)sizeof(BlobHeader)) return false;
  memcpy(&h, host, sizeof(BlobHeader));
  return h.magic == kBlobMagic && h.total_bytes == bytes;
}

// Per-environment sphere configurations, when the caller gives more than one: the blob's broad-phase bounds must cover them all.
cudaError_t set_sphere_cfgs(const cb200_rollout_io *io, const BlobHeader &h, FusedArgs &a) {
  if (io->sphere_configs == nullptr || io->num_sphere_configs <= 1) return cudaSuccess;
  if (h.n_sphere_cfgs != io->num_sphere_configs) return cudaErrorInvalidValue;
  a.sphere_cfgs = reinterpret_cast<const float4 *>(io->sphere_configs);
  a.n_sphere_cfgs = io->num_sphere_configs;
  return cudaSuccess;
}

// Lower-bound pyramid level of the ESDF (see voxel_sdf_grad): one thread per block of B^3 base corners (B = kMipBlock);
// the block of base corners [Bc, Bc+B-1] reads fine voxels [Bc, Bc+B] per axis (clipped to the grid).
__global__ void voxel_mip_kernel(VoxelSet vs, uint16_t *mip, int n_layers) {
  const long long per = vs.mip_stride;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < per * n_layers;
       t += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(t / per);
    long long c = t - (long long)k * per;
    const int nx = (int)vs.params[4 * k + 0], ny = (int)vs.params[4 * k + 1], nz = (int)vs.params[4 * k + 2];
    const int mx = (nx + kMipBlock - 1) >> kMipShift, my = (ny + kMipBlock - 1) >> kMipShift, mz = (nz + kMipBlock - 1) >> kMipShift;
    uint16_t outv = 0x7bffu;  // largest finite half: unused tail entries never cull anything wrongly (never read)
    if (c < (long long)mx * my * mz) {
      const int cz = (int)(c % mz), cy = (int)((c / mz) % my), cx = (int)(c / ((long long)mz * my));
      const uint16_t *feat = vs.features + (size_t)k * vs.n_voxels_per_layer;
      float m = 3.0e38f;
      const int B = kMipBlock;
      const int x1 = min(B * cx + B, nx - 1), y1 = min(B * cy + B, ny - 1), z1 = min(B * cz + B, nz - 1);
      for (int x = B * cx; x <= x1; ++x)
        for (int y = B * cy; y <= y1; ++y)
          for (int z = B * cz; z <= z1; ++z) m = fminf(m, load_half(feat + ((size_t)x * ny + y) * nz + z));
      outv = __half_as_ushort(__float2half_rd(m));  // m is itself a half value: exact
    }
    mip[(size_t)k * per + c] = outv;
  }
}

// Robot-sphere refresh (cb200_refresh_robot_spheres): configuration 0 of link_spheres [n_cfg, S, 4] -> the blob's sphere section,
// then warp w rebuilds the two broad-phase bounds of collision link w with the packer's bounding_ball.
struct SphereRefreshArgs {
  unsigned char *blob;
  const float *link_spheres;
  int32_t S, n_cfg, n_cl;
  int32_t off_spheres, off_padding, off_cl_start, off_cl_bound, off_cl_bound_scene;
};

// bounding_ball's farthest-ball scan over a warp: the largest distance, the lowest slot among equals (the serial scan's pick)
struct WarpFarthest {
  __device__ void operator()(double &best, int &arg) const {
    for (int o = 16; o > 0; o >>= 1) {
      const double b = __shfl_xor_sync(0xffffffffu, best, o);
      const int j = __shfl_xor_sync(0xffffffffu, arg, o);
      if (b > best || (b == best && j < arg)) {
        best = b;
        arg = j;
      }
    }
  }
};

__global__ void __launch_bounds__(128) refresh_robot_spheres_kernel(const SphereRefreshArgs a) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthreads = gridDim.x * blockDim.x;
  float *spheres = reinterpret_cast<float *>(a.blob + a.off_spheres);
  for (int i = tid; i < 4 * a.S; i += nthreads) spheres[i] = a.link_spheres[i];
  const int cl = tid >> 5, lane = threadIdx.x & 31;
  if (cl >= a.n_cl) return;  // whole warps
  const int16_t *cl_start = reinterpret_cast<const int16_t *>(a.blob + a.off_cl_start);
  const float *padding = reinterpret_cast<const float *>(a.blob + a.off_padding);
  const int s0 = cl_start[cl], s1 = cl_start[cl + 1];
  bounding_ball(a.link_spheres, padding, s0, s1, a.n_cfg, a.S, reinterpret_cast<float *>(a.blob + a.off_cl_bound) + 4 * cl, lane,
                32, WarpFarthest{});
  bounding_ball(a.link_spheres, (const float *)nullptr, s0, s1, a.n_cfg, a.S,
                reinterpret_cast<float *>(a.blob + a.off_cl_bound_scene) + 4 * cl, lane, 32, WarpFarthest{});
}

}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
// which kernel the last cb200_rollout_cost_grad / cb200_rollout_cost call of this thread launched (CB200_VARIANT_*; test / bench introspection)
static thread_local int g_last_variant = 0;

extern "C" {

int cb200_abi_version(void) { return CB200_ABI_VERSION; }
int cb200_last_rollout_variant(void) { return g_last_variant; }
int cb200_sm_arch(void) { return 90; }
const char *cb200_error_string(int err) { return cudaGetErrorString((cudaError_t)err); }

int cb200_device_info(int device, int *sm_count, int *max_smem_optin) {
  cudaError_t e = cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, device);
  if (e != cudaSuccess) return ret(e);
  return ret(cudaDeviceGetAttribute(max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
}

int cb200_kinematics_forward_spheres(float *link_pos, float *link_quat, float *batch_robot_spheres,
                                     float *batch_center_of_mass, float *global_cumul_mat, const float *joint_vec,
                                     const float *fixed_transform, const float *robot_spheres,
                                     const float *link_masses_com, const int8_t *joint_map_type,
                                     const int16_t *joint_map, const int16_t *link_map, const int16_t *tool_frame_map,
                                     const int16_t *link_sphere_map, const float *joint_offset_map,
                                     const int32_t *env_query_idx, int num_envs, int batch_size, int horizon,
                                     int n_joints, int num_spheres, int num_links, int n_tool_frames,
                                     int write_global_cumul, int compute_com, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(joint_vec);
  if (batch_size < 0 || num_links < 1 || horizon < 1) return ret(cudaErrorInvalidValue);
  if (compute_com != 0 && (batch_center_of_mass == nullptr || link_masses_com == nullptr)) return ret(cudaErrorInvalidValue);
  if (batch_size == 0) return ret(cudaSuccess);
  KinFwdArgs a{link_pos, link_quat, batch_robot_spheres, global_cumul_mat, joint_vec, fixed_transform, robot_spheres,
               joint_offset_map, joint_map_type, joint_map, link_map, tool_frame_map, link_sphere_map, env_query_idx,
               num_envs, batch_size, horizon, n_joints, num_spheres, num_links, n_tool_frames, write_global_cumul,
               link_masses_com, batch_center_of_mass};
  const size_t smem = (size_t)kWarpsPerCta * num_links * 12 * sizeof(float);
  void (*kern)(const KinFwdArgs) = compute_com != 0 ? kin_forward_kernel<true> : kin_forward_kernel<false>;
  if (const cudaError_t e = opt_in_smem(kern, smem); e != cudaSuccess) return e;
  const int grid = persistent_grid(kern, kWarpsPerCta * 32, smem, (batch_size + kWarpsPerCta - 1) / kWarpsPerCta);
  CB200_LAUNCH(kern, grid, kWarpsPerCta * 32, smem, (cudaStream_t)stream, a);
  return launch_status();
}

int cb200_kinematics_backward(float *grad_out, const float *grad_nlinks_pos, const float *grad_nlinks_quat,
                              const float *grad_spheres, const float *grad_center_of_mass,
                              const float *batch_center_of_mass, const float *grad_jacobian,
                              const float *global_cumul_mat, const float *robot_spheres, const float *link_masses_com,
                              const int16_t *link_map, const int16_t *joint_map, const int8_t *joint_map_type,
                              const int16_t *tool_frame_map, const int16_t *link_sphere_map,
                              const int16_t *link_chain_data, const int16_t *link_chain_offsets,
                              const int16_t *joint_links_data, const int16_t *joint_links_offsets,
                              const uint8_t *joint_affects_endeffector, const float *joint_offset_map,
                              const int32_t *env_query_idx, int num_envs, int batch_size, int horizon, int n_joints,
                              int num_spheres, int num_links, int n_tool_frames, int compute_com,
                              int compute_jacobian_grad, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(grad_out);
  (void)grad_jacobian;
  (void)link_chain_data;
  (void)link_chain_offsets;
  (void)joint_links_data;
  (void)joint_links_offsets;
  (void)joint_affects_endeffector;
  if (compute_jacobian_grad != 0 || num_links < 1 || num_links > kMaxLinks || horizon < 1) return ret(cudaErrorInvalidValue);
  if (compute_com != 0 && (grad_center_of_mass == nullptr || batch_center_of_mass == nullptr || link_masses_com == nullptr))
    return ret(cudaErrorInvalidValue);
  if (batch_size == 0) return ret(cudaSuccess);
  KinBwdArgs a{grad_out, grad_nlinks_pos, grad_nlinks_quat, num_spheres > 0 ? grad_spheres : nullptr, global_cumul_mat,
               robot_spheres, joint_offset_map, link_map, joint_map, tool_frame_map, link_sphere_map, joint_map_type,
               env_query_idx, num_envs, batch_size, horizon, n_joints, num_spheres, num_links, n_tool_frames,
               grad_center_of_mass, batch_center_of_mass, link_masses_com};
  void (*kern)(const KinBwdArgs) = compute_com != 0 ? kin_backward_kernel<true> : kin_backward_kernel<false>;
  const size_t per_warp = ((size_t)num_links * 12 + num_links * 8 + num_links + n_joints + 3) & ~(size_t)3;
  const size_t smem = ((((size_t)2 * num_links + 3) & ~(size_t)3) + kWarpsPerCta * per_warp) * sizeof(float);
  if (const cudaError_t e = opt_in_smem(kern, smem); e != cudaSuccess) return e;
  const int grid = persistent_grid(kern, kWarpsPerCta * 32, smem, (batch_size + kWarpsPerCta - 1) / kWarpsPerCta);
  CB200_LAUNCH(kern, grid, kWarpsPerCta * 32, smem, (cudaStream_t)stream, a);
  return launch_status();
}

int cb200_self_collision_distance(float *out_distance, float *out_vec, float *pair_distance, uint8_t *sparse_index,
                                  const float *robot_spheres, const float *sphere_padding, const float *weight,
                                  const int16_t *pair_locations, float *block_batch_max_value,
                                  int16_t *block_batch_max_index, int num_blocks_per_batch, int max_threads_per_block,
                                  int batch_size, int horizon, int nspheres, int num_collision_pairs,
                                  int store_pair_distance, int compute_grad, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(out_distance);
  (void)block_batch_max_value;
  (void)block_batch_max_index;
  (void)num_blocks_per_batch;
  (void)max_threads_per_block;
  const int N = batch_size * horizon;
  if (N == 0) return ret(cudaSuccess);
  if (N < 0 || nspheres < 1 || nspheres > 65535) return ret(cudaErrorInvalidValue);
  SelfArgs a{out_distance, out_vec, pair_distance, sparse_index, robot_spheres, sphere_padding, weight,
             reinterpret_cast<const uint32_t *>(pair_locations), N, nspheres, num_collision_pairs, store_pair_distance,
             compute_grad};
  if (num_collision_pairs <= 4096) {
    const size_t smem = (size_t)8 * nspheres * 16;
    if (const cudaError_t e = opt_in_smem(self_collision_kernel<32>, smem); e != cudaSuccess) return e;
    const int grid = persistent_grid(self_collision_kernel<32>, 256, smem, (N + 7) / 8);
    CB200_LAUNCH(self_collision_kernel<32>, grid, 256, smem, (cudaStream_t)stream, a);
  } else {
    const size_t smem = (size_t)nspheres * 16;
    const int grid = persistent_grid(self_collision_kernel<256>, 256, smem, N);
    CB200_LAUNCH(self_collision_kernel<256>, grid, 256, smem, (cudaStream_t)stream, a);
  }
  return launch_status();
}

static int scene_launch(float *distance, float *gradient, const float *spheres, const cb200_cuboid_set *cuboids,
                        const cb200_voxel_set *voxels, const float *weight, const float *eta, const float *speed_dt,
                        int speed_metric, const int32_t *env_query_idx, int B, int H, int S, int use_multi_env, int sweep,
                        cb200_stream_t stream) {
  CB200_DEVICE_GUARD(distance);
  const long long total = (long long)B * H * S;
  if (total == 0) return ret(cudaSuccess);
  if (total < 0 || (speed_metric && speed_dt == nullptr)) return ret(cudaErrorInvalidValue);
  SceneArgs a{distance, gradient, spheres, weight, eta, speed_dt, to_dev(cuboids), to_dev(voxels), env_query_idx,
              B, H, S, use_multi_env && env_query_idx != nullptr, sweep, speed_metric};
  const int grid = persistent_grid(scene_collision_kernel, 128, 0, (total + 127) / 128);
  CB200_LAUNCH(scene_collision_kernel, grid, 128, 0, (cudaStream_t)stream, a);
  return launch_status();
}

int cb200_sphere_obstacle_collision(float *distance, float *gradient, const float *spheres,
                                    const cb200_cuboid_set *cuboids, const cb200_voxel_set *voxels, const float *weight,
                                    const float *activation_distance, const int32_t *env_query_idx, int batch_size,
                                    int horizon, int num_spheres, int use_multi_env, cb200_stream_t stream) {
  return scene_launch(distance, gradient, spheres, cuboids, voxels, weight, activation_distance, nullptr, 0,
                      env_query_idx, batch_size, horizon, num_spheres, use_multi_env, 0, stream);
}

int cb200_swept_sphere_obstacle_collision(float *distance, float *gradient, const float *spheres,
                                          const cb200_cuboid_set *cuboids, const cb200_voxel_set *voxels,
                                          const float *weight, const float *activation_distance, const float *speed_dt,
                                          int enable_speed_metric, const int32_t *env_query_idx, int batch_size,
                                          int horizon, int num_spheres, int use_multi_env, cb200_stream_t stream) {
  return scene_launch(distance, gradient, spheres, cuboids, voxels, weight, activation_distance, speed_dt,
                      enable_speed_metric, env_query_idx, batch_size, horizon, num_spheres, use_multi_env, 1, stream);
}

int cb200_sphere_mesh_collision(float *distance, float *gradient, const float *spheres, const cb200_mesh_set *meshes,
                                const float *weight, const float *activation_distance, const float *speed_dt,
                                int enable_speed_metric, const int32_t *env_query_idx, int batch_size, int horizon,
                                int num_spheres, int use_multi_env, int sweep, int accumulate, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(distance);
  const long long total = (long long)batch_size * horizon * num_spheres;
  if (total == 0) return ret(cudaSuccess);
  MeshSet ms;
  if (total < 0 || meshes == nullptr || to_dev(meshes, ms) != cudaSuccess || (enable_speed_metric && speed_dt == nullptr))
    return ret(cudaErrorInvalidValue);
  MeshSceneArgs a{distance, gradient, spheres, weight, activation_distance, speed_dt, ms, env_query_idx, batch_size, horizon,
                  num_spheres, use_multi_env && env_query_idx != nullptr, sweep, enable_speed_metric, accumulate};
  const int grid = persistent_grid(mesh_collision_kernel, 128, 0, (total + 127) / 128);
  CB200_LAUNCH(mesh_collision_kernel, grid, 128, 0, (cudaStream_t)stream, a);
  return launch_status();
}

int cb200_tool_pose_distance(float *out_distance, float *out_position_distance, float *out_rotation_distance,
                             float *out_position_gradient, float *out_rotation_gradient, int32_t *out_goalset_idx,
                             const float *current_position, const float *current_quat, const float *goal_position,
                             const float *goal_quat, const int32_t *idxs_goal, const float *position_orientation_weight,
                             const float *terminal_pose_axes_weight_factor,
                             const float *non_terminal_pose_axes_weight_factor,
                             const float *terminal_pose_convergence_tolerance,
                             const float *non_terminal_pose_convergence_tolerance, int batch_size, int horizon,
                             int num_links, int num_goalset, int rotation_method, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(out_distance);
  const int total = batch_size * horizon * num_links;
  if (total == 0) return ret(cudaSuccess);
  if (total < 0 || num_goalset < 1 || rotation_method < 0 || rotation_method > 1) return ret(cudaErrorInvalidValue);
  PoseArgs a{out_distance, out_position_distance, out_rotation_distance, out_position_gradient, out_rotation_gradient,
             out_goalset_idx, current_position, current_quat, goal_position, goal_quat, position_orientation_weight,
             terminal_pose_axes_weight_factor, non_terminal_pose_axes_weight_factor,
             terminal_pose_convergence_tolerance, non_terminal_pose_convergence_tolerance, idxs_goal, batch_size,
             horizon, num_links, num_goalset, rotation_method};
  const int grid = persistent_grid(tool_pose_kernel, 128, 0, (total + 127) / 128);
  CB200_LAUNCH(tool_pose_kernel, grid, 128, 0, (cudaStream_t)stream, a);
  return launch_status();
}

int cb200_cspace_state_cost(float *out_cost, float *out_grad_p, float *out_grad_v, float *out_grad_a, float *out_grad_j,
                            float *out_grad_tau, const float *pos, const float *vel, const float *acc,
                            const float *jerk, const float *effort, const float *state_dt,
                            const float *target_joint_position, const int32_t *idxs_target_joint_position,
                            const float *p_b, const float *v_b, const float *a_b, const float *j_b,
                            const float *effort_b, const float *weight, const float *activation_distance,
                            const float *squared_l2_regularization_weights, const float *cspace_target_weight,
                            const float *cspace_non_terminal_weight_factor, const float *cspace_target_dof_weight,
                            int write_grad, int batch_size, int horizon, int dof, int retime_weights,
                            int retime_regularization_weights, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(out_cost);
  const int total = batch_size * horizon * dof;
  if (total == 0) return ret(cudaSuccess);
  if (total < 0) return ret(cudaErrorInvalidValue);
  CsStateArgs a{out_cost, out_grad_p, out_grad_v, out_grad_a, out_grad_j, out_grad_tau, pos, vel, acc, jerk, effort,
                state_dt, target_joint_position, p_b, v_b, a_b, j_b, effort_b, weight, activation_distance,
                squared_l2_regularization_weights, cspace_target_weight, cspace_non_terminal_weight_factor,
                cspace_target_dof_weight, idxs_target_joint_position, write_grad, batch_size, horizon, dof,
                retime_weights, retime_regularization_weights};
  const int grid = persistent_grid(cspace_state_kernel, 128, 0, (total + 127) / 128);
  CB200_LAUNCH(cspace_state_kernel, grid, 128, 0, (cudaStream_t)stream, a);
  return launch_status();
}

int cb200_cspace_position_cost(float *out_cost, float *out_grad_p, float *out_grad_tau, const float *pos,
                               const float *effort, const float *cspace_target, const int32_t *cspace_target_idx,
                               const float *p_b, const float *effort_b, const float *weight,
                               const float *activation_distance, const float *cspace_target_weight,
                               const float *cspace_target_dof_weight, const float *squared_l2_reg_weight,
                               const float *current_position, const float *current_velocity,
                               const int32_t *idxs_current_state, const float *v_b, const float *state_dt,
                               int write_grad, int batch_size, int horizon, int dof, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(out_cost);
  const int total = batch_size * horizon * dof;
  if (total == 0) return ret(cudaSuccess);
  if (total < 0) return ret(cudaErrorInvalidValue);
  CsPosArgs a{out_cost, out_grad_p, out_grad_tau, pos, effort, cspace_target, p_b, effort_b, weight,
              activation_distance, cspace_target_weight, cspace_target_dof_weight, squared_l2_reg_weight,
              current_position, current_velocity, v_b, state_dt, cspace_target_idx, idxs_current_state, write_grad,
              batch_size, horizon, dof};
  const int grid = persistent_grid(cspace_position_kernel, 128, 0, (total + 127) / 128);
  CB200_LAUNCH(cspace_position_kernel, grid, 128, 0, (cudaStream_t)stream, a);
  return launch_status();
}

// ---- robot blob -------------------------------------------------------------------------------
static int64_t blob_layout(const cb200_robot_sizes *sz, const int16_t *link_map, BlobHeader *h, int n_lp_cap) {
  const int nl = sz->num_links, D = sz->num_dof, S = sz->num_spheres, L = sz->num_tool_frames, P = sz->num_pairs;
  if (nl < 1 || nl > kMaxLinks || D < 0 || S < 0 || L < 0 || P < 0) return -1;
  int n_levels = 1;
  if (link_map != nullptr) {
    std::vector<int> depth(nl, 0);
    for (int l = 1; l < nl; ++l) {
      if (link_map[l] < 0 || link_map[l] >= l) return -2;
      depth[l] = depth[link_map[l]] + 1;
      n_levels = std::max(n_levels, depth[l] + 1);
    }
  } else {
    n_levels = nl;  // upper bound for sizing
  }
  int64_t off = sizeof(BlobHeader);
  auto take = [&](int64_t bytes) {
    int64_t o = off;
    off = (off + bytes + 15) & ~(int64_t)15;
    return (int32_t)o;
  };
  memset(h, 0, sizeof(*h));
  h->magic = kBlobMagic;
  h->nl = nl;
  h->D = D;
  h->S = S;
  h->L = L;
  h->P = P;
  h->n_levels = n_levels;
  h->off_fixed = take((int64_t)nl * 48);
  h->off_joff = take((int64_t)nl * 8);
  h->off_link_map = take((int64_t)nl * 2);
  h->off_joint_map = take((int64_t)nl * 2);
  h->off_joint_type = take(nl);
  h->off_tool_map = take((int64_t)L * 2);
  h->off_spheres = take((int64_t)S * 16);
  h->off_sph_link = take((int64_t)S * 2);
  h->off_padding = take((int64_t)S * 4);
  h->off_link_sph_off = take((int64_t)(nl + 1) * 2);
  h->off_link_sph_idx = take((int64_t)S * 2);
  h->off_level_off = take((int64_t)(nl + 1) * 2);  // sized for the worst case (n_levels <= nl)
  h->off_level_links = take((int64_t)nl * 2);
  h->off_anc_mask = take((int64_t)nl * 8);
  h->off_jl_off = take((int64_t)(D + 1) * 2);
  h->off_jl_idx = take((int64_t)nl * 2);
  h->off_limits = take((int64_t)10 * D * 4);
  // broad-phase tables, sized for the worst case (every link a collision link, every link pair checked)
  const int max_cl = std::min(nl, S);
  h->off_cl_link = take((int64_t)max_cl * 2);
  h->off_cl_start = take((int64_t)(max_cl + 1) * 2);
  h->off_cl_bound = take((int64_t)max_cl * 16);
  h->off_lp = take((int64_t)n_lp_cap * 4);
  h->off_fk_sched = take((int64_t)nl * 8);
  h->off_cl_bound_scene = take((int64_t)max_cl * 16);
  h->off_sph_cl = take((int64_t)S);
  h->smem_bytes = (int32_t)off;
  h->off_pairs = take((int64_t)P * 4);
  h->total_bytes = (int32_t)off;
  return off;
}

static int lp_cap(const cb200_robot_sizes *sz) {
  const int m = std::min(sz->num_links, sz->num_spheres);
  return std::min(m * (m - 1) / 2, std::max(sz->num_pairs, 0));
}

int cb200_voxel_mip_block(void) { return kMipBlock; }

int64_t cb200_voxel_mip_stride(const float *host_params, int num_layers) {
  if (host_params == nullptr || num_layers < 1) return -1;
  int64_t best = 1;
  for (int k = 0; k < num_layers; ++k) {
    const int64_t nx = (int64_t)host_params[4 * k], ny = (int64_t)host_params[4 * k + 1], nz = (int64_t)host_params[4 * k + 2];
    best = std::max(best, ((nx + kMipBlock - 1) >> kMipShift) * ((ny + kMipBlock - 1) >> kMipShift) * ((nz + kMipBlock - 1) >> kMipShift));
  }
  return best;
}

int cb200_voxel_build_mip(const cb200_voxel_set *vs, cb200_stream_t stream) {
  CB200_DEVICE_GUARD((vs != nullptr ? vs->mip : nullptr));
  if (vs == nullptr || vs->mip == nullptr || vs->mip_stride < 1 || vs->features == nullptr || vs->params == nullptr ||
      vs->max_n < 1 || vs->num_envs < 1)
    return ret(cudaErrorInvalidValue);
  const int n_layers = vs->max_n * vs->num_envs;
  const long long n = (long long)vs->mip_stride * n_layers;
  // grid-stride loop: one wave of resident CTAs on this device, fewer for small pyramids
  const int grid = persistent_grid(voxel_mip_kernel, 128, 0, (n + 127) / 128);
  CB200_LAUNCH(voxel_mip_kernel, grid, 128, 0, (cudaStream_t)stream, to_dev(vs), const_cast<uint16_t *>(vs->mip), n_layers);
  return launch_status();
}

int64_t cb200_robot_blob_bytes(const cb200_robot_sizes *sz) {
  BlobHeader h;
  return blob_layout(sz, nullptr, &h, lp_cap(sz));
}

int64_t cb200_pack_robot_blob(void *out, int64_t out_bytes, const cb200_robot_sizes *sz, const float *fixed_transforms,
                              const int16_t *link_map, const int16_t *joint_map, const int8_t *joint_map_type,
                              const float *joint_offset_map, const int16_t *tool_frame_map, const float *link_spheres,
                              const int16_t *link_sphere_map, const float *sphere_padding,
                              const int16_t *collision_pairs, const float *position_limits,
                              const float *velocity_limits, const float *acceleration_limits, const float *jerk_limits,
                              const float *effort_limits) {
  BlobHeader h;
  const int64_t total = blob_layout(sz, link_map, &h, lp_cap(sz));
  if (total < 0) return total;
  if (out_bytes < total) return -3;
  const int nl = h.nl, D = h.D, S = h.S, L = h.L, P = h.P;
  const int n_cfg = sz->num_sphere_configs > 1 ? sz->num_sphere_configs : 1;  // link_spheres is [n_cfg, S, 4]
  h.n_sphere_cfgs = n_cfg;
  unsigned char *o = static_cast<unsigned char *>(out);
  memset(o, 0, (size_t)total);
  memcpy(o, &h, sizeof(h));
  memcpy(o + h.off_fixed, fixed_transforms, (size_t)nl * 48);
  memcpy(o + h.off_joff, joint_offset_map, (size_t)nl * 8);
  memcpy(o + h.off_link_map, link_map, (size_t)nl * 2);
  memcpy(o + h.off_joint_map, joint_map, (size_t)nl * 2);
  memcpy(o + h.off_joint_type, joint_map_type, (size_t)nl);
  if (L) memcpy(o + h.off_tool_map, tool_frame_map, (size_t)L * 2);
  for (int l = 0; l < nl; ++l) {
    const int jt = joint_map_type[l];
    if (jt < -1 || jt > 5) return -4;
    if (jt >= 0 && (joint_map[l] < 0 || joint_map[l] >= D)) return -5;
  }
  for (int t = 0; t < L; ++t)
    if (tool_frame_map[t] < 0 || tool_frame_map[t] >= nl) return -6;
  if (S) {
    memcpy(o + h.off_spheres, link_spheres, (size_t)S * 16);
    memcpy(o + h.off_sph_link, link_sphere_map, (size_t)S * 2);
    memcpy(o + h.off_padding, sphere_padding, (size_t)S * 4);
  }
  // CSR link -> spheres
  int16_t *lso = reinterpret_cast<int16_t *>(o + h.off_link_sph_off);
  int16_t *lsi = reinterpret_cast<int16_t *>(o + h.off_link_sph_idx);
  int n = 0;
  for (int l = 0; l < nl; ++l) {
    lso[l] = (int16_t)n;
    for (int s = 0; s < S; ++s) {
      if (link_sphere_map[s] < 0 || link_sphere_map[s] >= nl) return -7;
      if (link_sphere_map[s] == l) lsi[n++] = (int16_t)s;
    }
  }
  lso[nl] = (int16_t)n;
  // depth levels + ancestor masks
  std::vector<int> depth(nl, 0);
  unsigned long long *anc = reinterpret_cast<unsigned long long *>(o + h.off_anc_mask);
  anc[0] = 1ull;
  for (int l = 1; l < nl; ++l) {
    depth[l] = depth[link_map[l]] + 1;
    anc[l] = anc[link_map[l]] | (1ull << l);
  }
  int16_t *lvo = reinterpret_cast<int16_t *>(o + h.off_level_off);
  int16_t *lvl = reinterpret_cast<int16_t *>(o + h.off_level_links);
  n = 0;
  for (int lev = 0; lev < h.n_levels; ++lev) {
    lvo[lev] = (int16_t)n;
    for (int l = 0; l < nl; ++l)
      if (depth[l] == lev) lvl[n++] = (int16_t)l;
  }
  lvo[h.n_levels] = (int16_t)n;
  {  // FK compose schedule: two independent links (same depth level) per step
    uint32_t *sched = reinterpret_cast<uint32_t *>(o + h.off_fk_sched);
    int steps = 0;
    for (int lev = 1; lev < h.n_levels; ++lev) {
      for (int i = lvo[lev]; i < lvo[lev + 1]; i += 2) {
        const uint32_t l0 = (uint32_t)lvl[i], p0 = (uint32_t)link_map[l0];
        sched[2 * steps] = (l0 * 48u) | ((p0 * 48u) << 16);
        sched[2 * steps + 1] = 0xffffu;
        if (i + 1 < lvo[lev + 1]) {
          const uint32_t l1 = (uint32_t)lvl[i + 1], p1 = (uint32_t)link_map[l1];
          sched[2 * steps + 1] = (l1 * 48u) | ((p1 * 48u) << 16);
        }
        ++steps;
      }
    }
    reinterpret_cast<BlobHeader *>(o)->n_fk_steps = steps;
  }
  // CSR joint -> links
  int16_t *jlo = reinterpret_cast<int16_t *>(o + h.off_jl_off);
  int16_t *jli = reinterpret_cast<int16_t *>(o + h.off_jl_idx);
  n = 0;
  for (int d = 0; d < D; ++d) {
    jlo[d] = (int16_t)n;
    for (int l = 0; l < nl; ++l)
      if (joint_map_type[l] >= 0 && joint_map[l] == d) jli[n++] = (int16_t)l;
  }
  jlo[D] = (int16_t)n;
  float *lim = reinterpret_cast<float *>(o + h.off_limits);
  const float *srcs[5] = {position_limits, velocity_limits, acceleration_limits, jerk_limits, effort_limits};
  for (int k = 0; k < 5; ++k)
    for (int i = 0; i < 2 * D; ++i) lim[k * 2 * D + i] = srcs[k] ? srcs[k][i] : (i < D ? -1e30f : 1e30f);
  for (int p = 0; p < P; ++p) {
    const int i = collision_pairs[2 * p], j = collision_pairs[2 * p + 1];
    if (i < 0 || j < 0 || i >= S || j >= S) return -8;
  }
  if (P) memcpy(o + h.off_pairs, collision_pairs, (size_t)P * 4);
  // ---- self-collision broad phase: collision links = maximal runs of consecutive spheres on one link
  {
    std::vector<int> cl_link, cl_start, cl_of_sphere(S, 0);
    bool ok = S > 0 && P > 0;
    for (int s0 = 0; s0 < S; ++s0) {
      if (s0 == 0 || link_sphere_map[s0] != link_sphere_map[s0 - 1]) {
        for (int l : cl_link) ok = ok && (l != link_sphere_map[s0]);  // a link's spheres must be contiguous
        cl_link.push_back(link_sphere_map[s0]);
        cl_start.push_back(s0);
      }
      cl_of_sphere[s0] = (int)cl_link.size() - 1;
    }
    cl_start.push_back(S);
    const int n_cl = (int)cl_link.size();
    std::vector<unsigned char> checked((size_t)n_cl * n_cl, 0);
    std::vector<uint32_t> lps;
    long long covered = 0;
    if (ok) {
      for (int p = 0; p < P && ok; ++p) {
        const int i = collision_pairs[2 * p], j = collision_pairs[2 * p + 1];
        const int a = cl_of_sphere[i], b = cl_of_sphere[j];
        ok = (i < j) && (a < b);
        if (ok && !checked[(size_t)a * n_cl + b]) {
          checked[(size_t)a * n_cl + b] = 1;
          lps.push_back((uint32_t)a | ((uint32_t)b << 16));
          covered += (long long)(cl_start[a + 1] - cl_start[a]) * (cl_start[b + 1] - cl_start[b]);
        }
      }
      ok = ok && covered == P && (int)lps.size() <= lp_cap(sz);  // list == union of full link x link blocks
    }
    if (ok) {
      std::sort(lps.begin(), lps.end(), [](uint32_t x, uint32_t y) {
        return ((x & 0xffffu) != (y & 0xffffu)) ? (x & 0xffffu) < (y & 0xffffu) : (x >> 16) < (y >> 16);
      });
      BlobHeader *hh = reinterpret_cast<BlobHeader *>(o);
      hh->n_cl = n_cl;
      hh->n_lp = (int32_t)lps.size();
      int16_t *cll = reinterpret_cast<int16_t *>(o + h.off_cl_link);
      int16_t *cls = reinterpret_cast<int16_t *>(o + h.off_cl_start);
      float *clb = reinterpret_cast<float *>(o + h.off_cl_bound);
      for (int a = 0; a < n_cl; ++a) {
        cll[a] = (int16_t)cl_link[a];
        cls[a] = (int16_t)cl_start[a];
        // bounding spheres of the enabled sphere balls: padded radii for self collision, raw radii for the scene
        bounding_ball(link_spheres, sphere_padding, cl_start[a], cl_start[a + 1], n_cfg, S, clb + 4 * a);
        bounding_ball(link_spheres, nullptr, cl_start[a], cl_start[a + 1], n_cfg, S,
                      reinterpret_cast<float *>(o + h.off_cl_bound_scene) + 4 * a);
      }
      cls[n_cl] = (int16_t)S;
      memcpy(o + h.off_lp, lps.data(), lps.size() * 4);
      for (int s0 = 0; s0 < S; ++s0) o[h.off_sph_cl + s0] = (unsigned char)cl_of_sphere[s0];
    }
  }
  return total;
}

int cb200_refresh_robot_spheres(void *robot_blob, const void *robot_blob_host, int32_t robot_blob_bytes, const float *link_spheres,
                                int32_t num_sphere_configs, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(robot_blob);
  BlobHeader h;
  if (robot_blob == nullptr || link_spheres == nullptr || !read_blob_header(robot_blob_host, robot_blob_bytes, h) ||
      num_sphere_configs != h.n_sphere_cfgs)
    return ret(cudaErrorInvalidValue);
  if (h.S == 0) return ret(cudaSuccess);
  const SphereRefreshArgs a{static_cast<unsigned char *>(robot_blob), link_spheres, h.S, h.n_sphere_cfgs, h.n_cl, h.off_spheres,
                            h.off_padding, h.off_cl_start, h.off_cl_bound, h.off_cl_bound_scene};
  const int grid = std::max(1, (h.n_cl * 32 + 127) / 128);  // a warp per collision link (none when n_lp == 0: n_cl == 0)
  CB200_LAUNCH(refresh_robot_spheres_kernel, grid, 128, 0, (cudaStream_t)stream, a);
  return launch_status();
}

}  // extern "C"

// One call of the fused rollout launcher as the kernel selection, the kernel table and the launch see it (prepare_rollout).
struct RolloutShape {
  BlobHeader h;
  long long N;                         // rows: batch x H
  int H, scene;                        // waypoints per trajectory; obstacle types present: bit 0 cuboids, bit 1 voxel grids
  bool mesh, traj, spline, arm_sized;  // meshes present; trajectory mode; rows from knots in the kernel; arm builds apply
  bool dynamics, dynamics_ok;          // inverse dynamics asked for (io->dynamics); with what the kernel needs (a.dyn set)
  int grad_floats, cost_floats;        // shared floats of a row: gradient kernels' standard layout, cost-only kernels
};

// Rollout kernel families, in the order of their CB200_VARIANT_*; arm rows and arm pairs both report the arm build.
enum class Family { Standard, ArmRows, ArmPairs, Big, Team2, Team4, Traj, TrajDyn };
constexpr int kFamilyVariant[] = {CB200_VARIANT_STANDARD, CB200_VARIANT_ARM,   CB200_VARIANT_ARM,  CB200_VARIANT_BIG,
                                  CB200_VARIANT_TEAM2,    CB200_VARIANT_TEAM4, CB200_VARIANT_TRAJ, CB200_VARIANT_TRAJ_DYN};

// k(std::integral_constant<int, SCENE>) for SCENE = scene: 0..3, or 7 where the family has a mesh build (MESH); else nullptr.
template <bool MESH, typename K>
static const void *by_scene(int scene, K k) {
  using std::integral_constant;
  if constexpr (MESH) if (scene == 7) return (const void *)k(integral_constant<int, 7>{});
  const void *const builds[4] = {(const void *)k(integral_constant<int, 0>{}), (const void *)k(integral_constant<int, 1>{}),
                                 (const void *)k(integral_constant<int, 2>{}), (const void *)k(integral_constant<int, 3>{})};
  return scene >= 0 && scene < 4 ? builds[scene] : nullptr;
}

// The kernel of family f for this call, and the one place that names a rollout kernel instantiation.  Kernels are specialised on
// the obstacle types present so that e.g. the IK kernel carries no ESDF code: the fused kernel's instruction footprint is what
// limits it.  Mesh scenes take one build per family, SCENE = 7, which checks at run time whether cuboids and ESDF grids are
// present; the team, arm, fused-dynamics and in-kernel spline builds have none.  nullptr: no such build.
static const void *rollout_kernel(Family f, bool grad, const RolloutShape &r) {
  const int s = r.mesh ? 7 : r.scene;
  switch (f) {
    case Family::Standard:
      if (r.spline) return grad ? by_scene<false>(s, [](auto c) { return rollout_fused_kernel<c, true>; }) : nullptr;
      return by_scene<true>(s, [=](auto c) { return grad ? rollout_fused_kernel<c, false> : rollout_cost_kernel<c>; });
    case Family::ArmRows:
      return by_scene<false>(s, [=](auto c) { return grad ? rollout_fused_kernel<c, false, 3> : rollout_cost_kernel<c, 3>; });
    case Family::ArmPairs:  // never against an ESDF: SCENE 0 and 1 only
      if (s > 1) return nullptr;
      if (!grad) return (const void *)(s ? rollout_cost_kernel<1, 3, 2> : rollout_cost_kernel<0, 3, 2>);
      return (const void *)(s ? rollout_fused_kernel<1, false, 3, 2> : rollout_fused_kernel<0, false, 3, 2>);
    case Family::Big:
      if (r.arm_sized)
        return by_scene<true>(s, [=](auto c) { return grad ? rollout_fused_big_kernel<c, true> : rollout_cost_big_kernel<c, true>; });
      return by_scene<true>(s, [=](auto c) { return grad ? rollout_fused_big_kernel<c> : rollout_cost_big_kernel<c>; });
    case Family::Team2: return grad ? by_scene<false>(s, [](auto c) { return rollout_fused_team_kernel<c, 2>; }) : nullptr;
    case Family::Team4: return grad ? by_scene<false>(s, [](auto c) { return rollout_fused_team_kernel<c, 4>; }) : nullptr;
    case Family::Traj:
      if (!grad) return nullptr;
      if (r.spline && r.arm_sized) return by_scene<false>(s, [](auto c) { return rollout_traj_kernel<c, true, true>; });
      if (r.spline) return by_scene<false>(s, [](auto c) { return rollout_traj_kernel<c, true>; });
      if (r.arm_sized) return by_scene<true>(s, [](auto c) { return rollout_traj_kernel<c, false, true>; });
      return by_scene<true>(s, [](auto c) { return rollout_traj_kernel<c, false>; });
    case Family::TrajDyn: return grad ? by_scene<false>(s, [](auto c) { return rollout_traj_dyn_kernel<c>; }) : nullptr;
  }
  return nullptr;
}

// Family f planned for this call: its kernel, the shared floats of one of its rows (a.eval_floats) and its CTA shape.
struct RolloutPlan { Family family; const void *kernel; int row_floats; Plan plan; };

// The kernel family of this call, planned.  The rule reads top to bottom, and a family whose plan does not fit falls to the next
// candidate: team -> big -> the fused-dynamics, trajectory, arm or standard kernel.  The cost-only launch (!grad) follows the
// gradient launch's rule, row size included, except that it takes the big kernel where the gradient launch takes the team kernel.
static cudaError_t select_rollout(const RolloutShape &r, bool grad, const DevInfo &d, RolloutPlan &out) {
  const BlobHeader &h = r.h;
  auto plan = [&](Family f, RolloutPlan &p) {
    const bool team = f == Family::Team2 || f == Family::Team4, dyn = f == Family::TrajDyn;
    const int team_size = f == Family::Team4 ? 4 : 2;
    const int big_floats = grad ? big_smem_floats(h.nl, h.D, h.S, h.L, h.n_cl) : r.cost_floats;
    p.family = f;
    p.kernel = rollout_kernel(f, grad, r);
    p.row_floats = team ? (big_floats + team_extra_floats(team_size, h.nl) + 3) & ~3
                        : f == Family::Big ? big_floats : grad ? r.grad_floats : r.cost_floats;
    const size_t halo_bytes = r.traj ? (size_t)2 * h.S * sizeof(float4) : 0;  // trajectory kernels: the neighbouring waypoints
    const PlanKey key{p.kernel, d.ordinal, (size_t)h.smem_bytes + halo_bytes, (f == Family::ArmPairs ? 2 : 1) * p.row_floats,
                      r.traj ? r.H : 0, dyn ? h.nl : 0, dyn ? h.D : 0};
    return cached_plan(key, d, [=](const PlanKey &k, size_t limit) {
      if (dyn) return plan_dyn(k, limit);
      return team ? plan_team(k, limit, team_size) : plan_warps(k, limit, f == Family::Big ? kBigWarps : kWarpsPerCta);
    }, p.plan);
  };
  // big robots (humanoids) and ESDF scenes, discrete mode: the list-based kernel with up to 16 warps per SM (see
  // rollout_fused_big_kernel).  CB200_BIG = 0 / 1 forces it off / on.  Default: on when a row of the standard layout exceeds
  // 8 KB, and against an ESDF for robots that have no 80-register arm build (or too few rows to fill it).
  // (arms against an ESDF: the 80-register arm build of the standard kernel is faster at full batches -- Franka + 256^3 ESDF,
  //  16,384 rows: 0.0793 vs 0.0864 ms -- so they come here only when rows are scarce enough for two warps per row)
  // (an 18-warp build -- 576 threads, 96 registers, small spills -- measured 0.237 ms on G1-29 against 0.219 ms for 16 warps)
  const int big_env = env_int("CB200_BIG", -1);
  const long long slots = (long long)d.sm_count * kBigWarps;
  const bool big_fit = !r.traj && !r.spline && h.n_lp > 0 && h.P > 0;
  const bool big_want = big_env >= 0 ? big_env != 0
                                     : ((size_t)r.grad_floats * sizeof(float) > 8192 ||
                                        ((r.scene & 2) != 0 && (!r.arm_sized || r.N * 2 <= slots)));
  if (big_fit && big_want) {
    RolloutPlan big;
    cudaError_t e = plan(Family::Big, big);
    if (e != cudaSuccess) return e;
    // Small batches: a team of warps per row (rollout_fused_team_kernel) when the rows would leave at least half of the
    // resident warp slots idle.  CB200_TEAM = 0 / 2 / 4 forces the team size.  The team kernel has no mesh build: mesh scenes
    // stay on the big kernel, and so do cost-only launches.
    if (grad && !r.mesh && h.nl <= 64) {
      const int team_env = env_int("CB200_TEAM", -1);
      // Measured rule.  Small robots (row <= 8 KB, here because of the ESDF): two warps per
      // row while that leaves warp slots free.  Humanoids: four warps per row while that leaves slots free, then two -- always
      // when the one-warp plan is shared-memory limited (G1-43: 11 rows per SM; 8 teams of 2 warps are 16 warps
      // at 8,192 rows), otherwise (G1-29) up to about two rows per warp slot.
      const bool small_robot = (size_t)r.grad_floats * sizeof(float) <= 8192;
      const bool smem_limited = big.plan.nw > 0 && big.plan.nw * big.plan.per_sm < kBigWarps;
      int team = 0;
      if (team_env >= 0) team = team_env;
      else if (small_robot) team = (r.N * 2 <= slots) ? 2 : 0;
      else if (r.N * 4 <= slots) team = 4;
      else if (smem_limited || r.N <= 2 * slots) team = 2;
      if (team == 2 || team == 4) {
        e = plan(team == 4 ? Family::Team4 : Family::Team2, out);
        if (e != cudaSuccess || out.plan.nw > 0) return e;
      }
    }
    if (big.plan.nw > 0) {
      out = big;
      return cudaSuccess;
    }
  }
  if (r.dynamics && !r.dynamics_ok) return cudaErrorInvalidValue;
  Family f = r.dynamics ? Family::TrajDyn : r.traj ? Family::Traj : Family::Standard;
  if (!r.traj && !r.spline && !r.mesh && r.arm_sized) {
    // arms (few links / spheres): the row state is ~3 KB, so residency is register-bound; their 80-register builds keep 24
    // instead of 16 warps per SM resident and are ~7 % faster on the IK workload (slower for humanoids, where shared memory
    // bounds residency anyway).
    // Rows per warp: 2 for arms of <= 16 links (one link per lane of a half-warp in the sparse J^T) from 1.5 rows per resident
    // warp slot of the arm build (3 CTAs of kWarpsPerCta warps per SM) up; with fewer rows a warp per row is faster (Franka +
    // cuboids, H100 SXM at 400 W: 0.0183 vs 0.0255 ms at 1.0 rows per slot, 0.0274 vs 0.0270 ms at 1.5, 0.0324 vs 0.0271 ms at
    // 2.0).  Not against an ESDF: that build spills (140 B) and measured 2 % slower (franka_16384_esdf).  CB200_ARM_PAIRS = 0 / 1
    // forces one / two rows per warp.
    // Mesh scenes of arms stay on the 128-register build, one row per warp: an 80-register mesh build spilled 172 B (DESIGN.md
    // section 4), so none is built.
    const int pairs_env = env_int("CB200_ARM_PAIRS", -1);
    const bool pairs = h.nl <= 16 && (r.scene & 2) == 0 &&
                       (pairs_env >= 0 ? pairs_env != 0 : 2LL * r.N >= 3LL * d.sm_count * 3 * kWarpsPerCta);
    f = pairs ? Family::ArmPairs : Family::ArmRows;
  }
  const cudaError_t e = plan(f, out);
  if (e != cudaSuccess) return e;
  return out.plan.nw > 0 ? cudaSuccess : cudaErrorInvalidConfiguration;
}

// Checks a call's arguments, fills `a` and `r` and runs the expanded spline schedule; r.N == 0 with status 0: nothing to launch.
static int prepare_rollout(const cb200_rollout_cfg *cfg, const cb200_rollout_io *io, bool grad, cb200_stream_t stream,
                           FusedArgs &a, RolloutShape &r) {
  if (cfg == nullptr || io == nullptr || io->robot_blob == nullptr || io->cost == nullptr || (grad && io->grad_q == nullptr) ||
      io->batch_size < 0 || io->horizon < 1)
    return ret(cudaErrorInvalidValue);
  if (!grad && (io->q == nullptr || io->spline != nullptr || io->dynamics != nullptr || cfg->use_sweep != 0))
    return ret(cudaErrorInvalidValue);
  const cb200_spline_input *sp = io->spline;
  if (sp == nullptr && io->q == nullptr) return ret(cudaErrorInvalidValue);
  int spline_steps = 0;
  if (sp != nullptr) {
    if (sp->knots == nullptr || sp->start_position == nullptr || sp->start_velocity == nullptr ||
        sp->start_acceleration == nullptr || sp->start_jerk == nullptr || sp->start_idx == nullptr ||
        sp->goal_idx == nullptr || sp->traj_dt == nullptr || sp->use_implicit_goal_state == nullptr ||
        sp->goal_position == nullptr || sp->goal_velocity == nullptr || sp->goal_acceleration == nullptr ||
        sp->goal_jerk == nullptr || sp->n_knots < 1 || sp->degree < 3 || sp->degree > 5)
      return ret(cudaErrorInvalidValue);
    spline_steps = (io->horizon - 1) / (sp->n_knots + sp->degree + 1);
    if (sp->grad_knots != nullptr &&
        (io->grad_vel == nullptr || io->grad_acc == nullptr || io->grad_jerk == nullptr || io->horizon - 1 < 5 ||
         spline_steps < 1 || spline_steps > 32))
      return ret(cudaErrorInvalidValue);
  }
  if (io->goal_position != nullptr && (io->goal_quat == nullptr || cfg->num_goalset < 1)) return ret(cudaErrorInvalidValue);
  r.H = io->horizon;
  r.N = (long long)io->batch_size * io->horizon;
  if (r.N == 0) return ret(cudaSuccess);
  if (!read_blob_header(io->robot_blob_host, io->robot_blob_bytes, r.h)) return ret(cudaErrorInvalidValue);
  const BlobHeader &h = r.h;
  a.cfg = *cfg;
  a.q = io->q;
  a.vel = io->vel;
  a.acc = io->acc;
  a.jerk = io->jerk;
  a.dt = io->dt;
  a.blob = static_cast<const unsigned char *>(io->robot_blob);
  a.cuboids = to_dev(io->cuboids);
  a.voxels = to_dev(io->voxels);
  a.env_query_idx = io->env_query_idx;
  a.goal_position = io->goal_position;
  a.goal_quat = io->goal_quat;
  a.idxs_goal = io->idxs_goal;
  a.pose_axes_t = io->pose_axes_terminal;
  a.pose_axes_nt = io->pose_axes_non_terminal;
  a.pose_tol_t = io->pose_tol_terminal;
  a.pose_tol_nt = io->pose_tol_non_terminal;
  a.cost = io->cost;
  a.self_cost = io->self_cost;
  a.scene_cost = io->scene_cost;
  a.pose_cost = io->pose_cost;
  a.cspace_cost = io->cspace_cost;
  if (grad) {
    a.grad_q = io->grad_q;
    a.grad_vel = io->grad_vel;
    a.grad_acc = io->grad_acc;
    a.grad_jerk = io->grad_jerk;
  }
  a.link_pos = io->link_pos;
  a.link_quat = io->link_quat;
  a.robot_spheres = io->robot_spheres;
  a.pose_goalset_idx = io->pose_goalset_idx;
  a.B = io->batch_size;
  a.H = io->horizon;
  if (cfg->cspace_target_weight > 0.0f && cfg->cspace_type != 0) {
    if (io->cspace_target == nullptr) return ret(cudaErrorInvalidValue);
    a.cs_target = io->cspace_target;
    a.cs_target_idx = io->idxs_cspace_target;
    a.cs_target_dofw = io->cspace_target_dof_weight;
  }
  if (io->current_position != nullptr) {
    if (io->current_state_dt == nullptr) return ret(cudaErrorInvalidValue);
    if (cfg->cspace_type == 1) {  // only the POSITION cost has a current-state block
      a.cur_pos = io->current_position;
      a.cur_vel = io->current_velocity;
      a.cur_idx = io->idxs_current_state;
      a.cur_dt = io->current_state_dt;
    }
  }
  if (set_sphere_cfgs(io, h, a) != cudaSuccess) return ret(cudaErrorInvalidValue);
  a.blob_smem_bytes = h.smem_bytes;
  r.grad_floats = eval_smem_floats(h.nl, h.D, h.S, h.L, h.n_cl);
  r.cost_floats = cost_smem_floats(h.nl, h.D, h.S, h.n_cl, h.n_lp == 0);
  const bool expand = sp != nullptr && sp->out_position != nullptr && sp->out_velocity != nullptr &&
                      sp->out_acceleration != nullptr && sp->out_jerk != nullptr && sp->out_dt != nullptr;
  // mesh obstacles: scene bit 2.  The in-kernel spline schedule and the fused-dynamics kernel have no mesh build; they refuse mesh
  // scenes rather than drop the meshes (the expanded schedule and the host-composed dynamics cost support them).
  if (cfg->scene_weight > 0.0f && to_dev(io->meshes, a.meshes) != cudaSuccess) return ret(cudaErrorInvalidValue);
  r.mesh = a.meshes.inv_pose != nullptr;
  if (r.mesh && ((sp != nullptr && !expand) || io->dynamics != nullptr)) return ret(cudaErrorInvalidValue);
  if (expand) {
    // expanded schedule: knots -> state with the stand-alone spline kernel, then the plain rollout kernels read it
    const int rc = cb200_bspline_forward(sp->out_position, sp->out_velocity, sp->out_acceleration, sp->out_jerk, sp->out_dt,
                                         sp->knots, sp->start_position, sp->start_velocity, sp->start_acceleration,
                                         sp->start_jerk, sp->goal_position, sp->goal_velocity, sp->goal_acceleration,
                                         sp->goal_jerk, sp->start_idx, sp->goal_idx, sp->traj_dt,
                                         sp->use_implicit_goal_state, io->batch_size, io->horizon, h.D, sp->n_knots,
                                         sp->degree, stream);
    if (rc != 0) return ret((cudaError_t)rc);
    a.q = sp->out_position;
    a.vel = sp->out_velocity;
    a.acc = sp->out_acceleration;
    a.jerk = sp->out_jerk;
    a.dt = sp->out_dt;
  } else if (sp != nullptr) {
    a.spl = FusedArgs::Spline{sp->knots, sp->start_position, sp->start_velocity, sp->start_acceleration, sp->start_jerk,
                              sp->goal_position, sp->goal_velocity, sp->goal_acceleration, sp->goal_jerk, sp->traj_dt,
                              sp->start_idx, sp->goal_idx, sp->use_implicit_goal_state, sp->out_position,
                              sp->out_velocity, sp->out_acceleration, sp->out_jerk, sp->n_knots, sp->degree, spline_steps};
  }
  r.traj = cfg->use_sweep != 0;
  r.spline = a.spl.knots != nullptr;
  if (r.traj && cfg->use_speed_metric && a.dt == nullptr && !r.spline) return ret(cudaErrorInvalidValue);
  r.scene = (cfg->scene_weight > 0.0f ? ((a.cuboids.inv_pose ? 1 : 0) | (a.voxels.inv_pose ? 2 : 0)) : 0);
  r.arm_sized = h.nl <= 24 && h.S <= 128;
  // inverse dynamics inside the trajectory kernel: rows must come from caller-provided states (or the expanded spline schedule,
  // which arrives here with a.spl.knots == nullptr) and the STATE c-space cost must be on, else select_rollout refuses the call
  const cb200_dynamics_params *dp = io->dynamics;
  r.dynamics = dp != nullptr;
  r.dynamics_ok = dp != nullptr && dp->link_masses_com != nullptr && dp->link_inertias != nullptr && dp->gravity != nullptr &&
                  r.traj && cfg->cspace_type == 2 && !r.spline && a.vel != nullptr && a.acc != nullptr;
  if (r.dynamics_ok) a.dyn = FusedArgs::Dyn{dp->link_masses_com, dp->link_inertias, dp->gravity};
  return 0;
}

// cb200_rollout_cost_grad (grad) and cb200_rollout_cost (!grad): one launcher, one kernel selection.  The cost-only launch takes
// the cost-only twin of the kernel the gradient launch would take (the big kernel where that is the team kernel) and ignores the
// gradient outputs; it covers discrete rows from caller-provided positions, without the fused dynamics.
static int rollout_launch(const cb200_rollout_cfg *cfg, const cb200_rollout_io *io, cb200_stream_t stream, bool grad) {
  CB200_DEVICE_GUARD((io != nullptr ? io->cost : nullptr));
  FusedArgs a{};
  RolloutShape r{};
  int rc = prepare_rollout(cfg, io, grad, stream, a, r);
  if (rc != 0 || r.N == 0) return rc;
  const DevInfo &d = dev_info();
  RolloutPlan c;
  if (const cudaError_t e = select_rollout(r, grad, d, c); e != cudaSuccess) return ret(e);
  const Plan &p = c.plan;
  long long grid, B = io->batch_size, resident = (long long)d.sm_count * p.per_sm;  // resident: CTAs of one wave
  int block = p.nw * 32;
  a.eval_floats = c.row_floats;
  // CB200_QUEUE = 0: static striding even when the caller gives a ticket counter
  int32_t *const counter = env_int("CB200_QUEUE", 1) != 0 ? io->work_counter : nullptr;
  if (c.family == Family::Team2 || c.family == Family::Team4) {  // at most one CTA per SM
    const int team = c.family == Family::Team4 ? 4 : 2, nteams = p.nw / team;
    // spread the rows over all SMs first: fewer teams per CTA rather than fewer CTAs
    const int launch_teams = (r.N + nteams - 1) / nteams < d.sm_count ? (int)((r.N + d.sm_count - 1) / d.sm_count) : nteams;
    grid = std::min((r.N + launch_teams - 1) / launch_teams, (long long)d.sm_count);
    block = launch_teams * team * 32;
    a.work_counter = counter;
  } else if (c.family == Family::TrajDyn) {  // a CTA per dynamics chunk of R waypoints, no counter
    grid = std::min(resident, B * ((r.H + p.R - 1) / p.R));
  } else {  // a warp per row (standard, arm, big), per pair of rows (paired arm build) or per waypoint of a trajectory tile
    const int rows = c.family == Family::ArmPairs ? 2 : 1;
    const long long units = (r.N + rows - 1) / rows;
    const long long need = r.traj ? B * ((r.H + p.nw - 1) / p.nw) : (units + p.nw - 1) / p.nw;
    grid = std::min(resident, need);
    // big: always a counter; the others: none when each row / pair / tile has its own warp / CTA, or when int tickets overflow
    if (c.family == Family::Big || (need > resident && !(r.traj && need > 0x3fffffffLL))) a.work_counter = counter;
  }
  const int g = (int)std::max(grid, 1LL);
  g_last_variant = kFamilyVariant[(int)c.family] | (grad ? 0 : CB200_VARIANT_COST_ONLY);
  if (c.family == Family::TrajDyn)
    CB200_LAUNCH(((void (*)(const FusedArgs, const int))c.kernel), g, block, p.smem, (cudaStream_t)stream, a, p.R);
  else
    CB200_LAUNCH(((void (*)(const FusedArgs))c.kernel), g, block, p.smem, (cudaStream_t)stream, a);
  rc = launch_status();
  // the adjoint of the spline front end runs right behind the rollout kernel on the same stream
  const cb200_spline_input *sp = io->spline;
  if (rc != 0 || sp == nullptr || sp->grad_knots == nullptr) return rc;
  return ret((cudaError_t)cb200_bspline_backward(sp->grad_knots, io->grad_q, io->grad_vel, io->grad_acc, io->grad_jerk,
                                                 sp->traj_dt, sp->goal_idx, sp->use_implicit_goal_state, io->batch_size,
                                                 io->horizon, r.h.D, sp->n_knots, sp->degree, stream));
}

extern "C" {

int cb200_rollout_cost_grad(const cb200_rollout_cfg *cfg, const cb200_rollout_io *io, cb200_stream_t stream) {
  return rollout_launch(cfg, io, stream, true);
}

int cb200_rollout_cost(const cb200_rollout_cfg *cfg, const cb200_rollout_io *io, cb200_stream_t stream) {
  return rollout_launch(cfg, io, stream, false);
}

int cb200_rollout_validate(const cb200_rollout_io *io, uint8_t *valid, int32_t check_bounds, int32_t check_self,
                           int32_t check_scene, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(valid);
  if (io == nullptr || valid == nullptr || io->q == nullptr || io->robot_blob == nullptr || io->spline != nullptr ||
      io->dynamics != nullptr || io->current_position != nullptr || io->batch_size < 0 || io->horizon < 1)
    return ret(cudaErrorInvalidValue);
  const long long N = (long long)io->batch_size * io->horizon;
  if (N == 0) return ret(cudaSuccess);
  BlobHeader h;
  if (N > 0x7fffffffLL || !read_blob_header(io->robot_blob_host, io->robot_blob_bytes, h)) return ret(cudaErrorInvalidValue);
  FusedArgs a{};
  a.cfg.self_weight = 1.0f;
  a.cfg.scene_weight = 1.0f;
  a.cfg.scene_activation = 0.0f;
  a.q = io->q;
  a.blob = static_cast<const unsigned char *>(io->robot_blob);
  a.env_query_idx = io->env_query_idx;
  a.B = io->batch_size;
  a.H = io->horizon;
  a.blob_smem_bytes = h.smem_bytes;
  a.eval_floats = cost_smem_floats(h.nl, h.D, h.S, h.n_cl, h.n_lp == 0);
  if (set_sphere_cfgs(io, h, a) != cudaSuccess) return ret(cudaErrorInvalidValue);
  int scene = 0;
  if (check_scene) {
    a.cuboids = to_dev(io->cuboids);
    a.voxels = to_dev(io->voxels);
    if (to_dev(io->meshes, a.meshes) != cudaSuccess) return ret(cudaErrorInvalidValue);
    scene = a.meshes.inv_pose ? 7 : (a.cuboids.inv_pose ? 1 : 0) | (a.voxels.inv_pose ? 2 : 0);
  }
  const void *kernel = by_scene<true>(scene, [](auto c) { return rollout_validate_kernel<c>; });
  const DevInfo &d = dev_info();
  Plan p;
  const PlanKey key{kernel, d.ordinal, (size_t)h.smem_bytes, a.eval_floats, 0, 0, 0};
  if (const cudaError_t e = cached_plan(key, d, [](const PlanKey &k, size_t limit) { return plan_warps(k, limit, kWarpsPerCta); }, p);
      e != cudaSuccess)
    return ret(e);
  if (p.nw == 0) return ret(cudaErrorInvalidConfiguration);
  const long long resident = (long long)d.sm_count * p.per_sm, need = (N + p.nw - 1) / p.nw;
  if (need > resident) a.work_counter = env_int("CB200_QUEUE", 1) != 0 ? io->work_counter : nullptr;
  const int checks = (check_bounds ? kCheckBounds : 0) | (check_self ? kCheckSelf : 0) | (check_scene ? kCheckScene : 0);
  g_last_variant = CB200_VARIANT_VALIDATE;
  CB200_LAUNCH(((void (*)(const FusedArgs, uint8_t *, const int))kernel), (int)std::max(std::min(resident, need), 1LL), p.nw * 32,
               p.smem, (cudaStream_t)stream, a, valid, checks);
  return launch_status();
}

}  // extern "C"
