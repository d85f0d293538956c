// cb200_trajectory.cu -- B-spline knot -> state kernels and their adjoint (SURVEY.md 8f rank 1), the position (clique) and
// acceleration control-space transitions (below), C ABI.
//
// Replaces the reference's three trajectory launches
//   interpolate_bspline_kernel            (kernels/trajectory/bspline/bspline_kernel.cuh:87-149)
//   interpolate_bspline_single_dt_kernel  (:216-270)
//   bspline_backward_kernel               (:326-373)
// Both are pure HBM streams: the forward writes 4 x [B,T,D] floats from a [B,nk,D] read, the adjoint reads
// 4 x [B,T,D] (each row (DEG+1) times, from L1/L2) and writes [B,nk,D].  One thread per output element with the
// dof index fastest so every warp touches consecutive addresses; no shared memory, no shuffles.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/curobo_b200.h"
#include "cb200_bspline.cuh"
#include "cb200_launch.h"

namespace {
using namespace cb200::bspline;
using cb200::capped_grid;
using cb200::launch_status;
using cb200::ret;

struct FwdArgs {
  float *out_p, *out_v, *out_a, *out_j, *out_dt;
  const float *u;
  const float *sp, *sv, *sa, *sj, *gp, *gv, *ga, *gj;
  const int32_t *start_idx, *goal_idx;
  const float *traj_dt;                   // [n_goal] indexed by goal_idx, or a single value (single-dt mode)
  const uint8_t *implicit;                // [n_goal]
  const int32_t *interpolation_horizon;   // single-dt mode: per-batch horizon; nullptr otherwise
  int B, T, D, n_knots;
};

template <int DEG>
__global__ void __launch_bounds__(256) bspline_forward_kernel(const __grid_constant__ FwdArgs a) {
  const long long n = (long long)a.B * a.T * a.D;
  for (long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x; tid < n; tid += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(tid % a.D);
    const int h = (int)((tid / a.D) % a.T);
    const int b = (int)(tid / ((long long)a.D * a.T));
    const int s_row = __ldg(a.start_idx + b), g_row = __ldg(a.goal_idx + b);
    int padded = a.T;
    float dt;
    if (a.interpolation_horizon != nullptr) {  // bspline_kernel.cuh:255-258
      padded = min(__ldg(a.interpolation_horizon + b), a.T - 1) + 1;
      dt = __ldg(a.traj_dt);
    } else {
      dt = __ldg(a.traj_dt + g_row);
    }
    const int steps = (padded - 1) / (a.n_knots + DEG + 1);
    const ControlPolygon<DEG> cp = make_polygon<DEG>(a.u, b, d, a.D, a.n_knots, dt, steps, a.implicit[g_row] != 0, a.sp, a.sv,
                                                     a.sa, a.sj, s_row, a.gp, a.gv, a.ga, a.gj, g_row);
    const State4 s = evaluate<DEG>(cp, h, steps);
    a.out_p[tid] = s.p;
    a.out_v[tid] = s.v;
    a.out_a[tid] = s.a;
    a.out_j[tid] = s.j;
    if (h == 0 && d == 0) a.out_dt[b] = dt;
  }
}

struct BwdArgs {
  float *out;
  const float *gp, *gv, *ga, *gj;
  const float *traj_dt;
  const int32_t *dt_idx;
  const uint8_t *implicit;
  int B, T, D, n_knots;
};

template <int DEG>
__global__ void __launch_bounds__(256) bspline_backward_kernel(const __grid_constant__ BwdArgs a) {
  const long long n = (long long)a.B * a.n_knots * a.D;
  const int horizon = a.T - 1;
  const int steps = horizon / (a.n_knots + DEG + 1);
  for (long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x; tid < n; tid += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(tid % a.D);
    const int k = (int)((tid / a.D) % a.n_knots);
    const int b = (int)(tid / ((long long)a.D * a.n_knots));
    const int row = __ldg(a.dt_idx + b);
    const float dt = __ldg(a.traj_dt + row);
    const bool implicit = a.implicit[row] != 0;
    const size_t base = (size_t)b * a.T * a.D + d;
    const float *gp = a.gp, *gv = a.gv, *ga = a.ga, *gj = a.gj;
    const int D = a.D;
    auto G = [=](int h, int which) -> float {
      const float *src = which == 0 ? gp : which == 1 ? gv : which == 2 ? ga : gj;
      return __ldg(src + base + (size_t)h * D);
    };
    a.out[tid] = knot_gradient<DEG>(k, steps, a.n_knots, horizon, implicit, dt, G);
  }
}

int launch_forward(const FwdArgs &a, int degree, cudaStream_t stream) {
  if (a.B <= 0 || a.T <= 0 || a.D <= 0 || a.n_knots <= 0) return ret(cudaErrorInvalidValue);
  const long long n = (long long)a.B * a.T * a.D;
  const int grid = capped_grid((n + 255) / 256, 8);  // 8 x 256 threads / SM resident: a whole number of waves
  switch (degree) {
    case 3: CB200_LAUNCH(bspline_forward_kernel<3>, grid, 256, 0, stream, a); break;
    case 4: CB200_LAUNCH(bspline_forward_kernel<4>, grid, 256, 0, stream, a); break;
    case 5: CB200_LAUNCH(bspline_forward_kernel<5>, grid, 256, 0, stream, a); break;
    default: return ret(cudaErrorInvalidValue);
  }
  return launch_status();
}

// ------------------------------------------------------------------------------------------------
// Position (clique) and acceleration control spaces.  Replaces the reference's legacy launches
//   position_clique_loop_idx_fwd_kernel  (kernels/trajectory/legacy/differentiation_position_kernel.cuh:18-231, 406-466)
//   position_clique_loop_idx_bwd_kernel  (:236-401)
//   acceleration_loop_idx[_rk2]_kernel   (integration_acceleration_kernel.cuh:13-139)
// The clique kernels are HBM streams like the B-spline ones above and use the same layout: one thread per output element,
// dof fastest, so every load and store of a warp is contiguous; the 5-row stencil reads of neighbouring rows are served
// by L1.  (The reference's adjoint puts the action index fastest, so its neighbouring threads stride by D.)  The
// integrator runs one thread per (b, d) with running sums, so it needs no per-horizon instantiation and has no horizon
// limit.  The arithmetic is the reference's, operation for operation, including its double-precision literals.
// ------------------------------------------------------------------------------------------------
struct CliqueFwdArgs {
  float *out_p, *out_v, *out_a, *out_j, *out_dt;
  const float *u, *sp, *sv, *sa, *gp;
  const int32_t *start_idx, *goal_idx;
  const float *traj_dt;      // [n_goal], indexed through goal_idx
  const uint8_t *implicit;   // [n_goal], indexed through goal_idx
  int B, H, D;
};

// The stencil pads the trajectory before its first action with the start state at waypoint 1 and three waypoints
// extrapolated backwards from it (waypoints 0, -1, -2) at zero jerk.  Same expressions as the reference
// (differentiation_position_kernel.cuh:83-91), including `2.0 * dt * v` in double: the same expression trees give the
// same FMA contraction, so positions match bit for bit.
constexpr float kStartJerk = 0.0f;
__device__ __forceinline__ float back1(float p, float v, float a, float dt) {
  return -(3.0f / 2) * a * dt * dt - (7.0f / 6) * dt * dt * dt * kStartJerk - dt * v + p;
}
__device__ __forceinline__ float back2(float p, float v, float a, float dt) {
  return -2.0f * a * dt * dt - (4.0f / 3) * dt * dt * dt * kStartJerk - 2.0 * dt * v + p;
}
__device__ __forceinline__ float back3(float p, float v, float a, float dt) {
  return (3.0f / 2) * (-1 * a * (dt * dt) - (dt * dt * dt) * kStartJerk) - 3.0f * dt * v + p;
}

__global__ void __launch_bounds__(256) clique_forward_kernel(const __grid_constant__ CliqueFwdArgs a) {
  const int D = a.D, H = a.H, n_act = a.H - 4;
  const long long n = (long long)a.B * H * D;
  for (long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x; tid < n; tid += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(tid % D);
    const int h = (int)((tid / D) % H);
    const int b = (int)(tid / ((long long)D * H));
    const int s_row = __ldg(a.start_idx + b), g_row = __ldg(a.goal_idx + b);
    const float dt = __ldg(a.traj_dt + g_row);
    const bool use_goal = a.implicit[g_row] != 0;
    const float dt_inv = 1.0 / dt;
    const float *u = a.u + (size_t)b * n_act * D + d;
    // in[k] = waypoint h - 2 + k; waypoint w >= 2 is action w - 2
    float in[5];
    if (h <= 3) {
      // rows 0..3 (reference branches h == 0..3, tested before the end-of-horizon ones): start padding, then actions
      const size_t s = (size_t)s_row * D + d;
      const float p = __ldg(a.sp + s), v = __ldg(a.sv + s), acc = __ldg(a.sa + s);
      const float w_m2 = back3(p, v, acc, dt), w_m1 = back2(p, v, acc, dt), w_0 = back1(p, v, acc, dt);
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        const int w = h - 2 + k;
        in[k] = w >= 2 ? __ldg(u + (size_t)(w - 2) * D) : w == 1 ? p : w == 0 ? w_0 : w == -1 ? w_m1 : w_m2;
      }
    } else {
      // interior and end rows: waypoints past the last action repeat it; with the implicit goal the last action is
      // replaced by the goal position.  At H = 8 row 3 took the branch above and so reads the raw last action.
      const float last = use_goal ? __ldg(a.gp + (size_t)g_row * D + d) : __ldg(u + (size_t)(n_act - 1) * D);
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        const int i = h - 4 + k;
        in[k] = i >= n_act - 1 ? last : __ldg(u + (size_t)i * D);
      }
    }
    a.out_p[tid] = in[2];
    a.out_v[tid] = ((0.083333333f) * in[0] - (0.666666667f) * in[1] + (0.666666667f) * in[3] + (-0.083333333f) * in[4]) * dt_inv;
    a.out_a[tid] = ((-0.083333333f) * in[0] + (1.333333333f) * in[1] + (-2.5f) * in[2] + (1.333333333f) * in[3] +
                    (-0.083333333f) * in[4]) * dt_inv * dt_inv;
    a.out_j[tid] = ((-(1.0f / 2.0f)) * in[0] + in[1] - in[3] + ((1.0f / 2.0f)) * in[4]) * (dt_inv * dt_inv * dt_inv);
    if (h == 0 && d == 0) a.out_dt[b] = dt;
  }
}

struct CliqueBwdArgs {
  float *out;
  const float *gp, *gv, *ga, *gj;
  const float *traj_dt;
  const int32_t *dt_idx;
  const uint8_t *implicit;
  int B, H, D;
};

// d loss / d action i: action i is waypoint i + 2, which the stencils of rows i .. i + 4 read.  The coefficients are the
// reference's (differentiation_position_kernel.cuh:343-390): unsuffixed, so the velocity and acceleration sums (and the
// last action's jerk sum) are evaluated in double.
__global__ void __launch_bounds__(256) clique_backward_kernel(const __grid_constant__ CliqueBwdArgs a) {
  const int D = a.D, H = a.H, n_act = a.H - 4;
  const long long n = (long long)a.B * n_act * D;
  for (long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x; tid < n; tid += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(tid % D);
    const int i = (int)((tid / D) % n_act);
    const int b = (int)(tid / ((long long)D * n_act));
    const int row = __ldg(a.dt_idx + b);
    const float dt = __ldg(a.traj_dt + row);
    const bool use_goal = a.implicit[row] != 0;
    const float dt_inv = 1.0f / dt;
    const float dt_inv_2 = dt_inv * dt_inv;
    const float dt_inv_3 = dt_inv_2 * dt_inv;
    const size_t base = ((size_t)b * H + i) * D + d;   // gradient row i, the first of the five
    const float *gp = a.gp + base, *gv = a.gv + base, *ga = a.ga + base, *gj = a.gj + base;
    auto G = [D](const float *g, int k) { return __ldg(g + (size_t)k * D); };
    float out = G(gp, 2);
    if (i < n_act - 1) {
      out += (-0.0833333330000000 * G(gv, 0) + 0.666666667000000 * G(gv, 1) + 0 * G(gv, 2) - 0.666666667000000 * G(gv, 3) +
              0.0833333330000000 * G(gv, 4)) * dt_inv;
      out += (-0.0833333330000000 * G(ga, 0) + 1.33333333300000 * G(ga, 1) + (-2.50000000000000) * G(ga, 2) +
              1.33333333300000 * G(ga, 3) + (-0.0833333330000000) * G(ga, 4)) * dt_inv_2;
      out += (0.5f * G(gj, 0) - 1.0f * G(gj, 1) + 1.0f * G(gj, 3) - 0.5f * G(gj, 4)) * dt_inv_3;
    } else if (use_goal) {
      out = 0.0f;   // the goal replaces the last action in every row that reads it
    } else {
      // the last action also stands in for waypoints H-2 and H-1
      out += G(gp, 3) + G(gp, 4);
      out += (-0.0833333330000000 * G(gv, 0) + 0.583333334000000 * G(gv, 1) + 0.583333334000000 * G(gv, 2) -
              0.0833333330000000 * G(gv, 3) + 0.0 * G(gv, 4)) * dt_inv;
      out += (-0.0833333330000000 * G(ga, 0) + 1.25000000000000 * G(ga, 1) + (-1.25000000000000) * G(ga, 2) +
              0.0833333330000000 * G(ga, 3)) * dt_inv_2;
      out += (0.5 * G(gj, 0) - 0.5 * G(gj, 1) - 0.5 * G(gj, 2) + 0.5 * G(gj, 3)) * dt_inv_3;
    }
    a.out[tid] = out;
  }
}

struct IntegrateArgs {
  float *out_p, *out_v, *out_a, *out_j;
  const float *u, *sp, *sv, *sa;
  const int32_t *start_idx;
  const float *traj_dt;      // [H], indexed by waypoint
  int B, H, D;
};

// Semi-implicit Euler from the start state: acc[h] = u[h-1], vel += acc * dt[h], pos += vel * dt[h],
// jerk[h] = (acc[h] - acc[h-1]) / dt[h], jerk[0] = 0 (integration_acceleration_kernel.cuh:49-61).
__global__ void __launch_bounds__(128) acceleration_integrate_kernel(const __grid_constant__ IntegrateArgs a) {
  const int D = a.D, H = a.H;
  const long long n = (long long)a.B * D;
  for (long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x; tid < n; tid += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(tid % D);
    const int b = (int)(tid / D);
    const size_t s = (size_t)__ldg(a.start_idx + b) * D + d;
    float pos = __ldg(a.sp + s), vel = __ldg(a.sv + s), acc = __ldg(a.sa + s);
    size_t o = (size_t)b * H * D + d;
    a.out_p[o] = pos;
    a.out_v[o] = vel;
    a.out_a[o] = acc;
    a.out_j[o] = 0.0f;
    for (int h = 1; h < H; ++h) {
      const float dt = __ldg(a.traj_dt + h);
      const float acc_h = __ldg(a.u + o);   // u[h-1]
      o += D;
      vel = vel + acc_h * dt;
      pos = pos + vel * dt;
      a.out_p[o] = pos;
      a.out_v[o] = vel;
      a.out_a[o] = acc_h;
      a.out_j[o] = (acc_h - acc) / dt;
      acc = acc_h;
    }
  }
}
}  // namespace

extern "C" {

int cb200_bspline_forward(float *out_position, float *out_velocity, float *out_acceleration, float *out_jerk, float *out_dt,
                          const float *u_position, const float *start_position, const float *start_velocity,
                          const float *start_acceleration, const float *start_jerk, const float *goal_position,
                          const float *goal_velocity, const float *goal_acceleration, const float *goal_jerk,
                          const int32_t *start_idx, const int32_t *goal_idx, const float *traj_dt,
                          const uint8_t *use_implicit_goal_state, int batch_size, int padded_horizon, int dof, int n_knots,
                          int bspline_degree, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(out_position);
  FwdArgs a{out_position, out_velocity, out_acceleration, out_jerk, out_dt, u_position, start_position, start_velocity,
            start_acceleration, start_jerk, goal_position, goal_velocity, goal_acceleration, goal_jerk, start_idx, goal_idx,
            traj_dt, use_implicit_goal_state, nullptr, batch_size, padded_horizon, dof, n_knots};
  return launch_forward(a, bspline_degree, (cudaStream_t)stream);
}

int cb200_bspline_single_dt(float *out_position, float *out_velocity, float *out_acceleration, float *out_jerk, float *out_dt,
                            const float *u_position, const float *knot_dt, const float *start_position,
                            const float *start_velocity, const float *start_acceleration, const float *start_jerk,
                            const float *goal_position, const float *goal_velocity, const float *goal_acceleration,
                            const float *goal_jerk, const int32_t *start_idx, const int32_t *goal_idx,
                            const float *interpolation_dt, const uint8_t *use_implicit_goal_state,
                            const int32_t *interpolation_horizon, int batch_size, int max_out_tsteps, int dof, int n_knots,
                            int bspline_degree, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(out_position);
  (void)knot_dt;  // carried by the reference signature, never read by its kernel (bspline_kernel.cuh:216-270)
  if (interpolation_horizon == nullptr) return ret(cudaErrorInvalidValue);
  FwdArgs a{out_position, out_velocity, out_acceleration, out_jerk, out_dt, u_position, start_position, start_velocity,
            start_acceleration, start_jerk, goal_position, goal_velocity, goal_acceleration, goal_jerk, start_idx, goal_idx,
            interpolation_dt, use_implicit_goal_state, interpolation_horizon, batch_size, max_out_tsteps, dof, n_knots};
  return launch_forward(a, bspline_degree, (cudaStream_t)stream);
}

int cb200_bspline_backward(float *out_grad_knots, const float *grad_position, const float *grad_velocity,
                           const float *grad_acceleration, const float *grad_jerk, const float *traj_dt,
                           const int32_t *dt_idx, const uint8_t *use_implicit_goal_state, int batch_size, int padded_horizon,
                           int dof, int n_knots, int bspline_degree, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(out_grad_knots);
  const int horizon = padded_horizon - 1;
  // same argument checks as the reference launcher (trajectory_kernel_launch.cu:592-627)
  if (batch_size <= 0 || dof <= 0 || n_knots <= 0 || horizon < 5) return ret(cudaErrorInvalidValue);
  if (bspline_degree < 3 || bspline_degree > 5) return ret(cudaErrorInvalidValue);
  const int steps = horizon / (n_knots + bspline_degree + 1);
  if (steps <= 0 || steps > 32) return ret(cudaErrorInvalidValue);
  BwdArgs a{out_grad_knots, grad_position, grad_velocity, grad_acceleration, grad_jerk, traj_dt, dt_idx, use_implicit_goal_state,
            batch_size, padded_horizon, dof, n_knots};
  const long long n = (long long)batch_size * n_knots * dof;
  const int grid = capped_grid((n + 127) / 128, 8);
  switch (bspline_degree) {
    case 3: CB200_LAUNCH(bspline_backward_kernel<3>, grid, 128, 0, (cudaStream_t)stream, a); break;
    case 4: CB200_LAUNCH(bspline_backward_kernel<4>, grid, 128, 0, (cudaStream_t)stream, a); break;
    default: CB200_LAUNCH(bspline_backward_kernel<5>, grid, 128, 0, (cudaStream_t)stream, a); break;
  }
  return launch_status();
}

int cb200_position_clique_forward(float *out_position, float *out_velocity, float *out_acceleration, float *out_jerk,
                                  float *out_dt, const float *u_position, const float *start_position,
                                  const float *start_velocity, const float *start_acceleration, const float *goal_position,
                                  const float *goal_velocity, const float *goal_acceleration, const int32_t *start_idx,
                                  const int32_t *goal_idx, const float *traj_dt, const uint8_t *use_implicit_goal_state,
                                  int batch_size, int horizon, int dof, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(out_position);
  (void)goal_velocity;       // carried by the reference signature, never read by its kernel
  (void)goal_acceleration;
  if (batch_size == 0) return 0;
  // horizon >= 8: the reference's rows 1..3 read actions 1..3 for any horizon (past the row's actions below 8)
  if (batch_size < 0 || dof <= 0 || horizon < 8) return ret(cudaErrorInvalidValue);
  CliqueFwdArgs a{out_position, out_velocity, out_acceleration, out_jerk, out_dt, u_position, start_position, start_velocity,
                  start_acceleration, goal_position, start_idx, goal_idx, traj_dt, use_implicit_goal_state, batch_size,
                  horizon, dof};
  const int grid = capped_grid(((long long)batch_size * horizon * dof + 255) / 256, 8);
  CB200_LAUNCH(clique_forward_kernel, grid, 256, 0, (cudaStream_t)stream, a);
  return launch_status();
}

int cb200_position_clique_backward(float *out_grad_position, const float *grad_position, const float *grad_velocity,
                                   const float *grad_acceleration, const float *grad_jerk, const float *traj_dt,
                                   const int32_t *dt_idx, const uint8_t *use_implicit_goal_state, int batch_size, int horizon,
                                   int dof, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(out_grad_position);
  if (batch_size == 0) return 0;
  if (batch_size < 0 || dof <= 0 || horizon < 8) return ret(cudaErrorInvalidValue);
  CliqueBwdArgs a{out_grad_position, grad_position, grad_velocity, grad_acceleration, grad_jerk, traj_dt, dt_idx,
                  use_implicit_goal_state, batch_size, horizon, dof};
  const int grid = capped_grid(((long long)batch_size * (horizon - 4) * dof + 255) / 256, 8);
  CB200_LAUNCH(clique_backward_kernel, grid, 256, 0, (cudaStream_t)stream, a);
  return launch_status();
}

int cb200_acceleration_integrate(float *out_position, float *out_velocity, float *out_acceleration, float *out_jerk,
                                 const float *u_acc, const float *start_position, const float *start_velocity,
                                 const float *start_acceleration, const int32_t *start_idx, const float *traj_dt,
                                 int batch_size, int horizon, int dof, int use_rk2, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(out_position);
  (void)use_rk2;   // both reference kernels compute the same semi-implicit Euler step
  if (batch_size == 0) return 0;
  if (batch_size < 0 || dof <= 0 || horizon < 1) return ret(cudaErrorInvalidValue);
  IntegrateArgs a{out_position, out_velocity, out_acceleration, out_jerk, u_acc, start_position, start_velocity,
                  start_acceleration, start_idx, traj_dt, batch_size, horizon, dof};
  const int grid = capped_grid(((long long)batch_size * dof + 127) / 128, 8);
  CB200_LAUNCH(acceleration_integrate_kernel, grid, 128, 0, (cudaStream_t)stream, a);
  return launch_status();
}

}  // extern "C"
