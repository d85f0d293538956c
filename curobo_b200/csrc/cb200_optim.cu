// cb200_optim.cu -- optimizer-side kernels of the solve loop (SURVEY.md 8f rank 2), C ABI.
//
//   cb200_lbfgs_step    replaces kernel_lbfgs_step / kernel_lbfgs_step_shared_memory
//                       (curobo/_src/curobolib/kernels/optimization/lbfgs/lbfgs_step_kernel.cuh:39-199)
//   cb200_line_search   replaces kernel_line_search (optimization/line_search/line_search_kernel.cuh:60-199)
//   cb200_mppi_sample   replaces the torch particle construction of ParticleOptCore.sample_actions
//   cb200_mppi_update   replaces the torch softmax / weighted sums / blends of MPPI._update_distribution (DIAG_A)
//
// The reference launches ONE CTA OF v_dim THREADS PER PROBLEM (optimization_config.py:54-70,76-127): 16,384 CTAs of
// 7 threads for the IK headline.  Here the mapping follows the problem size instead:
//   v_dim <= 32 : a group of G = 4/8/16/32 lanes owns a problem, 32/G problems per warp, persistent grid;
//                 reductions are shuffle trees inside the group (no shared memory, no __syncthreads); the history is
//                 staged once into shared memory while it is being rolled.
//   v_dim  > 32 : one CTA per problem, thread per variable (block reduction through shared memory).
// In both, sums are associated exactly like the reference's block_reduce_sum (shuffle-down tree per 32 consecutive
// elements, then the same tree over the per-warp sums; common/block_warp_reductions.cuh:44-105), so results are
// bit-compatible with the reference kernels.
//
// Both are HBM streams.  Per problem the step reads 2*m*V + 4*V + m floats and writes 2*m*V + 3*V + m (the history is
// physically rolled, as the reference's buffers are; QuasiNewtonBuffers readers expect the newest pair in slot m-1);
// the line search reads n*(2V+1) + V and writes 5V + 2n + O(1).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/curobo_b200.h"
#include "cb200_launch.h"

namespace {
using cb200::launch_status;
using cb200::opt_in_smem;
using cb200::persistent_grid;
using cb200::ret;

constexpr unsigned kFull = 0xffffffffu;

// ---- reductions ----------------------------------------------------------------------------------------------------
// Shuffle-down tree over a group of G lanes (absent elements hold 0, which the reference's masked tree skips:
// x + 0 == x), result of the group's lane 0 broadcast to the whole group.
template <int G>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int off = G / 2; off > 0; off >>= 1) v += __shfl_down_sync(kFull, v, off, G);
  return __shfl_sync(kFull, v, 0, G);
}
template <int G>
__device__ __forceinline__ float group_max(float v) {
#pragma unroll
  for (int off = G / 2; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(kFull, v, off, G));
  return v;
}

// CTA-wide sum in the reference's order; `data` = 32 floats of shared memory, every thread gets the result.
__device__ __forceinline__ float block_sum(float v, float *data) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(kFull, v, off);
  __syncthreads();  // previous readers of data[] are done
  if (lane == 0) data[warp] = v;
  __syncthreads();
  float w = (lane < nwarps) ? data[lane] : 0.0f;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) w += __shfl_down_sync(kFull, w, off);
  return __shfl_sync(kFull, w, 0);
}
__device__ __forceinline__ float block_max(float v, float *data) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(kFull, v, off));
  __syncthreads();
  if (lane == 0) data[warp] = v;
  __syncthreads();
  float w = (lane < nwarps) ? data[lane] : -INFINITY;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) w = fmaxf(w, __shfl_xor_sync(kFull, w, off));
  return w;
}

// ---- L-BFGS step ---------------------------------------------------------------------------------------------------
struct LbfgsArgs {
  float *step_vec, *rho, *y_buf, *s_buf, *x_0, *grad_0;
  const float *q, *grad_q;
  float epsilon;
  int B, m, V, stable;
  // optional fused line-search set-up (LineSearchStrategy._prepare_search_points, line_search_strategy.py:136-199):
  // x_set[b, j, :] = q[b, :] + magnitudes[j] * scale_action(step)
  float *x_set;                 // [B, n_ls, V] or null
  float *step_scaled;           // [B, V] or null: the clamped step the line search must be given
  const float *magnitudes;      // [n_ls]
  const float *step_max;        // [action_dim] or null (no clamping)
  int n_ls, action_dim, fix_terminal_from;  // elements >= fix_terminal_from are frozen (V when unused)
};

__device__ __forceinline__ float new_rho(float numerator, int stable) {
  float r = (float)(1.0 / (double)numerator);  // the reference divides in double (lbfgs_step_helpers.cuh:134)
  if (stable && numerator <= 0.0f) r = 0.0f;
  return r;
}
__device__ __forceinline__ float gamma_scale(float numerator, float denominator, float epsilon, int stable) {
  float var1 = numerator / denominator;
  if (stable && (isinf(var1) || isnan(var1))) var1 = epsilon;
  return var1 < 0.0f ? 0.0f : var1;  // curobo::common::relu
}

template <int G>
__global__ void __launch_bounds__(128) lbfgs_step_group_kernel(const __grid_constant__ LbfgsArgs a) {
  CB200_EXTERN_SHARED float smem[];
  constexpr int P = 32 / G;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int sub = lane / G, t = lane % G;
  const int m = a.m, V = a.V;
  // per warp: y[m][32], s[m][32], rho[P][32], alpha[P][32]
  float *sy = smem + (size_t)warp * (2 * m * 32 + 2 * P * 32);
  float *ss = sy + m * 32;
  float *srho = ss + m * 32;
  float *salpha = srho + P * 32;
  const size_t BV = (size_t)a.B * V;
  const long long groups = ((long long)a.B + P - 1) / P;
  for (long long wg = (long long)blockIdx.x * nwarps + warp; wg < groups; wg += (long long)gridDim.x * nwarps) {
    const long long b = wg * P + sub;
    const bool valid = b < a.B;
    const bool act = valid && t < V;
    const size_t idx = (size_t)b * V + t;
    float gq = 0.0f, y = 0.0f, s = 0.0f, qt = 0.0f;
    if (act) {
      gq = a.grad_q[idx];
      qt = a.q[idx];
      y = gq - a.grad_0[idx];
      s = qt - a.x_0[idx];
      a.grad_0[idx] = gq;
      a.x_0[idx] = qt;
    }
    const float numerator = group_sum<G>(y * s);
    // roll the history left by one while staging it (each thread touches only its own column: in place is safe)
    for (int i = 0; i < m - 1; ++i) {
      float yy = 0.0f, sv = 0.0f;
      if (act) {
        yy = a.y_buf[(size_t)(i + 1) * BV + idx];
        sv = a.s_buf[(size_t)(i + 1) * BV + idx];
        a.y_buf[(size_t)i * BV + idx] = yy;
        a.s_buf[(size_t)i * BV + idx] = sv;
      }
      sy[i * 32 + lane] = yy;
      ss[i * 32 + lane] = sv;
    }
    sy[(m - 1) * 32 + lane] = y;
    ss[(m - 1) * 32 + lane] = s;
    if (act) {
      a.y_buf[(size_t)(m - 1) * BV + idx] = y;
      a.s_buf[(size_t)(m - 1) * BV + idx] = s;
    }
    // rho: roll + append
    const float rnew = new_rho(numerator, a.stable);
    for (int i0 = 0; i0 < m; i0 += G) {
      const int i = i0 + t;
      float r = 0.0f;
      if (valid && i < m) r = (i < m - 1) ? a.rho[(size_t)(i + 1) * a.B + b] : rnew;
      __syncwarp();  // all reads of this chunk before any write (lane t+1 owns the slot lane t just read)
      if (valid && i < m) {
        a.rho[(size_t)i * a.B + b] = r;
        srho[sub * 32 + i] = r;
      }
    }
    __syncwarp();
    // two-loop recursion
    for (int i = m - 1; i >= 0; --i) {
      const float cs = ss[i * 32 + lane], cy = sy[i * 32 + lane], cr = srho[sub * 32 + i];
      const float al = group_sum<G>(gq * cs) * cr;
      gq = gq - al * cy;
      if (t == 0) salpha[sub * 32 + i] = al;
    }
    __syncwarp();
    const float denominator = group_sum<G>(y * y);
    gq = gamma_scale(numerator, denominator, a.epsilon, a.stable) * gq;
    for (int i = 0; i < m; ++i) {
      const float cy = sy[i * 32 + lane], cs = ss[i * 32 + lane], cr = srho[sub * 32 + i], al = salpha[sub * 32 + i];
      const float beta = group_sum<G>(gq * cy) * cr;
      gq = gq + (al - beta) * cs;
    }
    float step = -gq;
    if (act) a.step_vec[idx] = step;
    if (a.x_set != nullptr) {
      if (a.step_max != nullptr) {  // scale_action (line_search_strategy.py:214-240)
        const float ratio = act ? fabsf(step) / a.step_max[t % a.action_dim] : 0.0f;
        const float sc = fmaxf(group_max<G>(ratio), 1.0f);
        step = step / sc;
      }
      if (t >= a.fix_terminal_from) step = 0.0f;
      if (act) {
        if (a.step_scaled != nullptr) a.step_scaled[idx] = step;
        for (int j = 0; j < a.n_ls; ++j) a.x_set[((size_t)b * a.n_ls + j) * V + t] = qt + a.magnitudes[j] * step;
      }
    }
    __syncwarp();  // smem reuse in the next iteration
  }
}

// v_dim > 32: CTA per problem, thread per variable; history re-read from L1/L2 after the roll.
__global__ void lbfgs_step_block_kernel(const __grid_constant__ LbfgsArgs a) {
  CB200_EXTERN_SHARED float smem[];  // alpha[m] + rho[m]
  __shared__ float data[32];
  const int t = threadIdx.x, m = a.m, V = a.V;
  const int b = blockIdx.x;
  const bool act = t < V;
  float *salpha = smem, *srho = smem + m;
  const size_t BV = (size_t)a.B * V;
  const size_t idx = (size_t)b * V + t;
  float gq = 0.0f, y = 0.0f, s = 0.0f, qt = 0.0f;
  if (act) {
    gq = a.grad_q[idx];
    qt = a.q[idx];
    y = gq - a.grad_0[idx];
    s = qt - a.x_0[idx];
    a.grad_0[idx] = gq;
    a.x_0[idx] = qt;
    for (int i = 0; i < m - 1; ++i) {
      a.y_buf[(size_t)i * BV + idx] = a.y_buf[(size_t)(i + 1) * BV + idx];
      a.s_buf[(size_t)i * BV + idx] = a.s_buf[(size_t)(i + 1) * BV + idx];
    }
    a.y_buf[(size_t)(m - 1) * BV + idx] = y;
    a.s_buf[(size_t)(m - 1) * BV + idx] = s;
  }
  const float numerator = block_sum(y * s, data);
  if (t < m) srho[t] = (t < m - 1) ? a.rho[(size_t)(t + 1) * a.B + b] : new_rho(numerator, a.stable);
  __syncthreads();
  if (t < m) a.rho[(size_t)t * a.B + b] = srho[t];
  for (int i = m - 1; i >= 0; --i) {
    const float cs = act ? a.s_buf[(size_t)i * BV + idx] : 0.0f, cy = act ? a.y_buf[(size_t)i * BV + idx] : 0.0f;
    const float al = block_sum(gq * cs, data) * srho[i];
    gq = gq - al * cy;
    if (t == 0) salpha[i] = al;
  }
  const float denominator = block_sum(y * y, data);  // also orders salpha writes before the reads below
  gq = gamma_scale(numerator, denominator, a.epsilon, a.stable) * gq;
  for (int i = 0; i < m; ++i) {
    const float cy = act ? a.y_buf[(size_t)i * BV + idx] : 0.0f, cs = act ? a.s_buf[(size_t)i * BV + idx] : 0.0f;
    const float beta = block_sum(gq * cy, data) * srho[i];
    gq = gq + (salpha[i] - beta) * cs;
  }
  float step = -gq;
  if (act) a.step_vec[idx] = step;
  if (a.x_set != nullptr) {
    if (a.step_max != nullptr) {
      const float ratio = act ? fabsf(step) / a.step_max[t % a.action_dim] : 0.0f;
      step = step / fmaxf(block_max(ratio, data), 1.0f);
    }
    if (t >= a.fix_terminal_from) step = 0.0f;
    if (act) {
      if (a.step_scaled != nullptr) a.step_scaled[idx] = step;
      for (int j = 0; j < a.n_ls; ++j) a.x_set[((size_t)b * a.n_ls + j) * V + t] = qt + a.magnitudes[j] * step;
    }
  }
}

// ---- line search ---------------------------------------------------------------------------------------------------
struct LineSearchArgs {
  float *best_cost, *best_action;
  int16_t *best_iteration, *current_iteration;
  uint8_t *converged;
  int convergence_iteration;
  float cost_delta_threshold, cost_relative_threshold;
  float *exploration_cost, *exploration_action, *exploration_gradient;
  int32_t *exploration_idx;
  float *selected_cost, *selected_action, *selected_gradient;
  int32_t *selected_idx;
  const float *search_cost, *search_action, *search_gradient, *step_direction, *magnitudes;
  float c_1, c_2;
  int strong_wolfe, approx_wolfe, n, V, B;
};

struct WolfePick {
  int selected, exploration;
};
// candidate flags (bit i = candidate i) -> indices (line_search_helpers.cuh:46-76)
__device__ __forceinline__ WolfePick pick_indices(unsigned m_armijo, unsigned m_wolfe, int strong, int approx) {
  const int id1 = m_armijo ? 31 - __clz(m_armijo) : 0;
  const int id = m_wolfe ? 31 - __clz(m_wolfe) : 0;
  WolfePick p;
  p.selected = strong ? id : (id == 0 ? id1 : id);
  p.exploration = (approx && !strong && p.selected == 0) ? 1 : p.selected;
  return p;
}
__device__ __forceinline__ void wolfe_flags(float alpha, float c_0, float c_val, float g_val, float g_0, float c_1, float c_2,
                                            int strong, bool &armijo, bool &wolfe) {
  const float c1_alpha_g0 = c_1 * alpha * g_0;
  const float c2_g0 = c_2 * g_0;
  const float c2_abs_g0 = c_2 * fabsf(g_0);
  armijo = c_val <= (c_0 + c1_alpha_g0);
  const bool curv = strong ? (fabsf(g_val) <= c2_abs_g0) : (g_val >= c2_g0);
  wolfe = armijo & curv;
}
// best / convergence bookkeeping by one thread (line_search_helpers.cuh:22-44,95-140); returns update_best
__device__ __forceinline__ bool bookkeeping(const LineSearchArgs &a, long long b, float sel_cost) {
  const float cur_best = a.best_cost[b];
  const int cur_it = (int)a.current_iteration[b] + 1;
  int best_it = a.best_iteration[b];
  const float delta = cur_best - sel_cost;
  const float rel = delta / (cur_best + 1e-6f);
  const bool upd = delta > a.cost_delta_threshold && rel > a.cost_relative_threshold;
  best_it = upd ? cur_it : best_it;
  a.converged[b] = (uint8_t)(best_it + a.convergence_iteration < cur_it);
  a.best_iteration[b] = (int16_t)best_it;
  a.current_iteration[b] = (int16_t)cur_it;
  if (upd) a.best_cost[b] = sel_cost;
  return upd;
}

template <int G>
__global__ void __launch_bounds__(128) line_search_group_kernel(const __grid_constant__ LineSearchArgs a) {
  constexpr int P = 32 / G;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int sub = lane / G, t = lane % G;
  const int n = a.n, V = a.V;
  const long long groups = ((long long)a.B + P - 1) / P;
  for (long long wg = (long long)blockIdx.x * nwarps + warp; wg < groups; wg += (long long)gridDim.x * nwarps) {
    const long long b = wg * P + sub;
    const bool valid = b < a.B;
    const bool act = valid && t < V;
    const float sv = act ? a.step_direction[(size_t)b * V + t] : 0.0f;
    // directional derivatives g_i . p; lane t of the group keeps candidate (chunk base + t)'s, flags are gathered
    // with one ballot per chunk of G candidates (n <= G in every shipped configuration: 4 candidates)
    unsigned m_armijo = 0u, m_wolfe = 0u;
    const unsigned gmask = (G == 32) ? kFull : ((1u << G) - 1u);
    const float c_0 = valid ? a.search_cost[(size_t)b * n] : 0.0f;
    float g_0 = 0.0f;
    for (int c0 = 0; c0 < n; c0 += G) {
      float g_mine = 0.0f;
      const int c_end = min(c0 + G, n);
      for (int i = c0; i < c_end; ++i) {
        const float g = act ? a.search_gradient[((size_t)b * n + i) * V + t] : 0.0f;
        const float r = group_sum<G>(g * sv);
        if (i == 0) g_0 = r;
        if (i - c0 == t) g_mine = r;
      }
      bool ar = false, wo = false;
      const int c = c0 + t;
      if (valid && c < n)
        wolfe_flags(a.magnitudes[c], c_0, a.search_cost[(size_t)b * n + c], g_mine, g_0, a.c_1, a.c_2, a.strong_wolfe, ar, wo);
      const unsigned ba = __ballot_sync(kFull, ar), bw = __ballot_sync(kFull, wo);
      m_armijo |= ((ba >> (sub * G)) & gmask) << c0;
      m_wolfe |= ((bw >> (sub * G)) & gmask) << c0;
    }
    const WolfePick pk = pick_indices(m_armijo, m_wolfe, a.strong_wolfe, a.approx_wolfe);
    int upd = 0;
    if (valid && t == 0) {
      const float sel_cost = a.search_cost[(size_t)b * n + pk.selected];
      a.exploration_cost[b] = a.search_cost[(size_t)b * n + pk.exploration];
      a.selected_cost[b] = sel_cost;
      upd = bookkeeping(a, b, sel_cost) ? 1 : 0;
    }
    upd = __shfl_sync(kFull, upd, 0, G);
    if (act) {
      const size_t o = (size_t)b * V + t;
      const size_t es = ((size_t)b * n + pk.exploration) * V + t, ss = ((size_t)b * n + pk.selected) * V + t;
      a.exploration_action[o] = a.search_action[es];
      a.exploration_gradient[o] = a.search_gradient[es];
      const float sa = a.search_action[ss];
      a.selected_action[o] = sa;
      a.selected_gradient[o] = a.search_gradient[ss];
      if (upd) a.best_action[o] = sa;
    }
    if (valid)
      for (int c = t; c < n; c += G) {
        a.exploration_idx[(size_t)b * n + c] = pk.exploration;
        a.selected_idx[(size_t)b * n + c] = pk.selected;
      }
  }
}

// V > 32: CTA per problem
__global__ void line_search_block_kernel(const __grid_constant__ LineSearchArgs a) {
  __shared__ float data[32];
  __shared__ float g_step[32];
  __shared__ int sh_sel, sh_exp, sh_upd;
  const int t = threadIdx.x, n = a.n, V = a.V;
  const long long b = blockIdx.x;
  const bool act = t < V;
  const float sv = act ? a.step_direction[(size_t)b * V + t] : 0.0f;
  for (int i = 0; i < n; ++i) {
    const float g = act ? a.search_gradient[((size_t)b * n + i) * V + t] : 0.0f;
    const float r = block_sum(g * sv, data);
    if (t == 0) g_step[i] = r;
  }
  __syncthreads();
  if (t < 32) {
    bool ar = false, wo = false;
    if (t < n) wolfe_flags(a.magnitudes[t], a.search_cost[(size_t)b * n], a.search_cost[(size_t)b * n + t], g_step[t], g_step[0], a.c_1, a.c_2, a.strong_wolfe, ar, wo);
    const unsigned ba = __ballot_sync(kFull, ar), bw = __ballot_sync(kFull, wo);
    if (t == 0) {
      const WolfePick pk = pick_indices(ba, bw, a.strong_wolfe, a.approx_wolfe);
      sh_sel = pk.selected;
      sh_exp = pk.exploration;
      const float sel_cost = a.search_cost[(size_t)b * n + pk.selected];
      a.exploration_cost[b] = a.search_cost[(size_t)b * n + pk.exploration];
      a.selected_cost[b] = sel_cost;
      sh_upd = bookkeeping(a, b, sel_cost) ? 1 : 0;
    }
  }
  __syncthreads();
  const int sel = sh_sel, ex = sh_exp;
  if (act) {
    const size_t o = (size_t)b * V + t;
    const size_t es = ((size_t)b * n + ex) * V + t, ss = ((size_t)b * n + sel) * V + t;
    a.exploration_action[o] = a.search_action[es];
    a.exploration_gradient[o] = a.search_gradient[es];
    const float sa = a.search_action[ss];
    a.selected_action[o] = sa;
    a.selected_gradient[o] = a.search_gradient[ss];
    if (sh_upd) a.best_action[o] = sa;
  }
  if (t < n) {
    a.exploration_idx[(size_t)b * n + t] = ex;
    a.selected_idx[(size_t)b * n + t] = sel;
  }
}

template <int G>
int launch_lbfgs_group(const LbfgsArgs &a, cudaStream_t stream) {
  constexpr int P = 32 / G;
  const int block = 128, nwarps = block / 32;
  const size_t smem = (size_t)nwarps * (2 * a.m * 32 + 2 * P * 32) * sizeof(float);
  if (const cudaError_t e = opt_in_smem(lbfgs_step_group_kernel<G>, smem); e != cudaSuccess) return e;
  const long long groups = ((long long)a.B + P - 1) / P;
  const int grid = persistent_grid(lbfgs_step_group_kernel<G>, block, smem, (groups + nwarps - 1) / nwarps);
  CB200_LAUNCH(lbfgs_step_group_kernel<G>, grid, block, smem, stream, a);
  return launch_status();
}
template <int G>
int launch_ls_group(const LineSearchArgs &a, cudaStream_t stream) {
  constexpr int P = 32 / G;
  const int block = 128, nwarps = block / 32;
  const long long groups = ((long long)a.B + P - 1) / P;
  const int grid = persistent_grid(line_search_group_kernel<G>, block, 0, (groups + nwarps - 1) / nwarps);
  CB200_LAUNCH(line_search_group_kernel<G>, grid, block, 0, stream, a);
  return launch_status();
}

// ---- MPPI sample -----------------------------------------------------------------------------------------------------
// ParticleOptCore.sample_actions (optim/components/particle_opt_core.py:409-441) for DIAG_A covariance and CLAMP squash:
// per problem, Ns particles mean + noise * scale, then n_neg copies of -mean, then zeros; every element clamped to
// max(min(a, high), low).  One thread per element of actions [P, Np, H, D], d fastest.  The explicit roundings keep torch's
// two (mul, then add) under --fmad=true, so the actions equal the reference's bit for bit.
struct MppiSampleArgs {
  float *actions;
  const float *mean, *scale, *noise, *lows, *highs;
  int total, Np, Ns, n_neg, HD, D, noise_stride;  // noise_stride: floats between problems' sample sets (0: one shared set)
};

__global__ void __launch_bounds__(256) mppi_sample_kernel(const __grid_constant__ MppiSampleArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.total) return;
  const int d = i % a.D, hd = i % a.HD, pj = i / a.HD;
  const int j = pj % a.Np, p = pj / a.Np;
  float v = 0.0f;
  if (j < a.Ns)
    v = __fadd_rn(a.mean[p * a.HD + hd], __fmul_rn(a.noise[p * a.noise_stride + j * a.HD + hd], a.scale[p * a.D + d]));
  else if (j < a.Ns + a.n_neg)
    v = -a.mean[p * a.HD + hd];
  a.actions[i] = fmaxf(fminf(v, a.highs[d]), a.lows[d]);
}

// ---- MPPI update -----------------------------------------------------------------------------------------------------
// MPPI._update_distribution (optim/particle/mppi.py:200-248) with jit_mean_cov_diag_a (mppi.py:722-757), per problem:
//   total_j = discount * sum_h cost[j, h]          (the reference sums the horizon, then broadcasts gamma_seq over it)
//   w = softmax(-total / beta)                     (max subtracted)
//   best = a[argmax_j w_j]                         (lowest index on ties, torch.argmax)
//   cov_upd[d] = mean_h sum_j w_j (a_j[h,d] - mean_old[h,d])^2,  cov = (1-s_c) cov + s_c cov_upd + kappa,  scale = sqrt(cov)
//   mean = (1-s_m) mean + s_m sum_j w_j a_j
// The library builds with --prec-sqrt=false; scale takes the correctly rounded square root torch.sqrt gives (the host SIMT
// emulation's std::sqrt is correctly rounded too).
#ifdef CB200_SIMT_EMULATION
inline float sqrt_rn(float x) { return std::sqrt(x); }
#else
__device__ __forceinline__ float sqrt_rn(float x) { return __fsqrt_rn(x); }
#endif
// Every sum runs in one fixed order (per-lane serial, then a fixed shuffle tree), so runs and graph replays are bit-identical.
struct MppiUpdateArgs {
  const float *actions, *cost;
  float *mean, *cov, *scale, *best;
  int P, Np, H, D;
  float neg_inv_beta, discount, step_mean, keep_mean, step_cov, keep_cov, kappa;
  int update_cov, best_mode;
};

// the particle's softmax argument -total / beta
__device__ __forceinline__ float mppi_exponent(const MppiUpdateArgs &a, long long p, int j) {
  const float *c = a.cost + ((size_t)p * a.Np + j) * a.H;
  float s = 0.0f;
  for (int h = 0; h < a.H; ++h) s = __fadd_rn(s, c[h]);
  return __fmul_rn(a.neg_inv_beta, __fmul_rn(a.discount, s));
}

// (weight, index) of the larger weight, the lower index on ties
__device__ __forceinline__ void argmax_merge(float &w, int &j, float ow, int oj) {
  if (ow > w || (ow == w && oj < j)) {
    w = ow;
    j = oj;
  }
}

// mean / best for element v of problem p from the weights w[Np]; returns the element's covariance-update sum
__device__ __forceinline__ float mppi_element(const MppiUpdateArgs &a, long long p, int v, const float *w, int best_j) {
  const int V = a.H * a.D;
  const float *act = a.actions + (size_t)p * a.Np * V + v;
  const float mo = a.mean[(size_t)p * V + v];
  float m = 0.0f, c = 0.0f;
  for (int j = 0; j < a.Np; ++j) {
    const float x = act[(size_t)j * V], wj = w[j];
    const float dl = __fsub_rn(x, mo);
    m = __fadd_rn(m, __fmul_rn(wj, x));
    c = __fadd_rn(c, __fmul_rn(wj, __fmul_rn(dl, dl)));
  }
  a.mean[(size_t)p * V + v] = __fadd_rn(__fmul_rn(a.keep_mean, mo), __fmul_rn(a.step_mean, m));
  if (a.best_mode) a.best[(size_t)p * V + v] = act[(size_t)best_j * V];
  return c;
}

// covariance of dimension d from the per-element sums sv[H*D]
__device__ __forceinline__ void mppi_cov(const MppiUpdateArgs &a, long long p, int d, const float *sv) {
  float s = 0.0f;
  for (int h = 0; h < a.H; ++h) s = __fadd_rn(s, sv[h * a.D + d]);
  const size_t o = (size_t)p * a.D + d;
  const float upd = __fdiv_rn(s, (float)a.H);
  const float cv = __fadd_rn(__fadd_rn(__fmul_rn(a.keep_cov, a.cov[o]), __fmul_rn(a.step_cov, upd)), a.kappa);
  a.cov[o] = cv;
  a.scale[o] = sqrt_rn(cv);
}

// small problems (Np * V <= kMppiGroupElems): a group of G lanes owns a problem, 128 / G problems per CTA, no __syncthreads
constexpr int kMppiGroupElems = 2048, kMppiGroupSmem = 256;  // group path also needs Np + V <= kMppiGroupSmem
template <int G>
__global__ void __launch_bounds__(128) mppi_update_group_kernel(const __grid_constant__ MppiUpdateArgs a) {
  CB200_EXTERN_SHARED float smem[];
  const int t = threadIdx.x % G, grp = threadIdx.x / G;
  const int Np = a.Np, D = a.D, V = a.H * a.D;
  float *w = smem + (size_t)grp * (Np + V), *sv = w + Np;  // weights, then the covariance-update sums
  const long long p = (long long)blockIdx.x * (128 / G) + grp;
  const bool valid = p < a.P;
  float mx = -INFINITY;
  for (int j = t; j < Np; j += G) {
    const float x = valid ? mppi_exponent(a, p, j) : 0.0f;
    w[j] = x;
    mx = fmaxf(mx, x);
  }
  mx = group_max<G>(mx);
  float se = 0.0f;
  for (int j = t; j < Np; j += G) {
    const float e = expf(__fsub_rn(w[j], mx));
    w[j] = e;
    se = __fadd_rn(se, e);
  }
  se = group_sum<G>(se);
  float bw = -1.0f;
  int bj = 0;
  for (int j = t; j < Np; j += G) {
    const float wj = __fdiv_rn(w[j], se);
    w[j] = wj;
    argmax_merge(bw, bj, wj, j);
  }
#pragma unroll
  for (int off = G / 2; off > 0; off >>= 1) {
    const float ow = __shfl_xor_sync(kFull, bw, off, G);
    const int oj = __shfl_xor_sync(kFull, bj, off, G);
    argmax_merge(bw, bj, ow, oj);
  }
  __syncwarp();  // every lane's weights before any lane reads them all
  if (valid)
    for (int v = t; v < V; v += G) sv[v] = mppi_element(a, p, v, w, bj);
  if (a.update_cov) {
    __syncwarp();
    if (valid)
      for (int d = t; d < D; d += G) mppi_cov(a, p, d, sv);
  }
}

// larger problems: one CTA per problem, block reductions through shared memory (Np + V floats, within the default 48 KB)
constexpr int kMppiBlock = 256, kMppiMaxSmemFloats = 48 * 1024 / 4;
__global__ void __launch_bounds__(kMppiBlock) mppi_update_block_kernel(const __grid_constant__ MppiUpdateArgs a) {
  CB200_EXTERN_SHARED float smem[];
  __shared__ float data[32];
  __shared__ float arg_w[32];
  __shared__ int arg_j[32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, nt = blockDim.x;
  const int Np = a.Np, D = a.D, V = a.H * a.D;
  float *w = smem, *sv = smem + Np;
  const long long p = blockIdx.x;
  float mx = -INFINITY;
  for (int j = t; j < Np; j += nt) {
    const float x = mppi_exponent(a, p, j);
    w[j] = x;
    mx = fmaxf(mx, x);
  }
  mx = block_max(mx, data);
  float se = 0.0f;
  for (int j = t; j < Np; j += nt) {
    const float e = expf(__fsub_rn(w[j], mx));
    w[j] = e;
    se = __fadd_rn(se, e);
  }
  se = block_sum(se, data);
  float bw = -1.0f;
  int bj = 0;
  for (int j = t; j < Np; j += nt) {
    const float wj = __fdiv_rn(w[j], se);
    w[j] = wj;
    argmax_merge(bw, bj, wj, j);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float ow = __shfl_xor_sync(kFull, bw, off);
    const int oj = __shfl_xor_sync(kFull, bj, off);
    argmax_merge(bw, bj, ow, oj);
  }
  if (lane == 0) {
    arg_w[warp] = bw;
    arg_j[warp] = bj;
  }
  __syncthreads();  // also orders every thread's weights before the reads below
  bw = -1.0f;
  bj = 0;
  for (int k = 0; k < (nt >> 5); ++k) argmax_merge(bw, bj, arg_w[k], arg_j[k]);
  for (int v = t; v < V; v += nt) sv[v] = mppi_element(a, p, v, w, bj);
  if (a.update_cov) {
    __syncthreads();
    for (int d = t; d < D; d += nt) mppi_cov(a, p, d, sv);
  }
}

template <int G>
int launch_mppi_group(const MppiUpdateArgs &a, cudaStream_t stream) {
  constexpr int NG = 128 / G;
  const size_t smem = (size_t)NG * (a.Np + a.H * a.D) * sizeof(float);
  CB200_LAUNCH(mppi_update_group_kernel<G>, (a.P + NG - 1) / NG, 128, smem, stream, a);
  return launch_status();
}
}  // namespace

extern "C" {

int cb200_lbfgs_step(float *step_vec, float *rho_buffer, float *y_buffer, float *s_buffer, const float *q,
                     const float *grad_q, float *x_0, float *grad_0, float epsilon, int batch_size, int history_m,
                     int v_dim, int stable_mode, float *x_set, float *step_scaled, const float *search_magnitudes, int n_linesearch,
                     const float *action_step_max, int action_dim, int fix_terminal_action, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(step_vec);
  // argument checks of the reference launcher (cuda_core_backend/optimization.py:173-176; lbfgs.py:171-173)
  if (step_vec == nullptr || rho_buffer == nullptr || y_buffer == nullptr || s_buffer == nullptr || q == nullptr ||
      grad_q == nullptr || x_0 == nullptr || grad_0 == nullptr || batch_size < 0 || v_dim < 1 || v_dim > 1024 ||
      history_m < 1 || history_m > 31)
    return ret(cudaErrorInvalidValue);
  if (x_set != nullptr && (search_magnitudes == nullptr || n_linesearch < 1 || (action_step_max != nullptr && action_dim < 1)))
    return ret(cudaErrorInvalidValue);
  if (batch_size == 0) return ret(cudaSuccess);
  LbfgsArgs a{step_vec, rho_buffer, y_buffer, s_buffer, x_0, grad_0, q, grad_q, epsilon, batch_size, history_m, v_dim,
              stable_mode, x_set, step_scaled, search_magnitudes, action_step_max, n_linesearch, action_dim < 1 ? 1 : action_dim,
              (fix_terminal_action && action_dim > 0 && v_dim > action_dim) ? v_dim - action_dim : v_dim};
  cudaStream_t st = (cudaStream_t)stream;
  if (v_dim <= 4) return launch_lbfgs_group<4>(a, st);
  if (v_dim <= 8) return launch_lbfgs_group<8>(a, st);
  if (v_dim <= 16) return launch_lbfgs_group<16>(a, st);
  if (v_dim <= 32) return launch_lbfgs_group<32>(a, st);
  const int block = (v_dim + 31) / 32 * 32;
  CB200_LAUNCH(lbfgs_step_block_kernel, batch_size, block, 2 * history_m * sizeof(float), st, a);
  return launch_status();
}

int cb200_line_search(float *best_cost, float *best_action, int16_t *best_iteration, int16_t *current_iteration,
                      uint8_t *converged_global, int convergence_iteration, float cost_delta_threshold,
                      float cost_relative_threshold, float *exploration_cost, float *exploration_action,
                      float *exploration_gradient, int32_t *exploration_idx, float *selected_cost,
                      float *selected_action, float *selected_gradient, int32_t *selected_idx, const float *search_cost,
                      const float *search_action, const float *search_gradient, const float *step_direction,
                      const float *search_magnitudes, float armijo_threshold_c_1, float curvature_threshold_c_2,
                      int strong_wolfe, int approx_wolfe, int n_linesearch, int opt_dim, int batchsize,
                      cb200_stream_t stream) {
  CB200_DEVICE_GUARD(best_cost);
  if (best_cost == nullptr || best_action == nullptr || best_iteration == nullptr || current_iteration == nullptr ||
      converged_global == nullptr || exploration_cost == nullptr || exploration_action == nullptr ||
      exploration_gradient == nullptr || exploration_idx == nullptr || selected_cost == nullptr ||
      selected_action == nullptr || selected_gradient == nullptr || selected_idx == nullptr || search_cost == nullptr ||
      search_action == nullptr || search_gradient == nullptr || step_direction == nullptr ||
      search_magnitudes == nullptr || n_linesearch < 1 || n_linesearch > 32 || opt_dim < 1 || opt_dim > 1024 ||
      batchsize < 0)
    return ret(cudaErrorInvalidValue);
  if (batchsize == 0) return ret(cudaSuccess);
  LineSearchArgs a{best_cost, best_action, best_iteration, current_iteration, converged_global, convergence_iteration,
                   cost_delta_threshold, cost_relative_threshold, exploration_cost, exploration_action,
                   exploration_gradient, exploration_idx, selected_cost, selected_action, selected_gradient, selected_idx,
                   search_cost, search_action, search_gradient, step_direction, search_magnitudes, armijo_threshold_c_1,
                   curvature_threshold_c_2, strong_wolfe, approx_wolfe, n_linesearch, opt_dim, batchsize};
  cudaStream_t st = (cudaStream_t)stream;
  if (opt_dim <= 4) return launch_ls_group<4>(a, st);
  if (opt_dim <= 8) return launch_ls_group<8>(a, st);
  if (opt_dim <= 16) return launch_ls_group<16>(a, st);
  if (opt_dim <= 32) return launch_ls_group<32>(a, st);
  const int block = (opt_dim + 31) / 32 * 32;
  CB200_LAUNCH(line_search_block_kernel, batchsize, block, 0, st, a);
  return launch_status();
}

int cb200_mppi_sample(float *actions, const float *mean, const float *scale, const float *noise, const float *lows,
                      const float *highs, int num_problems, int num_particles, int num_sampled, int num_neg, int horizon,
                      int action_dim, int noise_per_problem, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(actions);
  if (actions == nullptr || mean == nullptr || scale == nullptr || noise == nullptr || lows == nullptr || highs == nullptr ||
      num_problems < 0 || num_particles < 1 || num_sampled < 1 || num_neg < 0 || num_sampled + num_neg > num_particles ||
      horizon < 1 || action_dim < 1 ||
      (long long)num_problems * num_particles * horizon * action_dim > 0x7fffffffLL)
    return ret(cudaErrorInvalidValue);
  if (num_problems == 0) return ret(cudaSuccess);
  const int HD = horizon * action_dim, total = num_problems * num_particles * HD;
  MppiSampleArgs a{actions, mean, scale, noise, lows, highs, total, num_particles, num_sampled, num_neg, HD, action_dim,
                   noise_per_problem ? num_sampled * HD : 0};
  CB200_LAUNCH(mppi_sample_kernel, (total + 255) / 256, 256, 0, (cudaStream_t)stream, a);
  return launch_status();
}

int cb200_mppi_update(const float *actions, const float *cost, float *mean, float *cov, float *scale, float *best,
                      int num_problems, int num_particles, int horizon, int action_dim, float beta, float step_size_mean,
                      float step_size_cov, float kappa, float discount, int update_cov, int best_mode, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(mean);
  const long long V = (long long)horizon * action_dim;
  if (actions == nullptr || cost == nullptr || mean == nullptr || (update_cov && (cov == nullptr || scale == nullptr)) ||
      (best_mode && best == nullptr) || num_problems < 0 || num_particles < 1 || horizon < 1 || action_dim < 1 ||
      !(beta > 0.0f) || num_particles + V > kMppiMaxSmemFloats)
    return ret(cudaErrorInvalidValue);
  if (num_problems == 0) return ret(cudaSuccess);
  // the coefficients as torch forms them: Python-double scalars rounded once to float
  MppiUpdateArgs a{actions, cost, mean, cov, scale, best, num_problems, num_particles, horizon, action_dim,
                   (float)(-1.0 / (double)beta), discount, step_size_mean, (float)(1.0 - (double)step_size_mean),
                   step_size_cov, (float)(1.0 - (double)step_size_cov), kappa, update_cov ? 1 : 0, best_mode ? 1 : 0};
  cudaStream_t st = (cudaStream_t)stream;
  if ((long long)num_particles * V <= kMppiGroupElems && num_particles + V <= kMppiGroupSmem) {
    if (V <= 8) return launch_mppi_group<8>(a, st);
    if (V <= 16) return launch_mppi_group<16>(a, st);
    return launch_mppi_group<32>(a, st);
  }
  CB200_LAUNCH(mppi_update_block_kernel, num_problems, kMppiBlock, (num_particles + V) * sizeof(float), st, a);
  return launch_status();
}

}  // extern "C"
