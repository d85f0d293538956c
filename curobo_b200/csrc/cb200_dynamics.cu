// cb200_dynamics.cu -- RNEA inverse dynamics + adjoint kernels (SURVEY.md 8f rank 3), C ABI.
//
// Replaces rnea_forward_kernel / rnea_backward_kernel (curobo/_src/curobolib/kernels/dynamics/, launched by
// backends/cuda_core_backend/dynamics.py:24-250).  One thread per (seed x waypoint) row -- rows are independent and
// there are tens of thousands of them, so tree-level parallelism inside a row (the reference's threads_per_batch > 1
// path with shared-memory atomics) is not needed to fill the machine, and the serial order makes every sum
// deterministic.  A row's per-link spatial vectors live in a TRANSPOSED shared-memory tile
// [array][link][component][row-in-CTA]: consecutive threads touch consecutive words, no bank conflicts.
// HBM traffic per row: forward 3*D*4 in, D*4 + nl*80 (cache) out; adjoint D*4*3 + nl*80 in, 3*D*4 out.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <type_traits>

#include "../../include/curobo_b200.h"
#include "cb200_launch.h"
#include "cb200_dynamics.cuh"

namespace {
using namespace cb200::dyn;
using cb200::capped_grid;
using cb200::dev_info;
using cb200::launch_status;
using cb200::opt_in_smem;
using cb200::ret;

struct TileStore {  // [arr][link][comp][rows] floats in shared memory
  float *base;
  int rows, t, nl;
  __device__ __forceinline__ float get(int arr, int k, int c) const { return base[((size_t)(arr * nl + k) * 6 + c) * rows + t]; }
  __device__ __forceinline__ void set(int arr, int k, int c, float v) { base[((size_t)(arr * nl + k) * 6 + c) * rows + t] = v; }
};

struct FwdArgs {
  Model M;
  float *tau, *cache;
  const float *q, *qd, *qdd, *f_ext;
  int B;
};
__global__ void rnea_forward_rows(const __grid_constant__ FwdArgs a) {
  CB200_EXTERN_SHARED float smem[];
  TileStore S{smem, (int)blockDim.x, (int)threadIdx.x, a.M.nl};
  const int D = a.M.D, nl = a.M.nl;
  for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < a.B; row += (long long)gridDim.x * blockDim.x)
    rnea_forward_row(a.M, S, a.q + row * D, a.qd + row * D, a.qdd + row * D, a.f_ext ? a.f_ext + row * nl * 6 : nullptr,
                     a.tau + row * D, a.cache + row * nl * kCacheFloatsPerLink);
}

struct BwdArgs {
  Model M;
  float *gq, *gqd, *gqdd, *grad_f_ext;
  const float *grad_tau, *q, *qd, *cache;
  int B;
};
__global__ void rnea_backward_rows(const __grid_constant__ BwdArgs a) {
  CB200_EXTERN_SHARED float smem[];
  TileStore S{smem, (int)blockDim.x, (int)threadIdx.x, a.M.nl};
  const int D = a.M.D, nl = a.M.nl;
  for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < a.B; row += (long long)gridDim.x * blockDim.x)
    rnea_backward_row(a.M, S, a.grad_tau + row * D, a.q + row * D, a.qd + row * D, a.cache + row * nl * kCacheFloatsPerLink,
                      a.gq + row * D, a.gqd + row * D, a.gqdd + row * D, a.grad_f_ext ? a.grad_f_ext + row * nl * 6 : nullptr);
}

// ---------------------------------------------------------------------------------------------------------------------
// CTA-phased kernels (the default path).  A CTA of 128 threads owns R rows (R = 32 / 16 / 8) as W = 128 / R workers per
// row; a thread is (worker w, row r).  Work that does not depend on the tree recursion -- staging the inputs, sin/cos of
// every joint, f = I a + v x* I v, the local adjoint terms, every gradient dot product, the cache traffic -- runs over
// (link, row) pairs on all W workers; only the two recursions remain serial and they run LEVEL-synchronously (the links of
// one depth level spread over the workers, one barrier per level).  The leaf -> root passes PULL: a link sums its
// children's contributions in level order instead of children adding into the parent, so no two workers write the same
// slot and every sum keeps the reference's serial order (rnea_forward_kernel.cuh:225-270, rnea_backward_kernel.cuh:296-460;
// children of a level-l link are exactly the level-(l+1) links that name it as parent -- kinematics_params.py:259-288).
// Shared memory per CTA: [NA][nl][6][R+1] spatial vectors + [nl][2][R+1] sin/cos + [NIO][D][R+1] joint-space rows.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kThreads = 128;

// The robot's constants copied into the CTA's shared memory: every later access is a broadcast shared-memory load instead
// of a chain of dependent global loads (level_links -> joint_map -> joint_offset ...) on the serial recursion.
__device__ __forceinline__ Model stage_model(const Model &G, float *dst) {
  const int nl = G.nl, t = threadIdx.x, n = blockDim.x;
  float *ft = dst, *mc = ft + 12 * nl, *in = mc + 4 * nl, *jo = in + 8 * nl, *gr = jo + 2 * nl;
  int16_t *jm = reinterpret_cast<int16_t *>(gr + 6), *lm = jm + nl, *ll = lm + nl, *ls = ll + nl;
  int8_t *jt = reinterpret_cast<int8_t *>(gr + 6 + (3 * nl + G.n_levels + 1 + 1) / 2);
  for (int i = t; i < 12 * nl; i += n) ft[i] = G.fixed_transforms[i];
  for (int i = t; i < 4 * nl; i += n) mc[i] = G.masses_com[i];
  for (int i = t; i < 8 * nl; i += n) in[i] = G.inertias[i];
  for (int i = t; i < 2 * nl; i += n) jo[i] = G.joint_offset[i];
  for (int i = t; i < 6; i += n) gr[i] = G.gravity[i];
  for (int i = t; i < nl; i += n) {
    jm[i] = G.joint_map[i];
    lm[i] = G.link_map[i];
    ll[i] = G.level_links[i];
    jt[i] = G.joint_type[i];
  }
  for (int i = t; i <= G.n_levels; i += n) ls[i] = G.level_starts[i];
  return Model{ft, mc, in, jt, jm, lm, jo, gr, ls, ll, nl, G.D, G.n_levels};
}
inline int model_smem_floats_host(int nl, int n_levels) { return (12 + 4 + 8 + 2) * nl + 6 + (3 * nl + n_levels + 2) / 2 + (nl + 3) / 4; }

template <class L>
struct Cta {
  float *T, *SC, *IO;
  int nl, D, RS, r, w;
  const Model &M;
  __device__ __forceinline__ float &at(int arr, int k, int c) const { return T[((arr * nl + k) * 6 + c) * RS + r]; }
  __device__ __forceinline__ void load(int arr, int k, float *o) const {
#pragma unroll
    for (int c = 0; c < 6; ++c) o[c] = at(arr, k, c);
  }
  __device__ __forceinline__ void store(int arr, int k, const float *x) const {
#pragma unroll
    for (int c = 0; c < 6; ++c) at(arr, k, c) = x[c];
  }
  __device__ __forceinline__ float &io(int arr, int d) const { return IO[(arr * D + d) * RS + r]; }
  __device__ __forceinline__ Rp rp(int k, int jt) const {  // local transform of link k from the staged sin/cos (or travel)
    const float x = SC[(k * 2 + 0) * RS + r], c = SC[(k * 2 + 1) * RS + r];
    return local_Rp_sc<L>(M.fixed_transforms + 12 * k, jt, x, c, x);
  }
  // sin/cos (revolute) or travel (prismatic) of every link of this row; q staged in io(0, .)
  __device__ __forceinline__ void stage_joint_angles(int W) const {
    for (int k = w; k < nl; k += W) {
      const int jt = M.joint_type[k], ji = M.joint_map[k];
      float qe = 0.0f, sn = 0.0f, cs = 1.0f;
      if (jt >= 0 && ji >= 0) qe = L::f(M.joint_offset + 2 * k) * io(0, ji) + L::f(M.joint_offset + 2 * k + 1);
      if (jt >= 3) sincosf(qe, &sn, &cs);
      SC[(k * 2 + 0) * RS + r] = jt >= 3 ? sn : qe;
      SC[(k * 2 + 1) * RS + r] = cs;
    }
  }
};

template <int R>
__global__ void __launch_bounds__(kThreads) rnea_forward_cta(const __grid_constant__ FwdArgs a) {
  using L = LdPlain;  // constants staged into shared memory
  constexpr int RS = R + 1, W = kThreads / R;
  CB200_EXTERN_SHARED __align__(16) float smem[];
  const int nl = a.M.nl, D = a.M.D;
  const Model M = stage_model(a.M, smem + ((2 * 6 + 2) * nl + 4 * D) * RS);
  Cta<L> S{smem, smem + 2 * nl * 6 * RS, smem + (2 * 6 + 2) * nl * RS, nl, D, RS, (int)threadIdx.x % R, (int)threadIdx.x / R, M};
  __syncthreads();
  float g[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) g[i] = L::f(M.gravity + i);
  for (long long row0 = (long long)blockIdx.x * R; row0 < a.B; row0 += (long long)gridDim.x * R) {
    const int nrows = (int)((a.B - row0) < R ? (a.B - row0) : R);
    const bool live = S.r < nrows;
    for (int i = threadIdx.x; i < R * D; i += kThreads) {  // coalesced: the CTA's rows are contiguous
      const int rr = i / D, d = i - rr * D;
      const bool ok = rr < nrows;
      const size_t gi = (size_t)(row0 + rr) * D + d;
      S.IO[(0 * D + d) * RS + rr] = ok ? a.q[gi] : 0.0f;
      S.IO[(1 * D + d) * RS + rr] = ok ? a.qd[gi] : 0.0f;
      S.IO[(2 * D + d) * RS + rr] = ok ? a.qdd[gi] : 0.0f;
      S.IO[(3 * D + d) * RS + rr] = 0.0f;
    }
    __syncthreads();
    S.stage_joint_angles(W);
    __syncthreads();
    for (int lv = 0; lv < M.n_levels; ++lv) {  // root -> leaves: v, a
      for (int idx = M.level_starts[lv] + S.w; idx < M.level_starts[lv + 1]; idx += W) {
        const int k = M.level_links[idx], jt = M.joint_type[k], ji = M.joint_map[k], par = M.link_map[k];
        const bool root = (par < 0) || (par == k), moving = (jt >= 0) && (ji >= 0);
        const float mul = moving ? L::f(M.joint_offset + 2 * k) : 1.0f;
        const float qd_eff = moving ? mul * S.io(1, ji) : 0.0f, qdd_eff = moving ? mul * S.io(2, ji) : 0.0f;
        const Rp t = S.rp(k, jt);
        float v[6], ac[6], tmp[6];
        if (root) {
#pragma unroll
          for (int i = 0; i < 6; ++i) v[i] = 0.0f;
          Xv(t, g, ac);
        } else {
          S.load(0, par, tmp);
          Xv(t, tmp, v);
          S.load(1, par, tmp);
          Xv(t, tmp, ac);
        }
        if (jt >= 0) {
          const int s = s_index(jt);
          add6(v, s, qd_eff);
          add6(ac, s, qdd_eff);
          motion_cross_S_add(ac, v, s, qd_eff);
        }
        S.store(0, k, v);
        S.store(1, k, ac);
      }
      __syncthreads();
    }
    for (int k = S.w; k < nl; k += W) {  // every (link, row): cache v, a; f = I a + v x* (I v) [- f_ext]
      float v[6], ac[6], Ia[6], Iv[6], x[6];
      S.load(0, k, v);
      S.load(1, k, ac);
      if (live) {
        float4 *ck = reinterpret_cast<float4 *>(a.cache + ((size_t)(row0 + S.r) * nl + k) * kCacheFloatsPerLink);
        ck[0] = make_float4(v[0], v[1], v[2], v[3]);
        ck[1] = make_float4(v[4], v[5], ac[0], ac[1]);
        ck[2] = make_float4(ac[2], ac[3], ac[4], ac[5]);
      }
      inertia_times<L>(M.masses_com + 4 * k, M.inertias + 8 * k, ac, Ia);
      inertia_times<L>(M.masses_com + 4 * k, M.inertias + 8 * k, v, Iv);
      force_cross(v, Iv, x);
      const float *fe = (a.f_ext != nullptr && live) ? a.f_ext + ((size_t)(row0 + S.r) * nl + k) * 6 : nullptr;
#pragma unroll
      for (int i = 0; i < 6; ++i) ac[i] = Ia[i] + x[i] - (fe ? fe[i] : 0.0f);
      S.store(1, k, ac);
    }
    __syncthreads();
    for (int lv = M.n_levels - 2; lv >= 0; --lv) {  // leaves -> root: a link pulls its children's wrenches
      const int c0 = M.level_starts[lv + 1], c1 = M.level_starts[lv + 2];
      for (int idx = M.level_starts[lv] + S.w; idx < c0; idx += W) {
        const int k = M.level_links[idx];
        float f[6];
        S.load(1, k, f);
        bool any = false;
        for (int ci = c0; ci < c1; ++ci) {
          const int c = M.level_links[ci];
          if (M.link_map[c] != k) continue;
          const Rp t = S.rp(c, M.joint_type[c]);
          float fc[6], x[6];
          S.load(1, c, fc);
          XTf(t, fc, x);
#pragma unroll
          for (int i = 0; i < 6; ++i) f[i] += x[i];
          any = true;
        }
        if (any) S.store(1, k, f);
      }
      __syncthreads();
    }
    for (int k = S.w; k < nl; k += W) {  // every (link, row): cache f, joint torque
      float f[6];
      S.load(1, k, f);
      if (live) {
        float4 *ck = reinterpret_cast<float4 *>(a.cache + ((size_t)(row0 + S.r) * nl + k) * kCacheFloatsPerLink + kCacheF);
        ck[0] = make_float4(f[0], f[1], f[2], f[3]);
        ck[1] = make_float4(f[4], f[5], 0.0f, 0.0f);
      }
      const int jt = M.joint_type[k], ji = M.joint_map[k];
      if (jt >= 0 && ji >= 0) atomicAdd(&S.io(3, ji), L::f(M.joint_offset + 2 * k) * pick6(f, s_index(jt)));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nrows * D; i += kThreads) {
      const int rr = i / D, d = i - rr * D;
      a.tau[(size_t)row0 * D + i] = S.IO[(3 * D + d) * RS + rr];
    }
    __syncthreads();
  }
}

template <int R>
__global__ void __launch_bounds__(kThreads) rnea_backward_cta(const __grid_constant__ BwdArgs a) {
  using L = LdNc;  // constants read in place through the read-only path (measured faster than staging for the adjoint)
  constexpr int RS = R + 1, W = kThreads / R;
  CB200_EXTERN_SHARED __align__(16) float smem[];
  const int nl = a.M.nl, D = a.M.D;
  const Model &M = a.M;
  Cta<L> S{smem, smem + 5 * nl * 6 * RS, smem + (5 * 6 + 2) * nl * RS, nl, D, RS, (int)threadIdx.x % R, (int)threadIdx.x / R, M};
  float g[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) g[i] = L::f(M.gravity + i);
  for (long long row0 = (long long)blockIdx.x * R; row0 < a.B; row0 += (long long)gridDim.x * R) {
    const int nrows = (int)((a.B - row0) < R ? (a.B - row0) : R);
    const bool live = S.r < nrows;
    for (int i = threadIdx.x; i < R * D; i += kThreads) {
      const int rr = i / D, d = i - rr * D;
      const bool ok = rr < nrows;
      const size_t gi = (size_t)(row0 + rr) * D + d;
      S.IO[(0 * D + d) * RS + rr] = ok ? a.q[gi] : 0.0f;
      S.IO[(1 * D + d) * RS + rr] = ok ? a.qd[gi] : 0.0f;
      S.IO[(2 * D + d) * RS + rr] = ok ? a.grad_tau[gi] : 0.0f;
      S.IO[(3 * D + d) * RS + rr] = 0.0f;
      S.IO[(4 * D + d) * RS + rr] = 0.0f;
      S.IO[(5 * D + d) * RS + rr] = 0.0f;
    }
    for (int k = S.w; k < nl; k += W) {  // the forward pass's v, a, f of every (link, row)
      float4 c0 = make_float4(0, 0, 0, 0), c1 = c0, c2 = c0, c3 = c0, c4 = c0;
      if (live) {
        const float4 *ck = reinterpret_cast<const float4 *>(a.cache + ((size_t)(row0 + S.r) * nl + k) * kCacheFloatsPerLink);
        c0 = __ldg(ck), c1 = __ldg(ck + 1), c2 = __ldg(ck + 2), c3 = __ldg(ck + 3), c4 = __ldg(ck + 4);
      }
      const float v[6] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y}, ac[6] = {c1.z, c1.w, c2.x, c2.y, c2.z, c2.w};
      const float f[6] = {c3.x, c3.y, c3.z, c3.w, c4.x, c4.y};
      S.store(0, k, v);
      S.store(1, k, ac);
      S.store(2, k, f);
    }
    __syncthreads();
    S.stage_joint_angles(W);
    __syncthreads();
    for (int lv = 0; lv < M.n_levels; ++lv) {  // root -> leaves: f_bar; the dX^T/dq term of grad_q
      for (int idx = M.level_starts[lv] + S.w; idx < M.level_starts[lv + 1]; idx += W) {
        const int k = M.level_links[idx], jt = M.joint_type[k], ji = M.joint_map[k], par = M.link_map[k];
        const bool root = (par < 0) || (par == k), moving = (jt >= 0) && (ji >= 0);
        const float mul = moving ? L::f(M.joint_offset + 2 * k) : 1.0f;
        const int s = jt >= 0 ? s_index(jt) : 0;
        float fk[6], fbar[6] = {0, 0, 0, 0, 0, 0}, gq1 = 0.0f;
        S.load(2, k, fk);
        if (moving) add6(fbar, s, mul * S.io(2, ji));
        if (!root) {
          const Rp t = S.rp(k, jt);
          float fp[6], X[6];
          S.load(2, par, fp);
          Xv(t, fp, X);
#pragma unroll
          for (int i = 0; i < 6; ++i) fbar[i] += X[i];
          if (moving) gq1 = mul * dot_crf_S(X, fk, s);
        }
        S.store(2, k, fbar);
        S.at(3, k, 0) = gq1;
      }
      __syncthreads();
    }
    for (int k = S.w; k < nl; k += W) {  // every (link, row): the adjoint terms that do not involve the children
      const float *mc = M.masses_com + 4 * k, *in = M.inertias + 8 * k;
      float v[6], fbar[6], ab[6], t1[6], t2[6], vb[6];
      S.load(0, k, v);
      S.load(2, k, fbar);
      const float gq1 = S.at(3, k, 0);
      if (a.grad_f_ext != nullptr && live) {
        float *ge = a.grad_f_ext + ((size_t)(row0 + S.r) * nl + k) * 6;
#pragma unroll
        for (int i = 0; i < 6; ++i) ge[i] = -fbar[i];
      }
      inertia_times<L>(mc, in, fbar, ab);  // a_bar += I f_bar
      inertia_times<L>(mc, in, v, t1);
      force_cross(fbar, t1, t2);  // v_bar -= crf(f_bar) I v
#pragma unroll
      for (int i = 0; i < 6; ++i) vb[i] = 0.0f - t2[i];
      motion_cross(v, fbar, t1);
      inertia_times<L>(mc, in, t1, t2);  // v_bar -= I crm(v) f_bar
#pragma unroll
      for (int i = 0; i < 6; ++i) vb[i] -= t2[i];
      S.store(3, k, ab);
      S.store(4, k, vb);
      S.at(2, k, 0) = gq1;
    }
    __syncthreads();
    for (int lv = M.n_levels - 1; lv >= 0; --lv) {  // leaves -> root: a link pulls its children's a_bar, v_bar
      const int c0 = M.level_starts[lv + 1], c1 = (lv + 1 < M.n_levels) ? M.level_starts[lv + 2] : c0;
      for (int idx = M.level_starts[lv] + S.w; idx < c0; idx += W) {
        const int k = M.level_links[idx], jt = M.joint_type[k], ji = M.joint_map[k];
        float ab[6] = {0, 0, 0, 0, 0, 0}, vb[6] = {0, 0, 0, 0, 0, 0}, x[6], y[6];
        for (int ci = c0; ci < c1; ++ci) {
          const int c = M.level_links[ci];
          if (M.link_map[c] != k) continue;
          const Rp t = S.rp(c, M.joint_type[c]);
          S.load(3, c, x);
          XTf(t, x, y);
#pragma unroll
          for (int i = 0; i < 6; ++i) ab[i] += y[i];
          S.load(4, c, x);
          XTf(t, x, y);
#pragma unroll
          for (int i = 0; i < 6; ++i) vb[i] += y[i];
        }
        S.load(3, k, x);
        S.load(4, k, y);
#pragma unroll
        for (int i = 0; i < 6; ++i) {
          ab[i] += x[i];
          vb[i] += y[i];
        }
        if (jt >= 0 && ji >= 0) force_cross_S_add(vb, s_index(jt), L::f(M.joint_offset + 2 * k) * S.io(1, ji), ab);
        S.store(3, k, ab);
        S.store(4, k, vb);
      }
      __syncthreads();
    }
    for (int k = S.w; k < nl; k += W) {  // every moving (link, row): the three joint-space gradients
      const int jt = M.joint_type[k], ji = M.joint_map[k], par = M.link_map[k];
      if (jt < 0 || ji < 0) continue;
      const bool root = (par < 0) || (par == k);
      const float mul = L::f(M.joint_offset + 2 * k);
      const int s = s_index(jt);
      float v[6], ab[6], vb[6], fx[6], X[6], u[6];
      S.load(0, k, v);
      S.load(3, k, ab);
      S.load(4, k, vb);
      const Rp t = S.rp(k, jt);
      force_cross(v, ab, fx);
      const float gqdd = mul * pick6(ab, s);
      const float gqd = (0.0f - mul * pick6(fx, s)) + mul * pick6(vb, s);
      float gq;
      if (!root) {
        S.load(1, par, u);
        Xv(t, u, X);
        gq = S.at(2, k, 0) - mul * dot_crm_S(ab, X, s);
        S.load(0, par, u);
        Xv(t, u, X);
        gq -= mul * dot_crm_S(vb, X, s);
      } else {
        Xv(t, g, X);
        gq = 0.0f - mul * dot_crm_S(ab, X, s);
      }
      atomicAdd(&S.io(3, ji), gq);
      atomicAdd(&S.io(4, ji), gqd);
      atomicAdd(&S.io(5, ji), gqdd);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nrows * D; i += kThreads) {
      const int rr = i / D, d = i - rr * D;
      a.gq[(size_t)row0 * D + i] = S.IO[(3 * D + d) * RS + rr];
      a.gqd[(size_t)row0 * D + i] = S.IO[(4 * D + d) * RS + rr];
      a.gqdd[(size_t)row0 * D + i] = S.IO[(5 * D + d) * RS + rr];
    }
    __syncthreads();
  }
}

struct CtaPlan {
  int R = 0, smem = 0, grid = 0;
};
// rows per CTA: the largest of 32 / 16 / 8 that keeps two CTAs per SM resident, halved while the grid would leave SMs idle
CtaPlan plan_cta(int B, int floats_per_row, int model_floats, bool adjoint) {
  const cb200::DevInfo &d = dev_info();
  const int max_smem = d.max_smem, sms = d.sm_count;
  CtaPlan p;
  auto bytes = [&](int R) { return (floats_per_row * (R + 1) + model_floats) * (int)sizeof(float); };
  // tuning (scripts/bench_dynamics.py, not repeated on H100): the adjoint is fastest at 16 rows per CTA, the forward pass at 32 once
  // the grid is several CTAs per SM deep; never fewer than three resident CTAs per SM when a smaller tile allows it
  int R = adjoint ? 16 : 32;
  while (R > 8 && 3 * (bytes(R) + 1024) > max_smem) R >>= 1;
  while (R > 16 && ((long long)B + R - 1) / R < 4LL * sms) R >>= 1;
  while (R > 8 && ((long long)B + R - 1) / R < 1LL * sms) R >>= 1;
  if (const char *e = getenv("CB200_RNEA_R")) {  // tuning knob: force the rows per CTA
    const int v = atoi(e);
    if (v == 8 || v == 16 || v == 32) R = v;
  }
  if (bytes(R) > max_smem) return p;
  p.R = R;
  p.smem = bytes(R);
  p.grid = capped_grid(((long long)B + R - 1) / R, 32);
  return p;
}
inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// rows per CTA: the largest of 128 / 64 / 32 whose tile leaves room for two CTAs per SM, else the largest of 32 .. 4 that fits
template <class K>
int pick_rows(K kern, int floats_per_row, int &smem_out) {
  const int max_smem = dev_info().max_smem;
  for (int rows = 128; rows >= 4; rows >>= 1) {  // below a warp for very large trees: correctness first on this path
    const int smem = floats_per_row * rows * (int)sizeof(float);
    if (smem * 2 + 4096 <= max_smem || (rows <= 32 && smem <= max_smem) || rows == 4) {
      if (smem > max_smem) return 0;
      if (opt_in_smem(kern, smem) != cudaSuccess) continue;
      smem_out = smem;
      return rows;
    }
  }
  return 0;
}

bool model_ok(const Model &M) {
  return M.fixed_transforms && M.masses_com && M.inertias && M.joint_type && M.joint_map && M.link_map && M.joint_offset &&
         M.gravity && M.level_starts && M.level_links && M.nl >= 1 && M.nl <= 1024 && M.D >= 1 && M.n_levels >= 1;
}
}  // namespace

extern "C" {

int cb200_rnea_forward(float *tau, const float *q, const float *qd, const float *qdd, const float *fixed_transforms,
                       const float *link_masses_com, const float *link_inertias, const int8_t *joint_map_type,
                       const int16_t *joint_map, const int16_t *link_map, const float *joint_offset_map,
                       const float *gravity, const int16_t *level_starts, const int16_t *level_links, float *forward_cache,
                       int batch_size, int num_links, int num_dof, int n_levels, const float *f_ext, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(tau);
  Model M{fixed_transforms, link_masses_com, link_inertias, joint_map_type, joint_map, link_map, joint_offset_map, gravity,
          level_starts,     level_links,     num_links,     num_dof,        n_levels};
  if (!model_ok(M) || tau == nullptr || q == nullptr || qd == nullptr || qdd == nullptr || forward_cache == nullptr ||
      batch_size < 0)
    return ret(cudaErrorInvalidValue);
  if (batch_size == 0) return ret(cudaSuccess);
  FwdArgs a{M, tau, forward_cache, q, qd, qdd, f_ext, batch_size};
  const CtaPlan p = plan_cta(batch_size, (2 * 6 + 2) * num_links + 4 * num_dof, model_smem_floats_host(num_links, n_levels), false);
  if (p.R != 0 && aligned16(forward_cache) && getenv("CB200_RNEA_ROWS") == nullptr) {
    auto cta = [&](auto R) {  // false: the shared-memory opt-in failed, the rows kernel below runs instead
      if (opt_in_smem(rnea_forward_cta<R>, p.smem) != cudaSuccess) return false;
      CB200_LAUNCH(rnea_forward_cta<R>, p.grid, kThreads, p.smem, (cudaStream_t)stream, a);
      return true;
    };
    if ((p.R == 32 && cta(std::integral_constant<int, 32>{})) || (p.R == 16 && cta(std::integral_constant<int, 16>{})) ||
        (p.R == 8 && cta(std::integral_constant<int, 8>{})))
      return launch_status();
  }
  int smem = 0;  // very large trees: one thread per row over a two-array tile
  const int rows = pick_rows(rnea_forward_rows, 2 * num_links * 6, smem);
  if (rows == 0) return ret(cudaErrorInvalidConfiguration);
  CB200_LAUNCH(rnea_forward_rows, capped_grid(((long long)batch_size + rows - 1) / rows, 8), rows, smem, (cudaStream_t)stream, a);
  return launch_status();
}

int cb200_rnea_backward(float *grad_q, float *grad_qd, float *grad_qdd, const float *grad_tau, const float *q,
                        const float *qd, const float *fixed_transforms, const float *link_masses_com,
                        const float *link_inertias, const int8_t *joint_map_type, const int16_t *joint_map,
                        const int16_t *link_map, const float *joint_offset_map, const float *gravity,
                        const int16_t *level_starts, const int16_t *level_links, const float *forward_cache, int batch_size,
                        int num_links, int num_dof, int n_levels, float *grad_f_ext, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(grad_q);
  Model M{fixed_transforms, link_masses_com, link_inertias, joint_map_type, joint_map, link_map, joint_offset_map, gravity,
          level_starts,     level_links,     num_links,     num_dof,        n_levels};
  if (!model_ok(M) || grad_q == nullptr || grad_qd == nullptr || grad_qdd == nullptr || grad_tau == nullptr || q == nullptr ||
      qd == nullptr || forward_cache == nullptr || batch_size < 0)
    return ret(cudaErrorInvalidValue);
  if (batch_size == 0) return ret(cudaSuccess);
  BwdArgs a{M, grad_q, grad_qd, grad_qdd, grad_f_ext, grad_tau, q, qd, forward_cache, batch_size};
  const CtaPlan p = plan_cta(batch_size, (5 * 6 + 2) * num_links + 6 * num_dof, 0, true);
  if (p.R != 0 && aligned16(forward_cache) && getenv("CB200_RNEA_ROWS") == nullptr) {
    auto cta = [&](auto R) {
      if (opt_in_smem(rnea_backward_cta<R>, p.smem) != cudaSuccess) return false;
      CB200_LAUNCH(rnea_backward_cta<R>, p.grid, kThreads, p.smem, (cudaStream_t)stream, a);
      return true;
    };
    if ((p.R == 32 && cta(std::integral_constant<int, 32>{})) || (p.R == 16 && cta(std::integral_constant<int, 16>{})) ||
        (p.R == 8 && cta(std::integral_constant<int, 8>{})))
      return launch_status();
  }
  int smem = 0;
  const int rows = pick_rows(rnea_backward_rows, 5 * num_links * 6, smem);
  if (rows == 0) return ret(cudaErrorInvalidConfiguration);
  CB200_LAUNCH(rnea_backward_rows, capped_grid(((long long)batch_size + rows - 1) / rows, 8), rows, smem, (cudaStream_t)stream, a);
  return launch_status();
}

}  // extern "C"
