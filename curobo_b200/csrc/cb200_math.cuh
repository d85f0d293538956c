// cb200_math.cuh -- scalar building blocks of the rollout hot path, usable from host and device.
//
// Everything here is per-(sphere | link | tool frame | dof) arithmetic with no thread cooperation, so it
// is compiled for the host as well and unit-tested on the CPU against oracle/ (tests/test_host_math.py)
// before any GPU time is spent.  Warp-cooperative code lives in cb200_warp.cuh.
//
// Reference arithmetic restated (not copied) from:
//   FK local transform      curobo/_src/curobolib/kernels/kinematics/kinematics_forward_helper.cuh:316-393
//   matrix -> quaternion    curobo/_src/curobolib/kernels/common/quaternion_util.cuh:52-58,110-158
//   quat grad -> omega      curobo/_src/curobolib/kernels/common/quaternion_util.cuh:86-103
//   collision activation    curobo/_src/geom/collision/wp_collision_common.py:12-37
//   cuboid SDF              curobo/_src/geom/data/data_cuboid.py:547-628
//   ESDF trilinear SDF      curobo/_src/geom/data/data_voxel.py:790-1069,1163-1215
//   tool-pose cost          curobo/_src/cost/wp_tool_pose.py:66-295,457-692
//   c-space costs           curobo/_src/cost/wp_cspace_state.py:21-285, wp_cspace_position.py:232-362,
//                           warp_bound_util.py:9-100
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#define CB_HD __host__ __device__ __forceinline__

namespace cb200 {

enum : int { JT_FIXED = -1, JT_XP = 0, JT_YP = 1, JT_ZP = 2, JT_XR = 3, JT_YR = 4, JT_ZR = 5 };

struct V3 {
  float x, y, z;
};
CB_HD V3 mk3(float x, float y, float z) { return V3{x, y, z}; }
CB_HD V3 operator+(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
CB_HD V3 operator-(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
CB_HD V3 operator*(float s, V3 a) { return V3{s * a.x, s * a.y, s * a.z}; }
CB_HD V3 operator*(V3 a, float s) { return V3{s * a.x, s * a.y, s * a.z}; }
CB_HD float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
CB_HD V3 cross(V3 a, V3 b) { return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
CB_HD float norm(V3 a) { return sqrtf(dot(a, a)); }

struct Q4 {  // quaternion stored x,y,z,w (Warp convention)
  float x, y, z, w;
};
CB_HD Q4 qmul(Q4 a, Q4 b) {
  return Q4{a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x,
            a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
CB_HD Q4 qconj(Q4 a) { return Q4{-a.x, -a.y, -a.z, a.w}; }
// wp.quat_rotate: v*(2w^2-1) + 2w (qv x v) + 2 qv (qv . v)
CB_HD V3 qrot(Q4 q, V3 v) {
  V3 qv = mk3(q.x, q.y, q.z);
  float c = 2.0f * q.w * q.w - 1.0f;
  V3 cr = cross(qv, v);
  float d = dot(qv, v);
  return mk3(v.x * c + cr.x * q.w * 2.0f + qv.x * d * 2.0f, v.y * c + cr.y * q.w * 2.0f + qv.y * d * 2.0f,
             v.z * c + cr.z * q.w * 2.0f + qv.z * d * 2.0f);
}

// ----------------------------------------------------------------------------------------------
// FK: local link transform  local = fixed * J(theta), written to o[12] (row-major 3x4).
// f may alias o.  theta already includes the (scale, bias) of joint_offset_map.
// ----------------------------------------------------------------------------------------------
CB_HD void local_link_transform(const float *f, int jt, float theta, float *o) {
  float m[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) m[i] = f[i];
  if (jt >= JT_XR) {
    float s, c;
    sincosf(theta, &s, &c);
    // rotate the two columns other than the axis: col_i' = c col_i + s col_j ; col_j' = c col_j - s col_i
    // with (i,j) = (y,z) for X, (z,x) for Y, (x,y) for Z.
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      float a0 = m[4 * r + 0], a1 = m[4 * r + 1], a2 = m[4 * r + 2];
      float b0 = a0, b1 = a1, b2 = a2;
      if (jt == JT_XR) {
        b1 = c * a1 + s * a2;
        b2 = c * a2 - s * a1;
      } else if (jt == JT_YR) {
        b2 = c * a2 + s * a0;
        b0 = c * a0 - s * a2;
      } else {
        b0 = c * a0 + s * a1;
        b1 = c * a1 - s * a0;
      }
      m[4 * r + 0] = b0;
      m[4 * r + 1] = b1;
      m[4 * r + 2] = b2;
    }
  } else if (jt >= JT_XP) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      float ax = (jt == JT_XP) ? m[4 * r + 0] : ((jt == JT_YP) ? m[4 * r + 1] : m[4 * r + 2]);
      m[4 * r + 3] += ax * theta;
    }
  }
#pragma unroll
  for (int i = 0; i < 12; ++i) o[i] = m[i];
}

// Rotation part of a row-major 3x4 transform -> quaternion (x,y,z,w) with w >= 0.
CB_HD Q4 quat_from_transform(const float *t) {
  const float t0 = t[0], t1 = t[1], t2 = t[2], t3 = t[4], t4 = t[5], t5 = t[6], t6 = t[8], t7 = t[9], t8 = t[10];
  Q4 q;
  float n, s;
  if (t8 < 0.0f) {
    if (t0 > t4) {
      n = 1.0f + t0 - t4 - t8;
      s = 0.5f * rsqrtf(n);
      q = Q4{n * s, (t1 + t3) * s, (t6 + t2) * s, -(t5 - t7) * s};
    } else {
      n = 1.0f - t0 + t4 - t8;
      s = 0.5f * rsqrtf(n);
      q = Q4{(t1 + t3) * s, n * s, (t5 + t7) * s, -(t6 - t2) * s};
    }
  } else {
    if (t0 < -t4) {
      n = 1.0f - t0 - t4 + t8;
      s = 0.5f * rsqrtf(n);
      q = Q4{(t6 + t2) * s, (t5 + t7) * s, n * s, -(t1 - t3) * s};
    } else {
      n = 1.0f + t0 + t4 + t8;
      s = 0.5f * rsqrtf(n);
      q = Q4{(t5 - t7) * s, (t6 - t2) * s, (t1 - t3) * s, -n * s};
    }
  }
  float inv = rsqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  if (q.w < 0.0f) inv = -inv;
  return Q4{q.x * inv, q.y * inv, q.z * inv, q.w * inv};
}

// omega = 1/2 E(q)^T g, g given w,x,y,z
CB_HD V3 quat_grad_to_omega(Q4 q, float gw, float gx, float gy, float gz) {
  return mk3(0.5f * (-q.x * gw + q.w * gx + q.z * gy - q.y * gz), 0.5f * (-q.y * gw - q.z * gx + q.w * gy + q.x * gz),
             0.5f * (-q.z * gw + q.y * gx - q.x * gy + q.w * gz));
}

// ----------------------------------------------------------------------------------------------
// Scene collision
// ----------------------------------------------------------------------------------------------
struct SdfGrad {
  float sdf;
  V3 n;  // "gradient" as the reference defines it: -d sdf/dp normalised (pointing into the obstacle)
};

// returns (cost, slope); pen <= 0 -> (0,0)
CB_HD void collision_activation(float pen, float eta, float &cost, float &slope) {
  if (pen <= 0.0f) {
    cost = 0.0f;
    slope = 0.0f;
  } else if (pen > eta) {
    cost = pen - 0.5f * eta;
    slope = 1.0f;
  } else {
    cost = 0.5f * pen * pen / eta;
    slope = pen / eta;
  }
}

CB_HD SdfGrad cuboid_sdf_grad(V3 p, float dx, float dy, float dz) {
  const float eps = 1e-6f;
  float hx = dx * 0.5f, hy = dy * 0.5f, hz = dz * 0.5f;
  float qx = fabsf(p.x) - hx, qy = fabsf(p.y) - hy, qz = fabsf(p.z) - hz;
  float cx = fmaxf(qx, 0.0f), cy = fmaxf(qy, 0.0f), cz = fmaxf(qz, 0.0f);
  float od = sqrtf(cx * cx + cy * cy + cz * cz);
  float maxq = fmaxf(qx, fmaxf(qy, qz));
  SdfGrad r;
  r.sdf = od + fminf(maxq, 0.0f);
  float gx = 0.0f, gy = 0.0f, gz = 0.0f;
  if (od > eps) {
    float inv = -1.0f / od;
    gx = cx * inv;
    gy = cy * inv;
    gz = cz * inv;
    if (p.x < 0.0f) gx = -gx;
    if (p.y < 0.0f) gy = -gy;
    if (p.z < 0.0f) gz = -gz;
  } else {
    if (fabsf(qx - maxq) < eps) {
      gx = (p.x < 0.0f) ? 1.0f : -1.0f;
    } else if (fabsf(qy - maxq) < eps) {
      gy = (p.y < 0.0f) ? 1.0f : -1.0f;
    } else {
      gz = (p.z < 0.0f) ? 1.0f : -1.0f;
    }
  }
  r.n = mk3(gx, gy, gz);
  return r;
}

CB_HD float load_half(const uint16_t *p) {
#ifdef __CUDA_ARCH__
  return __half2float(__ushort_as_half(__ldg(p)));
#else
  __half_raw hr;
  hr.x = *p;
  return __half2float(__half(hr));
#endif
}

// Boundary case of the trilinear sample (some of the 8 corners outside the grid): validity-weighted
// interpolation (data_voxel.py:919-1069).  Rare (spheres at the rim of the grid) -> kept out of line so the
// hot path stays small in the instruction cache.
static __host__ __device__ __noinline__ void voxel_sdf_boundary(const uint16_t *feat, long long base, long long sx, long long sy, bool x0k, bool x1k, bool y0k,
                        bool y1k, bool z0k, bool z1k, float fx, float fy, float fz, float inv, float max_dist,
                        float &sdf, float &gx, float &gy, float &gz) {
  const float fx1 = 1.0f - fx, fy1 = 1.0f - fy, fz1 = 1.0f - fz;
  float s[8], v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    int cx = (c >> 2) & 1, cy = (c >> 1) & 1, cz = c & 1;
    bool ok = (cx ? x1k : x0k) && (cy ? y1k : y0k) && (cz ? z1k : z0k);
    s[c] = max_dist;
    v[c] = 0.0f;
    if (ok) {
      s[c] = load_half(feat + base + cx * sx + cy * sy + cz);
      v[c] = 1.0f;
    }
  }
  float w[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) w[c] = (((c >> 2) & 1) ? fx : fx1) * (((c >> 1) & 1) ? fy : fy1) * ((c & 1) ? fz : fz1);
  float ws = 0.0f, vsum = 0.0f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    vsum += s[c] * w[c] * v[c];
    ws += w[c] * v[c];
  }
  if (ws <= 0.0f) {
    sdf = max_dist;
    gx = gy = gz = 0.0f;
    return;
  }
  sdf = vsum / ws;
  float gs, gw, wt;
  gs = gw = 0.0f;
#pragma unroll
  for (int c = 0; c < 4; ++c) {  // x: pairs (c, c+4) weighted by (y,z) bilinear weights
    wt = (((c >> 1) & 1) ? fy : fy1) * ((c & 1) ? fz : fz1);
    if (v[c] > 0.0f && v[c + 4] > 0.0f) {
      gs += (s[c + 4] - s[c]) * wt;
      gw += wt;
    }
  }
  gx = gw > 0.0f ? gs / gw * inv : 0.0f;
  gs = gw = 0.0f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    int c = ((k >> 1) << 2) | (k & 1);  // (x, y=0, z)
    wt = (((c >> 2) & 1) ? fx : fx1) * ((c & 1) ? fz : fz1);
    if (v[c] > 0.0f && v[c + 2] > 0.0f) {
      gs += (s[c + 2] - s[c]) * wt;
      gw += wt;
    }
  }
  gy = gw > 0.0f ? gs / gw * inv : 0.0f;
  gs = gw = 0.0f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    int c = k << 1;  // (x, y, z=0)
    wt = (((c >> 2) & 1) ? fx : fx1) * (((c >> 1) & 1) ? fy : fy1);
    if (v[c] > 0.0f && v[c + 1] > 0.0f) {
      gs += (s[c + 1] - s[c]) * wt;
      gw += wt;
    }
  }
  gz = gw > 0.0f ? gs / gw * inv : 0.0f;
}

// Trilinear ESDF sample + analytic gradient; feat points at the layer start (flat, z fastest).
// `need_below`: the caller only uses the normal when sdf < need_below (pen = r + eta - sdf > 0), so the gradient
// (two thirds of the arithmetic) is skipped otherwise -- the returned sdf is computed identically either way.
// `mip` (optional): min-pooled lower bounds, one fp16 per block of kMipBlock^3 base corners (cb200_voxel_build_mip).  A
// trilinear (or validity-weighted boundary) sample is a convex combination of its valid corner values, so
// mip[block] >= need_below proves sdf >= need_below and the eight scattered corner loads are skipped -- exact for the
// discrete test `pen = r + eta - sdf > 0`; the returned sdf is then only a lower bound, so swept sampling (which
// advances by the distance itself) must pass mip = nullptr.
constexpr int kMipShift = 3;                  // blocks of 8x8x8 base corners (4^3 measured the same: r18)
constexpr int kMipBlock = 1 << kMipShift;
CB_HD SdfGrad voxel_sdf_grad(V3 p, const uint16_t *feat, int nx, int ny, int nz, float vs, float max_dist,
                             float need_below = 3.0e38f, const uint16_t *mip = nullptr) {
  SdfGrad out;
  out.n = mk3(0.f, 0.f, 0.f);
  float sdf, gx, gy, gz;
  if (nx < 2 || ny < 2 || nz < 2) {
    // nearest-voxel lookup, zero gradient (data_voxel.py:825-829 + world_to_voxel_idx :709-724)
    int ix = (int)((p.x + (float)nx * vs * 0.5f) / vs);
    int iy = (int)((p.y + (float)ny * vs * 0.5f) / vs);
    int iz = (int)((p.z + (float)nz * vs * 0.5f) / vs);
    bool ok = ix >= 0 && ix < nx && iy >= 0 && iy < ny && iz >= 0 && iz < nz;
    sdf = ok ? load_half(feat + ((size_t)ix * ny + iy) * nz + iz) : max_dist;
    gx = gy = gz = 0.0f;
  } else {
    const float inv = 1.0f / vs;
    float vx = p.x * inv + (float)nx * 0.5f - 0.5f;
    float vy = p.y * inv + (float)ny * 0.5f - 0.5f;
    float vz = p.z * inv + (float)nz * 0.5f - 0.5f;
    float flx = floorf(vx), fly = floorf(vy), flz = floorf(vz);
    int x0 = (int)flx, y0 = (int)fly, z0 = (int)flz;
    float fx = vx - flx, fy = vy - fly, fz = vz - flz;
    float fx1 = 1.0f - fx, fy1 = 1.0f - fy, fz1 = 1.0f - fz;
    bool x0k = x0 >= 0 && x0 < nx, x1k = x0 + 1 >= 0 && x0 + 1 < nx;
    bool y0k = y0 >= 0 && y0 < ny, y1k = y0 + 1 >= 0 && y0 + 1 < ny;
    bool z0k = z0 >= 0 && z0 < nz, z1k = z0 + 1 >= 0 && z0 + 1 < nz;
    const long long sx = (long long)ny * nz, sy = nz;
    const long long base = (long long)x0 * sx + (long long)y0 * sy + z0;
    if (!((x0k || x1k) && (y0k || y1k) && (z0k || z1k))) {
      out.sdf = max_dist;  // all 8 corners outside the grid: weight_sum == 0 -> max_dist (data_voxel.py:1019-1020)
      return out;
    }
    if (mip != nullptr) {
      const int my = (ny + kMipBlock - 1) >> kMipShift, mz = (nz + kMipBlock - 1) >> kMipShift;
      const int cx = (x0 < 0 ? 0 : x0) >> kMipShift, cy = (y0 < 0 ? 0 : y0) >> kMipShift, cz = (z0 < 0 ? 0 : z0) >> kMipShift;
      const float lb = load_half(mip + ((size_t)cx * my + cy) * mz + cz);
      if (!(lb < need_below)) {
        out.sdf = lb >= max_dist ? max_dist : lb;
        return out;
      }
    }
    if (x0k && x1k && y0k && y1k && z0k && z1k) {
      const uint16_t *b = feat + base;
      float s000 = load_half(b), s001 = load_half(b + 1);
      float s010 = load_half(b + sy), s011 = load_half(b + sy + 1);
      float s100 = load_half(b + sx), s101 = load_half(b + sx + 1);
      float s110 = load_half(b + sx + sy), s111 = load_half(b + sx + sy + 1);
      sdf = s000 * fx1 * fy1 * fz1 + s001 * fx1 * fy1 * fz + s010 * fx1 * fy * fz1 + s011 * fx1 * fy * fz +
            s100 * fx * fy1 * fz1 + s101 * fx * fy1 * fz + s110 * fx * fy * fz1 + s111 * fx * fy * fz;
      if (!(sdf < need_below)) {
        out.sdf = sdf >= max_dist ? max_dist : sdf;
        return out;
      }
      gx = ((s100 - s000) * fy1 * fz1 + (s101 - s001) * fy1 * fz + (s110 - s010) * fy * fz1 + (s111 - s011) * fy * fz) * inv;
      gy = ((s010 - s000) * fx1 * fz1 + (s011 - s001) * fx1 * fz + (s110 - s100) * fx * fz1 + (s111 - s101) * fx * fz) * inv;
      gz = ((s001 - s000) * fx1 * fy1 + (s011 - s010) * fx1 * fy + (s101 - s100) * fx * fy1 + (s111 - s110) * fx * fy) * inv;
    } else {
      voxel_sdf_boundary(feat, base, sx, sy, x0k, x1k, y0k, y1k, z0k, z1k, fx, fy, fz, inv, max_dist, sdf, gx, gy, gz);
    }
  }
  if (sdf >= max_dist) {
    out.sdf = max_dist;
    return out;
  }
  out.sdf = sdf;
  V3 g = mk3(-gx, -gy, -gz);
  float l = norm(g);
  if (l > 1e-6f) out.n = (1.0f / l) * g;
  return out;
}

// ----------------------------------------------------------------------------------------------
// Obstacle set views (mirror of include/curobo_b200.h structs; kept POD so they pass by value)
// ----------------------------------------------------------------------------------------------
struct CuboidSet {
  const float *dims;
  const float *inv_pose;
  const uint8_t *enable;
  const int32_t *count;
  int32_t max_n, num_envs;
};
struct VoxelSet {
  const float *params;
  const float *inv_pose;
  const uint8_t *enable;
  const int32_t *count;
  const uint16_t *features;
  int32_t n_voxels_per_layer, max_n, num_envs;
  float max_dist;
  const uint16_t *mip;   // optional lower-bound pyramid level [num_envs*max_n][mip_stride], see voxel_sdf_grad
  int32_t mip_stride;
};

CB_HD float ldgf(const float *p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

struct ObsFrame {  // world -> obstacle transform
  V3 p;
  Q4 q;
  bool ident;  // q == (0, 0, 0, 1): the obstacle is axis-aligned with the world (the usual case for ESDF grids and tables)
};
CB_HD ObsFrame load_obs_frame(const float *inv_pose8) {
  ObsFrame f;
  f.p = mk3(ldgf(inv_pose8 + 0), ldgf(inv_pose8 + 1), ldgf(inv_pose8 + 2));
  f.q = Q4{ldgf(inv_pose8 + 4), ldgf(inv_pose8 + 5), ldgf(inv_pose8 + 6), ldgf(inv_pose8 + 3)};
  f.ident = f.q.x == 0.0f && f.q.y == 0.0f && f.q.z == 0.0f && f.q.w == 1.0f;
  return f;
}
// world point -> obstacle frame, obstacle-frame vector -> world.  With the identity rotation qrot returns its argument bit for bit
// (v * 1 + 0 + 0), so skipping it changes no result; the branch is uniform (every lane looks at the same obstacle).
CB_HD V3 to_obstacle(const ObsFrame &f, V3 pw) { return f.ident ? pw + f.p : qrot(f.q, pw) + f.p; }
CB_HD V3 from_obstacle(const ObsFrame &f, V3 v) { return f.ident ? v : qrot(qconj(f.q), v); }

// One obstacle abstraction so discrete and swept code is written once.
struct Obstacle {
  int kind;  // 0 cuboid, 1 voxel, 2 mesh
  float a, b, c;  // cuboid dims | mesh bounding-box extents
  const uint16_t *feat;
  const uint16_t *mip;
  int nx, ny, nz;
  float vs, max_dist;
  const float4 *mnodes, *mtris;  // mesh BVH (cb200_mesh.cuh)
};
struct MeshSet;
// mesh SDF through the BVH (cb200_mesh.cuh); declared here so that obstacle_sdf can dispatch to it
CB_HD SdfGrad mesh_sdf_grad(const float4 *nodes, const float4 *tris, V3 p, float max_distance, float need_below);
template <int SCENE>
CB_HD SdfGrad obstacle_sdf(const Obstacle &o, V3 p, float need_below = 3.0e38f, bool use_mip = false) {
  if ((SCENE & 4) && (SCENE == 4 || o.kind == 2)) {
    // data_mesh.py:671-677: max_distance = max(half the bounding-box diagonal, query_distance); the callers pass the query
    // distance (sphere radius + activation distance) as `need_below`
    const float half_diag = 0.5f * sqrtf(o.a * o.a + o.b * o.b + o.c * o.c);
    return mesh_sdf_grad(o.mnodes, o.mtris, p, fmaxf(half_diag, need_below), need_below);
  }
  if (SCENE == 1) return cuboid_sdf_grad(p, o.a, o.b, o.c);
  if (SCENE == 2) return voxel_sdf_grad(p, o.feat, o.nx, o.ny, o.nz, o.vs, o.max_dist, need_below, use_mip ? o.mip : nullptr);
  if (o.kind == 0) return cuboid_sdf_grad(p, o.a, o.b, o.c);
  return voxel_sdf_grad(p, o.feat, o.nx, o.ny, o.nz, o.vs, o.max_dist, need_below, use_mip ? o.mip : nullptr);
}

// Iterate every enabled obstacle of env `env` (cuboids then voxel grids) and call fn(frame, obstacle).
// SCENE is a compile-time mask (bit 0: cuboids, bit 1: voxel grids) so specialised kernels carry no dead code.
// Mesh obstacles (SCENE bit 2) come through `ms`, a pointer to a MeshSet (cb200_mesh.cuh) or null.
template <int SCENE, typename Fn, typename Meshes = MeshSet>
CB_HD void for_each_obstacle(const CuboidSet &cs, const VoxelSet &vx, int env, Fn fn, const Meshes *ms = nullptr) {
  if ((SCENE & 1) && cs.inv_pose != nullptr) {
    int ce = env < cs.num_envs ? env : 0;
    int n = cs.count[ce];
    if (n > cs.max_n) n = cs.max_n;
    #pragma unroll 1
    for (int i = 0; i < n; ++i) {
      int k = ce * cs.max_n + i;
      if (cs.enable[k] != 1) continue;
      Obstacle o;
      o.kind = 0;
      o.a = ldgf(cs.dims + 4 * k + 0);
      o.b = ldgf(cs.dims + 4 * k + 1);
      o.c = ldgf(cs.dims + 4 * k + 2);
      o.feat = nullptr;
      o.mip = nullptr;
      o.nx = o.ny = o.nz = 0;
      o.vs = 0.f;
      o.max_dist = 0.f;
      fn(load_obs_frame(cs.inv_pose + 8 * k), o);
    }
  }
  if ((SCENE & 2) && vx.inv_pose != nullptr) {
    int ve = env < vx.num_envs ? env : 0;
    int n = vx.count[ve];
    if (n > vx.max_n) n = vx.max_n;
    #pragma unroll 1
    for (int i = 0; i < n; ++i) {
      int k = ve * vx.max_n + i;
      if (vx.enable[k] != 1) continue;
      Obstacle o;
      o.kind = 1;
      o.a = o.b = o.c = 0.f;
      o.nx = (int)ldgf(vx.params + 4 * k + 0);
      o.ny = (int)ldgf(vx.params + 4 * k + 1);
      o.nz = (int)ldgf(vx.params + 4 * k + 2);
      o.vs = ldgf(vx.params + 4 * k + 3);
      o.feat = vx.features + (size_t)k * vx.n_voxels_per_layer;
      o.mip = vx.mip ? vx.mip + (size_t)k * vx.mip_stride : nullptr;
      o.max_dist = vx.max_dist;
      fn(load_obs_frame(vx.inv_pose + 8 * k), o);
    }
  }
  if constexpr ((SCENE & 4) != 0) {
    if (ms != nullptr && ms->inv_pose != nullptr) {
      int me = env < ms->num_envs ? env : 0;
      int n = ms->count[me];
      if (n > ms->max_n) n = ms->max_n;
      #pragma unroll 1
      for (int i = 0; i < n; ++i) {
        int k = me * ms->max_n + i;
        if (ms->enable[k] != 1) continue;
        Obstacle o;
        o.kind = 2;
        o.a = ldgf(ms->dims + 4 * k + 0);
        o.b = ldgf(ms->dims + 4 * k + 1);
        o.c = ldgf(ms->dims + 4 * k + 2);
        o.feat = nullptr;
        o.mip = nullptr;
        o.nx = o.ny = o.nz = 0;
        o.vs = 0.f;
        o.max_dist = 0.f;
        o.mnodes = ms->nodes + 2 * (size_t)ms->node_off[k];
        o.mtris = ms->tris + 8 * (size_t)ms->tri_off[k];
        fn(load_obs_frame(ms->inv_pose + 8 * k), o);
      }
    }
  }
}

// Discrete sphere-vs-scene: returns weighted cost, adds weighted world-frame gradient to g.
// (wp_collision_kernel.py:112-166)
template <int SCENE = 3, typename Meshes = MeshSet>
CB_HD float sphere_scene_discrete(V3 c, float r, float eta, float w, const CuboidSet &cs, const VoxelSet &vx, int env,
                                  V3 &g, const Meshes *ms = nullptr) {
  float cost = 0.0f;
  if (r < 0.0f) return 0.0f;
  const float radj = r + eta;
  for_each_obstacle<SCENE>(cs, vx, env, [&](const ObsFrame &f, const Obstacle &o) {
    V3 lp = to_obstacle(f, c);
    SdfGrad sg = obstacle_sdf<SCENE>(o, lp, radj, true);
    float pen = radj - sg.sdf;
    if (pen > 0.0f) {
      float ac, as;
      collision_activation(pen, eta, ac, as);
      V3 gw = from_obstacle(f, sg.n);
      cost += w * ac;
      g = g + (w * as) * gw;
    }
  }, ms);
  return cost;
}

// Swept sphere-vs-scene (wp_sweep_collision_kernel.py:137-260).  prev/next are the same sphere at
// h-1 / h+1 (has_prev / has_next false at the trajectory ends).
template <int SCENE = 3, typename Meshes = MeshSet>
CB_HD float sphere_scene_swept(V3 c, float r, float eta, float w, bool has_prev, V3 prev, bool has_next, V3 next,
                               const CuboidSet &cs, const VoxelSet &vx, int env, V3 &g, const Meshes *ms = nullptr) {
  float cost = 0.0f;
  if (r < 0.0f) return 0.0f;
  const float radj = r + eta;
  for_each_obstacle<SCENE>(cs, vx, env, [&](const ObsFrame &f, const Obstacle &o) {
    V3 lc = to_obstacle(f, c);
    float csum = 0.0f;
    V3 gsum = mk3(0.f, 0.f, 0.f);
    {
      SdfGrad sg = obstacle_sdf<SCENE>(o, lc, radj);
      float pen = radj - sg.sdf;
      if (pen > 0.0f) {
        float ac, as;
        collision_activation(pen, eta, ac, as);
        csum += ac;
        gsum = gsum + as * sg.n;
      }
    }
#pragma unroll 1
    for (int dir = 0; dir < 2; ++dir) {
      if (!(dir == 0 ? has_prev : has_next)) continue;
      V3 ln = to_obstacle(f, dir == 0 ? prev : next);
      float half = norm(ln - lc) * 0.5f;
      float inv_half = 1.0f / fmaxf(half, 0.001f);
      float jump = 0.0f;
#pragma unroll 1
      for (int it = 0; it < 3; ++it) {
        if (jump >= half) break;
        float t = 1.0f - 0.5f * jump * inv_half;
        V3 pt = t * lc + (1.0f - t) * ln;
        SdfGrad sg = obstacle_sdf<SCENE>(o, pt, radj);
        float pen = radj - sg.sdf;
        if (pen > 0.0f) {
          float ac, as;
          collision_activation(pen, eta, ac, as);
          csum += ac;
          gsum = gsum + as * sg.n;
          jump += pen;
        } else {
          jump += (-pen >= 1000.0f) ? radj : fmaxf(-pen, radj);
        }
      }
    }
    if (csum > 0.0f) {
      cost += w * csum;
      g = g + w * from_obstacle(f, gsum);
    }
  }, ms);
  return cost;
}

// Speed metric post-process of one sphere's summed (cost, grad) (wp_speed_metric.py:36-93).
CB_HD void speed_metric(V3 prev, V3 cur, V3 next, float dt, float &d, V3 &g) {
  if (dt < 1e-6f) dt = 1e-6f;
  V3 vel = (0.5f / dt) * (next - prev);
  float sv = norm(vel);
  if (sv < 1e-3f) return;
  if (d <= 0.0f) return;
  V3 acc = (1.0f / (dt * dt)) * (prev + next - 2.0f * cur);
  V3 nv = (1.0f / sv) * vel;
  V3 curv = (1.0f / (sv * sv)) * acc;
  V3 og = g - dot(nv, g) * nv;
  V3 oc = curv - dot(nv, curv) * nv;
  g = sv * (og - d * oc);
  d = sv * d;
}

// ----------------------------------------------------------------------------------------------
// Tool-pose cost for one tool frame (project_distance_to_goal = 0)
// ----------------------------------------------------------------------------------------------
struct PoseOut {
  float pos_cost, rot_cost, pos_err, rot_err;
  V3 g_pos;
  float gq_w, gq_x, gq_y, gq_z;  // quaternion-rate gradient, wxyz
  int goal_idx;
};

CB_HD PoseOut tool_pose_cost(V3 cp, Q4 cq /*xyzw*/, const float *goal_pos /*[n_goalset,3]*/,
                             const float *goal_quat /*[n_goalset,4] wxyz*/, int n_goalset, float w_pos, float w_rot,
                             const float *axes_base /*[L,6] or null*/, int frame, float tol_p, float tol_r,
                             int method) {
  float ax[6] = {1.f, 1.f, 1.f, 1.f, 1.f, 1.f};
  if (axes_base != nullptr) {  // NB: test the BASE pointer; never form (null + offset)
    for (int i = 0; i < 6; ++i) ax[i] = ldgf(axes_base + 6 * frame + i);
  }
  tol_p = tol_p * tol_p;
  tol_r = tol_r * tol_r;
  float best = -1.0f;
  PoseOut o;
  o.pos_cost = o.rot_cost = -1.0f;
  o.g_pos = mk3(0, 0, 0);
  V3 best_rg = mk3(0, 0, 0);
  o.goal_idx = 0;
  o.rot_err = -1.0f;
  #pragma unroll 1
  for (int g = 0; g < n_goalset; ++g) {
    V3 gp = mk3(ldgf(goal_pos + 3 * g), ldgf(goal_pos + 3 * g + 1), ldgf(goal_pos + 3 * g + 2));
    Q4 gq = Q4{ldgf(goal_quat + 4 * g + 1), ldgf(goal_quat + 4 * g + 2), ldgf(goal_quat + 4 * g + 3), ldgf(goal_quat + 4 * g)};
    V3 d = cp - gp;
    V3 wd = mk3(d.x * ax[0], d.y * ax[1], d.z * ax[2]);
    float pd = 0.5f * w_pos * dot(wd, wd);
    V3 pg = mk3(w_pos * ax[0] * ax[0] * d.x, w_pos * ax[1] * ax[1] * d.y, w_pos * ax[2] * ax[2] * d.z);
    if (pd < tol_p) {
      pd = 0.0f;
      pg = mk3(0, 0, 0);
    }
    Q4 qd = qmul(cq, qconj(gq));
    float rd, ang;
    V3 rg = mk3(0, 0, 0);
    if (method == 0) {
      V3 v = mk3(ax[3] * qd.x, ax[4] * qd.y, ax[5] * qd.z);
      float vl = norm(v);
      ang = 2.0f * atan2f(vl, fabsf(qd.w));
      if (w_rot == 0.0f) ang = 0.0f;
      V3 axis = (vl < 1e-15f) ? mk3(0, 0, 0) : (1.0f / vl) * v;
      V3 om = ang * axis;
      rd = w_rot * dot(om, om);
      if (rd < tol_r) {
        rd = 0.0f;
      } else {
        float sf = (qd.w < 0.0f) ? -2.0f : 2.0f;
        rg = (sf * w_rot) * om;
      }
    } else {
      if (qd.w < 0.0f) qd = Q4{-qd.x, -qd.y, -qd.z, -qd.w};
      V3 v = mk3(qd.x, qd.y, qd.z);
      float vn = norm(v);
      float ha = atan2f(vn, fabsf(qd.w));
      if (w_rot == 0.0f) ha = 0.0f;
      float ga = 2.0f * ha;
      V3 tv;
      if (vn < 1e-10f) {
        tv = 2.0f * v;
      } else if (fabsf(ha) < 1e-15f) {
        tv = (2.0f * (1.0f + vn * vn / (6.0f * qd.w * qd.w))) * v;
      } else {
        tv = (ga / (2.0f * sinf(ha))) * v;
      }
      V3 wt = mk3(ax[3] * tv.x, ax[4] * tv.y, ax[5] * tv.z);
      ang = norm(wt);
      rd = w_rot * dot(wt, wt);
      if (rd < tol_r) {
        rd = 0.0f;
      } else {
        rg = (2.0f * w_rot) * wt;
      }
    }
    float tot = pd + rd;
    if (best < 0.0f || tot < best) {
      best = tot;
      o.goal_idx = g;
      o.pos_cost = pd;
      o.rot_cost = rd;
      o.g_pos = pg;
      best_rg = rg;
      o.rot_err = ang;
    }
  }
  o.pos_err = (w_pos > 0.0f) ? sqrtf(2.0f * o.pos_cost / w_pos) : 0.0f;
  Q4 rate = qmul(cq, Q4{best_rg.x, best_rg.y, best_rg.z, 0.0f});
  o.gq_w = rate.w;
  o.gq_x = rate.x;
  o.gq_y = rate.y;
  o.gq_z = rate.z;
  return o;
}

// ----------------------------------------------------------------------------------------------
// C-space costs (per dof)
// ----------------------------------------------------------------------------------------------
CB_HD void bound_cost(float x, float lo, float hi, float act, float w, float &cost, float &grad) {
  float range = hi - lo;
  lo = lo + act * range;
  hi = hi - act * range;
  float d;
  if (x < lo)
    d = x - lo;
  else if (x > hi)
    d = x - hi;
  else
    return;
  float wv = w * d;
  cost += 0.5f * wv * d;
  grad += wv;
}
CB_HD void l2_reg(float v, float w, float &cost, float &grad) {
  float wv = w * v;
  cost += 0.5f * wv * v;
  grad += wv;
}

// ----------------------------------------------------------------------------------------------
// Broad-phase bound of a collision link: the blob packer (host) and cb200_refresh_robot_spheres (device) both call
// bounding_ball, so a refreshed blob holds the bytes a fresh pack would.
// ----------------------------------------------------------------------------------------------
// fp64 spelled, on the device, with round-to-nearest operations: nvcc cannot contract them into FMAs, so the device rounds every
// step exactly as the host code (x86-64 without FMA, also the host emulation of the kernels) does.
#ifdef __CUDA_ARCH__
CB_HD double bb_add(double a, double b) { return __dadd_rn(a, b); }
CB_HD double bb_sub(double a, double b) { return __dsub_rn(a, b); }
CB_HD double bb_mul(double a, double b) { return __dmul_rn(a, b); }
CB_HD double bb_div(double a, double b) { return __ddiv_rn(a, b); }
CB_HD double bb_sqrt(double a) { return __dsqrt_rn(a); }
#else
CB_HD double bb_add(double a, double b) { return a + b; }
CB_HD double bb_sub(double a, double b) { return a - b; }
CB_HD double bb_mul(double a, double b) { return a * b; }
CB_HD double bb_div(double a, double b) { return a / b; }
CB_HD double bb_sqrt(double a) { return sqrt(a); }
#endif

// Ball j of the slots (configuration j / m, sphere s_begin + j % m) of link_spheres [n_cfg, S, 4]: centre and radius
// (+ padding[s] when padding is given); false when the radius is negative (a disabled sphere).
CB_HD bool bb_ball(const float *link_spheres, const float *padding, int s_begin, int m, int S, int j, double *b) {
  const int cfg = j / m, s = s_begin + (j - cfg * m);
  const float *p = link_spheres + ((size_t)cfg * S + s) * 4;
  b[3] = bb_add((double)p[3], padding ? (double)padding[s] : 0.0);
  b[0] = p[0];
  b[1] = p[1];
  b[2] = p[2];
  return !(b[3] < 0);
}

// The ball farthest from c (max |p - c| + r; the lowest slot among equals) over the slots lane, lane + nlanes, ...;
// `reduce(best, arg)` combines the lanes' candidates (nothing to combine for one lane).
struct SerialFarthest {
  CB_HD void operator()(double &, int &) const {}
};
template <class Reduce>
CB_HD double bb_farthest(const float *ls, const float *padding, int s_begin, int m, int S, int n_slots, const double *c, int lane,
                         int nlanes, const Reduce &reduce, int &arg) {
  double best = -1, b[4];
  arg = -1;
  for (int j = lane; j < n_slots; j += nlanes) {
    if (!bb_ball(ls, padding, s_begin, m, S, j, b)) continue;
    const double dx = bb_sub(b[0], c[0]), dy = bb_sub(b[1], c[1]), dz = bb_sub(b[2], c[2]);
    const double d = bb_add(bb_sqrt(bb_add(bb_add(bb_mul(dx, dx), bb_mul(dy, dy)), bb_mul(dz, dz))), b[3]);
    if (d > best) {
      best = d;
      arg = j;
    }
  }
  reduce(best, arg);
  return best;
}

// Near-minimal ball enclosing the balls (p_s, r_s [+ padding_s]) with radius >= 0 of spheres [s_begin, s_end) of every
// configuration of link_spheres [n_cfg, S, 4]: Badoiu-Clarkson iterations from the centroid (move the centre 1/(k+1) of the way
// towards the farthest ball), then R = max(|p - c| + r) exactly for the final centre, inflated against fp32 rounding of the world
// transform.  out = (cx, cy, cz, R), written by lane 0; R = -1 when no sphere is enabled.  A tighter ball only prunes more; it is
// never unsafe.  Lanes 0..nlanes-1 share the farthest-ball scans through `reduce` and compute everything else redundantly.
template <class Reduce = SerialFarthest>
CB_HD void bounding_ball(const float *link_spheres, const float *padding, int s_begin, int s_end, int n_cfg, int S, float *out,
                         int lane = 0, int nlanes = 1, const Reduce &reduce = Reduce()) {
  const int m = s_end - s_begin, n_slots = (n_cfg < 1 ? 1 : n_cfg) * m;
  double c[3] = {0, 0, 0}, b[4];
  int n = 0;
  for (int j = 0; j < n_slots; ++j) {
    if (!bb_ball(link_spheres, padding, s_begin, m, S, j, b)) continue;
    c[0] = bb_add(c[0], b[0]);
    c[1] = bb_add(c[1], b[1]);
    c[2] = bb_add(c[2], b[2]);
    ++n;
  }
  if (n == 0) {
    if (lane == 0) {
      out[0] = out[1] = out[2] = 0.0f;
      out[3] = -1.0f;
    }
    return;
  }
  for (int k = 0; k < 3; ++k) c[k] = bb_div(c[k], (double)n);
  int arg;
  double best_R = bb_farthest(link_spheres, padding, s_begin, m, S, n_slots, c, lane, nlanes, reduce, arg);
  double best_c[3] = {c[0], c[1], c[2]};
  for (int it = 1; it <= 200; ++it) {
    const double R = bb_farthest(link_spheres, padding, s_begin, m, S, n_slots, c, lane, nlanes, reduce, arg);
    if (R < best_R) {
      best_R = R;
      for (int k = 0; k < 3; ++k) best_c[k] = c[k];
    }
    // step towards the farthest ball's centre, 1/(it+1) of the current radius, never past the centre
    bb_ball(link_spheres, padding, s_begin, m, S, arg, b);
    const double dx = bb_sub(b[0], c[0]), dy = bb_sub(b[1], c[1]), dz = bb_sub(b[2], c[2]);
    const double d = bb_sqrt(bb_add(bb_add(bb_mul(dx, dx), bb_mul(dy, dy)), bb_mul(dz, dz)));
    if (d < 1e-12) break;
    const double step = bb_div(R, bb_add((double)it, 1.0));
    const double mv = bb_div(d < step ? d : step, d);
    c[0] = bb_add(c[0], bb_mul(dx, mv));
    c[1] = bb_add(c[1], bb_mul(dy, mv));
    c[2] = bb_add(c[2], bb_mul(dz, mv));
  }
  const double Rf = bb_farthest(link_spheres, padding, s_begin, m, S, n_slots, best_c, lane, nlanes, reduce, arg);
  const float o[3] = {(float)best_c[0], (float)best_c[1], (float)best_c[2]};
  // centre was rounded to fp32: re-measure from the rounded centre
  const double cr[3] = {(double)o[0], (double)o[1], (double)o[2]};
  const double Rr = bb_farthest(link_spheres, padding, s_begin, m, S, n_slots, cr, lane, nlanes, reduce, arg);
  if (lane == 0) {
    out[0] = o[0];
    out[1] = o[1];
    out[2] = o[2];
    out[3] = (float)bb_add(bb_mul(Rf < Rr ? Rr : Rf, 1.0 + 1e-4), 1e-5);
  }
}

}  // namespace cb200
