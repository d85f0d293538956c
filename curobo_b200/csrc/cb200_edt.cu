// cb200_edt.cu -- exact 3-D nearest-site transform kernels (SURVEY.md 8f rank 4), C ABI.
//
// Replaces the reference's five PBA+ launches + final copy (backends/cuda_core_backend/pba.py:60-124) with three in-place
// passes and no transposes: z is the contiguous axis of the [nx, ny, nz] grid, so
//   pass 1  floods along z      a WARP per row: 32 consecutive voxels per step, the nearest site on either side found with
//                               one ballot + bit scan + shuffle per 32 voxels (no serial walk, fully coalesced),
//   pass 2  envelopes along y   32 columns adjacent in z per CTA: every row of the shared-memory tile is one 128-byte line,
//   pass 3  envelopes along x   columns adjacent in (y, z): same.
// The envelope passes run the BANDED schedule of cb200_edt.cuh: a CTA of 8 warps owns a tile of 32 columns, thread
// (band, column) builds the hull of its band's rows, one thread per column joins the band hulls by their common tangents,
// thread (band, column) fills its band's rows.  Round 1 ran one thread per column (0.18 + 0.18 + 0.35 ms at 256^3, 6 warps
// resident per SM: 9 % of the HBM bound).  The only HBM traffic is one coalesced read and one coalesced write of the grid per
// pass: 3 x 8 B per voxel (the reference moves 6 x 8 B plus its stack look-ups).  Every pass is in place (a tile is fully
// staged before its first row is written back), so the scratch `buffer` of the reference interface is not touched.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/curobo_b200.h"
#include "cb200_launch.h"
#include "cb200_edt.cuh"
#include "cb200_math.cuh"

namespace {
using namespace cb200::edt;
using cb200::capped_grid;
using cb200::launch_status;
using cb200::opt_in_smem;
using cb200::ret;

// pass 1.  A warp per z-row; CHUNKS x 32 >= nz.  v[c] = the row's voxels c * 32 + lane.  Forward: the last site at or
// before a voxel = highest set bit of the chunk's site ballot at or below the lane (else the carry of the earlier chunks);
// backward: the first site at or after it = lowest set bit at or above the lane (else the carry of the later chunks).  The
// nearer of the two wins, ties go to the later site (flood_column's rule, i.e. the reference's backward sweep).
template <int CHUNKS>
__device__ __forceinline__ void flood_row_load(const int *p, int nz, int lane, int (&v)[CHUNKS]) {
#pragma unroll
  for (int c = 0; c < CHUNKS; ++c) {
    const int i = c * 32 + lane;
    v[c] = (c * 32 < nz && i < nz) ? p[i] : -1;
  }
}
template <int CHUNKS>
__device__ __forceinline__ void flood_row_solve(int *p, int nz, int lane, const int (&v)[CHUNKS]) {
  int f[CHUNKS];
  int carry = kEmpty;
#pragma unroll
  for (int c = 0; c < CHUNKS; ++c) {
    const unsigned m = __ballot_sync(0xffffffffu, v[c] >= 0);
    const unsigned below = m & (0xffffffffu >> (31 - lane));
    const int src = below ? 31 - __clz((int)below) : 0;
    const int got = __shfl_sync(0xffffffffu, v[c], src);
    f[c] = below ? got : carry;
    if (m) carry = __shfl_sync(0xffffffffu, v[c], 31 - __clz((int)m));
  }
  carry = kEmpty;
#pragma unroll
  for (int c = CHUNKS - 1; c >= 0; --c) {
    const int i = c * 32 + lane;
    const unsigned m = __ballot_sync(0xffffffffu, v[c] >= 0);
    const unsigned above = m >> lane;
    const int src = above ? lane + __ffs((int)above) - 1 : 0;
    const int got = __shfl_sync(0xffffffffu, v[c], src);
    const int nb = above ? got : carry;
    if (m) carry = __shfl_sync(0xffffffffu, v[c], __ffs((int)m) - 1);
    if (c * 32 < nz && i < nz) {
      const int fw = f[c];
      const int db = nb < 0 ? 0x7fffffff : (coord<2>(nb) > i ? coord<2>(nb) - i : i - coord<2>(nb));
      const int df = fw < 0 ? 0x7fffffff : (coord<2>(fw) > i ? coord<2>(fw) - i : i - coord<2>(fw));
      const int r = df < db ? fw : nb;
      p[i] = r < 0 ? kEmpty : r;
    }
  }
}
// A warp takes TWO rows per step (both rows' loads in flight before either is solved): the pass is a pure stream, and the loads
// in flight per SM are what bound it.
template <int CHUNKS>
__global__ void __launch_bounds__(256) edt_flood_z_kernel(int *__restrict__ grid, int nz, long long nrows) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long row = 2 * warp0; row < nrows; row += 2 * nwarps) {
    int *p0 = grid + row * nz;
    const bool two = row + 1 < nrows;  // warp-uniform
    int *p1 = two ? p0 + nz : p0;
    int v0[CHUNKS], v1[CHUNKS];
    flood_row_load<CHUNKS>(p0, nz, lane, v0);
    if (two) flood_row_load<CHUNKS>(p1, nz, lane, v1);
    flood_row_solve<CHUNKS>(p0, nz, lane, v0);
    if (two) flood_row_solve<CHUNKS>(p1, nz, lane, v1);
  }
}

// passes 2 and 3: the banded schedule (cb200_edt.cuh).  The per-thread work of every phase is a member of BandedEnvelope --
// the host emulation (tests/hostmath) executes the same members thread by thread between the same barriers.
template <int AXIS>
__global__ void __launch_bounds__(kBands *kLanes) edt_envelope_kernel(const __grid_constant__ BandedEnvelope<AXIS> pass) {
  CB200_EXTERN_SHARED int tile[];
  const int lane = threadIdx.x & 31, band = threadIdx.x >> 5;
  const long long ntiles = pass.e.ntiles();
  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
    pass.phase_load_and_hull(tile, t, band, lane);
    __syncthreads();
    pass.phase_join(tile, t, band, lane);
    __syncthreads();
    pass.phase_fill(tile, t, band, lane);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) edt_distance_kernel(const int *__restrict__ sites, __half *__restrict__ out, int ny, int nz,
                                                            long long total, float voxel_size, float empty_value) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = sites[i];
    const int z = (int)(i % nz), y = (int)((i / nz) % ny), x = (int)(i / ((long long)nz * ny));
    const float d = v < 0 ? empty_value : sqrtf((float)site_distance_sq(v, x, y, z)) * voxel_size;
    out[i] = __float2half_rn(d);
  }
}

// The stages either side of the transform for a DENSE signed-distance source at the ESDF's own resolution (the reference reads
// its block-sparse TSDF through a hash table at the same places: builder_esdf.py:193-404 seeding, :410-503 distance + sign).
// sdf > 1e9 = unobserved.
__global__ void __launch_bounds__(256) esdf_seed_sites_kernel(const float *__restrict__ sdf, int *__restrict__ sites, int ny, int nz,
                                                               long long total, float voxel_size, float truncation) {
  const float surface = voxel_size * 0.9f, trunc_edge = -(truncation - voxel_size * 1.1f);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const float d = sdf[i];
    int out = -1;
    if (!(d > 1e9f) && (fabsf(d) <= surface || d < trunc_edge)) {  // surface voxel or truncation boundary (builder_esdf.py:255-261)
      const int z = (int)(i % nz), y = (int)((i / nz) % ny), x = (int)(i / ((long long)nz * ny));
      out = pack(x, y, z);
    }
    sites[i] = out;
  }
}

// The reference's DEFAULT seeding (mapper_cfg.py:103 seeding_method = "gather"; seed_esdf_sites_gather_kernel, builder_esdf.py:
// 308-404 with _check_seed_at_world_pos :267-306): an ESDF voxel is a site when the seed rule holds in the TSDF voxel that
// contains its centre OR one of the six points half an ESDF voxel away along the axes.  For the dense case (ESDF grid == TSDF grid)
// the probes land on the voxel itself and on neighbours -- which ones is decided by float32 rounding of
// int((world - origin) / voxel + n / 2), so the arithmetic is spelled with IEEE intrinsics in the reference's order (no FMA
// contraction, no approximate division): the dilated band is then the reference's band, voxel for voxel.
__device__ __forceinline__ bool seed_rule_at_world(const float *__restrict__ sdf, int nx, int ny, int nz, float wx, float wy, float wz,
                                                   float ox, float oy, float oz, float voxel_size, float surface, float trunc_edge) {
  const int gx = (int)__fadd_rn(__fdiv_rn(__fsub_rn(wx, ox), voxel_size), __fmul_rn((float)nx, 0.5f));
  const int gy = (int)__fadd_rn(__fdiv_rn(__fsub_rn(wy, oy), voxel_size), __fmul_rn((float)ny, 0.5f));
  const int gz = (int)__fadd_rn(__fdiv_rn(__fsub_rn(wz, oz), voxel_size), __fmul_rn((float)nz, 0.5f));
  if (gx < 0 || gx >= nx || gy < 0 || gy >= ny || gz < 0 || gz >= nz) return false;
  const float d = sdf[((long long)gx * ny + gy) * nz + gz];
  if (d > 1e9f) return false;
  return fabsf(d) <= surface || d < trunc_edge;
}
__global__ void __launch_bounds__(256) esdf_seed_sites_gather_kernel(const float *__restrict__ sdf, int *__restrict__ sites, int nx,
                                                                      int ny, int nz, long long total, float voxel_size,
                                                                      float truncation, float ox, float oy, float oz) {
  const float surface = __fmul_rn(voxel_size, 0.9f), trunc_edge = -__fsub_rn(truncation, __fmul_rn(voxel_size, 1.1f));
  const float half = __fmul_rn(voxel_size, 0.5f);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(i % nz), y = (int)((i / nz) % ny), x = (int)(i / ((long long)nz * ny));
    // centre = origin + (idx + 0.5 - n * 0.5) * voxel, in that order (builder_esdf.py:333-335)
    const float cx = __fadd_rn(ox, __fmul_rn(__fsub_rn(__fadd_rn((float)x, 0.5f), __fmul_rn((float)nx, 0.5f)), voxel_size));
    const float cy = __fadd_rn(oy, __fmul_rn(__fsub_rn(__fadd_rn((float)y, 0.5f), __fmul_rn((float)ny, 0.5f)), voxel_size));
    const float cz = __fadd_rn(oz, __fmul_rn(__fsub_rn(__fadd_rn((float)z, 0.5f), __fmul_rn((float)nz, 0.5f)), voxel_size));
    const bool hit = seed_rule_at_world(sdf, nx, ny, nz, cx, cy, cz, ox, oy, oz, voxel_size, surface, trunc_edge) ||
                     seed_rule_at_world(sdf, nx, ny, nz, __fadd_rn(cx, half), cy, cz, ox, oy, oz, voxel_size, surface, trunc_edge) ||
                     seed_rule_at_world(sdf, nx, ny, nz, __fsub_rn(cx, half), cy, cz, ox, oy, oz, voxel_size, surface, trunc_edge) ||
                     seed_rule_at_world(sdf, nx, ny, nz, cx, __fadd_rn(cy, half), cz, ox, oy, oz, voxel_size, surface, trunc_edge) ||
                     seed_rule_at_world(sdf, nx, ny, nz, cx, __fsub_rn(cy, half), cz, ox, oy, oz, voxel_size, surface, trunc_edge) ||
                     seed_rule_at_world(sdf, nx, ny, nz, cx, cy, __fadd_rn(cz, half), ox, oy, oz, voxel_size, surface, trunc_edge) ||
                     seed_rule_at_world(sdf, nx, ny, nz, cx, cy, __fsub_rn(cz, half), ox, oy, oz, voxel_size, surface, trunc_edge);
    sites[i] = hit ? pack(x, y, z) : -1;
  }
}

__device__ __forceinline__ float round_half_away(float v) { return v < 0.0f ? -floorf(0.5f - v) : floorf(v + 0.5f); }

__global__ void __launch_bounds__(256) esdf_signed_distance_kernel(const int *__restrict__ sites, const float *__restrict__ static_sdf,
                                                                    const float *__restrict__ combined_sdf, __half *__restrict__ out,
                                                                    int nx, int ny, int nz, long long total, float voxel_size,
                                                                    float skip_steps) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = sites[i];
    if (v < 0) {
      out[i] = __float2half_rn(1e4f);
      continue;
    }
    const int z = (int)(i % nz), y = (int)((i / nz) % ny), x = (int)(i / ((long long)nz * ny));
    const int sx = coord<0>(v), sy = coord<1>(v), sz = coord<2>(v);
    const float dx = (float)(x - sx), dy = (float)(y - sy), dz = (float)(z - sz);
    const float dist_voxels = sqrtf(dx * dx + dy * dy + dz * dz);
    float edt = dist_voxels * voxel_size;
    float sgn_src = 1e10f;
    if (dist_voxels > 1.0f && skip_steps > 0.0f && static_sdf != nullptr) {  // the voxel next to the site, towards the query
      const float inv = 1.0f / dist_voxels;
      const int ax = sx + (int)round_half_away(dx * inv * skip_steps), ay = sy + (int)round_half_away(dy * inv * skip_steps),
                az = sz + (int)round_half_away(dz * inv * skip_steps);
      if (ax >= 0 && ax < nx && ay >= 0 && ay < ny && az >= 0 && az < nz) sgn_src = static_sdf[((long long)ax * ny + ay) * nz + az];
    }
    if (sgn_src > 1e9f && combined_sdf != nullptr) sgn_src = combined_sdf[i];
    if (!(sgn_src > 1e9f) && sgn_src < 0.0f) edt = -edt;
    out[i] = __float2half_rn(edt);
  }
}

// Depth -> TSDF for a DENSE grid at the ESDF's resolution: the voxel-centric projective update of the reference's camera
// integrator (perception/mapper/kernel/builder/builder_camera_integrate.py:399-489, integrate_voxels_kernel) with the dense
// index in place of (block pool index, local index); the block discovery / allocation phases 1-3 of the block-sparse store (hash
// table) are out of scope.  block_data[i] = (sum of sdf * weight, sum of weight) as two fp16, accumulated in fp32 and rounded
// once per call, as the reference does.  Voxel centre = (idx + 0.5 - n / 2) * voxel_size + origin (builder_coord.py:57-66).
struct TsdfCameras {
  const float *intrinsics;  // [C, 3, 3]
  const float *position;    // [C, 3]
  const float *quaternion;  // [C, 4] wxyz, camera -> world
  const float *depth;       // [C, H, W] metres
  int num, height, width;
};
__global__ void __launch_bounds__(256) tsdf_integrate_depth_kernel(__half *__restrict__ block_data, int nx, int ny, int nz,
                                                                    long long total, float voxel_size, float ox, float oy, float oz,
                                                                    TsdfCameras cams, float depth_min, float depth_max,
                                                                    float truncation) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(i % nz), y = (int)((i / nz) % ny), x = (int)(i / ((long long)nz * ny));
    const float wx = ((float)x + 0.5f - (float)nx * 0.5f) * voxel_size + ox, wy = ((float)y + 0.5f - (float)ny * 0.5f) * voxel_size + oy,
                wz = ((float)z + 0.5f - (float)nz * 0.5f) * voxel_size + oz;
    float total_sw = 0.0f, total_w = 0.0f;
    for (int c = 0; c < cams.num; ++c) {
      const float *cp = cams.position + 3 * c, *cq = cams.quaternion + 4 * c, *K = cams.intrinsics + 9 * c;
      // wp.quat_rotate(quat_inverse(q), v): v (2 w^2 - 1) + 2 w (qv x v) + 2 qv (qv . v) with qv = -(x, y, z)
      const float qx = -cq[1], qy = -cq[2], qz = -cq[3], qw = cq[0];
      const float vx = wx - cp[0], vy = wy - cp[1], vz = wz - cp[2];
      const float cc = 2.0f * qw * qw - 1.0f;
      const float crx = qy * vz - qz * vy, cry = qz * vx - qx * vz, crz = qx * vy - qy * vx;
      const float d = qx * vx + qy * vy + qz * vz;
      const float xc = vx * cc + crx * qw * 2.0f + qx * d * 2.0f, yc = vy * cc + cry * qw * 2.0f + qy * d * 2.0f,
                  zc = vz * cc + crz * qw * 2.0f + qz * d * 2.0f;
      if (!(zc > depth_min)) continue;
      const float fx = K[0], fy = K[4], cx = K[2], cy = K[5];
      // (IEEE divisions: the library is built with approximate division, and the pixel index must not depend on it)
      const float u = __fdiv_rn(fx * xc, zc) + cx, v = __fdiv_rn(fy * yc, zc) + cy;
      const int px = (int)u, py = (int)v;  // truncation towards zero, as wp.int32(float)
      if (px < 0 || px >= cams.width || py < 0 || py >= cams.height) continue;
      const float depth = cams.depth[((long long)c * cams.height + py) * cams.width + px];
      if (!(depth >= depth_min && depth <= depth_max)) continue;
      const float sdf = depth - zc;
      if (!(sdf >= -truncation)) continue;
      const float sdf_clamped = fminf(sdf, truncation);
      const float coverage = __fdiv_rn(fx * voxel_size, zc) * __fdiv_rn(fy * voxel_size, zc);
      const float weight = fmaxf(coverage, 1.0f);  // compute_tsdf_weight == 1 (wp_integrate_common.py:57-105)
      total_sw += sdf_clamped * weight;
      total_w += weight;
    }
    if (total_w > 0.0f) {
      const float old_sw = __half2float(block_data[2 * i]), old_w = __half2float(block_data[2 * i + 1]);
      block_data[2 * i] = __float2half_rn(old_sw + total_sw);
      block_data[2 * i + 1] = __float2half_rn(old_w + total_w);
    }
  }
}

// Robot pixels of depth images, masked before the images reach the integrator above: the reference's RobotSegmenter
// (perception/robot_segmenter.py:35-366, rays of geom/cv.py:47-157) without its [pixels x spheres] distance matrix.  One CTA per
// 32 x 8 pixel tile of one image, warp = tile row (one 128-byte line of depth / filtered):
//   1. every thread deprojects its pixel and moves it into the robot frame; a block reduction gives the box of the tile's
//      candidate points (depth > 0 and finite),
//   2. the CTA keeps the image's spheres whose distance to that box is under r + threshold, compacted into shared memory,
//   3. every candidate pixel scans the kept spheres and stops at the first hit.
// A tile without a candidate skips 2 and 3.  The cull is exact: box and pixel distances round the same way (seg_dist2), and for a
// point inside the box every per-axis box gap is at most the point's rounded offset (rounding is monotone), so a sphere a pixel
// hits is never culled.
constexpr int kSegTileW = 32, kSegTileH = 8, kSegThreads = kSegTileW * kSegTileH, kSegWarps = kSegThreads / 32;
struct SegmentArgs {
  const float *depth;       // [B, H, W] metres
  const float *intrinsics;  // [B, 3, 3]
  const float *position;    // [B, 3]
  const float *quaternion;  // [B, 4] wxyz, camera -> robot base
  const float *spheres;     // [1 or B, S, 4]
  uint8_t *mask;            // [B, H, W]
  float *filtered;          // [B, H, W]
  int height, width, tiles_x, tiles_per_image;
  int sphere_stride;        // floats between two images' spheres: 0 when one robot state serves every image
  int num_spheres;
  float threshold;
};
// |d|^2 in round-to-nearest steps that the compiler cannot contract, so that the cull and the pixel test round alike
__device__ __forceinline__ float seg_dist2(float dx, float dy, float dz) {
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}
__global__ void __launch_bounds__(kSegThreads) segment_robot_depth_kernel(const SegmentArgs a) {
  using namespace cb200;
  CB200_EXTERN_SHARED __align__(16) float smem[];  // kept spheres: (centre, (r + threshold)^2)
  __shared__ float warp_box[kSegWarps][7];         // lo xyz, hi xyz, any candidate
  __shared__ int kept;
  float4 *survivors = reinterpret_cast<float4 *>(smem);
  const unsigned full = 0xffffffffu;
  const float inf = __int_as_float(0x7f800000);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int img = blockIdx.x / a.tiles_per_image, tile = blockIdx.x - img * a.tiles_per_image;
  const int tile_y = tile / a.tiles_x;
  const int u = (tile - tile_y * a.tiles_x) * kSegTileW + lane, v = tile_y * kSegTileH + warp;
  const bool inside = u < a.width && v < a.height;
  const long long pix = ((long long)img * a.height + v) * a.width + u;
  const float d = inside ? a.depth[pix] : 0.0f;
  // the reference masks depth > 0 only; an infinite depth puts the point at infinity and NaN fails every comparison, so
  // neither is ever masked there.  Tested on the bits: the library flushes subnormals to zero, and `d > 0.0f` would drop a
  // subnormal positive depth that the reference can mask.
  const int dbits = __float_as_int(d);
  const bool cand = dbits > 0 && dbits < 0x7f800000;
  V3 p = mk3(0.0f, 0.0f, 0.0f);
  if (cand) {
    const float *K = a.intrinsics + 9 * img, *cp = a.position + 3 * img, *cq = a.quaternion + 4 * img;
    // ray ((u - cx) / fx, (v - cy) / fy, 1) times the depth (get_projection_rays, project_depth_using_rays); IEEE divisions,
    // as in tsdf_integrate_depth_kernel
    const V3 pc = mk3(__fmul_rn(__fdiv_rn(__fsub_rn((float)u, K[2]), K[0]), d), __fmul_rn(__fdiv_rn(__fsub_rn((float)v, K[5]), K[4]), d), d);
    p = qrot(Q4{cq[1], cq[2], cq[3], cq[0]}, pc) + mk3(cp[0], cp[1], cp[2]);
  }
  float lo[3] = {cand ? p.x : inf, cand ? p.y : inf, cand ? p.z : inf};
  float hi[3] = {cand ? p.x : -inf, cand ? p.y : -inf, cand ? p.z : -inf};
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      lo[k] = fminf(lo[k], __shfl_xor_sync(full, lo[k], off));
      hi[k] = fmaxf(hi[k], __shfl_xor_sync(full, hi[k], off));
    }
  }
  const unsigned warp_cand = __ballot_sync(full, cand);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) warp_box[warp][k] = lo[k], warp_box[warp][3 + k] = hi[k];
    warp_box[warp][6] = warp_cand ? 1.0f : 0.0f;
  }
  if (threadIdx.x == 0) kept = 0;
  __syncthreads();
  bool any = false;
#pragma unroll
  for (int w = 0; w < kSegWarps; ++w) {
#pragma unroll
    for (int k = 0; k < 3; ++k) lo[k] = fminf(lo[k], warp_box[w][k]), hi[k] = fmaxf(hi[k], warp_box[w][3 + k]);
    any = any || warp_box[w][6] != 0.0f;
  }
  bool hit = false;
  if (any) {  // the same for every thread of the CTA
    const float *sph = a.spheres + (long long)img * a.sphere_stride;
    for (int base = 0; base < a.num_spheres; base += kSegThreads) {
      const int k = base + (int)threadIdx.x;
      bool keep = false;
      float4 s = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      if (k < a.num_spheres) {
        const float cx = sph[4 * k], cy = sph[4 * k + 1], cz = sph[4 * k + 2], reach = sph[4 * k + 3] + a.threshold;
        if (reach > 0.0f) {  // a disabled sphere (radius -100) never masks
          const float gx = fmaxf(fmaxf(__fsub_rn(lo[0], cx), __fsub_rn(cx, hi[0])), 0.0f);
          const float gy = fmaxf(fmaxf(__fsub_rn(lo[1], cy), __fsub_rn(cy, hi[1])), 0.0f);
          const float gz = fmaxf(fmaxf(__fsub_rn(lo[2], cz), __fsub_rn(cz, hi[2])), 0.0f);
          s = make_float4(cx, cy, cz, __fmul_rn(reach, reach));
          keep = seg_dist2(gx, gy, gz) < s.w;
        }
      }
      const unsigned m = __ballot_sync(full, keep);
      int slot = 0;
      if (lane == 0 && m != 0u) slot = atomicAdd(&kept, __popc(m));
      slot = __shfl_sync(full, slot, 0);
      if (keep) survivors[slot + __popc(m & ((1u << lane) - 1u))] = s;
    }
    __syncthreads();
    const int n = kept;
    if (cand) {
      for (int j = 0; j < n; ++j) {
        const float4 s = survivors[j];
        if (seg_dist2(__fsub_rn(p.x, s.x), __fsub_rn(p.y, s.y), __fsub_rn(p.z, s.z)) < s.w) {
          hit = true;
          break;
        }
      }
    }
  }
  if (inside) {
    a.mask[pix] = hit ? 1 : 0;
    a.filtered[pix] = hit ? 0.0f : d;
  }
}

// combined SDF of the dynamic (depth) and static channels: wp_tsdf_sample.py:22-97 (sample_dynamic_sdf / sample_combined_sdf):
// sum_sdf_w / sum_w where the weight exceeds min_weight, else 1e10 (unobserved); min with the static SDF when there is one.
__global__ void __launch_bounds__(256) tsdf_combined_sdf_kernel(const __half *__restrict__ block_data, const float *__restrict__ static_sdf,
                                                                 float *__restrict__ out, long long total, float min_weight) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const float sw = __half2float(block_data[2 * i]), w = __half2float(block_data[2 * i + 1]);
    float d = w > min_weight ? __fdiv_rn(sw, w) : 1e10f;
    if (static_sdf != nullptr) d = fminf(d, static_sdf[i]);
    out[i] = d;
  }
}

// World cuboids -> the STATIC channel of the dense TSDF: the per-voxel step of the reference's obstacle stamping
// (stamp_sdf_kernel, perception/mapper/kernel/builder/builder_stamp.py:263-315, with the cuboid overloads is_obs_enabled /
// load_obstacle_transform / compute_local_sdf of geom/data/data_cuboid.py:461-545) without the block enumeration / allocation in
// front of it: min over the enabled cuboids of the box SDF at the voxel centre; where |min| <= truncation the voxel takes
// clamp(min(existing, min), +-truncation), rounded through fp16 as the reference's static_block_data stores it.  static_sdf is
// float32 (> 1e9 = nothing stamped), the format DenseESDFBuilder takes.
__global__ void __launch_bounds__(256) tsdf_stamp_cuboids_kernel(float *__restrict__ static_sdf, int nx, int ny, int nz, long long total,
                                                                  float voxel_size, float ox, float oy, float oz, float truncation,
                                                                  cb200::CuboidSet cs, int env) {
  using namespace cb200;
  int ncub = cs.count[env];
  if (ncub > cs.max_n) ncub = cs.max_n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(i % nz), y = (int)((i / nz) % ny), x = (int)(i / ((long long)nz * ny));
    const V3 c = mk3(((float)x + 0.5f - (float)nx * 0.5f) * voxel_size + ox, ((float)y + 0.5f - (float)ny * 0.5f) * voxel_size + oy,
                     ((float)z + 0.5f - (float)nz * 0.5f) * voxel_size + oz);
    float min_sdf = 1e10f;
    for (int k = 0; k < ncub; ++k) {
      const int kk = env * cs.max_n + k;
      if (cs.enable[kk] != 1) continue;
      const ObsFrame f = load_obs_frame(cs.inv_pose + 8 * kk);
      const SdfGrad sg = cuboid_sdf_grad(to_obstacle(f, c), cs.dims[4 * kk], cs.dims[4 * kk + 1], cs.dims[4 * kk + 2]);
      min_sdf = fminf(min_sdf, sg.sdf);
    }
    if (fabsf(min_sdf) <= truncation) {
      const float final_sdf = fminf(static_sdf[i], min_sdf);
      static_sdf[i] = __half2float(__float2half_rn(fminf(fmaxf(final_sdf, -truncation), truncation)));
    }
  }
}

bool dims_ok(int nx, int ny, int nz) {
  return nx >= 1 && ny >= 1 && nz >= 1 && nx <= kMaxDim && ny <= kMaxDim && nz <= kMaxDim &&
         (long long)nx * ny * nz <= 2147483647LL;
}
}  // namespace

extern "C" {

int cb200_pba3d(int32_t *site_index, int32_t *buffer, int nx, int ny, int nz, int m3, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(site_index);
  (void)buffer;  // the reference's ping-pong scratch: every pass here is in place
  (void)m3;      // the reference's colour-kernel block height
  if (site_index == nullptr || !dims_ok(nx, ny, nz)) return ret(cudaErrorInvalidValue);
  const cudaStream_t st = (cudaStream_t)stream;
  const Plan p = make_plan(site_index, nx, ny, nz);
  const BandedEnvelope<1> by{p.y};
  const BandedEnvelope<0> bx{p.x};
  const int smem_y = by.smem_ints() * (int)sizeof(int), smem_x = bx.smem_ints() * (int)sizeof(int);
  if (opt_in_smem(edt_envelope_kernel<1>, smem_y) != cudaSuccess || opt_in_smem(edt_envelope_kernel<0>, smem_x) != cudaSuccess)
    return ret(cudaErrorInvalidConfiguration);
  const long long nrows = (long long)nx * ny;
  const int zgrid = capped_grid((nrows + 15) / 16, 32);  // 8 warps per CTA, two rows per warp and step
  if (nz <= 128) {
    CB200_LAUNCH(edt_flood_z_kernel<4>, zgrid, 256, 0, st, site_index, nz, nrows);
  } else if (nz <= 256) {
    CB200_LAUNCH(edt_flood_z_kernel<8>, zgrid, 256, 0, st, site_index, nz, nrows);
  } else if (nz <= 512) {
    CB200_LAUNCH(edt_flood_z_kernel<16>, zgrid, 256, 0, st, site_index, nz, nrows);
  } else {
    CB200_LAUNCH(edt_flood_z_kernel<32>, zgrid, 256, 0, st, site_index, nz, nrows);
  }
  CB200_LAUNCH(edt_envelope_kernel<1>, capped_grid(by.e.ntiles(), 32), kBands * kLanes, smem_y, st, by);
  CB200_LAUNCH(edt_envelope_kernel<0>, capped_grid(bx.e.ntiles(), 32), kBands * kLanes, smem_x, st, bx);
  return launch_status();
}

int cb200_edt_unsigned_distance(const int32_t *site_index, uint16_t *distance_fp16, int nx, int ny, int nz, float voxel_size,
                                float empty_value, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(distance_fp16);
  if (site_index == nullptr || distance_fp16 == nullptr || !dims_ok(nx, ny, nz) || !(voxel_size > 0.0f))
    return ret(cudaErrorInvalidValue);
  const long long total = (long long)nx * ny * nz;
  const long long blocks = (total + 255) / 256;
  CB200_LAUNCH(edt_distance_kernel, capped_grid(blocks, 32), 256, 0, (cudaStream_t)stream, site_index, reinterpret_cast<__half *>(distance_fp16),
               ny, nz, total, voxel_size, empty_value);
  return launch_status();
}

int cb200_esdf_seed_sites(const float *combined_sdf, int32_t *site_index, int nx, int ny, int nz, float voxel_size,
                          float truncation_distance, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(site_index);
  if (combined_sdf == nullptr || site_index == nullptr || !dims_ok(nx, ny, nz) || !(voxel_size > 0.0f))
    return ret(cudaErrorInvalidValue);
  const long long total = (long long)nx * ny * nz;
  CB200_LAUNCH(esdf_seed_sites_kernel, capped_grid((total + 255) / 256, 32), 256, 0, (cudaStream_t)stream, combined_sdf, site_index, ny, nz,
               total, voxel_size, truncation_distance);
  return launch_status();
}

int cb200_esdf_seed_sites_gather(const float *combined_sdf, int32_t *site_index, int nx, int ny, int nz, float voxel_size,
                                 float truncation_distance, const float *origin, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(site_index);
  if (combined_sdf == nullptr || site_index == nullptr || origin == nullptr || !dims_ok(nx, ny, nz) || !(voxel_size > 0.0f))
    return ret(cudaErrorInvalidValue);
  const long long total = (long long)nx * ny * nz;
  CB200_LAUNCH(esdf_seed_sites_gather_kernel, capped_grid((total + 255) / 256, 32), 256, 0, (cudaStream_t)stream, combined_sdf, site_index, nx,
               ny, nz, total, voxel_size, truncation_distance, origin[0], origin[1], origin[2]);
  return launch_status();
}

int cb200_esdf_signed_distance(const int32_t *site_index, const float *static_sdf, const float *combined_sdf,
                               uint16_t *distance_fp16, int nx, int ny, int nz, float voxel_size, float adjacent_skip_steps,
                               cb200_stream_t stream) {
  CB200_DEVICE_GUARD(distance_fp16);
  if (site_index == nullptr || distance_fp16 == nullptr || !dims_ok(nx, ny, nz) || !(voxel_size > 0.0f))
    return ret(cudaErrorInvalidValue);
  const long long total = (long long)nx * ny * nz;
  CB200_LAUNCH(esdf_signed_distance_kernel, capped_grid((total + 255) / 256, 32), 256, 0, (cudaStream_t)stream, site_index, static_sdf,
               combined_sdf, reinterpret_cast<__half *>(distance_fp16), nx, ny, nz, total, voxel_size, adjacent_skip_steps);
  return launch_status();
}

int cb200_tsdf_integrate_depth(uint16_t *block_data_fp16, int nx, int ny, int nz, float voxel_size, const float *origin,
                               int num_cameras, const float *intrinsics, const float *cam_positions,
                               const float *cam_quaternions, const float *depth_images, int image_height, int image_width,
                               float depth_min, float depth_max, float truncation_distance, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(block_data_fp16);
  if (block_data_fp16 == nullptr || origin == nullptr || intrinsics == nullptr || cam_positions == nullptr ||
      cam_quaternions == nullptr || depth_images == nullptr || !dims_ok(nx, ny, nz) || !(voxel_size > 0.0f) || num_cameras < 1 ||
      image_height < 1 || image_width < 1 || !(truncation_distance > 0.0f))
    return ret(cudaErrorInvalidValue);
  const long long total = (long long)nx * ny * nz;
  const TsdfCameras cams{intrinsics, cam_positions, cam_quaternions, depth_images, num_cameras, image_height, image_width};
  CB200_LAUNCH(tsdf_integrate_depth_kernel, capped_grid((total + 255) / 256, 32), 256, 0, (cudaStream_t)stream,
               reinterpret_cast<__half *>(block_data_fp16), nx, ny, nz, total, voxel_size, origin[0], origin[1], origin[2], cams,
               depth_min, depth_max, truncation_distance);
  return launch_status();
}

int cb200_segment_robot_depth(const float *depth, int batch, int height, int width, const float *intrinsics,
                              const float *cam_positions, const float *cam_quaternions, const float *robot_spheres, int robot_batch,
                              int num_spheres, float distance_threshold, uint8_t *mask, float *filtered, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(filtered);
  if (depth == nullptr || intrinsics == nullptr || cam_positions == nullptr || cam_quaternions == nullptr ||
      robot_spheres == nullptr || mask == nullptr || filtered == nullptr || batch < 1 || height < 1 || width < 1 ||
      num_spheres < 0 || (robot_batch != 1 && robot_batch != batch))
    return ret(cudaErrorInvalidValue);
  const int tiles_x = (width + kSegTileW - 1) / kSegTileW;
  const long long tiles_per_image = (long long)tiles_x * ((height + kSegTileH - 1) / kSegTileH);
  // one flat grid (the host emulation of tests/simt launches along x only): its x extent bounds the batch
  if (tiles_per_image * batch > 2147483647LL) return ret(cudaErrorInvalidValue);
  const long long smem = (long long)num_spheres * (long long)sizeof(float4);
  cudaFuncAttributes fa;
  if (cudaFuncGetAttributes(&fa, segment_robot_depth_kernel) != cudaSuccess) return ret(cudaErrorInvalidConfiguration);
  if (smem + (long long)fa.sharedSizeBytes > (long long)cb200::dev_info().max_smem) return ret(cudaErrorInvalidValue);
  if (opt_in_smem(segment_robot_depth_kernel, (size_t)smem) != cudaSuccess) return ret(cudaErrorInvalidConfiguration);
  const SegmentArgs a{depth, intrinsics, cam_positions, cam_quaternions, robot_spheres, mask, filtered, height, width, tiles_x,
                      (int)tiles_per_image, robot_batch == 1 ? 0 : 4 * num_spheres, num_spheres, distance_threshold};
  CB200_LAUNCH(segment_robot_depth_kernel, tiles_per_image * batch, kSegThreads, (size_t)smem, (cudaStream_t)stream, a);
  return launch_status();
}

int cb200_tsdf_stamp_cuboids(float *static_sdf, int nx, int ny, int nz, float voxel_size, const float *origin,
                             float truncation_distance, const cb200_cuboid_set *cuboids, int env_idx, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(static_sdf);
  if (static_sdf == nullptr || origin == nullptr || cuboids == nullptr || cuboids->inv_pose == nullptr || cuboids->dims == nullptr ||
      cuboids->enable == nullptr || cuboids->count == nullptr || cuboids->max_n < 1 || env_idx < 0 || env_idx >= cuboids->num_envs ||
      !dims_ok(nx, ny, nz) || !(voxel_size > 0.0f) || !(truncation_distance > 0.0f))
    return ret(cudaErrorInvalidValue);
  const long long total = (long long)nx * ny * nz;
  const cb200::CuboidSet cs{cuboids->dims, cuboids->inv_pose, cuboids->enable, cuboids->count, cuboids->max_n, cuboids->num_envs};
  CB200_LAUNCH(tsdf_stamp_cuboids_kernel, capped_grid((total + 255) / 256, 32), 256, 0, (cudaStream_t)stream, static_sdf, nx, ny, nz, total,
               voxel_size, origin[0], origin[1], origin[2], truncation_distance, cs, env_idx);
  return launch_status();
}

int cb200_tsdf_combined_sdf(const uint16_t *block_data_fp16, const float *static_sdf, float *combined_sdf, long long num_voxels,
                            float min_weight, cb200_stream_t stream) {
  CB200_DEVICE_GUARD(combined_sdf);
  if (block_data_fp16 == nullptr || combined_sdf == nullptr || num_voxels < 1) return ret(cudaErrorInvalidValue);
  CB200_LAUNCH(tsdf_combined_sdf_kernel, capped_grid((num_voxels + 255) / 256, 32), 256, 0, (cudaStream_t)stream,
               reinterpret_cast<const __half *>(block_data_fp16), static_sdf, combined_sdf, num_voxels, min_weight);
  return launch_status();
}

}  // extern "C"
