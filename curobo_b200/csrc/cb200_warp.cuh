// cb200_warp.cuh -- warp-cooperative stages of one rollout evaluation (device only).
//
// One warp owns one (seed x waypoint) evaluation.  Its working set lives in a private slice of shared
// memory (`EvalSmem`): the cumulative link transforms never leave the SM, sphere positions and sphere
// gradients are produced and consumed in place, and the J^T backward runs on per-link force/torque
// accumulators instead of walking a joint chain per sphere.
#pragma once
#include "cb200_blob.h"
#include "cb200_math.cuh"

namespace cb200 {

constexpr unsigned kFull = 0xffffffffu;

// View of the blob once it sits in shared memory (pointers into smem) + the pair list in global memory.
struct RobotView {
  int nl, D, S, L, P, n_levels;
  const float *fixed;
  const float *joff;
  const int16_t *link_map;
  const int16_t *joint_map;
  const int8_t *joint_type;
  const int16_t *tool_map;
  const float4 *spheres;
  const int16_t *sph_link;
  const float *padding;
  const int16_t *link_sph_off;
  const int16_t *link_sph_idx;
  const int16_t *level_off;
  const int16_t *level_links;
  const unsigned long long *anc_mask;
  const int16_t *jl_off;
  const int16_t *jl_idx;
  const float *limits;
  const uint32_t *pairs;  // global memory: one packed (i | j<<16) word per pair
  int n_cl, n_lp;
  const int16_t *cl_link;
  const int16_t *cl_start;
  const float4 *cl_bound;
  const uint32_t *lp;
  int n_fk_steps;
  const uint32_t *fk_sched;
  const float4 *cl_bound_scene;
  const uint8_t *sph_cl;
};

__device__ __forceinline__ RobotView make_robot_view(const unsigned char *smem_blob, const unsigned char *gmem_blob) {
  const BlobHeader *h = reinterpret_cast<const BlobHeader *>(smem_blob);
  RobotView v;
  v.nl = h->nl;
  v.D = h->D;
  v.S = h->S;
  v.L = h->L;
  v.P = h->P;
  v.n_levels = h->n_levels;
  v.fixed = reinterpret_cast<const float *>(smem_blob + h->off_fixed);
  v.joff = reinterpret_cast<const float *>(smem_blob + h->off_joff);
  v.link_map = reinterpret_cast<const int16_t *>(smem_blob + h->off_link_map);
  v.joint_map = reinterpret_cast<const int16_t *>(smem_blob + h->off_joint_map);
  v.joint_type = reinterpret_cast<const int8_t *>(smem_blob + h->off_joint_type);
  v.tool_map = reinterpret_cast<const int16_t *>(smem_blob + h->off_tool_map);
  v.spheres = reinterpret_cast<const float4 *>(smem_blob + h->off_spheres);
  v.sph_link = reinterpret_cast<const int16_t *>(smem_blob + h->off_sph_link);
  v.padding = reinterpret_cast<const float *>(smem_blob + h->off_padding);
  v.link_sph_off = reinterpret_cast<const int16_t *>(smem_blob + h->off_link_sph_off);
  v.link_sph_idx = reinterpret_cast<const int16_t *>(smem_blob + h->off_link_sph_idx);
  v.level_off = reinterpret_cast<const int16_t *>(smem_blob + h->off_level_off);
  v.level_links = reinterpret_cast<const int16_t *>(smem_blob + h->off_level_links);
  v.anc_mask = reinterpret_cast<const unsigned long long *>(smem_blob + h->off_anc_mask);
  v.jl_off = reinterpret_cast<const int16_t *>(smem_blob + h->off_jl_off);
  v.jl_idx = reinterpret_cast<const int16_t *>(smem_blob + h->off_jl_idx);
  v.limits = reinterpret_cast<const float *>(smem_blob + h->off_limits);
  v.pairs = reinterpret_cast<const uint32_t *>(gmem_blob + h->off_pairs);
  v.n_cl = h->n_cl;
  v.n_lp = h->n_lp;
  v.cl_link = reinterpret_cast<const int16_t *>(smem_blob + h->off_cl_link);
  v.cl_start = reinterpret_cast<const int16_t *>(smem_blob + h->off_cl_start);
  v.cl_bound = reinterpret_cast<const float4 *>(smem_blob + h->off_cl_bound);
  v.lp = reinterpret_cast<const uint32_t *>(smem_blob + h->off_lp);
  v.n_fk_steps = h->n_fk_steps;
  v.fk_sched = reinterpret_cast<const uint32_t *>(smem_blob + h->off_fk_sched);
  v.cl_bound_scene = reinterpret_cast<const float4 *>(smem_blob + h->off_cl_bound_scene);
  v.sph_cl = reinterpret_cast<const uint8_t *>(smem_blob + h->off_sph_cl);
  return v;
}

// Per-warp scratch (floats).  Layout computed identically on host (cb200_eval_smem_floats).
struct EvalSmem {
  float *cumul;   // [nl*12]
  float4 *sph;    // [S] world spheres (x,y,z,r)
  float4 *gsph;   // [S] padded spheres during self-collision, then sphere gradients
  float *ft;      // [nl*8]  F.xyz,_ ,T.xyz,_   (torque about the link origin)
  float *contrib; // [nl]
  float *qv;      // [D]
  float *gqv;     // [D]  c-space position gradient
  float *pose_g;  // [L*8]  g_pos.xyz,_, omega.xyz,_
  float4 *bc;     // [n_cl] world-frame bounding spheres of the collision links (self-collision broad phase)
  uint32_t *cmask;  // [n_cl] scene broad phase: bit i set <=> cuboid i may touch a sphere of the link
  float4 *glist;    // big-robot layout only: (g.xyz, sphere index) of the spheres with a non-zero gradient; gsph == nullptr there
};
__host__ __device__ inline int eval_smem_floats(int nl, int D, int S, int L, int n_cl) {
  int n = nl * 12 + S * 8 + nl * 8 + n_cl * 4;   // float4-aligned part
  n += nl + D + D + L * 8 + n_cl;
  return (n + 3) & ~3;
}
__device__ __forceinline__ EvalSmem carve_eval_smem(float *base, int nl, int D, int S, int L, int n_cl) {
  EvalSmem e;
  e.cumul = base;
  e.sph = reinterpret_cast<float4 *>(base + nl * 12);
  e.gsph = e.sph + S;
  e.ft = base + nl * 12 + S * 8;
  e.bc = reinterpret_cast<float4 *>(e.ft + nl * 8);
  e.contrib = e.ft + nl * 8 + n_cl * 4;
  e.qv = e.contrib + nl;
  e.gqv = e.qv + D;
  e.pose_g = e.gqv + D;
  e.cmask = reinterpret_cast<uint32_t *>(e.pose_g + L * 8);
  e.glist = nullptr;
  return e;
}

// Row state of the big-robot kernel (humanoids): no dense sphere-gradient array and no padded sphere copy -- the two [S] float4
// arrays that make a humanoid row 17-27 KB -- but a short list of the spheres that actually carry a gradient.  6.4 KB less per
// row for G1-29, 10.8 KB for G1-43: 16 instead of 10 resident rows per SM.
constexpr int kGradListCap = 96;
__host__ __device__ inline int big_smem_floats(int nl, int D, int S, int L, int n_cl) {
  int n = nl * 12 + S * 4 + nl * 8 + n_cl * 4 + kGradListCap * 4;  // float4-aligned part
  n += nl + D + D + L * 8 + n_cl;
  return (n + 3) & ~3;
}
__device__ __forceinline__ EvalSmem carve_big_smem(float *base, int nl, int D, int S, int L, int n_cl) {
  EvalSmem e;
  e.cumul = base;
  e.sph = reinterpret_cast<float4 *>(base + nl * 12);
  e.gsph = nullptr;
  e.ft = base + nl * 12 + S * 4;
  e.bc = reinterpret_cast<float4 *>(e.ft + nl * 8);
  e.glist = e.bc + n_cl;
  e.contrib = reinterpret_cast<float *>(e.glist + kGradListCap);
  e.qv = e.contrib + nl;
  e.gqv = e.qv + D;
  e.pose_g = e.gqv + D;
  e.cmask = reinterpret_cast<uint32_t *>(e.pose_g + L * 8);
  return e;
}

// Row state of the cost-only kernels (rollout_cost_kernel, rollout_cost_big_kernel): nothing the gradient alone reads -- no sphere
// gradients or gradient list, no force / torque accumulators, no c-space or pose gradients.  `ft` is only the 64-byte index
// scratch of the second-level self-collision cull.  The padded sphere copy stays for robots without a link-pair list (n_lp == 0),
// whose pair scan reads it; the others rebuild padded radii from the padding table.
constexpr int kCullScratchFloats = 16;
__host__ __device__ inline int cost_smem_floats(int nl, int D, int S, int n_cl, bool padded_copy) {
  int n = nl * 12 + S * (padded_copy ? 8 : 4) + kCullScratchFloats + n_cl * 4;  // float4-aligned part
  n += D + n_cl;
  return (n + 3) & ~3;
}
__device__ __forceinline__ EvalSmem carve_cost_smem(float *base, int nl, int D, int S, int n_cl, bool padded_copy) {
  EvalSmem e;
  e.cumul = base;
  e.sph = reinterpret_cast<float4 *>(base + nl * 12);
  e.gsph = padded_copy ? e.sph + S : nullptr;
  e.ft = base + nl * 12 + S * (padded_copy ? 8 : 4);
  e.bc = reinterpret_cast<float4 *>(e.ft + kCullScratchFloats);
  e.qv = reinterpret_cast<float *>(e.bc + n_cl);
  e.cmask = reinterpret_cast<uint32_t *>(e.qv + D);
  e.contrib = e.gqv = e.pose_g = nullptr;
  e.glist = nullptr;
  return e;
}

// Lanes of one row.  W = 32: the whole warp.  W = 16 (paired arm build): half h = lane >> 4 of the warp owns a row of its own,
// and the two halves may diverge, so every collective of a row names the row's lanes only.  In the helpers below `lane` is the
// lane within the row (0 .. W-1) and ballots come back in row-local bits.  W = 32 spells exactly the full-warp intrinsics.
template <int W>
__device__ __forceinline__ unsigned row_mask() {
  static_assert(W == 32 || W == 16, "a row is a warp or a half-warp");
  return W == 32 ? kFull : 0xffffu << (threadIdx.x & 16u);
}
#ifdef CB200_SIMT_EMULATION
// Host emulation build (tests/simt): there a warp collective is a meeting of all 32 lane threads, whatever its mask, while the
// two halves of a paired warp may be on different paths.  A half-warp's collectives therefore meet on a named barrier of their
// own (id = the half's index in the CTA: 16 ids for the <= 8-warp CTAs of the paired build), values passing through a CTA-wide
// slot array: publish, meet, read the half's 16 slots, meet again so the slots can be reused.
template <class T, class F>
inline T half_exchange(T v, F pick) {
  static unsigned long long slot[16 * 16];
  const int t = threadIdx.x;
  unsigned long long bits = 0;
  std::memcpy(&bits, &v, sizeof(T));
  slot[t] = bits;
  simt::named_barrier(t >> 4, 16);
  const unsigned long long got = pick(slot + (t & ~15));
  simt::named_barrier(t >> 4, 16);
  T r;
  std::memcpy(&r, &got, sizeof(T));
  return r;
}
#endif
template <int W>
__device__ __forceinline__ void row_sync() {
  if (W == 32) {
    __syncwarp();
  } else {
#ifdef CB200_SIMT_EMULATION
    simt::named_barrier(threadIdx.x >> 4, 16);
#else
    __syncwarp(row_mask<W>());
#endif
  }
}
template <int W>
__device__ __forceinline__ unsigned row_ballot(bool p) {
  if (W == 32) return __ballot_sync(kFull, p);
#ifdef CB200_SIMT_EMULATION
  return half_exchange((unsigned)p, [](const unsigned long long *s) {
    unsigned long long m = 0;
    for (int i = 0; i < 16; ++i) m |= (s[i] & 1ull) << i;
    return m;
  });
#else
  const unsigned m = row_mask<W>();
  return (__ballot_sync(m, p) & m) >> (threadIdx.x & 16u);
#endif
}
// value of row lane `src`
template <int W>
__device__ __forceinline__ uint32_t row_shfl(uint32_t v, int src) {
  if (W == 32) return __shfl_sync(kFull, v, src);
#ifdef CB200_SIMT_EMULATION
  return half_exchange(v, [src](const unsigned long long *s) { return s[src & 15]; });
#else
  return __shfl_sync(row_mask<W>(), v, src, W);
#endif
}
// value of row lane `lane ^ o` (o < W)
template <int W, class T>
__device__ __forceinline__ T row_shfl_xor(T v, int o) {
  if (W == 32) return __shfl_xor_sync(kFull, v, o);
#ifdef CB200_SIMT_EMULATION
  const int me = threadIdx.x & 15;
  return half_exchange(v, [me, o](const unsigned long long *s) { return s[me ^ o]; });
#else
  return __shfl_xor_sync(row_mask<W>(), v, o);
#endif
}
// REDUX over the row's lanes: OP 0 = add, 1 = min, 2 = max
template <int W, int OP>
__device__ __forceinline__ unsigned row_reduce(unsigned v) {
  if (W == 32) return OP == 0 ? __reduce_add_sync(kFull, v) : OP == 1 ? __reduce_min_sync(kFull, v) : __reduce_max_sync(kFull, v);
#ifdef CB200_SIMT_EMULATION
  return half_exchange(v, [](const unsigned long long *s) {
    unsigned r = (unsigned)s[0];
    for (int i = 1; i < 16; ++i) {
      const unsigned x = (unsigned)s[i];
      r = OP == 0 ? r + x : OP == 1 ? (x < r ? x : r) : (x > r ? x : r);
    }
    return (unsigned long long)r;
  });
#else
  const unsigned m = row_mask<W>();
  return OP == 0 ? __reduce_add_sync(m, v) : OP == 1 ? __reduce_min_sync(m, v) : __reduce_max_sync(m, v);
#endif
}

template <int W = 32>
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = W / 2; o > 0; o >>= 1) v += row_shfl_xor<W>(v, o);
  return v;
}

// ----------------------------------------------------------------------------------------------
// FK: local transforms (one lane per link) then level-synchronous chain compose
// (12 lanes per link, two links per step).  cumul[l] = cumul[parent[l]] * local[l].
// Reference semantics: kinematics_forward_helper.cuh:316-512.
// ----------------------------------------------------------------------------------------------
template <int W = 32>
__device__ __forceinline__ void warp_fk_compose(const RobotView &rv, const EvalSmem &es, int lane);
template <int W = 32>
__device__ __forceinline__ void warp_fk(const RobotView &rv, const EvalSmem &es, int lane) {
  // local transforms go to a scratch buffer (the not-yet-written world-sphere area) when it is large enough,
  // so a compose step needs one warp barrier instead of two; otherwise they are composed in place.
  const bool scratch = rv.S * 4 >= rv.nl * 12;
  float *loc = scratch ? reinterpret_cast<float *>(es.sph) : es.cumul;
  #pragma unroll 1
  for (int l = lane; l < rv.nl; l += W) {
    int jt = rv.joint_type[l];
    float th = 0.0f;
    if (jt >= 0) th = rv.joff[2 * l] * es.qv[rv.joint_map[l]] + rv.joff[2 * l + 1];
    local_link_transform(rv.fixed + 12 * l, jt, th, (l == 0 ? es.cumul : loc) + 12 * l);
  }
  row_sync<W>();
  warp_fk_compose<W>(rv, es, lane);
}

// second half of warp_fk: the level-scheduled compose (the local transforms are in place; see warp_fk)
template <int W>
__device__ __forceinline__ void warp_fk_compose(const RobotView &rv, const EvalSmem &es, int lane) {
  const bool scratch = rv.S * 4 >= rv.nl * 12;
  const float *loc = scratch ? reinterpret_cast<const float *>(es.sph) : es.cumul;
  // compose: 12 lanes per link, two links (same depth level) per step; the schedule holds byte offsets.  A whole warp does the
  // two links at once (half-warp per link); a half-warp row does slot 0, then slot 1 -- the schedule is the robot's, so both
  // rows of a warp take the same branches here.
  const int half = lane >> 4, k = lane & 15;
  const bool lane_ok = k < 12;
  const uint32_t row_off = (uint32_t)(k >> 2) * 16u, col_off = (uint32_t)(k & 3) * 4u, k_off = (uint32_t)k * 4u;
  const float cw = ((k & 3) == 3) ? 1.0f : 0.0f;
  unsigned char *cumb = reinterpret_cast<unsigned char *>(es.cumul);
  const unsigned char *locb = reinterpret_cast<const unsigned char *>(loc);
#pragma unroll 1
  for (int st = 0; st < rv.n_fk_steps; ++st) {
#pragma unroll
    for (int pass = 0; pass < 32 / W; ++pass) {
      const int sub = W == 32 ? half : pass;
      const uint32_t w = rv.fk_sched[2 * st + sub];
      const uint32_t l_off = w & 0xffffu, p_off = w >> 16;
      if (W == 16 && l_off == 0xffffu) continue;  // empty slot (same for every row)
      const bool act = lane_ok && (l_off != 0xffffu);
      float out = 0.0f;
      if (act) {
        const float4 pr = *reinterpret_cast<const float4 *>(cumb + p_off + row_off);
        const float *Lm = reinterpret_cast<const float *>(locb + l_off + col_off);
        out = pr.x * Lm[0] + pr.y * Lm[4] + pr.z * Lm[8] + cw * pr.w;
      }
      if (!scratch) row_sync<W>();
      if (act) *reinterpret_cast<float *>(cumb + l_off + k_off) = out;
      row_sync<W>();
    }
  }
}

// Spheres: world position of every robot sphere; also the self-collision (padded radius) copy in gsph.
// Reference: kinematics_forward_helper.cuh:218-254, kinematics_util.cuh:39-49.
// `cfg_spheres` != nullptr: the row's link-sphere configuration in global memory (num_envs > 1,
// kinematics_forward_helper.cuh:232-233) instead of the blob's set.
template <int W = 32>
__device__ __forceinline__ void warp_spheres(const RobotView &rv, const EvalSmem &es, int lane, float4 *out_global,
                                             const float4 *cfg_spheres = nullptr) {
  #pragma unroll 1
  for (int s = lane; s < rv.S; s += W) {
    const float *T = es.cumul + 12 * rv.sph_link[s];
    const float4 p = cfg_spheres != nullptr ? __ldg(cfg_spheres + s) : rv.spheres[s];
    const float4 r0 = *reinterpret_cast<const float4 *>(T), r1 = *reinterpret_cast<const float4 *>(T + 4),
                 r2 = *reinterpret_cast<const float4 *>(T + 8);
    float4 w;
    w.x = r0.x * p.x + r0.y * p.y + r0.z * p.z + r0.w;
    w.y = r1.x * p.x + r1.y * p.y + r1.z * p.z + r1.w;
    w.z = r2.x * p.x + r2.y * p.y + r2.z * p.z + r2.w;
    w.w = p.w;
    es.sph[s] = w;
    if (out_global != nullptr) out_global[s] = w;
    if (es.gsph != nullptr) {
      w.w = p.w + rv.padding[s];
      es.gsph[s] = w;
    }
  }
}

// ----------------------------------------------------------------------------------------------
// Self collision over an explicit pair list: f = (ri+rj)^2 - |pi-pj|^2 (padded radii, both >= 0),
// arg-max over pairs with f > 0, first pair wins ties.
// Reference: self_collision_helper.cuh:61-71,227-277; collision_pair.cuh:55-57.
// Returns f_max (0 if none) and the pair (i,j) to every lane.
// ----------------------------------------------------------------------------------------------
template <int W = 32>
__device__ __forceinline__ float warp_self_collision_pairs(const float4 *psph, const uint32_t *pairs, int P, int lane,
                                                           int &bi, int &bj) {
  float best = 0.0f;
  uint32_t best_p = 0xffffffffu;
  #pragma unroll 1
  for (int p = lane; p < P; p += W) {
    const uint32_t pr = __ldg(pairs + p);
    const float4 a = psph[pr & 0xffffu], b = psph[pr >> 16];
    const float rs = a.w + b.w;
    const float dx = a.x - b.x, dy = a.y - b.y, dz = a.z - b.z;
    float f = rs * rs - (dx * dx + dy * dy + dz * dz);
    if (!(a.w >= 0.0f && b.w >= 0.0f)) f = 0.0f;
    if (f > best) {
      best = f;
      best_p = (uint32_t)p;
    }
  }
  // positive floats order like their bit patterns
  const uint32_t fb = row_reduce<W, 2>(__float_as_uint(best));
  const uint32_t cand = (__float_as_uint(best) == fb && best > 0.0f) ? best_p : 0xffffffffu;
  const uint32_t win = row_reduce<W, 1>(cand);
  bi = bj = 0;
  if (win == 0xffffffffu) return 0.0f;
  const uint32_t pr = __ldg(pairs + win);
  bi = (int)(pr & 0xffffu);
  bj = (int)(pr >> 16);
  return __uint_as_float(fb);
}

// ----------------------------------------------------------------------------------------------
// Self collision with a link-level broad phase.  The reference's pair list is the union of
// (spheres of link a) x (spheres of link b) over the checked link pairs, and only pairs with
// f = (ri+rj)^2 - |pi-pj|^2 > 0 can matter (the running max starts at 0, self_collision_helper.cuh:239,264).
// If the bounding spheres of two links are disjoint no sphere pair of that block has f > 0, so the block is
// skipped -- the result (f_max and the arg-max pair, ties to the first pair in list order = smallest (i,j))
// is identical to scanning the whole list.  Lanes test 32 link pairs at a time; surviving blocks are scanned
// with lanes over the flattened |a| x |b| tile.
// ----------------------------------------------------------------------------------------------
// PADDED_COPY = false (big-robot layout): the padded sphere is rebuilt from the world sphere + the padding table on every read.
// World-frame bounding sphere of every collision link (es.bc), over the W lanes of a row, or of a team of warps sharing one
// (W = TEAM x 32, `lane` = the lane within the team).
template <int W = 32>
__device__ __forceinline__ void link_bounds(const RobotView &rv, const EvalSmem &es, int lane) {
  #pragma unroll 1
  for (int a = lane; a < rv.n_cl; a += W) {
    const float4 c = rv.cl_bound[a];
    const float *T = es.cumul + 12 * rv.cl_link[a];
    es.bc[a] = make_float4(T[0] * c.x + T[1] * c.y + T[2] * c.z + T[3], T[4] * c.x + T[5] * c.y + T[6] * c.z + T[7],
                           T[8] * c.x + T[9] * c.y + T[10] * c.z + T[11], c.w);
  }
}

template <bool PADDED_COPY>
__device__ __forceinline__ float4 padded_sphere(const RobotView &rv, const EvalSmem &es, int i) {
  if (PADDED_COPY) return es.gsph[i];
  float4 x = es.sph[i];
  x.w += rv.padding[i];
  return x;
}

// base0 / stride: the slice of the link-pair list this warp scans (a team of warps sharing one row takes interleaved
// slices); idx_scratch: 64 bytes of per-warp scratch for the second-level cull (default: the row's idle force / torque area);
// key_out: the warp's reduced arg-max key (f bits | ~i | ~j), 0 when nothing is positive.
// CULL2 = false (arm build of the IK kernel: links of <= ~10 spheres): blocks are scanned whole -- the second-level cull's code is
// 1.6 KB of the row's instruction footprint, which is what that kernel is short of.
// ANY = true (validity rows): the row only asks whether some pair has f > 0, so the scan stops at the first block boundary where
// a lane holds one (a warp vote); the returned f and pair are then those of the blocks scanned so far.
template <bool PADDED_COPY = true, bool CULL2 = true, int W = 32, bool ANY = false>
__device__ __forceinline__ float warp_self_collision_tiles(const RobotView &rv, const EvalSmem &es, int lane, int &bi,
                                                           int &bj, int base0 = 0, int stride = W,
                                                           unsigned char *idx_scratch = nullptr,
                                                           unsigned long long *key_out = nullptr, bool fill_bounds = true) {
  static_assert(W == 32 || !CULL2, "the second-level cull is written for whole-warp rows");
  if (fill_bounds) {
    link_bounds<W>(rv, es, lane);
    row_sync<W>();
  }
  unsigned long long key = 0ull;  // f bits | ~i | ~j : max = largest f, then smallest i, then smallest j
  #pragma unroll 1
  for (int base = base0; base < rv.n_lp; base += stride) {
    uint32_t pr = 0;
    bool hit = false;
    if (base + lane < rv.n_lp) {
      pr = rv.lp[base + lane];
      const float4 A = es.bc[pr & 0xffffu], B = es.bc[pr >> 16];
      const float dx = A.x - B.x, dy = A.y - B.y, dz = A.z - B.z, rs = A.w + B.w;
      hit = (A.w >= 0.0f) && (B.w >= 0.0f) && (dx * dx + dy * dy + dz * dz < rs * rs);
    }
    unsigned m = row_ballot<W>(hit);
    while (m) {
      if (ANY && row_ballot<W>(key != 0ull) != 0u) break;
      const int src = __ffs(m) - 1;
      m &= m - 1;
      const uint32_t q = row_shfl<W>(pr, src);
      const int a = q & 0xffffu, b = q >> 16;
      const int sa = rv.cl_start[a], na = rv.cl_start[a + 1] - sa;
      const int sb = rv.cl_start[b], nb = rv.cl_start[b + 1] - sb;
      if (CULL2 && es.ft != nullptr && na <= 32 && nb <= 32 && na * nb > 64) {  // (a block of <= 2 passes is cheaper to scan
                                                                        // than to cull; the lists are staged in es.ft)
        // Second-level cull (exact): a pair (i, j) with f > 0 has |p_i - c_b| < r_i + R_b and |p_j - c_a| < r_j + R_a
        // (bounds enclose the padded sphere balls), so only spheres that reach the OTHER link's bound can matter.
        // Most blocks that survive the bound-vs-bound test have none on one side and are dropped here; the rest are
        // scanned over the compacted candidate lists (indices staged in the idle force/torque scratch).
        const float4 A = es.bc[a], B = es.bc[b];
        bool ca = false, cb = false;
        if (lane < na) {
          const float4 x = padded_sphere<PADDED_COPY>(rv, es, sa + lane);
          const float dx = x.x - B.x, dy = x.y - B.y, dz = x.z - B.z, rs = x.w + B.w;
          ca = (x.w >= 0.0f) && (dx * dx + dy * dy + dz * dz < rs * rs);
        }
        if (lane < nb) {
          const float4 y = padded_sphere<PADDED_COPY>(rv, es, sb + lane);
          const float dx = y.x - A.x, dy = y.y - A.y, dz = y.z - A.z, rs = y.w + A.w;
          cb = (y.w >= 0.0f) && (dx * dx + dy * dy + dz * dz < rs * rs);
        }
        const unsigned ma = __ballot_sync(kFull, ca), mb = __ballot_sync(kFull, cb);
        if (ma == 0u || mb == 0u) continue;
        unsigned char *ia = idx_scratch != nullptr ? idx_scratch : reinterpret_cast<unsigned char *>(es.ft), *ib = ia + 32;
        const unsigned lt = (1u << lane) - 1u;
        if (ca) ia[__popc(ma & lt)] = (unsigned char)lane;
        if (cb) ib[__popc(mb & lt)] = (unsigned char)lane;
        __syncwarp();
        const int na2 = __popc(ma), nb2 = __popc(mb);
        const float inv_nb2 = 1.0f / (float)nb2;
        #pragma unroll 1
        for (int t = lane; t < na2 * nb2; t += 32) {
          const int io = (int)(((float)t + 0.5f) * inv_nb2);
          const int i = sa + ia[io], j = sb + ib[t - io * nb2];
          const float4 x = padded_sphere<PADDED_COPY>(rv, es, i), y = padded_sphere<PADDED_COPY>(rv, es, j);
          const float rs = x.w + y.w;
          const float dx = x.x - y.x, dy = x.y - y.y, dz = x.z - y.z;
          const float f = rs * rs - (dx * dx + dy * dy + dz * dz);
          if (f > 0.0f) {  // candidates already have non-negative radii
            const unsigned long long k = ((unsigned long long)__float_as_uint(f) << 32) |
                                         ((unsigned long long)(0xffffu - (unsigned)i) << 16) | (0xffffu - (unsigned)j);
            key = k > key ? k : key;
          }
        }
        __syncwarp();  // the index scratch is rewritten for the next block
        continue;
      }
      const float inv_nb = 1.0f / (float)nb;
      #pragma unroll 1
      for (int t = lane; t < na * nb; t += W) {
        const int io = (int)(((float)t + 0.5f) * inv_nb);
        const int i = sa + io, j = sb + (t - io * nb);
        const float4 x = padded_sphere<PADDED_COPY>(rv, es, i), y = padded_sphere<PADDED_COPY>(rv, es, j);
        const float rs = x.w + y.w;
        const float dx = x.x - y.x, dy = x.y - y.y, dz = x.z - y.z;
        const float f = rs * rs - (dx * dx + dy * dy + dz * dz);
        if (f > 0.0f && x.w >= 0.0f && y.w >= 0.0f) {
          const unsigned long long k = ((unsigned long long)__float_as_uint(f) << 32) |
                                       ((unsigned long long)(0xffffu - (unsigned)i) << 16) | (0xffffu - (unsigned)j);
          key = k > key ? k : key;
        }
      }
    }
    if (ANY && row_ballot<W>(key != 0ull) != 0u) break;
  }
#pragma unroll
  for (int o = W / 2; o > 0; o >>= 1) {
    const unsigned long long other = row_shfl_xor<W>(key, o);
    key = other > key ? other : key;
  }
  if (key_out != nullptr) *key_out = key;
  bi = bj = 0;
  if (key == 0ull) return 0.0f;
  bi = 0xffff - (int)((key >> 16) & 0xffffu);
  bj = 0xffff - (int)(key & 0xffffu);
  return __uint_as_float((uint32_t)(key >> 32));
}

// ----------------------------------------------------------------------------------------------
// J^T backward on link force/torque accumulators.
//   per link k:    F_k = sum g_s ,  T_k = sum (p_s - o_k) x g_s   (+ tool-frame g_pos / omega)
//   per joint link j: (F,T)_sub = sum over descendants k of shift_to_o_j(F_k, T_k)
//   revolute: s * a_j . T_sub      prismatic: s * a_j . F_sub
// Algebraically the reference's per-sphere chain walk (kinematics_backward_helper.cuh:15-183,
// kinematics_joint_util.cuh:12-67): g.(a x (p-o_j)) = a.((p-o_j) x g).
// gq_out[d] = gqv[d] + sum over links driven by joint d.
// ----------------------------------------------------------------------------------------------
template <int W = 32>
__device__ __forceinline__ void warp_fk_upsweep(const RobotView &rv, const EvalSmem &es, int lane, float *gq_out);
template <int W = 32>
__device__ __forceinline__ void warp_fk_backward(const RobotView &rv, const EvalSmem &es, int lane, float *gq_out) {
  #pragma unroll 1
  for (int k = lane; k < rv.nl; k += W) {
    const float *Tk = es.cumul + 12 * k;
    const V3 o = mk3(Tk[3], Tk[7], Tk[11]);
    V3 F = mk3(0, 0, 0), T = mk3(0, 0, 0);
    #pragma unroll 1
    for (int i = rv.link_sph_off[k]; i < rv.link_sph_off[k + 1]; ++i) {
      const int s = rv.link_sph_idx[i];
      const float4 g4 = es.gsph[s];
      const V3 g = mk3(g4.x, g4.y, g4.z);
      if (g.x == 0.0f && g.y == 0.0f && g.z == 0.0f) continue;
      const float4 p4 = es.sph[s];
      F = F + g;
      T = T + cross(mk3(p4.x, p4.y, p4.z) - o, g);
    }
    for (int e = 0; e < rv.L; ++e) {
      if (rv.tool_map[e] != k) continue;
      F = F + mk3(es.pose_g[8 * e + 0], es.pose_g[8 * e + 1], es.pose_g[8 * e + 2]);
      T = T + mk3(es.pose_g[8 * e + 4], es.pose_g[8 * e + 5], es.pose_g[8 * e + 6]);
    }
    float *ft = es.ft + 8 * k;
    ft[0] = F.x;
    ft[1] = F.y;
    ft[2] = F.z;
    ft[4] = T.x;
    ft[5] = T.y;
    ft[6] = T.z;
  }
  row_sync<W>();
  warp_fk_upsweep<W>(rv, es, lane, gq_out);
}

// second half of the J^T backward: per-link (F, T) accumulators in es.ft -> joint gradients
template <int W>
__device__ __forceinline__ void warp_fk_upsweep(const RobotView &rv, const EvalSmem &es, int lane, float *gq_out) {
  #pragma unroll 1
  for (int j = lane; j < rv.nl; j += W) {
    const int jt = rv.joint_type[j];
    float res = 0.0f;
    if (jt >= 0) {
      const float *Tj = es.cumul + 12 * j;
      const V3 oj = mk3(Tj[3], Tj[7], Tj[11]);
      V3 F = mk3(0, 0, 0), T = mk3(0, 0, 0);
      #pragma unroll 1
      for (int k = j; k < rv.nl; ++k) {
        if (!((rv.anc_mask[k] >> j) & 1ull)) continue;
        const float *ft = es.ft + 8 * k;
        const V3 Fk = mk3(ft[0], ft[1], ft[2]);
        const float *Tk = es.cumul + 12 * k;
        const V3 ok = mk3(Tk[3], Tk[7], Tk[11]);
        F = F + Fk;
        T = T + mk3(ft[4], ft[5], ft[6]) + cross(ok - oj, Fk);
      }
      const int ax = (jt >= JT_XR) ? jt - JT_XR : jt;
      const V3 a = mk3(Tj[ax], Tj[4 + ax], Tj[8 + ax]);
      res = rv.joff[2 * j] * ((jt >= JT_XR) ? dot(a, T) : dot(a, F));
    }
    es.contrib[j] = res;
  }
  row_sync<W>();
  for (int d = lane; d < rv.D; d += W) {
    float g = es.gqv[d];
    for (int i = rv.jl_off[d]; i < rv.jl_off[d + 1]; ++i) g += es.contrib[rv.jl_idx[i]];
    gq_out[d] = g;
  }
}

// Dense fallback, out of line: rarely taken, and inlining it would only bloat the instruction footprint of the
// hot path.  Views are rebuilt from raw pointers so that the caller's RobotView/EvalSmem stay in registers.
template <int W = 32>
static __device__ __noinline__ void warp_fk_backward_cold(const unsigned char *smem_blob, const unsigned char *gmem_blob,
                                                          float *eval_base, int lane, float *gq_out) {
  const RobotView rv = make_robot_view(smem_blob, gmem_blob);
  const EvalSmem es = carve_eval_smem(eval_base, rv.nl, rv.D, rv.S, rv.L, rv.n_cl);
  warp_fk_backward<W>(rv, es, lane, gq_out);
}

// ----------------------------------------------------------------------------------------------
// Same J^T backward, transposed for SPARSE sphere gradients (the common case: self-collision touches two
// spheres, scene collision only the colliding ones): lanes own links (up to 64 = 2 per lane); every sphere
// or tool frame with a non-zero gradient is broadcast to the warp and each lane whose link is an ancestor
// adds  s * a . ((p - o) x g [+ omega])  (revolute) or  s * a . g  (prismatic)  -- the reference's per-sphere
// chain walk (kinematics_backward_helper.cuh:15-99) with the chain laid across lanes.
// Returns false (nothing written) when the gradient is dense; the caller then uses warp_fk_backward.
// ----------------------------------------------------------------------------------------------
// SMALL = true (arm build: <= 24 links, so one link per lane, and <= 128 spheres): the second link slot is compiled out and the
// tool frames ride through the same broadcast loop as the spheres (entries S .. S + L - 1) -- one copy of the accumulate code
// instead of two; the row's instruction footprint is what that kernel is short of.
// W = 16 (half-warp rows): SMALL only, and the robot has <= 16 links.
template <bool SMALL = false, int W = 32>
__device__ __forceinline__ bool warp_fk_backward_sparse(const RobotView &rv, const EvalSmem &es, int lane, float *gq_out,
                                                        int nnz) {
  static_assert(W == 32 || SMALL, "half-warp rows take the one-link-per-lane form");
  if (nnz > 2 * rv.nl) return false;  // nnz = spheres with a non-zero gradient (counted by the caller)
  if (SMALL) {
    float sc = 0.0f;
    V3 ax = mk3(0, 0, 0), og = mk3(0, 0, 0);
    int jt = -1;
    if (lane < rv.nl) {
      jt = rv.joint_type[lane];
      if (jt >= 0) {
        const float *Tj = es.cumul + 12 * lane;
        const int a = (jt >= JT_XR) ? jt - JT_XR : jt;
        ax = mk3(Tj[a], Tj[4 + a], Tj[8 + a]);
        og = mk3(Tj[3], Tj[7], Tj[11]);
        sc = rv.joff[2 * lane];
      }
    }
    float acc = 0.0f;
    const int n_entries = rv.S + rv.L;
#pragma unroll 1
    for (int base = 0; base < n_entries; base += W) {
      const int s = base + lane;
      bool nz = false;
      if (s < rv.S) {
        const float4 g = es.gsph[s];
        nz = (g.x != 0.0f) || (g.y != 0.0f) || (g.z != 0.0f);
      } else if (s < n_entries) {
        const float *pg = es.pose_g + 8 * (s - rv.S);
        nz = pg[0] != 0.0f || pg[1] != 0.0f || pg[2] != 0.0f || pg[4] != 0.0f || pg[5] != 0.0f || pg[6] != 0.0f;
      }
      unsigned m = row_ballot<W>(nz);
      while (m) {
        const int ss = base + __ffs(m) - 1;
        m &= m - 1;
        V3 p, g, om = mk3(0, 0, 0);
        int k;
        if (ss < rv.S) {
          const float4 g4 = es.gsph[ss], p4 = es.sph[ss];
          k = rv.sph_link[ss];
          p = mk3(p4.x, p4.y, p4.z);
          g = mk3(g4.x, g4.y, g4.z);
        } else {
          const float *pg = es.pose_g + 8 * (ss - rv.S);
          k = rv.tool_map[ss - rv.S];
          const float *Tk = es.cumul + 12 * k;
          p = mk3(Tk[3], Tk[7], Tk[11]);
          g = mk3(pg[0], pg[1], pg[2]);
          om = mk3(pg[4], pg[5], pg[6]);
        }
        if (jt >= 0 && ((rv.anc_mask[k] >> lane) & 1ull))
          acc += (jt >= JT_XR) ? sc * (dot(ax, cross(p - og, g)) + dot(ax, om)) : sc * dot(ax, g);
      }
    }
    if (lane < rv.nl) es.contrib[lane] = acc;
    row_sync<W>();
    for (int d = lane; d < rv.D; d += W) {
      float g = es.gqv[d];
      for (int i = rv.jl_off[d]; i < rv.jl_off[d + 1]; ++i) g += es.contrib[rv.jl_idx[i]];
      gq_out[d] = g;
    }
    return true;
  }
  const int nu = rv.nl > 32 ? 2 : 1;
  // per-lane link constants (slot 0: link lane, slot 1: link lane + 32)
  V3 ax[2], og[2];
  float sc[2];
  int jt[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int j = lane + 32 * u;
    jt[u] = -1;
    if (u >= nu) continue;
    sc[u] = 0.0f;
    ax[u] = og[u] = mk3(0, 0, 0);
    if (j < rv.nl) {
      jt[u] = rv.joint_type[j];
      if (jt[u] >= 0) {
        const float *Tj = es.cumul + 12 * j;
        const int a = (jt[u] >= JT_XR) ? jt[u] - JT_XR : jt[u];
        ax[u] = mk3(Tj[a], Tj[4 + a], Tj[8 + a]);
        og[u] = mk3(Tj[3], Tj[7], Tj[11]);
        sc[u] = rv.joff[2 * j];
      }
    }
  }
  float acc[2] = {0.0f, 0.0f};
  auto add = [&](unsigned long long mask, V3 p, V3 g, V3 om) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = lane + 32 * u;
      if (u < nu && jt[u] >= 0 && ((mask >> j) & 1ull)) {
        acc[u] += (jt[u] >= JT_XR) ? sc[u] * (dot(ax[u], cross(p - og[u], g)) + dot(ax[u], om)) : sc[u] * dot(ax[u], g);
      }
    }
  };
  #pragma unroll 1
  for (int base = 0; base < rv.S; base += 32) {
    const int s = base + lane;
    bool nz = false;
    if (s < rv.S) {
      const float4 g = es.gsph[s];
      nz = (g.x != 0.0f) || (g.y != 0.0f) || (g.z != 0.0f);
    }
    unsigned m = __ballot_sync(kFull, nz);
    while (m) {
      const int ss = base + __ffs(m) - 1;
      m &= m - 1;
      const float4 g4 = es.gsph[ss], p4 = es.sph[ss];
      add(rv.anc_mask[rv.sph_link[ss]], mk3(p4.x, p4.y, p4.z), mk3(g4.x, g4.y, g4.z), mk3(0, 0, 0));
    }
  }
  #pragma unroll 1
  for (int t = 0; t < rv.L; ++t) {
    const float *pg = es.pose_g + 8 * t;
    const V3 g = mk3(pg[0], pg[1], pg[2]), om = mk3(pg[4], pg[5], pg[6]);
    if (g.x == 0.0f && g.y == 0.0f && g.z == 0.0f && om.x == 0.0f && om.y == 0.0f && om.z == 0.0f) continue;
    const int k = rv.tool_map[t];
    const float *Tk = es.cumul + 12 * k;
    add(rv.anc_mask[k], mk3(Tk[3], Tk[7], Tk[11]), g, om);
  }
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int j = lane + 32 * u;
    if (j < rv.nl) es.contrib[j] = acc[u];
  }
  __syncwarp();
  for (int d = lane; d < rv.D; d += 32) {
    float g = es.gqv[d];
    for (int i = rv.jl_off[d]; i < rv.jl_off[d + 1]; ++i) g += es.contrib[rv.jl_idx[i]];
    gq_out[d] = g;
  }
  return true;
}

// ----------------------------------------------------------------------------------------------
// Big-robot layout: the sphere gradients of a row live in a short list (es.glist: g.xyz + sphere index, in sphere order) instead
// of a dense [S] array.  The list is consumed either by the sparse J^T (lanes own links, entries broadcast) or -- when a row
// fills it -- drained into the per-link (F, T) accumulators, deterministically in list order.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void warp_zero_ft(const RobotView &rv, const EvalSmem &es, int lane) {
  for (int k = lane; k < rv.nl * 2; k += 32) reinterpret_cast<float4 *>(es.ft)[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncwarp();
}
__device__ __forceinline__ void warp_drain_list_to_ft(const RobotView &rv, const EvalSmem &es, int lane, int n) {
#pragma unroll 1
  for (int i = 0; i < n; ++i) {
    const float4 g4 = es.glist[i];
    const int s = __float_as_int(g4.w);
    const float4 p4 = es.sph[s];
    const int k = rv.sph_link[s];
    const float *Tk = es.cumul + 12 * k;
    const V3 g = mk3(g4.x, g4.y, g4.z);
    const V3 tq = cross(mk3(p4.x - Tk[3], p4.y - Tk[7], p4.z - Tk[11]), g);
    if (lane < 6) {
      const float v = lane == 0 ? g.x : lane == 1 ? g.y : lane == 2 ? g.z : lane == 3 ? tq.x : lane == 4 ? tq.y : tq.z;
      es.ft[8 * k + lane + (lane >= 3 ? 1 : 0)] += v;
    }
    __syncwarp();
  }
}
// dense finish: tool-frame gradients into the accumulators (one lane, frame order), then the up-sweep
__device__ __forceinline__ void warp_fk_backward_from_ft(const RobotView &rv, const EvalSmem &es, int lane, float *gq_out) {
  if (lane == 0) {
    for (int t = 0; t < rv.L; ++t) {
      float *ft = es.ft + 8 * rv.tool_map[t];
      const float *pg = es.pose_g + 8 * t;
      ft[0] += pg[0];
      ft[1] += pg[1];
      ft[2] += pg[2];
      ft[4] += pg[4];
      ft[5] += pg[5];
      ft[6] += pg[6];
    }
  }
  __syncwarp();
  warp_fk_upsweep(rv, es, lane, gq_out);
}
// sparse J^T over a list of (gradient, sphere) entries (the transposed chain walk of warp_fk_backward_sparse with the list as
// the source): lane j (and j + 32) accumulates the contribution to joint link j; `with_tools` adds the tool-frame gradients.
__device__ __forceinline__ void warp_list_accumulate(const RobotView &rv, const EvalSmem &es, int lane, const float4 *list, int n,
                                                     bool with_tools, float (&acc)[2]) {
  const int nu = rv.nl > 32 ? 2 : 1;
  V3 ax[2], og[2];
  float sc[2];
  int jt[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int j = lane + 32 * u;
    jt[u] = -1;
    if (u >= nu) continue;
    sc[u] = 0.0f;
    ax[u] = og[u] = mk3(0, 0, 0);
    if (j < rv.nl) {
      jt[u] = rv.joint_type[j];
      if (jt[u] >= 0) {
        const float *Tj = es.cumul + 12 * j;
        const int a = (jt[u] >= JT_XR) ? jt[u] - JT_XR : jt[u];
        ax[u] = mk3(Tj[a], Tj[4 + a], Tj[8 + a]);
        og[u] = mk3(Tj[3], Tj[7], Tj[11]);
        sc[u] = rv.joff[2 * j];
      }
    }
  }
  acc[0] = acc[1] = 0.0f;
  auto add = [&](unsigned long long mask, V3 p, V3 g, V3 om) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = lane + 32 * u;
      if (u < nu && jt[u] >= 0 && ((mask >> j) & 1ull)) {
        acc[u] += (jt[u] >= JT_XR) ? sc[u] * (dot(ax[u], cross(p - og[u], g)) + dot(ax[u], om)) : sc[u] * dot(ax[u], g);
      }
    }
  };
#pragma unroll 1
  for (int i = 0; i < n; ++i) {
    const float4 g4 = list[i];
    const int s = __float_as_int(g4.w);
    const float4 p4 = es.sph[s];
    add(rv.anc_mask[rv.sph_link[s]], mk3(p4.x, p4.y, p4.z), mk3(g4.x, g4.y, g4.z), mk3(0, 0, 0));
  }
  if (with_tools) {
#pragma unroll 1
    for (int t = 0; t < rv.L; ++t) {
      const float *pg = es.pose_g + 8 * t;
      const V3 g = mk3(pg[0], pg[1], pg[2]), om = mk3(pg[4], pg[5], pg[6]);
      if (g.x == 0.0f && g.y == 0.0f && g.z == 0.0f && om.x == 0.0f && om.y == 0.0f && om.z == 0.0f) continue;
      const int k = rv.tool_map[t];
      const float *Tk = es.cumul + 12 * k;
      add(rv.anc_mask[k], mk3(Tk[3], Tk[7], Tk[11]), g, om);
    }
  }
}

// sparse J^T over the list (the transposed chain walk of warp_fk_backward_sparse with the list as the source)
// SMALL: as in warp_fk_backward_sparse (<= 24 links: one link per lane; tool frames go through the same loop as the list).
template <bool SMALL = false>
__device__ __forceinline__ void warp_fk_backward_list(const RobotView &rv, const EvalSmem &es, int lane, float *gq_out, int n) {
  if (SMALL) {
    float sc = 0.0f;
    V3 ax = mk3(0, 0, 0), og = mk3(0, 0, 0);
    int jt = -1;
    if (lane < rv.nl) {
      jt = rv.joint_type[lane];
      if (jt >= 0) {
        const float *Tj = es.cumul + 12 * lane;
        const int a = (jt >= JT_XR) ? jt - JT_XR : jt;
        ax = mk3(Tj[a], Tj[4 + a], Tj[8 + a]);
        og = mk3(Tj[3], Tj[7], Tj[11]);
        sc = rv.joff[2 * lane];
      }
    }
    float acc = 0.0f;
#pragma unroll 1
    for (int i = 0; i < n + rv.L; ++i) {
      V3 p, g, om = mk3(0, 0, 0);
      int k;
      if (i < n) {
        const float4 g4 = es.glist[i];
        const int s = __float_as_int(g4.w);
        const float4 p4 = es.sph[s];
        k = rv.sph_link[s];
        p = mk3(p4.x, p4.y, p4.z);
        g = mk3(g4.x, g4.y, g4.z);
      } else {
        const float *pg = es.pose_g + 8 * (i - n);
        k = rv.tool_map[i - n];
        const float *Tk = es.cumul + 12 * k;
        p = mk3(Tk[3], Tk[7], Tk[11]);
        g = mk3(pg[0], pg[1], pg[2]);
        om = mk3(pg[4], pg[5], pg[6]);
        if (g.x == 0.0f && g.y == 0.0f && g.z == 0.0f && om.x == 0.0f && om.y == 0.0f && om.z == 0.0f) continue;
      }
      if (jt >= 0 && ((rv.anc_mask[k] >> lane) & 1ull))
        acc += (jt >= JT_XR) ? sc * (dot(ax, cross(p - og, g)) + dot(ax, om)) : sc * dot(ax, g);
    }
    if (lane < rv.nl) es.contrib[lane] = acc;
    __syncwarp();
    for (int d = lane; d < rv.D; d += 32) {
      float g = es.gqv[d];
      for (int i = rv.jl_off[d]; i < rv.jl_off[d + 1]; ++i) g += es.contrib[rv.jl_idx[i]];
      gq_out[d] = g;
    }
    return;
  }
  const int nu = rv.nl > 32 ? 2 : 1;
  V3 ax[2], og[2];
  float sc[2];
  int jt[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int j = lane + 32 * u;
    jt[u] = -1;
    if (u >= nu) continue;
    sc[u] = 0.0f;
    ax[u] = og[u] = mk3(0, 0, 0);
    if (j < rv.nl) {
      jt[u] = rv.joint_type[j];
      if (jt[u] >= 0) {
        const float *Tj = es.cumul + 12 * j;
        const int a = (jt[u] >= JT_XR) ? jt[u] - JT_XR : jt[u];
        ax[u] = mk3(Tj[a], Tj[4 + a], Tj[8 + a]);
        og[u] = mk3(Tj[3], Tj[7], Tj[11]);
        sc[u] = rv.joff[2 * j];
      }
    }
  }
  float acc[2] = {0.0f, 0.0f};
  auto add = [&](unsigned long long mask, V3 p, V3 g, V3 om) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = lane + 32 * u;
      if (u < nu && jt[u] >= 0 && ((mask >> j) & 1ull)) {
        acc[u] += (jt[u] >= JT_XR) ? sc[u] * (dot(ax[u], cross(p - og[u], g)) + dot(ax[u], om)) : sc[u] * dot(ax[u], g);
      }
    }
  };
#pragma unroll 1
  for (int i = 0; i < n; ++i) {
    const float4 g4 = es.glist[i];
    const int s = __float_as_int(g4.w);
    const float4 p4 = es.sph[s];
    add(rv.anc_mask[rv.sph_link[s]], mk3(p4.x, p4.y, p4.z), mk3(g4.x, g4.y, g4.z), mk3(0, 0, 0));
  }
#pragma unroll 1
  for (int t = 0; t < rv.L; ++t) {
    const float *pg = es.pose_g + 8 * t;
    const V3 g = mk3(pg[0], pg[1], pg[2]), om = mk3(pg[4], pg[5], pg[6]);
    if (g.x == 0.0f && g.y == 0.0f && g.z == 0.0f && om.x == 0.0f && om.y == 0.0f && om.z == 0.0f) continue;
    const int k = rv.tool_map[t];
    const float *Tk = es.cumul + 12 * k;
    add(rv.anc_mask[k], mk3(Tk[3], Tk[7], Tk[11]), g, om);
  }
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int j = lane + 32 * u;
    if (j < rv.nl) es.contrib[j] = acc[u];
  }
  __syncwarp();
  for (int d = lane; d < rv.D; d += 32) {
    float g = es.gqv[d];
    for (int i = rv.jl_off[d]; i < rv.jl_off[d + 1]; ++i) g += es.contrib[rv.jl_idx[i]];
    gq_out[d] = g;
  }
}

// ----------------------------------------------------------------------------------------------
// Bulk async copy (TMA 1-D) of the blob prefix into shared memory, completion on an mbarrier.
// ----------------------------------------------------------------------------------------------
#ifdef CB200_SIMT_EMULATION
// host emulation build (tests/simt): no TMA engine -- the CTA's threads copy the blob and meet at a barrier
__device__ __forceinline__ void stage_blob_to_smem(unsigned char *dst, const unsigned char *src, uint32_t bytes,
                                                   unsigned long long *mbar) {
  (void)mbar;
  for (uint32_t i = threadIdx.x; i < bytes; i += blockDim.x) dst[i] = src[i];
  __syncthreads();
}
#else
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void stage_blob_to_smem(unsigned char *dst, const unsigned char *src, uint32_t bytes,
                                                   unsigned long long *mbar) {
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(mbar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(mbar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(mbar))
                 : "memory");
  }
  // every thread waits for phase 0 of the barrier
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(mbar))
        : "memory");
  }
}
#endif  // CB200_SIMT_EMULATION

}  // namespace cb200
