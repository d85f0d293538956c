"""Robot segmentation of depth images (cb200_segment_robot_depth, curobo_b200.perception.RobotSegmenter).

(1) The kernel equals the float64 oracle (oracle/robot_mask_oracle.py) on rendered scenes of Franka, G1-29 and G1-43 -- the
robot's spheres, a back wall, a box and zero / NaN / inf pixels -- with one robot state for every image and one per image; masks
may differ only at pixels whose margin is within 1e-5 m of the threshold, which must be under 0.1 % of the pixels, and
`filtered` is where(mask, 0, depth) bit for bit.  (2) The reference's own outputs (tests/golden/robot_mask_reference_golden.npz).
(3) The tile cull is exact on adversarial tiles: far walls behind silhouettes, spheres 1e-4 m outside and inside a tile's
inflated box, tiles without a valid pixel, image sizes that are not multiples of the tile.  (4) Attached objects are masked
and disabled links are not when the segmenter shares a RolloutEngine's link spheres.  (5) Graph capture.  (6) The refusals."""
import dataclasses
import os

import numpy as np
import pytest
import torch

from helpers import random_q
from curobo_b200 import lib as cblib
from curobo_b200.backends import pba as pba_cu
from curobo_b200.perception import RobotSegmenter
from curobo_b200.robot_model import load_robot
from curobo_b200.rollout import RolloutConfig, RolloutEngine
from oracle import robot_mask_oracle as M
from oracle import rollout_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
INVALID = 1  # cudaErrorInvalidValue
EPS = 1e-5
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "robot_mask_reference_golden.npz")


def T(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t.to(dt) if dt is not None else t


def robot_q(rm, n, seed):
    return random_q(rm, n, seed=seed, scale=0.3)


def spheres_of(rm, q, link_spheres=None):
    if link_spheres is not None:
        rm = dataclasses.replace(rm, link_spheres=np.asarray(link_spheres)[:1])
    return O.fk_forward(rm, q)[1].astype(np.float32)                           # [n, S, 4]


def scene(spheres, n_img, hw, seed, invalid=(0.02, 0.005, 0.005), extra=()):
    """Cameras on the +x side of the robot looking at it, a back wall behind it and a box beside it; image b renders
    spheres[b] (or spheres[0] when one state serves every image) plus `extra` spheres, each 5 mm inside its collision sphere
    as a real surface is, so that no robot pixel lies on the threshold when it is 0."""
    spheres = np.concatenate([spheres, np.broadcast_to(np.asarray(extra, np.float32).reshape(1, -1, 4),
                                                       (len(spheres), len(extra), 4))], 1) if len(extra) else spheres
    spheres = np.concatenate([spheres[..., :3], spheres[..., 3:] - 0.005], -1)
    live = spheres[0][spheres[0][:, 3] > 0]
    c = 0.5 * (live[:, :3].min(0) + live[:, :3].max(0))
    ext = float(np.max(live[:, :3].max(0) - live[:, :3].min(0)))
    dist = 1.4 * ext + 1.0
    eyes = [c + dist * np.array([np.cos(a), np.sin(a), 0.35]) for a in np.linspace(-0.5, 0.5, n_img)]
    K, pos, quat = M.cameras(eyes, c, hw)
    wall = (c - np.array([0.8 * ext + 0.5, 0.0, 0.0]), np.array([1.0, 0.0, 0.0]))
    boxes = [(c + np.array([-0.1, 0.45 * ext + 0.25, -0.3 * ext]), c + np.array([0.1, 0.45 * ext + 0.45, -0.1 * ext]))]
    depth = np.stack([M.render_depth(K[b:b + 1], pos[b:b + 1], quat[b:b + 1], hw,
                                     spheres=spheres[b if len(spheres) > 1 else 0], wall=wall,
                                     boxes=boxes, invalid=invalid, seed=seed + b)[0] for b in range(n_img)])
    return K, pos, quat, depth


def run_kernel(depth, K, pos, quat, spheres, thr):
    b, h, w = depth.shape
    mask = torch.empty((b, h, w), dtype=torch.bool, device=DEV)
    filt = torch.empty((b, h, w), dtype=torch.float32, device=DEV)
    pba_cu.launch_segment_robot_depth(T(depth), T(K), T(pos), T(quat), T(spheres), thr, mask, filt)
    return mask.cpu().numpy(), filt.cpu().numpy()


def check(mask, filt, depth, K, pos, quat, spheres, thr, what=""):
    want, _, margin = M.robot_mask(depth, K, pos, quat, spheres, thr)
    near = np.abs(np.nan_to_num(margin, nan=1.0, posinf=1.0, neginf=-1.0)) <= EPS
    assert near.mean() < 1e-3, f"{what}: {near.mean():.4%} of pixels within {EPS} m of the threshold"
    bad = np.argwhere((mask != want) & ~near)
    assert bad.size == 0, f"{what}: {len(bad)} pixels differ from the oracle, e.g. {bad[:5].tolist()}"
    ref = np.where(mask, np.float32(0), depth).astype(np.float32)
    assert np.array_equal(filt.view(np.uint32), ref.view(np.uint32)), f"{what}: filtered is not where(mask, 0, depth)"
    return int(near.sum()), float(want.mean())


@pytest.mark.parametrize("robot", ["franka", "g1_29", "g1_43"])
@pytest.mark.parametrize("per_image", [False, True])
def test_kernel_vs_oracle(robot, per_image, n_img=2, hw=(480, 640), thresholds=(0.05, 0.0)):
    rm = load_robot(robot)
    q = robot_q(rm, n_img if per_image else 1, seed=3)
    sph = spheres_of(rm, q)
    K, pos, quat, depth = scene(sph, n_img, hw, seed=7)
    for thr in thresholds:
        mask, filt = run_kernel(depth, K, pos, quat, sph, thr)
        near, share = check(mask, filt, depth, K, pos, quat, sph, thr, f"{robot} thr {thr}")
        assert 0.01 < share < 0.6, f"{robot}: {share:.2%} of pixels masked; the scene does not exercise the mask"
        print(f"{robot} robot batch {len(q)} thr {thr}: {share:.2%} masked, {near} pixels within {EPS} m of the threshold")


def test_segmenter_vs_oracle(robot="franka", n_img=2, hw=(480, 640)):
    """get_robot_mask: FK drop-in then the kernel, for q [dof], [1, dof] and [B, dof]."""
    rm = load_robot(robot)
    seg = RobotSegmenter(rm, DEV, distance_threshold=0.03)
    q = robot_q(rm, n_img, seed=5)
    sph = spheres_of(rm, q)
    K, pos, quat, depth = scene(sph, n_img, hw, seed=9)
    for qq, s in ((q[0], sph[:1]), (q[:1], sph[:1]), (q, sph)):
        mask, filt = seg.get_robot_mask(T(depth), T(K), T(pos), T(quat), T(qq))
        assert mask.dtype == torch.bool and filt.dtype == torch.float32 and tuple(mask.shape) == depth.shape
        check(mask.cpu().numpy(), filt.cpu().numpy(), depth, K, pos, quat, s, 0.03, f"q {qq.shape}")


def test_reference_golden():
    g = np.load(GOLDEN)
    for name in sorted({k.split("/")[0] for k in g.files}):
        c = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}
        mask, filt = run_kernel(c["depth"], c["K"], c["pos"], c["quat"], c["spheres"], float(c["threshold"]))
        want = c["mask"].astype(bool)
        near = np.abs(np.nan_to_num(c["margin"], nan=1.0, posinf=1.0, neginf=-1.0)) <= EPS
        bad = np.argwhere((mask != want) & ~near)
        assert bad.size == 0, f"{name}: {len(bad)} pixels differ from the reference, e.g. {bad[:5].tolist()}"
        assert np.array_equal(filt.view(np.uint32), np.where(mask, np.float32(0), c["depth"]).astype(np.float32).view(np.uint32))


def adversarial_case(hw=(37, 45), seed=0):
    """One camera at the origin looking down +z with fx = fy = 1 and cx = cy = 0, so pixel (u, v) at depth d is (u d, v d, d):
    tile boxes are known exactly.  Tiles of near silhouettes (d = 1) over a far wall (d = 40), a tile with no valid pixel, and
    spheres placed 1e-4 m outside and inside the inflated box of single tiles."""
    H, W = hw
    rng = np.random.default_rng(seed)
    K = np.array([[[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1]]], np.float32)
    pos = np.zeros((1, 3), np.float32)
    quat = np.array([[1.0, 0, 0, 0]], np.float32)
    depth = np.full((1, H, W), 40.0, np.float32)
    depth[0, 8:16, :] = np.where(rng.random((8, W)) < 0.3, np.float32(1.0), np.float32(40.0))       # silhouettes on a far wall
    depth[0, 0:8, 0:32] = np.array([0.0, np.nan, np.inf, -1.0], np.float32)[rng.integers(0, 4, (8, 32))]  # no valid pixel
    depth[0, 16:24, 0:32] = 0.5                                                                       # a flat tile
    depth[0, 24:32, 32:] = 2.0                                                                        # a partial tile
    thr = 0.02
    sph = []
    # the flat tile's box: x in [0, 15.5], y in [8, 11.5], z = 0.5; corner (15.5, 11.5, 0.5)
    corner = np.array([31 * 0.5, 23 * 0.5, 0.5])
    d = np.array([1.0, 1.0, 1.0]) / np.sqrt(3.0)
    for r, gap in ((0.3, 1e-4), (0.25, -1e-4)):
        sph.append(np.r_[corner + d * (r + thr + gap), r])
    # the partial tile's box: x in [64, 88], y in [48, 62], z = 2; spheres beyond its far corner, above its face
    corner = np.array([44 * 2.0, 31 * 2.0, 2.0])
    sph.append(np.r_[corner + d * (0.4 + thr + 1e-4), 0.4])
    sph.append(np.r_[corner + d * (0.4 + thr - 1e-4), 0.4])
    sph.append(np.r_[70.0, 54.0, 2.0 - (0.3 + thr + 1e-4), 0.3])
    sph.append(np.r_[70.0, 54.0, 2.0 - (0.3 + thr - 1e-4), 0.3])
    # silhouettes: spheres around near points, and one at the far wall that only far points reach
    for _ in range(12):
        u, v = rng.integers(0, W), rng.integers(8, 16)
        sph.append(np.r_[u * 1.0 + rng.normal(0, 0.3), v * 1.0 + rng.normal(0, 0.3), 1.0 + rng.normal(0, 0.1), 0.2])
    sph.append(np.r_[20 * 40.0, 12 * 40.0, 40.0, 1.0])
    sph.append(np.r_[0.0, 0.0, 0.0, -100.0])                                      # disabled
    return depth, K, pos, quat, np.asarray(sph, np.float32)[None], thr


def test_cull_exact_on_adversarial_tiles():
    depth, K, pos, quat, sph, thr = adversarial_case()
    mask, filt = run_kernel(depth, K, pos, quat, sph, thr)
    check(mask, filt, depth, K, pos, quat, sph, thr, "adversarial")
    assert not mask[0, 0:8, 0:32].any()
    assert mask[0, 23, 31] and mask[0, 31, 44]                                    # the spheres 1e-4 m inside hit their corners
    assert mask[0, 8:16].any() and not mask[0, 8:16].all()
    # the same with each inside sphere alone, so that no other sphere can keep the tile alive
    for k in (1, 3, 5):
        one = sph[:, k:k + 1]
        m, f = run_kernel(depth, K, pos, quat, one, thr)
        check(m, f, depth, K, pos, quat, one, thr, f"sphere {k}")
        assert m.sum() >= 1
    for k in (0, 2, 4):
        m, _ = run_kernel(depth, K, pos, quat, sph[:, k:k + 1], thr)
        assert not m.any()
    for hw in ((1, 1), (9, 33), (17, 63)):                                         # sizes that are not multiples of the tile
        d = np.ascontiguousarray(depth[:, :hw[0], :hw[1]])
        m, f = run_kernel(d, K, pos, quat, sph, thr)
        check(m, f, d, K, pos, quat, sph, thr, f"{hw}")



def test_cull_exact_at_one_ulp():
    """A tile whose box corners are not pixels: valid pixels A (3, 6), B (10, 3), C (5, 1) at one depth, so B lies on the box's
    x = max face but at no corner.  A sphere beyond that face and below the depth plane has the same per-axis gaps to the box as
    to B, so the cull's bound equals B's distance.  With r the smallest float whose square exceeds that distance B is masked by
    one step of r; with the next float down nothing is.  The points are reproduced in float32 with the kernel's operations
    (identity camera pose), so the expected mask is exact and a cull that rounds differently from the pixel test would fail."""
    f = np.float32
    fx, fy, cx, cy, d = f(1.3), f(1.3), f(0.37), f(0.61), f(1.37)
    K = np.array([[[fx, 0, cx], [0, fy, cy], [0, 0, 1]]], np.float32)
    pos, quat = np.zeros((1, 3), np.float32), np.array([[1.0, 0, 0, 0]], np.float32)
    depth = np.zeros((1, 8, 32), np.float32)
    for u, v in ((3, 6), (10, 3), (5, 1)):
        depth[0, v, u] = d
    pb = np.array([((f(10) - cx) / fx) * d, ((f(3) - cy) / fy) * d, d], np.float32)
    c = np.array([pb[0] + f(0.0123), pb[1], pb[2] - f(0.0071)], np.float32)
    dx, dy, dz = pb - c
    dist2 = (dx * dx + dy * dy) + dz * dz
    r = f(np.sqrt(np.float64(dist2)))
    while r * r > dist2:
        r = np.nextafter(r, f(0))
    while r * r <= dist2:
        r = np.nextafter(r, f(1))
    r_miss = np.nextafter(r, f(0))
    assert r_miss * r_miss <= dist2 < r * r
    for radius, want in ((r, True), (r_miss, False)):
        sph = np.array([[[c[0], c[1], c[2], radius]]], np.float32)
        mask, filt = run_kernel(depth, K, pos, quat, sph, 0.0)
        assert bool(mask[0, 3, 10]) is want and mask.sum() == int(want), f"r {radius!r}: mask {np.argwhere(mask).tolist()}"
        assert np.array_equal(filt.view(np.uint32), np.where(mask, f(0), depth).view(np.uint32))


def test_subnormal_depth_is_a_candidate():
    """d > 0 holds for a subnormal depth, as in the reference, although the library flushes subnormals to zero."""
    K = np.array([[[500.0, 0, 16], [0, 500.0, 4], [0, 0, 1]]], np.float32)
    pos, quat = np.full((1, 3), 0.5, np.float32), np.array([[1.0, 0, 0, 0]], np.float32)
    depth = np.zeros((1, 8, 32), np.float32)
    depth[0, 2, 7] = np.float32(1e-40)
    depth[0, 5, 20] = 1.0
    sph = np.array([[[0.5, 0.5, 0.5, 0.1]]], np.float32)
    mask, filt = run_kernel(depth, K, pos, quat, sph, 0.0)
    check(mask, filt, depth, K, pos, quat, sph, 0.0, "subnormal")
    assert mask[0, 2, 7] and mask.sum() == 1

def test_attached_object_and_disabled_link(hw=(240, 320)):
    rm = load_robot("franka")
    eng = RolloutEngine(rm, RolloutConfig(), DEV)
    seg = RobotSegmenter(rm, DEV, distance_threshold=0.02, link_spheres=eng.link_spheres)
    q = robot_q(rm, 1, seed=11)
    obj = np.array([[0.0, 0.0, 0.12, 0.06], [0.0, 0.04, 0.17, 0.04]], np.float32)   # in the attached_object link's frame
    plain = spheres_of(rm, q, eng.link_spheres.cpu().numpy())
    eng.attach_object_spheres(T(obj))
    attached = spheres_of(rm, q, eng.link_spheres.cpu().numpy())
    eng.detach_object_spheres()
    obj_idx = np.nonzero((attached[0, :, 3] > 0) & (plain[0, :, 3] <= 0))[0]
    assert obj_idx.size == 2
    K, pos, quat, depth = scene(attached, 2, hw, seed=13, invalid=(0.0, 0.0, 0.0))
    _, _, m_obj = M.robot_mask(depth, K, pos, quat, attached[:, obj_idx], 0.02)
    _, _, m_rob = M.robot_mask(depth, K, pos, quat, plain, 0.02)
    only_obj = (m_obj > EPS) & (m_rob < -EPS)
    assert only_obj.sum() > 10

    mask, filt = seg.get_robot_mask(T(depth), T(K), T(pos), T(quat), T(q))
    mask = mask.cpu().numpy().copy()
    check(mask, filt.cpu().numpy(), depth, K, pos, quat, plain, 0.02, "detached")
    assert not mask[only_obj].any()

    eng.attach_object_spheres(T(obj))
    mask, filt = seg.get_robot_mask(T(depth), T(K), T(pos), T(quat), T(q))
    mask = mask.cpu().numpy().copy()
    check(mask, filt.cpu().numpy(), depth, K, pos, quat, attached, 0.02, "attached")
    assert mask[only_obj].all()

    link = "panda_hand"
    hand = np.nonzero(rm.link_sphere_idx_map == rm.link_names.index(link))[0]
    _, _, m_hand = M.robot_mask(depth, K, pos, quat, attached[:, hand], 0.02)
    eng.disable_link_spheres(link)
    disabled = spheres_of(rm, q, eng.link_spheres.cpu().numpy())
    _, _, m_rest = M.robot_mask(depth, K, pos, quat, disabled, 0.02)
    only_hand = (m_hand > EPS) & (m_rest < -EPS)
    assert only_hand.sum() > 10
    mask2, filt2 = seg.get_robot_mask(T(depth), T(K), T(pos), T(quat), T(q))
    mask2 = mask2.cpu().numpy().copy()
    check(mask2, filt2.cpu().numpy(), depth, K, pos, quat, disabled, 0.02, "disabled")
    assert mask[only_hand].all() and not mask2[only_hand].any()


def test_graph_capture_and_replay(hw=(480, 640)):
    rm = load_robot("franka")
    seg = RobotSegmenter(rm, DEV)
    q0, q1 = robot_q(rm, 2, seed=21)
    K, pos, quat, d0 = scene(spheres_of(rm, q0[None]), 2, hw, seed=3)
    d1 = scene(spheres_of(rm, q1[None]), 2, hw, seed=4)[3]
    depth, q = T(d0), T(q0)
    K, pos, quat = T(K), T(pos), T(quat)
    seg.get_robot_mask(depth, K, pos, quat, q)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        seg.get_robot_mask(depth, K, pos, quat, q)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        mask, filt = seg.get_robot_mask(depth, K, pos, quat, q)
    depth.copy_(T(d1))
    q.copy_(T(q1))
    g.replay()
    torch.cuda.synchronize()
    got_m, got_f = mask.clone(), filt.clone()
    want_m, want_f = seg.get_robot_mask(T(d1), K, pos, quat, T(q1))
    assert torch.equal(got_m, want_m) and torch.equal(got_f.view(torch.int32), want_f.view(torch.int32))
    assert got_m.any()


def test_refusals():
    L = cblib.load()
    b, h, w, s = 2, 16, 40, 8
    depth = T(np.ones((b, h, w), np.float32))
    K, pos, quat = T(np.tile(np.eye(3, dtype=np.float32), (b, 1, 1))), T(np.zeros((b, 3), np.float32)), \
        T(np.tile(np.array([1.0, 0, 0, 0], np.float32), (b, 1)))
    sph = T(np.zeros((b, s, 4), np.float32))
    mask = T(np.full((b, h, w), 7, np.uint8))
    filt = T(np.full((b, h, w), -3.0, np.float32))
    big = T(np.zeros((1, 14600, 4), np.float32))                         # 233,600 bytes of spheres: beyond the 227 KB opt-in

    def call(depth_p=depth.data_ptr(), batch=b, height=h, width=w, sph_p=sph.data_ptr(), rb=1, ns=s, mask_p=mask.data_ptr()):
        return L.cb200_segment_robot_depth(depth_p, batch, height, width, K.data_ptr(), pos.data_ptr(), quat.data_ptr(), sph_p,
                                           rb, ns, 0.05, mask_p, filt.data_ptr(), None)
    assert call(rb=3) == INVALID and call(rb=0) == INVALID
    assert call(depth_p=None) == INVALID and call(sph_p=None) == INVALID and call(mask_p=None) == INVALID
    assert call(sph_p=big.data_ptr(), ns=14600) == INVALID
    assert call(batch=1 << 15, height=8 << 10, width=32 << 10) == INVALID     # 2^35 tiles of 32 x 8 pixels
    assert call(ns=-1) == INVALID and call(height=0) == INVALID
    if DEV != "cpu":
        torch.cuda.synchronize()
    assert (mask.cpu() == 7).all() and (filt.cpu() == -3.0).all()                # nothing was launched
    assert call(rb=b) == 0 and call() == 0
    with pytest.raises(ValueError):
        pba_cu.launch_segment_robot_depth(depth, K, pos, quat, T(np.zeros((3, s, 4), np.float32)), 0.05, mask, filt)
    with pytest.raises(ValueError):
        pba_cu.launch_segment_robot_depth(depth, K, pos, quat, sph, 0.05, mask.view(torch.int8), filt)


Q_CAMERA = np.array([0.0, -0.3, 0.0, -2.0, 0.0, 1.8, 0.785], np.float32)     # Franka's retracted pose, the pose the cameras see
Q_INTO_BOX = np.array([1.5, -0.3, 0.0, -2.0, 0.0, 1.8, 0.785], np.float32)   # the same pose turned 1.5 rad about the base axis


def mapping_scene(rm, voxel, hw):
    """Franka at Q_CAMERA, a back wall, and a 16 cm box where the hand is at Q_INTO_BOX, seen by two cameras; the dense grid
    (1.6 m cube) around robot and box.  Returns spheres at both poses, the box, cameras, depth and the grid."""
    sph = spheres_of(rm, Q_CAMERA[None])
    into = spheres_of(rm, Q_INTO_BOX[None])[0]
    hand = into[rm.link_sphere_idx_map == rm.link_names.index("panda_hand")]
    box = (hand[:, :3].mean(0) - 0.08, hand[:, :3].mean(0) + 0.08)
    live = sph[0][sph[0][:, 3] > 0]
    lo, hi = np.minimum(live[:, :3].min(0), box[0]), np.maximum(live[:, :3].max(0), box[1])
    c = 0.5 * (lo + hi)
    eyes = [c + 2.2 * np.array([np.cos(a), np.sin(a), 0.45]) for a in (-0.35, 0.35)]
    K, pos, quat = M.cameras(eyes, c, hw)
    shrunk = np.concatenate([sph[0][:, :3], sph[0][:, 3:] - 0.005], -1)       # the surface 5 mm inside the collision spheres
    depth = M.render_depth(K, pos, quat, hw, spheres=shrunk, wall=((lo[0] - 0.6, 0.0, 0.0), (1.0, 0.0, 0.0)), boxes=[box])
    n = int(round(1.6 / voxel))
    return sph, into, box, K, pos, quat, depth, (n, n, n), tuple(float(v) for v in c)


def voxel_centres(shape, voxel, origin):
    idx = np.stack(np.meshgrid(*[np.arange(k) for k in shape], indexing="ij"), -1).astype(np.float64)
    return (idx + 0.5 - np.asarray(shape) / 2.0) * voxel + np.asarray(origin)


def test_segmented_depth_to_esdf_and_collision_checker(voxel=0.02, hw=(480, 640)):
    """Depth -> DenseTSDF -> combined SDF -> DenseESDFBuilder -> RobotCollisionChecker(voxel=...) with and without the robot's
    pixels masked: unsegmented, the robot maps itself as an obstacle; segmented, no voxel inside its spheres is negative, the box
    region is the same voxel for voxel, the camera's q is valid, and a q into the box is invalid in both maps."""
    from curobo_b200.collision import RobotCollisionChecker
    from curobo_b200.esdf import DenseESDFBuilder, DenseTSDF
    rm = load_robot("franka")
    sph, into, box, K, pos, quat, depth, shape, origin = mapping_scene(rm, voxel, hw)
    trunc = 3 * voxel
    seg = RobotSegmenter(rm, DEV, distance_threshold=0.03)
    mask, filtered = seg.get_robot_mask(T(depth), T(K), T(pos), T(quat), T(Q_CAMERA))
    assert mask.any()
    maps = {}
    for name, d in (("plain", T(depth)), ("segmented", filtered)):
        tsdf = DenseTSDF(shape, voxel, trunc, DEV, origin=origin)
        tsdf.integrate(d, T(K), T(pos), T(quat))
        combined = tsdf.combined_sdf().clone()
        esdf = DenseESDFBuilder(shape, voxel, trunc, DEV, origin=origin)
        esdf.compute(combined)
        ck = RobotCollisionChecker(rm, DEV, voxel=esdf.to_voxel_data())
        valid = ck.validate(T(np.stack([Q_CAMERA, Q_INTO_BOX])[:, None])).cpu().numpy()[:, 0].copy()
        maps[name] = (combined.cpu().numpy().copy(), valid)
    x = voxel_centres(shape, voxel, origin)
    live = sph[0][sph[0][:, 3] > 0]
    inside = np.zeros(shape, bool)
    for s in live:
        inside |= np.linalg.norm(x - s[:3], axis=-1) < s[3]
    box_region = np.all((x >= box[0] - trunc) & (x <= box[1] + trunc), -1)      # the voxels the box's surface reaches
    in_box = np.all((x >= box[0]) & (x <= box[1]), -1)
    plain, seg_map = maps["plain"][0], maps["segmented"][0]
    print(f"voxels inside the robot: {inside.sum()}, negative unsegmented: {(plain[inside] < 0).sum()}, segmented: "
          f"{(seg_map[inside] < 0).sum()}; box region {box_region.sum()} voxels, negative {(plain[box_region] < 0).sum()}; "
          f"valid (camera q, q into the box): unsegmented {maps['plain'][1]}, segmented {maps['segmented'][1]}")
    assert (plain[inside] < 0).sum() >= 10                                       # the robot maps itself as an obstacle
    assert not (seg_map[inside] < 0).any()                                        # ... and no longer does
    diff = box_region & (plain.view(np.uint32) != seg_map.view(np.uint32))
    assert not diff.any(), f"{diff.sum()} box-region voxels differ, e.g. at {x[diff][:4].round(3).tolist()} (box {box})"
    assert (plain[in_box] < 0).sum() >= 10                                        # the box is in both maps
    assert list(maps["plain"][1]) == [False, False]
    assert list(maps["segmented"][1]) == [True, False]
