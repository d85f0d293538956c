"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the reference's robot segmentation of depth images and a float64 renderer
of the scenes the tests segment.

    deproject      <- get_projection_rays + project_depth_using_rays  geom/cv.py:47-157 (depth_to_meter = 1: depth in metres)
    to_robot_frame <- Pose.batch_transform_points (camera -> robot base, quaternion wxyz)
    robot_mask     <- _mask_spheres_image_cdist  perception/robot_segmenter.py:336-366: mask = depth > 0 and
                      max_s(r_s - |p - c_s|) > -threshold, filtered = where(mask, 0, depth)
`robot_mask` also returns the margin max_s(r_s + threshold - |p - c_s|) of every pixel, so that a test can set aside the pixels
whose verdict float32 rounding may flip.
"""
import numpy as np

F = np.float64


def deproject(depth, K):
    """depth [B,H,W], K [B,3,3] -> camera-frame points [B,H,W,3]: ((u - cx) / fx d, (v - cy) / fy d, d) at integer (u, v)."""
    depth = np.asarray(depth, F)
    K = np.asarray(K, F)
    B, H, W = depth.shape
    v, u = np.meshgrid(np.arange(H, dtype=F), np.arange(W, dtype=F), indexing="ij")
    x = (u[None] - K[:, 0, 2, None, None]) / K[:, 0, 0, None, None]
    y = (v[None] - K[:, 1, 2, None, None]) / K[:, 1, 1, None, None]
    with np.errstate(invalid="ignore"):
        return np.stack([x * depth, y * depth, depth], -1)


def quat_matrix(q):
    """wxyz (unit) -> rotation matrix [..., 3, 3]."""
    w, x, y, z = (np.asarray(q, F)[..., i] for i in range(4))
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def to_robot_frame(points, pos, quat):
    """points [B,...,3] in the camera frame -> robot base frame: R(q) p + t per image."""
    R = quat_matrix(quat)
    pts = np.asarray(points, F)
    B = pts.shape[0]
    with np.errstate(invalid="ignore"):
        out = np.einsum("bij,bnj->bni", R, pts.reshape(B, -1, 3)) + np.asarray(pos, F)[:, None, :]
    return out.reshape(pts.shape)


def robot_mask(depth, K, pos, quat, spheres, threshold):
    """depth [B,H,W], spheres [1 or B, S, 4] -> (mask bool [B,H,W], filtered [B,H,W] in depth's dtype, margin float64 [B,H,W])."""
    depth = np.asarray(depth)
    p = to_robot_frame(deproject(depth, K), pos, quat)                          # [B,H,W,3]
    sph = np.broadcast_to(np.asarray(spheres, F), (depth.shape[0],) + np.asarray(spheres).shape[1:])
    B, H, W = depth.shape
    margin = np.full((B, H, W), -np.inf)
    with np.errstate(invalid="ignore", over="ignore"):
        for s in range(sph.shape[1]):
            dist = np.linalg.norm(p - sph[:, s, None, None, :3], axis=-1)
            margin = np.fmax(margin, sph[:, s, None, None, 3] + threshold - dist)
        finite = np.isfinite(p).all(-1)
        mask = (depth > 0) & finite & (margin > 0)
    filtered = np.where(mask, np.zeros((), depth.dtype), depth)
    return mask, filtered, margin


def render_depth(K, pos, quat, hw, spheres=(), wall=None, boxes=(), invalid=(0.0, 0.0, 0.0), seed=0):
    """z-depth images [B,H,W] float32 of balls, a plane and axis-aligned boxes, seen by pinhole cameras (K [B,3,3], pos [B,3],
    quat [B,4] wxyz camera -> world), ray through the pixel's integer coordinates.  spheres [S,4] (r <= 0: not drawn);
    wall = (point, normal); boxes = [(lo xyz, hi xyz), ...]; invalid = shares of pixels set to 0, NaN and +inf.  Pixels that hit
    nothing are 0."""
    H, W = hw
    K, pos = np.asarray(K, F), np.asarray(pos, F)
    B = K.shape[0]
    R = quat_matrix(quat)
    rng = np.random.default_rng(seed)
    out = np.zeros((B, H, W), np.float32)
    for b in range(B):
        ray = deproject(np.ones((1, H, W)), K[b:b + 1])[0] @ R[b].T                  # world direction with camera z = 1
        e = pos[b]
        t = np.full((H, W), np.inf)
        for c in np.asarray(spheres, F).reshape(-1, 4):
            if c[3] <= 0:
                continue
            oc = e - c[:3]
            a = (ray * ray).sum(-1)
            bb = 2 * (ray @ oc)
            cc = oc @ oc - c[3] ** 2
            disc = bb * bb - 4 * a * cc
            with np.errstate(invalid="ignore"):
                th = (-bb - np.sqrt(disc)) / (2 * a)
            t = np.where((disc > 0) & (th > 0) & (th < t), th, t)
        if wall is not None:
            p0, n = np.asarray(wall[0], F), np.asarray(wall[1], F)
            den = ray @ n
            with np.errstate(divide="ignore", invalid="ignore"):
                th = ((p0 - e) @ n) / den
            t = np.where((np.abs(den) > 1e-12) & (th > 0) & (th < t), th, t)
        for lo, hi in boxes:
            lo, hi = np.asarray(lo, F), np.asarray(hi, F)
            with np.errstate(divide="ignore", invalid="ignore"):
                t1, t2 = (lo - e) / ray, (hi - e) / ray
            tn = np.nanmax(np.minimum(t1, t2), -1)
            tf = np.nanmin(np.maximum(t1, t2), -1)
            t = np.where((tn <= tf) & (tn > 0) & (tn < t), tn, t)
        img = np.where(np.isfinite(t), t, 0.0).astype(np.float32)
        r = rng.random((H, W))
        z, nan, inf = invalid
        img[r < z] = 0.0
        img[(r >= z) & (r < z + nan)] = np.nan
        img[(r >= z + nan) & (r < z + nan + inf)] = np.inf
        out[b] = img
    return out


def look_at(eye, target):
    """camera -> world quaternion (wxyz) of a camera at `eye` looking at `target` (x right, y down, z forward)."""
    zc = np.asarray(target, F) - np.asarray(eye, F)
    zc /= np.linalg.norm(zc)
    up = np.array([0.0, 0.0, 1.0]) if abs(zc[2]) < 0.9 else np.array([1.0, 0.0, 0.0])
    xc = np.cross(zc, up)
    xc /= np.linalg.norm(xc)
    yc = np.cross(zc, xc)
    Rm = np.stack([xc, yc, zc], 1)
    w = np.sqrt(max(0.0, 1.0 + np.trace(Rm))) / 2.0
    q = np.array([w, (Rm[2, 1] - Rm[1, 2]) / (4 * w), (Rm[0, 2] - Rm[2, 0]) / (4 * w), (Rm[1, 0] - Rm[0, 1]) / (4 * w)])
    return q / np.linalg.norm(q)


def cameras(eyes, target, hw, focal=0.9):
    """K [C,3,3], pos [C,3], quat [C,4] (float32) of pinhole cameras at `eyes` looking at `target`, focal = focal * width."""
    H, W = hw
    n = len(eyes)
    K = np.zeros((n, 3, 3), np.float32)
    pos = np.asarray(eyes, np.float32).reshape(n, 3)
    quat = np.zeros((n, 4), np.float32)
    for c in range(n):
        f = focal * W
        K[c] = [[f, 0, W / 2 - 0.5], [0, f, H / 2 - 0.5], [0, 0, 1]]
        quat[c] = look_at(eyes[c], target)
    return K, pos, quat
