"""Generate tests/golden/robot_mask_reference_golden.npz: the REFERENCE's own robot segmentation steps -- `get_projection_rays` and
`project_depth_using_rays` (geom/cv.py:47-157), the camera -> robot pose transform (the `compute_batch_transform_point` Warp kernel
behind Pose.batch_transform_points, geom/transform.py:571-601, run thread by thread under the pure-Python Warp stand-in
oracle/warp_shim) and `_mask_spheres_image_cdist` (perception/robot_segmenter.py:336-366) -- on the CPU in float32 with
`curobo_runtime.torch_jit` off.  Inputs: Franka's FK spheres (oracle/rollout_oracle.py) at a few q, two 48 x 64 cameras.  The
fixture stores inputs, the reference's mask and filtered depth, and the float64 oracle's margin of every pixel (so that a test can
set aside pixels within rounding of the threshold).  Needs /root/reference (authoring container only):

    python tests/golden/make_robot_mask_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]
import _reference_under_shim as R  # noqa: E402

R.STUB_PACKAGES = R.STUB_PACKAGES + ("lxml",)
R.prepare()
import torch  # noqa: E402
import warp as wp  # noqa: E402  (the stand-in)

import curobo._src.runtime as curobo_runtime  # noqa: E402

curobo_runtime.torch_jit = False
cv = R.ref("curobo._src.geom.cv")
transform = R.ref("curobo._src.geom.transform")
segmenter = R.ref("curobo._src.perception.robot_segmenter")

from curobo_b200.robot_model import load_robot  # noqa: E402
from oracle import robot_mask_oracle as M  # noqa: E402
from test_gpu_robot_segmenter import robot_q, scene, spheres_of  # noqa: E402

HW = (48, 64)


def reference_mask(depth, K, pos, quat, spheres, threshold):
    B, H, W = depth.shape
    rays = cv.get_projection_rays(H, W, torch.from_numpy(K), 1.0)
    pts = cv.project_depth_using_rays(torch.from_numpy(depth), rays).numpy().astype(np.float32)   # [B, H*W, 3]
    out = wp.from_numpy(np.zeros((B * H * W, 3), np.float32), dtype=wp.vec3)
    wp.launch(transform.compute_batch_transform_point, dim=B * H * W,
              inputs=[wp.from_numpy(pos, dtype=wp.vec3), wp.from_numpy(quat, dtype=wp.vec4),
                      wp.from_numpy(pts.reshape(-1, 3), dtype=wp.vec3), H * W, B], outputs=[out])
    world = torch.from_numpy(np.asarray(out.numpy(), np.float32).reshape(B, H * W, 3))
    mask, filt = segmenter._mask_spheres_image_cdist(torch.from_numpy(depth), torch.from_numpy(spheres), world, float(threshold))
    return mask.numpy(), filt.numpy().astype(np.float32)


def main():
    rm = load_robot("franka")
    q = robot_q(rm, 3, seed=1)
    one, per_image = spheres_of(rm, q[:1]), spheres_of(rm, q[1:3])
    ls = np.array(rm.link_spheres if rm.link_spheres.ndim == 3 else rm.link_spheres[None], np.float32)
    ls[:, rm.link_sphere_idx_map == rm.link_names.index("panda_hand"), 3] = -100.0
    disabled = spheres_of(rm, q[:1], ls)
    cases = {"batch1_thr005": (one, 0.05, (0.02, 0.005, 0.005)), "batchB_thr005": (per_image, 0.05, (0.02, 0.005, 0.005)),
             "batch1_thr0": (one, 0.0, (0.02, 0.005, 0.005)), "disabled_hand": (disabled, 0.05, (0.0, 0.0, 0.0)),
             "invalid_pixels": (one, 0.05, (0.1, 0.05, 0.05))}
    out = {}
    for name, (sph, thr, invalid) in cases.items():
        K, pos, quat, depth = scene(one if name == "disabled_hand" else sph, 2, HW, seed=len(out), invalid=invalid)
        out[name] = dict(K=K, pos=pos, quat=quat, depth=depth, spheres=sph, threshold=np.float32(thr))
    # a camera that sees no robot: the first scene's cameras turned to look along the wall
    K, pos, quat, depth = scene(one, 2, HW, seed=9)
    quat = np.stack([M.look_at(p, p + np.array([0.0, 1.0, -0.2])) for p in pos]).astype(np.float32)
    depth = M.render_depth(K, pos, quat, HW, spheres=one[0], wall=((-1.0, 0.0, 0.0), (1.0, 0.0, 0.0)),
                           boxes=[((-0.2, 3.0, -1.0), (0.2, 3.5, 2.0))], seed=9)
    out["no_robot"] = dict(K=K, pos=pos, quat=quat, depth=depth, spheres=one, threshold=np.float32(0.05))
    flat = {}
    for name, c in out.items():
        mask, filt = reference_mask(c["depth"], c["K"], c["pos"], c["quat"], c["spheres"], c["threshold"])
        _, _, margin = M.robot_mask(c["depth"], c["K"], c["pos"], c["quat"], c["spheres"], float(c["threshold"]))
        c.update(mask=mask, filtered=filt, margin=margin)
        for k, v in c.items():
            flat[f"{name}/{k}"] = v
        print(name, "masked", int(mask.sum()), "of", mask.size, "valid", int((c["depth"] > 0).sum()))
    np.savez_compressed(os.path.join(HERE, "robot_mask_reference_golden.npz"), **flat)


if __name__ == "__main__":
    main()
