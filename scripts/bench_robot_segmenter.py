"""Robot segmentation of depth images on the GPU: cb200_segment_robot_depth alone and RobotSegmenter.get_robot_mask (FK + kernel),
each replayed as a CUDA graph, the reference's formula restated in torch on the same GPU (cdist, max, where; fp32), and the depth ->
TSDF -> ESDF chain at 256^3 with and without segmentation in front of it.  Robots: Franka (65 spheres), G1-29 (400), G1-43 (674);
images: 1 x 480x640, 2 x 480x640, 4 x 720x1280 (the sizes of the depth cameras a robot carries).  Each timed launch follows an L2
flush; medians of alternating arms, CUDA events.  Prints one JSON line per workload with the card's name and power limit.

    python scripts/bench_robot_segmenter.py [--reps 30]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from curobo_b200.backends import pba as pba_cu  # noqa: E402
from curobo_b200.esdf import DenseESDFBuilder, DenseTSDF  # noqa: E402
from curobo_b200.perception import RobotSegmenter  # noqa: E402
from curobo_b200.robot_model import load_robot  # noqa: E402
from test_gpu_robot_segmenter import robot_q, scene, spheres_of  # noqa: E402

DEV = "cuda:0"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def timed(arms, reps, flush):
    """arms: name -> callable; alternating, each call after an L2 flush; median ms per arm."""
    out = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            out[k].append(a.elapsed_time(b))
    return {k: float(np.median(v)) for k, v in out.items()}


def cull_share(depth, K, pos, quat, sph, thr):
    """Mean share of spheres that survive a tile's cull (32 x 8 tiles, boxes of the candidate points), computed on the host."""
    from oracle import robot_mask_oracle as M
    p = M.to_robot_frame(M.deproject(depth, K), pos, quat)
    B, H, W = depth.shape
    live = sph[0][sph[0][:, 3] + thr > 0]
    shares = []
    for b in range(B):
        for y in range(0, H, 8):
            for x in range(0, W, 32):
                d = depth[b, y:y + 8, x:x + 32]
                ok = (d > 0) & np.isfinite(d)
                if not ok.any():
                    continue
                pts = p[b, y:y + 8, x:x + 32][ok]
                lo, hi = pts.min(0), pts.max(0)
                gap = np.maximum(np.maximum(lo - live[:, :3], live[:, :3] - hi), 0)
                shares.append(((gap ** 2).sum(1) < (live[:, 3] + thr) ** 2).mean())
    return float(np.mean(shares)) * len(live) / len(sph[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--robots", default="franka,g1_29,g1_43")
    args = ap.parse_args()
    name, pl = card()
    flush = torch.empty(64 << 20, dtype=torch.float32, device=DEV)          # 256 MB: larger than the 50 MB L2
    thr = 0.05
    for robot in args.robots.split(","):
        rm = load_robot(robot)
        q = robot_q(rm, 1, seed=3)
        sph = spheres_of(rm, q)
        seg = RobotSegmenter(rm, DEV, distance_threshold=thr)
        for n_img, hw in ((1, (480, 640)), (2, (480, 640)), (4, (720, 1280))):
            K, pos, quat, depth = scene(sph, n_img, hw, seed=1)
            tK, tp, tq, td, ts, tqj = (torch.as_tensor(a).to(DEV) for a in (K, pos, quat, depth, sph, q))
            mask = torch.empty(depth.shape, dtype=torch.bool, device=DEV)
            filt = torch.empty(depth.shape, dtype=torch.float32, device=DEV)
            H, W = hw
            rays = torch.stack(torch.meshgrid(torch.arange(W, device=DEV, dtype=torch.float32),
                                              torch.arange(H, device=DEV, dtype=torch.float32), indexing="xy"), -1)
            rays = torch.cat([(rays - tK[:, None, None, [0, 1], [2, 2]]) / tK[:, None, None, [0, 1], [0, 1]],
                              torch.ones((n_img, H, W, 1), device=DEV)], -1).view(n_img, -1, 3)
            w, x, y, z = tq.unbind(-1)
            Rm = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y), 2 * (x * y + w * z),
                              1 - 2 * (x * x + z * z), 2 * (y * z - w * x), 2 * (x * z - w * y), 2 * (y * z + w * x),
                              1 - 2 * (x * x + y * y)], -1).view(n_img, 3, 3)

            def torch_arm():
                pts = td.view(n_img, -1, 1) * rays
                pts = pts @ Rm.transpose(1, 2) + tp[:, None]
                s = ts.expand(n_img, -1, -1)
                dist = -(torch.cdist(pts, s[..., :3]) - s[..., 3].unsqueeze(1))
                m = (td > 0) & (dist.max(-1)[0].view(td.shape) > -thr)
                return m, torch.where(m, 0, td)

            def kernel_arm():
                pba_cu.launch_segment_robot_depth(td, tK, tp, tq, ts, thr, mask, filt)

            def graph_of(fn):
                # both GPU arms are replayed graphs, so that the events time the device and not the Python launcher
                fn()
                st = torch.cuda.Stream()
                st.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(st):
                    fn()
                torch.cuda.current_stream().wait_stream(st)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    fn()
                return g
            g = graph_of(lambda: seg.get_robot_mask(td, tK, tp, tq, tqj))
            gk = graph_of(kernel_arm)

            c = np.asarray(sph[0][sph[0][:, 3] > 0][:, :3]).mean(0)
            tsdf = DenseTSDF((256, 256, 256), 0.01, 0.04, DEV, origin=tuple(c))
            esdf = DenseESDFBuilder((256, 256, 256), 0.01, 0.04, DEV, origin=tuple(c))

            def chain(segment):
                def run():
                    tsdf.reset()
                    if segment:
                        pba_cu.launch_segment_robot_depth(td, tK, tp, tq, ts, thr, mask, filt)
                    tsdf.integrate(filt if segment else td, tK, tp, tq)
                    esdf.compute(tsdf.combined_sdf())
                return run
            arms = {"kernel": gk.replay, "graph": g.replay, "torch_cdist": torch_arm, "chain_segmented": chain(True),
                    "chain_plain": chain(False)}
            for fn in arms.values():                                            # warm-up
                fn()
            torch.cuda.synchronize()
            m_ref, f_ref = torch_arm()
            kernel_arm()
            torch.cuda.synchronize()
            agree = float((m_ref == mask).float().mean())
            ms = timed(arms, args.reps, flush)
            px = n_img * H * W
            S = sph.shape[1]
            bytes_moved = px * (4 + 4 + 1) + n_img * (9 + 3 + 4) * 4 + S * 16
            print(json.dumps({"robot": robot, "spheres": S, "images": n_img, "hw": list(hw), "card": name, "power_limit": pl,
                              "ms": {k: round(v, 4) for k, v in ms.items()},
                              "kernel_gpix_per_s": round(px / ms["kernel"] / 1e6, 3),
                              "kernel_bytes": bytes_moved, "kernel_gb_per_s": round(bytes_moved / ms["kernel"] / 1e6, 1),
                              "torch_cdist_matrix_mb": round(px * S * 4 / 2 ** 20, 1),
                              "cull_survivor_share": round(cull_share(depth[:1, :min(H, 240)], K[:1], pos[:1], quat[:1], sph, thr), 4),
                              "mask_agreement_with_torch": agree, "masked_share": float(mask.float().mean())}), flush=True)
            del g, gk, tsdf, esdf
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
