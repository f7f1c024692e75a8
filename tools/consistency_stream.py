"""Time the multi-view depth consistency check on tools/fusion_stream.py's ray-cast room (400 views at 224x224):

  * slam_utils.view_consistency_check (one kernel launch) against a torch restatement of the reference's per-view loop
    (per view and neighbour: torch.inverse, a matmul and F.grid_sample) on the same GPU, with their counts compared;
  * render (1 camera, 720x1280) and extract_mesh (4 cm voxel) of the map with and without min_consistent_views=2,
    through OnlineSLAM's own filtering step (_consistent_maps) on the room's maps.

Every timed call ends in a device synchronise; the card's name and power limit are read in the same run.

    python tools/consistency_stream.py [--views 400] [--iters 10] [--out FILE]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fusion_stream import room  # noqa: E402
from render_stream import card  # noqa: E402


def torch_loop(depth, intri, poses, threshold):
    """The reference's per-view loop, restated with torch operations: view i's pixels unprojected with K_i^-1 and T_i,
    moved into each neighbour j within 4 indices by T_j^-1, projected with K_j and compared with j's depth sampled by
    grid_sample (bilinear, zero padding, align_corners=True)."""
    n, H, W = depth.shape
    dev = depth.device
    yy, xx = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    pix = torch.stack([xx, yy, torch.ones_like(xx)]).float().reshape(3, -1)
    out = torch.zeros(n, H, W, dtype=torch.int32, device=dev)
    for i in range(n):
        cam = (torch.inverse(intri[i]) @ pix) * depth[i].reshape(1, -1)
        world = poses[i] @ torch.cat([cam, torch.ones_like(cam[:1])])
        agree = torch.zeros(H * W, device=dev)
        for j in range(max(0, i - 4), min(n, i + 5)):
            if j == i:
                continue
            c = (torch.inverse(poses[j]) @ world)[:3]
            z = c[2].clamp(min=1e-6)
            q = intri[j] @ c
            uv = (q[:2] / q[2:]).T.reshape(1, H, W, 2)
            g = torch.stack([uv[..., 0] / (W - 1) * 2 - 1, uv[..., 1] / (H - 1) * 2 - 1], -1)
            s = F.grid_sample(depth[j][None, None], g, mode="bilinear", align_corners=True).reshape(-1)
            agree += (((s - z).abs() < threshold) & (z > 0)).float()
        out[i] = agree.reshape(H, W).int()
    return out


def timed(f, iters):
    f()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        t = time.perf_counter()
        f()
        torch.cuda.synchronize()
        ts.append(1e3 * (time.perf_counter() - t))
    return round(float(np.median(ts)), 3), round(float(min(ts)), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=400)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from vista_slam_b200.slam import OnlineSLAM
    from vista_slam_b200.utils.slam_utils import view_consistency_check

    rows = [{"card": card()}]
    print(json.dumps(rows[0]), flush=True)
    maps = room(a.views)
    depth = maps["depth"] * maps["scale"][:, :, None]
    n, H, W = depth.shape

    def kernel():
        return view_consistency_check(depth, maps["intri"], maps["pose"], 0.05)

    def loop():
        return torch_loop(depth, maps["intri"], maps["pose"], 0.05)

    c_k, c_l = kernel(), loop()
    torch.cuda.synchronize()
    k_ms, t_ms = timed(kernel, a.iters), timed(loop, max(2, a.iters // 5))
    rows.append({"what": "view_consistency_check", "views": n, "H": H, "W": W, "kernel_ms": k_ms, "torch_loop_ms": t_ms,
                 "pixels_differing": int((c_k != c_l).sum()), "pixels": c_k.numel(),
                 "count_histogram": torch.bincount(c_k.reshape(-1).long(), minlength=9).tolist()})
    print(json.dumps(rows[-1]), flush=True)

    # OnlineSLAM's filtering step on the room's maps, without a session
    s = OnlineSLAM.__new__(OnlineSLAM)
    s.conf_thres, s.consistency_thres = 0.5, 0.05
    from vista_slam_b200.fusion import fuse_views
    from vista_slam_b200.render import render_views
    pose = maps["pose"][:1]
    K = torch.tensor([[600.0, 0, 639.5], [0, 600.0, 359.5], [0, 0, 1]], device="cuda")[None]
    for k in (None, 2):
        def rend():
            m = s._consistent_maps(dict(maps), k or 0)
            return render_views(m, s.conf_thres, pose, K, (720, 1280))

        def mesh():
            m = s._consistent_maps(dict(maps), k or 0)
            return fuse_views(m, s.conf_thres, 0.04)
        r_ms, m_ms = timed(rend, a.iters), timed(mesh, a.iters)
        faces = len(mesh()["faces"])
        rows.append({"what": "render_and_extract_mesh", "min_consistent_views": k, "render_1cam_720x1280_ms": r_ms,
                     "extract_mesh_4cm_ms": m_ms, "faces": faces})
        print(json.dumps(rows[-1]), flush=True)
    rows.append({"peak_mib": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)})
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
