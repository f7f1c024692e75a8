"""Time fusion.fuse_views per stage on a synthetic room and on a replayed SLAM run.

The room: --views views at 224x224 along a seeded camera path through a 6 x 3 x 8 box room with a few boxes inside,
depths ray-cast in float64, every pixel confident.  The replayed run: tools/render_stream.replayed_slam over a --views
224x224 stream.  For each map and voxel size, the allocation (both sta_fusion_bricks calls), integration and meshing are timed
between device synchronisations with CUDA events, median of --iters calls after a warm-up, with the brick, vertex and
face counts and the peak device memory.  The card's name and power limit are read in the same run.

    python tools/fusion_stream.py [--views 400] [--iters 10] [--voxels 0.04,0.02]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import slam_oracle as so  # noqa: E402
from render_stream import card, replayed_slam  # noqa: E402

BOXES = [((-3.0, -1.5, -4.0), (3.0, 1.5, 4.0), True),  # the room, seen from inside
         ((-2.5, -1.5, 1.0), (-1.0, -0.7, 2.5), False), ((0.8, -1.5, -2.5), (2.2, 0.2, -1.0), False),
         ((-0.4, -1.5, -0.4), (0.4, -1.0, 0.4), False)]


def _look_at(eye, target):
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross((0.0, -1.0, 0.0), z)
    x /= np.linalg.norm(x)
    P = np.eye(4)
    P[:3, :3] = np.stack([x, np.cross(z, x), z], 1)
    P[:3, 3] = eye
    return P


def room(views, H=224, W=224, seed=0):
    """maps of `views` ray-cast views of the room (float32 on the GPU)."""
    r = np.random.default_rng(seed)
    K = np.array([[200.0, 0, W / 2 - 0.5], [0, 200.0, H / 2 - 0.5], [0, 0, 1]])
    yy, xx = np.mgrid[0:H, 0:W]
    ray = np.linalg.inv(K) @ np.stack([xx.ravel(), yy.ravel(), np.ones(H * W)])
    poses, depths, imgs = [], [], []
    for k in range(views):
        a = 2 * np.pi * k / views
        eye = np.array([1.6 * np.cos(a), 0.2 * np.sin(3 * a), 2.5 * np.sin(a)]) + r.normal(0, 0.05, 3)
        target = np.array([0.0, -0.5, 0.0]) + r.normal(0, 0.3, 3)
        P = _look_at(eye, target)
        d = P[:3, :3] @ ray
        best = np.full(H * W, np.inf)
        col = np.zeros((3, H * W))
        for bi, (lo, hi, inside) in enumerate(BOXES):
            lo, hi = np.array(lo)[:, None], np.array(hi)[:, None]
            with np.errstate(divide="ignore", invalid="ignore"):
                t0, t1 = (lo - eye[:, None]) / d, (hi - eye[:, None]) / d
            tn, tf = np.minimum(t0, t1).max(0), np.maximum(t0, t1).min(0)
            t = np.where(inside, tf, np.where((tn <= tf) & (tn > 0), tn, np.inf))
            hit = t < best
            best[hit] = t[hit]
            p = eye[:, None] + d * t
            col[:, hit] = (0.5 * np.sin(3 * p[:, hit] + bi)).clip(-1, 1)
        poses.append(P)
        depths.append(np.where(np.isfinite(best), best, 0.0).reshape(H, W))
        imgs.append(col.reshape(3, H, W))
    f32 = lambda x: torch.as_tensor(np.asarray(x, np.float32)).cuda()
    return {"pose": f32(poses), "scale": torch.ones(views, 1, device="cuda"), "depth": f32(depths),
            "conf": f32(np.stack(depths) > 0), "intri": f32([K] * views), "images": f32(imgs)}


def stages(maps, thres, voxel):
    """One fuse_views split into its three stages, each closed by a synchronisation: (ms per stage, counts)."""
    from vista_slam_b200 import fusion
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    out = fusion.fuse_views(maps, thres, voxel, min_weight=10 ** 9)  # allocation and integration; no cube is meshed
    ev[1].record()
    torch.cuda.synchronize()
    keys = fusion.brick_keys(out["bricks"])
    ev[2].record()
    mesh = fusion._mesh(keys, out["tsdf"], out["weight"], out["color"], voxel, 1.0)
    ev[3].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]), ev[2].elapsed_time(ev[3]), (len(keys), len(mesh["vertices"]), len(mesh["faces"]))


def alloc_only(maps, thres, voxel):
    """The allocation stage alone (as fuse_views runs it, up to the brick count)."""
    from vista_slam_b200 import fusion
    try:
        fusion.fuse_views(maps, thres, voxel, max_bricks=1)
    except ValueError:
        pass


def timed(f, iters):
    f()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        f()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def measure(name, maps, thres, voxel, iters):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    alloc = timed(lambda: alloc_only(maps, thres, voxel), iters)
    runs = [stages(maps, thres, voxel) for _ in range(iters + 1)][1:]
    ai = float(np.median([r[0] for r in runs]))
    mesh = float(np.median([r[1] for r in runs]))
    total = timed(lambda: __import__("vista_slam_b200.fusion", fromlist=["x"]).fuse_views(maps, thres, voxel), iters)
    B, nv, nf = runs[-1][2]
    return {"map": name, "voxel": voxel, "views": int(maps["depth"].shape[0]), "bricks": B, "vertices": nv,
            "faces": nf, "alloc_ms": round(alloc, 3), "integrate_ms": round(ai - alloc, 3), "mesh_ms": round(mesh, 3),
            "fuse_views_ms": round(total, 3), "peak_mib": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=400)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--voxels", default="0.04,0.02")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    voxels = [float(x) for x in a.voxels.split(",")]
    rows = [{"card": card()}]
    print(json.dumps(rows[0]), flush=True)
    maps = room(a.views)
    for v in voxels:
        rows.append(measure("room", maps, 0.5, v, a.iters))
        print(json.dumps(rows[-1]), flush=True)
    stream = so.make_stream(seed=3, n_views=a.views, H=224, W=224)
    slam = replayed_slam(stream)
    images = so.stream_images(stream)
    for i in range(a.views):
        slam.step(so_value(images, i, stream))
    del stream
    m = slam._view_maps(None)
    pts = slam._export(0, slam.view_num, cloud=True)
    ext = float((pts["points"][:int(pts["count"].cpu())].max(0).values
                 - pts["points"][:int(pts["count"].cpu())].min(0).values).max())
    for div in (64, 128):
        rows.append(measure("replayed", m, slam.conf_thres, ext / div, a.iters))
        print(json.dumps(rows[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


def so_value(images, i, stream):
    return {"rgb": torch.from_numpy(images[i])[None].cuda(), "shape": torch.tensor([[stream["H"], stream["W"]]]),
            "gray": None, "view_name": "%04d.png" % i}


if __name__ == "__main__":
    main()
