"""Time fusion.raycast beside render_views on the same maps, and OnlineSLAM.render_surface end to end.

Maps: tools/fusion_stream.py's room (--views ray-cast 224x224 views, every pixel confident) and the replayed SLAM run of
tools/render_stream.replayed_slam over a --views 224x224 stream.  Cameras: C = 1, 8 and 32 of the map's own poses,
spread over its path, at --size (default 720x1280) with a 60 degree horizontal field of view.

  room       the volume fused once per voxel size (0.04 and 0.02 by default); raycast of it and render_views of the room's
             points (radius 0) from the same cameras, alternated call by call; and fuse_volume + raycast end to end.
  replayed   render_surface (fusion and ray cast) at 1/64 and 1/128 of the cloud's extent, beside render.

Each call is timed with CUDA events and closed by a synchronisation; the median of --iters calls after two warm-up
rounds.  The card's name and power limit are read in the same run.  One JSON line per row.

    python tools/raycast_stream.py [--views 400] [--iters 10] [--voxels 0.04,0.02] [--size 720x1280]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from fusion_stream import room, so_value  # noqa: E402
from oracle import slam_oracle as so  # noqa: E402
from render_stream import card, replayed_slam  # noqa: E402


def alternated(calls, iters):
    """Median ms of each call in `calls` (name -> fn), run in turn, each between CUDA events and a synchronisation."""
    times = {k: [] for k in calls}
    for it in range(iters + 2):  # two warm-up rounds
        for k, fn in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            if it >= 2:
                times[k].append(a.elapsed_time(b))
    return {k: round(float(np.median(v)), 3) for k, v in times.items()}


def cameras(poses, Ho, Wo):
    f = Wo / 2 / np.tan(np.deg2rad(30))
    K = torch.tensor([[f, 0, Wo / 2], [0, f, Ho / 2], [0, 0, 1]], dtype=torch.float32, device="cuda")
    n = len(poses)
    return K, {C: poses[torch.from_numpy(np.linspace(0, n - 1, C).astype(np.int64)).cuda()].contiguous() for C in (1, 8, 32)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=400)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--voxels", default="0.04,0.02")
    ap.add_argument("--size", default="720x1280")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from vista_slam_b200.fusion import fuse_volume, raycast
    from vista_slam_b200.render import render_views
    Ho, Wo = (int(x) for x in a.size.split("x"))
    rows = [{"card": card(), "size": "%dx%d" % (Ho, Wo), "iters": a.iters}]
    print(json.dumps(rows[0]), flush=True)

    maps = room(a.views)
    K, poses = cameras(maps["pose"], Ho, Wo)
    for v in (float(x) for x in a.voxels.split(",")):
        vol = fuse_volume(maps, 0.5, v)
        calls = {}
        for C, P in poses.items():
            calls["raycast_C%d" % C] = (lambda P=P: raycast(vol["bricks"], vol["tsdf"], vol["weight"], vol["color"], v, P,
                                                            K, (Ho, Wo)))
            calls["render_views_C%d" % C] = lambda P=P: render_views(maps, 0.5, P, K, (Ho, Wo))
        calls["fuse_volume_and_raycast_C1"] = lambda: raycast(
            *(lambda o: (o["bricks"], o["tsdf"], o["weight"], o["color"]))(fuse_volume(maps, 0.5, v)), v, poses[1], K,
            (Ho, Wo))
        med = alternated(calls, a.iters)
        hit = float((raycast(vol["bricks"], vol["tsdf"], vol["weight"], vol["color"], v, poses[8], K, (Ho, Wo))["depth"]
                     > 0).float().mean())
        rows.append({"map": "room", "views": a.views, "voxel": v, "bricks": int(vol["bricks"].shape[0]),
                     "hit_fraction_C8": round(hit, 3), "ms": med})
        print(json.dumps(rows[-1]), flush=True)
        del vol

    stream = so.make_stream(seed=3, n_views=a.views, H=224, W=224)
    slam = replayed_slam(stream)
    images = so.stream_images(stream)
    for i in range(a.views):
        slam.step(so_value(images, i, stream))
    del stream, images
    ex = slam._export(0, slam.view_num, cloud=True)
    pts = ex["points"][:int(ex["count"].cpu())]
    ext = float((pts.max(0).values - pts.min(0).values).max())
    del ex, pts
    K, poses = cameras(slam._export(0, slam.view_num, cloud=False)["pose"], Ho, Wo)
    for div in (64, 128):
        v = ext / div
        calls = {}
        for C in (1, 8):
            calls["render_surface_C%d" % C] = lambda C=C: slam.render_surface(poses[C], K, (Ho, Wo), v)
            calls["render_C%d" % C] = lambda C=C: slam.render(poses[C], K, (Ho, Wo))
        med = alternated(calls, a.iters)
        rows.append({"map": "replayed", "views": slam.view_num, "voxel": round(v, 5), "extent_over": div, "ms": med})
        print(json.dumps(rows[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
