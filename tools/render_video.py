"""The frames of the reference's scripts/video.py, drawn on the GPU by the map renderer (vista_slam_b200/render.py).

    python tools/render_video.py FOLDER --out DIR [--size 480x720] [--radius 0] [--follow] [--camera w2c.npy]
                                 [--surface VOXEL [--min-weight N]]

FOLDER holds what OnlineSLAM.save_data_all and log_intermediate_results write: trajectory{_k}.npy, scales{_k}.npy,
depths.npy, confs.npz, intrinsics.npy, images.npy and view_graph.npz.  Frame v shows views 0..v with the poses of the
first intermediate trajectory whose index is >= v (the final trajectory after the last), the current camera's frustum
at scale 1.0, the previous one at 0.8 and the others at 0.1, and the graph's edges among views <= v; at each PGO index
an extra frame v_pgo shows the new trajectory.  Cameras: --follow is video.py's offset camera (20 degrees about x, then
[0, 0.3, 5]) composed with the current view's world-to-camera; --camera is a fixed 4x4 world-to-camera; by default a
fixed camera above the camera centres looks along their mean up axis (-y of the poses), backed off until every centre
is in frame.  Colours are the images' (not video.py's /1.5 shading); frames are PNG when cv2 imports, .npy otherwise.
With --surface VOXEL each frame draws, instead of point splats, the map fused into a TSDF volume of that voxel size
and ray-cast with a headlight (fusion.fuse_volume, fusion.raycast; min_weight --min-weight); the lines are drawn by
render_views over the same map with every point masked out and kept where they are nearer than the surface.
Prints each frame's render time (device time, the call synchronised)."""
import argparse
import glob
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from vista_slam_b200.fusion import fuse_volume, raycast  # noqa: E402
from vista_slam_b200.render import camera_frusta, concat_lines, graph_segments, render_views  # noqa: E402

CAMERA_COLOR = (0.6, 0.8, 1.0)
CUR_CAMERA_COLOR = (0.0745, 0.3137, 0.1059)
PRE_CAMERA_COLOR = (0.0431, 0.4627, 0.6274)


def follow_offset():
    a = np.deg2rad(20.0)
    off = np.eye(4)
    off[:3, :3] = [[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]]
    off[:3, 3] = [0, 0.3, 5]
    return off


def overhead_w2c(traj, K, Ho, Wo):
    """World-to-camera of a camera above the centres, looking along their mean up axis (-y of the poses), at a distance
    that puts every centre in the Ho x Wo image."""
    centres = traj[:, :3, 3]
    up = -traj[:, :3, 1].mean(0)
    up /= np.linalg.norm(up)
    fwd = -up  # look down onto the trajectory
    ref = traj[0, :3, 2] - traj[0, :3, 2].dot(fwd) * fwd
    if np.linalg.norm(ref) < 1e-6:
        ref = np.eye(3)[np.argmin(np.abs(fwd))]
    down = ref / np.linalg.norm(ref)  # image rows along the first camera's viewing direction
    right = np.cross(down, fwd)
    R = np.stack([right, down, fwd])  # rows: camera axes in the world
    mid = centres.mean(0)
    local = (centres - mid) @ R.T
    half = max(np.abs(local[:, 0]).max() / (Wo / 2 / K[0, 0]), np.abs(local[:, 1]).max() / (Ho / 2 / K[1, 1]), 1e-3)
    eye = mid - fwd * (half * 1.2 + np.abs(local[:, 2]).max())
    w2c = np.eye(4)
    w2c[:3, :3], w2c[:3, 3] = R, -R @ eye
    return w2c


def surface_frame(maps, thres, c2w, K, size, lines, voxel, min_weight):
    """The fused surface of maps ray-cast from c2w [1,4,4], with lines drawn by render_views over the same map with
    every point masked out (conf -inf), each pixel taking the nearer of the two."""
    vol = fuse_volume(maps, thres, voxel)
    surf = raycast(vol["bricks"], vol["tsdf"], vol["weight"], vol["color"], voxel, c2w, K, size, min_weight=min_weight)
    bare = dict(maps, conf=torch.full_like(maps["conf"], float("-inf")))
    ln = render_views(bare, thres, c2w, K, size, lines=lines)
    front = (ln["depth"] > 0) & ((surf["depth"] == 0) | (ln["depth"] < surf["depth"]))
    return {"rgb": torch.where(front[..., None], ln["rgb"], surf["rgb"]),
            "depth": torch.where(front, ln["depth"], surf["depth"])}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("folder")
    ap.add_argument("--out", required=True)
    ap.add_argument("--size", default="480x720")
    ap.add_argument("--radius", type=int, default=0)
    ap.add_argument("--follow", action="store_true")
    ap.add_argument("--camera", default=None)
    ap.add_argument("--surface", type=float, default=None, metavar="VOXEL")
    ap.add_argument("--min-weight", type=float, default=1.0)
    a = ap.parse_args(argv)
    Ho, Wo = (int(x) for x in a.size.lower().split("x"))
    F = a.folder
    pgo_idx = sorted(int(os.path.basename(p)[len("scales_"):-len(".npy")]) for p in glob.glob(os.path.join(F, "scales_*.npy")))
    if not pgo_idx:
        raise SystemExit("no scales_<k>.npy in %s: run with log_intermediate_results" % F)
    dev = torch.device("cuda")
    depths = torch.from_numpy(np.load(os.path.join(F, "depths.npy"))).to(dev)
    confs_npz = np.load(os.path.join(F, "confs.npz"), allow_pickle=True)
    confs = torch.from_numpy(confs_npz["confs"]).to(dev)
    thres = float(confs_npz["thres"])
    intri_np = np.load(os.path.join(F, "intrinsics.npy"))
    intri = torch.from_numpy(intri_np).to(dev)
    images = torch.from_numpy(np.load(os.path.join(F, "images.npy"))).to(dev).permute(0, 3, 1, 2) * 2 - 1
    vg = np.load(os.path.join(F, "view_graph.npz"), allow_pickle=True)
    view_graph, loop_min_dist = vg["view_graph"].item(), int(vg["loop_min_dist"])
    H, W = depths.shape[1:]
    # the output camera's intrinsics: a 60 degree horizontal field of view
    f = Wo / 2 / np.tan(np.deg2rad(30))
    K = np.array([[f, 0, Wo / 2], [0, f, Ho / 2], [0, 0, 1]])
    fixed = np.load(a.camera) if a.camera else None
    os.makedirs(a.out, exist_ok=True)
    try:
        import cv2
    except ImportError:
        cv2 = None

    def load(k):
        if k is None:
            return np.load(os.path.join(F, "trajectory.npy")), np.load(os.path.join(F, "scales.npy"))
        return np.load(os.path.join(F, "trajectory_%d.npy" % k)), np.load(os.path.join(F, "scales_%d.npy" % k))

    pgo_i = 0
    traj, scales = load(pgo_idx[0])
    overhead = None

    def frame(v, traj, scales, name, pre):
        nonlocal overhead
        n = v + 1
        maps = {"pose": torch.from_numpy(traj[:n]).float().to(dev), "scale": torch.from_numpy(scales[:n]).float().reshape(n, 1).to(dev),
                "depth": depths[:n], "conf": confs[:n], "intri": intri[:n], "images": images[:n].contiguous()}
        parts = [camera_frusta(traj[v:v + 1], intri_np[v], H, W, 1.0, CUR_CAMERA_COLOR)]
        small = [i for i in range(n) if i != v and i != pre]
        if pre is not None:
            parts.append(camera_frusta(traj[pre:pre + 1], intri_np[pre], H, W, 0.8, PRE_CAMERA_COLOR))
        if small:
            parts.append(camera_frusta(traj[small], intri_np[small], H, W, 0.1, CAMERA_COLOR))
        parts.append(graph_segments(traj, view_graph, loop_min_dist, range(n)))
        w2c_v = np.linalg.inv(traj[v].astype(np.float64))
        if a.follow:
            w2c = follow_offset() @ w2c_v
        elif fixed is not None:
            w2c = fixed
        else:
            if overhead is None:
                overhead = overhead_w2c(np.load(os.path.join(F, "trajectory.npy")).astype(np.float64), K, Ho, Wo)
            w2c = overhead
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        c2w = np.linalg.inv(w2c)[None]
        if a.surface is None:
            out = render_views(maps, thres, c2w, K, (Ho, Wo), point_radius=a.radius, lines=concat_lines(*parts))
        else:
            out = surface_frame(maps, thres, c2w, K, (Ho, Wo), concat_lines(*parts), a.surface, a.min_weight)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        rgb = out["rgb"][0].cpu().numpy()
        if cv2 is not None:
            cv2.imwrite(os.path.join(a.out, name + ".png"), (rgb[..., ::-1] * 255).round().astype(np.uint8))
        else:
            np.save(os.path.join(a.out, name + ".npy"), rgb)
        print("%s: %d views, %.2f ms" % (name, n, ms), flush=True)

    length = pgo_idx[-1] + 1
    for v in range(length):
        frame(v, traj, scales, "%04d" % v, v - 1 if v > 0 else None)
        if v == pgo_idx[pgo_i]:
            if pgo_i == len(pgo_idx) - 1:
                traj, scales = load(None)
            else:
                pgo_i += 1
                traj, scales = load(pgo_idx[pgo_i])
            frame(v, traj, scales, "%04d_pgo" % v, v - 1 if v > 0 else None)


if __name__ == "__main__":
    main()
