"""Time of OnlineSLAM.render on a 400-view 224 x 224 map, beside what a host viewer pays today for the same map.

The map is the seeded synthetic stream of oracle/slam_oracle.make_stream (planted trajectory with loops, smooth depths,
about half of the pixels confident) replayed through OnlineSLAM with the frontend replaced, as the GPU tests do.  The
renders are 720 x 1280 from C = 1, 8 and 32 cameras (the views' own poses, spread over the trajectory) at point radius 0
and 1, with no lines and with every view's frustum (8 segments) and every graph edge.  The host viewer's cost is
_export(cloud=True) and the copy of the points and colours to the host.  The two are timed alternately in one process,
each call between device synchronisations; the card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from oracle import slam_oracle as so  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def replayed_slam(stream):
    from vista_slam_b200.slam import OnlineSLAM

    class _Frontend(torch.nn.Module):
        def _encode_image(self, image, image_shape, normalize=False):
            return torch.zeros(1, 1, 1024, device="cuda"), None

    class _Loops:
        def __init__(self):
            self.calls, self.loop_dist_min = 0, 5

        def detect_loop(self, image, farthest_neighbor):
            c = stream["loops"][self.calls]
            self.calls += 1
            return list(c)

    class Replay(OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return _Frontend()

        def _regress_keyframe(self, i, js):
            E = [stream["edges"][(i, j)] for j in js]
            keep = [k for k, (j, e) in enumerate(zip(js, E)) if so.keep_edge(e["conf"], i, j, self.rel_pose_thres)]
            conf = torch.from_numpy(np.stack([np.stack([E[k]["confs"][r] for k in keep]) for r in range(2)])).cuda()
            return [float(e["conf"]) for e in E], keep, {
                "pose": torch.from_numpy(np.stack([e["pose"] for e in E])).cuda(),
                "pose_conf": torch.tensor([float(e["conf"]) for e in E], dtype=torch.float32, device="cuda"),
                "conf": conf,
                "depths": torch.from_numpy(np.stack([np.stack([E[k]["depths"][r] for k in keep]) for r in range(2)])).cuda(),
                "intri": torch.from_numpy(np.stack([E[k]["intri"] for k in keep])).cuda(),
                "conf_mean": conf.mean(dim=(2, 3)).contiguous()}

    slam = Replay("unused", os.path.join(ROOT, "tests", "golden", "loop_vocab.txt"), loop_dist_min=5, pgo_every=100000)
    slam.lc_detector = _Loops()
    return slam


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=400)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--size", default="720x1280")
    a = ap.parse_args()
    Ho, Wo = (int(x) for x in a.size.split("x"))
    from vista_slam_b200.render import camera_frusta, concat_lines, graph_segments
    print("card:", card(), flush=True)
    t0 = time.perf_counter()
    stream = so.make_stream(seed=3, n_views=a.views, H=224, W=224)
    images = so.stream_images(stream)
    slam = replayed_slam(stream)
    for i in range(a.views):
        slam.step({"rgb": torch.from_numpy(images[i])[None].cuda(), "shape": torch.tensor([[224, 224]]), "gray": None,
                   "view_name": "%05d" % i})
    del stream
    print("map built in %.1f s: %d views, %d nodes" % (time.perf_counter() - t0, slam.view_num, slam.num_nodes), flush=True)
    n = slam.view_num
    ex = slam._export(0, n, cloud=False)
    traj, intri = ex["pose"].cpu().numpy(), ex["intri"].cpu().numpy()
    confident = int((ex["conf"] > slam.conf_thres).sum())
    lines = concat_lines(camera_frusta(traj, intri, 224, 224, 0.1, (0.6, 0.8, 1.0)),
                         graph_segments(traj, slam.get_view_graph(), 5, range(n)))
    lines = tuple(torch.from_numpy(x).cuda() for x in lines)
    f = Wo / 2 / np.tan(np.deg2rad(30))
    K = torch.tensor([[f, 0, Wo / 2], [0, f, Ho / 2], [0, 0, 1]], dtype=torch.float32, device="cuda")
    poses = {C: torch.from_numpy(traj[np.linspace(0, n - 1, C).astype(int)]).cuda() for C in (1, 8, 32)}

    def host_viewer():
        out = slam._export(0, n, cloud=True)
        m = int(out["count"])
        return out["points"][:m].cpu(), out["colors"][:m].cpu()

    cases = [(C, r, ln) for C in (1, 8, 32) for r in (0, 1) for ln in (False, True)]
    calls = {c: (lambda c=c: slam.render(poses[c[0]], K, (Ho, Wo), point_radius=c[1], lines=lines if c[2] else None))
             for c in cases}
    calls["host"] = host_viewer
    times = {k: [] for k in calls}
    for it in range(a.iters + 2):  # two warm-up rounds
        for k, fn in calls.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if it >= 2:
                times[k].append(time.perf_counter() - t0)
    med = {k: float(np.median(v) * 1e3) for k, v in times.items()}
    res = {"card": card(), "views": n, "map": "224x224", "confident_points": confident, "segments": int(lines[0].shape[0]),
           "out": "%dx%d" % (Ho, Wo), "iters": a.iters,
           "render_ms": {"C%d_r%d_%s" % (C, r, "lines" if ln else "points"): med[(C, r, ln)] for C, r, ln in cases},
           "host_viewer_export_cloud_and_copy_ms": med["host"]}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
