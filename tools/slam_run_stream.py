"""Per-keyframe latency of the drop-in OnlineSLAM (vista_slam_b200/slam.py) at 224 x 224, and of save_data_all.

Random-init weights of the reference architecture and synthetic textured frames (a shifting smooth texture plus noise),
the golden DBoW3 vocabulary for loop detection.  Each step is split, with a device synchronisation around every part,
into the frontend (encoder + gated edge regression), loop detection and the graph update; the step totals include
those synchronisations.  save_data_all (every file, PLY included) is timed at 100 and at 400 views.
Prints the card's name and power limit.  The reference's host path is not measured here (it needs pypose)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def stats(v):
    v = np.sort(np.asarray(v) * 1e3)
    return {"median_ms": float(np.median(v)), "p90_ms": float(v[int(0.9 * (len(v) - 1))]), "n": int(len(v))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    from vista_slam_b200.slam import OnlineSLAM
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    torch.manual_seed(0)
    model = STA().cuda().eval()
    parts = {"frontend": [], "lc": [], "graph": []}

    def timed(name, f, *args):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = f(*args)
        torch.cuda.synchronize()
        if timing[0]:
            parts[name][-1] += time.perf_counter() - t0
        return r

    timing = [False]

    class Timed(OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return model

        def add_view(self, *args):
            return timed("frontend", super().add_view, *args)

        def _regress_keyframe(self, i, js):
            return timed("frontend", super()._regress_keyframe, i, js)

        def _add_keyframe(self, *args):
            return timed("graph", super()._add_keyframe, *args)

    H = W = 224
    g = torch.Generator().manual_seed(1)
    base = torch.rand(1, 3, H // 8, W // 4, generator=g)

    def frame(i):
        img = torch.nn.functional.interpolate(base.roll(i % (W // 4), dims=3)[..., :W // 8], size=(H, W), mode="bilinear")
        img = ((img * 2 - 1) + 0.05 * torch.randn(1, 3, H, W, generator=g)).clamp(-1, 1).cuda()
        return {"rgb": img, "shape": torch.tensor([[H, W]]), "gray": ((img[0].mean(0) + 1) / 2).contiguous(),
                "view_name": "%05d" % i}

    vocab = os.path.join(ROOT, "tests", "golden", "loop_vocab.txt")
    print("card:", card(), flush=True)
    # the defaults of OnlineSLAM, with PGO only at the end (pgo_every = 500) as in run.py's default configs
    slam = Timed("unused", vocab)
    lc = slam.lc_detector
    orig_detect = lc.detect_loop

    def detect(*args):
        return timed("lc", orig_detect, *args)

    lc.detect_loop = detect
    total, save = [], {}
    for i in range(a.views):
        timing[0] = i >= a.warmup
        for p in parts.values():
            p.append(0.0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        slam.step(frame(i))
        torch.cuda.synchronize()
        if timing[0]:
            total.append(time.perf_counter() - t0)
        if slam.view_num in (100, a.views):
            with tempfile.TemporaryDirectory() as d:
                slam.save_data_all(d)  # warm
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                slam.save_data_all(d)
                save[slam.view_num] = time.perf_counter() - t0
    res = {"card": card(), "size": "224x224", "views": a.views, "step_total": stats(total),
           **{"step_" + k: stats(v[a.warmup:]) for k, v in parts.items()},
           "save_data_all_ms": {str(k): 1e3 * v for k, v in save.items()}, "nodes": slam.num_nodes, "edges": slam.num_edges}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
