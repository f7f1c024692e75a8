"""Per-keyframe step latency of OnlineSLAM on a live-shaped stream, with pose-graph optimisation synchronous
(pgo_background = False) and on a side stream (pgo_background = True), on the default (dense at these sizes) and the
block-sparse route.

224 x 224 synthetic textured frames, random-init weights of the reference architecture, the golden DBoW3 vocabulary,
pgo_every = 50 (run_live.py's setting: each PGO optimises a window of 100 views plus the loop-related views).  After a
warm-up run of every (route, mode), the runs alternate off / on per route in one process.  A step is timed on the host
clock up to a synchronise of the current (main) stream, which does not wait for the background PGO's side stream; the
total includes the final wait_pgo().  The final node / edge tables of the two modes must be equal bit for bit.
Prints one JSON line with the card's name and power limit."""
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


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def stats(v):
    v = np.sort(np.asarray(v) * 1e3)
    q = lambda p: float(v[int(p * (len(v) - 1))])
    return {"p50_ms": q(0.5), "p90_ms": q(0.9), "p99_ms": q(0.99), "max_ms": float(v[-1]), "n": int(len(v))}


def tables(slam):
    G = slam._graph
    N, E, V = slam.num_nodes, slam.num_edges, slam.view_num
    return {"pose": G.pose[:N].cpu().numpy().tobytes(), "edges": G.edges[:E].cpu().numpy().tobytes(),
            "meas": G.meas[:E].cpu().numpy().tobytes(), "weight": G.weight[:E].cpu().numpy().tobytes(),
            "best_node": G.best_node[:V].cpu().numpy().tobytes()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=60)
    ap.add_argument("--pgo-every", type=int, default=50)
    a = ap.parse_args()
    from vista_slam_b200.slam import OnlineSLAM
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    torch.manual_seed(0)
    model = STA().cuda().eval()

    class Live(OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return model

    H = W = 224
    g = torch.Generator().manual_seed(1)
    base = torch.rand(1, 3, H // 8, W // 4, generator=g)
    frames = []
    for i in range(a.keyframes):
        img = torch.nn.functional.interpolate(base.roll(i % (W // 4), dims=3)[..., :W // 8], size=(H, W), mode="bilinear")
        img = ((img * 2 - 1) + 0.05 * torch.randn(1, 3, H, W, generator=g)).clamp(-1, 1).cuda()
        frames.append({"rgb": img, "shape": torch.tensor([[H, W]]), "gray": ((img[0].mean(0) + 1) / 2).contiguous(),
                       "view_name": "%05d" % i})
    vocab = os.path.join(ROOT, "tests", "golden", "loop_vocab.txt")

    def run(route, background, n):
        slam = Live("unused", vocab, max_view_num=max(n, 400) * 2, pgo_every=a.pgo_every)
        slam.pgo_route, slam.pgo_background = route, background
        main_stream = torch.cuda.current_stream()
        lat, pgo = [], 0
        torch.cuda.synchronize()
        t_all = time.perf_counter()
        for i in range(n):
            t0 = time.perf_counter()
            pgo += slam.step(frames[i], force_pgo=(i == n - 1))
            main_stream.synchronize()
            lat.append(time.perf_counter() - t0)
        slam.wait_pgo()
        torch.cuda.synchronize()
        total = time.perf_counter() - t_all
        return slam, lat, total, pgo

    print("card:", card(), flush=True)
    routes = {"default": None, "sparse": "sparse"}
    for route in routes.values():
        for bg in (False, True):
            run(route, bg, a.warmup)
    res = {"card": card(), "size": "224x224", "keyframes": a.keyframes, "pgo_every": a.pgo_every}
    for name, route in routes.items():
        out = {}
        for bg in (False, True):
            slam, lat, total, pgo = run(route, bg, a.keyframes)
            out["on" if bg else "off"] = dict(step=stats(lat), total_s=total, pgos=pgo, nodes=slam.num_nodes,
                                              edges=slam.num_edges, tables=tables(slam))
            del slam
            torch.cuda.empty_cache()
        assert out["on"].pop("tables") == out["off"].pop("tables"), "background PGO changed the graph (%s route)" % name
        res[name] = out
        print(name, json.dumps(out), flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
