"""OnlineSLAM.step against step_many at 224 x 224: milliseconds per keyframe over a 400-keyframe stream.

The stream of tools/slam_run_stream.py: random-init weights of the reference architecture, synthetic textured frames,
the golden DBoW3 vocabulary, OnlineSLAM's defaults with pgo_every = 500 and force_pgo on the last keyframe.  One
process alternates whole runs of `step` and of `step_many` in chunks of 8, 16, 32 and 64 keyframes, after a warm-up
run of each; every run is timed from its first call to a device synchronise after its last.  Loop detection is timed
on its own in the same way (detect_loop per frame against detect_loops per chunk) for its share.  The graphs are
compared: integer tables exactly, node poses as the largest absolute difference.  Prints the card's name and power
limit, then one JSON line."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=400)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--chunks", default="8,16,32,64")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from vista_slam_b200.slam import OnlineSLAM
    from vista_slam_b200.loop_detector import LoopDetector
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    torch.manual_seed(0)
    model = STA().cuda().eval()
    vocab = os.path.join(ROOT, "tests", "golden", "loop_vocab.txt")

    class Slam(OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return model

    H = W = 224
    g = torch.Generator().manual_seed(1)
    base = torch.rand(1, 3, H // 8, W // 4, generator=g)
    values = []
    for i in range(a.views):
        img = torch.nn.functional.interpolate(base.roll(i % (W // 4), dims=3)[..., :W // 8], size=(H, W), mode="bilinear")
        img = ((img * 2 - 1) + 0.05 * torch.randn(1, 3, H, W, generator=g)).clamp(-1, 1).cuda()
        values.append({"rgb": img, "shape": torch.tensor([[H, W]]), "gray": ((img[0].mean(0) + 1) / 2).contiguous(),
                       "view_name": "%05d" % i})
    chunks = [int(c) for c in a.chunks.split(",")]
    n = a.views

    def run(chunk):
        slam = Slam("unused", vocab, pgo_every=500)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if chunk is None:
            for i, v in enumerate(values):
                slam.step(v, force_pgo=(i == n - 1))
        else:
            for c in range(0, n, chunk):
                slam.step_many(values[c:c + chunk], force_pgo=(c + chunk >= n))
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        G = slam._graph
        N, E = slam.num_nodes, slam.num_edges
        tables = {"node_to_view": G.node_to_view[:N].cpu().numpy(), "edges": G.edges[:E].cpu().numpy(),
                  "best_node": G.best_node[:n].cpu().numpy(), "pose": G.pose[:N].cpu().numpy()}
        del slam
        torch.cuda.empty_cache()
        return dt, tables

    def run_lc(chunk):
        det = LoopDetector(vocab, 40, 40, 5)
        grays = [v["gray"] for v in values]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if chunk is None:
            for i, x in enumerate(grays):
                det.detect_loop(x, max(0, i - 3))
        else:
            for c in range(0, n, chunk):
                det.detect_loops(grays[c:c + chunk], [max(0, i - 3) for i in range(c, min(n, c + chunk))])
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    print("card:", card(), flush=True)
    modes = [None] + chunks
    name = {m: "step" if m is None else "step_many_%d" % m for m in modes}
    for m in modes:  # warm-up: every shape and CUDA graph of every mode
        run(m)
        run_lc(m)
    times = {name[m]: [] for m in modes}
    lc = {name[m]: [] for m in modes}
    tables = {}
    for _ in range(a.rounds):
        for m in modes:
            dt, tables[name[m]] = run(m)
            times[name[m]].append(dt)
            lc[name[m]].append(run_lc(m))
    ref = tables["step"]
    res = {"card": card(), "size": "%dx%d" % (H, W), "views": n, "rounds": a.rounds, "modes": {}}
    for m in modes:
        t = tables[name[m]]
        agree = all(t[k].shape == ref[k].shape and np.array_equal(t[k], ref[k]) for k in ("node_to_view", "edges", "best_node"))
        ms = 1e3 * min(times[name[m]]) / n
        lc_ms = 1e3 * min(lc[name[m]]) / n
        res["modes"][name[m]] = {
            "ms_per_keyframe": round(ms, 3), "ms_per_keyframe_all": [round(1e3 * x / n, 3) for x in times[name[m]]],
            "lc_ms_per_keyframe": round(lc_ms, 3), "lc_share": round(lc_ms / ms, 3), "graph_integers_equal_step": agree,
            "max_pose_diff_vs_step": float(np.abs(t["pose"] - ref["pose"]).max()) if agree else None,
            "speedup_vs_step": round(1e3 * min(times["step"]) / n / ms, 3)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
