"""Pose-graph optimisation on OnlineSLAM-shaped graphs: the dense route against the block-sparse route of PoseGraphOpt.

The graphs come from the drop-in OnlineSLAM replayed over oracle/slam_oracle.py::make_stream, with the frontend, the
keyframe regression and the loop detector substituted as tests/test_slam_gpu.py does, every edge kept
(rel_pose_thres = 0) and pgo_every above the run length, so that no PGO runs during the replay.  The graph only grows,
so the tables after view v are the graph of a v-view run; each size takes the prefix whose node count first reaches
it, with every node optimised.  Per size and route, after a warm-up step: the plan (sparse route: host analysis and
upload), one LM step, and a whole optimize() from a fresh PoseGraphOpt (plan included), each timed from its first call
to a device synchronise.  The dense route is timed once per size.  Prints the card's name and power limit, then one
JSON line per size: fill (nonzero 7x7 blocks of L against A's lower triangle), elimination-tree levels, device bytes of
each route, the timed step's losses and Cholesky flag, and the largest |node difference| between the two routes'
optimize() results where both run."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def timed(f):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = f()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dense", default="500,1000,2000,3600")
    ap.add_argument("--sparse", default="500,1000,2000,3600,7200,14400")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import test_slam_gpu as tsg
    from oracle import slam_oracle as so
    from vista_slam_b200 import _lib
    from vista_slam_b200.pose_graph import PoseGraphOpt
    dense_sizes = [int(s) for s in a.dense.split(",") if s]
    sparse_sizes = [int(s) for s in a.sparse.split(",") if s]
    target = max(dense_sizes + sparse_sizes)
    views = int(target / 6.5) + 20
    stream = so.make_stream(n_views=views)
    slam = tsg._replay_slam(stream, max_view_num=views + 10, pgo_every=10 ** 6, rel_pose_thres=0.0)
    images = so.stream_images(stream)
    counts = []
    for i in range(views):
        slam.step(tsg._value(images, i, stream))
        counts.append((slam.num_nodes, slam.num_edges))
        if slam.num_nodes >= target:
            break
    G = slam._graph
    print("card:", card())
    L = _lib.lib()
    for size in sorted(set(dense_sizes + sparse_sizes)):
        N, E = next(c for c in counts if c[0] >= size)
        nodes, edges, meas, weight = G.pose[:N].clone(), G.edges[:E], G.meas[:E], G.weight[:E]
        opt = torch.arange(N, device="cuda")
        rec = {"nodes": N, "edges": E}
        e_host, o_host = edges.cpu().numpy(), np.arange(N, dtype=np.int64)
        st = (ctypes.c_int64 * 5)()
        _lib.check(L.sta_pg_plan_analyze(e_host.ctypes.data, E, N, o_host.ctypes.data, N, st, *([None] * 6)), "analyze")
        rec.update(l_blocks=int(st[0]), a_blocks=int(st[1]), fill=round(st[0] / st[1], 3), levels=int(st[2]),
                   updates=int(st[3]))
        results = {}
        for route, sizes in (("dense", dense_sizes), ("sparse", sparse_sizes)):
            if size not in sizes:
                continue
            if route == "dense" and N > _lib.PG_DENSE_MAX_OPT:
                rec["dense"] = "refused: more than %d optimised nodes" % _lib.PG_DENSE_MAX_OPT
                continue

            def fresh():
                g = PoseGraphOpt(nodes, opt)
                g.sparse = route == "sparse"
                return g
            g = fresh()
            r = {}
            if route == "sparse":
                plan, r["plan_ms"] = timed(lambda: g.plan(edges))
                r["device_bytes"] = plan.info()["device_bytes"]
            else:
                r["device_bytes"] = int(L.sta_pose_graph_scratch_bytes(N, E, N))
            g.lm_step(edges, meas, weight, 1e-4)  # warm-up
            step, r["step_ms"] = timed(lambda: g.lm_step(edges, meas, weight, 1e-4))
            r["step_loss"], r["step_ok"] = [step[1], step[2]], step[4]
            g = fresh()
            losses, r["optimize_ms"] = timed(lambda: g.optimize(edges, meas, weight))
            r["iterations"] = len(losses)
            r["loss"] = [losses[0], losses[-1]]
            results[route] = g.get_nodes()
            rec[route] = r
            del g
            torch.cuda.empty_cache()
        if len(results) == 2:
            rec["max_abs_node_diff"] = float((results["dense"] - results["sparse"]).abs().max())
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
