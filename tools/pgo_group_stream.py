"""Pose-graph optimisation of several graphs at once: PoseGraphOpt.optimize_group against each graph's own optimize().

The graphs are OnlineSLAM-shaped: tools/pgo_stream.py's generator (the drop-in OnlineSLAM replayed over
oracle/slam_oracle.py::make_stream, every edge kept, no PGO during the replay), one stream seed per graph, each graph the
prefix whose node count first reaches the size, every node optimised.  Per size and group size G, after a warm-up:

  * step: G solo LM steps (PoseGraphOpt.lm_step, one read-back each) against one group step (one launch sequence, one
    read-back);
  * optimize: each graph's optimize() back to back against one optimize_group, with the plateau rule (each graph stops
    on its own) and with a fixed number of iterations (patience above steps, so both arms run 20 steps per graph).

The arms alternate, each sample ends in a device synchronise, and the median of --reps samples is printed.  The live
case replays S = 8 sessions (pgo_every past their length) and times one SLAMSessions.optimize over all of them against
eight pose_graph_optimize calls, from the same restored state.  Prints the card's name and power limit, then one JSON
line per measurement; each line also says whether the group's nodes equal the solo runs' bit for bit."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def timed(f):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = f()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t) * 1e3


def alternate(arms, reps):
    """{name: (result of the last sample, median ms)} of arms {name: f}, alternated after one warm-up sample each."""
    ms = {k: [] for k in arms}
    out = {}
    for r in range(reps + 1):
        for k, f in arms.items():
            out[k], t = timed(f)
            if r:
                ms[k].append(t)
    return {k: (out[k], round(statistics.median(ms[k]), 3)) for k in arms}


def graphs_at(sizes, seeds):
    """{size: [(nodes, edges, meas, weight), ...] one per seed}."""
    import test_slam_gpu as tsg
    from oracle import slam_oracle as so
    target = max(sizes)
    views = int(target / 6.5) + 20
    out = {s: [] for s in sizes}
    for seed in seeds:
        stream = so.make_stream(seed=seed, n_views=views)
        slam = tsg._replay_slam(stream, max_view_num=views + 10, pgo_every=10 ** 6, rel_pose_thres=0.0)
        images = so.stream_images(stream)
        counts = []
        for i in range(views):
            slam.step(tsg._value(images, i, stream))
            counts.append((slam.num_nodes, slam.num_edges))
            if slam.num_nodes >= target:
                break
        G = slam._graph
        for s in sizes:
            N, E = next(c for c in counts if c[0] >= s)
            out[s].append((G.pose[:N].clone(), G.edges[:E].clone(), G.meas[:E].clone(), G.weight[:E].clone()))
        del slam
        torch.cuda.empty_cache()
    return out


def group_case(size, probs, reps):
    from vista_slam_b200.pose_graph import PoseGraphOpt, _DenseGroup
    G = len(probs)
    opts = [torch.arange(p[0].shape[0], device="cuda") for p in probs]
    rec = {"size": size, "G": G, "nodes": [int(p[0].shape[0]) for p in probs], "edges": [int(p[1].shape[0]) for p in probs]}

    def fresh():
        return [PoseGraphOpt(p[0], o) for p, o in zip(probs, opts)]

    # one LM step
    solo_g, grp_g = fresh(), fresh()
    dense = _DenseGroup(grp_g, [p[1] for p in probs], [p[2] for p in probs], [p[3] for p in probs])
    r = alternate({"solo": lambda: [g.lm_step(p[1], p[2], p[3], 1e-4)[0] for g, p in zip(solo_g, probs)],
                   "group": lambda: [c[0] for c in dense.step(list(range(G)), [1e-4] * G)]}, reps)
    rec["step_ms"] = {"solo": r["solo"][1], "group": r["group"][1]}
    rec["step_equal"] = all(torch.equal(a, b) for a, b in zip(r["solo"][0], r["group"][0]))
    del dense, solo_g, grp_g
    # whole optimisations, with the plateau rule and with a fixed 20 iterations
    for name, kw in (("optimize", {}), ("optimize_fixed20", {"patience": 10 ** 6})):
        box = {}

        def solo():
            gs = fresh()
            box["solo"] = ([g.optimize(p[1], p[2], p[3], **kw) for g, p in zip(gs, probs)], [g.nodes for g in gs])

        def group():
            gs = fresh()
            box["group"] = (PoseGraphOpt.optimize_group(gs, [p[1] for p in probs], [p[2] for p in probs],
                                                        [p[3] for p in probs], **kw), [g.nodes for g in gs])
        r = alternate({"solo": solo, "group": group}, reps)
        rec[name + "_ms"] = {"solo": r["solo"][1], "group": r["group"][1]}
        rec[name + "_iterations"] = {"solo_total": sum(len(h) for h in box["solo"][0]),
                                     "group": max(len(h) for h in box["group"][0])}
        rec[name + "_equal"] = (box["solo"][0] == box["group"][0] and
                                all(torch.equal(a, b) for a, b in zip(box["solo"][1], box["group"][1])))
        box.clear()
        torch.cuda.empty_cache()
    for k in ("step_ms", "optimize_ms", "optimize_fixed20_ms"):
        rec[k]["solo_over_group"] = round(rec[k]["solo"] / rec[k]["group"], 3)
    return rec


def live_case(S, views, reps):
    from oracle import slam_oracle as so
    from test_sessions_gpu import _replay_sessions
    from test_slam_gpu import _value
    streams = [so.make_stream(seed=100 + k, n_views=views) for k in range(S)]
    ses = _replay_sessions(streams, pgo_every=10 ** 6, verbose=True, max_view_num=views + 10)
    ses.step({k: [_value(so.stream_images(s), i, s) for i in range(views)] for k, s in enumerate(streams)})
    saved = [(s._graph.pose[:s.num_nodes].clone(), set(s.loop_related_views)) for s in ses.sessions]

    def restore():
        for s, (pose, lrv) in zip(ses.sessions, saved):
            s._graph.pose[:s.num_nodes] = pose
            s.loop_related_views = set(lrv)

    def per_session():
        restore()
        torch.cuda.synchronize()
        t = time.perf_counter()
        for s in ses.sessions:
            s.pose_graph_optimize()
        torch.cuda.synchronize()
        return [s._graph.pose[:s.num_nodes].clone() for s in ses.sessions], (time.perf_counter() - t) * 1e3

    def together():
        restore()
        torch.cuda.synchronize()
        t = time.perf_counter()
        ses.optimize(range(S))
        torch.cuda.synchronize()
        return [s._graph.pose[:s.num_nodes].clone() for s in ses.sessions], (time.perf_counter() - t) * 1e3

    import contextlib
    import io
    ms = {"per_session": [], "together": []}
    with contextlib.redirect_stdout(io.StringIO()):  # the PGO messages
        for r in range(reps + 1):
            a, ta = per_session()
            b, tb = together()
            if r:
                ms["per_session"].append(ta)
                ms["together"].append(tb)
    rec = {"live_sessions": S, "views": views, "nodes": [s.num_nodes for s in ses.sessions],
           "ms": {k: round(statistics.median(v), 3) for k, v in ms.items()},
           "equal": all(torch.equal(x, y) for x, y in zip(a, b))}
    rec["ms"]["per_session_over_together"] = round(rec["ms"]["per_session"] / rec["ms"]["together"], 3)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="500,1000")
    ap.add_argument("--groups", default="1,2,4,8")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--live-views", type=int, default=80)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from pgo_stream import card
    print("card:", card(), flush=True)
    sizes = [int(s) for s in a.sizes.split(",") if s]
    groups = [int(g) for g in a.groups.split(",") if g]
    probs = graphs_at(sizes, range(1, max(groups) + 1)) if sizes else {}
    for size in sizes:
        for G in groups:
            print(json.dumps(group_case(size, probs[size][:G], a.reps)), flush=True)
            torch.cuda.empty_cache()
    if a.live_views:
        print(json.dumps(live_case(8, a.live_views, a.reps)), flush=True)


if __name__ == "__main__":
    main()
