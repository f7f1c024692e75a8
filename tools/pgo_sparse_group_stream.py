"""Pose-graph optimisation of several graphs at once on the block-sparse route: one sta_pose_graph_lm_step_sparse_group
launch sequence per LM iteration against each graph's own sparse steps, and against the dense group.

The graphs are those of tools/pgo_group_stream.py: OnlineSLAM-shaped (the drop-in OnlineSLAM replayed over
oracle/slam_oracle.py::make_stream, every edge kept, no PGO during the replay), one stream seed per graph, each graph the
prefix whose node count first reaches the size, every node optimised.  Per size and group size G, after a warm-up:

  * step: G solo sparse LM steps (PoseGraphOpt.lm_step, one read-back each), one sparse group step and one dense group
    step (one launch sequence and one read-back each);
  * optimize: each graph's own optimize() on the sparse route back to back, one optimize_group of sparse-route graphs
    and one of dense-route graphs, with the plateau rule and with a fixed 20 iterations (patience above steps);
  * plan: building the G member plans (host analysis and one upload each, as every optimize() does) and the group plans
    over them, timed apart from the steps.

The dense arm runs up to --dense-max nodes: its scratch grows as (7 n)^2 per graph and its step as n^3.  The arms
alternate, each sample ends in a device synchronise, and the median of --reps samples is printed.  The live case
replays 8 sessions of --live-views keyframes (pgo_every past their length) and times one SLAMSessions.optimize over all
of them with every session on the dense route, then on the sparse route, and the sparse route one session at a time,
from the same restored state.  Prints the card's name and power limit, then one JSON line per measurement; each line says
whether the sparse group's results equal the solo sparse runs' bit for bit, and how far the dense route's nodes are from
the sparse route's."""
import argparse
import contextlib
import io
import json
import statistics
import time

import torch

from pgo_group_stream import alternate, graphs_at, timed


def _fresh(probs, route):
    from vista_slam_b200.pose_graph import PoseGraphOpt
    return [PoseGraphOpt(p[0], torch.arange(p[0].shape[0], device="cuda"), route=route) for p in probs]


def _max_diff(a, b):
    return max(float((x - y).abs().max()) for x, y in zip(a, b))


def group_case(size, probs, reps, dense_max):
    from vista_slam_b200.pose_graph import PoseGraphOpt, _DenseGroup, _SparseGroup, _SparsePlan
    G = len(probs)
    E, P, W = [p[1] for p in probs], [p[2] for p in probs], [p[3] for p in probs]
    dense_on = size <= dense_max
    rec = {"size": size, "G": G, "nodes": [int(p[0].shape[0]) for p in probs], "edges": [int(e.shape[0]) for e in E]}

    # plans: the members' (host analysis + upload), then the group plans over them (the members' plans already built,
    # so _SparseGroup's construction is the group plans alone)
    t_plans, t_group = [], []
    for r in range(reps + 1):
        _, t = timed(lambda: [_SparsePlan(e, p[0].shape[0], torch.arange(p[0].shape[0])) for e, p in zip(E, probs)])
        gs = _fresh(probs, "sparse")
        for g, e in zip(gs, E):
            g.plan(e)
        sg, t2 = timed(lambda: _SparseGroup(gs, E, P, W))
        if r:
            t_plans.append(t)
            t_group.append(t2)
        rec["group_plan_info"] = sg.plan_info()
        del sg, gs
    rec["plan_ms"] = {"members": round(statistics.median(t_plans), 3), "group_plans": round(statistics.median(t_group), 3)}

    # one LM step
    solo_g, sgs = _fresh(probs, "sparse"), _fresh(probs, "sparse")
    sparse = _SparseGroup(sgs, E, P, W)
    arms = {"solo_sparse": lambda: [g.lm_step(e, p, w, 1e-4)[0] for g, e, p, w in zip(solo_g, E, P, W)],
            "sparse_group": lambda: [c[0] for c in sparse.step(list(range(G)), [1e-4] * G)]}
    if dense_on:
        dense = _DenseGroup(_fresh(probs, None), E, P, W)
        arms["dense_group"] = lambda: [c[0] for c in dense.step(list(range(G)), [1e-4] * G)]
    r = alternate(arms, reps)
    rec["step_ms"] = {k: v[1] for k, v in r.items()}
    rec["step_equal"] = all(torch.equal(a, b) for a, b in zip(r["solo_sparse"][0], r["sparse_group"][0]))
    if dense_on:
        rec["step_dense_max_abs_diff"] = _max_diff(r["dense_group"][0], r["sparse_group"][0])
        del dense
    del sparse, solo_g, sgs
    torch.cuda.empty_cache()

    # whole optimisations, with the plateau rule and with a fixed 20 iterations
    for name, kw in (("optimize", {}), ("optimize_fixed20", {"patience": 10 ** 6})):
        box = {}

        def solo():
            gs = _fresh(probs, "sparse")
            box["solo_sparse"] = ([g.optimize(e, p, w, **kw) for g, e, p, w in zip(gs, E, P, W)], [g.nodes for g in gs])

        def group(route, key):
            gs = _fresh(probs, route)
            box[key] = (PoseGraphOpt.optimize_group(gs, E, P, W, **kw), [g.nodes for g in gs])

        arms = {"solo_sparse": solo, "sparse_group": lambda: group("sparse", "sparse_group")}
        if dense_on:
            arms["dense_group"] = lambda: group(None, "dense_group")
        r = alternate(arms, reps)
        rec[name + "_ms"] = {k: v[1] for k, v in r.items()}
        rec[name + "_iterations"] = {"solo_total": sum(len(h) for h in box["solo_sparse"][0]),
                                     "group": max(len(h) for h in box["sparse_group"][0])}
        rec[name + "_equal"] = (box["solo_sparse"][0] == box["sparse_group"][0] and
                                all(torch.equal(a, b) for a, b in zip(box["solo_sparse"][1], box["sparse_group"][1])))
        if dense_on:
            rec[name + "_dense_max_abs_diff"] = _max_diff(box["dense_group"][1], box["sparse_group"][1])
        box.clear()
        torch.cuda.empty_cache()
    for k in ("step_ms", "optimize_ms", "optimize_fixed20_ms"):
        rec[k]["solo_over_sparse_group"] = round(rec[k]["solo_sparse"] / rec[k]["sparse_group"], 3)
        if dense_on:
            rec[k]["dense_group_over_sparse_group"] = round(rec[k]["dense_group"] / rec[k]["sparse_group"], 3)
    return rec


def live_case(S, views, reps):
    from oracle import slam_oracle as so
    from test_sessions_gpu import _replay_sessions
    from test_slam_gpu import _value
    streams = [so.make_stream(seed=100 + k, n_views=views) for k in range(S)]
    ses = _replay_sessions(streams, pgo_every=10 ** 6, verbose=True, max_view_num=views + 10)
    ses.step({k: [_value(so.stream_images(s), i, s) for i in range(views)] for k, s in enumerate(streams)})
    saved = [(s._graph.pose[:s.num_nodes].clone(), set(s.loop_related_views)) for s in ses.sessions]

    def run(route, together):
        for s, (pose, lrv) in zip(ses.sessions, saved):
            s._graph.pose[:s.num_nodes] = pose
            s.loop_related_views = set(lrv)
            s.pgo_route = route
        torch.cuda.synchronize()
        t = time.perf_counter()
        if together:
            ses.optimize(range(S))
        else:
            for s in ses.sessions:
                s.pose_graph_optimize()
        torch.cuda.synchronize()
        return [s._graph.pose[:s.num_nodes].clone() for s in ses.sessions], (time.perf_counter() - t) * 1e3

    arms = {"dense_together": (None, True), "sparse_together": ("sparse", True), "sparse_per_session": ("sparse", False)}
    ms = {k: [] for k in arms}
    out = {}
    with contextlib.redirect_stdout(io.StringIO()):  # the PGO messages
        for r in range(reps + 1):
            for k, (route, together) in arms.items():
                out[k], t = run(route, together)
                if r:
                    ms[k].append(t)
    rec = {"live_sessions": S, "views": views, "nodes": [s.num_nodes for s in ses.sessions],
           "ms": {k: round(statistics.median(v), 3) for k, v in ms.items()},
           "sparse_equal": all(torch.equal(x, y) for x, y in zip(out["sparse_together"], out["sparse_per_session"])),
           "dense_max_abs_diff": _max_diff(out["dense_together"], out["sparse_together"])}
    rec["ms"]["dense_over_sparse"] = round(rec["ms"]["dense_together"] / rec["ms"]["sparse_together"], 3)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="500,1000,2000")
    ap.add_argument("--groups", default="1,2,4,8,16")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dense-max", type=int, default=1000, help="largest size the dense-group arm runs at")
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
            print(json.dumps(group_case(size, probs[size][:G], a.reps, a.dense_max)), flush=True)
            torch.cuda.empty_cache()
    if a.live_views:
        print(json.dumps(live_case(8, a.live_views, a.reps)), flush=True)


if __name__ == "__main__":
    main()
