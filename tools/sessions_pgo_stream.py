"""PGO in a live SLAMSessions server on one H100: synchronous optimize, per-session background PGOs grouped per call,
and optimize(due, background=True); and the cost of graph insertion per keyframe against per edge chunk.

Each of S sessions runs its own seeded 224 x 224 textured stream (tools/sessions_stream.py), random-init weights of the
reference architecture and the golden DBoW3 vocabulary.  Live-shaped: one keyframe per session per call, pgo_every = 50
(run_live.py's setting).  For S in --sessions and both routes (default: dense at these sizes; sparse), one process
alternates whole runs of three arms after a warm-up run of each:

  (a) sync:      pgo_every beyond the stream (the window of pgo_every = 50 kept), and every 50 keyframes
                 sessions.optimize(due) (INTEGRATION.md §5's former recipe: every camera waits while the due graphs
                 optimise);
  (b) per_session: pgo_background = True and pgo_every = 50 in every session: the due PGOs of one step call start as
                 one group run at the end of the call;
  (c) background: as (a) with sessions.optimize(due, background=True).

A call's latency is timed on the host up to a synchronise of the main stream (not the PGO's side stream); a run's total
ends with every session's wait_pgo and a device synchronise.  Every arm's final tables must be equal bit for bit.

Insertion: --chunk keyframes per session per call (SLAMSessions.step, pgo_every beyond the stream), with the
sta_graph_add_keyframes calls counted and their host-to-stream time (CUDA events around each call on the main stream);
"before" drives the same queued keyframes through sta_graph_add_keyframe one keyframe at a time.  Prints the card's name
and power limit, then one JSON line."""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sessions_stream import VOCAB, card, stream  # noqa: E402


def stats(v):
    v = np.sort(np.asarray(v) * 1e3)
    q = lambda p: round(float(v[int(p * (len(v) - 1))]), 2)
    return {"p50_ms": q(0.5), "p90_ms": q(0.9), "p99_ms": q(0.99), "max_ms": round(float(v[-1]), 2), "calls": len(v)}


def tables(ses):
    out = []
    for s in ses.sessions:
        G = s._graph
        N, E = s.num_nodes, s.num_edges
        out.append(b"".join(t.cpu().numpy().tobytes() for t in (G.pose[:N], G.edges[:E], G.meas[:E], G.weight[:E],
                                                                 G.best_node[:s.view_num])))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", default="2,4,8")
    ap.add_argument("--views", type=int, default=200)
    ap.add_argument("--pgo-every", type=int, default=50)
    ap.add_argument("--chunk", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from vista_slam_b200 import _lib
    from vista_slam_b200.sessions import SLAMSessions
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    sizes = [int(s) for s in a.sessions.split(",")]
    n, P, C, Smax = a.views, a.pgo_every, a.chunk, max(sizes)
    print("card:", card(), flush=True)
    torch.manual_seed(0)
    model = copy.deepcopy(STA().eval()).cuda()
    streams = [stream(1 + k, n) for k in range(Smax)]

    def run(arm, S, route, views, lat=None):
        ses = SLAMSessions("unused", VOCAB, S, frontend=model, pgo_every=P if arm == "per_session" else 10 ** 9)
        for s in ses.sessions:
            s.pgo_route = route
            s.pgo_background = arm == "per_session"
            s.pgo_window_size = 2 * P  # the optimised window of pgo_every = P in every arm
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t in range(views):
            c0 = time.perf_counter()
            last = t == views - 1
            ses.step({k: [streams[k][t]] for k in range(S)}, force_pgo=range(S) if last and arm == "per_session" else ())
            if arm != "per_session" and ((t + 1) % P == 0 or last):
                ses.optimize(range(S), background=arm == "background")
            if lat is not None:
                torch.cuda.current_stream().synchronize()
                lat.append(time.perf_counter() - c0)
        for s in ses.sessions:
            s.wait_pgo()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        return dt, tables(ses)

    arms = ["sync", "per_session", "background"]
    res = {"card": card(), "size": "224x224", "views_per_session": n, "pgo_every": P, "rounds": a.rounds, "live": {},
           "insertion": {}}
    for route in (None, "sparse"):
        for S in sizes:  # warm-up
            for arm in arms:
                run(arm, S, route, min(n, P + 5))
        for S in sizes:
            times, lat, ref, equal = {x: [] for x in arms}, {x: [] for x in arms}, None, {}
            for _ in range(a.rounds):
                for arm in arms:
                    dt, tab = run(arm, S, route, n, lat[arm])
                    times[arm].append(round(dt, 3))
                    ref = tab if ref is None else ref
                    equal[arm] = tab == ref
            res["live"]["%s/S=%d" % (route or "dense", S)] = {
                arm: dict(stats(lat[arm]), seconds_all=times[arm], tables_equal=equal[arm]) for arm in arms}
            print(json.dumps({"%s/S=%d" % (route or "dense", S): res["live"]["%s/S=%d" % (route or "dense", S)]}),
                  flush=True)

    # insertion: chunked calls, grouped against one keyframe at a time
    L = _lib.lib()
    grouped = L.sta_graph_add_keyframes

    def per_keyframe(tab, count, scratch, nbytes, stream_):
        for t in range(count):
            e = tab[t]
            rc = L.sta_graph_add_keyframe(e.graph, e.view, e.n, e.js, e.cand, e.first_j, e.node0, e.edge0, e.H, e.W,
                                          e.pose, e.pose_conf, e.confs, e.depths, e.intri, e.conf_mean, stream_)
            if rc:
                return rc
        return 0

    def chunked(S, mode):
        calls, spans = [], []
        fn = grouped if mode == "after" else per_keyframe

        def timed(tab, count, scratch, nbytes, stream_):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            h0 = time.perf_counter()
            e0.record()
            rc = fn(tab, count, scratch, nbytes, stream_)
            e1.record()
            spans.append((time.perf_counter() - h0, e0, e1))
            calls.append(count)
            return rc

        L.sta_graph_add_keyframes = timed
        try:
            ses = SLAMSessions("unused", VOCAB, S, frontend=model, pgo_every=10 ** 9)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for c in range(0, n, C):
                ses.step({k: streams[k][c:c + C] for k in range(S)})
            torch.cuda.synchronize()
            total = time.perf_counter() - t0
        finally:
            L.sta_graph_add_keyframes = grouped
        host = sum(h for h, _, _ in spans)
        dev = sum(e0.elapsed_time(e1) for _, e0, e1 in spans) / 1e3
        launches = 2 * sum(calls) if mode == "before" else 2 * len(calls)
        step_calls = (n + C - 1) // C
        return {"insert_host_ms_per_call": round(1e3 * host / step_calls, 3),
                "insert_stream_ms_per_call": round(1e3 * dev / step_calls, 3),
                "insert_launches_per_call": round(launches / step_calls, 1), "keyframes": sum(calls),
                "total_s": round(total, 3)}, tables(ses)

    for S in sizes:
        chunked(S, "before")
        chunked(S, "after")
        r, ok = {"before": [], "after": []}, True
        for _ in range(a.rounds):
            for mode in ("before", "after"):
                out, tab = chunked(S, mode)
                r[mode].append(out)
                ref = tab if mode == "before" else ref
                ok = ok and (mode == "before" or tab == ref)
        res["insertion"]["S=%d" % S] = {"before": r["before"], "after": r["after"], "tables_equal": ok}
        print(json.dumps({"insertion S=%d" % S: res["insertion"]["S=%d" % S]}), flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
