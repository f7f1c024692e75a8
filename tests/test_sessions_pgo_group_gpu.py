"""GPU: grouped keyframe insertion (sta_graph_add_keyframes), background group runs (PoseGraphOpt.start_group) and
SLAMSessions' background PGOs (optimize(ks, background=True), due PGOs of one step call started as one run).

None of them adds numerics: every table, node pose and loss history is compared bit for bit with the per-keyframe,
synchronous or solo path it groups.  Background runs are slowed with the _Events stand-in of
test_pgo_background_gpu.py, so that they overlap later keyframes."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import slam_oracle as so
from test_pgo_background_gpu import _assert_identical, _Events, _full
from test_pose_graph_group_gpu import SPECS, _problem, _t
from test_pose_graph import make_graph
from test_sessions_gpu import _plan, _replay_sessions, _streams
from test_slam_batch_gpu import _files
from test_slam_gpu import _value
from test_slam_graph_fp64_gpu import _batch, _graph

pytestmark = pytest.mark.gpu

TABLES = ("pose", "depth", "conf", "intri", "cmean", "node_to_view", "node_to_connected_view", "best_node", "best_mean",
          "edges", "meas", "weight")


def _L():
    from vista_slam_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------------ sta_graph_add_keyframes
def _rot(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


class _Seq:
    """A graph's keyframes with OnlineSLAM's host bookkeeping: per keyframe (view, js, first_j, node0, edge0, batch,
    keep)."""

    def __init__(self, H, W, seed):
        self.H, self.W, self.seed = H, W, seed
        self.v2n, self.nodes, self.edges, self.kfs = {}, 0, 0, []
        self.rng = np.random.default_rng(seed)

    def add(self, view, js, bad_rotation=False):
        K = len(js) + 1  # one candidate row more than kept: cand is not the identity map
        poses = np.tile(np.eye(4, dtype=np.float32), (K, 1, 1))
        for r in range(K):
            poses[r, :3, :3] = _rot(self.rng)
            poses[r, :3, 3] = self.rng.normal(size=3)
        if bad_rotation:
            poses[1, :3, :3] *= 1.01
        keep = list(range(1, K))
        batch, keep = _batch(poses, self.H, self.W, self.seed * 1000 + len(self.kfs), keep=keep)
        v2n = {v: list(self.v2n.get(v, [])) for v in set(js) | {view}}
        first_j, n_scale = [], len(js) - 1
        for k, j in enumerate(js):
            v2n[view].append(self.nodes + 2 * k)
            first_j.append(v2n[j][0] if v2n[j] else -1)
            n_scale += first_j[-1] >= 0
            v2n[j].append(self.nodes + 2 * k + 1)
        self.v2n.update(v2n)
        self.kfs.append((view, list(js), first_j, self.nodes, self.edges, batch, keep))
        self.nodes += 2 * len(js)
        self.edges += n_scale + len(js)


def _entry(g, kf):
    L = _L()
    view, js, first_j, node0, edge0, batch, keep = kf
    n = len(js)
    arrays = ((ctypes.c_int64 * n)(*js), (ctypes.c_int * n)(*keep), (ctypes.c_int * n)(*first_j))
    e = L.StaGraphKeyframe(g.h, view, n, node0, edge0, g.H, g.W, *arrays,
                           *[batch[k].data_ptr() for k in ("pose", "pose_conf", "conf", "depths", "intri", "conf_mean")])
    return e, arrays


def _per_keyframe(g, kf):
    L = _L()
    e, arrays = _entry(g, kf)
    L.check(L.lib().sta_graph_add_keyframe(g.h, e.view, e.n, *arrays, e.node0, e.edge0, e.H, e.W, e.pose, e.pose_conf,
                                           e.confs, e.depths, e.intri, e.conf_mean, L.cur_stream()),
            "sta_graph_add_keyframe")


def _grouped(pairs, scratch_pad=0):
    """sta_graph_add_keyframes over [(graph, keyframe), ...]; returns its status."""
    L = _L()
    ents = [_entry(g, kf) for g, kf in pairs]
    tab = (L.StaGraphKeyframe * len(ents))(*[e for e, _ in ents])
    need = int(L.lib().sta_graph_add_keyframes_scratch_bytes(tab, len(ents)))
    assert need > 0, L.lib().sta_last_error()
    scratch = torch.empty((need + scratch_pad + 7) // 8, dtype=torch.float64, device="cuda")
    return L.lib().sta_graph_add_keyframes(tab, len(ents), L.ptr(scratch), need + scratch_pad, L.cur_stream())


def _sequences(H, W):
    # graph a: 18 consecutive keyframes of up to 3 neighbours, loop edges back to views 0 and 2, a keyframe whose loop
    # views have no node (first_j = -1), one of n = 1 and one of n = STA_GRAPH_MAX_KEYFRAME_EDGES
    a = _Seq(H, W, 1)
    for i in range(1, 17):
        js = list(range(max(0, i - 3), i)) + ([0] if i in (9, 13) else []) + ([2] if i == 15 else [])
        a.add(i, js)
    a.add(40, [20, 21, 3])                       # views 20 and 21 have no node: first_j = -1
    a.add(41, [40])                              # n = 1
    a.add(60, list(range(0, 17)) + list(range(22, 37)))  # n = 32: 17 edges with a first node, 15 without
    # graph b: a short chain; graph c: a rotation that is not orthonormal in its second keyframe
    b = _Seq(H, W, 2)
    for i in range(1, 13):
        b.add(i, list(range(max(0, i - 2), i)))
    c = _Seq(H, W, 3)
    c.add(1, [0])
    c.add(2, [0, 1], bad_rotation=True)
    c.add(3, [1, 2])
    return a, b, c


def _interleave(seqs):
    out, at = [], [0] * len(seqs)
    while any(t < len(s.kfs) for t, s in zip(at, seqs)):
        for k, s in enumerate(seqs):
            for _ in range(1 + k % 2):  # uneven interleaving
                if at[k] < len(s.kfs):
                    out.append((k, s.kfs[at[k]]))
                    at[k] += 1
    return out


def _snap(g):
    torch.cuda.synchronize()
    return {k: getattr(g, k).cpu().numpy().copy() for k in TABLES}


def _same(x, y):
    for k in TABLES:
        assert x[k].tobytes() == y[k].tobytes(), k


def _twin(*caps):
    """A graph whose map store (which sta_graph_create leaves as the allocation held it) is filled with a sentinel,
    so that twin graphs compare bit for bit everywhere, rows no keyframe wrote included."""
    g = _graph(*caps)
    for t in (g.depth, g.conf, g.intri):
        t.fill_(-7.0)
    return g


def test_add_keyframes_equals_per_keyframe():
    H, W = 24, 40
    seqs = _sequences(H, W)
    caps = [(2 * s.nodes + 8, s.edges + 8, 64) for s in seqs]
    per = [_twin(n, e, v, H, W) for n, e, v in caps]
    grp = [_twin(n, e, v, H, W) for n, e, v in caps]
    for s, g in zip(seqs, per):
        for kf in s.kfs:
            _per_keyframe(g, kf)
    order = _interleave(seqs)
    M = _L().GRAPH_MAX_GROUP_KEYFRAMES
    assert len(seqs[0].kfs) >= 16 and len(order) > M
    # three graphs interleaved, in calls of at most STA_GRAPH_MAX_GROUP_KEYFRAMES
    for c0 in range(0, len(order), M):
        assert _grouped([(grp[k], kf) for k, kf in order[c0:c0 + M]]) == 0, _L().lib().sta_last_error()
    for s, g1, g2 in zip(seqs, per, grp):
        t1, t2 = _snap(g1), _snap(g2)
        _same(t1, t2)
        assert (t2["node_to_view"][:s.nodes] >= 0).all() and (t2["edges"][:s.edges] >= 0).all()
    assert [g.flags() for g in per] == [g.flags() for g in grp] == [0, 0, _L().GRAPH_FLAG_NOT_SO3]
    # one graph, all of its 19 keyframes in one call: scale edges reach nodes inserted earlier in the same launch
    a = seqs[0]
    one = _twin(*caps[0], H, W)
    assert _grouped([(one, kf) for kf in a.kfs]) == 0
    _same(_snap(one), _snap(per[0]))


def test_add_keyframes_refusals():
    L = _L()
    lib = L.lib()
    H, W = 24, 40
    a, b, _ = _sequences(H, W)
    ga, gb = _graph(2 * a.nodes, a.edges + 4, 64, H, W), _graph(2 * b.nodes, b.edges, 64, H, W)
    assert _grouped([(ga, kf) for kf in a.kfs[:4]] + [(gb, kf) for kf in b.kfs[:3]]) == 0
    before = (_snap(ga), _snap(gb))
    nxt_a, nxt_b = a.kfs[4:6], b.kfs[3:5]

    def refused(pairs, what, scratch="auto"):
        ents = [_entry(g, kf) for g, kf in pairs]
        for e, kfp in zip(ents, [kf for _, kf in pairs]):
            for name, v in what.get(id(kfp), {}).items():
                setattr(e[0], name, v)
        tab = (L.StaGraphKeyframe * max(1, len(ents)))(*[e for e, _ in ents])
        buf = torch.empty(1 << 16, dtype=torch.float64, device="cuda")
        if scratch == "auto":
            rc = lib.sta_graph_add_keyframes(tab, len(ents), L.ptr(buf), buf.numel() * 8, L.cur_stream())
        else:
            rc = lib.sta_graph_add_keyframes(tab, len(ents), *scratch(buf), L.cur_stream())
        assert rc != 0
        if scratch == "auto":
            assert lib.sta_graph_add_keyframes_scratch_bytes(tab, len(ents)) == 0
        return lib.sta_last_error()

    good = [(ga, nxt_a[0]), (gb, nxt_b[0]), (ga, nxt_a[1]), (gb, nxt_b[1])]
    k0 = id(nxt_a[1])  # the bad keyframe is the third of the call: the first two must not go in either
    host = _batch(np.tile(np.eye(4, dtype=np.float32), (4, 1, 1)), H, W, 5)[0]
    cases = [
        ({"graph": None}, b"null"), ({"n": 0}, b"kept edges"), ({"n": 33}, b"kept edges"), ({"H": H + 1}, b"map size"),
        ({"pose": host["pose"].cpu().data_ptr()}, b"device memory"), ({"conf_mean": None}, b"null device input"),
        ({"js": None}, b"null"), ({"view": 64}, b"view index"), ({"view": 0}, b"earlier view"),
        ({"node0": nxt_a[1][3] + 2}, b"continue"), ({"edge0": nxt_a[1][4] - 1}, b"continue"),
        ({"node0": 2 * a.nodes - 1}, b"capacity"),
    ]
    for change, msg in cases:
        assert msg in refused(good, {k0: change}), change
    # per-edge fields of the keyframe: j not earlier, a negative candidate, a first node not yet in the graph
    for field, k, v, msg in (("js", 0, 10 ** 6, b"earlier view"), ("cand", 1, -1, b"candidate"),
                             ("first_j", 0, 10 ** 6, b"first node"), ("first_j", 0, -2, b"first node")):
        ents = [_entry(g, kf) for g, kf in good]
        getattr(ents[2][0], field)[k] = v
        tab = (L.StaGraphKeyframe * 4)(*[e for e, _ in ents])
        buf = torch.empty(1 << 16, dtype=torch.float64, device="cuda")
        assert lib.sta_graph_add_keyframes(tab, 4, L.ptr(buf), buf.numel() * 8, L.cur_stream()) != 0
        assert msg in lib.sta_last_error(), field
    # count, table and scratch
    tab = (L.StaGraphKeyframe * 33)(*([_entry(ga, nxt_a[0])[0]] * 33))
    buf = torch.empty(1 << 16, dtype=torch.float64, device="cuda")
    for cnt in (0, -1, 33):
        assert lib.sta_graph_add_keyframes(tab, cnt, L.ptr(buf), buf.numel() * 8, L.cur_stream()) != 0
        assert lib.sta_graph_add_keyframes_scratch_bytes(tab, cnt) == 0
    assert lib.sta_graph_add_keyframes(None, 1, L.ptr(buf), buf.numel() * 8, L.cur_stream()) != 0
    need = lib.sta_graph_add_keyframes_scratch_bytes((L.StaGraphKeyframe * 4)(*[_entry(g, kf)[0] for g, kf in good]), 4)
    assert need > 0
    assert b"null scratch" in refused(good, {}, scratch=lambda buf: (None, need))
    assert b"smaller" in refused(good, {}, scratch=lambda buf: (L.ptr(buf), need - 1))
    after = (_snap(ga), _snap(gb))
    _same(before[0], after[0])
    _same(before[1], after[1])
    assert ga.flags() == gb.flags() == 0
    # and the good call still goes in
    assert _grouped(good) == 0


# ------------------------------------------------------------------------------------------------ start_group
@pytest.fixture(scope="module")
def pg_problems():
    ps = [_problem(s) for s in SPECS[:5]]
    from vista_slam_b200 import _lib
    n = _lib.PG_DENSE_MAX_OPT + 40
    _, init, edges, meas, weights = make_graph(np.random.default_rng(21), n_nodes=n + 1, n_loops=60, noise=0.01,
                                               meas_noise=0.001)
    ps.append((_t(init, torch.float32), torch.arange(1, n + 1), _t(edges), _t(meas, torch.float32),
               _t(weights, torch.float32)))
    return ps


def _graphs(ps, routes):
    from vista_slam_b200.pose_graph import PoseGraphOpt
    return [PoseGraphOpt(p[0], p[1], route=r) for p, r in zip(ps, routes)]


@pytest.mark.parametrize("routes", ["dense", "sparse", "mixed"])
def test_start_group_equals_optimize_group(pg_problems, routes, monkeypatch):
    from vista_slam_b200.pose_graph import PoseGraphOpt
    if routes == "mixed":
        ps, rs = pg_problems, [None, "sparse", None, "sparse", None, None]  # the last one is past the dense limit
    else:
        ps, rs = pg_problems[:5], [routes] * 5
    args = lambda ps: ([p[2] for p in ps], [p[3] for p in ps], [p[4] for p in ps])
    ref = _graphs(ps, rs)
    want = PoseGraphOpt.optimize_group(ref, *args(ps))
    solo = []
    for p, r in zip(ps, rs):
        g = _graphs([p], [r])[0]
        solo.append((g.optimize(p[2], p[3], p[4]), g.get_nodes()))
    assert len({len(h) for h in want}) > 1  # graphs leave the group at different iterations
    _Events(monkeypatch, every=3)
    gs = _graphs(ps, rs)
    run = PoseGraphOpt.start_group(gs, *args(ps))
    polls, seen_done = 0, set()
    while not run.poll():
        polls += 1
        seen_done |= {k for k in range(len(gs)) if run.graph_done(k)}
    assert polls > len(max(want, key=len))  # the stand-in made polls answer "not yet"
    assert run.done and run.losses == want and len(seen_done) > 0
    for k, (g, r) in enumerate(zip(gs, ref)):
        assert run.graph_losses(k) == want[k] == solo[k][0] and run.graph_done(k)
        assert torch.equal(g.get_nodes(), r.get_nodes()) and torch.equal(g.get_nodes(), solo[k][1])
    # start(): a group of one with start()'s surface
    g = _graphs(ps[:1], rs[:1])[0]
    one = g.start(ps[0][2], ps[0][3], ps[0][4])
    assert one.wait() == want[0] == one.losses and one.done and one.stream is not None
    assert torch.equal(g.get_nodes(), ref[0].get_nodes())


def test_start_group_one_pinned_copy_and_launch_per_iteration(pg_problems, monkeypatch):
    import vista_slam_b200.pose_graph as P
    ps = pg_problems[:4]
    launches, orig = [], P._Group.launch

    def launch(self, active, dampings):
        launches.append(list(active))
        return orig(self, active, dampings)

    monkeypatch.setattr(P._Group, "launch", launch)
    reads = []
    monkeypatch.setattr(P, "_read_info", lambda t: reads.append(1) or t.cpu())
    gs = _graphs(ps, [None] * 4)
    run = P.PoseGraphOpt.start_group(gs, [p[2] for p in ps], [p[3] for p in ps], [p[4] for p in ps])
    losses = run.wait()
    assert len(launches) == max(len(h) for h in losses) and not reads
    assert [len(a) for a in launches] == [sum(len(h) > t for h in losses) for t in range(len(launches))]


# ------------------------------------------------------------------------------------------------ sessions
def _stepped(streams, **kw):
    ses = _replay_sessions(streams, pgo_every=1000, **kw)
    ses.step({k: [_value(so.stream_images(s), i, s) for i in range(s["n_views"])] for k, s in enumerate(streams)})
    return ses


def _three():
    return [so.make_stream(seed=3, n_views=20), so.make_stream(seed=8, n_views=14), so.make_stream(seed=21, n_views=1)]


def test_optimize_background_equals_synchronous(tmp_path, monkeypatch, capsys):
    import vista_slam_b200.pose_graph as P
    streams = _three()
    sync, bg = _stepped(streams), _stepped(streams)
    capsys.readouterr()
    sync.optimize([0, 1, 2])
    want_msgs = capsys.readouterr().out.splitlines()
    ev = _Events(monkeypatch)
    ev.hold = 10 ** 9
    bg.optimize([0, 1, 2], background=True)
    assert [s.pgo_pending for s in bg.sessions] == [True, True, False]  # session 2 has no edges: messages only
    assert bg[0]._pgo_run[0].stream is bg[1]._pgo_run[0].stream  # one shared run
    assert bg[0].loop_related_views == set()
    shown = bg[0].get_view(3).pose
    counts = {"read_info": 0, "synchronize": 0, "event_sync": 0}

    def counter(key, orig):
        def f(*a, **kw):
            counts[key] += 1
            return orig(*a, **kw)
        return f

    monkeypatch.setattr(P, "_read_info", counter("read_info", P._read_info))
    monkeypatch.setattr(torch.cuda, "synchronize", counter("synchronize", torch.cuda.synchronize))
    monkeypatch.setattr(torch.cuda.Event, "synchronize", counter("event_sync", torch.cuda.Event.synchronize))
    for s in bg.sessions:
        s._pgo_poll()
        assert torch.equal(bg[0].get_view(3).pose, shown)  # the poses from before the run
    assert counts == dict.fromkeys(counts, 0) and bg[0].pgo_pending
    bg[1].wait_pgo()  # waiting through one session finishes the shared run; the other folds at its next poll
    assert not bg[1].pgo_pending and bg[0].pgo_pending and counts["event_sync"] > 0
    bg[0]._pgo_poll()
    assert not bg[0].pgo_pending
    assert sorted(capsys.readouterr().out.splitlines()) == sorted(want_msgs)
    for k in range(3):
        _assert_identical(_full(bg[k]), _full(sync[k]))
        if k == 2:
            continue  # no node to export
        bg[k].save_data_all(str(tmp_path / "bg" / str(k)))
        sync[k].save_data_all(str(tmp_path / "sync" / str(k)))
        assert _files(tmp_path / "bg" / str(k)) == _files(tmp_path / "sync" / str(k))
    assert not torch.equal(bg[0].get_view(3).pose, shown)


def test_optimize_background_lifecycle(tmp_path, monkeypatch):
    streams = _three()[:2]
    ev = _Events(monkeypatch)
    # save_data_all, a second optimize and reset while pending
    sync, bg = _stepped(streams), _stepped(streams)
    ev.hold = 10 ** 9
    bg.optimize([0, 1], background=True)
    bg[0].save_data_all(str(tmp_path / "bg"))  # folds session 0 (waits for the shared run)
    sync.optimize([0, 1])
    sync[0].save_data_all(str(tmp_path / "sync"))
    assert _files(tmp_path / "bg") == _files(tmp_path / "sync")
    ev.hold = 10 ** 9
    assert bg[1].pgo_pending
    bg.optimize([1, 0])  # folds session 1's pending PGO first, then optimises now
    sync.optimize([1, 0])
    assert not any(s.pgo_pending for s in bg.sessions)
    for k in range(2):
        _assert_identical(_full(bg[k]), _full(sync[k]))
    ev.hold = 10 ** 9
    bg.optimize([0, 1], background=True)
    bg[0].reset()  # discarded, once its queued work is done with the tables
    assert not bg[0].pgo_pending and bg[1].pgo_pending
    bg[1].wait_pgo()
    sync.optimize([0, 1])
    _assert_identical(_full(bg[1]), _full(sync[1]))


def _sessions_run(shape, background, folder, pgo_every=4, per_call=None):
    streams = _streams()
    images = [so.stream_images(s) for s in streams]
    lengths = [s["n_views"] for s in streams]
    ses = _replay_sessions(streams, pgo_every=pgo_every)
    for s in ses.sessions:
        s.pgo_background = background
    at, flags = [0, 0, 0], {k: [] for k in range(3)}
    for call in _plan(shape, lengths):
        values = {k: [_value(images[k], i, streams[k]) for i in range(at[k], at[k] + m)] for k, m in call.items()}
        force = {k for k, m in call.items() if m and at[k] + m == lengths[k]}
        before = len(per_call[1]) if per_call else 0
        out = ses.step(values, force_pgo=force, log_intermediate_results=True,
                       output_folders={k: os.path.join(folder, str(k)) for k in range(3)})
        if per_call:
            per_call[0].append(len(per_call[1]) - before)
        for k in out:
            flags[k] += out[k]
        at = [a + call.get(k, 0) for k, a in enumerate(at)]
    for s in ses.sessions:
        s.wait_pgo()
    return ses, flags


@pytest.mark.parametrize("shape,pgo_every", [("ones", 4), ("uneven", 4), ("uneven", 2)])
def test_step_groups_background_pgos_per_call(shape, pgo_every, tmp_path, monkeypatch):
    import vista_slam_b200.pose_graph as P
    sync, flags_sync = _sessions_run(shape, False, str(tmp_path / "sync"), pgo_every)
    starts, orig = [], P.PoseGraphOpt.start_group
    runs, rinit = [], P.PoseGraphRun.__init__

    def start_group(*a, **kw):
        starts.append(len(a[0]))
        return orig(*a, **kw)

    def init(self, graphs, *a, **kw):
        runs.append(len(list(graphs)))
        return rinit(self, graphs, *a, **kw)

    monkeypatch.setattr(P.PoseGraphOpt, "start_group", staticmethod(start_group))
    monkeypatch.setattr(P.PoseGraphRun, "__init__", init)
    _Events(monkeypatch, every=3)
    per_call = ([], starts)
    bg, flags_bg = _sessions_run(shape, True, str(tmp_path / "bg"), pgo_every, per_call)
    assert flags_bg == flags_sync and all(any(f) for f in flags_sync.values())
    # every background PGO went through a group run, and some of them shared one
    assert runs == starts and sum(starts) == sum(sum(f) for f in flags_sync.values()) and max(starts) > 1
    if shape == "ones":
        assert max(per_call[0]) == 1  # one group run per call in which sessions fall due
    if pgo_every == 2:
        assert max(per_call[0]) > 1  # a session fell due twice in one call: its second PGO started the first group
    for k in range(3):
        _assert_identical(_full(bg[k]), _full(sync[k]))
        assert _files(tmp_path / "bg" / str(k)) == _files(tmp_path / "sync" / str(k))


def _counted(monkeypatch):
    L = _L().lib()
    counts = {"one": 0, "group": [], "read": 0}
    one, grp = L.sta_graph_add_keyframe, L.sta_graph_add_keyframes

    def f_one(*a):
        counts["one"] += 1
        return one(*a)

    def f_grp(tab, n, *a):
        counts["group"].append(n)
        return grp(tab, n, *a)

    monkeypatch.setattr(L, "sta_graph_add_keyframe", f_one)
    monkeypatch.setattr(L, "sta_graph_add_keyframes", f_grp)
    return counts


def _added(monkeypatch):
    """Views whose keyframe queued an insertion, per session object."""
    import vista_slam_b200.slam as S
    seen, orig = [], S.OnlineSLAM._add_keyframe

    def add(self, i, *a):
        seen.append((id(self), i))
        return orig(self, i, *a)

    monkeypatch.setattr(S.OnlineSLAM, "_add_keyframe", add)
    return seen


def test_insertion_calls_per_edge_chunk(monkeypatch):
    import vista_slam_b200.pose_graph as P
    from test_slam_batch_gpu import _replay_slam
    from vista_slam_b200.keyframe import KeyframeFrontend
    stream = so.make_stream(n_views=30)
    images = so.stream_images(stream)
    counts, added = _counted(monkeypatch), _added(monkeypatch)
    reads = []
    monkeypatch.setattr(P, "_read_info", lambda t: reads.append(1) or t.cpu())
    slam, ref = _replay_slam(stream, pgo_every=1000), _replay_slam(stream, pgo_every=1000)
    vs = [_value(images, i, stream) for i in range(stream["n_views"])]
    slam.step_many(vs[:20])
    # one call per edge chunk with a kept edge: the chunks step_many ran
    loops = stream["loops"]
    items = [(i, list(range(max(0, i - slam.neighbor_edge_num), i)) + [j for j, _ in loops[i][:slam.loop_edge_num]])
             for i in range(20)]
    views = {i for _, i in added}
    chunks = [c for c in KeyframeFrontend.edge_chunks(items) if any(items[t][0] in views for t in c)]
    assert counts["one"] == 0 and len(counts["group"]) == len(chunks) > 1 and max(counts["group"]) > 1
    assert counts["group"] == [sum(items[t][0] in views for t in c) for c in chunks]
    # step: a group of one per keyframe with kept edges
    counts["group"].clear()
    added.clear()
    for v in vs[20:]:
        slam.step(v)
    assert counts["one"] == 0 and counts["group"] == [1] * len(added) and len(added) > 0
    for v in vs:
        ref.step(v)
    _assert_identical(_full(slam), _full(ref))
    # sessions: one call per edge chunk of the call, spanning sessions
    counts["group"].clear()
    added.clear()
    streams = _streams()
    ses = _replay_sessions(streams, pgo_every=1000)
    ses.step({k: [_value(so.stream_images(s), i, s) for i in range(s["n_views"])] for k, s in enumerate(streams)})
    assert counts["one"] == 0 and len(counts["group"]) > 1 and max(counts["group"]) > 1
    assert sum(counts["group"]) == len(added)
    assert not reads


def test_insertion_flushes_before_pgo_and_capacity(monkeypatch):
    from test_slam_batch_gpu import _replay_slam
    stream = so.make_stream()
    images = so.stream_images(stream)
    vs = [_value(images, i, stream) for i in range(stream["n_views"])]
    counts = _counted(monkeypatch)
    a, b = _replay_slam(stream, pgo_every=5), _replay_slam(stream, pgo_every=5)
    a.step_many(vs)
    for v in vs:
        b.step(v)
    _assert_identical(_full(a), _full(b))
    assert counts["one"] == 0
    # capacity: the IndexError leaves the tables as step leaves them
    c, d = _replay_slam(stream, max_view_num=2), _replay_slam(stream, max_view_num=2)
    with pytest.raises(IndexError):
        c.step_many(vs)
    with pytest.raises(IndexError):
        for v in vs:
            d.step(v)
    _assert_identical(_full(c), _full(d))


def test_real_frontend_background_group_equals_synchronous(cuda_model, monkeypatch):
    from test_sessions_gpu import _frames, _real_sessions
    lengths = [9, 6, 11]
    frames = [_frames(n, 31 + k) for k, n in enumerate(lengths)]
    _Events(monkeypatch, every=3)
    out = []
    for background in (False, True):
        ses = _real_sessions(cuda_model, 3, {}, pgo_every=4)
        for s in ses.sessions:
            s.pgo_background = background
        flags = ses.step({k: st[:5] for k, st in enumerate(frames)})
        flags2 = ses.step({k: st[5:] for k, st in enumerate(frames)})
        ses.optimize(range(3), background=background)
        for s in ses.sessions:
            s.wait_pgo()
        out.append((ses, flags, flags2))
    (a, fa, ga), (b, fb, gb) = out
    assert fa == fb and ga == gb and any(any(f) for f in fa.values())
    for k in range(3):
        _assert_identical(_full(a[k]), _full(b[k]))
