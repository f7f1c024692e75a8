"""GPU: background pose-graph optimisation (OnlineSLAM.pgo_background, PoseGraphOpt.start, sta_graph_replay_nodes).

A background PGO must leave the graph exactly as the synchronous one: after wait_pgo(), every table, the host
bookkeeping, the step flags, the LM loss histories and every file save_data_all writes are compared bit for bit with a
twin run with pgo_background = False.  To make runs overlap later keyframes on a fast GPU, torch.cuda.Event.query is
made to answer as a slower GPU would (_Events): False for a number of calls, or on all but every n-th call."""
import ctypes
import os

import pytest
import torch

from oracle import slam_oracle as so
from test_sessions_gpu import _frames, _plan, _replay_sessions, _streams
from test_sessions_gpu import _tables as _all_tables
from test_slam_batch_gpu import _LoopsMany, _files, _real_slam, _state
from test_slam_batch_gpu import _replay_slam as _replay
from test_slam_gpu import _value

pytestmark = pytest.mark.gpu


class _Events:
    """torch.cuda.Event.query answering False for the next `hold` calls, then True only on every `every`-th call
    whose event has really completed.  Waiting on an event (Event.synchronize) ends the hold."""

    def __init__(self, monkeypatch, every=1):
        self.hold, self.every, self.n = 0, every, 0
        real_query, real_sync = torch.cuda.Event.query, torch.cuda.Event.synchronize

        def query(ev):
            if self.hold > 0:
                self.hold -= 1
                return False
            self.n += 1
            return real_query(ev) if self.n % self.every == 0 else False

        def synchronize(ev):
            self.hold = 0
            return real_sync(ev)

        monkeypatch.setattr(torch.cuda.Event, "query", query)
        monkeypatch.setattr(torch.cuda.Event, "synchronize", synchronize)


def _record_losses(monkeypatch):
    import vista_slam_b200.pose_graph as P
    made, init = [], P._LMState.__init__

    def rec(self, *a, **kw):
        init(self, *a, **kw)
        made.append(self)

    monkeypatch.setattr(P._LMState, "__init__", rec)
    return made


def _replays(monkeypatch):
    from vista_slam_b200 import _lib
    L = _lib.lib()
    counts, orig = [], L.sta_graph_replay_nodes

    def wrap(g, n, t, s):
        counts.append(n)
        return orig(g, n, t, s)

    monkeypatch.setattr(L, "sta_graph_replay_nodes", wrap)
    return counts


def _full(slam):
    out = _state(slam)
    out.update({"table_" + k: v for k, v in _all_tables(slam).items()})
    return out


def _assert_identical(a, b):
    assert a["host"] == b["host"]
    for k in a:
        if k != "host":
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
            assert a[k].tobytes() == b[k].tobytes(), k


def _drive(slam, stream, driver, folder):
    images = so.stream_images(stream)
    n = stream["n_views"]
    flags, pending = [], 0
    if driver == "step":
        for i in range(n):
            flags.append(slam.step(_value(images, i, stream), force_pgo=(i == n - 1), log_intermediate_results=True,
                                   output_folder=folder))
            pending += slam.pgo_pending
    else:
        for t0 in range(0, n, 4):
            vs = [_value(images, i, stream) for i in range(t0, min(n, t0 + 4))]
            flags += slam.step_many(vs, force_pgo=(t0 + 4 >= n), log_intermediate_results=(t0 % 8 == 0),
                                    output_folder=folder)
            pending += slam.pgo_pending
    return flags, pending


@pytest.mark.parametrize("every", [1, 4])
@pytest.mark.parametrize("driver", ["step", "step_many"])
@pytest.mark.parametrize("route", [None, "sparse"])
def test_background_equals_synchronous(route, driver, every, tmp_path, monkeypatch):
    stream = so.make_stream()
    losses = _record_losses(monkeypatch)
    sync = _replay(stream, pgo_every=3)
    sync.pgo_route = route
    flags_sync, _ = _drive(sync, stream, driver, str(tmp_path / "sync"))
    sync.save_data_all(str(tmp_path / "sync_final"))
    want = [list(s.losses) for s in losses]
    losses.clear()

    _Events(monkeypatch, every)
    replayed = _replays(monkeypatch)
    bg = _replay(stream, pgo_every=3)
    bg.pgo_route, bg.pgo_background = route, True
    flags_bg, pending = _drive(bg, stream, driver, str(tmp_path / "bg"))
    if every > 1:
        assert pending > 0 and sum(replayed) > 0  # runs overlapped later keyframes, whose nodes were replayed
    bg.wait_pgo()
    assert not bg.pgo_pending
    bg.save_data_all(str(tmp_path / "bg_final"))
    assert flags_bg == flags_sync and sum(flags_sync) >= 5
    assert [list(s.losses) for s in losses] == want and len(want) == sum(flags_sync)
    _assert_identical(_full(bg), _full(sync))
    assert _files(tmp_path / "bg") == _files(tmp_path / "sync")
    assert _files(tmp_path / "bg_final") == _files(tmp_path / "sync_final")
    assert set(bg.get_time_dict()) == set(sync.get_time_dict()) and bg.time_dict["pgo"] > 0


class _Pending:
    """A stand-in pending run that never finishes: _add_keyframe records the triples of the nodes it inserts."""

    def poll(self):
        return False


def test_replay_nodes_equals_insertion_after_the_roots():
    from vista_slam_b200 import _lib
    stream = so.make_stream()
    images = so.stream_images(stream)
    n, K = stream["n_views"], 8
    a, b = _replay(stream, pgo_every=1000), _replay(stream, pgo_every=1000)
    for i in range(K):
        a.step(_value(images, i, stream))
        b.step(_value(images, i, stream))
    N0 = a.num_nodes
    # new root poses: every node so far moved and rescaled, quaternions renormalised with w >= 0
    p = a._graph.pose[:N0].clone()
    d = torch.randn(N0, 8, generator=torch.Generator().manual_seed(4)).cuda() * 0.1
    q = p[:, 3:7] + d[:, 3:7]
    q = q / q.norm(dim=1, keepdim=True)
    q = torch.where(q[:, 3:4] < 0, -q, q)
    roots = torch.cat([p[:, :3] + d[:, :3], q, p[:, 7:] * (1 + d[:, 7:].abs())], 1).contiguous()
    a._graph.pose[:N0] = roots  # then a inserts the rest of the keyframes from the new roots
    rec = []
    b._pgo_run = (_Pending(), None, rec)
    for i in range(K, n):
        a.step(_value(images, i, stream))
        b.step(_value(images, i, stream))
    b._pgo_run = None
    G = b._graph
    view, cview = G.node_to_view.cpu().numpy(), G.node_to_connected_view.cpu().numpy()
    assert len(rec) > 0 and all(t[0] >= N0 for t in rec) and any(t[1] < N0 for t in rec)
    assert any(t[1] == t[0] + 1 for t in rec)  # a new view's first node, derived from its j node
    assert any(abs(view[t[0]] - cview[t[0]]) > b.neighbor_edge_num for t in rec)  # loop-closure nodes
    G.pose[:N0] = roots
    assert G.pose[N0:b.num_nodes].cpu().numpy().tobytes() != a._graph.pose[N0:a.num_nodes].cpu().numpy().tobytes()
    flat = (ctypes.c_int * (3 * len(rec)))(*[x for t in rec for x in t])
    L = _lib.lib()
    _lib.check(L.sta_graph_replay_nodes(G.h, len(rec), flat, _lib.cur_stream()), "sta_graph_replay_nodes")
    assert a.num_nodes == b.num_nodes
    assert G.pose[:b.num_nodes].cpu().numpy().tobytes() == a._graph.pose[:a.num_nodes].cpu().numpy().tobytes()
    _assert_identical(_full(a), _full(b))

    # refusals, before any launch: the poses stay as they are
    before = G.pose.clone()
    M, E = G.max_nodes, G.max_edges
    for bad in ([M, 0, 0], [-1, 0, 0], [5, M, 0], [5, -1, 0], [5, 5, 0], [5, 0, E], [5, 0, -1]):
        t = (ctypes.c_int * 6)(4, 0, 0, *bad)
        assert L.sta_graph_replay_nodes(G.h, 2, t, _lib.cur_stream()) != 0, bad
    assert L.sta_graph_replay_nodes(G.h, -1, flat, _lib.cur_stream()) != 0
    assert L.sta_graph_replay_nodes(G.h, 1, None, _lib.cur_stream()) != 0
    assert L.sta_graph_replay_nodes(G.h, 0, None, _lib.cur_stream()) == 0
    assert torch.equal(G.pose, before)


class _QuietLoops(_LoopsMany):
    """The replayed loop detector without its stand-in read-back (a device-wide synchronise)."""

    def detect_loop(self, image, farthest_neighbor):
        c = self.loops[self.calls]
        self.calls += 1
        return list(c)


def test_pending_run_does_not_wait(monkeypatch):
    import vista_slam_b200.pose_graph as P
    stream = so.make_stream()
    images = so.stream_images(stream)
    ev = _Events(monkeypatch)
    bg = _replay(stream, pgo_every=6)
    bg.pgo_background = True
    bg.lc_detector = _QuietLoops(stream["loops"], 5)
    for i in range(5):
        bg.step(_value(images, i, stream))
    ev.hold = 10 ** 9
    assert bg.step(_value(images, 5, stream)) and bg.pgo_pending  # view 6 is due: launched, and held from here on
    side = bg._pgo_run[0].stream
    shown = bg.get_view(3).pose
    counts = {"read_info": 0, "synchronize": 0, "empty_cache": 0, "side_sync": 0, "event_sync": 0}

    def counter(key, orig=None, cond=None):
        def f(*a, **kw):
            if cond is None or cond(*a):
                counts[key] += 1
            return orig(*a, **kw)
        return f

    monkeypatch.setattr(P, "_read_info", counter("read_info", P._read_info))
    monkeypatch.setattr(torch.cuda, "synchronize", counter("synchronize", torch.cuda.synchronize))
    monkeypatch.setattr(torch.cuda, "empty_cache", counter("empty_cache", torch.cuda.empty_cache))
    monkeypatch.setattr(torch.cuda.Stream, "synchronize",
                        counter("side_sync", torch.cuda.Stream.synchronize, lambda s: s.cuda_stream == side.cuda_stream))
    monkeypatch.setattr(torch.cuda.Event, "synchronize", counter("event_sync", torch.cuda.Event.synchronize))
    for i in range(6, 11):
        bg.step(_value(images, i, stream))
        assert bg.pgo_pending
        v = bg.get_view(3)
        assert torch.equal(v.pose, shown)  # the poses from before the run
    assert counts == dict.fromkeys(counts, 0)
    bg.wait_pgo()
    assert not bg.pgo_pending and counts["event_sync"] > 0
    assert not torch.equal(bg.get_view(3).pose, shown)

    sync = _replay(stream, pgo_every=6)
    for i in range(11):
        sync.step(_value(images, i, stream))
    _assert_identical(_full(bg), _full(sync))


def _launched(slam, stream, upto, ev):
    """Step keyframes 0 .. upto - 1, each background PGO held pending until something waits for it."""
    images = so.stream_images(stream)
    ev.hold = 10 ** 9
    for i in range(upto):
        slam.step(_value(images, i, stream))


def test_lifecycle_while_pending(monkeypatch):
    stream = so.make_stream()
    images = so.stream_images(stream)
    ev = _Events(monkeypatch)

    def pair(**kw):
        bg, sync = _replay(stream, **kw), _replay(stream, **kw)
        bg.pgo_background = True
        return bg, sync

    # reset: the pending result is discarded; the next keyframes run as after a synchronous PGO and a reset
    bg, sync = pair(pgo_every=5)
    _launched(bg, stream, 12, ev)
    _launched(sync, stream, 12, ev)
    assert bg.pgo_pending
    bg.reset()
    sync.reset()
    assert not bg.pgo_pending
    for s in (bg, sync):  # the loop detector is not reset: restart the replayed one with the views
        s.lc_detector = _LoopsMany(stream["loops"], 5)
    for i in range(7):
        bg.step(_value(images, i, stream))
        sync.step(_value(images, i, stream))
    bg.wait_pgo()
    _assert_identical(_full(bg), _full(sync))

    # pose_graph_optimize: folds the pending run first, then optimises now
    bg, sync = pair(pgo_every=5)
    _launched(bg, stream, 13, ev)
    _launched(sync, stream, 13, ev)
    assert bg.pgo_pending
    bg.pose_graph_optimize()
    sync.pose_graph_optimize()
    assert not bg.pgo_pending
    _assert_identical(_full(bg), _full(sync))

    # a capacity IndexError while a run is pending
    bg, sync = pair(pgo_every=2, max_view_num=2)
    for s in (bg, sync):
        with pytest.raises(IndexError):
            _launched(s, stream, stream["n_views"], ev)
    assert bg.pgo_pending
    bg.wait_pgo()
    _assert_identical(_full(bg), _full(sync))


def _sessions_run(shape, background, folder):
    streams = _streams()
    images = [so.stream_images(s) for s in streams]
    lengths = [s["n_views"] for s in streams]
    ses = _replay_sessions(streams, pgo_every=4)
    for s in ses.sessions:
        s.pgo_background = background
    at, flags = [0, 0, 0], {k: [] for k in range(3)}
    for call in _plan(shape, lengths):
        values = {k: [_value(images[k], i, streams[k]) for i in range(at[k], at[k] + m)] for k, m in call.items()}
        force = {k for k, m in call.items() if m and at[k] + m == lengths[k]}
        out = ses.step(values, force_pgo=force, log_intermediate_results=True,
                       output_folders={k: os.path.join(folder, str(k)) for k in range(3)})
        for k in out:
            flags[k] += out[k]
        at = [a + call.get(k, 0) for k, a in enumerate(at)]
    ses.optimize([0, 2])  # folds their pending runs first
    for s in ses.sessions:
        s.wait_pgo()
    return ses, flags


@pytest.mark.parametrize("shape", ["ones", "uneven"])
def test_sessions_background_equals_synchronous(shape, tmp_path, monkeypatch):
    _Events(monkeypatch, every=3)
    bg, flags_bg = _sessions_run(shape, True, str(tmp_path / "bg"))
    sync, flags_sync = _sessions_run(shape, False, str(tmp_path / "sync"))
    assert flags_bg == flags_sync and all(any(f) for f in flags_sync.values())
    for k in range(3):
        _assert_identical(_full(bg[k]), _full(sync[k]))
        assert _files(tmp_path / "bg" / str(k)) == _files(tmp_path / "sync" / str(k))


def test_real_frontend_background_equals_synchronous(cuda_model, monkeypatch):
    frames = _frames(12, 9)
    _Events(monkeypatch, every=3)
    runs = []
    for background in (False, True):
        s = _real_slam(cuda_model, 0.75, {})
        s.pgo_background = background
        flags = [s.step(v, force_pgo=(i == len(frames) - 1)) for i, v in enumerate(frames)]
        s.wait_pgo()
        runs.append((s, flags))
    (a, fa), (b, fb) = runs
    assert fa == fb and sum(fa) >= 2 and a.num_edges > 0
    _assert_identical(_full(a), _full(b))
