"""GPU: the dense Sim(3) LM step over a group of graphs (sta_pose_graph_lm_step_group), PoseGraphOpt.optimize_group and
SLAMSessions.optimize.

  * optimize_group leaves every graph bit for bit as its own optimize() does, with the same loss history, for groups of
    1, 3 and 8 planted graphs (oracle/pose_graph_oracle.py algebra) of different sizes, optimised sets and edge counts,
    in any order, and when a block-sparse-route graph shares the call;
  * a one-graph group launch and sta_pose_graph_lm_step give the same output and info bit for bit;
  * one info read-back per group iteration;
  * every refusal of the C entry point and of optimize_group comes before any launch;
  * SLAMSessions.optimize leaves replayed sessions (and sessions on the real frontend) as per-session
    pose_graph_optimize() does: tables, loop_related_views, messages and time_dict keys."""
import random

import numpy as np
import pytest
import torch

from oracle import slam_oracle as so
from test_pose_graph import make_graph  # planted graphs in the algebra of oracle/pose_graph_oracle.py

pytestmark = pytest.mark.gpu


def _t(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t.to(dtype) if dtype is not None else t).cuda()


# (seed, nodes, loops, init noise, measurement noise, optimised set); odd node counts (25, 33) put the next graph's
# scratch carve past an unaligned opt_map end
SPECS = [
    (7, 60, 15, 0.05, 0.0, "all_but_0"),    # converges to the planted answer
    (40, 12, 3, 1.5, 0.02, "all_but_0"),     # rejected steps from the first one on, then the plateau rule stops it
    (6, 40, 10, 0.05, 0.02, "all_but_0"),    # inconsistent measurements: plateaus after a few steps
    (11, 25, 4, 0.1, 0.01, "window"),       # fixed nodes: only the last 10 are optimised, unrelated edges present
    (12, 90, 30, 0.05, 0.01, "all"),        # every node optimised (gauge left free, damping keeps A definite)
    (13, 8, 1, 0.2, 0.0, "all_but_0"),
    (14, 33, 0, 0.1, 0.03, "window"),
    (15, 120, 40, 0.03, 0.005, "all_but_0"),
]


def _problem(spec):
    seed, n, loops, noise, mnoise, which = spec
    gt, init, edges, meas, weights = make_graph(np.random.default_rng(seed), n_nodes=n, n_loops=loops, noise=noise,
                                                meas_noise=mnoise)
    opt = {"all_but_0": list(range(1, n)), "window": list(range(n - 10, n)), "all": list(range(n))}[which]
    return (_t(init, torch.float32), torch.tensor(opt), _t(edges), _t(meas, torch.float32), _t(weights, torch.float32))


@pytest.fixture(scope="module")
def problems():
    return [_problem(s) for s in SPECS]


def _solo(p, **kw):
    from vista_slam_b200.pose_graph import PoseGraphOpt
    nodes, opt, edges, meas, w = p
    g = PoseGraphOpt(nodes, opt)
    return g.optimize(edges, meas, w, **kw), g.get_nodes()


def _group(ps, **kw):
    from vista_slam_b200.pose_graph import PoseGraphOpt
    gs = [PoseGraphOpt(p[0], p[1]) for p in ps]
    losses = PoseGraphOpt.optimize_group(gs, [p[2] for p in ps], [p[3] for p in ps], [p[4] for p in ps], **kw)
    return losses, [g.get_nodes() for g in gs]


def _info_rows(monkeypatch):
    """Every info row read back, in order."""
    import vista_slam_b200.pose_graph as P
    rows, orig = [], P._read_info

    def read(t):
        out = orig(t)
        rows.extend(out.reshape(-1, 4).tolist())
        return out

    monkeypatch.setattr(P, "_read_info", read)
    return rows


def test_group_equals_solo(problems, monkeypatch):
    rows = _info_rows(monkeypatch)
    solo = [_solo(p) for p in problems]
    # the planted graph is recovered, the noisy ones plateau early, and graph 1 had its steps rejected
    assert solo[0][0][-1] < 1e-9 and len(solo[2][0]) < 20
    assert any(r[1] > 1.5 * r[0] for r in rows) and len(solo[1][0]) == 3 and len(set(solo[1][0])) == 1
    assert len({len(h) for h, _ in solo}) > 1  # the graphs leave the group at different iterations
    for members in ([3], [0, 1, 2], list(range(8))):
        losses, nodes = _group([problems[k] for k in members])
        for k, h, x in zip(members, losses, nodes):
            assert h == solo[k][0], (members, k)
            assert torch.equal(x, solo[k][1]), (members, k)
    # a permuted group: the same per-graph results
    order = list(range(8))
    random.Random(3).shuffle(order)
    losses, nodes = _group([problems[k] for k in order])
    for k, h, x in zip(order, losses, nodes):
        assert h == solo[k][0] and torch.equal(x, solo[k][1]), k
    # a fixed number of iterations (no plateau stop): still the solo results
    solo20 = [_solo(p, patience=100) for p in problems[:4]]
    losses, nodes = _group(problems[:4], patience=100)
    assert all(len(h) == 20 for h in losses)
    for (h, x), h2, x2 in zip(solo20, losses, nodes):
        assert h == h2 and torch.equal(x, x2)


def test_group_with_a_sparse_route_graph(problems):
    from vista_slam_b200 import _lib
    n = _lib.PG_DENSE_MAX_OPT + 40
    gt, init, edges, meas, weights = make_graph(np.random.default_rng(21), n_nodes=n + 1, n_loops=60, noise=0.01,
                                                meas_noise=0.001)
    big = (_t(init, torch.float32), torch.arange(1, n + 1), _t(edges), _t(meas, torch.float32), _t(weights, torch.float32))
    ps = [problems[0], big, problems[3]]
    solo = [_solo(p) for p in ps]
    losses, nodes = _group(ps)
    from vista_slam_b200.pose_graph import PoseGraphOpt
    assert PoseGraphOpt(big[0], big[1]).sparse and len(solo[1][0]) > 1
    for (h, x), h2, x2 in zip(solo, losses, nodes):
        assert h == h2 and torch.equal(x, x2)


def _table(entries):
    from vista_slam_b200 import _lib
    tab = (_lib.StaPgGraph * max(1, len(entries)))()
    for k, (nodes, opt, edges, meas, w, out, damping) in enumerate(entries):
        tab[k] = _lib.StaPgGraph(nodes.data_ptr(), edges.data_ptr(), meas.data_ptr(), w.data_ptr(), opt.data_ptr(),
                                 out.data_ptr(), nodes.shape[0], edges.shape[0], opt.shape[0], damping)
    return tab


def test_entry_points_agree(problems):
    from vista_slam_b200 import _lib
    L = _lib.lib()
    for p, damping in ((problems[0], 1e-4), (problems[3], 0.3), (problems[7], 2e-6)):
        nodes, opt, edges, meas, w = p
        opt = opt.cuda()
        Nn, E, No = nodes.shape[0], edges.shape[0], opt.shape[0]
        out1, out2 = torch.full_like(nodes, float("nan")), torch.full_like(nodes, float("nan"))
        info1 = torch.full((4,), float("nan"), dtype=torch.float64, device="cuda")
        info2 = torch.full((1, 4), float("nan"), dtype=torch.float64, device="cuda")
        s1 = torch.empty(int(L.sta_pose_graph_scratch_bytes(Nn, E, No)) // 8 + 1, dtype=torch.float64, device="cuda")
        _lib.check(L.sta_pose_graph_lm_step(_lib.ptr(nodes), Nn, _lib.ptr(edges), _lib.ptr(meas), _lib.ptr(w), E, _lib.ptr(opt),
                                            No, damping, 1e-6, 1e32, _lib.ptr(out1), _lib.ptr(info1), _lib.ptr(s1),
                                            _lib.cur_stream()))
        tab = _table([(nodes, opt, edges, meas, w, out2, damping)])
        need = int(L.sta_pose_graph_group_scratch_bytes(tab, 1))
        assert need >= int(L.sta_pose_graph_scratch_bytes(Nn, E, No))
        s2 = torch.empty(need // 8 + 1, dtype=torch.float64, device="cuda")
        _lib.check(L.sta_pose_graph_lm_step_group(tab, 1, 1e-6, 1e32, _lib.ptr(info2), _lib.ptr(s2), need, _lib.cur_stream()))
        assert torch.equal(out1, out2) and torch.equal(info1, info2[0])
        assert info1[3] == 1.0 and info1[1] < info1[0]


def test_one_read_back_per_group_iteration(problems, monkeypatch):
    import vista_slam_b200.pose_graph as P
    counts = [0]
    orig = P._read_info

    def read(t):
        counts[0] += 1
        return orig(t)

    monkeypatch.setattr(P, "_read_info", read)
    losses, _ = _group(problems)
    assert counts[0] == max(len(h) for h in losses) and len({len(h) for h in losses}) > 1


def test_group_refusals(problems):
    from vista_slam_b200 import _lib
    from vista_slam_b200.pose_graph import PoseGraphOpt
    L = _lib.lib()
    # the C entry point: a status and a message, nothing launched (outputs keep their sentinel)
    base = [problems[0], problems[3]]
    outs = [torch.full_like(p[0], float("nan")) for p in base]
    ents = [(p[0], p[1].cuda(), p[2], p[3], p[4], o, 1e-4) for p, o in zip(base, outs)]
    info = torch.full((_lib.PG_GROUP_MAX + 1, 4), float("nan"), dtype=torch.float64, device="cuda")
    good = _table(ents)
    need = int(L.sta_pose_graph_group_scratch_bytes(good, 2))
    scratch = torch.empty(need // 8 + 1, dtype=torch.float64, device="cuda")
    st = _lib.cur_stream()

    def refused(tab, G, msg, info_p=_lib.ptr(info), scratch_p=_lib.ptr(scratch), nbytes=need):
        assert L.sta_pose_graph_lm_step_group(tab, G, 1e-6, 1e32, info_p, scratch_p, nbytes, st) != 0
        assert msg.encode() in L.sta_last_error(), L.sta_last_error()

    def bad(k, **kw):
        t = _table(ents)
        for f, v in kw.items():
            setattr(t[k], f, v)
        return t

    refused(None, 2, "null graph table")
    refused(good, 2, "null pointer", info_p=None)
    refused(good, 2, "null pointer", scratch_p=None)
    refused(good, 0, "STA_PG_GROUP_MAX")
    refused(good, _lib.PG_GROUP_MAX + 1, "STA_PG_GROUP_MAX")
    for f in ("nodes", "edges", "meas", "weights", "opt_idx", "nodes_out"):
        refused(bad(1, **{f: None}), 2, "null pointer")
    for f in ("num_nodes", "num_edges", "num_opt"):
        refused(bad(0, **{f: 0}), 2, "empty problem")
    refused(bad(1, num_opt=ents[1][0].shape[0] + 1), 2, "empty problem")
    refused(bad(0, num_opt=_lib.PG_DENSE_MAX_OPT + 1, num_nodes=_lib.PG_DENSE_MAX_OPT + 1), 2, "3657 optimised nodes")
    refused(good, 2, "scratch smaller", nbytes=need - 1)
    torch.cuda.synchronize()
    assert all(torch.isnan(o).all() for o in outs) and torch.isnan(info).all()
    assert L.sta_pose_graph_lm_step_group(good, 2, 1e-6, 1e32, _lib.ptr(info), _lib.ptr(scratch), need, st) == 0
    torch.cuda.synchronize()
    assert not any(torch.isnan(o).any() for o in outs) and not torch.isnan(info[:2]).any() and torch.isnan(info[2:]).all()

    # optimize_group: ValueError before any launch, every graph untouched
    gs = [PoseGraphOpt(p[0], p[1]) for p in base]
    before = [g.nodes.clone() for g in gs]
    e, m, w = [p[2] for p in base], [p[3] for p in base], [p[4] for p in base]
    import vista_slam_b200.pose_graph as P
    calls = [0]
    orig = P._DenseGroup.step

    def step(self, *a):
        calls[0] += 1
        return orig(self, *a)

    P._DenseGroup.step = step
    try:
        with pytest.raises(ValueError, match="twice"):
            PoseGraphOpt.optimize_group([gs[0], gs[0]], e, m, w)
        with pytest.raises(ValueError, match="one row per edge"):
            PoseGraphOpt.optimize_group(gs, e, [m[0], m[1][:-1]], w)
        with pytest.raises(ValueError, match="one row per edge"):
            PoseGraphOpt.optimize_group(gs, e, m, [w[0][:-2], w[1]])
        with pytest.raises(ValueError, match="one entry per graph"):
            PoseGraphOpt.optimize_group(gs, e, m, w[:1])
        other = PoseGraphOpt(base[1][0], base[1][1])
        if torch.cuda.device_count() > 1:
            other = PoseGraphOpt(base[1][0].to("cuda:1"), base[1][1])
        else:  # one device here: a host tensor stands for the other device
            other.nodes = other.nodes.cpu()
        with pytest.raises(ValueError, match="one device"):
            PoseGraphOpt.optimize_group([gs[0], other], e, m, w)
    finally:
        P._DenseGroup.step = orig
    assert calls[0] == 0
    assert all(torch.equal(g.nodes, b) for g, b in zip(gs, before))


# ------------------------------------------------------------------------------------------------ sessions
@pytest.fixture
def replay_streams():
    """Three replayed sessions: two of 20 and 14 views, one that holds only its first keyframe."""
    return [so.make_stream(seed=3, n_views=20), so.make_stream(seed=8, n_views=14), so.make_stream(seed=21, n_views=1)]


def _stepped(streams):
    from test_sessions_gpu import _replay_sessions
    from test_slam_gpu import _value
    ses = _replay_sessions(streams, pgo_every=1000)
    ses.step({k: [_value(so.stream_images(s), i, s) for i in range(s["n_views"])] for k, s in enumerate(streams)})
    return ses


def _tables(s):
    G = s._graph
    return {"pose": G.pose[:s.num_nodes].cpu().numpy(), "edges": G.edges[:s.num_edges].cpu().numpy(),
            "meas": G.meas[:s.num_edges].cpu().numpy(), "weight": G.weight[:s.num_edges].cpu().numpy(),
            "best_node": G.best_node[:s.view_num].cpu().numpy(), "node_to_view": G.node_to_view.cpu().numpy()}


def test_sessions_optimize_equals_per_session_pgo(replay_streams, capsys):
    ses, twin = _stepped(replay_streams), _stepped(replay_streams)
    assert [s.num_edges > 0 for s in ses.sessions] == [True, True, False] and ses[2].num_nodes == 0
    assert any(s.loop_related_views for s in ses.sessions)
    assert all(_tables(a)["pose"].tobytes() == _tables(b)["pose"].tobytes() for a, b in zip(ses.sessions, twin.sessions))
    before = [_tables(s)["pose"] for s in ses.sessions]
    capsys.readouterr()
    ses.optimize([0, 1, 2])
    got = capsys.readouterr().out.splitlines()
    for s in twin.sessions:
        s.pose_graph_optimize()
    want = capsys.readouterr().out.splitlines()
    assert sorted(got) == sorted(want) and len(got) == 6
    for a, b, p0 in zip(ses.sessions, twin.sessions, before):
        ta, tb = _tables(a), _tables(b)
        for k in ta:
            np.testing.assert_array_equal(ta[k], tb[k], err_msg=k)
        assert a.loop_related_views == b.loop_related_views == set()
        assert set(a.get_time_dict()) == set(b.get_time_dict())
        assert a.time_dict["pgo"] > 0
    assert not np.array_equal(_tables(ses[0])["pose"], before[0])  # the PGO moved the poses


def test_sessions_optimize_refusals(replay_streams):
    ses = _stepped(replay_streams)
    p0 = _tables(ses[0])["pose"]
    lrv = set(ses[0].loop_related_views)
    for bad in ([0, 3], [1, 1], [-1], ["0"]):
        with pytest.raises(ValueError, match="session"):
            ses.optimize(bad)
    assert np.array_equal(_tables(ses[0])["pose"], p0) and ses[0].loop_related_views == lrv
    ses.optimize([])
    assert ses[0].loop_related_views == lrv


def test_sessions_optimize_real_frontend(cuda_model):
    from test_sessions_gpu import _frames, _real_sessions
    lengths = [9, 6, 11]
    streams = [_frames(n, 31 + k) for k, n in enumerate(lengths)]
    ses = _real_sessions(cuda_model, 3, {}, pgo_every=1000)
    ses.step({k: st for k, st in enumerate(streams)})
    assert all(s.num_edges > 0 for s in ses.sessions)
    saved = [(s._graph.pose[:s.num_nodes].clone(), set(s.loop_related_views)) for s in ses.sessions]
    want = []
    for s in ses.sessions:
        s.pose_graph_optimize()
        want.append(s._graph.pose[:s.num_nodes].clone())
    for s, (pose, lrv) in zip(ses.sessions, saved):
        s._graph.pose[:s.num_nodes] = pose
        s.loop_related_views = lrv
    ses.optimize(range(3))
    for s, w in zip(ses.sessions, want):
        assert torch.equal(s._graph.pose[:s.num_nodes], w)
        assert s.loop_related_views == set()
