"""GPU: the block-sparse LM step over a group of plans (sta_pose_graph_lm_step_sparse_group), the route choice of
PoseGraphOpt, optimize_group over block-sparse-route graphs, and OnlineSLAM / SLAMSessions with pgo_route = "sparse".

  * every active member's nodes_out, info row and last update equal sta_pose_graph_lm_step_sparse on its own plan bit
    for bit, in groups of 1, 2, 3, 8 and 16 graphs of different sizes, level counts and windows, in any order and with
    members sitting steps out; inactive members' outputs and info rows keep their NaN sentinels;
  * the launches per step depend on the level count only, not on G;
  * optimize_group leaves route="sparse" graphs as their own optimize() does: plateau exits at different iterations,
    a fixed 20 steps, more than PG_GROUP_MAX graphs, mixed dense and sparse groups, one read-back per iteration;
  * route choice and its refusals; the golden SLAM replay and SLAMSessions.optimize on the sparse route;
  * every refusal of the C entry points comes before any launch."""
import ctypes
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import pose_graph_oracle as pg
from test_pose_graph import make_graph
from test_pose_graph_sparse_gpu import planted

pytestmark = pytest.mark.gpu


def _t(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t.to(dtype) if dtype is not None else t).cuda()


# (n, windowed, seed): sizes and windows that give different level counts, node and edge counts; every graph has
# repeated node pairs and an optimised node without a related edge (planted())
PLANTED = [(40, False, 1), (60, True, 2), (90, False, 3), (130, False, 4), (25, False, 5), (33, True, 6), (200, False, 7),
           (70, True, 8), (48, False, 9), (110, True, 10), (17, False, 11), (150, False, 12), (64, False, 13),
           (81, True, 14), (300, False, 15), (55, False, 16)]


class _Member:
    """One planted graph with its plan, device inputs and the solo step's results at its own damping."""

    def __init__(self, spec, k):
        from vista_slam_b200 import _lib
        from vista_slam_b200.pose_graph import _SparsePlan
        init, edges, meas, weights, opt = planted(*spec)
        self.nodes, self.edges = _t(init, torch.float32), _t(edges)
        self.meas, self.weights = _t(meas, torch.float32), _t(weights, torch.float32)
        self.plan = _SparsePlan(self.edges, self.nodes.shape[0], torch.tensor(opt))
        self.n_opt, self.damping = len(opt), 1e-4 * (1 + k)
        self.levels = self.plan.info()["levels"]
        L = _lib.lib()
        self.out = torch.full_like(self.nodes, float("nan"))
        self.info = torch.full((4,), float("nan"), dtype=torch.float64, device="cuda")
        _lib.check(L.sta_pose_graph_lm_step_sparse(self.plan.h, _lib.ptr(self.nodes), _lib.ptr(self.meas),
                                                   _lib.ptr(self.weights), self.damping, 1e-6, 1e32, _lib.ptr(self.out),
                                                   _lib.ptr(self.info), _lib.cur_stream()), "solo step")
        self.delta = self.last_delta()
        assert not torch.isnan(self.out).any() and self.info[3] == 1.0

    def last_delta(self):
        from vista_slam_b200 import _lib
        d = torch.empty(7 * self.n_opt, dtype=torch.float64, device="cuda")
        _lib.check(_lib.lib().sta_pg_plan_last_delta(self.plan.h, _lib.ptr(d), _lib.cur_stream()), "last delta")
        return d

    def step(self, out, active=True):
        from vista_slam_b200 import _lib
        if not active:
            return _lib.StaPgSparseStep(None, None, None, None, 0.0, 0)
        return _lib.StaPgSparseStep(self.nodes.data_ptr(), self.meas.data_ptr(), self.weights.data_ptr(), out.data_ptr(),
                                    self.damping, 1)


@pytest.fixture(scope="module")
def members():
    return [_Member(s, k) for k, s in enumerate(PLANTED)]


def _group_plan(plans):
    from vista_slam_b200 import _lib
    L = _lib.lib()
    h = ctypes.c_void_p()
    tab = (ctypes.c_void_p * len(plans))(*[p.h for p in plans])
    _lib.check(L.sta_pg_group_plan_create(tab, len(plans), ctypes.byref(h)), "group plan")
    return h


def _plan_info(h):
    from vista_slam_b200 import _lib
    v = (ctypes.c_int64 * 4)()
    _lib.check(_lib.lib().sta_pg_group_plan_info(h, v), "group plan info")
    return [int(x) for x in v]


def _run_group(ms, active):
    """One group step of ms with the given active flags into NaN-filled outputs -> (outs, info [G][4])."""
    from vista_slam_b200 import _lib
    L = _lib.lib()
    h = _group_plan([m.plan for m in ms])
    try:
        outs = [torch.full_like(m.nodes, float("nan")) for m in ms]
        info = torch.full((len(ms), 4), float("nan"), dtype=torch.float64, device="cuda")
        steps = (_lib.StaPgSparseStep * len(ms))(*[m.step(o, a) for m, o, a in zip(ms, outs, active)])
        _lib.check(L.sta_pose_graph_lm_step_sparse_group(h, steps, 1e-6, 1e32, _lib.ptr(info), _lib.cur_stream()),
                   "group step")
        torch.cuda.synchronize()
    finally:
        L.sta_pg_group_plan_destroy(h)
    return outs, info


def test_c_group_step_equals_solo_steps(members):
    rnd = random.Random(7)
    cases = [([3], [True]), ([0, 1], [True, True]), ([4, 2, 10], [True, False, True]),
             (list(range(8)), [True] * 8), (list(range(16)), [True] * 16)]
    perm = list(range(16))
    rnd.shuffle(perm)
    cases.append((perm, [rnd.random() < 0.6 for _ in perm]))
    sub = rnd.sample(range(16), 8)
    cases.append((sub, [k % 3 != 1 for k in range(8)]))
    cases.append((list(reversed(range(16))), [False] * 15 + [True]))
    assert len({m.levels for m in members}) > 3  # the members have different level counts
    for idx, active in cases:
        ms = [members[k] for k in idx]
        outs, info = _run_group(ms, active)
        for m, o, row, a in zip(ms, outs, info, active):
            if a:
                assert torch.equal(o, m.out) and torch.equal(row, m.info), idx
                assert torch.equal(m.last_delta(), m.delta), idx
            else:
                assert torch.isnan(o).all() and torch.isnan(row).all(), idx


def test_no_active_member_launches_nothing(members):
    outs, info = _run_group(members[:3], [False] * 3)
    assert all(torch.isnan(o).all() for o in outs) and torch.isnan(info).all()


def test_launches_per_step_do_not_grow_with_the_group(members):
    deepest = max(members, key=lambda m: m.levels)
    one = _group_plan([deepest.plan])
    full = _group_plan([m.plan for m in members])
    from vista_slam_b200 import _lib
    try:
        i1, i16 = _plan_info(one), _plan_info(full)
    finally:
        _lib.lib().sta_pg_group_plan_destroy(one)
        _lib.lib().sta_pg_group_plan_destroy(full)
    assert i1[0] == 1 and i16[0] == 16
    assert i1[1] == i16[1] == deepest.levels
    assert i1[2] == i16[2] == 4 * deepest.levels + 6
    assert 0 < i1[3] < i16[3] < 1 << 20  # small tables: the member plans keep their arrays and scratch


# ------------------------------------------------------------------------------------------------ optimize_group
SPECS = [  # (seed, nodes, loops, init noise, measurement noise, optimised set), as tests/test_pose_graph_group_gpu.py
    (7, 60, 15, 0.05, 0.0, "all_but_0"),
    (40, 12, 3, 1.5, 0.02, "all_but_0"),
    (6, 40, 10, 0.05, 0.02, "all_but_0"),
    (11, 25, 4, 0.1, 0.01, "window"),
    (12, 90, 30, 0.05, 0.01, "all"),
    (13, 8, 1, 0.2, 0.0, "all_but_0"),
    (14, 33, 0, 0.1, 0.03, "window"),
    (15, 120, 40, 0.03, 0.005, "all_but_0"),
]


def _problem(spec):
    seed, n, loops, noise, mnoise, which = spec
    _, init, edges, meas, weights = make_graph(np.random.default_rng(seed), n_nodes=n, n_loops=loops, noise=noise,
                                               meas_noise=mnoise)
    opt = {"all_but_0": list(range(1, n)), "window": list(range(n - 10, n)), "all": list(range(n))}[which]
    return (_t(init, torch.float32), torch.tensor(opt), _t(edges), _t(meas, torch.float32), _t(weights, torch.float32))


@pytest.fixture(scope="module")
def problems():
    return [_problem(s) for s in SPECS]


def _solo(p, route, **kw):
    from vista_slam_b200.pose_graph import PoseGraphOpt
    nodes, opt, edges, meas, w = p
    g = PoseGraphOpt(nodes, opt, route=route)
    return g.optimize(edges, meas, w, **kw), g.get_nodes()


def _group(ps, routes, **kw):
    from vista_slam_b200.pose_graph import PoseGraphOpt
    gs = [PoseGraphOpt(p[0], p[1], route=r) for p, r in zip(ps, routes)]
    losses = PoseGraphOpt.optimize_group(gs, [p[2] for p in ps], [p[3] for p in ps], [p[4] for p in ps], **kw)
    return losses, [g.get_nodes() for g in gs]


def _count_read_backs(monkeypatch):
    import vista_slam_b200.pose_graph as P
    counts, orig = [0], P._read_info

    def read(t):
        counts[0] += 1
        return orig(t)

    monkeypatch.setattr(P, "_read_info", read)
    return counts


def test_optimize_group_sparse_equals_solo(problems, monkeypatch):
    solo = [_solo(p, "sparse") for p in problems]
    assert len({len(h) for h, _ in solo}) > 1  # the graphs leave the group at different iterations
    counts = _count_read_backs(monkeypatch)
    for members in ([3], [0, 1, 2], list(range(8))):
        counts[0] = 0
        losses, nodes = _group([problems[k] for k in members], ["sparse"] * len(members))
        assert counts[0] == max(len(h) for h in losses)
        for k, h, x in zip(members, losses, nodes):
            assert h == solo[k][0] and torch.equal(x, solo[k][1]), (members, k)
    order = list(range(8))
    random.Random(5).shuffle(order)
    losses, nodes = _group([problems[k] for k in order], ["sparse"] * 8)
    for k, h, x in zip(order, losses, nodes):
        assert h == solo[k][0] and torch.equal(x, solo[k][1]), k
    # a fixed number of iterations (no plateau stop)
    solo20 = [_solo(p, "sparse", patience=100) for p in problems[:5]]
    losses, nodes = _group(problems[:5], ["sparse"] * 5, patience=100)
    assert all(len(h) == 20 for h in losses)
    for (h, x), h2, x2 in zip(solo20, losses, nodes):
        assert h == h2 and torch.equal(x, x2)


def test_optimize_group_sparse_chunks_and_mixed_groups(problems, monkeypatch):
    from vista_slam_b200 import _lib
    from vista_slam_b200 import pose_graph as P
    solo_s = [_solo(p, "sparse") for p in problems]
    solo_d = [_solo(p, None) for p in problems]
    sizes = []
    init = P._SparseGroup.__init__

    def recording(self, *a, **kw):
        init(self, *a, **kw)
        sizes.append([c1 - c0 for c0, c1, _ in self.chunks])
    monkeypatch.setattr(P._SparseGroup, "__init__", recording)
    counts = _count_read_backs(monkeypatch)
    # more than PG_GROUP_MAX sparse graphs: two group plans
    n = _lib.PG_GROUP_MAX + 3
    idx = [k % 8 for k in range(n)]
    losses, nodes = _group([problems[k] for k in idx], ["sparse"] * n)
    assert sizes[-1] == [_lib.PG_GROUP_MAX, 3] and counts[0] == max(len(h) for h in losses)
    for k, h, x in zip(idx, losses, nodes):
        assert h == solo_s[k][0] and torch.equal(x, solo_s[k][1]), k
    # mixed: dense and sparse members interleaved, one read-back per iteration for all of them
    for routes in (["sparse", None] * 4, [None] * 7 + ["sparse"], ["sparse", "dense", "dense", "sparse", None, "sparse",
                                                                   "sparse", "dense"]):
        counts[0] = 0
        losses, nodes = _group(problems, routes)
        assert counts[0] == max(len(h) for h in losses)
        for k, (r, h, x) in enumerate(zip(routes, losses, nodes)):
            want = solo_s[k] if r == "sparse" else solo_d[k]
            assert h == want[0] and torch.equal(x, want[1]), (routes, k)


# ------------------------------------------------------------------------------------------------ route choice
@pytest.mark.parametrize("n", [40, 60])
@pytest.mark.parametrize("window", [False, True])
def test_sparse_route_agrees_with_dense_on_small_graphs(n, window):
    """The tolerances of test_routes_agree_on_small_graphs, with route="sparse" instead of a lowered limit."""
    from vista_slam_b200.pose_graph import PoseGraphOpt
    init, edges, meas, weights, opt = planted(n, window, seed=n + window)
    args = (_t(edges), _t(meas, torch.float32), _t(weights, torch.float32))
    mk = lambda route: PoseGraphOpt(_t(init, torch.float32), torch.tensor(opt), route=route)
    dense, sparse = mk(None), mk("sparse")
    assert not dense.sparse and sparse.sparse and not mk("dense").sparse
    c_d, d0, d1, dn, ok_d = dense.lm_step(*args, 1e-4)
    c_s, s0, s1, sn, ok_s = sparse.lm_step(*args, 1e-4)
    assert ok_d and ok_s and s0 == d0
    ref, r0, r1, delta = pg.lm_step(init, edges, meas, weights, opt, 1e-4)
    assert abs(s1 - r1) < 1e-6 * max(1.0, r0) and abs(sn - np.linalg.norm(delta)) < 1e-8 * max(1.0, np.linalg.norm(delta))
    got = c_s.cpu().numpy().astype(np.float64)
    for v in range(len(init)):
        assert np.allclose(pg.sim3_matrix(got[v]), pg.sim3_matrix(ref[v]), atol=2e-6), v
    losses_d, losses_s = mk("dense").optimize(*args), mk("sparse").optimize(*args)
    assert len(losses_s) == len(losses_d)
    np.testing.assert_allclose(losses_s, losses_d, rtol=1e-6, atol=0)


def test_route_refusals_and_default(monkeypatch):
    from vista_slam_b200 import _lib
    from vista_slam_b200.pose_graph import PoseGraphOpt
    big = torch.zeros(_lib.PG_DENSE_MAX_OPT + 1, 8, device="cuda")
    big[:, 6] = big[:, 7] = 1.0
    with pytest.raises(ValueError, match="route='dense'"):
        PoseGraphOpt(big, route="dense")
    assert PoseGraphOpt(big, route="sparse").sparse and PoseGraphOpt(big).sparse
    assert not PoseGraphOpt(big[:-1], route="dense").sparse and not PoseGraphOpt(big[:-1]).sparse
    for bad in ("Sparse", "block", 1, True):
        with pytest.raises(ValueError, match="route"):
            PoseGraphOpt(big[:10], route=bad)
    small = big[:40]
    monkeypatch.setattr(_lib, "PG_DENSE_MAX_OPT", 39)
    assert PoseGraphOpt(small).sparse and not PoseGraphOpt(small[:39]).sparse
    with pytest.raises(ValueError, match="route='dense'"):
        PoseGraphOpt(small, route="dense")
    monkeypatch.setattr(_lib, "PG_DENSE_MAX_OPT", 40)
    assert not PoseGraphOpt(small).sparse and PoseGraphOpt(small, route="sparse").sparse


# ------------------------------------------------------------------------------------------------ SLAM
def test_golden_slam_replay_on_the_sparse_route(tmp_path, monkeypatch):
    import test_slam_gpu as tsg
    from vista_slam_b200 import pose_graph as P
    golden = dict(np.load(os.path.join(GOLDEN_DIR, "slam_graph.npz")))
    built, init = [], P._SparsePlan.__init__

    def counting(self, *a):
        init(self, *a)
        built.append(self)
    monkeypatch.setattr(P._SparsePlan, "__init__", counting)
    replay = tsg._replay_slam

    def sparse_replay(*a, **kw):
        slam = replay(*a, **kw)
        assert slam.pgo_route is None
        slam.pgo_route = "sparse"
        return slam
    monkeypatch.setattr(tsg, "_replay_slam", sparse_replay)
    tsg.test_golden_replay(golden, tmp_path, monkeypatch)
    assert len(built) == len(golden["pgo_num_edges"])  # every PGO took the sparse route, one plan each


def test_sessions_optimize_sparse_route_equals_per_session_pgo(capsys):
    from oracle import slam_oracle as so
    from test_pose_graph_group_gpu import _stepped, _tables
    streams = [so.make_stream(seed=3, n_views=20), so.make_stream(seed=8, n_views=14), so.make_stream(seed=21, n_views=1)]
    ses, twin = _stepped(streams), _stepped(streams)
    for s in ses.sessions + twin.sessions:
        s.pgo_route = "sparse"
    assert any(s.loop_related_views for s in ses.sessions)
    before = [_tables(s)["pose"] for s in ses.sessions]
    capsys.readouterr()
    ses.optimize(range(len(streams)))
    got = capsys.readouterr().out.splitlines()
    for s in twin.sessions:
        s.pose_graph_optimize()
    want = capsys.readouterr().out.splitlines()
    assert sorted(got) == sorted(want) and len(got) == 2 * len(streams)
    for a, b in zip(ses.sessions, twin.sessions):
        ta, tb = _tables(a), _tables(b)
        for k in ta:
            np.testing.assert_array_equal(ta[k], tb[k], err_msg=k)
        assert a.loop_related_views == b.loop_related_views == set()
    assert not np.array_equal(_tables(ses[0])["pose"], before[0])


# ------------------------------------------------------------------------------------------------ refusals
def test_group_refusals(members):
    from vista_slam_b200 import _lib
    L = _lib.lib()
    ms = members[:3]
    out = ctypes.c_void_p()
    tab = (ctypes.c_void_p * 3)(ms[0].plan.h, ms[1].plan.h, ms[0].plan.h)
    assert L.sta_pg_group_plan_create(tab, 3, ctypes.byref(out)) == 2
    assert b"named twice" in L.sta_last_error() and out.value is None
    h = _group_plan([m.plan for m in ms])
    try:
        outs = [torch.full_like(m.nodes, float("nan")) for m in ms]
        info = torch.full((3, 4), float("nan"), dtype=torch.float64, device="cuda")
        st = _lib.cur_stream()

        def steps(k=None, field=None):
            t = (_lib.StaPgSparseStep * 3)(*[m.step(o) for m, o in zip(ms, outs)])
            if k is not None:
                setattr(t[k], field, None)
            return t

        def refused(gp, tab, info_p, msg):
            assert L.sta_pose_graph_lm_step_sparse_group(gp, tab, 1e-6, 1e32, info_p, st) == 2
            assert msg in L.sta_last_error(), L.sta_last_error()

        refused(None, steps(), _lib.ptr(info), b"null pointer")
        refused(h, None, _lib.ptr(info), b"null pointer")
        refused(h, steps(), None, b"null pointer")
        for f in ("nodes", "meas", "weights", "nodes_out"):
            refused(h, steps(2, f), _lib.ptr(info), b"active member")
        torch.cuda.synchronize()
        assert all(torch.isnan(o).all() for o in outs) and torch.isnan(info).all()
        # an inactive member's null pointers are never read
        t = steps(1, "nodes")
        t[1].active = 0
        _lib.check(L.sta_pose_graph_lm_step_sparse_group(h, t, 1e-6, 1e32, _lib.ptr(info), st), "group step")
        torch.cuda.synchronize()
        assert torch.isnan(outs[1]).all() and torch.isnan(info[1]).all()
        assert torch.equal(outs[0], ms[0].out) and torch.equal(outs[2], ms[2].out)
        if torch.cuda.device_count() > 1:
            with torch.cuda.device(1):
                assert L.sta_pose_graph_lm_step_sparse_group(h, steps(), 1e-6, 1e32, _lib.ptr(info), st) == 2
                assert b"another device" in L.sta_last_error()
                other = ctypes.c_void_p()
                tab = (ctypes.c_void_p * 1)(ms[0].plan.h)
                assert L.sta_pg_group_plan_create(tab, 1, ctypes.byref(other)) == 2
                assert b"another device" in L.sta_last_error()
    finally:
        L.sta_pg_group_plan_destroy(h)
