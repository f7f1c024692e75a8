"""CPU: the block-sparse route of the pose-graph LM step without a GPU.

  * the sparse oracle (oracle/pose_graph_sparse_oracle.py) equals the dense oracle on planted graphs;
  * the host analysis of the library's plan (sta_pg_plan_analyze): the ordering is a permutation of the optimised nodes,
    L's block pattern is the boolean elimination's under that ordering, every update reads only columns of earlier
    elimination-tree levels, and malformed problems are refused with a message;
  * the header declares the new entry points and the dense limit that _lib mirrors.
"""
import ctypes
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from oracle import pose_graph_oracle as pg
from oracle import pose_graph_sparse_oracle as pgs
from test_pose_graph import make_graph


def analyze(edges, num_nodes, opt_idx):
    """sta_pg_plan_analyze: (stats dict, order, level, colptr, blk_row, upd_ptr, upd)."""
    from vista_slam_b200 import _lib
    L = _lib.lib()
    e = np.ascontiguousarray(edges, dtype=np.int64).reshape(-1, 2)
    o = np.ascontiguousarray(opt_idx, dtype=np.int64)
    st = (ctypes.c_int64 * 5)()
    rc = L.sta_pg_plan_analyze(e.ctypes.data, len(e), num_nodes, o.ctypes.data, len(o), st, *([None] * 6))
    if rc != 0:
        raise RuntimeError(L.sta_last_error().decode())
    nl, na, nlev, nupd, nbytes = map(int, st)
    n = len(o)
    order, level = np.empty(n, np.int32), np.empty(n, np.int32)
    colptr, blk_row = np.empty(n + 1, np.int32), np.empty(nl, np.int32)
    upd_ptr, upd = np.empty(nl + 1, np.int64), np.empty(2 * nupd, np.int32)
    rc = L.sta_pg_plan_analyze(e.ctypes.data, len(e), num_nodes, o.ctypes.data, len(o), st,
                               *[a.ctypes.data for a in (order, level, colptr, blk_row, upd_ptr, upd)])
    assert rc == 0
    stats = {"l_blocks": nl, "a_blocks": na, "levels": nlev, "updates": nupd, "device_bytes": nbytes}
    return stats, order, level, colptr, blk_row, upd_ptr, upd.reshape(-1, 2)


def boolean_elimination(edges, opt_idx, order):
    """Lower block pattern of the Cholesky factor of P A P^T, by dense boolean elimination."""
    opt_map = pg.split_nodes(int(max(edges.max(), max(opt_idx))) + 1, opt_idx)
    n = len(opt_idx)
    pos = np.empty(n, np.int64)
    pos[np.asarray(order)] = np.arange(n)
    M = np.eye(n, dtype=bool)
    for i, j in edges:
        a, b = opt_map[i], opt_map[j]
        if a >= 0 and b >= 0:
            M[pos[a], pos[b]] = M[pos[b], pos[a]] = True
    for k in range(n):
        rows = np.nonzero(M[k + 1:, k])[0] + k + 1
        M[np.ix_(rows, rows)] = True
    return np.tril(M)


def slam_shaped_edges(n_views=40, per_view=6, seed=0):
    """Edges like OnlineSLAM's: each keyframe adds nodes for its views, scale edges to each view's first node, pose
    edges to the previous three keyframes and an occasional loop closure."""
    rng = np.random.default_rng(seed)
    first, edges, nn = {}, [], 0
    for i in range(1, n_views):
        for j in [j for j in range(max(0, i - 3), i)] + ([int(rng.integers(0, i - 8))] if i > 12 and i % 4 == 0 else []):
            a, b = nn, nn + 1
            nn += 2
            for v, node in ((i, a), (j, b)):
                if v in first:
                    edges.append((node, first[v]))
                else:
                    first[v] = node
            edges.append((a, b))
    return np.array(edges, np.int64), nn


def graphs():
    rng = np.random.default_rng(21)
    _, init, edges, _, _ = make_graph(rng, n_nodes=60, n_loops=15)
    yield "planted", edges, 60, list(range(1, 60))
    yield "planted-window", edges, 60, list(range(30, 60))
    e, nn = slam_shaped_edges()
    yield "slam-shaped", e, nn, list(range(nn))
    # two components, repeated pairs, an isolated optimised node, unrelated edges, scrambled optimised order
    e2 = np.concatenate([edges[:40], edges[:40] + 60, edges[:5], [[0, 1], [2, 3]]])
    opt = list(rng.permutation(np.r_[10:60, 70:120, 121]))
    yield "mixed", e2, 122, opt
    r = rng.integers(0, 50, size=(120, 2))
    yield "random", r[r[:, 0] != r[:, 1]], 50, list(range(50))


@pytest.mark.parametrize("window", [False, True])
def test_sparse_oracle_equals_dense_oracle(window):
    rng = np.random.default_rng(31)
    gt, init, edges, meas, weights = make_graph(rng, n_nodes=14, n_loops=4, noise=0.05, meas_noise=0.02)
    opt_idx = list(range(9, 14)) if window else list(range(1, 14))
    A, g, loss = pg.build_normal_equations(init, edges, meas, weights, opt_idx)
    As, gs, losss = pgs.build_normal_equations(init, edges, meas, weights, opt_idx)
    assert np.allclose(As.toarray(), A, rtol=1e-13, atol=1e-13 * np.abs(A).max())
    assert np.array_equal(gs, g) and losss == loss
    n1, l0, l1, d = pg.lm_step(init, edges, meas, weights, opt_idx, 1e-4)
    n2, s0, s1, ds = pgs.lm_step(init, edges, meas, weights, opt_idx, 1e-4)
    assert s0 == l0 and abs(s1 - l1) <= 1e-12 * l0
    assert np.allclose(ds, d, rtol=0, atol=1e-12 * np.abs(d).max())
    assert np.allclose(n2, n1, rtol=0, atol=1e-12)
    nodes, losses = pg.optimize(init, edges, meas, weights, opt_idx)
    snodes, slosses = pgs.optimize(init, edges, meas, weights, opt_idx)
    assert len(slosses) == len(losses)
    assert np.allclose(slosses, losses, rtol=1e-10, atol=1e-14)
    assert np.allclose(snodes, nodes, rtol=0, atol=1e-10)


def test_sparse_oracle_refuses_an_indefinite_system():
    rng = np.random.default_rng(32)
    gt, init, edges, meas, weights = make_graph(rng, n_nodes=8, n_loops=2, noise=0.05, meas_noise=0.02)
    weights[3] = -100.0
    with pytest.raises(np.linalg.LinAlgError):
        pg.lm_step(init, edges, meas, weights, list(range(1, 8)), 1e-4)
    with pytest.raises(np.linalg.LinAlgError):
        pgs.lm_step(init, edges, meas, weights, list(range(1, 8)), 1e-4)


@pytest.mark.parametrize("name,edges,num_nodes,opt_idx", list(graphs()), ids=[g[0] for g in graphs()])
def test_plan_ordering_pattern_and_levels(name, edges, num_nodes, opt_idx):
    stats, order, level, colptr, blk_row, upd_ptr, upd = analyze(edges, num_nodes, opt_idx)
    n = len(opt_idx)
    assert sorted(order.tolist()) == list(range(n))                       # a permutation of the optimised nodes
    assert analyze(edges, num_nodes, opt_idx)[1].tolist() == order.tolist()  # deterministic
    # L's block pattern, column by column: diagonal first, then rows ascending
    want = boolean_elimination(np.asarray(edges), opt_idx, order)
    got = np.zeros((n, n), bool)
    for K in range(n):
        rows = blk_row[colptr[K]:colptr[K + 1]]
        assert rows[0] == K and (np.diff(rows) > 0).all()
        got[rows, K] = True
    assert np.array_equal(got, want)
    assert stats["l_blocks"] == colptr[n] == want.sum() and stats["levels"] == level.max() + 1
    # A's lower blocks are a subset of L's
    assert stats["a_blocks"] <= stats["l_blocks"]
    # elimination tree levels: parent = first off-diagonal row, strictly higher level
    for K in range(n):
        if colptr[K + 1] - colptr[K] > 1:
            assert level[blk_row[colptr[K] + 1]] > level[K]
    # updates: block (I, K) gets L_Ij L_Kj^T for exactly the j < K with both blocks nonzero, ascending, and reads only
    # columns of earlier levels
    col_of = np.repeat(np.arange(n), np.diff(colptr))
    assert upd_ptr[-1] == stats["updates"] == len(upd)
    for b in range(colptr[n]):
        I, K = blk_row[b], col_of[b]
        u = upd[upd_ptr[b]:upd_ptr[b + 1]]
        js = col_of[u[:, 0]]
        assert np.array_equal(js, col_of[u[:, 1]]) and (np.diff(js) > 0).all()
        assert (blk_row[u[:, 0]] == I).all() and (blk_row[u[:, 1]] == K).all()
        assert np.array_equal(js, np.nonzero(want[I, :K] & want[K, :K])[0])
        assert (level[js] < level[K]).all()


def test_plan_refusals():
    e = np.array([[0, 1], [1, 2], [2, 3]], np.int64)
    for edges, nn, opt, msg in ((e, 4, [1, 2, 2], "repeated"),
                                (e, 4, [1, 4], "optimised index 4 outside"),
                                (e, 4, [-1, 2], "optimised index -1 outside"),
                                (np.array([[0, 1], [1, 5]]), 4, [1], "edge 1 has endpoint 5 outside"),
                                (np.array([[0, -1]]), 4, [1], "endpoint -1 outside"),
                                (e, 4, [], "empty problem"),
                                (np.zeros((0, 2)), 4, [1], "empty problem")):
        with pytest.raises(RuntimeError, match=msg):
            analyze(edges, nn, opt)


def test_plan_statistics_grow_with_the_factor_not_the_square():
    e, nn = slam_shaped_edges(n_views=400)
    stats = analyze(e, nn, list(range(nn)))[0]
    # the dense route would hold (7 nn)^2 doubles; the plan holds a few blocks per node
    assert nn > 2000 and stats["l_blocks"] < 10 * stats["a_blocks"]
    assert stats["device_bytes"] < 8 * (7 * nn) ** 2 / 20


def test_header_declares_the_sparse_route_and_the_dense_limit():
    from vista_slam_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "sta_b200.h")).read()
    for name in ("sta_pg_plan_create", "sta_pg_plan_destroy", "sta_pg_plan_info", "sta_pg_plan_analyze",
                 "sta_pose_graph_lm_step_sparse", "sta_pg_plan_last_delta"):
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert hasattr(_lib.lib(), name)
    assert int(re.search(r"STA_PG_DENSE_MAX_OPT\s*=\s*(\d+)", hdr).group(1)) == _lib.PG_DENSE_MAX_OPT == 3657
    # the dense route's shared-memory right-hand side: 7 x 8 bytes per node within 200 KB
    assert 7 * 8 * _lib.PG_DENSE_MAX_OPT <= 200 * 1024 < 7 * 8 * (_lib.PG_DENSE_MAX_OPT + 1)
