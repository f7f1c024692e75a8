"""GPU: the block-sparse route of PoseGraphOpt (csrc/pose_graph_sparse.cu) against the dense route and the oracles.

Small problems are sent down the sparse route by lowering _lib.PG_DENSE_MAX_OPT, which PoseGraphOpt reads in its
constructor; the last test runs a graph beyond the dense route's limit as it is shipped.
"""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import pose_graph_oracle as pg
from oracle import pose_graph_sparse_oracle as pgs
from oracle import slam_oracle as so
from test_pose_graph import make_graph

pytestmark = pytest.mark.gpu
U = np.finfo(np.float64).eps / 2


def _t(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t.to(dtype) if dtype is not None else t).cuda()


@pytest.fixture
def sparse_route(monkeypatch):
    """Every PoseGraphOpt built while active takes the sparse route; yields the list of plans built."""
    from vista_slam_b200 import _lib
    from vista_slam_b200 import pose_graph as P
    monkeypatch.setattr(_lib, "PG_DENSE_MAX_OPT", 0)
    built = []
    init = P._SparsePlan.__init__

    def counting(self, *a):
        init(self, *a)
        built.append(self)
    monkeypatch.setattr(P._SparsePlan, "__init__", counting)
    return built


def planted(n, window, seed):
    """Two planted components (the second offset by n // 2), three repeated node pairs with their own measurements,
    and an isolated last node that is optimised but has no related edge.  Windowed: two windows of optimised nodes, so
    that edges among fixed nodes are unrelated.  Returns fp32-rounded inputs in float64 and the optimised indices."""
    rng = np.random.default_rng(seed)
    h = n // 2
    _, i1, e1, m1, w1 = make_graph(rng, n_nodes=h, n_loops=5, noise=0.05, meas_noise=0.02)
    _, i2, e2, m2, w2 = make_graph(rng, n_nodes=n - h - 1, n_loops=5, noise=0.05, meas_noise=0.02)
    edges = np.concatenate([e1, e2 + h])
    meas, weights = np.concatenate([m1, m2]), np.concatenate([w1, w2])
    dup = rng.choice(len(edges), 3, replace=False)
    dmeas = np.array([pg.sim3_mul(pg.sim3_exp(rng.normal(size=7) * 0.02), meas[k]) for k in dup])
    edges, meas = np.concatenate([edges, edges[dup]]), np.concatenate([meas, dmeas])
    weights = np.concatenate([weights, 0.5 + rng.random((3, 7))])
    lone = pg.sim3_exp(rng.normal(size=7) * 0.3)
    init = np.concatenate([i1, i2, lone[None]])
    opt = list(range(h - 8, h)) + list(range(n - 12, n)) if window else [v for v in range(n) if v not in (0, h)]
    r32 = lambda a: a.astype(np.float32).astype(np.float64)
    return r32(init), edges, r32(meas), r32(weights), opt


def _graph(init, opt):
    from vista_slam_b200.pose_graph import PoseGraphOpt
    return PoseGraphOpt(_t(init, torch.float32), torch.tensor(opt))


def _args(edges, meas, weights):
    return _t(edges), _t(meas, torch.float32), _t(weights, torch.float32)


@pytest.mark.parametrize("n", [40, 60])
@pytest.mark.parametrize("window", [False, True])
def test_routes_agree_on_small_graphs(n, window, monkeypatch):
    from vista_slam_b200 import _lib
    init, edges, meas, weights, opt = planted(n, window, seed=n + window)
    args = _args(edges, meas, weights)
    dense = _graph(init, opt)
    assert not dense.sparse
    monkeypatch.setattr(_lib, "PG_DENSE_MAX_OPT", 0)
    sparse = _graph(init, opt)
    assert sparse.sparse
    c_d, d0, d1, dn, ok_d = dense.lm_step(*args, 1e-4)
    c_s, s0, s1, sn, ok_s = sparse.lm_step(*args, 1e-4)
    assert ok_d and ok_s
    assert s0 == d0  # same residuals, same fixed-order reduction
    ref, r0, r1, delta = pg.lm_step(init, edges, meas, weights, opt, 1e-4)
    assert abs(s1 - r1) < 1e-6 * max(1.0, r0) and abs(sn - np.linalg.norm(delta)) < 1e-8 * max(1.0, np.linalg.norm(delta))
    got = c_s.cpu().numpy().astype(np.float64)
    for v in range(len(init)):
        assert np.allclose(pg.sim3_matrix(got[v]), pg.sim3_matrix(ref[v]), atol=2e-6), v  # fp32 output rounding
    ld = _graph(init, opt)
    ld.sparse = False
    losses_d = ld.optimize(*args)
    losses_s = _graph(init, opt).optimize(*args)
    assert len(losses_s) == len(losses_d)
    np.testing.assert_allclose(losses_s, losses_d, rtol=1e-6, atol=0)


def test_golden_slam_replay_through_the_sparse_route(sparse_route, tmp_path, monkeypatch):
    import test_slam_gpu as tsg
    golden = dict(np.load(os.path.join(GOLDEN_DIR, "slam_graph.npz")))
    tsg.test_golden_replay(golden, tmp_path, monkeypatch)
    assert len(sparse_route) == len(golden["pgo_num_edges"])  # one plan per PGO, reused across its iterations


def test_solver_backward_error(sparse_route):
    """Residual of the device's update d (fp64, read back from the plan) in the oracle's fp64 normal equations:
    ||(A + damping) d + g||.

    Bound: the Cholesky factorisation and the two triangular solves are backward stable -- the computed d solves
    (A_d + dA) d = -g_d with |dA| <= gamma(3m + 1) |L| |L^T| (Higham, Accuracy and Stability of Numerical Algorithms,
    Thm 10.4; m = 7 n_opt, gamma(k) = k u / (1 - k u)), and || |L| |L^T| ||_2 <= m ||A||_2 (Thm 10.5).  A_d, g_d are the
    device's normal equations: the same fp32 inputs, but residuals and Jacobians evaluated in closed form where the
    oracle takes matrix exponentials.  Their relative difference from the oracle's is bounded by the cancellation in the
    closed-form coefficients of W (u / theta^2 for a residual rotation angle theta >= theta_min), the series truncated
    below |sigma| = 1e-2 (sigma^5 / 720 <= 1.4e-13) and 64 u for the roundings of one product chain:
      ||(A + damping) d + g|| <= (gamma(3m + 1) m + eps) ||A||_2 ||d|| + eps ||g||,  eps = 64 u + u / theta_min^2 + 1.4e-13."""
    from vista_slam_b200 import _lib
    rng = np.random.default_rng(41)
    _, init, edges, meas, weights = make_graph(rng, n_nodes=50, n_loops=12, noise=0.3, meas_noise=0.1)
    r32 = lambda a: a.astype(np.float32).astype(np.float64)
    init, meas, weights = r32(init), r32(meas), r32(weights)
    opt = list(range(1, 50))
    A, g, _ = pg.build_normal_equations(init, edges, meas, weights, opt)
    Ad = A.copy()
    Ad[np.diag_indices_from(Ad)] = np.clip(np.diag(A), 1e-6, 1e32) * (1.0 + 1e-4)
    theta = min(np.linalg.norm(pg.edge_residual(meas[e], init[i], init[j])[3:6]) for e, (i, j) in enumerate(edges))
    assert theta > 1e-3
    m = Ad.shape[0]
    gam = (3 * m + 1) * U / (1 - (3 * m + 1) * U)
    eps = 64 * U + U / theta ** 2 + 1.4e-13
    gr = _graph(init, opt)
    cand, l0, l1, dn, ok = gr.lm_step(*_args(edges, meas, weights), 1e-4)
    assert ok and len(sparse_route) == 1
    d = torch.empty(m, dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib().sta_pg_plan_last_delta(sparse_route[0].h, _lib.ptr(d), _lib.cur_stream()), "last delta")
    d = d.cpu().numpy()
    assert abs(np.linalg.norm(d) - dn) <= 1e-12 * dn
    res = np.linalg.norm(Ad @ d + g)
    bound = (gam * m + eps) * np.linalg.norm(Ad, 2) * np.linalg.norm(d) + eps * np.linalg.norm(g)
    assert res <= bound, (res, bound)


def test_indefinite_system_is_reported_and_rejected(monkeypatch):
    from vista_slam_b200 import _lib
    rng = np.random.default_rng(42)
    _, init, edges, meas, weights = make_graph(rng, n_nodes=40, n_loops=8, noise=0.05, meas_noise=0.02)
    weights[5] = -100.0  # edge (6, 5): both endpoints optimised
    opt = list(range(1, 40))
    args = _args(edges, meas, weights)
    assert not _graph(init, opt).lm_step(*args, 1e-4)[4]
    monkeypatch.setattr(_lib, "PG_DENSE_MAX_OPT", 0)
    g = _graph(init, opt)
    before = g.get_nodes()
    cand, l0, l1, dn, ok = g.lm_step(*args, 1e-4)
    assert not ok
    losses = g.optimize(*args, steps=2)
    assert losses == [l0, l0] and torch.equal(g.get_nodes(), before)  # both steps rejected, nodes untouched


def test_sparse_route_is_deterministic(sparse_route):
    init, edges, meas, weights, opt = planted(60, False, seed=5)
    args = _args(edges, meas, weights)
    a, b = _graph(init, opt), _graph(init, opt)
    la, lb = a.optimize(*args), b.optimize(*args)
    assert la == lb and torch.equal(a.get_nodes(), b.get_nodes())
    assert len(sparse_route) == 2


def test_online_slam_beyond_the_dense_limit(tmp_path, monkeypatch):
    """A drop-in OnlineSLAM replay whose final force_pgo optimises more than STA_PG_DENSE_MAX_OPT nodes (every edge kept,
    pgo_every above the run length, so the window covers the whole graph).

    Bounds: graph tables against the oracle replay as in tests/test_slam_gpu.py, except node poses: a node pose is a
    chain of up to 2 V float32 Sim(3) products (V = 560 views), each within 5e-7 relative of the float64 product on the
    same inputs, on translations up to 3: 2 V x 5e-7 x 3 = 1.7e-3.  The PGO result against the sparse oracle's optimize
    on the device's own pre-PGO tables: the oracle keeps its iterates in float64 while the device rounds each accepted
    iterate to float32 (6e-8 relative), and at most 20 iterations each start from such a rounding: 20 x 6e-8 x 3 = 3.6e-6
    per element, taken as 1e-5 to leave the LM contraction a factor of 3."""
    import test_slam_gpu as tsg
    import vista_slam_b200.slam as S
    from vista_slam_b200 import _lib
    V = 560
    stream = so.make_stream(n_views=V)
    calls = []

    class RecordingPGO(S.PoseGraphOpt):
        def optimize(self, edges, poses, weight, **kw):
            rec = {"opt": self.idxs_opt.cpu().numpy(), "nodes": self.nodes.cpu().numpy(), "sparse": self.sparse,
                   "edges": edges.cpu().numpy(), "meas": poses.cpu().numpy(), "weight": weight.cpu().numpy()}
            rec["losses"] = super().optimize(edges, poses, weight, **kw)
            rec["result"] = self.nodes.cpu().numpy()
            calls.append(rec)
            return rec["losses"]

    monkeypatch.setattr(S, "PoseGraphOpt", RecordingPGO)
    slam = tsg._replay_slam(stream, max_view_num=600, pgo_every=100000, rel_pose_thres=0.0)
    images = so.stream_images(stream)
    for i in range(V):
        slam.step(tsg._value(images, i, stream), force_pgo=(i == V - 1))
    assert len(calls) == 1
    c = calls[0]
    N, E = slam.num_nodes, slam.num_edges
    assert len(c["opt"]) == N > _lib.PG_DENSE_MAX_OPT and c["sparse"]
    # the dense route still refuses this problem, with today's message
    from vista_slam_b200.pose_graph import PoseGraphOpt
    dense = PoseGraphOpt(_t(c["nodes"]), _t(c["opt"]))
    assert dense.sparse
    dense.sparse = False
    with pytest.raises(RuntimeError, match="more than 3657 optimised nodes"):
        dense.lm_step(*_args(c["edges"], c["meas"], c["weight"]), 1e-4)
    del dense
    torch.cuda.empty_cache()
    # graph tables before the PGO against the oracle replay (its final PGO through the sparse oracle)
    graph, _, pgos = pgs.run(stream, pgo_every=100000, max_view_num=600, rel_pose_thres=0.0)
    assert (graph.num_nodes, graph.num_edges) == (N, E) and len(pgos) == 1
    np.testing.assert_array_equal(c["opt"], pgos[0]["opt_idx"])
    np.testing.assert_array_equal(c["edges"], graph.edges[:E])
    np.testing.assert_allclose(c["meas"], graph.meas[:E], atol=tsg.POSE_TOL, rtol=0)
    np.testing.assert_allclose(c["weight"], graph.weight[:E], atol=tsg.SCALE_TOL, rtol=0)
    np.testing.assert_allclose(c["nodes"], pgos[0]["nodes"], atol=1.7e-3, rtol=0)
    # the PGO on the device's own inputs against the sparse oracle
    ref, ref_losses = pgs.optimize(c["nodes"].astype(np.float64), c["edges"], c["meas"].astype(np.float64),
                                   c["weight"].astype(np.float64), c["opt"])
    assert len(ref_losses) == len(c["losses"])
    np.testing.assert_allclose(c["result"], ref, atol=1e-5, rtol=0)
