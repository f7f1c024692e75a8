"""GPU: the Sim(3) pose-graph LM step (csrc/pose_graph.cuh, pose_graph.cu, pose_graph_sparse.cu) against the float64
oracle at every branch of its closed-form algebra and at the sizes SLAM runs it.

  (a) planted residuals (tests/test_pose_graph_fp64_cpu.py CASES: every w_coeffs / sim3_log branch, q_w < 0, a
      quaternion scaled by 1.7, translations of 1e3), read in fp64 through the block-sparse route's last delta, and
      through the dense and group routes' info rows and nodes_out; two-edge graphs reach J_l(r)^-1 of both edges;
  (b) the dense route at num_opt = 1 ... 3657 (order 7 ... 25 599) against the sparse oracle, the sparse route at 3657,
      and a full optimize() at 1000 nodes;
  (c) a group of {3657, 1, 37, 5} optimised nodes plus a graph with no related edge, each with its own damping;
  (d) dmin / dmax that bind, on the dense, group and sparse routes.
"""
import numpy as np
import pytest
import scipy.sparse.linalg as spla
import torch

from oracle import pose_graph_oracle as pg
from oracle import pose_graph_sparse_oracle as pgs
from test_pose_graph import make_graph
from test_pose_graph_fp64_cpu import CASES, F32, U, case_bound, case_weight, one_edge_reference, planted_node, solve_bound

pytestmark = pytest.mark.gpu
IDENT = np.array([0, 0, 0, 0, 0, 0, 1, 1.0])


def _t(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t.to(dtype) if dtype is not None else t).cuda()


def _args(edges, meas, weights):
    return _t(edges), _t(meas, torch.float32), _t(weights, torch.float32)


def _graph(init, opt):
    from vista_slam_b200.pose_graph import PoseGraphOpt
    return PoseGraphOpt(_t(init, torch.float32), torch.tensor(opt))


@pytest.fixture
def sparse_route(monkeypatch):
    """Every PoseGraphOpt built while active takes the block-sparse route; yields the list of plans built."""
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


def _last_delta(plan, m):
    from vista_slam_b200 import _lib
    d = torch.empty(m, dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib().sta_pg_plan_last_delta(plan.h, _lib.ptr(d), _lib.cur_stream()), "last delta")
    return d.cpu().numpy()


def _group_step(problems, dampings, dmin=1e-6, dmax=1e32):
    """One sta_pose_graph_lm_step_group launch over problems [(init, edges, meas, weights, opt)] -> per graph
    (nodes_out, info row)."""
    from vista_slam_b200.pose_graph import _DenseGroup
    gs = [_graph(p[0], p[4]) for p in problems]
    args = [_args(*p[1:4]) for p in problems]
    grp = _DenseGroup(gs, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args], dmin=dmin, dmax=dmax)
    res = grp.step(list(range(len(gs))), dampings)
    info = grp.info.cpu().numpy()
    return [(r[0].cpu().numpy().astype(np.float64), info[k]) for k, r in enumerate(res)]


def _aligned(got, ref):
    """got with each quaternion's sign matched to ref's: q and -q are one rotation, the oracle returns q_w >= 0 and the
    device keeps the sign of q_delta q_X."""
    got = got.copy()
    flip = np.sum(got[:, 3:7] * ref[:, 3:7], axis=1) < 0
    got[flip, 3:7] *= -1
    return got


def _node_bound(ref, eta):
    """Per element of nodes_out: the fp32 rounding of the reference, 16 u for the oracle's own rounding (its quaternion
    comes from a rotation matrix), plus eta (an fp64 error in delta) times the node's sensitivity to delta,
    2 (1 + |t|_inf + s) (Y = Exp(delta) X: t moves by d_tau + d_phi x t + d_sigma t)."""
    sens = 2.0 * (1.0 + np.abs(ref[:, :3]).max(axis=1) + np.abs(ref[:, 7]))
    return F32 * np.abs(ref) + 16 * U * (1.0 + np.abs(ref)) + eta * sens[:, None]


# ------------------------------------------------------------------------------------------------ (a) planted branches
def _one_edge(case):
    X = planted_node(case).astype(np.float64)
    return np.stack([IDENT, X]), np.array([[0, 1]], dtype=np.int64), IDENT[None].copy(), case_weight(case)[None], [1]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_planted_residual_read_in_fp64(case, sparse_route):
    """One edge from a fixed identity node onto X with T = identity, damping 0: the error is X itself and the sparse
    route's delta is -r = -Log(X) in fp64 (J_l(r) r = r).  Bound per element: (e_r + e_solve) ||r||, e_r the case's
    residual bound (test_pose_graph_fp64_cpu.case_bound: kappa(W) (64 u + u / theta^2) + the series truncation and the
    dropped theta^2 terms), e_solve = kappa_2(A) (gamma(22) 7 + 64 u).  For the sigma-series cases this is >= 10x below
    the effect of the s4 term (test_series_bound_notices_a_dropped_term).  Measured on an H100 80GB HBM3: at most
    9.4e-14 ||r|| (the sigma-series cases, the C series truncation) against bounds of 2.0e-13 ||r|| and up."""
    nodes, edges, meas, w, opt = _one_edge(case)
    r_ref, d_ref, l_ref, A = one_edge_reference(case, w[0])
    nr = np.linalg.norm(r_ref)
    bound = (case_bound(r_ref) + solve_bound(A)) * nr
    g = _graph(nodes, opt)
    out, l0, l1, dn, ok = g.lm_step(*_args(edges, meas, w), 0.0)
    assert ok and len(sparse_route) == 1
    d = _last_delta(sparse_route[0], 7)
    err = np.abs(d + r_ref).max()
    print(f"{case[0]}: |delta + r| = {err / nr:.2e} ||r||, bound {bound / nr:.2e} ||r||")
    assert err <= bound, (err, bound)
    if np.linalg.norm(r_ref[3:6]) == 0.0:  # the update then runs sim3_exp's th < 1e-8 branch
        assert np.linalg.norm(d[3:6]) < 1e-8
    lb = np.sum(w[0] * (2 * np.abs(r_ref) * bound + bound ** 2)) + 16 * U * l_ref
    assert abs(l0 - l_ref) <= lb, (l0, l_ref, lb)
    ref_nodes = pg.apply_update(nodes, opt, d_ref)
    got = _aligned(out.cpu().numpy().astype(np.float64), ref_nodes)
    assert np.all(np.abs(got - ref_nodes) <= _node_bound(ref_nodes, bound + 64 * U * nr))


def test_planted_residuals_dense_and_group():
    """The same one-edge graphs through the dense route (one graph each) and the group route (16 + 5 graphs in two
    launches): loss before l0 = r^T W r and |delta| = ||r|| in fp64 from the info rows, nodes_out per element, all
    within the bounds of test_planted_residual_read_in_fp64."""
    probs = [_one_edge(c) for c in CASES]
    refs = [one_edge_reference(c, p[3][0]) for c, p in zip(CASES, probs)]
    dense = []
    for p in probs:
        out, l0, l1, dn, ok = _graph(p[0], p[4]).lm_step(*_args(*p[1:4]), 0.0)
        assert ok
        dense.append((out.cpu().numpy().astype(np.float64), np.array([l0, l1, dn, 1.0])))
    group = _group_step(probs[:16], [0.0] * 16) + _group_step(probs[16:], [0.0] * (len(probs) - 16))
    for case, p, (r_ref, d_ref, l_ref, A), dres, gres in zip(CASES, probs, refs, dense, group):
        nr = np.linalg.norm(r_ref)
        bound = (case_bound(r_ref) + solve_bound(A)) * nr
        lb = np.sum(p[3][0] * (2 * np.abs(r_ref) * bound + bound ** 2)) + 16 * U * l_ref
        ref_nodes = pg.apply_update(p[0], p[4], d_ref)
        for route, (got, info) in (("dense", dres), ("group", gres)):
            assert info[3] == 1.0, (case[0], route)
            assert abs(info[0] - l_ref) <= lb, (case[0], route, info[0], l_ref, lb)
            assert abs(info[2] - nr) <= np.sqrt(7) * bound, (case[0], route, info[2], nr)
            got = _aligned(got, ref_nodes)
            assert np.all(np.abs(got - ref_nodes) <= _node_bound(ref_nodes, bound + 64 * U * nr)), (case[0], route)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_two_edges_reach_the_jacobian(case, sparse_route):
    """Fixed nodes I and Y, optimised node X; edges (I, X) with T = identity (residual: the planted case) and (Y, X) with a
    generic residual rho (theta 0.6, sigma 0.2), weights 1 and 0.3..2.7.  delta = -A^-1 g depends on J_l(r)^-1 of both
    edges.  Against the oracle's np.linalg.solve, normwise (first order):
      ||d - d_ref|| <= kappa_2(A) (2 e_J + gamma(22) 7 + 64 u) ||d_ref|| + ||A^-1|| ||dg||,
      e_J = kappa(J_l(r_e)) (64 u + e_r ||r_e||)  (relative error of J_e),
      ||dg|| <= sum_e ||J_e|| w_max (e_J + e_r) ||r_e||."""
    X = planted_node(case).astype(np.float64)
    rng = np.random.default_rng(7)
    Y = pg.sim3_exp(rng.normal(size=7) * 0.5).astype(np.float32).astype(np.float64)
    rho = np.concatenate([[0.3, -0.2, 0.1], 0.6 * np.array([0.0, 0.6, 0.8]), [0.2]])
    T2 = pg.sim3_mul(pg.sim3_mul(pg.sim3_exp(rho), pg.sim3_inv(X)), Y).astype(np.float32).astype(np.float64)
    nodes = np.stack([IDENT, Y, X])
    edges = np.array([[0, 2], [1, 2]], dtype=np.int64)
    meas = np.stack([IDENT, T2])
    w = np.stack([case_weight(case), np.linspace(0.3, 2.7, 7)]).astype(np.float32).astype(np.float64)
    A, g, _ = pg.build_normal_equations(nodes, edges, meas, w, [2])
    d_ref = -np.linalg.solve(A, g)
    dg, eJmax = 0.0, 0.0
    for e in range(2):
        r, _, J = pg.edge_jacobians(meas[e], nodes[edges[e, 0]], nodes[edges[e, 1]])
        er = case_bound(r)
        eJ = np.linalg.cond(pg.sim3_jl(r)) * (64 * U + er * np.linalg.norm(r))
        dg += np.linalg.norm(J, 2) * w[e].max() * (eJ + er) * np.linalg.norm(r)
        eJmax = max(eJmax, eJ)
    kap = np.linalg.cond(A)
    bound = kap * (2 * eJmax + (22 * U) * 7 + 64 * U) * np.linalg.norm(d_ref) + np.linalg.norm(np.linalg.inv(A), 2) * dg
    gr = _graph(nodes, [2])
    _, _, _, _, ok = gr.lm_step(*_args(edges, meas, w), 0.0)
    assert ok
    d = _last_delta(sparse_route[0], 7)
    err = np.linalg.norm(d - d_ref)
    print(f"{case[0]}: |d - d_ref| = {err / np.linalg.norm(d_ref):.2e} ||d_ref||, bound {bound / np.linalg.norm(d_ref):.2e}")
    assert err <= bound, (err, bound)


# ------------------------------------------------------------------------------------------------ (b) production sizes
def production_graph(n_opt, seed):
    """A planted trajectory of n_opt + 1 nodes (node 0 fixed): odometry (i+1, i), skips (i+2, i), n_opt // 3 random
    loop closures and a closure onto node 0 from every 10th node, measurements with noise 0.01, initial guess with
    noise 0.02, weights 0.5..1.5.  Short steps (translation 0.02, scale 0.005 per step) keep the translations near 1 at
    3657 nodes and the closures onto the fixed node tie the chain down: kappa_1(A) stays near 1e4 where a 0.3 step
    gives 1e7.  fp32-rounded inputs in float64."""
    rng = np.random.default_rng(seed)
    n = n_opt + 1
    gt = [IDENT.copy()]
    for _ in range(n - 1):
        xi = np.concatenate([rng.normal(size=3) * 0.02, rng.normal(size=3) * 0.1, rng.normal(size=1) * 0.005])
        gt.append(pg.sim3_mul(gt[-1], pg.sim3_exp(xi)))
    edges = [(i + 1, i) for i in range(n - 1)] + [(i + 2, i) for i in range(n - 2)]
    for _ in range(max(1, n_opt // 3)):
        i, j = sorted(rng.choice(n, size=2, replace=False))
        edges.append((int(j), int(i)))
    edges += [(v, 0) for v in range(10, n, 10)]
    edges = np.array(edges, dtype=np.int64)
    meas = np.array([pg.sim3_mul(pg.sim3_exp(rng.normal(size=7) * 0.01), pg.sim3_mul(pg.sim3_inv(gt[j]), gt[i]))
                     for i, j in edges])
    weights = 0.5 + rng.random((len(edges), 7))
    init = np.array([gt[0]] + [pg.sim3_mul(pg.sim3_exp(rng.normal(size=7) * 0.02), gt[v]) for v in range(1, n)])
    r32 = lambda a: a.astype(np.float32).astype(np.float64)
    return r32(init), edges, r32(meas), r32(weights), list(range(1, n))


def oracle_step(init, edges, meas, weights, opt, damping, dmin=1e-6, dmax=1e32):
    """pose_graph_sparse_oracle.lm_step, keeping what the bounds need: the LU factor's 1-norm condition estimate
    (scipy.sparse.linalg.onenormest of A^-1 through the factor; A symmetric, so ||.||_2 <= ||.||_1), ||A||_1, ||g||,
    the smallest residual rotation angle and the largest translation."""
    A, g, l0 = pgs.build_normal_equations(init, edges, meas, weights, opt)
    Ad = pgs.damp(A, damping, dmin, dmax)
    lu = spla.splu(Ad, permc_spec="MMD_AT_PLUS_A", diag_pivot_thresh=0.0, options={"SymmetricMode": True})
    assert np.array_equal(lu.perm_r, lu.perm_c) and (lu.U.diagonal() > 0).all()
    d = -lu.solve(g)
    nodes = pg.apply_update(init, opt, d)
    inv = spla.LinearOperator(Ad.shape, matvec=lu.solve, rmatvec=lu.solve, dtype=np.float64)
    rel = pg.related_edges(edges, opt)
    th = [np.linalg.norm(pg.edge_residual(meas[e], init[edges[e, 0]], init[edges[e, 1]])[3:6]) for e in np.nonzero(rel)[0]]
    return dict(nodes=nodes, l0=l0, l1=pg.graph_loss(nodes, edges, meas, weights, opt), d=d, g=g, m=Ad.shape[0],
                A1=spla.norm(Ad, 1), Ainv1=spla.onenormest(inv), theta=min(th) if th else np.inf,
                wsum=float(weights[rel].sum()), tmax=float(np.abs(init[:, :3]).max()), E=int(rel.sum()), diag=A.diagonal())


def check_step(ref, out, l0, l1, dn, what):
    """The device's step against oracle_step's.  eps = 64 u + u / theta_min^2 + 1.4e-13 (test_solver_backward_error's
    model of the closed-form residuals and Jacobians against the oracle's expm).
      l0:  |l0 - l0_ref| <= (2 eps + 7 E u) l0_ref                         (r^T W r, E related edges summed)
      |d|: |dn - ||d_ref||| <= ||A^-1|| ((gamma(3m+1) m + eps) ||A|| ||d|| + eps ||g||)   (Higham Thm 10.4/10.5)
      nodes_out: fp32 rounding of the reference + eta (1 + |t| + s) 2, eta the same forward bound with Higham's
           worst-case gamma(3m+1) m replaced by the probabilistic 16 sqrt(3m+1) u (Higham & Mary 2019), plus eps |d|
      l1:  evaluated at fp32-rounded nodes: residual components move by rho = 4 (2^-24 + eta) (1 + 2 t_max), so
           |l1 - l1_ref| <= 2 sqrt(l1_ref W) rho + W rho^2 + (2 eps + 7 E u) l1_ref,  W = sum of the related weights.
    Returns the observed / bound ratios."""
    m, d = ref["m"], ref["d"]
    th = ref["theta"]
    eps = 64 * U + (U / th ** 2 if th >= 1e-4 else 1e-12) + 1.4e-13
    nd = np.linalg.norm(d)
    gam = (3 * m + 1) * U / (1 - (3 * m + 1) * U)
    fwd = ref["Ainv1"] * ((gam * m + eps) * ref["A1"] * nd + eps * np.linalg.norm(ref["g"]))
    eta = ref["Ainv1"] * ((16 * np.sqrt(3 * m + 1) * U + eps) * ref["A1"] * nd + eps * np.linalg.norm(ref["g"])) + eps * nd
    red = 7 * ref["E"] * U
    b_l0 = (2 * eps + red) * ref["l0"]
    rho = 4 * (F32 + eta) * (1 + 2 * ref["tmax"])
    b_l1 = 2 * np.sqrt(ref["l1"] * ref["wsum"]) * rho + ref["wsum"] * rho ** 2 + (2 * eps + red) * ref["l1"]
    got = _aligned(out.cpu().numpy().astype(np.float64) if torch.is_tensor(out) else out, ref["nodes"])
    nb = _node_bound(ref["nodes"], eta)
    ratios = dict(l0=abs(l0 - ref["l0"]) / b_l0 if b_l0 else float(l0 != ref["l0"]),
                  l1=abs(l1 - ref["l1"]) / b_l1 if b_l1 else float(l1 != ref["l1"]),
                  dn=abs(dn - nd) / fwd if fwd else float(dn != nd),
                  nodes=float((np.abs(got - ref["nodes"]) / nb).max()))
    print(what, {k: f"{v:.2e}" for k, v in ratios.items()}, f"kappa_1 ~ {ref['A1'] * ref['Ainv1']:.1e}")
    assert all(v <= 1.0 for v in ratios.values()), (what, ratios)
    return ratios


SIZES = [1, 4, 5, 9, 10, 147, 1000, 3657]
_CACHE = {}


def production(n_opt, damping=1e-4):
    """production_graph(n_opt) and its oracle step, computed once per module."""
    key = (n_opt, damping)
    if key not in _CACHE:
        p = production_graph(n_opt, seed=n_opt)
        _CACHE[key] = (p, oracle_step(*p, damping))
    return _CACHE[key]


@pytest.mark.parametrize("n_opt", SIZES)
def test_dense_route_at_production_sizes(n_opt):
    """One dense LM step (damping 1e-4) at orders 7 n_opt = 7 ... 25 599 (straddling multiples of the 32-wide panels;
    at 3657 the solve holds 204 792 bytes of right-hand side in its 204 800-byte budget) against the sparse oracle,
    bounds of check_step."""
    import time
    (init, edges, meas, weights, opt), ref = production(n_opt)
    g = _graph(init, opt)
    assert not g.sparse
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out, l0, l1, dn, ok = g.lm_step(*_args(edges, meas, weights), 1e-4)
    print(f"dense step at {n_opt} optimised nodes: {1e3 * (time.perf_counter() - t0):.1f} ms (incl. first launches)")
    assert ok
    check_step(ref, out, l0, l1, dn, f"dense {n_opt}")
    if n_opt == 3657:  # the block-sparse route on the same inputs: the same nodes within 2 fp32 ulps
        from vista_slam_b200 import _lib
        _lib.PG_DENSE_MAX_OPT, keep = 0, _lib.PG_DENSE_MAX_OPT
        try:
            s = _graph(init, opt)
        finally:
            _lib.PG_DENSE_MAX_OPT = keep
        assert s.sparse
        out_s, s0, s1, sn, ok_s = s.lm_step(*_args(edges, meas, weights), 1e-4)
        assert ok_s and s0 == l0
        check_step(ref, out_s, s0, s1, sn, "sparse 3657")
        a, b = out.cpu().numpy(), out_s.cpu().numpy()
        assert np.all(np.abs(a - b) <= 2 * np.spacing(np.maximum(np.abs(a), np.abs(b)))), np.abs(a - b).max()


def test_optimize_at_1000_nodes_against_the_oracle_history():
    """PoseGraphOpt.optimize (LM with trust region and plateau stop) at 1000 optimised nodes against
    pose_graph_sparse_oracle.optimize: the same number of iterations, the first loss within check_step's l0 bound, and
    every later loss within its l1 bound.  The device rounds each accepted iterate to fp32 and the next steps contract
    that perturbation (by at least 1/2 per step here), so rho is twice one rounding's."""
    (init, edges, meas, weights, opt), ref = production(1000)
    g = _graph(init, opt)
    losses = g.optimize(*_args(edges, meas, weights))
    _, ref_losses = pgs.optimize(init, edges, meas, weights, opt)
    assert len(losses) == len(ref_losses), (losses, ref_losses)
    rho = 2 * 4 * F32 * (1 + 2 * ref["tmax"])
    for k, (a, b) in enumerate(zip(losses, ref_losses)):
        lb = 2 * np.sqrt(b * ref["wsum"]) * rho + ref["wsum"] * rho ** 2 + 1e-10 * b
        assert abs(a - b) <= lb, (k, a, b, lb)


# ------------------------------------------------------------------------------------------------ (c) mixed group
def _no_related_edge_graph():
    """Six nodes, edges among the first five only, the sixth (isolated) optimised: no related edge, A = 0 clamped to
    dmin, g = 0, delta = 0, both losses 0."""
    _, init, edges, meas, weights = make_graph(np.random.default_rng(3), n_nodes=5, n_loops=1, noise=0.05,
                                               meas_noise=0.01)
    init = np.concatenate([init, pg.sim3_exp(np.full(7, 0.1))[None]])
    r32 = lambda a: a.astype(np.float32).astype(np.float64)
    return r32(init), edges, r32(meas), r32(weights), [5]


def test_group_of_mixed_sizes_against_the_oracle():
    """One group launch over {3657, 1, 37, 5} optimised nodes and the graph with no related edge, dampings 1e-4, 0.3,
    2.0, 1e-2, 0.5: every info row and nodes_out against the oracle (check_step), not only against the solo step.  The
    panel loop runs to order 25 599 while the small graphs return at their own order."""
    probs = [production(3657)[0], production_graph(1, 11), production_graph(37, 12), production_graph(5, 13),
             _no_related_edge_graph()]
    damp = [1e-4, 0.3, 2.0, 1e-2, 0.5]
    res = _group_step(probs, damp)
    for k, (p, dk, (out, info)) in enumerate(zip(probs, damp, res)):
        ref = production(3657)[1] if k == 0 else oracle_step(*p, dk)
        assert info[3] == 1.0
        check_step(ref, out, info[0], info[1], info[2], f"group member {k} ({len(p[4])} optimised)")
    out, info = res[4]
    assert info[0] == info[1] == info[2] == 0.0 and np.array_equal(out[:5], probs[4][0][:5])


# ------------------------------------------------------------------------------------------------ (d) damping clamp
def test_binding_diagonal_clamp_on_every_route(sparse_route, monkeypatch):
    """dmin = 1, dmax = 10 with weights 0.29 x 10^-3 .. 10^0.5, so that both bounds clamp diagonal entries of A (and
    dmin alone sets the isolated node's), damping 1: dense, group and sparse against the oracle's damp (clamp, then
    scale by 1 + damping), bounds of check_step; the sparse route's delta as well.  The largest diagonal entry stays
    below 2 dmax, so the damped diagonal is at least A's and the system stays definite (clamping entries far above
    dmax makes it indefinite)."""
    from vista_slam_b200 import _lib
    rng = np.random.default_rng(17)
    _, init, edges, meas, weights = make_graph(rng, n_nodes=40, n_loops=10, noise=0.05, meas_noise=0.02)
    weights = 0.29 * 10.0 ** rng.uniform(-3.0, 0.5, size=weights.shape)
    init = np.concatenate([init, pg.sim3_exp(np.full(7, 0.2))[None]])  # node 40: optimised, no edge
    r32 = lambda a: a.astype(np.float32).astype(np.float64)
    p = (r32(init), edges, r32(meas), r32(weights), list(range(1, 41)))
    ref = oracle_step(*p, 1.0, dmin=1.0, dmax=10.0)
    assert (ref["diag"] < 1.0).sum() > 7 and (ref["diag"] > 10.0).sum() > 7 and ref["diag"].max() < 20.0  # both bounds bind, not only the lone node
    monkeypatch.setattr(_lib, "PG_DENSE_MAX_OPT", 3657)
    dense = _graph(p[0], p[4])
    assert not dense.sparse
    out, l0, l1, dn, ok = dense.lm_step(*_args(*p[1:4]), 1.0, dmin=1.0, dmax=10.0)
    assert ok
    check_step(ref, out, l0, l1, dn, "dense clamp")
    other = production_graph(9, 21)
    (out_g, info), _ = _group_step([p, other], [1.0, 1e-4], dmin=1.0, dmax=10.0)
    check_step(ref, out_g, info[0], info[1], info[2], "group clamp")
    monkeypatch.setattr(_lib, "PG_DENSE_MAX_OPT", 0)
    s = _graph(p[0], p[4])
    assert s.sparse
    out_s, s0, s1, sn, ok_s = s.lm_step(*_args(*p[1:4]), 1.0, dmin=1.0, dmax=10.0)
    assert ok_s
    check_step(ref, out_s, s0, s1, sn, "sparse clamp")
    d = _last_delta(sparse_route[-1], ref["m"])
    m, th = ref["m"], ref["theta"]
    eps = 64 * U + U / th ** 2 + 1.4e-13
    gam = (3 * m + 1) * U / (1 - (3 * m + 1) * U)
    fwd = ref["Ainv1"] * ((gam * m + eps) * ref["A1"] * np.linalg.norm(ref["d"]) + eps * np.linalg.norm(ref["g"]))
    assert np.linalg.norm(d - ref["d"]) <= fwd
    # the isolated node: delta = 0 exactly, its pose copied through Exp(0)
    assert np.all(d[-7:] == 0.0)
