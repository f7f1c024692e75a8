"""CPU companion of tests/test_pose_graph_fp64_gpu.py: the planted Sim(3) residuals that steer the LM step's closed-form
algebra (csrc/pose_graph.cuh) through each of its branches, their error bounds, and the oracle pinned at those cases.

  * A numpy mirror of w_coeffs / w_matrix / sim3_log (statement for statement, same branch tests) names the branches
    each planted residual reaches; the test asserts them, so the case list cannot drift away from the branches it is
    meant to cover.
  * The oracle (oracle/pose_graph_oracle.py, which evaluates W and J_l as matrix exponentials) is pinned at every case
    against scipy.linalg.expm of the 4x4 generator and by J_l(r) r = r.
  * The bound of each case (case_bound) is checked on the mirror, and for the sigma-series cases it is shown to be at
    least 10x below the effect of the smallest series term the kernel keeps, so a dropped term is noticed.
"""
import numpy as np
import pytest
from scipy.linalg import expm

from oracle import pose_graph_oracle as pg

U = np.finfo(np.float64).eps / 2
F32 = np.finfo(np.float32).eps / 2  # fp32 unit roundoff (2^-24)

# name, sigma, theta, tau (residual translation), rotation axis, modifier of the stored quaternion, and the branches the
# kernel takes (checked by test_cases_reach_their_branches on the mirror):
#   C: "series" (|sigma| < 1e-2) or "expm1";  AB: "small-theta series", "small-theta closed" (theta < 1e-4) or "closed";
#   log: "n<1e-12" (theta = 0 exactly) or "atan2";  flip: the stored q_w < 0
# sigma-series cases sit at theta = 0 exactly or theta >= 0.1, clear of the u / theta^2 cancellation of the closed forms
_T = np.array([0.4, -0.3, 0.5])
_AX = np.array([0.48, -0.6, 0.64])  # unit
CASES = [
    ("s+0.0099_t0", 0.0099, 0.0, _T, _AX, None, ("series", "small-theta series", "n<1e-12", False)),
    ("s-0.0099_t0", -0.0099, 0.0, _T, _AX, None, ("series", "small-theta series", "n<1e-12", False)),
    ("s+0.0099_t0.5", 0.0099, 0.5, _T, _AX, None, ("series", "closed", "atan2", False)),
    ("s-0.0099_t1", -0.0099, 1.0, _T, _AX, None, ("series", "closed", "atan2", False)),
    ("s+0.0101_t0", 0.0101, 0.0, _T, _AX, None, ("expm1", "small-theta closed", "n<1e-12", False)),
    ("s-0.0101_t0.3", -0.0101, 0.3, _T, _AX, None, ("expm1", "closed", "atan2", False)),
    ("s0_t0", 0.0, 0.0, _T, _AX, None, ("series", "small-theta series", "n<1e-12", False)),
    ("s0_t1", 0.0, 1.0, _T, _AX, None, ("series", "closed", "atan2", False)),
    ("s+2.5_t0", 2.5, 0.0, _T, _AX, None, ("expm1", "small-theta closed", "n<1e-12", False)),
    ("s-2.5_t3", -2.5, 3.0, _T, _AX, None, ("expm1", "closed", "atan2", False)),
    ("s+2.5_tpi", 2.5, np.pi - 1e-3, _T, _AX, None, ("expm1", "closed", "atan2", False)),
    ("t5e-5_s+0.0099", 0.0099, 5e-5, _T, _AX, None, ("series", "small-theta series", "atan2", False)),
    ("t5e-5_s+2.5", 2.5, 5e-5, _T, _AX, None, ("expm1", "small-theta closed", "atan2", False)),
    ("t2e-4_s0", 0.0, 2e-4, _T, _AX, None, ("series", "closed", "atan2", False)),
    ("t2e-4_s-0.3", -0.3, 2e-4, _T, _AX, None, ("expm1", "closed", "atan2", False)),
    ("t1_s0.2", 0.2, 1.0, _T, _AX, None, ("expm1", "closed", "atan2", False)),
    ("tpi_s0", 0.0, np.pi - 1e-3, _T, _AX, None, ("series", "closed", "atan2", False)),
    ("qw<0", 0.1, 2.0, _T, _AX, "flip", ("expm1", "closed", "atan2", True)),
    ("q*1.7", -0.3, 0.7, _T, _AX, "x1.7", ("expm1", "closed", "atan2", False)),
    ("q*1.7_qw<0_t0", 0.05, 0.0, _T, _AX, "flip x1.7", ("expm1", "small-theta closed", "n<1e-12", True)),
    ("tau1e3", 0.05, 0.4, np.array([1e3, -7e2, 4e2]), _AX, None, ("expm1", "closed", "atan2", False)),
]
SERIES = [c for c in CASES if c[6][0] == "series" and c[1] != 0.0]


def case_weight(case):
    """Edge weight of the one-edge graph (fp32 values, as the device reads them): 1, except at tau = 1e3, where
    weighting tau by 1e-4 keeps the 7x7 normal matrix near kappa 2e7 (unit weights: 2e11) and its diagonal above the LM
    clamp's dmin = 1e-6 (a weight of 1e-6 puts it at 9.6e-7, where the clamp changes the system)."""
    w = np.array([1e-4] * 3 + [1.0] * 4) if case[0] == "tau1e3" else np.ones(7)
    return w.astype(np.float32).astype(np.float64)


# ------------------------------------------------------------------------------- mirror of csrc/pose_graph.cuh
def w_coeffs(sigma, theta):
    """pose_graph.cuh w_coeffs, statement for statement; also returns the branch names (C, AB)."""
    es = np.exp(sigma)
    small_s = abs(sigma) < 1e-2
    s1 = sigma
    s2 = s1 * s1
    s3 = s2 * s1
    s4 = s2 * s2
    C = 1.0 + s1 / 2 + s2 / 6 + s3 / 24 + s4 / 120 if small_s else np.expm1(sigma) / sigma
    if theta < 1e-4:
        if small_s:
            A = 0.5 + s1 / 3 + s2 / 8 + s3 / 30 + s4 / 144
            B = 1.0 / 6 + s1 / 8 + s2 / 20 + s3 / 72 + s4 / 336
            ab = "small-theta series"
        else:
            A = (es * (sigma - 1.0) + 1.0) / s2
            B = (es * (s2 - 2.0 * sigma + 2.0) - 2.0) / (2.0 * s3)
            ab = "small-theta closed"
    else:
        den, sn, cs = s2 + theta * theta, np.sin(theta), np.cos(theta)
        A = (es * (sigma * sn - theta * cs) + theta) / (theta * den)
        B = (C - (es * (sigma * cs + theta * sn) - sigma) / den) / (theta * theta)
        ab = "closed"
    return C, A, B, ("series" if small_s else "expm1", ab)


def w_matrix(phi, sigma, coeffs=w_coeffs):
    th = np.sqrt(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2])
    C, A, B, br = coeffs(sigma, th)
    return C * np.eye(3) + A * pg.hat(phi) + B * (np.outer(phi, phi) - th * th * np.eye(3)), br


def sim3_load(p32):
    """pose_graph.cuh sim3_load: fp32 data in fp64, quaternion renormalised."""
    p = np.asarray(p32, dtype=np.float32).astype(np.float64)
    q = p[3:7] / np.sqrt(np.sum(p[3:7] * p[3:7]))
    return p[:3], q, p[7]


def sim3_log(t, q, s, coeffs=w_coeffs):
    """pose_graph.cuh sim3_log (the 3x3 cofactor inverse replaced by a solve); returns (xi, branch names)."""
    flip = bool(q[3] < 0)
    if flip:
        q = -q
    n = np.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2])
    k = 2.0 if n < 1e-12 else 2.0 * np.arctan2(n, q[3]) / n
    phi, sigma = k * q[:3], np.log(s)
    W, (cb, ab) = w_matrix(phi, sigma, coeffs)
    return np.concatenate([np.linalg.solve(W, t), phi, [sigma]]), (cb, ab, "n<1e-12" if n < 1e-12 else "atan2", flip)


def w_coeffs_without_s4(sigma, theta):
    """w_coeffs with the s4 term of the C series dropped: the defect the sigma-series cases must catch."""
    C, A, B, br = w_coeffs(sigma, theta)
    if abs(sigma) < 1e-2:
        C -= sigma ** 4 / 120
    return C, A, B, br


# ------------------------------------------------------------------------------- planted inputs and their bounds
def planted_xi(case):
    _, sigma, theta, tau, axis, _, _ = case
    return np.concatenate([tau, theta * axis, [sigma]])


def planted_node(case):
    """The stored (fp32) Sim(3) node whose Log is the case's residual: oracle Exp of the planted tangent, then the case's
    modifier of the stored quaternion (sign flip, scale by 1.7; both leave the rotation unchanged)."""
    X = pg.sim3_exp(planted_xi(case))
    mod = case[5] or ""
    if "flip" in mod:
        X[3:7] = -X[3:7]
    if "x1.7" in mod:
        X[3:7] *= 1.7
    return X.astype(np.float32)


def oracle_w(r):
    aug = np.zeros((6, 6))
    aug[:3, :3] = r[6] * np.eye(3) + pg.hat(r[3:6])
    aug[:3, 3:] = np.eye(3)
    return expm(aug)[:3, 3:]


def case_bound(r):
    """Relative bound e_r on the kernel's residual r = Log(X) against the oracle's, |r_k - r_ref_k| <= e_r ||r_ref||_2,
    from the error model of test_pose_graph_sparse_gpu.py::test_solver_backward_error applied to tau = W^-1 t:
      e_r = kappa(W) (64 u + u / theta^2 [theta >= 1e-4 branch]) + ||W^-1|| (trunc + drop)
      trunc = 1.1 |sigma|^5 / 720 (1 + theta + theta^2)   the first series term left out, below |sigma| = 1e-2
                                                          (tail <= 1.1 x it), on C, A Phi and B Phi^2
      drop  = e^max(sigma, 0) (theta^3 / 24 + theta^4 / 120)   0 < theta < 1e-4: the theta^2 corrections of A and B
                                                          (|sin(u th)/th - u| <= u^3 th^2 / 6, |(1 - cos u th)/th^2 - u^2/2|
                                                          <= u^4 th^2 / 24, integrated against e^(u sigma) over [0, 1])."""
    sigma, th = r[6], np.linalg.norm(r[3:6])
    W = oracle_w(r)
    e = 64 * U + (U / th ** 2 if th >= 1e-4 else 0.0)
    trunc = 1.1 * abs(sigma) ** 5 / 720 * (1 + th + th * th) if abs(sigma) < 1e-2 else 0.0
    drop = np.exp(max(sigma, 0.0)) * (th ** 3 / 24 + th ** 4 / 120) if 0 < th < 1e-4 else 0.0
    return np.linalg.cond(W) * e + np.linalg.norm(np.linalg.inv(W), 2) * (trunc + drop)


def solve_bound(A):
    """Relative forward error of a backward-stable 7x7 Cholesky solve: kappa_2(A) gamma(3m + 1) m, m = 7 (Higham,
    Thm 10.4 / 10.5), plus 64 u kappa_2(A) for the roundings of the kernel's J = J_l^-1 Ad_A that enter A and g."""
    m = A.shape[0]
    gam = (3 * m + 1) * U / (1 - (3 * m + 1) * U)
    return np.linalg.cond(A) * (gam * m + 64 * U)


def one_edge_reference(case, weight):
    """Oracle answers of the one-edge graph [identity (fixed), X (optimised)], edge (0, 1), T = identity:
    (r, delta = -A^-1 g, loss = r^T W r, A)."""
    X = planted_node(case).astype(np.float64)
    I = np.array([0, 0, 0, 0, 0, 0, 1, 1.0])
    nodes = np.stack([I, X])
    edges = np.array([[0, 1]], dtype=np.int64)
    A, g, loss = pg.build_normal_equations(nodes, edges, I[None], weight[None], [1])
    assert np.diag(A).min() > 1e-6  # the LM diagonal clamp does not bind: delta = -r
    return pg.edge_residual(I, I, X), -np.linalg.solve(A, g), loss, A


# ------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_cases_reach_their_branches(case):
    t, q, s = sim3_load(planted_node(case))
    _, br = sim3_log(t, q, s)
    assert br == case[6], (case[0], br)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_pinned_against_expm(case):
    """The oracle's Log at the stored node: expm of its generator is the node's matrix, and J_l(r) r = r."""
    X = planted_node(case).astype(np.float64)
    r = pg.sim3_log(X)
    M = pg.sim3_matrix(X)
    scale = max(1.0, np.abs(M).max())
    assert np.abs(expm(pg.sim3_generator(r)) - M).max() <= 1e-13 * scale * max(1.0, np.linalg.norm(r))
    assert np.abs(r - planted_xi(case)).max() <= 1e-5 * max(1.0, np.linalg.norm(r))  # fp32 storage of the node
    assert np.abs(pg.sim3_jl(r) @ r - r).max() <= 1e-13 * max(1.0, np.linalg.norm(r)) ** 2
    assert np.abs(pg.sim3_matrix(pg.sim3_exp(r)) - M).max() <= 1e-13 * scale * max(1.0, np.linalg.norm(r))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_mirror_within_the_case_bound(case):
    t, q, s = sim3_load(planted_node(case))
    r, _ = sim3_log(t, q, s)
    ref = pg.sim3_log(planted_node(case).astype(np.float64))
    assert np.abs(r - ref).max() <= case_bound(ref) * np.linalg.norm(ref)


@pytest.mark.parametrize("case", SERIES, ids=[c[0] for c in SERIES])
def test_series_bound_notices_a_dropped_term(case):
    """The whole delta bound of the GPU test (residual + 7x7 solve) is at least 10x below what the smallest term kept in
    the C series (sigma^4 / 120) moves tau by; the mirror with that term dropped falls outside it."""
    ref, _, _, A = one_edge_reference(case, case_weight(case))
    bound = (case_bound(ref) + solve_bound(A)) * np.linalg.norm(ref)
    effect = case[1] ** 4 / 120 * np.abs(np.linalg.solve(oracle_w(ref), np.linalg.solve(oracle_w(ref), sim3_load(
        planted_node(case))[0]))).max()  # d tau = -W^-1 dC W^-1 t
    assert 10 * bound <= effect, (bound, effect)
    t, q, s = sim3_load(planted_node(case))
    bad, _ = sim3_log(t, q, s, coeffs=w_coeffs_without_s4)
    assert np.abs(bad - ref).max() > bound
