"""ORACLE -- test infrastructure, not product code (only tests/ and tools/ may import it).

Sparse restatement of the Levenberg-Marquardt step of oracle/pose_graph_oracle.py, for graphs where the dense numpy
normal equations (7 n_opt square) are too slow or too large: the same per-edge residuals and Jacobians
(pose_graph_oracle.edge_jacobians), A = J^T W J assembled as a scipy.sparse matrix, the same damping, and the solve by
scipy.sparse.linalg (a sparse LU with symmetric, diagonal pivoting, which for a symmetric matrix is its LDL^T
factorisation: every pivot is positive exactly when the matrix is positive definite, so an indefinite system raises
numpy.linalg.LinAlgError as np.linalg.cholesky does in the dense oracle).  The update, the losses and the optimize loop
are those of the dense oracle.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import pose_graph_oracle as pg
from oracle import slam_oracle as so

_II, _JJ = np.meshgrid(np.arange(7), np.arange(7), indexing="ij")


def build_normal_equations(nodes, edges, meas, weights, opt_idx):
    """(A as scipy.sparse CSC, g, loss) -- the sparse twin of pose_graph_oracle.build_normal_equations."""
    opt_map = pg.split_nodes(len(nodes), opt_idx)
    n = len(opt_idx)
    rows, cols, vals = [], [], []
    g = np.zeros(7 * n)
    loss = 0.0
    for e in np.nonzero(pg.related_edges(edges, opt_idx))[0]:
        i, j = int(edges[e, 0]), int(edges[e, 1])
        r, Ji, Jj = pg.edge_jacobians(meas[e], nodes[i], nodes[j])
        W = np.diag(weights[e])
        loss += float(r @ W @ r)
        blocks = [(opt_map[i], Ji), (opt_map[j], Jj)]
        for a, Ja in blocks:
            if a < 0:
                continue
            g[7 * a:7 * a + 7] += Ja.T @ W @ r
            for b, Jb in blocks:
                if b < 0:
                    continue
                rows.append(7 * a + _II.ravel())
                cols.append(7 * b + _JJ.ravel())
                vals.append((Ja.T @ W @ Jb).ravel())
    if rows:
        rows, cols, vals = np.concatenate(rows), np.concatenate(cols), np.concatenate(vals)
    A = sp.coo_matrix((vals, (rows, cols)), shape=(7 * n, 7 * n)).tocsc()  # duplicates are summed
    return A, g, loss


def damp(A, damping, dmin=1e-6, dmax=1e32):
    """pp.optim.LM.step's damping: diagonal clamped to [dmin, dmax], then scaled by 1 + damping."""
    d = np.clip(A.diagonal(), dmin, dmax) * (1.0 + damping)
    return (A - sp.diags(A.diagonal()) + sp.diags(d)).tocsc()


def spd_solve(A, b):
    """x = A^-1 b for a symmetric positive definite sparse A; LinAlgError if A is not positive definite."""
    lu = spla.splu(A, permc_spec="MMD_AT_PLUS_A", diag_pivot_thresh=0.0, options={"SymmetricMode": True})
    if not (np.array_equal(lu.perm_r, lu.perm_c) and (lu.U.diagonal() > 0).all()):
        raise np.linalg.LinAlgError("Matrix is not positive definite")
    return lu.solve(b)


def lm_step(nodes, edges, meas, weights, opt_idx, damping, dmin=1e-6, dmax=1e32):
    """pose_graph_oracle.lm_step with the sparse normal equations and solve.  Returns (new_nodes, loss_before,
    loss_after, delta)."""
    A, g, loss0 = build_normal_equations(nodes, edges, meas, weights, opt_idx)
    delta = -spd_solve(damp(A, damping, dmin, dmax), g)
    new_nodes = pg.apply_update(nodes, opt_idx, delta)
    return new_nodes, loss0, pg.graph_loss(new_nodes, edges, meas, weights, opt_idx), delta


def optimize(nodes, edges, meas, weights, opt_idx, steps=20, patience=3, decreasing=1e-4, radius=1e4):
    """pose_graph_oracle.optimize (same trust-region and plateau rules) over the sparse lm_step."""
    losses = []
    stall = 0
    for _ in range(steps):
        new_nodes, l0, l1, delta = lm_step(nodes, edges, meas, weights, opt_idx, 1.0 / radius)
        if l1 <= l0:
            nodes = new_nodes
            radius = min(radius * 2.0, 1e32)
        else:
            radius = max(radius * 0.5, 1e-32)
            l1 = l0
        losses.append(l1)
        stall = stall + 1 if (l0 - l1) < decreasing else 0
        if stall >= patience:
            break
    return nodes, losses


def _pgo(graph, opt_idx):
    """slam_oracle.pgo with the sparse optimize."""
    E, N = graph.num_edges, graph.num_nodes
    edges = graph.edges[:E]
    related = pg.related_edges(edges, opt_idx)
    out, _ = optimize(graph.pose[:N].astype(np.float64), edges, graph.meas[:E].astype(np.float64),
                      graph.weight[:E].astype(np.float64), opt_idx)
    graph.pose[:N] = out.astype(np.float32)
    return related


def run(stream, **kw):
    """slam_oracle.run with every PGO solved by the sparse oracle (same arguments and results): for runs whose PGO is
    too large for the dense numpy normal equations."""
    dense = so.pgo
    so.pgo = _pgo
    try:
        return so.run(stream, **kw)
    finally:
        so.pgo = dense
