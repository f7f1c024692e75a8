"""Drop-in vista_slam/eval/eval_traj.py: Sim(3) alignment of an estimated trajectory and its APE, as evo computes them,
without evo or matplotlib.

A few hundred poses at most, so this stays host numpy float64.  In place of evo trajectory objects the aligned estimate
and the reference come back as float64 [n, 4, 4] arrays.  `full_traj_eval` / `traj_eval_and_plot` create
`plot_parent_dir` as the reference does but draw no plot."""
import os

import numpy as np

APE_KEYS = ("rmse", "mean", "median", "std", "min", "max", "sse")


def _umeyama_sim3(x, y):
    """evo's umeyama_alignment with scale: x, y [3, n] -> (R, t, c) minimising |y - (c R x + t)|."""
    m, n = x.shape
    mx, my = x.mean(axis=1), y.mean(axis=1)
    sigma_x = 1.0 / n * (np.linalg.norm(x - mx[:, None]) ** 2)
    outer = np.zeros((m, m))
    for i in range(n):
        outer += np.outer(y[:, i] - my, x[:, i] - mx)
    cov = np.multiply(1.0 / n, outer)
    u, d, v = np.linalg.svd(cov)
    if np.count_nonzero(d > np.finfo(d.dtype).eps) < m - 1:
        raise ValueError("Degenerate covariance rank, Umeyama alignment is not possible")
    s = np.eye(m)
    if np.linalg.det(u) * np.linalg.det(v) < 0.0:
        s[m - 1, m - 1] = -1
    r = u.dot(s).dot(v)
    c = 1 / sigma_x * np.trace(np.diag(d).dot(s))
    t = my - np.multiply(c, r.dot(mx))
    return r, t, c


def _as_pose(p):
    if hasattr(p, "detach"):
        p = p.detach().cpu().numpy()
    return np.asarray(p, np.float64)


def align_traj(traj_est_all, traj_ref_all):
    """traj_est_all, traj_ref_all: sequences of [4, 4] poses (numpy arrays or tensors).  Poses whose reference sum is not
    finite are skipped.  Returns (r_a [3,3], t_a [3], s, aligned estimate [n,4,4], reference [n,4,4]): the estimate's
    positions are aligned to the reference's with a Sim(3) Umeyama fit, and the aligned poses are [r_a | t_a] [R | s t]."""
    est, ref = [], []
    for i in range(len(traj_ref_all)):
        val = traj_ref_all[i].sum()
        if np.isnan(float(val)) or np.isinf(float(val)):
            print(f"Nan or Inf found in gt poses, skipping {i}th pose!")
            continue
        est.append(_as_pose(traj_est_all[i]))
        ref.append(_as_pose(traj_ref_all[i]))
    est, ref = np.stack(est), np.stack(ref)
    r_a, t_a, s = _umeyama_sim3(est[:, :3, 3].T, ref[:, :3, 3].T)
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = r_a, t_a
    scaled = est.copy()
    scaled[:, :3, 3] *= s
    return r_a, t_a, s, np.stack([T.dot(p) for p in scaled]), ref


def traj_eval_and_plot(traj_est, traj_ref, plot_parent_dir, plot_name):
    """APE of the translation part: {rmse, mean, median, std, min, max, sse} of |t_est - t_ref|.  No plot is drawn."""
    if not os.path.exists(plot_parent_dir):
        os.makedirs(plot_parent_dir)
    est, ref = np.asarray(traj_est, np.float64), np.asarray(traj_ref, np.float64)
    e = np.linalg.norm(ref[:, :3, 3] - est[:, :3, 3], axis=1)
    sse = float(np.dot(e, e))
    return {"rmse": float(np.sqrt(sse / len(e))), "mean": float(np.mean(e)), "median": float(np.median(e)),
            "std": float(np.std(e)), "min": float(np.min(e)), "max": float(np.max(e)), "sse": sse}


def full_traj_eval(traj_est, traj_ref, plot_parent_dir, plot_name):
    """-> (aligned estimate [n,4,4], reference [n,4,4], r_a, t_a, s, APE statistics)."""
    r_a, t_a, s, traj_est, traj_ref = align_traj(traj_est, traj_ref)
    if not os.path.exists(plot_parent_dir):
        os.makedirs(plot_parent_dir)
    ape_statistics = traj_eval_and_plot(traj_est, traj_ref, plot_parent_dir, plot_name)
    return traj_est, traj_ref, r_a, t_a, s, ape_statistics
