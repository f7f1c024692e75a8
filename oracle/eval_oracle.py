"""numpy / scipy restatement of the SLAM evaluation (vista_slam/eval/eval_traj.py and eval_recon.py with what they call
in evo, open3d and pykdtree), one function per stage so that each can be fed the GPU's own inputs; plus the seeded
synthetic scene the tests and tools/eval_stream.py evaluate.

The third-party steps are restated from the libraries' published behaviour:
  * evo: PoseTrajectory3D.align(correct_scale=True) = umeyama_alignment with scale, then scale the translations and
    left-multiply [R_a | t_a]; APE translation_part statistics (rmse, mean, median, std, min, max, sse);
  * open3d voxel_down_sample: min_bound = min - v/2, key = floor((p - min_bound) / v), the mean of each voxel's points
    (summed in input order here; open3d's output order is its hash order, this is ascending key order);
  * open3d registration_icp point-to-point: nearest target strictly within the radius, fitness / inlier_rmse, Eigen's
    umeyama without scaling, stop when both changes are below 1e-6, at most 30 iterations;
  * pykdtree: exact nearest-neighbour distances (scipy.spatial.cKDTree here).
Distances are (dx dx + dy dy) + dz dz in float64, as the device computes them."""
import os

import numpy as np
import torch
from scipy.spatial import cKDTree

VOXEL, ICP_DIST, ICP_ITERS, ICP_EPS, MAX_ERROR = 0.05, 0.1, 30, 1e-6, 0.5
INT_MAX = 2 ** 31 - 1


# ------------------------------------------------------------------------------------------------ trajectory
def umeyama(x, y, with_scale):
    """evo.core.geometry.umeyama_alignment: x, y [3, n] -> (R, t, c) minimising |y - (c R x + t)|."""
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
    c = 1 / sigma_x * np.trace(np.diag(d).dot(s)) if with_scale else 1.0
    t = my - np.multiply(c, r.dot(mx))
    return r, t, c


def align_traj(traj_est_all, traj_ref_all):
    """(R_a, t_a, s, aligned estimate [n,4,4], reference [n,4,4]); poses whose reference sum is not finite are skipped."""
    est, ref = [], []
    for i in range(len(traj_ref_all)):
        val = traj_ref_all[i].sum()
        if np.isnan(val) or np.isinf(val):
            continue
        est.append(np.asarray(traj_est_all[i], np.float64))
        ref.append(np.asarray(traj_ref_all[i], np.float64))
    est, ref = np.stack(est), np.stack(ref)
    r, t, s = umeyama(est[:, :3, 3].T, ref[:, :3, 3].T, True)
    scaled = est.copy()
    scaled[:, :3, 3] *= s
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = r, t
    return r, t, s, np.stack([T.dot(p) for p in scaled]), ref


def ape_statistics(est, ref):
    e = np.linalg.norm(ref[:, :3, 3] - est[:, :3, 3], axis=1)
    return {"rmse": float(np.sqrt(np.dot(e, e) / len(e))), "mean": float(np.mean(e)), "median": float(np.median(e)),
            "std": float(np.std(e)), "min": float(np.min(e)), "max": float(np.max(e)), "sse": float(np.dot(e, e))}


def full_traj_eval(traj_est, traj_ref):
    r, t, s, est, ref = align_traj(traj_est, traj_ref)
    return est, ref, r, t, s, ape_statistics(est, ref)


# ------------------------------------------------------------------------------------------------ clouds
def local_points(depths, intrinsics):
    """slam_utils.compute_local_pointclouds (torch, float32)."""
    N, H, W = depths.shape
    y, x = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    pix = torch.stack((x, y, torch.ones_like(x)), dim=-1).float().reshape(-1, 3)
    if intrinsics.ndim == 2:
        cam = torch.matmul(torch.inverse(intrinsics), pix.T).T.reshape(1, H, W, 3).repeat(N, 1, 1, 1)
    else:
        cam = torch.matmul(torch.inverse(intrinsics)[:, None], pix[None, :, :, None].expand(N, -1, -1, -1))
        cam = cam.squeeze(-1).reshape(N, H, W, 3)
    return cam * depths[..., None]


def world_points(cam, poses):
    h = torch.cat([cam, torch.ones_like(cam[:, :, :, 0:1])], dim=-1)
    return torch.matmul(poses[:, None, None, :, :], h[..., None]).squeeze(-1)[..., :3]


def clouds(gt_depths, gt_poses, gt_intri, est_depths, est_poses, est_intris, est_masks):
    """eval_recon.py:130-141 on float32 torch CPU tensors -> (gt points, estimated points) float32 numpy [n,3]."""
    gt = world_points(local_points(gt_depths, gt_intri), gt_poses).numpy()
    est = world_points(local_points(est_depths, est_intris), est_poses).numpy()
    gm = (gt_depths > 0).numpy().astype(bool)
    em = est_masks.numpy().astype(bool)
    return gt[gm], est[em & gm]


def transform(p, T):
    """p <- T[:3, :3] p + T[:3, 3] with each operation rounded on its own, float64."""
    p = np.asarray(p, np.float64)
    out = np.empty_like(p)
    for r in range(3):
        out[:, r] = ((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3]
    return out


def initial_alignment(R, t, s):
    T = np.eye(4)
    T[:3, :3] = s * np.asarray(R, np.float64)
    T[:3, 3] = np.asarray(t, np.float64).reshape(3)
    return T


def voxel_down(p, v):
    """open3d voxel_down_sample, voxel points in ascending (kx, ky, kz) order, each the input-order sum / count."""
    p = np.asarray(p, np.float64)
    if v <= 0.0:
        raise ValueError("voxel_size <= 0")
    if len(p) == 0:
        return np.zeros((0, 3))
    mn = p.min(axis=0) - v * 0.5
    mx = p.max(axis=0) + v * 0.5
    if v * INT_MAX < (mx - mn).max():
        raise ValueError("voxel_size is too small")
    key = np.floor((p - mn) / v).astype(np.int64)
    order = np.lexsort((key[:, 2], key[:, 1], key[:, 0]))
    ks = key[order]
    head = np.ones(len(p), bool)
    head[1:] = (ks[1:] != ks[:-1]).any(axis=1)
    vid = np.empty(len(p), np.int64)
    vid[order] = np.cumsum(head) - 1
    nv = int(head.sum())
    sums = np.zeros((nv, 3))
    np.add.at(sums, vid, p)  # unbuffered, in input order
    cnt = np.bincount(vid, minlength=nv).astype(np.float64)
    return sums / cnt[:, None]


def dist2(a, b):
    d = a - b
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def nearest(ref, q, radius=np.inf, workers=1):
    """(distance clipped to radius, index or -1) of each query's nearest ref point strictly within radius."""
    ref, q = np.asarray(ref, np.float64), np.asarray(q, np.float64)
    if len(ref) == 0 or len(q) == 0:
        return np.full(len(q), float(radius)), np.full(len(q), -1, np.int64)
    _, j = cKDTree(ref).query(q, k=1, distance_upper_bound=np.nextafter(radius, np.inf), workers=workers)
    ok = j < len(ref)
    jj = np.where(ok, j, 0)
    d2 = dist2(q, ref[jj])
    ok &= d2 < radius * radius
    return np.where(ok, np.sqrt(d2), float(radius)), np.where(ok, j, -1).astype(np.int64)


def icp_update(src, dst, corr):
    """Eigen::umeyama(src, dst, false) over the correspondences (identity when there are none)."""
    m = corr >= 0
    if not m.any():
        return np.eye(4)
    x, y = src[m], dst[corr[m]]
    mx, my = x.mean(axis=0), y.mean(axis=0)
    cov = (y - my).T.dot(x - mx) / len(x)
    u, _, vt = np.linalg.svd(cov)
    S = np.eye(3)
    if np.linalg.det(u) * np.linalg.det(vt) < 0:
        S[2, 2] = -1
    T = np.eye(4)
    T[:3, :3] = u.dot(S).dot(vt)
    T[:3, 3] = my - T[:3, :3].dot(mx)
    return T


def icp(src, dst, max_dist=ICP_DIST, max_iter=ICP_ITERS, eps=ICP_EPS):
    """open3d registration_icp (point-to-point, identity start) -> {transformation, fitness, inlier_rmse, iterations}."""
    src, dst = np.asarray(src, np.float64).copy(), np.asarray(dst, np.float64)

    def evaluate(p):
        d, j = nearest(dst, p, max_dist)
        m = j >= 0
        n = int(m.sum())
        if n == 0:
            return j, 0.0, 0.0
        return j, n / len(p), float(np.sqrt((d[m] ** 2).sum() / n))

    T = np.eye(4)
    corr, fit, rmse = evaluate(src)
    it = 0
    for it in range(1, max_iter + 1):
        U = icp_update(src, dst, corr)
        T = U.dot(T)
        src = transform(src, U)
        f0, r0 = fit, rmse
        corr, fit, rmse = evaluate(src)
        if abs(f0 - fit) < eps and abs(r0 - rmse) < eps:
            break
    return {"transformation": T, "fitness": fit, "inlier_rmse": rmse, "iterations": it}


def chamfer(ref, est, max_error=MAX_ERROR, workers=1):
    """chamfer_distance_RMSE -> (chamfer, rmse accuracy, rmse completeness, dist1, dist2)."""
    d1, _ = nearest(ref, est, np.inf, workers)
    d2, _ = nearest(est, ref, np.inf, workers)
    d1, d2 = np.clip(d1, 0, max_error), np.clip(d2, 0, max_error)
    r1, r2 = np.sqrt(np.mean(d1 ** 2)), np.sqrt(np.mean(d2 ** 2))
    return 0.5 * r1 + 0.5 * r2, r1, r2, d1, d2


def eval_recon_points(gt_pts, est_pts, R, t, s, workers=1):
    """eval_recon.py:143-178 from the two clouds on: every stage's output."""
    est = transform(est_pts, initial_alignment(R, t, s))
    est_down, gt_down = voxel_down(est, VOXEL), voxel_down(gt_pts, VOXEL)
    reg = icp(est_down, gt_down)
    est_final = transform(est, reg["transformation"])
    ch, r1, r2, _, _ = chamfer(np.asarray(gt_pts, np.float64), est_final, MAX_ERROR, workers)
    return {"est_aligned": est, "est_down": est_down, "gt_down": gt_down, "icp": reg, "est_final": est_final,
            "rmse_acc": r1, "rmse_comp": r2, "chamfer": ch}


def load(folder):
    c = np.load(os.path.join(folder, "confs.npz"))
    return {"gt_depths": np.load(os.path.join(folder, "gt_depths.npy")), "gt_poses": np.load(os.path.join(folder, "gt_poses.npy")),
            "gt_intrinsic": np.load(os.path.join(folder, "gt_intrinsics.npy")),
            "unscaled_depths": np.load(os.path.join(folder, "depths.npy")),
            "scales": np.load(os.path.join(folder, "scales.npy"))[..., None],
            "intrinsics": np.load(os.path.join(folder, "intrinsics.npy")), "confs": c["confs"], "conf_thres": c["thres"].item(),
            "poses": np.load(os.path.join(folder, "trajectory.npy"))}


def eval_recon_from_saved_data(folder, rel_est_gt=None, workers=1):
    """eval_recon_from_saved_data -> (stage outputs, gt cloud, estimated cloud)."""
    d = load(folder)
    gt_depths = torch.from_numpy(d["gt_depths"]).float()
    gt_poses = torch.from_numpy(d["gt_poses"]).float()
    est_poses = torch.from_numpy(d["poses"]).float()
    gt, est = clouds(gt_depths, gt_poses, torch.from_numpy(d["gt_intrinsic"]),
                     torch.from_numpy(d["unscaled_depths"] * d["scales"]).float(), est_poses,
                     torch.from_numpy(d["intrinsics"]).float(), torch.from_numpy(d["confs"] > d["conf_thres"]).float())
    if rel_est_gt is None:
        R, t, s, _, _ = align_traj(est_poses, gt_poses)
    else:
        R, t, s = rel_est_gt
    return eval_recon_points(gt, est, R, t, s, workers), gt, est


# ------------------------------------------------------------------------------------------------ synthetic scene
ROOM = (np.array([-2.0, -2.0, 0.0]), np.array([2.0, 2.0, 2.5]))
BOXES = [(np.array([-1.5, -1.5, 0.0]), np.array([-0.9, -0.8, 0.8])), (np.array([0.8, 0.5, 0.0]), np.array([1.4, 1.3, 1.2])),
         (np.array([-0.3, 1.0, 0.0]), np.array([0.3, 1.6, 0.5])), (np.array([0.9, -1.6, 0.6]), np.array([1.6, -1.1, 1.4]))]


def _rot(axis, ang):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K.dot(K)


def camera_pose(k, n):
    th = 2 * np.pi * 0.9 * k / n
    c = np.array([0.6 * np.cos(th), 0.6 * np.sin(th), 1.2 + 0.1 * np.sin(3 * th)])
    yaw, pitch = th + np.pi / 2 + 0.3 * np.sin(2 * th), -0.15 + 0.05 * np.cos(th)
    z = np.array([np.cos(yaw) * np.cos(pitch), np.sin(yaw) * np.cos(pitch), np.sin(pitch)])
    x = np.array([np.sin(yaw), -np.cos(yaw), 0.0])
    y = np.cross(z, x)
    P = np.eye(4)
    P[:3, :3] = np.stack([x, y, z], axis=1)
    P[:3, 3] = c
    return P


def render(P, K, H, W):
    """fp64 ray cast of the room and its boxes: depth along the camera z axis."""
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    dc = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1).reshape(-1, 3)
    d = dc.dot(P[:3, :3].T)
    o = P[:3, 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        t_room = np.where(d > 0, (ROOM[1] - o) * inv, (ROOM[0] - o) * inv).min(axis=1)
        t = t_room
        for lo, hi in BOXES:
            t1, t2 = (lo - o) * inv, (hi - o) * inv
            tn, tf = np.minimum(t1, t2).max(axis=1), np.maximum(t1, t2).min(axis=1)
            t = np.where((tn <= tf) & (tn > 0) & (tn < t), tn, t)
    return t.reshape(H, W)  # dc has z = 1: the ray parameter is the depth


def make_scene(n_views=24, H=48, W=64, seed=0, nan_view=7):
    """Seeded synthetic evaluation scene in save_data_all's arrays: ground truth and a perturbed estimate."""
    rng = np.random.default_rng(seed)
    f = 0.8 * W
    K = np.array([[f, 0, (W - 1) / 2], [0, f, (H - 1) / 2], [0, 0, 1]])
    sg, Roff, toff = 1.3, _rot([0.2, -0.3, 0.9], np.deg2rad(25.0)), np.array([0.4, -0.2, 0.1])
    gt_depths = np.empty((n_views, H, W), np.float32)
    gt_poses = np.empty((n_views, 4, 4), np.float32)
    est_poses = np.empty((n_views, 4, 4), np.float32)
    depths = np.empty((n_views, H, W), np.float32)
    intr = np.empty((n_views, 3, 3), np.float32)
    scales = rng.uniform(0.7, 1.4, size=(n_views, 1)).astype(np.float32)
    confs = rng.uniform(1.0, 10.0, size=(n_views, H, W)).astype(np.float32)
    for k in range(n_views):
        P = camera_pose(k, n_views)
        gd = render(P, K, H, W)
        gt = gd.copy()
        if k % 5 == 2:  # a hole in the ground truth
            gt[H // 4:H // 4 + max(1, H // 8), W // 3:W // 3 + max(1, W // 6)] = 0.0
        gt_poses[k] = P
        if k == nan_view:  # a view without ground truth
            gt[:] = 0.0
            gt_poses[k, 0, 3] = np.nan
        gt_depths[k] = gt
        dr = _rot([0.1, 0.4, 1.0], np.deg2rad(0.8) * k / n_views)
        E = np.eye(4)
        E[:3, :3] = Roff.dot(dr).dot(P[:3, :3])
        E[:3, 3] = sg * Roff.dot(P[:3, 3]) + toff + 0.02 * k / n_views * np.array([1.0, -0.5, 0.3])
        est_poses[k] = E
        Ke = K.copy()
        Ke[0, 0] *= 1 + 0.004 * rng.standard_normal()
        Ke[1, 1] *= 1 + 0.004 * rng.standard_normal()
        Ke[0, 2] += 0.2 * rng.standard_normal()
        Ke[1, 2] += 0.2 * rng.standard_normal()
        intr[k] = Ke
        de = sg * gd * (1 + 0.01 * rng.standard_normal(gd.shape))
        far = rng.choice(H * W, size=max(2, H * W // 200), replace=False)  # far outliers: clipped at 0.5
        de.reshape(-1)[far] *= 3.0
        confs[k].reshape(-1)[far] = 9.0
        depths[k] = (de / scales[k]).astype(np.float32)
    return {"trajectory": est_poses, "scales": scales, "depths": depths, "intrinsics": intr, "confs": confs, "thres": 4.2,
            "gt_poses": gt_poses, "gt_depths": gt_depths, "gt_intrinsics": K.astype(np.float32)}


def write_scene(scene, folder):
    """The files save_data_all writes (with gt_*), minus images and the PLY."""
    os.makedirs(folder, exist_ok=True)
    n = len(scene["trajectory"])
    np.savez(os.path.join(folder, "view_graph.npz"), view_graph={v: [v - 1] if v else [] for v in range(n)}, loop_min_dist=40,
             view_names=["%04d.png" % v for v in range(n)])
    for k in ("trajectory", "scales", "depths", "intrinsics", "gt_poses", "gt_depths", "gt_intrinsics"):
        np.save(os.path.join(folder, k + ".npy"), scene[k])
    np.savez(os.path.join(folder, "confs.npz"), confs=scene["confs"], thres=scene["thres"])
