"""Drop-in vista_slam/eval/eval_recon.py: reconstruction accuracy, completeness and Chamfer distance of a saved SLAM run,
on the GPU (csrc/recon.cu), without open3d, pykdtree or munch.

eval_recon follows the reference step by step:
  1. clouds: ground truth where gt_depth > 0 (shared gt intrinsics), estimate where the mask is set and gt_depth > 0,
     unprojected and moved to the world in fp32, in (view, row, column) order -> fp64;
  2. the estimate moved by (s R, t) in fp64;
  3. open3d's voxel_down_sample(0.05) of both clouds (voxels in ascending key order rather than open3d's hash order);
  4. open3d's point-to-point registration_icp from the downsampled estimate to the downsampled ground truth
     (correspondences strictly within 0.1, identity start, at most 30 iterations, stop when fitness and inlier RMSE both
     change by less than 1e-6).  The nearest neighbours and the moments run on the device; the 3 x 3 SVD and the
     convergence test on the host, one read-back per iteration;
  5. the ICP transformation applied to the full-resolution estimate;
  6. nearest-neighbour distances both ways, clipped to [0, 0.5]: rmse_acc (estimate -> ground truth), rmse_comp
     (ground truth -> estimate), chamfer = 0.5 rmse_acc + 0.5 rmse_comp.

Differences from the reference's types: load_data returns a `View` (dict with attribute access) in place of a
munch.Munch; the clouds eval_recon returns in place of open3d `points` are fp64 CUDA tensors [n, 3];
chamfer_distance_RMSE takes [n, 3] arrays or tensors, and returns its distances as fp64 CUDA tensors.  Ground-truth and
estimated intrinsics must be float32: the reference's torch.matmul raises on any other dtype."""
import ctypes
import os

import numpy as np
import torch

from .. import _lib
from ..slam import View

VOXEL_SIZE, ICP_MAX_DIST, ICP_MAX_ITER, ICP_EPS, MAX_ERROR = 0.05, 0.1, 30, 1e-6, 0.5


def load_data(output_foler, load_view_graph=True,
              load_gt_depths=True, load_gt_poses=True, load_gt_intrinsic=True,
              load_unscaled_depths=True, load_scales=True,
              load_intrinsics=True, load_confs=True, load_poses=True):
    """eval_recon.py:7-35: the files of save_data_all as host numpy arrays, in a View."""
    data = {}
    if load_view_graph:
        view_graph_npz = np.load(os.path.join(output_foler, "view_graph.npz"), allow_pickle=True)
        data["view_graph"] = view_graph_npz["view_graph"].item()
        data["loop_min_dist"] = view_graph_npz["loop_min_dist"].item()
        data["view_names"] = view_graph_npz["view_names"].tolist()
    if load_gt_depths:
        data["gt_depths"] = np.load(os.path.join(output_foler, "gt_depths.npy"))
    if load_gt_poses:
        data["gt_poses"] = np.load(os.path.join(output_foler, "gt_poses.npy"))
    if load_gt_intrinsic:
        data["gt_intrinsic"] = np.load(os.path.join(output_foler, "gt_intrinsics.npy"))
    if load_unscaled_depths:
        data["unscaled_depths"] = np.load(os.path.join(output_foler, "depths.npy"))
    if load_scales:
        data["scales"] = np.load(os.path.join(output_foler, "scales.npy"))[..., None]  # [N, 1, 1]
    if load_intrinsics:
        data["intrinsics"] = np.load(os.path.join(output_foler, "intrinsics.npy"))
    if load_confs:
        confs_npz = np.load(os.path.join(output_foler, "confs.npz"))
        data["confs"] = confs_npz["confs"]
        data["conf_thres"] = confs_npz["thres"].item()
    if load_poses:
        data["poses"] = np.load(os.path.join(output_foler, "trajectory.npy"))
    return View(data)


def transform_to_world_coordinates(cam_coords, poses):
    """eval_recon.py:78-86: (N, H, W, 3) camera points -> world points with poses (N, 4, 4), on the tensors' device."""
    cam_coords_h = torch.cat([cam_coords, torch.ones_like(cam_coords[:, :, :, 0:1])], dim=-1)
    points_world = torch.matmul(poses[:, None, None, :, :], cam_coords_h[..., None])
    return points_world.squeeze(-1)[..., :3]


# ------------------------------------------------------------------------------------------------ device stages
def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def _f32(x, name):
    t = torch.as_tensor(x)
    return t.to(device=_dev(), dtype=torch.float32).contiguous()


def _intrinsics(x, name):
    t = torch.as_tensor(x)
    if t.dtype != torch.float32:
        raise TypeError("%s must be float32 (got %s): the reference's torch.matmul with float32 pixel coordinates raises "
                        "on any other dtype" % (name, t.dtype))
    return t.to(_dev()).contiguous()


def _points(p):
    """[n, 3] array / tensor (or anything with .points) -> contiguous fp64 CUDA tensor."""
    p = getattr(p, "points", p)
    t = torch.as_tensor(np.asarray(p) if not isinstance(p, torch.Tensor) else p)
    t = t.to(device=_dev(), dtype=torch.float64).reshape(-1, 3).contiguous()
    return t


def _scratch(nbytes):
    return torch.empty((int(nbytes) + 15) // 16 * 2, dtype=torch.float64, device=_dev())


def world_clouds(gt_depths, gt_poses, gt_intri, depths, scales, est_poses, est_intris, confs, thres):
    """Both clouds as fp64 CUDA tensors (ground truth, estimate).  depths are multiplied by scales [N] in fp32 when
    scales is given; the estimate keeps confs > thres and gt_depths > 0."""
    gd, gp, gk = _f32(gt_depths, "gt_depths"), _f32(gt_poses, "gt_poses"), _intrinsics(gt_intri, "gt_intri")
    d, ep, ek, c = _f32(depths, "depths"), _f32(est_poses, "est_poses"), _intrinsics(est_intris, "est_intris"), _f32(confs, "confs")
    sc = None if scales is None else _f32(scales, "scales").reshape(-1)
    N, H, W = gd.shape
    if (tuple(d.shape) != (N, H, W) or tuple(c.shape) != (N, H, W) or tuple(gp.shape) != (N, 4, 4)
            or tuple(ep.shape) != (N, 4, 4) or tuple(gk.shape) != (3, 3) or tuple(ek.shape) != (N, 3, 3)
            or (sc is not None and sc.numel() != N)):
        raise ValueError("shape mismatch: gt_depths / depths / confs [N,H,W], poses [N,4,4], gt_intri [3,3], "
                         "est_intris [N,3,3], scales [N]")
    L = _lib.lib()
    gt = torch.empty(N * H * W, 3, dtype=torch.float64, device=_dev())
    est = torch.empty_like(gt)
    cnt = torch.zeros(2, dtype=torch.int64, device=_dev())
    scratch = _scratch(L.sta_eval_clouds_scratch_bytes(N, H))
    _lib.check(L.sta_eval_clouds(N, H, W, _lib.ptr(gd), _lib.ptr(gp), _lib.ptr(gk), _lib.ptr(d), _lib.ptr(sc), _lib.ptr(ep),
                                 _lib.ptr(ek), _lib.ptr(c), float(thres), _lib.ptr(gt), _lib.ptr(est), _lib.ptr(cnt),
                                 _lib.ptr(scratch), _lib.cur_stream()), "sta_eval_clouds")
    n0, n1 = cnt.tolist()
    return gt[:n0], est[:n1]


def transform_points_(pts, T):
    """In place on an fp64 CUDA [n, 3] tensor: p <- T[:3, :3] p + T[:3, 3]."""
    m = (ctypes.c_double * 12)(*np.asarray(T, np.float64)[:3, :4].reshape(-1).tolist())
    _lib.check(_lib.lib().sta_transform_points(_lib.ptr(pts), len(pts), m, _lib.cur_stream()), "sta_transform_points")
    return pts


def voxel_down_sample(pts, voxel_size):
    """open3d PointCloud.voxel_down_sample on an fp64 CUDA [n, 3] tensor."""
    pts = _points(pts)
    L = _lib.lib()
    out = torch.empty_like(pts)
    cnt = ctypes.c_int64()
    scratch = _scratch(L.sta_voxel_scratch_bytes(len(pts)))
    _lib.check(L.sta_voxel_down(_lib.ptr(pts), len(pts), float(voxel_size), _lib.ptr(out), ctypes.byref(cnt), _lib.ptr(scratch),
                                _lib.cur_stream()), "sta_voxel_down")
    return out[:cnt.value]


class NnIndex:
    """Device nearest-neighbour index over one fp64 [n, 3] cloud (sta_nn_*)."""

    def __init__(self, pts):
        self.pts = _points(pts)
        h = ctypes.c_void_p()
        _lib.check(_lib.lib().sta_nn_create(_lib.ptr(self.pts), len(self.pts), ctypes.byref(h), _lib.cur_stream()),
                   "sta_nn_create")
        self.h = h

    def __del__(self):
        if getattr(self, "h", None) and _lib._lib is not None:
            _lib.lib().sta_nn_destroy(self.h)
            self.h = None

    def query(self, q, radius):
        """(distance to the nearest point strictly within radius, or radius; its index, or -1) per query."""
        q = _points(q)
        L = _lib.lib()
        dist = torch.empty(len(q), dtype=torch.float64, device=_dev())
        idx = torch.empty(len(q), dtype=torch.int64, device=_dev())
        scratch = _scratch(L.sta_nn_query_scratch_bytes(len(q)))
        _lib.check(L.sta_nn_query(self.h, _lib.ptr(q), len(q), float(radius), _lib.ptr(dist), _lib.ptr(idx), _lib.ptr(scratch),
                                  _lib.cur_stream()), "sta_nn_query")
        return dist, idx


def _umeyama_rigid(m):
    """Eigen::umeyama without scaling from the moments of sta_icp_moments (identity without correspondences)."""
    n = m[0]
    if n == 0:
        return np.eye(4)
    mx, my, cov = m[2:5] / n, m[5:8] / n, m[8:17].reshape(3, 3) / n
    u, _, vt = np.linalg.svd(cov)
    S = np.eye(3)
    if np.linalg.det(u) * np.linalg.det(vt) < 0:
        S[2, 2] = -1
    T = np.eye(4)
    T[:3, :3] = u.dot(S).dot(vt)
    T[:3, 3] = my - T[:3, :3].dot(mx)
    return T


def registration_icp(source, target, max_correspondence_distance=ICP_MAX_DIST, max_iteration=ICP_MAX_ITER,
                     relative_fitness=ICP_EPS, relative_rmse=ICP_EPS):
    """open3d registration_icp, point-to-point, identity start -> {transformation, fitness, inlier_rmse, iterations}."""
    src = _points(source).clone()
    ix = NnIndex(target)
    L = _lib.lib()
    mom = torch.empty(17, dtype=torch.float64, device=_dev())
    scratch = _scratch(L.sta_icp_scratch_bytes(len(src)))

    def evaluate():
        _lib.check(L.sta_icp_moments(ix.h, _lib.ptr(ix.pts), _lib.ptr(src), len(src), float(max_correspondence_distance),
                                     _lib.ptr(mom), _lib.ptr(scratch), _lib.cur_stream()), "sta_icp_moments")
        m = mom.cpu().numpy()
        if m[0] == 0:
            return m, 0.0, 0.0
        return m, m[0] / len(src), float(np.sqrt(m[1] / m[0]))

    T = np.eye(4)
    m, fit, rmse = evaluate()
    it = 0
    for it in range(1, max_iteration + 1):
        U = _umeyama_rigid(m)
        T = U.dot(T)
        transform_points_(src, U)
        f0, r0 = fit, rmse
        m, fit, rmse = evaluate()
        if abs(f0 - fit) < relative_fitness and abs(r0 - rmse) < relative_rmse:
            break
    return {"transformation": T, "fitness": fit, "inlier_rmse": rmse, "iterations": it}


def chamfer_distance_RMSE(pcd_ref, pcd_est, max_error):
    """eval_recon.py:89-105 -> (chamfer, rmse of dist1, rmse of dist2, dist1, dist2): dist1 is each estimated point's
    nearest-neighbour distance in the reference cloud, dist2 the reverse, both clipped to [0, max_error]."""
    ref, est = _points(pcd_ref), _points(pcd_est)
    L = _lib.lib()
    d1, _ = NnIndex(ref).query(est, max_error)
    d2, _ = NnIndex(est).query(ref, max_error)
    ss = torch.empty(2, dtype=torch.float64, device=_dev())
    scratch = _scratch(L.sta_reduce_scratch_bytes())
    for k, d in enumerate((d1, d2)):
        _lib.check(L.sta_sum_sq_clipped(_lib.ptr(d), len(d), float(max_error), _lib.ptr(ss[k:]), _lib.ptr(scratch),
                                        _lib.cur_stream()), "sta_sum_sq_clipped")
    s1, s2 = ss.tolist()
    rmse1 = float(np.sqrt(s1 / len(d1))) if len(d1) else float("nan")
    rmse2 = float(np.sqrt(s2 / len(d2))) if len(d2) else float("nan")
    return 0.5 * rmse1 + 0.5 * rmse2, rmse1, rmse2, d1, d2


def _initial(rel_R, rel_t, rel_s):
    T = np.eye(4)
    T[:3, :3] = float(rel_s) * np.asarray(torch.as_tensor(rel_R).cpu(), np.float64).reshape(3, 3)
    T[:3, 3] = np.asarray(torch.as_tensor(rel_t).cpu(), np.float64).reshape(3)
    return T


def _recon(gt_pts, est_pts, rel_R, rel_t, rel_s, tick):
    transform_points_(est_pts, _initial(rel_R, rel_t, rel_s))
    tick("align")
    est_down, gt_down = voxel_down_sample(est_pts, VOXEL_SIZE), voxel_down_sample(gt_pts, VOXEL_SIZE)
    tick("downsample")
    reg = registration_icp(est_down, gt_down, ICP_MAX_DIST)
    tick("icp")
    transform_points_(est_pts, reg["transformation"])
    chamfer_dist, rmse_acc, rmse_comp, _, _ = chamfer_distance_RMSE(gt_pts, est_pts, max_error=MAX_ERROR)
    tick("chamfer")
    return rmse_acc, rmse_comp, chamfer_dist, gt_pts, est_pts


def eval_recon(gt_depths, gt_poses, gt_intri,
               est_depths, est_poses, est_intris, est_masks,
               rel_R, rel_t, rel_s):
    """eval_recon.py:108-178 -> (rmse_acc, rmse_comp, chamfer, gt points, estimated points); the points are fp64 CUDA
    tensors [n, 3].  gt_depths / est_depths / est_masks [N,H,W], poses [N,4,4], gt_intri [3,3], est_intris [N,3,3]."""
    assert len(gt_depths) == len(est_depths) == len(est_masks) == len(est_poses) == len(gt_poses)
    mask = (torch.as_tensor(est_masks) != 0).to(torch.float32)
    gt_pts, est_pts = world_clouds(gt_depths, gt_poses, gt_intri, est_depths, None, est_poses, est_intris, mask, 0.5)
    return _recon(gt_pts, est_pts, rel_R, rel_t, rel_s, lambda name: None)


def _from_saved_data(output_folder, rel_est_gt, tick):
    data = load_data(f"{output_folder}", load_view_graph=False)
    tick("load")
    gt_poses = torch.from_numpy(data.gt_poses).float()
    est_poses = torch.from_numpy(data.poses).float()
    if rel_est_gt is not None:
        rel_R, rel_t, rel_s = rel_est_gt
    else:
        from .eval_traj import align_traj
        rel_R, rel_t, rel_s, _, _ = align_traj(est_poses, gt_poses)
    scales = data.scales.reshape(len(data.scales), -1)[:, 0]
    gt_pts, est_pts = world_clouds(data.gt_depths, gt_poses, torch.from_numpy(data.gt_intrinsic), data.unscaled_depths,
                                   scales, est_poses, torch.from_numpy(data.intrinsics).float(), data.confs, data.conf_thres)
    tick("clouds")
    return _recon(gt_pts, est_pts, rel_R, rel_t, rel_s, tick)


def eval_recon_from_saved_data(output_folder, rel_est_gt: list | None = None):
    """eval_recon.py:181-206: rel_est_gt is None or [R, t, s] of the estimate relative to the ground truth (None: aligned
    from the trajectories)."""
    return _from_saved_data(output_folder, rel_est_gt, lambda name: None)
