"""Pointmap consumers on the GPU -- same names and argument meaning as vista_slam/utils/slam_utils.py, for the
functions OnlineSLAM calls on the head outputs right after the STA boundary (SURVEY.md section 8(f) rank 2):

    estimate_intrinsic_from_pts3d               slam_utils.py:8-79    (slam.py:184)
    estimate_scale_with_depth_and_confidence    slam_utils.py:168-190 (slam.py:224)
    view_consistency_check                      slam_utils.py:346-419 (the map's multi-view depth consistency;
                                                OnlineSLAM.view_consistency and min_consistent_views)

plus `pointmap_consumers`, the fused form of slam.py:181-185 + pose_graph.py:41 (intrinsics, depth maps and the
per-view confidence mean in ONE pass over the pointmaps, no host synchronisation), and `scale_and_confidence`
(slam.py:224-227 in one pass).  CUDA tensors only: there is no CPU fallback -- a CPU tensor raises."""
import torch

from .. import _lib

_scratch = {}


def _scratch_for(device, V):
    key = (device.index, max(int(V), 1))
    buf = _scratch.get(key)
    if buf is None:
        nbytes = int(_lib.lib().sta_pointmap_scratch_bytes(key[1]))
        buf = torch.empty(nbytes // 8, dtype=torch.float64, device=device)
        _scratch[key] = buf
    return buf


def _f32_cuda(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor (the CUDA library has no CPU path)" % name)
    return t.detach().to(torch.float32).contiguous()


def pointmap_consumers(pts3d, confidence, shared_intrinsic=False):
    """pts3d [B,H,W,3], confidence [B,H,W] -> (K [3,3] | [B,3,3], depths [B,H,W], conf_mean [B]); one kernel pass."""
    pts3d = _f32_cuda(pts3d, "pts3d")
    confidence = _f32_cuda(confidence, "confidence")
    B, H, W, three = pts3d.shape
    if three != 3 or tuple(confidence.shape) != (B, H, W):
        raise RuntimeError("expected pts3d [B,H,W,3] and confidence [B,H,W]")
    dev = pts3d.device
    K = torch.empty((3, 3) if shared_intrinsic else (B, 3, 3), dtype=torch.float32, device=dev)
    depth = torch.empty((B, H, W), dtype=torch.float32, device=dev)
    cmean = torch.empty((B,), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().sta_pointmap_consumers(_lib.ptr(pts3d), _lib.ptr(confidence), B, H, W,
                                                     1 if shared_intrinsic else 0, _lib.ptr(K), _lib.ptr(depth),
                                                     _lib.ptr(cmean), _lib.ptr(_scratch_for(dev, B)), _lib.cur_stream()),
                   "sta_pointmap_consumers")
    return K, depth, cmean


def estimate_intrinsic_from_pts3d(pts3d, confidence, shared_intrinsic=False):
    """Drop-in for slam_utils.py:8-79: K [3,3] if shared else [B,3,3]."""
    return pointmap_consumers(pts3d, confidence, shared_intrinsic)[0]


def scale_and_confidence(Di, Dj, ci, cj):
    """(scale, scale_conf) of slam.py:224-227 as two 0-d CUDA tensors; one kernel pass."""
    Di, Dj, ci, cj = [_f32_cuda(t, n).reshape(-1) for t, n in ((Di, "Di"), (Dj, "Dj"), (ci, "ci"), (cj, "cj"))]
    n = Di.numel()
    if not (Dj.numel() == n and ci.numel() == n and cj.numel() == n and n > 0):
        raise RuntimeError("Di, Dj, ci, cj must have the same non-zero number of elements")
    out = torch.empty(2, dtype=torch.float32, device=Di.device)
    with torch.cuda.device(Di.device):
        _lib.check(_lib.lib().sta_depth_scale(_lib.ptr(Di), _lib.ptr(Dj), _lib.ptr(ci), _lib.ptr(cj), n, _lib.ptr(out),
                                              _lib.ptr(_scratch_for(Di.device, 1)), _lib.cur_stream()), "sta_depth_scale")
    return out[0], out[1]


def estimate_scale_with_depth_and_confidence(Di, Dj, ci, cj):
    """Drop-in for slam_utils.py:168-190: scalar s with Dj ~ s * Di."""
    return scale_and_confidence(Di, Dj, ci, cj)[0]


def view_consistency_check(depth, intrinsics, poses, threshold=0.05):
    """Drop-in for slam_utils.py:346-419: depth [n,H,W], intrinsics [n,3,3], poses [n,4,4] camera-to-world ->
    int32 [n,H,W], per pixel the number of views within 4 indices whose depth agrees with the pixel's reprojection
    within `threshold` (absolute).  Computed in float32 (inputs are cast) by one kernel launch (csrc/consistency.cu),
    with the reference's quirks: a point projecting outside a neighbour samples 0 there, a non-finite projection never
    agrees, and the window is clipped at the ends of the sequence.  No host synchronisation."""
    depth = _f32_cuda(depth, "depth")
    intrinsics = _f32_cuda(intrinsics, "intrinsics")
    poses = _f32_cuda(poses, "poses")
    if depth.dim() != 3:
        raise RuntimeError("expected depth [n,H,W], got %s" % (tuple(depth.shape),))
    n, H, W = depth.shape
    if tuple(intrinsics.shape) != (n, 3, 3) or tuple(poses.shape) != (n, 4, 4):
        raise RuntimeError("expected intrinsics [n,3,3] and poses [n,4,4] for depth [n,H,W]")
    if intrinsics.device != depth.device or poses.device != depth.device:
        raise RuntimeError("depth, intrinsics and poses must be on one device")
    count = torch.empty((n, H, W), dtype=torch.int32, device=depth.device)
    if n == 0:
        return count
    with torch.cuda.device(depth.device):
        _lib.check(_lib.lib().sta_view_consistency(_lib.ptr(depth), _lib.ptr(intrinsics), _lib.ptr(poses), n, H, W,
                                                   float(threshold), _lib.ptr(count), _lib.cur_stream()),
                   "sta_view_consistency")
    return count
