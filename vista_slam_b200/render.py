"""Images of the SLAM map from any camera, drawn on the device (csrc/render.cu, `sta_render`).

The map is what OnlineSLAM._export returns without the cloud -- pose [V,4,4] (scale dropped), scale [V,1], depth and
conf [V,H,W] (unscaled), intri [V,3,3] -- plus images [V,3,H,W] in [-1, 1].  Every pixel with conf > conf_thres is the
PLY's point of save_data_all, bit for bit, splatted into a z-buffer; line segments (camera frusta, pose-graph edges) are
depth-tested in the same buffer, so points hide the lines behind them.  Ties at equal depth go to the lower id, so an
image does not depend on scheduling.  There is no shading, anti-aliasing or disc splat: a point covers a square of
(2 point_radius + 1)^2 pixels at every depth.

camera_frusta and graph_segments build the lines of scripts/video.py: a camera's 8 frustum segments (open3d's
LineSet.create_camera_visualization(...).lines[:8]) and the view graph's neighbour and loop edges (get_edge_lineset)."""
import ctypes
import numbers

import numpy as np
import torch

from . import _lib

NEIGHBOR_EDGE_COLOR = (0.0, 0.0, 1.0)
LOOP_EDGE_COLOR = (1.0, 0.5, 0.0)
_MAP_KEYS = ("pose", "scale", "depth", "conf", "intri", "images")


def _tensor(x, name, dtype=None):
    if not isinstance(x, (torch.Tensor, np.ndarray)):
        raise ValueError("%s must be a tensor or an array" % name)
    t = torch.as_tensor(x)
    if dtype is not None and not (t.is_floating_point() and t.dtype != torch.float16):
        raise ValueError("%s must be a float32 or float64 array, not %s" % (name, t.dtype))
    return t


def _w2c(poses):
    """World-to-camera of camera-to-world [C,4,4] (bottom row 0 0 0 1): [A^-1 | -A^-1 t] with A^-1 from the adjugate,
    in float64; cast to float32.  Only elementwise operations (no solver, matmul or reduction), so there is no host
    synchronisation and each camera's result does not depend on how many cameras share the call."""
    a = [[poses[:, i, j] for j in range(3)] for i in range(3)]
    t = [poses[:, i, 3] for i in range(3)]
    # cofactors: adj[i][j] = cofactor of a[j][i]
    adj = [[a[(j + 1) % 3][(i + 1) % 3] * a[(j + 2) % 3][(i + 2) % 3] - a[(j + 1) % 3][(i + 2) % 3] * a[(j + 2) % 3][(i + 1) % 3]
            for j in range(3)] for i in range(3)]
    det = a[0][0] * adj[0][0] + a[0][1] * adj[1][0] + a[0][2] * adj[2][0]
    inv = [[adj[i][j] / det for j in range(3)] for i in range(3)]
    rows = [torch.stack(inv[i] + [-(inv[i][0] * t[0] + inv[i][1] * t[1] + inv[i][2] * t[2])], dim=-1) for i in range(3)]
    last = torch.zeros_like(rows[0])
    last[:, 3] = 1.0
    return torch.stack(rows + [last], dim=1).to(torch.float32).contiguous()


def _check_maps(maps):
    """The arrays of a `maps` dict (module docstring) as tensors, and V, H, W; ValueError for a missing key, a shape
    or a dtype other than float32.  Devices are the caller's to check."""
    if not isinstance(maps, dict) or any(k not in maps for k in _MAP_KEYS):
        raise ValueError("maps must be a dict with keys %s" % (_MAP_KEYS,))
    m = {k: _tensor(maps[k], "maps[%r]" % k) for k in _MAP_KEYS}
    if m["depth"].dim() != 3:
        raise ValueError("maps['depth'] must be [V,H,W], got %s" % (tuple(m["depth"].shape),))
    V, H, W = m["depth"].shape
    want = {"pose": (V, 4, 4), "scale": (V, 1), "depth": (V, H, W), "conf": (V, H, W), "intri": (V, 3, 3),
            "images": (V, 3, H, W)}
    for k, shape in want.items():
        got = tuple(m[k].shape)
        if got != shape and not (k == "scale" and got == (V,)):
            raise ValueError("maps[%r] must be %s, got %s" % (k, shape, got))
        if m[k].dtype != torch.float32:
            raise ValueError("maps[%r] must be float32, not %s" % (k, m[k].dtype))
    return m, V, H, W


def render_views(maps, conf_thres, poses, K, size, point_radius=0, near=1e-3, lines=None, background=(1.0, 1.0, 1.0)):
    """Render `maps` (module docstring; every array float32 on one CUDA device) from C cameras.

    poses [C,4,4]: camera-to-world (the convention of trajectory.npy, get_view().pose and frame_trajectory()["pose"]),
    host or device, inverted on the map's device in float64.  K: [C,3,3] or one [3,3] for all.  size: (Ho, Wo).
    lines: (segs [L,2,3] world endpoints, colors [L,3]) or None.  A point or segment is drawn where its camera-frame z
    is at least near.  Returns {rgb [C,Ho,Wo,3] float32, depth [C,Ho,Wo] float32 (camera z, 0 where empty), index
    [C,Ho,Wo] int64 (v H W + row W + col of the point drawn, V H W + l for segment l, -1 where empty)} on the map's
    device, with no host synchronisation.  Shapes, dtypes, devices and ranges are checked first (ValueError)."""
    m, V, H, W = _check_maps(maps)
    if not (isinstance(size, (tuple, list)) and len(size) == 2 and all(isinstance(s, numbers.Integral) for s in size)):
        raise ValueError("size must be (Ho, Wo)")
    Ho, Wo = int(size[0]), int(size[1])
    if not (1 <= Ho <= _lib.RENDER_MAX_SIDE and 1 <= Wo <= _lib.RENDER_MAX_SIDE):
        raise ValueError("output size %s outside [1, %d]" % ((Ho, Wo), _lib.RENDER_MAX_SIDE))
    if not isinstance(point_radius, numbers.Integral) or not 0 <= point_radius <= _lib.RENDER_MAX_RADIUS:
        raise ValueError("point_radius must be an integer in [0, %d]" % _lib.RENDER_MAX_RADIUS)
    if not (isinstance(near, numbers.Real) and np.isfinite(near) and near > 0):
        raise ValueError("near must be a positive finite number")
    if not (isinstance(conf_thres, numbers.Real) and np.isfinite(conf_thres)):
        raise ValueError("conf_thres must be a finite number")
    P = _tensor(poses, "poses", float)
    if P.dim() != 3 or tuple(P.shape[1:]) != (4, 4):
        raise ValueError("poses must be [C,4,4], got %s" % (tuple(P.shape),))
    C = P.shape[0]
    if not 1 <= C <= _lib.RENDER_MAX_SIDE:
        raise ValueError("1 to %d cameras per call, got %d" % (_lib.RENDER_MAX_SIDE, C))
    Kt = _tensor(K, "K", float)
    if tuple(Kt.shape) == (3, 3):
        Kt = Kt.expand(C, 3, 3)
    if tuple(Kt.shape) != (C, 3, 3):
        raise ValueError("K must be [3,3] or [C,3,3] with C = %d, got %s" % (C, tuple(Kt.shape)))
    if len(background) != 3:
        raise ValueError("background must be 3 numbers")
    segs = cols = None
    L = 0
    if lines is not None:
        if not (isinstance(lines, (tuple, list)) and len(lines) == 2):
            raise ValueError("lines must be (segs [L,2,3], colors [L,3])")
        segs, cols = _tensor(lines[0], "segs", float), _tensor(lines[1], "line colors", float)
        L = segs.shape[0] if segs.dim() == 3 else -1
        if tuple(segs.shape[1:]) != (2, 3) or tuple(cols.shape) != (L, 3):
            raise ValueError("lines must be (segs [L,2,3], colors [L,3]), got %s and %s"
                             % (tuple(segs.shape), tuple(cols.shape)))
    if V > 65535:
        raise ValueError("at most 65535 views per render, got %d" % V)
    if V * H * W + L >= 2 ** 32 - 1:
        raise ValueError("V H W + L = %d ids do not fit the 32-bit key id" % (V * H * W + L))
    dev = m["depth"].device
    if dev.type != "cuda" or any(m[k].device != dev for k in _MAP_KEYS):
        raise ValueError("the map arrays must all be on one CUDA device")

    w2c = _w2c(P.to(dev, torch.float64))
    Kd = Kt.to(dev, torch.float32).contiguous()
    if L > 0:
        segs = segs.to(dev, torch.float32).contiguous()
        cols = cols.to(dev, torch.float32).contiguous()
    else:
        segs = cols = None
    m = {k: t.contiguous() for k, t in m.items()}
    rgb = torch.empty(C, Ho, Wo, 3, dtype=torch.float32, device=dev)
    depth = torch.empty(C, Ho, Wo, dtype=torch.float32, device=dev)
    index = torch.empty(C, Ho, Wo, dtype=torch.int64, device=dev)
    Lb = _lib.lib()
    nbytes = int(Lb.sta_render_scratch_bytes(C, Ho, Wo))
    scratch = torch.empty(nbytes // 8, dtype=torch.int64, device=dev)
    bg = (ctypes.c_float * 3)(*[float(b) for b in background])
    with torch.cuda.device(dev):
        _lib.check(Lb.sta_render(
            _lib.ptr(m["depth"]), _lib.ptr(m["conf"]), _lib.ptr(m["pose"]), _lib.ptr(m["scale"]), _lib.ptr(m["intri"]),
            _lib.ptr(m["images"]), V, H, W, float(conf_thres), _lib.ptr(w2c), _lib.ptr(Kd), C, Ho, Wo, int(point_radius),
            float(near), _lib.ptr(segs), _lib.ptr(cols), L, bg, _lib.ptr(scratch), nbytes, _lib.ptr(rgb),
            _lib.ptr(depth), _lib.ptr(index), _lib.cur_stream()), "sta_render")
    return {"rgb": rgb, "depth": depth, "index": index}


def camera_frusta(poses, K, H, W, scale, color):
    """The 8 segments per camera that scripts/video.py draws (create_camera_visualization(...).lines[:8]): the centre
    to the image corners (0,0), (W,0), (W,H), (0,H) at depth `scale`, then around that rectangle.  poses [N,4,4]
    camera-to-world, K [3,3] or [N,3,3].  Returns (segs [8N,2,3], colors [8N,3]) float32 numpy arrays."""
    P = np.asarray(poses, dtype=np.float64).reshape(-1, 4, 4)
    Ks = np.broadcast_to(np.asarray(K, dtype=np.float64), (len(P), 3, 3))
    pix = np.array([[0.0, 0.0, 1.0], [W, 0.0, 1.0], [W, H, 1.0], [0.0, H, 1.0]])
    segs = []
    for p, k in zip(P, Ks):
        cam = np.concatenate([np.zeros((1, 3)), pix @ np.linalg.inv(k).T * scale])  # centre, then the 4 corners
        w = cam @ p[:3, :3].T + p[:3, 3]
        for a, b in ((0, 1), (0, 2), (0, 3), (0, 4), (1, 2), (2, 3), (3, 4), (4, 1)):
            segs.append((w[a], w[b]))
    segs = np.asarray(segs, dtype=np.float32).reshape(-1, 2, 3)
    return segs, np.tile(np.asarray(color, dtype=np.float32), (len(segs), 1))


def graph_segments(poses, view_graph, loop_min_dist, views):
    """The edges scripts/video.py draws for `views` (get_edge_lineset of each): from the centre of view v to that of
    each connected view nv <= v in view_graph[v], loop orange if |v - nv| >= loop_min_dist and neighbour blue
    otherwise.  poses [V,4,4] camera-to-world, indexed by view.  Returns (segs [L,2,3], colors [L,3]) float32."""
    P = np.asarray(poses, dtype=np.float64)
    segs, cols = [], []
    for v in views:
        for nv in view_graph[v]:
            if nv > v:
                continue
            segs.append((P[v, :3, 3], P[nv, :3, 3]))
            cols.append(LOOP_EDGE_COLOR if abs(v - nv) >= loop_min_dist else NEIGHBOR_EDGE_COLOR)
    return np.asarray(segs, dtype=np.float32).reshape(-1, 2, 3), np.asarray(cols, dtype=np.float32).reshape(-1, 3)


def concat_lines(*parts):
    """One (segs, colors) pair of several, for render_views' `lines`."""
    return (np.concatenate([p[0] for p in parts]).reshape(-1, 2, 3), np.concatenate([p[1] for p in parts]).reshape(-1, 3))
