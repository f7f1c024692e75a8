"""GPU: ray casting of the fused TSDF volume (csrc/raycast.cu, fusion.raycast, OnlineSLAM.render_surface).

  1. A planted plane where every float32 operation is exact: every pixel hits, depth within one float32 ulp, normal
     exactly (0, 0, -1), colour within one ulp.
  2. Sphere, torus and noisy fields with saddles, random cameras, C in {1, 3, 17}, min_weight 1 and 2 over partial
     weights, against the float64 oracle (oracle/raycast_oracle.py): hit / miss equal on every unambiguous pixel; where
     both hit, depth within 1e-4 v + 1e-6 z, colour within 1e-5, normal within 1e-3.
  3. Every hit lies in a cube that marching cubes meshes, within sqrt(3) v of that cube's vertices.
  4. Fused scenes: the 26-view ray-cast sphere and the fusion-stream room from new cameras against analytic depths.
  5. The same bits on every call and for C cameras as for C one-camera calls, inputs unmodified, no host
     synchronisation in _raycast.
  6. OnlineSLAM: render_surface equals fuse_volume + raycast bit for bit, views and min_consistent_views honoured,
     background PGO equal to synchronous, the session unchanged, fuse_volume + _mesh equal to fuse_views; the real
     frontend gives a non-empty image.
  7. tools/render_video.py --surface writes the frame sequence."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import fusion_oracle as fo
from oracle import raycast_oracle as ro
from oracle import slam_oracle as so
from test_fusion_gpu import _K, _look_at, _replayed, _voxel_of
from test_raycast_cpu import _field_volume
from test_slam_batch_gpu import _frames_224
from test_slam_gpu import VOCAB, _replay_slam, _value

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _t(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def _cast(vol, v, poses, K, size, **kw):
    from vista_slam_b200.fusion import raycast
    b, T, Wt, C = vol
    out = raycast(_t(b), _t(T), _t(Wt), _t(C), v, _t(poses, torch.float32), _t(K, torch.float32), size, **kw)
    return {k: x.cpu().numpy() for k, x in out.items()}


def _random_cameras(r, C, dist=(2.4, 3.2)):
    eyes = r.normal(size=(C, 3))
    eyes *= r.uniform(*dist, (C, 1)) / np.linalg.norm(eyes, axis=1, keepdims=True)
    return np.stack([_look_at(e, r.normal(0, 0.1, 3), up=(0.0, 0.0, 1.0) if abs(e[2]) < 2.0 else (0.0, 1.0, 0.0))
                     for e in eyes]).astype(np.float32)


# ------------------------------------------------------------------------------------------------ (1)
def test_planted_plane_exact():
    v = 0.25
    vol = _field_volume(lambda X: np.clip((8.5 * v - X[..., 2]) / (4 * v), -1, 1), v, np.array([-16, -16, 0]),
                        np.array([15, 15, 15]))
    b, T, Wt, _ = vol
    C = np.full(T.shape + (3,), 0.375, np.float32)
    K = np.array([[8.0, 0, 8], [0, 8.0, 6], [0, 0, 1]], np.float32)
    out = _cast((b, T, Wt, C), v, np.eye(4, dtype=np.float32)[None], K, (12, 16))
    zp = np.float32(8.5 * v)
    assert (out["depth"] > 0).all()
    assert (np.abs(out["depth"] - zp) <= np.spacing(zp)).all(), np.abs(out["depth"] - zp).max()
    np.testing.assert_array_equal(out["normal"], np.broadcast_to(np.float32([0, 0, -1]), out["normal"].shape))
    assert (np.abs(out["color"] - np.float32(0.375)) <= np.spacing(np.float32(0.375))).all()


# ------------------------------------------------------------------------------------------------ (2)
def _volume(shape, seed):
    r = np.random.default_rng(seed)
    if shape == "sphere":
        v = 0.1
        vol = _field_volume(lambda X: np.linalg.norm(X, axis=-1) - 1.0, v, np.array([-14] * 3), np.array([13] * 3))
    elif shape == "torus":
        v = 0.05
        f = lambda X: np.hypot(np.hypot(X[..., 0], X[..., 1]) - 1.0, X[..., 2]) - 0.4
        vol = _field_volume(f, v, np.array([-32, -32, -10]), np.array([31, 31, 9]))
    else:  # a sphere's distance field with noise on the samples near it: saddles everywhere
        v = 0.05
        vol = _field_volume(lambda X: np.linalg.norm(X, axis=-1) - 1.0, v, np.array([-32] * 3), np.array([31] * 3))
        T = vol[1]
        T += (0.08 * r.uniform(-1, 1, T.shape) * (np.abs(T) < 0.3)).astype(np.float32)
    b, T, _, X = vol
    # partial weights: blobs of weight 1 that min_weight 2 cuts out, and a few unobserved samples
    Xd = X.astype(np.float64)
    Wt = np.where(np.sin(4 * Xd[..., 0] + seed) + np.sin(3 * Xd[..., 1]) > 0.8, 1.0, 2.0).astype(np.float32)
    Wt[r.uniform(size=T.shape) < 1e-3] = 0.0
    C = (0.5 + 0.25 * np.sin(3.0 * X.astype(np.float64))).astype(np.float32)
    return (b, T, Wt, C), v


@pytest.mark.parametrize("shape, C, mw, seed", [
    ("sphere", 1, 1, 0), ("sphere", 17, 2, 1), ("torus", 3, 1, 2), ("torus", 17, 2, 3), ("noisy", 3, 2, 4),
    ("noisy", 17, 1, 5), ("noisy", 1, 1, 6)])
def test_random_fields_against_fp64(shape, C, mw, seed):
    vol, v = _volume(shape, seed)
    r = np.random.default_rng(100 + seed)
    poses = _random_cameras(r, C)
    Ho, Wo = (24, 32) if C > 3 else (48, 64)
    K = np.stack([_K(r.uniform(30, 60) * Wo / 64, Wo / 2 - r.uniform(0, 1), Ho / 2 - r.uniform(0, 1)) for _ in range(C)])
    got = _cast(vol, v, poses, K, (Ho, Wo), min_weight=mw)
    want = ro.raycast(fo.key(vol[0]), *vol[1:], v, poses, K, (Ho, Wo), min_weight=mw)
    clean = ~want["ambiguous"]
    gh = got["depth"] > 0
    assert want["hit"][clean].sum() > 0.05 * clean.size
    np.testing.assert_array_equal(gh[clean], want["hit"][clean])
    both = gh & want["hit"]
    z = want["depth"][both]
    ratio = np.abs(got["depth"][both] - z) / (1e-4 * v + 1e-6 * z)
    assert ratio.max() <= 1, ratio.max()
    assert np.abs(got["color"][both] - want["color"][both]).max() <= 1e-5
    assert np.abs(got["normal"][both] - want["normal"][both]).max() <= 1e-3
    assert np.abs(got["rgb"][both] - want["rgb"][both]).max() <= 1e-3
    miss = ~gh
    assert (got["color"][miss] == 1.0).all() and (got["rgb"][miss] == 1.0).all() and (got["normal"][miss] == 0).all()
    print("%s C=%d mw=%d: %d px, %d hit, %d ambiguous, depth error up to %.2f of its bound" % (
        shape, C, mw, gh.size, gh.sum(), (~clean).sum(), ratio.max()))


# ------------------------------------------------------------------------------------------------ (3)
def test_hits_lie_in_meshed_cubes_near_their_vertices():
    from scipy.spatial import cKDTree
    from vista_slam_b200.fusion import marching_cubes
    vol, v = _volume("noisy", 7)
    b, T, Wt, C = vol
    # every sample observed: no step of a ray crosses an unmeshed cube between two meshed ones
    Wt = np.ones_like(Wt)
    vol = (b, T, Wt, C)
    mesh = marching_cubes(_t(b), _t(T), _t(Wt), _t(C), v)
    verts = mesh["vertices"].cpu().numpy().astype(np.float64)
    r = np.random.default_rng(8)
    poses = _random_cameras(r, 3)
    K = _K(50.0, 31.5, 23.5)
    got = _cast(vol, v, poses, K, (48, 64))
    V = ro._Volume(fo.key(b), T, Wt, C, v, 1)
    tree = cKDTree(verts)
    checked = 0
    for c in range(3):
        row, col = np.nonzero(got["depth"][c] > 0)
        P = poses[c].astype(np.float64)
        dc = np.stack([(col - K[0, 2]) / K[0, 0], (row - K[1, 2]) / K[1, 1], np.ones(len(col))], -1)
        p = P[:3, 3] + got["depth"][c][row, col][:, None].astype(np.float64) * (dc @ P[:3, :3].T)
        for q in p:
            # the cells within 1e-4 v of the hit
            cands = {tuple(np.floor((q + (np.array(o) - 1) * 1e-4 * v) / v).astype(int)) for o in np.ndindex(3, 3, 3)}
            ok = False
            for cell in cands:
                pc = (np.array(cell) + 0.5) * v
                valid, g, _ = V.corners(pc[None])
                signs = V.T[g[0]] < 0
                if not (valid[0] and signs.any() and not signs.all()):
                    continue  # marching cubes' case 0 or 255, or an unmeshed cube
                near = tree.query_ball_point(q, np.sqrt(3) * v + 1e-6)
                lo, hi = np.array(cell) * v - 1e-5 * v, (np.array(cell) + 1) * v + 1e-5 * v
                if any(((verts[i] >= lo) & (verts[i] <= hi)).all() for i in near):
                    ok = True
                    break
            assert ok, (c, q)
            checked += 1
    assert checked > 1000


# ------------------------------------------------------------------------------------------------ (4)
def _sphere_maps(R=1.0, H=64, W=64, f=60.0):
    """test_fusion_gpu's 26 ray-cast views of a sphere of radius R."""
    K = _K(f, W / 2 - 0.5, H / 2 - 0.5).astype(np.float64)
    dirs = [np.array(d, np.float64) for d in np.ndindex(3, 3, 3) if d != (1, 1, 1)]
    poses, depths = [], []
    for d in dirs:
        d = (d - 1) / np.linalg.norm(d - 1)
        P = _look_at(3.0 * d, np.zeros(3), up=(0.0, 0.0, 1.0) if abs(d[2]) < 0.9 else (0.0, 1.0, 0.0))
        yy, xx = np.mgrid[0:H, 0:W]
        ray = np.linalg.inv(K) @ np.stack([xx.ravel(), yy.ravel(), np.ones(H * W)])
        rw = P[:3, :3] @ ray
        o = P[:3, 3][:, None]
        a, b, c = (rw * rw).sum(0), 2 * (o * rw).sum(0), (o * o).sum() - R * R
        disc = b * b - 4 * a * c
        poses.append(P)
        depths.append(np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), 0.0).reshape(H, W))
    V = len(poses)
    d = np.stack(depths).astype(np.float32)
    maps = {"pose": np.stack(poses).astype(np.float32), "scale": np.ones((V, 1), np.float32), "depth": d,
            "conf": np.where(d > 0, 1.0, 0.0).astype(np.float32), "intri": np.stack([K] * V).astype(np.float32),
            "images": np.zeros((V, 3, H, W), np.float32)}
    return {k: _t(x) for k, x in maps.items()}


def _erode(mask, r=2):
    out = mask.copy()
    H, W = mask.shape
    pad = np.pad(mask, r, constant_values=False)
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            out &= pad[r + dy:r + dy + H, r + dx:r + dx + W]
    return out


def test_fused_sphere_from_new_cameras():
    from vista_slam_b200.fusion import fuse_volume, raycast
    R, v = 1.0, 0.04
    vol = fuse_volume(_sphere_maps(R), 0.5, v)
    r = np.random.default_rng(9)
    poses = _random_cameras(r, 4, dist=(2.5, 3.5))
    K = _K(70.0, 39.5, 29.5)
    out = raycast(vol["bricks"], vol["tsdf"], vol["weight"], vol["color"], v, _t(poses), _t(K), (60, 80))
    depth = out["depth"].cpu().numpy()
    for c in range(4):
        P = poses[c].astype(np.float64)
        row, col = np.mgrid[0:60, 0:80]
        d = np.stack([(col - K[0, 2]) / K[0, 0], (row - K[1, 2]) / K[1, 1], np.ones((60, 80))], -1) @ P[:3, :3].T
        o = P[:3, 3]
        disc = (d @ o) ** 2 - (d * d).sum(-1) * (o @ o - R * R)
        hit = depth[c] > 0
        p = o + depth[c][hit][:, None] * d[hit]
        dist = np.abs(np.linalg.norm(p, axis=1) - R)
        assert dist.max() <= 4 * v and dist.mean() < 0.5 * v, (dist.max(), dist.mean())
        inner = _erode(disc > 0)
        assert inner.sum() > 500 and hit[inner].all(), (~hit[inner]).sum()


def _box_depth(eye, d, boxes):
    """Analytic depth (ray parameter) and (box, face) id of rays eye + t d [n,3] in fusion_stream's room."""
    best = np.full(len(d), np.inf)
    face = np.full(len(d), -1)
    for bi, (lo, hi, inside) in enumerate(boxes):
        lo, hi = np.array(lo), np.array(hi)
        with np.errstate(divide="ignore", invalid="ignore"):
            t0, t1 = (lo - eye) / d, (hi - eye) / d
        tn, tf = np.minimum(t0, t1), np.maximum(t0, t1)
        t = np.where(inside, tf.min(1), np.where((tn.max(1) <= tf.min(1)) & (tn.max(1) > 0), tn.max(1), np.inf))
        ax = np.where(inside, tf.argmin(1), tn.argmax(1))
        sel = t < best
        best[sel] = t[sel]
        face[sel] = bi * 6 + ax[sel] * 2 + (d[sel, ax[sel]] > 0)
    return best, face


def test_fused_room_from_new_cameras_against_the_analytic_depth():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import fusion_stream as fs
    from vista_slam_b200.fusion import fuse_volume, raycast
    v = 0.04
    vol = fuse_volume(fs.room(100), 0.5, v)
    Ho, Wo = 96, 128
    K = _K(100.0, Wo / 2 - 0.5, Ho / 2 - 0.5).astype(np.float64)
    r = np.random.default_rng(12)
    poses = []
    for k in range(4):
        a = 2 * np.pi * (k + 0.37) / 4
        eye = np.array([1.2 * np.cos(a), 0.1, 2.0 * np.sin(a)]) + r.normal(0, 0.05, 3)
        poses.append(fs._look_at(eye, np.array([0.0, -0.5, 0.0]) + r.normal(0, 0.3, 3)))
    poses = np.stack(poses)
    out = raycast(vol["bricks"], vol["tsdf"], vol["weight"], vol["color"], v, _t(poses, torch.float32),
                  _t(K, torch.float32), (Ho, Wo))
    depth = out["depth"].cpu().numpy()
    errs = []
    for c in range(4):
        P = poses[c]
        row, col = np.mgrid[0:Ho, 0:Wo]
        d = (np.stack([(col - K[0, 2]) / K[0, 0], (row - K[1, 2]) / K[1, 1], np.ones((Ho, Wo))], -1) @ P[:3, :3].T)
        t, face = _box_depth(P[:3, 3], d.reshape(-1, 3), fs.BOXES)
        face = face.reshape(Ho, Wo)
        same = np.ones((Ho, Wo), bool)
        pad = np.pad(face, 2, constant_values=-2)
        for dy in range(-2, 3):
            for dx in range(-2, 3):
                same &= pad[2 + dy:2 + dy + Ho, 2 + dx:2 + dx + Wo] == face
        keep = same & np.isfinite(t.reshape(Ho, Wo))
        assert keep.sum() > 0.5 * keep.size
        # the camera z of the analytic hit is its ray parameter (the ray's camera-frame z is 1)
        errs.append(np.abs(depth[c][keep] - t.reshape(Ho, Wo)[keep]) * np.linalg.norm(d[keep], axis=-1))
    e = np.concatenate(errs)
    print("room: median %.4f v, p99 %.3f v" % (np.median(e) / v, np.percentile(e, 99) / v))
    assert np.median(e) < v / 4 and np.percentile(e, 99) < 4 * v


# ------------------------------------------------------------------------------------------------ (5)
def test_deterministic_camera_independent_read_only_and_no_sync():
    from vista_slam_b200.fusion import _raycast, brick_keys
    vol, v = _volume("noisy", 10)
    t = [_t(x) for x in vol]
    before = [x.clone() for x in t]
    keys = brick_keys(t[0]).contiguous()
    poses = _t(_random_cameras(np.random.default_rng(11), 5))
    K = _t(np.stack([_K(40.0 + 3 * c, 31.5, 23.5) for c in range(5)]), torch.float32)
    args = (keys, t[1], t[2], t[3], v, 2.0, poses, K, (48, 64), 1e-3, (0.0, 0.25, 1.0))
    a = _raycast(*args)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = _raycast(*args)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in a:
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k
    for c in range(5):
        one = _raycast(keys, t[1], t[2], t[3], v, 2.0, poses[c:c + 1], K[c:c + 1], (48, 64), 1e-3, (0.0, 0.25, 1.0))
        for k in a:
            assert torch.equal(one[k][0].view(torch.int32), a[k][c].view(torch.int32)), (k, c)
    for x, y in zip(t, before):
        assert torch.equal(x, y)
    assert (a["depth"] > 0).any() and (a["depth"] == 0).any()


# ------------------------------------------------------------------------------------------------ (6)
def _same(a, b):
    for k in a:
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k


def _cams(slam, ks):
    views = [slam.get_view(k) for k in ks]
    return torch.stack([x.pose for x in views]).cuda(), torch.stack([x.intri for x in views]).cuda()


def test_render_surface_equals_fuse_volume_and_raycast_read_only():
    from vista_slam_b200.fusion import _mesh, brick_keys, fuse_views, fuse_volume, raycast
    slam, stream = _replayed()
    v, _ = _voxel_of(slam)
    P, K = _cams(slam, range(0, 18, 4))
    size = (stream["H"], stream["W"])
    G = slam._graph
    tables = {k: getattr(G, k).clone() for k in ("pose", "depth", "conf", "intri", "cmean", "node_to_view",
                                                    "node_to_connected_view", "best_node", "best_mean", "edges", "meas",
                                                    "weight")}
    times = dict(slam.time_dict)
    host = (dict(slam.view_to_node), list(slam.node_to_connected_view), slam.num_nodes, slam.num_edges, slam.view_num)
    got = slam.render_surface(P, K, size, v, min_weight=2)
    vol = fuse_volume(slam._view_maps(None), slam.conf_thres, v)
    _same(got, raycast(vol["bricks"], vol["tsdf"], vol["weight"], vol["color"], v, P, K, size, min_weight=2))
    assert (got["depth"] > 0).sum() > 0.2 * got["depth"].numel()
    _same(got, slam.render_surface(P, K, size, v, min_weight=2))
    # views and min_consistent_views
    part = slam.render_surface(P, K, size, v, views=range(3, 12), min_consistent_views=2)
    maps = slam._consistent_maps(slam._view_maps(range(3, 12)), 2)
    vol2 = fuse_volume(maps, slam.conf_thres, v)
    _same(part, raycast(vol2["bricks"], vol2["tsdf"], vol2["weight"], vol2["color"], v, P, K, size))
    assert not torch.equal(part["depth"], slam.render_surface(P, K, size, v)["depth"])
    # fuse_volume + _mesh is fuse_views
    whole = fuse_views(slam._view_maps(None), slam.conf_thres, v, min_weight=2)
    mesh = _mesh(brick_keys(vol["bricks"]).contiguous(), vol["tsdf"], vol["weight"], vol["color"], float(np.float32(v)), 2.0)
    for k in ("bricks", "tsdf", "weight", "color"):
        assert torch.equal(whole[k], vol[k]), k
    for k in mesh:
        assert torch.equal(whole[k], mesh[k]), k
    for k, t in tables.items():
        assert torch.equal(getattr(G, k).view(torch.uint8), t.view(torch.uint8)), k
    assert slam.time_dict == times
    assert host == (dict(slam.view_to_node), list(slam.node_to_connected_view), slam.num_nodes, slam.num_edges,
                    slam.view_num)
    with pytest.raises(IndexError):
        slam.render_surface(P, K, size, v, views=range(0, slam.view_num + 1))


def test_background_pgo_render_surface_equals_synchronous():
    stream = so.make_stream()
    images = so.stream_images(stream)
    sync = _replay_slam(stream)
    bg = _replay_slam(stream)
    bg.pgo_background = True
    for i in range(14):
        sync.step(_value(images, i, stream))
        bg.step(_value(images, i, stream))
    bg.wait_pgo()
    v, _ = _voxel_of(sync)
    P, K = _cams(sync, [2, 9])
    a = sync.render_surface(P, K, (stream["H"], stream["W"]), v)
    b = bg.render_surface(P, K, (stream["H"], stream["W"]), v)
    _same(a, b)


def test_real_frontend_render_surface(cuda_model):
    import vista_slam_b200.slam as S

    class Run(S.OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return cuda_model

    slam = Run("unused", VOCAB, verbose=False, loop_dist_min=4, pgo_every=5, rel_pose_thres=0.5)
    frames = _frames_224(12)
    for i in range(12):
        slam.step(frames[i], force_pgo=(i == 11))
    ex = slam._export(0, slam.view_num, cloud=False)
    d = (ex["depth"] * ex["scale"][:, :, None])[ex["conf"] > slam.conf_thres]
    v = float(d[d > 0].median()) / 16.0
    P, K = _cams(slam, [0, slam.view_num - 1])
    out = slam.render_surface(P, K, (112, 112), v)
    print("real frontend: %d of %d pixels hit" % (int((out["depth"] > 0).sum()), out["depth"].numel()))
    assert (out["depth"] > 0).any()
    assert torch.isfinite(out["rgb"]).all()


# ------------------------------------------------------------------------------------------------ (7)
def test_render_video_surface_makes_the_frame_sequence(tmp_path):
    stream = so.make_stream()
    images = so.stream_images(stream)
    slam = _replay_slam(stream)
    n = stream["n_views"]
    run = tmp_path / "run"
    pgo_at = []
    for i in range(n):
        if slam.step(_value(images, i, stream), force_pgo=(i == n - 1), log_intermediate_results=True,
                     output_folder=str(run)):
            pgo_at.append(i)
    slam.save_data_all(str(run))
    v, _ = _voxel_of(slam)
    out = tmp_path / "frames"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "render_video.py"), str(run), "--out", str(out),
                        "--size", "96x128", "--surface", repr(v), "--min-weight", "1"], capture_output=True, text=True,
                       cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    files = sorted(os.listdir(out))
    names = {os.path.splitext(f)[0] for f in files}
    assert names == {"%04d" % k for k in range(n)} | {"%04d_pgo" % k for k in pgo_at}, files
