"""GPU: the map renderer (csrc/render.cu, vista_slam_b200/render.py, OnlineSLAM.render).

  1. Planted scenes where every float32 operation is exact (power-of-two focal lengths, integer principal points,
     identity or axis-permutation poses, power-of-two depths): occluders, ties, radius 0 / 1 / 2, a camera facing away,
     the near plane, segments in front of and behind a plane of points.  rgb, depth and index bit for bit.
  2. Random scenes against the float64 oracle (oracle/render_oracle.py) at C = 1, 3, 17.  Unambiguous pixels: index
     equal, depth within 1e-6 relative, rgb bit-equal to the winner's (img + 1) / 2.  Ambiguous pixels (a candidate
     within 1e-3 px of a pixel boundary, or the two nearest depths within 1e-5 relative): index among the oracle's
     candidates.
  3. A replayed OnlineSLAM run: view k from its own pose and intrinsics lands every confident pixel on itself.
  4. Every drawn point is the PLY's point of _export(cloud=True): it projects into the splat's footprint and has its
     colour, on the replayed run and on a run of the real frontend.
  5. Repeated calls and one-camera calls give the same bits; render leaves the graph and time_dict as they were and
     does not synchronise with the host.
  6. After a background PGO is folded, a render equals the synchronous run's.
  7. Tracked frames' poses render one image each.
  8. Refusals: a view without a node (IndexError), size, radius and id range (ValueError), before any launch.
  9. tools/render_video.py makes the whole frame sequence from the files of a run with log_intermediate_results."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import render_oracle as ro
from oracle import slam_oracle as so
from test_slam_batch_gpu import _frames_224
from test_slam_gpu import VOCAB, _replay_slam, _value

pytestmark = pytest.mark.gpu


def _dev(maps):
    return {k: torch.as_tensor(np.ascontiguousarray(v, dtype=np.float32)).cuda() for k, v in maps.items()}


def _grid_maps(depths, pose=None, seed=0):
    """Views of H x W pixels with K = I: pixel (col, row) at depth d is (col d, row d, d) in the view's frame; every
    pixel confident unless its depth is 0; images random in [-1, 1] on a 2^-7 grid."""
    d = np.asarray(depths, np.float32)
    V, H, W = d.shape
    r = np.random.default_rng(seed)
    return {"pose": np.tile(np.eye(4, dtype=np.float32) if pose is None else pose, (V, 1, 1)),
            "scale": np.ones((V, 1), np.float32), "depth": d, "conf": np.where(d > 0, 10.0, 0.0).astype(np.float32),
            "intri": np.tile(np.eye(3, dtype=np.float32), (V, 1, 1)),
            "images": (np.rint(r.uniform(-128, 128, (V, 3, H, W))) / 128).astype(np.float32)}


def _K(f, cx, cy):
    return np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]], np.float64)


def _render(maps, poses, K, size, **kw):
    from vista_slam_b200.render import render_views
    out = render_views(_dev(maps), 4.2, torch.as_tensor(np.asarray(poses, np.float64)), torch.as_tensor(K), size, **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _oracle(maps, poses, K, size, radius=0, near=1e-3, lines=None):
    C = len(poses)
    w2c = np.linalg.inv(np.asarray(poses, np.float64))
    Ks = np.broadcast_to(np.asarray(K, np.float64), (C, 3, 3))
    segs, cols = lines if lines is not None else (None, None)
    return ro.render(maps, 4.2, w2c, Ks, size, radius=radius, near=near, segs=segs, seg_colors=cols)


def _assert_exact(got, want):
    np.testing.assert_array_equal(got["index"], want["index"])
    np.testing.assert_array_equal(got["depth"], want["depth"].astype(np.float32))
    np.testing.assert_array_equal(got["rgb"], want["rgb"])


# ------------------------------------------------------------------------------------------------ (1)
PERM = np.array([[0, 1, 0, 0], [0, 0, 1, 0], [1, 0, 0, 0], [0, 0, 0, 1]], np.float64)  # axis permutation, det +1


@pytest.mark.parametrize("radius", [0, 1, 2])
@pytest.mark.parametrize("frame", ["identity", "permuted"])
def test_planted_scenes_bit_for_bit(radius, frame):
    # view 0: a 4 x 4 plane at z = 2 with one occluder at z = 1 and one pixel at z = 2 tying with view 1's;
    # view 1: a pixel in front of the plane (z = 1) and one at the plane's depth (a tie at the same image position)
    d0 = np.full((4, 4), 2.0)
    d0[1, 2] = 1.0
    d1 = np.zeros((4, 4))
    d1[2, 1], d1[3, 3] = 1.0, 2.0
    P = np.eye(4) if frame == "identity" else PERM
    maps = _grid_maps(np.stack([d0, d1]), pose=P.astype(np.float32))
    K = _K(4.0, 8.0, 8.0)
    segs = np.array([[[-1.0, 0.5, 1.0], [1.0, 0.5, 1.0]],    # in front of the plane: x 4 .. 12 on row 10, z = 1
                     [[-2.0, 4.0, 4.0], [2.0, 4.0, 4.0]],    # behind it: x 6 .. 10 on row 12, z = 4
                     [[0.0, 0.0, 0.5], [0.0, 0.0, -1.0]]])   # crosses the near plane (0.25): clipped, on pixel (8, 8)
    segs_w = segs @ P[:3, :3].T  # the same segments in the permuted world
    cols = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])
    poses = np.stack([P, P @ np.diag([-1.0, 1.0, -1.0, 1.0])])  # camera 1 faces away from everything
    got = _render(maps, poses, K, (24, 24), point_radius=radius, near=0.25, lines=(segs_w, cols))
    want = _oracle(_grid_maps(np.stack([d0, d1])), np.stack([np.eye(4), np.diag([-1.0, 1, -1, 1])]), K, (24, 24),
                   radius=radius, near=0.25, lines=(segs, cols))
    _assert_exact(got, want)
    HW = 16
    # camera 1 faces away from every point and from segments 0 and 1; the far end of segment 2 (z = -1) is in front
    assert set(np.unique(got["index"][1]).tolist()) <= {-1, 2 * HW + 2}
    assert ((got["index"][1] == -1) == (got["depth"][1] == 0)).all() and (got["rgb"][1][got["index"][1] == -1] == 1).all()
    idx = got["index"][0]
    assert idx[8 + 4, 8 + 8] == 1 * 4 + 2 and got["depth"][0, 12, 16] == 1.0  # the occluder
    assert idx[8 + 12, 8 + 12] == 15  # tie at z = 2 with view 1's (3, 3): the lower id
    assert idx[10, 4] == 2 * HW and got["depth"][0, 10, 4] == 1.0  # the front segment, left of the plane
    if radius < 2:  # (at radius 2 the front segment's footprint reaches row 12)
        assert idx[12, 8] == 4  # the plane's point hides the segment behind it
    if radius == 0:
        assert idx[12, 6] == 2 * HW + 1 and got["depth"][0, 12, 6] == 4.0  # beside the point, the segment shows
    assert idx[8, 8] == 2 * HW + 2 and got["depth"][0, 8, 8] == 0.5  # the clipped segment, in front of point 0
    for v, row, col in ((0, 3, 1), (1, 2, 1)):  # pixels no line reaches
        i = v * HW + row * 4 + col
        np.testing.assert_array_equal(got["rgb"][0, 8 + 4 * row, 8 + 4 * col], (maps["images"][v, :, row, col] + 1) / 2)
        assert idx[8 + 4 * row, 8 + 4 * col] == i


# ------------------------------------------------------------------------------------------------ (2)
def _random_scene(seed, C):
    r = np.random.default_rng(seed)
    V, H, W = 3, 12, 16
    maps = {"pose": np.zeros((V, 4, 4), np.float32), "scale": r.uniform(0.8, 1.25, (V, 1)).astype(np.float32),
            "depth": r.uniform(1.0, 3.0, (V, H, W)).astype(np.float32),
            "conf": r.uniform(1.0, 8.0, (V, H, W)).astype(np.float32),
            "intri": np.zeros((V, 3, 3), np.float32), "images": r.uniform(-1, 1, (V, 3, H, W)).astype(np.float32)}
    for v in range(V):
        maps["pose"][v] = np.eye(4)
        maps["pose"][v, :3, :3] = so._rotvec_to_rot(0.2 * r.standard_normal(3))
        maps["pose"][v, :3, 3] = 0.3 * r.standard_normal(3)
        maps["intri"][v] = _K(r.uniform(12, 18), W / 2, H / 2)
    poses = np.zeros((C, 4, 4))
    for c in range(C):
        poses[c] = np.eye(4)
        poses[c, :3, :3] = so._rotvec_to_rot(0.15 * r.standard_normal(3))
        poses[c, :3, 3] = 0.4 * r.standard_normal(3) - [0, 0, 1.0]
    K = np.stack([_K(r.uniform(20, 40), r.uniform(20, 28), r.uniform(16, 24)) for _ in range(C)])
    return maps, poses, K


@pytest.mark.parametrize("C", [1, 3, 17])
@pytest.mark.parametrize("radius", [0, 1])
def test_random_scenes_against_fp64(C, radius):
    maps, poses, K = _random_scene(100 + C, C)
    size = (40, 48)
    got = _render(maps, poses, K, size, point_radius=radius)
    want = _oracle(maps, poses, K, size, radius=radius)
    amb = want["ambiguous"]
    sure = ~amb
    np.testing.assert_array_equal(got["index"][sure], want["index"][sure])
    hit = sure & (want["index"] >= 0)
    assert hit.sum() > 100
    rel = np.abs(got["depth"][hit] - want["depth"][hit]) / want["depth"][hit]
    assert rel.max() <= 1e-6, rel.max()
    imgs = maps["images"]
    H, W = imgs.shape[2:]
    ids = got["index"][hit]
    v, pix = ids // (H * W), ids % (H * W)
    np.testing.assert_array_equal(got["rgb"][hit], (imgs[v, :, pix // W, pix % W] + np.float32(1)) / np.float32(2))
    for c, y, x in zip(*np.nonzero(amb)):
        assert got["index"][c, y, x] in want["accept"][(c, y, x)], (c, y, x)
    print("C=%d r=%d: %d of %d pixels ambiguous" % (C, radius, amb.sum(), amb.size))


# ------------------------------------------------------------------------------------------------ (3) (4)
def _replayed(n=None, **over):
    stream = so.make_stream()
    slam = _replay_slam(stream, **over)
    images = so.stream_images(stream)
    n = stream["n_views"] if n is None else n
    for i in range(n):
        slam.step(_value(images, i, stream), force_pgo=(i == n - 1))
    return slam, stream


def test_self_view_lands_every_pixel_on_itself():
    slam, stream = _replayed()
    H, W = stream["H"], stream["W"]
    for k in (0, 7, stream["n_views"] - 1):
        view = slam.get_view(k, filter_outlier=False)
        out = slam.render(view.pose[None], view.intri, (H, W), views=range(k, k + 1))
        ex = slam._export(k, 1, cloud=False)
        conf = ex["conf"][0].cpu().numpy()
        mask = conf > slam.conf_thres
        idx = out["index"][0].cpu().numpy()
        np.testing.assert_array_equal(idx[mask], np.flatnonzero(mask.reshape(-1)))
        assert (idx[~mask] == -1).all()
        want = (ex["depth"][0] * ex["scale"][0]).cpu().numpy()
        np.testing.assert_allclose(out["depth"][0].cpu().numpy()[mask], want[mask], rtol=2e-6, atol=0)
        img = slam.imgs[k].float().numpy()
        np.testing.assert_array_equal(out["rgb"][0].cpu().numpy()[mask], ((img + 1) / 2).transpose(1, 2, 0)[mask])
        assert (out["rgb"][0].cpu().numpy()[~mask] == 1).all()


def _check_against_ply(slam, poses, K, size, radius, slack=0.0):
    """Every drawn point against the PLY: its fp64 projection within the footprint (radius + 0.5 px, plus 1e-3 px and
    `slack` times the float32 rounding of the projection, |x| f / z ulps, for far-out points of random weights) and
    its colour bit for bit.  Returns the render and the number of drawn pixels."""
    n = slam.view_num
    out = slam.render(poses, K, size, point_radius=radius, views=range(n))
    ex = slam._export(0, n, cloud=True)
    cnt = int(ex["count"])
    pts, cols = ex["points"][:cnt].cpu().numpy().astype(np.float64), ex["colors"][:cnt].cpu().numpy()
    conf = ex["conf"].cpu().numpy().reshape(-1)
    confident = np.flatnonzero(conf > slam.conf_thres)
    assert len(confident) == cnt
    idx = out["index"].cpu().numpy()
    w2c = np.linalg.inv(np.asarray(poses, np.float64))
    Ks = np.broadcast_to(np.asarray(K, np.float64), (len(w2c), 3, 3))
    drawn = 0
    for c in range(len(w2c)):
        ys, xs = np.nonzero((idx[c] >= 0) & (idx[c] < len(conf)))
        rank = np.searchsorted(confident, idx[c][ys, xs])
        np.testing.assert_array_equal(confident[rank], idx[c][ys, xs])
        q = pts[rank] @ w2c[c, :3, :3].T + w2c[c, :3, 3]
        uvw = q @ Ks[c].T
        u, v = uvw[:, 0] / uvw[:, 2], uvw[:, 1] / uvw[:, 2]
        f = np.abs(Ks[c]).max()
        tol = radius + 0.5 + 1e-3 + slack * 6e-8 * f * np.abs(q).sum(1) / np.abs(q[:, 2])
        assert (np.abs(u - xs) <= tol).all() and (np.abs(v - ys) <= tol).all()
        np.testing.assert_array_equal(out["rgb"][c].cpu().numpy()[ys, xs], cols[rank])
        drawn += len(ys)
    return out, drawn


def test_render_agrees_with_the_ply():
    slam, stream = _replayed()
    view = slam.get_view(3)
    back = view.pose.numpy().astype(np.float64) @ np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, -2.0], [0, 0, 0, 1]])
    poses = np.stack([view.pose.numpy(), back])
    _, drawn = _check_against_ply(slam, poses, view.intri.numpy(), (64, 80), 1)
    assert drawn > 1000


def test_real_frontend_render_agrees_with_the_ply_and_tracked_frames_render(cuda_model):
    import vista_slam_b200.slam as S

    class Run(S.OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return cuda_model

    slam = Run("unused", VOCAB, verbose=False, loop_dist_min=4, pgo_every=5, rel_pose_thres=0.5)
    frames = _frames_224(14)
    for i in range(12):
        slam.step(frames[i], force_pgo=(i == 11))
    view = slam.get_view(5)
    _, drawn = _check_against_ply(slam, view.pose[None].numpy(), view.intri.numpy(), (224, 224), 0, slack=64)
    print("real frontend: %d pixels drawn" % drawn)
    # (7) tracked frames: one image per frame trajectory pose
    slam.track(frames[12:14])
    traj = slam.frame_trajectory()
    out = slam.render(traj["pose"], view.intri, (120, 160), point_radius=1)
    assert out["rgb"].shape == (2, 120, 160, 3) and out["depth"].shape == (2, 120, 160)
    assert out["index"].shape == (2, 120, 160) and out["index"].dtype == torch.int64


# ------------------------------------------------------------------------------------------------ (5)
def test_deterministic_one_camera_calls_read_only_and_no_sync():
    slam, stream = _replayed()
    G = slam._graph
    tables = {k: getattr(G, k).clone() for k in ("pose", "depth", "conf", "intri", "cmean", "node_to_view",
                                                    "node_to_connected_view", "best_node", "best_mean", "edges", "meas",
                                                    "weight")}
    times = dict(slam.time_dict)
    host = (dict(slam.view_to_node), list(slam.node_to_connected_view), slam.num_nodes, slam.num_edges, slam.view_num)
    views = [slam.get_view(k) for k in range(0, 18, 3)]
    K = torch.stack([v.intri for v in views]).cuda()
    P = torch.stack([v.pose for v in views]).double().cuda()
    g = torch.Generator().manual_seed(11)  # a scene of its own, whatever ran before in the session
    segs = torch.randn(40, 2, 3, generator=g).cuda()
    cols = torch.rand(40, 3, generator=g).cuda()
    a = slam.render(P, K, (48, 64), point_radius=2, lines=(segs, cols))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = slam.render(P, K, (48, 64), point_radius=2, lines=(segs, cols))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    for c in range(len(views)):
        one = slam.render(P[c:c + 1], K[c], (48, 64), point_radius=2, lines=(segs, cols))
        for k in a:
            assert torch.equal(one[k][0], a[k][c]), (k, c)
    assert (a["index"] >= 0).any()
    # bytes, not values: the rows past the inserted nodes are never written and may hold NaN bit patterns
    for k, t in tables.items():
        assert torch.equal(getattr(G, k).view(torch.uint8), t.view(torch.uint8)), k
    assert slam.time_dict == times
    assert host == (dict(slam.view_to_node), list(slam.node_to_connected_view), slam.num_nodes, slam.num_edges,
                    slam.view_num)


# ------------------------------------------------------------------------------------------------ (6)
def test_background_pgo_render_equals_synchronous():
    stream = so.make_stream()
    images = so.stream_images(stream)
    sync = _replay_slam(stream)
    bg = _replay_slam(stream)
    bg.pgo_background = True
    n = 14
    for i in range(n):
        sync.step(_value(images, i, stream))
        bg.step(_value(images, i, stream))
    bg.wait_pgo()
    view = sync.get_view(9)
    poses = np.stack([view.pose.numpy(), np.eye(4)])
    a = sync.render(poses, view.intri, (48, 64), point_radius=1)
    b = bg.render(poses, view.intri, (48, 64), point_radius=1)
    for k in a:
        assert torch.equal(a[k], b[k]), k


# ------------------------------------------------------------------------------------------------ (8)
def test_refusals_before_any_launch():
    from vista_slam_b200.render import render_views
    slam, stream = _replayed(n=5)
    pose, K = slam.get_view(2).pose[None], slam.get_view(2).intri
    with pytest.raises(IndexError):
        slam.render(pose, K, (32, 40), views=range(0, 6))
    for kw in (dict(size=(0, 40)), dict(size=(32, 9000)), dict(point_radius=5), dict(point_radius=-1)):
        args = dict(size=(32, 40))
        args.update(kw)
        with pytest.raises(ValueError):
            slam.render(pose, K, **args)
    with pytest.raises(ValueError, match="view"):
        slam.render(pose, K, (32, 40), views=[0, 1])
    V, H, W = 65535, 256, 257
    big = {"pose": torch.eye(4, device="cuda").expand(V, 4, 4), "scale": torch.ones(1, 1, device="cuda").expand(V, 1),
           "depth": torch.ones(1, 1, 1, device="cuda").expand(V, H, W),
           "conf": torch.ones(1, 1, 1, device="cuda").expand(V, H, W),
           "intri": torch.eye(3, device="cuda").expand(V, 3, 3),
           "images": torch.zeros(1, 1, 1, 1, device="cuda").expand(V, 3, H, W)}
    with pytest.raises(ValueError, match="32-bit"):
        render_views(big, 4.2, pose, K, (32, 40))


# ------------------------------------------------------------------------------------------------ (9)
def test_render_video_makes_the_frame_sequence(tmp_path):
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
    out = tmp_path / "frames"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "render_video.py"), str(run), "--out", str(out),
                        "--size", "96x128", "--radius", "1"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    files = sorted(os.listdir(out))
    names = {os.path.splitext(f)[0] for f in files}
    assert names == {"%04d" % v for v in range(n)} | {"%04d_pgo" % v for v in pgo_at}, files
    r2 = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "render_video.py"), str(run), "--out",
                         str(tmp_path / "follow"), "--size", "48x64", "--follow"], capture_output=True, text=True, cwd=ROOT)
    assert r2.returncode == 0, r2.stderr[-3000:]
    assert len(os.listdir(tmp_path / "follow")) == len(files)
