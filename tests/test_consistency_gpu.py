"""GPU: multi-view depth consistency (csrc/consistency.cu, slam_utils.view_consistency_check, OnlineSLAM.view_consistency
and min_consistent_views on render / extract_mesh / save_mesh / save_data_all).

  1. Planted exact scenes (power-of-two K, plane depths and shifts, every float32 operation exact): counts bit-equal to
     the hand values and to the float64 oracle, the off-image, behind-the-camera and non-finite quirks included.
  2. The reference golden (tests/golden/consistency.npz): counts equal on every pixel the oracle marks unambiguous, and
     on every pixel of the exact scenes.
  3. Random ray-cast scenes up to 64 views against the oracle on unambiguous pixels; the same bits on repeated calls.
  4. A replayed OnlineSLAM run, synchronous and with background PGO: view_consistency is view_consistency_check of the
     stacked get_view outputs bit for bit, the session is left as it was, None and 0 give the existing outputs, k > 0
     gives render_views / fuse_views of the maps with conf -inf where the count is below k, the PLY is the ordered
     subset, and a planted bad keyframe drops out at k = 1.
  5. The real frontend: counts within [0, 8], the filtered PLY an ordered subset of the unfiltered one.
  6. Refusals before any launch."""
import os

import numpy as np
import pytest
import torch

from oracle import consistency_oracle as co
from test_consistency_cpu import K8, _pose, _shifted_planes
from test_fusion_gpu import _replayed, _voxel_of
from test_slam_batch_gpu import _frames_224
from test_slam_gpu import VOCAB, _replay_slam, _value
from oracle import slam_oracle as so

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "consistency.npz")


def _check(d, K, T, thr=0.05):
    from vista_slam_b200.utils.slam_utils import view_consistency_check
    out = view_consistency_check(torch.from_numpy(np.asarray(d)).cuda(), torch.from_numpy(np.asarray(K)).cuda(),
                                 torch.from_numpy(np.asarray(T)).cuda(), thr)
    assert out.dtype == torch.int32 and out.is_cuda
    return out.cpu().numpy()


# ------------------------------------------------------------------------------------------------ (1)
def _planted():
    flip = np.diag([-1.0, 1.0, -1.0])
    d2 = np.full((2, 6, 10), 4.0, np.float32)
    behind = (d2, np.tile(K8, (2, 1, 1)), np.stack([_pose(np.eye(3), [0, 0, 0]), _pose(flip, [5.0, 0, 0])]))
    half = (d2, np.tile(K8, (2, 1, 1)), np.stack([_pose(np.eye(3), [0, 0, 0]), _pose(flip, [2.0, 0, 0])]))
    d3 = np.full((3, 6, 10), 2.0, np.float32)
    d3[0, 3, 4] = 0.0
    nan = (d3, np.tile(K8, (3, 1, 1)),
           np.stack([_pose(np.eye(3), [0.5, 0, 0]), _pose(np.eye(3), [0.5, 0, 0]), _pose(np.eye(3), [0.75, 0, 0])]))
    yy, xx = np.meshgrid(np.arange(6), np.arange(10), indexing="ij")
    return [
        ("shift", _shifted_planes((0.0, 2.0, 4.5, 5.0)), None),
        ("ladder", _shifted_planes(tuple(0.5 * k for k in range(11))), None),
        ("half", _shifted_planes((0.0, 0.25)), None),
        ("behind", behind, np.ones((2, 6, 10), np.int32)),
        ("behind_on_image", half, None),
        ("nan", nan, None),
        ("single", _shifted_planes((0.0,)), np.zeros((1, 6, 10), np.int32)),
    ], ((xx < 4) | (yy == 5)).astype(np.int32)


def test_planted_exact_scenes_bit_for_bit():
    scenes, behind_on_image_0 = _planted()
    for name, (d, K, T), hand in scenes:
        want, amb = co.view_consistency(d, K, T)
        assert not amb.any(), name
        got = _check(d, K, T)
        np.testing.assert_array_equal(got, want, err_msg=name)
        if hand is not None:
            np.testing.assert_array_equal(got, hand, err_msg=name)
        if name == "behind_on_image":
            np.testing.assert_array_equal(got[0], behind_on_image_0)
        if name == "nan":
            assert got[0, 3, 4] == 0 and got[0, 3, 5] == 2 and got[1, 3, 4] == 1


# ------------------------------------------------------------------------------------------------ (2)
def test_reference_golden():
    g = dict(np.load(GOLDEN))
    thr = float(g["threshold"])
    for name in g["names"]:
        d, K, T, want = g[name + "_depth"], g[name + "_intri"], g[name + "_pose"], g[name + "_count"]
        got = _check(d, K, T, thr)
        _, amb = co.view_consistency(d, K, T, thr)
        unamb = ~amb.any(-1)
        assert (got[unamb] == want[unamb]).all(), (name, int((got != want)[unamb].sum()))
        if name in g["exact"]:
            np.testing.assert_array_equal(got, want, err_msg=name)
        print("%-14s device != reference on %d of %d pixels (%d ambiguous)" % (name, int((got != want).sum()), got.size,
                                                                             int((~unamb).sum())))


# ------------------------------------------------------------------------------------------------ (3)
@pytest.mark.parametrize("seed, n, H, W", [(1, 2, 20, 24), (2, 9, 31, 47), (3, 17, 40, 56), (4, 64, 48, 64)])
def test_random_scenes_against_fp64(seed, n, H, W):
    d, K, T = co.raycast_scene(seed, n, H, W)
    thr = [0.05, 0.02, 0.1, 0.05][seed - 1]
    want, amb = co.view_consistency(d, K, T, thr)
    a = _check(d, K, T, thr)
    b = _check(d, K, T, thr)
    np.testing.assert_array_equal(a, b)
    unamb = ~amb.any(-1)
    assert (a[unamb] == want[unamb]).all(), int((a != want)[unamb].sum())
    # the smaller threshold puts more tests near a tie than the golden's 0.05 (0.23 % at 0.02)
    tests = sum(min(n - 1, i + 4) - max(0, i - 4) for i in range(n)) * H * W
    assert amb.sum() < 1e-2 * tests
    assert (a >= 0).all() and (a <= 8).all() and a.max() == min(8, n - 1)


# ------------------------------------------------------------------------------------------------ (4)
def _stacked_check(slam, views):
    from vista_slam_b200.utils.slam_utils import view_consistency_check
    vs = [slam.get_view(v) for v in views]
    return view_consistency_check(torch.stack([v.depth for v in vs]).cuda(), torch.stack([v.intri for v in vs]).cuda(),
                                  torch.stack([v.pose for v in vs]).cuda(), slam.consistency_thres)


def _filtered(maps, counts, k):
    maps = dict(maps)
    maps["conf"] = maps["conf"].masked_fill(counts < k, float("-inf"))
    return maps


def _cams(slam):
    ex = slam._export(0, 2, cloud=False)
    return ex["pose"], ex["intri"], (slam._graph.H, slam._graph.W)


def test_replayed_run(tmp_path):
    from vista_slam_b200.fusion import fuse_views
    from vista_slam_b200.render import render_views
    from vista_slam_b200.slam import read_ply
    slam, stream = _replayed()
    n = slam.view_num
    v, _ = _voxel_of(slam)
    G = slam._graph
    names = ("pose", "depth", "conf", "intri", "cmean", "node_to_view", "node_to_connected_view", "best_node",
             "best_mean", "edges", "meas", "weight")
    tables = {k: getattr(G, k).clone() for k in names}
    host = (dict(slam.view_to_node), list(slam.node_to_connected_view), slam.num_nodes, slam.num_edges, slam.view_num)

    c = slam.view_consistency()
    assert c.shape == (n, G.H, G.W) and c.dtype == torch.int32
    assert torch.equal(c, _stacked_check(slam, range(n)))
    assert torch.equal(slam.view_consistency(range(3, 11)), _stacked_check(slam, range(3, 11)))
    assert torch.equal(slam.view_consistency(), c)
    print("replayed counts:", np.bincount(c.cpu().numpy().ravel(), minlength=9))

    poses, K, size = _cams(slam)
    base_r = slam.render(poses, K, size)
    base_m = slam.extract_mesh(v)
    for k0 in (None, 0):
        r = slam.render(poses, K, size, min_consistent_views=k0)
        m = slam.extract_mesh(v, min_consistent_views=k0)
        for a, b in list(zip(r.values(), base_r.values())) + list(zip(m.values(), base_m.values())):
            assert torch.equal(a, b)
    maps = slam._view_maps(None)
    for k in (1, 2, 4):
        r = slam.render(poses, K, size, min_consistent_views=k)
        want = render_views(_filtered(maps, c, k), slam.conf_thres, poses, K, size)
        for key in want:
            assert torch.equal(r[key], want[key]), (k, key)
        m = slam.extract_mesh(v, min_consistent_views=k)
        want = fuse_views(_filtered(maps, c, k), slam.conf_thres, v)
        for key in want:
            assert torch.equal(m[key], want[key]), (k, key)
    path = slam.save_mesh(str(tmp_path / "mesh2"), v, min_consistent_views=2)
    assert os.path.exists(path)

    # save_data_all: the PLY is the ordered subset, every other file unchanged
    slam.save_data_all(str(tmp_path / "all"))
    slam.save_data_all(str(tmp_path / "none"), min_consistent_views=0)
    slam.save_data_all(str(tmp_path / "k2"), min_consistent_views=2)
    files = sorted(os.listdir(tmp_path / "all"))
    assert files == sorted(os.listdir(tmp_path / "k2"))
    for f in files:
        a = open(tmp_path / "all" / f, "rb").read()
        assert a == open(tmp_path / "none" / f, "rb").read(), f
        if f != "pointcloud.ply":
            assert a == open(tmp_path / "k2" / f, "rb").read(), f
    P, C = read_ply(str(tmp_path / "all" / "pointcloud.ply"))
    P2, C2 = read_ply(str(tmp_path / "k2" / "pointcloud.ply"))
    keep = (c[maps["conf"] > slam.conf_thres] >= 2).cpu().numpy()
    assert len(keep) == len(P) and 0 < keep.sum() < len(P)
    np.testing.assert_array_equal(P2.view(np.uint32), P[keep].view(np.uint32))
    np.testing.assert_array_equal(C2, C[keep])

    for k, t in tables.items():
        assert torch.equal(getattr(G, k).view(torch.uint8), t.view(torch.uint8)), k
    assert host == (dict(slam.view_to_node), list(slam.node_to_connected_view), slam.num_nodes, slam.num_edges,
                    slam.view_num)

    # a planted bad keyframe: view b's depth x 1000 puts its points far beyond every neighbour's surface, so none of
    # its map pixels agrees (its zeroed pixels sit at the camera centre and may still agree through off-image samples)
    b = 7
    G.depth[int(G.best_node[b])] *= 1000.0
    c = slam.view_consistency()
    maps = slam._view_maps(None)
    assert (c[b][maps["conf"][b] > slam.conf_thres] == 0).all()
    r = slam.render(poses, K, size, min_consistent_views=1)
    idx = r["index"][r["index"] >= 0]
    hw = G.H * G.W
    assert not ((idx >= b * hw) & (idx < (b + 1) * hw)).any()
    slam.save_data_all(str(tmp_path / "bad"), min_consistent_views=1, save_view_graph=False, save_images=False)
    P1, _ = read_ply(str(tmp_path / "bad" / "pointcloud.ply"))
    used = maps["conf"] > slam.conf_thres
    assert len(P1) == int(((c >= 1) & used).sum()) <= int(used.sum()) - int(used[b].sum())


def test_background_pgo_equals_synchronous():
    stream = so.make_stream()
    images = so.stream_images(stream)
    sync = _replay_slam(stream)
    bg = _replay_slam(stream)
    bg.pgo_background = True
    for i in range(14):
        sync.step(_value(images, i, stream))
        bg.step(_value(images, i, stream))
    c = bg.view_consistency()  # whatever the PGO's state, the views it shows
    assert c.shape[0] == 14
    bg.wait_pgo()
    assert torch.equal(bg.view_consistency(), sync.view_consistency())
    assert torch.equal(bg.view_consistency(), _stacked_check(bg, range(14)))
    poses, K, size = _cams(sync)
    a = sync.render(poses, K, size, min_consistent_views=2)
    b = bg.render(poses, K, size, min_consistent_views=2)
    for key in a:
        assert torch.equal(a[key], b[key]), key


# ------------------------------------------------------------------------------------------------ (5)
def test_real_frontend(cuda_model, tmp_path):
    import vista_slam_b200.slam as S
    from vista_slam_b200.slam import read_ply

    class Run(S.OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return cuda_model

    slam = Run("unused", VOCAB, verbose=False, loop_dist_min=4, pgo_every=5, rel_pose_thres=0.5)
    frames = _frames_224(12)
    for i in range(12):
        slam.step(frames[i], force_pgo=(i == 11))
    ex = slam._export(0, slam.view_num, cloud=False)
    d = (ex["depth"] * ex["scale"][:, :, None])[ex["conf"] > slam.conf_thres]
    slam.consistency_thres = 0.05 * float(d[d > 0].median())  # random-weight maps: a threshold at the map's scale
    c = slam.view_consistency()
    assert int(c.min()) >= 0 and int(c.max()) <= 8
    print("real frontend counts:", np.bincount(c.cpu().numpy().ravel(), minlength=9))
    slam.save_data_all(str(tmp_path / "a"))
    slam.save_data_all(str(tmp_path / "b"), min_consistent_views=1)
    P, C = read_ply(str(tmp_path / "a" / "pointcloud.ply"))
    P1, C1 = read_ply(str(tmp_path / "b" / "pointcloud.ply"))
    keep = (c[ex["conf"] > slam.conf_thres] >= 1).cpu().numpy()
    np.testing.assert_array_equal(P1.view(np.uint32), P[keep].view(np.uint32))
    np.testing.assert_array_equal(C1, C[keep])


# ------------------------------------------------------------------------------------------------ (6)
def test_refusals_before_any_launch(tmp_path):
    from vista_slam_b200.utils.slam_utils import view_consistency_check
    d = torch.ones(3, 4, 5, device="cuda")
    K = torch.eye(3, device="cuda").repeat(3, 1, 1)
    T = torch.eye(4, device="cuda").repeat(3, 1, 1)
    for args in ((d[0], K, T), (d, K[:2], T), (d, K, T[:, :3]), (d.cpu(), K, T), (d, K.cpu(), T)):
        with pytest.raises(RuntimeError):
            view_consistency_check(*args)
    for args, thr in (((d[:, :1], K, T), 0.05), ((d[:, :, :1], K, T), 0.05), ((d, K, T), float("nan"))):
        with pytest.raises(RuntimeError, match="sta_view_consistency"):
            view_consistency_check(*args, threshold=thr)
    assert view_consistency_check(d[:0], K[:0], T[:0]).shape == (0, 4, 5)
    slam, _ = _replayed(n=5)
    poses, K2, size = _cams(slam)
    for k in (-1, 9, 1.5, True):
        with pytest.raises(ValueError, match="min_consistent_views"):
            slam.render(poses, K2, size, min_consistent_views=k)
        with pytest.raises(ValueError, match="min_consistent_views"):
            slam.extract_mesh(0.1, min_consistent_views=k)
        with pytest.raises(ValueError, match="min_consistent_views"):
            slam.save_mesh(str(tmp_path / "m"), 0.1, min_consistent_views=k)
        with pytest.raises(ValueError, match="min_consistent_views"):
            slam.save_data_all(str(tmp_path / "s"), min_consistent_views=k)
    assert not os.path.exists(tmp_path / "m") and not os.path.exists(tmp_path / "s")
    with pytest.raises(IndexError):
        slam.view_consistency(range(0, 6))
