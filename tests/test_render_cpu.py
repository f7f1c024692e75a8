"""CPU: the map renderer's float64 oracle (oracle/render_oracle.py) on hand-computed scenes, the line builders of
vista_slam_b200/render.py against video.py's geometry and colour rule, and the refusals of render_views and sta_render
that come before anything needs CUDA.

The hand scenes use a map camera with K = I at the origin, so map pixel (col, row) at depth d is the world point
(col d, row d, d), and render cameras with power-of-two focal lengths: every position below is exact."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import render_oracle as ro


def _maps(depths, images=None):
    """A map of V views of one row: depths [V][W], every pixel confident, K = I, identity pose, scale 1."""
    d = np.asarray(depths, np.float32)[:, None, :]
    V, _, W = d.shape
    img = np.zeros((V, 3, 1, W), np.float32) if images is None else np.asarray(images, np.float32)
    return {"pose": np.tile(np.eye(4, dtype=np.float32), (V, 1, 1)), "scale": np.ones((V, 1), np.float32), "depth": d,
            "conf": np.full_like(d, 10.0), "intri": np.tile(np.eye(3, dtype=np.float32), (V, 1, 1)), "images": img}


def _K(f, cx, cy):
    return np.array([[[f, 0, cx], [0, f, cy], [0, 0, 1]]], np.float64)


EYE = np.eye(4)[None]


def test_occlusion_picks_the_nearer_point():
    img = np.stack([np.full((3, 1, 1), -1.0), np.full((3, 1, 1), 0.5)])
    out = ro.render(_maps([[2.0], [1.0]], img), 4.2, EYE, _K(4, 2, 2), (5, 5))
    assert out["index"][0, 2, 2] == 1 and out["depth"][0, 2, 2] == 1.0
    np.testing.assert_array_equal(out["rgb"][0, 2, 2], [0.75, 0.75, 0.75])
    assert (out["index"][0] >= 0).sum() == 1 and out["rgb"][0, 0, 0].tolist() == [1, 1, 1]
    assert not out["ambiguous"].any()


def test_equal_depth_goes_to_the_lower_id():
    out = ro.render(_maps([[2.0], [2.0]]), 4.2, EYE, _K(4, 2, 2), (5, 5))
    assert out["index"][0, 2, 2] == 0
    assert out["ambiguous"][0, 2, 2] and out["accept"][(0, 2, 2)] == {0, 1}


def test_radius_at_the_image_border():
    # map pixel 0 lands on (0, 0), pixel 1 on (4, 0): footprints are cut by the border
    for r, covered in ((0, {(0, 0), (0, 4)}),
                       (1, {(0, 0), (0, 1), (1, 0), (1, 1), (0, 3), (0, 4), (1, 3), (1, 4)}),
                       (2, {(y, x) for y in range(3) for x in range(5)})):
        out = ro.render(_maps([[1.0, 2.0]]), 4.2, EYE, _K(4, 0, 0), (6, 5), radius=r)
        got = {(int(y), int(x)) for y, x in zip(*np.nonzero(out["index"][0] >= 0))}
        assert got == covered, r
    # at r = 2 the two footprints overlap in columns 2: the nearer point (id 0, depth 1) wins
    assert out["index"][0, 0, 2] == 0 and out["index"][0, 0, 3] == 1


def test_point_behind_the_camera_and_the_near_plane():
    turn = np.diag([-1.0, 1.0, -1.0, 1.0])[None]  # looks along -z: the points are behind it
    out = ro.render(_maps([[1.0, 2.0, 4.0]]), 4.2, turn, _K(4, 4, 4), (9, 9))
    assert (out["index"] == -1).all() and (out["depth"] == 0).all() and (out["rgb"] == 1).all()
    out = ro.render(_maps([[1.0, 2.0, 4.0]]), 4.2, EYE, _K(4, 4, 4), (16, 16), near=1.5)
    assert sorted(out["index"][out["index"] >= 0].tolist()) == [1, 2]


def test_segment_steps_with_constant_depth_and_is_hidden_behind_points():
    segs = np.array([[[-1.0, 0.0, 2.0], [1.0, 0.0, 2.0]]])  # x from 2 to 6 on row 4 at z = 2
    out = ro.render(_maps([[1.0]]), 4.2, EYE, _K(4, 4, 4), (9, 9), segs=segs, seg_colors=[[0.0, 0.0, 1.0]])
    assert out["index"][0, 4, 4] == 0  # the point at z = 1 in front of the segment
    for x in (2, 3, 5, 6):
        assert out["index"][0, 4, x] == 1 and out["depth"][0, 4, x] == 2.0
        np.testing.assert_array_equal(out["rgb"][0, 4, x], [0, 0, 1])
    assert (out["index"][0] >= 0).sum() == 5
    # a segment crossing the near plane is cut there, a segment wholly behind it is dropped
    cross = np.array([[[0.0, 0.0, -1.0], [0.0, 0.0, 4.0]]])
    assert len(ro.segment_samples(cross[0, 0], cross[0, 1], np.eye(4), _K(4, 4, 4)[0], 9, 9, 0, 0.5)) >= 1
    assert ro.segment_samples(np.array([0.0, 0, -2]), np.array([0.0, 0, -1]), np.eye(4), _K(4, 4, 4)[0], 9, 9, 0, 0.5) == []


def test_camera_frusta_geometry():
    from vista_slam_b200.render import camera_frusta
    pose = np.eye(4)
    pose[:3, 3] = [1, 2, 3]
    K = np.array([[2.0, 0, 1], [0, 2.0, 1], [0, 0, 1]])
    segs, cols = camera_frusta(pose[None], K, 2, 2, 2.0, (0.1, 0.2, 0.3))
    c = np.array([1, 2, 3])
    corners = c + 2.0 * np.array([[-0.5, -0.5, 1], [0.5, -0.5, 1], [0.5, 0.5, 1], [-0.5, 0.5, 1]])
    want = [(c, corners[k]) for k in range(4)] + [(corners[k], corners[(k + 1) % 4]) for k in range(4)]
    np.testing.assert_allclose(segs, np.array(want), atol=1e-6)
    assert segs.dtype == np.float32 and cols.shape == (8, 3)
    np.testing.assert_allclose(cols, np.tile([0.1, 0.2, 0.3], (8, 1)), atol=1e-7)
    segs2, _ = camera_frusta(np.stack([pose, pose]), np.stack([K, K]), 2, 2, 2.0, (0, 0, 0))
    assert segs2.shape == (16, 2, 3)


def test_graph_segments_follow_the_video_colour_rule():
    from vista_slam_b200.render import graph_segments
    poses = np.tile(np.eye(4), (6, 1, 1))
    poses[:, 0, 3] = np.arange(6)
    vg = {0: [1], 1: [0, 2], 2: [1, 3], 3: [2, 0], 4: [3], 5: [4, 1]}
    segs, cols = graph_segments(poses, vg, 3, range(5))
    # edges (v, nv) with nv <= v: (1,0), (2,1), (3,2), (3,0) loop, (4,3)
    np.testing.assert_array_equal(segs[:, 0, 0], [1, 2, 3, 3, 4])
    np.testing.assert_array_equal(segs[:, 1, 0], [0, 1, 2, 0, 3])
    np.testing.assert_array_equal(cols, [[0, 0, 1]] * 3 + [[1, 0.5, 0]] + [[0, 0, 1]])
    assert graph_segments(poses, vg, 3, range(1))[0].shape == (0, 2, 3)


def _cpu_maps(V=2, H=4, W=5):
    return {"pose": torch.eye(4).repeat(V, 1, 1), "scale": torch.ones(V, 1), "depth": torch.ones(V, H, W),
        "conf": torch.ones(V, H, W), "intri": torch.eye(3).repeat(V, 1, 1), "images": torch.zeros(V, 3, H, W)}


@pytest.mark.parametrize("change, match", [
    (dict(size=(0, 8)), "output size"), (dict(size=(8, 8193)), "output size"), (dict(size=8), "size"),
    (dict(point_radius=5), "point_radius"), (dict(point_radius=-1), "point_radius"), (dict(near=0.0), "near"),
    (dict(poses=torch.eye(4)), "poses"), (dict(poses=torch.eye(4).repeat(8193, 1, 1)), "cameras"),
    (dict(K=torch.eye(3).repeat(2, 1, 1)), "K must be"), (dict(lines=(torch.zeros(2, 3), torch.zeros(2, 3))), "lines"),
    (dict(lines=(torch.zeros(2, 2, 3), torch.zeros(3, 3))), "lines"), (dict(background=(1, 1)), "background"),
    (dict(maps_f64=True), "float32"), (dict(maps_bad_shape=True), "images"), (dict(maps_big=True), "32-bit"),
    (dict(maps_many_views=True), "65535"), ({}, "CUDA device")])
def test_render_views_refusals(change, match):
    from vista_slam_b200.render import render_views
    maps = _cpu_maps()
    if change.pop("maps_f64", False):
        maps["conf"] = maps["conf"].double()
    if change.pop("maps_bad_shape", False):
        maps["images"] = maps["images"][:, :2]
    if change.pop("maps_big", False):  # 65535 views of 256 x 257: ids past 2^32 - 1 (stride-0 views, no memory)
        V, H, W = 65535, 256, 257
        maps = {"pose": torch.eye(4).expand(V, 4, 4), "scale": torch.ones(1, 1).expand(V, 1),
                "depth": torch.ones(1, 1, 1).expand(V, H, W), "conf": torch.ones(1, 1, 1).expand(V, H, W),
                "intri": torch.eye(3).expand(V, 3, 3), "images": torch.zeros(1, 1, 1, 1).expand(V, 3, H, W)}
    if change.pop("maps_many_views", False):
        V = 65536
        maps = {"pose": torch.eye(4).expand(V, 4, 4), "scale": torch.ones(1, 1).expand(V, 1),
                "depth": torch.ones(1, 1, 1).expand(V, 1, 1), "conf": torch.ones(1, 1, 1).expand(V, 1, 1),
                "intri": torch.eye(3).expand(V, 3, 3), "images": torch.zeros(1, 1, 1, 1).expand(V, 3, 1, 1)}
    args = dict(poses=torch.eye(4)[None], K=torch.eye(3), size=(8, 8))
    args.update(change)
    with pytest.raises(ValueError, match=match):
        render_views(maps, 0.5, **args)


def _abi_call(lib, **over):
    fake = ctypes.c_void_p(256)  # never dereferenced: every case is refused before any CUDA call
    a = dict(depth=fake, conf=fake, pose=fake, scale=fake, intri=fake, imgs=fake, V=1, H=4, W=4, thres=0.5, w2c=fake, K=fake,
             C=1, Ho=8, Wo=8, r=0, near=1e-3, segs=None, cols=None, L=0, bg=(ctypes.c_float * 3)(1, 1, 1), scratch=fake,
             nbytes=1 << 20, rgb=fake, depth_out=fake, index=fake)
    a.update(over)
    return lib.sta_render(a["depth"], a["conf"], a["pose"], a["scale"], a["intri"], a["imgs"], a["V"], a["H"], a["W"], a["thres"],
                        a["w2c"], a["K"], a["C"], a["Ho"], a["Wo"], a["r"], a["near"], a["segs"], a["cols"], a["L"], a["bg"],
                        a["scratch"], a["nbytes"], a["rgb"], a["depth_out"], a["index"], None)


@pytest.mark.parametrize("over, match", [
    (dict(C=0), b"cameras"), (dict(Ho=8193), b"cameras"), (dict(Wo=0), b"cameras"), (dict(r=5), b"radius"),
    (dict(r=-1), b"radius"), (dict(near=0.0), b"near"), (dict(near=-1.0), b"near"), (dict(V=65536), b"65535"),
    (dict(V=65535, H=256, W=257), b"32-bit"), (dict(V=0, L=-1), b"segment count"), (dict(H=0), b"map size"),
    (dict(L=2), b"null segments"), (dict(depth=None), b"null map"), (dict(rgb=None), b"null output"),
    (dict(w2c=None), b"null camera"), (dict(scratch=ctypes.c_void_p(260)), b"misaligned"), (dict(scratch=None), b"scratch"),
    (dict(nbytes=8 * 64 - 8), b"smaller")])
def test_abi_refusals_before_any_cuda_call(over, match):
    from vista_slam_b200 import _lib
    lib = _lib.lib()
    assert lib.sta_render_scratch_bytes(3, 8, 8) == 3 * 64 * 8 and lib.sta_render_scratch_bytes(0, 8, 8) == 0
    assert _abi_call(lib, **over) == 2
    assert match in lib.sta_last_error()
    assert lib.sta_version() == 2
