"""CPU: the ray-casting oracle (oracle/raycast_oracle.py) against closed forms -- an axis-aligned plane, a sphere's
distance field, a surface seen from behind -- and the refusals of fusion.raycast, OnlineSLAM.render_surface and
sta_raycast that come before anything needs CUDA."""
import ctypes
import types

import numpy as np
import pytest
import torch

from oracle import fusion_oracle as fo
from oracle import raycast_oracle as ro


def _field_volume(f, v, lo, hi, weight=None, band=None):
    """Bricks covering lattice [lo, hi] per axis, sorted by key, tsdf = f(x) at the float32 lattice points (float32),
    weight 1 (or weight(ijk)), colour = x.  band: keep only the bricks whose centre has |f| < band.  Returns
    (bricks [B,3] int32, tsdf, weight, color)."""
    bl, bh = np.floor_divide(lo, 8), np.floor_divide(hi, 8)
    b = np.stack(np.meshgrid(*[np.arange(bl[k], bh[k] + 1) for k in range(3)], indexing="ij"), -1).reshape(-1, 3)
    if band is not None:
        b = b[np.abs(f((b + 0.5) * 8 * v)) < band]
    b = b[np.argsort(fo.key(b))]
    ijk = fo.sample_coords(fo.key(b))
    X = (ijk.astype(np.float32) * np.float32(v)).astype(np.float64)
    T = f(X).astype(np.float32)
    Wt = np.ones_like(T) if weight is None else weight(ijk).astype(np.float32)
    return b.astype(np.int32), T, Wt, X.astype(np.float32)


def _K(f, cx, cy):
    return np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]], np.float64)


def _cast(vol, v, poses, K, size, **kw):
    b, T, Wt, C = vol
    return ro.raycast(fo.key(b), T, Wt, C, v, poses, K, size, **kw)


def test_plane_depth_and_normal():
    v = 0.125
    zp = 2.0 + 0.5 * v  # half-way between samples
    vol = _field_volume(lambda X: np.clip((zp - X[..., 2]) / (4 * v), -1, 1), v, np.array([-16, -16, 8]),
                        np.array([15, 15, 23]))
    out = _cast(vol, v, np.eye(4)[None], _K(16.0, 8, 6), (12, 16))
    # (the centre ray has a sample exactly on the plane: a crossing at a step boundary, flagged ambiguous, and hit)
    assert out["hit"].all() and out["ambiguous"].sum() == 1
    np.testing.assert_allclose(out["depth"], zp, rtol=0, atol=1e-12)
    np.testing.assert_allclose(out["normal"], np.broadcast_to([0.0, 0.0, -1.0], out["normal"].shape), atol=1e-12)
    # the colour is the position: x = z (col - cx) / f at the hit
    col = np.arange(16)
    np.testing.assert_allclose(out["color"][0, 3, :, 0], zp * (col - 8) / 16.0, atol=1e-6)
    # a headlight: the centre ray meets the plane head-on
    np.testing.assert_allclose(out["rgb"][0, 6, 8], out["color"][0, 6, 8], atol=1e-12)


def _look_at(eye, target, up=(0.0, 1.0, 0.0)):
    z = np.asarray(target, np.float64) - eye
    z /= np.linalg.norm(z)
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    P = np.eye(4)
    P[:3, :3] = np.stack([x, np.cross(z, x), z], 1)
    P[:3, 3] = eye
    return P


def test_sphere_distance_field_against_the_analytic_intersection():
    # the interpolant's gradient errs by about 0.65 v / R: 1/128 keeps it well under 1e-2 rad; bricks only near the
    # surface
    R, v = 1.0, 1.0 / 128
    vol = _field_volume(lambda X: np.linalg.norm(X, axis=-1) - R, v, np.array([-144] * 3), np.array([143] * 3),
                        band=16 * v)
    poses = np.stack([_look_at(np.array(e, np.float64), np.zeros(3)) for e in ([0.3, 0.2, -3.0], [2.5, 1.0, 1.2])])
    K = _K(24.0, 15.5, 11.5)
    out = _cast(vol, v, poses, K, (24, 32))
    for c in range(2):
        P = poses[c]
        row, col = np.mgrid[0:24, 0:32]
        dc = np.stack([(col - K[0, 2]) / K[0, 0], (row - K[1, 2]) / K[1, 1], np.ones((24, 32))], -1)
        d = dc @ P[:3, :3].T
        o = P[:3, 3]
        a, bq, cq = (d * d).sum(-1), 2 * (d @ o), o @ o - R * R
        disc = bq * bq - 4 * a * cq
        zs = (-bq - np.sqrt(np.maximum(disc, 0))) / (2 * a)
        clear = (disc > 0.05) & ~out["ambiguous"][c]  # away from the silhouette
        assert clear.sum() > 100
        assert out["hit"][c][clear].all()
        p = o + out["depth"][c][..., None] * d
        want = p / np.linalg.norm(p, axis=-1, keepdims=True)
        # the hit within v^2 / R of the sphere, and its depth too where the ray meets the sphere at 60 degrees or less
        # (the trilinear interpolant of |x| - R lies above it by up to about 3 v^2 / (8 R))
        assert np.abs(np.linalg.norm(p[clear], axis=-1) - R).max() <= v * v / R
        head_on = clear & (-(want * d).sum(-1) / np.linalg.norm(d, axis=-1) >= 0.5)
        assert head_on.sum() > 100
        assert np.abs(out["depth"][c][head_on] - zs[head_on]).max() <= v * v / R
        cos = np.clip((out["normal"][c] * want).sum(-1), -1, 1)
        assert np.arccos(cos[clear]).max() <= 1e-2
        assert not out["hit"][c][disc < 0].any()


def test_a_surface_seen_from_behind_is_passed_through():
    """T = -(z - 1.05)(z - 2.05): negative at the camera, a - to + crossing at 1.05, a + to - crossing at 2.05.  The ray
    starts inside the valid negative region and hits the second one, where the interpolant between samples 2.0 and
    2.1 is zero at 2.0 + 0.1 * 0.0475 / 0.1."""
    v = 0.1
    vol = _field_volume(lambda X: -(X[..., 2] - 1.05) * (X[..., 2] - 2.05), v, np.array([-16, -16, -8]),
                        np.array([15, 15, 31]))
    out = _cast(vol, v, np.eye(4)[None], _K(8.0, 4, 3), (6, 8))
    assert out["hit"].all()
    np.testing.assert_allclose(out["depth"], 2.0475, rtol=0, atol=1e-6)  # the samples are float32
    np.testing.assert_allclose(out["normal"][..., 2], -1.0, atol=1e-9)
    # with the far surface gone (zero weight beyond z = 1.6) nothing is hit
    vol2 = _field_volume(lambda X: -(X[..., 2] - 1.05) * (X[..., 2] - 2.05), v, np.array([-16, -16, -8]),
                         np.array([15, 15, 31]), weight=lambda ijk: (ijk[..., 2] <= 16).astype(np.float32))
    out2 = _cast(vol2, v, np.eye(4)[None], _K(8.0, 4, 3), (6, 8))
    assert not out2["hit"].any()
    np.testing.assert_array_equal(out2["rgb"], 1.0)
    np.testing.assert_array_equal(out2["depth"], 0.0)


def test_min_weight_and_empty_volume_miss():
    v = 0.125
    zp = 2.0 + 0.5 * v
    vol = _field_volume(lambda X: np.clip((zp - X[..., 2]) / (4 * v), -1, 1), v, np.array([-16, -16, 8]),
                        np.array([15, 15, 23]))
    assert not _cast(vol, v, np.eye(4)[None], _K(16.0, 8, 6), (12, 16), min_weight=2)["hit"].any()
    empty = (np.zeros((0, 3), np.int32), np.zeros((0, 8, 8, 8), np.float32), np.zeros((0, 8, 8, 8), np.float32),
             np.zeros((0, 8, 8, 8, 3), np.float32))
    out = _cast(empty, v, np.eye(4)[None], _K(16.0, 8, 6), (4, 5), background=(0.0, 0.5, 1.0))
    assert not out["hit"].any()
    np.testing.assert_array_equal(out["rgb"][0, 0, 0], [0.0, 0.5, 1.0])


# ------------------------------------------------------------------------------------------------ refusals
def _vol_args(B=2):
    return dict(bricks=torch.zeros(B, 3, dtype=torch.int32), tsdf=torch.zeros(B, 8, 8, 8),
                weight=torch.zeros(B, 8, 8, 8), color=torch.zeros(B, 8, 8, 8, 3), voxel_size=0.1,
                poses=torch.eye(4)[None], K=torch.eye(3), size=(4, 5))


@pytest.mark.parametrize("change, match", [
    (dict(voxel_size=0.0), "voxel_size"), (dict(voxel_size=float("nan")), "voxel_size"),
    (dict(min_weight=0.5), "min_weight"), (dict(bricks=torch.zeros(2, 2)), "bricks"),
    (dict(tsdf=torch.zeros(2, 8, 8, 7)), "tsdf"), (dict(color=torch.zeros(2, 8, 8, 8)), "color"),
    (dict(weight=torch.zeros(2, 8, 8, 8, dtype=torch.float64)), "weight"), ({}, "CUDA device")])
def test_raycast_volume_refusals(change, match):
    from vista_slam_b200.fusion import raycast
    args = _vol_args()
    args.update(change)
    with pytest.raises(ValueError, match=match):
        raycast(**args)


@pytest.mark.parametrize("change, match", [
    (dict(size=(0, 5)), "output size"), (dict(size=(4, 8193)), "output size"), (dict(size=(4,)), "size"),
    (dict(near=0.0), "near"), (dict(near=float("inf")), "near"), (dict(poses=torch.eye(4)), "poses"),
    (dict(poses=torch.eye(4, dtype=torch.int64)[None]), "poses"), (dict(K=torch.eye(3).repeat(2, 1, 1)), "K"),
    (dict(poses=torch.eye(4).expand(8193, 4, 4)), "cameras"), (dict(background=(1.0, 1.0)), "background"),
    (dict(background=(1.0, 1.0, float("nan"))), "background")])
def test_raycast_camera_refusals(change, match):
    from vista_slam_b200.fusion import _check_cameras
    args = dict(poses=torch.eye(4)[None], K=torch.eye(3), size=(4, 5), near=1e-3, background=(1.0, 1.0, 1.0))
    args.update(change)
    with pytest.raises(ValueError, match=match):
        _check_cameras(dev=torch.device("cpu"), **args)


@pytest.mark.parametrize("change, match, exc", [
    (dict(voxel_size=0.0), "voxel_size", ValueError), (dict(trunc=0.5), "trunc", ValueError),
    (dict(min_weight=0), "min_weight", ValueError), (dict(min_consistent_views=9), "min_consistent_views", ValueError),
    (dict(size=(0, 5)), "output size", ValueError), (dict(K=torch.eye(4)), "K", ValueError),
    (dict(background=(1.0,)), "background", ValueError)])
def test_render_surface_refusals_before_any_work(change, match, exc):
    from vista_slam_b200.slam import OnlineSLAM

    def no_work(*a, **k):
        raise AssertionError("work started before the arguments were checked")

    fake = types.SimpleNamespace(device=torch.device("cpu"), _graph=None, _view_maps=no_work,
                                 _consistent_maps=no_work, conf_thres=1.0)
    args = dict(poses=torch.eye(4)[None], K=torch.eye(3), size=(4, 5), voxel_size=0.1)
    args.update(change)
    with pytest.raises(exc, match=match):
        OnlineSLAM.render_surface(fake, **args)


FAKE = ctypes.c_void_p(256)  # never dereferenced: every case is refused before any CUDA call


def _raycast_call(lib, **over):
    a = dict(B=4, voxel=0.1, mw=1.0, C=1, Ho=4, Wo=5, near=1e-3, keys=FAKE, cams=FAKE, scratch=FAKE, nbytes=1 << 10,
             rgb=FAKE)
    a.update(over)
    bg = (ctypes.c_float * 3)(1.0, 1.0, 1.0)
    return lib.sta_raycast(a["keys"], a["B"], FAKE, FAKE, FAKE, a["voxel"], a["mw"], a["cams"], FAKE, a["C"], a["Ho"],
                           a["Wo"], a["near"], bg, a["scratch"], a["nbytes"], a["rgb"], FAKE, FAKE, FAKE, None)


@pytest.mark.parametrize("over, match", [
    (dict(C=0), b"8192"), (dict(C=8193), b"8192"), (dict(Ho=0), b"8192"), (dict(Wo=8193), b"8192"),
    (dict(B=-1), b"brick count"), (dict(B=(1 << 20) + 1), b"brick count"), (dict(voxel=0.0), b"voxel"),
    (dict(voxel=float("nan")), b"voxel"), (dict(mw=0.5), b"min_weight"), (dict(near=0.0), b"near"),
    (dict(near=float("inf")), b"near"), (dict(keys=None), b"null volume"), (dict(cams=None), b"null camera"),
    (dict(rgb=None), b"null output"), (dict(scratch=None), b"scratch"), (dict(scratch=ctypes.c_void_p(264)), b"misaligned"),
    (dict(nbytes=16), b"smaller"), ({}, b"device memory")])
def test_abi_refusals_before_any_cuda_call(over, match):
    from vista_slam_b200 import _lib
    lib = _lib.lib()
    assert _raycast_call(lib, **over) == 2
    assert match in lib.sta_last_error()
    assert lib.sta_version() == 2


def test_scratch_query():
    from vista_slam_b200 import _lib
    lib = _lib.lib()
    assert lib.sta_raycast_scratch_bytes(-1) == 0 and lib.sta_raycast_scratch_bytes((1 << 20) + 1) == 0
    assert lib.sta_raycast_scratch_bytes(0) == 32 and lib.sta_raycast_scratch_bytes(1 << 20) == 32
