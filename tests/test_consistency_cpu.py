"""CPU: the multi-view depth consistency's float64 oracle (oracle/consistency_oracle.py) against the reference's golden
counts (tests/golden/consistency.npz, tools/make_golden_consistency.py) and on hand-computed scenes, the new C entry
point's export, and the refusals of view_consistency_check, min_consistent_views and sta_view_consistency that come
before anything needs CUDA.

The hand scenes are fronto-parallel planes at z = 4 seen by 10 x 6 cameras with K = [[8, 0, 4], [0, 8, 2], [0, 0, 1]]
moved along x: a point of view i at pixel column x lands in view j at column x + 2 (t_i - t_j), exactly."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import consistency_oracle as co

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "consistency.npz")
K8 = np.array([[8, 0, 4], [0, 8, 2], [0, 0, 1]], np.float32)


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _pose(R, t):
    T = np.eye(4, dtype=np.float32)
    T[:3, :3], T[:3, 3] = R, t
    return T


def _window_sizes(n):
    return np.array([min(n - 1, i + 4) - max(0, i - 4) for i in range(n)])


def test_oracle_matches_the_reference_golden(golden):
    g = golden
    thr = float(g["threshold"])
    tests = ambiguous = 0
    for name in g["names"]:
        d, K, T, want = g[name + "_depth"], g[name + "_intri"], g[name + "_pose"], g[name + "_count"]
        got, amb = co.view_consistency(d, K, T, thr)
        unamb = ~amb.any(-1)
        assert (got[unamb] == want[unamb]).all(), (name, int((got != want)[unamb].sum()))
        tests += int(_window_sizes(d.shape[0]).sum()) * d.shape[1] * d.shape[2]
        ambiguous += int(amb.sum())
        if name in g["exact"]:
            assert not amb.any() and (got == want).all(), name
    assert ambiguous < 1e-3 * tests, (ambiguous, tests)


def test_golden_pins_the_quirks(golden):
    g = golden
    # the 180-degree neighbour: whole rows of 6 (every neighbour agrees, the flipped one through off-image samples)
    assert (g["flipped_count"] == 6).sum() >= 8
    # coincident centres: view 0's depth-0 pixels land at (K c)_z = 0 in view 1 and on c = (-1/4, 0, 0) in view 2
    assert (g["coincident_count"][0, 1:3, 2:5] == 0).all()
    # overflow: (1, 0) overflows in the unnormalisation (no agreement), (0, 1) is finite and far off-image (agrees)
    np.testing.assert_array_equal(g["overflow_count"][0], [[0, 0], [1, 0]])


def _shifted_planes(ts, depth=4.0):
    n = len(ts)
    d = np.full((n, 6, 10), depth, np.float32)
    return d, np.tile(K8, (n, 1, 1)), np.stack([_pose(np.eye(3), [t, 0, 0]) for t in ts])


@pytest.mark.parametrize("ts", [(0.0, 0.5), (0.0, 2.0, 4.5, 5.0), tuple(0.5 * k for k in range(11)), (0.0, 0.0, 0.0)])
def test_oracle_on_shifted_planes(ts):
    """Column x of view i agrees with view j iff x + 2 (t_i - t_j) lies in [0, W - 1]: on the image (borders included)
    the sample is the plane's depth, one or more whole columns beyond it the sample is 0."""
    d, K, T = _shifted_planes(ts)
    got, amb = co.view_consistency(d, K, T)
    n, H, W = d.shape
    want = np.zeros((n, H, W), np.int32)
    for i in range(n):
        for j in range(max(0, i - 4), min(n, i + 5)):
            if j != i:
                u = np.arange(W) + 2 * (ts[i] - ts[j])
                want[i] += ((u >= 0) & (u <= W - 1)).astype(np.int32)[None, :]
    np.testing.assert_array_equal(got, want)
    assert not amb.any()


def test_oracle_half_pixel_blend_and_window_clip():
    """A half-pixel shift blends the plane with the zero padding half a column outside the image (sample 2, disagree)
    and is exact elsewhere; with 11 views the window of view 0 holds views 1..4 only."""
    d, K, T = _shifted_planes((0.0, 0.25))
    got, _ = co.view_consistency(d, K, T)
    assert (got[0, :, 0] == 0).all() and (got[0, :, 1:] == 1).all()
    assert (got[1, :, -1] == 0).all() and (got[1, :, :-1] == 1).all()
    d, K, T = _shifted_planes((0.0,) * 11)
    got, _ = co.view_consistency(d, K, T)
    np.testing.assert_array_equal(got[:, 0, 0], _window_sizes(11))


def test_oracle_off_image_behind_the_camera_agrees():
    """View 1 is turned 180 degrees about y and moved to x = 5: each view's points lie behind the other, z clamps to
    1e-6, and they land 10 columns to the left of the image, where the sample is 0 -- so every pixel agrees."""
    flip = np.diag([-1.0, 1.0, -1.0])
    d = np.full((2, 6, 10), 4.0, np.float32)
    K = np.tile(K8, (2, 1, 1))
    T = np.stack([_pose(np.eye(3), [0, 0, 0]), _pose(flip, [5.0, 0, 0])])
    got, amb = co.view_consistency(d, K, T)
    assert (got == 1).all() and not amb.any()
    # at x = 2 the flipped camera sees view 0's point (x, y) at column x - 4 and row 4 - y: where that is on the image
    # the sample is 4 against z = 1e-6, no agreement; off the image (x < 4 or y = 5) it still agrees
    T[1, 0, 3] = 2.0
    got, _ = co.view_consistency(d, K, T)
    yy, xx = np.meshgrid(np.arange(6), np.arange(10), indexing="ij")
    np.testing.assert_array_equal(got[0], ((xx < 4) | (yy == 5)).astype(np.int32))


def test_oracle_non_finite_projection_never_agrees():
    """A depth-0 pixel is the camera centre; a neighbour with the same centre sees it at c = 0, so u = 0 / 0: no
    agreement even though the clamped z (1e-6) is below the threshold.  A neighbour 1/4 to the side sees it at
    c = (-1/4, 0, 0): u = -2 / 0 = -inf, also no agreement."""
    d = np.full((3, 6, 10), 2.0, np.float32)
    d[0, 3, 4] = 0.0
    K = np.tile(K8, (3, 1, 1))
    T = np.stack([_pose(np.eye(3), [0.5, 0, 0]), _pose(np.eye(3), [0.5, 0, 0]), _pose(np.eye(3), [0.75, 0, 0])])
    got, amb = co.view_consistency(d, K, T)
    assert got[0, 3, 4] == 0 and not amb.any()
    # beside it both neighbours agree (view 2 sees the plane one column to the left); view 1's pixel over the hole
    # samples view 0's 0 there and agrees with view 2 only
    assert got[0, 3, 5] == 2 and got[1, 3, 4] == 1


def test_oracle_single_view_is_zero():
    d, K, T = _shifted_planes((0.0,))
    got, amb = co.view_consistency(d, K, T)
    assert (got == 0).all() and not amb.any()


def test_symbol_is_exported():
    from vista_slam_b200 import _lib
    lib = _lib.lib()
    assert hasattr(lib, "sta_view_consistency")
    assert lib.sta_view_consistency.argtypes is not None
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "sta_b200.h")).read()
    assert "int sta_view_consistency(" in hdr
    from vista_slam_b200.utils import slam_utils
    assert callable(slam_utils.view_consistency_check)


FAKE = ctypes.c_void_p(256)  # never dereferenced: every case is refused before any CUDA call


@pytest.mark.parametrize("over, match", [
    (dict(n=0), b"view count"), (dict(n=65536), b"view count"), (dict(H=1), b"at least 2"), (dict(W=1), b"at least 2"),
    (dict(n=4096, H=1024, W=512), b"2^31"), (dict(thr=float("nan")), b"finite"), (dict(thr=float("inf")), b"finite"),
    (dict(depth=None), b"null"), (dict(out=None), b"null"), ({}, b"device memory")])
def test_abi_refusals_before_any_cuda_call(over, match):
    from vista_slam_b200 import _lib
    lib = _lib.lib()
    a = dict(n=2, H=4, W=4, thr=0.05, depth=FAKE, out=FAKE)
    a.update(over)
    assert lib.sta_view_consistency(a["depth"], FAKE, FAKE, a["n"], a["H"], a["W"], a["thr"], a["out"], None) == 2
    assert match in lib.sta_last_error()


def test_python_refusals_of_cpu_tensors_and_shapes():
    from vista_slam_b200.utils.slam_utils import view_consistency_check
    d, K, T = (torch.from_numpy(x) for x in _shifted_planes((0.0, 0.5)))
    with pytest.raises(RuntimeError, match="CUDA"):
        view_consistency_check(d, K, T)


@pytest.mark.parametrize("k", [-1, 9, 1.0, True, "2", 2.5])
def test_min_consistent_views_refusals(k):
    from vista_slam_b200.slam import _min_consistent_views
    with pytest.raises(ValueError, match="min_consistent_views"):
        _min_consistent_views(k)


def test_min_consistent_views_accepts_none_and_integers():
    from vista_slam_b200.slam import _min_consistent_views
    assert _min_consistent_views(None) == 0
    assert [_min_consistent_views(k) for k in (0, 1, 8, np.int64(3))] == [0, 1, 8, 3]


def test_product_does_not_name_the_checker():
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vista_slam_b200")
    for f in ("slam.py", os.path.join("utils", "slam_utils.py"), os.path.join("csrc", "consistency.cu")):
        src = open(os.path.join(root, f)).read()
        assert "oracle" not in src.replace("oracle/", "").lower(), f
