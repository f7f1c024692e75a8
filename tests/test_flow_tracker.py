"""Keyframe flow tracker -- CPU side.

The numpy oracle (oracle/flow_tracker_oracle.py: pyrDown, Scharr, cornerMinEigenVal, the sequential greedy corner
selection, fixed-point pyramidal LK and FlowTracker.compute_disparity) against golden outputs of the UNMODIFIED
reference tracker (vista_slam/flow_tracker.py with cv2, tools/make_golden_flow.py) on the seeded sequences, plus
known answers, the size refusals of the C ABI and the absence of a CPU path.  The CUDA kernels are held bit-exact to
this oracle by tests/test_flow_gpu.py."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import flow_tracker_oracle as orc

G = np.load(os.path.join(GOLDEN_DIR, "flow.npz"))
SEQS = orc.sequences()
THRESHOLD = 5.0

# Oracle vs cv2 4.13 on these sequences, measured when the goldens were made.  The oracle sums the LK normal equations
# exactly; cv2 sums them in fp32 (SIMD order), so a point whose minimum eigenvalue or determinant sits at its threshold,
# or whose window sits at the bounds, can flip status: 0 to 2 points per frame, at most 0.52 % of a frame's points.
# Where statuses agree, tracked positions differ by at most 5.2e-3 px (a point wandering through a 70-px jump), and by
# more than 1e-3 px for at most 1.3 % of a frame's points.  A flipped point changes the mean disparity by up to
# 0.39 %; with equal statuses the means agree to 1e-4.  Corner lists are identical except on the low-contrast frames
# of sequence (e), where cv2's fp32 box filter puts one more corner (1 of 353) over the quality threshold.
CORNER_SETDIFF_FRAC = 0.006
STATUS_FLIP_FRAC = 0.011
POS_MAX = 0.011
POS_FRAC_ABOVE_1E3 = 0.026
MEAN_REL_EQUAL_STATUS = 1e-3
MEAN_REL_FLIPPED = 8e-3


def _golden(name, t):
    n = int(G[name + "__tracked"][t])
    nc = int(G[name + "__ncorners"][t])
    return dict(decision=bool(G[name + "__decision"][t]), mean=float(G[name + "__mean"][t]), tracked=n,
                next_pts=G[name + "__next_pts"][t, :max(n, 0)], status=G[name + "__status"][t, :max(n, 0)],
                corners=G[name + "__corners"][t, :nc])


@pytest.mark.parametrize("name", sorted(SEQS))
def test_oracle_matches_reference_goldens(name):
    """Decisions equal on every frame; corners, LK status / positions (tracked from the golden's own keyframe corners)
    and the mean disparity within the bounds above."""
    tr = orc.FlowTrackerOracle(THRESHOLD)
    kf_corners_equal = True
    for t, img in enumerate(SEQS[name]):
        g = _golden(name, t)
        kf_pyr = getattr(tr, "kf_pyr", None)
        assert tr.compute_disparity(img) == g["decision"], (name, t)
        if g["tracked"] >= 0:
            kf_pts = _golden(name, t - 1)["corners"]
            nxt, st = orc.lk_track(kf_pyr, orc.pyramid(img), kf_pts)
            st = st[:, 0]
            flips = st != g["status"]
            assert flips.mean() <= STATUS_FLIP_FRAC, (name, t, int(flips.sum()))
            both = (st == 1) & (g["status"] == 1)
            err = np.abs(nxt.reshape(-1, 2)[both] - g["next_pts"][both]).max(-1)
            assert err.max(initial=0) <= POS_MAX, (name, t, err.max(initial=0))
            assert (err > 1e-3).sum() <= POS_FRAC_ABOVE_1E3 * len(err), (name, t)
            if not np.isnan(g["mean"]):
                exact = kf_corners_equal and not flips.any()
                bound = MEAN_REL_EQUAL_STATUS if exact else MEAN_REL_FLIPPED
                assert abs(tr.last_mean_disparity - g["mean"]) <= bound * g["mean"], (name, t)
        else:
            assert tr.last_track is None
        kp = np.zeros((0, 2), np.float32) if tr.kf_pts is None else tr.kf_pts.reshape(-1, 2)
        diff = set(map(tuple, kp.tolist())) ^ set(map(tuple, g["corners"].tolist()))
        assert len(diff) <= CORNER_SETDIFF_FRAC * max(len(kp), 1), (name, t, len(diff))
        kf_corners_equal = np.array_equal(kp, g["corners"])


def test_goldens_cover_every_branch():
    dec = {k: G[k] for k in G.files if k.endswith("__decision")}
    assert sum(int(v.sum()) for v in dec.values()) > 10 and sum(int((~v).sum()) for v in dec.values()) > 20
    assert (G["a_224x224__decision"][1:]).sum() >= 2                            # the threshold is crossed repeatedly
    assert (G["d_384x512__ncorners"] == 1000).all()                             # the cap applies
    e_tracked = [int((G["e_jump_224x224__status"][t] == 1).sum()) for t in range(len(SEQS["e_jump_224x224"]))]
    assert any(0 <= n < 10 and G["e_jump_224x224__tracked"][t] >= 10 for t, n in enumerate(e_tracked))  # case 2
    assert (G["e_jump_224x224__ncorners"] == 6).any()                           # a keyframe with < 10 corners
    assert (G["f_flat_ties_128x160__ncorners"][:2] == 0).all()                  # kf_pts is None
    assert orc.num_levels(168, 224) == 3 and orc.num_levels(169, 169) == 4 and orc.num_levels(168, 168) == 3


def test_mean_disparity_is_the_mean_of_absolute_components():
    """flow_tracker.py:50: norm over the axis of size 1 of (N, 1, 2) points gives |dx| and |dy| separately."""
    kf = np.array([[[10.0, 20.0]], [[30.0, 40.0]]], np.float32)
    nxt = kf + np.array([[[3.0, 4.0]], [[-6.0, 8.0]]], np.float32)
    m, mean = orc.mean_disparity(kf, nxt, np.array([[1], [1]], np.uint8))
    assert m == 2 and mean == pytest.approx((3 + 4 + 6 + 8) / 4.0)          # 5.25, not the Euclidean mean 7.5
    m, mean = orc.mean_disparity(kf, nxt, np.array([[0], [1]], np.uint8))
    assert m == 1 and mean == pytest.approx(7.0)
    shifted = kf + np.array([3.0, 0.0], np.float32)
    assert orc.mean_disparity(kf, shifted, np.ones((2, 1), np.uint8))[1] == pytest.approx(1.5)


def test_pyr_down_and_scharr_known_answers():
    a = np.arange(36, dtype=np.uint8).reshape(6, 6) * 7
    # pyrDown of a linear ramp with REFLECT_101: interior samples are exact, (sum + 128) >> 8 rounds
    d = orc.pyr_down(a)
    assert d.shape == (3, 3) and d[1, 1] == a[2, 2]
    b = np.zeros((5, 7), np.uint8)
    b[2, 3] = 255
    d = orc.pyr_down(b)
    assert d.shape == (3, 4) and d[1, 1] == (6 * 4 * 255 + 128) >> 8 and d[0, 0] == 0
    s = orc.scharr(b).astype(int)
    assert s[2, 2, 0] == 10 * 255 and s[2, 4, 0] == -10 * 255 and s[1, 3, 1] == 10 * 255 and s[3, 3, 1] == -10 * 255
    assert s[1, 2, 0] == 3 * 255 and s[2, 3].tolist() == [0, 0]


def test_corner_tie_order_keeps_the_highest_index():
    pts = orc.good_features(orc.tie_frame()).reshape(-1, 2)
    # four exactly tied maxima at (32..33, 32..33); the highest linear index, (33, 33), wins and suppresses the others
    ys, xs, vals = orc.corner_candidates(orc.tie_frame())
    top = vals == vals[0]
    assert top.sum() >= 4 and (ys[0], xs[0]) == (33, 33)
    assert pts[0].tolist() == [33.0, 33.0]
    assert not any(abs(x - 33) < 8 and abs(y - 33) < 8 and (x, y) != (33, 33) for x, y in pts.tolist())


@pytest.mark.parametrize("name", ["d_384x512", "f_flat_ties_128x160"])
def test_corners_are_spaced_and_capped(name):
    for img in SEQS[name]:
        p = orc.good_features(img)
        if p is None:
            continue
        p = p.reshape(-1, 2).astype(np.float64)
        assert len(p) <= 1000
        d2 = ((p[:, None] - p[None]) ** 2).sum(-1) + np.eye(len(p)) * 1e9
        assert d2.min() >= 64


def test_lk_recovers_an_integer_shift():
    scene = orc.make_scene(3, 200, 200, octaves=(12, 6, 3), gains=(1.0, 0.6, 0.4))
    a = np.clip(np.rint(scene[20:180, 20:180]), 0, 255).astype(np.uint8)
    b = np.clip(np.rint(scene[17:177, 22:182]), 0, 255).astype(np.uint8)   # content moves by (-2, +3)
    p = orc.good_features(a)
    inner = ((p[:, 0] > 30) & (p[:, 0] < 130)).all(-1)
    nxt, st = orc.lk_track(orc.pyramid(a), orc.pyramid(b), p[inner])
    assert st.all()
    np.testing.assert_allclose(nxt - p[inner], np.broadcast_to(np.float32([-2.0, 3.0]), nxt.shape), atol=0.01)


def test_c_abi_refuses_bad_sizes_and_null_groups_before_touching_the_gpu():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    h = ctypes.c_void_p()
    for H, W in ((31, 224), (224, 16), (2049, 64), (64, 4096)):
        assert L.sta_flow_create(H, W, ctypes.byref(h)) == 2 and not h.value
        assert b"[32, 2048]" in L.sta_last_error()
        assert L.sta_flow_scratch_bytes(H, W) == 0
        assert L.sta_op_good_features(None, H, W, None, None, None, None) == 2
        assert L.sta_op_lk_track(None, None, H, W, None, 0, None, None, None, None) == 2
    assert L.sta_flow_scratch_bytes(224, 224) > 2 * (224 + 42) ** 2
    assert L.sta_flow_track_group(None, 1, None, None, 0, None, None) == 2
    assert L.sta_flow_promote_group(None, 1, None, None) == 2


def test_flow_tracker_has_no_cpu_path():
    from vista_slam_b200.flow_tracker import FlowTracker
    tr = FlowTracker(5.0)
    assert tr.min_disparity == 5.0 and tr.last_kf is None and tr.kf_pts is None and tr.kf_gray is None
    assert tr.last_mean_disparity is None
    with pytest.raises(NotImplementedError):
        tr.compute_disparity(np.zeros((64, 64), np.uint8), visualize=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        tr.compute_disparity(torch.zeros(64, 64, dtype=torch.uint8))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="CUDA"):
            tr.compute_disparity(np.zeros((64, 64), np.uint8))
