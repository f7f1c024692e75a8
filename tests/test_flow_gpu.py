"""Keyframe flow tracker -- GPU side (csrc/flow.cu through the C ABI and vista_slam_b200/flow_tracker.py).

The kernels are bit-exact with the numpy oracle (oracle/flow_tracker_oracle.py): the same corners in the same order,
the same LK status and bit-identical next points, on every golden sequence and on two further sizes.  FlowTracker's
decisions equal the unmodified reference's (tests/golden/flow.npz) on every frame, within the oracle-vs-cv2 bounds of
tests/test_flow_tracker.py for the mean disparity."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import flow_tracker_oracle as orc

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(GOLDEN_DIR, "flow.npz"))
SEQS = orc.sequences()
THRESHOLD = 5.0
MEAN_REL_FLIPPED = 8e-3   # tests/test_flow_tracker.py: the oracle's mean vs cv2's when a point's status flips


def _extra_sequences():
    """Two sizes beyond the goldens: odd sides (3 pyramid levels above the base) and the smallest accepted frame."""
    s1 = orc.make_scene(21, 301 + 80, 419 + 80)
    s2 = orc.make_scene(22, 33 + 80, 45 + 80, octaves=(6, 3), gains=(1.0, 0.6))
    return {"odd_301x419": [orc.warp_frame(s1, 301, 419, 0.7 * t, -0.4 * t, 0.002 * t) for t in range(4)],
            "small_33x45": [orc.warp_frame(s2, 33, 45, 0.5 * t, 0.3 * t) for t in range(4)],
            "ties_64x64": [orc.tie_frame(), np.roll(orc.tie_frame(), 1, axis=1)]}


ALL = dict(SEQS, **_extra_sequences())


@pytest.mark.parametrize("name", sorted(ALL))
def test_kernels_bit_exact_with_oracle(name):
    from vista_slam_b200.flow_tracker import calc_optical_flow_pyr_lk, good_features_to_track
    frames = ALL[name]
    for t, img in enumerate(frames):
        ref = orc.good_features(img)
        got = good_features_to_track(img)
        if ref is None:
            assert got is None, (name, t)
            continue
        got = got.cpu().numpy()
        assert got.shape == ref.shape and np.array_equal(got, ref), (name, t)
        if t + 1 < len(frames):
            nxt_ref, st_ref = orc.lk_track(orc.pyramid(img), orc.pyramid(frames[t + 1]), ref)
            nxt, st = calc_optical_flow_pyr_lk(img, frames[t + 1], got)
            assert np.array_equal(st.cpu().numpy(), st_ref), (name, t)
            assert np.array_equal(nxt.cpu().numpy().view(np.uint32), nxt_ref.view(np.uint32)), (name, t)


def _run(name, feed):
    from vista_slam_b200.flow_tracker import FlowTracker
    tr = FlowTracker(THRESHOLD)
    out = []
    for img in SEQS[name]:
        d = tr.compute_disparity(feed(img))
        kp = tr.kf_pts
        out.append((d, tr.last_mean_disparity, None if kp is None else kp.cpu().numpy(), tr.kf_gray.cpu().numpy()))
    return out


@pytest.mark.parametrize("name", sorted(SEQS))
def test_flow_tracker_matches_reference_and_oracle(name):
    got = _run(name, lambda img: img)                                                # numpy uint8, uploaded
    ora = orc.FlowTrackerOracle(THRESHOLD)
    for t, (img, (d, mean, kp, kf_gray)) in enumerate(zip(SEQS[name], got)):
        assert d == bool(G[name + "__decision"][t]), (name, t)
        assert ora.compute_disparity(img) == d, (name, t)
        ref_kp = ora.kf_pts
        assert (kp is None) == (ref_kp is None) and (kp is None or np.array_equal(kp, ref_kp)), (name, t)
        assert np.array_equal(kf_gray, ora.kf_gray), (name, t)
        gm = float(G[name + "__mean"][t])
        if np.isnan(gm):
            continue
        # the device sums |dx| + |dy| in fp64; numpy's mean is an fp32 pairwise sum
        assert mean == pytest.approx(ora.last_mean_disparity, rel=1e-6), (name, t)
        assert abs(mean - gm) <= MEAN_REL_FLIPPED * gm, (name, t)


def test_fp32_gray_from_preprocessing_equals_uint8_path():
    from vista_slam_b200.datasets.slam_images_only import SLAM_image_only
    from vista_slam_b200.flow_tracker import FlowTracker
    ds = SLAM_image_only([], resolution=(224, 224))
    scene = orc.make_scene(31, 480 + 120, 640 + 120)
    grays = []
    for t in range(8):
        g = orc.warp_frame(scene, 480, 640, 2.5 * t, 1.0 * t, 0.002 * t)
        rgb = np.stack([g, np.roll(g, 3, 1), 255 - g], -1)
        grays.append(ds.process_image(rgb)["gray"])
    a, b = FlowTracker(THRESHOLD), FlowTracker(THRESHOLD)
    for g in grays:
        da = a.compute_disparity(g)
        db = b.compute_disparity((g.squeeze(0).cpu().numpy() * 255).astype(np.uint8))
        assert da == db and a.last_mean_disparity == b.last_mean_disparity
        assert torch.equal(a.kf_gray, b.kf_gray)
        assert (a.kf_pts is None and b.kf_pts is None) or torch.equal(a.kf_pts, b.kf_pts)


def test_two_runs_are_bit_identical():
    for name in ("a_224x224", "d_384x512"):
        r1 = _run(name, lambda img: torch.from_numpy(img).cuda())
        r2 = _run(name, lambda img: torch.from_numpy(img).cuda())
        for x, y in zip(r1, r2):
            assert x[0] == y[0] and x[1] == y[1]
            assert (x[2] is None and y[2] is None) or np.array_equal(x[2], y[2])


def test_group_promoted_keyframe_equals_fresh_keyframe():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    f0, f1 = SEQS["b_192x256"][0], SEQS["b_192x256"][3]
    H, W = f0.shape
    d0, d1 = torch.from_numpy(f0).cuda(), torch.from_numpy(f1).cuda()
    s = _lib.cur_stream()

    def tracker():
        h = ctypes.c_void_p()
        _lib.check(L.sta_flow_create(H, W, ctypes.byref(h)))
        return h

    def keyframe(h):
        gray = torch.empty(H, W, dtype=torch.uint8, device="cuda")
        der = torch.empty(H, W, 2, dtype=torch.int16, device="cuda")
        pts = torch.empty(1000, 2, dtype=torch.float32, device="cuda")
        cnt = torch.empty(1, dtype=torch.int32, device="cuda")
        _lib.check(L.sta_flow_keyframe_level0(h, _lib.ptr(gray), _lib.ptr(der), s))
        _lib.check(L.sta_flow_keyframe_points(h, _lib.ptr(pts), _lib.ptr(cnt), s))
        n = int(cnt.item())
        return gray.cpu().numpy(), der.cpu().numpy(), pts[:n].cpu().numpy()

    a, b = tracker(), tracker()
    ta, tb = (ctypes.c_void_p * 1)(a.value), (ctypes.c_void_p * 1)(b.value)
    frame0 = (ctypes.c_int * 1)(0)
    try:
        stats = _lib.StaFlowStats()
        _lib.check(L.sta_flow_set_keyframe_group(ta, 1, _lib.ptr(d0), 0, s))
        _lib.check(L.sta_flow_track_group(ta, 1, None, _lib.ptr(d1), 0, ctypes.byref(stats), s))
        assert stats.n_corners == len(orc.good_features(f0)) and stats.n_tracked >= 10
        _lib.check(L.sta_flow_promote_group(ta, 1, frame0, s))
        _lib.check(L.sta_flow_set_keyframe_group(tb, 1, _lib.ptr(d1), 0, s))
        ka, kb = keyframe(a), keyframe(b)
        assert np.array_equal(ka[0], f1) and np.array_equal(ka[0], kb[0])
        assert np.array_equal(ka[1], kb[1]) and np.array_equal(ka[1], orc.scharr(f1))
        assert np.array_equal(ka[2], kb[2]) and np.array_equal(ka[2], orc.good_features(f1).reshape(-1, 2))
        assert L.sta_flow_promote_group(ta, 1, frame0, s) == 2   # nothing tracked since the last promotion
    finally:
        L.sta_flow_destroy(a)
        L.sta_flow_destroy(b)


def test_frame_size_change_is_refused():
    from vista_slam_b200.flow_tracker import FlowTracker
    tr = FlowTracker(THRESHOLD)
    assert tr.compute_disparity(SEQS["a_224x224"][0])
    with pytest.raises(ValueError):
        tr.compute_disparity(SEQS["b_192x256"][0])
