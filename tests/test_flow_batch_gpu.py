"""Batched keyframe selection -- GPU side: FlowTracker.compute_disparities, compute_disparities_group and
SLAM_image_only.process_images against the one-frame calls.

The batched path promises the one-frame loop's results with no tolerance: the same decisions, last_mean_disparity
equal with ==, and kf_pts / kf_gray equal with torch.equal after every call, whatever the round length, the chunking,
the input form or the other trackers of a group."""
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


def _extra_sequences():
    """test_flow_gpu.py's further sizes: odd sides, the smallest accepted frame, tied maxima."""
    s1 = orc.make_scene(21, 301 + 80, 419 + 80)
    s2 = orc.make_scene(22, 33 + 80, 45 + 80, octaves=(6, 3), gains=(1.0, 0.6))
    return {"odd_301x419": [orc.warp_frame(s1, 301, 419, 0.7 * t, -0.4 * t, 0.002 * t) for t in range(4)],
            "small_33x45": [orc.warp_frame(s2, 33, 45, 0.5 * t, 0.3 * t) for t in range(4)],
            "ties_64x64": [orc.tie_frame(), np.roll(orc.tie_frame(), 1, axis=1)]}


ALL = dict(SEQS, **_extra_sequences())


def _tracker():
    from vista_slam_b200.flow_tracker import FlowTracker
    return FlowTracker(THRESHOLD)


def _state(tr):
    kp = tr.kf_pts
    return tr.last_mean_disparity, None if kp is None else kp.clone(), tr.kf_gray.clone()


def _assert_state(tr, st, where):
    mean, kp, gray = st
    assert tr.last_mean_disparity == mean, where
    got = tr.kf_pts
    assert (got is None) == (kp is None), where
    assert kp is None or torch.equal(got, kp), where
    assert torch.equal(tr.kf_gray, gray), where


def _sequential(frames):
    """Decisions and the state after every frame of the one-frame loop."""
    tr = _tracker()
    dec, states = [], []
    for f in frames:
        dec.append(tr.compute_disparity(f))
        states.append(_state(tr))
    return dec, states


def _gray_frames(frames):
    """The fp32 gray of process_images over RGB versions of the frames, (F, 1, h, w) CUDA."""
    from vista_slam_b200.datasets.slam_images_only import SLAM_image_only
    ds = SLAM_image_only([], resolution=(224, 224))
    rgb = np.stack([np.stack([g, np.roll(g, 3, 1), 255 - g], -1) for g in frames])
    return ds.process_images(rgb)["gray"]


FEEDS = {
    "numpy": lambda frames: list(frames),
    "stacked_u8": lambda frames: torch.from_numpy(np.stack(frames)).cuda(),
}


@pytest.mark.parametrize("feed", sorted(FEEDS))
@pytest.mark.parametrize("name", sorted(ALL))
@pytest.mark.parametrize("round_len", [1, 2, 3, 1000])
def test_whole_sequence_equals_one_frame_loop(name, feed, round_len, monkeypatch):
    from vista_slam_b200 import flow_tracker as ft
    monkeypatch.setattr(ft, "ROUND", round_len)
    frames = ALL[name]
    dec, states = _sequential(frames)
    if name in SEQS:
        assert dec == [bool(v) for v in G[name + "__decision"]], name
    tr = _tracker()
    got = tr.compute_disparities(FEEDS[feed](frames))
    assert got == dec, (name, feed, round_len)
    _assert_state(tr, states[-1], (name, feed, round_len))


@pytest.mark.parametrize("name", sorted(SEQS))
@pytest.mark.parametrize("round_len", [2, 1000])
def test_fp32_gray_of_process_images(name, round_len, monkeypatch):
    from vista_slam_b200 import flow_tracker as ft
    monkeypatch.setattr(ft, "ROUND", round_len)
    gray = _gray_frames(SEQS[name])
    dec, states = _sequential([gray[i] for i in range(gray.shape[0])])
    tr = _tracker()
    assert tr.compute_disparities(gray) == dec, name
    _assert_state(tr, states[-1], name)


@pytest.mark.parametrize("name", sorted(ALL))
@pytest.mark.parametrize("round_len", [1, 3, 1000])
def test_random_chunks_mixed_with_single_calls(name, round_len, monkeypatch):
    from vista_slam_b200 import flow_tracker as ft
    monkeypatch.setattr(ft, "ROUND", round_len)
    frames = ALL[name]
    dec, states = _sequential(frames)
    rng = np.random.default_rng(sum(map(ord, name)) + round_len)
    tr = _tracker()
    i = 0
    while i < len(frames):
        c = int(rng.integers(1, 6))
        chunk = frames[i:i + c]
        feed = FEEDS["numpy" if rng.integers(2) else "stacked_u8"]
        assert tr.compute_disparities(feed(chunk)) == dec[i:i + len(chunk)], (name, i)
        i += len(chunk)
        _assert_state(tr, states[i - 1], (name, i))
        if i < len(frames):
            assert tr.compute_disparity(frames[i]) == dec[i], (name, i)
            _assert_state(tr, states[i], (name, i))
            i += 1


def test_every_promotion_cause_occurs():
    """The golden sequences promote for all three reasons: a keyframe with fewer than 10 corners, fewer than 10
    points tracked, and the mean above the threshold (which test_whole_sequence_equals_one_frame_loop covers)."""
    causes = set()
    for name, frames in SEQS.items():
        dec, states = _sequential(frames)
        for i in range(1, len(frames)):
            if not dec[i]:
                continue
            prev_pts = states[i - 1][1]
            if prev_pts is None or len(prev_pts) < 10:
                causes.add("few_corners")
            elif states[i][0] is None:
                causes.add("few_tracked")
            else:
                assert states[i][0] > THRESHOLD
                causes.add("mean")
    assert causes == {"few_corners", "few_tracked", "mean"}


def _streams(n):
    """n seeded 224x224 streams of 12 frames; stream 0 is the golden sequence e (every promotion cause)."""
    out = [list(SEQS["e_jump_224x224"])]
    for k in range(1, n):
        scene = orc.make_scene(100 + k, 224 + 120, 224 + 120)
        out.append([orc.warp_frame(scene, 224, 224, (1.2 + 0.3 * k) * t, 0.5 * t, 0.002 * t) for t in range(12)])
    return out


def _few_corner_prefix(frames):
    """The shortest prefix after which the tracker's keyframe has fewer than 10 corners."""
    tr = _tracker()
    for i, f in enumerate(frames):
        tr.compute_disparity(f)
        kp = tr.kf_pts
        if kp is None or len(kp) < 10:
            return i + 1
    raise AssertionError("no keyframe with fewer than 10 corners")


@pytest.mark.parametrize("n", [1, 3, 8])
def test_group_equals_each_trackers_own_run(n):
    from vista_slam_b200.flow_tracker import compute_disparities_group
    streams = _streams(n)
    # tracker states before the group calls: fresh, mid-sequence, and with a keyframe of fewer than 10 corners
    starts = [_few_corner_prefix(streams[0])] + [0 if k % 2 else 3 + k % 4 for k in range(1, n)]
    group, twins = [_tracker() for _ in range(n)], [_tracker() for _ in range(n)]
    for k in range(n):
        for f in streams[k][:starts[k]]:
            group[k].compute_disparity(f)
            twins[k].compute_disparity(f)
    pos = list(starts)
    for take in (1, 4, 100):  # one frame per tracker (the live case), then several, then the rest
        chunks = [streams[k][pos[k]:pos[k] + take] for k in range(n)]
        got = compute_disparities_group(group, chunks)
        for k in range(n):
            assert got[k] == [twins[k].compute_disparity(f) for f in chunks[k]], (n, k, take)
            _assert_state(group[k], _state(twins[k]), (n, k, take))
            pos[k] += len(chunks[k])


def test_group_with_fresh_trackers_and_stacked_frames():
    from vista_slam_b200.flow_tracker import compute_disparities_group
    streams = _streams(4)
    group = [_tracker() for _ in range(4)]
    got = compute_disparities_group(group, [torch.from_numpy(np.stack(s)).cuda() for s in streams])
    for k in range(4):
        dec, states = _sequential(streams[k])
        assert got[k] == dec, k
        _assert_state(group[k], states[-1], k)


def test_refusals_leave_trackers_unchanged():
    from vista_slam_b200.flow_tracker import compute_disparities_group
    a_frames, b_frames = SEQS["a_224x224"], SEQS["b_192x256"]
    a, twin, other = _tracker(), _tracker(), _tracker()
    for f in a_frames[:3]:
        a.compute_disparity(f)
        twin.compute_disparity(f)
    with pytest.raises(ValueError):
        compute_disparities_group([a, a], [a_frames[3:4], a_frames[4:5]])
    with pytest.raises(ValueError):
        compute_disparities_group([a, other], [a_frames[3:4], b_frames[:1]])
    with pytest.raises(ValueError):
        a.compute_disparities(b_frames[:2])
    with pytest.raises(ValueError):
        a.compute_disparities([a_frames[3], b_frames[3]])
    with pytest.raises(ValueError):
        compute_disparities_group([a, other], [a_frames[3:4], [a_frames[4].astype(np.float32) / 255]])
    assert other.last_kf is None
    assert a.compute_disparities([]) == [] and compute_disparities_group([a, other], [[], []]) == [[], []]
    _assert_state(a, _state(twin), "after refusals")
    for f in a_frames[3:]:
        assert a.compute_disparity(f) == twin.compute_disparity(f)
        _assert_state(a, _state(twin), "after refusals")


def test_c_group_refusals_come_before_any_launch():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    s = _lib.cur_stream()
    hs = []
    for H, W in ((64, 64), (64, 64), (64, 80)):
        h = ctypes.c_void_p()
        _lib.check(L.sta_flow_create(H, W, ctypes.byref(h)))
        hs.append(h.value)
    try:
        frames = torch.zeros(2, 64, 64, dtype=torch.uint8, device="cuda")
        stats = (_lib.StaFlowStats * 3)()
        arr = lambda *v: (ctypes.c_void_p * len(v))(*v)  # noqa: E731
        assert L.sta_flow_track_group(arr(hs[0]), 1, None, _lib.ptr(frames), 0, stats, s) == 2  # no keyframe
        _lib.check(L.sta_flow_set_keyframe_group(arr(hs[0], hs[1]), 2, _lib.ptr(frames), 0, s))
        assert L.sta_flow_set_keyframe_group(arr(hs[0], hs[0]), 2, _lib.ptr(frames), 0, s) == 2  # repeated
        assert L.sta_flow_track_group(arr(hs[0], hs[2]), 2, None, _lib.ptr(frames), 0, stats, s) == 2  # mixed sizes
        assert L.sta_flow_track_group(arr(hs[0], hs[1], hs[0]), 3, None, _lib.ptr(frames), 0, stats, s) == 2  # split
        assert L.sta_flow_track_group(arr(hs[0]), 0, None, _lib.ptr(frames), 0, stats, s) == 2
        assert L.sta_flow_track_group(arr(hs[0]), 1, None, None, 0, stats, s) == 2
        held = (ctypes.c_int * 1)(1)
        assert L.sta_flow_track_group(arr(hs[0]), 1, held, None, 0, stats, s) == 2  # holds nothing
        assert L.sta_flow_promote_group(arr(hs[0]), 1, (ctypes.c_int * 1)(0), s) == 2  # no group track
        _lib.check(L.sta_flow_track_group(arr(hs[0], hs[0]), 2, None, _lib.ptr(frames), 0, stats, s))
        assert L.sta_flow_promote_group(arr(hs[0]), 1, (ctypes.c_int * 1)(2), s) == 2  # no such frame
        _lib.check(L.sta_flow_promote_group(arr(hs[0]), 1, (ctypes.c_int * 1)(0), s))
        two = (ctypes.c_int * 2)(1, 1)
        assert L.sta_flow_track_group(arr(hs[0], hs[0]), 2, two, None, 0, stats, s) == 2  # holds one frame
        _lib.check(L.sta_flow_track_group(arr(hs[0]), 1, held, None, 0, stats, s))
        torch.cuda.synchronize()
    finally:
        for h in hs:
            L.sta_flow_destroy(ctypes.c_void_p(h))


@pytest.mark.parametrize("portrait", [False, True])
@pytest.mark.parametrize("F", [1, 5])
@pytest.mark.parametrize("resolution", [(224, 224), (256, 192)])
def test_process_images_equals_process_image(portrait, F, resolution):
    from vista_slam_b200.datasets.slam_images_only import SLAM_image_only
    ds = SLAM_image_only([], resolution=resolution)
    H, W = (640, 480) if portrait else (480, 640)
    scene = orc.make_scene(40 + F, H + 80, W + 80)
    rgb = []
    for t in range(F):
        g = orc.warp_frame(scene, H, W, 1.5 * t, -0.7 * t, 0.001 * t)
        rgb.append(np.stack([g, np.roll(g, 5, 0), 255 - g], -1))
    names = ["/data/frame_%03d.png" % t for t in range(F)]
    for batch in (rgb, torch.from_numpy(np.stack(rgb)).cuda()):
        out = ds.process_images(batch, names)
        assert out["rgb"].shape[0] == F and out["gray"].shape[:2] == (F, 1)
        assert out["img_name"] == [os.path.basename(n) for n in names]
        for t in range(F):
            one = ds.process_image(rgb[t], names[t])
            assert torch.equal(out["rgb"][t], one["rgb"]) and torch.equal(out["gray"][t], one["gray"]), (F, t)


def test_two_runs_are_bit_identical():
    for name in ("a_224x224", "d_384x512", "e_jump_224x224"):
        runs = []
        for _ in range(2):
            tr = _tracker()
            dec = tr.compute_disparities(SEQS[name])
            runs.append((dec, _state(tr)))
        (d1, s1), (d2, s2) = runs
        assert d1 == d2 and s1[0] == s2[0] and torch.equal(s1[2], s2[2])
        assert (s1[1] is None and s2[1] is None) or torch.equal(s1[1], s2[1])
