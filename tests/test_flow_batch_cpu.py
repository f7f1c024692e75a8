"""Batched keyframe selection -- CPU side: the group entry points are declared and exported, the Python surface refuses
bad arguments with ValueError before touching the device, and without CUDA it raises instead of falling back."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT

NEW = ("sta_flow_set_keyframe_group", "sta_flow_track_group", "sta_flow_promote_group", "sta_preprocess_rgb8_many")


def test_group_entry_points_are_declared_and_exported():
    from vista_slam_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "sta_b200.h")).read()
    declared = set(re.findall(r"\b(sta_[a-z0-9_]+)\s*\(", hdr))
    L = _lib.lib()
    for name in NEW:
        assert name in declared, name
        assert hasattr(L, name) and getattr(L, name).argtypes, name


def test_c_refusals_need_no_device():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    stats = (_lib.StaFlowStats * 1)()
    assert L.sta_flow_track_group(None, 1, None, None, 0, stats, None) == 2
    assert L.sta_flow_track_group((_lib.c_void_p * 1)(None), 1, None, None, 0, stats, None) == 2
    assert L.sta_flow_set_keyframe_group(None, 0, None, 0, None) == 2
    assert L.sta_flow_promote_group((_lib.c_void_p * 1)(None), 1, None, None) == 2
    assert L.sta_preprocess_rgb8_many(None, 0, 480, 640, 224, 224, 10, 10, None, None, None, None) == 2
    assert b"frame count" in L.sta_last_error()


def _trackers(n):
    from vista_slam_b200.flow_tracker import FlowTracker
    return [FlowTracker(5.0) for _ in range(n)]


def test_group_arguments_are_checked_on_the_host():
    from vista_slam_b200.flow_tracker import compute_disparities_group
    a, b = _trackers(2)
    f, g = np.zeros((64, 64), np.uint8), np.zeros((64, 80), np.uint8)
    with pytest.raises(ValueError):
        compute_disparities_group([a, a], [[f], [f]])          # a repeated tracker
    with pytest.raises(ValueError):
        compute_disparities_group([a, b], [[f], [g]])          # frames of different sizes
    with pytest.raises(ValueError):
        compute_disparities_group([a, b], [[f], [f.astype(np.float32)]])
    with pytest.raises(ValueError):
        compute_disparities_group([a, b], [[f]])               # one list per tracker
    with pytest.raises(ValueError):
        a.compute_disparities([f, g])
    with pytest.raises(ValueError):
        a.compute_disparities(torch.zeros(2, 1, 64, 64, dtype=torch.uint8))  # neither stacked form
    with pytest.raises(ValueError):
        a.compute_disparities([np.zeros((64, 64, 3), np.uint8)])
    assert a.compute_disparities([]) == []
    assert compute_disparities_group([a, b], [[], []]) == [[], []]
    assert a.last_kf is None and b.last_kf is None


def test_no_cpu_fallback(monkeypatch):
    from vista_slam_b200.flow_tracker import compute_disparities_group
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    a, b = _trackers(2)
    frames = [np.zeros((64, 64), np.uint8)] * 3
    with pytest.raises(RuntimeError):
        a.compute_disparities(frames)
    with pytest.raises(RuntimeError):
        compute_disparities_group([a, b], [frames, frames[:1]])
    assert a.last_kf is None


def test_round_length_is_a_module_constant():
    from vista_slam_b200 import flow_tracker
    import inspect
    assert isinstance(flow_tracker.ROUND, int) and flow_tracker.ROUND >= 1
    assert list(inspect.signature(flow_tracker.FlowTracker.compute_disparities).parameters) == ["self", "frames"]


def test_process_images_arguments_are_checked_on_the_host():
    from vista_slam_b200.datasets.slam_images_only import SLAM_image_only
    ds = SLAM_image_only([], resolution=(224, 224))
    with pytest.raises(ValueError):
        ds.process_images([np.zeros((48, 64, 3), np.uint8), np.zeros((64, 48, 3), np.uint8)])
    with pytest.raises(ValueError):
        ds.process_images([np.zeros((48, 64), np.uint8)])
    with pytest.raises(ValueError):
        ds.process_images(np.zeros((2, 48, 64, 3), np.float32))
    with pytest.raises(ValueError):
        ds.process_images([np.zeros((48, 64, 3), np.uint8)], img_names=["a", "b"])
    with pytest.raises(ValueError):
        ds.process_images([])
