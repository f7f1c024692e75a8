"""CPU: the grouped keyframe insertion is declared and exported, refuses null arguments before touching a device, and
PoseGraphOpt.start_group refuses what optimize_group refuses."""
import os
import re

import pytest
import torch

from conftest import ROOT


def test_grouped_insertion_is_declared_and_exported():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "sta_b200.h")).read()
    assert "int sta_graph_add_keyframes(const StaGraphKeyframe* kfs, int count, void* scratch, size_t scratch_bytes, " \
           "void* stream);" in hdr
    assert "size_t sta_graph_add_keyframes_scratch_bytes(const StaGraphKeyframe* kfs, int count);" in hdr
    assert int(re.search(r"STA_GRAPH_MAX_GROUP_KEYFRAMES\s*=\s*(\d+)", hdr).group(1)) == _lib.GRAPH_MAX_GROUP_KEYFRAMES
    for name in ("sta_graph_add_keyframes", "sta_graph_add_keyframes_scratch_bytes", "sta_graph_add_keyframe"):
        assert hasattr(L, name)
    # the ctypes mirror has the header's field order
    body = re.search(r"typedef struct StaGraphKeyframe \{(.*?)\} StaGraphKeyframe;", hdr, re.S).group(1)
    fields = re.findall(r"\*?\s*(\w+)\s*[,;]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert fields == [f for f, _ in _lib.StaGraphKeyframe._fields_]


def test_null_arguments_are_refused():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    assert L.sta_graph_add_keyframes(None, 1, None, 0, None) != 0
    assert L.sta_graph_add_keyframes_scratch_bytes(None, 1) == 0
    tab = (_lib.StaGraphKeyframe * 2)()  # every field null
    for count in (1, 2):
        assert L.sta_graph_add_keyframes(tab, count, None, 0, None) != 0
        assert b"null" in L.sta_last_error()
        assert L.sta_graph_add_keyframes_scratch_bytes(tab, count) == 0
    for count in (0, -1, _lib.GRAPH_MAX_GROUP_KEYFRAMES + 1):
        assert L.sta_graph_add_keyframes(tab, count, None, 0, None) != 0
        assert L.sta_graph_add_keyframes_scratch_bytes(tab, count) == 0
    assert L.sta_graph_add_keyframe(None, 1, 1, None, None, None, 0, 0, 1, 1, None, None, None, None, None, None, None) != 0


class _Stand:
    """What the group checks read of a PoseGraphOpt: its nodes' device."""

    def __init__(self, device="cpu"):
        self.nodes = torch.zeros(3, 8, device=device)
        self.sparse = False


def _raises_both(graphs, edges, poses, weights, match):
    from vista_slam_b200.pose_graph import PoseGraphOpt
    with pytest.raises(ValueError, match=match):
        PoseGraphOpt.optimize_group(graphs, edges, poses, weights)
    with pytest.raises(ValueError, match=match):
        PoseGraphOpt.start_group(graphs, edges, poses, weights)


def test_start_group_refusals_match_optimize_group():
    e, p, w = torch.zeros(4, 2, dtype=torch.int64), torch.zeros(4, 8), torch.zeros(4, 7)
    a, b = _Stand(), _Stand()
    _raises_both([a, b], [e], [p, p], [w, w], "one entry per graph")
    _raises_both([a, a], [e, e], [p, p], [w, w], "named twice")
    _raises_both([a, _Stand("meta")], [e, e], [p, p], [w, w], "one device")
    _raises_both([a, b], [e, e], [p, p[:3]], [w, w], "one row per edge")
    _raises_both([a], [e], [p], [w[:2]], "one row per edge")
