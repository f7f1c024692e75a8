"""CPU: the gated regression across caches yields one result per keyframe, in order, also when a keyframe without
candidate edges (another session's first view) sits between two keyframes of one edge chunk."""
from vista_slam_b200.keyframe import MAX_EDGES, KeyframeFrontend, regress_keyframes_gated_group


class _Cache(KeyframeFrontend):
    def _regress_chunk(self, items, rel_pose_thres, pad):
        for c, i, js in items:
            yield c, i, list(js), pad


def test_group_regression_yields_align_with_items():
    a, b = _Cache(None), _Cache(None)
    items = [(a, 5, [4, 3, 2]), (b, 0, []), (b, 1, [0]), (a, 6, list(range(MAX_EDGES))), (b, 2, [1, 0]), (a, 0, [])]
    out = list(regress_keyframes_gated_group(items, 0.5))
    assert out == [(a, 5, [4, 3, 2], True), None, (b, 1, [0], True), (a, 6, list(range(MAX_EDGES)), True),
                   (b, 2, [1, 0], True), None]
    one = list(regress_keyframes_gated_group([(b, 0, []), (b, 1, [0]), (b, 2, [1, 0])], 0.5))
    assert one == [None, (b, 1, [0], False), (b, 2, [1, 0], False)]
