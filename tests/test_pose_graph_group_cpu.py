"""CPU: the argument checks of sta_pose_graph_group_scratch_bytes and the refusals of sta_pose_graph_lm_step_group, which
both come before anything reaches the device (the descriptor pointers below are never dereferenced)."""
import ctypes

import pytest

from vista_slam_b200 import _lib

FAKE = 4096  # stands for a device pointer


def _graph(num_nodes=40, num_edges=90, num_opt=39):
    return _lib.StaPgGraph(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, num_nodes, num_edges, num_opt, 1e-4)


def _table(*graphs):
    return (_lib.StaPgGraph * len(graphs))(*graphs)


def test_group_scratch_bytes():
    L = _lib.lib()
    a, b = _graph(), _graph(300, 700, 120)
    one = L.sta_pose_graph_group_scratch_bytes(_table(a), 1)
    # a group of one holds the one-graph step's scratch
    assert one >= L.sta_pose_graph_scratch_bytes(40, 90, 39) > 8 * (7 * 39) ** 2
    two = L.sta_pose_graph_group_scratch_bytes(_table(a, b), 2)
    assert two == L.sta_pose_graph_group_scratch_bytes(_table(b, a), 2)
    assert two >= L.sta_pose_graph_scratch_bytes(40, 90, 39) + L.sta_pose_graph_scratch_bytes(300, 700, 120) - 256
    full = L.sta_pose_graph_group_scratch_bytes(_table(*[a] * _lib.PG_GROUP_MAX), _lib.PG_GROUP_MAX)
    assert full > _lib.PG_GROUP_MAX * (one - 256)
    # every graph's part starts on a 256-byte boundary, odd node counts included (its fp64 arrays stay aligned)
    odd = _table(_graph(25, 40, 10), _graph(33, 51, 33), _graph(7, 3, 1))
    assert L.sta_pose_graph_group_scratch_bytes(odd, 3) % 256 == 0
    edge = _graph(_lib.PG_DENSE_MAX_OPT, 10, _lib.PG_DENSE_MAX_OPT)
    assert L.sta_pose_graph_group_scratch_bytes(_table(edge), 1) > 8 * (7 * _lib.PG_DENSE_MAX_OPT) ** 2


@pytest.mark.parametrize("case", ["null_table", "G0", "G_over", "G_negative", "nodes", "edges", "meas", "weights",
                                  "opt_idx", "nodes_out", "no_nodes", "no_edges", "no_opt", "negative", "opt_over_nodes",
                                  "over_dense_limit"])
def test_group_refusals(case):
    L = _lib.lib()
    G = 2
    tab = _table(_graph(), _graph(300, 700, 120))
    if case == "null_table":
        tab = None
    elif case == "G0":
        G = 0
    elif case == "G_over":
        tab, G = _table(*[_graph()] * (_lib.PG_GROUP_MAX + 1)), _lib.PG_GROUP_MAX + 1
    elif case == "G_negative":
        G = -1
    elif case in ("nodes", "edges", "meas", "weights", "opt_idx", "nodes_out"):
        setattr(tab[1], case, None)
    else:
        tab[1] = {"no_nodes": _graph(0, 90, 0), "no_edges": _graph(40, 0, 39), "no_opt": _graph(40, 90, 0),
                  "negative": _graph(40, -5, 39), "opt_over_nodes": _graph(40, 90, 41),
                  "over_dense_limit": _graph(_lib.PG_DENSE_MAX_OPT + 1, 90, _lib.PG_DENSE_MAX_OPT + 1)}[case]
    assert L.sta_pose_graph_group_scratch_bytes(tab, G) == 0
    info = scratch = ctypes.c_void_p(FAKE)
    assert L.sta_pose_graph_lm_step_group(tab, G, 1e-6, 1e32, info, scratch, 1 << 40, None) == 2
    assert b"requirement failed" in L.sta_last_error()


def test_group_step_refuses_its_buffers():
    L = _lib.lib()
    tab = _table(_graph(), _graph(300, 700, 120))
    need = L.sta_pose_graph_group_scratch_bytes(tab, 2)
    p = ctypes.c_void_p(FAKE)
    for info, scratch, nbytes, msg in ((None, p, need, b"null pointer"), (p, None, need, b"null pointer"),
                                       (p, ctypes.c_void_p(FAKE + 4), need, b"aligned"),
                                       (p, p, need - 1, b"scratch smaller")):
        assert L.sta_pose_graph_lm_step_group(tab, 2, 1e-6, 1e32, info, scratch, nbytes, None) == 2
        assert msg in L.sta_last_error()
