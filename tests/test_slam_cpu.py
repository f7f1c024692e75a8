"""CPU: the numpy restatement of OnlineSLAM's graph bookkeeping and export (oracle/slam_oracle.py) against the unmodified
reference's record (tests/golden/slam_graph.npz, tools/make_golden_slam.py), the import hygiene of
vista_slam_b200.slam, and the new C-ABI symbols.

Bounds: integers, masks and point order must be equal.  Floats: the reference sums the depth-scale reductions in float32
(torch) where the oracle sums in float64, so a scale may differ by a few float32 ulps; node poses inherit that through
the Sim(3) products and the PGO.  Poses, measurements and weights are compared at 2e-5 absolute (values are O(1)),
points at 1e-4 absolute (translation O(1) plus depth O(3) times a relative error of a few ulps)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN_DIR, ROOT
from oracle import slam_oracle as so

CFG = dict(rel_pose_thres=0.75, neighbor_edge_num=3, loop_edge_num=3, pgo_every=6)


@pytest.fixture(scope="module")
def g():
    return dict(np.load(os.path.join(GOLDEN_DIR, "slam_graph.npz")))


@pytest.fixture(scope="module")
def run():
    stream = so.make_stream()
    return stream, so.run(stream, **CFG)


def test_oracle_graph_equals_reference(g, run):
    stream, (graph, kf, pgos) = run
    N, E = len(g["node_to_view"]), len(g["edges"])
    assert graph.num_nodes == N and graph.num_edges == E
    np.testing.assert_array_equal(graph.node_to_view[:N], g["node_to_view"])
    np.testing.assert_array_equal(graph.node_to_connected_view[:N], g["node_to_connected_view"])
    np.testing.assert_array_equal(graph.edges[:E], g["edges"])
    np.testing.assert_allclose(graph.meas[:E], g["meas"], atol=2e-5, rtol=0)
    np.testing.assert_allclose(graph.weight[:E], g["weight"], atol=2e-5, rtol=0)
    for t, r in enumerate(kf):
        assert r["num_nodes"] == g["kf_num_nodes"][t] and r["num_edges"] == g["kf_num_edges"][t]
        n = r["num_nodes"]
        np.testing.assert_allclose(r["pose"], g["kf_pose"][t, :n], atol=2e-5, rtol=0)
        np.testing.assert_array_equal(r["best_node"], g["kf_best_node"][t, :t + 1])
    # PGO: node sets, related masks, weights (the PoseGraphOpt per-edge pairing) and results
    assert len(pgos) == len(g["pgo_num_edges"]) >= 3
    o_ptr = r_ptr = n_ptr = 0
    for p, ne, nn in zip(pgos, g["pgo_num_edges"], g["pgo_num_nodes"]):
        no = len(p["opt_idx"])
        np.testing.assert_array_equal(p["opt_idx"], g["pgo_opt_idx"][o_ptr:o_ptr + no])
        np.testing.assert_array_equal(p["related"], g["pgo_related"][r_ptr:r_ptr + ne])
        np.testing.assert_allclose(graph.weight[:ne][p["related"]], g["pgo_weight"][r_ptr:r_ptr + ne][p["related"]], atol=2e-5,
                                   rtol=0)
        np.testing.assert_allclose(p["nodes"], g["pgo_nodes"][n_ptr:n_ptr + nn], atol=2e-5, rtol=0)
        np.testing.assert_allclose(p["result"], g["pgo_result"][n_ptr:n_ptr + nn], atol=2e-5, rtol=0)
        o_ptr, r_ptr, n_ptr = o_ptr + no, r_ptr + ne, n_ptr + nn


def test_oracle_export_equals_reference(g, run):
    stream, (graph, _, _) = run
    ex = so.export(graph, stream["n_views"], 4.2, so.stream_images(stream))
    np.testing.assert_allclose(ex["trajectory"], g["out_trajectory"], atol=2e-5, rtol=0)
    np.testing.assert_allclose(ex["scales"], g["out_scales"], atol=2e-5, rtol=0)
    np.testing.assert_array_equal(ex["depths"], g["out_depths"])
    np.testing.assert_array_equal(ex["confs"], g["out_confs"])
    np.testing.assert_array_equal(ex["intrinsics"], g["out_intrinsics"])
    assert len(ex["points"]) == len(g["ply_points"])
    np.testing.assert_allclose(ex["points"], g["ply_points"], atol=1e-4, rtol=0)
    np.testing.assert_allclose(ex["colors"], g["ply_colors"], atol=1e-6, rtol=0)
    assert float(g["out_confs_thres"]) == 4.2
    assert list(g["out_files"]) == ["confs.npz", "depths.npy", "images.npy", "intrinsics.npy", "pointcloud.ply",
                                    "scales.npy", "trajectory.npy", "view_graph.npz"]


def test_reference_behaviours_pinned_by_the_golden(g):
    # node 0 is view 1's first node, node 1 view 0's; view 0 keeps the identity and view 1 gets identity o sim3_10
    assert g["node_to_view"][0] == 1 and g["node_to_view"][1] == 0
    np.testing.assert_array_equal(g["kf_pose"][1, 1], [0, 0, 0, 0, 0, 0, 1, 1])
    np.testing.assert_allclose(g["kf_pose"][1, 0], g["meas"][0], atol=1e-6)
    # the edge i - j = 1 is always kept: every view v >= 1 has a node connected to v - 1
    ptr = np.concatenate([[0], np.cumsum(g["out_view_graph_len"])])
    for v in range(1, len(ptr) - 1):
        assert v - 1 in g["out_view_graph"][ptr[v]:ptr[v + 1]]
    # the loop-related VIEW ids entered the first PGO after a loop as NODE ids
    stream = so.make_stream()
    loop_views = {v for i in range(stream["n_views"]) for j, _ in stream["loops"][i][:3]
                  for v in (i, j) if so.keep_edge(stream["edges"][(i, j)]["conf"], i, j, 0.75)}
    assert loop_views and loop_views <= set(g["pgo_opt_idx"].tolist())


def test_make_golden_slam_regenerates_the_golden(tmp_path, g):
    if not os.path.isdir("/root/reference/vista_slam"):
        pytest.skip("the reference tree is not present")
    out = tmp_path / "slam_graph.npz"
    subprocess.run([sys.executable, os.path.join(ROOT, "tools", "make_golden_slam.py"), str(out)], check=True,
                   capture_output=True)
    new = np.load(out)
    assert sorted(new.files) == sorted(g)
    for k in g:
        assert new[k].dtype == g[k].dtype and new[k].shape == g[k].shape, k
        assert new[k].tobytes() == g[k].tobytes(), k


def test_slam_module_imports_without_pypose_munch_colorama_open3d():
    code = ("import sys\n"
            "for m in ('pypose', 'munch', 'colorama', 'open3d'):\n"
            "    sys.modules[m] = None  # any import of them raises\n"
            "import vista_slam_b200.slam as s\n"
            "assert s.OnlineSLAM\n"
            "assert not any(m in sys.modules and sys.modules[m] is not None for m in ('pypose', 'munch', 'colorama', 'open3d'))\n")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=ROOT)


def test_graph_symbols_are_exported():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    for name in ("sta_graph_create", "sta_graph_destroy", "sta_graph_tables", "sta_graph_reset", "sta_graph_flags",
                 "sta_graph_add_keyframe", "sta_graph_export_scratch_bytes", "sta_graph_export"):
        assert hasattr(L, name), name
    assert L.sta_version() == 2
    assert L.sta_graph_export_scratch_bytes(2, 32) >= 2 * 32 * 12 + 8


def test_compaction_order_is_view_row_column():
    conf = np.array([[[5.0, 1.0], [4.2, 7.0]], [[9.0, 4.3], [0.0, 4.2]]])
    np.testing.assert_array_equal(so.compact(conf, 4.2), [0, 3, 4, 5])
    assert len(so.compact(np.zeros((2, 3, 3)), 4.2)) == 0
