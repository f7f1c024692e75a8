"""GPU: the drop-in OnlineSLAM (vista_slam_b200/slam.py) with its device pose graph (csrc/slam_graph.cu).

The frontend is substituted by overriding load_frontend, the per-keyframe regression through `_regress_keyframe`, and
the loop detector by assigning `lc_detector`; everything else is the class as users run it.

Bounds (per element, absolute; poses, measurements and points are O(1) to O(10)):
  * node poses, edge measurements, PGO results: 1e-4.  A node pose is a chain of at most 2 V = 40 float32 Sim(3)
    products (each within about 8 float32 ulps, 5e-7 relative, of the float64 product on the same inputs) on
    translations up to 3, and the scale edges take a depth-scale reduction summed in a different order (a few ulps):
    40 x 5e-7 x 3 = 6e-5.
  * scales and weights: 1e-5 (one reduction, relative error of a few ulps on values up to 3).
  * points: 1e-3 + 4e-4 |p| per point.  1e-3 is the translation bound plus the pose bound times a local point norm up to
    10; 4e-4 |p| = 4 POSE_TOL |p| covers the rotation: four quaternion components within POSE_TOL put |dq| within
    2 POSE_TOL, and a unit quaternion moved by dq rotates a vector by at most 2 |dq| |p|.  Random-init weights give
    degenerate intrinsics and points up to |p| ~ 1e5, where this term dominates.
Integers, masks, point counts and point order must be equal."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import slam_oracle as so

pytestmark = pytest.mark.gpu
VOCAB = os.path.join(GOLDEN_DIR, "loop_vocab.txt")
CFG = dict(max_view_num=400, neighbor_edge_num=3, loop_edge_num=3, loop_dist_min=5, conf_thres=4.2, rel_pose_thres=0.75,
           pgo_every=6)
POSE_TOL, SCALE_TOL, PT_TOL = 1e-4, 1e-5, 1e-3


class _Frontend(torch.nn.Module):
    def _encode_image(self, image, image_shape, normalize=False):
        return torch.zeros(1, 1, 1024, device="cuda"), None


class _Loops:
    def __init__(self, loops, loop_dist_min):
        self.loops, self.loop_dist_min, self.calls = loops, loop_dist_min, 0

    def detect_loop(self, image, farthest_neighbor):
        torch.cuda.synchronize()  # the real detector reads its candidates back here
        c = self.loops[self.calls]
        self.calls += 1
        return list(c)


def _batch(stream, i, js, rel_pose_thres):
    E = [stream["edges"][(i, j)] for j in js]
    keep = [k for k, (j, e) in enumerate(zip(js, E)) if so.keep_edge(e["conf"], i, j, rel_pose_thres)]
    dev = "cuda"
    conf = torch.from_numpy(np.stack([np.stack([E[k]["confs"][r] for k in keep]) for r in range(2)])).to(dev)
    return [float(e["conf"]) for e in E], keep, {
        "pose": torch.from_numpy(np.stack([e["pose"] for e in E])).to(dev),
        "pose_conf": torch.tensor([float(e["conf"]) for e in E], dtype=torch.float32, device=dev),
        "conf": conf,
        "depths": torch.from_numpy(np.stack([np.stack([E[k]["depths"][r] for k in keep]) for r in range(2)])).to(dev),
        "intri": torch.from_numpy(np.stack([E[k]["intri"] for k in keep])).to(dev),
        "conf_mean": conf.mean(dim=(2, 3)).contiguous()}


def _replay_slam(stream, cfg=CFG, **over):
    from vista_slam_b200.slam import OnlineSLAM

    class ReplaySLAM(OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return _Frontend()

        def _regress_keyframe(self, i, js):
            return _batch(stream, i, js, self.rel_pose_thres)

    c = dict(cfg)
    c.update(over)
    slam = ReplaySLAM("unused", VOCAB, verbose=True, **c)
    slam.lc_detector = _Loops(stream["loops"], c["loop_dist_min"])
    return slam


def _assert_points(got, want):
    bound = PT_TOL + 4 * POSE_TOL * np.linalg.norm(want, axis=1, keepdims=True)
    err = np.abs(got - want)
    assert (err <= bound).all(), float((err / bound).max())


def _value(images, i, stream):
    return {"rgb": torch.from_numpy(images[i])[None].cuda(), "shape": torch.tensor([[stream["H"], stream["W"]]]), "gray": None,
            "view_name": "%04d.png" % i}


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN_DIR, "slam_graph.npz")))


def test_golden_replay(golden, tmp_path, monkeypatch):
    import vista_slam_b200.slam as S
    g = golden
    stream = so.make_stream()
    pgo_calls = []

    class RecordingPGO(S.PoseGraphOpt):
        def optimize(self, edges, poses, weight, **kw):
            rec = {"opt_idx": self.idxs_opt.cpu().numpy(), "related": self.get_related_edge_idxs(edges).cpu().numpy(),
                   "nodes": self.nodes.cpu().numpy()}
            out = super().optimize(edges, poses, weight, **kw)
            rec["result"] = self.nodes.cpu().numpy()
            pgo_calls.append(rec)
            return out

    monkeypatch.setattr(S, "PoseGraphOpt", RecordingPGO)
    slam = _replay_slam(stream)
    n = stream["n_views"]
    for i in range(n):
        slam.step(_value(so.stream_images(stream), i, stream), force_pgo=(i == n - 1))
        assert slam.num_nodes == g["kf_num_nodes"][i] and slam.num_edges == g["kf_num_edges"][i]
        N = slam.num_nodes
        np.testing.assert_allclose(slam._graph.pose[:N].cpu().numpy(), g["kf_pose"][i, :N], atol=POSE_TOL, rtol=0)
        np.testing.assert_array_equal(slam._graph.best_node[:i + 1].cpu().numpy(), g["kf_best_node"][i, :i + 1])
    G = slam._graph
    N, E = slam.num_nodes, slam.num_edges
    np.testing.assert_array_equal(G.node_to_view[:N].cpu().numpy(), g["node_to_view"])
    np.testing.assert_array_equal(G.node_to_connected_view[:N].cpu().numpy(), g["node_to_connected_view"])
    np.testing.assert_array_equal(G.edges[:E].cpu().numpy(), g["edges"])
    np.testing.assert_allclose(G.meas[:E].cpu().numpy(), g["meas"], atol=POSE_TOL, rtol=0)
    np.testing.assert_allclose(G.weight[:E].cpu().numpy(), g["weight"], atol=SCALE_TOL, rtol=0)
    assert (G.node_to_view[N:] == -1).all() and (G.edges[E:] == -1).all()
    # PGO: node sets and related masks exactly, inputs and results within the pose bound
    assert len(pgo_calls) == len(g["pgo_num_edges"])
    o = r = m = 0
    for c, ne, nn in zip(pgo_calls, g["pgo_num_edges"], g["pgo_num_nodes"]):
        no = len(c["opt_idx"])
        np.testing.assert_array_equal(c["opt_idx"], g["pgo_opt_idx"][o:o + no])
        np.testing.assert_array_equal(c["related"], g["pgo_related"][r:r + ne])
        np.testing.assert_allclose(c["nodes"], g["pgo_nodes"][m:m + nn], atol=POSE_TOL, rtol=0)
        np.testing.assert_allclose(c["result"], g["pgo_result"][m:m + nn], atol=POSE_TOL, rtol=0)
        o, r, m = o + no, r + ne, m + nn
    # save_data_all: same files, keys, shapes, dtypes; values within bounds; point count and order exact
    slam.save_data_all(str(tmp_path))
    assert sorted(os.listdir(tmp_path)) == list(g["out_files"])
    for f, tol in (("trajectory", POSE_TOL), ("scales", SCALE_TOL), ("images", 0), ("depths", 0), ("intrinsics", 0)):
        a = np.load(tmp_path / (f + ".npy"))
        assert a.dtype == g["out_" + f].dtype and a.shape == g["out_" + f].shape, f
        np.testing.assert_allclose(a, g["out_" + f], atol=tol, rtol=0)
    c = np.load(tmp_path / "confs.npz")
    assert sorted(c.files) == ["confs", "thres"] and float(c["thres"]) == float(g["out_confs_thres"])
    np.testing.assert_array_equal(c["confs"], g["out_confs"])
    vg = np.load(tmp_path / "view_graph.npz", allow_pickle=True)
    assert sorted(vg.files) == ["loop_min_dist", "view_graph", "view_names"]
    graph = vg["view_graph"].item()
    assert isinstance(graph, dict) and sorted(graph) == list(range(n))
    np.testing.assert_array_equal([u for v in range(n) for u in graph[v]], g["out_view_graph"])
    assert int(vg["loop_min_dist"]) == int(g["out_loop_min_dist"])
    np.testing.assert_array_equal(vg["view_names"], g["out_view_names"])
    pts, cols = S.read_ply(tmp_path / "pointcloud.ply")
    assert len(pts) == len(g["ply_points"])
    _assert_points(pts, g["ply_points"])
    np.testing.assert_array_equal(cols, np.rint(np.clip(g["ply_colors"], 0, 1) * 255).astype(np.uint8))
    # get_view: attribute and key access, filtered depth
    v = slam.get_view(3)
    assert v.pose.shape == (4, 4) and v["intri"].shape == (3, 3)
    best = int(g["kf_best_node"][-1, 3])
    s = float(g["out_scales"][3, 0])
    want = g["out_depths"][3] * s
    want[g["out_confs"][3] < 4.2] = 0
    np.testing.assert_allclose(v.depth.numpy(), want, atol=POSE_TOL, rtol=0)
    assert best == int(slam._graph.best_node[3])
    assert slam.imgs[2].device.type == "cpu"
    img, pcl = slam.get_pointmap_vis(2)
    assert img.dtype == np.uint8 and pcl.shape == (stream["H"], stream["W"], 3)


def test_loop_related_views_only_when_verbose_and_reset_keeps_the_loop_detector(golden):
    stream = so.make_stream()
    quiet = _replay_slam(stream)
    quiet.verbose = False
    for i in range(13):  # view 12 adds two loop closure edges
        quiet.step(_value(so.stream_images(stream), i, stream))
    assert quiet.loop_related_views == set()
    loud = _replay_slam(stream)
    for i in range(13):
        loud.step(_value(so.stream_images(stream), i, stream))
    assert loud.loop_related_views == {12, 2, 3}
    det = loud.lc_detector
    loud.reset()
    assert loud.lc_detector is det and det.calls == 13 and loud.view_num == 0 and loud.num_nodes == 0
    assert int(loud._graph.best_node[0]) == -1 and (loud._graph.edges[:8] == -1).all()


def test_graph_update_and_export_do_not_synchronise(golden):
    stream = so.make_stream()
    slam = _replay_slam(stream)
    for i in range(4):
        slam.step(_value(so.stream_images(stream), i, stream))
    batches = [_batch(stream, i, list(range(max(0, i - 3), i)) + [j for j, _ in stream["loops"][i][:3]], 0.75)
               for i in (4, 5)]
    torch.cuda.synchronize()
    slam.view_num = 6
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i, (_, keep, batch) in zip((4, 5), batches):
            slam._add_keyframe(i, list(range(max(0, i - 3), i)), keep, batch)
        slam.imgs.extend([slam.imgs.device_stack()[0]] * 2)
        out = slam._export(0, 6, cloud=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert int(out["count"]) > 0


def test_refusals(golden):
    from vista_slam_b200 import _lib
    stream = so.make_stream()
    # capacity: max_view_num = 1 -> 9 nodes; the reference raises IndexError there
    small = _replay_slam(stream, max_view_num=1)
    with pytest.raises(IndexError):
        for i in range(6):
            small.step(_value(so.stream_images(stream), i, stream))
    slam = _replay_slam(stream)
    for i in range(3):
        slam.step(_value(so.stream_images(stream), i, stream))
    _, keep, batch = _batch(stream, 3, [0, 1, 2], 0.75)
    nodes, edges = slam.num_nodes, slam.num_edges
    # the C entry point refuses before any launch too
    n = len(keep)
    import ctypes
    args = ((ctypes.c_int64 * n)(*[[0, 1, 2][k] for k in keep]), (ctypes.c_int * n)(*keep), (ctypes.c_int * n)(*([-1] * n)))
    rc = _lib.lib().sta_graph_add_keyframe(slam._graph.h, 3, n, *args, slam._graph.max_nodes - 1, 0, stream["H"], stream["W"],
                                            *[_lib.ptr(batch[k]) for k in ("pose", "pose_conf", "conf", "depths", "intri",
                                                                          "conf_mean")], _lib.cur_stream())
    assert rc != 0 and b"capacity" in _lib.lib().sta_last_error()
    # map size other than the graph's
    bad = dict(batch, conf=batch["conf"][..., :-1].contiguous(), depths=batch["depths"][..., :-1].contiguous())
    with pytest.raises(RuntimeError, match="map size"):
        slam._add_keyframe(3, [0, 1, 2], keep, bad)
    # host memory as input
    with pytest.raises(RuntimeError, match="device memory"):
        slam._add_keyframe(3, [0, 1, 2], keep, {k: v.cpu() for k, v in batch.items()})
    assert (slam.num_nodes, slam.num_edges) == (nodes, edges)
    torch.cuda.synchronize()
    assert int(slam._graph.node_to_view[nodes]) == -1
    # a planted non-orthonormal rotation raises ValueError at the next read-back
    s2 = so.make_stream()
    s2["edges"][(3, 2)]["pose"] = s2["edges"][(3, 2)]["pose"].copy()
    s2["edges"][(3, 2)]["pose"][:3, :3] *= np.float32(1.01)
    bad_slam = _replay_slam(s2)
    for i in range(4):
        bad_slam.step(_value(so.stream_images(s2), i, s2))
    with pytest.raises(ValueError, match="orthonormal"):
        bad_slam.step(_value(so.stream_images(s2), 4, s2))


@pytest.mark.parametrize("case", ["random", "ties", "empty"])
def test_export_compaction_against_oracle(case, tmp_path):
    stream = so.make_stream(seed=11, n_views=8, H=24, W=72)
    r = np.random.default_rng(5)
    for e in stream["edges"].values():
        if case == "empty":
            e["confs"] = (r.random(e["confs"].shape) * 4.0).astype(np.float32)  # all below 4.2
        else:
            e["confs"] = (1.0 + 8.0 * r.random(e["confs"].shape)).astype(np.float32)
            if case == "ties":
                e["confs"][r.random(e["confs"].shape) < 0.3] = np.float32(4.2)  # conf == conf_thres is excluded
    slam = _replay_slam(stream, pgo_every=1000)
    images = so.stream_images(stream)
    n_views = stream["n_views"]
    for i in range(n_views):
        slam.step(_value(images, i, stream), force_pgo=(i == n_views - 1))  # so.run ends with a PGO too
    out = slam._export(0, stream["n_views"], cloud=True)
    cm = {}
    for i in range(1, stream["n_views"]):
        for j in list(range(max(0, i - 3), i)) + [j for j, _ in stream["loops"][i][:3]]:
            cm[(i, j)] = stream["edges"][(i, j)]["confs"].astype(np.float64).mean(axis=(1, 2))
    graph, _, _ = so.run(stream, pgo_every=1000, cmeans={k: torch.tensor(v).float().numpy() for k, v in cm.items()})
    np.testing.assert_array_equal(slam._graph.best_node[:stream["n_views"]].cpu().numpy(), graph.best_node[:stream["n_views"]])
    ex = so.export(graph, stream["n_views"], 4.2, images)
    n = int(out["count"])
    assert n == len(ex["points"]) and (n == 0) == (case == "empty")
    _assert_points(out["points"][:n].cpu().numpy(), ex["points"])
    np.testing.assert_allclose(out["colors"][:n].cpu().numpy(), ex["colors"], atol=1e-6, rtol=0)
    slam.save_data_all(str(tmp_path))
    pts, _ = __import__("vista_slam_b200.slam", fromlist=["read_ply"]).read_ply(tmp_path / "pointcloud.ply")
    assert len(pts) == n


def test_end_to_end_against_oracle(cuda_model, tmp_path):
    """About 12 keyframes at 224 x 224 through the real frontend (synthetic checkpoint), the real loop detector (golden
    DBoW3 vocabulary) and the device graph, then the oracle replayed on that run's own frontend outputs."""
    import vista_slam_b200.slam as S
    recorded = {}

    class Run(S.OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return cuda_model

        def _regress_keyframe(self, i, js):
            conf_host, keep, b = super()._regress_keyframe(i, js)
            recorded[i] = (list(js), conf_host, keep, {k: v.cpu().numpy().copy() for k, v in b.items()})
            return conf_host, keep, b

    slam = Run("unused", VOCAB, verbose=True, loop_dist_min=4, pgo_every=5, rel_pose_thres=0.5)
    g = torch.Generator().manual_seed(3)
    H = W = 224
    base = torch.rand(1, 3, H // 8, W // 8, generator=g)
    n = 12
    for i in range(n):
        img = torch.nn.functional.interpolate(base.roll(i, dims=3), size=(H, W), mode="bilinear") * 2 - 1
        img = (img + 0.05 * torch.rand(1, 3, H, W, generator=g)).clamp(-1, 1).cuda()
        gray = ((img[0].mean(0) + 1) / 2).contiguous()
        slam.step({"rgb": img, "shape": torch.tensor([[H, W]]), "gray": gray, "view_name": "%d" % i}, force_pgo=(i == n - 1))
    # the oracle on the recorded outputs
    stream = {"n_views": n, "H": H, "W": W, "loops": [], "edges": {}, "seed": 0}
    cmeans = {}
    for i in range(n):
        js, conf_host, keep, b = recorded.get(i, ([], [], [], {}))
        nb = max(0, i - 3)
        stream["loops"].append([(j, 0.0) for j in js[i - nb:]])
        for k, j in enumerate(js):
            e = {"pose": b["pose"][k], "conf": np.float32(conf_host[k])}
            if k in keep:
                p = keep.index(k)
                e.update(confs=b["conf"][:, p], depths=b["depths"][:, p], intri=b["intri"][p])
                cmeans[(i, j)] = b["conf_mean"][:, p]
            stream["edges"][(i, j)] = e
    graph, kf, _ = so.run(stream, rel_pose_thres=0.5, pgo_every=5, cmeans=cmeans)
    N, E = slam.num_nodes, slam.num_edges
    assert (N, E) == (graph.num_nodes, graph.num_edges) and N > 0
    G = slam._graph
    np.testing.assert_array_equal(G.node_to_view[:N].cpu().numpy(), graph.node_to_view[:N])
    np.testing.assert_array_equal(G.edges[:E].cpu().numpy(), graph.edges[:E])
    np.testing.assert_array_equal(G.best_node[:n].cpu().numpy(), graph.best_node[:n])
    np.testing.assert_allclose(G.weight[:E].cpu().numpy(), graph.weight[:E], atol=SCALE_TOL, rtol=1e-5)
    np.testing.assert_allclose(G.meas[:E].cpu().numpy(), graph.meas[:E], atol=POSE_TOL, rtol=1e-5)
    np.testing.assert_allclose(G.pose[:N].cpu().numpy(), graph.pose[:N], atol=POSE_TOL, rtol=1e-4)
    ex = so.export(graph, n, slam.conf_thres, slam.imgs.device_stack().cpu().numpy())
    out = slam._export(0, n, cloud=True)
    m = int(out["count"])
    assert m == len(ex["points"])
    _assert_points(out["points"][:m].cpu().numpy(), ex["points"])
    t = slam.get_time_dict()
    assert t["total"] > 0 and set(t) >= {"encoder", "decoder", "lc", "pgo", "graph_construction"}
