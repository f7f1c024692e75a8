"""Golden record of the UNMODIFIED reference OnlineSLAM (vista_slam/slam.py) on a seeded replay -> tests/golden/slam_graph.npz.

Runs only where the reference tree is present.  The reference code is imported unchanged; only its inputs are substituted:
  * in-memory stand-ins in sys.modules for pypose (oracle/pypose_stub.py: float64 arithmetic of
    oracle/pose_graph_oracle.py), munch, colorama, open3d (captures the point cloud it is asked to write) and
    vista_slam.loop_detector (replays the stream's loop candidates); xformers as in tools/ref_import.py;
  * the device is the CPU;
  * the STA frontend is replaced by the seeded per-edge stream of oracle/slam_oracle.py::make_stream (a planted trajectory
    with loops, pose confidences on both sides of rel_pose_thres, smooth positive depths, confidences away from
    conf_thres and from best-node ties, 32 x 40 maps), and pgo_every = 6 so that PGO runs several times.

Recorded: the graph after every keyframe, every PGO's inputs and result, and every file save_data_all writes."""
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from oracle import pypose_stub  # noqa: E402
from oracle import slam_oracle as so  # noqa: E402

CFG = dict(max_view_num=400, neighbor_edge_num=3, loop_edge_num=3, loop_dist_min=5, loop_nms=40, loop_cand_thresh_neighbor=5,
           conf_thres=4.2, rel_pose_thres=0.75, flow_thres=5.0, pgo_every=6)
PLY = {}


def _install_stubs(stream):
    pypose_stub.install()

    class Munch(dict):
        __getattr__ = dict.__getitem__

    sys.modules["munch"] = types.SimpleNamespace(Munch=Munch)

    class _Empty:
        def __getattr__(self, k):
            return ""

    sys.modules["colorama"] = types.SimpleNamespace(Fore=types.SimpleNamespace(
        CYAN="c", BLUE="b", YELLOW="y", GREEN="g", RED="r", MAGENTA="m"), Style=types.SimpleNamespace(RESET_ALL=""))

    class PointCloud:
        pass

    def write_point_cloud(path, pcd):
        PLY["path"] = os.path.basename(path)
        PLY["points"] = np.asarray(pcd.points)
        PLY["colors"] = np.asarray(pcd.colors)
        return True

    sys.modules["open3d"] = types.SimpleNamespace(geometry=types.SimpleNamespace(PointCloud=PointCloud),
                                                  utility=types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a)),
                                                  io=types.SimpleNamespace(write_point_cloud=write_point_cloud))

    class LoopDetector:
        def __init__(self, vocab_path, loop_dist_min, loop_nms, loop_cand_thresh_neighbor):
            self.loop_dist_min, self.loop_nms, self.loop_cand_thresh_neighbor = loop_dist_min, loop_nms, loop_cand_thresh_neighbor
            self.calls = 0

        def detect_loop(self, image, farthest_neighbor):
            c = stream["loops"][self.calls]
            self.calls += 1
            return list(c)

    sys.modules["vista_slam.loop_detector"] = types.SimpleNamespace(LoopDetector=LoopDetector)


def main(out_path=os.path.join(ROOT, "tests", "golden", "slam_graph.npz")):
    stream = so.make_stream()
    _install_stubs(stream)
    from tools.ref_import import REFERENCE_ROOT, _install_xformers_shim
    _install_xformers_shim()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import pypose as pp
    from vista_slam.slam import OnlineSLAM

    class _Frontend(torch.nn.Module):
        def _encode_image(self, image, image_shape, normalize=False):
            return torch.zeros(1), torch.zeros(1)

    class ReplaySLAM(OnlineSLAM):
        device = property(lambda self: torch.device("cpu"), lambda self, v: None)

        def load_frontend(self, ckpt_path):
            return _Frontend()

        def regress_two_views(self, i, j):
            e = stream["edges"][(i, j)]
            se3 = pp.mat2SE3(torch.from_numpy(e["pose"])[None], atol=1e-3).data
            conf = torch.tensor([float(e["conf"])], dtype=torch.float32)
            if conf < self.rel_pose_thres and i - j != 1:
                return se3, conf, None, None, None
            return se3, conf, torch.from_numpy(e["confs"]), torch.from_numpy(e["intri"]), torch.from_numpy(e["depths"])

    slam = ReplaySLAM("unused.pth", "unused.txt", verbose=True, **CFG)
    images = so.stream_images(stream)
    n = stream["n_views"]
    rec = {"kf_num_nodes": [], "kf_num_edges": [], "kf_pose": [], "kf_best_node": [], "kf_best_mean": []}
    for i in range(n):
        value = {"rgb": torch.from_numpy(images[i])[None], "shape": torch.tensor([[stream["H"], stream["W"]]]), "gray": None,
                 "view_name": "%04d.png" % i}
        slam.step(value, force_pgo=(i == n - 1))
        nodes, edges = slam.pose_graph_nodes, slam.pose_graph_edges
        rec["kf_num_nodes"].append(nodes.num_nodes)
        rec["kf_num_edges"].append(edges.num_edges)
        rec["kf_pose"].append(nodes.poses.tensor()[:nodes.num_nodes].numpy().copy())
        rec["kf_best_node"].append([nodes.view_to_best_node[v][0] for v in range(n)])
        rec["kf_best_mean"].append([nodes.view_to_best_node[v][1] for v in range(n)])
    nodes, edges = slam.pose_graph_nodes, slam.pose_graph_edges
    N, E = nodes.num_nodes, edges.num_edges
    out = {"kf_num_nodes": np.array(rec["kf_num_nodes"], np.int64), "kf_num_edges": np.array(rec["kf_num_edges"], np.int64),
           "kf_pose": np.stack([np.pad(p, ((0, N - len(p)), (0, 0))) for p in rec["kf_pose"]]).astype(np.float32),
           "kf_best_node": np.array(rec["kf_best_node"], np.int64),
           "kf_best_mean": np.array(rec["kf_best_mean"], np.float64),
           "node_to_view": np.array(nodes.node_to_view[:N], np.int64),
           "node_to_connected_view": np.array(nodes.node_to_connected_view[:N], np.int64),
           "edges": edges.edges[:E].numpy(), "meas": edges.poses.tensor()[:E].numpy(), "weight": edges.confs[:E].numpy()}
    calls = pypose_stub.LM_CALLS
    out["pgo_num_edges"] = np.array([c["num_edges"] for c in calls], np.int64)
    out["pgo_num_nodes"] = np.array([len(c["nodes"]) for c in calls], np.int64)
    for k in ("opt_idx", "related", "nodes", "result", "weight"):
        out["pgo_" + k] = np.concatenate([c[k] for c in calls])
    with tempfile.TemporaryDirectory() as d:
        slam.save_data_all(d)
        for f in ("trajectory", "scales", "images", "depths", "intrinsics"):
            out["out_" + f] = np.load(os.path.join(d, f + ".npy"))
        c = np.load(os.path.join(d, "confs.npz"))
        out["out_confs"], out["out_confs_thres"] = c["confs"], c["thres"]
        vg = np.load(os.path.join(d, "view_graph.npz"), allow_pickle=True)
        graph = vg["view_graph"].item()
        out["out_view_graph_len"] = np.array([len(graph[v]) for v in range(n)], np.int64)
        out["out_view_graph"] = np.array([u for v in range(n) for u in graph[v]], np.int64)
        out["out_loop_min_dist"] = vg["loop_min_dist"]
        out["out_view_names"] = vg["view_names"]
        out["out_files"] = np.array(sorted(os.listdir(d) + [PLY["path"]]))
    out["ply_points"], out["ply_colors"] = PLY["points"], PLY["colors"]
    np.savez_compressed(out_path, **out)
    print("wrote", out_path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main(*sys.argv[1:])
