"""ORACLE -- test infrastructure, not product code (only tests/ and tools/ may import it).

numpy restatement of OnlineSLAM's graph bookkeeping and map export (vista_slam/slam.py:108-140,191-412 over
vista_slam/pose_graph.py:5-54), and the seeded per-edge stream that stands in for the STA frontend in
tools/make_golden_slam.py and the GPU tests.

Arithmetic follows the reference's storage: node poses, edge measurements, weights and maps are float32 values; Sim(3)
products are evaluated in float64 on those values (oracle/pose_graph_oracle.py) and stored as float32, as the PyPose
stand-in (oracle/pypose_stub.py) does when the unmodified reference runs.  The depth-scale reductions and the
confidence means run in float64 and are stored as float32 (the reference sums in float32 with torch)."""
import numpy as np

from oracle import pose_graph_oracle as pg

ID_POSE_CONF = 2.0  # PoseGraphEdges.id_pose_conf


# ---------------------------------------------------------------------------------------------- seeded stream
def _rotvec_to_rot(v):
    th = np.linalg.norm(v)
    if th < 1e-12:
        return np.eye(3)
    k = pg.hat(v / th)
    return np.eye(3) + np.sin(th) * k + (1 - np.cos(th)) * k @ k


def make_stream(seed=7, n_views=20, H=32, W=40, neighbor_edge_num=3, loop_every=4, loop_min_gap=8, rel_pose_thres=0.75,
                conf_thres=4.2):
    """A planted trajectory that comes back near its start (loops), and per candidate edge (i, j) what
    regress_two_views returns: relative pose [4,4] (orthonormal fp32 rotation), pose confidence on both sides of
    rel_pose_thres, and for every edge the maps [2,H,W] (row 0 view i, row 1 view j) of positive smooth depths and
    confidences (about half of them above conf_thres) at least 0.05 from conf_thres, with per-map offsets that keep confidence means apart, plus the shared
    intrinsics [3,3].  Loop candidates: every loop_every-th view from 2 loop_every on gets up to two earlier views at least
    loop_min_gap back.  Returns a dict; edges are keyed (i, j)."""
    rng = np.random.default_rng(seed)
    cams = []
    for v in range(n_views):
        a = 2 * np.pi * v / (0.75 * n_views)
        R = _rotvec_to_rot(np.array([0.05 * np.sin(a), a * 0.3, 0.02 * np.cos(a)]))
        t = np.array([np.cos(a) - 1.0, 0.1 * np.sin(2 * a), np.sin(a)])
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, t
        cams.append(T)
    loops = []
    for i in range(n_views):
        c = []
        if i >= 2 * loop_every and i % loop_every == 0:
            far = [j for j in range(0, i - loop_min_gap)]
            pick = rng.choice(far, size=min(2, len(far)), replace=False) if far else []
            c = [(int(j), float(0.2 + 0.5 * rng.random())) for j in pick]
            c.sort(key=lambda x: -x[1])
        loops.append(c)
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    edges = {}
    for i in range(1, n_views):
        js = list(range(max(0, i - neighbor_edge_num), i)) + [j for j, _ in loops[i]]
        for j in js:
            r = np.random.default_rng([seed, i, j])
            T = np.linalg.inv(cams[j]) @ cams[i]  # pose_i = pose_j o T_ij
            T[:3, :3] = T[:3, :3] @ _rotvec_to_rot(0.01 * r.standard_normal(3))
            T[:3, 3] += 0.01 * r.standard_normal(3)
            pose = T.astype(np.float32)
            while True:
                conf = 0.3 + 0.9 * r.random()
                if abs(conf - rel_pose_thres) > 0.02:
                    break
            depths, confs = [], []
            for row in range(2):
                d = 1.5 + 0.5 * np.sin(xx / W * 3.0 + r.random() * 6) * np.cos(yy / H * 2.0 + r.random() * 6) + r.random()
                c = 1.0 + 6.0 * (0.5 + 0.5 * np.sin(xx / (3.0 + 4 * r.random()) + yy / (2.0 + 3 * r.random())))
                c = c + 0.37 * r.random()
                # on a 2^-8 / 2^-6 grid, so that the golden record of the maps compresses
                d, c = np.rint(d * 256) / 256, np.rint(c * 64) / 64
                c = np.where(np.abs(c - conf_thres) < 0.05, conf_thres + 0.1, c)
                depths.append(d)
                confs.append(c)
            fx = W * (0.9 + 0.2 * r.random())
            fy = H * (0.9 + 0.2 * r.random())
            K = np.array([[fx, 0, W / 2.0], [0, fy, H / 2.0], [0, 0, 1]])
            edges[(i, j)] = {"pose": pose, "conf": np.float32(conf), "depths": np.stack(depths).astype(np.float32),
                             "confs": np.stack(confs).astype(np.float32), "intri": K.astype(np.float32)}
    return {"n_views": n_views, "H": H, "W": W, "loops": loops, "edges": edges, "seed": seed}


def keep_edge(conf, i, j, rel_pose_thres):
    """slam.py:169,195."""
    return not (float(conf) < rel_pose_thres and i - j != 1)


def conf_mean(c):
    return np.float32(np.mean(c, dtype=np.float64))


def depth_scale(Di, Dj, ci, cj):
    """estimate_scale_with_depth_and_confidence (slam_utils.py:168-190) and (ci cj).sqrt().mean() (slam.py:227)."""
    Di, Dj, ci, cj = (np.asarray(x, np.float64).reshape(-1) for x in (Di, Dj, ci, cj))
    w = np.maximum(ci * cj, 1e-6)
    return np.float32((w * Di * Dj).sum() / (w * Di * Di).sum()), np.float32(np.sqrt(ci * cj).mean())


def _mul32(a, b):
    return pg.sim3_mul(np.asarray(a, np.float64), np.asarray(b, np.float64)).astype(np.float32)


# ---------------------------------------------------------------------------------------------- graph
class Graph:
    """PoseGraphNodes + PoseGraphEdges + the bookkeeping of connect_view_i_j, in numpy."""

    def __init__(self, max_nodes, max_edges):
        self.pose = np.zeros((max_nodes, 8), np.float32)
        self.pose[:, 6:] = 1.0
        self.node_to_view = -np.ones(max_nodes, np.int64)
        self.node_to_connected_view = -np.ones(max_nodes, np.int64)
        self.view_to_node = {}
        self.best_node = -np.ones(max_nodes, np.int64)
        self.best_mean = np.full(max_nodes, -100.0, np.float32)
        self.maps = []  # (depth, conf, intri) per node
        self.cmean = []
        self.edges = -np.ones((max_edges, 2), np.int64)
        self.meas = np.zeros((max_edges, 8), np.float32)
        self.meas[:, 6:] = 1.0
        self.weight = np.ones((max_edges, 7), np.float32)
        self.num_nodes = self.num_edges = 0

    def add_node(self, v, depth, conf, intri, other, cmean=None):
        n = self.num_nodes
        if n >= len(self.pose):
            raise IndexError("node capacity")
        self.maps.append((depth, conf, intri))
        self.node_to_view[n], self.node_to_connected_view[n] = v, other
        self.view_to_node.setdefault(v, []).append(n)
        m = conf_mean(conf) if cmean is None else np.float32(cmean)
        self.cmean.append(m)
        if m > self.best_mean[v]:
            self.best_mean[v], self.best_node[v] = m, n
        self.num_nodes += 1
        return n

    def add_edge(self, i, j, meas, w):
        e = self.num_edges
        if e >= len(self.edges):
            raise IndexError("edge capacity")
        self.edges[e] = (i, j)
        self.meas[e] = meas
        self.weight[e] = w
        self.num_edges += 1

    def connect(self, i, j, pose44, conf, confs, intri, depths, cmeans=None):
        """connect_view_i_j (slam.py:205-239) for a kept edge."""
        se3 = np.concatenate([pose44[:3, 3], pg.rot_to_quat(np.asarray(pose44[:3, :3], np.float64)), [1.0]]).astype(np.float32)
        nodes = {}
        i_new = True
        for r, (v, other) in enumerate(((i, j), (j, i))):
            n = self.add_node(v, depths[r], confs[r], intri, other, None if cmeans is None else cmeans[r])
            nodes[v] = n
            if len(self.view_to_node[v]) > 1:
                if v == i:
                    i_new = False
                f = self.view_to_node[v][0]
                s, sc = depth_scale(depths[r], self.maps[f][0], confs[r], self.maps[f][1])
                sim3 = np.array([0, 0, 0, 0, 0, 0, 1, s], np.float32)
                self.add_edge(n, f, sim3, [ID_POSE_CONF] * 6 + [sc])
                self.pose[n] = _mul32(self.pose[f], sim3)
        if i_new:
            self.pose[nodes[i]] = _mul32(self.pose[nodes[j]], se3)
        self.add_edge(nodes[i], nodes[j], se3, [np.float32(conf)] * 7)


def pgo_node_set(graph, view_num, pgo_window_size, loop_related_views):
    """slam.py:115-121: the nodes of the views in the window, plus the loop-related VIEW ids taken as node ids."""
    s = set()
    for v in range(max(0, view_num - pgo_window_size), view_num):
        s.update(graph.view_to_node.get(v, []))
    s.update(loop_related_views)
    return np.array(sorted(s), np.int64)


def pgo(graph, opt_idx):
    """slam.py:123-138 with PoseGraphOpt's per-edge weights; returns (related mask, weights used)."""
    E, N = graph.num_edges, graph.num_nodes
    edges = graph.edges[:E]
    related = pg.related_edges(edges, opt_idx)
    w = graph.weight[:E].astype(np.float64)
    out, _ = pg.optimize(graph.pose[:N].astype(np.float64), edges, graph.meas[:E].astype(np.float64), w, opt_idx)
    graph.pose[:N] = out.astype(np.float32)
    return related


def run(stream, rel_pose_thres=0.75, neighbor_edge_num=3, loop_edge_num=3, pgo_every=6, max_view_num=400, verbose=True,
        cmeans=None):
    """OnlineSLAM.step over the stream (force_pgo at the last view).  cmeans: optional {(i, j): [2] conf means} to use
    instead of recomputing them (a device run's own).  Returns (graph, per-keyframe records, PGO records)."""
    max_nodes = max_view_num * (neighbor_edge_num * 2 + loop_edge_num)
    max_edges = max_view_num * ((neighbor_edge_num * 2 + loop_edge_num - 1) + (neighbor_edge_num * 2 + loop_edge_num) // 2 + 1)
    g = Graph(max_nodes, max_edges)
    loop_related = set()
    kf, pgos = [], []
    n = stream["n_views"]
    for i in range(n):
        js = list(range(max(0, i - neighbor_edge_num), i)) + [j for j, _ in stream["loops"][i][:loop_edge_num]]
        for j in js:
            e = stream["edges"][(i, j)]
            if not keep_edge(e["conf"], i, j, rel_pose_thres):
                continue
            if i - j > neighbor_edge_num and verbose:
                loop_related.update((i, j))
            g.connect(i, j, e["pose"], e["conf"], e["confs"], e["intri"], e["depths"],
                      None if cmeans is None else cmeans[(i, j)])
        view_num = i + 1
        if view_num % pgo_every == 0 or i == n - 1:
            opt_idx = pgo_node_set(g, view_num, 2 * pgo_every, loop_related)
            nodes_in = g.pose[:g.num_nodes].copy()
            related = pgo(g, opt_idx)
            pgos.append({"opt_idx": opt_idx, "related": related, "num_edges": g.num_edges, "nodes": nodes_in,
                         "result": g.pose[:g.num_nodes].copy()})
            loop_related = set()
        kf.append({"num_nodes": g.num_nodes, "num_edges": g.num_edges, "pose": g.pose[:g.num_nodes].copy(),
                   "best_node": g.best_node[:view_num].copy()})
    return g, kf, pgos


# ---------------------------------------------------------------------------------------------- export
def export(graph, view_num, conf_thres, images):
    """save_data_all (slam.py:353-412): per view through its best node; images [N,3,H,W] in [-1, 1]."""
    poses, scales, depths, confs, intris = [], [], [], [], []
    for v in range(view_num):
        b = int(graph.best_node[v])
        X = graph.pose[b].astype(np.float64)
        P = np.eye(4)
        P[:3, :3] = pg.quat_to_rot(X[3:7])
        P[:3, 3] = X[:3]
        poses.append(P)
        scales.append([X[7]])
        d, c, K = graph.maps[b]
        depths.append(d)
        confs.append(c)
        intris.append(K)
    poses, scales = np.array(poses), np.array(scales)
    depths, confs, intris = np.array(depths), np.array(confs), np.array(intris)
    masks = confs > conf_thres
    N, H, W = depths.shape
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    pix = np.stack([xx, yy, np.ones_like(xx)], -1).reshape(-1, 3).astype(np.float64)
    pts = []
    for v in range(N):
        cam = pix @ np.linalg.inv(intris[v].astype(np.float64)).T * (depths[v].astype(np.float64) * scales[v, 0]).reshape(-1, 1)
        pts.append((cam @ poses[v][:3, :3].T + poses[v][:3, 3]).reshape(H, W, 3))
    pts = np.array(pts)
    imgs = (np.transpose(np.asarray(images, np.float64), (0, 2, 3, 1)) + 1.0) / 2.0
    return {"trajectory": poses, "scales": scales, "depths": depths, "confs": confs, "intrinsics": intris,
            "points": pts[masks], "colors": imgs[masks], "masks": masks}


def compact(conf, thres):
    """The (view, row, column) order of world_points[masks] (slam.py:407): flat indices of conf > thres."""
    return np.flatnonzero(np.asarray(conf).reshape(-1) > thres)


def stream_images(stream):
    """Seeded images [N,3,H,W] in [-1, 1] for the stream's views: smooth 8-bit patterns (32 levels) with a per-view,
    per-channel phase, normalised as the dataset does (u8 / 255 * 2 - 1), so that the images and the colours derived from
    them compress in the golden record."""
    r = np.random.default_rng([stream["seed"], 99])
    N, H, W = stream["n_views"], stream["H"], stream["W"]
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    ph = r.random((N, 3, 2)) * 6.0
    u8 = 8 * np.rint(15.9 + 15.9 * np.sin(xx / 5.0 + ph[..., 0, None, None]) * np.cos(yy / 7.0 + ph[..., 1, None, None]))
    return (u8.astype(np.float32) / 255.0 * 2.0 - 1.0).astype(np.float32)
