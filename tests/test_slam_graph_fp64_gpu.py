"""GPU: the device pose graph and its map export (csrc/slam_graph.cu, cloud.cuh, pointmap.cuh) against float64 per
element, driven through the C ABI (slam._Graph and _lib) one kernel step at a time.

Every float64 reference is computed from the device's own stored inputs, read back from its tables, so that a bound
covers one step and cannot hide an error inside the drift of a chain (the bounds and the mirror:
tests/test_slam_graph_fp64_cpu.py):
  (a) edge measurements: the rotation cases of the CPU file as pose rows; STA_GRAPH_FLAG_NOT_SO3 exactly for the
      flagged ones, kept until sta_graph_reset;
  (b) node poses: every node against the fp64 product of its stored parent and stored measurement, on planted parents
      (translations of 1e3, scales of 1e-2 and 1e2, q_w < 0) and chains that take sim3_mul's sign flip;
  (c) scale edges against fp64 sums over the stored maps at 224 x 224, 384 x 512 and 37 x 1001, with the clamp and
      cancelling sums planted;
  (d) a keyframe of 32 kept edges, all with a first node of view j (63 scale edges), against the oracle's bookkeeping;
  (e) node and edge tables filled exactly, one more refused before any launch, a reset beyond 65,536 slots;
  (f) sta_graph_replay_nodes over more than 512 triples (three launches and more);
  (g) sta_graph_export at widths around 256 and 512, row counts around 1024, a view sub-range, and at production
      size (400 views of 224 x 224 in a graph of 3600 nodes);
  (h) eval_recon.world_clouds at W = 512 and 513 against the torch reference of tests/test_eval_gpu.py.
Each test prints the largest err / bound of its checks ("worst <check> <ratio>")."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import eval_oracle as eo
from oracle import pose_graph_oracle as pg
from oracle import slam_oracle as so
from test_eval_gpu import _assert_close_f32
from test_pgo_background_gpu import _Pending, _assert_identical, _full
from test_slam_batch_gpu import _replay_slam as _replay
from test_slam_gpu import _value
from test_slam_graph_fp64_cpu import (C_PT, C_ROT, F32, Q_ABS, ROT_CASES, SIM3_CASES, _ratio, inv3, random_pairs,
                                      rot_to_quat, scale_errs, scale_stats_ref, sim3_err, sim3_mul64, unproject_ref)

pytestmark = pytest.mark.gpu


def _lib():
    from vista_slam_b200 import _lib
    return _lib


def _report(name, r):
    print("worst %s %.4g" % (name, r))
    assert r <= 1.0, (name, r)


def _graph(max_nodes, max_edges, max_views, H, W):
    from vista_slam_b200.slam import _Graph
    return _Graph(max_nodes, max_edges, max_views, H, W, torch.device("cuda"))


def _plan(node0, edge0, first_j):
    """graph_link_kernel's order for one keyframe: scale edges [(edge, new node, other)], pose edges
    [(edge, ni, nj, k)], derived nodes [(node, parent, edge)] in derivation order, and the next free edge."""
    e, scale, pose, derived = edge0, [], [], []
    for k, f in enumerate(first_j):
        ni = node0 + 2 * k
        if k > 0:
            scale.append((e, ni, node0))
            derived.append((ni, node0, e))
            e += 1
        if f >= 0:
            scale.append((e, ni + 1, f))
            derived.append((ni + 1, f, e))
            e += 1
        pose.append((e, ni, ni + 1, k))
        if k == 0:
            derived.append((ni, ni + 1, e))
        e += 1
    return scale, pose, derived, e


def _maps(n, H, W, gen, plant=True):
    """[2, n, H, W] depth and confidence maps (fp32, CUDA): depths in [0.5, 3.5], confidences in [1, 8]; planted: 40 %
    negative depths (sum w Di Dj cancels) and 5 % of pixels with ci cj < 1e-6 (the clamp)."""
    d = 0.5 + 3 * torch.rand(2, n, H, W, generator=gen, device="cuda")
    c = 1 + 7 * torch.rand(2, n, H, W, generator=gen, device="cuda")
    if plant:
        d = torch.where(torch.rand(d.shape, generator=gen, device="cuda") < 0.4, -d, d)
        tiny = torch.rand(c.shape, generator=gen, device="cuda") < 0.05
        c = torch.where(tiny, 1e-3 * torch.rand(c.shape, generator=gen, device="cuda"), c)
    return d.contiguous(), c.contiguous()


def _batch(poses, H, W, seed, keep=None, conf_mean=None, plant=True):
    """A keyframe's device batch: pose rows [K,4,4] (fp32), pose confidences, the maps of the kept rows, intrinsics and
    confidence means (planted or the maps' fp32 means)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    K = len(poses)
    keep = list(range(K)) if keep is None else keep
    n = len(keep)
    d, c = _maps(n, H, W, gen, plant)
    r = np.random.default_rng(seed)
    intri = np.zeros((n, 3, 3), np.float32)
    intri[:, 0, 0], intri[:, 1, 1] = W * r.uniform(0.8, 1.2, n), H * r.uniform(0.8, 1.2, n)
    intri[:, 0, 2], intri[:, 1, 2], intri[:, 2, 2] = W / 2, H / 2, 1
    cm = c.mean(dim=(2, 3)) if conf_mean is None else torch.as_tensor(np.asarray(conf_mean, np.float32)).cuda()
    return {"pose": torch.from_numpy(np.asarray(poses, np.float32)).cuda(),
            "pose_conf": torch.from_numpy(r.uniform(0.3, 1.2, K).astype(np.float32)).cuda(), "conf": c, "depths": d,
            "intri": torch.from_numpy(intri).cuda(), "conf_mean": cm.contiguous()}, keep


def _add(g, view, js, first_j, node0, edge0, batch, keep):
    n = len(js)
    L = _lib()
    b = batch
    return L.lib().sta_graph_add_keyframe(
        g.h, view, n, (ctypes.c_int64 * n)(*js), (ctypes.c_int * n)(*keep), (ctypes.c_int * n)(*first_j), node0, edge0, g.H,
        g.W, *[L.ptr(b[k]) for k in ("pose", "pose_conf", "conf", "depths", "intri", "conf_mean")], L.cur_stream())


class _Builder:
    """Keyframes into a device graph with OnlineSLAM's host bookkeeping (first node of view j), the oracle Graph's
    bookkeeping alongside when asked, and the plans of every keyframe."""

    def __init__(self, g, oracle=None):
        self.g, self.oracle = g, oracle
        self.v2n, self.nodes, self.edges = {}, 0, 0
        self.scale, self.pose, self.derived = [], [], []

    def add(self, view, js, batch, keep, first_j=None):
        if first_j is None:
            v2n = {v: list(self.v2n.get(v, [])) for v in set(js) | {view}}
            first_j = []
            for k, j in enumerate(js):
                v2n[view].append(self.nodes + 2 * k)
                first_j.append(v2n[j][0] if v2n[j] else -1)
                v2n[j].append(self.nodes + 2 * k + 1)
            self.v2n.update(v2n)
        _lib().check(_add(self.g, view, js, first_j, self.nodes, self.edges, batch, keep), "sta_graph_add_keyframe")
        sc, po, de, e = _plan(self.nodes, self.edges, first_j)
        self.scale += sc
        self.pose += [(e_, ni, nj, batch, keep[k]) for e_, ni, nj, k in po]
        self.derived += de
        if self.oracle is not None:
            host = {k: v.cpu().numpy() for k, v in batch.items()}
            for k, j in enumerate(js):
                c = keep[k]
                self.oracle.connect(view, j, host["pose"][c], host["pose_conf"][c], host["conf"][:, k], host["intri"][k],
                                    host["depths"][:, k], host["conf_mean"][:, k])
        self.nodes += 2 * len(js)
        self.edges = e
        return first_j


def _tables(g):
    return {k: getattr(g, k).cpu().numpy() for k in ("pose", "depth", "conf", "intri", "cmean", "node_to_view",
                                                      "node_to_connected_view", "best_node", "best_mean", "edges", "meas",
                                                      "weight")}


def _check_nodes(g, derived):
    """Worst err / bound of the derived nodes [(node, parent, edge)].  Their scales must stay in fp32's normal range,
    where a bound relative to the magnitude holds (a chain of small scale edges underflows: a property of the data)."""
    pose, meas = g.pose.cpu().numpy(), g.meas.cpu().numpy()
    nodes = [d[0] for d in derived]
    assert (pose[nodes, 6] >= 0).all()  # kept with q_w >= 0
    assert (np.abs(pose[nodes, 7]) >= 1e-30).all()
    return max(sim3_err(pose[n], pose[p], meas[e]) for n, p, e in derived)


def _check_pose_edges(g, pose_edges):
    meas, weight, edges = g.meas.cpu().numpy(), g.weight.cpu().numpy(), g.edges.cpu().numpy()
    worst = 0.0
    for e, ni, nj, batch, row in pose_edges:
        M = batch["pose"][row].cpu().numpy()
        q, _, _, _ = rot_to_quat(M)
        assert list(edges[e]) == [ni, nj]
        assert meas[e, :3].tobytes() == M[:3, 3].tobytes() and meas[e, 7] == 1.0
        assert (weight[e] == batch["pose_conf"][row].item()).all()
        worst = max(worst, _ratio(np.abs(meas[e, 3:7] - q), 2.0 ** -23 * np.abs(q) + Q_ABS))
    return worst


def _check_scale_edges(g, scale_edges):
    meas, weight, edges = g.meas.cpu().numpy(), g.weight.cpu().numpy(), g.edges.cpu().numpy()
    worst = [0.0, 0.0]
    for e, nn, no in scale_edges:
        assert list(edges[e]) == [nn, no]
        assert (meas[e, :7] == [0, 0, 0, 0, 0, 0, 1]).all() and (weight[e, :6] == 2.0).all()
        st = scale_stats_ref(g.depth[nn].double(), g.depth[no].double(), g.conf[nn].double(), g.conf[no].double(), xp=torch)
        es, ec = scale_errs(meas[e, 7], weight[e, 6], st)
        worst = [max(worst[0], es), max(worst[1], ec)]
    return worst


def _pose44(q, t):
    M = np.eye(4)
    M[:3, :3], M[:3, 3] = pg.quat_to_rot(np.asarray(q, np.float64)), t
    return M.astype(np.float32)


# ------------------------------------------------------------------------------- (a) edge measurements
def test_edge_quaternions_and_the_so3_flag():
    L = _lib()
    H = W = 4
    g = _graph(128, 128, 64, H, W)
    accepted = [c for c in ROT_CASES if c[2][2]]
    flagged = [c for c in ROT_CASES if not c[2][2]]
    assert 0 < len(accepted) <= 32 and flagged
    poses = [c[1] for c in accepted][::-1]  # candidate rows in reverse: edge k reads row K - 1 - k
    batch, _ = _batch(poses, H, W, 1)
    keep = list(range(len(poses)))[::-1]
    b = _Builder(g)
    b.add(1, [0] * len(keep), batch, keep, first_j=[-1] * len(keep))
    torch.cuda.synchronize()
    assert g.flags() == 0
    worst = _check_pose_edges(g, b.pose)
    for name, M, _ in flagged:
        L.check(L.lib().sta_graph_reset(g.h, L.cur_stream()), "sta_graph_reset")
        assert g.flags() == 0
        b = _Builder(g)
        bad, _ = _batch([M], H, W, 2)
        b.add(2, [1], bad, [0], first_j=[-1])
        torch.cuda.synchronize()
        assert g.flags() == L.GRAPH_FLAG_NOT_SO3, name
        good, _ = _batch([accepted[0][1]], H, W, 3)  # an accepted rotation afterwards leaves the flag set
        b.add(3, [2], good, [0], first_j=[-1])
        torch.cuda.synchronize()
        assert g.flags() == L.GRAPH_FLAG_NOT_SO3, name
        worst = max(worst, _check_pose_edges(g, b.pose))  # the quaternion is stored all the same
    L.check(L.lib().sta_graph_reset(g.h, L.cur_stream()), "sta_graph_reset")
    torch.cuda.synchronize()
    assert g.flags() == 0 and (g.edges == -1).all()
    _report("edge_quaternion", worst)


# ------------------------------------------------------------------------------- (b) node poses
def test_node_poses_against_their_stored_parents():
    H = W = 4
    a_rows = [c[1] for c in SIM3_CASES]
    b_rows = [c[2] for c in SIM3_CASES]
    R = len(a_rows) + 1
    roots = np.stack(a_rows + [a_rows[4].copy()])
    roots[-1, 3:7] = -roots[-1, 3:7]  # a parent stored with q_w < 0 (a PGO result may be): the scale edge's product flips
    g = _graph(400, 600, 200, H, W)
    g.pose[:R] = torch.from_numpy(roots).cuda()
    gen = torch.Generator(device="cuda").manual_seed(0)
    g.depth[:R], g.conf[:R] = 0.5 + 3 * torch.rand(R, H, W, generator=gen, device="cuda"), 1 + torch.rand(R, H, W, generator=gen, device="cuda")
    b = _Builder(g)
    b.nodes = R
    view = 1
    for c, (a_row, b_row) in enumerate(zip(roots, b_rows + [b_rows[4]])):  # pose[nj] = root c (rescaled), pose[ni] = it x b
        batch, keep = _batch([_pose44(b_row[3:7], b_row[:3])], H, W, 10 + c, plant=False)
        b.add(view, [0], batch, keep, first_j=[c])
        view += 1
    # chains: each keyframe's first edge hangs from the previous keyframe's view-i node; 3 edges, so that the k > 0 nodes
    # take the scale edge to node0; translations up to 1e3 and rotations past 90 degrees
    qa, qb = random_pairs(40, seed=5)
    prev = b.nodes - 2
    for c in range(40):
        rows = [_pose44(qb[c, 3:7], qb[c, :3]), _pose44(qa[c, 3:7], qa[c, :3]), _pose44(qb[(c + 1) % 40, 3:7], qa[c, :3])]
        batch, keep = _batch(rows, H, W, 100 + c, plant=False)
        node0 = b.nodes
        b.add(view, [0, 0, 0], batch, keep, first_j=[prev, -1, prev + 1])
        prev = node0
        view += 1
    torch.cuda.synchronize()
    pose, meas = g.pose.cpu().numpy(), g.meas.cpu().numpy()
    flips = [sim3_mul64(pose[p], meas[e])[2] for _, p, e in b.derived]
    scale_edge = {e for e, _, _ in b.scale}
    assert any(f and e in scale_edge for f, (_, _, e) in zip(flips, b.derived))
    assert sum(f and e not in scale_edge for f, (_, _, e) in zip(flips, b.derived)) >= 3
    assert np.abs(pose[:b.nodes, :3]).max() >= 1e3 and pose[:b.nodes, 7].min() <= 0.011 and pose[:b.nodes, 7].max() >= 99
    _report("node_pose", _check_nodes(g, b.derived))
    _report("edge_quaternion", _check_pose_edges(g, b.pose))


# ------------------------------------------------------------------------------- (c) scale edges
@pytest.mark.parametrize("H,W", [(224, 224), (384, 512), (37, 1001)])
def test_scale_edges_against_fp64_sums(H, W):
    g = _graph(16, 16, 8, H, W)
    b = _Builder(g)
    rows = [_pose44(q[3:7], q[:3]) for q in random_pairs(3, seed=H)[0]]
    for view, js in ((1, [0]), (2, [1, 0]), (3, [2, 0, 1])):
        batch, keep = _batch(rows[:len(js)], H, W, view * 7 + W)
        b.add(view, js, batch, keep)
        torch.cuda.synchronize()
        for k, j in enumerate(js):  # the stored maps are the inputs, bit for bit
            for r in range(2):
                slot = b.nodes - 2 * len(js) + 2 * k + r
                assert torch.equal(g.depth[slot].view(torch.int32), batch["depths"][r, k].view(torch.int32))
                assert torch.equal(g.conf[slot].view(torch.int32), batch["conf"][r, k].view(torch.int32))
    assert len(b.scale) == 3 + 5  # view 2: k = 1 and both js; view 3: k = 1, 2 and all three js
    es, ec = _check_scale_edges(g, b.scale)
    _report("scale %dx%d" % (H, W), es)
    _report("scale_conf %dx%d" % (H, W), ec)
    _report("node_pose", _check_nodes(g, b.derived))


# ------------------------------------------------------------------------------- (d) a full keyframe
def test_full_keyframe_against_the_oracle_bookkeeping():
    H, W = 56, 64
    V = 33
    g = _graph(2 * 31 + 64 + 8, 200, 64, H, W)
    oracle = so.Graph(200, 200)
    b = _Builder(g, oracle)
    r = np.random.default_rng(3)
    pr = random_pairs(64, seed=9)[0]
    for v in range(1, V):  # view v with js = [v - 1]; every node's confidence mean is 3.0 or 3.5 (ties)
        batch, keep = _batch([_pose44(pr[v, 3:7], pr[v, :3])], H, W, v, conf_mean=[[3.0], [3.0 + 0.5 * (v % 3 == 0)]],
                             plant=False)  # scale edges near 0.8 along the chain of views, clear of underflow
        b.add(v, [v - 1], batch, keep)
    K = 40
    keep = sorted(r.choice(K, 32, replace=False).tolist())
    rows = [_pose44(pr[k, 3:7], pr[k, :3] * 10) for k in range(K)]
    js = list(range(1, V))
    cm = np.full((2, 32), 3.0, np.float32)
    cm[0, 5] = cm[0, 9] = 4.0  # view V: a tie for the best mean; the first node wins
    cm[1, ::4] = 3.5  # views j: some new best means, the rest tie the current one
    batch, keep = _batch(rows, H, W, 77, keep=keep, conf_mean=cm)
    first_j = b.add(V, js, batch, keep)
    assert len(first_j) == 32 and min(first_j) >= 0
    torch.cuda.synchronize()
    assert b.edges == oracle.num_edges and b.nodes == oracle.num_nodes
    N, E = oracle.num_nodes, oracle.num_edges
    assert sum(1 for e, nn, _ in b.scale if nn >= N - 64) == 63
    np.testing.assert_array_equal(g.node_to_view[:N].cpu().numpy(), oracle.node_to_view[:N])
    np.testing.assert_array_equal(g.node_to_connected_view[:N].cpu().numpy(), oracle.node_to_connected_view[:N])
    np.testing.assert_array_equal(g.edges[:E].cpu().numpy(), oracle.edges[:E])
    np.testing.assert_array_equal(g.best_node[:V + 1].cpu().numpy(), oracle.best_node[:V + 1])
    assert int(g.best_node[V]) == N - 64 + 2 * 5  # the first of the tied nodes
    np.testing.assert_array_equal(g.cmean[:N].cpu().numpy(), np.array(oracle.cmean, np.float32))
    for k in range(32):
        for rr in range(2):
            slot = N - 64 + 2 * k + rr
            assert torch.equal(g.depth[slot].view(torch.int32), batch["depths"][rr, k].view(torch.int32))
            assert torch.equal(g.conf[slot].view(torch.int32), batch["conf"][rr, k].view(torch.int32))
            assert torch.equal(g.intri[slot], batch["intri"][k])
    _report("edge_quaternion", _check_pose_edges(g, b.pose))
    es, ec = _check_scale_edges(g, b.scale)
    _report("scale full keyframe", es)
    _report("scale_conf full keyframe", ec)
    _report("node_pose", _check_nodes(g, b.derived))


# ------------------------------------------------------------------------------- (e) capacities
def _snapshot(g):
    return {k: v.tobytes() for k, v in _tables(g).items()}


def test_capacities_exactly_full_and_one_more_refused():
    L = _lib()
    H = W = 8
    g = _graph(6, 6, 4, H, W)  # kf 1: nodes 0-1, edge 0; kf 2: nodes 2-5, edges 1-5 (3 scale, 2 pose)
    oracle = so.Graph(6, 6)
    b = _Builder(g, oracle)
    pr = random_pairs(4, seed=2)[0]
    b1, k1 = _batch([_pose44(pr[0, 3:7], pr[0, :3])], H, W, 1)
    b.add(1, [0], b1, k1)
    b2, k2 = _batch([_pose44(pr[1, 3:7], pr[1, :3]), _pose44(pr[2, 3:7], pr[2, :3])], H, W, 2)
    b.add(2, [1, 0], b2, k2)
    torch.cuda.synchronize()
    assert (b.nodes, b.edges) == (g.max_nodes, g.max_edges) == (oracle.num_nodes, oracle.num_edges)
    np.testing.assert_array_equal(g.node_to_view.cpu().numpy(), oracle.node_to_view)
    np.testing.assert_array_equal(g.edges.cpu().numpy(), oracle.edges)
    assert list(g.edges[5].cpu().numpy()) == [4, 5] and int(g.node_to_view[5]) == 0 and int(g.node_to_connected_view[5]) == 2
    assert torch.equal(g.depth[5], b2["depths"][1, 1]) and torch.equal(g.intri[5], b2["intri"][1])
    _report("node_pose", _check_nodes(g, b.derived))
    _report("edge_quaternion", _check_pose_edges(g, b.pose))
    _report("scale capacity", max(_check_scale_edges(g, b.scale)))
    before, flags = _snapshot(g), g.flags()
    # one node more (node0 + 2n = max_nodes + 1), one edge more (edge0 + n_scale + n = max_edges + 1)
    rc = _add(g, 2, [1, 0], [0, 1], 3, 0, b2, k2)
    assert rc != 0 and b"node capacity" in L.lib().sta_last_error()
    rc = _add(g, 2, [1, 0], [-1, 1], 0, 3, b2, k2)
    assert rc != 0 and b"edge capacity" in L.lib().sta_last_error()
    torch.cuda.synchronize()
    assert _snapshot(g) == before and g.flags() == flags


def test_reset_beyond_one_grid_pass():
    L = _lib()
    g = _graph(70_000, 200_000, 66_000, 1, 1)  # 256 x 256 threads per pass: 1, 3 and 2 passes over the three tables
    for name, val in (("pose", 7.0), ("cmean", 7.0), ("node_to_view", 5), ("node_to_connected_view", 5), ("best_node", 5),
                      ("best_mean", 7.0), ("edges", 5), ("meas", 7.0), ("weight", 7.0)):
        getattr(g, name).fill_(val)
    L.check(L.lib().sta_graph_reset(g.h, L.cur_stream()), "sta_graph_reset")
    torch.cuda.synchronize()
    ident = torch.tensor([0, 0, 0, 0, 0, 0, 1, 1.0], device="cuda")
    assert (g.pose == ident).all() and (g.meas == ident).all() and (g.weight == 1).all()
    assert (g.node_to_view == -1).all() and (g.node_to_connected_view == -1).all() and (g.cmean == 0).all()
    assert (g.edges == -1).all() and (g.best_node == -1).all() and (g.best_mean == -100).all()
    assert g.flags() == 0


# ------------------------------------------------------------------------------- (f) replay
def test_replay_over_many_launches():
    L = _lib()
    stream = so.make_stream(n_views=160)
    images = so.stream_images(stream)
    n, K = stream["n_views"], 8
    a, b = _replay(stream, pgo_every=1000), _replay(stream, pgo_every=1000)
    for i in range(K):
        a.step(_value(images, i, stream))
        b.step(_value(images, i, stream))
    N0 = a.num_nodes
    p = a._graph.pose[:N0].clone()
    d = torch.randn(N0, 8, generator=torch.Generator().manual_seed(4)).cuda() * 0.1
    q = p[:, 3:7] + d[:, 3:7]
    q = q / q.norm(dim=1, keepdim=True)
    q = torch.where(q[:, 3:4] < 0, -q, q)
    roots = torch.cat([p[:, :3] + d[:, :3] * 100, q, p[:, 7:] * (1 + d[:, 7:].abs())], 1).contiguous()
    a._graph.pose[:N0] = roots
    rec = []
    b._pgo_run = (_Pending(), None, rec)
    for i in range(K, n):
        a.step(_value(images, i, stream))
        b.step(_value(images, i, stream))
    b._pgo_run = None
    assert len(rec) > 512  # three launches of kReplayChunk = 256 triples or more
    launch = {}
    for t, (node, _, _) in enumerate(rec):
        launch[node] = t // 256
    assert any(launch.get(par, t // 256) < t // 256 for t, (_, par, _) in enumerate(rec) if t >= 512)
    G = b._graph
    G.pose[:N0] = roots
    flat = (ctypes.c_int * (3 * len(rec)))(*[x for t in rec for x in t])
    L.check(L.lib().sta_graph_replay_nodes(G.h, len(rec), flat, L.cur_stream()), "sta_graph_replay_nodes")
    assert G.pose[:b.num_nodes].cpu().numpy().tobytes() == a._graph.pose[:a.num_nodes].cpu().numpy().tobytes()
    _assert_identical(_full(a), _full(b))
    _report("node_pose replay", _check_nodes(G, rec))


# ------------------------------------------------------------------------------- (g) export
def _export_graph(V, H, W, per_view, seed, max_views=None, max_edges=1):
    """A graph whose tables are written directly: V views of per_view nodes each, random poses (t up to 1e2, scales in
    [0.1, 10], quaternions up to 1e-3 off unit), intrinsics, depths in [-0.5, 4] and confidences in [0, 8]; best node
    of each view random among its nodes."""
    N = V * per_view
    g = _graph(N, max_edges, max_views or V, H, W)
    gen = torch.Generator(device="cuda").manual_seed(seed)

    def u(*s):
        return torch.rand(*s, generator=gen, device="cuda")

    q = torch.randn(N, 4, generator=gen, device="cuda")
    q = q / q.norm(dim=1, keepdim=True) * (1 + 1e-3 * (2 * u(N, 1) - 1))
    g.pose.copy_(torch.cat([200 * u(N, 3) - 100, q, 10 ** (2 * u(N, 1) - 1)], 1))
    K = torch.zeros(N, 3, 3, device="cuda")
    K[:, 0, 0], K[:, 1, 1] = W * (0.8 + 0.4 * u(N)), H * (0.8 + 0.4 * u(N))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = u(N) - 0.5, W / 2 + 10 * u(N) - 5, H / 2 + 10 * u(N) - 5, 1
    g.intri.copy_(K)
    g.depth.copy_(4.5 * u(N, H, W) - 0.5)
    g.conf.copy_(8 * u(N, H, W))
    best = torch.arange(V, device="cuda") * per_view + (u(V) * per_view).long().clamp_max(per_view - 1)
    g.best_node[:V] = best
    imgs = (2 * u(V, 3, H, W) - 1).contiguous()
    return g, imgs


def _run_export(g, view0, nv, thres, imgs):
    L = _lib()
    H, W = g.H, g.W

    def f32(*s):
        return torch.empty(*s, dtype=torch.float32, device="cuda")

    out = {"pose": f32(nv, 4, 4), "scale": f32(nv, 1), "depth": f32(nv, H, W), "conf": f32(nv, H, W), "intri": f32(nv, 3, 3),
           "points": f32(nv * H * W, 3), "colors": f32(nv * H * W, 3), "count": torch.zeros(1, dtype=torch.int64, device="cuda")}
    nbytes = int(L.lib().sta_graph_export_scratch_bytes(nv, H))
    scratch = torch.empty((nbytes + 7) // 8, dtype=torch.int64, device="cuda")
    L.check(L.lib().sta_graph_export(g.h, view0, nv, float(thres), L.ptr(imgs), L.ptr(out["pose"]), L.ptr(out["scale"]),
                                     L.ptr(out["depth"]), L.ptr(out["conf"]), L.ptr(out["intri"]), L.ptr(out["points"]),
                                     L.ptr(out["colors"]), L.ptr(out["count"]), L.ptr(scratch), L.cur_stream()),
            "sta_graph_export")
    return out


def _bits(t):
    return t.contiguous().view(torch.int32)


def _check_export(g, view0, nv, thres, imgs, name, chunk=1 << 22):
    """Export views view0 .. view0 + nv - 1 (imgs: the images of all views) and check every output."""
    imgs = imgs[view0:view0 + nv].contiguous()
    out = _run_export(g, view0, nv, thres, imgs)
    b = g.best_node[view0:view0 + nv]
    p = g.pose[b]
    assert torch.equal(_bits(out["scale"][:, 0]), _bits(p[:, 7]))
    for k, table in (("intri", g.intri), ("depth", g.depth), ("conf", g.conf)):
        assert torch.equal(_bits(out[k]), _bits(table[b])), k
    P = out["pose"]
    assert torch.equal(_bits(P[:, :3, 3]), _bits(p[:, :3]))
    assert (P[:, 3] == torch.tensor([0, 0, 0, 1.0], device="cuda")).all()
    x, y, z, w = p[:, 3:7].double().unbind(1)
    ax, ay, az, aw = x.abs(), y.abs(), z.abs(), w.abs()
    ref = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                       2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                       2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    mag = torch.stack([1 + 2 * (ay * ay + az * az), 2 * (ax * ay + az * aw), 2 * (ax * az + ay * aw),
                       2 * (ax * ay + az * aw), 1 + 2 * (ax * ax + az * az), 2 * (ay * az + ax * aw),
                       2 * (ax * az + ay * aw), 2 * (ay * az + ax * aw), 1 + 2 * (ax * ax + ay * ay)], 1).view(-1, 3, 3)
    r_rot = float(((P[:, :3, :3].double() - ref).abs() / (C_ROT * F32 * mag)).max())
    # the kept pixels in (view, row, column) order: conf > thres (a NaN or a confidence at the threshold is not kept)
    idx = (out["conf"] > torch.tensor(thres, dtype=torch.float32, device="cuda")).flatten().nonzero()[:, 0]
    n = int(out["count"])
    assert n == len(idx)
    H, W = g.H, g.W
    Ki = inv3(out["intri"].double())
    Pd, s = P.double(), out["scale"][:, 0].double()
    worst = 0.0
    for c0 in range(0, n, chunk):
        i = idx[c0:c0 + chunk]
        v, row, col = i // (H * W), (i // W) % H, i % W
        ds = out["depth"].flatten()[i].double() * s[v]
        refp, S = unproject_ref([k[v] for k in Ki], Pd[v], col.double(), row.double(), ds)
        got = out["points"][c0:c0 + len(i)].double()
        for c in range(3):
            worst = max(worst, float(((got[:, c] - refp[c]).abs() / (C_PT * F32 * S[c])).max()))
        col_ref = (imgs[v, :, row, col] + 1) / 2
        assert torch.equal(_bits(out["colors"][c0:c0 + len(i)]), _bits(col_ref))
    _report("export_rotation " + name, r_rot)
    _report("export_point " + name, worst)
    return out, n


@pytest.mark.parametrize("W", [255, 256, 257, 512, 513])
def test_export_across_row_widths(W):
    H, V, thres = 3, 7, 4.2
    g, imgs = _export_graph(V, H, W, 2, W)
    b = g.best_node[:V]
    conf = g.conf[b].clone()
    conf[0] = thres - 1  # nothing
    conf[1] = thres + 1  # everything
    conf[2] = thres - 1
    conf[2, :, min(256, W - 1)] = thres + 1  # only column 256 (the first of the second pass)
    conf[3] = thres - 1
    conf[3, :, W - 1] = thres + 1  # only the last column
    conf[4, 0, ::3] = thres  # at the threshold: not kept
    conf[4, 1, ::5] = float("nan")
    for v in range(V):
        g.conf[b[v]] = conf[v]
    out, n = _check_export(g, 0, V, thres, imgs, "W=%d" % W)
    counts = [(out["conf"][v] > thres).sum().item() for v in range(V)]
    assert counts[:4] == [0, H * W, H, H] and n == sum(counts)


@pytest.mark.parametrize("V,H", [(3, 100), (8, 256), (7, 433)])
def test_export_across_row_counts(V, H):
    g, imgs = _export_graph(V, H, 40, 3, V * H)
    _check_export(g, 0, V, 4.2, imgs, "rows=%d" % (V * H))


def test_export_of_a_view_range():
    g, imgs = _export_graph(10, 20, 300, 2, 5)
    _, n = _check_export(g, 3, 5, 4.2, imgs, "views 3-7")
    assert n > 0


def test_export_at_production_size():
    """OnlineSLAM's defaults: max_view_num = 400 -> 3600 nodes, 5200 edges, 3600 views; 400 views of 224 x 224."""
    V, H, W = 400, 224, 224
    g, imgs = _export_graph(V, H, W, 9, 400, max_views=3600, max_edges=5200)
    _, n = _check_export(g, 0, V, 4.2, imgs, "400x224x224")
    assert n > 8_000_000


# ------------------------------------------------------------------------------- (h) reconstruction clouds
@pytest.mark.parametrize("W", [512, 513])
def test_reconstruction_clouds_across_two_row_passes(W):
    from vista_slam_b200.eval import eval_recon as R
    s = eo.make_scene(n_views=4, H=6, W=W, nan_view=99)
    confs = s["confs"].copy()
    confs[0] = 1.0
    confs[0, :, 256] = 9.0  # only column 256
    confs[1] = 9.0  # everything
    confs[2] = 1.0
    confs[2, :, W - 1] = 9.0  # only the last column
    gt, est = R.world_clouds(s["gt_depths"], s["gt_poses"], s["gt_intrinsics"], s["depths"], s["scales"].reshape(-1),
                             s["trajectory"], s["intrinsics"], confs, s["thres"])
    tg, te = eo.clouds(torch.from_numpy(s["gt_depths"]), torch.from_numpy(s["gt_poses"]), torch.from_numpy(s["gt_intrinsics"]),
                       torch.from_numpy(s["depths"] * s["scales"][:, :, None]), torch.from_numpy(s["trajectory"]),
                       torch.from_numpy(s["intrinsics"]), torch.from_numpy(confs > s["thres"]).float())
    assert len(gt) == len(tg) and len(est) == len(te) and len(est) > 0
    _assert_close_f32(gt.cpu().numpy(), tg.astype(np.float64))
    _assert_close_f32(est.cpu().numpy(), te.astype(np.float64))
