"""GPU: TSDF fusion and marching cubes (csrc/fusion.cu, vista_slam_b200/fusion.py, OnlineSLAM.extract_mesh / save_mesh).

  1. Planted scenes where every float32 operation is exact (power-of-two voxel, focal lengths and depths at half
     voxels, integer principal points, identity or axis-permutation poses), one and two views, with a far point that
     falls outside the brick range: bricks, tsdf, weight, colour, vertices and faces bit for bit against the oracle
     (vertex colours beside the far point's column to one float32 rounding).
  2. Random scenes against the float64 oracle (oracle/fusion_oracle.py): brick sets equal up to cube faces within 1e-4 v
     of a brick boundary; on unambiguous samples weight equal, tsdf and colour within 1e-5; faces equal as vertex-key
     triples on cubes whose corners are unambiguous, vertices within 1e-5 v plus the move that a float32 tsdf error of
     2e-6 causes on the vertex's edge; and the mesh of the device's own volume
     equal to the oracle's marching cubes of it.
  3. Topology on analytic volumes and a noisy sphere full of saddles, through marching_cubes: a closed oriented manifold (every undirected edge in two
     faces, every directed edge in at most one), Euler characteristic 2 (sphere) and 0 (torus), positive signed volume
     within 2 % of the analytic one, every vertex on the linear zero crossing of its edge.
  4. A sphere fused from 26 ray-cast views: every vertex within trunc of the sphere, mean distance below v / 2.
  5. A replayed OnlineSLAM run: the same bits on every call, the session left as it was, every vertex within trunc + v
     of the PLY cloud, background PGO equal to synchronous, save_mesh's file equal to the tensors.
  6. The real frontend: a non-empty mesh, no edge in more than two faces.
  7. Refusals before any launch."""
import numpy as np
import pytest
import torch

from oracle import fusion_oracle as fo
from oracle import slam_oracle as so
from test_slam_batch_gpu import _frames_224
from test_slam_gpu import VOCAB, _replay_slam, _value

pytestmark = pytest.mark.gpu


def _dev(maps):
    return {k: torch.as_tensor(np.ascontiguousarray(v, dtype=np.float32)).cuda() for k, v in maps.items()}


def _K(f, cx, cy):
    return np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]], np.float32)


def _fuse(maps, voxel, **kw):
    from vista_slam_b200.fusion import fuse_views
    out = fuse_views(_dev(maps), 0.5, voxel, **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


# ------------------------------------------------------------------------------------------------ (1)
def _planted(two_views, far_point):
    """A fronto-parallel plane at z = 8.5 v (v = 1/4) seen by an 8 x 8 camera at the origin (f = 8, c = (4, 4)) and
    optionally by a second one rotated 90 degrees about z and moved to (1/2, 1/4, -1/2); images on a 2^-3 grid."""
    v = 0.25
    H = W = 8
    r = np.random.default_rng(3)
    poses = [np.eye(4, dtype=np.float32)]
    depths = [np.full((H, W), 8.5 * v, np.float32)]
    if two_views:
        P = np.eye(4, dtype=np.float32)
        P[:3, :3] = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]
        P[:3, 3] = [0.5, 0.25, -0.5]
        poses.append(P)
        depths.append(np.full((H, W), 8.5 * v + 0.5, np.float32))
    V = len(poses)
    d = np.stack(depths)
    conf = np.ones((V, H, W), np.float32)
    conf[0, 0, 0] = 0.25  # below the threshold
    if far_point:
        d[0, 7, 7] = 1e30  # its bricks fall outside [-2^20, 2^20 - 1]: skipped by the allocation
    maps = {"pose": np.stack(poses), "scale": np.ones((V, 1), np.float32), "depth": d, "conf": conf,
            "intri": np.stack([_K(8, 4, 4)] * V), "images": (np.rint(r.uniform(-8, 8, (V, 3, H, W))) / 8).astype(np.float32)}
    return maps, v


@pytest.mark.parametrize("two_views", [False, True])
@pytest.mark.parametrize("far_point", [False, True])
def test_planted_scenes_bit_for_bit(two_views, far_point):
    maps, v = _planted(two_views, far_point)
    got = _fuse(maps, v)
    want = fo.fuse(maps, 0.5, v)
    np.testing.assert_array_equal(got["bricks"], want["bricks"])
    assert want["sure"] == want["maybe"]
    for k in ("tsdf", "weight", "color"):
        np.testing.assert_array_equal(got[k], want[k].astype(np.float32), err_msg=k)
    mesh = fo.marching_cubes(want["bricks"], want["tsdf"], want["weight"], want["color"], v)
    assert len(mesh["faces"]) > 0
    np.testing.assert_array_equal(got["vertices"], mesh["vertices"].astype(np.float32))
    if far_point:
        # the far pixel's t = 1 beside t = -1/8 puts vertices at fractions such as 1/9, where the float32 colour
        # interpolation rounds once more than the float64 one
        np.testing.assert_allclose(got["vertex_colors"], mesh["vertex_colors"], rtol=2.0 ** -23, atol=0)
    else:
        np.testing.assert_array_equal(got["vertex_colors"], mesh["vertex_colors"].astype(np.float32))
    np.testing.assert_array_equal(got["faces"], mesh["faces"])
    # the plane's vertices lie on it, half-way between samples (the far point's pixel adds a surface of its own)
    if not far_point:
        np.testing.assert_array_equal(got["vertices"][:, 2], np.full(len(got["vertices"]), 8.5 * v, np.float32))


# ------------------------------------------------------------------------------------------------ (2)
def _look_at(eye, target, up=(0.0, 1.0, 0.0)):
    z = np.asarray(target, np.float64) - eye
    z /= np.linalg.norm(z)
    x = np.cross(up, z)
    if np.linalg.norm(x) < 1e-6:
        x = np.cross((1.0, 0.0, 0.0), z)
    x /= np.linalg.norm(x)
    P = np.eye(4)
    P[:3, :3] = np.stack([x, np.cross(z, x), z], 1)
    P[:3, 3] = eye
    return P


def _random_scene(seed, V=3, H=20, W=24):
    r = np.random.default_rng(seed)
    poses, depths = [], []
    for _ in range(V):
        P = _look_at(r.normal(0, 0.15, 3) + [0, 0, -1.0], r.normal(0, 0.05, 3))
        poses.append(P)
        yy, xx = np.mgrid[0:H, 0:W]
        depths.append(1.0 + 0.1 * np.sin(xx / 4.0 + r.uniform(0, 6)) * np.cos(yy / 5.0) + r.uniform(-0.02, 0.02, (H, W)))
    maps = {"pose": np.stack(poses).astype(np.float32), "scale": r.uniform(0.9, 1.1, (V, 1)).astype(np.float32),
            "depth": np.stack(depths).astype(np.float32), "conf": r.uniform(0, 2, (V, H, W)).astype(np.float32),
            "intri": np.stack([_K(20.0, W / 2 - 0.5, H / 2 - 0.5)] * V),
            "images": r.uniform(-1, 1, (V, 3, H, W)).astype(np.float32)}
    maps["depth"] /= maps["scale"][:, :, None]
    return maps


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_scenes_against_fp64(seed):
    maps = _random_scene(seed)
    v = 0.03
    got = _fuse(maps, v, trunc=0.09)
    want = fo.fuse(maps, 0.5, v, trunc=0.09)
    gk = set(fo.key(got["bricks"]).tolist())
    assert want["sure"] <= gk <= want["maybe"]
    # samples of the bricks both have
    common = np.intersect1d(fo.key(got["bricks"]), want["keys"])
    gi = np.searchsorted(fo.key(got["bricks"]), common)
    wi = np.searchsorted(want["keys"], common)
    amb = want["ambiguous"][wi]
    ok = ~amb
    np.testing.assert_array_equal(got["weight"][gi][ok], want["weight"][wi][ok])
    np.testing.assert_allclose(got["tsdf"][gi][ok], want["tsdf"][wi][ok], rtol=0, atol=1e-5)
    np.testing.assert_allclose(got["color"][gi][ok], want["color"][wi][ok], rtol=0, atol=1e-5)
    print("seed %d: %d bricks, %d of %d samples ambiguous" % (seed, len(gk), amb.sum(), amb.size))
    # the device mesh is the oracle's marching cubes of the device volume
    own = fo.marching_cubes(got["bricks"], got["tsdf"], got["weight"], got["color"], v)
    np.testing.assert_array_equal(got["faces"], own["faces"])
    np.testing.assert_allclose(got["vertices"], own["vertices"], rtol=0, atol=1e-6 * v + 1e-6)
    np.testing.assert_allclose(got["vertex_colors"], own["vertex_colors"], rtol=0, atol=1e-6)
    # against the oracle volume's mesh: faces as vertex-key triples on cubes whose corners are all unambiguous
    ref = fo.marching_cubes(want["bricks"], want["tsdf"], want["weight"], want["color"], v)
    assert len(ref["faces"]) > 0

    def clean_cubes(mesh):
        keep = []
        for c in mesh["face_cubes"]:
            ok_c = True
            for o in range(8):
                q = c + [o & 1, o >> 1 & 1, o >> 2]
                b = np.floor_divide(q, 8)
                j = np.searchsorted(want["keys"], fo.key(b))
                if j >= len(want["keys"]) or want["keys"][j] != fo.key(b):
                    ok_c = False
                    break
                loc = q - 8 * b
                if want["ambiguous"][j, loc[2], loc[1], loc[0]]:
                    ok_c = False
                    break
            keep.append(ok_c)
        return np.array(keep, bool)

    def triples(mesh, keep):
        vk = mesh["vertex_keys"]
        return {tuple(map(tuple, vk[f])) for f in mesh["faces"][keep]}

    a, b = triples(own, clean_cubes(own)), triples(ref, clean_cubes(ref))
    assert a == b
    # vertices of the edges both meshes have
    pos_own = {tuple(k): p for k, p in zip(own["vertex_keys"], own["vertices"])}
    pos_ref = {tuple(k): p for k, p in zip(ref["vertex_keys"], ref["vertices"])}
    shared = {k for t in a for k in t}
    Tr = want["tsdf"].reshape(-1)

    def tval(q):
        bb = np.floor_divide(q, 8)
        loc = q - 8 * bb
        return Tr[np.searchsorted(want["keys"], fo.key(bb)) * 512 + loc[2] * 64 + loc[1] * 8 + loc[0]]

    for k in shared:
        # a tsdf error dT moves a vertex by v dT / |T_a - T_b|: 1e-5 v, plus 2e-6 v / |T_a - T_b| for the tsdf's own
        # float32 error (3e-5 v on an edge whose tsdf difference is 0.1)
        q = np.array(k[:3])
        q2 = q.copy()
        q2[k[3]] += 1
        tol = v * (1e-5 + 2e-6 / abs(tval(q) - tval(q2)))
        assert np.abs(pos_own[k] - pos_ref[k]).max() <= tol, k


# ------------------------------------------------------------------------------------------------ (3)
def _field_volume(f, v, lo, hi):
    """Bricks covering lattice [lo, hi] per axis, sorted by key, weight 1, tsdf = f(x) at the float32 lattice points,
    colour = x."""
    bl, bh = np.floor_divide(lo, 8), np.floor_divide(hi, 8)
    b = np.stack(np.meshgrid(*[np.arange(bl[k], bh[k] + 1) for k in range(3)], indexing="ij"), -1).reshape(-1, 3)
    b = b[np.argsort(fo.key(b))]
    ijk = fo.sample_coords(fo.key(b))
    X = (ijk.astype(np.float32) * np.float32(v)).astype(np.float64)
    T = f(X).astype(np.float32)
    return b.astype(np.int32), T, np.ones_like(T), X.astype(np.float32)


def _mc(b, T, Wt, C, v, **kw):
    from vista_slam_b200.fusion import marching_cubes
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a)).cuda()
    out = marching_cubes(t(b), t(T), t(Wt), t(C), v, **kw)
    return {k: x.cpu().numpy() for k, x in out.items()}


def _topology(V, F):
    e = np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]])
    directed = {tuple(x) for x in e.tolist()}
    assert len(directed) == len(e), "a directed edge is in two faces"
    und = np.sort(e, 1)
    _, counts = np.unique(und, axis=0, return_counts=True)
    assert (counts == 2).all(), "an edge is not in exactly two faces"
    used = np.unique(F)
    assert len(used) == len(V)
    return len(V) - len(counts) + len(F)


def _signed_volume(V, F):
    a, b, c = V[F[:, 0]].astype(np.float64), V[F[:, 1]].astype(np.float64), V[F[:, 2]].astype(np.float64)
    return np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0


def _check_against_oracle_mc(vol, v, got):
    own = fo.marching_cubes(*vol, v)
    np.testing.assert_array_equal(got["faces"], own["faces"])
    np.testing.assert_allclose(got["vertices"], own["vertices"], rtol=0, atol=2e-6 * max(1.0, np.abs(own["vertices"]).max()))
    # each vertex on the linear zero crossing of its edge
    return own


@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_topology_of_analytic_volumes(shape):
    if shape == "sphere":
        R, v = 1.0, 0.1
        vol = _field_volume(lambda X: np.linalg.norm(X, axis=-1) - R, v, np.array([-14] * 3), np.array([13] * 3))
        want_chi, want_vol = 2, 4.0 / 3.0 * np.pi * R ** 3
    else:
        R, r, v = 1.0, 0.4, 0.05
        f = lambda X: np.hypot(np.hypot(X[..., 0], X[..., 1]) - R, X[..., 2]) - r
        vol = _field_volume(f, v, np.array([-32, -32, -10]), np.array([31, 31, 9]))
        want_chi, want_vol = 0, 2 * np.pi ** 2 * R * r ** 2
    got = _mc(*vol, v)
    chi = _topology(got["vertices"], got["faces"])
    assert chi == want_chi
    sv = _signed_volume(got["vertices"], got["faces"])
    assert sv > 0 and abs(sv - want_vol) <= 0.02 * want_vol, (sv, want_vol)
    _check_against_oracle_mc(vol, v, got)


@pytest.mark.parametrize("seed", [0, 1])
def test_topology_of_random_fields_with_saddles(seed):
    """A sphere's distance field with uniform noise of +-0.08 on the samples near it (1.6 steps of the field per voxel):
    many cube faces are ambiguous (saddles), and the zero set stays well inside the volume."""
    v = 0.05
    vol = _field_volume(lambda X: np.linalg.norm(X, axis=-1) - 1.0, v, np.array([-32] * 3), np.array([31] * 3))
    T = vol[1]
    T += (0.08 * np.random.default_rng(seed).uniform(-1, 1, T.shape) * (np.abs(T) < 0.3)).astype(np.float32)
    got = _mc(*vol, v)
    assert len(got["faces"]) > 0
    _topology(got["vertices"], got["faces"])
    assert _signed_volume(got["vertices"], got["faces"]) > 0
    own = _check_against_oracle_mc(vol, v, got)
    # vertices on the linear zero crossing: interpolating the field along each vertex's edge gives 0
    keys = fo.key(vol[0])
    Tf = T.reshape(-1)

    def tval(q):
        bb = np.floor_divide(q, 8)
        loc = q - 8 * bb
        return Tf[np.searchsorted(keys, fo.key(bb)) * 512 + loc[2] * 64 + loc[1] * 8 + loc[0]]

    for (i, j, kk, ax), p in zip(own["vertex_keys"], got["vertices"]):
        q = np.array([i, j, kk])
        q2 = q.copy()
        q2[ax] += 1
        xa, xb = np.float32(q[ax]) * np.float32(v), np.float32(q2[ax]) * np.float32(v)
        s = (np.float64(p[ax]) - xa) / (np.float64(xb) - xa)
        assert 0 <= s <= 1 and abs(tval(q) + s * (tval(q2) - tval(q))) <= 1e-5


# ------------------------------------------------------------------------------------------------ (4)
def test_fused_sphere_from_ray_cast_views():
    R, H, W, f = 1.0, 64, 64, 60.0
    K = _K(f, W / 2 - 0.5, H / 2 - 0.5).astype(np.float64)
    dirs = [np.array(d, np.float64) for d in np.ndindex(3, 3, 3) if d != (1, 1, 1)]
    poses, depths = [], []
    for d in dirs:
        d = (d - 1) / np.linalg.norm(d - 1)
        P = _look_at(3.0 * d, np.zeros(3), up=(0.0, 0.0, 1.0) if abs(d[2]) < 0.9 else (0.0, 1.0, 0.0))
        yy, xx = np.mgrid[0:H, 0:W]
        ray = np.linalg.inv(K) @ np.stack([xx.ravel(), yy.ravel(), np.ones(H * W)])  # camera frame, z = 1
        rw = P[:3, :3] @ ray
        o = P[:3, 3][:, None]
        a, b, c = (rw * rw).sum(0), 2 * (o * rw).sum(0), (o * o).sum() - R * R
        disc = b * b - 4 * a * c
        t = np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), 0.0)
        poses.append(P)
        depths.append(t.reshape(H, W))
    V = len(poses)
    d = np.stack(depths).astype(np.float32)
    maps = {"pose": np.stack(poses).astype(np.float32), "scale": np.ones((V, 1), np.float32), "depth": d,
            "conf": np.where(d > 0, 1.0, 0.0).astype(np.float32), "intri": np.stack([K] * V).astype(np.float32),
            "images": np.zeros((V, 3, H, W), np.float32)}
    v = 0.04
    got = _fuse(maps, v)
    dist = np.abs(np.linalg.norm(got["vertices"].astype(np.float64), axis=1) - R)
    assert len(dist) > 1000
    assert dist.max() <= 4 * v and dist.mean() < 0.5 * v, (dist.max(), dist.mean())
    print("sphere: %d vertices, %d faces, mean %.4f v, max %.3f v" % (len(dist), len(got["faces"]), dist.mean() / v,
                                                                     dist.max() / v))


# ------------------------------------------------------------------------------------------------ (5)
def _replayed(n=None):
    stream = so.make_stream()
    slam = _replay_slam(stream)
    images = so.stream_images(stream)
    n = stream["n_views"] if n is None else n
    for i in range(n):
        slam.step(_value(images, i, stream), force_pgo=(i == n - 1))
    return slam, stream


def _voxel_of(slam):
    """1/64 of the cloud's extent between its 2nd and 98th percentiles per axis, and the cloud."""
    ex = slam._export(0, slam.view_num, cloud=True)
    pts = ex["points"][:int(ex["count"].cpu())]
    lo, hi = np.percentile(pts.cpu().numpy(), [2, 98], axis=0)
    return float((hi - lo).max()) / 64.0, pts


def test_replayed_run_is_deterministic_read_only_and_near_the_cloud(tmp_path):
    from vista_slam_b200.eval.eval_recon import NnIndex
    from vista_slam_b200.slam import read_mesh_ply
    slam, stream = _replayed()
    v, pts = _voxel_of(slam)
    G = slam._graph
    tables = {k: getattr(G, k).clone() for k in ("pose", "depth", "conf", "intri", "cmean", "node_to_view",
                                                    "node_to_connected_view", "best_node", "best_mean", "edges", "meas",
                                                    "weight")}
    times = dict(slam.time_dict)
    host = (dict(slam.view_to_node), list(slam.node_to_connected_view), slam.num_nodes, slam.num_edges, slam.view_num)
    a = slam.extract_mesh(v)
    b = slam.extract_mesh(v)
    for k in a:
        assert torch.equal(a[k].view(torch.uint8) if a[k].is_floating_point() else a[k],
                           b[k].view(torch.uint8) if b[k].is_floating_point() else b[k]), k
    assert len(a["faces"]) > 100
    for k, t in tables.items():
        assert torch.equal(getattr(G, k).view(torch.uint8), t.view(torch.uint8)), k
    assert slam.time_dict == times
    assert host == (dict(slam.view_to_node), list(slam.node_to_connected_view), slam.num_nodes, slam.num_edges,
                    slam.view_num)
    nn = NnIndex(pts.double().contiguous())
    _, idx = nn.query(a["vertices"].double().contiguous(), 4 * v + v + 1e-6)
    assert (idx >= 0).all(), int((idx < 0).sum())
    path = slam.save_mesh(str(tmp_path), v)
    V, C, F = read_mesh_ply(path)
    np.testing.assert_array_equal(V, a["vertices"].cpu().numpy())
    np.testing.assert_array_equal(F, a["faces"].cpu().numpy())
    np.testing.assert_array_equal(C, np.rint(np.clip(a["vertex_colors"].cpu().double().numpy(), 0, 1) * 255))


def test_background_pgo_mesh_equals_synchronous():
    stream = so.make_stream()
    images = so.stream_images(stream)
    sync = _replay_slam(stream)
    bg = _replay_slam(stream)
    bg.pgo_background = True
    for i in range(14):
        sync.step(_value(images, i, stream))
        bg.step(_value(images, i, stream))
    bg.wait_pgo()
    v, _ = _voxel_of(sync)
    a = sync.extract_mesh(v, min_weight=2)
    b = bg.extract_mesh(v, min_weight=2)
    for k in a:
        assert torch.equal(a[k], b[k]), k


# ------------------------------------------------------------------------------------------------ (6)
def test_real_frontend_mesh_is_an_edge_manifold(cuda_model):
    import vista_slam_b200.slam as S

    class Run(S.OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return cuda_model

    slam = Run("unused", VOCAB, verbose=False, loop_dist_min=4, pgo_every=5, rel_pose_thres=0.5)
    frames = _frames_224(12)
    for i in range(12):
        slam.step(frames[i], force_pgo=(i == 11))
    ex = slam._export(0, slam.view_num, cloud=False)
    d = (ex["depth"] * ex["scale"][:, :, None])[ex["conf"] > slam.conf_thres]
    v = float(d[d > 0].median()) / 16.0  # the typical used depth sets the scale; random-weight maps have far outliers
    mesh = slam.extract_mesh(v)
    F = mesh["faces"].cpu().numpy()
    w = mesh["weight"]
    print("real frontend: voxel %.4g, %d bricks, %d observed samples, max weight %d, %d negative" % (
        v, len(mesh["bricks"]), int((w > 0).sum()), int(w.max()) if w.numel() else 0, int((mesh["tsdf"][w > 0] < 0).sum())))
    assert len(F) > 0
    e = np.sort(np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]]), 1)
    _, counts = np.unique(e, axis=0, return_counts=True)
    assert counts.max() <= 2


# ------------------------------------------------------------------------------------------------ (7)
def test_refusals_before_any_launch():
    from vista_slam_b200.fusion import fuse_views
    slam, stream = _replayed(n=5)
    v, _ = _voxel_of(slam)
    with pytest.raises(IndexError):
        slam.extract_mesh(v, views=range(0, 6))
    for kw in (dict(trunc=4.5 * v), dict(trunc=0.0), dict(min_weight=0), dict(voxel_size=-1.0)):
        args = dict(voxel_size=v)
        args.update(kw)
        with pytest.raises(ValueError):
            slam.extract_mesh(**args)
    maps = slam._view_maps(None)
    with pytest.raises(ValueError, match="max_bricks = 1"):
        fuse_views(maps, slam.conf_thres, v, max_bricks=1)
