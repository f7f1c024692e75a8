"""CPU: the TSDF fusion's float64 oracle (oracle/fusion_oracle.py) on hand-computed scenes, the generated
marching-cubes table (tools/make_mc_table.py, csrc/mc_table.h) through its topology, the mesh PLY round trip, and the
refusals of fuse_views, marching_cubes and the sta_fusion_* entry points that come before anything needs CUDA.

The hand scenes are fronto-parallel planes seen by cameras with K = I at the origin (or moved along z), so a sample
(x, y, z) projects to pixel (floor(x / z + 0.5), floor(y / z + 0.5)) and its sdf is d - z."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import fusion_oracle as fo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_mc_table as mct  # noqa: E402


def _plane(depths, conf=None, poses=None, H=4, W=4, images=None):
    """V views of a plane at camera depth depths[v] over every pixel; K = I."""
    V = len(depths)
    d = np.stack([np.full((H, W), z, np.float32) for z in depths])
    return {"pose": np.stack(poses).astype(np.float32) if poses is not None else np.tile(np.eye(4, dtype=np.float32), (V, 1, 1)),
            "scale": np.ones((V, 1), np.float32), "depth": d,
            "conf": np.ones_like(d) if conf is None else np.asarray(conf, np.float32),
            "intri": np.tile(np.eye(3, dtype=np.float32), (V, 1, 1)),
            "images": np.zeros((V, 3, H, W), np.float32) if images is None else np.asarray(images, np.float32)}


def _sample(vol, q):
    """(tsdf, weight, color) of lattice point q, or None when its brick does not exist."""
    b = np.floor_divide(q, 8)
    j = np.searchsorted(vol["keys"], fo.key(b))
    if j >= len(vol["keys"]) or vol["keys"][j] != fo.key(b):
        return None
    x, y, z = np.asarray(q) - 8 * b
    return vol["tsdf"][j, z, y, x], vol["weight"][j, z, y, x], vol["color"][j, z, y, x]


def test_one_view_plane_has_the_analytic_tsdf():
    v, d = 0.25, 2.0
    tau = 4 * v
    vol = fo.fuse(_plane([d]), 0.5, v)
    # the sample on the optical axis at every depth around the plane
    for k in range(-3, 13):
        z = k * v
        s = _sample(vol, (0, 0, k))
        if z > d + tau or z <= 0:
            assert s is None or s[1] == 0, (k, s)
            continue
        assert s is not None and s[1] == 1, k
        assert s[0] == min(1.0, (d - z) / tau), k
    # only samples within the truncation band behind the plane are observed
    assert vol["weight"][vol["tsdf"] < 0].size > 0 and (vol["tsdf"][vol["weight"] > 0] >= -1).all()


def test_two_views_average_and_the_far_side_is_skipped():
    v = 0.25
    tau = 4 * v
    back = np.eye(4)
    back[2, 3] = -1.0  # the second camera one unit behind the first: the plane at camera depth 3
    img = np.stack([np.full((3, 4, 4), -1.0), np.full((3, 4, 4), 1.0)])
    vol = fo.fuse(_plane([2.0, 3.0], poses=[np.eye(4), back], images=img), 0.5, v)
    s = _sample(vol, (0, 0, 6))  # z = 1.5: sdf 0.5 in both views
    assert s[1] == 2 and s[0] == 0.5 and (s[2] == 0.5).all()
    s = _sample(vol, (0, 0, 11))  # z = 2.75 > d + tau in neither view, t = -0.75
    assert s[1] == 2 and s[0] == -0.75
    assert _sample(vol, (0, 0, 13)) is None or _sample(vol, (0, 0, 13))[1] == 0  # z = 3.25 > 2 + tau


def test_a_pixel_below_the_threshold_contributes_nothing():
    v = 0.25
    conf = np.ones((2, 4, 4), np.float32)
    conf[1] = 0.25  # the second view is below the threshold everywhere
    img = np.stack([np.full((3, 4, 4), -1.0), np.full((3, 4, 4), 1.0)])
    one = fo.fuse(_plane([2.0], images=img[:1]), 0.5, v)
    two = fo.fuse(_plane([2.0, 1.0], conf=conf, images=img), 0.5, v)
    np.testing.assert_array_equal(one["keys"], two["keys"])
    for k in ("tsdf", "weight", "color"):
        np.testing.assert_array_equal(one[k], two[k])


def test_far_and_non_finite_points_allocate_nothing():
    v = 0.25
    maps = _plane([2.0, 1e30, np.inf])
    alone = fo.fuse(_plane([2.0]), 0.5, v)
    vol = fo.fuse(maps, 0.5, v)
    np.testing.assert_array_equal(vol["keys"], alone["keys"])


def test_oracle_marching_cubes_of_a_plane():
    v = 0.25
    vol = fo.fuse(_plane([2.125], H=8, W=8), 0.5, v)
    mesh = fo.marching_cubes(vol["bricks"], vol["tsdf"], vol["weight"], vol["color"], v)
    assert len(mesh["faces"]) > 0
    np.testing.assert_array_equal(mesh["vertices"][:, 2], 2.125)
    assert (mesh["vertex_keys"][:, 3] == 2).all()
    # faces wind counter-clockwise seen from the camera (outside, towards -z)
    V, F = mesh["vertices"], mesh["faces"]
    n = np.cross(V[F[:, 1]] - V[F[:, 0]], V[F[:, 2]] - V[F[:, 0]])
    assert (n[:, 2] < 0).all()
    # min_weight above every weight meshes nothing
    assert len(fo.marching_cubes(vol["bricks"], vol["tsdf"], vol["weight"], vol["color"], v, min_weight=2)["faces"]) == 0


# ------------------------------------------------------------------------------------------------ the table
def test_generated_table_matches_the_committed_header():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "make_mc_table.py"), "--check"], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    num, tris = fo.mc_table()
    for c in range(256):
        want = mct.case_triangles(c)
        assert num[c] == len(want)
        assert [tuple(tris[c, 3 * k:3 * k + 3]) for k in range(num[c])] == want
        assert (tris[c, 3 * num[c]:] == -1).all()


def _crossing(case):
    out = set()
    for e in range(12):
        a, b = mct.edge_corners(e)
        if (case >> a & 1) != (case >> b & 1):
            out.add(e)
    return out


@pytest.mark.parametrize("case", range(256))
def test_every_case_has_closed_loops_over_its_crossing_edges(case):
    crossing = _crossing(case)
    loops = mct.case_loops(case)
    used = [e for loop in loops for e in loop]
    assert sorted(used) == sorted(crossing)  # every crossing edge in exactly one loop
    for loop in loops:
        assert len(loop) >= 3
        # consecutive edges (and the last to the first) share a face: the loop closes
        for a, b in zip(loop, loop[1:] + loop[:1]):
            ca, cb = set(mct.edge_corners(a)), set(mct.edge_corners(b))
            assert any(ca | cb <= set(f) for f in mct.faces()), (case, loop)
    tris = mct.case_triangles(case)
    assert all(e in crossing for t in tris for e in t)  # no triangle on a non-crossing edge
    assert len(tris) == sum(len(loop) - 2 for loop in loops)
    # no fan diagonal lies on a cube face, where the neighbouring cube could draw it too
    loop_edges = {frozenset((a, b)) for loop in loops for a, b in zip(loop, loop[1:] + loop[:1])}
    for t in tris:
        for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
            assert frozenset((a, b)) in loop_edges or not mct.share_face(a, b), (case, t)


def test_ambiguous_face_keeps_inside_corners_apart():
    # corners 0 and 3 are diagonal on the z = 0 face: two separate loops, each around one corner
    loops = mct.case_loops(1 | 8)
    assert len(loops) == 2
    assert {frozenset(loop) for loop in loops} == {frozenset({0, 4, 8}), frozenset({1, 5, 11})}


# ------------------------------------------------------------------------------------------------ mesh PLY
def test_mesh_ply_round_trip(tmp_path):
    from vista_slam_b200.slam import read_mesh_ply, write_mesh_ply
    r = np.random.default_rng(0)
    V = r.normal(size=(50, 3)).astype(np.float32)
    C = r.uniform(-0.1, 1.1, (50, 3)).astype(np.float32)
    F = r.integers(0, 50, (80, 3)).astype(np.int32)
    path = str(tmp_path / "mesh.ply")
    write_mesh_ply(path, V, C, F)
    v, c, f = read_mesh_ply(path)
    np.testing.assert_array_equal(v, V)
    np.testing.assert_array_equal(f, F)
    np.testing.assert_array_equal(c, np.rint(np.clip(C.astype(np.float64), 0, 1) * 255).astype(np.uint8))
    with open(path, "rb") as fh:
        head = fh.read(400).split(b"end_header")[0].decode()
    assert "element face 80" in head and "property list uchar int vertex_indices" in head
    write_mesh_ply(path, np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3), np.int32))
    v, c, f = read_mesh_ply(path)
    assert v.shape == (0, 3) and f.shape == (0, 3)


# ------------------------------------------------------------------------------------------------ refusals
def _cpu_maps(V=2, H=4, W=5):
    return {"pose": torch.eye(4).repeat(V, 1, 1), "scale": torch.ones(V, 1), "depth": torch.ones(V, H, W),
            "conf": torch.ones(V, H, W), "intri": torch.eye(3).repeat(V, 1, 1), "images": torch.zeros(V, 3, H, W)}


@pytest.mark.parametrize("change, match", [
    (dict(voxel_size=0.0), "voxel_size"), (dict(voxel_size=float("nan")), "voxel_size"), (dict(trunc=0.41), "trunc"),
    (dict(trunc=0.0), "trunc"), (dict(trunc=-0.1), "trunc"), (dict(min_weight=0), "min_weight"),
    (dict(min_weight=0.5), "min_weight"), (dict(max_bricks=0), "max_bricks"), (dict(max_bricks=2 ** 20 + 1), "max_bricks"),
    (dict(conf_thres=float("inf")), "conf_thres"), (dict(maps_f64=True), "float32"), (dict(maps_bad=True), "images"),
    (dict(maps_many=True), "65535"), ({}, "CUDA device")])
def test_fuse_views_refusals(change, match):
    from vista_slam_b200.fusion import fuse_views
    maps = _cpu_maps()
    if change.pop("maps_f64", False):
        maps["depth"] = maps["depth"].double()
    if change.pop("maps_bad", False):
        maps["images"] = maps["images"][:, :2]
    if change.pop("maps_many", False):
        V = 65536
        maps = {"pose": torch.eye(4).expand(V, 4, 4), "scale": torch.ones(1, 1).expand(V, 1),
                "depth": torch.ones(1, 1, 1).expand(V, 1, 1), "conf": torch.ones(1, 1, 1).expand(V, 1, 1),
                "intri": torch.eye(3).expand(V, 3, 3), "images": torch.zeros(1, 1, 1, 1).expand(V, 3, 1, 1)}
    args = dict(conf_thres=0.5, voxel_size=0.1)
    args.update(change)
    with pytest.raises(ValueError, match=match):
        fuse_views(maps, **args)


@pytest.mark.parametrize("change, match", [
    (dict(voxel_size=0.0), "voxel_size"), (dict(min_weight=0.9), "min_weight"), (dict(bricks=torch.zeros(2, 2)), "bricks"),
    (dict(tsdf=torch.zeros(2, 8, 8, 7)), "tsdf"), (dict(color=torch.zeros(2, 8, 8, 8)), "color"),
    (dict(weight=torch.zeros(2, 8, 8, 8, dtype=torch.float64)), "weight"), ({}, "CUDA device")])
def test_marching_cubes_refusals(change, match):
    from vista_slam_b200.fusion import marching_cubes
    args = dict(bricks=torch.zeros(2, 3, dtype=torch.int32), tsdf=torch.zeros(2, 8, 8, 8), weight=torch.zeros(2, 8, 8, 8),
                color=torch.zeros(2, 8, 8, 8, 3), voxel_size=0.1)
    args.update(change)
    with pytest.raises(ValueError, match=match):
        marching_cubes(**args)


FAKE = ctypes.c_void_p(256)  # never dereferenced: every case is refused before any CUDA call


def _bricks_call(lib, **over):
    a = dict(V=1, H=4, W=4, voxel=0.1, trunc=0.4, cap=0, scratch=FAKE, nbytes=1 << 20, counts=FAKE, keys=None)
    a.update(over)
    return lib.sta_fusion_bricks(FAKE, FAKE, FAKE, FAKE, FAKE, a["V"], a["H"], a["W"], 0.5, a["voxel"], a["trunc"],
                                 a["cap"], a["scratch"], a["nbytes"], a["keys"], a["counts"], None)


def _integrate_call(lib, **over):
    a = dict(V=1, H=4, W=4, B=4, voxel=0.1, trunc=0.4, scratch=FAKE, nbytes=1 << 20, tsdf=FAKE, depth=FAKE)
    a.update(over)
    return lib.sta_fusion_integrate(a["depth"], FAKE, FAKE, FAKE, FAKE, FAKE, a["V"], a["H"], a["W"], 0.5, FAKE, a["B"],
                                    a["voxel"], a["trunc"], a["scratch"], a["nbytes"], a["tsdf"], FAKE, FAKE, None)


def _mesh_call(lib, **over):
    a = dict(B=4, voxel=0.1, mw=1.0, nv=0, nf=0, scratch=FAKE, nbytes=1 << 20, verts=None, counts=FAKE)
    a.update(over)
    return lib.sta_fusion_mesh(FAKE, a["B"], FAKE, FAKE, FAKE, a["voxel"], a["mw"], a["nv"], a["nf"], a["scratch"],
                               a["nbytes"], a["verts"], a["verts"], None, a["counts"], None)


@pytest.mark.parametrize("call, over, match", [
    ("bricks", dict(V=0), b"65535"), ("bricks", dict(H=65536), b"65535"), ("bricks", dict(voxel=0.0), b"voxel"),
    ("bricks", dict(trunc=0.41), b"trunc"), ("bricks", dict(trunc=0.0), b"trunc"), ("bricks", dict(cap=-1), b"capacity"),
    ("bricks", dict(cap=1 << 31), b"capacity"), ("bricks", dict(cap=8), b"null keys_out"),
    ("bricks", dict(counts=None), b"null"), ("bricks", dict(scratch=ctypes.c_void_p(264)), b"misaligned"),
    ("bricks", dict(nbytes=8), b"smaller"), ("bricks", {}, b"device memory"),
    ("integrate", dict(V=0), b"65535"), ("integrate", dict(trunc=0.5), b"trunc"), ("integrate", dict(B=-1), b"brick count"),
    ("integrate", dict(B=(1 << 20) + 1), b"brick count"), ("integrate", dict(depth=None), b"null input"),
    ("integrate", dict(tsdf=None), b"null output"), ("integrate", dict(scratch=None), b"scratch"),
    ("integrate", dict(nbytes=8), b"smaller"), ("integrate", {}, b"device memory"),
    ("mesh", dict(B=-1), b"brick count"), ("mesh", dict(voxel=float("inf")), b"voxel"), ("mesh", dict(mw=0.5), b"min_weight"),
    ("mesh", dict(nv=-1), b"negative"), ("mesh", dict(nv=5), b"null vertex"), ("mesh", dict(counts=None), b"null counts"),
    ("mesh", dict(scratch=ctypes.c_void_p(264)), b"misaligned"), ("mesh", dict(nbytes=8), b"smaller"),
    ("mesh", {}, b"device memory")])
def test_abi_refusals_before_any_cuda_call(call, over, match):
    from vista_slam_b200 import _lib
    lib = _lib.lib()
    fn = {"bricks": _bricks_call, "integrate": _integrate_call, "mesh": _mesh_call}[call]
    assert fn(lib, **over) == 2
    assert match in lib.sta_last_error()
    assert lib.sta_version() == 2


def test_scratch_queries():
    from vista_slam_b200 import _lib
    lib = _lib.lib()
    assert lib.sta_fusion_bricks_scratch_bytes(0, 4, 4, 0) == 0 and lib.sta_fusion_bricks_scratch_bytes(1, 4, 4, -1) == 0
    assert lib.sta_fusion_bricks_scratch_bytes(1, 4, 4, 1000) > lib.sta_fusion_bricks_scratch_bytes(1, 4, 4, 0) > 0
    assert lib.sta_fusion_integrate_scratch_bytes(10, 33) == 144 + 4 * 10 * 2  # dmax [33] padded to 16 bytes, 2 words
    assert lib.sta_fusion_mesh_scratch_bytes(-1) == 0 and lib.sta_fusion_mesh_scratch_bytes(2) > 2 * 512 * 9
    # a 400-view 224 x 224 map fits a few GB even at its worst, 8 distinct bricks for every pixel
    assert lib.sta_fusion_bricks_scratch_bytes(400, 224, 224, 8 * 400 * 224 * 224) < 4.5 * 2 ** 30
