"""CPU: the numpy restatement of the SLAM evaluation (oracle/eval_oracle.py) on planted answers and against the unmodified
reference's record (tests/golden/eval.npz, tools/make_golden_eval.py), and the import hygiene of the drop-in modules.

Bounds: the oracle and the golden run the same float64 arithmetic on the same scene, so counts and the ICP iteration
count are equal and floats agree to 1e-12."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, ROOT
from oracle import eval_oracle as eo


def _rot(axis, ang):
    return eo._rot(axis, ang)


def test_umeyama_recovers_a_planted_sim3_and_refuses_degenerate_input():
    rng = np.random.default_rng(1)
    x = rng.standard_normal((3, 40))
    R, t, s = _rot([0.3, -1, 0.4], 1.1), np.array([0.5, -2.0, 1.0]), 1.7
    r, tt, c = eo.umeyama(x, s * R.dot(x) + t[:, None], True)
    np.testing.assert_allclose(r, R, atol=1e-12)
    np.testing.assert_allclose(tt, t, atol=1e-12)
    assert abs(c - s) < 1e-12
    # a reflection in the data: the fit stays a rotation
    y = np.diag([1.0, 1.0, -1.0]).dot(x)
    r, _, _ = eo.umeyama(x, y, True)
    assert abs(np.linalg.det(r) - 1) < 1e-12
    with pytest.raises(ValueError):
        eo.umeyama(np.ones((3, 5)), np.ones((3, 5)), True)  # every position the same: rank 0


def test_align_traj_skips_non_finite_poses_and_ape_statistics():
    n = 6
    ref = np.tile(np.eye(4), (n, 1, 1))
    ref[:, :3, 3] = np.random.default_rng(0).standard_normal((n, 3))
    est = ref.copy()
    ref[2, 0, 0] = np.nan
    r, t, s, al, rf = eo.align_traj(est, ref)
    assert len(al) == n - 1 and abs(s - 1) < 1e-12
    err = np.array([0.0, 3.0, 4.0])
    a = np.tile(np.eye(4), (3, 1, 1))
    b = a.copy()
    b[:, 0, 3] = err
    st = eo.ape_statistics(a, b)
    assert st["sse"] == 25.0 and st["max"] == 4.0 and st["min"] == 0.0 and st["median"] == 3.0
    assert abs(st["rmse"] - np.sqrt(25 / 3)) < 1e-15 and abs(st["mean"] - 7 / 3) < 1e-15


def test_voxel_down_sample_on_hand_built_clouds():
    v = 0.5
    # min_bound = (-1.25, ...): -1.0 and -0.76 share voxel 0, -0.75 starts voxel 1 (the boundary belongs to the upper one)
    p = np.array([[-1.0, 0, 0], [0.26, 0, 0], [-0.76, 0, 0], [-0.75, 0, 0], [0.3, 0, 0]])
    out = eo.voxel_down(p, v)
    np.testing.assert_array_equal(out[:, 0], [(-1.0 + -0.76) / 2, -0.75, (0.26 + 0.3) / 2])
    one = eo.voxel_down(np.array([[3.0, -2.0, 1.0]]), v)  # a single point is its own voxel
    np.testing.assert_array_equal(one, [[3.0, -2.0, 1.0]])
    with pytest.raises(ValueError, match="too small"):
        eo.voxel_down(np.array([[0.0, 0, 0], [1e9, 0, 0]]), 1e-9)
    with pytest.raises(ValueError):
        eo.voxel_down(p, 0.0)


def _room_cloud():
    sc = eo.make_scene(n_views=8, H=24, W=32, seed=5, nan_view=-1)
    gt, _ = eo.clouds(torch.from_numpy(sc["gt_depths"]), torch.from_numpy(sc["gt_poses"]), torch.from_numpy(sc["gt_intrinsics"]),
                      torch.from_numpy(sc["gt_depths"]), torch.from_numpy(sc["gt_poses"]),
                      torch.from_numpy(np.repeat(sc["gt_intrinsics"][None], 8, 0)), torch.ones(8, 24, 32))
    return eo.voxel_down(gt, 0.05)


def test_icp_recovers_a_planted_rigid_motion_and_stops():
    dst = _room_cloud()
    M = np.eye(4)
    M[:3, :3], M[:3, 3] = _rot([1, 2, 3], np.deg2rad(0.5)), [0.01, -0.008, 0.005]
    src = eo.transform(dst, np.linalg.inv(M))
    r = eo.icp(src, dst, max_iter=100, eps=0.0)
    np.testing.assert_allclose(r["transformation"], M, atol=1e-9)
    assert r["fitness"] == 1.0
    r = eo.icp(src, dst)
    assert 1 < r["iterations"] < 30
    far = eo.icp(src + 100.0, dst)
    assert far["iterations"] == 1 and far["fitness"] == 0.0 and far["inlier_rmse"] == 0.0
    np.testing.assert_array_equal(far["transformation"], np.eye(4))


def test_chamfer_clips_a_far_outlier_at_half():
    ref = np.zeros((1, 3))
    ch, r1, r2, d1, d2 = eo.chamfer(ref, np.array([[0.0, 0.0, 0.0], [10.0, 0.0, 0.0]]))
    np.testing.assert_array_equal(d1, [0.0, 0.5])
    assert r1 == np.sqrt(0.125) and r2 == 0.0 and ch == 0.5 * r1


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN_DIR, "eval.npz")))


@pytest.fixture(scope="module")
def scene_dir():
    with tempfile.TemporaryDirectory() as d:
        eo.write_scene(eo.make_scene(), d)
        yield d


def test_oracle_equals_reference_golden(golden, scene_dir):
    g = golden
    est = list(np.load(os.path.join(scene_dir, "trajectory.npy")))
    ref = list(np.load(os.path.join(scene_dir, "gt_poses.npy")))
    _, _, r, t, s, st = eo.full_traj_eval(est, ref)
    np.testing.assert_allclose(r, g["r_a"], atol=1e-12, rtol=0)
    np.testing.assert_allclose(t, g["t_a"], atol=1e-12, rtol=0)
    assert abs(s - g["s"]) < 1e-12
    for k, v in st.items():
        assert abs(v - g["ape_" + k]) < 1e-12, k
    for tag, rel in (("", [r, t, s]), ("self_", None)):
        o, gt, e = eo.eval_recon_from_saved_data(scene_dir, rel)
        assert len(gt) == g[tag + "n_gt"] and len(e) == g[tag + "n_est"]
        assert o["icp"]["iterations"] == g[tag + "icp_iterations"]
        assert abs(o["icp"]["fitness"] - g[tag + "icp_fitness"]) < 1e-12
        np.testing.assert_allclose(o["icp"]["transformation"], g[tag + "icp_transformation"], atol=1e-12, rtol=0)
        for k in ("rmse_acc", "rmse_comp", "chamfer"):
            assert abs(o[k] - g[tag + k]) < 1e-12, k
    # the scene exercises what the golden pins: outliers clip at 0.5, holes, a skipped pose, conf on both sides
    assert 0 < g["n_est"] < g["n_gt"] and g["icp_iterations"] > 1


def test_make_golden_eval_regenerates_the_golden(tmp_path, golden):
    if not os.path.isdir("/root/reference/vista_slam"):
        pytest.skip("the reference tree is not present")
    out = tmp_path / "eval.npz"
    subprocess.run([sys.executable, os.path.join(ROOT, "tools", "make_golden_eval.py"), str(out)], check=True, capture_output=True)
    new = np.load(out)
    assert sorted(new.files) == sorted(golden)
    for k in golden:
        assert new[k].dtype == golden[k].dtype and new[k].shape == golden[k].shape, k
        assert new[k].tobytes() == golden[k].tobytes(), k


def test_eval_modules_import_without_evo_open3d_pykdtree_munch_matplotlib():
    code = ("import sys\n"
            "mods = ('evo', 'open3d', 'pykdtree', 'munch', 'matplotlib')\n"
            "for m in mods:\n"
            "    sys.modules[m] = None  # any import of them raises\n"
            "import vista_slam_b200.eval.eval_traj as t, vista_slam_b200.eval.eval_recon as r\n"
            "assert t.full_traj_eval and t.align_traj and t.traj_eval_and_plot\n"
            "assert r.load_data and r.transform_to_world_coordinates and r.chamfer_distance_RMSE and r.eval_recon\n"
            "assert r.eval_recon_from_saved_data\n"
            "assert not any(sys.modules.get(m) is not None for m in mods)\n")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=ROOT)


def test_drop_in_trajectory_eval_equals_golden(golden, scene_dir, tmp_path):
    from vista_slam_b200.eval.eval_traj import full_traj_eval
    est = list(np.load(os.path.join(scene_dir, "trajectory.npy")))
    ref = list(np.load(os.path.join(scene_dir, "gt_poses.npy")))
    al, rf, r, t, s, st = full_traj_eval(est, ref, str(tmp_path / "plots"), "traj")
    assert os.path.isdir(tmp_path / "plots") and al.shape == rf.shape == (len(est) - 1, 4, 4) and al.dtype == np.float64
    np.testing.assert_allclose(r, golden["r_a"], atol=1e-12, rtol=0)
    np.testing.assert_allclose(t, golden["t_a"], atol=1e-12, rtol=0)
    assert abs(s - golden["s"]) < 1e-12
    assert all(abs(st[k] - golden["ape_" + k]) < 1e-12 for k in st)
    with pytest.raises(ValueError):
        full_traj_eval([np.eye(4)] * 3, [np.eye(4)] * 3, str(tmp_path), "x")


def test_recon_symbols_are_exported():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    for name in ("sta_op_radix_sort", "sta_eval_clouds", "sta_voxel_down", "sta_nn_create", "sta_nn_query", "sta_nn_destroy",
                 "sta_op_moments", "sta_icp_moments", "sta_transform_points", "sta_sum_sq_clipped"):
        assert hasattr(L, name), name
    assert L.sta_version() == 2
