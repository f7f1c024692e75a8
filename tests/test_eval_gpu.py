"""GPU: the reconstruction evaluation kernels (csrc/recon.cu) and the drop-in eval modules against numpy, the oracle
(oracle/eval_oracle.py) and the reference's golden (tests/golden/eval.npz).

Bounds: the sort, counts, point order, voxel points and nearest-neighbour distances are exact (the device computes the
same correctly rounded operations in a fixed order); cKDTree computes its own distances, so it is within 1 ulp.  ICP
sums its moments in another order than numpy: transformations to 1e-9.  The clouds are unprojected in fp32 with K^-1
from the fp64 adjugate where torch inverts in fp32: points within 8 fp32 ulps of the point's largest coordinate, and the
whole-function metrics to 1e-5 relative."""
import os
import tempfile

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import eval_oracle as eo

pytestmark = pytest.mark.gpu


def _lib():
    from vista_slam_b200 import _lib
    return _lib


def _sort(keys, nbits, idx=None):
    L = _lib()
    n = len(keys)
    k = torch.as_tensor(keys.view(np.int64)).cuda()
    i = None if idx is None else torch.as_tensor(idx.astype(np.int32)).cuda()
    ko, io = torch.empty_like(k), torch.empty(n, dtype=torch.int32, device="cuda")
    s = torch.empty(int(L.lib().sta_sort_scratch_bytes(n)) // 8 + 2, dtype=torch.int64, device="cuda")
    L.check(L.lib().sta_op_radix_sort(L.ptr(k), L.ptr(i), n, nbits, L.ptr(ko), L.ptr(io), L.ptr(s), L.cur_stream()))
    return ko.cpu().numpy().view(np.uint64), io.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("n,nbits", [(0, 8), (1, 1), (4097, 1), (4097, 63), (100003, 17), (1 << 25, 40), (77777, 64)])
def test_radix_sort_is_stable_and_equals_numpy(n, nbits):
    rng = np.random.default_rng(n + nbits)
    hi = np.uint64((1 << nbits) - 1) if nbits < 64 else np.uint64(2 ** 64 - 1)
    keys = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n, dtype=np.uint64)
    keys &= hi
    if n > 10:
        keys[::3] = keys[0]  # many duplicates
    ko, io = _sort(keys, nbits)
    want = np.argsort(keys, kind="stable")
    np.testing.assert_array_equal(io, want)
    np.testing.assert_array_equal(ko, keys[want])


def test_radix_sort_sorts_only_the_low_bits_and_carries_indices():
    keys = np.array([0x100 + 3, 2, 0x200 + 3, 1], np.uint64)
    ko, io = _sort(keys, 8, idx=np.array([10, 11, 12, 13]))
    np.testing.assert_array_equal(io, [13, 11, 10, 12])


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN_DIR, "eval.npz")))


@pytest.fixture(scope="module")
def scene_dir():
    with tempfile.TemporaryDirectory() as d:
        eo.write_scene(eo.make_scene(), d)
        yield d


def _gpu_clouds(folder):
    from vista_slam_b200.eval import eval_recon as R
    d = R.load_data(folder, load_view_graph=False)
    return R.world_clouds(d.gt_depths, d.gt_poses, d.gt_intrinsic, d.unscaled_depths, d.scales.reshape(-1), d.poses,
                          d.intrinsics, d.confs, d.conf_thres)


def _torch_clouds(folder):
    d = eo.load(folder)
    return eo.clouds(torch.from_numpy(d["gt_depths"]), torch.from_numpy(d["gt_poses"]), torch.from_numpy(d["gt_intrinsic"]),
                     torch.from_numpy(d["unscaled_depths"] * d["scales"]), torch.from_numpy(d["poses"]),
                     torch.from_numpy(d["intrinsics"]), torch.from_numpy(d["confs"] > d["conf_thres"]).float())


def _assert_close_f32(got, want, ulps=8):
    scale = np.abs(want).max(axis=1, keepdims=True)
    assert (np.abs(got - want) <= ulps * np.spacing(scale.astype(np.float32)).astype(np.float64)).all()


def test_clouds_counts_order_and_points(scene_dir, golden):
    gt, est = _gpu_clouds(scene_dir)
    tg, te = _torch_clouds(scene_dir)
    assert len(gt) == len(tg) == golden["n_gt"] and len(est) == len(te) == golden["n_est"]
    _assert_close_f32(gt.cpu().numpy(), tg.astype(np.float64))
    _assert_close_f32(est.cpu().numpy(), te.astype(np.float64))


def test_voxel_downsampling_is_bit_exact_with_the_oracle(scene_dir):
    from vista_slam_b200.eval import eval_recon as R
    gt, est = _gpu_clouds(scene_dir)
    for p in (gt, est):
        np.testing.assert_array_equal(R.voxel_down_sample(p, 0.05).cpu().numpy(), eo.voxel_down(p.cpu().numpy(), 0.05))
    # 20 M points over a wide range, with negative coordinates and far outliers
    rng = np.random.default_rng(7)
    big = torch.from_numpy(rng.uniform(-30, 20, size=(20_000_000, 3))).cuda()
    big[:100] *= 1e4
    np.testing.assert_array_equal(R.voxel_down_sample(big, 0.05).cpu().numpy(), eo.voxel_down(big.cpu().numpy(), 0.05))
    # keys wider than 64 bits take the two-pass path
    wide = torch.tensor([[0.0, 0.0, 0.0], [1e6, 1e6, 1e6], [0.01, 0.0, 0.0], [1e6, 1e6 + 0.01, 1e6]], dtype=torch.float64).cuda()
    np.testing.assert_array_equal(R.voxel_down_sample(wide, 1e-3).cpu().numpy(), eo.voxel_down(wide.cpu().numpy(), 1e-3))


def _brute(ref, q, r):
    d2 = ((q[:, None, 0] - ref[None, :, 0]) ** 2 + (q[:, None, 1] - ref[None, :, 1]) ** 2) + (q[:, None, 2] - ref[None, :, 2]) ** 2
    j = d2.argmin(axis=1)
    best = d2[np.arange(len(q)), j]
    ok = best < r * r
    return np.where(ok, np.sqrt(best), r), np.where(ok, j, -1)


@pytest.mark.parametrize("radius", [0.1, 0.5])
def test_nearest_neighbour_is_exact_against_brute_force(radius):
    from vista_slam_b200.eval.eval_recon import NnIndex
    rng = np.random.default_rng(3)
    for n, m in ((1, 5), (33, 100), (20000, 3000)):
        ref = rng.uniform(-1, 1, size=(n, 3))
        if n > 100:
            ref[:50] = ref[50:100]  # duplicates
            ref[-3:] = [[1e6, 0, 0], [-1e5, 3e5, 0], [0, 0, 7e4]]  # outliers stretch the Morton box
        q = np.concatenate([rng.uniform(-1.2, 1.2, size=(m, 3)), ref[:7]])  # some queries equal a point
        d, j = NnIndex(torch.from_numpy(ref).cuda()).query(torch.from_numpy(q).cuda(), radius)
        bd, bj = _brute(ref, q, radius)
        np.testing.assert_array_equal(d.cpu().numpy(), bd)
        dj = j.cpu().numpy()
        np.testing.assert_array_equal(dj >= 0, bj >= 0)
        ok = dj >= 0
        np.testing.assert_array_equal(eo.dist2(q[ok], ref[dj[ok]]), eo.dist2(q[ok], ref[bj[ok]]))  # ties: any index
        k = min(n, 7)
        assert (d.cpu().numpy()[-k:] == 0).all()


def test_nearest_neighbour_at_5m_points_within_one_ulp_of_ckdtree():
    from scipy.spatial import cKDTree
    from vista_slam_b200.eval.eval_recon import NnIndex
    rng = np.random.default_rng(11)
    ref = rng.normal(size=(5_000_000, 3)) * [3.0, 2.0, 1.0]
    ref[:1000] = ref[1000:2000]
    ref[-20:] *= 1e4
    q = rng.normal(size=(1_000_000, 3)) * [3.0, 2.0, 1.0]
    d, _ = NnIndex(torch.from_numpy(ref).cuda()).query(torch.from_numpy(q).cuda(), 0.5)
    want = np.minimum(cKDTree(ref).query(q, workers=-1)[0], 0.5)
    got = d.cpu().numpy()
    assert (np.abs(got - want) <= np.spacing(want)).all()


def test_nearest_neighbour_in_an_empty_cloud_is_clipped():
    from vista_slam_b200.eval.eval_recon import NnIndex
    d, j = NnIndex(torch.zeros(0, 3, dtype=torch.float64).cuda()).query(torch.ones(5, 3, dtype=torch.float64).cuda(), 0.5)
    assert (d.cpu().numpy() == 0.5).all() and (j.cpu().numpy() == -1).all()


def test_moments_against_numpy():
    L = _lib()
    rng = np.random.default_rng(2)
    src, dst = rng.normal(size=(5000, 3)), rng.normal(size=(700, 3))
    corr = rng.integers(-1, 700, size=5000)
    s, t, c = (torch.from_numpy(a).cuda() for a in (src, dst, corr))
    out = torch.empty(17, dtype=torch.float64, device="cuda")
    scr = torch.empty(int(L.lib().sta_reduce_scratch_bytes()) // 8 + 2, dtype=torch.float64, device="cuda")
    L.check(L.lib().sta_op_moments(L.ptr(s), L.ptr(t), L.ptr(c), 5000, L.ptr(out), L.ptr(scr), L.cur_stream()))
    o = out.cpu().numpy()
    m = corr >= 0
    x, y = src[m], dst[corr[m]]
    assert o[0] == m.sum()
    np.testing.assert_allclose(o[1], eo.dist2(x, y).sum(), rtol=1e-12)
    np.testing.assert_allclose(o[2:5], x.sum(0), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(o[5:8], y.sum(0), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(o[8:].reshape(3, 3), (y - y.mean(0)).T.dot(x - x.mean(0)), rtol=1e-10, atol=1e-10)


def test_icp_on_the_gpus_downsampled_clouds_matches_the_oracle(scene_dir, golden):
    from vista_slam_b200.eval import eval_recon as R
    gt, est = _gpu_clouds(scene_dir)
    R.transform_points_(est, eo.initial_alignment(golden["r_a"], golden["t_a"], golden["s"]))
    ed, gd = R.voxel_down_sample(est, 0.05), R.voxel_down_sample(gt, 0.05)
    got = R.registration_icp(ed, gd, 0.1)
    want = eo.icp(ed.cpu().numpy(), gd.cpu().numpy())
    assert got["iterations"] == want["iterations"] == golden["icp_iterations"]
    assert got["fitness"] == want["fitness"]
    np.testing.assert_allclose(got["transformation"], want["transformation"], atol=1e-9, rtol=0)
    far = R.registration_icp(ed[:50] + 100.0, gd, 0.1)
    assert far["iterations"] == 1 and far["fitness"] == 0.0
    np.testing.assert_array_equal(far["transformation"], np.eye(4))


def test_whole_functions_on_the_golden_scene(scene_dir, golden, tmp_path):
    from vista_slam_b200.eval.eval_recon import eval_recon_from_saved_data
    from vista_slam_b200.eval.eval_traj import full_traj_eval
    est = list(np.load(os.path.join(scene_dir, "trajectory.npy")))
    ref = list(np.load(os.path.join(scene_dir, "gt_poses.npy")))
    _, _, r, t, s, st = full_traj_eval(est, ref, str(tmp_path), "traj")
    np.testing.assert_allclose(r, golden["r_a"], atol=1e-9, rtol=0)
    np.testing.assert_allclose(t, golden["t_a"], atol=1e-9, rtol=0)
    assert abs(s - golden["s"]) < 1e-9 and all(abs(st[k] - golden["ape_" + k]) < 1e-9 for k in st)
    for tag, rel in (("", [r, t, s]), ("self_", None)):
        acc, comp, ch, gp, ep = eval_recon_from_saved_data(scene_dir, rel_est_gt=rel)
        assert gp.dtype == ep.dtype == torch.float64 and gp.is_cuda and gp.shape == (golden[tag + "n_gt"], 3)
        for k, v in (("rmse_acc", acc), ("rmse_comp", comp), ("chamfer", ch)):
            assert abs(v - golden[tag + k]) <= 1e-5 * golden[tag + k], (k, v, golden[tag + k])
    # two runs are bit-identical
    again = eval_recon_from_saved_data(scene_dir, rel_est_gt=[r, t, s])
    first = eval_recon_from_saved_data(scene_dir, rel_est_gt=[r, t, s])
    assert again[:3] == first[:3] and torch.equal(again[4], first[4])


def test_eval_recon_with_tensors_and_the_refusals(scene_dir, golden):
    from vista_slam_b200 import _lib as L
    from vista_slam_b200.eval import eval_recon as R
    d = eo.load(scene_dir)
    args = [torch.from_numpy(d["gt_depths"]), torch.from_numpy(d["gt_poses"]), torch.from_numpy(d["gt_intrinsic"]),
            torch.from_numpy(d["unscaled_depths"] * d["scales"]), torch.from_numpy(d["poses"]), torch.from_numpy(d["intrinsics"]),
            torch.from_numpy(d["confs"] > d["conf_thres"]).float(), golden["r_a"], golden["t_a"], golden["s"]]
    acc, comp, ch, _, _ = R.eval_recon(*args)
    assert abs(ch - golden["chamfer"]) <= 1e-5 * golden["chamfer"]
    bad = list(args)
    bad[2] = bad[2].double()
    with pytest.raises(TypeError, match="float32"):
        R.eval_recon(*bad)
    bad = list(args)
    bad[5] = bad[5][:-1]
    with pytest.raises(ValueError, match="shape"):
        R.world_clouds(*bad[:4], None, *bad[4:7], 0.5)
    with pytest.raises(RuntimeError, match="too small"):
        R.voxel_down_sample(torch.tensor([[0.0, 0, 0], [1e9, 0, 0]], dtype=torch.float64), 1e-9)
    with pytest.raises(RuntimeError, match="voxel_size <= 0"):
        R.voxel_down_sample(torch.zeros(3, 3, dtype=torch.float64), 0.0)
    host = torch.zeros(4, 3, dtype=torch.float64)
    out = torch.zeros(4, 3, dtype=torch.float64, device="cuda")
    cnt = __import__("ctypes").c_int64()
    assert L.lib().sta_voxel_down(L.ptr(host), 4, 0.05, L.ptr(out), cnt, L.ptr(out), None) == 2
    assert b"device memory" in L.lib().sta_last_error()


def test_end_to_end_online_slam_then_both_evaluations(cuda_model, tmp_path):
    """12 keyframes at 224 x 224 through the drop-in OnlineSLAM (synthetic checkpoint), save_data_all with ground truth,
    then both drop-in evaluations against the oracle on the same files."""
    import vista_slam_b200.slam as S
    from vista_slam_b200.eval.eval_recon import eval_recon_from_saved_data
    from vista_slam_b200.eval.eval_traj import full_traj_eval

    class Run(S.OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return cuda_model

    slam = Run("unused", os.path.join(GOLDEN_DIR, "loop_vocab.txt"), loop_dist_min=4, pgo_every=5, rel_pose_thres=0.5)
    g = torch.Generator().manual_seed(3)
    H = W = 224
    base = torch.rand(1, 3, H // 8, W // 8, generator=g)
    n = 12
    for i in range(n):
        img = torch.nn.functional.interpolate(base.roll(i, dims=3), size=(H, W), mode="bilinear") * 2 - 1
        img = (img + 0.05 * torch.rand(1, 3, H, W, generator=g)).clamp(-1, 1).cuda()
        gray = ((img[0].mean(0) + 1) / 2).contiguous()
        slam.step({"rgb": img, "shape": torch.tensor([[H, W]]), "gray": gray, "view_name": "%d" % i}, force_pgo=(i == n - 1))
    est_poses = [slam.get_view(i, return_depth=False, return_intri=False).pose.numpy() for i in range(n)]
    scene = eo.make_scene(n_views=n, H=H, W=W, seed=4, nan_view=-1)
    gt_poses = list(scene["gt_poses"])
    # ground-truth positions planted as a Sim(3) of the estimate's, so the alignment is well posed
    for i in range(n):
        gt_poses[i] = gt_poses[i].copy()
        gt_poses[i][:3, 3] = 0.7 * est_poses[i][:3, 3] + [0.1, 0.2, 0.3] + 0.01 * np.sin(i)
    out = str(tmp_path / "run")
    slam.save_data_all(out, gt_poses=gt_poses, gt_depths=list(scene["gt_depths"]), gt_intrinsics=scene["gt_intrinsics"])
    _, _, r, t, s, st = full_traj_eval(est_poses, gt_poses, out, "traj")
    _, _, ro, to, so, sto = eo.full_traj_eval(est_poses, gt_poses)
    np.testing.assert_allclose(r, ro, atol=1e-9)
    assert abs(s - so) < 1e-9 and abs(st["rmse"] - sto["rmse"]) < 1e-9
    acc, comp, ch, gp, ep = eval_recon_from_saved_data(out, rel_est_gt=[r, t, s])
    o, ogt, oest = eo.eval_recon_from_saved_data(out, [r, t, s], workers=-1)
    assert len(gp) == len(ogt) and len(ep) == len(oest)
    for k, v in (("rmse_acc", acc), ("rmse_comp", comp), ("chamfer", ch)):
        assert abs(v - o[k]) <= 1e-5 * max(o[k], 1e-12), (k, v, o[k])
