"""GPU: the batched keyframe step (SURVEY.md 8(f) rank 1, vista_slam_b200/keyframe.py -> sta_regress_pairs) against
the per-edge call sequence of OnlineSLAM.regress_two_views (slam.py:153-189) issued through the reference-shaped
module methods, against the fused pair path (hence, transitively, the oracle / golden vectors of test_model_gpu.py),
and against the numpy oracle of the pointmap consumers."""
import numpy as np
import pytest
import torch

from oracle import slam_utils_oracle as orc
from oracle.sta_oracle import make_images

pytestmark = pytest.mark.gpu


def maxn(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def test_batched_edges_match_per_edge_reference_sequence(cuda_model):
    from vista_slam_b200.keyframe import KeyframeFrontend
    from vista_slam_b200.utils import slam_utils as su
    H, W = 64, 80
    imgs, _ = make_images(4, H, W, 99)
    ts = torch.tensor([[H, W]])
    kf = KeyframeFrontend(cuda_model)
    for b in range(4):
        assert kf.add_view(imgs[b:b + 1].cuda(), ts) == b
    i, js = 3, [2, 1, 0]
    res = kf.regress_views(i, js)
    assert res["pose"].shape == (3, 4, 4) and res["pts3d"].shape == (2, 3, H, W, 3) and res["intri"].shape == (3, 3, 3)
    grid = torch.cartesian_prod(torch.arange(H // 16), torch.arange(W // 16)).view(1, -1, 2).cuda()
    for e, j in enumerate(js):
        fi, fj = kf.enc_features[i], kf.enc_features[j]
        d_ij, d_ji = cuda_model._decode_stereo(fi, fj, grid, grid)
        pose = cuda_model.head_pose_s(d_ij[-1][:, 0, :])
        r_ij = cuda_model.head_pts([fi] + [t[:, 1:, :] for t in d_ij], ts)
        r_ji = cuda_model.head_pts([fj] + [t[:, 1:, :] for t in d_ji], ts)
        # same kernels on the same operands; batching only changes tile scheduling -> tight bounds
        assert maxn(res["pose"][e:e + 1], pose["pose"]) < 5e-3
        assert maxn(res["pose_conf"][e:e + 1], pose["conf"]) < 2e-3
        assert maxn(res["pts3d"][0, e:e + 1], r_ij["pts3d"]) < 2e-2
        assert maxn(res["pts3d"][1, e:e + 1], r_ji["pts3d"]) < 2e-2
        assert maxn(res["conf"][0, e:e + 1], r_ij["conf"]) < 2e-2
        # pointmap consumers of THIS step's outputs: numpy oracle on the same pointmaps
        pcls = torch.cat([res["pts3d"][0, e:e + 1], res["pts3d"][1, e:e + 1]], dim=0)
        confs = torch.cat([res["conf"][0, e:e + 1], res["conf"][1, e:e + 1]], dim=0)
        K_ref = orc.estimate_intrinsic_from_pts3d(pcls.cpu().numpy(), confs.cpu().numpy(), True)
        assert np.allclose(res["intri"][e].cpu().numpy(), K_ref, rtol=1e-4, atol=1e-4)
        assert torch.equal(res["depths"][:, e], pcls[..., 2])
        assert np.allclose(res["conf_mean"][:, e].cpu().numpy(), confs.reshape(2, -1).double().mean(1).cpu().numpy(),
                           rtol=1e-5)
        assert np.allclose(su.estimate_intrinsic_from_pts3d(pcls, confs, True).cpu().numpy(), K_ref, rtol=1e-4, atol=1e-4)
    # the keyframe path really is graph-replayed (4 encodes of one shape: eager, capture + replay, replay, replay)
    from vista_slam_b200 import _lib
    assert _lib.lib().sta_graph_replays(cuda_model._handle) >= 3
    r2 = kf.regress_views(i, js)   # second use of this (K, H, W): captured and replayed
    r3 = kf.regress_views(i, js)   # replayed
    for k in ("pose", "pts3d", "conf", "intri", "depths"):
        assert torch.equal(r2[k], r3[k]), k            # replays are deterministic
        assert maxn(r2[k], res[k]) < 1e-6, k           # and equal the eager first run
    # K = 1 convenience form keeps the reference's return convention
    pose, pconf, confs, intri, depths = kf.regress_two_views(3, 2)
    assert pose.shape == (1, 4, 4) and confs.shape == (2, H, W) and intri.shape == (3, 3) and depths.shape == (2, H, W)
    assert maxn(pose, res["pose"][0:1]) < 5e-3


def test_keyframe_step_equals_fused_pair_path(cuda_model):
    from vista_slam_b200.keyframe import KeyframeFrontend
    H, W = 48, 64
    img1, img2 = make_images(2, H, W, 5)
    main, sup = cuda_model.forward_pairs(img1.cuda(), img2.cuda())
    ts = torch.tensor([[H, W]])
    for b in range(2):
        kf = KeyframeFrontend(cuda_model)
        kf.add_view(img1[b:b + 1].cuda(), ts)
        kf.add_view(img2[b:b + 1].cuda(), ts)
        r = kf.regress_views(0, [1])
        assert maxn(r["pts3d"][0], main["pts3d_pred"][b:b + 1]) < 2e-2
        assert maxn(r["pts3d"][1], sup["pts3d_pred"][b:b + 1]) < 2e-2
        assert maxn(r["pose"], main["relative_pose"][b:b + 1]) < 5e-3
        assert maxn(r["pose_ji"], sup["relative_pose"][b:b + 1]) < 5e-3


def test_keyframe_step_vs_oracle_on_the_cached_features(cuda_model, state_dict):
    """Oracle parity of sta_regress_pairs (not just self-consistency): the cached encoder features go through the oracle's
    decode_stereo / head_pts / head_pose on the CPU (bf16-operand emulation) and are compared with the batched step."""
    from oracle.sta_oracle import StaOracle, token_positions
    from test_model_gpu import TOL_EMU
    from vista_slam_b200.keyframe import KeyframeFrontend
    H, W = 64, 80
    imgs, _ = make_images(3, H, W, 123)
    ts = torch.tensor([[H, W]])
    kf = KeyframeFrontend(cuda_model)
    for b in range(3):
        kf.add_view(imgs[b:b + 1].cuda(), ts)
    i, js = 2, [1, 0]
    res = kf.regress_views(i, js)
    orc = StaOracle(state_dict, emulate_bf16=True)
    pos = token_positions(1, H // 16, W // 16)
    for e, j in enumerate(js):
        fi, fj = kf.enc_features[i].cpu(), kf.enc_features[j].cpu()
        with torch.no_grad():
            d_ij, d_ji = orc.decode_stereo(fi, fj, pos, pos)
            pose = orc.head_pose(d_ij[-1][:, 0, :])
            r_ij = orc.head_pts([fi] + [t[:, 1:, :] for t in d_ij], H, W)
            r_ji = orc.head_pts([fj] + [t[:, 1:, :] for t in d_ji], H, W)
        assert maxn(res["pose"][e:e + 1], pose["pose"]) < TOL_EMU["relative_pose"]
        assert maxn(res["pose_conf"][e:e + 1], pose["conf"]) < TOL_EMU["relative_pose_conf"]
        assert maxn(res["pts3d"][0, e:e + 1], r_ij["pts3d"]) < TOL_EMU["pts3d_pred"]
        assert maxn(res["pts3d"][1, e:e + 1], r_ji["pts3d"]) < TOL_EMU["pts3d_pred"]
        assert maxn(res["conf"][0, e:e + 1], r_ij["conf"]) < TOL_EMU["conf"]
        assert maxn(res["conf"][1, e:e + 1], r_ji["conf"]) < TOL_EMU["conf"]
        # (the intrinsics of these random-weight pointmaps are ill-conditioned -- focal ~ 1e-3 -- so they are compared on
        # IDENTICAL pointmaps in the test above, not across the two implementations)


def test_gated_keyframe_step_keeps_the_reference_early_out(cuda_model):
    """slam.py:169-170: an edge with rel_pose_conf < thres that is not the immediate neighbour (i - j != 1) is rejected
    BEFORE the DPT heads.  The gated batched step must (a) return None for exactly those edges, (b) give the kept edges
    the same results as the ungated batch, with one host synchronisation for the whole keyframe."""
    from vista_slam_b200.keyframe import KeyframeFrontend
    H, W = 64, 80
    imgs, _ = make_images(5, H, W, 321)
    ts = torch.tensor([[H, W]])
    kf = KeyframeFrontend(cuda_model)
    for b in range(5):
        kf.add_view(imgs[b:b + 1].cuda(), ts)
    i, js = 4, [3, 2, 1, 0]
    full = kf.regress_views(i, js)
    confs = full["pose_conf"].cpu()
    # threshold between the candidates' confidences: rejects some non-neighbour edges, keeps others
    order = sorted(float(c) for c in confs[1:])
    thres = 0.5 * (order[0] + order[1]) if order[0] != order[1] else order[0] + 1e-6
    out = kf.regress_views_gated(i, js, thres)
    assert len(out) == 4
    n_rej = 0
    for e, j in enumerate(js):
        pose, pconf, cf, intri, depths = out[e]
        assert torch.equal(pose[0], full["pose"][e]) and torch.equal(pconf[0], full["pose_conf"][e])
        rejected = float(confs[e]) < thres and i - j != 1
        if rejected:
            n_rej += 1
            assert cf is None and intri is None and depths is None
        else:
            # same kernels on the same decoder hooks; only the DPT batch composition differs
            assert maxn(cf, full["conf"][:, e]) < 2e-2
            assert maxn(depths, full["depths"][:, e]) < 2e-2
            assert maxn(intri, full["intri"][e]) < 2e-2
    assert 1 <= n_rej <= 2
    # everything rejected except the immediate neighbour (which the reference always keeps)
    out = kf.regress_views_gated(i, js, 2.0)
    assert out[0][2] is not None and all(o[2] is None for o in out[1:])
    # nothing rejected == the ungated batch, bit for bit (same tile routes)
    out = kf.regress_views_gated(i, js, -1.0)
    for e in range(4):
        assert torch.equal(out[e][2], full["conf"][:, e]) and torch.equal(out[e][4], full["depths"][:, e])


def test_gated_finish_after_another_call_is_refused(cuda_model):
    """sta_regress_pairs_finish reads the decoder hooks _begin left in the workspace.  An encode of the same image size
    in between carves that workspace again (without reallocating it), so _finish must refuse instead of running the DPT
    heads on overwritten hooks."""
    import ctypes
    from vista_slam_b200 import _lib
    from vista_slam_b200.keyframe import KeyframeFrontend
    H, W = 64, 80
    imgs, _ = make_images(3, H, W, 7)
    ts = torch.tensor([[H, W]])
    kf = KeyframeFrontend(cuda_model)
    for b in range(3):
        kf.add_view(imgs[b:b + 1].cuda(), ts)
    L, h = _lib.lib(), cuda_model._handle
    f32 = dict(device="cuda", dtype=torch.float32)
    fi, fj = torch.cat(kf.enc_features[:2]), torch.cat(kf.enc_features[1:])
    pose, pconf = torch.empty(2, 2, 4, 4, **f32), torch.empty(2, 2, **f32)
    pts, conf = torch.empty(2, 2, H, W, 3, **f32), torch.empty(2, 2, H, W, **f32)
    idx = (ctypes.c_int * 2)(0, 1)

    def begin():
        _lib.check(L.sta_regress_pairs_begin(h, _lib.ptr(fi), _lib.ptr(fj), 2, H, W, _lib.ptr(pose), _lib.ptr(pconf),
                                             _lib.cur_stream()), "sta_regress_pairs_begin")

    def finish():
        return L.sta_regress_pairs_finish(h, idx, 2, _lib.ptr(pts), _lib.ptr(conf), None, None, None, None,
                                          _lib.cur_stream())

    begin()
    assert finish() == 0
    begin()
    cuda_model._encode_image(imgs[:1].cuda(), ts, normalize=False)
    with pytest.raises(RuntimeError, match="sta_regress_pairs_begin"):
        _lib.check(finish(), "sta_regress_pairs_finish")
    torch.cuda.synchronize()
