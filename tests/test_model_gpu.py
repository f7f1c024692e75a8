"""GPU: the whole STA path through the module surface -> C ABI -> sm_90a kernels, against the golden vectors
produced by the UNMODIFIED reference (fp32, CPU; tools/make_golden.py) and against the oracle on the same inputs.

Parity protocol (DESIGN.md section 4):
  (1) production precision (bf16 tensor-core operands, fp32 accumulation): bf16 operands cannot meet rtol 1e-3
      against an fp32 reference (SURVEY.md D6), so the bounds are fixed at about twice the deviation of the bf16
      kernels, per output (all four golden cases), for the maximum and the median error, and the
      deviation from fp32 must be statistically the same as that of the oracle run with the same operand precision
      (|cuda - fp32| ~ |emu - fp32|): a kernel bug does not hide inside the bf16 noise floor.
  (2) split-precision parity mode (precision="x3": the same tensor-core kernels with (hi | lo | hi) x (hi | hi | lo)
      operands, ~17 significant bits): north_star's tolerance itself -- pointmaps 1e-3, pose 1e-4 -- against the
      fp32 reference goldens at every size incl. cfg-1 (224x224) and a cfg-2 pair (512x384).
Max-normalised error = max|a-b| / max|b|; median-normalised = median|a-b| / max|b|.
"""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from oracle.sta_oracle import StaOracle, make_images

pytestmark = pytest.mark.gpu

KEYS = {"pts3d_pred": "pts3d", "conf": "conf", "relative_pose": "pose", "relative_pose_conf": "pose_conf"}
CASES = ["pair_64x80", "pair_b2_48x64", "pair_224x224", "pair_384x512"]
# bf16 production mode: bounds on the max-normalised deviation over the four golden cases and both views, about twice
# the deviation of bf16 tensor-core kernels (pts3d / conf / pose / pose_conf).
TOL_EMU = {"pts3d_pred": 3.3e-2, "conf": 2.7e-2, "relative_pose": 3.2e-2, "relative_pose_conf": 4.0e-3}
TOL_FP32 = {"pts3d_pred": 4.7e-2, "conf": 3.1e-2, "relative_pose": 5.4e-2, "relative_pose_conf": 5.8e-3}
# median-normalised, dense outputs only
TOL_MED_FP32 = {"pts3d_pred": 3.4e-3, "conf": 2.2e-3}
# trunk features vs the fp32 reference
TOL_FEAT = {"enc_feat1": 1.6e-2, "dec": 2.0e-2}
# north_star: "pointmaps rtol 1e-3, pose params rtol 1e-4" -- met by the split-precision parity mode
TOL_X3 = {"pts3d_pred": 1e-3, "conf": 1e-3, "relative_pose": 1e-4, "relative_pose_conf": 1e-4}


def maxn(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def medn(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).abs().median() / b.abs().max().clamp_min(1e-30))


def golden_case(case):
    g = np.load(os.path.join(GOLDEN_DIR, case + ".npz"))
    meta = json.loads(str(g["meta"]))
    img1, img2 = make_images(meta["B"], meta["H"], meta["W"], meta["image_seed"])
    if meta.get("bf16_images"):  # cfg-2 feeds bf16 images; the golden was generated from exactly these values
        img1, img2 = img1.bfloat16().float(), img2.bfloat16().float()
    return g, meta, img1, img2


@pytest.mark.parametrize("case", CASES)
def test_forward_pairs_vs_reference_golden_and_oracle(cuda_model, state_dict, case):
    """Production (bf16) precision on every golden: cfg-1 224x224 and one cfg-2 512x384 pair included."""
    g, meta, img1, img2 = golden_case(case)
    main, sup = cuda_model.forward_pairs(img1.cuda(), img2.cuda())
    with torch.no_grad():
        o_main, o_sup = StaOracle(state_dict, emulate_bf16=True).forward_pair(img1, img2)
    for res, orc, pre in ((main, o_main, "main_"), (sup, o_sup, "support_")):
        for k, gk in KEYS.items():
            gold = torch.from_numpy(g[pre + gk])
            e_emu, e_fp32 = maxn(res[k], orc[k]), maxn(res[k], gold)
            assert e_emu < TOL_EMU[k], (pre, k, e_emu)
            assert e_fp32 < TOL_FP32[k], (pre, k, e_fp32)
            if k in TOL_MED_FP32:
                # dense outputs: the deviation from fp32 is the operand-precision noise floor, not more --
                # compare with what the oracle shows at the same operand precision (max and median)
                assert medn(res[k], gold) < TOL_MED_FP32[k], (pre, k)
                assert e_fp32 < 1.6 * maxn(orc[k], gold) + 1e-4, (pre, k, e_fp32, maxn(orc[k], gold))
                assert medn(res[k], gold) < 1.25 * medn(orc[k], gold) + 1e-5, (pre, k)


def test_cfg2_batch16_pair0_is_the_golden_pair(cuda_model):
    """cfg-2 proper: 16 bf16 512x384 pairs in one call -- full-size GEMM grids, 128-row attention tiles,
    full DPT pyramid -- with pair 0 = the pair the unmodified reference was run on."""
    g, meta, img1, img2 = golden_case("pair_384x512")
    H, W = meta["H"], meta["W"]
    o1, o2 = make_images(15, H, W, 99)
    b1 = torch.cat([img1, o1]).bfloat16().cuda()
    b2 = torch.cat([img2, o2]).bfloat16().cuda()
    main, sup = cuda_model.forward_pairs(b1, b2)
    for res, pre in ((main, "main_"), (sup, "support_")):
        for k, gk in KEYS.items():
            gold = torch.from_numpy(g[pre + gk])
            assert maxn(res[k][:1], gold) < TOL_FP32[k], (pre, k, maxn(res[k][:1], gold))
            if k in TOL_MED_FP32:
                assert medn(res[k][:1], gold) < TOL_MED_FP32[k], (pre, k)
    # and the pair's result does not depend on its batch neighbours (same tile route at 8 pairs: bit-identical)
    m8, s8 = cuda_model.forward_pairs(b1[:8], b2[:8])
    assert torch.equal(m8["pts3d_pred"][0], main["pts3d_pred"][0]) and torch.equal(s8["relative_pose"][0], sup["relative_pose"][0])


@pytest.mark.parametrize("case", CASES)
def test_split_precision_mode_meets_north_star_tolerance(cuda_model_x3, case):
    """precision='x3' (the same tensor-core kernels, ~17-bit operands) vs the fp32 reference golden:
    pointmaps 1e-3, pose 1e-4 (BASELINE.json north_star), at every size incl. cfg-1 and a cfg-2 pair."""
    g, meta, img1, img2 = golden_case(case)
    main, sup = cuda_model_x3.forward_pairs(img1.cuda(), img2.cuda())
    for res, pre in ((main, "main_"), (sup, "support_")):
        for k, gk in KEYS.items():
            gold = torch.from_numpy(g[pre + gk])
            e = maxn(res[k], gold)
            assert e < TOL_X3[k], (case, pre, k, e)
    # elementwise, the way the survey measured the reference's own bf16 deviation (SURVEY.md App. D)
    gold = torch.from_numpy(g["main_pts3d"])
    assert torch.allclose(main["pts3d_pred"].cpu(), gold, rtol=1e-3, atol=1e-3 * float(gold.abs().max()) * 1e-1)
    # trunk features through the reference-shaped sub-entry points
    B, H, W = meta["B"], meta["H"], meta["W"]
    ts = torch.tensor([[H, W]] * B)
    f1, p1 = cuda_model_x3._encode_image(img1.cuda(), ts, normalize=False)
    f2, p2 = cuda_model_x3._encode_image(img2.cuda(), ts, normalize=False)
    d1, _ = cuda_model_x3._decode_stereo(f1, f2, p1, p2, layers=(12,))
    assert maxn(f1, torch.from_numpy(g["enc_feat1"])) < 1e-3
    assert maxn(d1[12], torch.from_numpy(g["dec1_12"])) < 1e-3


def test_sub_entry_points_match_reference_golden_and_fused_path(cuda_model):
    """the slam.py call sequence (slam.py:144,162-180): _encode_image -> _decode_stereo -> head_pose_s / head_pts."""
    g = np.load(os.path.join(GOLDEN_DIR, "pair_64x80.npz"))
    meta = json.loads(str(g["meta"]))
    B, H, W = meta["B"], meta["H"], meta["W"]
    img1, img2 = make_images(B, H, W, meta["image_seed"])
    ts = torch.tensor([[H, W]] * B)
    f1, p1 = cuda_model._encode_image(img1.cuda(), ts, normalize=False)
    f2, p2 = cuda_model._encode_image(img2.cuda(), ts, normalize=False)
    assert f1.shape == (B, (H // 16) * (W // 16), 1024) and p1.dtype == torch.int64
    assert torch.equal(p1.cpu(), torch.from_numpy(g["pos1"]))
    assert maxn(f1, torch.from_numpy(g["enc_feat1"])) < TOL_FEAT["enc_feat1"]
    d1, d2 = cuda_model._decode_stereo(f1, f2, p1, p2)
    assert len(d1) == 13 and len(d2) == 13 and d1[0].shape == (B, (H // 16) * (W // 16) + 1, 768)
    for k, t in (("dec1_6", d1[6]), ("dec1_9", d1[9]), ("dec1_12", d1[12]), ("dec2_12", d2[12])):
        assert maxn(t, torch.from_numpy(g[k])) < TOL_FEAT["dec"], k
    pts = cuda_model.head_pts([f1] + [t[:, 1:, :] for t in d1], ts)
    pose = cuda_model.head_pose_s(d1[-1][:, 0, :])
    main, _ = cuda_model.forward_pairs(img1.cuda(), img2.cuda())
    # same kernels, same order -> the decomposed path reproduces the fused one up to the fp32->bf16 hand-over
    assert maxn(pts["pts3d"], main["pts3d_pred"]) < 2e-2
    assert maxn(pose["pose"], main["relative_pose"]) < 5e-3
    out = cuda_model({"main_view": {"img": img1.cuda(), "true_shape": ts},
                      "neighbor_views": [{"img": img2.cuda(), "true_shape": ts}], "loop_views": []})
    assert set(out) == {"main_views", "support_views"}
    assert set(out["main_views"][0]) == {"pts3d_pred", "conf", "relative_pose", "relative_pose_conf"}
    assert out["main_views"][0]["pts3d_pred"].shape == (B, H, W, 3)


def test_pose_is_a_rigid_transform(cuda_model):
    img1, img2 = make_images(3, 64, 96, 5)
    main, sup = cuda_model.forward_pairs(img1.cuda(), img2.cuda())
    for res in (main, sup):
        P = res["relative_pose"].double().cpu()
        R = P[:, :3, :3]
        assert (R @ R.transpose(1, 2) - torch.eye(3, dtype=torch.float64)).abs().max() < 1e-5  # pp.mat2SE3 atol 1e-3
        assert (torch.det(R) - 1).abs().max() < 1e-5
        assert torch.equal(P[:, 3], torch.tensor([[0., 0., 0., 1.]], dtype=torch.float64).expand(3, 4))
        assert ((res["relative_pose_conf"] > 0) & (res["relative_pose_conf"] < 1)).all()
        assert (res["conf"] >= 1).all()


def test_full_size_properties_cfg2(cuda_model):
    """cfg-2 size (16 pairs, 512x384 bf16): size-independent properties -- finiteness, batch invariance (a pair's
    result does not depend on its batch neighbours) and view symmetry (swapping the views swaps the outputs)."""
    B, H, W = 16, 384, 512
    g = torch.Generator().manual_seed(3)
    i1 = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).bfloat16().cuda()
    i2 = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).bfloat16().cuda()
    main, sup = cuda_model.forward_pairs(i1, i2)
    for res in (main, sup):
        assert res["pts3d_pred"].shape == (B, H, W, 3) and torch.isfinite(res["pts3d_pred"]).all()
        assert torch.isfinite(res["relative_pose"]).all()
    again, _ = cuda_model.forward_pairs(i1, i2)
    assert torch.equal(again["pts3d_pred"], main["pts3d_pred"])         # deterministic kernels (no atomics)
    # no cross-pair op: a pair's result does not depend on its batch neighbours.  Bit-identical as long as the same
    # tile route is taken (8 vs 16 pairs); a single pair takes the small-problem route (128-wide tiles, split-K with a
    # fixed but different fp32 summation order), so it agrees to the bf16 rounding level instead.
    m8, s8 = cuda_model.forward_pairs(i1[4:12], i2[4:12])
    assert torch.equal(m8["pts3d_pred"][1], main["pts3d_pred"][5])
    assert torch.equal(s8["relative_pose"][1], sup["relative_pose"][5])
    m1, s1 = cuda_model.forward_pairs(i1[5:6], i2[5:6])
    assert maxn(m1["pts3d_pred"][0], main["pts3d_pred"][5]) < 2e-2
    assert maxn(s1["relative_pose"][0], sup["relative_pose"][5]) < 5e-3
    m2, s2 = cuda_model.forward_pairs(i2, i1)                             # swapped views
    assert torch.equal(m2["pts3d_pred"], sup["pts3d_pred"]) and torch.equal(s2["conf"], main["conf"])


def test_host_entry_point_matches_device_entry_point(cuda_model):
    img1, img2 = make_images(2, 64, 80, 9)
    h1, h2 = img1.bfloat16().pin_memory(), img2.bfloat16().pin_memory()
    out = cuda_model.forward_pairs_host(h1, h2)
    main, sup = cuda_model.forward_pairs(h1.cuda(), h2.cuda())
    assert torch.equal(out["pts3d"][0], main["pts3d_pred"].cpu()) and torch.equal(out["pose"][1], sup["relative_pose"].cpu())


def test_ragged_and_edge_shapes(cuda_model):
    # smallest image (1 token), odd token grids (crop path of refinenet4), portrait batch, B chunking (> 16 pairs)
    for (B, H, W) in ((1, 16, 16), (2, 48, 80), (1, 80, 48), (17, 32, 32)):
        img1, img2 = make_images(B, H, W, 11)
        main, sup = cuda_model.forward_pairs(img1.cuda(), img2.cuda())
        shape = (B, H, W, 3) if W >= H else (B, W, H, 3)  # portrait batches come back transposed to landscape (misc.py:58-61)
        assert main["pts3d_pred"].shape == shape and torch.isfinite(main["pts3d_pred"]).all(), (B, H, W)
    with pytest.raises(AssertionError):
        cuda_model._encode_image(torch.zeros(1, 3, 30, 32, device="cuda"), None, normalize=False)
