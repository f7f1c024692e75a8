"""CPU: the checkers of tests/test_layers_gpu.py and tests/test_pose_head_gpu.py reject the mis-indexings they are there
to catch.  Each case builds a reference the way the GPU test does, plants one indexing error in a copy of it, and
asserts that the helper the GPU test uses refuses the copy while accepting the reference itself."""
import math

import pytest
import torch

from test_layers_gpu import (EPI_BF16, EPI_PIXSHUF, Layer, _sparse_rows, check_bound, check_exact, conv_cols,
                             make_operands, pixshuf, tau)
from test_pose_head_gpu import check_pose, project64


def _linear_bound(A, W):
    ref = A.double() @ W.double().t()
    S = A.double().abs() @ W.double().abs().t()
    return ref, 2.0 ** -8 * ref.abs() + tau(A.shape[1]) * S


def test_one_tile_row_shifted_by_one_fails_the_float64_bound():
    g = torch.Generator().manual_seed(0)
    A = torch.randn(300, 256, generator=g).bfloat16()
    W = (torch.randn(256, 256, generator=g) / 16).bfloat16()
    ref, bound = _linear_bound(A, W)
    check_bound("reference", ref, ref, bound)
    got = ref.clone()
    got[128 + 16:128 + 32] = ref[128 + 17:128 + 33]  # one 16-row group of the second tile reads the next row
    with pytest.raises(AssertionError):
        check_bound("row shift", got, ref, bound)


def test_two_images_swapped_fails_the_planted_check():
    e = Layer("conv", EPI_BF16, N=64, K=9 * 64, conv=(3, 20, 12, 64))
    o = make_operands(e, "planted", 1, dev="cpu")
    Wp = o["W"].double()
    ref = torch.stack([(conv_cols(o["A"][i:i + 1]) @ Wp.t()).view(20, 12, 64) for i in range(3)])
    check_exact("reference", ref.clone(), ref)
    got = ref[[0, 2, 1]]
    with pytest.raises(AssertionError):
        check_exact("images swapped", got, ref)


def test_one_k_block_dropped_fails_the_planted_check():
    g = torch.Generator().manual_seed(2)
    M, N, K = 200, 256, 768
    A = torch.randint(-2, 3, (M, K), generator=g).float()
    W = _sparse_rows(N, K, g, "cpu")
    ref = A.double() @ W.double().t()
    for kb in (0, 5, K // 64 - 1):
        A2 = A.clone()
        A2[:, kb * 64:(kb + 1) * 64] = 0
        with pytest.raises(AssertionError):
            check_exact("k-block %d dropped" % kb, A2.double() @ W.double().t(), ref)


def test_one_pixel_shuffle_sub_pixel_transposed_fails_the_planted_check():
    e = Layer("act0T", EPI_PIXSHUF, 2 * 3 * 5, 4 * 4 * 128, 128, ps=(4, 128, 2, 3, 5))
    o = make_operands(e, "planted", 3, dev="cpu")
    y = o["A"].double() @ o["W"].double().t()
    ref = pixshuf(y, *e.ps)
    k, cout = 4, 128
    v = y.view(-1, k, k, cout).clone()
    v[:, 1, 2], v[:, 2, 1] = y.view(-1, k, k, cout)[:, 2, 1], y.view(-1, k, k, cout)[:, 1, 2]  # (kh, kw) = (1, 2) <-> (2, 1)
    with pytest.raises(AssertionError):
        check_exact("sub-pixel transposed", pixshuf(v.view(-1, k * k * cout), *e.ps), ref)


def test_pose_with_the_wrong_determinant_sign_is_rejected():
    g = torch.Generator().manual_seed(4)
    q1, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    q2, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    M = (q1 @ torch.diag(torch.tensor([1.0, 0.6, 0.3], dtype=torch.float64)) @ q2).unsqueeze(0)
    ref = project64(M)
    ref.update(t=torch.zeros(1, 3, dtype=torch.float64), err_t=torch.ones(1, 3, dtype=torch.float64),
               conf=torch.full((1,), 0.5, dtype=torch.float64), err_conf=torch.ones(1, dtype=torch.float64),
               dA=torch.full((1,), 1e-6, dtype=torch.float64))
    pose = torch.eye(4, dtype=torch.float64).unsqueeze(0)
    pose[0, :3, :3] = ref["R"][0]
    check_pose("reference", pose, ref["conf"], ref)
    # R = V diag(1, 1, -det(V U^T)) U^T: the projection with the determinant correction of the wrong sign
    A = torch.nn.functional.normalize(M, dim=-1).transpose(-1, -2)
    u, _, vh = torch.linalg.svd(A)
    v = vh.transpose(-1, -2)
    d = -torch.det(v @ u.transpose(-1, -2))
    bad = pose.clone()
    bad[0, :3, :3] = (torch.cat([v[:, :, :2], v[:, :, 2:] * d.view(-1, 1, 1)], 2) @ u.transpose(-1, -2))[0]
    with pytest.raises(AssertionError):
        check_pose("wrong determinant sign", bad, ref["conf"], ref)
    # and with the sign forced into SO(3) by flipping a column: fails the rotation bound instead
    bad2 = pose.clone()
    bad2[0, :3, :3] = bad[0, :3, :3] @ torch.diag(torch.tensor([1.0, -1.0, 1.0], dtype=torch.float64)) * -1
    if math.isclose(float(torch.det(bad2[0, :3, :3])), 1.0, abs_tol=1e-9):
        with pytest.raises(AssertionError):
            check_pose("flipped", bad2, ref["conf"], ref)
