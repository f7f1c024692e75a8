"""CPU: the FP8 mode's recipe in the oracle (oracle/fp8_oracle.py) -- power-of-two scales, e4m3 range and rounding, and
how far the emulated mode moves the outputs from the fp32 reference goldens."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from oracle.fp8_oracle import (Fp8Oracle, dequantize_blocks, dequantize_rows, fp8_scale, quantize_blocks,
                               quantize_rows)
from oracle.sta_oracle import make_images

KEYS = {"pts3d_pred": "pts3d", "conf": "conf", "relative_pose": "pose", "relative_pose_conf": "pose_conf"}
# Max-normalised deviation from the fp32 goldens (median-normalised for the dense outputs), worst of both views, of the
# recipe emulated on this oracle with seed-0 random weights (DESIGN.md section 5).  Bounds are 1.6x these.
DEV = {
    "pair_224x224": {"pts3d_pred": (1.35e-1, 1.6e-2), "conf": (1.22e-1, 1.2e-2), "relative_pose": (2.00e-1, None),
                     "relative_pose_conf": (4.8e-2, None)},
    "pair_64x80": {"pts3d_pred": (1.12e-1, 1.1e-2), "conf": (9.7e-2, 1.1e-2), "relative_pose": (8.0e-2, None),
                   "relative_pose_conf": (1.9e-2, None)},
}


def _groups(seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(64, 1024, generator=g)
    x = x * torch.exp2(torch.randint(-30, 30, (64, 8, 1), generator=g).float()).repeat_interleave(128, 1).reshape(64, 1024)
    x[3, 128:256] = 0.0  # an all-zero group
    return x


def test_scales_are_powers_of_two_and_codes_in_range():
    x = _groups(0)
    q, s = quantize_rows(x)
    m, e = torch.frexp(s)
    assert bool((m == 0.5).all()), "scales are powers of two"
    assert float(s[3, 1]) == 1.0, "an all-zero group has scale 1"
    deq = dequantize_rows(q, s)
    assert float(q.float().abs().max()) <= 448.0
    g = x.reshape(64, 8, 128)
    amax = g.abs().amax(-1)
    nz = amax > 0
    # smallest e with amax <= 448 * 2^e: it fits, and half the scale would not
    assert bool((amax <= 448 * s).all()) and bool((amax[nz] > 224 * s[nz]).all())
    # round to nearest: the error is at most half an e4m3 ulp at the value's binade (3 mantissa bits, subnormals 2^-9)
    v = g / s[..., None]
    ulp = torch.exp2(torch.clamp(torch.floor(torch.log2(v.abs().clamp_min(1e-30))), min=-6) - 3)
    err = (deq.reshape(64, 8, 128) - g).abs() / s[..., None]
    assert bool((err <= 0.5 * ulp + 1e-12).all())


def test_scale_at_a_power_of_two_boundary():
    # amax exactly 448 * 2^e takes scale 2^e; the next fp32 value above takes 2^(e + 1)
    for e in (-20, -3, 0, 5):
        b = torch.tensor([448.0 * 2.0 ** e], dtype=torch.float32)
        s, inv = fp8_scale(b)
        assert float(s) == 2.0 ** e and float(inv) == 2.0 ** -e
        s2, _ = fp8_scale(torch.nextafter(b, torch.tensor([float("inf")])))
        assert float(s2) == 2.0 ** (e + 1)
    x = torch.zeros(1, 128)
    x[0, 7] = -448.0 * 8
    q, s = quantize_rows(x)
    assert float(s) == 8.0 and float(q.float()[0, 7]) == -448.0


def test_weight_blocks():
    g = torch.Generator().manual_seed(1)
    w = torch.randn(256, 384, generator=g) / 20
    w[128:, :128] *= 1000
    q, s = quantize_blocks(w)
    assert s.shape == (2, 3) and float(s[1, 0]) > 100 * float(s[0, 0])
    # half an e4m3 ulp of the top binade [256, 448] (32) per block scale
    bound = 16 * s.repeat_interleave(128, 0).repeat_interleave(128, 1)
    assert bool(((dequantize_blocks(q, s) - w).abs() <= bound).all())


@pytest.mark.parametrize("case", sorted(DEV))
def test_oracle_deviation_from_fp32_goldens(state_dict, case):
    g = np.load(os.path.join(GOLDEN_DIR, case + ".npz"))
    meta = json.loads(str(g["meta"]))
    img1, img2 = make_images(meta["B"], meta["H"], meta["W"], meta["image_seed"])
    with torch.no_grad():
        main, sup = Fp8Oracle(state_dict).forward_pair(img1, img2)
    for k, gk in KEYS.items():
        mx, md = DEV[case][k]
        for res, pre in ((main, "main_"), (sup, "support_")):
            gold = torch.from_numpy(g[pre + gk])
            d = (res[k].float() - gold).abs()
            scale = float(gold.abs().max())
            assert float(d.max()) / scale < 1.6 * mx, (case, pre, k, float(d.max()) / scale)
            if md is not None:
                assert float(d.median()) / scale < 1.6 * md, (case, pre, k, float(d.median()) / scale)
