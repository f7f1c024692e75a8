"""GPU: the FP8 mode (STA(precision="fp8"), include/sta_b200.h STA_PRECISION_FP8) -- the bf16 quantiser, tile offsets
and a planted long sum of its GEMM (every launch at the model's sizes: tests/test_layers_fp8_gpu.py), the whole model against the CPU restatement of the recipe (oracle/fp8_oracle.py) and the fp32
goldens, its effect on the other modes, its memory, and OnlineSLAM on top of it."""
import ctypes
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR
from oracle.fp8_oracle import Fp8Oracle, dequantize_blocks, dequantize_rows, quantize_blocks, quantize_rows
from oracle.sta_oracle import make_images
from test_gemm_schedule_gpu import _copies, _tile_rows
from test_model_gpu import KEYS, golden_case, maxn, medn

pytestmark = pytest.mark.gpu

from vista_slam_b200 import _lib  # noqa: E402
from vista_slam_b200._lib import EPI_F32, EPI_GELU_FP8, EPI_ROPE, StaGemmFp8Desc  # noqa: E402

DEV = "cuda"
CASES = ["pair_64x80", "pair_b2_48x64", "pair_224x224", "pair_384x512"]
# FP8 model against the fp8 oracle: max-normalised deviation over the four goldens and both views, about twice what was
# measured for the dense outputs (pts3d 7.0e-2, conf 4.8e-2 on an H100).  The kernels and the oracle round the same
# recipe from slightly different fp32 values (LayerNorm, GEMM sums), so each carries its own e4m3 noise; the pose of a
# single token through an SVD amplifies it most on the smallest golden (12 tokens: the oracle's own pose deviation from
# fp32 is 4-13x bf16's there and changes by 3x with the host's BLAS; the kernels' reached 0.79), so the pose bounds are
# also allowed POSE_FACTOR x the oracle's own deviation from fp32, and that golden's pose is only checked to be a rigid
# transform.  That deviation is ill-conditioning, not the pose head: on that golden the head kernel matches a float64
# head on the FP8 model's own pose tokens with err / bound < 1e-4 (tests/test_pose_head_gpu.py), while those tokens
# are 11% from the bf16 model's and the resulting rotations differ by up to 0.82 (H100 80GB HBM3, 700 W).
# Sample 0's tokens give det A < 0 with sigma2 - sigma3 = 0.17, so a token error reaches R amplified by 2 / 0.17 = 12.
TOL_ORACLE = {"pts3d_pred": 1.5e-1, "conf": 1.5e-1, "relative_pose": 2.5e-1, "relative_pose_conf": 6e-2}
POSE_FACTOR = 4.0
ILL_CONDITIONED_POSE = {"pair_b2_48x64"}
# dense outputs against fp32: max and median deviation relative to the oracle's own (largest measured: 1.27x median,
# pair_64x80 main view)
MAX_VS_ORACLE, MED_VS_ORACLE = 1.6, 1.3


def _u8(q):
    return q.view(torch.uint8)


def _operands(M, N, K, g):
    """exactly known e4m3 operands with varied power-of-two scales: (codes, scales, dequantised fp64) of A and W"""
    a = torch.randn(M, K, generator=g) * torch.exp2(torch.randint(-4, 5, (M, 1), generator=g).float())
    w = torch.randn(N, K, generator=g) / math.sqrt(K) * torch.exp2(torch.randint(-3, 4, (N // 128, 1), generator=g).float()
                                                                    ).repeat_interleave(128, 0)
    aq, as_ = quantize_rows(a)
    wq, ws = quantize_blocks(w)
    return aq, as_, dequantize_rows(aq, as_).double(), wq, ws, dequantize_blocks(wq, ws).double()


def _gemm(epi, aq, as_, wq, ws, M, N, K, bias, out, resid=None, out_scale=None, pos=None, rope_cols=0):
    d = StaGemmFp8Desc()
    d.epi, d.M, d.N, d.K = epi, M, N, K
    d.A, d.lda, d.a_scale = aq.data_ptr(), K, as_.data_ptr()
    d.W, d.ldw, d.w_scale = wq.data_ptr(), K, ws.data_ptr()
    d.bias = bias.data_ptr()
    d.out, d.ldo = out.data_ptr(), N
    d.resid = None if resid is None else resid.data_ptr()
    d.out_scale = None if out_scale is None else out_scale.data_ptr()
    if pos is not None:
        d.pos, d.rope_cols = pos.data_ptr(), rope_cols
    _lib.check(_lib.lib().sta_op_gemm_fp8(ctypes.byref(d), _lib.cur_stream()), "sta_op_gemm_fp8")


def _dev(*ts):
    return [_u8(t).to(DEV) if t.dtype == torch.float8_e4m3fn else t.to(DEV) for t in ts]


def test_quant_bf16_is_bit_identical_to_cpu():
    g = torch.Generator().manual_seed(5)
    rows, C = 301, 1024
    x = (torch.randn(rows, C, generator=g) * torch.exp2(torch.randint(-20, 20, (rows, C // 128), generator=g).float()
                                                          ).repeat_interleave(128, 1)).bfloat16()
    x[7, 256:384] = 0
    q, s = torch.empty(rows, C, dtype=torch.uint8, device=DEV), torch.empty(rows, C // 128, device=DEV)
    _lib.check(_lib.lib().sta_op_quant_fp8(x.to(DEV).data_ptr(), rows, C, q.data_ptr(), s.data_ptr(), _lib.cur_stream()))
    torch.cuda.synchronize()
    q_ref, s_ref = quantize_rows(x.float())
    assert torch.equal(q.cpu(), _u8(q_ref)) and torch.equal(s.cpu(), s_ref)


@pytest.mark.parametrize("epi,N,K", [(EPI_ROPE, 3072, 1024), (EPI_F32, 1024, 1024), (EPI_GELU_FP8, 4096, 1024),
                                     (EPI_F32, 768, 3072)])
def test_block_is_bit_identical_at_any_tile_offset(epi, N, K):
    g = torch.Generator().manual_seed(N + K + epi)
    for mt in _tile_rows(N):
        M = 128 * mt
        aq, as_, _, wq, ws, _ = _operands(M, N, K, g)
        pos = torch.randint(0, 32, (M, 2), generator=g, dtype=torch.int32)
        offs = _copies(mt)
        aq8 = _u8(aq).clone()
        for o in offs:
            aq8[128 * o:128 * o + 128] = aq8[:128]
            as_[128 * o:128 * o + 128] = as_[:128]
            pos[128 * o:128 * o + 128] = pos[:128]
        bias = torch.randn(N, generator=g)
        A, As, Wd, Wsd, Bd, P = aq8.to(DEV), as_.to(DEV), _u8(wq).to(DEV), ws.to(DEV), bias.to(DEV), pos.to(DEV)

        def run(rows):
            a, sa = A[:rows].contiguous(), As[:rows].contiguous()
            if epi == EPI_F32:
                x = torch.ones(rows, N, device=DEV)
                _gemm(epi, a, sa, Wd, Wsd, rows, N, K, Bd, x, resid=x)
                return [x]
            if epi == EPI_ROPE:
                o = torch.full((rows, N), float("nan"), device=DEV, dtype=torch.bfloat16)
                _gemm(epi, a, sa, Wd, Wsd, rows, N, K, Bd, o, pos=P[:rows].contiguous(), rope_cols=2048)  # enc.qkv
                return [o]
            q, s = torch.empty(rows, N, dtype=torch.uint8, device=DEV), torch.empty(rows, N // 128, device=DEV)
            _gemm(epi, a, sa, Wd, Wsd, rows, N, K, Bd, q, out_scale=s)
            return [q, s]

        alone, big = run(128), run(M)
        torch.cuda.synchronize()
        for a, b in zip(alone, big):
            for o in offs:
                assert torch.equal(b[128 * o:128 * o + 128], a), "tile offset %d of %d" % (o, mt)


def test_planted_long_sum_holds_fp32_accuracy():
    # K = 4096: one large product (2^16) in k-block 0, then 31 k-blocks of 128 products 2^-6 each: 65536 + 62 exactly.
    # A single tensor-core accumulator over all of K would drop the small products.
    M, N, K = 128, 128, 4096
    a = torch.zeros(M, K)
    w = torch.zeros(N, K)
    a[:, 0], w[:, 0] = 256.0, 256.0
    a[:, 128:], w[:, 128:] = 1.0, 2.0 ** -6
    aq, wq = a.to(torch.float8_e4m3fn), w.to(torch.float8_e4m3fn)
    as_ = torch.ones(M, K // 128)
    ws = torch.ones(N // 128, K // 128)
    aqd, asd, wqd, wsd = _dev(aq, as_, wq, ws)
    x = torch.zeros(M, N, device=DEV)
    _gemm(EPI_F32, aqd, asd, wqd, wsd, M, N, K, torch.zeros(N, device=DEV), x)
    torch.cuda.synchronize()
    assert bool((x == 65598.0).all()), float((x - 65598.0).abs().max())


# ------------------------------------------------------------------------------------------------ model
@pytest.fixture(scope="module")
def fp8_model(state_dict):
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    m = STA(precision="fp8")
    m.load_state_dict(state_dict, strict=True)
    m.eval()
    m._ready(torch.empty(1, device=DEV))
    return m


def _oracle_bound(k, orc, gold):
    if k in ("relative_pose", "relative_pose_conf"):
        return max(TOL_ORACLE[k], POSE_FACTOR * maxn(orc, gold))
    return TOL_ORACLE[k]


@pytest.mark.parametrize("case", CASES)
def test_forward_pairs_vs_fp8_oracle_and_fp32_golden(fp8_model, state_dict, case):
    g, meta, img1, img2 = golden_case(case)
    main, sup = fp8_model.forward_pairs(img1.cuda(), img2.cuda())
    with torch.no_grad():
        o_main, o_sup = Fp8Oracle(state_dict).forward_pair(img1, img2)
    rec = {}
    for res, orc, pre in ((main, o_main, "main_"), (sup, o_sup, "support_")):
        for k, gk in KEYS.items():
            gold = torch.from_numpy(g[pre + gk])
            rec[pre + gk] = [maxn(res[k], orc[k]), maxn(res[k], gold), maxn(orc[k], gold), medn(res[k], gold),
                             medn(orc[k], gold)]
    print("fp8 model", case, json.dumps(rec))
    for res, orc, pre in ((main, o_main, "main_"), (sup, o_sup, "support_")):
        for k, gk in KEYS.items():
            gold = torch.from_numpy(g[pre + gk])
            if k == "relative_pose" and case in ILL_CONDITIONED_POSE:
                P = res[k].double().cpu()
                R = P[:, :3, :3]
                assert (R @ R.transpose(1, 2) - torch.eye(3, dtype=torch.float64)).abs().max() < 1e-5
                assert (torch.det(R) - 1).abs().max() < 1e-5
                continue
            assert maxn(res[k], orc[k]) < _oracle_bound(k, orc[k], gold), (pre, k)
            if k in ("pts3d_pred", "conf"):
                # the deviation from fp32 is the recipe's, not more: the pattern of test_model_gpu.py
                assert maxn(res[k], gold) < MAX_VS_ORACLE * maxn(orc[k], gold) + 1e-4, (pre, k)
                assert medn(res[k], gold) < MED_VS_ORACLE * medn(orc[k], gold) + 1e-5, (pre, k)


def test_cfg2_batch16_pair0_is_the_golden_pair(fp8_model, state_dict):
    g, meta, img1, img2 = golden_case("pair_384x512")
    H, W = meta["H"], meta["W"]
    o1, o2 = make_images(15, H, W, 99)
    main, sup = fp8_model.forward_pairs(torch.cat([img1, o1]).bfloat16().cuda(), torch.cat([img2, o2]).bfloat16().cuda())
    one_m, one_s = fp8_model.forward_pairs(img1.bfloat16().cuda(), img2.bfloat16().cuda())
    with torch.no_grad():
        o_main, o_sup = Fp8Oracle(state_dict).forward_pair(img1, img2)
    for res, orc, pre in ((main, o_main, "main_"), (sup, o_sup, "support_")):
        for k, gk in KEYS.items():
            gold = torch.from_numpy(g[pre + gk])
            assert maxn(res[k][:1], orc[k]) < _oracle_bound(k, orc[k], gold), (pre, k)
            if k in ("pts3d_pred", "conf"):
                assert maxn(res[k][:1], gold) < MAX_VS_ORACLE * maxn(orc[k], gold) + 1e-4, (pre, k)
    m8, s8 = fp8_model.forward_pairs(torch.cat([img1, o1])[:8].bfloat16().cuda(), torch.cat([img2, o2])[:8].bfloat16().cuda())
    assert torch.equal(m8["pts3d_pred"][0], main["pts3d_pred"][0]) and torch.equal(s8["relative_pose"][0], sup["relative_pose"][0])
    assert maxn(one_m["pts3d_pred"][0], main["pts3d_pred"][0]) < 5e-2


def test_every_entry_point_runs(fp8_model):
    img1, img2 = make_images(2, 64, 80, 9)
    B, H, W = 2, 64, 80
    ts = torch.tensor([[H, W]] * B)
    main, _ = fp8_model.forward_pairs(img1.cuda(), img2.cuda())
    f1, p1 = fp8_model._encode_image(img1.cuda(), ts, normalize=False)
    f2, p2 = fp8_model._encode_image(img2.cuda(), ts, normalize=False)
    d1, d2 = fp8_model._decode_stereo(f1, f2, p1, p2)
    pts = fp8_model.head_pts([f1] + [t[:, 1:, :] for t in d1], ts)
    pose = fp8_model.head_pose_s(d1[-1][:, 0, :])
    assert maxn(pts["pts3d"], main["pts3d_pred"]) < 5e-2 and maxn(pose["pose"], main["relative_pose"]) < 2e-2
    out = fp8_model({"main_view": {"img": img1.cuda(), "true_shape": ts},
                     "neighbor_views": [{"img": img2.cuda(), "true_shape": ts}], "loop_views": []})
    assert out["main_views"][0]["pts3d_pred"].shape == (B, H, W, 3)
    h1, h2 = img1.bfloat16().pin_memory(), img2.bfloat16().pin_memory()
    host = fp8_model.forward_pairs_host(h1, h2)
    dm, ds = fp8_model.forward_pairs(h1.cuda(), h2.cuda())
    assert torch.equal(host["pts3d"][0], dm["pts3d_pred"].cpu()) and torch.equal(host["pose"][1], ds["relative_pose"].cpu())


def test_bf16_model_is_untouched_by_an_fp8_model(cuda_model, state_dict):
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    img1, img2 = make_images(2, 64, 80, 21)
    before = cuda_model.forward_pairs(img1.cuda(), img2.cuda())
    m = STA(precision="fp8")
    m.load_state_dict(state_dict, strict=True)
    m.eval()
    m.forward_pairs(img1.cuda(), img2.cuda())
    after = cuda_model.forward_pairs(img1.cuda(), img2.cuda())
    for b, a in zip(before, after):
        for k in b:
            assert torch.equal(b[k], a[k]), k


def test_device_bytes_fp8_below_bf16(state_dict):
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    img1, img2 = make_images(2, 64, 80, 22)
    got = {}
    for prec in ("bf16", "fp8"):
        m = STA(precision=prec)
        m.load_state_dict(state_dict, strict=True)
        m.eval()
        m.forward_pairs(img1.cuda(), img2.cuda())
        torch.cuda.synchronize()
        got[prec] = m.device_bytes
        del m
    trunk = 24 * 12 * 1024 ** 2 + 12 * 16 * 768 ** 2  # trunk weights: 415,236,096
    assert got["bf16"] - got["fp8"] >= 0.95 * trunk, got  # half of their bf16 bytes


def test_online_slam_on_the_fp8_frontend(state_dict, tmp_path):
    from vista_slam_b200.slam import OnlineSLAM
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA

    class Fp8Slam(OnlineSLAM):  # the recipe of INTEGRATION.md section 5
        def load_frontend(self, ckpt_path):
            m = STA(precision="fp8")
            m.load_state_dict(state_dict, strict=True)
            return m.to(self.device).eval()

    H = W = 224
    g = torch.Generator().manual_seed(1)
    base = torch.rand(1, 3, H // 8, W // 4, generator=g)
    values = []
    for i in range(24):
        img = F.interpolate(base.roll(3 * i, dims=3)[..., :W // 8], size=(H, W), mode="bilinear")
        img = ((img * 2 - 1) + 0.05 * torch.randn(1, 3, H, W, generator=g)).clamp(-1, 1).cuda()
        values.append({"rgb": img, "shape": torch.tensor([[H, W]]), "gray": ((img[0].mean(0) + 1) / 2).contiguous(),
                       "view_name": "%05d" % i})
    vocab = os.path.join(GOLDEN_DIR, "loop_vocab.txt")
    slam = Fp8Slam("unused", vocab, pgo_every=500)
    for v in values[:8]:
        slam.step(v)
    slam.step_many(values[8:], force_pgo=True)
    torch.cuda.synchronize()
    N, E, V = slam.num_nodes, slam.num_edges, slam.view_num
    assert V > 1 and N > 0 and E > 0
    G = slam._graph
    ntv = G.node_to_view[:N].cpu()
    assert bool(((ntv >= 0) & (ntv < V)).all())
    edges = G.edges[:E].cpu()
    assert bool(((edges >= 0) & (edges < N)).all())
    assert bool(torch.isfinite(G.pose[:N]).all())
    out = tmp_path / "run"
    slam.save_data_all(str(out))
    files = [f for f in out.rglob("*") if f.is_file()]
    assert files and all(f.stat().st_size > 0 for f in files), files
