"""GPU: every bf16 GEMM and implicit-GEMM convolution launch the model makes, at the model's shapes, against float64 with a
bound on every output element, against planted integer answers bit for bit, and with NaN canaries around every output;
plus the bandwidth kernels (patch im2col, bilinear upsample, stride-2 im2col, LayerNorm, fp32 -> bf16 cast) at the same
sizes.

The launch list is layer_catalogue(): it restates run_encoder (runtime.cu:892-920), run_decoder (runtime.cu:927-1002) and
run_dpt (runtime.cu:1029-1106) one launch at a time.  A layer added to runtime.cu gets its line there.
off_model_layers() runs the same checks on launches the model does not make: other shapes and epilogue combinations.

Float64 check.  Random operands (weights scaled by 1/sqrt(K) as the model's are), the reference is the float64 product of
exactly the bf16 operands the kernel reads (cuBLAS DGEMM; convolutions as F.unfold + matmul).  Per element:

    |got - ref| <= u_out |ref| + tau(K) S,    S = sum_k |a_k w_k| + |bias| + sum |skip|

  * u_out = 2^-8 for bf16 outputs (round to nearest: half an ulp is at most 2^-8 of the value), 2^-23 for fp32 outputs.
  * tau(K) = TAU_STEP (K / 16 + 8), TAU_STEP = 2^-22.  The tensor cores add each k16 group of exact bf16 products to an
    fp32 accumulator; one such addition costs at most an ulp of the running sum (2^-23 of it, or 2^-22 if both the group
    sum and the addition truncate), and |running sum| <= S.  A tile makes K / 16 additions; the bias, the skip tensors,
    the split-K partial sums (at most 8) and the fp32 epilogue arithmetic make at most 8 more.
    Largest err / bound measured: see MEASURED_RATIO.
  * GELU scales the tau term by max|gelu'| = 1.13 and adds 2^-20 for the kernel's fitted gelu (5e-7 absolute).
  * RoPE: both elements of a rotated pair get tau (S_a + S_b), plus 2^-21 (|pos| + 2) (|a| + |b|) for the fp32 angle of
    the kernel's table (one ulp of pos * inv_freq) and the fp32 rotation.
  * EPI_HEAD: the hidden layer's bound is carried through the 1x1 (sum_c |w_jc| tau S_c, plus 2^-18 sum_c |w_jc h_c| for
    the two fp32 64-term chains) and the post-process, whose gradient is at most e^d (d = |xyz|) for pts3d and e^conf for
    conf; the fp32 post-process itself gets 2^-20 of the value.
  * x3 (split-precision parity mode): the operands are the (hi | lo | hi) x (hi | hi | lo) expansions along K, the
    reference is their float64 product (so K is 3K in tau), the output is hi + lo with u_out = 2^-16.

Planted answers.  Small integer operands, biases and skip tensors, sparse enough that S <= 256 for every output: every
partial sum and every output is then an integer that bf16 and fp32 hold exactly in any summation order, and the kernel
must reproduce the integer reference exactly.  Weight rows are random and distinct, each with nonzeros in several
k-blocks; convolution inputs carry single-pixel deltas at 16-row and 8-column tile borders and image edges, and every
image has its own pattern.  GELU rows are planted at pre-activations >= 6, where the kernel's gelu is the identity in
fp32; RoPE rows at position (0, 0), where the rotation is the identity.  EPI_HEAD gets power-of-two 1x1 weights, so the
four logits are exact and only the post-process's rounding is left (2^-20 of the value).

Canaries.  Outputs, relu copies and pixel-shuffle targets have a trailing image or three trailing rows, and every
row-strided output has 64 padding columns (32 for fp32); all of it is NaN and must keep its bits.  The decoder_embed
output's pose-token rows are not addressed either."""
import ctypes
import math
from dataclasses import dataclass, replace

import pytest
import torch
import torch.nn.functional as F

from vista_slam_b200._lib import EPI_BF16, EPI_F32, EPI_GELU, EPI_HEAD, EPI_PIXSHUF, EPI_ROPE, StaGemmDesc

pytestmark = pytest.mark.gpu

TAU_STEP = 2.0 ** -22
# Largest err / bound of the float64 checks, H100 80GB HBM3 (700 W power limit), all three sizes and the off-model
# layers:
#   fp32-output layers, where the tau term dominates: 0.027 in the catalogue (dec.proj at cfg-2), 0.042 off the model
#   (f32_inplace_M24576_N1024_K256): tau grows with K / 16 while random roundings grow with its square root, so K = 256
#   comes closest; tau is a worst case ~24x above what the tensor cores show on random operands;
#   bf16 outputs: 0.994 -- the output rounding, which u_out = 2^-8 covers exactly, with little room left;
#   x3: 0.27; EPI_HEAD: 0.0017; planted EPI_HEAD against its 2^-20 post-process bound: 0.18.
MEASURED_RATIO = {"f32_out": 0.042, "bf16_out": 0.994, "x3": 0.27, "head": 0.0017, "head_planted": 0.18}
GELU_SLOPE = 1.1289
SPLITK_BYTES = 48 << 20  # StaModel::kSplitKBytes (runtime.cu): the model's split-K workspace


def tau(K):
    return TAU_STEP * (K / 16 + 8)


# ---------------------------------------------------------------------------------------------------------------------
# the catalogue
# ---------------------------------------------------------------------------------------------------------------------

@dataclass(frozen=True)
class Layer:
    name: str
    epi: int
    M: int = 0                # linear: rows of A
    N: int = 0
    K: int = 0                # logical reduction length
    conv: tuple = None        # (nimg, H, W, Cin): 3x3 implicit-GEMM convolution, padding 1
    bias: bool = True
    resid: str = ""           # "" | "inplace" (fp32 residual stream, out += ...) | "skip" (a tensor of the out type)
    resid2: bool = False
    relu_main: int = 0
    relu_copy: bool = False
    rope_cols: int = 0
    pos_grid: tuple = None    # RoPE positions: (samples, h, w, with_pose_token) as launch_make_positions builds them
    pos_rand: int = 0         # RoPE positions without a grid: uniform in [-1, pos_rand) on each axis
    rowmap_n: int = 0
    ps: tuple = None          # EPI_PIXSHUF: (k, cout, nimg, h, w)
    taps: int = 1             # K = taps x channels (act3c reads stride-2 im2col rows): x3 splits each tap
    splitk: bool = True       # pass the model's split-K workspace


def layer_catalogue(h, w, nimg, pairs, dpt_nimg):
    """The sta_op_gemm launches of one forward pass: encoder over nimg images of h x w tokens, decoder over `pairs`
    pairs (2 * pairs samples), DPT over a pass of dpt_nimg images."""
    n = h * w
    L = []
    # run_encoder (runtime.cu:892-920), bf16 mode
    T = nimg * n
    enc_pos = (nimg, h, w, 0)
    L += [Layer("enc.patch_embed", EPI_F32, T, 1024, 768),
          Layer("enc.qkv", EPI_ROPE, T, 3072, 1024, rope_cols=2048, pos_grid=enc_pos),
          Layer("enc.proj", EPI_F32, T, 1024, 1024, resid="inplace"),
          Layer("enc.fc1", EPI_GELU, T, 4096, 1024),
          Layer("enc.fc2", EPI_F32, T, 1024, 4096, resid="inplace")]
    # run_decoder (runtime.cu:927-1002): S = 2 pairs samples of n + 1 rows (pose token first)
    S = 2 * pairs
    Td = S * (n + 1)
    dec_pos = (S, h, w, 1)
    L += [Layer("dec.decoder_embed", EPI_F32, S * n, 768, 1024, rowmap_n=n),
          Layer("dec.qkv", EPI_ROPE, Td, 2304, 768, rope_cols=1536, pos_grid=dec_pos),
          Layer("dec.proj", EPI_F32, Td, 768, 768, resid="inplace"),
          Layer("dec.projk|projv", EPI_ROPE, Td, 1536, 768, rope_cols=768, pos_grid=dec_pos),
          Layer("dec.projq", EPI_ROPE, Td, 768, 768, rope_cols=768, pos_grid=dec_pos),
          Layer("dec.cproj", EPI_F32, Td, 768, 768, resid="inplace"),
          Layer("dec.fc1", EPI_GELU, Td, 3072, 768),
          Layer("dec.fc2", EPI_F32, Td, 768, 3072, resid="inplace")]
    # run_dpt (runtime.cu:1029-1106) over dpt_nimg images
    m = dpt_nimg
    T = m * n
    h4, w4 = (h + 1) // 2, (w + 1) // 2
    LH, LW = [4 * h, 2 * h, h, h4], [4 * w, 2 * w, w, w4]
    L += [Layer("dpt.act0", EPI_BF16, T, 128, 1024),
          Layer("dpt.act0T", EPI_PIXSHUF, T, 4 * 4 * 128, 128, ps=(4, 128, m, h, w)),
          Layer("dpt.act1", EPI_BF16, T, 192, 768),
          Layer("dpt.act1T", EPI_PIXSHUF, T, 2 * 2 * 192, 192, ps=(2, 192, m, h, w)),
          Layer("dpt.act2", EPI_BF16, T, 384, 768),
          Layer("dpt.act3", EPI_BF16, T, 768, 768),
          Layer("dpt.act3c", EPI_BF16, m * h4 * w4, 768, 9 * 768, taps=9)]
    for i, cin in enumerate((128, 192, 384, 768)):
        L.append(Layer("dpt.layer%d_rn" % (i + 1), EPI_BF16, N=256, K=9 * cin, conv=(m, LH[i], LW[i], cin), bias=False,
                       relu_copy=True))
    for lvl in (3, 2, 1, 0):
        g = (m, LH[lvl], LW[lvl], 256)
        p = "dpt.refinenet%d." % (lvl + 1)
        if lvl != 3:
            L += [Layer(p + "rcu1.conv1", EPI_BF16, N=256, K=2304, conv=g, relu_main=1),
                  Layer(p + "rcu1.conv2", EPI_BF16, N=256, K=2304, conv=g, resid="skip", resid2=True, relu_copy=True)]
        L += [Layer(p + "rcu2.conv1", EPI_BF16, N=256, K=2304, conv=g, relu_main=1),
              Layer(p + "rcu2.conv2", EPI_BF16, N=256, K=2304, conv=g, resid="skip"),
              Layer(p + "out_conv", EPI_BF16, m * LH[lvl] * LW[lvl], 256, 256)]
    L += [Layer("dpt.head.0", EPI_BF16, N=128, K=2304, conv=(m, 8 * h, 8 * w, 256)),
          Layer("dpt.head.2", EPI_HEAD, N=128, K=1152, conv=(m, 16 * h, 16 * w, 128))]
    return L


def off_model_layers():
    """sta_op_gemm launches the model does not make: ragged and other shapes, tile counts from one CTA to many waves,
    epilogue combinations the catalogue lacks (two skip tensors on a linear layer, relu on a linear layer's output, an
    fp32 output with its own skip tensor, the in-place fp32 update without a split-K workspace), RoPE at random
    positions, partly past the shared-memory table, and small convolutions, pixel shuffles and a head."""
    L = [Layer("linear_M%d_N%d_K%d" % s, EPI_BF16, *s)
         for s in ((128, 256, 64), (300, 512, 192), (128, 256, 1024), (8192, 1024, 1024), (1000, 384, 768),
                   (24608, 768, 768), (777, 512, 256), (4096, 768, 768), (300, 384, 192))]
    L += [Layer("f32_inplace_M%d_N%d_K%d" % s, EPI_F32, *s, resid="inplace")
          for s in ((777, 512, 256), (4096, 768, 768), (300, 384, 192), (777, 320, 256), (5000, 1024, 256),
                    (24576, 1024, 256))]
    L += [Layer("f32_inplace_M196_N1024_K1024_no_splitk_ws", EPI_F32, 196, 1024, 1024, resid="inplace", splitk=False),
          Layer("f32_M777_N512_K256", EPI_F32, 777, 512, 256),
          Layer("f32_M196_N1024_K1024", EPI_F32, 196, 1024, 1024),
          Layer("f32_skip_M777_N512_K256", EPI_F32, 777, 512, 256, resid="skip"),
          Layer("f32_rowmap_7x111_N512_K256", EPI_F32, 777, 512, 256, rowmap_n=111),
          Layer("skip2_relu_copy_M777_N512_K256", EPI_BF16, 777, 512, 256, resid="skip", resid2=True, relu_copy=True),
          Layer("skip2_relu_copy_M500_N256_K256", EPI_BF16, 500, 256, 256, resid="skip", resid2=True, relu_copy=True),
          Layer("relu_main_M777_N512_K256", EPI_BF16, 777, 512, 256, relu_main=1),
          Layer("no_bias_M777_N384_K256", EPI_BF16, 777, 384, 256, bias=False),
          Layer("gelu_M777_N512_K256", EPI_GELU, 777, 512, 256),
          Layer("gelu_M4096_N768_K768", EPI_GELU, 4096, 768, 768),
          Layer("gelu_M196_N1024_K1024", EPI_GELU, 196, 1024, 1024),
          Layer("gelu_M5000_N1024_K256", EPI_GELU, 5000, 1024, 256),
          Layer("rope_M777_N768_K256", EPI_ROPE, 777, 768, 256, rope_cols=512, pos_rand=40),
          Layer("rope_M500_N768_K256", EPI_ROPE, 500, 768, 256, rope_cols=512, pos_rand=70),
          Layer("rope_M196_N1024_K1024", EPI_ROPE, 196, 1024, 1024, rope_cols=768, pos_rand=14),
          Layer("rope_M5000_N1024_K256", EPI_ROPE, 5000, 1024, 256, rope_cols=768, pos_rand=70),
          Layer("pixshuf_k2_C128_64_2x5x7", EPI_PIXSHUF, 70, 256, 128, ps=(2, 64, 2, 5, 7)),
          Layer("pixshuf_k2_C192_192_2x6x10", EPI_PIXSHUF, 120, 768, 192, ps=(2, 192, 2, 6, 10))]
    L += [Layer("conv_%dx%dx%d_C%d_%d_skip_relu_copy" % g, EPI_BF16, N=g[4], K=9 * g[3], conv=g[:4], resid="skip",
                relu_copy=True)
          for g in ((2, 8, 16, 64, 256), (3, 14, 14, 128, 256), (2, 24, 32, 256, 256), (1, 20, 36, 256, 128))]
    L += [Layer("conv_2x14x18_C128_256_skip", EPI_BF16, N=256, K=1152, conv=(2, 14, 18, 128), resid="skip"),
          Layer("conv_2x14x18_C256_256_no_bias_relu_main", EPI_BF16, N=256, K=2304, conv=(2, 14, 18, 256), bias=False,
                relu_main=1),
          Layer("head_2x32x48", EPI_HEAD, N=128, K=1152, conv=(2, 32, 48, 128))]
    return L


# the off-model layers also checked in the split-precision (x3) parity mode
OFF_MODEL_X3 = {"linear_M777_N512_K256", "linear_M4096_N768_K768", "linear_M300_N384_K192",
                "f32_inplace_M777_N512_K256", "f32_inplace_M4096_N768_K768", "f32_inplace_M300_N384_K192",
                "skip2_relu_copy_M500_N256_K256", "gelu_M777_N512_K256", "gelu_M4096_N768_K768", "rope_M500_N768_K256",
                "pixshuf_k2_C192_192_2x6x10", "conv_2x14x18_C128_256_skip"}


# (id, h, w, trunk images, pairs, DPT images, x3 checked)
SIZES = [("keyframe14x14", 14, 14, 1, 1, 1, True),
         ("odd3x5", 3, 5, 2, 1, 2, True),
         ("cfg2_24x32", 24, 32, 32, 16, 16, False)]
CFG2_CHECKED_IMAGES = (0, 15)  # float64 convolution references at cfg-2: the first and the last image of the pass


# ---------------------------------------------------------------------------------------------------------------------
# helpers that need no GPU (tests/test_layers_cpu.py feeds them mis-indexed outputs)
# ---------------------------------------------------------------------------------------------------------------------

def err_ratio(got, ref, bound):
    """max |got - ref| / bound (float64); NaN or Inf in got gives NaN / Inf"""
    r = ((got.double() - ref).abs() / bound).max()
    return float(r)


def check_bound(name, got, ref, bound):
    ratio = err_ratio(got, ref, bound)
    print("layer bound %-44s worst err / bound = %.4f" % (name, ratio), flush=True)
    assert ratio <= 1.0, "%s: err / bound = %s at %s" % (name, ratio, _worst(got, ref, bound))
    return ratio


def _worst(got, ref, bound):
    r = ((got.double() - ref).abs() / bound).nan_to_num(float("inf"))
    i = int(r.reshape(-1).argmax())
    idx = []
    for s in reversed(ref.shape):
        idx.append(i % s)
        i //= s
    idx = tuple(reversed(idx))
    return "%s: got %r ref %r bound %r" % (idx, float(got[idx]), float(ref[idx]), float(bound[idx]))


def check_exact(name, got, ref):
    """planted answers: got must equal the integer reference exactly"""
    g = got.double()
    bad = g != ref
    if bool(bad.any()):
        idx = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d elements differ from the planted answer; first %s: got %r want %r" % (
            name, int(bad.sum()), bad.numel(), idx, float(g[idx]), float(ref[idx])))


def pixshuf(y, k, cout, nimg, h, w):
    """GEMM rows [nimg h w][(kh, kw, co)] -> NHWC [nimg][h k][w k][cout] (ConvTranspose2d with kernel = stride = k)"""
    return (y.reshape(nimg, h, w, k, k, cout).permute(0, 1, 3, 2, 4, 5).reshape(nimg, h * k, w * k, cout))


def conv_cols(x, stride=1):
    """NHWC [n][H][W][C] -> im2col rows [n OH OW][9 C] in (kh, kw, c) order, float64, padding 1"""
    n, H, W, C = x.shape
    u = F.unfold(x.permute(0, 3, 1, 2).double(), 3, padding=1, stride=stride)  # [n][C 9][L]
    return u.view(n, C, 9, -1).permute(0, 3, 2, 1).reshape(-1, 9 * C)


def inv_freq64(device):
    return 100.0 ** (-torch.arange(16, device=device, dtype=torch.float64) / 16)


def rope64(x, pos, rope_cols):
    """float64 2-D RoPE of columns [0, rope_cols) of x [rows][N] (64-wide heads: y-half then x-half, pairs (i, i + 16))
    with exact angles; also the pair partner of every rotated column (for the bounds)"""
    out = x.clone()
    rows = x.shape[0]
    heads = rope_cols // 64
    v = x[:, :rope_cols].reshape(rows, heads, 64)
    o = out[:, :rope_cols].view(rows, heads, 64)
    inv = inv_freq64(x.device)
    for axis in range(2):
        ang = pos[:, axis].double()[:, None] * inv[None, :]
        c, s = ang.cos()[:, None, :], ang.sin()[:, None, :]
        a = v[..., axis * 32: axis * 32 + 16]
        b = v[..., axis * 32 + 16: axis * 32 + 32]
        o[..., axis * 32: axis * 32 + 16] = a * c - b * s
        o[..., axis * 32 + 16: axis * 32 + 32] = b * c + a * s
    return out


def rope_pair_sum(x, rope_cols):
    """x_i + x_partner(i) on the rotated columns, x elsewhere"""
    out = x.clone()
    rows = x.shape[0]
    v = x[:, :rope_cols].reshape(rows, rope_cols // 32, 2, 16)
    out[:, :rope_cols] = (v + v.flip(2)).reshape(rows, rope_cols)
    return out


def head_post(o):
    """EPI_HEAD post-process of logits [..][4] (postprocess.py:37-58): pts3d, conf"""
    xyz = o[..., :3]
    d = xyz.norm(dim=-1, keepdim=True)
    return xyz / d.clamp_min(1e-8) * torch.expm1(d), 1.0 + o[..., 3].exp()


def head_bound(o, err_o):
    """bounds on pts3d / conf from bounds err_o [..][4] on the logits o (post-process gradient <= e^d, e^cf)"""
    d = o[..., :3].norm(dim=-1, keepdim=True)
    e3 = err_o[..., :3].sum(-1, keepdim=True)
    pts, conf = head_post(o)
    bp = torch.exp(d + e3) * e3 + 2.0 ** -20 * pts.abs() + 1e-30
    bc = torch.exp(o[..., 3] + err_o[..., 3]) * err_o[..., 3] + 2.0 ** -20 * conf
    return bp, bc


def positions(grid, device):
    """the model's RoPE positions (launch_make_positions): (y, x) per token, (-1, -1) for a sample's pose token"""
    samples, h, w, with_pose = grid
    t = torch.arange(h * w, device=device)
    p = torch.stack([t // w, t % w], 1)
    if with_pose:
        p = torch.cat([torch.full((1, 2), -1, device=device, dtype=p.dtype), p])
    return p.repeat(samples, 1).int().contiguous()


# ---------------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------------

def split_act(x, taps=1):
    """(hi | lo | hi) along the last dim, per tap: the split-precision activation layout"""
    s = x.shape
    v = x.reshape(*s[:-1], taps, s[-1] // taps)
    hi = v.bfloat16()
    lo = (v - hi.float()).bfloat16()
    return torch.cat([hi, lo, hi], -1).reshape(*s[:-1], 3 * s[-1])


def split_w(w, taps=1):
    """(hi | hi | lo) along K, per tap: the split-precision weight layout"""
    s = w.shape
    v = w.reshape(s[0], taps, s[1] // taps)
    hi = v.bfloat16()
    lo = (v - hi.float()).bfloat16()
    return torch.cat([hi, hi, lo], -1).reshape(s[0], 3 * s[1])


def merge3(o, n):
    assert torch.equal(o[..., :n], o[..., 2 * n:3 * n]), "hi copies differ"
    return o[..., :n].double() + o[..., n:2 * n].double()


def _sparse_rows(N, K, g, dev, positive=False, nz=6):
    """N random distinct weight rows with nz nonzeros of magnitude 1 or 2, spread over the k-blocks of 64"""
    nkb = K // 64
    Wt = torch.zeros(N, K, device=dev)
    start = torch.randint(0, nkb, (N,), generator=g, device=dev)
    for j in range(nz):
        blk = (start + (j * nkb) // nz) % nkb
        col = blk * 64 + torch.randint(0, 64, (N,), generator=g, device=dev)
        val = torch.randint(1, 3, (N,), generator=g, device=dev).float()
        if not positive:
            val = val * (torch.randint(0, 2, (N,), generator=g, device=dev) * 2 - 1)
        Wt[torch.arange(N, device=dev), col] += val
    return Wt


def _deltas(x, g):
    """single-pixel deltas at 16-row / 8-column tile borders and image edges, in every image"""
    n, H, W, C = x.shape
    ys = sorted({y for y in (0, 15, 16, 31, 32, H - 1) if 0 <= y < H})
    xs = sorted({v for v in (0, 7, 8, 15, 16, W - 1) if 0 <= v < W})
    for i in range(n):
        for y in ys:
            for v in xs:
                x[i, y, v] += torch.randint(-2, 3, (C,), generator=g, device=x.device).float()
    return x


def make_operands(e, kind, seed, dev="cuda"):
    """logical fp32 operands of layer e: 'random' (normal, weights / sqrt(K)) or 'planted' (small integers)"""
    g = torch.Generator(device=dev).manual_seed(seed)
    planted = kind == "planted"
    positive = planted and e.epi == EPI_GELU
    o = {}
    if e.conv:
        nimg, H, W, Cin = e.conv
        if planted:
            o["A"] = _deltas(torch.randint(-1, 2, (nimg, H, W, Cin), generator=g, device=dev).float(), g)
        else:
            o["A"] = torch.randn(nimg, H, W, Cin, generator=g, device=dev)
        rows = (nimg, H, W)
    else:
        if planted:
            lo = 0 if positive else -2
            o["A"] = torch.randint(lo, 3, (e.M, e.K), generator=g, device=dev).float()
        else:
            o["A"] = torch.randn(e.M, e.K, generator=g, device=dev)
        rows = (e.M,)
    if planted:
        o["W"] = _sparse_rows(e.N, e.K, g, dev, positive)
    else:
        o["W"] = torch.randn(e.N, e.K, generator=g, device=dev) / math.sqrt(e.K)
    cout = e.ps[1] if e.ps else e.N  # the pixel shuffle adds one bias per output channel
    if e.bias:
        o["bias"] = (torch.randint(6, 10, (cout,), generator=g, device=dev).float() if positive else
                     torch.randint(-4, 5, (cout,), generator=g, device=dev).float() if planted else
                     torch.randn(cout, generator=g, device=dev))
    out_rows = (e.M // e.rowmap_n * (e.rowmap_n + 1),) if e.rowmap_n else rows
    for key, on in (("resid", bool(e.resid)), ("resid2", e.resid2)):
        if on:
            o[key] = (torch.randint(-4, 5, out_rows + (cout,), generator=g, device=dev).float() if planted else
                      torch.randn(out_rows + (cout,), generator=g, device=dev))
    if e.epi == EPI_HEAD:
        if planted:
            hw = torch.zeros(4, 128, device=dev)
            for j in range(4):
                idx = torch.randperm(128, generator=g, device=dev)[:8]
                hw[j, idx] = (torch.randint(0, 2, (8,), generator=g, device=dev) * 2 - 1).float() * 2.0 ** -6
            o["head_w"] = hw
            o["head_b"] = torch.tensor([0.25, -0.25, 0.5, -0.5], device=dev)
        else:
            o["head_w"] = torch.randn(4, 128, generator=g, device=dev) / math.sqrt(128)
            o["head_b"] = torch.randn(4, generator=g, device=dev) * 0.1
    if e.rope_cols:
        o["pos"] = (torch.zeros(e.M, 2, dtype=torch.int32, device=dev) if planted else
                    positions(e.pos_grid, dev) if e.pos_grid else
                    torch.randint(-1, e.pos_rand, (e.M, 2), generator=g, device=dev, dtype=torch.int32))
    return o


def _phys(x, split, taps=1):
    return split_act(x, taps) if split else x.bfloat16()


def _logical(xp, split, n):
    return merge3(xp, n) if split else xp.double()


# ---------------------------------------------------------------------------------------------------------------------
# launch + canaries
# ---------------------------------------------------------------------------------------------------------------------

_WS = {}


def _splitk_ws():
    if "ws" not in _WS:
        _WS["ws"] = torch.zeros(SPLITK_BYTES // 4, device="cuda")
    return _WS["ws"]


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), device="cuda", dtype=dtype)


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def gemm_desc(**kw):
    """StaGemmDesc with the given fields; tensors stand for their data pointers"""
    d = StaGemmDesc()
    for k, v in kw.items():
        setattr(d, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    return d


def run_gemm(d, what="sta_op_gemm"):
    from vista_slam_b200._lib import check, cur_stream, lib
    check(lib().sta_op_gemm(ctypes.byref(d), cur_stream()), what)


def run_layer(e, o, split):
    """Launch layer e on the physical form of operands o (bf16, or the x3 layout when split).  Every output sits in a
    NaN-filled buffer with trailing rows / a trailing image and padding columns; the unaddressed part must keep its
    bits.  Returns the logical outputs (float64) and the physical operands the kernel read."""
    m = 3 if split else 1
    conv = e.conv is not None
    A = _phys(o["A"], split, e.taps)
    if conv:
        Wp = (split_w(o["W"], 9) if split else o["W"].bfloat16()).contiguous()
    else:
        Wp = (split_w(o["W"], e.taps) if split else o["W"].bfloat16()).contiguous()
    Kp = m * e.K
    d = StaGemmDesc()
    d.conv3x3, d.epi = int(conv), e.epi
    d.A, d.lda = A.data_ptr(), (0 if conv else Kp)
    d.W, d.ldw = Wp.data_ptr(), Kp
    d.N, d.K = e.N, Kp
    d.split_precision = int(split)
    if e.splitk:
        d.splitk_ws, d.splitk_ws_bytes = _splitk_ws().data_ptr(), SPLITK_BYTES
    keep = [A, Wp]
    if conv:
        nimg, H, W, Cin = e.conv
        d.nimg, d.H, d.Wd, d.Cin = nimg, H, W, m * Cin
        rows = (nimg, H, W)
        M = nimg * H * W
    else:
        d.M = e.M
        rows = (e.M,)
        M = e.M
    if e.bias:
        d.bias = o["bias"].data_ptr()
    outs, checks = {}, []   # checks: (buffer, before, addressed mask)

    def buffer(shape, dtype, addressed_slices):
        buf = _nan(shape, dtype)
        mask = torch.zeros(shape, dtype=torch.bool, device="cuda")
        for sl in addressed_slices:
            mask[sl] = True
        return buf, mask

    if e.epi == EPI_HEAD:
        nimg, H, W, _ = e.conv
        pts, mp = buffer((nimg + 1, H, W, 3), torch.float32, [slice(0, nimg)])
        cf, mc = buffer((nimg + 1, H, W), torch.float32, [slice(0, nimg)])
        hw = o["head_w"].t().contiguous()
        keep.append(hw)
        d.head_w, d.head_b, d.pts3d, d.conf = hw.data_ptr(), o["head_b"].data_ptr(), pts.data_ptr(), cf.data_ptr()
        checks += [(pts, pts.clone(), mp), (cf, cf.clone(), mc)]
    elif e.epi == EPI_PIXSHUF:
        k, cout, nimg, h, w = e.ps
        out, mo = buffer((nimg + 1, h * k, w * k, m * cout), torch.bfloat16, [slice(0, nimg)])
        d.out, d.ps_k, d.ps_cout, d.ps_h, d.ps_w = out.data_ptr(), k, cout, h, w
        checks.append((out, out.clone(), mo))
    else:
        f32 = e.epi == EPI_F32
        width = e.N if f32 else m * e.N
        ldo = width + (32 if f32 else 64)
        out_rows = (M // e.rowmap_n * (e.rowmap_n + 1)) if e.rowmap_n else M
        flat = (out_rows + 3, ldo)
        addr = (slice(0, out_rows), slice(0, width))
        if conv:
            nimg = e.conv[0]
            shape = (nimg + 1,) + rows[1:] + (ldo,)
            addr = (slice(0, nimg), slice(None), slice(None), slice(0, width))
        else:
            shape = flat
        out, mo = buffer(shape, torch.float32 if f32 else torch.bfloat16, [addr])
        if e.rowmap_n:
            mo[:out_rows].view(-1, e.rowmap_n + 1, ldo)[:, 0] = False  # pose-token rows
        if e.resid == "inplace":
            out[addr] = o["resid"]
            d.resid = out.data_ptr()
        d.out, d.ldo = out.data_ptr(), ldo
        checks.append((out, out.clone(), mo))
        for key in ("resid", "resid2"):
            if key in o and e.resid == "skip":
                s = _nan(shape, out.dtype)
                s[addr] = o[key] if f32 else _phys(o[key], split)
                keep.append(s)
                setattr(d, key, s.data_ptr())
                o[key + "_phys"] = s[addr]
        if e.relu_copy:
            out2, m2 = buffer(shape, torch.bfloat16, [addr])
            d.out2 = out2.data_ptr()
            checks.append((out2, out2.clone(), m2))
        d.relu_main = e.relu_main
        d.rowmap_n = e.rowmap_n
    if e.rope_cols:
        d.pos, d.rope_cols = o["pos"].data_ptr(), e.rope_cols
    run_gemm(d, "sta_op_gemm " + e.name)
    torch.cuda.synchronize()
    for buf, before, mask in checks:
        assert torch.equal(_bits(buf)[~mask], _bits(before)[~mask]), "%s: wrote outside the addressed output" % e.name
    # logical outputs
    if e.epi == EPI_HEAD:
        outs["pts3d"], outs["conf"] = pts[:-1].double(), cf[:-1].double()
    elif e.epi == EPI_PIXSHUF:
        outs["out"] = _logical(out[:-1], split, e.ps[1])
    else:
        got = out[addr]
        if e.rowmap_n:
            got = got.reshape(-1, e.rowmap_n + 1, width)[:, 1:].reshape(-1, width)
        outs["out"] = got.double() if e.epi == EPI_F32 else _logical(got, split, e.N)
        if e.relu_copy:
            outs["relu"] = _logical(out2[addr], split, e.N)
    return outs, A, Wp


# ---------------------------------------------------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------------------------------------------------

def _gemm64(A, Wp, e, images=None):
    """float64 A W^T and |A| |W|^T from the physical operands; convolutions image by image (only `images` if given)"""
    W64 = Wp.double()
    if e.conv is None:
        A64 = A.double()
        return A64 @ W64.t(), A64.abs() @ W64.abs().t()
    base, S = [], []
    for i in (range(A.shape[0]) if images is None else images):
        cols = conv_cols(A[i:i + 1])
        base.append(cols @ W64.t())
        S.append(cols.abs_() @ W64.abs().t())
        del cols
    nimg, H, W, _ = e.conv
    shp = (-1, H, W, e.N)
    return torch.cat(base).view(shp), torch.cat(S).view(shp)


def reference(e, o, A, Wp, split, images=None):
    """float64 outputs and the bound on |got - ref| for each"""
    u_out = 2.0 ** -16 if split else 2.0 ** -8
    t = tau((3 if split else 1) * e.K)
    base, S = _gemm64(A, Wp, e, images)
    sel = (lambda x: x) if images is None else (lambda x: x[list(images)])
    o["_S_max"] = float(S.max())  # the products alone (planted construction check)
    if e.bias:
        b = o["bias"].double()
        if e.ps:
            b = b.repeat(e.ps[0] ** 2)
        base = base + b
        S = S + b.abs()
    for key in ("resid", "resid2"):
        if key in o:
            r = o[key + "_phys"] if e.resid == "skip" else o[key]
            r = _logical(r, split, e.N) if e.resid == "skip" else r.double()
            if e.rowmap_n:
                r = r.reshape(-1, e.rowmap_n + 1, e.N)[:, 1:].reshape(-1, e.N)
            r = sel(r)
            base = base + r
            S = S + r.abs()
    if e.epi == EPI_F32:
        return {"out": (base, 2.0 ** -23 * base.abs() + t * S)}
    if e.epi == EPI_GELU:
        ref = F.gelu(base)
        return {"out": (ref, u_out * ref.abs() + GELU_SLOPE * t * S + 2.0 ** -20)}
    if e.epi == EPI_ROPE:
        pos = o["pos"]
        ref = rope64(base, pos, e.rope_cols)
        S2 = rope_pair_sum(S, e.rope_cols)
        ang = torch.zeros_like(base)
        ang[:, :e.rope_cols] = (2.0 ** -21 * (pos.abs().max(1).values.double() + 2))[:, None] * \
            rope_pair_sum(base.abs(), e.rope_cols)[:, :e.rope_cols]
        return {"out": (ref, u_out * ref.abs() + t * S2 + ang)}
    if e.epi == EPI_PIXSHUF:
        ref = pixshuf(base, *e.ps)
        return {"out": (ref, u_out * ref.abs() + t * pixshuf(S, *e.ps))}
    if e.epi == EPI_HEAD:
        hid = base.clamp_min(0)
        w4 = o["head_w"].double()
        b4 = o["head_b"].double()
        logits = hid @ w4.t() + b4
        err = (t * S) @ w4.abs().t() + 2.0 ** -18 * (hid @ w4.abs().t()) + 2.0 ** -24 * b4.abs()
        pts, conf = head_post(logits)
        bp, bc = head_bound(logits, err)
        return {"pts3d": (pts, bp), "conf": (conf, bc)}
    # EPI_BF16
    ref = base.clamp_min(0) if e.relu_main else base
    res = {"out": (ref, u_out * ref.abs() + t * S)}
    if e.relu_copy:
        rr = base.clamp_min(0)
        res["relu"] = (rr, u_out * rr.abs() + t * S)
    return res


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------

def _cases(x3_only):
    cases = [(sid, e) for sid, h, w, nimg, pairs, dn, x3 in SIZES if x3 or not x3_only
             for e in layer_catalogue(h, w, nimg, pairs, dn)]
    cases += [("off_model", e) for e in off_model_layers() if e.name in OFF_MODEL_X3 or not x3_only]
    return [pytest.param(sid, e, id="%s-%s" % (sid, e.name)) for sid, e in cases]


def _seed(sid, e, salt):
    return (sum(map(ord, sid + e.name)) * 7919 + salt) % (1 << 31)


def _images(sid, e):
    if sid.startswith("cfg2") and e.conv is not None:
        return CFG2_CHECKED_IMAGES
    return None


def _restrict(got, e, images):
    if images is None:
        return got
    return got[list(images)]


@pytest.fixture(autouse=True)
def _no_tf32():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("sid,e", _cases(False))
def test_layer_within_float64_bound_bf16(sid, e):
    o = make_operands(e, "random", _seed(sid, e, 1))
    outs, A, Wp = run_layer(e, o, split=False)
    images = _images(sid, e)
    refs = reference(e, o, A, Wp, False, images)
    for key, (ref, bound) in refs.items():
        check_bound("%s %s bf16 %s" % (sid, e.name, key), _restrict(outs[key], e, images), ref, bound)


@pytest.mark.parametrize("sid,e", _cases(True))
def test_layer_within_float64_bound_x3(sid, e):
    o = make_operands(e, "random", _seed(sid, e, 2))
    outs, A, Wp = run_layer(e, o, split=True)
    refs = reference(e, o, A, Wp, True)
    for key, (ref, bound) in refs.items():
        check_bound("%s %s x3 %s" % (sid, e.name, key), outs[key], ref, bound)


@pytest.mark.parametrize("sid,e", _cases(False))
def test_layer_planted_integers_bit_for_bit(sid, e):
    o = make_operands(e, "planted", _seed(sid, e, 3))
    outs, A, Wp = run_layer(e, o, split=False)
    # GELU rows are planted at pre-activations >= 6, where the kernel's fp32 gelu is the identity
    refs = reference(replace(e, epi=EPI_BF16) if e.epi == EPI_GELU else e, o, A, Wp, False)
    # products <= _S_max, |bias| <= 9, two skip tensors <= 4 each
    assert o["_S_max"] + 9 + 8 <= 256, "construction: S = %g" % o["_S_max"]
    if e.epi == EPI_GELU:
        assert float(refs["out"][0].min()) >= 6.0, "construction: a GELU pre-activation below 6"
    for key, (ref, _) in refs.items():
        name = "%s %s planted %s" % (sid, e.name, key)
        if e.epi == EPI_HEAD:  # exact logits; the fp32 post-process rounds
            check_bound(name, outs[key], ref, 2.0 ** -20 * ref.abs() + 1e-30)
        else:
            check_exact(name, outs[key], ref)


# ---------------------------------------------------------------------------------------------------------------------
# bandwidth kernels at the catalogue's sizes
# ---------------------------------------------------------------------------------------------------------------------

def _upsample_shapes():
    """(nimg, H, W, C) of run_dpt's sta_op_upsample2x-shaped calls: the refinenet3..1 outputs (C = 256) and head.0's
    output (C = 128), at every size; widths where the 4-pixel run or the block's pixel pass is ragged included"""
    out = []
    for sid, h, w, nimg, pairs, dn, _ in SIZES:
        out += [(sid, dn, h, w, 256), (sid, dn, 2 * h, 2 * w, 256), (sid, dn, 4 * h, 4 * w, 256),
                (sid, dn, 8 * h, 8 * w, 128)]
    out += [("ragged", 2, 5, 33, 256), ("ragged", 1, 3, 37, 128), ("ragged", 2, 1, 1, 256)]
    out += [("off_model", 2, 7, 9, 64), ("off_model", 1, 12, 16, 256), ("off_model", 3, 5, 3, 128),
            ("off_model", 2, 24, 32, 128), ("off_model", 1, 1, 40, 64)]
    return out


def _bilinear64(x):
    """align_corners=True bilinear x2 of NHWC float64 x with exact coordinates"""
    return F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)


@pytest.mark.parametrize("sid,nimg,H,W,C", _upsample_shapes())
def test_upsample2x_within_float64_bound(sid, nimg, H, W, C):
    """|got - ref| <= 2^-8 |ref| + 2^-12 max|x|: the output rounding, plus the kernel's fp32 coordinates (one ulp of
    the scale and one of dst * scale move the sample point by at most 2^-15 of a pixel for H, W <= 192, and the fp32
    floor may take the neighbouring cell at an exact grid point, where the interpolant is continuous) and its fp32
    arithmetic."""
    from vista_slam_b200._lib import check, cur_stream, lib
    g = torch.Generator(device="cuda").manual_seed(H * 1000 + W + C)
    x = torch.randn(nimg, H, W, C, generator=g, device="cuda").bfloat16()
    out = _nan((nimg + 1, 2 * H, 2 * W, C), torch.bfloat16)
    before = out.clone()
    check(lib().sta_op_upsample2x(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), nimg, H, W, C,
                                  cur_stream()))
    torch.cuda.synchronize()
    assert torch.equal(_bits(out[nimg:]), _bits(before[nimg:])), "wrote past the last image"
    ref = torch.cat([_bilinear64(x[i:i + 1].double()) for i in range(nimg)])
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -12 * float(x.float().abs().max())
    check_bound("upsample2x %s %dx%dx%dx%d" % (sid, nimg, H, W, C), out[:nimg], ref, bound)


@pytest.mark.parametrize("nimg,H,W,C", [(1, 14, 14, 768), (2, 3, 5, 768), (16, 24, 32, 768), (2, 7, 9, 768),
                                        (2, 3, 5, 2304), (1, 1, 1, 768), (2, 7, 10, 64)])
def test_im2col_3x3_s2_is_exact(nimg, H, W, C):
    """act3c's input: a pure copy of channel vectors, so it must equal the unfold of the input exactly"""
    from vista_slam_b200._lib import check, cur_stream, lib
    g = torch.Generator(device="cuda").manual_seed(H * W + C)
    x = torch.randn(nimg, H, W, C, generator=g, device="cuda").bfloat16()
    OH, OW = (H + 1) // 2, (W + 1) // 2
    rows = nimg * OH * OW
    out = _nan((rows + 3, 9 * C), torch.bfloat16)
    before = out.clone()
    check(lib().sta_op_im2col_3x3_s2(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), nimg, H, W, C,
                                     cur_stream()))
    torch.cuda.synchronize()
    assert torch.equal(_bits(out[rows:]), _bits(before[rows:]))
    check_exact("im2col s2 %dx%dx%dx%d" % (nimg, H, W, C), out[:rows], conv_cols(x, stride=2))


@pytest.mark.parametrize("src", ["fp32", "bf16"])
@pytest.mark.parametrize("sid,B,H,W", [(sid, nimg, 16 * h, 16 * w) for sid, h, w, nimg, _, _, _ in SIZES] +
                         [("off_model", 2, 32, 48)])
def test_patch_im2col_is_exact(sid, B, H, W, src):
    """patch_embed's input: the 16 x 16 patches of a [B][3][H][W] image as rows [B h w][768] in F.unfold's (c, ky, kx)
    order.  A bf16 image is copied exactly, an fp32 one rounded to the nearest bf16."""
    from vista_slam_b200._lib import check, cur_stream, lib
    g = torch.Generator(device="cuda").manual_seed(B * H + W)
    img = torch.rand(B, 3, H, W, generator=g, device="cuda") * 2 - 1
    if src == "bf16":
        img = img.bfloat16()
    rows = B * (H // 16) * (W // 16)
    out = _nan((rows + 3, 768), torch.bfloat16)
    before = out.clone()
    check(lib().sta_op_patch_im2col(ctypes.c_void_p(img.data_ptr()), int(src == "bf16"), B, H, W,
                                    ctypes.c_void_p(out.data_ptr()), cur_stream()))
    torch.cuda.synchronize()
    assert torch.equal(_bits(out[rows:]), _bits(before[rows:]))
    want = F.unfold(img.float(), 16, stride=16).transpose(1, 2).reshape(-1, 768).bfloat16()
    assert torch.equal(_bits(out[:rows]), _bits(want))


def _ln_cases():
    out = []
    for sid, h, w, nimg, pairs, dn, _ in SIZES:
        n = h * w
        S = 2 * pairs
        out += [(sid + "-enc", nimg * n, 1024, "single", 0), (sid + "-dec_norm1|norm_y", S * (n + 1), 768, "dual", 0),
                (sid + "-dec_norm_drop_pose", S * (n + 1), 768, "single", n + 1)]
    return out + [("off_model-dual_C1024", 1000, 1024, "dual", 0)]


def layernorm64(x, g, b, eps=1e-6):
    """float64 LayerNorm of fp32 rows x with gain g and bias b, and the bound of the kernel's fp32 arithmetic,
    2^-16 (|g| (|z| + max|x_row| / std) + |b|), without the output rounding"""
    x64 = x.double()
    mu = x64.mean(1, keepdim=True)
    std = (x64.var(1, unbiased=False, keepdim=True) + eps).sqrt()
    z = (x64 - mu) / std
    xmax = x64.abs().max(1, keepdim=True).values / std
    gg, bb = g.double(), b.double()
    return z * gg + bb, 2.0 ** -16 * (gg.abs() * (z.abs() + xmax) + bb.abs())


@pytest.mark.parametrize("sid,rows,C,form,drop", _ln_cases())
def test_layernorm_within_float64_bound(sid, rows, C, form, drop):
    """|got - ref| <= 2^-8 |ref| + 2^-16 (|g| (|z| + max|x_row| / std) + |b|), z the float64 normalised value: the bf16
    output rounding, plus the fp32 mean, variance and normalisation (a few ulps of the row's magnitude after scaling
    by rstd)."""
    from vista_slam_b200._lib import check, cur_stream, lib
    g = torch.Generator(device="cuda").manual_seed(rows + C + drop)
    x = torch.randn(rows, C, generator=g, device="cuda") * 3 + 0.5
    params = [torch.randn(C, generator=g, device="cuda") for _ in range(4)]
    out_rows = rows // drop * (drop - 1) if drop else rows
    outs = [_nan((out_rows + 3, C), torch.bfloat16) for _ in range(2 if form == "dual" else 1)]
    befores = [t.clone() for t in outs]
    P = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    dual = form == "dual"
    check(lib().sta_op_layernorm(P(x), rows, C, 1e-6, P(params[0]), P(params[1]), P(outs[0]),
                                 P(params[2]) if dual else None, P(params[3]) if dual else None,
                                 P(outs[1]) if dual else None, drop, cur_stream()))
    torch.cuda.synchronize()
    keep = (torch.arange(rows, device="cuda") % drop) != 0 if drop else slice(None)
    for i, o in enumerate(outs):
        ref, b32 = layernorm64(x, params[2 * i], params[2 * i + 1])
        ref, b32 = ref[keep], b32[keep]
        bound = 2.0 ** -8 * ref.abs() + b32
        assert torch.equal(_bits(o[out_rows:]), _bits(befores[i][out_rows:]))
        check_bound("layernorm %s out%d" % (sid, i + 1), o[:out_rows], ref, bound)


@pytest.mark.parametrize("sid,rows,C,drop", [(s, S * (h * w + 1), 768, h * w + 1) for s, h, w, _, p, _, _ in SIZES
                                             for S in (2 * p,)] + [("enc_features", 196, 1024, 0)])
def test_cast_f32_bf16_is_round_to_nearest(sid, rows, C, drop):
    """the decoder hooks (pose row dropped) and the encoder features: the bf16 rounding of each fp32 value, exactly"""
    from vista_slam_b200._lib import check, cur_stream, lib
    g = torch.Generator(device="cuda").manual_seed(rows + C)
    x = torch.randn(rows, C, generator=g, device="cuda") * torch.exp2(torch.randint(-20, 20, (rows, 1), generator=g,
                                                                                    device="cuda").float())
    out_rows = rows // drop * (drop - 1) if drop else rows
    out = _nan((out_rows + 3, C), torch.bfloat16)
    before = out.clone()
    check(lib().sta_op_cast_f32_bf16(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), rows, C, drop,
                                     cur_stream()))
    torch.cuda.synchronize()
    want = x.view(-1, drop, C)[:, 1:].reshape(-1, C) if drop else x
    assert torch.equal(_bits(out[out_rows:]), _bits(before[out_rows:]))
    assert torch.equal(_bits(out[:out_rows]), _bits(want.bfloat16().contiguous()))
