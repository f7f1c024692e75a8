"""GPU: every launch of the FP8 mode (STA(precision="fp8")) at the model's shapes -- the e4m3 GEMMs (A_FP8 x EPI_F32 /
EPI_ROPE / EPI_GELU_FP8) and the two quantisers -- against float64 with a bound on every output element, against planted
answers bit for bit, and with NaN canaries around every output; the e4m3 weights the loader packs, bit for bit against
oracle/fp8_oracle.py; and a probe that pins down how the FP8 tensor-core instruction accumulates.

The launch list is fp8_catalogue(): it restates the FP8 branches of run_encoder (runtime.cu:898-907) and run_decoder
(runtime.cu:942-958) one launch at a time, at the sizes of tests/test_layers_gpu.py plus one OnlineSLAM.step_many chunk.
Every EPI_F32 launch gets the model's 48 MiB split-K workspace poisoned with NaN, and the test asserts that split-K ran
with the factor the rule of gemm.cu (restated in split_factor) predicts, or did not run.

Float64 check.  Random e4m3 codes with power-of-two scales that differ per row and k-block (activations) and per
128 x 128 block (weights); a scale applied to the wrong row, k-block or block moves the result far outside the bound.
The reference is the float64 product of the dequantised operands, plus bias and residual.  Per element:

    |got - ref| <= u_out |ref| + T,   T = EPS_BLK P + 2^-23 (K / 128 + 8) S,
    P = sum_k |a_k w_k|,   S = P + |bias| (+ |resid|)

  * The kernel runs one wgmma k-block of 128 (four k32 instructions) into a zeroed block accumulator, then folds it into
    the fp32 tile as acc = fma(blk, a_scale[row] w_scale, acc).  The scales are powers of two, so the products of the
    dequantised operands are exact and only the block sum and the folds round.
  * EPS_BLK bounds the block sum: |blk - exact| <= EPS_BLK P_blk, P_blk = sum over the block of |a_k w_k|.  It is derived
    from test_wgmma_e4m3_accumulation_probe, which records how the instruction accumulates (see PROBE_* below).  Bias and
    residual never pass through the tensor core, so only the fp32 term applies to them.
  * The fp32 arithmetic after it: K / 128 folds, the bias add, and on the split-K route at most 8 partial sums and the
    residual add; each rounds by at most 2^-24 of a partial sum, and every partial sum is at most S.  2^-23 per step
    covers that twice over.  u_out = 2^-23 for the fp32 stream, 2^-8 for bf16 (RoPE) outputs.
  * RoPE: both elements of a rotated pair get T_a + T_b, plus 2^-21 (|pos| + 2) (|a| + |b|) for the fp32 angle of
    the kernel's table and the fp32 rotation, as in test_layers_gpu.py.
  * GELU_FP8: the fp32 value the kernel quantises is within B = 1.1289 T + 2^-20 + 2^-23 |gelu| of the exact-erf
    gelu of the float64 pre-activation (max |gelu'| = 1.1289; 2^-20 for the fitted gelu_erf, 5e-7 absolute; the last
    rounding).  LayerNorm-fp8: B = 2^-16 (|g| (|z| + max|x_row| / std) + |b|), the fp32 part of the bound of
    test_layers_gpu.py::test_layernorm_within_float64_bound.
  * e4m3 outputs (check_codes): a group's scale must equal fp8_scale of the float64 amax over its 128 columns, unless
    that amax lies within the group's largest B of a boundary 448 * 2^e (then the neighbouring scale is accepted too).
    Where the scales agree, every code must be the round-to-nearest-even, saturating e4m3 value of ref / s, unless
    ref / s lies within B / s of a rounding midpoint: then every code RNE takes on [ref - B, ref + B] / s is accepted.
    The elements each exception admits are counted and must stay below MAX_EXCEPTION_FRAC of the output.
  * quant_fp8 is bit-identical to oracle/fp8_oracle.py quantize_rows.
  * EPS_BLK is a worst case, far above what random operands reach (MEASURED_RATIO).  The fp32 and RoPE checks still
    catch a misapplied scale, a dropped k-block or k32 slice because the operands' power-of-two scales differ by up to
    2^11 between rows, k-blocks and weight blocks, so such a fault moves an output by many times its bound
    (tests/test_layers_fp8_cpu.py).  Operands with uniform scales would not give that margin: keep the spread.

Planted answers.  Small-integer codes with power-of-two scales: every product is a multiple of 2^-2 (1 in GELU rows), the
block sums are small integers, and every output is exact in fp32 and bf16 in any summation order.  Weight rows are
distinct, with nonzeros in several k-blocks under different block scales.  RoPE rows sit at position (0, 0).  GELU rows
sit at pre-activations in [6, 15] (where gelu_erf is the identity in fp32; integers below 16 lie on the e4m3 grid at any
power-of-two scale) or exactly 0; one row's largest value is exactly 448 (scale 1), another's 480 (scale 2).  A second
planted GELU_FP8 set covers the nonlinear region: codes -1, 0, 1 with scales 1/2 and 1 give exact pre-activations, all
multiples of 2^-2 in [-6, 6], so every code, negative ones included, and every scale is held to RNE(gelu_erf64 / s)
with only the fitted gelu's slack.

Canaries.  Every output has three trailing rows of NaN (e4m3 code 0x7F, NaN scales, NaN past the fp32 stream's M rows)
that must keep their bits; one RoPE output also has 64 padding columns."""
import ctypes
import math
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from oracle.fp8_oracle import fp8_scale, quantize_blocks, quantize_rows
from test_layers_gpu import (GELU_SLOPE, SIZES, SPLITK_BYTES, _bits, _nan, check_bound, check_exact, positions,
                             rope64, rope_pair_sum)
from vista_slam_b200._lib import EPI_F32, EPI_GELU_FP8, EPI_ROPE, StaGemmFp8Desc

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn
NAN_E4M3 = 0x7F
# How one wgmma m64n128k32 e4m3 instruction accumulates, recorded by test_wgmma_e4m3_accumulation_probe on an H100 80GB
# HBM3 (700 W power limit): its 33 terms (the accumulator and 32 exact products) are aligned to the exponent E of the
# largest and each is truncated toward zero to a multiple of 2^(E - PROBE_KEPT_BITS); the sum of those is exact in fp32.
# A product below 2^-13 of the largest term is lost; 1.5 x 2^-5 beside 2^8 keeps 2^-5, with either sign.
PROBE_KEPT_BITS = 13
# So one instruction is off by less than 33 x 2^-13 of its largest term, which is at most S_blk; a k-block is four.
EPS_BLK = 4 * 33 * 2.0 ** -PROBE_KEPT_BITS
# Largest err / bound of the float64 checks, H100 80GB HBM3 (700 W power limit), all four sizes: fp32-output layers
# 0.021 (enc.proj at cfg-2), RoPE outputs 0.096 (enc.qkv at cfg-2; the bf16 output rounding dominates).  Largest share
# of an output's codes an exception admitted: LayerNorm-fp8 8.4e-3, planted nonlinear GELU_FP8 1.6e-3 (values within
# the fitted gelu's 2^-20 of a subnormal midpoint), random GELU_FP8 all of them.  The file (145 cases with
# tests/test_layers_fp8_cpu.py) runs in about 8 s.
MEASURED_RATIO = {"f32_out": 0.021, "rope": 0.096}
# Largest share of an output's e4m3 codes that a midpoint or scale-boundary exception may admit:
#   ln: LayerNorm-fp8 (8.4e-3 measured);
#   gelu_nonlinear: GELU_FP8 on exact pre-activations in [-6, 6] (test_fp8_gelu_planted_nonlinear_codes), where only
#     the fitted gelu and its rounding are left (1.6e-3 measured);
#   gelu_random: GELU_FP8 on random operands.  There the worst-case block term EPS_BLK sum|a w| is wider than an e4m3
#     step on most elements (sum|a w| is many times |gelu|), so that check is a bound on each code's value, no tighter;
#     the codes are pinned by the planted tests above.
MAX_EXCEPTION_FRAC = {"ln": 0.02, "gelu_nonlinear": 5e-3, "gelu_random": 1.0}
# Split-K factors the catalogue's EPI_F32 launches take on a 132-SM H100 (gemm.cu:93-103).
SPLIT_FACTORS_COVERED = {1, 2, 3, 4, 5, 8}


def fold_tau(K):
    """the fp32 steps after the tensor core: K / 128 folds, bias, split-K partials, residual"""
    return 2.0 ** -23 * (K / 128 + 8)


# ---------------------------------------------------------------------------------------------------------------------
# the catalogue
# ---------------------------------------------------------------------------------------------------------------------

@dataclass(frozen=True)
class Fp8Launch:
    name: str
    kind: str                 # "gemm" | "ln" | "quant"
    epi: int = -1
    M: int = 0                # rows
    N: int = 0                # gemm: output columns; ln / quant: C
    K: int = 0
    rope_cols: int = 0
    pos_grid: tuple = None    # RoPE positions: (samples, h, w, with_pose_token) as launch_make_positions builds them
    dual: bool = False        # ln: the decoder's second affine output (norm_y)


def fp8_catalogue(h, w, nimg, pairs):
    """The FP8-mode launches of one forward pass through the trunk: encoder over nimg images of h x w tokens, decoder
    over `pairs` pairs (2 * pairs samples of h w + 1 rows, the pose token first)."""
    T = nimg * h * w
    enc_pos = (nimg, h, w, 0)
    L = [  # run_encoder, FP8 branch
        Fp8Launch("enc.norm1", "ln", M=T, N=1024),                                          # runtime.cu:899
        Fp8Launch("enc.qkv", "gemm", EPI_ROPE, T, 3072, 1024, 2048, enc_pos),               # runtime.cu:900
        Fp8Launch("enc.attn_out", "quant", M=T, N=1024),                                    # runtime.cu:903
        Fp8Launch("enc.proj", "gemm", EPI_F32, T, 1024, 1024),                              # runtime.cu:904
        Fp8Launch("enc.norm2", "ln", M=T, N=1024),                                          # runtime.cu:905
        Fp8Launch("enc.fc1", "gemm", EPI_GELU_FP8, T, 4096, 1024),                          # runtime.cu:906
        Fp8Launch("enc.fc2", "gemm", EPI_F32, T, 1024, 4096),                               # runtime.cu:907
    ]
    S = 2 * pairs
    Td = S * (h * w + 1)
    dec_pos = (S, h, w, 1)
    L += [  # run_decoder, FP8 branch
        Fp8Launch("dec.norm1|norm_y", "ln", M=Td, N=768, dual=True),                        # runtime.cu:943
        Fp8Launch("dec.qkv", "gemm", EPI_ROPE, Td, 2304, 768, 1536, dec_pos),               # runtime.cu:944
        Fp8Launch("dec.attn_out", "quant", M=Td, N=768),                                    # runtime.cu:947
        Fp8Launch("dec.proj", "gemm", EPI_F32, Td, 768, 768),                               # runtime.cu:948
        Fp8Launch("dec.projk|projv", "gemm", EPI_ROPE, Td, 1536, 768, 768, dec_pos),        # runtime.cu:949
        Fp8Launch("dec.norm2", "ln", M=Td, N=768),                                          # runtime.cu:950
        Fp8Launch("dec.projq", "gemm", EPI_ROPE, Td, 768, 768, 768, dec_pos),               # runtime.cu:951
        Fp8Launch("dec.cross_attn_out", "quant", M=Td, N=768),                              # runtime.cu:954
        Fp8Launch("dec.cproj", "gemm", EPI_F32, Td, 768, 768),                              # runtime.cu:955
        Fp8Launch("dec.norm3", "ln", M=Td, N=768),                                          # runtime.cu:956
        Fp8Launch("dec.fc1", "gemm", EPI_GELU_FP8, Td, 3072, 768),                          # runtime.cu:957
        Fp8Launch("dec.fc2", "gemm", EPI_F32, Td, 768, 3072),                               # runtime.cu:958
    ]
    return L


# (id, h, w, trunk images, pairs): test_layers_gpu.SIZES (keyframe, odd, cfg-2) and one OnlineSLAM.step_many chunk of
# four keyframes and three edge pairs
FP8_SIZES = [(sid, h, w, nimg, pairs) for sid, h, w, nimg, pairs, _, _ in SIZES] + [("step_many4_14x14", 14, 14, 4, 3)]


def split_factor(e, sms):
    """gemm.cu:93-103: the split-K factor of an EPI_F32 launch with the model's workspace (1 = not split)"""
    if e.kind != "gemm" or e.epi != EPI_F32:
        return 1
    m_tiles, nkb = (e.M + 127) // 128, e.K // 128
    tiles = m_tiles * (e.N // 128)
    if tiles >= sms:
        return 1
    ks = min(sms // tiles, 8, nkb // 2)
    return ks if ks >= 2 and ks * m_tiles * 128 * e.N * 4 <= SPLITK_BYTES else 1


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------------
# helpers that need no GPU (tests/test_layers_fp8_cpu.py feeds them faulty outputs)
# ---------------------------------------------------------------------------------------------------------------------

def dequant_rows(q, s):
    """e4m3 codes [rows][K] (float8 or uint8) and scales [rows][K / 128] -> float64"""
    q = q.view(E4M3) if q.dtype == torch.uint8 else q
    return (q.float().double().view(q.shape[0], -1, 128) * s.double()[..., None]).view(q.shape)


def dequant_blocks(q, s):
    q = q.view(E4M3) if q.dtype == torch.uint8 else q
    N, K = q.shape
    return (q.float().double().view(N // 128, 128, K // 128, 128) * s.double()[:, None, :, None]).view(N, K)


def e4m3_ord(codes):
    """e4m3 codes (uint8) -> integers monotonic in the value (sign-magnitude; -0 = +0)"""
    c = codes.to(torch.int32)
    return torch.where(c >= 128, -(c - 128), c)


def _rne_range(v, b):
    """ord range of the codes RNE takes on [v - b, v + b] (RNE and saturation are monotonic)"""
    lo_x = (v - b).float()
    lo_x = torch.where(lo_x.double() > v - b, torch.nextafter(lo_x, torch.full_like(lo_x, -math.inf)), lo_x)
    hi_x = (v + b).float()
    hi_x = torch.where(hi_x.double() < v + b, torch.nextafter(hi_x, torch.full_like(hi_x, math.inf)), hi_x)
    enc = lambda x: e4m3_ord(x.clamp(-448, 448).to(E4M3).view(torch.uint8))  # noqa: E731
    return enc(lo_x), enc(hi_x)


def check_codes(name, q, s, ref, bound, max_frac):
    """e4m3 output q (uint8 [rows][C]) with scales s ([rows][C / 128]) against the float64 reference of the fp32 values
    the kernel quantised, each known to `bound`.  Returns the share of codes that an exception admitted."""
    rows, C = ref.shape
    G = C // 128
    r3, b3 = ref.view(rows, G, 128), bound.view(rows, G, 128)
    amax, bmax = r3.abs().amax(-1), b3.amax(-1)
    s_ref = fp8_scale(amax.float())[0]
    s = s.float()
    e = torch.round(torch.log2(amax.clamp_min(1e-300) / 448.0))
    near = ((448.0 * torch.exp2(e) - amax).abs() <= bmax) & (amax > 0)
    neighbour = (s == 2 * s_ref) | (s == 0.5 * s_ref)
    bad = (s != s_ref) & ~(near & neighbour)
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d scales wrong; first %s: got %r want %r (amax %r)" % (
            name, int(bad.sum()), bad.numel(), i, float(s[i]), float(s_ref[i]), float(amax[i])))
    same = (s == s_ref)[..., None].expand(rows, G, 128)
    sd = s.double()[..., None]
    lo, hi = _rne_range(r3 / sd, b3 / sd)
    got = e4m3_ord(q.view(rows, G, 128))
    wrong = same & ((got < lo) | (got > hi))
    if bool(wrong.any()):
        i = tuple(wrong.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d codes wrong; first %s: got ord %d, allowed [%d, %d] (ref / s = %r)" % (
            name, int(wrong.sum()), wrong.numel(), i, int(got[i]), int(lo[i]), int(hi[i]), float(r3[i] / sd[i[:2]])))
    n_mid = int((same & (lo != hi)).sum())
    n_scale = int((~same).sum())
    frac = (n_mid + n_scale) / ref.numel()
    print("codes %-44s midpoint exceptions %d, scale exceptions %d of %d (%.2e)" % (name, n_mid, n_scale, ref.numel(),
                                                                                   frac), flush=True)
    assert frac <= max_frac, "%s: exceptions admit %.3g of the codes" % (name, frac)
    return frac


def check_canaries(name, buf, before, mask):
    """the unaddressed part (mask False) of an output buffer must keep its bits"""
    b = buf.view(torch.uint8) if buf.element_size() == 1 else _bits(buf)
    b0 = before.view(torch.uint8) if before.element_size() == 1 else _bits(before)
    assert torch.equal(b[~mask], b0[~mask]), "%s: wrote outside the addressed output" % name


def make_fp8_operands(e, kind, seed, dev="cuda"):
    """e4m3 codes + power-of-two scales of a gemm launch: 'random', 'planted' or, for GELU_FP8, 'planted_nonlinear'
    (see the module docstring)"""
    g = torch.Generator(device=dev).manual_seed(seed)
    M, N, K = e.M, e.N, e.K
    nkb = K // 128
    ri = lambda lo, hi, shape: torch.randint(lo, hi, shape, generator=g, device=dev)  # noqa: E731
    o = {}
    if kind == "random":
        o["aq"] = (torch.randn(M, K, generator=g, device=dev) * 64).clamp(-448, 448).to(E4M3)
        o["as"] = torch.exp2(ri(-10, -4, (M, nkb)).float())
        o["wq"] = (torch.randn(N, K, generator=g, device=dev) * 64).clamp(-448, 448).to(E4M3)
        o["ws"] = torch.exp2(ri(-3, 4, (N // 128, nkb)).float() - 6 - round(math.log2(math.sqrt(K))))
        o["bias"] = torch.randn(N, generator=g, device=dev) * 0.1
        if e.epi == EPI_F32:
            o["resid"] = torch.randn(M, N, generator=g, device=dev)
        if e.epi == EPI_ROPE:
            o["pos"] = positions(e.pos_grid, dev)
        return o
    if kind == "planted_nonlinear":
        # a in {-1, 0, 1} x {1/2, 1}, four weights +-1 x {1/2, 1} per row, bias a multiple of 1/4 in [-2, 2]:
        # pre-activations are multiples of 1/4 in [-6, 6], exact in any summation order
        o["aq"] = ri(-1, 2, (M, K)).float().to(E4M3)
        o["as"] = torch.exp2(ri(-1, 1, (M, nkb)).float())
        Wt = torch.zeros(N, K, device=dev)
        start = ri(0, nkb, (N,))
        for j in range(4):
            col = ((start + (j * nkb) // 4) % nkb) * 128 + ri(0, 128, (N,))
            Wt[torch.arange(N, device=dev), col] = (ri(0, 2, (N,)) * 2 - 1).float()
        o["wq"] = Wt.to(E4M3)
        o["ws"] = torch.exp2(ri(-1, 1, (N // 128, nkb)).float())
        o["bias"] = ri(-8, 9, (N,)).float() / 4
        return o
    gelu = e.epi == EPI_GELU_FP8
    # GELU: a, w >= 0, products <= 4, two per row, bias 6 or 7: pre-activations in [6, 15].  Otherwise |products| <= 8
    # on the grid 2^-2, four per row, |bias| <= 4: |outputs| <= 36, exact in bf16.
    o["aq"] = (ri(0, 2, (M, K)) if gelu else ri(-2, 3, (M, K))).float().to(E4M3)
    o["as"] = torch.exp2(ri(0, 2, (M, nkb)).float() if gelu else ri(-1, 2, (M, nkb)).float())
    nz = 2 if gelu else 4
    Wt = torch.zeros(N, K, device=dev)
    start = ri(0, nkb, (N,))
    rows = torch.arange(N, device=dev)
    for j in range(nz):
        col = ((start + (j * nkb) // nz) % nkb) * 128 + ri(0, 128, (N,))
        val = torch.ones(N, device=dev) if gelu else (ri(0, 2, (N,)) * 2 - 1).float()
        Wt[rows, col] = val
    o["ws"] = torch.exp2(ri(0, 2, (N // 128, nkb)).float() if gelu else ri(-1, 2, (N // 128, nkb)).float())
    o["bias"] = (ri(6, 8, (N,)) if gelu else ri(-4, 5, (N,))).float()
    if gelu:
        # column n0 reads only k_star: 448 in row 0 (scale 1), 480 = 240 x 2 in the last row, 0 elsewhere
        n0, k_star = N - 128 + 5, K - 1
        Wt[:, k_star] = 0
        Wt[n0] = 0
        Wt[n0, k_star] = 1
        o["ws"][n0 // 128, nkb - 1] = 1
        aq = o["aq"].float()
        aq[:, k_star] = 0
        aq[0, k_star], aq[M - 1, k_star] = 448, 240
        o["aq"] = aq.to(E4M3)
        o["as"][0, nkb - 1], o["as"][M - 1, nkb - 1] = 1, 2
        o["bias"][n0] = 0
    o["wq"] = Wt.to(E4M3)
    if e.epi == EPI_F32:
        o["resid"] = ri(-4, 5, (M, N)).float()
    if e.epi == EPI_ROPE:
        o["pos"] = torch.zeros(M, 2, dtype=torch.int32, device=dev)
    return o


def gemm_reference(e, o, rope_cols=None):
    """float64 output of a gemm launch and the bound on |got - ref| (GELU_FP8: on the fp32 value before quantisation)"""
    A64, W64 = dequant_rows(o["aq"], o["as"]), dequant_blocks(o["wq"], o["ws"])
    base = A64 @ W64.t() + o["bias"].double()
    # EPS_BLK applies to the products (the tensor-core block sums), the fp32 steps to everything that is summed
    T = EPS_BLK * (A64.abs() @ W64.abs().t())
    del A64, W64
    S = T / EPS_BLK + o["bias"].double().abs()
    if e.epi == EPI_F32:
        base += o["resid"].double()
        S += o["resid"].double().abs()
    T += fold_tau(e.K) * S
    del S
    if e.epi == EPI_F32:
        return base, 2.0 ** -23 * base.abs() + T
    if e.epi == EPI_ROPE:
        rc = e.rope_cols if rope_cols is None else rope_cols
        pos = o["pos"]
        ref = rope64(base, pos, rc)
        ang = torch.zeros_like(base)
        ang[:, :rc] = (2.0 ** -21 * (pos.abs().max(1).values.double() + 2))[:, None] * \
            rope_pair_sum(base.abs(), rc)[:, :rc]
        return ref, 2.0 ** -8 * ref.abs() + rope_pair_sum(T, rc) + ang
    ref = F.gelu(base)
    return ref, GELU_SLOPE * T + 2.0 ** -20 + 2.0 ** -23 * ref.abs()


def gelu_planted_reference(o):
    """GELU_FP8 on 'planted_nonlinear' operands: the pre-activations are exact (multiples of 2^-2 in [-6, 6]), so the
    fp32 value the kernel quantises is within 2^-20 + 2^-23 |gelu| of the exact-erf gelu"""
    pre = dequant_rows(o["aq"], o["as"]) @ dequant_blocks(o["wq"], o["ws"]).t() + o["bias"].double()
    assert float(pre.abs().max()) <= 6 and bool((pre * 4 == (pre * 4).round()).all()), "construction: pre-activations"
    ref = F.gelu(pre)
    return pre, ref, 2.0 ** -20 + 2.0 ** -23 * ref.abs()


# ---------------------------------------------------------------------------------------------------------------------
# launches
# ---------------------------------------------------------------------------------------------------------------------

_WS = {}


def _splitk_ws():
    if "ws" not in _WS:
        _WS["ws"] = torch.empty(SPLITK_BYTES // 4, device="cuda")
    return _WS["ws"]


def _u8(t):
    return t.view(torch.uint8)


def run_gemm(e, o, ldo_pad=0):
    """Launch gemm e on operands o the way linear_fp8 (runtime.cu:593-607) does, with the model's split-K workspace
    poisoned with NaN; check the canaries and the split-K factor.  Returns the output (and scales for GELU_FP8)."""
    from vista_slam_b200._lib import check, cur_stream, lib
    M, N, K = e.M, e.N, e.K
    ws = _splitk_ws()
    ws.fill_(float("nan"))
    d = StaGemmFp8Desc()
    d.epi, d.M, d.N, d.K = e.epi, M, N, K
    d.A, d.lda, d.a_scale = _u8(o["aq"]).data_ptr(), K, o["as"].data_ptr()
    d.W, d.ldw, d.w_scale = _u8(o["wq"]).data_ptr(), K, o["ws"].data_ptr()
    d.bias = o["bias"].data_ptr()
    d.splitk_ws, d.splitk_ws_bytes = ws.data_ptr(), SPLITK_BYTES
    checks = []
    if e.epi == EPI_F32:   # the fp32 residual stream, updated in place
        out = _nan((M + 3, N), torch.float32)
        out[:M] = o["resid"]
        d.out, d.ldo, d.resid = out.data_ptr(), N, out.data_ptr()
        mask = torch.zeros(out.shape, dtype=torch.bool, device="cuda")
        mask[:M] = True
        checks.append((out, out.clone(), mask))
        res = (out,)
    elif e.epi == EPI_ROPE:
        ldo = N + ldo_pad
        out = _nan((M + 3, ldo), torch.bfloat16)
        d.out, d.ldo = out.data_ptr(), ldo
        d.pos, d.rope_cols = o["pos"].data_ptr(), e.rope_cols
        mask = torch.zeros(out.shape, dtype=torch.bool, device="cuda")
        mask[:M, :N] = True
        checks.append((out, out.clone(), mask))
        res = (out,)
    else:
        q = torch.full((M + 3, N), NAN_E4M3, dtype=torch.uint8, device="cuda")
        s = _nan((M + 3, N // 128), torch.float32)
        d.out, d.ldo, d.out_scale = q.data_ptr(), N, s.data_ptr()
        for buf in (q, s):
            mask = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
            mask[:M] = True
            checks.append((buf, buf.clone(), mask))
        res = (q, s)
    check(lib().sta_op_gemm_fp8(ctypes.byref(d), cur_stream()), "sta_op_gemm_fp8 " + e.name)
    torch.cuda.synchronize()
    for buf, before, mask in checks:
        check_canaries(e.name, buf, before, mask)
    ks = split_factor(e, _sms())
    if ks > 1:
        rows = (M + 127) // 128 * 128
        used = ws[:ks * rows * N].view(ks, rows, N)
        assert bool(torch.isfinite(used[:, :M]).all()), "%s: split-K x%d did not write every partial" % (e.name, ks)
        assert bool(ws[ks * rows * N:].isnan().all()), "%s: split-K wrote past %d partials" % (e.name, ks)
    else:
        assert bool(ws.isnan().all()), "%s: split-K ran, the rule predicts no split" % e.name
    if e.epi == EPI_GELU_FP8:
        return res[0][:M], res[1][:M]
    return res[0][:M, :N]


def run_ln(e, x, params):
    """sta_op_layernorm_fp8 as ln_fp8 (runtime.cu:630-636) calls it; checks the canaries"""
    from vista_slam_b200._lib import check, cur_stream, lib
    rows, C = e.M, e.N
    outs = [(torch.full((rows + 3, C), NAN_E4M3, dtype=torch.uint8, device="cuda"), _nan((rows + 3, C // 128), torch.float32))
            for _ in range(2 if e.dual else 1)]
    befores = [(q.clone(), s.clone()) for q, s in outs]
    P = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    g1, b1, g2, b2 = params
    q2, s2 = outs[1] if e.dual else (None, None)
    check(lib().sta_op_layernorm_fp8(P(x), rows, C, 1e-6, P(g1), P(b1), P(outs[0][0]), P(outs[0][1]),
                                     P(g2) if e.dual else None, P(b2) if e.dual else None, P(q2), P(s2), cur_stream()),
          "sta_op_layernorm_fp8 " + e.name)
    torch.cuda.synchronize()
    for (q, s), (q0, s0) in zip(outs, befores):
        for buf, before in ((q, q0), (s, s0)):
            mask = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
            mask[:rows] = True
            check_canaries(e.name, buf, before, mask)
    return [(q[:rows], s[:rows]) for q, s in outs]


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------

def _cases(kinds):
    return [pytest.param(sid, e, id="%s-%s" % (sid, e.name))
            for sid, h, w, nimg, pairs in FP8_SIZES for e in fp8_catalogue(h, w, nimg, pairs) if e.kind in kinds]


def _seed(sid, e, salt):
    return (sum(map(ord, sid + e.name)) * 7919 + salt) % (1 << 31)


@pytest.fixture(autouse=True)
def _no_tf32():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("sid,e", _cases(("gemm",)))
def test_fp8_gemm_within_float64_bound(sid, e):
    o = make_fp8_operands(e, "random", _seed(sid, e, 1))
    got = run_gemm(e, o)
    ref, bound = gemm_reference(e, o)
    name = "%s %s" % (sid, e.name)
    if e.epi == EPI_GELU_FP8:
        q, s = got
        check_codes(name, q, s, ref, bound, MAX_EXCEPTION_FRAC["gelu_random"])
    else:
        check_bound(name, got, ref, bound)


@pytest.mark.parametrize("sid,e", _cases(("gemm",)))
def test_fp8_gemm_planted_bit_for_bit(sid, e):
    o = make_fp8_operands(e, "planted", _seed(sid, e, 2))
    got = run_gemm(e, o)
    A64, W64 = dequant_rows(o["aq"], o["as"]), dequant_blocks(o["wq"], o["ws"])
    ref = A64 @ W64.t() + o["bias"].double()
    name = "%s %s planted" % (sid, e.name)
    if e.epi == EPI_F32:
        check_exact(name, got, ref + o["resid"].double())
    elif e.epi == EPI_ROPE:  # position (0, 0): the rotation is the identity
        assert float(ref.abs().max()) <= 36 and bool((ref * 4 == (ref * 4).round()).all()), "construction"
        check_exact(name, got, ref)
    else:
        big = ref.abs() > 15
        assert bool(((ref == 0) | ((ref >= 6) & (ref <= 15)) | big).all()), "construction: pre-activations"
        assert float(ref[0].max()) == 448 and float(ref[-1].max()) == 480, "construction: 448 / 480 rows"
        q, s = got
        q_ref, s_ref = quantize_rows(ref.float())
        check_exact(name + " scales", s, s_ref.double())
        assert float(s[0, -1]) == 1 and float(s[-1, -1]) == 2
        bad = _u8(q_ref) != q
        if bool(bad.any()):
            i = tuple(bad.nonzero()[0].tolist())
            raise AssertionError("%s: %d codes differ; first %s: got %d want %d" % (name, int(bad.sum()), i, int(q[i]),
                                                                                   int(_u8(q_ref)[i])))


@pytest.mark.parametrize("sid,e", [c for c in _cases(("gemm",)) if c.values[1].epi == EPI_GELU_FP8])
def test_fp8_gelu_planted_nonlinear_codes(sid, e):
    """GELU_FP8 where gelu is not the identity: exact pre-activations, multiples of 2^-2 in [-6, 6], so every scale and
    code is checked against RNE(gelu_erf64 / s) with only the fitted gelu's 2^-20 + 2^-23 |gelu| of slack; negative
    codes included"""
    o = make_fp8_operands(e, "planted_nonlinear", _seed(sid, e, 5))
    q, s = run_gemm(e, o)
    pre, ref, bound = gelu_planted_reference(o)
    assert float(pre.min()) < -3 and float(pre.max()) > 3 and bool((ref < -0.1).any()), "construction: coverage"
    check_codes("%s %s planted nonlinear" % (sid, e.name), q, s, ref, bound, MAX_EXCEPTION_FRAC["gelu_nonlinear"])
    assert bool((q > 0x80).any()), "construction: no negative code"


@pytest.mark.parametrize("sid,e", _cases(("ln",)))
def test_layernorm_fp8_within_float64_bound(sid, e):
    g = torch.Generator(device="cuda").manual_seed(_seed(sid, e, 3))
    rows, C = e.M, e.N
    x = torch.randn(rows, C, generator=g, device="cuda") * 3 + torch.randn(rows, 1, generator=g, device="cuda")
    params = [1 + 0.3 * torch.randn(C, generator=g, device="cuda") if i % 2 == 0 else
              0.1 * torch.randn(C, generator=g, device="cuda") for i in range(4)]
    outs = run_ln(e, x, params)
    x64 = x.double()
    mu = x64.mean(1, keepdim=True)
    std = (x64.var(1, unbiased=False, keepdim=True) + 1e-6).sqrt()
    z = (x64 - mu) / std
    xmax = x64.abs().max(1, keepdim=True).values / std
    for i, (q, s) in enumerate(outs):
        gg, bb = params[2 * i].double(), params[2 * i + 1].double()
        ref = z * gg + bb
        bound = 2.0 ** -16 * (gg.abs() * (z.abs() + xmax) + bb.abs())
        check_codes("%s %s out%d" % (sid, e.name, i + 1), q, s, ref, bound, MAX_EXCEPTION_FRAC["ln"])


@pytest.mark.parametrize("sid,e", _cases(("quant",)))
def test_quant_fp8_bit_identical_to_oracle(sid, e):
    from vista_slam_b200._lib import check, cur_stream, lib
    g = torch.Generator(device="cuda").manual_seed(_seed(sid, e, 4))
    rows, C = e.M, e.N
    x = (torch.randn(rows, C, generator=g, device="cuda") *
         torch.exp2(torch.randint(-20, 20, (rows, C // 128), generator=g, device="cuda").float()).repeat_interleave(128, 1))
    x[rows // 2, :128] = 0  # an all-zero group: scale 1
    x = x.bfloat16()
    q = torch.full((rows + 3, C), NAN_E4M3, dtype=torch.uint8, device="cuda")
    s = _nan((rows + 3, C // 128), torch.float32)
    q0, s0 = q.clone(), s.clone()
    check(lib().sta_op_quant_fp8(x.data_ptr(), rows, C, q.data_ptr(), s.data_ptr(), cur_stream()), "sta_op_quant_fp8")
    torch.cuda.synchronize()
    for buf, before in ((q, q0), (s, s0)):
        mask = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
        mask[:rows] = True
        check_canaries(e.name, buf, before, mask)
    q_ref, s_ref = quantize_rows(x.float())
    assert torch.equal(q[:rows], _u8(q_ref)) and torch.equal(_bits(s[:rows]), _bits(s_ref))


def test_rope_output_with_padded_row_stride():
    """one RoPE launch (dec.projk|projv at the keyframe size) into rows of N + 64 columns: the padding keeps its bits"""
    e = [x for x in fp8_catalogue(14, 14, 1, 1) if x.name == "dec.projk|projv"][0]
    o = make_fp8_operands(e, "random", 11)
    got = run_gemm(e, o, ldo_pad=64)
    ref, bound = gemm_reference(e, o)
    check_bound("keyframe14x14 dec.projk|projv ldo N + 64", got, ref, bound)


def test_catalogue_takes_every_split_factor():
    """the catalogue's EPI_F32 launches cover split-K factors 1, 2, 3, 4, 5 and 8 on a 132-SM H100 (each launch asserts
    the factor it took)"""
    sms = _sms()
    if sms != 132:
        pytest.skip("split factors are listed for 132 SMs; this device has %d" % sms)
    got = {split_factor(e, sms) for _, h, w, nimg, pairs in FP8_SIZES for e in fp8_catalogue(h, w, nimg, pairs)
           if e.kind == "gemm" and e.epi == EPI_F32}
    assert got == SPLIT_FACTORS_COVERED, got


# ---------------------------------------------------------------------------------------------------------------------
# the packed e4m3 weights (pack_linear_fp8_kernel, runtime.cu:63-81), read back through sta_weight_slot
# ---------------------------------------------------------------------------------------------------------------------

TRUNK_ENC = ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2")
TRUNK_DEC = ("attn.qkv", "attn.proj", "cross_attn.projq", "cross_attn.projk", "cross_attn.projv", "cross_attn.proj",
             "mlp.fc1", "mlp.fc2")


def trunk_weight_names():
    """the 192 weights the FP8 mode stores as e4m3: 24 x 4 encoder, 12 x 8 decoder (projk and projv share one matrix)"""
    return (["enc_blocks.%d.%s.weight" % (i, n) for i in range(24) for n in TRUNK_ENC] +
            ["dec_block.%d.%s.weight" % (i, n) for i in range(12) for n in TRUNK_DEC])


def _device_view(ptr, shape, typestr):
    class _View:
        __cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2}
    return torch.as_tensor(_View(), device="cuda")


class _Handle:
    """a bare library model handle: tensors are loaded one by one, nothing runs"""

    def __init__(self, precision):
        from vista_slam_b200 import _lib
        self.L = _lib.lib()
        self.h = ctypes.c_void_p()
        _lib.check(self.L.sta_create_ex(ctypes.byref(self.h), precision), "sta_create_ex")

    def load(self, name, t):
        from vista_slam_b200 import _lib
        src = t.detach().float().contiguous().cuda()
        torch.cuda.synchronize()
        shape = (ctypes.c_int64 * src.dim())(*src.shape)
        _lib.check(self.L.sta_load_tensor(self.h, name.encode(), src.data_ptr(), shape, src.dim(), 1), name)
        torch.cuda.synchronize()

    def slot(self, name):
        p, ld, s = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_void_p()
        rc = self.L.sta_weight_slot(self.h, name.encode(), ctypes.byref(p), ctypes.byref(ld), ctypes.byref(s))
        return rc, p.value, ld.value, s.value

    def fp8_weight(self, name, rows, cols):
        rc, p, ld, s = self.slot(name)
        assert rc == 0 and p and s and ld == cols, (name, rc, ld)
        q = _device_view(p, (rows, ld), "|u1")[:, :cols]
        sc = _device_view(s, (rows // 128, ld // 128), "<f4")
        return q, sc

    def close(self):
        self.L.sta_destroy(self.h)


def _check_packed(h, name, w, oracle_dev):
    q, s = h.fp8_weight(name, *w.shape)
    q_ref, s_ref = quantize_blocks(w.to(oracle_dev))
    q_ref, s_ref = _u8(q_ref).cuda(), s_ref.cuda()
    assert torch.equal(_bits(s), _bits(s_ref)), "%s: block scales differ at %s" % (name, (s != s_ref).nonzero()[:4].tolist())
    bad = q != q_ref
    assert not bool(bad.any()), "%s: %d codes differ, first at %s" % (name, int(bad.sum()), bad.nonzero()[0].tolist())
    return s


def test_packed_trunk_weights_bit_identical_to_oracle(state_dict):
    from vista_slam_b200._lib import PRECISION_FP8
    h = _Handle(PRECISION_FP8)
    try:
        names = trunk_weight_names()
        assert len(names) == 192
        for n in names:
            h.load(n, state_dict[n])
        for n in names:  # after every load: a slot written by its neighbour's pack shows here
            _check_packed(h, n, state_dict[n].cuda(), "cuda")
    finally:
        h.close()


def test_packed_weights_planted_blocks():
    """blocks with amax exactly 448 * 2^e, one fp32 ulp above it, all zeros, and below 448 * 2^-126 (fp32 subnormals
    included); projk and projv of one block, whose scale rows share one array"""
    from vista_slam_b200._lib import PRECISION_BF16, PRECISION_FP8
    g = torch.Generator().manual_seed(3)
    w = torch.randn(1024, 4096, generator=g) * 0.02

    def blk(i, j):
        return w[128 * i:128 * i + 128, 128 * j:128 * j + 128]
    blk(0, 0)[7, 9] = 448 * 2.0 ** -3
    blk(0, 1)[3, 100] = -torch.nextafter(torch.tensor(448 * 2.0 ** -3), torch.tensor(math.inf))
    blk(1, 0).zero_()
    blk(1, 1).copy_(torch.randn(128, 128, generator=g) * 2.0 ** -122)
    blk(1, 1)[0, :8] = torch.tensor([2.0 ** -130, -2.0 ** -140, 2.0 ** -149, 0, 3 * 2.0 ** -135, 2.0 ** -126, 1e-40, -1e-39])
    blk(2, 2)[0, 0] = 448 * 2.0 ** 4
    blk(2, 3)[127, 127] = torch.nextafter(torch.tensor(448 * 2.0 ** 4), torch.tensor(math.inf))
    want = {(0, 0): 2.0 ** -3, (0, 1): 2.0 ** -2, (1, 0): 1.0, (1, 1): 2.0 ** -126, (2, 2): 16.0, (2, 3): 32.0}
    pk = torch.randn(768, 768, generator=g) * 0.05
    pv = torch.randn(768, 768, generator=g) * 0.05
    pk[0, 0], pv[0, 0] = 448 * 2.0 ** -2, 448 * 2.0 ** -5  # distinct block (0, 0) scales
    h = _Handle(PRECISION_FP8)
    try:
        name = "enc_blocks.5.mlp.fc2.weight"
        h.load(name, w)
        h.load("dec_block.3.cross_attn.projk.weight", pk)
        h.load("dec_block.3.cross_attn.projv.weight", pv)
        s = _check_packed(h, name, w, "cpu")
        for (i, j), v in want.items():
            assert float(s[i, j]) == v, ((i, j), float(s[i, j]), v)
        sk = _check_packed(h, "dec_block.3.cross_attn.projk.weight", pk, "cpu")
        sv = _check_packed(h, "dec_block.3.cross_attn.projv.weight", pv, "cpu")
        assert float(sk[0, 0]) == 2.0 ** -2 and float(sv[0, 0]) == 2.0 ** -5
        # the lookup: an unknown name fails; a bf16 weight and an ignored tensor have no scales
        assert h.slot("enc_blocks.5.mlp.fc3.weight")[0] != 0
        rc, p, ld, sp = h.slot("decoder_embed.weight")
        assert rc == 0 and p and ld == 1024 and not sp
        rc, p, ld, sp = h.slot("enc_norm.weight")
        assert rc == 0 and not p and not sp
    finally:
        h.close()
    h = _Handle(PRECISION_BF16)
    try:
        rc, p, ld, sp = h.slot(name)
        assert rc == 0 and p and ld == 4096 and not sp
    finally:
        h.close()


# ---------------------------------------------------------------------------------------------------------------------
# accumulator probe
# ---------------------------------------------------------------------------------------------------------------------

# One 128 x 128 x 128 launch, unit scales, no bias.  Row m of A holds a large value in k = 0 and one small value s in
# every k >= 1; column n of W holds w0 in k = 0 and +-1 on a span of k.  So out[m][n] = L w0 +- len(span) s exactly, with
# the large product and the small ones in one k32 instruction ("one", "same"), in consecutive instructions ("next"), or
# both ("all": 127 small products over the four instructions of the k-block).
PROBE_SMALL = [2.0 ** -i for i in range(10)] + [1.5 * 2.0 ** -i for i in range(9)]
PROBE_LARGE = (1.0, 256.0)
PROBE_W0 = (1.0, 256.0)
PROBE_SPANS = {"one": range(1, 2), "same": range(1, 32), "next": range(32, 64), "all": range(1, 128)}


def probe_layout():
    rows = [(L, s) for L in PROBE_LARGE for s in PROBE_SMALL]
    cols = [(span, sign, w0) for span in PROBE_SPANS for sign in (1, -1) for w0 in PROBE_W0]
    A = torch.zeros(128, 128, dtype=torch.float64)
    W = torch.zeros(128, 128, dtype=torch.float64)
    for m, (L, s) in enumerate(rows):
        A[m, 0], A[m, 1:] = L, s
    for n, (span, sign, w0) in enumerate(cols):
        W[n, 0] = w0
        W[n, list(PROBE_SPANS[span])] = sign
    return rows, cols, A, W


def run_probe():
    from vista_slam_b200._lib import check, cur_stream, lib
    rows, cols, A, W = probe_layout()
    aq, wq = A.float().to(E4M3).cuda(), W.float().to(E4M3).cuda()
    assert torch.equal(aq.float().double().cpu(), A) and torch.equal(wq.float().double().cpu(), W)
    ones = torch.ones(128, 1, device="cuda")
    out = torch.zeros(128, 128, device="cuda")
    bias = torch.zeros(128, device="cuda")
    d = StaGemmFp8Desc()
    d.epi, d.M, d.N, d.K = EPI_F32, 128, 128, 128
    d.A, d.lda, d.a_scale = _u8(aq).data_ptr(), 128, ones.data_ptr()
    d.W, d.ldw, d.w_scale = _u8(wq).data_ptr(), 128, ones.data_ptr()
    d.bias, d.out, d.ldo = bias.data_ptr(), out.data_ptr(), 128
    check(lib().sta_op_gemm_fp8(ctypes.byref(d), cur_stream()), "probe")
    torch.cuda.synchronize()
    return rows, cols, out.cpu().double(), A @ W.t()


def wgmma_e4m3_model(P):
    """the recorded accumulation of one k-block: P [..][128] exact products, four k32 instructions into an accumulator
    that starts at zero"""
    c = torch.zeros(P.shape[:-1], dtype=torch.float64)
    for i in range(4):
        terms = torch.cat([c[..., None], P[..., 32 * i:32 * i + 32]], -1)
        _, e = torch.frexp(terms.abs().amax(-1, keepdim=True))
        g = torch.exp2((e - 1 - PROBE_KEPT_BITS).double())
        c = (torch.trunc(terms / g) * g).sum(-1)
    return c


def test_wgmma_e4m3_accumulation_probe():
    """Every probe output equals the recorded model (wgmma_e4m3_model) exactly: the alignment to the largest term, the
    13 bits kept below it, truncation toward zero, and the accumulator of the previous instruction aligned like a
    product.  If the hardware accumulates differently, this test says so and EPS_BLK must be derived anew."""
    rows, cols, got, exact = run_probe()
    _, _, A, W = probe_layout()
    want = wgmma_e4m3_model(A[:, None, :] * W[None, :, :])
    lines = []
    for n, (span, sign, w0) in enumerate(cols):
        for m, (L, s) in enumerate(rows):
            if got[m, n] != want[m, n]:
                lines.append("%s %+d large %g small %g: got %r, model %r, exact %r" % (
                    span, sign, L * w0, s, float(got[m, n]), float(want[m, n]), float(exact[m, n])))
    assert not lines, "the e4m3 wgmma accumulates unlike the recorded model:\n" + "\n".join(lines[:40])
    # the facts EPS_BLK rests on, in the probe's own terms
    m = rows.index((256.0, 2.0 ** -5))
    assert float(got[m, cols.index(("one", 1, 1.0))]) == 256 + 2.0 ** -5          # 2^-13 of the largest: kept
    m = rows.index((256.0, 2.0 ** -6))
    assert float(got[m, cols.index(("one", 1, 1.0))]) == 256                        # 2^-14: lost
    m = rows.index((256.0, 1.5 * 2.0 ** -5))
    assert float(got[m, cols.index(("one", -1, 1.0))]) == 256 - 2.0 ** -5          # truncated toward zero
    assert float(got[m, cols.index(("one", 1, 1.0))]) == 256 + 2.0 ** -5
    m = rows.index((256.0, 1.0))
    assert float(got[m, cols.index(("next", 1, 256.0))]) == 65536                   # the accumulator counts as a term
