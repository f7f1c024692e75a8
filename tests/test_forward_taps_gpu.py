"""GPU: the model's own forward, launch by launch, against float64.  The runtime's buffer taps (sta_set_taps,
include/sta_b200.h) copy the output of every launch of run_encoder, run_decoder, decode_with_poses, run_dpt and
forward_chunk; each launch is then checked on the operands it actually read -- the tapped outputs of the launches before
it, the weights from the state dict (rounded to bf16, or the e4m3 blocks read back through sta_weight_slot in FP8 mode)
-- with the op-level bound of its launch kind from tests/test_layers_gpu.py, tests/test_layers_fp8_gpu.py,
tests/test_attention_gpu.py and tests/test_pose_head_gpu.py.  Every reference starts from the kernel's own input, so
errors do not compound and those tight bounds apply unchanged to the model's buffers, strides, weight slots, LayerNorm
parameters, positions, partner samples and hook offsets.  A wiring slip (norm2's parameters read for norm3, the pose
token at (0, 0), cross-attention on its own sample, norm_y after self-attention) moves the launch it touches far past its
bound, where the end-to-end checks of tests/test_model_gpu.py see a few per cent after 36 blocks and the DPT.

Exact checks: the positions, the patches (F.unfold), the pose-token rows (init_pose_token bit for bit), the hooks (the
RNE bf16 of the stream, pose rows dropped), the stride-2 im2col, and the zero padding channels of act0 (96 -> 128).

Tap-list completeness: with every name of TAP_PATTERNS tapped (null destinations, counting only), the firings of the
primary names sum to the forward's sta_launch_count delta, so a launch added without a tap fails here.

The packed bf16 and x3 weights: every one of the 665 slots read back through sta_weight_slot equals the packing of the
fp32 state dict (RNE bf16 hi, and hi | hi | lo in x3) bit for bit, padding zero; plus planted ties and nonzero lo parts."""
import ctypes
import gc

import pytest
import torch
import torch.nn.functional as F

from oracle.fp8_oracle import quantize_rows
from oracle.sta_oracle import make_images
from test_attention_gpu import _check_bound as attention_check_bound
from test_layers_fp8_gpu import (MAX_EXCEPTION_FRAC, Fp8Launch, _device_view, _Handle, check_codes, gemm_reference)
from test_layers_gpu import (CFG2_CHECKED_IMAGES, EPI_BF16, EPI_F32, EPI_GELU, EPI_HEAD, EPI_PIXSHUF, EPI_ROPE, Layer,
                             _bilinear64, _bits, check_bound, check_exact, conv_cols, layernorm64, positions, reference)
from test_pose_head_gpu import check_pose, head_pose64
from vista_slam_b200._lib import EPI_GELU_FP8, PRECISION_BF16, PRECISION_X3, StaTap, check, cur_stream, lib

pytestmark = pytest.mark.gpu

# Largest err / bound per launch kind over every case of this file, H100 80GB HBM3 (700 W power limit); the file ran in
# 44 s there.  bf16 outputs sit near 1 as in tests/test_layers_gpu.py: the output rounding, which 2^-8 covers exactly.
# "ln_fp8_codes" and "gelu_fp8_codes" are the shares of e4m3 codes an exception admitted (check_codes; GELU_FP8 on the
# model's operands is a value bound, MAX_EXCEPTION_FRAC["gelu_random"]).  "pose" is ~0: its bound is dominated by the
# 2^-16 LayerNorm term of the kernel's own dec_norm, so it pins down which token the head reads, not its last bits.
MEASURED_RATIO = {"attention": 0.66, "bf16_out": 0.991, "conv": 0.979, "f32_out": 0.024, "gelu": 0.978, "rope": 0.981,
                  "ln": 0.988, "pixshuf": 0.994, "upsample": 0.915, "head": 0.0007, "pose": 0.0, "fp8_f32": 0.005,
                  "fp8_rope": 0.058, "ln_fp8_codes": 0.0091, "gelu_fp8_codes": 1.0}

ENC_BF16 = ("ln1", "qkv", "att", "x_attn", "ln2", "hid", "x")
ENC_FP8 = ("ln1.q", "ln1.s", "qkv", "att", "att8.q", "att8.s", "x_attn", "ln2.q", "ln2.s", "hid.q", "hid.s", "x")
DEC_BF16 = ("ln1", "lny", "qkv", "att", "x_self", "kvc", "ln2", "qc", "catt", "x_cross", "ln3", "hid", "x")
DEC_FP8 = ("ln1.q", "ln1.s", "lny.q", "lny.s", "qkv", "att", "att8.q", "att8.s", "x_self", "kvc", "ln2.q", "ln2.s", "qc",
           "catt", "catt8.q", "catt8.s", "x_cross", "ln3.q", "ln3.s", "hid.q", "hid.s", "x")
DPT = (["dpt.a0", "dpt.l1", "dpt.a1", "dpt.l2", "dpt.l3", "dpt.a3", "dpt.col4", "dpt.l4"] +
       ["dpt.rn%d.%s" % (i, k) for i in range(4) for k in ("raw", "relu")] +
       ["dpt.ref%d.%s" % (lvl, k) for lvl in (3, 2, 1, 0)
        for k in (() if lvl == 3 else ("t1", "s_raw", "s_relu")) + ("t2", "o", "up", "path")] +
       ["dpt.hc1", "dpt.hup", "dpt.pts3d", "dpt.conf"])
ENCODE = ["patches", "pos.enc", "enc.embed"]
DECODE = ["dec.hook0", "pos.dec", "dec.embed", "dec.pose_tok", "dec.hook1", "dec.hook2", "dec.hook3", "pose", "pose_conf"]
# every tap name of runtime.cu, blocks as %d (tests/test_forward_taps_cpu.py scans the source for this set); dec.out is
# the per-layer output copy of sta_decode, which no forward below takes
TAP_PATTERNS = sorted(set(ENCODE + ["enc.%d." + n for n in ENC_BF16 + ENC_FP8] + DECODE +
                           ["dec.%d." + n for n in DEC_BF16 + DEC_FP8] + DPT + ["dec.out"]))


def is_secondary(name):
    """a second output of a launch whose first output has its own tap: FP8 scales, norm_y, relu copies, pose conf"""
    return name.endswith((".s", "relu", "pose_conf", "dpt.conf")) or ".lny" in name


def forward_names(fp8, enc_blocks=range(24), dec_blocks=range(12), encode=True, dpt=True):
    """the tap names of one forward, for the given blocks"""
    enc, dec = (ENC_FP8, DEC_FP8) if fp8 else (ENC_BF16, DEC_BF16)
    names = list(ENCODE) if encode else []
    if encode:
        names += ["enc.%d.%s" % (l, n) for l in enc_blocks for n in enc]
    names += DECODE + ["dec.%d.%s" % (l, n) for l in dec_blocks for n in dec]
    return names + (DPT if dpt else [])


# ---------------------------------------------------------------------------------------------------------------------
# running a forward with taps
# ---------------------------------------------------------------------------------------------------------------------

def run_tapped(model, names, call):
    """call() once counting bytes (null destinations), then once into buffers of exactly that size.  Returns
    {name: uint8 tensor}, {name: firings} and call()'s result.  The taps are cleared in any case."""
    L, h = lib(), model._handle
    arr = (StaTap * len(names))()
    keep = [n.encode() for n in names]
    for i, n in enumerate(keep):
        arr[i].name = n
    try:
        check(L.sta_set_taps(h, arr, len(names)), "sta_set_taps")
        call()
        torch.cuda.synchronize()
        sizes = [arr[i].written for i in range(len(names))]
        bufs = [torch.empty(max(s, 1), dtype=torch.uint8, device="cuda") for s in sizes]
        for i, b in enumerate(bufs):
            arr[i].dst, arr[i].capacity, arr[i].written, arr[i].fired = b.data_ptr(), sizes[i], 0, 0
        check(L.sta_set_taps(h, arr, len(names)), "sta_set_taps")
        out = call()
        torch.cuda.synchronize()
        assert [arr[i].written for i in range(len(names))] == sizes, "a tap wrote a different size the second time"
        fired = {n: arr[i].fired for i, n in enumerate(names)}
        return {n: bufs[i][:sizes[i]] for i, n in enumerate(names)}, fired, out
    finally:
        L.sta_set_taps(h, None, 0)


def _same_outputs(a, b):
    for x, y in zip(a, b):
        assert torch.equal(_bits(x.contiguous()), _bits(y.contiguous())), "outputs with taps differ from outputs without"


def bf(t, *shape):
    return t.view(torch.bfloat16).view(*shape)


def f32(t, *shape):
    return t.view(torch.float32).view(*shape)


# ---------------------------------------------------------------------------------------------------------------------
# weights as the kernels read them
# ---------------------------------------------------------------------------------------------------------------------

DPT_P = "downstream_head_pts.dpt."


class Weights:
    def __init__(self, sd, model):
        self.sd, self.model = sd, model

    def f(self, name):
        return self.sd[name].cuda().float()

    def lin(self, name, rows_pad=0):
        """[N][K] bf16 (a 1x1 convolution's [N][K][1][1] too), zero rows up to rows_pad"""
        w = self.f(name)
        w = w.reshape(w.shape[0], -1)
        if rows_pad:
            w = F.pad(w, (0, 0, 0, rows_pad - w.shape[0]))
        return w.bfloat16()

    def bias(self, name, pad=0):
        b = self.f(name)
        return F.pad(b, (0, pad - b.shape[0])) if pad else b

    def conv3(self, name, cin_pad=0):
        """[Cout][Cin][3][3] -> [Cout][9 Cin_pad] in conv_cols' (kh, kw, c) order, bf16"""
        w = self.f(name).permute(0, 2, 3, 1)
        if cin_pad:
            w = F.pad(w, (0, cin_pad - w.shape[-1]))
        return w.reshape(w.shape[0], -1).bfloat16()

    def convT(self, name, k, c_pad):
        """ConvTranspose2d [Cin][Cout][k][k] -> GEMM rows [(kh k + kw) Cout_pad + co][Cin_pad], bf16"""
        w = self.f(name)
        cin, cout = w.shape[:2]
        out = torch.zeros(k, k, c_pad, c_pad, device="cuda")
        out[:, :, :cout, :cin] = w.permute(2, 3, 1, 0)
        return out.reshape(k * k * c_pad, c_pad).bfloat16()

    def fp8(self, name, rows, cols):
        """e4m3 codes [rows][cols] and block scales of a trunk weight, from the model's arena"""
        p, ld, s = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_void_p()
        check(lib().sta_weight_slot(self.model._handle, name.encode(), ctypes.byref(p), ctypes.byref(ld),
                                    ctypes.byref(s)), name)
        assert ld.value == cols and s.value
        return (_device_view(p.value, (rows, cols), "|u1"),
                _device_view(s.value, (rows // 128, cols // 128), "<f4"))


# ---------------------------------------------------------------------------------------------------------------------
# the checks of one tapped forward
# ---------------------------------------------------------------------------------------------------------------------

class Checker:
    def __init__(self, taps, W, fp8, h, w, S, images=None):
        self.t, self.W, self.fp8 = taps, W, fp8
        self.h, self.w, self.S = h, w, S
        self.N = h * w
        self.images = images
        self.worst = {}

    def record(self, kind, ratio):
        self.worst[kind] = max(self.worst.get(kind, 0.0), ratio)

    # ---- launch kinds ----
    def ln(self, name, x, g, b):
        """bf16 LayerNorm output, or the e4m3 codes + scales of an FP8 one, of fp32 rows x"""
        ref, b32 = layernorm64(x, self.W.f(g), self.W.f(b))
        if self.fp8:
            C = x.shape[1]
            q, s = self.t[name + ".q"].view(-1, C), f32(self.t[name + ".s"], -1, C // 128)
            self.record("ln_fp8_codes", check_codes(name, q, s, ref, b32, MAX_EXCEPTION_FRAC["ln"]))
            return
        got = bf(self.t[name], ref.shape[0], -1)
        self.record("ln", check_bound(name, got, ref, 2.0 ** -8 * ref.abs() + b32))

    def gemm(self, kind, name, A, Wp, bias, got, resid=None, pos=None, rope_cols=0, rowmap_n=0, epi=None):
        M, K = A.shape
        e = Layer(name, epi, M, Wp.shape[0], K, bias=bias is not None, resid="inplace" if resid is not None else "",
                  rope_cols=rope_cols, rowmap_n=rowmap_n)
        o = {"bias": bias} if bias is not None else {}
        if resid is not None:
            o["resid"] = resid
        if pos is not None:
            o["pos"] = pos
        ref, bound = reference(e, o, A, Wp, False)["out"]
        self.record(kind, check_bound(name, got, ref, bound))
        return ref

    def gemm_fp8(self, name, a_name, K, wname, rows, bias, got_name, epi, resid=None, pos=None, rope_cols=0):
        """an e4m3 GEMM on the tapped codes + scales a_name (K wide) and the packed weight wname ([rows][K])"""
        aq, as_ = self.t[a_name + ".q"], self.t[a_name + ".s"]
        wq, ws = self.W.fp8(wname, rows, K)
        M = aq.numel() // K
        o = {"aq": aq.view(M, K), "as": f32(as_, M, K // 128), "wq": wq, "ws": ws, "bias": bias}
        if resid is not None:
            o["resid"] = resid
        if pos is not None:
            o["pos"] = pos
        e = Fp8Launch(name, "gemm", epi, M, rows, K, rope_cols)
        ref, bound = gemm_reference(e, o)
        if epi == EPI_GELU_FP8:
            q, s = self.t[got_name + ".q"].view(M, rows), f32(self.t[got_name + ".s"], M, rows // 128)
            self.record("gelu_fp8_codes", check_codes(name, q, s, ref, bound, MAX_EXCEPTION_FRAC["gelu_random"]))
            return
        got = f32(self.t[got_name], M, rows) if epi == EPI_F32 else bf(self.t[got_name], M, rows)
        self.record("fp8_f32" if epi == EPI_F32 else "fp8_rope", check_bound(name, got, ref, bound))

    def attention(self, name, q, k, v, heads, shift):
        """q, k, v [samples][n][heads 64] views of the tapped projections"""
        S, n = q.shape[:2]
        seen = [x.float().reshape(S, n, heads, 64) for x in (q, k, v)]
        out = bf(self.t[name], S, n, heads, 64).double()
        self.record("attention", attention_check_bound(name, "bf16", out, seen, shift))

    def quant(self, name, src):
        q_ref, s_ref = quantize_rows(src.float())
        q, s = self.t[name + ".q"].view(q_ref.shape), f32(self.t[name + ".s"], *s_ref.shape)
        assert torch.equal(q, q_ref.view(torch.uint8)) and torch.equal(_bits(s), _bits(s_ref)), name

    def conv(self, kind, name, A, Wp, bias, got, relu_main=0, skip=None, skip2=None, got_relu=None):
        nimg, H, Wd, Cin = A.shape
        e = Layer(name, EPI_BF16, N=Wp.shape[0], K=9 * Cin, conv=(nimg, H, Wd, Cin), bias=bias is not None,
                  resid="skip" if skip is not None else "", resid2=skip2 is not None, relu_main=relu_main,
                  relu_copy=got_relu is not None)
        o = {"bias": bias} if bias is not None else {}
        for key, s in (("resid", skip), ("resid2", skip2)):
            if s is not None:
                o[key] = o[key + "_phys"] = s
        refs = reference(e, o, A, Wp, False, self.images)
        sel = (lambda x: x) if self.images is None else (lambda x: x[list(self.images)])
        ref, bound = refs["out"]
        self.record(kind, check_bound(name, sel(got), ref, bound))
        if got_relu is not None:
            ref, bound = refs["relu"]
            self.record(kind, check_bound(name + " relu", sel(got_relu), ref, bound))

    def upsample(self, name, x, got, OH, OW):
        imgs = range(x.shape[0]) if self.images is None else self.images
        ref = torch.cat([_bilinear64(x[i:i + 1].double())[:, :OH, :OW] for i in imgs])
        bound = 2.0 ** -8 * ref.abs() + 2.0 ** -12 * float(x.float().abs().max())
        self.record("upsample", check_bound(name, got[list(imgs)], ref, bound))

    # ---- the model's stages ----
    def encoder(self, images, blocks):
        t, W, S, N, h, w = self.t, self.W, self.S, self.N, self.h, self.w
        T = S * N
        want = F.unfold(images.float(), 16, stride=16).transpose(1, 2).reshape(-1, 768).bfloat16()
        assert torch.equal(_bits(bf(t["patches"], T, 768)), _bits(want)), "patches"
        pos = t["pos.enc"].view(torch.int32).view(T, 2)
        assert torch.equal(pos, positions((S, h, w, 0), "cuda")), "pos.enc"
        x = lambda n: f32(t[n], T, 1024)  # noqa: E731
        self.gemm("f32_out", "enc.embed", bf(t["patches"], T, 768), W.lin("patch_embed.proj.weight"),
                  W.f("patch_embed.proj.bias"), x("enc.embed"), epi=EPI_F32)
        for l in blocks:
            p, P = "enc_blocks.%d." % l, "enc.%d." % l
            xin = x("enc.embed") if l == 0 else x("enc.%d.x" % (l - 1))
            self.ln(P + "ln1", xin, p + "norm1.weight", p + "norm1.bias")
            if self.fp8:
                self.gemm_fp8(P + "qkv", P + "ln1", 1024, p + "attn.qkv.weight", 3072, W.f(p + "attn.qkv.bias"), P + "qkv",
                              EPI_ROPE, pos=pos, rope_cols=2048)
            else:
                self.gemm("rope", P + "qkv", bf(t[P + "ln1"], T, 1024), W.lin(p + "attn.qkv.weight"),
                          W.f(p + "attn.qkv.bias"), bf(t[P + "qkv"], T, 3072), pos=pos, rope_cols=2048, epi=EPI_ROPE)
            qkv = bf(t[P + "qkv"], S, N, 3072)
            self.attention(P + "att", qkv[..., :1024], qkv[..., 1024:2048], qkv[..., 2048:], 16, 0)
            if self.fp8:
                self.quant(P + "att8", bf(t[P + "att"], T, 1024))
                self.gemm_fp8(P + "x_attn", P + "att8", 1024, p + "attn.proj.weight", 1024, W.f(p + "attn.proj.bias"),
                              P + "x_attn", EPI_F32, resid=xin)
                self.ln(P + "ln2", x(P + "x_attn"), p + "norm2.weight", p + "norm2.bias")
                self.gemm_fp8(P + "hid", P + "ln2", 1024, p + "mlp.fc1.weight", 4096, W.f(p + "mlp.fc1.bias"), P + "hid",
                              EPI_GELU_FP8)
                self.gemm_fp8(P + "x", P + "hid", 4096, p + "mlp.fc2.weight", 1024, W.f(p + "mlp.fc2.bias"), P + "x",
                              EPI_F32, resid=x(P + "x_attn"))
                continue
            self.gemm("f32_out", P + "x_attn", bf(t[P + "att"], T, 1024), W.lin(p + "attn.proj.weight"),
                      W.f(p + "attn.proj.bias"), x(P + "x_attn"), resid=xin, epi=EPI_F32)
            self.ln(P + "ln2", x(P + "x_attn"), p + "norm2.weight", p + "norm2.bias")
            self.gemm("gelu", P + "hid", bf(t[P + "ln2"], T, 1024), W.lin(p + "mlp.fc1.weight"),
                      W.f(p + "mlp.fc1.bias"), bf(t[P + "hid"], T, 4096), epi=EPI_GELU)
            self.gemm("f32_out", P + "x", bf(t[P + "hid"], T, 4096), W.lin(p + "mlp.fc2.weight"),
                      W.f(p + "mlp.fc2.bias"), x(P + "x"), resid=x(P + "x_attn"), epi=EPI_F32)
        if 23 in blocks:
            want = x("enc.23.x").bfloat16()
            assert torch.equal(_bits(bf(t["dec.hook0"], T, 1024)), _bits(want)), "dec.hook0"

    def decoder(self, blocks, B):
        t, W, S, N, h, w = self.t, self.W, self.S, self.N, self.h, self.w
        M = N + 1
        Td = S * M
        pos = t["pos.dec"].view(torch.int32).view(Td, 2)
        assert torch.equal(pos, positions((S, h, w, 1), "cuda")), "pos.dec"
        x = lambda n: f32(t[n], Td, 768)  # noqa: E731
        rows = lambda v: v.view(S, M, -1)[:, 1:].reshape(S * N, -1)  # noqa: E731  (pose rows dropped)
        self.gemm("f32_out", "dec.embed", bf(t["dec.hook0"], S * N, 1024), W.lin("decoder_embed.weight"),
                  W.f("decoder_embed.bias"), rows(x("dec.embed")), rowmap_n=N, epi=EPI_F32)
        tok = x("dec.pose_tok").view(S, M, 768)
        assert torch.equal(_bits(tok[:, 0]), _bits(W.f("init_pose_token").view(1, 768).expand(S, 768))), "pose token"
        assert torch.equal(_bits(tok[:, 1:]), _bits(x("dec.embed").view(S, M, 768)[:, 1:])), "dec.pose_tok rows"
        for l in blocks:
            p, P = "dec_block.%d." % l, "dec.%d." % l
            xin = x("dec.pose_tok") if l == 0 else x("dec.%d.x" % (l - 1))
            self.ln(P + "ln1", xin, p + "norm1.weight", p + "norm1.bias")
            self.ln(P + "lny", xin, p + "norm_y.weight", p + "norm_y.bias")
            kvb = torch.cat([W.f(p + "cross_attn.projk.bias"), W.f(p + "cross_attn.projv.bias")])
            if self.fp8:
                self.gemm_fp8(P + "qkv", P + "ln1", 768, p + "attn.qkv.weight", 2304, W.f(p + "attn.qkv.bias"), P + "qkv",
                              EPI_ROPE, pos=pos, rope_cols=1536)
            else:
                self.gemm("rope", P + "qkv", bf(t[P + "ln1"], Td, 768), W.lin(p + "attn.qkv.weight"),
                          W.f(p + "attn.qkv.bias"), bf(t[P + "qkv"], Td, 2304), pos=pos, rope_cols=1536, epi=EPI_ROPE)
            qkv = bf(t[P + "qkv"], S, M, 2304)
            self.attention(P + "att", qkv[..., :768], qkv[..., 768:1536], qkv[..., 1536:], 12, 0)
            if self.fp8:
                self.quant(P + "att8", bf(t[P + "att"], Td, 768))
                self.gemm_fp8(P + "x_self", P + "att8", 768, p + "attn.proj.weight", 768, W.f(p + "attn.proj.bias"),
                              P + "x_self", EPI_F32, resid=xin)
                self.gemm_fp8(P + "kvc", P + "lny", 768, p + "cross_attn.projk.weight", 1536, kvb, P + "kvc", EPI_ROPE,
                              pos=pos, rope_cols=768)
                self.ln(P + "ln2", x(P + "x_self"), p + "norm2.weight", p + "norm2.bias")
                self.gemm_fp8(P + "qc", P + "ln2", 768, p + "cross_attn.projq.weight", 768,
                              W.f(p + "cross_attn.projq.bias"), P + "qc", EPI_ROPE, pos=pos, rope_cols=768)
            else:
                self.gemm("f32_out", P + "x_self", bf(t[P + "att"], Td, 768), W.lin(p + "attn.proj.weight"),
                          W.f(p + "attn.proj.bias"), x(P + "x_self"), resid=xin, epi=EPI_F32)
                Wkv = torch.cat([W.lin(p + "cross_attn.projk.weight"), W.lin(p + "cross_attn.projv.weight")])
                self.gemm("rope", P + "kvc", bf(t[P + "lny"], Td, 768), Wkv, kvb, bf(t[P + "kvc"], Td, 1536), pos=pos,
                          rope_cols=768, epi=EPI_ROPE)
                self.ln(P + "ln2", x(P + "x_self"), p + "norm2.weight", p + "norm2.bias")
                self.gemm("rope", P + "qc", bf(t[P + "ln2"], Td, 768), W.lin(p + "cross_attn.projq.weight"),
                          W.f(p + "cross_attn.projq.bias"), bf(t[P + "qc"], Td, 768), pos=pos, rope_cols=768,
                          epi=EPI_ROPE)
            kv = bf(t[P + "kvc"], S, M, 1536)
            self.attention(P + "catt", bf(t[P + "qc"], S, M, 768), kv[..., :768], kv[..., 768:], 12, B)
            if self.fp8:
                self.quant(P + "catt8", bf(t[P + "catt"], Td, 768))
                self.gemm_fp8(P + "x_cross", P + "catt8", 768, p + "cross_attn.proj.weight", 768,
                              W.f(p + "cross_attn.proj.bias"), P + "x_cross", EPI_F32, resid=x(P + "x_self"))
                self.ln(P + "ln3", x(P + "x_cross"), p + "norm3.weight", p + "norm3.bias")
                self.gemm_fp8(P + "hid", P + "ln3", 768, p + "mlp.fc1.weight", 3072, W.f(p + "mlp.fc1.bias"), P + "hid",
                              EPI_GELU_FP8)
                self.gemm_fp8(P + "x", P + "hid", 3072, p + "mlp.fc2.weight", 768, W.f(p + "mlp.fc2.bias"), P + "x", EPI_F32,
                              resid=x(P + "x_cross"))
            else:
                self.gemm("f32_out", P + "x_cross", bf(t[P + "catt"], Td, 768), W.lin(p + "cross_attn.proj.weight"),
                          W.f(p + "cross_attn.proj.bias"), x(P + "x_cross"), resid=x(P + "x_self"), epi=EPI_F32)
                self.ln(P + "ln3", x(P + "x_cross"), p + "norm3.weight", p + "norm3.bias")
                self.gemm("gelu", P + "hid", bf(t[P + "ln3"], Td, 768), W.lin(p + "mlp.fc1.weight"),
                          W.f(p + "mlp.fc1.bias"), bf(t[P + "hid"], Td, 3072), epi=EPI_GELU)
                self.gemm("f32_out", P + "x", bf(t[P + "hid"], Td, 3072), W.lin(p + "mlp.fc2.weight"),
                          W.f(p + "mlp.fc2.bias"), x(P + "x"), resid=x(P + "x_cross"), epi=EPI_F32)
            if l in (5, 8):
                q = 1 if l == 5 else 2
                want = rows(x(P + "x")).bfloat16()
                assert torch.equal(_bits(bf(t["dec.hook%d" % q], S * N, 768)), _bits(want)), "dec.hook%d" % q
        if 11 in blocks:
            xo = x("dec.11.x")
            # the final norm, pose rows dropped: dec.hook3
            ref, b32 = layernorm64(xo, W.f("dec_norm.weight"), W.f("dec_norm.bias"))
            got = bf(t["dec.hook3"], S * N, 768)
            self.record("ln", check_bound("dec.hook3", got, rows(ref), 2.0 ** -8 * rows(ref).abs() + rows(b32)))
            # the pose heads on the dec_norm-ed pose rows (the kernel normalises them itself, in fp32)
            tok, tok_err = (r.view(S, M, 768)[:, 0] for r in (ref, b32))
            pref = head_pose64(self.W.sd, tok, tok_err)
            worst, _ = check_pose("pose", f32(t["pose"], S, 4, 4), f32(t["pose_conf"], S), pref)
            self.record("pose", worst)

    def dpt(self, nimg):
        """the DPT of all nimg images (the tapped calls in order: views, halves)"""
        t, W, N, h, w = self.t, self.W, self.N, self.h, self.w
        T = nimg * N
        h4, w4 = (h + 1) // 2, (w + 1) // 2
        LH, LW = [4 * h, 2 * h, h, h4], [4 * w, 2 * w, w, w4]
        P = DPT_P + "act_postprocess."
        hook = [bf(t["dec.hook0"], -1, 1024)] + [bf(t["dec.hook%d" % q], -1, 768) for q in (1, 2, 3)]
        assert all(x.shape[0] == T for x in hook)
        a0 = bf(t["dpt.a0"], T, 128)
        self.gemm("bf16_out", "dpt.a0", hook[0], W.lin(P + "0.0.weight")[:96], W.f(P + "0.0.bias"), a0[:, :96],
                  epi=EPI_BF16)
        assert not bool(a0[:, 96:].float().any()), "dpt.a0: padding channels 96..127 not zero"
        l1 = bf(t["dpt.l1"], nimg, 4 * h, 4 * w, 128)
        self.pixshuf("dpt.l1", a0, W.convT(P + "0.1.weight", 4, 128), W.bias(P + "0.1.bias", 128), l1, 4, 128, nimg, 96)
        assert not bool(l1[..., 96:].float().any()), "dpt.l1: padding channels 96..127 not zero"
        a1 = bf(t["dpt.a1"], T, 192)
        self.gemm("bf16_out", "dpt.a1", hook[1], W.lin(P + "1.0.weight"), W.f(P + "1.0.bias"), a1, epi=EPI_BF16)
        l2 = bf(t["dpt.l2"], nimg, 2 * h, 2 * w, 192)
        self.pixshuf("dpt.l2", a1, W.convT(P + "1.1.weight", 2, 192), W.f(P + "1.1.bias"), l2, 2, 192, nimg, 192)
        l3 = bf(t["dpt.l3"], nimg, h, w, 384)
        self.gemm("bf16_out", "dpt.l3", hook[2], W.lin(P + "2.0.weight"), W.f(P + "2.0.bias"), l3.reshape(T, 384),
                  epi=EPI_BF16)
        a3 = bf(t["dpt.a3"], nimg, h, w, 768)
        self.gemm("bf16_out", "dpt.a3", hook[3], W.lin(P + "3.0.weight"), W.f(P + "3.0.bias"), a3.reshape(T, 768),
                  epi=EPI_BF16)
        col4 = bf(t["dpt.col4"], nimg * h4 * w4, 9 * 768)
        check_exact("dpt.col4", col4, conv_cols(a3, stride=2))
        l4 = bf(t["dpt.l4"], nimg, h4, w4, 768)
        self.gemm("bf16_out", "dpt.l4", col4, W.conv3(P + "3.1.weight"), W.f(P + "3.1.bias"), l4.reshape(-1, 768),
                  epi=EPI_BF16)
        lin = [l1, l2, l3, l4]
        raw, relu = [], []
        for i in range(4):
            shape = (nimg, LH[i], LW[i], 256)
            raw.append(bf(t["dpt.rn%d.raw" % i], *shape))
            relu.append(bf(t["dpt.rn%d.relu" % i], *shape))
            self.conv("conv", "dpt.rn%d" % i, lin[i], W.conv3(DPT_P + "scratch.layer_rn.%d.weight" % i,
                                                              lin[i].shape[-1]), None, raw[i], got_relu=relu[i])
        path = None
        for lvl in (3, 2, 1, 0):
            r = DPT_P + "scratch.refinenet%d." % (lvl + 1)
            R = "dpt.ref%d." % lvl
            shape = (nimg, LH[lvl], LW[lvl], 256)
            g = lambda n, s=shape: bf(t[R + n], *s)  # noqa: E731
            if lvl == 3:
                s_raw, s_relu = raw[3], relu[3]
            else:
                self.conv("conv", R + "t1", relu[lvl], W.conv3(r + "resConfUnit1.conv1.weight"),
                          W.f(r + "resConfUnit1.conv1.bias"), g("t1"), relu_main=1)
                s_raw, s_relu = g("s_raw"), g("s_relu")
                self.conv("conv", R + "s", g("t1"), W.conv3(r + "resConfUnit1.conv2.weight"),
                          W.f(r + "resConfUnit1.conv2.bias"), s_raw, skip=raw[lvl], skip2=path, got_relu=s_relu)
            self.conv("conv", R + "t2", s_relu, W.conv3(r + "resConfUnit2.conv1.weight"),
                      W.f(r + "resConfUnit2.conv1.bias"), g("t2"), relu_main=1)
            self.conv("conv", R + "o", g("t2"), W.conv3(r + "resConfUnit2.conv2.weight"),
                      W.f(r + "resConfUnit2.conv2.bias"), g("o"), skip=s_raw)
            self.gemm("bf16_out", R + "up", g("o").reshape(-1, 256), W.lin(r + "out_conv.weight"),
                      W.f(r + "out_conv.bias"), g("up").reshape(-1, 256), epi=EPI_BF16)
            OH, OW = (LH[2], LW[2]) if lvl == 3 else (2 * LH[lvl], 2 * LW[lvl])
            path = bf(t[R + "path"], nimg, OH, OW, 256)
            self.upsample(R + "path", g("up"), path, OH, OW)
        H8, W8 = 8 * h, 8 * w
        hc1 = bf(t["dpt.hc1"], nimg, H8, W8, 128)
        self.conv("conv", "dpt.hc1", path, W.conv3(DPT_P + "head.0.weight"), W.f(DPT_P + "head.0.bias"), hc1)
        hup = bf(t["dpt.hup"], nimg, 2 * H8, 2 * W8, 128)
        self.upsample("dpt.hup", hc1, hup, 2 * H8, 2 * W8)
        e = Layer("dpt.head", EPI_HEAD, N=128, K=1152, conv=(nimg, 2 * H8, 2 * W8, 128))
        o = {"bias": W.f(DPT_P + "head.2.bias"), "head_w": W.f(DPT_P + "head.4.weight").view(4, 128),
             "head_b": W.f(DPT_P + "head.4.bias")}
        refs = reference(e, o, hup, W.conv3(DPT_P + "head.2.weight"), False, self.images)
        sel = (lambda v: v) if self.images is None else (lambda v: v[list(self.images)])
        got = {"pts3d": f32(t["dpt.pts3d"], nimg, 2 * H8, 2 * W8, 3), "conf": f32(t["dpt.conf"], nimg, 2 * H8, 2 * W8)}
        for key, (ref, bound) in refs.items():
            self.record("head", check_bound("dpt." + key, sel(got[key]).double(), ref, bound))

    def pixshuf(self, name, A, Wp, bias, got, k, cout, nimg, real):
        """the transposed convolution (kernel = stride = k) as a GEMM with the pixel-shuffle epilogue; channels from
        `real` on are padding (checked to be zero by the caller)"""
        e = Layer(name, EPI_PIXSHUF, A.shape[0], Wp.shape[0], A.shape[1], ps=(k, cout, nimg, self.h, self.w))
        ref, bound = reference(e, {"bias": bias}, A, Wp, False)["out"]
        self.record("pixshuf", check_bound(name, got[..., :real], ref[..., :real], bound[..., :real]))


def _report(c, what):
    for kind, r in sorted(c.worst.items()):
        print("forward taps %-32s %-16s worst %.4f (recorded %s)" % (what, kind, r, MEASURED_RATIO.get(kind)),
              flush=True)


@pytest.fixture(autouse=True)
def _no_tf32():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.fixture(autouse=True)
def _release_memory():
    """The cfg-2 taps and float64 references take gigabytes; hand them back to the device after each test, so that
    the library's own allocations in later suites do not find them held by PyTorch's cache."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def fp8_model(state_dict):
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    m = STA(precision="fp8")
    m.load_state_dict(state_dict, strict=True)
    m.eval()
    m._ready(torch.empty(1, device="cuda"))
    yield m
    torch.cuda.synchronize()
    lib().sta_destroy(m._handle)  # its weights and its cfg-2 workspace
    m._handle = None


def _model(request, precision):
    return request.getfixturevalue("cuda_model" if precision == "bf16" else "fp8_model")


# (id, precision, B pairs, H, W, encoder blocks, decoder blocks, DPT images checked)
FORWARDS = [("64x80", "bf16", 1, 64, 80, range(24), range(12), None),
            ("64x80", "fp8", 1, 64, 80, range(24), range(12), None),
            ("48x80", "bf16", 1, 48, 80, range(24), range(12), None),
            ("224x224", "bf16", 1, 224, 224, range(24), range(12), None),
            ("cfg2_384x512", "bf16", 16, 384, 512, (0, 11, 23), (0, 5, 11), CFG2_CHECKED_IMAGES),
            ("cfg2_384x512", "fp8", 16, 384, 512, (0, 11, 23), (0, 5, 11), CFG2_CHECKED_IMAGES)]


def _needed(blocks, depth):
    """the blocks whose output x a check of `blocks` reads"""
    return sorted(set(blocks) | {b - 1 for b in blocks if b > 0} | {depth - 1})


@pytest.mark.parametrize("sid,precision,B,H,W,enc_blocks,dec_blocks,images",
                         [pytest.param(*f, id="%s-%s" % f[:2]) for f in FORWARDS])
def test_forward_pairs_launch_by_launch(request, state_dict, sid, precision, B, H, W, enc_blocks, dec_blocks, images):
    model = _model(request, precision)
    fp8 = precision == "fp8"
    img1, img2 = (x.cuda() for x in make_images(B, H, W, seed=B * 1000 + H + W))
    plain = model.forward_pairs(img1, img2)
    names = forward_names(fp8, _needed(enc_blocks, 24), _needed(dec_blocks, 12))
    taps, fired, out = run_tapped(model, names, lambda: model.forward_pairs(img1, img2))
    _same_outputs([v for d in plain for v in d.values()], [v for d in out for v in d.values()])
    h, w = H // 16, W // 16
    c = Checker(taps, Weights(state_dict, model), fp8, h, w, 2 * B, images)
    c.encoder(torch.cat([img1, img2]), enc_blocks)
    c.decoder(dec_blocks, B)
    c.dpt(2 * B)
    # the DPT wrote the caller's maps: view 0 then view 1
    got = torch.stack([d["pts3d_pred"] for d in out]).reshape(2 * B, H, W, 3)
    assert torch.equal(_bits(got.contiguous()), _bits(f32(taps["dpt.pts3d"], 2 * B, H, W, 3))), "dpt.pts3d"
    _report(c, "%s %s" % (sid, precision))


def test_forward_pairs_host_dpt_halves(cuda_model, state_dict):
    """B = 2: each view's DPT runs as two parts, the second at first = 1 of the hooks"""
    B, H, W = 2, 64, 80
    img1, img2 = make_images(B, H, W, seed=7)
    img1, img2 = img1.pin_memory(), img2.pin_memory()
    plain = cuda_model.forward_pairs_host(img1, img2)
    plain = {k: v.clone() for k, v in plain.items()}
    names = forward_names(False)
    taps, fired, out = run_tapped(cuda_model, names, lambda: cuda_model.forward_pairs_host(img1, img2))
    assert fired["dpt.a0"] == 4 and fired["dpt.pts3d"] == 4, "two DPT parts per view"
    _same_outputs(list(plain.values()), list(out.values()))
    c = Checker(taps, Weights(state_dict, cuda_model), False, H // 16, W // 16, 2 * B)
    c.encoder(torch.cat([img1, img2]).cuda(), range(24))
    c.decoder(range(12), B)
    c.dpt(2 * B)
    _report(c, "host B=2")


def _regress(model, fi, fj, K, H, W):
    pose = torch.empty(2, K, 4, 4, device="cuda")
    pconf = torch.empty(2, K, device="cuda")
    pts = torch.empty(2, K, H, W, 3, device="cuda")
    conf = torch.empty(2, K, H, W, device="cuda")
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    check(lib().sta_regress_pairs(model._handle, P(fi), P(fj), K, H, W, P(pose), P(pconf), P(pts), P(conf), None, None,
                                  None, None, cur_stream()), "sta_regress_pairs")
    return pose, pconf, pts, conf


def test_regress_pairs_keyframe_edges(cuda_model, state_dict):
    """the SLAM keyframe path: K = 3 edges of 14 x 14 tokens from encoder features, graphed when untapped"""
    K, H, W = 3, 224, 224
    N = (H // 16) * (W // 16)
    g = torch.Generator(device="cuda").manual_seed(3)
    fi, fj = (torch.randn(K, N, 1024, generator=g, device="cuda") for _ in range(2))
    L = lib()
    for _ in range(3):  # seen, captured, replayed
        plain = _regress(cuda_model, fi, fj, K, H, W)
    torch.cuda.synchronize()
    replays = L.sta_graph_replays(cuda_model._handle)
    names = forward_names(False, encode=False)
    taps, fired, out = run_tapped(cuda_model, names, lambda: _regress(cuda_model, fi, fj, K, H, W))
    assert L.sta_graph_replays(cuda_model._handle) == replays, "a tapped call replayed a graph"
    _same_outputs(plain, out)
    _regress(cuda_model, fi, fj, K, H, W)
    torch.cuda.synchronize()
    assert L.sta_graph_replays(cuda_model._handle) == replays + 1, "cleared taps: the graph replays again"
    want = torch.cat([fi, fj]).reshape(-1, 1024).bfloat16()
    assert torch.equal(_bits(bf(taps["dec.hook0"], 2 * K * N, 1024)), _bits(want)), "dec.hook0"
    c = Checker(taps, Weights(state_dict, cuda_model), False, H // 16, W // 16, 2 * K)
    c.decoder(range(12), K)
    c.dpt(2 * K)
    _report(c, "regress K=3")


@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_every_launch_has_one_tap(request, precision):
    """every name fires; the primary names' firings are the launches the forward counts"""
    model = _model(request, precision)
    img1, img2 = (x.cuda() for x in make_images(2, 64, 80, seed=5))
    names = forward_names(precision == "fp8")
    model.forward_pairs(img1, img2)
    torch.cuda.synchronize()
    L, h = lib(), model._handle
    arr = (StaTap * len(names))()
    keep = [n.encode() for n in names]
    for i, n in enumerate(keep):
        arr[i].name = n
    check(L.sta_set_taps(h, arr, len(names)))
    try:
        l0 = L.sta_launch_count(h)
        model.forward_pairs(img1, img2)
        torch.cuda.synchronize()
        launches = L.sta_launch_count(h) - l0
    finally:
        L.sta_set_taps(h, None, 0)
    fired = {n: arr[i].fired for i, n in enumerate(names)}
    assert all(f > 0 for f in fired.values()), [n for n, f in fired.items() if f == 0]
    assert sum(f for n, f in fired.items() if not is_secondary(n)) == launches
    l0 = L.sta_launch_count(h)
    model.forward_pairs(img1, img2)
    assert L.sta_launch_count(h) - l0 == launches, "the tap copies were counted as launches"


def test_too_small_a_tap_is_refused_by_name(cuda_model):
    img1, img2 = (x.cuda() for x in make_images(1, 64, 80, seed=5))
    L, h = lib(), cuda_model._handle
    buf = torch.empty(64, dtype=torch.uint8, device="cuda")
    arr = (StaTap * 1)()
    arr[0].name, arr[0].dst, arr[0].capacity = b"enc.3.qkv", buf.data_ptr(), 64
    check(L.sta_set_taps(h, arr, 1))
    try:
        with pytest.raises(RuntimeError, match="enc.3.qkv"):
            cuda_model.forward_pairs(img1, img2)
    finally:
        L.sta_set_taps(h, None, 0)
    torch.cuda.synchronize()
    assert arr[0].written == 0 and arr[0].fired == 0


# ---------------------------------------------------------------------------------------------------------------------
# the packed bf16 and x3 weights, bit for bit (pack_linear_kernel, pack_conv3_kernel, pack_convT_kernel,
# transpose_f32_kernel and the PK_F32 copies, runtime.cu)
# ---------------------------------------------------------------------------------------------------------------------

def _parts(w, split):
    """RNE bf16 hi, and in x3 the lo part bf16(w - hi), as int16 bits"""
    hi = w.bfloat16()
    if not split:
        return [_bits(hi)]
    lo = (w - hi.float()).bfloat16()
    return [_bits(hi), _bits(hi), _bits(lo)]


def pack_linear(w, split, rows_pad=0):
    """[N][K] -> [N_pad][ldd] bits: (hi) or (hi | hi | lo), zero rows below N"""
    w = w.reshape(w.shape[0], -1).float()
    out = torch.cat(_parts(w, split), 1)
    return F.pad(out, (0, 0, 0, rows_pad - out.shape[0])) if rows_pad else out


def pack_conv3(w, split, cin_pad=0):
    """[Cout][Cin][3][3] -> [Cout][9][(3 x) Cin_pad] bits: per tap (hi) or (hi | hi | lo), each part Cin_pad wide"""
    v = w.float().permute(0, 2, 3, 1)
    if cin_pad:
        v = F.pad(v, (0, cin_pad - v.shape[-1]))
    return torch.cat(_parts(v, split), -1).reshape(w.shape[0], -1)


def pack_convT(w, split, k, c_pad):
    """[Cin][Cout][k][k] -> [(kh k + kw) Cout_pad + co][(3 x) Cin_pad] bits"""
    cin, cout = w.shape[:2]
    v = torch.zeros(k, k, c_pad, c_pad, device=w.device)
    v[:, :, :cout, :cin] = w.float().permute(2, 3, 1, 0)
    return torch.cat(_parts(v, split), -1).reshape(k * k * c_pad, -1)


def expected_slots(sd_keys, shapes):
    """name -> (kind, arguments) of the 665 state-dict keys, as build_registry (runtime.cu) registers them"""
    out = {}
    for n in sd_keys:
        s = shapes[n]
        if n.startswith("enc_norm.") or "_rn.weight" in n and "layer_rn" not in n or \
                "refinenet4.resConfUnit1" in n:
            out[n] = ("ignore",)
        elif n.endswith(".bias") or "norm" in n and n.endswith(".weight") or n.startswith("head_pose_s.") or \
                n == "init_pose_token":
            out[n] = ("f32",)
        elif n == DPT_P + "head.4.weight":
            out[n] = ("transpose",)
        elif n in (DPT_P + "act_postprocess.0.1.weight", DPT_P + "act_postprocess.1.1.weight"):
            out[n] = ("convT", s[2], 128 if s[0] == 96 else s[0])
        elif len(s) == 4 and s[2] == 3:
            out[n] = ("conv3", 128 if s[1] == 96 else 0)
        else:
            out[n] = ("linear", 128 if s[0] == 96 else 0)
    return out


def read_slot(model_handle, name, kind, shape, split):
    """the slot of `name` as bits (int16 for bf16 packings, int32 for fp32 ones), with its padding"""
    p, ld, s = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_void_p()
    check(lib().sta_weight_slot(model_handle, name.encode(), ctypes.byref(p), ctypes.byref(ld), ctypes.byref(s)), name)
    m = 3 if split else 1
    k = kind[0]
    if k == "ignore":
        return p.value, None
    n = 1
    for d in shape:
        n *= d
    if k in ("f32", "transpose"):
        pad = 128 if name.endswith(("act_postprocess.0.0.bias", "act_postprocess.0.1.bias")) else n
        return p.value, _device_view(p.value, (pad,), "<i4")
    if k == "linear":
        rows = kind[1] or shape[0]
        assert ld.value == m * (n // shape[0]), (name, ld.value)
        return p.value, _device_view(p.value, (rows, ld.value), "<i2")
    if k == "conv3":
        cin = kind[1] or shape[1]
        return p.value, _device_view(p.value, (shape[0], 9 * m * cin), "<i2")
    kk, cp = kind[1], kind[2]
    return p.value, _device_view(p.value, (kk * kk * cp, m * cp), "<i2")


def want_slot(w, kind, split):
    k = kind[0]
    if k == "f32":
        return w.float().reshape(-1).view(torch.int32)
    if k == "transpose":
        return w.float().reshape(w.shape[0], -1).t().contiguous().reshape(-1).view(torch.int32)
    if k == "linear":
        return pack_linear(w, split, kind[1])
    if k == "conv3":
        return pack_conv3(w, split, kind[1])
    return pack_convT(w, split, kind[1], kind[2])


def check_slot(name, got, want):
    if got.shape != want.shape:
        raise AssertionError("%s: slot shape %s, packing %s" % (name, tuple(got.shape), tuple(want.shape)))
    bad = got != want
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d packed elements differ; first at %s" % (name, int(bad.sum()), bad.numel(), i))


def _check_all_slots(handle, sd, split):
    kinds = expected_slots(list(sd.keys()), {n: tuple(v.shape) for n, v in sd.items()})
    assert len(kinds) == 665
    for n, kind in kinds.items():
        ptr, got = read_slot(handle, n, kind, tuple(sd[n].shape), split)
        if kind[0] == "ignore":
            assert ptr is None, "%s is ignored by the forward but has a slot" % n
            continue
        w = sd[n].cuda()
        want = want_slot(w, kind, split)
        if got.dim() == 1 and want.numel() < got.numel():  # a bias padded to 128 channels: zeros behind it
            want = F.pad(want, (0, got.numel() - want.numel()))
        check_slot(n, got, want)


@pytest.mark.parametrize("precision", ["bf16", "x3"])
def test_packed_weights_bit_identical(request, state_dict, precision):
    model = request.getfixturevalue("cuda_model" if precision == "bf16" else "cuda_model_x3")
    torch.cuda.synchronize()
    _check_all_slots(model._handle, state_dict, precision == "x3")


def _planted(shape, g):
    """values with exact bf16 ties (hi rounds to even, truncation does not) and values with a nonzero lo part"""
    n = 1
    for d in shape:
        n *= d
    e = torch.exp2(torch.randint(-6, 3, (n,), generator=g).float())
    odd = torch.randint(0, 128, (n,), generator=g).float() * 2 + 1  # 8-bit mantissa below 2^8, odd
    kind = torch.arange(n) % 3
    tie = (128 + (odd % 128)) * 2 + 1                        # 9 bits, last one set: exactly half a bf16 ulp off
    v = torch.where(kind == 0, tie * 2.0 ** -8, torch.where(kind == 1, (128 + odd % 128) * 2.0 ** -7 + 2.0 ** -15,
                                                            torch.randn(n, generator=g)))
    sign = torch.randint(0, 2, (n,), generator=g).float() * 2 - 1
    return (v * e * sign).view(shape)


@pytest.mark.parametrize("precision", [PRECISION_BF16, PRECISION_X3])
def test_packed_weights_planted_ties_and_lo_parts(state_dict, precision):
    split = precision == PRECISION_X3
    g = torch.Generator().manual_seed(11)
    names = ["dec_block.3.mlp.fc1.weight", "dec_block.3.cross_attn.projv.weight", DPT_P + "act_postprocess.0.0.weight",
             DPT_P + "act_postprocess.0.0.bias", DPT_P + "act_postprocess.0.1.weight",
             DPT_P + "act_postprocess.1.1.weight", DPT_P + "scratch.layer_rn.0.weight",
             DPT_P + "scratch.refinenet2.resConfUnit1.conv2.weight", DPT_P + "head.4.weight", "head_pose_s.fc_rot.weight"]
    kinds = expected_slots(names, {n: tuple(state_dict[n].shape) for n in names})
    h = _Handle(precision)
    try:
        planted = {n: _planted(tuple(state_dict[n].shape), g) for n in names}
        t = planted[names[0]].reshape(-1)
        w16 = t.bfloat16().float()
        assert bool((t[::3] != w16[::3]).all()), "construction: ties"
        for n in names:
            h.load(n, planted[n])
        for n in names:
            _, got = read_slot(h.h, n, kinds[n], tuple(planted[n].shape), split)
            want = want_slot(planted[n].cuda(), kinds[n], split)
            if got.dim() == 1 and want.numel() < got.numel():
                want = F.pad(want, (0, got.numel() - want.numel()))
            check_slot(n, got, want)
    finally:
        h.close()
