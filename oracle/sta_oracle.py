"""ORACLE -- test infrastructure, not product code.

A plain-PyTorch fp32 CPU restatement of the reference STA forward pass
(zhangganlin/vista-slam, vista_slam/sta_model).  Only tests/, __graft_entry__.smoke() and the
`cpu_baseline` / `--impl reference` legs of bench.py may import this module; the product path
(vista_slam_b200/) never does, and has no CPU fallback.

Pinning: the reference ships no tests or golden vectors for this path (SURVEY.md section 4), so the
oracle is pinned against the *unmodified reference itself*, imported in the build container by
tools/make_golden.py (xformers shimmed with SDPA).  The outputs of that run are committed under
tests/golden/ and tests/test_oracle_golden.py checks this restatement against them.

Every function cites the reference file:line it restates.  Two arithmetic modes:
  * emulate_bf16=False : pure fp32 -- the reference's CPU semantics (its CUDA path adds TF32).
  * emulate_bf16=True  : GEMM/conv operands and the activations the CUDA path stores as bf16 are
    rounded to bf16 (fp32 accumulate, fp32 residual stream / LayerNorm / softmax), i.e. the same
    operand precision as the CUDA kernels, so that parity can be checked below bf16's noise floor.
"""
import math

import torch
import torch.nn.functional as F

ENC_DIM, ENC_DEPTH, ENC_HEADS = 1024, 24, 16
DEC_DIM, DEC_DEPTH, DEC_HEADS = 768, 12, 12
LN_EPS = 1e-6          # sta_model.py:43
ROPE_BASE = 100.0      # 'RoPE100', sta_model.py:44,111-112
DPT_HOOKS = (0, 7, 10, 13)  # heads/dpt_head.py:112 with dec_depth = 12


# ----------------------------------------------------------------------------------------------
# state-dict layout (SURVEY.md App. C) and a deterministic synthetic checkpoint
# ----------------------------------------------------------------------------------------------
def state_dict_spec():
    """[(name, shape)] in the reference's state_dict order (665 entries, 438,455,505 parameters)."""
    s = [("init_pose_token", (1, 1, DEC_DIM)),
         ("patch_embed.proj.weight", (ENC_DIM, 3, 16, 16)), ("patch_embed.proj.bias", (ENC_DIM,))]

    def lin(p, o, i):
        return [(p + ".weight", (o, i)), (p + ".bias", (o,))]

    def ln(p, c):
        return [(p + ".weight", (c,)), (p + ".bias", (c,))]

    for i in range(ENC_DEPTH):
        p = "enc_blocks.%d." % i
        s += ln(p + "norm1", ENC_DIM) + lin(p + "attn.qkv", 3 * ENC_DIM, ENC_DIM) + lin(p + "attn.proj", ENC_DIM, ENC_DIM)
        s += ln(p + "norm2", ENC_DIM) + lin(p + "mlp.fc1", 4 * ENC_DIM, ENC_DIM) + lin(p + "mlp.fc2", ENC_DIM, 4 * ENC_DIM)
    s += ln("enc_norm", ENC_DIM) + lin("decoder_embed", DEC_DIM, ENC_DIM)
    for i in range(DEC_DEPTH):
        p = "dec_block.%d." % i
        s += ln(p + "norm1", DEC_DIM) + lin(p + "attn.qkv", 3 * DEC_DIM, DEC_DIM) + lin(p + "attn.proj", DEC_DIM, DEC_DIM)
        for n in ("projq", "projk", "projv", "proj"):
            s += lin(p + "cross_attn." + n, DEC_DIM, DEC_DIM)
        s += ln(p + "norm2", DEC_DIM) + ln(p + "norm3", DEC_DIM)
        s += lin(p + "mlp.fc1", 4 * DEC_DIM, DEC_DIM) + lin(p + "mlp.fc2", DEC_DIM, 4 * DEC_DIM) + ln(p + "norm_y", DEC_DIM)
    s += ln("dec_norm", DEC_DIM)
    d = "downstream_head_pts.dpt."
    dims = (96, 192, 384, 768)
    for i in range(4):
        s.append((d + "scratch.layer%d_rn.weight" % (i + 1), (256, dims[i], 3, 3)))
    for i in range(4):
        s.append((d + "scratch.layer_rn.%d.weight" % i, (256, dims[i], 3, 3)))
    for i in range(1, 5):
        p = d + "scratch.refinenet%d." % i
        s += [(p + "out_conv.weight", (256, 256, 1, 1)), (p + "out_conv.bias", (256,))]
        for u in ("resConfUnit1", "resConfUnit2"):
            for c in ("conv1", "conv2"):
                s += [(p + u + "." + c + ".weight", (256, 256, 3, 3)), (p + u + "." + c + ".bias", (256,))]
    s += [(d + "head.0.weight", (128, 256, 3, 3)), (d + "head.0.bias", (128,)),
          (d + "head.2.weight", (128, 128, 3, 3)), (d + "head.2.bias", (128,)),
          (d + "head.4.weight", (4, 128, 1, 1)), (d + "head.4.bias", (4,))]
    a = d + "act_postprocess."
    s += [(a + "0.0.weight", (96, ENC_DIM, 1, 1)), (a + "0.0.bias", (96,)),
          (a + "0.1.weight", (96, 96, 4, 4)), (a + "0.1.bias", (96,)),
          (a + "1.0.weight", (192, DEC_DIM, 1, 1)), (a + "1.0.bias", (192,)),
          (a + "1.1.weight", (192, 192, 2, 2)), (a + "1.1.bias", (192,)),
          (a + "2.0.weight", (384, DEC_DIM, 1, 1)), (a + "2.0.bias", (384,)),
          (a + "3.0.weight", (768, DEC_DIM, 1, 1)), (a + "3.0.bias", (768,)),
          (a + "3.1.weight", (768, 768, 3, 3)), (a + "3.1.bias", (768,))]
    h = "head_pose_s."
    s += lin(h + "mlp.0", 512, DEC_DIM) + lin(h + "mlp.2", 512, 512) + lin(h + "mlp.4", 512, 512)
    s += lin(h + "fc_t", 3, 512) + lin(h + "fc_conf.0", 1, 512) + lin(h + "fc_rot", 9, 512)
    return s


def make_state_dict(seed=0, dtype=torch.float32):
    """Deterministic random-init checkpoint with the reference's 665 keys (there is no network for the
    real frontend_sta_weights.pth).  Weights ~ N(0, 1/fan_in), small biases, LayerNorm near identity;
    the aliased `scratch.layer{i}_rn` / `scratch.layer_rn.{i-1}` entries share one tensor as in the
    reference (dpt_block.py:33-75)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in state_dict_spec():
        if "scratch.layer_rn." in name:  # alias of scratch.layer{i+1}_rn
            idx = int(name.split("scratch.layer_rn.")[1].split(".")[0])
            sd[name] = sd[name.replace("scratch.layer_rn.%d" % idx, "scratch.layer%d_rn" % (idx + 1))]
            continue
        if name == "init_pose_token":
            t = torch.randn(shape, generator=g) * 0.02
        elif "norm" in name and name.endswith(".weight"):
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif name.endswith(".bias"):
            t = 0.02 * torch.randn(shape, generator=g)
        else:
            if "act_postprocess.0.1" in name or "act_postprocess.1.1" in name:
                fan_in = shape[0]          # ConvTranspose2d: [Cin][Cout][k][k], k == stride -> one tap per output
            else:
                fan_in = 1
                for v in shape[1:]:
                    fan_in *= v
            t = torch.randn(shape, generator=g) / math.sqrt(fan_in)
            if name.endswith("head.4.weight"):
                # keep |xyz| (= log1p of the point distance, postprocess.py:37-48) and the confidence logit
                # in the O(1) range of a trained model instead of the O(10) a variance-preserving init gives
                t = t * 0.1
        sd[name] = t.to(dtype)
    return sd


def usable_cpus(cap=32):
    """Threads the CPU legs may use: CPU affinity and cgroup quota, not os.cpu_count() (a 128-core host whose
    container is limited to a few cores thrashes badly when torch spawns 128 threads)."""
    import os
    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except Exception:
        pass
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            txt = open(path).read().split()
            if path.endswith("cpu.max"):
                if txt[0] != "max":
                    n = min(n, max(1, int(int(txt[0]) / int(txt[1]))))
            else:
                q = int(txt[0])
                if q > 0:
                    per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
                    n = min(n, max(1, q // per))
            break
        except Exception:
            continue
    return max(1, min(n, cap))


def make_images(B, H, W, seed=1234):
    """Synthetic pair batch in [-1, 1] (range of ImgNorm, utils/image.py:13)."""
    g = torch.Generator().manual_seed(seed)
    img1 = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    img2 = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    return img1, img2


# ----------------------------------------------------------------------------------------------
# building blocks
# ----------------------------------------------------------------------------------------------
def _bf16(x):
    return x.to(torch.bfloat16).to(torch.float32)


def _id(x):
    return x


def token_positions(B, h, w):
    """PositionGetter, blocks/sta_blocks.py:235-247: pos[b, y*w + x] = (y, x), int64."""
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    return torch.stack([ys.reshape(-1), xs.reshape(-1)], dim=-1)[None].expand(B, -1, -1).clone()


def rope2d(t, pos):
    """RoPE2D.forward, pos_embed/pos_embed.py:149-185 (== curope kernels.cu:17-82).
    t: [B, heads, N, 64]; pos: [B, N, 2] int (y, x), negative positions allowed."""
    d_half = t.shape[-1] // 2          # 32 features per axis
    nfreq = d_half // 2                # 16 frequencies
    inv_freq = 1.0 / (ROPE_BASE ** (torch.arange(nfreq, dtype=torch.float32) / nfreq))
    out = []
    for axis in range(2):
        part = t[..., axis * d_half:(axis + 1) * d_half]
        ang = pos[:, :, axis].to(torch.float32)[:, None, :, None] * inv_freq  # [B,1,N,16]
        cos, sin = torch.cos(ang), torch.sin(ang)
        a, b = part[..., :nfreq], part[..., nfreq:]
        out += [a * cos - b * sin, b * cos + a * sin]
    return torch.cat(out, dim=-1)


class StaOracle:
    def __init__(self, state_dict, emulate_bf16=False):
        self.sd = {k: v.to(torch.float32) for k, v in state_dict.items()}
        self.emu = bool(emulate_bf16)
        self.q = _bf16 if self.emu else _id      # rounding applied where the CUDA path stores bf16
        self._wq = {}

    # -- parameter access (weights that feed tensor-core GEMMs are bf16-rounded in emulation) --
    def w(self, name):
        if not self.emu:
            return self.sd[name]
        if name not in self._wq:
            self._wq[name] = _bf16(self.sd[name])
        return self._wq[name]

    def p(self, name):
        return self.sd[name]

    def linear(self, x, prefix):
        return F.linear(x, self.w(prefix + ".weight"), self.p(prefix + ".bias"))

    def ln(self, x, prefix):
        return F.layer_norm(x, (x.shape[-1],), self.p(prefix + ".weight"), self.p(prefix + ".bias"), LN_EPS)

    def attention(self, q, k, v):
        """softmax(q k^T / sqrt(64)) v; q,k,v: [B, heads, N, 64]
        (xformers FMHA at sta_blocks.py:143 and the naive form at sta_blocks.py:201-205)."""
        s = (q @ k.transpose(-1, -2)) * 0.125
        if not self.emu:
            return s.softmax(dim=-1) @ v
        e = torch.exp(s - s.amax(dim=-1, keepdim=True))
        return (_bf16(e) @ v) / e.sum(dim=-1, keepdim=True)  # kernel: bf16 P operand, fp32 row sum

    def mlp(self, x, prefix):
        """Mlp, sta_blocks.py:58-79: fc1 -> exact (erf) GELU -> fc2."""
        h = self.q(F.gelu(self.linear(x, prefix + ".fc1")))
        return self.linear(h, prefix + ".fc2")

    def self_attn(self, xn, pos, prefix, heads):
        """XFormer_Attention.forward, sta_blocks.py:129-148."""
        B, N, C = xn.shape
        qkv = self.linear(xn, prefix + ".qkv").reshape(B, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
        q, k, v = self.q(rope2d(qkv[0], pos)), self.q(rope2d(qkv[1], pos)), self.q(qkv[2])
        o = self.q(self.attention(q, k, v).transpose(1, 2).reshape(B, N, C))
        return self.linear(o, prefix + ".proj")

    def cross_attn(self, xn, yn, xpos, ypos, prefix, heads):
        """CrossAttention.forward, sta_blocks.py:188-208 (key = value = norm_y(y))."""
        B, Nq, C = xn.shape
        Nk = yn.shape[1]
        q = self.linear(xn, prefix + ".projq").reshape(B, Nq, heads, C // heads).transpose(1, 2)
        k = self.linear(yn, prefix + ".projk").reshape(B, Nk, heads, C // heads).transpose(1, 2)
        v = self.linear(yn, prefix + ".projv").reshape(B, Nk, heads, C // heads).transpose(1, 2)
        q, k, v = self.q(rope2d(q, xpos)), self.q(rope2d(k, ypos)), self.q(v)
        o = self.q(self.attention(q, k, v).transpose(1, 2).reshape(B, Nq, C))
        return self.linear(o, prefix + ".proj")

    # -- encoder ------------------------------------------------------------------------------
    def encode_image(self, img):
        """_encode_image(..., normalize=False), sta_model.py:163-174 with PatchEmbedDust3R
        (patch_embed.py:17-27): Conv2d(3,1024,16,16) -> tokens, then 24 x Block (sta_blocks.py:166-169).
        enc_norm is skipped exactly like every reference call site (sta_model.py:259,267; slam.py:144)."""
        B, _, H, W = img.shape
        assert H % 16 == 0 and W % 16 == 0
        h, w = H // 16, W // 16
        x = F.conv2d(self.q(img.to(torch.float32)), self.w("patch_embed.proj.weight"), self.p("patch_embed.proj.bias"),
                     stride=16)
        x = x.flatten(2).transpose(1, 2)
        pos = token_positions(B, h, w)
        for i in range(ENC_DEPTH):
            p = "enc_blocks.%d" % i
            x = x + self.self_attn(self.q(self.ln(x, p + ".norm1")), pos, p + ".attn", ENC_HEADS)
            x = x + self.mlp(self.q(self.ln(x, p + ".norm2")), p + ".mlp")
        return x, pos

    # -- decoder ------------------------------------------------------------------------------
    def dec_block(self, x, y, xpos, ypos, i):
        """DecoderBlock.forward, sta_blocks.py:226-231."""
        p = "dec_block.%d" % i
        x = x + self.self_attn(self.q(self.ln(x, p + ".norm1")), xpos, p + ".attn", DEC_HEADS)
        yn = self.q(self.ln(y, p + ".norm_y"))
        x = x + self.cross_attn(self.q(self.ln(x, p + ".norm2")), yn, xpos, ypos, p + ".cross_attn", DEC_HEADS)
        x = x + self.mlp(self.q(self.ln(x, p + ".norm3")), p + ".mlp")
        return x

    def decode_stereo(self, feat1, feat2, pos1, pos2):
        """_decode_stereo, sta_model.py:177-244: decoder_embed, prepend the learned pose token at
        position (-1,-1), 12 symmetric blocks (both directions read the layer's inputs), dec_norm on the last."""
        B = feat1.shape[0]
        tok = self.p("init_pose_token").expand(B, -1, -1)
        f1 = torch.cat([tok, self.linear(self.q(feat1), "decoder_embed")], dim=1)
        f2 = torch.cat([tok, self.linear(self.q(feat2), "decoder_embed")], dim=1)
        neg = -torch.ones(B, 1, 2, dtype=pos1.dtype)
        p1, p2 = torch.cat([neg, pos1], dim=1), torch.cat([neg, pos2], dim=1)
        out1, out2 = [f1], [f2]
        for i in range(DEC_DEPTH):
            a, b = out1[-1], out2[-1]
            out1.append(self.dec_block(a, b, p1, p2, i))
            out2.append(self.dec_block(b, a, p2, p1, i))
        out1[-1] = self.ln(out1[-1], "dec_norm")
        out2[-1] = self.ln(out2[-1], "dec_norm")
        return out1, out2

    # -- heads --------------------------------------------------------------------------------
    def conv(self, x, prefix, bias=True, **kw):
        return F.conv2d(x, self.w(prefix + ".weight"), self.p(prefix + ".bias") if bias else None, **kw)

    def rcu(self, x, prefix):
        """ResidualConvUnit_custom.forward, dpt_block.py:121-142 (bn=False, non-in-place ReLU)."""
        o = self.q(F.relu(self.conv(self.q(F.relu(x)), prefix + ".conv1", padding=1)))
        return self.conv(o, prefix + ".conv2", padding=1) + x

    def head_pts(self, tokens14, H, W):
        """head_pts = transpose_to_landscape(PixelwiseTaskWithDPT) for landscape batches:
        utils/misc.py:48-61, dpt_head.py:34-66,90-95, dpt_block.py:264-450, postprocess.py:10-62.
        tokens14 = [enc_feat] + [dec_k[:, 1:, :]] (sta_model.py:271,275)."""
        h, w = H // 16, W // 16
        lay = []
        for hook in DPT_HOOKS:
            t = self.q(tokens14[hook].to(torch.float32))
            lay.append(t.transpose(1, 2).reshape(t.shape[0], t.shape[2], h, w))
        a = "downstream_head_pts.dpt.act_postprocess."
        s = "downstream_head_pts.dpt.scratch."
        l0 = self.q(self.conv(lay[0], a + "0.0"))
        l0 = self.q(F.conv_transpose2d(l0, self.w(a + "0.1.weight"), self.p(a + "0.1.bias"), stride=4))
        l1 = self.q(self.conv(lay[1], a + "1.0"))
        l1 = self.q(F.conv_transpose2d(l1, self.w(a + "1.1.weight"), self.p(a + "1.1.bias"), stride=2))
        l2 = self.q(self.conv(lay[2], a + "2.0"))
        l3 = self.q(self.conv(lay[3], a + "3.0"))
        l3 = self.q(self.conv(l3, a + "3.1", stride=2, padding=1))
        r = [self.q(self.conv(l, s + "layer_rn.%d" % i, bias=False, padding=1)) for i, l in enumerate((l0, l1, l2, l3))]

        def fuse(idx, path, layer):
            p = s + "refinenet%d" % idx
            if layer is None:
                x = path
            else:
                x = self.q(path + self.rcu(layer, p + ".resConfUnit1"))
            x = self.q(self.rcu(x, p + ".resConfUnit2"))
            return self.q(F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)), p

        up4, p4 = fuse(4, r[3], None)
        up4 = up4[:, :, :r[2].shape[2], :r[2].shape[3]]            # dpt_head.py:58
        path4 = self.q(self.conv(up4, p4 + ".out_conv"))
        up3, p3 = fuse(3, path4, r[2])
        path3 = self.q(self.conv(up3, p3 + ".out_conv"))
        up2, p2 = fuse(2, path3, r[1])
        path2 = self.q(self.conv(up2, p2 + ".out_conv"))
        up1, p1 = fuse(1, path2, r[0])
        path1 = self.q(self.conv(up1, p1 + ".out_conv"))
        hd = "downstream_head_pts.dpt.head."
        o = self.q(self.conv(path1, hd + "0", padding=1))
        o = self.q(F.interpolate(o, scale_factor=2, mode="bilinear", align_corners=True))
        o = F.relu(self.conv(o, hd + "2", padding=1))
        # the fused CUDA epilogue keeps the 128-channel activation and the 1x1 conv in fp32
        o = F.conv2d(o, self.p(hd + "4.weight"), self.p(hd + "4.bias"))
        fmap = o.permute(0, 2, 3, 1)
        xyz = fmap[..., 0:3]
        d = xyz.norm(dim=-1, keepdim=True)
        pts3d = xyz / d.clip(min=1e-8) * torch.expm1(d)              # postprocess.py:37-48, mode 'exp'
        conf = 1.0 + fmap[..., 3].exp()                              # postprocess.py:53-58, ('exp', 1, inf)
        return {"pts3d": pts3d, "conf": conf}

    def head_pose(self, tok):
        """PoseHead_small.forward, heads/pose_head.py:109-119 (+ svd_orthogonalize :38-57,
        convert_pose_to_4x4 :94-107).  Always fp32 (slam.py:164 disables autocast around it)."""
        x = tok.to(torch.float32)
        for i in (0, 2, 4):
            x = F.relu(F.linear(x, self.p("head_pose_s.mlp.%d.weight" % i), self.p("head_pose_s.mlp.%d.bias" % i)))
        t = F.linear(x, self.p("head_pose_s.fc_t.weight"), self.p("head_pose_s.fc_t.bias"))
        r9 = F.linear(x, self.p("head_pose_s.fc_rot.weight"), self.p("head_pose_s.fc_rot.bias"))
        conf = torch.sigmoid(F.linear(x, self.p("head_pose_s.fc_conf.0.weight"), self.p("head_pose_s.fc_conf.0.bias")))
        m = F.normalize(r9.reshape(-1, 3, 3), p=2, dim=-1).transpose(-1, -2)
        u, _, vh = torch.linalg.svd(m)
        v = vh.transpose(-1, -2)
        det = torch.det(v @ u.transpose(-1, -2))
        r = torch.cat([v[:, :, :2], v[:, :, 2:] * det.view(-1, 1, 1)], dim=2) @ u.transpose(-1, -2)
        pose = torch.zeros(x.shape[0], 4, 4)
        pose[:, :3, :3] = r
        pose[:, :3, 3] = t
        pose[:, 3, 3] = 1.0
        return {"pose": pose, "conf": conf.squeeze(-1)}

    def head_pts_ts(self, tokens14, true_shape):
        """head_pts with the reference's `transpose_to_landscape` wrapper (utils/misc.py:36-82, activate = landscape_only =
        True): landscape batches run the head at (H, W) = (min, max); all-portrait batches run it at (max, min) on the
        SAME token sequence and transpose the maps; mixed batches do both per sample."""
        ts = torch.as_tensor(true_shape)
        H, W = int(ts.min()), int(ts.max())
        height, width = ts.T
        land = width >= height

        def tr(d):
            return {k: v.swapaxes(1, 2) for k, v in d.items()}
        if bool(land.all()):
            return self.head_pts(tokens14, H, W)
        if bool((~land).all()):
            return tr(self.head_pts(tokens14, W, H))
        res_l = self.head_pts([t[land] for t in tokens14], H, W)
        res_p = tr(self.head_pts([t[~land] for t in tokens14], W, H))
        out = {}
        for k in res_l:
            x = res_l[k].new_empty((len(ts),) + tuple(res_l[k].shape[1:]))
            x[land] = res_l[k]
            x[~land] = res_p[k]
            out[k] = x
        return out

    def forward_views(self, main_img, main_ts, supports):
        """forward(views) for any number of support views (sta_model.py:247-291): `supports` = [(img, true_shape)], the
        neighbour views followed by the loop views (eval mode uses all loop candidates).  Returns (main_res, support_res),
        two lists of per-support dicts."""
        mf, mpos = self.encode_image(main_img)
        main_res, sup_res = [], []
        for img, ts in supports:
            nf, npos = self.encode_image(img)
            md, nd = self.decode_stereo(mf, nf, mpos, npos)
            for feat, dec, shape, bucket in ((nf, nd, ts, sup_res), (mf, md, main_ts, main_res)):
                pts = self.head_pts_ts([feat] + [t[:, 1:, :] for t in dec], shape)
                pose = self.head_pose(dec[-1][:, 0, :])
                bucket.append({"pts3d_pred": pts["pts3d"], "conf": pts["conf"], "relative_pose": pose["pose"],
                               "relative_pose_conf": pose["conf"]})
        return main_res, sup_res

    # -- forward(views) with one support view --------------------------------------------------
    def forward_pair(self, img1, img2):
        """forward(), sta_model.py:247-291, main view = img1, one support view = img2.
        Returns (main_view_dict, support_view_dict) with the reference's output keys."""
        H, W = img1.shape[-2:]
        f1, pos1 = self.encode_image(img1)
        f2, pos2 = self.encode_image(img2)
        d1, d2 = self.decode_stereo(f1, f2, pos1, pos2)
        res = []
        for feat, dec in ((f1, d1), (f2, d2)):
            pts = self.head_pts([feat] + [t[:, 1:, :] for t in dec], H, W)
            pose = self.head_pose(dec[-1][:, 0, :])
            res.append({"pts3d_pred": pts["pts3d"], "conf": pts["conf"], "relative_pose": pose["pose"],
                        "relative_pose_conf": pose["conf"]})
        return res[0], res[1]


# algorithmic FLOPs per pair, SURVEY.md section 8(d) (verified there against FlopCounterMode on the reference)
def flops_per_pair(H, W):
    h, w = H // 16, W // 16
    N = h * w
    M = N + 1
    P4 = ((h + 1) // 2) * ((w + 1) // 2)
    enc = 2 * N * 768 * 1024 + 24 * (24 * N * 1024 ** 2 + 4 * N * N * 1024)
    dec = 2 * (2 * N * 1024 * 768) + 24 * (32 * M * 768 ** 2 + 8 * M * M * 768)
    act = (2 * N * 1024 * 96 + 32 * N * 96 ** 2 + 2 * N * 768 * 192 + 8 * N * 192 ** 2 + 2 * N * 768 * 384 +
           2 * N * 768 ** 2 + 18 * P4 * 768 ** 2)
    rn = 18 * 256 * (16 * N * 96 + 4 * N * 192 + N * 384 + P4 * 768)
    refine = (2 * P4 + 4 * N + 16 * N + 64 * N) * 2 * 9 * 256 ** 2 + (4 * P4 + 4 * N + 16 * N + 64 * N) * 2 * 256 ** 2
    head = 2 * 64 * N * 9 * 256 * 128 + 2 * 256 * N * 9 * 128 ** 2 + 2 * 256 * N * 128 * 4
    pose = 2 * (768 * 512 + 2 * 512 ** 2 + 512 * 13)
    return 2 * enc + dec + 2 * (act + rn + refine + head) + 2 * pose
