"""Drop-in host-side mirror of vista_slam/sta_model/sta_model.py::SymmetricTwoViewAssociation.

Same class name, constructor defaults, attributes, 665-key state_dict and entry points
(`_encode_image`, `_decode_stereo`, `head_pose_s`, `head_pts`, `forward(views, loop_num)`,
`load_state_dict`, `set_freeze`) as the reference (sta_model.py:26-291), so that
vista_slam/slam.py:95-106,142-189 and sta_model/train.py:208,278 (inference) call it unchanged.

Nothing is computed in PyTorch: every entry point hands raw device pointers to the hand-written
sm_90a kernels behind the C ABI (include/sta_b200.h, csrc/).  PyTorch only owns the parameter
tensors, the input/output buffers and the CUDA stream.  There is no CPU or eager fallback: a
call on a non-CUDA tensor, or without the built library, raises.
"""
import ctypes
import math
import weakref

import torch
import torch.nn as nn

from .. import _lib

inf = float("inf")

_ENC_DIM, _DEC_DIM = 1024, 768


def _param_spec():
    """(name, shape) of every state_dict entry, in the reference's order (SURVEY.md App. C)."""
    E, D = _ENC_DIM, _DEC_DIM
    spec = [("init_pose_token", (1, 1, D)), ("patch_embed.proj.weight", (E, 3, 16, 16)), ("patch_embed.proj.bias", (E,))]

    def dense(prefix, n_out, n_in):
        spec.append((prefix + ".weight", (n_out, n_in)))
        spec.append((prefix + ".bias", (n_out,)))

    def norm(prefix, c):
        spec.append((prefix + ".weight", (c,)))
        spec.append((prefix + ".bias", (c,)))

    for i in range(24):
        b = "enc_blocks.%d" % i
        norm(b + ".norm1", E)
        dense(b + ".attn.qkv", 3 * E, E)
        dense(b + ".attn.proj", E, E)
        norm(b + ".norm2", E)
        dense(b + ".mlp.fc1", 4 * E, E)
        dense(b + ".mlp.fc2", E, 4 * E)
    norm("enc_norm", E)
    dense("decoder_embed", D, E)
    for i in range(12):
        b = "dec_block.%d" % i
        norm(b + ".norm1", D)
        dense(b + ".attn.qkv", 3 * D, D)
        dense(b + ".attn.proj", D, D)
        for nm in ("projq", "projk", "projv", "proj"):
            dense(b + ".cross_attn." + nm, D, D)
        norm(b + ".norm2", D)
        norm(b + ".norm3", D)
        dense(b + ".mlp.fc1", 4 * D, D)
        dense(b + ".mlp.fc2", D, 4 * D)
        norm(b + ".norm_y", D)
    norm("dec_norm", D)
    dpt = "downstream_head_pts.dpt."
    widths = (96, 192, 384, 768)
    for i, c in enumerate(widths):
        spec.append((dpt + "scratch.layer%d_rn.weight" % (i + 1), (256, c, 3, 3)))
    for i, c in enumerate(widths):  # same Parameters, second name (aliases)
        spec.append((dpt + "scratch.layer_rn.%d.weight" % i, (256, c, 3, 3)))
    for i in range(1, 5):
        r = dpt + "scratch.refinenet%d." % i
        spec.append((r + "out_conv.weight", (256, 256, 1, 1)))
        spec.append((r + "out_conv.bias", (256,)))
        for unit in ("resConfUnit1", "resConfUnit2"):
            for cv in ("conv1", "conv2"):
                spec.append((r + unit + "." + cv + ".weight", (256, 256, 3, 3)))
                spec.append((r + unit + "." + cv + ".bias", (256,)))
    for nm, shp in (("head.0", (128, 256, 3, 3)), ("head.2", (128, 128, 3, 3)), ("head.4", (4, 128, 1, 1))):
        spec.append((dpt + nm + ".weight", shp))
        spec.append((dpt + nm + ".bias", (shp[0],)))
    act = dpt + "act_postprocess."
    for nm, shp in (("0.0", (96, E, 1, 1)), ("0.1", (96, 96, 4, 4)), ("1.0", (192, D, 1, 1)), ("1.1", (192, 192, 2, 2)),
                    ("2.0", (384, D, 1, 1)), ("3.0", (768, D, 1, 1)), ("3.1", (768, 768, 3, 3))):
        spec.append((act + nm + ".weight", shp))
        spec.append((act + nm + ".bias", (shp[1] if nm in ("0.1", "1.1") else shp[0],)))
    ph = "head_pose_s."
    dense(ph + "mlp.0", 512, D)
    dense(ph + "mlp.2", 512, 512)
    dense(ph + "mlp.4", 512, 512)
    dense(ph + "fc_t", 3, 512)
    dense(ph + "fc_conf.0", 1, 512)
    dense(ph + "fc_rot", 9, 512)
    return spec


class _Node(nn.Module):
    """Parameter container; the module tree only exists to reproduce the reference's state_dict names."""


class _PatchEmbedNode(_Node):
    patch_size = (16, 16)


class _PoseHeadNode(_Node):
    """`model.head_pose_s(tok)` (heads/pose_head.py:109-119) -> {'pose': (B,4,4), 'conf': (B,)}."""

    def forward(self, pose_token):
        owner = self._owner()
        if owner is None:
            raise RuntimeError("head_pose_s lost its model")
        return owner._pose_head(pose_token)


def _attach(root, dotted, param):
    parts = dotted.split(".")
    node = root
    for key in parts[:-1]:
        child = node._modules.get(key)
        if child is None:
            if node is root and key == "patch_embed":
                child = _PatchEmbedNode()
            elif node is root and key == "head_pose_s":
                child = _PoseHeadNode()
            else:
                child = _Node()
            node.add_module(key, child)
        node = child
    node.register_parameter(parts[-1], param)


class SymmetricTwoViewAssociation(nn.Module):
    """H100-native STA frontend with the reference's module surface (sta_model.py:26-52 for the defaults)."""

    def __init__(self, img_size=(224, 224), patch_size=16, enc_embed_dim=1024, enc_depth=24, enc_num_heads=16,
                 dec_embed_dim=768, dec_depth=12, dec_num_heads=12, mlp_ratio=4, norm_layer=None, pos_embed="RoPE100",
                 output_mode="pts3d", head_type="dpt", depth_mode=("exp", -inf, inf), conf_mode=("exp", 1, inf),
                 freeze="none", landscape_only=True, patch_embed_cls="PatchEmbedDust3R", precision="bf16"):
        super().__init__()
        # `precision` is the one extension of the reference signature: "bf16" (production; every benchmark number),
        # "x3" = split-precision parity mode (include/sta_b200.h, STA_PRECISION_X3) used by the parity tests, or "fp8" =
        # e4m3 operands with block scales for the encoder and decoder linears (STA_PRECISION_FP8): an opt-in that changes
        # the numerics (INTEGRATION.md section 5).
        if precision not in ("bf16", "x3", "fp8"):
            raise ValueError("precision must be 'bf16', 'x3' or 'fp8'")
        self.precision = precision
        fixed = dict(patch_size=(patch_size, 16), enc_embed_dim=(enc_embed_dim, 1024), enc_depth=(enc_depth, 24),
                     enc_num_heads=(enc_num_heads, 16), dec_embed_dim=(dec_embed_dim, 768), dec_depth=(dec_depth, 12),
                     dec_num_heads=(dec_num_heads, 12), mlp_ratio=(mlp_ratio, 4), pos_embed=(pos_embed, "RoPE100"),
                     output_mode=(output_mode, "pts3d"), head_type=(head_type, "dpt"),
                     depth_mode=(tuple(depth_mode), ("exp", -inf, inf)), conf_mode=(tuple(conf_mode), ("exp", 1, inf)),
                     patch_embed_cls=(patch_embed_cls, "PatchEmbedDust3R"))
        for k, (got, want) in fixed.items():
            if got != want:
                raise NotImplementedError(
                    "the sm_90a kernels are specialised for the reference's default STA() configuration; "
                    "%s=%r is not supported (expected %r)" % (k, got, want))
        if norm_layer is not None:
            probe = norm_layer(8)
            if not isinstance(probe, nn.LayerNorm) or abs(probe.eps - 1e-6) > 1e-12:
                raise NotImplementedError("norm_layer must be LayerNorm(eps=1e-6)")
        self.img_size = img_size
        self.patch_size = patch_size
        self.enc_depth, self.enc_embed_dim = enc_depth, enc_embed_dim
        self.dec_depth, self.dec_embed_dim = dec_depth, dec_embed_dim
        self.pos_embed = pos_embed
        self.enc_pos_embed = None
        self.dec_pos_embed = None
        self.output_mode, self.head_type = output_mode, head_type
        self.depth_mode, self.conf_mode = tuple(depth_mode), tuple(conf_mode)
        self.landscape_only = landscape_only

        gen = torch.Generator().manual_seed(0)
        aliases = {}
        for name, shape in _param_spec():
            if ".scratch.layer_rn." in name:
                idx = int(name.split(".scratch.layer_rn.")[1].split(".")[0])
                _attach(self, name, aliases["layer%d_rn" % (idx + 1)])
                continue
            if name == "init_pose_token":
                t = torch.randn(shape, generator=gen) * 0.02
            elif len(shape) == 1:
                t = torch.ones(shape) if (".norm" in name or name.startswith(("enc_norm", "dec_norm"))) and \
                    name.endswith("weight") else torch.zeros(shape)
            else:
                fan_in = 1
                for v in shape[1:]:
                    fan_in *= v
                bound = 1.0 / math.sqrt(fan_in)
                t = (torch.rand(shape, generator=gen) * 2 - 1) * bound
            p = nn.Parameter(t, requires_grad=True)
            _attach(self, name, p)
            if ".scratch.layer" in name and "_rn." in name:
                aliases[name.split(".scratch.")[1].split(".")[0]] = p
        self.head_pose_s._owner = weakref.ref(self)
        self._handle = None
        self._uploaded_key = None
        self.set_freeze(freeze)

    # ------------------------------------------------------------------ reference API: housekeeping
    def load_state_dict(self, ckpt, **kw):  # sta_model.py:143-144
        out = super().load_state_dict(ckpt, **kw)
        self._uploaded_key = None
        self._weights_external = False  # an explicit checkpoint replaces broadcast weights
        return out

    def set_freeze(self, freeze):  # sta_model.py:148-161
        if freeze == "none":
            return
        if freeze == "encoder":
            for name, p in self.named_parameters():
                if name.startswith(("patch_embed.", "enc_blocks.")):
                    p.requires_grad = False
            return
        raise NotImplementedError("freeze=%s not implemented" % freeze)

    def _apply(self, fn, *a, **kw):  # .to() / .cuda() / .float(): weights must be re-packed
        out = super()._apply(fn, *a, **kw)
        self._uploaded_key = None
        return out

    def __del__(self):
        h = getattr(self, "_handle", None)
        if h is not None:
            try:
                _lib.lib().sta_destroy(h)
            except Exception:
                pass

    # ------------------------------------------------------------------ weights -> C library
    def _state_key(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _ready(self, like):
        """Create the C handle on the tensor's device and (re-)upload the packed weights if needed."""
        if not like.is_cuda:
            raise RuntimeError("vista_slam_b200 runs only on CUDA (sm_90a) tensors; there is no CPU path")
        L = _lib.lib()
        key = (like.device.index, self._state_key())
        if self._handle is not None and self._uploaded_key == key:
            return L
        if getattr(self, "_weights_external", False) and self._handle is not None:
            if self._uploaded_key is not None and self._uploaded_key[0] != like.device.index:
                raise RuntimeError("this replica's weights were broadcast to cuda:%s; it cannot run on cuda:%s"
                                   % (self._uploaded_key[0], like.device.index))
            return L  # broadcast weights: the local parameters are placeholders and must not overwrite the arena
        with torch.cuda.device(like.device):
            if self._handle is None:
                self._handle = self._create(L)
            # sta_load_tensor packs on the legacy default stream: make sure dtype conversions / copies issued on the
            # current (possibly non-blocking) torch stream have landed before the library reads the tensors
            torch.cuda.current_stream().synchronize()
            for name, t in self.state_dict().items():
                src = t.detach()
                on_dev = 1 if src.is_cuda else 0
                src = src.to(torch.float32).contiguous()
                if on_dev and src.data_ptr() != t.data_ptr():
                    torch.cuda.current_stream().synchronize()  # a conversion kernel was just enqueued on the torch stream
                shape = (ctypes.c_int64 * src.dim())(*src.shape)
                _lib.check(L.sta_load_tensor(self._handle, name.encode(), _lib.ptr(src), shape, src.dim(), on_dev),
                           "sta_load_tensor(%s)" % name)
            missing = L.sta_missing_tensors(self._handle)
            if missing != 0:
                raise RuntimeError("%d state-dict tensors missing after upload" % missing)
        self._uploaded_key = key
        return L

    def _create(self, L):
        h = ctypes.c_void_p()
        prec = {"bf16": _lib.PRECISION_BF16, "x3": _lib.PRECISION_X3, "fp8": _lib.PRECISION_FP8}[self.precision]
        _lib.check(L.sta_create_ex(ctypes.byref(h), prec), "sta_create_ex")
        return h

    def weight_arena(self):
        """uint8 CUDA tensor aliasing the library's packed-weight arena (for a NCCL broadcast)."""
        if self._handle is None:
            raise RuntimeError("model has no device handle yet")
        p, n = ctypes.c_void_p(), ctypes.c_int64()
        _lib.check(_lib.lib().sta_weight_arena(self._handle, ctypes.byref(p), ctypes.byref(n)), "sta_weight_arena")

        class _Arena:
            __cuda_array_interface__ = {"shape": (n.value,), "typestr": "|u1", "data": (p.value, False), "version": 2}

        return torch.as_tensor(_Arena(), device="cuda")

    def broadcast_weights(self, src=0, group=None, device=None):
        """One NCCL broadcast of the packed weight arena from rank `src` (per-rank independent inference
        afterwards).  Non-source ranks need no state dict."""
        import torch.distributed as dist
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if device.index is None:  # 'cuda' -> the concrete ordinal, so that _ready() computes the same key later
            device = torch.device("cuda", torch.cuda.current_device())
        probe = torch.empty(1, device=device)
        L = _lib.lib()
        if dist.get_rank(group) == src:
            self._ready(probe)
        else:
            with torch.cuda.device(device):
                if self._handle is None:
                    self._handle = self._create(L)
        with torch.cuda.device(device):
            arena = self.weight_arena()
            dist.broadcast(arena, src=src, group=group)
            torch.cuda.synchronize()
        if dist.get_rank(group) != src:
            _lib.check(L.sta_mark_all_loaded(self._handle), "sta_mark_all_loaded")
            self._uploaded_key = (device.index, self._state_key())
            # the arena now holds rank `src`'s weights, NOT this module's (random-init) parameters: never re-upload
            self._weights_external = True

    # ------------------------------------------------------------------ reference API: compute
    @torch.no_grad()
    def _encode_image(self, image, true_shape=None, normalize=True):
        """sta_model.py:163-174 -> (x (B,N,1024) fp32, pos (B,N,2) int64)."""
        L = self._ready(image)
        if image.dim() != 4 or image.shape[1] != 3:
            raise ValueError("image must be (B,3,H,W)")
        B, _, H, W = image.shape
        assert H % 16 == 0, "Input image height (%d) is not a multiple of patch size (16)." % H
        assert W % 16 == 0, "Input image width (%d) is not a multiple of patch size (16)." % W
        if image.dtype not in (torch.float32, torch.bfloat16):
            image = image.float()
        image = image.contiguous()
        N = (H // 16) * (W // 16)
        feat = torch.empty(B, N, 1024, device=image.device, dtype=torch.float32)
        pos = torch.empty(B, N, 2, device=image.device, dtype=torch.int64)
        with torch.cuda.device(image.device):
            _lib.check(L.sta_encode(self._handle, _lib.ptr(image), int(image.dtype == torch.bfloat16), B, H, W,
                                    _lib.ptr(feat), _lib.ptr(pos), _lib.cur_stream()), "sta_encode")
        if normalize:  # never used by the reference's callers (normalize=False at sta_model.py:259,267, slam.py:144)
            feat = torch.nn.functional.layer_norm(feat, (1024,), self.enc_norm.weight, self.enc_norm.bias, 1e-6)
        return feat, pos

    @torch.no_grad()
    def _decode_stereo(self, feat1, feat2, pose1, pose2, layers=None):
        """sta_model.py:177-244 -> (list[13] of (B,N+1,768), list[13]); `layers` (extension) restricts which
        of the 13 per-layer outputs are materialised (others are None)."""
        L = self._ready(feat1)
        B, N, C = feat1.shape
        if C != 1024 or feat2.shape != feat1.shape:
            raise ValueError("features must both be (B,N,1024)")
        want = range(13) if layers is None else layers
        f1, f2 = feat1.float().contiguous(), feat2.float().contiguous()
        p1, p2 = pose1.to(torch.int64).contiguous(), pose2.to(torch.int64).contiguous()
        outs = []
        arrs = []
        for _ in range(2):
            lst = [None] * 13
            arr = (ctypes.c_void_p * 13)()
            for i in want:
                lst[i] = torch.empty(B, N + 1, 768, device=f1.device, dtype=torch.float32)
                arr[i] = lst[i].data_ptr()
            outs.append(lst)
            arrs.append(arr)
        with torch.cuda.device(f1.device):
            _lib.check(L.sta_decode(self._handle, _lib.ptr(f1), _lib.ptr(f2), _lib.ptr(p1), _lib.ptr(p2), B, N,
                                    arrs[0], arrs[1], _lib.cur_stream()), "sta_decode")
        return outs[0], outs[1]

    @torch.no_grad()
    def _pose_head(self, tok):
        L = self._ready(tok)
        if tok.dim() != 2 or tok.shape[1] != 768:
            raise ValueError("pose token must be (B,768)")
        t = tok.float().contiguous()
        B = t.shape[0]
        pose = torch.empty(B, 4, 4, device=t.device, dtype=torch.float32)
        conf = torch.empty(B, device=t.device, dtype=torch.float32)
        with torch.cuda.device(t.device):
            _lib.check(L.sta_head_pose(self._handle, _lib.ptr(t), B, _lib.ptr(pose), _lib.ptr(conf), _lib.cur_stream()),
                       "sta_head_pose")
        return {"pose": pose, "conf": conf}

    @torch.no_grad()
    def _dpt(self, tokens, H, W):
        L = self._ready(tokens[0])
        t = [tokens[i].float().contiguous() for i in (0, 7, 10, 13)]  # hooks, heads/dpt_head.py:112
        B = t[0].shape[0]
        pts = torch.empty(B, H, W, 3, device=t[0].device, dtype=torch.float32)
        conf = torch.empty(B, H, W, device=t[0].device, dtype=torch.float32)
        with torch.cuda.device(t[0].device):
            _lib.check(L.sta_head_pts(self._handle, _lib.ptr(t[0]), _lib.ptr(t[1]), _lib.ptr(t[2]), _lib.ptr(t[3]), B, H, W,
                                      _lib.ptr(pts), _lib.ptr(conf), _lib.cur_stream()), "sta_head_pts")
        return {"pts3d": pts, "conf": conf}

    def head_pts(self, decout, true_shape):
        """transpose_to_landscape(PixelwiseTaskWithDPT), sta_model.py:135-137 + utils/misc.py:36-82."""
        ts = torch.as_tensor(true_shape)
        if not self.landscape_only:
            assert bool((ts[0:1] == ts).all()), "true_shape must be all identical"
            H, W = [int(v) for v in ts[0].tolist()]
            return self._dpt(decout, H, W)
        H, W = int(ts.min()), int(ts.max())
        height, width = ts.T
        is_landscape = width >= height
        if bool(is_landscape.all()):
            return self._dpt(decout, H, W)
        if bool((~is_landscape).all()):
            return {k: v.swapaxes(1, 2) for k, v in self._dpt(decout, W, H).items()}
        # only the hooked layers are read (heads/dpt_head.py:112); forward() passes None for the others
        res_l = self._dpt([None if d is None else d[is_landscape] for d in decout], H, W)
        res_p = {k: v.swapaxes(1, 2)
                 for k, v in self._dpt([None if d is None else d[~is_landscape] for d in decout], W, H).items()}
        out = {}
        for k in res_l:
            x = res_l[k].new_empty((len(ts),) + tuple(res_l[k].shape[1:]))
            x[is_landscape] = res_l[k]
            x[~is_landscape] = res_p[k]
            out[k] = x
        return out

    @torch.no_grad()
    def forward_pairs(self, img1, img2):
        """Fused fast path for a batch of B pairs (one support view): 2 encodes + symmetric decode + 2 DPT +
        2 pose heads in one C call.  Returns (main_dict, support_dict) with the reference's output keys."""
        L = self._ready(img1)
        if img1.shape != img2.shape or img1.dim() != 4 or img1.shape[1] != 3:
            raise ValueError("img1/img2 must both be (B,3,H,W)")
        if img1.dtype != img2.dtype or img1.dtype not in (torch.float32, torch.bfloat16):
            img1, img2 = img1.float(), img2.float()
        img1, img2 = img1.contiguous(), img2.contiguous()
        B, _, H, W = img1.shape
        dev = img1.device
        pts = torch.empty(2, B, H, W, 3, device=dev, dtype=torch.float32)
        conf = torch.empty(2, B, H, W, device=dev, dtype=torch.float32)
        pose = torch.empty(2, B, 4, 4, device=dev, dtype=torch.float32)
        pconf = torch.empty(2, B, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _lib.check(L.sta_forward_pairs(self._handle, _lib.ptr(img1), _lib.ptr(img2), int(img1.dtype == torch.bfloat16),
                                           B, H, W, _lib.ptr(pts), _lib.ptr(conf), _lib.ptr(pose), _lib.ptr(pconf),
                                           _lib.cur_stream()), "sta_forward_pairs")
        if self.landscape_only and H > W:
            # all-portrait batch: the reference's head wrapper returns the maps transposed to landscape
            # (transpose_to_landscape, utils/misc.py:48-61) -- same here, as a view
            pts, conf = pts.swapaxes(2, 3), conf.swapaxes(2, 3)
        return tuple({"pts3d_pred": pts[v], "conf": conf[v], "relative_pose": pose[v], "relative_pose_conf": pconf[v]}
                     for v in range(2))

    @torch.no_grad()
    def forward_pairs_host(self, img1, img2, out=None):
        """End-to-end variant with HOST tensors (pinned recommended): H2D copies, forward, D2H copies and a
        stream synchronise all happen inside the C call (sta_forward_pairs_host).  The maps come back in the image's own
        (H, W) orientation: no landscape transposition is applied to the caller's buffers."""
        if img1.is_cuda or img2.is_cuda:
            raise ValueError("forward_pairs_host takes host tensors")
        L = self._ready(torch.empty(1, device="cuda"))
        B, _, H, W = img1.shape
        if out is None:
            out = {"pts3d": torch.empty(2, B, H, W, 3).pin_memory(), "conf": torch.empty(2, B, H, W).pin_memory(),
                   "pose": torch.empty(2, B, 4, 4).pin_memory(), "pose_conf": torch.empty(2, B).pin_memory()}
        _lib.check(L.sta_forward_pairs_host(self._handle, _lib.ptr(img1), _lib.ptr(img2), int(img1.dtype == torch.bfloat16),
                                            B, H, W, _lib.ptr(out["pts3d"]), _lib.ptr(out["conf"]), _lib.ptr(out["pose"]),
                                            _lib.ptr(out["pose_conf"]), _lib.cur_stream()), "sta_forward_pairs_host")
        return out

    @torch.no_grad()
    def forward(self, views: dict, loop_num=0):
        """sta_model.py:247-291: main view against every neighbour / loop view."""
        main_view = views["main_view"]
        loop_candidates = views["loop_views"]
        if not self.training:
            loop_num = len(loop_candidates)
        support_views = views["neighbor_views"] + loop_candidates[:loop_num]
        main_res, support_res = [], []
        if len(support_views) == 1 and self.landscape_only and _same_landscape(main_view, support_views[0]):
            m, s = self.forward_pairs(main_view["img"], support_views[0]["img"])
            return {"main_views": [m], "support_views": [s]}
        main_feat, main_pos = self._encode_image(main_view["img"], main_view["true_shape"], normalize=False)
        for n_view in support_views:
            n_feat, n_pos = self._encode_image(n_view["img"], n_view["true_shape"], normalize=False)
            main_dec, n_dec = self._decode_stereo(main_feat, n_feat, main_pos, n_pos, layers=(6, 9, 12))
            for feat, dec, view, bucket in ((n_feat, n_dec, n_view, support_res), (main_feat, main_dec, main_view, main_res)):
                toks = [feat] + [None if t is None else t[:, 1:, :] for t in dec]
                pts = self.head_pts(toks, view["true_shape"])
                pose = self.head_pose_s(dec[-1][:, 0, :])
                bucket.append({"pts3d_pred": pts["pts3d"], "conf": pts["conf"], "relative_pose": pose["pose"],
                               "relative_pose_conf": pose["conf"]})
        return {"main_views": main_res, "support_views": support_res}

    @property
    def launch_count(self):
        return 0 if self._handle is None else int(_lib.lib().sta_launch_count(self._handle))

    @property
    def device_bytes(self):
        return 0 if self._handle is None else int(_lib.lib().sta_device_bytes(self._handle))


def _same_landscape(a, b):
    sa, sb = torch.as_tensor(a["true_shape"]), torch.as_tensor(b["true_shape"])
    if a["img"].shape != b["img"].shape:
        return False
    H, W = a["img"].shape[-2:]
    ok = bool((sa == sa.new_tensor([H, W])).all()) and bool((sb == sb.new_tensor([H, W])).all())
    return ok and W >= H
