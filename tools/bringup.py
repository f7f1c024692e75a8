"""GPU bring-up of the op-level kernels against plain torch fp32 references (run under gpurun).

    python tools/bringup.py            # runs every group in its own subprocess (a trap kills only that group)
    python tools/bringup.py <group>    # run one group in-process

Prints one line per check: name, max abs err, max ref magnitude, PASS/FAIL.
"""
import math
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

GROUPS = ["gemm_basic", "gemm_epi", "conv", "coalesced_epi", "attention", "misc", "x3", "perf"]


def report(name, got, ref, tol):
    import torch
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs().max().item()
    mag = ref.abs().max().item()
    bad = not math.isfinite(err) or err > tol * max(mag, 1e-6)
    print("%-44s err=%.3e ref_max=%.3e rel=%.2e %s" % (name, err, mag, err / max(mag, 1e-12), "FAIL" if bad else "PASS"),
          flush=True)
    return not bad


def gemm_desc(**kw):
    from vista_slam_b200._lib import StaGemmDesc
    d = StaGemmDesc()
    for k, v in kw.items():
        if hasattr(v, "data_ptr"):
            v = v.data_ptr()
        setattr(d, k, v)
    return d


def run_gemm(d):
    import ctypes
    from vista_slam_b200._lib import check, cur_stream, lib
    check(lib().sta_op_gemm(ctypes.byref(d), cur_stream()), "sta_op_gemm")


def group_gemm_basic():
    import torch
    from vista_slam_b200._lib import EPI_BF16
    torch.manual_seed(0)
    dev = "cuda"
    for (M, N, K) in [(128, 256, 64), (300, 512, 192), (128, 256, 1024), (8192, 1024, 1024), (1000, 384, 768),
                      (24608, 768, 768)]:
        A = torch.randn(M, K, device=dev).bfloat16()
        W = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
        bias = torch.randn(N, device=dev)
        out = torch.full((M, N), float("nan"), device=dev, dtype=torch.bfloat16)
        d = gemm_desc(conv3x3=0, epi=EPI_BF16, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=out, ldo=N)
        run_gemm(d)
        torch.cuda.synchronize()
        ref = A.float() @ W.float().t() + bias
        report("gemm bf16 M%d N%d K%d" % (M, N, K), out, ref, 1e-2)


def rope_ref(x, pos):
    """x: [rows, heads, 64] fp32, pos: [rows, 2] -> rotated (pos_embed.py:149-185 semantics)."""
    import torch
    inv = 1.0 / (100.0 ** (torch.arange(16, device=x.device, dtype=torch.float32) / 16))
    out = x.clone()
    for axis in range(2):
        ang = pos[:, axis].float()[:, None] * inv[None, :]
        cos = ang.cos()[:, None, :]
        sin = ang.sin()[:, None, :]
        a = x[..., axis * 32: axis * 32 + 16]
        b = x[..., axis * 32 + 16: axis * 32 + 32]
        out[..., axis * 32: axis * 32 + 16] = a * cos - b * sin
        out[..., axis * 32 + 16: axis * 32 + 32] = b * cos + a * sin
    return out


def group_gemm_epi():
    import torch
    import torch.nn.functional as F
    from vista_slam_b200._lib import EPI_BF16, EPI_F32, EPI_GELU, EPI_PIXSHUF, EPI_ROPE
    torch.manual_seed(1)
    dev = "cuda"
    M, N, K = 777, 512, 256
    A = torch.randn(M, K, device=dev).bfloat16()
    W = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=dev)
    base = A.float() @ W.float().t() + bias
    # GELU
    out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(epi=EPI_GELU, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=out, ldo=N))
    report("epi gelu", out, F.gelu(base), 1e-2)
    # BF16 + resid + resid2 + relu copy
    r1 = torch.randn(M, N, device=dev).bfloat16()
    r2 = torch.randn(M, N, device=dev).bfloat16()
    out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    out2 = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(epi=EPI_BF16, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=out, ldo=N, out2=out2,
                       resid=r1, resid2=r2))
    ref = base + r1.float() + r2.float()
    report("epi bf16 resid x2", out, ref, 1e-2)
    report("epi bf16 relu copy", out2, ref.relu(), 1e-2)
    out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(epi=EPI_BF16, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=out, ldo=N, relu_main=1))
    report("epi bf16 relu main", out, base.relu(), 1e-2)
    # N = 384: an odd number of 128-column tiles, no bias
    W3 = (torch.randn(384, K, device=dev) / math.sqrt(K)).bfloat16()
    out = torch.zeros(M, 384, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(epi=EPI_BF16, A=A, lda=K, W=W3, ldw=K, M=M, N=384, K=K, out=out, ldo=384))
    report("epi bf16 N384 (no bias)", out, A.float() @ W3.float().t(), 1e-2)
    # F32 with residual in place
    x = torch.randn(M, N, device=dev)
    x0 = x.clone()
    run_gemm(gemm_desc(epi=EPI_F32, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=x, ldo=N, resid=x))
    report("epi f32 resid in place", x, x0 + base, 2e-3)
    # F32 without residual (plain fp32 store) and with a separate residual tensor
    y = torch.zeros(M, N, device=dev)
    run_gemm(gemm_desc(epi=EPI_F32, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=y, ldo=N))
    report("epi f32 no resid", y, base, 2e-3)
    y = torch.zeros(M, N, device=dev)
    run_gemm(gemm_desc(epi=EPI_F32, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=y, ldo=N, resid=x0))
    report("epi f32 resid separate", y, x0 + base, 2e-3)
    # F32 with rowmap (decoder_embed): 7 samples x 111 tokens
    nt = 111
    xd = torch.zeros(7 * (nt + 1), N, device=dev)
    run_gemm(gemm_desc(epi=EPI_F32, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=xd, ldo=N, rowmap_n=nt))
    ref = torch.zeros(7, nt + 1, N, device=dev)
    ref[:, 1:] = base.view(7, nt, N)
    report("epi f32 rowmap", xd, ref.view(-1, N), 2e-3)
    # ROPE: N = 3*256 (4 heads), rope on first 512 columns, positions incl. -1
    C = 256
    Wq = (torch.randn(3 * C, K, device=dev) / math.sqrt(K)).bfloat16()
    bq = torch.randn(3 * C, device=dev)
    pos = torch.randint(-1, 40, (M, 2), device=dev, dtype=torch.int32)
    out = torch.zeros(M, 3 * C, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(epi=EPI_ROPE, A=A, lda=K, W=Wq, ldw=K, M=M, N=3 * C, K=K, bias=bq, out=out, ldo=3 * C, pos=pos,
                       rope_cols=2 * C))
    qkv = A.float() @ Wq.float().t() + bq
    ref = qkv.clone()
    ref[:, :2 * C] = rope_ref(qkv[:, :2 * C].reshape(M, 8, 64), pos).reshape(M, 2 * C)
    report("epi rope", out, ref, 1e-2)
    # small-problem route (SLAM mode: one 224x224 keyframe = 196 tokens): 128-wide single-CTA tiles, split-K for the
    # in-place fp32 layers (with scratch), TMA reduce-add without scratch
    Ms, Ks = 196, 1024
    As = torch.randn(Ms, Ks, device=dev).bfloat16()
    Wl = (torch.randn(1024, Ks, device=dev) / math.sqrt(Ks)).bfloat16()
    bl = torch.randn(1024, device=dev)
    refs = As.float() @ Wl.float().t() + bl
    ws = torch.zeros(8 * 256 * 1024, device=dev)
    for name, kw in (("split-K", dict(splitk_ws=ws, splitk_ws_bytes=ws.numel() * 4)), ("reduce-add", {})):
        xs = torch.randn(Ms, 1024, device=dev)
        x0s = xs.clone()
        run_gemm(gemm_desc(epi=EPI_F32, A=As, lda=Ks, W=Wl, ldw=Ks, M=Ms, N=1024, K=Ks, bias=bl, out=xs, ldo=1024, resid=xs,
                           **kw))
        report("small M196 f32 in place (%s)" % name, xs, x0s + refs, 2e-3)
    ys = torch.zeros(Ms, 1024, device=dev)
    run_gemm(gemm_desc(epi=EPI_F32, A=As, lda=Ks, W=Wl, ldw=Ks, M=Ms, N=1024, K=Ks, bias=bl, out=ys, ldo=1024,
                       splitk_ws=ws, splitk_ws_bytes=ws.numel() * 4))
    report("small M196 f32 no resid (split-K)", ys, refs, 2e-3)
    outs = torch.zeros(Ms, 1024, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(epi=EPI_GELU, A=As, lda=Ks, W=Wl, ldw=Ks, M=Ms, N=1024, K=Ks, bias=bl, out=outs, ldo=1024))
    report("small M196 gelu", outs, F.gelu(refs), 1e-2)
    poss = torch.randint(-1, 14, (Ms, 2), device=dev, dtype=torch.int32)
    run_gemm(gemm_desc(epi=EPI_ROPE, A=As, lda=Ks, W=Wl, ldw=Ks, M=Ms, N=1024, K=Ks, bias=bl, out=outs, ldo=1024, pos=poss,
                       rope_cols=768))
    refr = refs.clone()
    refr[:, :768] = rope_ref(refs[:, :768].reshape(Ms, 12, 64), poss).reshape(Ms, 768)
    report("small M196 rope", outs, refr, 1e-2)
    # the same epilogues on a problem wide enough to fill every SM with 128 x 128 tiles (TMA-store epilogue)
    Mw, Kw = 5000, 256
    Aw = torch.randn(Mw, Kw, device=dev).bfloat16()
    Ww = (torch.randn(1024, Kw, device=dev) / math.sqrt(Kw)).bfloat16()
    refw = Aw.float() @ Ww.float().t() + bl
    outw = torch.zeros(Mw, 1024, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(epi=EPI_GELU, A=Aw, lda=Kw, W=Ww, ldw=Kw, M=Mw, N=1024, K=Kw, bias=bl, out=outw, ldo=1024))
    report("wide M5000 gelu", outw, F.gelu(refw), 1e-2)
    posw = torch.randint(-1, 70, (Mw, 2), device=dev, dtype=torch.int32)
    run_gemm(gemm_desc(epi=EPI_ROPE, A=Aw, lda=Kw, W=Ww, ldw=Kw, M=Mw, N=1024, K=Kw, bias=bl, out=outw, ldo=1024, pos=posw,
                       rope_cols=768))
    refr = refw.clone()
    refr[:, :768] = rope_ref(refw[:, :768].reshape(Mw, 12, 64), posw).reshape(Mw, 768)
    report("wide M5000 rope (positions beyond the smem table)", outw, refr, 1e-2)
    xw = torch.randn(Mw, 1024, device=dev)
    xw0 = xw.clone()
    run_gemm(gemm_desc(epi=EPI_F32, A=Aw, lda=Kw, W=Ww, ldw=Kw, M=Mw, N=1024, K=Kw, bias=bl, out=xw, ldo=1024, resid=xw))
    report("wide M5000 f32 in place (reduce-add)", xw, xw0 + refw, 2e-3)
    # a full-size in-place fp32 layer: 24576 x 1024 = 1536 tiles, many waves of the persistent grid
    Mt, Kt = 24576, 256
    At = torch.randn(Mt, Kt, device=dev).bfloat16()
    Wt = (torch.randn(1024, Kt, device=dev) / math.sqrt(Kt)).bfloat16()
    bt = torch.randn(1024, device=dev)
    xt = torch.randn(Mt, 1024, device=dev)
    xt0 = xt.clone()
    run_gemm(gemm_desc(epi=EPI_F32, A=At, lda=Kt, W=Wt, ldw=Kt, M=Mt, N=1024, K=Kt, bias=bt, out=xt, ldo=1024, resid=xt))
    report("M24576 N1024 f32 in place (many waves)", xt, xt0 + At.float() @ Wt.float().t() + bt, 2e-3)
    # PIXSHUF: tokens (2 img, 5x7 grid), Cin 128, cout 64, k 2
    nimg, h, w, cin, cout, k = 2, 5, 7, 128, 64, 2
    At = torch.randn(nimg * h * w, cin, device=dev).bfloat16()
    Wt = (torch.randn(cin, cout, k, k, device=dev) / math.sqrt(cin))  # ConvTranspose2d weight layout
    bt = torch.randn(cout, device=dev)
    Wp = Wt.permute(2, 3, 1, 0).reshape(k * k * cout, cin).contiguous().bfloat16()
    out = torch.zeros(nimg, h * k, w * k, cout, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(epi=EPI_PIXSHUF, A=At, lda=cin, W=Wp, ldw=cin, M=nimg * h * w, N=k * k * cout, K=cin, bias=bt,
                       out=out, ps_k=k, ps_cout=cout, ps_h=h, ps_w=w))
    xin = At.float().view(nimg, h, w, cin).permute(0, 3, 1, 2)
    ref = F.conv_transpose2d(xin, Wp.float().view(k, k, cout, cin).permute(3, 2, 0, 1), bt, stride=k)
    report("epi pixshuf (ConvTranspose k=s)", out, ref.permute(0, 2, 3, 1), 1e-2)
    torch.cuda.synchronize()


def group_conv():
    import torch
    import torch.nn.functional as F
    from vista_slam_b200._lib import EPI_BF16, EPI_HEAD
    torch.manual_seed(2)
    dev = "cuda"
    for (nimg, H, W, Cin, Cout) in [(2, 8, 16, 64, 256), (3, 14, 14, 128, 256), (2, 24, 32, 256, 256),
                                    (1, 20, 36, 256, 128)]:
        x = torch.randn(nimg, H, W, Cin, device=dev).bfloat16()
        wt = (torch.randn(Cout, Cin, 3, 3, device=dev) / math.sqrt(9 * Cin))
        b = torch.randn(Cout, device=dev)
        wp = wt.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous().bfloat16()
        r1 = torch.randn(nimg, H, W, Cout, device=dev).bfloat16()
        out = torch.zeros(nimg, H, W, Cout, device=dev, dtype=torch.bfloat16)
        out2 = torch.zeros_like(out)
        run_gemm(gemm_desc(conv3x3=1, epi=EPI_BF16, A=x, W=wp, ldw=9 * Cin, N=Cout, K=9 * Cin, nimg=nimg, H=H, Wd=W,
                           Cin=Cin, bias=b, out=out, ldo=Cout, out2=out2, resid=r1))
        ref = F.conv2d(x.float().permute(0, 3, 1, 2), wp.float().view(Cout, 3, 3, Cin).permute(0, 3, 1, 2), b,
                       padding=1).permute(0, 2, 3, 1) + r1.float()
        report("conv3x3 %dx%dx%d C%d->%d" % (nimg, H, W, Cin, Cout), out, ref, 1e-2)
        report("   relu copy", out2, ref.relu(), 1e-2)
    # head: conv 128->128 + relu + 1x1 (128->4) + postprocess
    nimg, H, W = 2, 32, 48
    x = torch.randn(nimg, H, W, 128, device=dev).bfloat16()
    wt = torch.randn(128, 128, 3, 3, device=dev) / math.sqrt(9 * 128)
    b = torch.randn(128, device=dev) * 0.1
    wp = wt.permute(0, 2, 3, 1).reshape(128, 9 * 128).contiguous().bfloat16()
    w4 = torch.randn(4, 128, device=dev) / math.sqrt(128)
    b4 = torch.randn(4, device=dev) * 0.1
    w4t = w4.t().contiguous()
    pts = torch.zeros(nimg, H, W, 3, device=dev)
    conf = torch.zeros(nimg, H, W, device=dev)
    run_gemm(gemm_desc(conv3x3=1, epi=EPI_HEAD, A=x, W=wp, ldw=9 * 128, N=128, K=9 * 128, nimg=nimg, H=H, Wd=W, Cin=128,
                       bias=b, head_w=w4t, head_b=b4, pts3d=pts, conf=conf))
    hid = F.conv2d(x.float().permute(0, 3, 1, 2), wp.float().view(128, 3, 3, 128).permute(0, 3, 1, 2), b,
                   padding=1).relu()
    o = torch.einsum("nchw,oc->nhwo", hid, w4) + b4
    xyz = o[..., :3]
    dd = xyz.norm(dim=-1, keepdim=True)
    ref_pts = xyz / dd.clip(min=1e-8) * torch.expm1(dd)
    ref_conf = 1 + o[..., 3].exp()
    report("head conv+1x1+postprocess pts3d", pts, ref_pts, 5e-3)
    report("head conv+1x1+postprocess conf", conf, ref_conf, 5e-3)
    torch.cuda.synchronize()


def group_coalesced_epi():
    """Stores of the coalesced per-warp epilogue that the shapes of gemm_epi and conv do not reach."""
    import torch
    import torch.nn.functional as F
    from vista_slam_b200._lib import EPI_BF16, EPI_F32
    torch.manual_seed(6)
    dev = "cuda"
    # in-place fp32 residual update with N % 128 != 0: the epilogue loads the residual rows before it stores over them
    M, N, K = 777, 320, 256
    A = torch.randn(M, K, device=dev).bfloat16()
    W = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=dev)
    x = torch.randn(M, N, device=dev)
    x0 = x.clone()
    run_gemm(gemm_desc(epi=EPI_F32, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=x, ldo=N, resid=x))
    report("f32 resid in place N320", x, x0 + A.float() @ W.float().t() + bias, 2e-3)
    # conv with no bias, no residual, relu on the main output (the first conv of a DPT residual unit)
    nimg, H, W, Cin, Cout = 2, 14, 18, 256, 256
    x = torch.randn(nimg, H, W, Cin, device=dev).bfloat16()
    wp = (torch.randn(Cout, 9 * Cin, device=dev) / math.sqrt(9 * Cin)).bfloat16()
    out = torch.full((nimg, H, W, Cout), float("nan"), device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(conv3x3=1, epi=EPI_BF16, A=x, W=wp, ldw=9 * Cin, N=Cout, K=9 * Cin, nimg=nimg, H=H, Wd=W, Cin=Cin,
                       out=out, ldo=Cout, relu_main=1))
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wp.float().view(Cout, 3, 3, Cin).permute(0, 3, 1, 2), padding=1)
    report("conv3x3 no bias, relu main", out, ref.permute(0, 2, 3, 1).relu(), 1e-2)
    torch.cuda.synchronize()


def group_attention():
    import torch
    import torch.nn.functional as F
    from vista_slam_b200._lib import check, cur_stream, lib, ptr
    torch.manual_seed(3)
    dev = "cuda"
    L = lib()
    # launch_attention takes 128-row query tiles when that grid has at least one CTA per SM, else 64-row tiles.  On a
    # 132-SM H100, (2, 12, 769), (4, 12, 769) and (3, 16, 768) take 128 rows, the others 64; both kinds include ragged
    # last query and key tiles.
    for (batch, heads, n, shift) in [(2, 3, 128, 0), (2, 3, 196, 0), (2, 12, 769, 0), (4, 12, 769, 2), (3, 16, 768, 0),
                                     (2, 12, 197, 0), (2, 3, 130, 0), (2, 3, 257, 1), (3, 2, 1, 0), (2, 2, 901, 1)]:
        C = heads * 64
        qkv = torch.randn(batch, n, 3 * C, device=dev).bfloat16()
        out = torch.zeros(batch, n, C, device=dev, dtype=torch.bfloat16)
        check(L.sta_op_attention(ptr(qkv), 3 * C, 0, ptr(qkv), 3 * C, C, ptr(qkv), 3 * C, 2 * C, ptr(out), C, batch,
                                 heads, n, n, shift, 0.125, cur_stream()), "attention")
        torch.cuda.synchronize()
        q, k, v = [qkv[..., i * C:(i + 1) * C].float().view(batch, n, heads, 64).transpose(1, 2) for i in range(3)]
        if shift:
            idx = [(b + shift) % batch for b in range(batch)]
            k, v = k[idx], v[idx]
        ref = F.scaled_dot_product_attention(q, k, v, scale=0.125).transpose(1, 2).reshape(batch, n, C)
        report("attention b%d h%d n%d shift%d" % (batch, heads, n, shift), out, ref, 2e-2)
    # the online-softmax rescale: the keys of later tiles score much higher than those of earlier ones, so every new key
    # tile raises the running row maximum and rescales the accumulated O and l (factors far below 2^-8), for some rows
    # only in the ragged last tile.
    # 3 heads: 30 CTAs of 128 rows would leave SMs idle -> 64-row tiles; 16 heads: 160 CTAs -> 128-row tiles.
    batch, n = 2, 600
    for heads in (3, 16):
        C = heads * 64
        qkv = torch.randn(batch, n, 3 * C, device=dev)
        growth = 1.0 + 5.0 * (torch.arange(n, device=dev) // 128).float()           # key tile t scaled by 1 + 5t
        qkv[:, :, C:2 * C] *= growth[None, :, None]
        qkv[0, 590:, C:2 * C] *= 4.0                                                  # a further jump inside the last tile
        qkv = qkv.bfloat16()
        out = torch.zeros(batch, n, C, device=dev, dtype=torch.bfloat16)
        check(L.sta_op_attention(ptr(qkv), 3 * C, 0, ptr(qkv), 3 * C, C, ptr(qkv), 3 * C, 2 * C, ptr(out), C, batch, heads, n,
                                 n, 0, 0.125, cur_stream()), "attention")
        q, k, v = [qkv[..., i * C:(i + 1) * C].float().view(batch, n, heads, 64).transpose(1, 2) for i in range(3)]
        ref = F.scaled_dot_product_attention(q, k, v, scale=0.125).transpose(1, 2).reshape(batch, n, C)
        report("attention growing maxima (rescale path) h%d" % heads, out, ref, 2e-2)


def group_misc():
    import torch
    import torch.nn.functional as F
    from vista_slam_b200._lib import check, cur_stream, lib, ptr
    torch.manual_seed(4)
    dev = "cuda"
    L = lib()
    st = cur_stream()
    for C in (768, 1024):
        rows = 1000
        x = torch.randn(rows, C, device=dev) * 3 + 0.5
        g1, b1, g2, b2 = [torch.randn(C, device=dev) for _ in range(4)]
        o1 = torch.zeros(rows, C, device=dev, dtype=torch.bfloat16)
        o2 = torch.zeros_like(o1)
        check(L.sta_op_layernorm(ptr(x), rows, C, 1e-6, ptr(g1), ptr(b1), ptr(o1), ptr(g2), ptr(b2), ptr(o2), 0, st))
        report("layernorm C%d out1" % C, o1, F.layer_norm(x, (C,), g1, b1, 1e-6), 1e-2)
        report("layernorm C%d out2" % C, o2, F.layer_norm(x, (C,), g2, b2, 1e-6), 1e-2)
    # drop_first_of
    x = torch.randn(4 * 51, 768, device=dev)
    g1, b1 = torch.randn(768, device=dev), torch.randn(768, device=dev)
    o1 = torch.zeros(4 * 50, 768, device=dev, dtype=torch.bfloat16)
    check(L.sta_op_layernorm(ptr(x), 4 * 51, 768, 1e-6, ptr(g1), ptr(b1), ptr(o1), None, None, None, 51, st))
    report("layernorm drop pose row", o1, F.layer_norm(x, (768,), g1, b1, 1e-6).view(4, 51, 768)[:, 1:].reshape(-1, 768),
           1e-2)
    # patch im2col
    img = torch.rand(2, 3, 32, 48, device=dev) * 2 - 1
    o = torch.zeros(2 * 2 * 3, 768, device=dev, dtype=torch.bfloat16)
    check(L.sta_op_patch_im2col(ptr(img), 0, 2, 32, 48, ptr(o), st))
    ref = F.unfold(img, 16, stride=16).transpose(1, 2).reshape(-1, 768)
    report("patch im2col fp32", o, ref, 1e-2)
    imgb = img.bfloat16()
    check(L.sta_op_patch_im2col(ptr(imgb), 1, 2, 32, 48, ptr(o), st))
    report("patch im2col bf16", o, F.unfold(imgb.float(), 16, stride=16).transpose(1, 2).reshape(-1, 768), 1e-6)
    # upsample
    x = torch.randn(2, 7, 9, 64, device=dev).bfloat16()
    o = torch.zeros(2, 14, 18, 64, device=dev, dtype=torch.bfloat16)
    check(L.sta_op_upsample2x(ptr(x), ptr(o), 2, 7, 9, 64, st))
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True)
    report("upsample2x align_corners", o, ref.permute(0, 2, 3, 1), 1e-2)
    for (nimg, H, W, C) in [(1, 12, 16, 256), (3, 5, 3, 128), (2, 24, 32, 128), (1, 1, 40, 64)]:
        x = torch.randn(nimg, H, W, C, device=dev).bfloat16()
        o = torch.zeros(nimg, 2 * H, 2 * W, C, device=dev, dtype=torch.bfloat16)
        check(L.sta_op_upsample2x(ptr(x), ptr(o), nimg, H, W, C, st))
        ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True)
        report("upsample2x %dx%dx%dx%d" % (nimg, H, W, C), o, ref.permute(0, 2, 3, 1), 1e-2)
    # im2col s2
    x = torch.randn(2, 7, 10, 64, device=dev).bfloat16()
    o = torch.zeros(2 * 4 * 5, 9 * 64, device=dev, dtype=torch.bfloat16)
    check(L.sta_op_im2col_3x3_s2(ptr(x), ptr(o), 2, 7, 10, 64, st))
    ref = F.unfold(x.float().permute(0, 3, 1, 2), 3, padding=1, stride=2)  # [n, C*9, L] with (c, tap) order
    ref = ref.view(2, 64, 9, -1).permute(0, 3, 2, 1).reshape(-1, 9 * 64)
    report("im2col 3x3 s2", o, ref, 1e-6)
    # cast with drop
    x = torch.randn(3 * 11, 768, device=dev)
    o = torch.zeros(3 * 10, 768, device=dev, dtype=torch.bfloat16)
    check(L.sta_op_cast_f32_bf16(ptr(x), ptr(o), 33, 768, 11, st))
    report("cast drop", o, x.view(3, 11, 768)[:, 1:].reshape(-1, 768), 1e-2)
    # rope2d op
    tok = torch.randn(2, 50, 4, 64, device=dev).bfloat16()
    pos = torch.randint(-1, 30, (2, 50, 2), device=dev, dtype=torch.int64)
    ref = rope_ref(tok.float().view(100, 4, 64), pos.view(100, 2))
    check(L.sta_op_rope2d(ptr(tok), ptr(pos), 2, 50, 4, st))
    report("rope2d op", tok.view(100, 4, 64), ref, 1e-2)
    torch.cuda.synchronize()


def split_act(x):
    """fp32 [.., C] -> bf16 [.., 3C] = (hi | lo | hi): the activation layout of the split-precision parity mode."""
    import torch
    hi = x.bfloat16()
    lo = (x - hi.float()).bfloat16()
    return torch.cat([hi, lo, hi], dim=-1).contiguous()


def split_w(w):
    """fp32 [N, K] -> bf16 [N, 3K] = (hi | hi | lo): the weight layout of the split-precision parity mode."""
    import torch
    hi = w.bfloat16()
    lo = (w - hi.float()).bfloat16()
    return torch.cat([hi, hi, lo], dim=-1).contiguous()


def merge3(o, N, name):
    """(hi | lo | hi) rows -> fp32 hi + lo; the two hi copies must be identical."""
    import torch
    assert torch.equal(o[..., :N], o[..., 2 * N:3 * N]), name + ": hi copies differ"
    return o[..., :N].float() + o[..., N:2 * N].float()


def group_x3():
    """Split-precision parity mode of the SAME wgmma kernels (operands expanded along K, two-pass / three-store
    epilogues), against fp64 references on the un-rounded fp32 operands.  Bounds 1e-4 max-normalised: two orders of
    magnitude below the bf16 operand noise floor, so an indexing / epilogue error of any size cannot hide."""
    import ctypes
    import torch
    import torch.nn.functional as F
    from vista_slam_b200._lib import EPI_BF16, EPI_F32, EPI_GELU, EPI_PIXSHUF, EPI_ROPE, check, cur_stream, lib, ptr
    torch.manual_seed(7)
    dev = "cuda"
    TOL = 1e-4
    # small problem / many tiles / N % 256 != 0
    for (M, N, K) in [(777, 512, 256), (4096, 768, 768), (300, 384, 192)]:
        A = torch.randn(M, K, device=dev)
        W = torch.randn(N, K, device=dev) / math.sqrt(K)
        bias = torch.randn(N, device=dev)
        base = (A.double() @ W.double().t() + bias.double())
        A3, W3 = split_act(A), split_w(W)
        for epi, nm, fn in ((EPI_BF16, "bf16", lambda t: t), (EPI_GELU, "gelu", lambda t: F.gelu(t))):
            if epi == EPI_GELU and N % 256 != 0:
                continue  # the model has no GELU layer with N % 256 != 0
            out = torch.full((M, 3 * N), float("nan"), device=dev, dtype=torch.bfloat16)
            run_gemm(gemm_desc(epi=epi, A=A3, lda=3 * K, W=W3, ldw=3 * K, M=M, N=N, K=3 * K, bias=bias, out=out, ldo=3 * N,
                               split_precision=1))
            torch.cuda.synchronize()
            report("x3 gemm %s M%d N%d K%d" % (nm, M, N, K), merge3(out, N, nm), fn(base).float(), TOL)
        # fp32 output accumulating in place (residual stream)
        x = torch.randn(M, N, device=dev)
        x0 = x.clone()
        run_gemm(gemm_desc(epi=EPI_F32, A=A3, lda=3 * K, W=W3, ldw=3 * K, M=M, N=N, K=3 * K, bias=bias, out=x, ldo=N, resid=x,
                           split_precision=1))
        torch.cuda.synchronize()
        report("x3 gemm f32 resid in place M%d N%d K%d" % (M, N, K), x, (x0.double() + base).float(), TOL)
    # skip tensors + relu copy (staging epilogue), RoPE
    M, N, K = 500, 256, 256
    A = torch.randn(M, K, device=dev)
    W = torch.randn(N, K, device=dev) / math.sqrt(K)
    bias = torch.randn(N, device=dev)
    r1, r2 = torch.randn(M, N, device=dev), torch.randn(M, N, device=dev)
    out = torch.zeros(M, 3 * N, device=dev, dtype=torch.bfloat16)
    out2 = torch.zeros_like(out)
    run_gemm(gemm_desc(epi=EPI_BF16, A=split_act(A), lda=3 * K, W=split_w(W), ldw=3 * K, M=M, N=N, K=3 * K, bias=bias, out=out,
                       ldo=3 * N, out2=out2, resid=split_act(r1), resid2=split_act(r2), split_precision=1))
    torch.cuda.synchronize()
    # the skip tensors themselves carry 2^-17 relative representation error
    ref = (A.double() @ W.double().t() + bias.double() + r1.double() + r2.double()).float()
    report("x3 gemm bf16 resid x2", merge3(out, N, "resid"), ref, TOL)
    report("x3 gemm bf16 relu copy", merge3(out2, N, "relu"), ref.relu(), TOL)
    heads = 4
    N = heads * 64 * 3
    W = torch.randn(N, K, device=dev) / math.sqrt(K)
    bias = torch.randn(N, device=dev)
    pos = torch.stack([torch.randint(-1, 40, (M,), device=dev), torch.randint(-1, 70, (M,), device=dev)], 1).int().contiguous()
    out = torch.zeros(M, 3 * N, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(epi=EPI_ROPE, A=split_act(A), lda=3 * K, W=split_w(W), ldw=3 * K, M=M, N=N, K=3 * K, bias=bias, out=out,
                       ldo=3 * N, pos=pos, rope_cols=2 * heads * 64, split_precision=1))
    torch.cuda.synchronize()
    base = (A.double() @ W.double().t() + bias.double()).float()
    ref = base.clone()
    ref[:, :2 * heads * 64] = rope_ref(base[:, :2 * heads * 64].reshape(M, 2 * heads, 64), pos).reshape(M, -1)
    report("x3 gemm rope", merge3(out, N, "rope"), ref, TOL)
    # implicit-GEMM conv with a skip tensor
    nimg, H, Wd, Cin, Cout = 2, 14, 18, 128, 256
    x = torch.randn(nimg, H, Wd, Cin, device=dev)
    wt = torch.randn(Cout, Cin, 3, 3, device=dev) / math.sqrt(9 * Cin)
    b = torch.randn(Cout, device=dev)
    wp3 = torch.cat([split_w(wt[:, :, kh, kw]).view(Cout, 1, 3 * Cin) for kh in range(3) for kw in range(3)], 1)
    wp3 = wp3.reshape(Cout, 27 * Cin).contiguous()
    r1 = torch.randn(nimg, H, Wd, Cout, device=dev)
    out = torch.zeros(nimg, H, Wd, 3 * Cout, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(conv3x3=1, epi=EPI_BF16, A=split_act(x), W=wp3, ldw=27 * Cin, N=Cout, K=27 * Cin, nimg=nimg, H=H, Wd=Wd,
                       Cin=3 * Cin, bias=b, out=out, ldo=3 * Cout, resid=split_act(r1), split_precision=1))
    torch.cuda.synchronize()
    ref = (F.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), b.double(), padding=1).permute(0, 2, 3, 1) + r1.double()).float()
    report("x3 conv3x3 + skip", merge3(out, Cout, "conv"), ref, TOL)
    # ConvTranspose (k = stride = 2) as GEMM + pixel shuffle
    hh, ww, C = 6, 10, 192
    T = 2 * hh * ww
    a = torch.randn(T, C, device=dev)
    wT = torch.randn(C, C, 2, 2, device=dev) / math.sqrt(C)  # [Cin][Cout][k][k]
    bT = torch.randn(C, device=dev)
    wg = wT.permute(2, 3, 1, 0).reshape(4 * C, C).contiguous()  # [(kh,kw,co)][ci]
    out = torch.zeros(2, 2 * hh, 2 * ww, 3 * C, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(epi=EPI_PIXSHUF, A=split_act(a), lda=3 * C, W=split_w(wg), ldw=3 * C, M=T, N=4 * C, K=3 * C, bias=bT,
                       out=out, ps_k=2, ps_cout=C, ps_h=hh, ps_w=ww, split_precision=1))
    torch.cuda.synchronize()
    ref = F.conv_transpose2d(a.double().view(2, hh, ww, C).permute(0, 3, 1, 2), wT.double(), bT.double(), stride=2)
    report("x3 convT pixel-shuffle", merge3(out, C, "convT"), ref.permute(0, 2, 3, 1).float(), TOL)


def group_perf():
    import torch
    import torch.nn.functional as F
    from vista_slam_b200._lib import EPI_BF16, EPI_GELU, check, cur_stream, lib, ptr
    dev = "cuda"
    torch.manual_seed(5)

    def timeit(fn, n=10):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    def tile_times(d, flop):
        """Both tile shapes of a linear layer forced through tile_n (the automatic choice is the untagged time)."""
        if d.N % 256 or d.conv3x3:
            return ""
        res = []
        for tn in (128, 256):
            d.tile_n = tn
            ms = timeit(lambda: run_gemm(d))
            res.append("tile_n %d %.3f ms = %.0f TFLOP/s" % (tn, ms, flop / ms / 1e9))
        d.tile_n = 0
        return "   [" + ", ".join(res) + "]"

    # the cuBLAS kernel torch.matmul picks for the encoder's qkv shape (its name carries the tile shape)
    A = torch.randn(24576, 1024, device=dev).bfloat16()
    W = torch.randn(3072, 1024, device=dev).bfloat16()
    torch.matmul(A, W.t())
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        torch.matmul(A, W.t())
        torch.cuda.synchronize()
    names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    print("torch.matmul M24576 N3072 K1024 kernels:", names, flush=True)

    # trunk shapes, plus one grid of 200 tiles (between one and two tiles per SM on a 132-SM H100)
    for (M, N, K, epi) in [(24576, 3072, 1024, EPI_BF16), (24576, 4096, 1024, EPI_GELU), (24576, 1024, 4096, EPI_BF16),
                           (24576, 1024, 1024, EPI_BF16), (3200, 1024, 1024, EPI_BF16)]:
        A = torch.randn(M, K, device=dev).bfloat16()
        W = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
        bias = torch.randn(N, device=dev)
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        d = gemm_desc(epi=epi, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=out, ldo=N)
        ms = timeit(lambda: run_gemm(d))
        ms_t = timeit(lambda: torch.matmul(A, W.t()))
        print("gemm M%d N%d K%d epi%d: %.3f ms = %.0f TFLOP/s   (torch.matmul %.3f ms = %.0f TFLOP/s)%s" %
              (M, N, K, epi, ms, 2.0 * M * N * K / ms / 1e9, ms_t, 2.0 * M * N * K / ms_t / 1e9,
               tile_times(d, 2.0 * M * N * K)), flush=True)
    # epilogue variants on the trunk shapes
    from vista_slam_b200._lib import EPI_F32, EPI_ROPE
    M = 24576
    for (N, K, epi, name) in [(3072, 1024, EPI_ROPE, "rope (enc qkv)"), (1024, 1024, EPI_F32, "f32+resid (enc proj)"),
                              (1024, 4096, EPI_F32, "f32+resid (enc fc2)"), (2304, 768, EPI_ROPE, "rope (dec qkv)"),
                              (768, 768, EPI_F32, "f32+resid (dec proj)"), (3072, 768, EPI_GELU, "gelu (dec fc1)")]:
        A = torch.randn(M, K, device=dev).bfloat16()
        W = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
        bias = torch.randn(N, device=dev)
        if epi == EPI_F32:
            out = torch.zeros(M, N, device=dev)
            d = gemm_desc(epi=epi, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=out, ldo=N, resid=out)
        elif epi == EPI_ROPE:
            out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
            pos = torch.randint(0, 32, (M, 2), device=dev, dtype=torch.int32)
            d = gemm_desc(epi=epi, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=out, ldo=N, pos=pos,
                          rope_cols=2 * N // 3)
        else:
            out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
            d = gemm_desc(epi=epi, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=out, ldo=N)
        ms = timeit(lambda: run_gemm(d))
        print("gemm-epi %-22s M%d N%d K%d: %.3f ms = %.0f TFLOP/s%s" % (name, M, N, K, ms, 2.0 * M * N * K / ms / 1e9,
                                                                       tile_times(d, 2.0 * M * N * K)), flush=True)
    # Per-tile fixed cost: time(K) = a + b K over a K sweep at a trunk shape.  a is what a tile costs besides its
    # k-blocks (epilogue, pipeline fill and drain) where it is not hidden behind another tile's MMAs; a / time(1024) is
    # its share of a K = 1024 layer.
    M, N = 24576, 3072
    ks, ts = [256, 512, 1024, 2048], []
    for K in ks:
        A = torch.randn(M, K, device=dev).bfloat16()
        W = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
        bias = torch.randn(N, device=dev)
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        d = gemm_desc(epi=EPI_BF16, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=out, ldo=N)
        ts.append(timeit(lambda: run_gemm(d), n=20))
    n = len(ks)
    mk, mt = sum(ks) / n, sum(ts) / n
    slope = sum((k - mk) * (t - mt) for k, t in zip(ks, ts)) / sum((k - mk) ** 2 for k in ks)
    icpt = mt - slope * mk
    print("gemm K sweep M%d N%d: %s ms; fixed cost %.3f ms = %.0f %% of K=1024" %
          (M, N, " ".join("K%d %.3f" % (k, t) for k, t in zip(ks, ts)), icpt, 100.0 * icpt / ts[ks.index(1024)]),
          flush=True)
    # cfg-2 DPT 3x3 convolutions (run_dpt in runtime.cu: 16 images per pass, token grid 24 x 32), against cuDNN
    from vista_slam_b200._lib import EPI_HEAD
    for (H, W, Cin, Cout, name) in [(96, 128, 128, 256, "layer1_rn"), (48, 64, 192, 256, "layer2_rn"),
                                    (24, 32, 384, 256, "layer3_rn"), (12, 16, 768, 256, "layer4_rn"),
                                    (96, 128, 256, 256, "refinenet1 rcu"), (48, 64, 256, 256, "refinenet2 rcu"),
                                    (24, 32, 256, 256, "refinenet3 rcu"), (12, 16, 256, 256, "refinenet4 rcu"),
                                    (192, 256, 256, 128, "head.0"), (384, 512, 128, 128, "head.2 (+head epilogue)")]:
        nimg = 16
        x = torch.randn(nimg, H, W, Cin, device=dev).bfloat16()
        wp = (torch.randn(Cout, 9 * Cin, device=dev) / math.sqrt(9 * Cin)).bfloat16()
        b = torch.randn(Cout, device=dev)
        if Cout == 128 and H == 384:
            w4t = (torch.randn(4, 128, device=dev) / math.sqrt(128)).t().contiguous()
            b4 = torch.randn(4, device=dev)
            pts = torch.zeros(nimg, H, W, 3, device=dev)
            conf = torch.zeros(nimg, H, W, device=dev)
            d = gemm_desc(conv3x3=1, epi=EPI_HEAD, A=x, W=wp, ldw=9 * Cin, N=Cout, K=9 * Cin, nimg=nimg, H=H, Wd=W,
                          Cin=Cin, bias=b, head_w=w4t, head_b=b4, pts3d=pts, conf=conf)
        else:
            out = torch.zeros(nimg, H, W, Cout, device=dev, dtype=torch.bfloat16)
            d = gemm_desc(conv3x3=1, epi=EPI_BF16, A=x, W=wp, ldw=9 * Cin, N=Cout, K=9 * Cin, nimg=nimg, H=H, Wd=W,
                          Cin=Cin, bias=b, out=out, ldo=Cout)
        ms = timeit(lambda: run_gemm(d))
        xc = x.permute(0, 3, 1, 2)  # NCHW view of NHWC memory: cuDNN's channels-last path
        wc = wp.view(Cout, 3, 3, Cin).permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
        ms_t = timeit(lambda: F.conv2d(xc, wc, padding=1))
        fl = 2.0 * nimg * H * W * Cout * 9 * Cin
        print("conv3x3 %-24s %dx%dx%d C%d->%d: %.3f ms = %.0f TFLOP/s   (cuDNN conv2d %.3f ms = %.0f TFLOP/s)" %
              (name, nimg, H, W, Cin, Cout, ms, fl / ms / 1e9, ms_t, fl / ms_t / 1e9), flush=True)
    L = lib()
    for (batch, heads, n) in [(32, 16, 768), (32, 12, 769)]:
        C = heads * 64
        qkv = torch.randn(batch, n, 3 * C, device=dev).bfloat16()
        out = torch.zeros(batch, n, C, device=dev, dtype=torch.bfloat16)
        ms = timeit(lambda: check(L.sta_op_attention(ptr(qkv), 3 * C, 0, ptr(qkv), 3 * C, C, ptr(qkv), 3 * C, 2 * C,
                                                     ptr(out), C, batch, heads, n, n, 0, 0.125, cur_stream())))
        fl = 4.0 * batch * heads * n * n * 64
        print("attention b%d h%d n%d: %.3f ms = %.0f TFLOP/s" % (batch, heads, n, ms, fl / ms / 1e9), flush=True)
    # bandwidth kernels at the cfg-2 sizes (16 images per DPT pass, 32 images in the trunk)
    for (nimg, H, W, C) in [(16, 192, 256, 128), (16, 96, 128, 256), (16, 48, 64, 256)]:
        x = torch.randn(nimg, H, W, C, device=dev).bfloat16()
        o = torch.zeros(nimg, 2 * H, 2 * W, C, device=dev, dtype=torch.bfloat16)
        ms = timeit(lambda: check(L.sta_op_upsample2x(ptr(x), ptr(o), nimg, H, W, C, cur_stream())))
        gb = (x.numel() + o.numel()) * 2 / 1e9
        print("upsample2x %dx%dx%dx%d: %.3f ms = %.0f GB/s" % (nimg, H, W, C, ms, gb / ms * 1e3), flush=True)
    for (rows, C) in [(24576, 1024), (24608, 768)]:
        x = torch.randn(rows, C, device=dev)
        g = torch.randn(C, device=dev)
        b = torch.randn(C, device=dev)
        o = torch.zeros(rows, C, device=dev, dtype=torch.bfloat16)
        ms = timeit(lambda: check(L.sta_op_layernorm(ptr(x), rows, C, 1e-6, ptr(g), ptr(b), ptr(o), None, None, None, 0,
                                                     cur_stream())))
        gb = rows * C * 6 / 1e9
        print("layernorm %dx%d: %.3f ms = %.0f GB/s" % (rows, C, ms, gb / ms * 1e3), flush=True)


def main():
    if len(sys.argv) > 1:
        import torch
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
        for g in sys.argv[1:]:
            globals()["group_" + g]()
        return
    for g in GROUPS:
        print("=== group %s ===" % g, flush=True)
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), g], timeout=300)
            print("=== group %s exit %d (%.1fs) ===" % (g, r.returncode, time.time() - t0), flush=True)
        except subprocess.TimeoutExpired:
            print("=== group %s TIMEOUT ===" % g, flush=True)


if __name__ == "__main__":
    main()
