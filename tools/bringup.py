"""Timing of the op-level kernels on the GPU: the trunk's GEMMs and their epilogues against torch.matmul, the cfg-2 DPT
3x3 convolutions against cuDNN, attention, and the bandwidth kernels, at the model's cfg-2 shapes.

    python tools/bringup.py

Prints one line per shape with its time and rate.  Correctness of the same kernels is checked by the test suite
(tests/test_layers_gpu.py, tests/test_attention_gpu.py).
"""
import math
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


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


def main():
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


if __name__ == "__main__":
    main()
