"""GPU: the GEMM's tile schedule.  A CTA's tiles alternate between its two consumer warpgroups, so the same tile can be
computed by either warpgroup, first or last in a CTA, with the other warpgroup busy or idle.  A 128-row block computed
alone must come out bit-identical when it is embedded at other tile offsets of a larger problem, at tile counts below
the SM count, between one and two tiles per SM, odd per CTA, and far above (the cfg-2 encoder fc1).  Short K loops
(one k-block, fewer k-blocks than ring stages) and the split-K route are checked against a torch fp32 reference (the
RoPE rotation in float64), max-normalised: max |got - ref| <= 1e-2 max |ref| for bf16 outputs (their 2^-8 rounding),
2e-3 max |ref| for fp32 outputs (accumulation order only)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from test_layers_gpu import gemm_desc, rope64, run_gemm  # noqa: E402
from vista_slam_b200._lib import EPI_BF16, EPI_F32, EPI_GELU, EPI_HEAD, EPI_PIXSHUF, EPI_ROPE  # noqa: E402

DEV = "cuda"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tile_rows(N):
    """M-tile counts (128 rows each) for an N-wide layer: below the SM count, between SMs and 2 x SMs, odd per CTA."""
    nt = N // 128
    s = _sms()
    return [max(3, s // (2 * nt)), (3 * s // 2) // nt + 1, (3 * s + s // 2) // nt | 1]


def _copies(n):
    """Offsets for copies of block 0 among n blocks: first, middle, last, never two neighbours -- so a tile that read
    its neighbour's operands (the other warpgroup's ring stage) would come out different."""
    kept = []
    for o in (0, n // 2, n - 1):
        if all(abs(o - k) >= 2 for k in kept):
            kept.append(o)
    return kept


def _linear(epi, A, W, bias, out, pos=None, resid=None):
    M, K = A.shape
    N = W.shape[0]
    kw = {}
    if epi == EPI_ROPE:
        kw = dict(pos=pos, rope_cols=2 * N // 3)
    run_gemm(gemm_desc(epi=epi, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=out, ldo=N, resid=resid, **kw))


def _embed_linear(epi, N, K, m_tiles, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    M = 128 * m_tiles
    A = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    W = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=DEV, generator=g)
    pos = torch.randint(0, 32, (M, 2), device=DEV, dtype=torch.int32, generator=g)
    blk = slice(0, 128)
    offsets = _copies(m_tiles)
    for o in offsets:  # the block at every offset at once: each copy runs on its own tile slot
        A[128 * o:128 * o + 128] = A[blk]
        pos[128 * o:128 * o + 128] = pos[blk]
    f32 = epi == EPI_F32
    if f32:  # in-place fp32 residual stream: out += A W^T + b (bulk reduce-add)
        x = torch.randn(M, N, device=DEV, generator=g)
        for o in offsets:
            x[128 * o:128 * o + 128] = x[blk]
        alone = x[blk].clone()
        _linear(epi, A[blk].contiguous(), W, bias, alone, resid=alone)
        _linear(epi, A, W, bias, x, resid=x)
        big = x
    else:
        skip = None
        if epi == EPI_BF16:  # a skip tensor: the coalesced epilogue
            skip = torch.randn(M, N, device=DEV, generator=g).bfloat16()
            for o in offsets:
                skip[128 * o:128 * o + 128] = skip[blk]
        alone = torch.full((128, N), float("nan"), device=DEV, dtype=torch.bfloat16)
        big = torch.full((M, N), float("nan"), device=DEV, dtype=torch.bfloat16)
        _linear(epi, A[blk].contiguous(), W, bias, alone, pos=pos[blk].contiguous(),
                resid=None if skip is None else skip[blk].contiguous())
        _linear(epi, A, W, bias, big, pos=pos, resid=skip)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(alone.float()).all())
    for o in offsets:
        assert torch.equal(big[128 * o:128 * o + 128], alone), "tile offset %d of %d" % (o, m_tiles)


@pytest.mark.parametrize("epi,N,K", [(EPI_ROPE, 3072, 1024), (EPI_F32, 1024, 1024), (EPI_GELU, 4096, 1024),
                                     (EPI_BF16, 768, 768)])
def test_block_is_bit_identical_at_any_tile_offset(epi, N, K):
    for i, mt in enumerate(_tile_rows(N)):
        _embed_linear(epi, N, K, mt, seed=10 * epi + i)


def test_block_is_bit_identical_at_cfg2_fc1_scale():
    _embed_linear(EPI_GELU, 4096, 1024, 24576 // 128, seed=99)  # 6144 tiles


def _images(nimg, H, W, C, g):
    return torch.randn(nimg, H, W, C, device=DEV, generator=g).bfloat16()


def _img_counts(tiles_per_img):
    s = _sms()
    return [max(3, s // (2 * tiles_per_img)), (3 * s // 2) // tiles_per_img + 1, (3 * s + s // 2) // tiles_per_img | 1]


@pytest.mark.parametrize("epi", [EPI_BF16, EPI_HEAD])
def test_conv_image_is_bit_identical_at_any_batch_index(epi):
    # one 16 x 8-pixel tile per image and 128-channel tile: the image index is the tile index
    H, W, Cin = 16, 8, 128
    Cout = 128 if epi == EPI_HEAD else 256
    g = torch.Generator(device=DEV).manual_seed(40 + epi)
    wp = (torch.randn(Cout, 9 * Cin, device=DEV, generator=g) / math.sqrt(9 * Cin)).bfloat16()
    b = torch.randn(Cout, device=DEV, generator=g) * 0.1
    w4t = (torch.randn(4, 128, device=DEV, generator=g) / math.sqrt(128)).t().contiguous()
    b4 = torch.randn(4, device=DEV, generator=g) * 0.1

    def run(x, resid):
        n = x.shape[0]
        if epi == EPI_HEAD:
            pts = torch.full((n, H, W, 3), float("nan"), device=DEV)
            conf = torch.full((n, H, W), float("nan"), device=DEV)
            run_gemm(gemm_desc(conv3x3=1, epi=EPI_HEAD, A=x, W=wp, ldw=9 * Cin, N=128, K=9 * Cin, nimg=n, H=H, Wd=W,
                               Cin=Cin, bias=b, head_w=w4t, head_b=b4, pts3d=pts, conf=conf))
            return [pts, conf]
        out = torch.full((n, H, W, Cout), float("nan"), device=DEV, dtype=torch.bfloat16)
        out2 = torch.full_like(out, float("nan"))
        run_gemm(gemm_desc(conv3x3=1, epi=EPI_BF16, A=x, W=wp, ldw=9 * Cin, N=Cout, K=9 * Cin, nimg=n, H=H, Wd=W,
                           Cin=Cin, bias=b, out=out, ldo=Cout, out2=out2, resid=resid))
        return [out, out2]

    for nimg in _img_counts(Cout // 128):
        x = _images(nimg, H, W, Cin, g)
        r = torch.randn(nimg, H, W, Cout, device=DEV, generator=g).bfloat16()
        idx = _copies(nimg)
        for i in idx:
            x[i] = x[0]
            r[i] = r[0]
        alone = run(x[:1].contiguous(), r[:1].contiguous())
        big = run(x, r)
        torch.cuda.synchronize()
        for a, bb in zip(alone, big):
            assert bool(torch.isfinite(a.float()).all())
            for i in idx:
                assert torch.equal(bb[i], a[0]), "image %d of %d" % (i, nimg)


def test_pixel_shuffle_image_is_bit_identical_at_any_batch_index():
    # ConvTranspose2d(k = 2) as a GEMM over 8 x 16-token images (128 tokens = one M tile per image)
    k, cout, ph, pw, Cin = 2, 128, 8, 16, 256
    N = k * k * cout
    g = torch.Generator(device=DEV).manual_seed(77)
    W = (torch.randn(N, Cin, device=DEV, generator=g) / math.sqrt(Cin)).bfloat16()
    b = torch.randn(cout, device=DEV, generator=g)

    def run(A, n):
        out = torch.full((n, ph * k, pw * k, cout), float("nan"), device=DEV, dtype=torch.bfloat16)
        run_gemm(gemm_desc(epi=EPI_PIXSHUF, A=A, lda=Cin, W=W, ldw=Cin, M=A.shape[0], N=N, K=Cin, bias=b, out=out,
                           ldo=cout, ps_k=k, ps_cout=cout, ps_h=ph, ps_w=pw))
        return out

    for nimg in _img_counts(N // 128):
        A = torch.randn(nimg * ph * pw, Cin, device=DEV, generator=g).bfloat16()
        idx = _copies(nimg)
        for i in idx:
            A[i * 128:(i + 1) * 128] = A[:128]
        alone = run(A[:128].contiguous(), 1)
        big = run(A, nimg)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(alone.float()).all())
        for i in idx:
            assert torch.equal(big[i], alone[0]), "image %d of %d" % (i, nimg)


@pytest.mark.parametrize("K", [64, 192])  # one k-block; fewer k-blocks than ring stages
@pytest.mark.parametrize("epi", [EPI_BF16, EPI_GELU, EPI_F32, EPI_ROPE])
def test_short_k_loops(epi, K):
    g = torch.Generator(device=DEV).manual_seed(K + epi)
    M, N = 128 * (_sms() + 5) // 2 + 37, 384  # ragged last tile, both warpgroups busy
    A = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    W = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=DEV, generator=g)
    ref = A.float() @ W.float().t() + bias
    if epi == EPI_F32:
        x = torch.randn(M, N, device=DEV, generator=g)
        ref = ref + x
        _linear(epi, A, W, bias, x, resid=x)
        got, tol = x, 2e-3
    else:
        got = torch.full((M, N), float("nan"), device=DEV, dtype=torch.bfloat16)
        pos = torch.randint(0, 32, (M, 2), device=DEV, dtype=torch.int32, generator=g)
        _linear(epi, A, W, bias, got, pos=pos)
        if epi == EPI_GELU:
            ref = F.gelu(ref)
        if epi == EPI_ROPE:
            rc = 2 * N // 3
            ref = rope64(ref.double(), pos, rc)
        tol = 1e-2
    torch.cuda.synchronize()
    err = (got.float() - ref).abs().max().item()
    assert err <= tol * ref.abs().max().item(), err


def test_split_k_small_problem():
    # fewer tiles than SMs with a split-K workspace: partial tiles per k-range, summed in a fixed order
    g = torch.Generator(device=DEV).manual_seed(123)
    M, N, K = 200, 1024, 1024
    A = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    W = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=DEV, generator=g)
    x = torch.randn(M, N, device=DEV, generator=g)
    ref = x + A.float() @ W.float().t() + bias
    ws = torch.zeros(8 * 256 * N, device=DEV)
    run_gemm(gemm_desc(epi=EPI_F32, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=bias, out=x, ldo=N, resid=x,
                       splitk_ws=ws, splitk_ws_bytes=ws.numel() * 4))
    torch.cuda.synchronize()
    assert ws.abs().sum().item() > 0, "the split-K route was not taken"
    err = (x - ref).abs().max().item()
    assert err <= 2e-3 * ref.abs().max().item(), err


def test_rope_positions_beyond_the_shared_memory_table():
    # positions 63 and up are read from the global sin/cos table; warps whose rows are all below take the staged copy
    g = torch.Generator(device=DEV).manual_seed(321)
    M, N, K = 128 * 40 + 17, 384, 256
    A = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    W = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=DEV, generator=g)
    pos = torch.randint(0, 32, (M, 2), device=DEV, dtype=torch.int32, generator=g)
    far = torch.arange(M, device=DEV) % 256 >= 128  # every other tile: large positions
    pos[far] = torch.randint(60, 200, (int(far.sum()), 2), device=DEV, dtype=torch.int32, generator=g)
    pos[::7] = -1  # the pose-token position
    got = torch.full((M, N), float("nan"), device=DEV, dtype=torch.bfloat16)
    _linear(EPI_ROPE, A, W, bias, got, pos=pos)
    torch.cuda.synchronize()
    ref = A.float() @ W.float().t() + bias
    rc = 2 * N // 3
    ref = rope64(ref.double(), pos, rc)
    err = (got.float() - ref).abs().max().item()
    assert err <= 1e-2 * ref.abs().max().item(), err
