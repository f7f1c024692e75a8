"""GPU: the linear GEMM's two tile shapes give bit-identical results.  The 128 x 256 kernel (both consumer warpgroups
on one tile, one m64n256k16 wgmma per k16 step) and the 128 x 128 ping-pong kernel run the same k16 steps in the same
order for every output element and the same epilogue operations, so forcing tile_n = 256 or 128 (or leaving the choice
to the automatic rule) must not change a bit.  Checked for every trunk layer shape and epilogue the rule can route to
wide tiles, at cfg-2 and SLAM sizes, for M not a multiple of 128, tile counts below the SM count, between one and two
per SM and odd per CTA, and N = 768 (three wide tiles).  Rows past M and padding columns past N hold NaN canaries that
neither kernel may touch."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_layers_gpu import gemm_desc, run_gemm  # noqa: E402
from vista_slam_b200._lib import EPI_BF16, EPI_F32, EPI_GELU, EPI_ROPE  # noqa: E402

DEV = "cuda"
PAD_ROWS, PAD_COLS = 37, 64


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(epi, M, N, K, tile_n, seed, f32_in_place=True, relu=0, bias=True):
    """One layer on fresh seeded operands; returns the whole output buffer (canaries included)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    A = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    W = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
    b = torch.randn(N, device=DEV, generator=g) if bias else None
    pos = torch.randint(-1, 40, (M, 2), device=DEV, dtype=torch.int32, generator=g)
    pos[::7] = torch.randint(-1, 64, (len(range(0, M, 7)), 2), device=DEV, dtype=torch.int32, generator=g)  # past the staged table
    ldo = N + PAD_COLS
    kw = {}
    if epi == EPI_F32:
        out = torch.full((M + PAD_ROWS, ldo), float("nan"), device=DEV)
        if f32_in_place:
            out[:M, :N] = torch.randn(M, N, device=DEV, generator=g)
            kw["resid"] = out
    else:
        out = torch.full((M + PAD_ROWS, ldo), float("nan"), device=DEV, dtype=torch.bfloat16)
    if epi == EPI_ROPE:
        kw.update(pos=pos, rope_cols=2 * N // 3)
    run_gemm(gemm_desc(epi=epi, A=A, lda=K, W=W, ldw=K, M=M, N=N, K=K, bias=b, out=out, ldo=ldo,
                       relu_main=relu, tile_n=tile_n, **kw))
    torch.cuda.synchronize()
    return out


def _same(epi, M, N, K, seed, **kw):
    wide = _run(epi, M, N, K, 256, seed, **kw)
    narrow = _run(epi, M, N, K, 128, seed, **kw)
    auto = _run(epi, M, N, K, 0, seed, **kw)
    body = wide[:M, :N].float()
    assert bool(torch.isfinite(body).all()), "non-finite output in the M x N body"
    assert bool(torch.isnan(wide[M:].float()).all()) and bool(torch.isnan(wide[:, N:].float()).all()), "canary overwritten"
    bits = torch.int32 if epi == EPI_F32 else torch.int16
    assert torch.equal(wide.view(bits), narrow.view(bits)), "tile_n 256 differs from tile_n 128"
    assert torch.equal(auto.view(bits), narrow.view(bits)), "automatic choice differs from tile_n 128"


# (epi, M, N, K): the cfg-2 layer shapes with N % 256 == 0 (encoder M = 32 x 768 tokens, decoder M = 32 x 769) and
# the DPT head's 256-channel 1x1 conv, each forced to both tile shapes; which of them the automatic rule sends to
# 128 x 256 tiles is checked in test_gemm_wide_cpu.py
CFG2 = [
    (EPI_ROPE, 24576, 3072, 1024),   # enc qkv
    (EPI_GELU, 24576, 4096, 1024),   # enc fc1
    (EPI_F32, 24576, 1024, 4096),    # enc fc2 (in place)
    (EPI_F32, 24576, 1024, 1024),    # enc proj (in place)
    (EPI_ROPE, 24608, 2304, 768),    # dec qkv
    (EPI_ROPE, 24608, 1536, 768),    # dec cross-attention kv
    (EPI_GELU, 24608, 3072, 768),    # dec fc1
    (EPI_BF16, 16 * 48 * 64, 256, 256),  # refinenet out_conv
]


@pytest.mark.parametrize("epi,M,N,K", CFG2)
def test_cfg2_layer_is_bit_identical_across_tile_shapes(epi, M, N, K):
    _same(epi, M, N, K, seed=M + N + K + epi)


# SLAM sizes: one keyframe pair (2 x 196 tokens) and a batch of 16 pairs, forced either way
@pytest.mark.parametrize("epi,N,K", [(EPI_ROPE, 3072, 1024), (EPI_GELU, 4096, 1024), (EPI_F32, 1024, 4096),
                                     (EPI_ROPE, 2304, 768), (EPI_GELU, 3072, 768)])
@pytest.mark.parametrize("M", [392, 16 * 392 + 16])
def test_slam_layer_is_bit_identical_across_tile_shapes(epi, N, K, M):
    _same(epi, M, N, K, seed=7 * M + N)


@pytest.mark.parametrize("epi", [EPI_BF16, EPI_ROPE, EPI_F32, EPI_GELU])
def test_tile_counts_and_ragged_m(epi):
    # wide tiles of N = 1024: 4 per 128-row block
    s = _sms()
    below = max(3, s // 8)               # m-tiles: fewer wide tiles than SMs
    between = (3 * s // 2) // 4 + 1      # between one and two per SM
    odd = (3 * s) // 4 | 1               # about three per CTA, an odd tile count
    for i, mt in enumerate((below, between, odd)):
        _same(epi, 128 * mt - 40, 1024, 512, seed=100 * epi + i)  # M not a multiple of 128
    _same(epi, 24608, 1024, 256, seed=3 + epi)


def test_n768_three_wide_tiles():
    for epi in (EPI_BF16, EPI_ROPE, EPI_F32, EPI_GELU):
        _same(epi, 24608, 768, 768, seed=50 + epi)


def test_bf16_relu_plain_f32_and_no_bias():
    _same(EPI_BF16, 3000, 1024, 384, seed=61, relu=1)
    _same(EPI_F32, 3000, 1024, 384, seed=62, f32_in_place=False)
    _same(EPI_BF16, 3000, 512, 384, seed=63, bias=False)


def test_wide_tiles_are_refused_where_they_do_not_apply():
    with pytest.raises(RuntimeError, match="tile_n"):
        _run(EPI_BF16, 256, 384, 128, 256, seed=1)  # N % 256 != 0
    with pytest.raises(RuntimeError, match="tile_n"):
        _run(EPI_BF16, 256, 512, 128, 192, seed=1)  # not a tile shape
