"""CPU: the linear GEMM's automatic tile choice (sta_gemm_auto_tile_n) is a fixed function of the layer's shape and
routes exactly the intended cfg-2 layers to 128 x 256 tiles on a 132-SM H100."""
from vista_slam_b200 import _lib
from vista_slam_b200._lib import EPI_BF16, EPI_F32, EPI_GELU, EPI_HEAD, EPI_PIXSHUF, EPI_ROPE

SMS = 132
ENC_M, DEC_M = 32 * 768, 32 * 769  # cfg-2: 16 pairs, 24 x 32 tokens per image (+ one pose token in the decoder)

# (name, M, N, K, epi, expected tile_n)
CFG2 = [
    ("enc qkv", ENC_M, 3072, 1024, EPI_ROPE, 256),
    ("enc proj", ENC_M, 1024, 1024, EPI_F32, 128),  # N and K both short: the exposed epilogue costs more than it gains
    ("enc fc1", ENC_M, 4096, 1024, EPI_GELU, 256),
    ("enc fc2", ENC_M, 1024, 4096, EPI_F32, 256),
    ("dec qkv", DEC_M, 2304, 768, EPI_ROPE, 256),
    ("dec cross kv", DEC_M, 1536, 768, EPI_ROPE, 128),
    ("dec fc1", DEC_M, 3072, 768, EPI_GELU, 256),
    # 579 wide tiles (4.4 waves, 87.7 % of the slots used) against 1158 (8.8 waves, 97.5 %)
    ("dec proj / cross proj", DEC_M, 768, 768, EPI_F32, 128),
    ("dec fc2", DEC_M, 768, 3072, EPI_F32, 128),
    ("dec cross q", DEC_M, 768, 768, EPI_ROPE, 128),
    ("decoder_embed", ENC_M, 768, 1024, EPI_F32, 128),
    ("dpt act_postprocess.3", ENC_M, 768, 768, EPI_BF16, 128),
    ("dpt act_postprocess.2", ENC_M, 384, 768, EPI_BF16, 128),
    ("dpt refinenet out_conv", 16 * 48 * 64, 256, 256, EPI_BF16, 128),
]


def _rule(M, N, K, epi, sms=SMS):
    return _lib.lib().sta_gemm_auto_tile_n(M, N, K, epi, sms)


def test_cfg2_layers_route_as_intended():
    got = {name: _rule(M, N, K, epi) for name, M, N, K, epi, _ in CFG2}
    want = {name: t for name, _, _, _, _, t in CFG2}
    assert got == want


def test_rule_is_a_function_of_the_shape():
    first = [_rule(M, N, K, epi) for _, M, N, K, epi, _ in CFG2]
    for _ in range(3):
        assert [_rule(M, N, K, epi) for _, M, N, K, epi, _ in reversed(CFG2)] == first[::-1]


def test_small_and_unsupported_shapes_keep_128_wide_tiles():
    for M in (196, 392):  # one keyframe / one pair at 224 x 224
        for N, K, epi in ((3072, 1024, EPI_ROPE), (4096, 1024, EPI_GELU), (1024, 4096, EPI_F32), (2304, 768, EPI_ROPE)):
            assert _rule(M, N, K, epi) == 128, (M, N)
    assert _rule(ENC_M, 2304, 4096, EPI_BF16) == 256
    assert _rule(ENC_M, 384, 4096, EPI_BF16) == 128  # N % 256 != 0
    assert _rule(ENC_M, 4096, 1024, EPI_PIXSHUF) == 128
    assert _rule(ENC_M, 4096, 1024, EPI_HEAD) == 128
    assert _rule(0, 4096, 1024, EPI_BF16) == 128
