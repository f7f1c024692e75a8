"""GPU: every op-level kernel, called through the C ABI, against a plain PyTorch fp32 reference of the same op
on identical bf16-rounded operands.  Tolerances: outputs stored as bf16 -> 2^-8 relative rounding of the
largest value (max-normalised 1e-2 bound); fp32 outputs 2e-3 (accumulation order only)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import tools.bringup as bu  # noqa: E402  (shared check helpers; prints one line per check)


@pytest.fixture(autouse=True)
def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _collect(fn, capsys):
    fn()
    out = capsys.readouterr().out
    lines = [l for l in out.splitlines() if l.strip().endswith(("PASS", "FAIL"))]
    assert lines, out
    bad = [l for l in lines if l.endswith("FAIL")]
    assert not bad, "\n".join(bad)
    return lines


def test_gemm_shapes_and_tails(capsys):
    assert len(_collect(bu.group_gemm_basic, capsys)) == 6


def test_gemm_fused_epilogues(capsys):
    # gelu, residual x2 + relu copy, relu, BN=128 path, fp32 (in-place reduce-add, plain, separate residual), row map, RoPE, ConvT
    assert len(_collect(bu.group_gemm_epi, capsys)) == 20


def test_implicit_gemm_conv_and_head(capsys):
    assert len(_collect(bu.group_conv, capsys)) == 10


def test_coalesced_epilogue_in_place_and_relu_main(capsys):
    """In-place fp32 residual update with N % 128 != 0 (residual loads ahead of the aliasing stores) and a conv with
    no bias, no residual and relu on the main output."""
    assert len(_collect(bu.group_coalesced_epi, capsys)) == 2


def test_attention_self_and_cross(capsys):
    assert len(_collect(bu.group_attention, capsys)) == 12


def test_bandwidth_kernels(capsys):
    assert len(_collect(bu.group_misc, capsys)) == 15


def test_split_precision_mode_of_the_tensor_core_kernels(capsys):
    """x3 parity mode at op level: the same wgmma GEMM / implicit-conv kernels with (hi | lo | hi) x (hi | hi | lo) operands
    against fp64 references, 1e-4 max-normalised (100x below the bf16 floor)."""
    assert len(_collect(bu.group_x3, capsys)) == 13


def test_gemm_zero_and_identity_properties():
    """size-independent properties at full cfg-2 size: linearity in the bias and exactness on an identity weight."""
    from vista_slam_b200._lib import EPI_BF16
    dev = "cuda"
    M, K = 24576, 1024
    A = torch.randn(M, K, device=dev).bfloat16()
    W = torch.eye(K, device=dev).bfloat16()
    out = torch.empty(M, K, device=dev, dtype=torch.bfloat16)
    bu.run_gemm(bu.gemm_desc(epi=EPI_BF16, A=A, lda=K, W=W, ldw=K, M=M, N=K, K=K, out=out, ldo=K))
    torch.cuda.synchronize()
    assert torch.equal(out, A)  # identity weight, no bias: bit exact


def test_attention_uniform_values_property():
    """softmax rows sum to one: with V constant per head the output equals that constant (any n, incl. ragged tiles)."""
    from vista_slam_b200._lib import check, cur_stream, lib, ptr
    dev = "cuda"
    for n in (1, 127, 129, 769):
        C = 2 * 64
        qkv = torch.randn(2, n, 3 * C, device=dev).bfloat16()
        qkv[..., 2 * C:] = 0.5
        out = torch.zeros(2, n, C, device=dev, dtype=torch.bfloat16)
        check(lib().sta_op_attention(ptr(qkv), 3 * C, 0, ptr(qkv), 3 * C, C, ptr(qkv), 3 * C, 2 * C, ptr(out), C, 2, 2, n, n, 0,
                                     0.125, cur_stream()))
        torch.cuda.synchronize()
        assert torch.allclose(out.float(), torch.full_like(out, 0.5).float(), atol=4e-3), n


def test_error_reporting_through_the_abi():
    from vista_slam_b200._lib import EPI_BF16, EPI_GELU, EPI_ROPE, lib
    import ctypes
    A = torch.zeros(128, 64, device="cuda", dtype=torch.bfloat16)
    d = bu.gemm_desc(epi=EPI_BF16, A=A, lda=64, W=A, ldw=64, M=128, N=48, K=64, out=A, ldo=48)  # N % 32 != 0
    rc = lib().sta_op_gemm(ctypes.byref(d), None)
    assert rc != 0 and b"multiple of 32" in lib().sta_last_error()
    # GELU and RoPE have only the TMA-store epilogue: N % 128 != 0 is refused, not computed another way
    out = torch.zeros(128, 96, device="cuda", dtype=torch.bfloat16)
    for epi in (EPI_GELU, EPI_ROPE):
        d = bu.gemm_desc(epi=epi, A=A, lda=64, W=out, ldw=64, M=128, N=96, K=64, out=out, ldo=96)
        rc = lib().sta_op_gemm(ctypes.byref(d), None)
        assert rc != 0 and b"GELU / RoPE epilogues need" in lib().sta_last_error(), epi
