"""GPU: size-independent properties of the op-level kernels, called through the C ABI: an identity weight reproduces A
bit for bit, attention over constant values returns that constant, and refused GEMM arguments report why."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from test_layers_gpu import gemm_desc, run_gemm  # noqa: E402


def test_gemm_zero_and_identity_properties():
    """size-independent properties at full cfg-2 size: linearity in the bias and exactness on an identity weight."""
    from vista_slam_b200._lib import EPI_BF16
    dev = "cuda"
    M, K = 24576, 1024
    A = torch.randn(M, K, device=dev).bfloat16()
    W = torch.eye(K, device=dev).bfloat16()
    out = torch.empty(M, K, device=dev, dtype=torch.bfloat16)
    run_gemm(gemm_desc(epi=EPI_BF16, A=A, lda=K, W=W, ldw=K, M=M, N=K, K=K, out=out, ldo=K))
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
    d = gemm_desc(epi=EPI_BF16, A=A, lda=64, W=A, ldw=64, M=128, N=48, K=64, out=A, ldo=48)  # N % 32 != 0
    rc = lib().sta_op_gemm(ctypes.byref(d), None)
    assert rc != 0 and b"multiple of 32" in lib().sta_last_error()
    # GELU and RoPE have only the TMA-store epilogue: N % 128 != 0 is refused, not computed another way
    out = torch.zeros(128, 96, device="cuda", dtype=torch.bfloat16)
    for epi in (EPI_GELU, EPI_ROPE):
        d = gemm_desc(epi=epi, A=A, lda=64, W=out, ldw=64, M=128, N=96, K=64, out=out, ldo=96)
        rc = lib().sta_op_gemm(ctypes.byref(d), None)
        assert rc != 0 and b"GELU / RoPE epilogues need" in lib().sta_last_error(), epi
