"""CPU: the checkers of tests/test_layers_fp8_gpu.py reject the faults they are there to catch.  Each case builds the
reference the way the GPU test does, makes an "output" on the CPU with one planted fault, and asserts that the helper
the GPU test uses refuses it while accepting the fault-free output."""
import pytest
import torch
import torch.nn.functional as F

from oracle.fp8_oracle import quantize_rows
from test_layers_fp8_gpu import (E4M3, EPI_F32, EPI_GELU_FP8, EPI_ROPE, MAX_EXCEPTION_FRAC, NAN_E4M3, Fp8Launch,
                                 _rne_range, check_canaries, check_codes, dequant_blocks, dequant_rows,
                                 gelu_planted_reference, gemm_reference, make_fp8_operands)
from test_layers_gpu import check_bound, check_exact, rope64

M, N, K = 200, 384, 512


def _out(o, ws=None, a_scale=None, drop_kb=None, drop=128):
    """the float64 product the kernel would compute from operands o, with a fault: drop_kb drops `drop` columns of K
    from drop_kb * drop on"""
    A = dequant_rows(o["aq"], o["as"] if a_scale is None else a_scale)
    W = dequant_blocks(o["wq"], o["ws"] if ws is None else ws)
    if drop_kb is not None:
        A = A.clone()
        A[:, drop_kb * drop:(drop_kb + 1) * drop] = 0
    return A @ W.t() + o["bias"].double()


def _f32(o, **fault):
    return _out(o, **fault) + o["resid"].double()


E = Fp8Launch("f32", "gemm", EPI_F32, M, N, K)


@pytest.fixture(scope="module")
def f32_case():
    o = make_fp8_operands(E, "random", 1, dev="cpu")
    ref, bound = gemm_reference(E, o)
    check_bound("fault-free", _f32(o), ref, bound)
    return o, ref, bound


def test_one_weight_block_scale_doubled(f32_case):
    o, ref, bound = f32_case
    ws = o["ws"].clone()
    ws[1, 2] *= 2
    with pytest.raises(AssertionError):
        check_bound("block scale x2", _f32(o, ws=ws), ref, bound)


def test_one_k_block_dropped(f32_case):
    o, ref, bound = f32_case
    for kb in range(K // 128):
        with pytest.raises(AssertionError):
            check_bound("k-block %d dropped" % kb, _f32(o, drop_kb=kb), ref, bound)


def test_one_k32_slice_dropped(f32_case):
    """one wgmma k32 instruction of a k-block lost: still far outside the worst-case bound with these operands"""
    o, ref, bound = f32_case
    for sl in range(0, K // 32, 3):
        with pytest.raises(AssertionError):
            check_bound("k32 slice %d dropped" % sl, _f32(o, drop_kb=sl, drop=32), ref, bound)


def test_a_scale_of_the_next_row(f32_case):
    o, ref, bound = f32_case
    a_s = o["as"].clone()
    a_s[77] = o["as"][78]
    with pytest.raises(AssertionError):
        check_bound("row 77 scaled as row 78", _f32(o, a_scale=a_s), ref, bound)


def test_one_planted_k_block_dropped():
    o = make_fp8_operands(E, "planted", 2, dev="cpu")
    ref = _f32(o)
    check_exact("fault-free", ref.clone(), ref)
    for kb in range(K // 128):
        with pytest.raises(AssertionError):
            check_exact("k-block %d dropped" % kb, _f32(o, drop_kb=kb), ref)


def test_rope_over_two_thirds_instead_of_half():
    """dec.projk|projv rotates 768 of its 1536 columns; 2N/3 = 1024 is what an old hard-coded rope_cols did"""
    e = Fp8Launch("projk|projv", "gemm", EPI_ROPE, 114, 1536, 768, 768, (2, 7, 8, 1))
    o = make_fp8_operands(e, "random", 3, dev="cpu")
    ref, bound = gemm_reference(e, o)
    base = _out(o)
    check_bound("768 rotated", rope64(base, o["pos"], 768).bfloat16(), ref, bound)
    with pytest.raises(AssertionError):
        check_bound("1024 rotated", rope64(base, o["pos"], 1024).bfloat16(), ref, bound)


def _gelu_case():
    e = Fp8Launch("fc1", "gemm", EPI_GELU_FP8, M, 512, K)
    o = make_fp8_operands(e, "random", 4, dev="cpu")
    ref, bound = gemm_reference(e, o)
    q, s = quantize_rows(ref.float())
    return ref, bound, q.view(torch.uint8), s


def test_gelu_code_moved_one_step():
    ref, bound, q, s = _gelu_case()
    check_codes("fault-free", q, s, ref, bound, max_frac=1.0)
    # an element whose bound admits one code only (away from any midpoint)
    sd = s.double().repeat_interleave(128, 1)
    lo, hi = _rne_range(ref / sd, bound / sd)
    code = q.view(E4M3).float()
    i, j = [int(x) for x in ((lo == hi) & (code > 1) & (code < 400)).nonzero()[0]]
    bad = q.clone()
    bad[i, j] += 1  # the next e4m3 code up (positive, not at the top of the range)
    with pytest.raises(AssertionError):
        check_codes("code + 1", bad, s, ref, bound, max_frac=1.0)


def test_out_scale_in_the_neighbouring_n_tile():
    ref, bound, q, s = _gelu_case()
    ref[:, 256:384] = 4 * ref[:, 128:256]  # n-tile 2's scales are 4x n-tile 1's in every row
    bound[:, 256:384] = 4 * bound[:, 128:256]
    q, s = quantize_rows(ref.float())
    q = q.view(torch.uint8)
    assert bool((s[:, 2] == 4 * s[:, 1]).all())
    check_codes("fault-free", q, s, ref, bound, max_frac=1.0)
    bad = s.clone()
    bad[:, 2] = s[:, 1]  # n-tile 2 written with n-tile 1's scales
    with pytest.raises(AssertionError):
        check_codes("scales of n-tiles 1 and 2 swapped", q, bad, ref, bound, max_frac=1.0)


def _nonlinear_case():
    e = Fp8Launch("fc1", "gemm", EPI_GELU_FP8, M, 512, K)
    o = make_fp8_operands(e, "planted_nonlinear", 5, dev="cpu")
    pre, ref, bound = gelu_planted_reference(o)
    q, s = quantize_rows(ref.float())
    check_codes("fault-free", q.view(torch.uint8), s, ref, bound, MAX_EXCEPTION_FRAC["gelu_nonlinear"])
    return pre, ref, bound


@pytest.mark.parametrize("fault", ["sigmoid approximation", "gelu + 0.01", "tanh approximation"])
def test_planted_nonlinear_gelu_rejects_another_gelu(fault):
    """the planted GELU_FP8 set tells the exact-erf gelu from its common approximations and from a small offset"""
    pre, ref, bound = _nonlinear_case()
    if fault == "sigmoid approximation":
        bad = pre * torch.sigmoid(1.702 * pre)
    elif fault == "gelu + 0.01":
        bad = ref + 0.01
    else:
        bad = F.gelu(pre, approximate="tanh")
    q, s = quantize_rows(bad.float())
    with pytest.raises(AssertionError):
        check_codes(fault, q.view(torch.uint8), s, ref, bound, MAX_EXCEPTION_FRAC["gelu_nonlinear"])


def test_overwritten_canary():
    for buf in (torch.full((M + 3, N), NAN_E4M3, dtype=torch.uint8), torch.full((M + 3, N // 128), float("nan")),
                torch.full((M + 3, N), float("nan"), dtype=torch.bfloat16)):
        before = buf.clone()
        mask = torch.zeros(buf.shape, dtype=torch.bool)
        mask[:M] = True
        buf[:M] = 0
        check_canaries("fault-free", buf, before, mask)
        buf[M + 2, -1] = 0
        with pytest.raises(AssertionError):
            check_canaries("canary overwritten", buf, before, mask)
