"""CPU: the tap names of runtime.cu are exactly those tests/test_forward_taps_gpu.py checks, and its packing helpers
reject the mis-indexed layouts they are there to catch."""
import os
import re

import pytest
import torch

from test_forward_taps_gpu import (TAP_PATTERNS, check_slot, is_secondary, pack_conv3, pack_convT, pack_linear,
                                   want_slot)

RUNTIME = os.path.join(os.path.dirname(__file__), "..", "vista_slam_b200", "csrc", "runtime.cu")


def _indexless(name):
    """DPT level, layer_rn and hook indices as %d (the runtime formats some of them, names others)"""
    return re.sub(r"(rn|ref|hook)\d", r"\1%d", name)


def runtime_tap_names():
    """the names the runtime's tap calls format: tap(...) as given, tap_fp8(...) as .q and .s (tap_fp8's own tap
    calls, which append the suffix, are not names)"""
    src = open(RUNTIME).read()
    names = set()
    for fn, name in re.findall(r'\b(tap|tap_fp8)\(c{1,2}, [^;]*?"([^"]+)"', src):
        if not name.startswith("."):
            names |= {name + ".q", name + ".s"} if fn == "tap_fp8" else {name}
    return {_indexless(n) for n in names}


def test_runtime_tap_names_are_the_checked_list():
    got = runtime_tap_names()
    want = {_indexless(n) for n in TAP_PATTERNS}
    assert got == want, {"in runtime.cu only": sorted(got - want), "in the test only": sorted(want - got)}


def test_secondary_names_are_the_second_outputs():
    assert {n for n in TAP_PATTERNS if is_secondary(n)} == {
        "enc.%d.ln1.s", "enc.%d.att8.s", "enc.%d.ln2.s", "enc.%d.hid.s", "dec.%d.lny", "dec.%d.lny.q", "dec.%d.lny.s",
        "dec.%d.ln1.s", "dec.%d.att8.s", "dec.%d.ln2.s", "dec.%d.catt8.s", "dec.%d.ln3.s", "dec.%d.hid.s", "pose_conf",
        "dpt.conf", "dpt.rn0.relu", "dpt.rn1.relu", "dpt.rn2.relu", "dpt.rn3.relu", "dpt.ref2.s_relu",
        "dpt.ref1.s_relu", "dpt.ref0.s_relu"}


def _w(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g)


@pytest.mark.parametrize("split", [False, True])
def test_conv3_with_channel_major_taps_is_rejected(split):
    w = _w(8, 6, 3, 3)
    want = pack_conv3(w, split, 8)
    check_slot("reference", want.clone(), want)
    bad = pack_conv3(w.transpose(2, 3), split, 8)  # (kw, kh) order
    with pytest.raises(AssertionError):
        check_slot("kh <-> kw", bad, want)
    bad = want.clone()
    bad.view(8, 9, -1)[:, :, 7] = 1  # a nonzero padding channel
    with pytest.raises(AssertionError):
        check_slot("padding", bad, want)


@pytest.mark.parametrize("split", [False, True])
def test_convT_with_cin_and_cout_swapped_is_rejected(split):
    w = _w(6, 6, 2, 2, seed=1)
    want = pack_convT(w, split, 2, 8)
    with pytest.raises(AssertionError):
        check_slot("Cin <-> Cout", pack_convT(w.transpose(0, 1), split, 2, 8), want)
    with pytest.raises(AssertionError):
        check_slot("kh <-> kw", pack_convT(w.transpose(2, 3), split, 2, 8), want)


def test_x3_linear_with_lo_and_hi_swapped_is_rejected():
    w = _w(16, 32, seed=2)
    want = pack_linear(w, True)
    bad = torch.cat([want[:, 64:], want[:, :64]], 1)  # (lo | hi | hi)
    with pytest.raises(AssertionError):
        check_slot("lo first", bad, want)


def test_truncation_instead_of_round_to_nearest_even_is_rejected():
    tie = torch.tensor([[1 + 3 * 2.0 ** -8, 1 + 2.0 ** -8, -(1 + 3 * 2.0 ** -8), 1.0]])
    want = pack_linear(tie, False)
    trunc = (tie.view(torch.int32) & ~0xFFFF).view(torch.float32)  # bf16 by dropping the low 16 bits
    with pytest.raises(AssertionError):
        check_slot("truncated", trunc.bfloat16().view(torch.int16), want)
    assert want.view(torch.bfloat16).float().tolist() == [[1 + 2.0 ** -6, 1.0, -(1 + 2.0 ** -6), 1.0]]


def test_transposed_f32_head_weight_is_checked_transposed():
    w = _w(4, 128, 1, 1, seed=3)
    want = want_slot(w, ("transpose",), False)
    with pytest.raises(AssertionError):
        check_slot("not transposed", w.reshape(-1).view(torch.int32), want)
