"""CPU: the per-slot checker of tests/test_entry_points_gpu.py rejects the mistakes it is there to catch.

The batched entry points write pair p's view v at slot [v][p] of flat [2][B_total] buffers, chunk by chunk.  A wrong
offset, stride or index there writes a plausible answer for the wrong pair.  Each case here builds the outputs a
correct entry point would write from oracle references, plants one such mistake in a copy and asserts that
`check_slots` refuses the copy while accepting the correct outputs and the same outputs rounded to 17 significant
bits (about what the split-precision mode delivers)."""
import math

import pytest
import torch

from oracle.sta_oracle import StaOracle, make_images
from test_model_gpu import TOL_EMU, TOL_X3

# A slot's reference must differ from every other slot's reference in the same call by at least MARGIN times the bound,
# so that a slot written with another slot's answer fails by a wide margin rather than by luck.
MARGIN = 10.0
# Outputs held to that rule one by one.  The pose confidence is one scalar per slot: among a few dozen random pairs two
# lie within 1e-4 of each other, so no useful bound can separate every pair by it alone.  At the bf16 bounds only the
# pointmaps separate every pair (pose rows of two random pairs can differ by 0.1 max-normalised, 3x TOL_EMU).  Every
# slot is in addition held to the rule on its outputs taken together (check_slots).
STRICT_X3 = ("pts3d_pred", "conf", "relative_pose")
STRICT_BF16 = ("pts3d_pred",)
POSE_KEYS = ("relative_pose", "relative_pose_conf")


def seed_of(H, W, p):
    """The image seed of pair p at H x W: every pair of every size has its own images."""
    return 1_000_000 * (H // 16) + 1000 * (W // 16) + p


def pair_images(H, W, pairs):
    """img1, img2 [len(pairs), 3, H, W]: pair p is make_images(1, H, W, seed_of(H, W, p)), two different views."""
    ims = [make_images(1, H, W, seed_of(H, W, p)) for p in pairs]
    return torch.cat([a for a, _ in ims]), torch.cat([b for _, b in ims])


def oracle_pairs(orc, img1, img2):
    """The oracle's (main, support) dicts of every pair of a batch, one tuple per pair."""
    with torch.no_grad():
        m, s = orc.forward_pair(img1, img2)
    return [({k: v[b] for k, v in m.items()}, {k: v[b] for k, v in s.items()}) for b in range(img1.shape[0])]


def _maxn(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _margins(refs, key, tol, median=False):
    """[S, S] matrix: max|R_t - R_s| / max|R_s| / tol for slot references R (with median=True the median of |R_t - R_s|,
    over every 7th element); inf where t is s's own reference object (the same inputs planted twice)."""
    R = torch.stack([r[key].detach().reshape(-1).float().cpu() for r in refs])
    mx = R.abs().amax(1).clamp_min(1e-30)
    if median:
        R = R[:, ::7]
    out = torch.empty(len(refs), len(refs), dtype=torch.float64)
    for s in range(len(refs)):
        d = (R - R[s]).abs()
        out[s] = ((d.median(1).values if median else d.amax(1)) / mx[s] / tol).double()
        for t in range(len(refs)):
            if refs[t] is refs[s]:
                out[s, t] = math.inf
    return out


def check_slots(what, got, refs, tol, strict, med_tol=None, pose_scale=None):
    """Slot [v][p] of every output in `got` ({key: tensor [2, B, ...]}, as an entry point wrote it) against its own
    reference refs[p][v] ({pair index: (view 0 dict, view 1 dict)}), max-normalised, below tol[key] (and median-normalised
    below med_tol[key] where given).  Before that, the discrimination rule: for every checked slot, every other checked
    slot's reference differs from its own by at least MARGIN x tol in at least one output, and in each `strict` output on
    its own (an output with a median bound counts as told apart when either statistic is).  pose_scale[p] multiplies
    pair p's pose bounds in the comparison, not in the discrimination rule.  Returns the largest error / bound per
    output."""
    slots = [(p, v) for p in refs for v in (0, 1)]
    slot_refs = [refs[p][v] for p, v in slots]
    keys = list(tol)
    marg = {k: _margins(slot_refs, k, tol[k]) for k in keys}
    for k in (med_tol or {}):
        if k in marg:
            marg[k] = torch.maximum(marg[k], _margins(slot_refs, k, med_tol[k], median=True))
    joint = torch.stack([marg[k] for k in keys]).amax(0)
    for s, (p, v) in enumerate(slots):
        assert float(joint[s].min()) >= MARGIN, (what, "pair %d view %d: another slot's reference lies within %.3g bounds"
                                                 % (p, v, float(joint[s].min())))
        for k in strict:
            assert float(marg[k][s].min()) >= MARGIN, (what, k, "pair %d view %d: another slot's reference lies within "
                                                       "%.3g bounds" % (p, v, float(marg[k][s].min())))
    worst = {}
    for k in keys:
        for p, v in slots:
            a, b = got[k][v][p], refs[p][v][k]
            e = _maxn(a, b)
            t = tol[k] * (pose_scale.get(p, 1.0) if pose_scale and k in POSE_KEYS else 1.0)
            assert e < t, (what, "pair %d view %d" % (p, v), k, e, t)
            worst[k] = max(worst.get(k, 0.0), e / t)
            if med_tol and k in med_tol:
                a, b = a.detach().float().cpu(), b.detach().float().cpu()
                m = float((a - b).abs().median() / b.abs().max().clamp_min(1e-30))
                assert m < med_tol[k], (what, "pair %d view %d" % (p, v), k, "median", m)
    return worst


def stack_outputs(refs, B):
    """The [2][B] output buffers a correct entry point writes, from per-pair references."""
    return {k: torch.stack([torch.stack([refs[p][v][k] for p in range(B)]) for v in (0, 1)]) for k in refs[0][0]}


def round_bits(x, bits):
    """x (fp32) rounded to `bits` significant bits, to nearest."""
    i = x.contiguous().view(torch.int32)
    drop = 24 - bits
    r = ((i + (1 << (drop - 1))) >> drop) << drop
    return r.view(torch.float32)


B, H, W = 5, 32, 32
CHUNK = 3  # a chunk size that does not divide B: chunks of 3 and 2 pairs
MODES = {"x3": (TOL_X3, STRICT_X3), "bf16": (TOL_EMU, STRICT_BF16)}


@pytest.fixture(scope="module")
def refs(state_dict):
    img1, img2 = pair_images(H, W, range(B))
    return dict(enumerate(oracle_pairs(StaOracle(state_dict), img1, img2)))


@pytest.mark.parametrize("mode", list(MODES))
def test_correct_and_17_bit_outputs_pass(refs, mode):
    tol, strict = MODES[mode]
    got = stack_outputs(refs, B)
    check_slots("exact", got, refs, tol, strict)
    rounded = {k: round_bits(v, 17) for k, v in got.items()}
    assert any(not torch.equal(rounded[k], got[k]) for k in got)
    check_slots("17 bits", rounded, refs, tol, strict)


@pytest.mark.parametrize("mode", list(MODES))
def test_outputs_shifted_by_one_pair_fail(refs, mode):
    tol, strict = MODES[mode]
    got = stack_outputs(refs, B)
    for k, v in got.items():
        bad = dict(got)
        bad[k] = torch.cat([v[:, 1:], v[:, :1]], dim=1)
        with pytest.raises(AssertionError):
            check_slots("shifted " + k, bad, refs, tol, strict)


@pytest.mark.parametrize("mode", list(MODES))
def test_views_swapped_fail(refs, mode):
    tol, strict = MODES[mode]
    got = stack_outputs(refs, B)
    for p in (0, B - 1):
        bad = {k: v.clone() for k, v in got.items()}
        for k in bad:
            bad[k][0, p], bad[k][1, p] = got[k][1, p], got[k][0, p]
        with pytest.raises(AssertionError):
            check_slots("views swapped at pair %d" % p, bad, refs, tol, strict)


@pytest.mark.parametrize("mode", list(MODES))
def test_view_two_at_the_chunk_stride_fails(refs, mode):
    """The chunked writer with view 2 of chunk pair b0 + i at B_chunk + b0 + i instead of B_total + b0 + i."""
    tol, strict = MODES[mode]
    got = stack_outputs(refs, B)
    for k, v in got.items():
        flat = torch.full((2 * B,) + tuple(v.shape[2:]), float("nan"))
        for b0 in range(0, B, CHUNK):
            nb = min(CHUNK, B - b0)
            flat[b0:b0 + nb] = v[0, b0:b0 + nb]
            flat[nb + b0:nb + b0 + nb] = v[1, b0:b0 + nb]
        bad = dict(got)
        bad[k] = flat.view(v.shape)
        with pytest.raises(AssertionError):
            check_slots("view 2 at the chunk stride, " + k, bad, refs, tol, strict)


@pytest.mark.parametrize("mode", list(MODES))
def test_one_tile_from_another_pair_fails(refs, mode):
    """One 16 x 16 pixel tile of one pair's maps taken from another pair."""
    tol, strict = MODES[mode]
    got = stack_outputs(refs, B)
    for k in ("pts3d_pred", "conf"):
        for v, p, q in ((0, 2, 3), (1, 4, 0)):
            bad = dict(got)
            bad[k] = got[k].clone()
            bad[k][v, p, 16:32, 16:32] = got[k][v, q, 16:32, 16:32]
            with pytest.raises(AssertionError):
                check_slots("tile of pair %d in pair %d, %s" % (q, p, k), bad, refs, tol, strict)


@pytest.mark.parametrize("mode", list(MODES))
def test_finish_outputs_in_sorted_order_fail(refs, mode):
    """sta_regress_pairs_finish writes slot k for edge edge_idx[k]; outputs in sorted index order must fail."""
    tol, strict = MODES[mode]
    idx = [3, 0, 4, 1]
    want = {k: refs[e] for k, e in enumerate(idx)}
    good = stack_outputs(want, len(idx))
    check_slots("given order", good, want, tol, strict)
    srt = {k: refs[e] for k, e in enumerate(sorted(idx))}
    with pytest.raises(AssertionError):
        check_slots("sorted order", stack_outputs(srt, len(idx)), want, tol, strict)


def test_the_discrimination_rule_refuses_indistinguishable_pairs(refs):
    """Two slots whose references agree within the bound: the helper asserts instead of running a check that could not
    tell them apart -- unless they are the same reference object (the same inputs planted twice)."""
    near = {0: refs[0], 1: ({k: v * (1 + 1e-5) for k, v in refs[0][0].items()}, refs[1][1])}
    with pytest.raises(AssertionError, match="another slot"):
        check_slots("near copy", stack_outputs(near, 2), near, TOL_X3, STRICT_X3)
    same = {0: refs[0], 1: refs[0]}
    check_slots("planted twice", stack_outputs(same, 2), same, TOL_X3, STRICT_X3)
