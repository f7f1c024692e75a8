"""GPU: both attention kernels -- the wgmma flash-attention kernel (sta_op_attention) and the fp32 kernel of the
split-precision parity mode (sta_op_attention_split) -- against plain float64 attention computed from exactly the
operands each kernel sees, with a bound per output element, plus planted answers that must come out bit for bit,
schedule invariances of the kernel against itself, and the refusals of launch_attention.

Every call runs on NaN-filled buffers: the other heads' columns, the padding columns of every operand and output, and
three trailing output rows are never addressed, so a NaN in the output means a stray read and a changed canary bit a
stray write."""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from vista_slam_b200._lib import cur_stream, lib  # noqa: E402

DEV = "cuda"
SCALE = 0.125
LOG2E = 1.4426950408889634
KERNELS = ("bf16", "x3")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, g, s=1.0):
    return torch.randn(shape, device=DEV, generator=g) * s


def _away_from_zero(shape, g):
    """Values with 0.25 <= |v| <= 2: a planted output that picks up other keys' values at 2^-40 stays visibly exact."""
    mag = torch.rand(shape, device=DEV, generator=g) * 1.75 + 0.25
    return mag * (torch.randint(0, 2, shape, device=DEV, generator=g) * 2 - 1)


def _self(C):  # the model's self-attention: q | k | v of one [batch][n][3C] projection
    return dict(q=("qkv", 3 * C, 0), k=("qkv", 3 * C, C), v=("qkv", 3 * C, 2 * C), ldo=C)


def _cross(C):  # the decoder's cross-attention: q [batch][n][C], k | v of one [batch][n][2C] projection
    return dict(q=("q", C, 0), k=("kv", 2 * C, 0), v=("kv", 2 * C, C), ldo=C)


def _wide(C):  # the heads sit two heads in from the start of a wider projection; output rows have padding columns
    W = C + 256
    return dict(q=("qkv", 3 * W, 128), k=("qkv", 3 * W, W + 128), v=("qkv", 3 * W, 2 * W + 128), ldo=C + 40)


def _apart(C):  # K and V in separate buffers with different strides and offsets
    return dict(q=("q", C + 64, 64), k=("k", C + 16, 8), v=("v", C + 200, 136), ldo=C + 8)


def _operand(x, split):
    """fp32 values -> (hi, lo) bf16 as stored for the kernel (lo None for the bf16 kernel) and the fp32 values the kernel
    computes with: hi, or hi + lo added in fp32 as the split kernel forms them."""
    hi = x.bfloat16()
    if not split:
        return hi, None, hi.float()
    lo = (x - hi.float()).bfloat16()
    return hi, lo, hi.float() + lo.float()


def _attend(kernel, Q, K, V, shift=0, layout=_cross, scale=SCALE):
    """Run one kernel on Q [B][nq][H][64], K, V [B][nk][H][64] (fp32; rounded to the kernel's operands here), laid out by
    layout(64 H) = {q|k|v: (buffer, logical row width, column of head 0), ldo: logical output width}; operands naming
    the same buffer share it.  Buffers are NaN except the addressed columns; the output's unaddressed elements (padding
    columns, three trailing rows) must keep their bits.  Returns the output as float64 (hi + lo in split mode) and the
    operands as the kernel sees them (fp32)."""
    split = kernel == "x3"
    m = 3 if split else 1
    B, nq, H, _ = Q.shape
    nk = K.shape[1]
    C = 64 * H
    lay = layout(C)
    bufs, seen = {}, []
    for key, x, n in (("q", Q, nq), ("k", K, nk), ("v", V, nk)):
        name, width, col0 = lay[key]
        if name not in bufs:
            bufs[name] = torch.full((B, n, m * width), float("nan"), device=DEV, dtype=torch.bfloat16)
        buf = bufs[name]
        assert buf.shape[1] == n
        hi, lo, s = _operand(x.reshape(B, n, C), split)
        buf[..., col0:col0 + C] = hi
        if split:
            buf[..., width + col0:width + col0 + C] = lo
            buf[..., 2 * width + col0:2 * width + col0 + C] = hi
        seen.append(s.view(B, n, H, 64))
    ldo = lay["ldo"]
    out = torch.full((B * nq + 3, m * ldo), float("nan"), device=DEV, dtype=torch.bfloat16)
    before = out.clone()
    fn = lib().sta_op_attention_split if split else lib().sta_op_attention
    a = [(ctypes.c_void_p(bufs[lay[key][0]].data_ptr()), m * lay[key][1], lay[key][2]) for key in "qkv"]
    rc = fn(*a[0], *a[1], *a[2], ctypes.c_void_p(out.data_ptr()), m * ldo, B, H, nq, nk, shift, scale, cur_stream())
    assert rc == 0, lib().sta_last_error()
    torch.cuda.synchronize()
    addressed = torch.zeros(out.shape, dtype=torch.bool, device=DEV)
    for part in range(m):
        addressed[:B * nq, part * ldo:part * ldo + C] = True
    assert torch.equal(out.view(torch.int16)[~addressed], before.view(torch.int16)[~addressed]), \
        "wrote outside the addressed output"
    o = out[:B * nq].view(B, nq, m * ldo)
    if split:
        assert torch.equal(o[..., :C], o[..., 2 * ldo:2 * ldo + C]), "hi copies differ"
        res = o[..., :C].double() + o[..., ldo:ldo + C].double()
    else:
        res = o[..., :C].double()
    assert bool(torch.isfinite(res).all()), "NaN / Inf in the output: a read outside the addressed operands"
    return res.view(B, nq, H, 64), seen


def _scores(Q, K, b, shift, scale=SCALE):
    """float64 scale * q k^T of sample b against its K / V sample: [H][nq][nk]."""
    kb = (b + shift) % Q.shape[0]
    return torch.einsum("qhd,khd->hqk", Q[b].double(), K[kb].double()) * scale


def _reference(Q, K, V, shift, scale=SCALE):
    """float64 ref = P V and A = P |V| with P = softmax(scale Q K^T), one sample at a time; and the largest |score| in
    log2 units."""
    B = Q.shape[0]
    ref = torch.empty(Q.shape, dtype=torch.float64, device=DEV)
    A = torch.empty_like(ref)
    smax = 0.0
    for b in range(B):
        s = _scores(Q, K, b, shift, scale)
        smax = max(smax, s.abs().max().item() * LOG2E)
        p = torch.softmax(s, dim=-1)
        vb = V[(b + shift) % B].double()
        ref[b] = torch.einsum("hqk,khd->qhd", p, vb)
        A[b] = torch.einsum("hqk,khd->qhd", p, vb.abs())
    return ref, A, smax


def _check_bound(name, kernel, out, seen, shift):
    Q, K, V = seen
    ref, A, smax = _reference(Q, K, V, shift)
    assert smax <= 128.0, "%s: scores reach %.1f log2 units; the bounds assume |s| <= 128" % (name, smax)
    nk = K.shape[1]
    flush = nk * 2.0 ** -126 * V.abs().max().item()
    if kernel == "x3":
        bound = 2.0 ** -16 * ref.abs() + (nk + 64) * 2.0 ** -22 * A + flush
    else:
        bound = 2.0 ** -8 * ref.abs() + (2.0 ** -8 + 2.0 ** -12) * A + flush
    ratio = ((out - ref).abs() / bound).max().item()
    print("attention bound %-28s %-4s worst err / bound = %.3f" % (name, kernel, ratio), flush=True)
    assert ratio <= 1.0, "%s %s: err / bound = %.3f" % (name, kernel, ratio)
    return ratio


def _random_qkv(B, H, nq, nk, seed):
    g = _gen(seed)
    return _randn((B, nq, H, 64), g), _randn((B, nk, H, 64), g), _randn((B, nk, H, 64), g)


def _growth(B, H, n, seed):
    """Key tile t scaled by 1 + 2t and sample 0's keys 590.. by a further 1.5 (only in the ragged last tile): row maxima
    grow from tile to tile, for some rows only in the tail.  Scores stay within 128 log2 units."""
    Q, K, V = _random_qkv(B, H, n, n, seed)
    K *= (1.0 + 2.0 * (torch.arange(n, device=DEV) // 128).float())[None, :, None, None]
    K[0, 590:] *= 1.5
    return Q, K, V


# (id, batch, heads, nq, nk, kv_batch_shift, layout, generator)
_CASES = [
    # the model's calls at cfg-2 (16 pairs = 32 samples): encoder self, decoder self, decoder cross (partner shift 16)
    ("cfg2_enc_self", 32, 16, 768, 768, 0, _self, None),
    ("cfg2_dec_self", 32, 12, 769, 769, 0, _self, None),
    ("cfg2_dec_cross", 32, 12, 769, 769, 16, _cross, None),
    # and at 224 x 224 in SLAM mode (one pair): the 64-row route
    ("slam224_enc_self", 2, 16, 196, 196, 0, _self, None),
    ("slam224_dec_self", 2, 12, 197, 197, 0, _self, None),
    ("slam224_dec_cross", 2, 12, 197, 197, 1, _cross, None),
]
_CASES += [("ragged_n%d" % n, 2, 3, n, n, 1, _self, None)
           for n in (1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 257, 385, 1025)]
_CASES += [("nq%d_nk%d" % (nq, nk), 2, 3, nq, nk, 1, _cross, None) for nq, nk in ((1, 769), (769, 1), (300, 129))]
_CASES += [
    ("wide_heads2to5_ldo_pad", 2, 4, 200, 200, 1, _wide, None),
    ("k_v_apart", 3, 2, 300, 129, 2, _apart, None),
]
# both query-tile sizes with ragged last query and key tiles, cross-sample K / V (shift), a single row; and the
# online-softmax rescale under growing row maxima, at 64-row (3 heads) and 128-row tiles (16 heads)
_CASES += [("bringup_b%d_h%d_n%d_s%d" % (b, h, n, s), b, h, n, n, s, _self, None)
           for b, h, n, s in ((2, 3, 128, 0), (2, 3, 196, 0), (2, 12, 769, 0), (4, 12, 769, 2), (3, 16, 768, 0),
                              (2, 12, 197, 0), (2, 3, 130, 0), (2, 3, 257, 1), (3, 2, 1, 0), (2, 2, 901, 1))]
_CASES += [("bringup_growing_maxima_h%d" % h, 2, h, 600, 600, 0, _self, _growth) for h in (3, 16)]


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("case", _CASES, ids=[c[0] for c in _CASES])
def test_attention_within_per_element_bound_of_float64(case, kernel):
    """|out - ref| per element, ref = P V and A = P |V| in float64 from the operands the kernel sees, P = softmax(scale
    Q K^T), log2-domain scores within +-128.

    bf16 kernel: |out - ref| <= 2^-8 |ref| + (2^-8 + 2^-12) A.
      * bf16 has 8 significant bits, so rounding to nearest costs up to 2^-8 of the value (half an ulp just above a
        power of two, 2^-9 just below the next).  The output rounding costs up to 2^-8 |ref|.
      * Each weight 2^(s - m) is rounded to bf16 before P V while l sums the unrounded weights: the error is
        sum_j d_j w_j V_j with |d_j| <= 2^-8, at most 2^-8 A.  Over many keys the d_j cancel, but when a few keys
        hold the softmax (growing maxima) they do not: an allowance of 2^-9 for either rounding is exceeded there
        (err / (2^-9 |ref| + 2^-8 A) = 1.17 with 16 heads on an H100 SXM at 400 W, reproduced by an fp32 emulation of
        the kernel's roundings).
      * 2^-12 A covers ex2.approx (about 2^-22 relative), the fp32 scores (|s| <= 128 puts the exponent within
        2^-16), the rescale factors and the fp32 sums of l and P V.
    x3 kernel: |out - ref| <= 2^-16 |ref| + (nk + 64) 2^-22 A.
      * hi + lo of the output is within 2^-8 of 2^-8 of |out|.
      * The scores (64-term fp32 dot products of hi + lo operands, q pre-scaled), the exponent argument s - m and
        exp2f each cost a few 2^-24 of the weight, charged as 64 x 2^-22; the fp32 sequential sums of l and P V over nk
        keys cost at most nk 2^-24 each.
    Both bounds add nk 2^-126 max|V|: a weight or rescale factor below 2^-126 of the running maximum is flushed to 0 by
    ex2.approx.ftz, which only matters for entries that are themselves below 2^-100."""
    name, B, H, nq, nk, shift, layout, make = case
    seed = sum(map(ord, name))
    Q, K, V = make(B, H, nq, seed) if make else _random_qkv(B, H, nq, nk, seed)
    out, seen = _attend(kernel, Q, K, V, shift, layout)
    _check_bound(name, kernel, out, seen, shift)


# ---------------------------------------------------------------------------------------------------------------------
# planted answers
# ---------------------------------------------------------------------------------------------------------------------

def _target_weights(seen, shift, targets):
    """float64 softmax weight of key targets[b, i, h] in row (b, i, h), and its lead over the runner-up in log2 units."""
    Q, K, _ = seen
    w, lead = [], []
    for b in range(Q.shape[0]):
        s = _scores(Q, K, b, shift)                             # [H][nq][nk]
        t = targets[b].transpose(0, 1).unsqueeze(-1)            # [H][nq][1]
        w.append(torch.softmax(s, dim=-1).gather(-1, t))
        s = s * LOG2E
        st = s.gather(-1, t)
        lead.append(st - s.scatter(-1, t, -math.inf).max(dim=-1, keepdim=True).values)
    return torch.cat(w).min().item(), torch.cat(lead).min().item()


def _expect_planted(kernel, out, seen, shift, targets):
    _, _, V = seen
    B = V.shape[0]
    want = torch.stack([V[(b + shift) % B].gather(0, targets[b].unsqueeze(-1).expand(-1, -1, 64)) for b in range(B)])
    w, lead = _target_weights(seen, shift, targets)
    assert w >= 1.0 - 2.0 ** -24, "construction: the target's float64 weight is %.10f" % w
    bad = (out != want.double()).any(dim=-1)
    assert not bool(bad.any()), "%s: %d of %d rows differ from V[target]; first (sample, row, head): %s" % (
        kernel, int(bad.sum()), bad.numel(), tuple(bad.nonzero()[0].tolist()))
    return lead


# (batch, heads, shift): 64-row tiles (42 CTAs of 128 rows would leave SMs idle) and 128-row tiles (168 CTAs)
_PLANT_SHAPES = [(2, 3, 1), (4, 6, 2)]


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("B,H,shift", _PLANT_SHAPES)
def test_dominant_key_gives_its_value_bit_for_bit(kernel, B, H, shift):
    """Keys are random +-1 vectors and q_i = 8 k_t(i) for a target key t(i) of the partner sample: the target leads
    every other key by far more than 40 log2 units, so the output row is V[t(i)] exactly (its weight is 1 to 2^-24, the
    rest vanish in the bf16 / hi + lo rounding).  Targets: keys 0, 127, 128, one key in every stage of the 3-stage
    ring over two wraps (tiles 0-5), and 768, the only key of the ragged last tile (nk = 769); a different target per
    head, row and sample."""
    n = 769
    special = torch.tensor([0, 127, 128, 255, 261, 461, 612, 767, 768], device=DEV)
    g = _gen(11 + B)
    K = (torch.randint(0, 2, (B, n, H, 64), device=DEV, generator=g) * 2 - 1).float()
    V = _away_from_zero((B, n, H, 64), g)
    i = torch.arange(n, device=DEV)[None, :, None]
    h = torch.arange(H, device=DEV)[None, None, :]
    b = torch.arange(B, device=DEV)[:, None, None]
    targets = special[(i + 2 * h + 5 * b) % len(special)]       # [B][nq][H]
    Q = torch.empty(B, n, H, 64, device=DEV)
    for s in range(B):
        Q[s] = 8.0 * K[(s + shift) % B].gather(0, targets[s].unsqueeze(-1).expand(-1, -1, 64))
    out, seen = _attend(kernel, Q, K, V, shift, _self)
    lead = _expect_planted(kernel, out, seen, shift, targets)
    assert lead >= 40.0, "construction: lead %.1f log2 units" % lead


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("nk", [1, 65, 129, 700])
def test_masked_key_slots_never_enter_the_softmax(kernel, nk):
    """Masking canary: the target key's score is exactly 0 (q is 16 e_0 and the target's k_0 is 0) and every other
    real key scores -46 log2 units.  A zero-filled slot past nk that escaped the mask would score exactly 0 as well,
    take half the weight and halve the output; a correct kernel returns V[target] bit for bit.  Ragged last tiles hold
    1, 65, 1 and 60 real keys."""
    B, H, nq, shift = 2, 3, 200, 1
    g = _gen(nk)
    K = _randn((B, nk, H, 64), g)
    K[..., 0] = -16.0
    V = _away_from_zero((B, nk, H, 64), g)
    Q = torch.zeros(B, nq, H, 64, device=DEV)
    Q[..., 0] = 16.0
    choice = torch.tensor([0, nk - 1, nk // 2], device=DEV)
    tb = choice[(torch.arange(B, device=DEV)[:, None] * H + torch.arange(H, device=DEV)[None, :]) % 3]  # [B][H]
    for b in range(B):
        K[(b + shift) % B, tb[b], torch.arange(H, device=DEV), 0] = 0.0
    targets = tb[:, None, :].expand(B, nq, H).contiguous()
    out, seen = _attend(kernel, Q, K, V, shift, _cross)
    _expect_planted(kernel, out, seen, shift, targets)


# per key tile offsets of the scores in log2 units (the last entry is the ragged tail)
_READOUTS = [
    ("max_in_first_tile", 705, [8, 0, 0, 0, 0, 0]),
    ("max_in_last_tile", 705, [0, 2, 4, 6, 8, 10]),
    ("max_only_in_ragged_tail", 641, [0, 0, 0, 0, 0, 12]),
    ("jump_over_126", 705, [-68, 62, 62, 62, 62, 62]),
    ("all_scores_equal", 705, None),
]


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("name,nk,offsets", _READOUTS, ids=[r[0] for r in _READOUTS])
def test_rescale_readout_of_softmax_mass_per_key_tile(kernel, name, nk, offsets):
    """V one-hot by key tile, V[j, d] = [d == j // 128]: column d of the output is the softmax mass of key tile d, so
    every online-softmax rescale shows up in its own column.  Scores are offset per tile (q_0 = 8, k_0 = offset / log2 e
    plus noise in the other dimensions), with the row maximum in the first tile, the last tile, only in the ragged tail,
    after a jump of 130 log2 units (the rescale factor of the first tile's mass flushes to 0), or all scores equal.
    Checked against the per-element bounds of test_attention_within_per_element_bound_of_float64."""
    B, H, nq, shift = 2, 3, 130, 1
    g = _gen(nk + len(name))
    K = _randn((B, nk, H, 64), g, 0.5)
    Q = _randn((B, nq, H, 64), g, 0.5)
    if offsets is None:
        K[:] = K[:, :1]
    else:
        off = torch.tensor(offsets, device=DEV, dtype=torch.float32)[torch.arange(nk, device=DEV) // 128]
        Q[..., 0] = 8.0
        K[..., 0] = (off / LOG2E)[None, :, None]
    V = torch.zeros(B, nk, H, 64, device=DEV)
    V[:, torch.arange(nk, device=DEV), :, torch.arange(nk, device=DEV) // 128] = 1.0
    out, seen = _attend(kernel, Q, K, V, shift, _cross)
    _check_bound("readout_" + name, kernel, out, seen, shift)


# ---------------------------------------------------------------------------------------------------------------------
# schedule invariance: the kernel against itself, bit for bit
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("B,H,n,shift", [(3, 4, 300, 1), (6, 8, 385, 3)])
def test_rows_do_not_depend_on_sample_or_head_position(kernel, B, H, n, shift):
    """One (sample, head) problem computed alone (one sample, one head: 64-row tiles) and embedded at three (sample,
    head) positions of a larger batch among random neighbours: 36 CTAs of 128 rows (64-row tiles) and 192 (128-row
    tiles on a 132-SM H100)."""
    g = _gen(B * H)
    q0, k0, v0 = _randn((1, n, 1, 64), g), _randn((1, n, 1, 64), g), _randn((1, n, 1, 64), g)
    alone, _ = _attend(kernel, q0, k0, v0)
    Q, K, V = _random_qkv(B, H, n, n, B + H)
    spots = [(0, 0), (1, H - 1), (B - 1, H // 2)]
    for b, h in spots:
        Q[b, :, h] = q0[0, :, 0]
        K[(b + shift) % B, :, h] = k0[0, :, 0]
        V[(b + shift) % B, :, h] = v0[0, :, 0]
    big, _ = _attend(kernel, Q, K, V, shift)
    for b, h in spots:
        assert torch.equal(big[b, :, h], alone[0, :, 0]), (b, h)


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("B,H,shift", [(2, 3, 1), (4, 12, 2)])
def test_output_rows_move_with_permuted_query_rows(kernel, B, H, shift):
    """nq = 449 = 7 x 64 + 1.  Permuting the seven whole 64-row query blocks moves each block to another query tile and,
    with 128-row tiles (4 x 12 x 4 = 192 CTAs), to the other consumer warpgroup; the output rows must move with them.
    Single rows permuted inside each block come out bit-identical as well: every row runs the same instruction
    sequence."""
    n = 449
    Q, K, V = _random_qkv(B, H, n, n, 7 * B)
    base, _ = _attend(kernel, Q, K, V, shift)
    g = _gen(5)
    perm = torch.arange(n, device=DEV)
    blocks = torch.randperm(7, device=DEV, generator=g)
    perm[:448] = (blocks[:, None] * 64 + torch.arange(64, device=DEV)[None, :]).reshape(-1)
    moved, _ = _attend(kernel, Q[:, perm], K, V, shift)
    assert torch.equal(moved, base[:, perm]), "64-row blocks"
    inner = torch.arange(n, device=DEV)
    inner[:448] = (torch.arange(7, device=DEV)[:, None] * 64 + torch.stack(
        [torch.randperm(64, device=DEV, generator=g) for _ in range(7)])).reshape(-1)
    moved, _ = _attend(kernel, Q[:, inner], K, V, shift)
    assert torch.equal(moved, base[:, inner]), "rows inside 64-row blocks"


def test_64_row_and_128_row_tiles_give_identical_rows():
    """launch_attention takes 128-row query tiles (two consumer warpgroups per CTA) once they give every SM a CTA, else
    64-row tiles.  One problem alone (14 tiles of 128 rows) and replicated over enough samples to reach the SM count
    must give the same rows."""
    H, n = 2, 769
    tiles = (n + 127) // 128 * H
    reps = -(-_sms() // tiles)
    assert tiles < _sms() <= tiles * reps
    Q, K, V = _random_qkv(1, H, n, n, 3)
    alone, _ = _attend("bf16", Q, K, V)
    rep = [x.expand(reps, -1, -1, -1).contiguous() for x in (Q, K, V)]
    many, _ = _attend("bf16", *rep)
    for b in range(reps):
        assert torch.equal(many[b], alone[0]), b


@pytest.mark.parametrize("kernel", KERNELS)
def test_repeat_runs_are_identical_at_cfg2_encoder_size(kernel):
    Q, K, V = _random_qkv(32, 16, 768, 768, 17)
    first, _ = _attend(kernel, Q, K, V, 0, _self)
    second, _ = _attend(kernel, Q, K, V, 0, _self)
    assert torch.equal(first, second)


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------

_RB, _RH, _RN = 2, 2, 65
_RC = 64 * _RH

# (id, edit of the physical arguments given m = 3 in split mode else 1, message, split only)
_REFUSALS = [
    ("empty", lambda a, m: a.update(nk=0), "empty attention problem", False),
    ("stride_not_16B", lambda a, m: a.update(ldk=a["ldk"] + 4 * m), "row strides must be 16B multiples", False),
    ("col0_not_16B", lambda a, m: a.update(v_col0=a["v_col0"] + 4), "column offsets must be 16B multiples", False),
    ("split_stride_not_3x", lambda a, m: a.update(ldq=a["ldq"] + 8), "strides must be 3 x the logical width", True),
    ("shift_negative", lambda a, m: a.update(shift=-1), "kv_batch_shift must lie in [0, batch)", False),
    ("shift_batch", lambda a, m: a.update(shift=_RB), "kv_batch_shift must lie in [0, batch)", False),
    ("q_cols_past_row", lambda a, m: a.update(q_col0=64), "q head columns run past the row width", False),
    ("q_col0_negative", lambda a, m: a.update(q_col0=-8), "q head columns run past the row width", False),
    ("k_cols_past_row", lambda a, m: a.update(k_col0=_RC + 64), "k head columns run past the row width", False),
    ("v_cols_past_row", lambda a, m: a.update(v_col0=_RC + 8), "v head columns run past the row width", False),
    ("ldo_narrow", lambda a, m: a.update(ldo=m * (_RC - 64)), "output rows are narrower than 64 x heads", False),
    ("scale_nan", lambda a, m: a.update(scale=float("nan")), "scale must be finite and positive", False),
    ("scale_inf", lambda a, m: a.update(scale=float("inf")), "scale must be finite and positive", False),
    ("scale_zero", lambda a, m: a.update(scale=0.0), "scale must be finite and positive", False),
    ("scale_negative", lambda a, m: a.update(scale=-0.125), "scale must be finite and positive", False),
    # more CTAs than a grid dimension holds (the launch itself would fail, so nothing runs either way)
    ("grid", lambda a, m: a.update(batch=65536 if m == 3 else 1 << 30), "grid limits", False),
]


@pytest.mark.parametrize("kernel,edit,msg", [(k, r[1], r[2]) for r in _REFUSALS for k in KERNELS if k == "x3" or not r[3]],
                         ids=["%s-%s" % (r[0], k) for r in _REFUSALS for k in KERNELS if k == "x3" or not r[3]])
def test_out_of_range_arguments_are_refused_before_any_launch(kernel, edit, msg):
    """Each requirement of launch_attention, through both entry points (the (hi | lo | hi) stride rule only through the
    split one): non-zero return, the requirement's message, and an output canary that keeps its bits.  Every buffer
    sits inside an allocation with one buffer's worth of slack on each side."""
    m = 3 if kernel == "x3" else 1
    a = dict(ldq=m * _RC, q_col0=0, ldk=m * 2 * _RC, k_col0=0, v_col0=_RC, ldo=m * _RC, batch=_RB, shift=0,
             scale=SCALE)
    a["ldv"] = a["ldk"]
    edit(a, m)

    def slack(ld):
        t = torch.full((3 * _RB * _RN * ld,), float("nan"), device=DEV, dtype=torch.bfloat16)
        return t, ctypes.c_void_p(t.data_ptr() + 2 * _RB * _RN * ld)

    q, pq = slack(m * _RC)
    kv, pkv = slack(m * 2 * _RC)
    out, po = slack(m * _RC)
    before = out.clone()
    fn = lib().sta_op_attention_split if m == 3 else lib().sta_op_attention
    rc = fn(pq, a["ldq"], a["q_col0"], pkv, a["ldk"], a["k_col0"], pkv, a["ldv"], a["v_col0"], po, a["ldo"],
            a["batch"], _RH, _RN, a.get("nk", _RN), a["shift"], a["scale"], cur_stream())
    torch.cuda.synchronize()
    err = lib().sta_last_error().decode()
    assert rc != 0 and msg in err, (rc, err)
    assert torch.equal(out.view(torch.int16), before.view(torch.int16))
