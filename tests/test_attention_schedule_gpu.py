"""GPU: the persistent schedule of the wgmma attention kernel.  One CTA per SM walks the items (query tile, head,
sample) blockIdx.x, blockIdx.x + gridDim.x, ..; the Q tile is double-buffered, the K / V ring and its barrier phases run
on from one item to the next, the two consumer warpgroups take turns issuing their MMAs, a warpgroup with no valid row
in an item only passes its turns and releases the stages, and a last key tile of <= 16 keys takes one k16 step of P V.

Planted dominant keys (a different target key per sample, head and row) give answers that must come out bit for bit,
so a Q buffer, ring stage or phase carried wrongly from one item to the next shows up as a wrong row.  Every call runs
on the NaN-filled buffers and output canaries of test_attention_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from test_attention_gpu import (DEV, _attend, _away_from_zero, _cross, _expect_planted, _gen,  # noqa: E402
                                _random_qkv, _self, _sms)


def _planted(B, H, nq, nk, shift, targets, seed):
    """Keys are random +-1 vectors and q = 16 k_target of the row's K / V sample: the target leads every other key by
    more than 40 log2 units, so the output row is V[target] exactly.  targets: [B][nq][H] key indices."""
    g = _gen(seed)
    K = (torch.randint(0, 2, (B, nk, H, 64), device=DEV, generator=g) * 2 - 1).float()
    V = _away_from_zero((B, nk, H, 64), g)
    Q = torch.empty(B, nq, H, 64, device=DEV)
    for b in range(B):
        Q[b] = 16.0 * K[(b + shift) % B].gather(0, targets[b].unsqueeze(-1).expand(-1, -1, 64))
    return Q, K, V


def _check_planted(B, H, nq, nk, shift, layout, targets, seed):
    Q, K, V = _planted(B, H, nq, nk, shift, targets, seed)
    out, seen = _attend("bf16", Q, K, V, shift, layout)
    lead = _expect_planted("bf16", out, seen, shift, targets)
    assert lead >= 40.0, "construction: lead %.1f log2 units" % lead


@pytest.mark.parametrize("name,B,H,n,shift,layout", [
    ("cfg2_dec_self", 32, 12, 769, 0, _self),
    ("cfg2_dec_cross", 32, 12, 769, 16, _cross),
    ("cfg2_enc_self", 32, 16, 768, 0, _self),
])
def test_every_item_of_a_persistent_cta_gets_its_own_answer(name, B, H, n, shift, layout):
    """The model's shapes at cfg-2: about 20 (decoder) and 23 (encoder) items per CTA on a 132-SM H100.  Random targets
    per (sample, row, head), so no two neighbouring items or rows share an answer."""
    g = _gen(len(name) * 7 + H)
    targets = torch.randint(0, n, (B, n, H), device=DEV, generator=g)
    _check_planted(B, H, n, n, shift, layout, targets, len(name) + H)


def _grid_edges():
    s = _sms()
    # (id, rows per problem, copies): rows <= 64 with fewer copies than SMs take 64-row tiles (one item per copy),
    # otherwise 128-row tiles, one item per copy
    return [("sms_minus_1", 60, s - 1), ("sms", 100, s), ("sms_plus_1", 100, s + 1), ("2sms_plus_1", 100, 2 * s + 1)]


@pytest.mark.parametrize("edge", range(4), ids=["sms_minus_1", "sms", "sms_plus_1", "2sms_plus_1"])
def test_item_counts_at_the_grid_edges(edge):
    """Five different one-head problems (nk = 769: the one-key tail), each computed alone, then replicated as copy
    c = problem c % 5 so that the item count is SMs - 1, SMs, SMs + 1 or 2 SMs + 1.  Items i and i + SMs of one CTA hold
    different problems (SMs is not a multiple of 5 on an H100), and every copy must be bit-identical to its problem
    alone."""
    _, nq, copies = _grid_edges()[edge]
    nk, P = 769, 5
    assert _sms() % P != 0
    probs = []
    for i in range(P):
        g = _gen(100 + i)
        probs.append((torch.randn(1, nq, 1, 64, device=DEV, generator=g), torch.randn(1, nk, 1, 64, device=DEV, generator=g),
                      torch.randn(1, nk, 1, 64, device=DEV, generator=g)))
    alone = [_attend("bf16", *pr)[0] for pr in probs]
    idx = torch.arange(copies, device=DEV) % P
    Q, K, V = (torch.cat([probs[i][k] for i in idx.tolist()]) for k in range(3))
    many, _ = _attend("bf16", Q, K, V)
    for c in range(copies):
        assert torch.equal(many[c], alone[c % P][0]), "copy %d of %d" % (c, copies)


@pytest.mark.parametrize("r", [1, 15, 16, 17, 64, 127])
def test_ragged_key_tail_widths(r):
    """nk = 5 x 128 + r: tails of <= 16 keys take one k16 step of P V, wider ones all eight.  Half the rows target a key
    of the tail, the others keys of the full tiles.  nq = 257 on 4 x 12 samples x heads (144 items of 128 rows): the
    last query tile has one row, so its second warpgroup has none."""
    B, H, nq, shift = 4, 12, 257, 1
    nk = 5 * 128 + r
    g = _gen(r)
    tail = 640 + torch.randint(0, r, (B, nq, H), device=DEV, generator=g)
    body = torch.randint(0, 640, (B, nq, H), device=DEV, generator=g)
    pick = torch.randint(0, 2, (B, nq, H), device=DEV, generator=g).bool()
    _check_planted(B, H, nq, nk, shift, _cross, torch.where(pick, tail, body), 1000 + r)


@pytest.mark.parametrize("nq", [320, 321, 385])
def test_query_tails_with_an_empty_or_one_row_warpgroup(nq):
    """nq = 320 and 385 leave the second consumer warpgroup of the last 128-row query tile without a row (it only passes
    its turns and releases the ring stages), 321 leaves it one row; 4 x 12 samples x heads give 128-row tiles.  Checked
    bit for bit against the same rows computed with 64-row tiles (one sample, one head at a time is below the SM count)
    and against planted answers."""
    B, H, nk, shift = 4, 12, 700, 1
    Q, K, V = _random_qkv(B, H, nq, nk, nq)
    many, _ = _attend("bf16", Q, K, V, shift)
    for b, h in ((0, 0), (B - 1, H - 1), (1, 5)):
        kb = (b + shift) % B
        one, _ = _attend("bf16", Q[b:b + 1, :, h:h + 1], K[kb:kb + 1, :, h:h + 1], V[kb:kb + 1, :, h:h + 1])
        assert torch.equal(many[b, :, h], one[0, :, 0]), (b, h)
    g = _gen(nq + 1)
    _check_planted(B, H, nq, nk, shift, _cross, torch.randint(0, nk, (B, nq, H), device=DEV, generator=g), nq)
