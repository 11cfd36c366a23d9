"""Dense prefill attention (attn_prefill_tc.cu): the MMAs of a KV block cover only its valid
columns rounded up to 32 (32, 64, 96 or 128), and the result must be exactly what the full
128-column block gave.  The columns a narrower block drops carry P = 0, so O and the row sums
must not change in a single bit.

A token attends to the same keys whatever follows it in its sequence, but the width of the block
it sees does depend on that: the last own block of a q tile ends at min(q_len, t0 + q_tile).  So
the outputs of the first m tokens of a sequence must be bit-identical between the full sequence
and the same sequence cut to m tokens, for cuts that move the block across every width class.
Outputs must also not depend on the order of the work items or on how they are split between
launches.
"""
import math
import random

import pytest
import torch

from sutro_b200 import _lib as L

pytestmark = pytest.mark.gpu

DEV = "cuda"
HD = 128
SCALE = 1.0 / math.sqrt(HD)
HEADS = [(8, 8), (16, 8), (32, 8), (16, 2)]     # G = 1, 2, 4, 8
HEAD_IDS = ["G1", "G2", "G4", "G8"]
PREFIXES = [0, 15, 16, 17, 46]
N_LAYERS, LAYER, PREFIX_ROWS = 2, 1, 64


def i32(x):
    return torch.as_tensor(x, dtype=torch.int32).to(DEV)


def buffers(hq, hkv, T, seed):
    """Random dense qkv rows (32 spare rows: every 32-row TMA box stays on finite values) and a
    random prefix buffer."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    qkv = torch.randn(T + 32, (hq + 2 * hkv) * HD, generator=g).to(DEV, torch.bfloat16)
    pre = torch.randn(N_LAYERS, PREFIX_ROWS, 2 * hkv * HD, generator=g).to(DEV, torch.bfloat16)
    return qkv, pre


def run(qkv, pre, specs, q_start, hq, hkv, item_lists):
    """sb200_attn_prefill_dense, one launch per item list, into one output."""
    out = torch.zeros(qkv.shape[0], hq * HD, dtype=torch.bfloat16, device=DEV)
    d_qs, d_ql, d_past = i32(q_start), i32([n for _, n in specs]), i32([p for p, _ in specs])
    for items in item_lists:
        d_items = i32([x for it in items for x in it])
        L.check(L.lib().sb200_attn_prefill_dense(
            L.ptr(qkv), qkv.shape[0], L.ptr(out), L.ptr(pre), PREFIX_ROWS, N_LAYERS, LAYER,
            L.ptr(d_items), len(items), L.ptr(d_qs), L.ptr(d_ql), L.ptr(d_past), hq, hkv, SCALE,
            L.current_stream()))
    torch.cuda.synchronize()
    return out


def items_of(specs, qt):
    return [(i, t0) for i, (_, n) in enumerate(specs) for t0 in range(0, n, qt)]


def bits(t):
    return t.contiguous().view(torch.int16)


@pytest.mark.parametrize("past", PREFIXES)
@pytest.mark.parametrize("hq,hkv", HEADS, ids=HEAD_IDS)
def test_cut_sequences_are_bit_identical(hq, hkv, past):
    """One sequence of 600 own tokens and its cuts at every length that changes the width class
    of some q tile's last own block, all in one launch: the common tokens agree bit for bit."""
    qt = L.lib().sb200_attn_prefill_q_tile(hq, hkv)
    full = 600
    # the width of the block [128 b, ...) of a tile changes at lengths 128 b + 32 w + {0, 1}
    cuts = sorted({c for b in range(5) for w in range(4) for d in (0, 1, 16, 17)
                   for c in [128 * b + 32 * w + d] if 1 <= c < full} | {1, 2, qt - 1, qt, qt + 1})
    qkv_full, pre = buffers(hq, hkv, full, seed=hq * 131 + hkv * 7 + past)
    specs = [(past, full)] + [(past, c) for c in cuts]
    # every sequence starts with the same rows: copy the full sequence's rows to each cut
    q_start, T = [], 0
    for _, n in specs:
        q_start.append(T)
        T += n
    qkv = torch.randn(T + 32, qkv_full.shape[1]).to(DEV, torch.bfloat16)
    for s, (_, n) in zip(q_start, specs):
        qkv[s:s + n] = qkv_full[:n]
    items = items_of(specs, qt)
    out = run(qkv, pre, specs, q_start, hq, hkv, [items])
    ref = bits(out[:full])
    for s, (_, n) in zip(q_start[1:], specs[1:]):
        got = bits(out[s:s + n])
        bad = (got != ref[:n]).any(dim=1).nonzero().flatten().tolist()
        assert not bad, (f"cut {n}, prefix {past}: tokens {bad[:8]} differ from the full "
                         f"sequence's")


@pytest.mark.parametrize("hq,hkv", HEADS, ids=HEAD_IDS)
def test_item_order_and_launch_split_do_not_matter(hq, hkv):
    """A batch of sequences with every prefix length, run as one launch in order, as one launch
    with the items shuffled, and as three launches over a shuffled partition."""
    qt = L.lib().sb200_attn_prefill_q_tile(hq, hkv)
    rng = random.Random(hq * 10 + hkv)
    specs = [(rng.choice(PREFIXES), n) for n in (1, 15, 16, 17, 31, 33, 64, 97, 107, 128, 129,
                                                  255, 300, 513, 600)]
    q_start, T = [], 0
    for _, n in specs:
        q_start.append(T)
        T += n
    qkv, pre = buffers(hq, hkv, T, seed=hq + hkv)
    items = items_of(specs, qt)
    ref = run(qkv, pre, specs, q_start, hq, hkv, [items])[:T]
    shuffled = items[:]
    rng.shuffle(shuffled)
    one = run(qkv, pre, specs, q_start, hq, hkv, [shuffled])[:T]
    a, b = sorted(rng.sample(range(1, len(items)), 2))
    three = run(qkv, pre, specs, q_start, hq, hkv, [shuffled[:a], shuffled[a:b], shuffled[b:]])[:T]
    assert torch.equal(bits(one), bits(ref))
    assert torch.equal(bits(three), bits(ref))
