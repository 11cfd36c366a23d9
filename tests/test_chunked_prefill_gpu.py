"""Chunked prefill attention (`sb200_attn_prefill_chunked`): a sequence whose own tokens
[0, hist) were prefilled by earlier calls reads their K/V from the paged pool, and the rest from
the dense qkv rows of the current chunk.  With hist a multiple of
`sb200_attn_prefill_hist_align` every q tile, KV block, mask and rescale decision is that of the
unchunked call, so each output must be bit-identical to `sb200_attn_prefill_dense` over the whole
row.

The history gather re-swizzles every 16-byte chunk: the pool keeps chunk c of a token at
c ^ (pos & 7), the shared-memory tile wants it at c ^ ((pos - past) & 7).  The two differ whenever
the shared prefix's length is not a multiple of 8 (15, 17 and 46 here), so a gather that ignored
`past` would fail those cases; the test asserts that it runs them with history."""
import math

import pytest
import torch

from kv_layout import build_cache
from sutro_b200 import _lib as L

pytestmark = pytest.mark.gpu

DEV = "cuda"
HD = 128
SCALE = 1.0 / math.sqrt(HD)
HEADS = [(32, 8), (16, 8), (40, 8), (64, 8), (8, 8)]
PREFIXES = [0, 15, 16, 17, 46]
N_LAYERS, LAYER = 2, 1
SENTINEL = -12345.0     # bf16-exact


def i32(x):
    return torch.as_tensor(x, dtype=torch.int32).to(DEV)


def layout(hq, hkv):
    """Per sequence (hist, chunk length): several histories in one launch, chunks that end on and
    off q-tile and block edges, and a sequence without history."""
    a = L.lib().sb200_attn_prefill_hist_align(hq, hkv)
    qt = L.lib().sb200_attn_prefill_q_tile(hq, hkv)
    assert a % 128 == 0 and a % qt == 0 and a == 128 * qt // math.gcd(128, qt)
    if a == 128:
        return a, [(0, 300), (128, 1), (384, 129), (1024, 77), (256, 256)]
    return a, [(0, 60), (a, 1), (a, 311), (2 * a, qt + 3)]


def _launch(fn, qkv, pre, n_pre, q_start, q_len, past, hq, hkv, qt, out, *paged):
    """One launch; every argument array stays referenced until the launch has finished (a
    temporary freed before it would hand its memory to the next one)."""
    items = [(i, t0) for i, n in enumerate(q_len) for t0 in range(0, n, qt)]
    keep = [i32([x for it in items for x in it]), i32(q_start), i32(q_len), i32(past)]
    extra = []
    if paged:
        pool, pt, max_pages, slot, hist = paged
        keep += [i32(slot), i32(hist)]
        extra = [L.ptr(pool), L.ptr(pt), max_pages, L.ptr(keep[4]), L.ptr(keep[5])]
    L.check(fn(L.ptr(qkv), qkv.shape[0], L.ptr(out), L.ptr(pre), n_pre, N_LAYERS, LAYER,
               L.ptr(keep[0]), len(items), L.ptr(keep[1]), L.ptr(keep[2]), L.ptr(keep[3]), hq,
               hkv, SCALE, *extra, L.current_stream()))
    torch.cuda.synchronize()


def dense(qkv, pre, n_pre, q_start, q_len, past, hq, hkv, qt, out):
    _launch(L.lib().sb200_attn_prefill_dense, qkv, pre, n_pre, q_start, q_len, past, hq, hkv, qt,
            out)


def chunked(qkv, pre, n_pre, q_start, q_len, past, hq, hkv, qt, out, pool, pt, max_pages, slot,
            hist):
    _launch(L.lib().sb200_attn_prefill_chunked, qkv, pre, n_pre, q_start, q_len, past, hq, hkv,
            qt, out, pool, pt, max_pages, slot, hist)


def case(hq, hkv, past, seed):
    """Whole rows packed densely, their current chunks packed with a 7-row gap between them
    (rows the kernel must not write), and a pool holding each row's [prefix garbage | history]."""
    a, seqs = layout(hq, hkv)
    qt = L.lib().sb200_attn_prefill_q_tile(hq, hkv)
    g = torch.Generator().manual_seed(seed)
    w = (hq + 2 * hkv) * HD
    full_len = [h + n for h, n in seqs]
    full_start = [sum(full_len[:i]) for i in range(len(seqs))]
    full = torch.randn(sum(full_len) + 32, w, generator=g).to(DEV, torch.bfloat16)
    n_pre = max(past, 1)
    pre = torch.randn(N_LAYERS, n_pre, 2 * hkv * HD, generator=g).to(DEV, torch.bfloat16)
    ch_start, ch, t = [], [], 0
    for (h, n), s in zip(seqs, full_start):
        ch_start.append(t)
        ch.append(full[s + h:s + h + n])
        ch.append(torch.randn(7, w, generator=g).to(DEV, torch.bfloat16))
        t += n + 7
    chunk = torch.cat(ch + [torch.zeros(32, w, device=DEV, dtype=torch.bfloat16)])
    k_seqs, v_seqs = [], []
    for (h, _), s in zip(seqs, full_start):
        junk = torch.randn(past, hkv, HD, generator=g).to(DEV, torch.bfloat16)
        own = full[s:s + h, hq * HD:].view(h, 2, hkv, HD)
        k_seqs.append(torch.cat([junk, own[:, 0]]))
        v_seqs.append(torch.cat([junk, own[:, 1]]))
    n_pages = sum((k.shape[0] + 15) // 16 for k in k_seqs) + 8
    pool, pt, max_pages = build_cache(k_seqs, v_seqs, hkv, n_pages, DEV, seed=seed)
    return dict(a=a, qt=qt, seqs=seqs, full=full, full_start=full_start, pre=pre, n_pre=n_pre,
                chunk=chunk, ch_start=ch_start, pool=pool, pt=pt, max_pages=max_pages)


@pytest.mark.parametrize("past", PREFIXES)
@pytest.mark.parametrize("hq,hkv", HEADS, ids=[f"{q}_{k}" for q, k in HEADS])
def test_chunked_equals_dense_over_the_whole_row(hq, hkv, past):
    c = case(hq, hkv, past, seed=hq * 1000 + hkv * 10 + past)
    seqs, n = c["seqs"], len(c["seqs"])
    ref = torch.zeros(c["full"].shape[0], hq * HD, dtype=torch.bfloat16, device=DEV)
    dense(c["full"], c["pre"], c["n_pre"], c["full_start"], [h + m for h, m in seqs], [past] * n,
          hq, hkv, c["qt"], ref)
    out = torch.full((c["chunk"].shape[0], hq * HD), SENTINEL, dtype=torch.bfloat16, device=DEV)
    chunked(c["chunk"], c["pre"], c["n_pre"], c["ch_start"], [m for _, m in seqs], [past] * n,
            hq, hkv, c["qt"], out, c["pool"], c["pt"], c["max_pages"], list(range(n)),
            [h for h, _ in seqs])
    torch.cuda.synchronize()
    written = torch.zeros(out.shape[0], dtype=torch.bool, device=DEV)
    for (h, m), s, cs in zip(seqs, c["full_start"], c["ch_start"]):
        want = ref[s + h:s + h + m]
        got = out[cs:cs + m]
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (h, m)
        written[cs:cs + m] = True
    # no stray writes: every row outside the chunks keeps the sentinel
    assert (out[~written] == SENTINEL).all()
    # the history was really read from the pool; with past % 8 != 0 the pool's chunk order
    # (pos & 7) differs from the tile's ((pos - past) & 7) on every gathered token, so a verbatim
    # copy of the pool rows would have failed the comparison above
    assert sum(h > 0 for h, _ in seqs) >= 3
    gathered = torch.cat([torch.arange(h) for h, _ in seqs if h > 0])
    differs = ((past + gathered) & 7) != (gathered & 7)
    assert bool(differs.all()) == (past % 8 != 0) and bool(differs.any()) == (past % 8 != 0)
    print("CHUNKED", f"{hq}/{hkv}", f"past={past}", f"reswizzled={past % 8 != 0}")


def test_prefixes_include_ones_that_need_the_reswizzle():
    """Prefix lengths that are not multiples of 8 (and one that is not a multiple of 16, so a
    history block starts mid-page): the cases a gather that ignored `past` would fail."""
    assert [p for p in PREFIXES if p % 8] and [p for p in PREFIXES if p % 16 == 0 and p]


@pytest.mark.parametrize("hq,hkv", HEADS, ids=[f"{q}_{k}" for q, k in HEADS])
def test_no_history_is_the_dense_call(hq, hkv):
    """hist = 0 everywhere: byte-identical to sb200_attn_prefill_dense on the same rows."""
    c = case(hq, hkv, 46, seed=hq + hkv)
    seqs, n = c["seqs"], len(c["seqs"])
    q_len = [m for _, m in seqs]
    a = torch.full((c["chunk"].shape[0], hq * HD), SENTINEL, dtype=torch.bfloat16, device=DEV)
    b = a.clone()
    dense(c["chunk"], c["pre"], c["n_pre"], c["ch_start"], q_len, [46] * n, hq, hkv, c["qt"], a)
    chunked(c["chunk"], c["pre"], c["n_pre"], c["ch_start"], q_len, [46] * n, hq, hkv, c["qt"],
            b, c["pool"], c["pt"], c["max_pages"], list(range(n)), [0] * n)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_alignment_and_arguments():
    lib = L.lib()
    assert [lib.sb200_attn_prefill_hist_align(hq, hkv) for hq, hkv in HEADS] == \
        [128, 128, 3200, 128, 128]
    assert lib.sb200_attn_prefill_hist_align(12, 4) == 0
    one, two = i32([0]), i32([0, 0])
    rc = lib.sb200_attn_prefill_chunked(
        L.ptr(one), 1, L.ptr(one), None, 0, 1, 0, L.ptr(two), 1, L.ptr(one), L.ptr(one),
        L.ptr(one), 32, 8, SCALE, None, None, 0, None, None, L.current_stream())
    assert rc != 0 and b"required" in lib.sb200_last_error()
