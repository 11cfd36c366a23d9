"""Attention kernels checked bit for bit where the math allows it, and against fp64 elsewhere.

Covers the dense prefill attention (attn_prefill_tc.cu), the decode attention (attn_decode.cu)
and the fused QKV epilogue's dense K/V copy (gemm_wgmma.cu), all through the C ABI, at the four
GQA group sizes and the engine's scale 1/sqrt(128):

1. Masked rows do not matter.  Every location a kernel may load but must not use (rows past a
   sequence's end inside a 32-row TMA box, prefix rows at or after `past`, other kv heads, other
   layers, token slots past ctx_len, other slots' pages, page-table entries past the last page)
   is filled with finite decoys whose keys are aligned with the queries and whose values are
   about +-1000; the outputs of every query that cannot see them must not change in a single bit.
   NaN is placed only where no kernel loads anything.
2. Pointer attention.  Q and K are built so that every (token, head) has exactly one visible key
   that outscores every other visible key by > 40 log2 units; the output must then be exactly
   V[target].  Masked positions carry decoy keys that outscore the target, so a mask that leaks
   turns the output into V[decoy].
3. Tight numerics at engine-sized contexts (up to 4096 tokens, ~1000 prefix rows, hundreds of
   decode rows) against an fp64 softmax, with the per-element bound of `error_bound`.
4. The fused QKV epilogue writes post-norm/RoPE K and V both to the paged pool and, unswizzled,
   to the k/v columns of its output; the two copies must be identical, Q and K must be the exact
   norm -> RoPE of the projection at every served head layout and at positions up to 32,767, and
   the chain the engine runs (fused QKV -> dense prefill attention) must meet the bound of 3.
"""
import math
import random

import pytest
import torch

from sutro_b200 import _lib as L
from sutro_b200 import modelspec as MS
import bf16_ref as R
import kv_layout as KV

DEV = "cuda"
HD, PAGE = KV.HD, KV.PAGE
SCALE = 1.0 / math.sqrt(HD)
HEADS = [(8, 8), (16, 8), (32, 8), (16, 2)]     # G = 1, 2, 4, 8; (32, 8) is both real models
HEAD_IDS = ["G1", "G2", "G4", "G8"]


def bf(x):
    return x.to(torch.bfloat16)


def i32(x):
    return torch.as_tensor(x, dtype=torch.int32).to(DEV)


def starts(specs):
    out, acc = [], 0
    for _, n in specs:
        out.append(acc)
        acc += n
    return out, acc


# --------------------------------------------------------------------------- error bound
P_ROUND = 2.0 ** -8       # unit roundoff of bf16 (8 significant bits)
FP32_SLACK = 2.0 ** -12   # fp32 scores (up to a few thousand), ex2.approx, fp32 accumulation
MEAN_LIMIT = 0.3          # mean |err| / mean bound


def ulp_bf16(x):
    """Spacing of the bf16 numbers at |x|."""
    _, e = torch.frexp(x.abs())
    u = torch.ldexp(torch.ones_like(x), (e - 8).clamp(min=-133))
    return torch.where(x == 0, torch.full_like(x, 2.0 ** -133), u)


def error_bound(ref, mag):
    """Per-element bound on |got - ref| for both attention kernels.

    ref = sum_j p_j v_j / sum_j p_j in fp64, mag = sum_j p_j |v_j| / sum_j p_j.  The kernels
    compute p_j in fp32 (up to a common factor: the dense kernel rescales lazily, so its P may
    reach 2^8), round P to bf16 for the P.V MMA, accumulate O and l = sum_j p_j (unrounded) in
    fp32, and round O / l to bf16 once.  Rounding P moves each p_j by at most 2^-8 p_j whatever
    its scale, so before the last rounding the output is off by at most
        E = (2^-8 + 2^-12) * mag,
    2^-12 covering the fp32 scores (an fp32 score of a few thousand is off by ~1e-3, which moves p
    by ~1e-4 relative), ex2.approx and the fp32 accumulation.  The final rounding adds half an ulp of a
    value within E of ref:  |got - ref| <= ulp(|ref| + E) / 2 + E.  Written as c * 2^-9 * mag, the
    P term has c = 2: c ~ 1.25 covers long rows, but rows with a few keys and one dominant |v|
    reach c = 1.98 in a CPU emulation (test_error_bound_covers_emulated_p_rounding), so a smaller
    c would fail on correct kernels.
    """
    e = (P_ROUND + FP32_SLACK) * mag
    return 0.5 * ulp_bf16(ref.abs() + e) + e


def bound_ratios(got, ref, mag):
    got = got.double().reshape(ref.shape)
    err = (got - ref).abs()
    b = error_bound(ref, mag)
    return (err / b).max().item(), (err.mean() / b.mean()).item()


def assert_within_bound(got, ref, mag, what):
    assert torch.isfinite(got).all(), what
    worst, mean = bound_ratios(got, ref, mag)
    print(f"[attn bound] {what}: max err/bound {worst:.3f}, mean err / mean bound {mean:.3f}")
    assert worst <= 1.0, (what, worst)
    assert mean <= MEAN_LIMIT, (what, mean)


def attn_ref64(q, k, v, n_vis, hkv):
    """fp64 softmax(q k^T * scale) v.  q: [n, hq, 128]; k, v: [L, hkv, 128]; query i sees keys
    [0, n_vis[i]).  Returns (ref, mag) [n, hq, 128] fp64 (mag: see error_bound).  Chunked over
    queries so that the score matrix stays below 256 MB."""
    n, hq = q.shape[0], q.shape[1]
    G, Lk = hq // hkv, k.shape[0]
    dev = q.device
    kd, vd = k.double().to(dev), v.double().to(dev)
    va = vd.abs()
    n_vis = torch.as_tensor(n_vis, device=dev).long()
    pos = torch.arange(Lk, device=dev)
    ref = torch.empty(n, hq, HD, dtype=torch.float64, device=dev)
    mag = torch.empty_like(ref)
    step = max(1, (1 << 25) // (hq * Lk))
    for i0 in range(0, n, step):
        qc = q[i0:i0 + step].double().view(-1, hkv, G, HD)
        s = torch.einsum("chgd,lhd->chgl", qc, kd) * SCALE
        s = s.masked_fill(pos[None, None, None, :] >= n_vis[i0:i0 + step, None, None, None],
                          float("-inf"))
        p = torch.softmax(s, dim=-1)
        ref[i0:i0 + step] = torch.einsum("chgl,lhd->chgd", p, vd).reshape(-1, hq, HD)
        mag[i0:i0 + step] = torch.einsum("chgl,lhd->chgd", p, va).reshape(-1, hq, HD)
    return ref, mag


def test_error_bound_covers_emulated_p_rounding():
    """CPU emulation of the kernels' rounding points (P in fp32 at a random power-of-two scale up
    to 2^8, rounded to bf16, O and l accumulated in fp32, O / l rounded to bf16) stays within
    error_bound, with the mean ratio below MEAN_LIMIT, from 2 keys up to 4096."""
    g = torch.Generator().manual_seed(0)
    worst = 0.0
    for Lk in (2, 3, 5, 17, 33, 129, 1000, 4096):
        for gain in (1.0, 6.0):
            n = max(16, 40000 // Lk)
            q = bf(torch.randn(n, HD, generator=g) * gain).double()
            k = bf(torch.randn(Lk, HD, generator=g)).double()
            v = bf(torch.randn(Lk, HD, generator=g)).double()
            s = q @ k.T * SCALE
            p = torch.softmax(s, -1)
            ref, mag = p @ v, p @ v.abs()
            lazy = torch.exp2(torch.rand(n, 1, generator=g, dtype=torch.float64) * 8)
            p32 = (torch.exp(s - s.max(-1, keepdim=True).values) * lazy).float()
            o = bf(p32).float() @ v.float()
            got = bf(o / p32.sum(-1, keepdim=True))
            w, m = bound_ratios(got, ref, mag)
            assert w <= 1.0 and m <= MEAN_LIMIT, (Lk, gain, w, m)
            worst = max(worst, w)
    assert worst > 0.5   # the bound is not loose: some element comes close to it


# --------------------------------------------------------------------------- pointer construction
A_PTR, D_PTR = 20.0, 40.0     # address and decoy-channel amplitudes (exact in bf16)
N_ADDR = 1024                 # positions a pointer test may address


def address(j):
    """[n, 128]: A * (e_{j mod 32} + e_{32 + j div 32}) for j < 1024.  Two distinct addresses share
    at most one coordinate, so a query at its target's address scores 2A^2 against it and at most
    A^2 against any other key.  Dims 64..127 stay zero: they are the decoy channels."""
    j = torch.as_tensor(j).long().reshape(-1)
    assert int(j.max()) < N_ADDR
    x = torch.zeros(j.numel(), HD)
    r = torch.arange(j.numel())
    x[r, j % 32] = A_PTR
    x[r, 32 + j // 32] = A_PTR
    return x


def kv_address(pos, kvh):
    """Key of absolute position `pos` in kv head `kvh` (each head permutes the addresses)."""
    return address((torch.as_tensor(pos).long() + 389 * kvh) % N_ADDR)


def test_pointer_construction_is_sharp():
    """With all 1024 addresses visible, the fp64 softmax weight of the target is >= 1 - 2^-20
    and its score is > 40 log2 units above every other key; a decoy channel (D^2 = 1600 against
    2A^2 = 800) takes the same weight from the target when it is visible."""
    keys = address(torch.arange(N_ADDR)).double()
    s = keys @ keys.T * SCALE                            # [target, key]
    w = torch.softmax(s, -1).diagonal()
    assert w.min().item() >= 1 - 2.0 ** -20
    others = s.masked_fill(torch.eye(N_ADDR, dtype=torch.bool), float("-inf")).max(-1).values
    assert ((s.diagonal() - others) / math.log(2)).min().item() > 40
    q = address([700]).double()
    q[0, 64 + 5] = D_PTR
    dk = keys.clone()
    dk[3, 64 + 5] = D_PTR                                # key 3 carries the decoy channel 5
    p = torch.softmax((dk @ q[0]) * SCALE, -1)
    assert p[3].item() >= 1 - 2.0 ** -20


def pointer_candidates(vis_end, edges, G, rng):
    """Visible positions [0, vis_end] to point at: the edge positions first, then random ones
    until the G heads of a group can point at different keys."""
    cand = sorted({e for e in edges if 0 <= e <= vis_end})
    extra = [x for x in rng.sample(range(vis_end + 1), min(vis_end + 1, G + 4)) if x not in cand]
    return cand + extra[:max(0, G - len(cand))]


def pointer_value(n, kvh_count, gen):
    """bf16 V with |v| in [0.25, 2): never 0, so V[target] cannot be mistaken for a tiny leak."""
    sign = torch.where(torch.rand(n, kvh_count, HD, generator=gen) < 0.5, -1.0, 1.0)
    return bf(sign * (0.25 + 1.75 * torch.rand(n, kvh_count, HD, generator=gen)))


# --------------------------------------------------------------------------- launchers
def q_tiles(specs, hq, hkv):
    qt = L.lib().sb200_attn_prefill_q_tile(hq, hkv)
    return [x for i, (_, n) in enumerate(specs) for t0 in range(0, n, qt) for x in (i, t0)]


def run_dense(qkv, pre, prefix_rows, n_layers, layer, specs, hq, hkv):
    """sb200_attn_prefill_dense over sequences packed back to back; -> [T, hq, 128]."""
    q_start, T = starts(specs)
    items = q_tiles(specs, hq, hkv)
    out = torch.zeros(qkv.shape[0], hq * HD, dtype=torch.bfloat16, device=DEV)
    d_items, d_qs = i32(items), i32(q_start)
    d_ql, d_past = i32([n for _, n in specs]), i32([p for p, _ in specs])
    L.check(L.lib().sb200_attn_prefill_dense(
        L.ptr(qkv), qkv.shape[0], L.ptr(out), L.ptr(pre), prefix_rows if pre is not None else 0,
        n_layers, layer, L.ptr(d_items), len(items) // 2, L.ptr(d_qs), L.ptr(d_ql), L.ptr(d_past),
        hq, hkv, SCALE, L.current_stream()))
    torch.cuda.synchronize()
    return out[:T].view(T, hq, HD)


def run_decode(qkv, pool, pt, row_slot, ctx, hq, hkv):
    """sb200_attn_decode.  -> [B, hq, 128]."""
    B = qkv.shape[0]
    out = torch.zeros(B, hq * HD, dtype=torch.bfloat16, device=DEV)
    d_pt, d_rs, d_ctx = i32(pt), i32(row_slot), i32(ctx)
    L.check(L.lib().sb200_attn_decode(L.ptr(qkv), L.ptr(out), L.ptr(pool), L.ptr(d_pt),
                                      pt.shape[1], L.ptr(d_rs), L.ptr(d_ctx), B, hq, hkv, SCALE,
                                      L.current_stream()))
    torch.cuda.synchronize()
    return out.view(B, hq, HD)


# --------------------------------------------------------------------------- paged cache
def paged_cache(k_seqs, v_seqs, share=0, spare=4, seed=0):
    """Scatter per-sequence K/V ([L_i, hkv, 128] bf16) into a pool of shuffled pages.

    Sequences longer than `share` pages share their first `share` pages (their K/V there must be
    equal).  Every slot the sequences do not fill holds finite random values.  `spare` pages are
    referenced by no page-table entry; every entry past a sequence's last page points at one more
    page, the decoy page.  Returns (logical pool [pages, hkv, 2, 16, 128] on the device, page table
    [n, max_pages] on the host, decoy page id, spare page ids)."""
    g = torch.Generator().manual_seed(seed)
    hkv = k_seqs[0].shape[1]
    lens = [k.shape[0] for k in k_seqs]
    n_pages = [(l + PAGE - 1) // PAGE for l in lens]
    sharing = [share > 0 and l > share * PAGE for l in lens]
    total = share + sum(n - (share if s else 0) for n, s in zip(n_pages, sharing)) + 1 + spare
    order = iter(torch.randperm(total, generator=g).tolist())
    shared = [next(order) for _ in range(share)]
    pt = torch.full((len(lens), max(n_pages) + 2), -1, dtype=torch.long)
    for i, (n, s) in enumerate(zip(n_pages, sharing)):
        for p in range(n):
            pt[i, p] = shared[p] if s and p < share else next(order)
    decoy = next(order)
    spare_ids = [next(order) for _ in range(spare)]
    pt[pt < 0] = decoy
    logical = bf(torch.randn(total, hkv, 2, PAGE, HD, device=DEV))
    for i, (k, v) in enumerate(zip(k_seqs, v_seqs)):
        pos = torch.arange(lens[i])
        pages, r = pt[i][pos // PAGE].to(DEV), (pos % PAGE).to(DEV)
        logical[pages, :, 0, r] = k.to(DEV)
        logical[pages, :, 1, r] = v.to(DEV)
    return logical, pt, decoy, spare_ids


def first_touched(mod, pt_row, length):
    """[hkv]: the first position < length whose slot is marked in mod [pages, hkv, 16], else
    length."""
    pos = torch.arange(length)
    m = mod[pt_row[pos // PAGE], :, pos % PAGE]                    # [length, hkv]
    return torch.where(m, pos[:, None], length).min(0).values


def check_unchanged(out, base, unchanged, what):
    """Bits of the queries that cannot see the change must be equal; the others must move."""
    u = unchanged.to(out.device)
    assert torch.equal(out[u], base[u]), f"{what}: leaked into a query that cannot see it"
    if (~u).any():
        assert not torch.equal(out[~u], base[~u]), f"{what}: the decoys changed nothing visible"


def decoy_k(u, rows):
    """[rows, hkv, 128]: keys aligned with the queries' common direction u [hkv, 128]."""
    return bf((2 * u).expand(rows, *u.shape))


def decoy_v(rows, hkv):
    return bf(1000 * torch.where(torch.rand(rows, hkv, HD, device=DEV) < 0.5, -1.0, 1.0))


def queries(rows, hq, hkv, u, gain=1.0):
    """Random q rows [rows, (hq + 2 hkv) * 128] sharing the per-kv-head direction u (so a key
    along u dominates every query of its group); k/v columns random."""
    G = hq // hkv
    x = torch.randn(rows, (hq + 2 * hkv) * HD, device=DEV)
    x[:, :hq * HD] = gain * (x[:, :hq * HD] + 1.5 * u.repeat_interleave(G, 0).reshape(1, -1))
    return bf(x)


# --------------------------------------------------------------------------- 1. masked rows
def dense_unchanged(specs, hq, hkv, rows=(), pre_rows=(), kv_heads=None):
    """[T, hq] bool: queries that see none of the changed qkv rows / prefix rows of kv_heads."""
    q_start, T = starts(specs)
    G = hq // hkv
    heads = torch.tensor([kv_heads is None or h // G in kv_heads for h in range(hq)])
    m = torch.ones(T, hq, dtype=torch.bool)
    for s, (p, n) in enumerate(specs):
        own = [r - q_start[s] for r in rows if q_start[s] <= r < q_start[s] + n]
        first = 0 if any(r < p for r in pre_rows) else min(own, default=n)
        m[q_start[s] + first:q_start[s] + n, heads] = False
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("hq,hkv", HEADS, ids=HEAD_IDS)
def test_dense_prefill_masked_rows_do_not_leak(hq, hkv):
    """A past of 37 (odd: a mask off by one on odd columns shows), own lengths crossing the 16-,
    32-, 128- and 256-row boundaries, a 17-row sequence inside the previous one's last box, and
    40 padding rows of which the first 31 are in reach of the last sequence's boxes."""
    G, P, prefix_rows, n_layers, layer = hq // hkv, 37, 100, 3, 1
    specs = [(P, 300), (0, 161), (P, 17), (0, 140)]
    q_start, T = starts(specs)
    reach = T + 31                   # qkv rows [T, reach) can be loaded; later ones never are
    torch.manual_seed(G)
    u = torch.randn(hkv, HD, device=DEV)
    qkv = queries(T + 40, hq, hkv, u)
    pre = bf(torch.randn(n_layers, prefix_rows, 2 * hkv * HD, device=DEV))
    KVC = slice(hq * HD, None)       # k | v columns of qkv: the layout of a prefix row

    def run():
        return run_dense(qkv, pre, prefix_rows, n_layers, layer, specs, hq, hkv)

    def put(buf_rows, kv_heads=None):
        n = buf_rows.shape[0]
        k, v = buf_rows[:, :hkv * HD].view(n, hkv, HD), buf_rows[:, hkv * HD:].view(n, hkv, HD)
        hs = list(range(hkv)) if kv_heads is None else kv_heads
        k[:, hs] = decoy_k(u, n)[:, hs]
        v[:, hs] = decoy_v(n, hkv)[:, hs]

    base0 = run()
    # NaN where no box reaches: qkv k/v past the reach, prefix rows past P + 31, other layers
    qkv[reach:, KVC] = float("nan")
    pre[layer, P + 31:] = float("nan")
    pre[[i for i in range(n_layers) if i != layer]] = float("nan")
    base = run()
    assert torch.isfinite(base).all()
    assert torch.equal(base, base0), "rows outside every box / other layers changed the output"
    qkv0, pre0 = qkv.clone(), pre.clone()

    def restore():
        qkv.copy_(qkv0)
        pre.copy_(pre0)

    # prefix rows [P, P + 31): inside the last prefix box, masked for every sequence
    put(pre[layer, P:P + 31])
    check_unchanged(run(), base, dense_unchanged(specs, hq, hkv), "prefix rows >= past")
    restore()
    # the 31 rows after each sequence's last token (the next sequence's rows, or padding)
    for s, (_, n) in enumerate(specs):
        end = q_start[s] + n
        rows = range(end, min(end + 31, reach))
        put(qkv[end:end + len(rows), KVC])
        check_unchanged(run(), base, dense_unchanged(specs, hq, hkv, rows=rows),
                        f"box past the end of sequence {s}")
        restore()
    # own row j: the queries before j must not see it (tile, box and block boundaries)
    for s, js in ((0, (15, 16, 17, 31, 32, 33, 127, 128, 129, 255, 256)), (1, (1, 64, 127, 128))):
        for j in js:
            r = q_start[s] + j
            put(qkv[r:r + 1, KVC])
            check_unchanged(run(), base, dense_unchanged(specs, hq, hkv, rows=[r]),
                            f"own row {j} of sequence {s}")
            restore()
    # the k/v columns of kv head 0 only: the other kv heads' queries must not move
    if hkv > 1:
        put(qkv[:reach, KVC], kv_heads=[0])
        put(pre[layer, :P + 31], kv_heads=[0])
        check_unchanged(run(), base,
                        dense_unchanged(specs, hq, hkv, rows=range(reach), pre_rows=range(P + 31),
                                        kv_heads=[0]),
                        "kv head 0")
        restore()


def paged_decoys(logical, u, mod, page, r, kv_heads=None):
    """Decoy K (along u) and V (+-1000) into slots (page, r) of the logical pool; marks mod."""
    page, r = torch.as_tensor(page).reshape(-1), torch.as_tensor(r).reshape(-1)
    hkv = logical.shape[1]
    hs = torch.arange(hkv) if kv_heads is None else torch.tensor(kv_heads)
    n = page.numel()
    pd, rd, hd = page.to(DEV)[:, None], r.to(DEV)[:, None], hs.to(DEV)[None, :]
    logical[pd, hd, 0, rd] = decoy_k(u, n)[:, hs.to(DEV)]
    logical[pd, hd, 1, rd] = decoy_v(n, hkv)[:, hs.to(DEV)]
    mod[page[:, None], hs[None, :], r[:, None]] = True


def last_page_tails(pt, lens):
    """(pages, slots) of the unused slots in each sequence's last page."""
    pages, slots = [], []
    for i, l in enumerate(lens):
        for r in range(l % PAGE, PAGE if l % PAGE else 0):
            pages.append(int(pt[i, (l - 1) // PAGE]))
            slots.append(r)
    return pages, slots


def decode_case(lens, hq, hkv, share, seed):
    """Per-slot K/V (slots longer than `share` pages share those pages), queries for rows mapped
    to slots in reverse order."""
    torch.manual_seed(seed)
    kp = bf(torch.randn(share * PAGE, hkv, HD, device=DEV))
    vp = bf(torch.randn(share * PAGE, hkv, HD, device=DEV))
    ks, vs = [], []
    for l in lens:
        k = bf(torch.randn(l, hkv, HD, device=DEV))
        v = bf(torch.randn(l, hkv, HD, device=DEV))
        if share and l > share * PAGE:
            k[:share * PAGE], v[:share * PAGE] = kp, vp
        ks.append(k)
        vs.append(v)
    B = len(lens)
    row_slot = list(range(B - 1, -1, -1))
    ctx = [lens[s] for s in row_slot]
    return ks, vs, row_slot, ctx


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [2])      # the warp-per-(sequence, kv head) kernel
@pytest.mark.parametrize("hq,hkv", HEADS, ids=HEAD_IDS)
def test_decode_masked_slots_do_not_leak(hq, hkv, variant):
    G = hq // hkv
    lens = [1, 15, 16, 17, 33, 100, 129, 255, 256, 257, 600, 47]
    ks, vs, row_slot, ctx = decode_case(lens, hq, hkv, share=2, seed=20 + G)
    logical, pt, decoy_page, spare = paged_cache(ks, vs, share=2, seed=G)
    u = torch.randn(hkv, HD, device=DEV)
    qkv = queries(len(lens), hq, hkv, u)

    def run():
        return run_decode(qkv, KV.pack_tile(logical), pt, row_slot, ctx, hq, hkv)

    def unchanged(mod):
        m = torch.ones(len(lens), hq, dtype=torch.bool)
        for b, s in enumerate(row_slot):
            m[b] = (first_touched(mod, pt[s], ctx[b]) == ctx[b]).repeat_interleave(G)
        return m

    base = run()
    logical[spare] = float("nan")
    assert torch.equal(run(), base)
    saved = logical.clone()
    fresh = lambda: torch.zeros(logical.shape[0], hkv, PAGE, dtype=torch.bool)
    mod = fresh()
    paged_decoys(logical, u, mod, [decoy_page] * PAGE, list(range(PAGE)))
    check_unchanged(run(), base, unchanged(fresh()), "page-table entries past the last page")
    logical.copy_(saved)
    mod = fresh()
    paged_decoys(logical, u, mod, *last_page_tails(pt, lens))
    check_unchanged(run(), base, unchanged(mod), "slots at or after ctx_len")
    logical.copy_(saved)
    if hkv > 1:
        mod = fresh()
        n_pg = logical.shape[0]
        paged_decoys(logical, u, mod, torch.arange(n_pg).repeat_interleave(PAGE),
                     torch.arange(PAGE).repeat(n_pg), kv_heads=[hkv - 1])
        check_unchanged(run(), base, unchanged(mod), "last kv head")
        logical.copy_(saved)
    # the own (unshared) pages of slot 10, and one position in the middle of slot 9
    mod = fresh()
    pages = pt[10, 2:(lens[10] + PAGE - 1) // PAGE]
    paged_decoys(logical, u, mod, pages.repeat_interleave(PAGE), torch.arange(PAGE).repeat(len(pages)))
    paged_decoys(logical, u, mod, int(pt[9, 100 // PAGE]), 100 % PAGE)
    check_unchanged(run(), base, unchanged(mod), "pages of slots 9 and 10")


# --------------------------------------------------------------------------- 2. pointer attention
EDGES = (0, 15, 16, 31, 32, 127, 128, 255, 256)


class PointerQueries:
    """Targets and query vectors of one launch.  A few probed (token, head) pairs also get a decoy
    channel c (dim 64 + c of the query, unique in the launch): a key that carries the same channel
    scores D^2 = 1600 for that query only, above the target's 2A^2 = 800."""

    def __init__(self, hq, hkv, seed):
        self.hq, self.hkv, self.G = hq, hkv, hq // hkv
        self.rng = random.Random(seed)
        self.tgt = []          # per query row: [hq] absolute target positions
        self.probes = []       # (row, head, channel)

    def add_row(self, vis_end, edges, probe):
        """A query row that sees positions [0, vis_end]; probe: give one head a channel."""
        row = []
        for kvh in range(self.hkv):
            cand = pointer_candidates(vis_end, edges, self.G, self.rng)
            off = self.rng.randrange(len(cand))
            row += [cand[(off + h) % len(cand)] for h in range(self.G)]
        self.tgt.append(row)
        if probe:
            c = len(self.probes)
            assert c < HD - 64
            self.probes.append((len(self.tgt) - 1, len(self.tgt) % self.hq, c))
            return c
        return None

    def q(self):
        """[rows, hq, 128] fp32 (host)."""
        t = torch.tensor(self.tgt)
        kvh = torch.arange(self.hq) // self.G
        q = kv_address(t.reshape(-1), 0).view(len(self.tgt), self.hq, HD)
        for h in range(self.hq):   # address in the permutation of the head's kv head
            q[:, h] = kv_address(t[:, h], int(kvh[h]))
        for row, h, c in self.probes:
            q[row, h, 64 + c] = D_PTR
        return q


def qkv_rows(q, hkv):
    """q [rows, hq, 128] -> bf16 qkv rows with zero k/v columns."""
    rows, hq = q.shape[:2]
    x = torch.zeros(rows, (hq + 2 * hkv) * HD)
    x[:, :hq * HD] = q.reshape(rows, -1)
    return bf(x).to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("hq,hkv", HEADS, ids=HEAD_IDS)
def test_dense_prefill_pointer_is_exact(hq, hkv):
    """Targets at key 0, prefix row past-1, own row 0, the diagonal and the 15/16, 31/32,
    127/128 and 255/256 boundaries; decoys right after the diagonal and at prefix row `past`."""
    G, P, prefix_rows, t_pad = hq // hkv, 257, 300, 40
    specs = [(P, 260), (0, 300), (P, 1), (0, 33), (P, 129)]
    q_start, T = starts(specs)
    gen = torch.Generator().manual_seed(30 + G)
    pq = PointerQueries(hq, hkv, seed=G)
    probe_at = []
    for s, (p, n) in enumerate(specs):
        edges = EDGES + (p - 1, p)
        for t in range(n):
            c = pq.add_row(p + t, edges + (p + t,), probe=t in (0, 15, 31, 127, n - 1))
            if c is not None:
                probe_at.append((s, t, pq.probes[-1][1] // G, c))
    # keys: prefix row r holds position r, own row i of sequence s holds position past_s + i
    kv = torch.zeros(T + t_pad, 2 * hkv, HD)
    pre = torch.zeros(2, prefix_rows, 2 * hkv, HD)
    for h in range(hkv):
        pre[1, :, h] = kv_address(torch.arange(prefix_rows), h)
        for s, (p, n) in enumerate(specs):
            kv[q_start[s]:q_start[s] + n, h] = kv_address(p + torch.arange(n), h)
        kv[T:, h] = kv_address(torch.arange(t_pad) + 500, h)
    kv[:, hkv:] = pointer_value(T + t_pad, hkv, gen).float()
    pre[1, :, hkv:] = pointer_value(prefix_rows, hkv, gen).float()
    for s, t, h, c in probe_at:
        kv[q_start[s] + t + 1, h, 64 + c] = D_PTR          # the key right after the diagonal
        if specs[s][0] > 0 and t == specs[s][1] - 1:
            pre[1, specs[s][0], h, 64 + c] = D_PTR         # the first prefix row not in its past
    kv[T + 31:] = float("nan")                             # out of every box's reach
    pre[1, P + 31:] = float("nan")
    pre[0] = float("nan")                                  # another layer
    qkv = qkv_rows(pq.q(), hkv)
    qkv = torch.cat([qkv, torch.zeros(t_pad, qkv.shape[1], dtype=qkv.dtype, device=DEV)])
    qkv[:, hq * HD:] = bf(kv.reshape(T + t_pad, -1)).to(DEV)
    pre_d = bf(pre.reshape(2, prefix_rows, -1)).to(DEV)
    out = run_dense(qkv, pre_d, prefix_rows, 2, 1, specs, hq, hkv)
    # expected: V of the target position
    v_all = torch.cat([pre[1, :, hkv:], kv[:T, hkv:]])    # [prefix_rows + T, hkv, 128]
    tgt = torch.tensor(pq.tgt)
    idx = torch.empty_like(tgt)
    for s, (p, n) in enumerate(specs):
        blk = tgt[q_start[s]:q_start[s] + n]
        idx[q_start[s]:q_start[s] + n] = torch.where(blk < p, blk, prefix_rows + q_start[s] + blk - p)
    want = bf(v_all[idx, (torch.arange(hq) // G)[None, :]]).to(DEV)
    bad = (out != want).any(-1).nonzero()
    assert bad.numel() == 0, (len(bad), bad[:8].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [2])      # the warp-per-(sequence, kv head) kernel
@pytest.mark.parametrize("hq,hkv", HEADS, ids=HEAD_IDS)
def test_decode_pointer_is_exact(hq, hkv, variant):
    """Targets at the edges and at L-1; three pages of shared prefix, rows mapped to slots in
    reverse order, a decoy in the slot right after L-1 and in the page past the last one."""
    G = hq // hkv
    lens = [1, 2, 16, 17, 33, 49, 64, 129, 256, 257, 300, 600, 1000]
    share = 3
    gen = torch.Generator().manual_seed(50 + G)
    B = len(lens)
    row_slot = list(range(B - 1, -1, -1))
    ctx = [lens[s] for s in row_slot]
    pq = PointerQueries(hq, hkv, seed=200 + G)
    for b in range(B):
        pq.add_row(ctx[b] - 1, EDGES + (ctx[b] - 1,), probe=True)
    shared_v = pointer_value(share * PAGE, hkv, gen)
    ks, vs = [], []
    for l in lens:
        ks.append(bf(torch.stack([kv_address(torch.arange(l), h) for h in range(hkv)], 1)))
        v = pointer_value(l, hkv, gen)
        if l > share * PAGE:
            v[:share * PAGE] = shared_v
        vs.append(v)
    logical, pt, decoy_page, _ = paged_cache(ks, vs, share=share, seed=G)
    for row, head, c in pq.probes:
        s, l, h = row_slot[row], ctx[row], head // G
        if l % PAGE:
            logical[int(pt[s, l // PAGE]), h, 0, l % PAGE, 64 + c] = D_PTR
    logical[decoy_page, :, 0, :, 64:] = D_PTR
    out = run_decode(qkv_rows(pq.q(), hkv), KV.pack_tile(logical), pt, row_slot, ctx, hq, hkv)
    tgt = torch.tensor(pq.tgt)
    want = torch.stack([vs[row_slot[b]][tgt[b], torch.arange(hq) // G] for b in range(B)])
    bad = (out != want.to(DEV)).any(-1).nonzero()
    assert bad.numel() == 0, (len(bad), bad[:8].tolist())


# --------------------------------------------------------------------------- 3. numerics
RAMP_LOG2_PER_BLOCK = 12.0   # > the dense kernel's lazy-rescale threshold of 8 log2 units


def add_ramp(k, pos):
    """With q[..., 0] = 4, k[..., 0] = g * pos makes the scores rise by RAMP_LOG2_PER_BLOCK every
    128 keys, so a row's running maximum jumps past the rescale threshold block after block."""
    g = RAMP_LOG2_PER_BLOCK / 128 / (4 * SCALE / math.log(2))
    k[..., 0] = (g * pos.float().to(k.device))[:, None]


def dense_random(hq, hkv, specs, prefix_rows, seed, gain=1.0, ramp=False):
    """Random bf16 qkv (+ 32 zero rows) and prefix buffers; -> qkv, pre, (ref, mag)."""
    torch.manual_seed(seed)
    q_start, T = starts(specs)
    ldq = (hq + 2 * hkv) * HD
    x = torch.randn(T + 32, ldq, device=DEV)
    x[T:] = 0
    x[:, :hq * HD] *= gain
    pre = torch.randn(1, max(prefix_rows, 1), 2 * hkv * HD, device=DEV)
    if ramp:
        x[:, :hq * HD].view(-1, hq, HD)[..., 0] = 4.0
        add_ramp(pre[0, :, :hkv * HD].view(-1, hkv, HD), torch.arange(pre.shape[1]))
        for s, (p, n) in enumerate(specs):
            add_ramp(x[q_start[s]:q_start[s] + n, hq * HD:(hq + hkv) * HD].view(n, hkv, HD),
                     p + torch.arange(n))
    qkv, pre = bf(x), bf(pre)
    refs, mags = [], []
    for s, (p, n) in enumerate(specs):
        rows = qkv[q_start[s]:q_start[s] + n].view(n, hq + 2 * hkv, HD)
        k = torch.cat([pre[0, :p, :hkv * HD].view(p, hkv, HD), rows[:, hq:hq + hkv]])
        v = torch.cat([pre[0, :p, hkv * HD:].view(p, hkv, HD), rows[:, hq + hkv:]])
        r, m = attn_ref64(rows[:, :hq], k, v, p + 1 + torch.arange(n), hkv)
        refs.append(r)
        mags.append(m)
    return qkv, pre, (torch.cat(refs), torch.cat(mags))


DENSE_LONG = [(0, 4096), (1000, 3073), (1000, 129), (0, 641), (1000, 15), (0, 401), (1000, 31),
              (0, 161), (1000, 383)]
DENSE_MIX = [(0, 2049), (997, 1025), (0, 15), (997, 145), (0, 287), (997, 33), (0, 127),
             (997, 513), (0, 129)]                        # lengths = 1, 15, 17, 31, 33, 127, 129 mod 128
RAMP_SPECS = [(0, 4096), (1000, 1025), (1000, 33)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,hq,hkv,specs,gain,ramp", [pytest.param(*c, id=c[0]) for c in (
    ("G1", 8, 8, DENSE_MIX, 1.0, False),
    ("G2", 16, 8, DENSE_MIX, 1.0, False),
    ("G4-long", 32, 8, DENSE_LONG, 1.0, False),
    ("G8", 16, 2, DENSE_MIX, 1.0, False),
    ("G4-rescale", 32, 8, RAMP_SPECS, 3.0, True),
    ("G8-rescale", 16, 2, RAMP_SPECS, 3.0, True),
)])
def test_dense_prefill_error_bound(case, hq, hkv, specs, gain, ramp):
    prefix_rows = max(p for p, _ in specs) + 32
    qkv, pre, (ref, mag) = dense_random(hq, hkv, specs, prefix_rows, seed=len(case) + hq,
                                        gain=gain, ramp=ramp)
    out = run_dense(qkv, pre, prefix_rows, 1, 0, specs, hq, hkv)
    assert_within_bound(out, ref, mag, f"dense prefill {case}")


@pytest.mark.gpu
@pytest.mark.parametrize("hq,hkv", HEADS, ids=HEAD_IDS)
def test_decode_error_bound(hq, hkv):
    """Contexts up to 4096 over hundreds of rows (256 at the real models' shape)."""
    B = 256 if hq == 32 else 64
    g = torch.Generator().manual_seed(hq + hkv)
    fixed = [1, 15, 16, 17, 129, 2048, 4095, 4096]
    lens = fixed + torch.randint(1, 4097, (B - len(fixed),), generator=g).tolist()
    ks, vs, row_slot, ctx = decode_case(lens, hq, hkv, share=4, seed=70 + hq)
    logical, pt, _, _ = paged_cache(ks, vs, share=4, seed=hkv)
    pool = KV.pack_tile(logical)
    del logical
    qkv = bf(torch.randn(B, (hq + 2 * hkv) * HD, device=DEV))
    refs = [attn_ref64(qkv[b:b + 1, :hq * HD].view(1, hq, HD), ks[s], vs[s], [ctx[b]], hkv)
            for b, s in enumerate(row_slot)]
    ref, mag = torch.cat([r for r, _ in refs]), torch.cat([m for _, m in refs])
    out = run_decode(qkv, pool, pt, row_slot, ctx, hq, hkv)
    assert_within_bound(out, ref, mag, f"decode G{hq // hkv}")


# --------------------------------------------------------------------------- 4. fused QKV epilogue
def rope_tables(max_pos=4096, theta=1e6):
    inv = 1.0 / (theta ** (torch.arange(0, HD, 2, dtype=torch.float32) / HD))
    fr = torch.arange(max_pos, dtype=torch.float32)[:, None] * inv[None, :]
    return bf(fr.cos()).to(DEV), bf(fr.sin()).to(DEV)


def fused_qkv(a, m, w, qn, kn, cos, sin, tok_slot, tok_pos, pt, pool, hq, hkv, block_n, out):
    d_slot, d_pos, d_pt = i32(tok_slot), i32(tok_pos), i32(pt)
    L.check(L.lib().sb200_gemm_qkv_rope(
        L.ptr(a), a.shape[0], L.ptr(w), L.ptr(out), m, a.shape[1], block_n, L.ptr(qn), L.ptr(kn),
        L.ptr(cos), L.ptr(sin), L.ptr(d_slot), L.ptr(d_pos), L.ptr(d_pt), pt.shape[1],
        L.ptr(pool), hq, hkv, 1e-6, L.current_stream()))
    torch.cuda.synchronize()


# every head layout the engine serves: tiny-qwen3 / tiny-llama, tiny-qwen3-g4, qwen-3-0.6b and the
# embedding model, qwen-3-4b and llama-3.1-8b.  At hkv = 2 one 512-wide tile holds K and V.
SERVED_HEADS = [(4, 2), (8, 2), (16, 8), (32, 8)]
SERVED_HEAD_IDS = ["4_2", "8_2", "16_8", "32_8"]
_TABLES = {}


def model_rope_tables(name):
    """The engine's bf16 cos/sin tables of a real model at all 32,768 positions, on the GPU."""
    if name not in _TABLES:
        _TABLES[name] = tuple(t.to(DEV) for t in MS.rope_tables(MS.get_spec(name), KV.MAX_POS))
    return _TABLES[name]


@pytest.mark.gpu
@pytest.mark.parametrize("M", [77, 129, 300])
@pytest.mark.parametrize("qk_norm", [True, False], ids=["qk_norm", "no_norm"])
@pytest.mark.parametrize("block_n", [0, 128, 256, 512])
@pytest.mark.parametrize("hq,hkv", SERVED_HEADS, ids=SERVED_HEAD_IDS)
def test_qkv_epilogue_dense_kv_copy(hq, hkv, block_n, qk_norm, M):
    """Small-integer A and W make the projection exact.  The k/v columns of the output must be
    bit-identical to what the same launch wrote into the pool, V must be bf16(A Wv^T), Q and K
    must match linear -> bf16 -> RMSNorm -> RoPE bit for bit, at positions up to 32,767 with the
    tables of qwen-3-4b (with the norm) or llama-3.1-8b (without); with the norm, an output whose
    normed operand (dim i or i + 64) is tied may take either rounding of it (bf16_ref: the
    epilogue rounds x * rstd to bf16 and then uses exact bf16x2 products, so the window of the
    fp32 sum of squares and rsqrtf is all that matters).  Output rows >= M, pool slots no token
    maps to and the sentinel page every other page-table entry points at stay untouched.  K < 2,048
    and one tile per CTA: the consumer warpgroups run the epilogue math."""
    K, extra = 256, 40
    N = (hq + 2 * hkv) * HD
    torch.manual_seed(M + block_n + int(qk_norm) + hq + hkv)
    a = bf(torch.randint(-2, 3, (M + extra, K), device=DEV).float())
    w = bf(torch.randint(-1, 2, (N, K), device=DEV).float())
    qn = bf(torch.rand(HD, device=DEV) + 0.5) if qk_norm else None
    kn = bf(torch.rand(HD, device=DEV) + 0.5) if qk_norm else None
    cos, sin = model_rope_tables("qwen-3-4b" if qk_norm else "llama-3.1-8b")
    n_slots = 4
    tok_slot, tok_pos = KV.long_positions(M, n_slots, seed=M + hq)
    assert set(KV.EDGE_POSITIONS) <= set(tok_pos.tolist())
    assert (tok_pos >= 4096).float().mean() > 0.5
    pt, num_pages, sentinel = KV.sparse_page_table(tok_slot, tok_pos, n_slots, seed=M + block_n)
    pool = torch.full((num_pages, hkv, 2, PAGE, HD), -3.0, dtype=torch.bfloat16, device=DEV)
    out = torch.full((M + extra, N), 7.0, dtype=torch.bfloat16, device=DEV)
    fused_qkv(a, M, w, qn, kn, cos, sin, tok_slot, tok_pos, pt, pool, hq, hkv, block_n, out)

    lin = bf(a[:M].float() @ w.float().t()).view(M, hq + 2 * hkv, HD)   # exact, then rounded
    got = out[:M].view(M, hq + 2 * hkv, HD)
    assert torch.all(out[M:] == 7.0), "rows >= M written"
    logical = KV.unpack_tile(pool)
    page, r = pt[tok_slot, tok_pos // PAGE].to(DEV), (tok_pos % PAGE).to(DEV)
    written = torch.zeros(num_pages, PAGE, dtype=torch.bool, device=DEV)
    written[page, r] = True
    assert torch.all(logical.permute(0, 3, 1, 2, 4)[~written] == -3.0), "unmapped pool slots written"
    assert not written[sentinel].any() and torch.all(logical[sentinel] == -3.0), "sentinel written"
    assert torch.equal(got[:, hq:hq + hkv], logical[page, :, 0, r]), "dense K != paged K"
    assert torch.equal(got[:, hq + hkv:], logical[page, :, 1, r]), "dense V != paged V"
    assert torch.equal(got[:, hq + hkv:], lin[:, hq + hkv:]), "V != bf16(A Wv^T)"

    pos = tok_pos.to(DEV)
    for name, sl, nw in (("q", slice(0, hq), qn), ("k", slice(hq, hq + hkv), kn)):
        cands, tied = R.normed_rope_candidates(lin[:, sl], nw, 1e-6, R.QKV_NORM_DEPTH, cos[pos],
                                               sin[pos])
        R.assert_one_of(got[:, sl], cands, name)
        if qk_norm:
            print(f"[ties] fused QKV {hq}/{hkv} {name} M={M} block_n={block_n}: "
                  f"{tied.double().mean().item():.2e} tied")
            assert tied.double().mean().item() < 0.01, name


@pytest.mark.gpu
@pytest.mark.parametrize("hq,hkv", [(32, 8), (16, 2)], ids=["G4", "G8"])
def test_fused_qkv_into_dense_prefill(hq, hkv):
    """The engine's prefill chain: fused QKV (norm + RoPE, dense K/V copy) -> dense prefill
    attention, against an fp64 attention over the K/V the same launch wrote to the pool."""
    specs = [(0, 300), (0, 129), (0, 77), (0, 1)]
    q_start, T = starts(specs)
    K = 512
    N = (hq + 2 * hkv) * HD
    torch.manual_seed(hq)
    a = bf(torch.randn(T + 32, K, device=DEV))
    w = bf(torch.randn(N, K, device=DEV) / math.sqrt(K))
    qn = bf(torch.rand(HD, device=DEV) + 0.5)
    kn = bf(torch.rand(HD, device=DEV) + 0.5)
    cos, sin = rope_tables(4096)
    tok_slot = torch.cat([torch.full((n,), s) for s, (_, n) in enumerate(specs)])
    tok_pos = torch.cat([torch.arange(n) for _, n in specs])
    max_pages = 32
    pt = torch.randperm(len(specs) * max_pages + 8)[:len(specs) * max_pages].view(-1, max_pages)
    pool = torch.zeros(len(specs) * max_pages + 8, hkv, 2, PAGE, HD, dtype=torch.bfloat16,
                       device=DEV)
    qkv = torch.zeros(T + 32, N, dtype=torch.bfloat16, device=DEV)   # the engine zeroes it too
    fused_qkv(a, T, w, qn, kn, cos, sin, tok_slot, tok_pos, pt, pool, hq, hkv, 0, qkv)
    out = run_dense(qkv, None, 0, 1, 0, specs, hq, hkv)
    logical = KV.unpack_tile(pool)
    refs = []
    for s, (_, n) in enumerate(specs):
        p = torch.arange(n)
        k = logical[pt[s, p // PAGE].to(DEV), :, 0, (p % PAGE).to(DEV)]
        v = logical[pt[s, p // PAGE].to(DEV), :, 1, (p % PAGE).to(DEV)]
        q = qkv[q_start[s]:q_start[s] + n, :hq * HD].view(n, hq, HD)
        refs.append(attn_ref64(q, k, v, 1 + p, hkv))
    assert_within_bound(out, torch.cat([r for r, _ in refs]), torch.cat([m for _, m in refs]),
                        f"fused QKV -> dense prefill G{hq // hkv}")
