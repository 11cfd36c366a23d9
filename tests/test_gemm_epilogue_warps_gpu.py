"""The epilogue warps of the fused GEMM (gemm_wgmma.cu): SwiGLU and QKV with many tiles per CTA.

When a launch gives a CTA more than one tile and K >= 2048, the consumer warpgroups only stage
bf16(acc) and warps 9-11 run the SwiGLU or QKV math in place in the staging slab, store it, and
hand the slab back.  Otherwise the consumers run the math themselves.  These tests drive the
hand-off hard (dozens of tiles per CTA at the shortest K that takes the path, so every slab is
reused under backpressure) and require the results of the two paths, of every tile width and of
every batch that contains a row, to be bit-identical.
"""
import math

import pytest
import torch

from sutro_b200 import _lib as L
import bf16_ref as R
import kv_layout as KV
import test_attention_exact_gpu as AX

DEV = "cuda"
HD, PAGE = KV.HD, KV.PAGE
HQ, HKV = 32, 8
N_QKV = (HQ + 2 * HKV) * HD


def bf(x):
    return x.to(torch.bfloat16)


def i32(x):
    return torch.as_tensor(x, dtype=torch.int32).to(DEV)


def rope_tables(max_pos=4096, theta=1e6):
    inv = 1.0 / (theta ** (torch.arange(0, HD, 2, dtype=torch.float32) / HD))
    fr = torch.arange(max_pos, dtype=torch.float32)[:, None] * inv[None, :]
    return bf(fr.cos()).to(DEV), bf(fr.sin()).to(DEV)


def fused_qkv(a, m, w, qn, kn, cos, sin, tok_slot, tok_pos, pt, pool, block_n, out, hq=HQ,
              hkv=HKV):
    d_slot, d_pos, d_pt = i32(tok_slot), i32(tok_pos), i32(pt)
    L.check(L.lib().sb200_gemm_qkv_rope(
        L.ptr(a), a.shape[0], L.ptr(w), L.ptr(out), m, a.shape[1], block_n, L.ptr(qn), L.ptr(kn),
        L.ptr(cos), L.ptr(sin), L.ptr(d_slot), L.ptr(d_pos), L.ptr(d_pt), pt.shape[1],
        L.ptr(pool), hq, hkv, 1e-6, L.current_stream()))
    torch.cuda.synchronize()


def token_layout(M, n_slots, seed):
    """Distinct positions < 4096 per slot; page table over a shuffled pool with spare pages."""
    g = torch.Generator().manual_seed(seed)
    tok_slot = torch.arange(M) % n_slots
    tok_pos = torch.empty(M, dtype=torch.long)
    for s in range(n_slots):
        idx = (tok_slot == s).nonzero().flatten()
        tok_pos[idx] = torch.randperm(4095, generator=g)[:len(idx)]
    tok_pos[0] = 4095
    max_pages = 4096 // PAGE
    num_pages = n_slots * max_pages + 16
    pt = torch.randperm(num_pages, generator=g)[:n_slots * max_pages].view(n_slots, max_pages)
    return tok_slot, tok_pos, pt, num_pages


@pytest.mark.gpu
@pytest.mark.parametrize("qk_norm", [True, False], ids=["qk_norm", "no_norm"])
@pytest.mark.parametrize("block_n", [128, 256, 512])
@pytest.mark.parametrize("K", [2048, 2560])
@pytest.mark.parametrize("hq,hkv", AX.SERVED_HEADS, ids=AX.SERVED_HEAD_IDS)
def test_qkv_epilogue_warps_many_tiles(hq, hkv, K, block_n, qk_norm):
    """129 row tiles (the last one 77 rows) x up to 48 column tiles over the SMs, with K = 2048
    (the shortest K that takes the epilogue warps) or 2560, at every served head layout.  Small-
    integer A and W make the projection exact (fp32 sums of integers; only the rounding to bf16
    remains), so V must be bf16(A Wv^T) and Q and K must be one of the candidates of linear ->
    bf16 -> RMSNorm -> RoPE, with the tables of qwen-3-4b (norm) or llama-3.1-8b (no norm) at
    positions up to 32,767; the dense K/V copy must equal the paged one; rows >= M, pool slots no
    token maps to and the sentinel page of the unmapped page-table entries stay untouched."""
    M, extra = 129 * 128 - 51, 40
    N = (hq + 2 * hkv) * HD
    # more tiles than SMs (even at the widest tile) and K >= 2048: the epilogue warps run
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert K >= 2048 and math.ceil(M / 128) * math.ceil(N / 512) > sms
    torch.manual_seed(K + block_n + int(qk_norm) + hq + hkv)
    a = bf(torch.randint(-2, 3, (M + extra, K), device=DEV).float())
    w = bf(torch.randint(-1, 2, (N, K), device=DEV).float())
    qn = bf(torch.rand(HD, device=DEV) + 0.5) if qk_norm else None
    kn = bf(torch.rand(HD, device=DEV) + 0.5) if qk_norm else None
    cos, sin = AX.model_rope_tables("qwen-3-4b" if qk_norm else "llama-3.1-8b")
    tok_slot, tok_pos = KV.long_positions(M, 8, seed=K + block_n)
    assert set(KV.EDGE_POSITIONS) <= set(tok_pos.tolist())
    assert (tok_pos >= 4096).float().mean() > 0.5
    pt, num_pages, sentinel = KV.sparse_page_table(tok_slot, tok_pos, 8, seed=K + hq)
    pool = torch.full((num_pages, hkv, 2, PAGE, HD), -3.0, dtype=torch.bfloat16, device=DEV)
    out = torch.full((M + extra, N), 7.0, dtype=torch.bfloat16, device=DEV)
    fused_qkv(a, M, w, qn, kn, cos, sin, tok_slot, tok_pos, pt, pool, block_n, out, hq, hkv)

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
            assert tied.double().mean().item() < 0.01, name


@pytest.mark.gpu
def test_qkv_epilogue_warps_invariant():
    """Random operands at the model's K, norm on.  A 5,000-row batch (epilogue warps) gives the
    same bits at block_n 128, 256 and 512, and the same bits as its rows run alone: 77 rows (one
    tile per CTA, so the consumers run the math) and 1,500 rows (epilogue warps again, with other
    tiles on each CTA).  A slab handed over too early or reused too soon breaks this."""
    M, K = 5000, 2560
    torch.manual_seed(5)
    a = bf(torch.randn(M, K, device=DEV))
    w = bf(torch.randn(N_QKV, K, device=DEV) / math.sqrt(K))
    qn = bf(torch.rand(HD, device=DEV) + 0.5)
    kn = bf(torch.rand(HD, device=DEV) + 0.5)
    cos, sin = rope_tables(4096)
    tok_slot, tok_pos, pt, num_pages = token_layout(M, 4, seed=11)

    def run(lo, hi, block_n):
        pool = torch.zeros(num_pages, HKV, 2, PAGE, HD, dtype=torch.bfloat16, device=DEV)
        out = torch.zeros(hi - lo, N_QKV, dtype=torch.bfloat16, device=DEV)
        fused_qkv(a[lo:hi], hi - lo, w, qn, kn, cos, sin, tok_slot[lo:hi], tok_pos[lo:hi], pt,
                  pool, block_n, out)
        logical = KV.unpack_tile(pool)
        page = pt[tok_slot[lo:hi], tok_pos[lo:hi] // PAGE].to(DEV)
        r = (tok_pos[lo:hi] % PAGE).to(DEV)
        return out, logical[page, :, :, r]

    ref_out, ref_kv = run(0, M, 128)
    for block_n in (256, 512):
        out, kv = run(0, M, block_n)
        assert torch.equal(out, ref_out), f"block_n {block_n}: qkv differs from block_n 128"
        assert torch.equal(kv, ref_kv), f"block_n {block_n}: paged K/V differs from block_n 128"
    for lo, hi in ((1234, 1234 + 77), (3000, 4500)):
        for block_n in (0, 256):
            out, kv = run(lo, hi, block_n)
            assert torch.equal(out, ref_out[lo:hi]), f"rows {lo}:{hi} alone: qkv differs"
            assert torch.equal(kv, ref_kv[lo:hi]), f"rows {lo}:{hi} alone: paged K/V differs"


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [64, 128, 256])
@pytest.mark.parametrize("K", [2048, 2560])
def test_swiglu_epilogue_warps_match_consumer_path(K, block_n):
    """SwiGLU in place in the slab, at every tile width (BLOCK_N = 64 writes 64-byte output rows
    over the 128-byte input rows).  A 40-row-tile launch with many tiles per CTA (epilogue warps)
    must equal, bit for bit, the same rows run 128 at a time (one tile per CTA: the consumers run
    the math, the path the row-kernel and epilogue tests check against the oracle)."""
    M, N = 40 * 128 - 19, 2048
    torch.manual_seed(K + block_n)
    a = bf(torch.randn(M, K, device=DEV))
    w = bf(torch.randn(N, K, device=DEV) / math.sqrt(K))
    lib = L.lib()

    def run(lo, hi):
        out = torch.full((hi - lo, N // 2), 7.0, dtype=torch.bfloat16, device=DEV)
        L.check(lib.sb200_gemm_bf16_tn(L.ptr(a[lo:hi]), hi - lo, L.ptr(w), L.ptr(out), 0, hi - lo,
                                       N, K, N // 2, 2, block_n, L.current_stream()))
        torch.cuda.synchronize()
        return out

    full = run(0, M)
    parts = torch.cat([run(lo, min(lo + 128, M)) for lo in range(0, M, 128)])
    assert torch.equal(full, parts), f"block_n {block_n}: epilogue warps != consumer epilogue"
