"""GPU parity tests for the hand-written kernels, called through the C-ABI.

Each kernel is compared with a plain PyTorch restatement of the same op (fp32
math with the bf16 rounding points documented in the kernel headers).
"""
import math

import pytest
import torch

from sutro_b200 import _lib as L
import kv_layout as KV
from test_attention_exact_gpu import assert_within_bound, attn_ref64
from test_gemm_epilogue_gpu import (RESIDUAL_BF16, STORE_BF16, SWIGLU_BF16,
                                    assert_f32_within_bound, check_against_f32, interleave, tiles)

pytestmark = pytest.mark.gpu

DEV = "cuda"


def bf(x):
    return x.to(torch.bfloat16)


def stream():
    return L.current_stream()


# --------------------------------------------------------------------------- GEMM
def _gemm(a, w, epi=0, resid=None, block_n=0, m=None, out=None):
    M = a.shape[0] if m is None else m
    N, K = w.shape
    if out is None:
        if epi == 3:
            out = torch.zeros(M, N, dtype=torch.float32, device=DEV)
        elif epi == 2:
            out = torch.zeros(M, N // 2, dtype=torch.bfloat16, device=DEV)
        else:
            out = torch.zeros(M, N, dtype=torch.bfloat16, device=DEV)
    ldd = out.shape[1]
    L.check(L.lib().sb200_gemm_bf16_tn(L.ptr(a), a.shape[0], L.ptr(w), L.ptr(out), L.ptr(resid),
                                       M, N, K, ldd, epi, block_n, stream()))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("block_n", [64, 128, 256, 512, 0])  # 512 = the widest tile
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (128, 256, 256), (300, 768, 512),
                                   (1000, 1536, 2560), (77, 32 * 11, 192)])
def test_gemm_store_bf16(M, N, K, block_n):
    """bf16(acc) bit for bit, and the accumulator within the fp64 bound."""
    torch.manual_seed(M * 7 + N + K)
    a = bf(torch.randn(M, K, device=DEV))
    w = bf(torch.randn(N, K, device=DEV) / math.sqrt(K))
    acc = check_against_f32(a, w, STORE_BF16, M, block_n)
    assert_f32_within_bound(acc, a, w, f"store_bf16 {M}x{N}x{K} block_n={block_n}")


def test_gemm_exact_integers():
    """Small-integer operands: every partial sum is exact in fp32, so the result
    must be bit-identical to the reference whatever the accumulation order."""
    M, N, K = 384, 512, 1024
    torch.manual_seed(1)
    a = bf(torch.randint(-3, 4, (M, K), device=DEV).float())
    w = bf(torch.randint(-3, 4, (N, K), device=DEV).float())
    d = _gemm(a, w, 3)
    ref = a.float() @ w.float().t()
    assert torch.equal(d, ref)


@pytest.mark.parametrize("M,N,K,epi", [
    (32768, 19456, 2560, 3),     # gate/up shape of qwen-3-4b at a full prefill step (fp32 out)
    (32768, 2560, 9728, 0),      # down projection
    (32768, 6144, 2560, 0),      # QKV
    (32768, 2560, 4096, 1),      # O projection + residual
    (3584, 2560, 9728, 1),       # decode batch: down + residual
    (3584, 19456, 2560, 0),      # decode batch: gate/up rows
    (20000, 4096, 4096, 0),      # llama-3.1-8b width, M not a multiple of the tile
])
def test_gemm_exact_integers_at_the_benchmark_shapes(M, N, K, epi):
    """The shapes that earn the roofline number (multi-group raster, many waves, K up to
    9728), on small-integer operands: every partial sum is exact in fp32, so the kernel must
    agree BIT FOR BIT with a plain fp32 matmul (+ the documented bf16 rounding points),
    whatever tile shape or raster order the launcher picked."""
    torch.manual_seed(M + N + K)
    a = bf(torch.randint(-2, 3, (M, K), device=DEV).float())
    w = bf(torch.randint(-2, 3, (N, K), device=DEV).float())
    acc = a.float() @ w.float().t()          # exact: |sum| <= 4*9728 < 2^24
    if epi == 3:
        assert torch.equal(_gemm(a, w, 3), acc)
    elif epi == 0:
        assert torch.equal(_gemm(a, w, 0), bf(acc))
    else:
        r = bf(torch.randint(-64, 65, (M, N), device=DEV).float())
        out = r.clone()
        _gemm(a, w, 1, resid=out, out=out)
        assert torch.equal(out, bf(bf(acc).float() + r.float()))
    del acc


def test_gemm_swiglu_at_the_benchmark_shape():
    """SwiGLU at a full prefill step of qwen-3-4b, bit for bit under the SiLU tie rule against
    the fp32 accumulator of the same launch shape."""
    M, F, K = 16384, 9728, 2560
    torch.manual_seed(11)
    a = bf(torch.randn(M, K, device=DEV))
    w = bf(torch.randn(2 * F, K, device=DEV) / math.sqrt(K))
    check_against_f32(a, w, SWIGLU_BF16, M)


def test_gemm_tile_configurations_are_bit_identical():
    """Batch invariance of the GEMM: the launcher picks the tile shape from M (128x64 ...
    128x256), so a row's result must not depend on that choice — every configuration
    accumulates over K in the same order (k-blocks of 64, four K=16 wgmma steps each)."""
    torch.manual_seed(21)
    M, N, K = 300, 1536, 2560
    a = bf(torch.randn(M, K, device=DEV))
    w = bf(torch.randn(N, K, device=DEV) / math.sqrt(K))
    outs = {bn: _gemm(a, w, 3, block_n=bn) for bn in (64, 128, 256, 512)}
    for bn in (128, 256, 512):
        diff = (outs[bn] != outs[64]).float().mean().item()
        assert diff == 0.0, (bn, diff, (outs[bn] - outs[64]).abs().max().item())
    # and the rows of a small batch equal the same rows inside a big one
    big = bf(torch.randn(5000, K, device=DEV))
    big[1000:1000 + M] = a
    full = _gemm(big, w, 3)
    assert torch.equal(full[1000:1000 + M], outs[64])


def test_gemm_a_rows_larger_than_m():
    M, N, K = 200, 512, 256
    torch.manual_seed(2)
    a = bf(torch.randn(1024, K, device=DEV))
    w = bf(torch.randn(N, K, device=DEV) / 16)
    out = torch.full((1024, N), 7.0, dtype=torch.bfloat16, device=DEV)
    _gemm(a, w, 0, m=M, out=out)
    ref = bf(a[:M].float() @ w.float().t())
    assert torch.allclose(out[:M].float(), ref.float(), rtol=1.6e-2, atol=1e-3)
    assert torch.all(out[M:] == 7.0)  # rows past M untouched


@pytest.mark.parametrize("epi", [1, 2])
def test_gemm_cta_pair_fused_epilogues(epi):
    """residual / SwiGLU epilogues through the widest tile at a multi-wave shape."""
    M, N, K = 1500, 5120, 1024
    torch.manual_seed(7)
    a = bf(torch.randn(M, K, device=DEV))
    w = bf(torch.randn(N, K, device=DEV) / math.sqrt(K))
    r = bf(torch.randn(tiles(M), N, device=DEV))
    check_against_f32(a, w, epi, M, block_n=512, resid=r if epi == RESIDUAL_BF16 else None)


def test_gemm_residual():
    M, N, K = 260, 768, 512
    torch.manual_seed(3)
    a = bf(torch.randn(M, K, device=DEV))
    w = bf(torch.randn(N, K, device=DEV) / math.sqrt(K))
    r = bf(torch.randn(tiles(M), N, device=DEV))
    check_against_f32(a, w, RESIDUAL_BF16, M, resid=r)  # in place, as the engine does


def test_gemm_swiglu():
    M, F, K = 300, 640, 512
    torch.manual_seed(4)
    a = bf(torch.randn(M, K, device=DEV))
    wg = bf(torch.randn(F, K, device=DEV) / math.sqrt(K))
    wu = bf(torch.randn(F, K, device=DEV) / math.sqrt(K))
    acc = check_against_f32(a, interleave(wg, wu), SWIGLU_BF16, M)
    # the accumulator's even columns are the gate projection, the odd ones the up projection
    assert_f32_within_bound(acc[:, 0::2], a, wg, "swiglu gate")
    assert_f32_within_bound(acc[:, 1::2], a, wu, "swiglu up")


def test_gemm_f32_logits_partial_n_tile():
    M, N, K = 130, 32 * 37, 320  # N not a multiple of any tile width
    torch.manual_seed(5)
    a = bf(torch.randn(M, K, device=DEV))
    w = bf(torch.randn(N, K, device=DEV) / math.sqrt(K))
    for bn in (64, 128, 256, 512):
        assert_f32_within_bound(_gemm(a, w, 3, block_n=bn), a, w, f"logits block_n={bn}")


def test_gemm_bad_shape_reports_error():
    a = bf(torch.randn(16, 48, device=DEV))
    w = bf(torch.randn(32, 48, device=DEV))
    out = torch.zeros(16, 32, dtype=torch.bfloat16, device=DEV)
    rc = L.lib().sb200_gemm_bf16_tn(L.ptr(a), 16, L.ptr(w), L.ptr(out), 0, 16, 32, 48, 32, 0, 0,
                                    stream())
    assert rc != 0 and b"unsupported shape" in L.lib().sb200_last_error()


# --------------------------------------------------------------------------- row kernels
def test_embed_gather_and_l2norm():
    torch.manual_seed(0)
    table = bf(torch.randn(1000, 256, device=DEV))
    ids = torch.randint(0, 1000, (77,), dtype=torch.int32, device=DEV)
    out = torch.empty(77, 256, dtype=torch.bfloat16, device=DEV)
    L.check(L.lib().sb200_embed_gather(L.ptr(ids), L.ptr(table), L.ptr(out), 77, 256, stream()))
    torch.cuda.synchronize()
    assert torch.equal(out, table[ids.long()])
    o32 = torch.empty(77, 256, dtype=torch.float32, device=DEV)
    L.check(L.lib().sb200_l2_normalize_rows(L.ptr(out), L.ptr(o32), 77, 256, stream()))
    torch.cuda.synchronize()
    ref = torch.nn.functional.normalize(out.float(), dim=-1)
    assert torch.allclose(o32, ref, rtol=1e-5, atol=1e-6)


# --------------------------------------------------------------------------- fused QKV
def rope_tables(max_pos, theta=1e6):
    inv = 1.0 / (theta ** (torch.arange(0, KV.HD, 2, dtype=torch.float32) / KV.HD))
    fr = torch.arange(max_pos, dtype=torch.float32)[:, None] * inv[None, :]
    return bf(fr.cos()).to(DEV), bf(fr.sin()).to(DEV)


@pytest.mark.parametrize("block_n", [128, 256, 512, 0])
@pytest.mark.parametrize("qk_norm", [True, False])
def test_gemm_qkv_rope_fused_matches_unfused(qk_norm, block_n):
    """K1+K5 fused epilogue == plain QKV GEMM followed by rope_kv_write (same rounding
    points; only the order of the per-head sum of squares differs)."""
    torch.manual_seed(5)
    hq, hkv, T, K = 6, 2, 333, 320
    N = (hq + 2 * hkv) * KV.HD
    n_slots, max_pages, num_pages = 4, 12, 60
    a = bf(torch.randn(T, K, device=DEV))
    w = bf(torch.randn(N, K, device=DEV) / math.sqrt(K))
    qn = bf(torch.rand(KV.HD, device=DEV) + 0.5) if qk_norm else None
    kn = bf(torch.rand(KV.HD, device=DEV) + 0.5) if qk_norm else None
    cos, sin = rope_tables(256)
    tok_slot = torch.arange(T, dtype=torch.int32) % n_slots
    tok_pos = (torch.arange(T, dtype=torch.int32) // n_slots) + 5
    pt = torch.randperm(num_pages)[: n_slots * max_pages].view(n_slots, max_pages).to(torch.int32)
    d_slot, d_pos, d_pt = tok_slot.to(DEV), tok_pos.to(DEV), pt.to(DEV)
    # unfused path
    qkv_a = torch.zeros(T, N, dtype=torch.bfloat16, device=DEV)
    pool_a = torch.zeros(num_pages, hkv, 2, KV.PAGE, KV.HD, dtype=torch.bfloat16, device=DEV)
    L.check(L.lib().sb200_gemm_bf16_tn(L.ptr(a), T, L.ptr(w), L.ptr(qkv_a), 0, T, N, K, N, 0, 0,
                                       stream()))
    L.check(L.lib().sb200_rope_kv_write(L.ptr(qkv_a), L.ptr(qn), L.ptr(kn), L.ptr(cos), L.ptr(sin),
                                        L.ptr(d_slot), L.ptr(d_pos), L.ptr(d_pt), max_pages,
                                        L.ptr(pool_a), T, hq, hkv, 1e-6, stream()))
    # fused path
    qkv_b = torch.zeros(T, N, dtype=torch.bfloat16, device=DEV)
    pool_b = torch.zeros_like(pool_a)
    L.check(L.lib().sb200_gemm_qkv_rope(L.ptr(a), T, L.ptr(w), L.ptr(qkv_b), T, K, block_n,
                                        L.ptr(qn), L.ptr(kn), L.ptr(cos), L.ptr(sin),
                                        L.ptr(d_slot), L.ptr(d_pos), L.ptr(d_pt), max_pages,
                                        L.ptr(pool_b), hq, hkv, 1e-6, stream()))
    torch.cuda.synchronize()
    qa, qb = qkv_a[:, :hq * KV.HD].float(), qkv_b[:, :hq * KV.HD].float()
    assert torch.allclose(qa, qb, rtol=2e-2, atol=2e-2)
    assert (qa != qb).float().mean().item() < 0.01
    assert torch.allclose(pool_a.float(), pool_b.float(), rtol=2e-2, atol=2e-2)
    assert (pool_a != pool_b).float().mean().item() < 0.01
    assert torch.equal(pool_a[:, :, 1], pool_b[:, :, 1])          # V: pure copy, bit-exact


# --------------------------------------------------------------------------- attention
@pytest.mark.parametrize("variant", [2])   # the warp-per-(sequence, kv head) kernel
@pytest.mark.parametrize("hq,hkv", [(32, 8), (16, 8), (8, 8), (16, 2)])
def test_attn_decode(hq, hkv, variant):
    torch.manual_seed(hq * 100 + hkv)
    lens = [1, 15, 16, 17, 63, 64, 65, 130, 257, 600]
    B = len(lens)
    ks = [bf(torch.randn(l, hkv, KV.HD, device=DEV)) for l in lens]
    vs = [bf(torch.randn(l, hkv, KV.HD, device=DEV)) for l in lens]
    pool, pt, max_pages = KV.build_cache(ks, vs, hkv, 200, DEV)
    qkv = bf(torch.randn(B, (hq + 2 * hkv) * KV.HD, device=DEV))
    out = torch.zeros(B, hq * KV.HD, dtype=torch.bfloat16, device=DEV)
    # rows are mapped to slots through an indirection (reverse order)
    row_slot = torch.arange(B - 1, -1, -1, dtype=torch.int32, device=DEV)
    ctx = torch.tensor([lens[B - 1 - b] for b in range(B)], dtype=torch.int32, device=DEV)
    scale = 1.0 / math.sqrt(KV.HD)
    L.check(L.lib().sb200_attn_decode(L.ptr(qkv), L.ptr(out), L.ptr(pool), L.ptr(pt), max_pages,
                                      L.ptr(row_slot), L.ptr(ctx), B, hq, hkv, scale, stream()))
    torch.cuda.synchronize()
    refs = [attn_ref64(qkv[b:b + 1, :hq * KV.HD].view(1, hq, KV.HD), ks[B - 1 - b], vs[B - 1 - b],
                       [lens[B - 1 - b]], hkv) for b in range(B)]
    assert_within_bound(out, torch.cat([r for r, _ in refs]), torch.cat([m for _, m in refs]),
                        f"decode {hq}/{hkv}")


def _dense_case(hq, hkv, specs, prefix_rows, n_layers, layer, seed, q_gain=1.0, t_pad=7):
    """Random dense qkv / prefix buffers + the (items, q_start, q_len, past) arrays of
    sb200_attn_prefill_dense.  specs: [(past, new)] per sequence."""
    torch.manual_seed(seed)
    T = sum(q for _, q in specs)
    ldq = (hq + 2 * hkv) * KV.HD
    qkv = bf(torch.randn(T + t_pad, ldq, device=DEV))
    qkv[:, :hq * KV.HD] *= q_gain
    pre = bf(torch.randn(n_layers, max(prefix_rows, 1), 2 * hkv * KV.HD, device=DEV))
    qt = L.lib().sb200_attn_prefill_q_tile(hq, hkv)
    assert qt == 128 // (hq // hkv)
    q_start, items, acc = [], [], 0
    for i, (p, q) in enumerate(specs):
        q_start.append(acc)
        acc += q
        for t0 in range(0, q, qt):
            items += [i, t0]
    return qkv, pre, q_start, items, T


def _dense_ref(qkv, pre, layer, hq, hkv, specs, q_start):
    """fp64 reference of the dense prefill attention: (ref, mag) [T, hq, 128] (see
    test_attention_exact_gpu.error_bound)."""
    refs = []
    for i, (p, q) in enumerate(specs):
        rows = qkv[q_start[i]:q_start[i] + q].view(q, hq + 2 * hkv, KV.HD)
        k = torch.cat([pre[layer, :p, :hkv * KV.HD].view(p, hkv, KV.HD), rows[:, hq:hq + hkv]])
        v = torch.cat([pre[layer, :p, hkv * KV.HD:].view(p, hkv, KV.HD), rows[:, hq + hkv:]])
        refs.append(attn_ref64(rows[:, :hq], k, v, p + 1 + torch.arange(q), hkv))
    return torch.cat([r for r, _ in refs]), torch.cat([m for _, m in refs])


@pytest.mark.parametrize("hq,hkv", [(32, 8), (16, 8), (4, 4), (16, 2)])
def test_attn_prefill_dense_tcgen05(hq, hkv):
    """K3 on wgmma: new tokens attend to [dense shared prefix | own rows] (TMA-fed wgmma,
    S/O in registers) — against an fp32 softmax(QK^T)V over the same bf16 inputs."""
    specs = [(0, 1), (0, 16), (0, 17), (0, 100), (32, 5), (32, 70), (48, 200), (3, 33),
             (46, 111), (130, 140), (200, 300), (0, 129), (1, 128)]
    n_layers, layer, prefix_rows = 3, 1, 200
    qkv, pre, q_start, items, T = _dense_case(hq, hkv, specs, prefix_rows, n_layers, layer,
                                              seed=hq * 7 + hkv)
    out = torch.zeros(T, hq * KV.HD, dtype=torch.bfloat16, device=DEV)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=DEV)
    scale = 1.0 / math.sqrt(KV.HD)
    d_items, d_qs = i32(items), i32(q_start)
    d_ql, d_past = i32([q for _, q in specs]), i32([p for p, _ in specs])
    L.check(L.lib().sb200_attn_prefill_dense(
        L.ptr(qkv), qkv.shape[0], L.ptr(out), L.ptr(pre), prefix_rows, n_layers, layer,
        L.ptr(d_items), len(items) // 2, L.ptr(d_qs), L.ptr(d_ql), L.ptr(d_past), hq, hkv, scale,
        stream()))
    torch.cuda.synchronize()
    ref, mag = _dense_ref(qkv, pre, layer, hq, hkv, specs, q_start)
    assert_within_bound(out, ref, mag, f"dense prefill {hq}/{hkv}")


def test_attn_prefill_dense_rescale_and_no_prefix():
    """Large score magnitudes force the lazy running-max rescale of the register
    accumulator O; prefix_kv may be NULL when nothing has a past."""
    hq, hkv = 8, 2
    specs = [(0, 700), (0, 260), (0, 31)]
    qkv, pre, q_start, items, T = _dense_case(hq, hkv, specs, 0, 1, 0, seed=3, q_gain=6.0)
    out = torch.zeros(T, hq * KV.HD, dtype=torch.bfloat16, device=DEV)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=DEV)
    scale = 1.0 / math.sqrt(KV.HD)
    d_items, d_qs = i32(items), i32(q_start)
    d_ql, d_past = i32([q for _, q in specs]), i32([0] * len(specs))
    L.check(L.lib().sb200_attn_prefill_dense(
        L.ptr(qkv), qkv.shape[0], L.ptr(out), None, 0, 1, 0, L.ptr(d_items), len(items) // 2,
        L.ptr(d_qs), L.ptr(d_ql), L.ptr(d_past), hq, hkv, scale, stream()))
    torch.cuda.synchronize()
    ref, mag = _dense_ref(qkv, pre, 0, hq, hkv, specs, q_start)
    assert_within_bound(out, ref, mag, "dense prefill, q_gain 6")


def test_attn_prefill_dense_is_batch_invariant():
    """A sequence's output bits do not depend on which other sequences share the launch."""
    hq, hkv = 32, 8
    specs = [(46, 111), (46, 64), (46, 150), (0, 90)]
    qkv, pre, q_start, items, T = _dense_case(hq, hkv, specs, 46, 1, 0, seed=9)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=DEV)
    scale = 1.0 / math.sqrt(KV.HD)

    def run(sel):
        qt = L.lib().sb200_attn_prefill_q_tile(hq, hkv)
        its = [x for i in sel for t0 in range(0, specs[i][1], qt) for x in (sel.index(i), t0)]
        out = torch.zeros(T, hq * KV.HD, dtype=torch.bfloat16, device=DEV)
        d_items, d_qs = i32(its), i32([q_start[i] for i in sel])
        d_ql, d_past = i32([specs[i][1] for i in sel]), i32([specs[i][0] for i in sel])
        L.check(L.lib().sb200_attn_prefill_dense(
            L.ptr(qkv), qkv.shape[0], L.ptr(out), L.ptr(pre), 46, 1, 0, L.ptr(d_items),
            len(its) // 2, L.ptr(d_qs), L.ptr(d_ql), L.ptr(d_past), hq, hkv, scale, stream()))
        torch.cuda.synchronize()
        return out
    full = run([0, 1, 2, 3])
    for i in range(4):
        alone = run([i])
        lo, hi = q_start[i], q_start[i] + specs[i][1]
        assert torch.equal(alone[lo:hi], full[lo:hi])


# --------------------------------------------------------------------------- FSM mask
def test_fsm_build_mask_matches_python_walk():
    torch.manual_seed(0)
    n_states, vocab = 5, 1000
    trans = torch.randint(-1, n_states, (n_states, 256), dtype=torch.int32)
    trans[torch.rand(n_states, 256) < 0.5] = -1
    accept = torch.tensor([0, 1, 0, 1, 0], dtype=torch.uint8)
    lens = torch.randint(0, 5, (vocab,))
    off = torch.zeros(vocab + 1, dtype=torch.int32)
    off[1:] = torch.cumsum(lens, 0)
    blob = torch.randint(0, 256, (int(off[-1]),), dtype=torch.uint8)
    eos = 7
    words = (vocab + 31) // 32
    mask = torch.zeros(n_states, words, dtype=torch.int32, device=DEV)
    d_trans, d_acc, d_blob, d_off = trans.to(DEV), accept.to(DEV), blob.to(DEV), off.to(DEV)
    L.check(L.lib().sb200_fsm_build_mask(L.ptr(d_trans), L.ptr(d_acc), n_states,
                                         L.ptr(d_blob), L.ptr(d_off), vocab, eos,
                                         L.ptr(mask), words, stream()))
    torch.cuda.synchronize()
    mask = mask.cpu()
    for s in range(n_states):
        for t in range(vocab):
            if t == eos:
                ok = bool(accept[s])
            else:
                cur, bs = s, blob[off[t]:off[t + 1]].tolist()
                for b in bs:
                    cur = int(trans[cur, b])
                    if cur < 0:
                        break
                ok = len(bs) > 0 and cur >= 0
            bit = (int(mask[s, t // 32]) >> (t % 32)) & 1
            assert bit == int(ok), (s, t)
