"""Attention kernels at a GQA group of 5 (qwen-3-14b's 40 query heads over 8 KV heads, and the
tiny test model's 10 over 2).

A prefill q tile then holds QT = 25 tokens x 5 heads in 125 of its 128 wgmma rows.  Three things
differ from the other group sizes, and each has a check here:
- the Q tile's TMA boxes deliver 32,000 bytes, not 32 KiB;
- rows 125-127 are padding: their token index is 25, the first token of the NEXT q tile, so an
  item that stored them would overwrite another item's output.  Each work item is launched alone
  into a sentinel-filled output, and exactly its own tokens may change;
- q tiles start at multiples of 25, so a tile's causal frontier can fall anywhere inside a
  128-token KV block (asserted: some tiles straddle two blocks).
The masked-row, pointer, fp64-bound, invariance and fused-QKV checks of the other group sizes run
here unchanged at both G = 5 head layouts, through the functions of their own test modules.
"""
import pytest
import torch

import test_attention_exact_gpu as AX
import test_gemm_epilogue_warps_gpu as EW
import test_long_context_gpu as LC
import test_prefill_attention_widths_gpu as PW
from sutro_b200 import _lib as L

pytestmark = pytest.mark.gpu

DEV = "cuda"
HD = AX.HD
G5_HEADS = [(40, 8), (10, 2)]
G5_IDS = ["40_8", "10_2"]
QT = 25


def test_q_tile_is_25():
    assert L.lib().sb200_attn_prefill_q_tile(40, 8) == QT
    assert L.lib().sb200_attn_prefill_q_tile(10, 2) == QT


# --------------------------------------------------------------------------- prefill
@pytest.mark.parametrize("hq,hkv", G5_HEADS, ids=G5_IDS)
def test_dense_prefill_masked_rows_do_not_leak(hq, hkv):
    AX.test_dense_prefill_masked_rows_do_not_leak(hq, hkv)


@pytest.mark.parametrize("hq,hkv", G5_HEADS, ids=G5_IDS)
def test_dense_prefill_pointer_is_exact(hq, hkv):
    AX.test_dense_prefill_pointer_is_exact(hq, hkv)


def residue_specs():
    """Own lengths covering every residue mod 25 and 127/128/129/255/256/257, with prefixes of 0,
    15, 16, 17, 46 and 1,000 tokens in turn."""
    lens = [25 * (1 + (7 * r) % 11) + r for r in range(QT)] + [127, 128, 129, 255, 256, 257]
    prefixes = [0, 15, 16, 17, 46, 1000]
    return [(prefixes[i % len(prefixes)], n) for i, n in enumerate(lens)]


def straddling_tiles(specs):
    """(sequence, t0) of the q tiles whose tokens lie in two 128-token KV blocks."""
    return [(s, t0) for s, (_, n) in enumerate(specs) for t0 in range(0, n, QT)
            if t0 // 128 != (min(t0 + QT, n) - 1) // 128]


@pytest.mark.parametrize("hq,hkv", G5_HEADS, ids=G5_IDS)
def test_dense_prefill_error_bound(hq, hkv):
    specs = residue_specs()
    assert {n % QT for _, n in specs} == set(range(QT))
    assert {p for p, _ in specs} == {0, 15, 16, 17, 46, 1000}
    straddle = straddling_tiles(specs)
    assert len(straddle) >= 10, straddle
    prefix_rows = 1000 + 32
    qkv, pre, (ref, mag) = AX.dense_random(hq, hkv, specs, prefix_rows, seed=hq + 5)
    out = AX.run_dense(qkv, pre, prefix_rows, 1, 0, specs, hq, hkv)
    AX.assert_within_bound(out, ref, mag, f"dense prefill G5 {hq}/{hkv}")
    # the straddling tiles on their own, so a wrong frontier cannot hide in the mean
    q_start, _ = AX.starts(specs)
    rows = torch.tensor(sorted({q_start[s] + t for s, t0 in straddle
                                for t in range(t0, min(t0 + QT, specs[s][1]))}))
    AX.assert_within_bound(out[rows.to(DEV)], ref[rows.to(ref.device)], mag[rows.to(mag.device)],
                           f"dense prefill G5 {hq}/{hkv}, tiles across a KV block")


def test_dense_prefill_rescale_error_bound():
    AX.test_dense_prefill_error_bound("G5-rescale", 40, 8, AX.RAMP_SPECS, 3.0, True)


@pytest.mark.parametrize("own,past", [(32768, 0), (32768, 777)])
def test_dense_prefill_long_rows_within_fp64_bound(own, past):
    LC.test_dense_prefill_long_rows_within_fp64_bound(40, 8, own, past)


@pytest.mark.parametrize("hq,hkv", G5_HEADS, ids=G5_IDS)
def test_each_item_writes_only_its_own_tokens(hq, hkv):
    """Every work item launched alone into an output full of a sentinel: exactly the item's own
    tokens (up to 25) x all query heads change, and they equal the full launch's bits."""
    specs = [(46, 130), (0, 77), (17, 26), (0, 51), (1000, 300)]
    q_start, T = AX.starts(specs)
    prefix_rows = 1000 + 32
    qkv, pre, _ = AX.dense_random(hq, hkv, specs, prefix_rows, seed=hq * 3 + hkv)
    items = [(s, t0) for s, (_, n) in enumerate(specs) for t0 in range(0, n, QT)]
    d_qs = AX.i32(q_start)
    d_ql, d_past = AX.i32([n for _, n in specs]), AX.i32([p for p, _ in specs])
    sentinel = -12345.0

    def launch(item_list):
        out = torch.full((qkv.shape[0], hq * HD), sentinel, dtype=torch.bfloat16, device=DEV)
        d_items = AX.i32([x for it in item_list for x in it])
        L.check(L.lib().sb200_attn_prefill_dense(
            L.ptr(qkv), qkv.shape[0], L.ptr(out), L.ptr(pre), prefix_rows, 1, 0, L.ptr(d_items),
            len(item_list), L.ptr(d_qs), L.ptr(d_ql), L.ptr(d_past), hq, hkv, AX.SCALE,
            L.current_stream()))
        torch.cuda.synchronize()
        return out

    full = launch(items)
    assert not (full[:T] == sentinel).any()
    assert (full[T:] == sentinel).all()
    for s, t0 in items:
        out = launch([(s, t0)])
        changed = (out != sentinel).view(-1, hq, HD).any(-1)          # [rows, hq]
        want = torch.zeros_like(changed)
        r0, r1 = q_start[s] + t0, q_start[s] + min(t0 + QT, specs[s][1])
        want[r0:r1] = True
        assert torch.equal(changed, want), (s, t0, changed.nonzero()[:8].tolist())
        assert torch.equal(out[r0:r1], full[r0:r1]), (s, t0)


@pytest.mark.parametrize("past", PW.PREFIXES)
@pytest.mark.parametrize("hq,hkv", G5_HEADS, ids=G5_IDS)
def test_cut_sequences_are_bit_identical(hq, hkv, past):
    PW.test_cut_sequences_are_bit_identical(hq, hkv, past)


@pytest.mark.parametrize("hq,hkv", G5_HEADS, ids=G5_IDS)
def test_item_order_and_launch_split_do_not_matter(hq, hkv):
    PW.test_item_order_and_launch_split_do_not_matter(hq, hkv)


# --------------------------------------------------------------------------- decode
@pytest.mark.parametrize("hq,hkv", G5_HEADS, ids=G5_IDS)
def test_decode_masked_slots_do_not_leak(hq, hkv):
    AX.test_decode_masked_slots_do_not_leak(hq, hkv, 2)


@pytest.mark.parametrize("hq,hkv", G5_HEADS, ids=G5_IDS)
def test_decode_pointer_is_exact(hq, hkv):
    AX.test_decode_pointer_is_exact(hq, hkv, 2)


@pytest.mark.parametrize("hq,hkv", G5_HEADS, ids=G5_IDS)
def test_decode_error_bound(hq, hkv):
    AX.test_decode_error_bound(hq, hkv)


G5_DECODE_LENS = [1, 16, 17, 4095, 4096, 4097, 8193, 32768]


@pytest.mark.parametrize("hq,hkv", G5_HEADS, ids=G5_IDS)
def test_split_decode_within_fp64_bound_and_no_leaks(hq, hkv):
    """Single-split rows and split-KV rows in one launch; decoys past each context and NaN pages
    past each row's last page must not leak."""
    lens = G5_DECODE_LENS
    pool, pt, ks, vs = LC.paged_rows(lens, hkv, seed=hq + 5 * hkv)
    rows = list(range(len(lens)))
    torch.manual_seed(hq + 1)
    qkv = AX.bf(torch.randn(len(rows), (hq + 2 * hkv) * HD, device=DEV))
    out = LC.decode(qkv, pool, pt, rows, lens, hq, hkv)
    for b in rows:
        ref, mag = AX.attn_ref64(qkv[b:b + 1, :hq * HD].view(1, hq, HD), ks[b], vs[b], [lens[b]],
                                 hkv)
        AX.assert_within_bound(out[b:b + 1], ref, mag, f"decode G5 {hq}/{hkv} ctx {lens[b]}")


@pytest.mark.parametrize("hq,hkv", G5_HEADS, ids=G5_IDS)
def test_split_decode_is_batch_invariant(hq, hkv):
    LC.test_split_decode_is_batch_invariant(hq, hkv)


# --------------------------------------------------------------------------- fused QKV epilogue
@pytest.mark.parametrize("M", [77, 300])
@pytest.mark.parametrize("qk_norm", [True, False], ids=["qk_norm", "no_norm"])
@pytest.mark.parametrize("block_n", [0, 128, 256, 512])
def test_qkv_epilogue_dense_kv_copy(block_n, qk_norm, M):
    """The consumer path (K = 256) at 40/8, positions up to 32,767."""
    AX.test_qkv_epilogue_dense_kv_copy(40, 8, block_n, qk_norm, M)


@pytest.mark.parametrize("qk_norm", [True, False], ids=["qk_norm", "no_norm"])
@pytest.mark.parametrize("block_n", [128, 256, 512])
def test_qkv_epilogue_warps_many_tiles(block_n, qk_norm):
    """The epilogue-warp path (K = 2,048, more tiles than SMs) at 40/8."""
    EW.test_qkv_epilogue_warps_many_tiles(40, 8, 2048, block_n, qk_norm)


def test_fused_qkv_into_dense_prefill():
    AX.test_fused_qkv_into_dense_prefill(40, 8)
