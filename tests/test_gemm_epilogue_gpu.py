"""The GEMM's fused epilogues, bit for bit.

The residual epilogue (D = bf16(bf16(acc) + R)) loads R for a chunk of columns before it stores
any of them, with the row and column masks applied to the loads as well as the stores; the SwiGLU
epilogue pairs interleaved gate/up columns across lanes and stores N/2 columns.  These tests cover
the tails those masks guard (M not a multiple of the 128-row tile, M < 128, N not a multiple of
the tile width), every tile width, the in-place form the engine uses and an out-of-place
residual, and that no output row >= M is written.

Small-integer operands make every partial sum exact in fp32, so the epilogues are compared bit
for bit with a plain fp32 matmul plus the documented bf16 rounding (SiLU under bf16_ref's tie
rule).  On random data at the models' projection shapes, the STORE_F32 output of the same launch
shape is the accumulator the other epilogues round (one mainloop, and every tile width
accumulates in the same order), so each epilogue is checked bit for bit against the rounding of
that accumulator, and the accumulator itself against fp64.
"""
import math

import pytest
import torch

import bf16_ref as R
from sutro_b200 import _lib as L

pytestmark = pytest.mark.gpu

DEV = "cuda"
STORE_BF16, RESIDUAL_BF16, SWIGLU_BF16, STORE_F32 = 0, 1, 2, 3
BLOCK_NS = [64, 128, 256, 512]


def bf(x):
    return x.to(torch.bfloat16)


def ints(rows, cols, lo=-2, hi=3):
    return bf(torch.randint(lo, hi, (rows, cols), device=DEV).float())


def tiles(m):
    """Rows of an output buffer: whole 128-row tiles, so a kernel that ignored M would write
    into the buffer's own sentinel rows and never past it."""
    return (m + 127) // 128 * 128


def gemm(a, w, epi, m, block_n, resid=None, out=None):
    N, K = w.shape
    if out is None:
        cols = N // 2 if epi == SWIGLU_BF16 else N
        out = torch.full((tiles(m), cols), 7.0, device=DEV,
                         dtype=torch.float32 if epi == STORE_F32 else torch.bfloat16)
    L.check(L.lib().sb200_gemm_bf16_tn(L.ptr(a), a.shape[0], L.ptr(w), L.ptr(out), L.ptr(resid),
                                       m, N, K, out.shape[1], epi, block_n, L.current_stream()))
    torch.cuda.synchronize()
    return out


def interleave(wg, wu):
    """Gate/up weights as the SwiGLU epilogue takes them: row 2j is gate j, row 2j + 1 is up j."""
    return torch.stack([wg, wu], dim=1).reshape(2 * wg.shape[0], wg.shape[1]).contiguous()


def swiglu_cands(a, wg, wu):
    g = bf(a.float() @ wg.float().t())
    u = bf(a.float() @ wu.float().t())
    return R.swiglu_ref(g, u)


@pytest.mark.parametrize("block_n", BLOCK_NS)
@pytest.mark.parametrize("epi", [STORE_BF16, RESIDUAL_BF16, SWIGLU_BF16, STORE_F32])
@pytest.mark.parametrize("M", [300, 77, 129])
def test_row_and_column_tails_are_exact(M, epi, block_n):
    """M = 300 ends in a partial row tile, M = 77 is a single partial tile, M = 129 leaves one
    row in the second tile; N = 352 is not a multiple of any tile width (for SwiGLU: 2F = 352).
    A has exactly M rows; the output has whole tiles, and its rows >= M keep their sentinel."""
    torch.manual_seed(M * 10 + epi)
    N, K = 32 * 11, 448
    a = ints(M, K)
    if epi == SWIGLU_BF16:
        wg, wu = ints(N // 2, K), ints(N // 2, K)
        out = gemm(a, interleave(wg, wu), epi, M, block_n)
        cands, _ = swiglu_cands(a, wg, wu)
        R.assert_one_of(out[:M], cands, f"swiglu M={M} block_n={block_n}")
        assert torch.all(out[M:] == 7.0), "rows >= M written"
        return
    w = ints(N, K)
    acc = a.float() @ w.float().t()
    if epi == STORE_F32:
        out = gemm(a, w, epi, M, block_n)
        assert torch.equal(out[:M], acc)
    elif epi == STORE_BF16:
        out = gemm(a, w, epi, M, block_n)
        assert torch.equal(out[:M], bf(acc))
    else:
        r = ints(tiles(M), N, -64, 65)
        out = r.clone()
        gemm(a, w, epi, M, block_n, resid=out, out=out)   # in place, as the engine runs it
        assert torch.equal(out[:M], bf(bf(acc).float() + r[:M].float()))
        assert torch.equal(out[M:], r[M:]), "rows >= M written"
        return
    assert torch.all(out[M:] == 7.0), "rows >= M written"


@pytest.mark.parametrize("block_n", BLOCK_NS)
@pytest.mark.parametrize("M", [300, 77])
def test_residual_out_of_place_leaves_rows_past_m_untouched(M, block_n):
    """The residual is read from its own buffer, A has rows past M (a_rows > M), and no output
    row >= M is written."""
    torch.manual_seed(M + block_n)
    N, K = 480, 256
    a, w = ints(1024, K), ints(N, K)
    r = ints(1024, N, -64, 65)
    out = torch.full((1024, N), 7.0, dtype=torch.bfloat16, device=DEV)
    gemm(a, w, RESIDUAL_BF16, M, block_n, resid=r, out=out)
    acc = a[:M].float() @ w.float().t()
    assert torch.equal(out[:M], bf(bf(acc).float() + r[:M].float()))
    assert torch.all(out[M:] == 7.0)


# --------------------------------------------------------------------------- random data
def check_against_f32(a, w, epi, m, block_n=0, resid=None):
    """Run `epi` and STORE_F32 on the same A, W, M (so the same tile shape and accumulation
    order), check the epilogue bit for bit against the rounding of the fp32 accumulator, and
    return that accumulator [m, N].  resid: [tiles(m), N] bf16, updated in place."""
    acc_full = gemm(a, w, STORE_F32, m, block_n)
    acc = acc_full[:m]
    assert torch.all(acc_full[m:] == 7.0), "STORE_F32 wrote rows >= M"
    what = f"epi {epi} M={m} N={w.shape[0]} K={w.shape[1]}"
    if epi == STORE_BF16:
        out = gemm(a, w, epi, m, block_n)
        assert torch.equal(R.bits(out[:m]), R.bits(bf(acc))), what
    elif epi == RESIDUAL_BF16:
        r = resid.clone()
        gemm(a, w, epi, m, block_n, resid=resid, out=resid)
        assert torch.equal(R.bits(resid[:m]), R.bits(bf(bf(acc).float() + r[:m].float()))), what
        assert torch.equal(R.bits(resid[m:]), R.bits(r[m:])), "rows >= M written"
        return acc
    else:
        out = gemm(a, w, epi, m, block_n)
        cands, tied = R.swiglu_ref(bf(acc[:, 0::2]), bf(acc[:, 1::2]))
        R.assert_one_of(out[:m], cands, what)
        frac = tied.double().mean().item()
        print(f"[ties] swiglu M={m} 2F={w.shape[0]} K={w.shape[1]}: {frac:.2e} tied")
        assert frac < 0.01
    assert torch.all(out[m:] == 7.0), "rows >= M written"
    return acc


def assert_f32_within_bound(acc, a, w, what):
    ref, bound = R.gemm_f32_bound(a, w)
    ratio = ((acc.double() - ref).abs() / bound).max().item()
    print(f"[gemm f32] {what}: largest |acc - fp64| / bound {ratio:.2e} (c = {R.GEMM_C})")
    assert ratio <= 1.0, (what, ratio)


# (N, K, epilogue): gate/up (interleaved, 2F columns) and O / down with residual, for qwen-3-4b
# (d_model 2560, 32 q heads, d_ff 9728) and llama-3.1-8b (4096, 32, 14336)
PROJECTIONS = {
    "qwen4b-gate-up": (2 * 9728, 2560, SWIGLU_BF16),
    "qwen4b-o": (2560, 4096, RESIDUAL_BF16),
    "qwen4b-down": (2560, 9728, RESIDUAL_BF16),
    "llama8b-gate-up": (2 * 14336, 4096, SWIGLU_BF16),
    "llama8b-o": (4096, 4096, RESIDUAL_BF16),
    "llama8b-down": (4096, 14336, RESIDUAL_BF16),
}
PROJ_M = (1, 17, 200, 3584, 4096)


@pytest.mark.parametrize("name", list(PROJECTIONS))
def test_epilogues_round_the_f32_accumulator(name):
    """Random bf16 data at the models' projection shapes: STORE_BF16 == bf16(acc), RESIDUAL ==
    bf16(bf16(acc) + R) and SwiGLU under the tie rule, bit for bit against the STORE_F32 output of
    the same launch shape; that accumulator within the fp64 bound of bf16_ref.gemm_f32_bound."""
    N, K, epi = PROJECTIONS[name]
    gen = torch.Generator(device=DEV).manual_seed(N + K)
    w = bf(torch.randn(N, K, generator=gen, device=DEV) / math.sqrt(K))
    for m in PROJ_M:
        a = bf(torch.randn(m, K, generator=gen, device=DEV))
        resid = bf(torch.randn(tiles(m), N, generator=gen, device=DEV))
        check_against_f32(a, w, STORE_BF16, m)
        acc = check_against_f32(a, w, epi, m, resid=resid)
        assert_f32_within_bound(acc, a, w, f"{name} M={m}")


@pytest.mark.parametrize("N,K", [(151936, 2560), (128256, 4096)], ids=["qwen", "llama"])
def test_lm_head_f32_against_fp64(N, K):
    """The LM heads (STORE_F32 logits) at decode-sized M, against fp64."""
    gen = torch.Generator(device=DEV).manual_seed(N)
    w = bf(torch.randn(N, K, generator=gen, device=DEV) / math.sqrt(K))
    for m in (1, 17, 200):
        a = bf(torch.randn(m, K, generator=gen, device=DEV))
        acc = gemm(a, w, STORE_F32, m, 0)
        assert torch.all(acc[m:] == 7.0)
        assert_f32_within_bound(acc[:m], a, w, f"lm head N={N} M={m}")
