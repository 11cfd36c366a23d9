"""Edges of the GEMM's fused epilogues, bit for bit.

The residual epilogue (D = bf16(bf16(acc) + R)) loads R for a chunk of columns before it stores
any of them, with the row and column masks applied to the loads as well as the stores.  These
tests cover the tails those masks guard (M not a multiple of the 128-row tile, M < 128, N not a
multiple of the tile width), every tile width, the in-place form the engine uses and an
out-of-place residual, and that no output row >= M is written.

Small-integer operands make every partial sum exact in fp32, so STORE_BF16, RESIDUAL_BF16 and
STORE_F32 are compared bit for bit with a plain fp32 matmul plus the documented bf16 rounding.
"""
import pytest
import torch

from sutro_b200 import _lib as L

pytestmark = pytest.mark.gpu

DEV = "cuda"
STORE_BF16, RESIDUAL_BF16, STORE_F32 = 0, 1, 3
BLOCK_NS = [64, 128, 256, 512]


def bf(x):
    return x.to(torch.bfloat16)


def ints(rows, cols, lo=-2, hi=3):
    return bf(torch.randint(lo, hi, (rows, cols), device=DEV).float())


def gemm(a, w, epi, m, block_n, resid=None, out=None):
    N, K = w.shape
    if out is None:
        out = torch.zeros(m, N, dtype=torch.float32 if epi == STORE_F32 else torch.bfloat16,
                          device=DEV)
    L.check(L.lib().sb200_gemm_bf16_tn(L.ptr(a), a.shape[0], L.ptr(w), L.ptr(out), L.ptr(resid),
                                       m, N, K, out.shape[1], epi, block_n, L.current_stream()))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("block_n", BLOCK_NS)
@pytest.mark.parametrize("epi", [STORE_BF16, RESIDUAL_BF16, STORE_F32])
@pytest.mark.parametrize("M", [300, 77, 129])
def test_row_and_column_tails_are_exact(M, epi, block_n):
    """M = 300 ends in a partial row tile, M = 77 is a single partial tile, M = 129 leaves one
    row in the second tile; N = 352 is not a multiple of any tile width."""
    torch.manual_seed(M * 10 + epi)
    N, K = 32 * 11, 448
    a, w = ints(M, K), ints(N, K)
    acc = a.float() @ w.float().t()
    if epi == STORE_F32:
        assert torch.equal(gemm(a, w, epi, M, block_n), acc)
    elif epi == STORE_BF16:
        assert torch.equal(gemm(a, w, epi, M, block_n), bf(acc))
    else:
        r = ints(M, N, -64, 65)
        out = r.clone()
        gemm(a, w, epi, M, block_n, resid=out, out=out)   # in place, as the engine runs it
        assert torch.equal(out, bf(bf(acc).float() + r.float()))


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
