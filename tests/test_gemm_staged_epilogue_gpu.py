"""The GEMM's staged epilogues: bf16 results go through a shared-memory staging buffer and are
stored by TMA, and the residual is loaded into that buffer by TMA while the tile's mainloop runs.

These cases reach what the other epilogue tests do not: many tiles per CTA with fewer K blocks
than ring stages (so the staging buffer is reused, and a tile's residual load races the previous
tile's store, as soon as possible), an output row stride wider than N (TMA must clip at N, not at
the stride), and the fused QKV epilogue without the dense K/V copy, whose K/V columns of the
qkv buffer must stay untouched.  Small-integer operands keep every sum exact, so all checks are
bit for bit.
"""
import math
import os
import subprocess
import sys

import pytest
import torch

import bf16_ref as R
from sutro_b200 import _lib as L
from test_gemm_epilogue_gpu import (BLOCK_NS, RESIDUAL_BF16, STORE_BF16, SWIGLU_BF16, bf, gemm,
                                    interleave, ints, swiglu_cands, tiles)

pytestmark = pytest.mark.gpu

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("block_n", BLOCK_NS)
@pytest.mark.parametrize("K", [64, 128])
def test_many_tiles_per_cta_with_short_k(K, block_n):
    """129 row tiles (the last one partial) x a column tail: several tiles per CTA at every tile
    width, each with one or two K blocks, so consecutive tiles' stores, staging writes and
    in-place residual loads follow each other closely."""
    torch.manual_seed(K + block_n)
    M, N = 129 * 128 - 51, 1056
    a, w = ints(M, K), ints(N, K)
    acc = a.float() @ w.float().t()

    out = gemm(a, w, STORE_BF16, M, block_n)
    assert torch.equal(out[:M], bf(acc))
    assert torch.all(out[M:] == 7.0), "rows >= M written"

    r = ints(tiles(M), N, -64, 65)
    out = r.clone()
    gemm(a, w, RESIDUAL_BF16, M, block_n, resid=out, out=out)
    assert torch.equal(out[:M], bf(bf(acc).float() + r[:M].float()))
    assert torch.equal(out[M:], r[M:]), "rows >= M written"

    wg, wu = ints(N // 2, K), ints(N // 2, K)
    out = gemm(a, interleave(wg, wu), SWIGLU_BF16, M, block_n)
    cands, _ = swiglu_cands(a, wg, wu)
    R.assert_one_of(out[:M], cands, f"swiglu K={K} block_n={block_n}")
    assert torch.all(out[M:] == 7.0), "rows >= M written"


@pytest.mark.parametrize("block_n", BLOCK_NS)
@pytest.mark.parametrize("epi", [STORE_BF16, RESIDUAL_BF16, SWIGLU_BF16])
def test_row_stride_wider_than_n(epi, block_n):
    """ldd > N: the columns between N (N/2 for SwiGLU) and ldd, and the rows >= M, keep their
    sentinel."""
    torch.manual_seed(epi * 1000 + block_n)
    M, N, K = 300, 352, 192
    n_out = N // 2 if epi == SWIGLU_BF16 else N
    ldd = n_out + 40
    a = ints(M, K)
    out = torch.full((tiles(M), ldd), 7.0, dtype=torch.bfloat16, device=DEV)
    if epi == SWIGLU_BF16:
        wg, wu = ints(N // 2, K), ints(N // 2, K)
        gemm(a, interleave(wg, wu), epi, M, block_n, out=out)
        cands, _ = swiglu_cands(a, wg, wu)
        R.assert_one_of(out[:M, :n_out], cands, f"swiglu ldd={ldd} block_n={block_n}")
        assert torch.all(out[M:] == 7.0), "rows >= M written"
    else:
        w = ints(N, K)
        acc = a.float() @ w.float().t()
        if epi == STORE_BF16:
            gemm(a, w, epi, M, block_n, out=out)
            assert torch.equal(out[:M, :N], bf(acc))
            assert torch.all(out[M:] == 7.0), "rows >= M written"
        else:
            r = ints(tiles(M), N, -64, 65)
            out[:, :N] = r
            gemm(a, w, epi, M, block_n, resid=out, out=out)
            assert torch.equal(out[:M, :N], bf(bf(acc).float() + r[:M].float()))
            assert torch.equal(out[M:, :N], r[M:]), "rows >= M written"
    assert torch.all(out[:, n_out:] == 7.0), "columns past N written"


def test_row_stride_tma_cannot_address_is_rejected():
    """A bf16 row stride that is not a multiple of 16 bytes is reported, not run."""
    a, w = ints(64, 64), ints(64, 64)
    out = torch.zeros(64, 68, dtype=torch.bfloat16, device=DEV)
    rc = L.lib().sb200_gemm_bf16_tn(L.ptr(a), 64, L.ptr(w), L.ptr(out), 0, 64, 64, 64, 68,
                                    STORE_BF16, 0, L.current_stream())
    assert rc != 0 and b"16-byte" in L.lib().sb200_last_error()


# ----------------------------------------------------------------------- fused QKV, no dense copy
_QKV_RUN = """
import sys, torch
sys.path.insert(0, sys.argv[1])
from sutro_b200 import _lib as L
t = torch.load(sys.argv[2])
a, w, qkv, pool = t["a"].cuda(), t["w"].cuda(), t["qkv"].cuda(), t["pool"].cuda()
dev = {k: t[k].cuda() for k in ("qn", "kn", "cos", "sin", "slot", "pos", "pt")}
L.check(L.lib().sb200_gemm_qkv_rope(
    L.ptr(a), a.shape[0], L.ptr(w), L.ptr(qkv), a.shape[0], a.shape[1], t["block_n"],
    L.ptr(dev["qn"]), L.ptr(dev["kn"]), L.ptr(dev["cos"]), L.ptr(dev["sin"]), L.ptr(dev["slot"]),
    L.ptr(dev["pos"]), L.ptr(dev["pt"]), dev["pt"].shape[1], L.ptr(pool), t["hq"], t["hkv"], 1e-6,
    L.current_stream()))
torch.cuda.synchronize()
torch.save({"qkv": qkv.cpu(), "pool": pool.cpu()}, sys.argv[3])
"""


@pytest.mark.parametrize("block_n", [128, 256])
def test_qkv_without_dense_copy_leaves_kv_columns(block_n, tmp_path):
    """With SB200_QKV_DENSE=0 (read once per process, so the run is a subprocess), the q columns
    and the paged K/V equal those of the default run bit for bit, and the K/V columns of the qkv
    buffer keep their sentinel."""
    torch.manual_seed(block_n)
    hq, hkv, T, K = 6, 2, 333, 320
    N = (hq + 2 * hkv) * 128
    n_slots, max_pages, num_pages = 4, 12, 60
    inv = 1.0 / (1e6 ** (torch.arange(0, 128, 2, dtype=torch.float32) / 128))
    fr = torch.arange(256, dtype=torch.float32)[:, None] * inv[None, :]
    t = {
        "a": ints(T, K).cpu(), "w": bf(torch.randn(N, K) / math.sqrt(K)),
        "qkv": torch.full((T, N), 7.0, dtype=torch.bfloat16),
        "pool": torch.zeros(num_pages, hkv, 2, 16, 128, dtype=torch.bfloat16),
        "qn": bf(torch.rand(128) + 0.5), "kn": bf(torch.rand(128) + 0.5),
        "cos": bf(fr.cos()), "sin": bf(fr.sin()),
        "slot": torch.arange(T, dtype=torch.int32) % n_slots,
        "pos": torch.arange(T, dtype=torch.int32) // n_slots + 5,
        "pt": torch.randperm(num_pages)[: n_slots * max_pages].view(n_slots, max_pages)
                   .to(torch.int32),
        "block_n": block_n, "hq": hq, "hkv": hkv,
    }
    src, dst = tmp_path / "in.pt", tmp_path / "out.pt"
    torch.save(t, src)
    env = dict(os.environ, SB200_QKV_DENSE="0")
    flags = ["-s"] if sys.flags.no_user_site else []
    subprocess.run([sys.executable, *flags, "-c", _QKV_RUN, ROOT, str(src), str(dst)], env=env,
                   check=True, timeout=600)
    got = torch.load(dst)

    qkv, pool = t["qkv"].to(DEV), t["pool"].to(DEV)
    dev = {k: t[k].to(DEV) for k in ("a", "w", "qn", "kn", "cos", "sin", "slot", "pos", "pt")}
    L.check(L.lib().sb200_gemm_qkv_rope(
        L.ptr(dev["a"]), T, L.ptr(dev["w"]), L.ptr(qkv), T, K, block_n, L.ptr(dev["qn"]),
        L.ptr(dev["kn"]), L.ptr(dev["cos"]), L.ptr(dev["sin"]), L.ptr(dev["slot"]),
        L.ptr(dev["pos"]), L.ptr(dev["pt"]), max_pages, L.ptr(pool), hq, hkv, 1e-6,
        L.current_stream()))
    torch.cuda.synchronize()
    qkv, pool = qkv.cpu(), pool.cpu()
    assert torch.equal(R.bits(got["qkv"][:, :hq * 128]), R.bits(qkv[:, :hq * 128]))
    assert torch.all(got["qkv"][:, hq * 128:] == 7.0), "K/V columns written without dense copy"
    assert not torch.all(qkv[:, hq * 128:] == 7.0), "the default run writes the dense K/V"
    assert torch.equal(R.bits(got["pool"]), R.bits(pool))
