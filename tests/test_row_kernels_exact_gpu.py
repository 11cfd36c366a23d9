"""Row kernels (norm_rope.cu) bit for bit, at the model widths and head counts.

- RMSNorm at every register-resident instance (NV = 4, 10, 16), the two-pass one (long rows and
  every in-place call) and partial last vectors, on rows whose mean squares span 2^-40 (eps
  dominates) to 2^40, plus an all-zero row.
- The stand-alone RoPE/KV write at 12 to 64 heads per token (one to four passes of 16 heads),
  with and without q/k-norm, Qwen and llama-scaled tables, positions up to 32,767, shuffled
  2,049-entry page tables and a sentinel-filled pool.
- Embedding gathers from full-size tables, and the embedding head's L2 normalisation.

Rounding follows bf16_ref: every element must equal the fp64 reference rounded at the kernel's
rounding points, except where a pre-rounding value lies within the derived window of a bf16
midpoint; there either neighbour is accepted.  Rows, outputs and pool slots a launch must not
touch are sentinel-filled and checked, and every buffer has room for a whole partial CTA or page
past what the launch covers.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import bf16_ref as R
import kv_layout as KV
from sutro_b200 import _lib as L
from sutro_b200 import modelspec as MS

DEV = "cuda"
HD, PAGE = KV.HD, KV.PAGE
LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sutro_b200",
                   "libsutro_b200.so")
TIED_LIMIT = 0.01   # largest accepted fraction of tied elements (about 0.3 % at d = 5120)


def bf(x):
    return x.to(torch.bfloat16)


def i32(x):
    return torch.as_tensor(x, dtype=torch.int32).to(DEV)


def launch(name, *args):
    L.check(getattr(L.lib(), name)(*args, L.current_stream()))
    torch.cuda.synchronize()


# --------------------------------------------------------------------------- CPU self-check
def f32(x):
    return np.asarray(x, dtype=np.float32)


def perturb_ulps(x, k, rng):
    """fp32 x moved by k ulps, up or down at random (the worst case of a k-ulp intrinsic)."""
    x = f32(x)
    step = np.where(rng.random(x.shape) < 0.5, -1, 1).astype(np.int64) * np.asarray(k, np.int64)
    return (x.view(np.int32).astype(np.int64) + step).astype(np.int32).view(np.float32)


def bf16_rne(x):
    """fp32 -> nearest bf16 (ties to even), as fp32."""
    b = f32(x).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32)


def emulate_rms_scale(x, lanes, offsets, eps, rng):
    """fp32 x * rstd in a kernel's order.  lanes: [n_lanes, pairs, 2] dims summed by each lane as
    `ss += a*a + b*b` (-1 = padding), then one xor-butterfly level per offset; rsqrtf off by
    2 ulp."""
    xp = np.concatenate([x, np.zeros((x.shape[0], 1), np.float32)], 1)   # index -1 -> 0
    sq = xp * xp                                           # exact: bf16 squares
    ss = np.zeros((x.shape[0], lanes.shape[0]), np.float32)
    for p in range(lanes.shape[1]):
        ss = f32(ss + f32(sq[:, lanes[:, p, 0]] + sq[:, lanes[:, p, 1]]))
    for o in offsets:
        ss = f32(ss + ss[:, np.arange(lanes.shape[0]) ^ o])
    t = f32(f32(ss[:, :1] / np.float32(x.shape[1])) + np.float32(eps))
    rstd = perturb_ulps(1.0 / np.sqrt(t.astype(np.float64)), 2, rng)
    return f32(x * rstd)


def rms_lanes(d):
    vec = np.arange(32)[:, None] + 32 * np.arange((d // 8 + 31) // 32)[None, :]   # [lane, k]
    dims = vec[..., None] * 8 + np.arange(8)                                    # [lane, k, 8]
    dims = np.where(vec[..., None] < d // 8, dims, -1)
    return dims.reshape(32, -1, 2), (16, 8, 4, 2, 1)


def rope_lanes():
    l = np.arange(16)[:, None]
    pairs = np.stack([4 * l + np.arange(4), 64 + 4 * l + np.arange(4)], -1)     # [16, 4, 2]
    return pairs, (8, 4, 2, 1)


def qkv_lanes():
    q = np.arange(4)[:, None]
    lo = 8 * np.arange(16)[None, :] + 2 * q
    return np.stack([lo, lo + 1], -1), (1, 2)                                   # [4, 16, 2]


def test_tie_windows_cover_emulated_kernels():
    """numpy emulation of the fp32 order of rmsnorm_kernel, rope_kv_kernel's q/k-norm, the QKV
    epilogue's q/k-norm (rsqrtf 2 ulp off) and the SwiGLU epilogue's SiLU (__expf at its
    documented worst error, over every bf16 |g| < 88.7): every element outside
    bf16_ref's window rounds to what the reference says, and the windows stay narrow."""
    rng = np.random.default_rng(0)
    worst = 0.0
    cases = [(d, rms_lanes(d), R.rmsnorm_depth(d)) for d in (128, 1032, 2568, 4104, 5120)]
    cases += [(HD, rope_lanes(), R.ROPE_NORM_DEPTH), (HD, qkv_lanes(), R.QKV_NORM_DEPTH)]
    for d, (lanes, offsets), depth in cases:
        assert sum(offsets) == lanes.shape[0] - 1
        assert sorted(lanes[lanes >= 0].tolist()) == list(range(d))    # every dim exactly once
        for eps in (1e-6, 1e-5):
            rows = 400
            scale = 2.0 ** rng.integers(-20, 21, (rows, 1))
            x = bf(torch.from_numpy(rng.standard_normal((rows, d)) * scale)).float().numpy()
            y32 = emulate_rms_scale(x, lanes, offsets, eps, rng)
            x64 = torch.from_numpy(x).double()
            eps32 = float(np.float32(eps))
            y = x64 * torch.rsqrt(x64.square().mean(-1, keepdim=True) + eps32)
            near, _, tied = R.bf16_window(y, R.rms_delta(depth))
            got = torch.from_numpy(bf16_rne(y32)).double()
            assert torch.equal(got[~tied], near[~tied]), (d, eps)
            rel = ((torch.from_numpy(y32).double() - y).abs() / y.abs()).nan_to_num(0)
            worst = max(worst, (rel / R.rms_delta(depth)).max().item())
            assert tied.double().mean().item() < TIED_LIMIT, (d, tied.double().mean().item())
    assert worst <= 1.0
    print(f"[ties] RMSNorm emulation: largest error / window {worst:.3f}")

    g16 = np.arange(0, 1 << 16, dtype=np.uint32) << 16
    g = g16.view(np.float32)
    # beyond, exp(-g) overflows (g < 0: the result is -0) or 1 + exp(-g) rounds to 1 (s = g)
    g = g[np.isfinite(g) & (np.abs(g) < R.LN_FLT_MAX)]
    e = perturb_ulps(np.exp(-g.astype(np.float64)), np.floor(2 + 1.173 * np.abs(g)), rng)
    s = bf16_rne(f32(g / f32(np.float32(1.0) + e)))
    near, _, tied = R.silu_ref(torch.from_numpy(g.copy()).to(torch.bfloat16))
    assert torch.equal(torch.from_numpy(s)[~tied], near.float()[~tied])
    assert tied.double().mean().item() < TIED_LIMIT
    print(f"[ties] SiLU emulation over {g.size} bf16 values: {tied.double().mean().item():.2e} "
          f"tied")
    # past the overflow point F.silu gives -0, and so must the reference
    gneg = torch.tensor([-89.0, -1000.0, -88.5]).to(torch.bfloat16)
    near, _, _ = R.silu_ref(gneg)
    assert R.bits(near)[:2].tolist() == [-32768, -32768] and near[2].item() < 0


def test_bf16_window_rounds_to_nearest_even():
    y = torch.tensor([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 1.0 + 2 ** -9, -0.0, 0.0, 3.0 + 2 ** -30],
                     dtype=torch.float64)
    near, far, tied = R.bf16_window(y, 0.0)
    assert near.tolist() == [1.0, 1.0 + 4 * 2 ** -8, 1.0, 0.0, 0.0, 3.0]
    assert tied.tolist() == [True, True, False, False, False, False]
    assert far.tolist()[:2] == [1.0 + 2 ** -7, 1.0 + 2 * 2 ** -8]
    assert torch.signbit(near[3]) and not torch.signbit(near[4])
    assert torch.equal(near, y.to(torch.bfloat16).double())


@pytest.mark.skipif(not os.path.exists(LIB), reason="library not built")
def test_rope_kv_write_rejects_more_than_64_heads():
    """The head count is checked before any CUDA call, so this needs no GPU."""
    lib = ctypes.CDLL(LIB)
    lib.sb200_last_error.restype = ctypes.c_char_p
    rc = lib.sb200_rope_kv_write(None, None, None, None, None, None, None, None, 1, None, 1, 49, 8,
                                 ctypes.c_float(1e-6), None)
    assert rc == -1
    assert lib.sb200_last_error().decode() == \
        "rope_kv_write: at most 64 heads (q+k+v) per token, got 65"


# --------------------------------------------------------------------------- RMSNorm
RMS_WIDTHS = [128, 1024, 1032, 2560, 2568, 4096, 4104, 5120]
ROW_COUNTS = (1, 3, 5, 4097)
SPARE_ROWS = 8       # past `rows`: more than a partial 4-row CTA can reach
EXPS = list(range(-20, 21, 5))      # element scale 2^e: mean squares 2^-40 .. 2^40


def scaled_rows(rows, d, gen):
    """[rows, d] bf16; row i is N(0, 1) * 2^EXPS[i % 9], and the middle row (rows >= 3) is 0."""
    e = torch.tensor([EXPS[i % len(EXPS)] for i in range(rows)], device=DEV, dtype=torch.float32)
    x = torch.randn(rows, d, generator=gen, device=DEV) * torch.exp2(e)[:, None]
    if rows >= 3:
        x[rows // 2] = 0
    return bf(x)


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [1e-6, 1e-5])
@pytest.mark.parametrize("in_place", [False, True], ids=["out_of_place", "in_place"])
@pytest.mark.parametrize("d", RMS_WIDTHS)
def test_rmsnorm_exact(d, in_place, eps):
    """d = 128 .. 1024: NV = 4; 1032 .. 2560: NV = 10; 2568 .. 4096: NV = 16; 4104, 5120 and every
    in-place call: the two-pass kernel.  1032, 2568 and 4104 end in a partial last vector."""
    gen = torch.Generator(device=DEV).manual_seed(d * 3 + int(in_place))
    w = bf(torch.randn(d, generator=gen, device=DEV))
    depth = R.rmsnorm_depth(d)
    tied_n = total = 0
    for rows in ROW_COUNTS:
        x = torch.cat([scaled_rows(rows, d, gen),
                       bf(torch.randn(SPARE_ROWS, d, generator=gen, device=DEV))])
        if in_place:
            out = x.clone()
            launch("sb200_rmsnorm", L.ptr(out), L.ptr(w), L.ptr(out), rows, d, eps)
            spare = x[rows:]
        else:
            out = torch.full_like(x, -7.0)
            launch("sb200_rmsnorm", L.ptr(x), L.ptr(w), L.ptr(out), rows, d, eps)
            spare = torch.full_like(x[rows:], -7.0)
        near, far, tied = R.rmsnorm_ref(x[:rows], w, eps, depth)
        R.assert_one_of(out[:rows], [near, far], f"rmsnorm d={d} rows={rows}")
        assert torch.equal(R.bits(out[rows:]), R.bits(spare)), f"rows >= {rows} written"
        if rows >= 3:
            assert torch.all(out[rows // 2] == 0)
        tied_n += tied.sum().item()
        total += tied.numel()
    frac = tied_n / total
    print(f"[ties] rmsnorm d={d} {'in place' if in_place else 'out of place'} eps={eps}: "
          f"{frac:.2e} tied (window {R.rms_delta(depth):.2e})")
    assert frac < TIED_LIMIT


# --------------------------------------------------------------------------- RoPE / KV write
ROPE_HEADS = [(8, 2), (16, 8), (32, 8), (48, 8)]   # 12, 32, 48, 64 heads: 1 .. 4 passes of 16


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["qwen-3-4b", "llama-3.1-8b"])
@pytest.mark.parametrize("qk_norm", [True, False], ids=["qk_norm", "no_norm"])
@pytest.mark.parametrize("hq,hkv", ROPE_HEADS)
def test_rope_kv_write_exact(hq, hkv, qk_norm, model):
    """Q in place and K in the pool equal the op-by-op RoPE of the (q/k-normed) heads at
    positions up to 32,767 (the model's 32,768-row tables, the engine's 2,049-entry page table),
    the dense K columns equal the pool's K, V in the pool is a bit copy of the input, and pool
    slots no token maps to keep their sentinel, as does the page every unmapped entry points at."""
    spec = MS.get_spec(model)
    nh = hq + 2 * hkv
    T, n_slots, max_pages = 150, 3, KV.MAX_PAGES
    torch.manual_seed(nh * 2 + int(qk_norm) + len(model))
    tok_slot, tok_pos = KV.long_positions(T, n_slots, seed=nh + len(model))
    assert set(KV.EDGE_POSITIONS) <= set(tok_pos.tolist())
    assert (tok_pos >= 4096).float().mean() > 0.5
    pt, num_pages, sentinel = KV.sparse_page_table(tok_slot, tok_pos, n_slots, seed=nh)
    cos, sin = (t.to(DEV) for t in MS.rope_tables(spec, KV.MAX_POS))
    qkv = bf(torch.randn(T, nh * HD, device=DEV) * 3)
    qn = bf(torch.randn(HD, device=DEV)) if qk_norm else None
    kn = bf(torch.randn(HD, device=DEV)) if qk_norm else None
    pool = torch.full((num_pages, hkv, 2, PAGE, HD), -3.0, dtype=torch.bfloat16, device=DEV)
    orig = qkv.clone()
    d_slot, d_pos, d_pt = i32(tok_slot), i32(tok_pos), i32(pt)
    launch("sb200_rope_kv_write", L.ptr(qkv), L.ptr(qn), L.ptr(kn), L.ptr(cos),
           L.ptr(sin), L.ptr(d_slot), L.ptr(d_pos), L.ptr(d_pt), max_pages, L.ptr(pool),
           T, hq, hkv, spec.rms_eps)

    x = orig.view(T, nh, HD)
    got = qkv.view(T, nh, HD)
    pos = tok_pos.to(DEV)
    logical = KV.unpack_tile(pool)
    page, r = pt[tok_slot, tok_pos // PAGE].to(DEV), (tok_pos % PAGE).to(DEV)
    pool_k, pool_v = logical[page, :, 0, r], logical[page, :, 1, r]      # [T, hkv, 128]
    tied_n = 0
    for name, sl, nw, res in (("q", slice(0, hq), qn, got[:, :hq]),
                              ("k", slice(hq, hq + hkv), kn, pool_k)):
        cands, tied = R.normed_rope_candidates(x[:, sl], nw, spec.rms_eps, R.ROPE_NORM_DEPTH,
                                               cos[pos], sin[pos])
        R.assert_one_of(res, cands, f"{name} {hq}/{hkv}")
        tied_n += tied.sum().item()
    assert torch.equal(R.bits(got[:, hq:hq + hkv]), R.bits(pool_k)), "dense K != pool K"
    assert torch.equal(R.bits(pool_v), R.bits(x[:, hq + hkv:])), "pool V != input V"
    assert torch.equal(R.bits(got[:, hq + hkv:]), R.bits(x[:, hq + hkv:])), "dense V changed"
    written = torch.zeros(num_pages, PAGE, dtype=torch.bool, device=DEV)
    written[page, r] = True
    assert torch.all(logical.permute(0, 3, 1, 2, 4)[~written] == -3.0), "unmapped pool slots written"
    assert not written[sentinel].any() and torch.all(logical[sentinel] == -3.0), "sentinel written"
    frac = tied_n / (T * (hq + hkv) * HD)
    print(f"[ties] rope_kv_write {hq}/{hkv} {model} qk_norm={qk_norm}: {frac:.2e} tied")
    assert frac < TIED_LIMIT


# --------------------------------------------------------------------------- gathers
@pytest.mark.gpu
@pytest.mark.parametrize("vocab,d", [(151936, 2560), (128256, 4096), (151936, 1032)])
def test_embed_gather_exact(vocab, d):
    """Full-size tables; ids include 0, vocab - 1 and repeats; 1003 rows end in a partial CTA."""
    gen = torch.Generator(device=DEV).manual_seed(d)
    table = torch.randn(vocab, d, generator=gen, device=DEV, dtype=torch.bfloat16)
    rows = 1003
    ids = torch.randint(0, vocab, (rows,), generator=gen, device=DEV, dtype=torch.int32)
    ids[:6] = torch.tensor([0, vocab - 1, 0, vocab - 1, 17, 17], dtype=torch.int32)
    ids[-1] = vocab - 1
    out = torch.full((rows + SPARE_ROWS, d), -7.0, dtype=torch.bfloat16, device=DEV)
    launch("sb200_embed_gather", L.ptr(ids), L.ptr(table), L.ptr(out), rows, d)
    assert torch.equal(R.bits(out[:rows]), R.bits(table[ids.long()]))
    assert torch.all(out[rows:] == -7.0), "rows past `rows` written"


def l2_delta(d):
    """Relative bound of l2norm_kernel: the sum of squares runs through d/64 + 1 + 5 roundings
    (lane-strided bf16 pairs, 5 butterfly levels); sqrtf, 1 / x and x * inv round once each:
    ((d/64 + 6) / 2 + 3) u.  Doubled for safety."""
    return ((d + 63) // 64 + 6 + 6) * R.U32


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1024, 2560, 4096, 1032])
def test_l2_normalize_rows(d):
    """fp32 x / max(||x||, 1e-12) against fp64, element by element.  Row 0 is zero (zeros out),
    row 1 has a norm below 1e-12 (x * 1e12, as torch.nn.functional.normalize gives)."""
    gen = torch.Generator(device=DEV).manual_seed(d)
    rows = 1001
    x = scaled_rows(rows, d, gen)
    x[0] = 0
    x[1] = bf(torch.randn(d, generator=gen, device=DEV) * 2.0 ** -48)
    out = torch.full((rows + SPARE_ROWS, d), -7.0, device=DEV)
    launch("sb200_l2_normalize_rows", L.ptr(x), L.ptr(out), rows, d)
    x64 = x.double()
    norm = x64.norm(dim=-1, keepdim=True)
    assert norm[1].item() < 1e-12
    ref = x64 / norm.clamp_min(1e-12)
    assert torch.all(out[0] == 0)
    ratio = ((out[:rows].double() - ref).abs() / (l2_delta(d) * ref.abs()))
    ratio = torch.where(ref == 0, torch.where(out[:rows] == 0, 0.0, float("inf")), ratio)
    print(f"[l2norm] d={d}: largest error / bound {ratio.max().item():.3f}")
    assert ratio.max().item() <= 1.0
    tiny = torch.nn.functional.normalize(x[1:2].float(), dim=-1)
    assert torch.allclose(out[1:2], tiny, rtol=l2_delta(d), atol=0)
    assert torch.all(out[rows:] == -7.0), "rows past `rows` written"
