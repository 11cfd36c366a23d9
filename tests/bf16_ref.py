"""Test helper: exact references for kernels that round fp32 results to bf16.

Most rounding steps in the row kernels and GEMM epilogues are deterministic: a product of two
bf16 values is exact in fp32, and fp32 arithmetic followed by bf16 rounding of a sum of two bf16
values equals the correctly rounded bf16 sum (24 >= 2 * 8 + 2).  The inexact steps are the fp32
sum of squares with rsqrtf (RMSNorm) and __expf (SiLU).  For those the reference computes the
pre-rounding value y in fp64 and derives a relative bound delta on how far the kernel's fp32 value
can be from y.  When y lies within delta * |y| of a bf16 rounding midpoint it is *tied*: either
bf16 neighbour of y is accepted.  Every other element must round exactly as y does.

The bounds are first-order error analyses of the kernels' fp32 operation order, times a safety
factor of 2; test_row_kernels_exact_gpu.test_tie_windows_cover_emulated_kernels checks them
against a numpy emulation of that order with rsqrtf and __expf at their documented worst error.
"""
import torch

U32 = 2.0 ** -24          # unit roundoff of fp32
LN_FLT_MAX = 88.72283905206835   # exp(x) overflows fp32 above this


# --------------------------------------------------------------------------- rounding windows
def bf16_window(y, delta):
    """y: fp64 tensor; delta: float or tensor broadcastable to y.

    Returns (near, far, tied): near is y rounded to bf16 (to nearest, ties to even), far is the
    other bf16 neighbour of y where y is tied and equals near elsewhere; both fp64 holding bf16
    values, with y's sign (so 0 and -0 are kept apart)."""
    a = y.abs()
    _, e = torch.frexp(a)                                  # a = f * 2^e, f in [0.5, 1)
    ulp = torch.ldexp(torch.ones_like(a), (e - 8).clamp(min=-133))
    r = a / ulp                                            # exact: ulp is a power of two
    fl = torch.floor(r)
    frac = r - fl
    up = (frac > 0.5) | ((frac == 0.5) & (torch.remainder(fl, 2) == 1))
    lo, hi = fl * ulp, (fl + 1) * ulp
    near = torch.where(up, hi, lo)
    tied = ((frac - 0.5).abs() * ulp <= delta * a) & (a > 0)
    far = torch.where(tied, torch.where(up, lo, hi), near)
    return torch.copysign(near, y), torch.copysign(far, y), tied


def bits(t):
    """Raw bit patterns of a bf16 (int16) or fp32 (int32) tensor."""
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def assert_one_of(got, cands, what):
    """Every element of got must be bit-identical to the same element of one candidate."""
    g = bits(got)
    ok = torch.zeros_like(g, dtype=torch.bool)
    for c in cands:
        ok |= g == bits(c.to(got.dtype))
    if not bool(ok.all()):
        idx = (~ok).nonzero()[0].tolist()
        first = tuple(idx)
        raise AssertionError(f"{what}: {(~ok).sum().item()} of {ok.numel()} elements differ; first "
                             f"at {first}: got {got[first].item()!r}, expected one of "
                             f"{[c[first].item() for c in cands]}")


# --------------------------------------------------------------------------- RMSNorm
def rms_delta(depth):
    """Relative bound on |fp32 x * rstd - x / sqrt(mean(x^2) + eps)| for a kernel whose sum of
    squares runs through at most `depth` fp32 additions from any square to the total.

    Squares of bf16 values are exact in fp32.  A sum of nonnegative terms in which each term
    passes through at most `depth` roundings is within depth * u of the exact sum (u = 2^-24).
    Then `/ d` and `+ eps` round once each (depth + 2), the square root halves that, rsqrtf adds
    at most 2 ulp = 4u, and x * rstd rounds once more: (depth / 2 + 6) u.  Doubled for safety."""
    return (depth + 12) * U32


def rmsnorm_depth(d):
    """rmsnorm_kernel: lane l sums the squares of vectors l, l + 32, ... (8 elements each) as
    `ss += a*a + b*b`, four pairs per vector, then a 5-level xor butterfly."""
    return 4 * ((d + 255) // 256) + 1 + 5


ROPE_NORM_DEPTH = 4 + 1 + 4    # rope_kv_kernel: 4 pairs per lane of a half-warp, 4 levels
QKV_NORM_DEPTH = 16 + 1 + 2    # QKV epilogue: 16 pairs per lane of a quad, 2 levels


def rmsnorm_ref(x, w, eps, depth):
    """bf16(w * bf16(x * rsqrt(mean(x^2) + eps))) over the last dim of bf16 x.

    Returns (near, far, tied) as bf16 tensors: near from the correctly rounded inner value, far
    from its other neighbour where that value is tied (see bf16_window)."""
    x64 = x.double()
    eps32 = float(torch.tensor(eps, dtype=torch.float32))     # the kernel adds eps as fp32
    y = x64 * torch.rsqrt(x64.square().mean(-1, keepdim=True) + eps32)
    near, far, tied = bf16_window(y, rms_delta(depth))
    wf = w.float()
    # w * bf16(y) is a product of two bf16 values: exact in fp32, then rounded once
    return (wf * near.float()).to(torch.bfloat16), (wf * far.float()).to(torch.bfloat16), tied


# --------------------------------------------------------------------------- RoPE
def rope_ref(x, cos, sin):
    """x: [T, H, 128] bf16, cos/sin: [T, 64] bf16 — rotate-half RoPE, every op rounded to bf16."""
    c = torch.cat([cos, cos], -1)[:, None, :]
    s = torch.cat([sin, sin], -1)[:, None, :]
    rot = torch.cat([-x[..., 64:], x[..., :64]], -1)
    return (x * c) + (rot * s)


def normed_rope_candidates(x, w, eps, depth, cos, sin):
    """RoPE of the (optionally q/k-RMSNormed) heads x: [T, H, 128] bf16.

    Output dims i and i + 64 both depend on the normed dims i and i + 64, so where either is tied
    each combination of their two roundings is a candidate.  Returns (candidates, tied) with
    tied [T, H, 128] marking outputs that have more than one candidate."""
    if w is None:
        return [rope_ref(x, cos, sin)], torch.zeros_like(x, dtype=torch.bool)
    near, far, tied = rmsnorm_ref(x, w, eps, depth)
    cands = []
    for lo in (near, far):
        for hi in (near, far):
            cands.append(rope_ref(torch.cat([lo[..., :64], hi[..., 64:]], -1), cos, sin))
    t = tied[..., :64] | tied[..., 64:]
    return cands, torch.cat([t, t], -1)


# --------------------------------------------------------------------------- SiLU
def silu_delta(g):
    """Relative bound on |fp32 g / (1 + __expf(-g)) - silu(g)| for bf16 g (fp64 tensor).

    __expf(x) is within 2 + floor(1.173 |x|) ulp (CUDA Programming Guide, intrinsic functions),
    i.e. (4 + 2.346 |g|) u relative; 1 + e carries at most that error and rounds once, the
    division rounds once: (6 + 2.346 |g|) u.  Doubled for safety."""
    return (12 + 4.7 * g.abs()) * U32


def silu_ref(g):
    """bf16(silu(g)) for bf16 g: (near, far, tied) as bf16.  Follows F.silu's fp32 semantics
    where exp(-g) overflows fp32 (g < -88.72): the result is -0, not the tiny fp64 value."""
    g64 = g.double()
    s = g64 / (1.0 + torch.exp(-g64))
    s = torch.where(-g64 > LN_FLT_MAX, torch.zeros_like(s) * -1.0, s)
    near, far, tied = bf16_window(s, silu_delta(g64))
    return near.to(torch.bfloat16), far.to(torch.bfloat16), tied


def swiglu_ref(g, u):
    """SWIGLU_BF16 epilogue on the bf16 projections g, u: bf16(bf16(silu(g)) * u).
    Returns (candidates, tied)."""
    near, far, tied = silu_ref(g)
    uf = u.float()
    return [(near.float() * uf).to(torch.bfloat16), (far.float() * uf).to(torch.bfloat16)], tied


# --------------------------------------------------------------------------- fp32 GEMM accumulator
GEMM_C = 2.0


def gemm_f32_bound(a, w):
    """(ref, bound) for the fp32 accumulator of a @ w.T (bf16 operands), computed in fp64.

    bound = c * K * 2^-24 * sum_k |a_k w_k|.  With c = 1 this is the classic worst case of any
    fp32 summation order that rounds to nearest; the tensor cores' internal alignment and
    rounding of the products within one MMA step are not documented and may truncate, which
    doubles the per-addition error, hence c = 2."""
    a64, w64 = a.double(), w.double()
    ref = a64 @ w64.t()
    mag = a64.abs() @ w64.abs().t()
    return ref, GEMM_C * a.shape[1] * U32 * mag
