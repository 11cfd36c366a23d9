"""CPU oracle for temperature / top-k / top-p sampling.  TEST INFRASTRUCTURE (see
oracle/model_ref.py for who may import oracle/).

PARITY UNPINNED by the reference (`sampling_params` is an opaque dict forwarded to the
hosted service, sutro/sdk.py:203).  Semantics restated here are the customary ones
(vLLM / transformers logits processors): z = logit / T over the allowed tokens; top-k keeps
every token whose z is >= the k-th largest (ties kept); top-p then keeps the smallest set of
highest-z tokens whose softmax mass reaches top_p (ties kept); the token is drawn by inverse
CDF over the kept set in vocabulary order from one uniform u per (seed, row, step).
The generator is Philox4x32-10 (Salmon et al., SC'11), pinned by the Random123 known-answer
vectors in tests/test_sampler_oracle.py; the kept sets are checked there against
transformers' Temperature / TopK / TopP logits warpers.
"""
from __future__ import annotations

import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32_10(key, ctr):
    k0, k1 = key
    c0, c1, c2, c3 = ctr
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2
        hi0, lo0, hi1, lo1 = p0 >> 32, p0 & MASK, p1 >> 32, p1 & MASK
        c0, c1, c2, c3 = (hi1 ^ c1 ^ k0) & MASK, lo1, (hi0 ^ c3 ^ k1) & MASK, lo0
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return c0, c1, c2, c3


def philox4x32_10_np(key, ctr):
    """philox4x32_10 on numpy arrays: key = (k0, k1), ctr = (c0, c1, c2, c3), each an int or an
    array (broadcast), one counter per element.  Returns four uint64 arrays of 32-bit words."""
    k0, k1 = (np.asarray(k, dtype=np.uint64) for k in key)
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) for c in ctr)
    m0, m1, mask = np.uint64(M0), np.uint64(M1), np.uint64(MASK)
    s32 = np.uint64(32)
    for _ in range(10):
        p0, p1 = m0 * c0, m1 * c2                       # < 2^64: exact in uint64
        c0, c1, c2, c3 = (p1 >> s32) ^ c1 ^ k0, p1 & mask, (p0 >> s32) ^ c3 ^ k1, p0 & mask
        k0, k1 = (k0 + np.uint64(W0)) & mask, (k1 + np.uint64(W1)) & mask
    return c0, c1, c2, c3


def uniform(seed: int, row: int, step: int, seed_per_row: bool) -> float:
    r = row if seed_per_row else 0
    x = philox4x32_10((seed & MASK, (seed >> 32) & MASK), (r & MASK, (r >> 32) & MASK, step, 0))
    return float(np.float32(x[0] >> 8) * np.float32(1.0 / 16777216.0))


def uniform_np(seed: int, row, step, seed_per_row: bool) -> np.ndarray:
    """uniform() for arrays of rows and steps (float32)."""
    r = np.asarray(row, dtype=np.uint64) if seed_per_row else np.uint64(0)
    x0 = philox4x32_10_np((seed & MASK, (seed >> 32) & MASK),
                          (r & np.uint64(MASK), r >> np.uint64(32), step, 0))[0]
    return (x0 >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def scaled(logits: np.ndarray, temperature: float) -> np.ndarray:
    """z = logit * (1/T) in fp32, rounded as the kernel rounds it: 1/T first, then the product."""
    inv_t = np.float32(1) / np.float32(temperature)
    return (np.asarray(logits, dtype=np.float32) * inv_t).astype(np.float32)


def fkey(z: np.ndarray) -> np.ndarray:
    """Order-preserving uint32 image of float32 values (-0.0 taken as +0.0), as the kernel's."""
    z = np.asarray(z, dtype=np.float32)
    u = np.where(z == 0, np.float32(0), z).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def tau_expected(logits: np.ndarray, allowed: np.ndarray, temperature: float, top_k: int,
                 top_p: float):
    """-> (tau, margin): the key of the smallest kept z after top-k then top-p (0 when no filter
    is active; kept = allowed & fkey(z) >= tau), and, for top-p, how far the boundary is from
    being decided the other way: min(mass of the keys >= boundary - top_p*W, top_p*W - mass of
    the keys > boundary) / W (a side with no key beyond it does not count), in fp64 from the exact exp(z - zmax).  The top-k key is exact
    (margin inf without top-p).  Ties at the boundary are kept by both filters."""
    z = scaled(logits, temperature)
    keys = fkey(z)
    tau, margin = np.uint32(0), np.inf
    ka = np.sort(keys[allowed])[::-1]
    if top_k and 0 < top_k <= len(ka):
        tau = ka[top_k - 1]
    if top_p < 1.0:
        cand = allowed & (keys >= tau)
        zc = z[cand].astype(np.float64)
        w = np.exp(zc - zc.max())
        kc = keys[cand]
        uk, inv = np.unique(kc, return_inverse=True)       # ascending distinct keys
        mass = np.bincount(inv, weights=w)[::-1]            # per distinct key, descending
        cum = np.cumsum(mass)
        W = cum[-1]
        target = max(top_p, 0.0) * W
        j = int(np.searchsorted(cum, target, side="left"))
        j = min(j, len(cum) - 1)
        above = cum[j - 1] if j > 0 else 0.0
        # no key below the last group / above the first: that side cannot flip
        margin = min(cum[j] - target if j < len(cum) - 1 else np.inf,
                     target - above if j > 0 else np.inf) / W
        tau = max(tau, uk[::-1][j])
    return np.uint32(tau), float(margin)


def log_softmax(logits: np.ndarray, allowed: np.ndarray, temperature: float) -> np.ndarray:
    """fp64 log-softmax of z = fp32(logit * (1/T)) over the allowed tokens (-inf elsewhere);
    temperature <= 0 (greedy) uses the logits as they are."""
    z = scaled(logits, temperature) if temperature > 0 else np.asarray(logits, np.float32)
    z = np.where(allowed, z.astype(np.float64), -np.inf)
    zmax = z.max()
    return z - zmax - np.log(np.exp(z - zmax).sum())


def kept_set(logits: np.ndarray, allowed: np.ndarray, temperature: float, top_k: int,
             top_p: float):
    """-> (kept bool mask, weights exp(z - zmax) as float32)"""
    z = scaled(logits, temperature)
    z = np.where(allowed, z, -np.inf).astype(np.float32)
    zmax = z.max()
    w = np.exp(z - zmax, dtype=np.float32)
    w[~allowed] = 0
    keep = allowed.copy()
    if top_k and top_k > 0 and allowed.sum() > top_k:
        kth = np.sort(z[allowed])[-top_k]
        keep &= z >= kth
    if 0.0 < top_p < 1.0:
        zk = np.where(keep, z, -np.inf)
        order = np.argsort(-zk, kind="stable")
        mass = np.cumsum(w[order].astype(np.float64))
        total = mass[keep.sum() - 1]
        n = int(np.searchsorted(mass[:keep.sum()], top_p * total, side="left")) + 1
        thr = zk[order[min(n, keep.sum()) - 1]]
        keep &= z >= thr
    return keep, w


def sample(logits: np.ndarray, allowed: np.ndarray, temperature: float, top_k: int, top_p: float,
           u: float):
    """-> (token, slack): slack = distance of the draw from the nearest CDF boundary in units
    of total mass (a GPU/CPU disagreement is only acceptable when slack is ~fp32 rounding)."""
    keep, w = kept_set(logits, allowed, temperature, top_k, top_p)
    wk = np.where(keep, w, 0).astype(np.float64)
    cdf = np.cumsum(wk)
    total = cdf[-1]
    target = u * total
    tok = int(np.searchsorted(cdf, target, side="right"))
    tok = min(tok, len(cdf) - 1)
    while wk[tok] == 0 and tok > 0:          # target == total lands past the last kept token
        tok -= 1
    lo = cdf[tok] - wk[tok]
    slack = min(target - lo, cdf[tok] - target) / total
    return tok, float(slack)


def logprob(logits: np.ndarray, allowed: np.ndarray, temperature: float, tok: int) -> float:
    return float(log_softmax(logits, allowed, temperature)[tok])
