"""Pins the sampling oracle: Philox4x32-10 against the Random123 known-answer vectors,
and the top-k / top-p set semantics on hand-checkable distributions."""
import numpy as np

from oracle import sampler_ref as S


def test_philox4x32_10_random123_known_answers():
    assert S.philox4x32_10((0, 0), (0, 0, 0, 0)) == (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)
    f = 0xffffffff
    assert S.philox4x32_10((f, f), (f, f, f, f)) == (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)
    assert S.philox4x32_10((0xa4093822, 0x299f31d0), (0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344)) \
        == (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)


def test_top_k_and_top_p_sets():
    lg = np.log(np.array([0.5, 0.2, 0.15, 0.1, 0.05], dtype=np.float32))
    allowed = np.ones(5, dtype=bool)
    keep, _ = S.kept_set(lg, allowed, 1.0, 2, 1.0)
    assert keep.tolist() == [True, True, False, False, False]
    keep, _ = S.kept_set(lg, allowed, 1.0, 0, 0.6)          # 0.5 < 0.6 <= 0.7
    assert keep.tolist() == [True, True, False, False, False]
    keep, _ = S.kept_set(lg, allowed, 1.0, 0, 0.5)          # reached by the first token
    assert keep.tolist() == [True, False, False, False, False]
    allowed[0] = False                                       # mask first
    keep, _ = S.kept_set(lg, allowed, 1.0, 1, 1.0)
    assert keep.tolist() == [False, True, False, False, False]
    # ties at the threshold are kept
    lg2 = np.array([1.0, 1.0, 0.0], dtype=np.float32)
    keep, _ = S.kept_set(lg2, np.ones(3, dtype=bool), 1.0, 1, 1.0)
    assert keep.tolist() == [True, True, False]


def test_inverse_cdf_in_vocabulary_order_and_uniform_range():
    lg = np.log(np.array([0.25, 0.25, 0.5], dtype=np.float32))
    allowed = np.ones(3, dtype=bool)
    assert S.sample(lg, allowed, 1.0, 0, 1.0, 0.10)[0] == 0
    assert S.sample(lg, allowed, 1.0, 0, 1.0, 0.30)[0] == 1
    assert S.sample(lg, allowed, 1.0, 0, 1.0, 0.99)[0] == 2
    us = [S.uniform(7, r, s, True) for r in range(50) for s in range(4)]
    assert 0.0 <= min(us) and max(us) < 1.0 and 0.35 < np.mean(us) < 0.65
    assert S.uniform(7, 3, 1, False) == S.uniform(7, 9, 1, False)      # shared stream
    assert S.uniform(7, 3, 1, True) != S.uniform(7, 9, 1, True)


def test_kept_sets_match_transformers_logits_warpers():
    """The filter semantics against transformers' Temperature / TopK / TopP warpers (applied
    in that order, as `generate` does) on random logits: identical surviving-token sets.
    Logits are drawn without ties and top_p is kept away from cumulative-mass boundaries, where
    fp32 summation order decides membership."""
    import torch
    from transformers.generation.logits_process import (TemperatureLogitsWarper,
                                                        TopKLogitsWarper, TopPLogitsWarper)
    rng = np.random.default_rng(7)
    checked = 0
    for trial in range(60):
        vocab = int(rng.choice([50, 333, 2048]))
        logits = (rng.standard_normal(vocab) * rng.uniform(0.5, 4.0)).astype(np.float32)
        T = float(rng.choice([0.5, 0.9, 1.0, 1.7]))
        k = int(rng.choice([0, 1, 5, 40]))
        p = float(rng.choice([1.0, 0.95, 0.8, 0.3]))
        allowed = np.ones(vocab, dtype=bool)
        keep, _ = S.kept_set(logits, allowed, T, k, p)
        x = torch.from_numpy(logits)[None]
        x = TemperatureLogitsWarper(T)(None, x)
        if k > 0:
            x = TopKLogitsWarper(top_k=k)(None, x)
        if p < 1.0:
            probs = torch.softmax(x[0].double(), -1).sort(descending=True).values.cumsum(0)
            if (probs - p).abs().min() < 1e-4:      # boundary case: skip
                continue
            x = TopPLogitsWarper(top_p=p)(None, x)
        theirs = torch.isfinite(x[0]).numpy()
        assert (keep == theirs).all(), (trial, T, k, p, keep.sum(), theirs.sum())
        checked += 1
    assert checked > 40


def test_vectorised_philox_matches_the_scalar_one():
    f = 0xffffffff
    for key, ctr in [((0, 0), (0, 0, 0, 0)), ((f, f), (f, f, f, f)),
                     ((0xa4093822, 0x299f31d0), (0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344))]:
        assert tuple(int(x) for x in S.philox4x32_10_np(key, ctr)) == S.philox4x32_10(key, ctr)
    rows = np.array([0, 5, 2 ** 32 + 7, 2 ** 63 - 1], dtype=np.uint64)
    steps = np.array([0, 1, 2 ** 31 - 1, 12345])
    for spr in (False, True):
        u = np.broadcast_to(S.uniform_np(2 ** 40 + 3, rows, steps, spr), 4)
        assert [float(x) for x in u] == [S.uniform(2 ** 40 + 3, int(r), int(s), spr)
                                         for r, s in zip(rows, steps)]


def test_fkey_order_and_exact_thresholds():
    z = np.array([-np.inf, -3.0, -1e-40, -0.0, 0.0, 1e-40, 2.0, np.inf], dtype=np.float32)
    k = S.fkey(z)
    assert (np.diff(k.astype(np.int64)) >= 0).all() and k[3] == k[4]
    lg = np.array([5, 4, 4, 4, 1], dtype=np.float32)
    allowed = np.ones(5, dtype=bool)
    assert S.tau_expected(lg, allowed, 1.0, 3, 1.0) == (S.fkey(np.float32(4)), np.inf)
    assert S.tau_expected(lg, allowed, 1.0, 9, 1.0)[0] == 0                # k > allowed: off
    tau, margin = S.tau_expected(lg, allowed, 1.0, 0, 0.5)                 # 1 / 2.12 < 0.5
    assert tau == S.fkey(np.float32(4)) and abs(margin - (0.5 - 1 / 2.1219)) < 1e-3
    assert S.scaled(np.float32(3.0), 0.7) == np.float32(3.0) * (np.float32(1) / np.float32(0.7))
