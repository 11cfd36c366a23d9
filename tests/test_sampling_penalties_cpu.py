"""Presence / frequency / repetition penalties and min_p on the CPU: the reference
(tests/penalty_ref.py) against the libraries that define them, and the SDK's handling of the keys.

- penalty_ref.apply_penalties is bit-identical to vLLM's apply_penalties (its CPU path) at full
  Qwen vocabulary size, on logits with +-0, negatives, huge magnitudes and subnormals,
  heavy-repeat histories and penalties of both signs, repetition below and above 1.
- The reference's min_p kept set equals transformers' MinPLogitsWarper's except within a band of
  the threshold, where the two round the same comparison differently.
- Sutro.infer accepts the four keys, validates them with vLLM's ranges, and forwards only the
  non-neutral ones, so a job without them reaches the engine exactly as before.
"""
import numpy as np
import pytest
import torch

import penalty_ref as P
from oracle import sampler_ref as S
from sutro_b200 import engine as E
from sutro_b200.common import check_penalties
from sutro_b200.engine import GenerationResult
from sutro_b200.sdk import Sutro

QWEN = 151936


def _history(rng, n_rows, V):
    """Per-row prompt and output ids with heavy repeats (a small hot set) and some spread."""
    prompts, outputs = [], []
    for r in range(n_rows):
        hot = rng.integers(0, V, size=12)
        n_p, n_o = int(rng.integers(0, 600)), int(rng.integers(0, 200))
        if r % 8 == 0:
            n_o = 0                                   # empty output
        if r % 8 == 1:
            n_p = 0
        p = np.where(rng.random(n_p) < 0.7, rng.choice(hot, n_p), rng.integers(0, V, n_p))
        o = np.where(rng.random(n_o) < 0.8, rng.choice(hot, n_o), rng.integers(0, V, n_o))
        prompts.append(p.astype(np.int64))
        outputs.append(o.astype(np.int64))
    return prompts, outputs


def _logits(rng, n_rows, V, prompts, outputs):
    lg = (rng.standard_normal((n_rows, V)) * 6).astype(np.float32)
    for r in range(n_rows):
        hist = np.concatenate([prompts[r], outputs[r]])
        if len(hist):
            # the history's own logits take the special values too
            pick = rng.choice(hist, size=min(len(hist), 24))
            lg[r, pick[0::4]] = 0.0
            lg[r, pick[1::4]] = -0.0
            lg[r, pick[2::4]] = np.float32(3e38) * rng.choice([-1, 1])
            lg[r, pick[3::4]] = np.float32(1e-40) * rng.choice([-1, 1])
    flat = lg.reshape(-1)
    for val in (0.0, -0.0, 1e30, -1e30, 3.4e38, -3.4e38, 1e-42, -1e-42):
        flat[rng.integers(0, flat.size, 4000)] = np.float32(val)
    return lg


def _pad(seqs, V):
    n = max(1, max(len(s) for s in seqs))
    out = np.full((len(seqs), n), V, dtype=np.int64)      # vLLM pads with vocab_size
    for i, s in enumerate(seqs):
        out[i, :len(s)] = s
    return torch.from_numpy(out)


def test_apply_penalties_bit_identical_to_vllm():
    pytest.importorskip("vllm")
    from vllm.model_executor.layers.utils import apply_penalties as vllm_apply_penalties

    rng = np.random.default_rng(20261017)
    n_rows, V = 64, QWEN
    prompts, outputs = _history(rng, n_rows, V)
    lg = _logits(rng, n_rows, V, prompts, outputs)
    pres = rng.uniform(-2, 2, n_rows).astype(np.float32)
    freq = rng.uniform(-2, 2, n_rows).astype(np.float32)
    rep = rng.choice(np.float32([0.5, 0.9, 1.0, 1.1, 1.3, 2.0]), n_rows)
    pres[0:4], freq[0:4], rep[0:4] = 0, 0, 1            # neutral rows
    pres[4:8], freq[4:8] = 0, 0                         # repetition alone
    rep[8:12] = 1                                       # presence / frequency alone
    pres[12:16], freq[12:16] = -np.abs(pres[12:16]), -np.abs(freq[12:16])
    got = np.stack([P.apply_penalties(lg[r], prompts[r], outputs[r], float(pres[r]),
                                      float(freq[r]), float(rep[r])) for r in range(n_rows)])
    want = torch.from_numpy(lg.copy())
    vllm_apply_penalties(want, _pad(prompts, V), _pad(outputs, V), torch.from_numpy(pres),
                         torch.from_numpy(freq), torch.from_numpy(rep))
    want = want.numpy()
    assert got.dtype == np.float32
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))
    assert bad[0].size == 0, (bad[0][:5], bad[1][:5], got[bad][:5], want[bad][:5])
    # the penalties did something on every non-neutral row
    for r in range(4, n_rows):
        touched = (rep[r] != 1 and (len(prompts[r]) or len(outputs[r]))) or \
            (len(outputs[r]) and (pres[r] != 0 or freq[r] != 0))
        if touched:
            assert (got[r].view(np.uint32) != lg[r].view(np.uint32)).any(), r


def test_apply_penalties_neutral_and_zeroed_values_leave_logits_alone():
    rng = np.random.default_rng(1)
    lg = rng.standard_normal(1000).astype(np.float32)
    lg[:10] = -0.0
    hist = rng.integers(0, 1000, 50)
    for r in (1.0, 0.0, -1.0):            # a zeroed C struct: repetition <= 0 reads as off
        out = P.apply_penalties(lg, hist, hist, 0.0, 0.0, r)
        assert out.view(np.uint32).tolist() == lg.view(np.uint32).tolist()


def test_min_p_kept_set_matches_transformers_outside_a_band():
    from transformers import MinPLogitsWarper

    rng = np.random.default_rng(7)
    # the two sides round the same comparison (ours: z >= zmax + fp32(ln min_p); transformers:
    # softmax(z) >= min_p * max softmax(z), in fp32): they may differ within this band of z
    band = 1e-4
    n_band = n_diff = 0
    for i, min_p in enumerate([0.01, 0.05, 0.1, 0.3, 0.9, 1.0]):
        V = QWEN if i % 2 == 0 else 128256
        z = (rng.standard_normal(V) * (2 + 2 * i)).astype(np.float32)
        z[rng.integers(0, V, 64)] = z.max()             # ties at the maximum
        allowed = np.ones(V, dtype=bool)
        keep, _ = P.kept_set(z, allowed, 1.0, 0, 1.0, min_p)
        proc = MinPLogitsWarper(min_p=min_p)
        out = proc(None, torch.from_numpy(z.copy())[None])[0].numpy()
        ref = np.isfinite(out)
        thr = P.min_p_threshold(z, allowed, min_p)
        near = np.abs(z.astype(np.float64) - float(thr)) <= band * max(1.0, abs(float(thr)))
        n_band += int(near.sum())
        diff = keep != ref
        n_diff += int(diff.sum())
        assert not (diff & ~near).any(), (min_p, np.nonzero(diff & ~near)[0][:5])
        assert keep.sum() >= 1 and keep[np.argmax(z)]
        # the threshold the kernel reports keeps exactly this set
        tau, _ = P.tau_expected(z, allowed, 1.0, 0, 1.0, min_p)
        assert ((S.fkey(z) >= tau) == keep).all()
    print(f"min_p: {n_diff} disagreements, all among {n_band} tokens within the band")


def test_min_p_composes_with_top_k_and_top_p_as_the_largest_threshold():
    rng = np.random.default_rng(3)
    z = (rng.standard_normal(5000) * 3).astype(np.float32)
    allowed = rng.random(5000) < 0.8
    for k, p, m in [(50, 1.0, 0.1), (5, 1.0, 0.01), (0, 0.9, 0.2), (100, 0.5, 0.05)]:
        keep, _ = P.kept_set(z, allowed, 0.7, k, p, m)
        tau, margin = P.tau_expected(z, allowed, 0.7, k, p, m)
        if margin > 1e-6:
            assert ((S.fkey(S.scaled(z, 0.7)) >= tau) & allowed == keep).all(), (k, p, m)
        # min_p alone, then top-k on what it kept, equals both thresholds at once
        km, _ = P.kept_set(z, allowed, 0.7, 0, 1.0, m)
        kk, _ = P.kept_set(z, allowed, 0.7, k, 1.0, 0.0)
        if p == 1.0:
            assert (keep == (km & kk)).all()


def test_check_penalties_ranges():
    assert check_penalties() == (0.0, 0.0, 1.0, 0.0)
    assert check_penalties(-2, 2, 0.01, 1) == (-2.0, 2.0, 0.01, 1.0)
    for bad in [dict(presence_penalty=2.5), dict(presence_penalty=-2.01),
                dict(frequency_penalty=3), dict(frequency_penalty=float("nan")),
                dict(repetition_penalty=0), dict(repetition_penalty=-1),
                dict(repetition_penalty=float("inf")), dict(min_p=-0.1), dict(min_p=1.5)]:
        with pytest.raises(ValueError):
            check_penalties(**bad)


class _Stub:
    def __init__(self):
        self.calls = []

    def generate(self, rows, **kw):
        self.calls.append(kw)
        return GenerationResult([f"o{i}" for i in range(len(rows))], None, None, {})


def _client(tmp_path):
    c = Sutro(verbose=False, cache_dir=str(tmp_path))
    c.register_engine("qwen-3-4b", _Stub())
    return c


def test_sdk_accepts_and_forwards_the_penalty_keys(tmp_path):
    c = _client(tmp_path)
    c.infer(["x"], model="qwen-3-4b", sampling_params={
        "temperature": 0.7, "presence_penalty": 1.5, "frequency_penalty": 0.5,
        "repetition_penalty": 1.1, "min_p": 0.05, "max_tokens": 8})
    kw = c._engines["qwen-3-4b"].calls[0]
    assert (kw["presence_penalty"], kw["frequency_penalty"], kw["repetition_penalty"],
            kw["min_p"]) == (1.5, 0.5, 1.1, 0.05)


def test_sdk_neutral_penalties_reach_the_engine_as_an_old_job(tmp_path):
    c = _client(tmp_path)
    c.infer(["x"], model="qwen-3-4b", sampling_params={"max_tokens": 8})
    c.infer(["x"], model="qwen-3-4b", sampling_params={
        "max_tokens": 8, "presence_penalty": 0, "frequency_penalty": 0.0,
        "repetition_penalty": 1.0, "min_p": None})
    a, b = c._engines["qwen-3-4b"].calls
    assert a == b
    assert not {"presence_penalty", "frequency_penalty", "repetition_penalty", "min_p"} & set(a)


@pytest.mark.parametrize("sp", [{"presence_penalty": 2.5}, {"frequency_penalty": -3},
                                {"repetition_penalty": 0}, {"min_p": 1.2}, {"min_p": -0.5},
                                {"logit_bias": {1: 2.0}}, {"stop": ["x"]}])
def test_sdk_rejects_out_of_range_and_unknown_keys(tmp_path, sp):
    with pytest.raises(ValueError):
        _client(tmp_path).infer(["x"], model="qwen-3-4b", sampling_params=sp)


def test_zeroed_job_struct_is_neutral():
    job, args = E.JobC(), E.SampleArgsC()
    for o in (job, args):
        assert (o.presence_penalty, o.frequency_penalty, o.repetition_penalty, o.min_p) == \
            (0.0, 0.0, 0.0, 0.0)
    # repetition 0 (a zeroed struct) is read as off, like the oracle
    lg = np.arange(-5, 5, dtype=np.float32)
    assert (P.apply_penalties(lg, [1, 2], [3], 0.0, 0.0, job.repetition_penalty) == lg).all()
