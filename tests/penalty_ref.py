"""Test helper: the CPU reference for presence / frequency / repetition penalties and min_p, and
the one-row replay and greedy oracle of penalised jobs.

Semantics are vLLM's, whose sampling_params the hosted service takes:
  apply_penalties   vllm.model_executor.layers.utils.apply_penalties restated step by step in
                    fp32 (pinned bit for bit in tests/test_sampling_penalties_cpu.py)
  min_p             keep z >= zmax + fp32(ln min_p), applied before top-k / top-p as in vLLM v1;
                    every filter keeps an upper set of z, so the kept set is top-k / top-p
                    (oracle/sampler_ref.py) over the tokens min_p keeps
  prompt / output   the prompt is the tokens fed (prefix | row | suffix, the jump-forward
                    prefix included); the output is what the row has generated so far
The replay (PenalisedReplay) and the greedy oracle (generate_penalised) extend
tests/engine_replay.Replay and oracle/model_ref.RefModel without changing them.
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import torch

from engine_replay import Replay
from oracle import sampler_ref as S
from sutro_b200 import _lib as L

PENALTY_KEYS = ("presence_penalty", "frequency_penalty", "repetition_penalty")


def apply_penalties(logits: np.ndarray, prompt, output, presence_penalty: float = 0.0,
                    frequency_penalty: float = 0.0, repetition_penalty: float = 1.0) -> np.ndarray:
    """vLLM's apply_penalties for one row, in fp32, on a copy of `logits` [V]:
      repetition  l * (l > 0 ? fp32(1/r) : r) for every token of prompt ∪ output
      frequency   l - fp32(f * count), count = occurrences in the output (0 elsewhere)
      presence    l - fp32(p * (count > 0))
    Every vocabulary entry takes the three steps, as in vLLM (so with f or p negative, -0.0
    becomes +0.0 everywhere).  Neutral values (0, 0, 1, or repetition <= 0: a zeroed C struct)
    return the logits unchanged.  Ids outside [0, V) are ignored."""
    l = np.array(logits, dtype=np.float32, copy=True)
    r = np.float32(repetition_penalty if repetition_penalty > 0 else 1.0)
    f, p = np.float32(frequency_penalty), np.float32(presence_penalty)
    if f == 0 and p == 0 and r == 1:
        return l
    V = l.shape[-1]

    def counts(ids):
        ids = np.asarray(ids, dtype=np.int64).reshape(-1)
        ids = ids[(ids >= 0) & (ids < V)]
        return np.bincount(ids, minlength=V)[:V]
    out_cnt = counts(output)
    seen = (counts(prompt) > 0) | (out_cnt > 0)
    pen = np.where(seen, r, np.float32(1.0)).astype(np.float32)
    with np.errstate(over="ignore"):                   # +-inf, as in fp32 on the GPU
        l = l * np.where(l > 0, np.float32(1.0) / pen, pen).astype(np.float32)
        l = (l - f * out_cnt.astype(np.float32)).astype(np.float32)
        return (l - p * (out_cnt > 0).astype(np.float32)).astype(np.float32)


def log_min_p(min_p: float) -> np.float32:
    """fp32(ln min_p), as the host computes it for the kernel: in double, rounded once."""
    return np.float32(np.log(np.float64(np.float32(min(min_p, 1.0)))))


def min_p_threshold(z: np.ndarray, allowed: np.ndarray, min_p: float) -> np.float32:
    """The smallest z min_p keeps: fp32(zmax + fp32(ln min_p)), zmax over the allowed tokens."""
    zmax = np.float32(np.asarray(z, np.float32)[allowed].max())
    return np.float32(zmax + log_min_p(min_p))


def _min_p_allowed(logits, allowed, temperature, min_p):
    """(allowed tokens min_p keeps, the key of its threshold); min_p <= 0: (allowed, 0)."""
    if min_p <= 0:
        return allowed, np.uint32(0)
    z = S.scaled(logits, temperature)
    key = S.fkey(min_p_threshold(z, allowed, min_p))[()]
    return allowed & (S.fkey(z) >= key), np.uint32(key)


def kept_set(logits, allowed, temperature, top_k, top_p, min_p=0.0):
    """S.kept_set with min_p applied first: -> (kept bool mask, weights)."""
    keep, _ = _min_p_allowed(logits, allowed, temperature, min_p)
    return S.kept_set(logits, keep, temperature, top_k, top_p)


def tau_expected(logits, allowed, temperature, top_k, top_p, min_p=0.0):
    """S.tau_expected with min_p applied first: -> (key of the smallest kept z, top-p margin).
    The kept set is {allowed i : fkey(z_i) >= tau}, what the kernel reports as out_tau."""
    keep, key = _min_p_allowed(logits, allowed, temperature, min_p)
    tau, margin = S.tau_expected(logits, keep, temperature, top_k, top_p)
    return np.uint32(max(tau, key)), margin


@torch.no_grad()
def generate_penalised(model, prompt, max_new: int, eos_id: int, penalties: dict,
                       ignore_eos: bool = False):
    """Greedy decode of oracle/model_ref.RefModel (no schema) with `penalties`
    ({presence,frequency,repetition}_penalty) applied to every step's logits over the prompt and
    the output so far.  -> (tokens, margins, decision_pos), the margins of the penalised logits."""
    cache = [None] * model.spec.n_layers
    prompt = list(prompt)
    h = model._forward(prompt, 0, cache)[-1:]
    out, margins, dpos = [], [], []
    pos = len(prompt)
    while True:
        lg = (h @ model._lm_head().t())[0].float().numpy()
        lg = torch.from_numpy(apply_penalties(lg, prompt, out, **penalties))
        top = torch.topk(lg, 2)
        tok = int((lg == top.values[0]).nonzero()[0])      # lowest index wins exact ties
        margins.append(float(top.values[0] - top.values[1]))
        dpos.append(len(out))
        if tok == eos_id and not ignore_eos:
            break
        out.append(tok)
        if len(out) >= max_new:
            break
        h = model._forward([tok], pos, cache)
        pos += 1
    return SimpleNamespace(tokens=out, margins=margins, decision_pos=dpos)


class _PenaltyLib:
    """The library as the replay sees it: sb200_sample also gets the job's penalties and the
    replayed row's prompt (as one piece: the prefix holds all of it)."""

    def __init__(self, rep):
        self.rep, self.real = rep, L.lib()

    def __getattr__(self, name):
        return getattr(self.real, name)

    def sb200_sample(self, args_ref, stream):
        a = args_ref._obj
        for k, v in self.rep.pen.items():
            setattr(a, k, v)
        d_prompt, d_roff, d_nrow = self.rep.prompt_dev
        a.prompt_prefix, a.n_prompt_prefix = d_prompt.data_ptr(), d_prompt.numel()
        a.row_tokens, a.row_tok_off, a.slot_n_row_tok = (d_prompt.data_ptr(), d_roff.data_ptr(),
                                                        d_nrow.data_ptr())
        return self.real.sb200_sample(args_ref, stream)


class PenalisedReplay(Replay):
    """engine_replay.Replay for jobs with penalties and min_p: job() takes them as keyword
    arguments (the engine's names) and every sampling step of the replay applies them."""

    def __init__(self, eng):
        super().__init__(eng)
        self.pen = {}
        self.prompt_dev = None
        self.lib = _PenaltyLib(self)

    def job(self, rows, presence_penalty=0.0, frequency_penalty=0.0, repetition_penalty=1.0,
            min_p=0.0, **kw):
        self.pen = dict(presence_penalty=presence_penalty, frequency_penalty=frequency_penalty,
                        repetition_penalty=repetition_penalty, min_p=min_p)
        try:
            return super().job(rows, **kw)
        finally:
            self.pen = {}

    def row(self, prompt, *args, **kw):
        dev = self.dev
        self.prompt_dev = (torch.as_tensor(np.asarray(prompt, np.int32)).to(dev),
                           torch.zeros(2, dtype=torch.int64, device=dev),
                           torch.zeros(1, dtype=torch.int32, device=dev))
        return super().row(prompt, *args, **kw)
