"""Presence / frequency / repetition penalties and min_p on the GPU (sampler_fsm.cu).

1. Through `sb200_sample`, 512-row chunks at full vocabulary size: the penalty kernel's in-place
   logits are bit-identical to penalty_ref.apply_penalties (tests/penalty_ref.py), over
   histories that mix empty, one-token and repeat-heavy outputs, long prompts, masked and done
   rows; the greedy token is the reference's arg-max of the penalised, masked logits, and the row
   bookkeeping (ngen, out_tokens, out_len, done) follows it; `out_tau` is the reference's
   threshold for min_p alone and combined with top-k / top-p wherever the top-p margin allows.
   The same checks run at every size class of the row-history table (out_stride 1,024 to 8,192,
   tables up to 150 KB of shared memory): hashes at their design load, probe chains that wrap
   past the table's end, 32,000-token prompts and ids outside the vocabulary.
2. Neutral values give the same bytes and the same launch counts as a job without them.
3. Every row of a penalised job equals its one-row replay through the verified kernels
   (penalty_ref.PenalisedReplay over tests/engine_replay.py), bit for bit, in the engine's
   scheduling geometries, and at 2,048 to 8,192 new tokens on full-vocabulary tiny models, where
   the engine's table needs more than 48 KiB of shared memory.
4. A penalised row decoded alone equals the same row inside a shuffled batch.
5. Greedy with penalties equals the CPU model (penalty_ref.generate_penalised) up to the first
   near tie.
6. Sutro.infer, sb200_infer_text and sb200_model_infer agree on a penalised job.
"""
import ctypes as C
import dataclasses
from typing import Literal

import numpy as np
import pytest
import torch
from pydantic import BaseModel

import penalty_ref as P
from oracle import sampler_ref as S
from sutro_b200 import _lib as L
from sutro_b200 import engine as E
from sutro_b200 import modelspec as MS
from sutro_b200 import synth, vocab as VB

pytestmark = pytest.mark.gpu

DEV = "cuda"
SYS = synth.README_SYSTEM_PROMPT
TOP_P_MARGIN = 1e-4            # as in test_sampler_gpu.py
PEN = dict(presence_penalty=1.5, frequency_penalty=0.5, repetition_penalty=1.1)


class Sentiment(BaseModel):
    sentiment: Literal["positive", "neutral", "negative"]


def bits(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.float32)).view(np.uint32)


def dev(a, dtype=torch.int32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


# ------------------------------------------------------------------------ 1. the sample hook
HASH_MUL = 2654435761          # the kernel's hash: home(t) = (t * HASH_MUL) mod hash_size


def hash_size(stride):
    """Slots of the kernel's output-count hash: the smallest power of two >= 2 * out_stride
    (at least 32), so live rows (at most out_stride - 1 outputs) keep its load under 0.5."""
    h = 32
    while h < 2 * stride:
        h *= 2
    return h


def table_bytes(V, stride):
    """Dynamic shared memory of the penalty kernel: the prompt bitmap and 8 bytes a hash slot."""
    return (V + 31) // 32 * 4 + hash_size(stride) * 8


def wrap_cluster(V, H, rng, n_buckets=24, per_bucket=3):
    """Distinct tokens, per_bucket of them homed at each of the last n_buckets slots of an
    H-slot table (t = j * HASH_MUL^-1 mod H, plus multiples of H): linear probing must carry
    some of them past the last slot and around to slot 0."""
    inv = pow(HASH_MUL, -1, H)
    toks = []
    for j in range(H - n_buckets, H):
        base = j * inv % H
        toks += [base + int(k) * H for k in rng.choice((V - 1 - base) // H + 1, per_bucket,
                                                        replace=False)]
    return np.array(toks, np.int32)


def probes_wrap(tokens, V, H):
    """True if some probe chain must run past the table's last slot: for some m, more distinct
    in-range tokens are homed in the last m slots than those m slots hold (whatever the order of
    the insertions)."""
    t = np.unique(np.asarray(tokens, np.int64))
    t = t[(t >= 0) & (t < V)]
    home = (t.astype(np.uint64) * np.uint64(HASH_MUL)) % np.uint64(H)
    from_end = np.sort((H - home).astype(np.int64))          # 1 for the last slot
    return bool((np.arange(1, len(from_end) + 1) > from_end).any())


class Chunk:
    """B rows (512 by default) with their prompts, histories, masks and done flags, on the GPU.
    Row b is of kind b % 10: kinds 0-5 mix empty, one-token, repeat-heavy and stride - 1 outputs
    (mostly repeats) with prompts of up to 3,000 tokens; 6 holds stride - 1 distinct outputs (the
    hash at its design load); 7 a cluster homed in the table's last slots, so probes wrap to
    slot 0, with repeats mixed in; 8 a ~32,000-token prompt that overlaps the output; 9 ids
    outside [0, V) in the prompt and the output, which the kernel must ignore."""

    KINDS = 10

    def __init__(self, V, seed, B=512, stride=96):
        rng = np.random.default_rng(seed)
        self.V, self.B, self.stride, self.H = V, B, stride, hash_size(stride)
        self.raw = (rng.standard_normal((B, V)) * 4).astype(np.float32)
        self.pre = rng.integers(0, V, 40).astype(np.int32)
        self.suf = rng.integers(0, V, 9).astype(np.int32)
        rows, self.ngen, self.out = [], np.zeros(B, np.int32), np.zeros((B, stride), np.int32)
        bad = np.array([-1, -7, V, V + 1, 2 ** 31 - 1, -2 ** 31], np.int64)
        for b in range(B):
            hot = rng.integers(0, V, 6)
            kind = b % self.KINDS
            if kind < 6:
                n_row = [0, 3, 40, 3000, 200, 15][kind] + int(rng.integers(0, 8))
                row = np.where(rng.random(n_row) < 0.5, rng.choice(hot, n_row),
                               rng.integers(0, V, n_row))
                n = [0, 1, 80, 5, stride - 1, 30][kind]
                o = np.where(rng.random(n) < 0.85, rng.choice(hot, n), rng.integers(0, V, n))
            elif kind == 6:
                row = rng.integers(0, V, 20)
                o = rng.choice(V, stride - 1, replace=False)
            elif kind == 7:
                cl = wrap_cluster(V, self.H, rng)
                n = max(len(cl), min(stride - 1, 4 * len(cl)))
                o = np.concatenate([cl, np.where(rng.random(n - len(cl)) < 0.9,
                                                 rng.choice(cl, n - len(cl)),
                                                 rng.integers(0, V, n - len(cl)))])
                o = rng.permutation(o)
                row = np.where(rng.random(100) < 0.5, rng.choice(cl, 100), rng.integers(0, V, 100))
            elif kind == 8:
                n = min(stride - 1, 500)
                o = np.where(rng.random(n) < 0.6, rng.choice(hot, n), rng.integers(0, V, n))
                n_row = 32000 - int(rng.integers(0, 50))
                row = np.where(rng.random(n_row) < 0.3, rng.choice(o, n_row),
                               rng.integers(0, V, n_row))
            else:
                n = min(stride - 1, 300)
                o = np.where(rng.random(n) < 0.2, rng.choice(bad, n), rng.choice(hot, n))
                row = np.where(rng.random(400) < 0.2, rng.choice(bad, 400),
                               rng.integers(0, V, 400))
            rows.append(np.asarray(row).astype(np.int32))
            n = len(o)
            self.out[b, :n] = np.asarray(o).astype(np.int32)
            self.ngen[b] = n
            # the history's own logits take +-0 and ties at the maximum
            h = np.concatenate([rows[b], self.out[b, :n]])
            h = h[(h >= 0) & (h < V)]
            if len(h):
                self.raw[b, h[:3]] = np.float32([0.0, -0.0, self.raw[b].max()])[:len(h[:3])]
        self.raw[:, rng.integers(0, V, 64)] = -0.0                   # -0.0 outside the histories
        self.rows = rows
        self.roff = np.zeros(B + 1, np.int64)
        self.roff[1:] = np.cumsum([len(r) for r in rows])
        self.row_toks = np.concatenate(rows).astype(np.int32)
        self.n_row = np.array([len(r) for r in rows], np.int32)
        self.done = (np.arange(B) % 17 == 5).astype(np.int32)
        # every third row is masked to a random half of the vocabulary (one state per row)
        self.masked = np.arange(B) % 3 == 1
        self.allowed = np.ones((B, V), dtype=bool)
        self.allowed[self.masked] = rng.random((int(self.masked.sum()), V)) < 0.5
        self.state = np.where(self.masked, np.arange(B), -1).astype(np.int32)

    def prompt(self, b):
        return np.concatenate([self.pre, self.rows[b], self.suf])

    def run(self, T=0.0, k=0, p=1.0, **pen):
        B, V = self.B, self.V
        words = (V + 31) // 32
        pad = np.zeros((B, words * 32), dtype=bool)
        pad[:, :V] = self.allowed
        mask = np.packbits(pad, axis=-1, bitorder="little").view(np.int32)
        d = {"lg": dev(self.raw, torch.float32), "row_slot": dev(np.arange(B)),
             "state": dev(self.state), "ngen": dev(self.ngen), "next": dev(np.zeros(B)),
             "pos": dev(np.zeros(B)), "done": dev(self.done), "slot_row": dev(np.arange(B)),
             "maxnew": dev(np.full(B, self.stride)), "out": dev(self.out),
             "len": dev(np.zeros(B)), "mask": dev(mask),
             "trans": dev(np.tile(np.arange(B, dtype=np.int32)[:, None], (1, 256))),
             "final": dev(np.zeros(B), torch.uint8), "tb": dev(np.arange(V) % 256, torch.uint8),
             "to": dev(np.arange(V + 1)), "tau": dev(np.zeros(B)),
             "pre": dev(self.pre), "suf": dev(self.suf), "rt": dev(self.row_toks),
             "roff": dev(self.roff, torch.int64), "nrow": dev(self.n_row)}
        g = lambda n: d[n].data_ptr()  # noqa: E731
        a = E.SampleArgsC()
        a.logits, a.ldl, a.vocab, a.B = g("lg"), V, V, B
        a.row_slot, a.slot_state, a.slot_ngen = g("row_slot"), g("state"), g("ngen")
        a.slot_next_tok, a.slot_pos, a.slot_done = g("next"), g("pos"), g("done")
        a.slot_row, a.slot_maxnew, a.out_tokens, a.out_len = (g("slot_row"), g("maxnew"),
                                                              g("out"), g("len"))
        a.out_stride, a.mask_bits, a.mask_words = self.stride, g("mask"), words
        a.fsm_trans, a.fsm_final, a.tok_bytes, a.tok_off = g("trans"), g("final"), g("tb"), g("to")
        a.eos_id, a.ignore_eos = V - 1, 1
        a.temperature, a.top_k, a.top_p = T, k, p
        a.out_tau = g("tau")
        for name, v in pen.items():
            setattr(a, name, v)
        a.prompt_prefix, a.n_prompt_prefix = g("pre"), len(self.pre)
        a.prompt_suffix, a.n_prompt_suffix = g("suf"), len(self.suf)
        a.row_tokens, a.row_tok_off, a.slot_n_row_tok = g("rt"), g("roff"), g("nrow")
        L.check(L.lib().sb200_sample(C.byref(a), L.current_stream()))
        torch.cuda.synchronize()
        return {n: t.cpu().numpy() for n, t in d.items()}

    def penalised(self, b, presence_penalty=0.0, frequency_penalty=0.0, repetition_penalty=1.0,
                  **_):
        return P.apply_penalties(self.raw[b], self.prompt(b), self.out[b, :self.ngen[b]],
                                 presence_penalty, frequency_penalty, repetition_penalty)


CHUNKS = {}


def chunk(V):
    if V not in CHUNKS:
        CHUNKS[V] = Chunk(V, seed=V)
    return CHUNKS[V]


PEN_SETS = [dict(PEN), dict(presence_penalty=-1.0, frequency_penalty=-0.25, repetition_penalty=0.8),
            dict(repetition_penalty=1.7), dict(frequency_penalty=2.0)]


def check_penalised_greedy(c, pen):
    """One greedy sb200_sample over chunk c with penalties pen: penalised logits bit-identical to
    the reference, the reference's lowest-index arg-max drawn and booked, done rows untouched."""
    h = c.run(**pen)
    n_rewritten = 0
    for b in range(c.B):
        n = c.ngen[b]
        if c.done[b]:
            assert (bits(h["lg"][b]) == bits(c.raw[b])).all(), b        # done rows: untouched
            assert h["ngen"][b] == n and h["len"][b] == 0 and h["done"][b] == 1, b
            assert (h["out"][b] == c.out[b]).all(), b
            continue
        want = c.penalised(b, **pen)
        bad = np.nonzero(bits(h["lg"][b]) != bits(want))[0]
        assert bad.size == 0, (b, bad[:5], h["lg"][b][bad[:5]], want[bad[:5]])
        n_rewritten += int((bits(want) != bits(c.raw[b])).sum())
        z = np.where(c.allowed[b], want, -np.inf)
        tok = int(np.flatnonzero(z == z.max())[0])                     # lowest index wins ties
        assert h["next"][b] == tok, (b, h["next"][b], tok)
        # bookkeeping: the token appended after the history, the row done at out_stride tokens
        assert h["ngen"][b] == n + 1 and h["len"][b] == n + 1, (b, h["ngen"][b], h["len"][b])
        assert (h["out"][b, :n] == c.out[b, :n]).all() and h["out"][b, n] == tok, b
        assert h["done"][b] == int(n + 1 >= c.stride), b
    assert n_rewritten > 0
    return n_rewritten


@pytest.mark.parametrize("V", [151936, 128256])
@pytest.mark.parametrize("pi", range(len(PEN_SETS)))
def test_penalised_logits_and_greedy_token_are_exact(V, pi):
    c, pen = chunk(V), PEN_SETS[pi]
    n_rewritten = check_penalised_greedy(c, pen)
    print("PENALTIES", f"V={V}", pen, f"rewritten={n_rewritten}")


# out_stride at and around each doubling of the hash, up to the kernel's 8,192-token limit
TABLE_STRIDES = [1024, 1025, 2048, 2049, 4096, 4097, 8192]
_BIG = {}


def big_chunk(V, stride):
    """A 40-row chunk (the CPU reference stays quick at 8,192-token histories); the last one
    built is kept for the next penalty set."""
    if (V, stride) not in _BIG:
        _BIG.clear()
        _BIG[(V, stride)] = Chunk(V, seed=V + stride, B=40, stride=stride)
    return _BIG[(V, stride)]


@pytest.mark.parametrize("pi", [0, 1])                    # PEN_SETS[1] has the -0.0 pass
@pytest.mark.parametrize("V", [151936, 128256])
@pytest.mark.parametrize("stride", TABLE_STRIDES)
def test_penalty_tables_at_every_size_class(stride, V, pi):
    c, pen = big_chunk(V, stride), PEN_SETS[pi]
    # the regimes: past 48 KiB the launcher opts in to more shared memory (Qwen from 1,025
    # tokens, Llama from 2,049); hashes at their design load; probe chains that wrap; long
    # prompts; ids outside the vocabulary, all in rows that are not done
    tb = table_bytes(V, stride)
    assert (tb > 48 * 1024) == (stride > (1024 if V == 151936 else 2048)), tb
    live = [b for b in range(c.B) if not c.done[b]]
    outs = [c.out[b, :c.ngen[b]] for b in live]
    assert any(len(np.unique(o)) == stride - 1 for o in outs)
    assert any(probes_wrap(o, V, c.H) for o in outs)
    assert max(len(c.prompt(b)) for b in live) >= 32000
    assert any(((o < 0) | (o >= V)).any() for o in outs)
    n_rewritten = check_penalised_greedy(c, pen)
    print("PENALTY_TABLE", f"V={V}", f"stride={stride}", f"hash={c.H}", f"smem={tb}", pen,
          f"rewritten={n_rewritten}")


@pytest.mark.parametrize("V", [151936, 128256])
@pytest.mark.parametrize("T,k,p,m", [(0.7, 0, 1.0, 0.05), (1.0, 0, 1.0, 0.3), (0.7, 40, 1.0, 0.05),
                                     (0.7, 0, 0.9, 0.02), (1.3, 100, 0.8, 0.1), (0.7, 0, 1.0, 1.0)])
def test_min_p_threshold_alone_and_with_top_k_top_p(V, T, k, p, m):
    c = chunk(V)
    h = c.run(T=T, k=k, p=p, min_p=m, **PEN)
    checked = 0
    for b in range(c.B):
        if c.done[b]:
            continue
        lg = c.penalised(b, **PEN)
        assert (bits(h["lg"][b]) == bits(lg)).all(), b
        tau, margin = P.tau_expected(lg, c.allowed[b], T, k, p, m)
        if margin <= TOP_P_MARGIN:
            continue
        got = h["tau"].view(np.uint32)[b]
        assert got == tau, (b, got, tau)
        keep = c.allowed[b] & (S.fkey(S.scaled(lg, T)) >= tau)
        assert keep[int(h["next"][b])], b                              # drawn from the kept set
        checked += 1
    assert checked > 0.9 * (c.B - c.done.sum()), checked
    print("MIN_P", f"V={V}", (T, k, p, m), f"rows={checked}")


def test_penalties_refuse_outputs_longer_than_the_table():
    lg = torch.zeros(1, 64, device=DEV)
    z = torch.zeros(1, dtype=torch.int32, device=DEV)
    a = E.SampleArgsC()
    a.logits, a.ldl, a.vocab, a.B, a.out_stride = lg.data_ptr(), 64, 64, 1, 8193
    a.presence_penalty = 1.0
    for n in ("row_slot", "slot_state", "slot_ngen", "slot_next_tok", "slot_pos", "slot_done",
              "slot_row", "slot_maxnew", "out_tokens", "out_len", "row_tokens", "row_tok_off",
              "slot_n_row_tok"):
        setattr(a, n, z.data_ptr())
    assert L.lib().sb200_sample(C.byref(a), L.current_stream()) != 0
    err = L.lib().sb200_last_error()
    assert "8192" in (err.decode() if isinstance(err, bytes) else str(err))


# ---------------------------------------------------------------------------- engine jobs
def build(name, **kw):
    from sutro_b200.engine import LocalEngine
    spec = MS.get_spec(name)
    w = MS.make_weights(spec, seed=0, std=0.05)
    v = VB.build_vocab(spec.family, spec.vocab_size, seed=0, n_trained=600)
    kw.setdefault("kv_pages", 512)
    return LocalEngine(spec, MS.pack_for_engine(spec, w, "cuda"), v, device=0, **kw), w


_ENG = {}


def engine(name):
    if name not in _ENG:
        eng, w = build(name, max_slots=8, max_prefill_tokens=1024, logit_chunk_rows=3)
        _ENG[name] = (eng, w, P.PenalisedReplay(eng))
    return _ENG[name]


ROWS = synth.README_REVIEWS + synth.product_reviews(7, seed=7) + ["word " * 600, ""]


def test_neutral_values_are_the_old_job():
    eng, _, _ = engine("tiny-qwen3")
    for kw in [dict(), dict(temperature=0.8, top_k=20, top_p=0.9, seed=3),
               dict(json_schema=Sentiment.model_json_schema())]:
        base = eng.generate(ROWS, system_prompt=SYS, max_new_tokens=32, return_tokens=True,
                            return_logprobs=True, **kw)
        neut = eng.generate(ROWS, system_prompt=SYS, max_new_tokens=32, return_tokens=True,
                            return_logprobs=True, presence_penalty=0.0, frequency_penalty=0.0,
                            repetition_penalty=1.0, min_p=0.0, **kw)
        assert neut.out_tokens == base.out_tokens
        assert (bits(neut.cum_logprobs) == bits(base.cum_logprobs)).all()
        assert neut.stats["kernel_launches"] == base.stats["kernel_launches"]
    # with a penalty on, the penalty kernel adds one launch per sampler launch
    pen = eng.generate(ROWS, system_prompt=SYS, max_new_tokens=32, return_tokens=True, **PEN)
    heads = pen.stats["prefill_steps"] + pen.stats["decode_steps"]
    assert pen.stats["kernel_launches"]["sample"] >= 2 * heads


def replay_compare(eng, rep, rows, label, one_call=False, **kw):
    if one_call:
        res = eng.infer_one_call(rows, return_logprobs=True, **kw)
    else:
        res = eng.generate(rows, return_tokens=True, return_first_logits=True,
                           return_logprobs=True, **kw)
    reps = rep.job(rows, **kw)
    for i, r in enumerate(reps):
        assert res.out_tokens[i] == r.tokens, (label, i, res.out_tokens[i], r.tokens)
        if not one_call:      # the first-decision logits stay raw
            assert (bits(res.first_logits[i].numpy()) == bits(r.first_logits.numpy())).all()
        assert bits(res.cum_logprobs[i]) == bits(r.cum_logprob), (label, i)
    steps = sum(r.decode_steps for r in reps)
    print("PARITY", label, f"rows={len(rows)}", f"steps={steps}",
          f"truncated={res.stats['rows_truncated']}")
    return res


CASES = [
    ("greedy", dict()),
    ("sampled_minp", dict(temperature=0.8, top_k=30, top_p=0.9, seed=5, min_p=0.05)),
    ("schema_jump", dict(json_schema=Sentiment.model_json_schema())),
    ("schema_nojump_sampled", dict(json_schema=Sentiment.model_json_schema(), jump_forward=False,
                                   temperature=0.7, seed=2, min_p=0.1)),
    ("no_share", dict(share_prefix=False, temperature=0.7, seed=9)),
]


@pytest.mark.parametrize("name", ["tiny-qwen3", "tiny-qwen3-g4", "tiny-llama"])
@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_penalised_rows_match_the_replay(name, case):
    eng, _, rep = engine(name)
    kw = dict(dict(CASES)[case], **PEN)
    res = replay_compare(eng, rep, ROWS, f"{case}[{name}]", system_prompt=SYS, max_new_tokens=40,
                         **kw)
    assert res.stats["rows_truncated"] == 1          # the 600-word row


def full_vocab_engine(name, window):
    """A tiny model over its family's full-size vocabulary, with a window of `window` tokens."""
    from sutro_b200.engine import LocalEngine
    V = {"qwen3": 151936, "llama": 128256}[MS.get_spec(name).family]
    spec = dataclasses.replace(MS.with_vocab(MS.get_spec(name), V), max_position=window)
    w = MS.make_weights(spec, seed=0, std=0.05)
    v = VB.build_vocab(spec.family, V, seed=0)
    return LocalEngine(spec, MS.pack_for_engine(spec, w, "cuda"), v, device=0, kv_pages=2048,
                       max_slots=4, max_prefill_tokens=1024, logit_chunk_rows=2)


@pytest.mark.parametrize("name,max_new", [("tiny-qwen3", 2048), ("tiny-qwen3", 8192),
                                          ("tiny-llama", 2049)])
def test_long_penalised_jobs_match_the_replay(name, max_new):
    """The engine sizes the table by max_new_tokens: 2,048 (the SDK's default budget) and 8,192
    (the limit) at Qwen's vocabulary, 2,049 at Llama's, all past 48 KiB of shared memory.  Every
    row runs its whole budget (ignore_eos), so the hash ends at its design load."""
    eng = full_vocab_engine(name, window=max_new + 1024)
    try:
        tb = table_bytes(eng.spec.vocab_size, max_new)
        assert tb > 48 * 1024, tb
        rep = P.PenalisedReplay(eng)
        rows = [synth.README_REVIEWS[0], synth.product_reviews(2, seed=31)[1], "ok"]
        cases = [dict(), dict(temperature=0.8, top_k=30, top_p=0.9, seed=5, min_p=0.05)]
        for kw in (cases if name == "tiny-qwen3" else cases[1:]):
            res = replay_compare(eng, rep, rows, f"{name} max_new={max_new} smem={tb}",
                                 system_prompt=SYS, max_new_tokens=max_new, ignore_eos=True,
                                 **kw, **PEN)
            assert all(len(t) == max_new for t in res.out_tokens)
            assert res.stats["rows_truncated"] == 0
    finally:
        eng.close()
        torch.cuda.empty_cache()


def test_one_call_penalised_rows_match_the_replay():
    eng, _, rep = engine("tiny-qwen3")
    replay_compare(eng, rep, ROWS, "one_call", one_call=True, system_prompt=SYS,
                   max_new_tokens=40, temperature=0.7, seed=4, min_p=0.05, **PEN)


def test_penalised_row_alone_equals_it_inside_a_shuffled_batch():
    eng, _, _ = engine("tiny-qwen3-g4")
    rng = np.random.default_rng(0)
    kw = dict(system_prompt=SYS, max_new_tokens=48, return_tokens=True, return_logprobs=True,
              temperature=0.9, seed=11, seed_per_row=True, min_p=0.02, **PEN)
    rows = synth.product_reviews(12, seed=3)
    for target in (0, 5):
        alone = eng.generate([rows[target]], row_ids=[target], **kw)
        order = rng.permutation(len(rows))
        batch = eng.generate([rows[i] for i in order], row_ids=[int(i) for i in order], **kw)
        j = int(np.flatnonzero(order == target)[0])
        assert batch.out_tokens[j] == alone.out_tokens[0]
        assert bits(batch.cum_logprobs[j]) == bits(alone.cum_logprobs[0])


def test_greedy_penalties_match_the_cpu_model():
    from oracle.bpe_ref import RefTokenizer
    from oracle.model_ref import RefModel
    eng, w, _ = engine("tiny-qwen3")
    ref_tok, model = RefTokenizer(eng.vocab), RefModel(eng.spec, w)
    tpl = VB.chat_template(eng.spec.family, SYS)
    rows = synth.README_REVIEWS + synth.product_reviews(3, seed=13)
    res = eng.generate(rows, system_prompt=SYS, max_new_tokens=24, return_tokens=True,
                       ignore_eos=True, **PEN)
    compared = 0
    for row, got in zip(rows, res.out_tokens):
        r = P.generate_penalised(model, ref_tok.render(tpl, row), 24, eng.vocab.eos_id, PEN,
                                 ignore_eos=True)
        cut = next((p for p, m in zip(r.decision_pos, r.margins) if m < 0.06), len(r.tokens))
        assert got[:cut] == r.tokens[:cut], (row, got, r.tokens, r.margins)
        compared += cut
    assert compared > 0
    print("ORACLE", f"tokens_compared={compared}")


def test_real_size_penalised_rows_match_the_replay():
    from sutro_b200.engine import LocalEngine
    spec = MS.get_spec("qwen-3-4b")
    w = MS.make_engine_weights_on_device(spec, 0, "cuda")
    v = VB.build_vocab(spec.family, spec.vocab_size, seed=0)
    eng = LocalEngine(spec, w, v, device=0, kv_pages=256, max_slots=4, max_prefill_tokens=1024,
                      logit_chunk_rows=3)
    try:
        rows = [synth.README_REVIEWS[0], synth.product_reviews(3, seed=21)[1], "ok", ""]
        replay_compare(eng, P.PenalisedReplay(eng), rows, "real_size[qwen-3-4b]",
                       system_prompt=SYS, max_new_tokens=9, ignore_eos=True, temperature=0.7,
                       seed=1, min_p=0.05,
                       **PEN)
    finally:
        eng.close()
        del eng, w
        torch.cuda.empty_cache()


def test_sdk_one_call_and_c_host_agree(tmp_path):
    from sutro_b200.bundle import export_bundle
    from sutro_b200.engine import JobC, JobStatsC, ResultC
    from sutro_b200.sdk import Sutro
    eng, _, _ = engine("tiny-llama")
    rows = synth.README_REVIEWS + ["café naïve 東京"]
    sp = dict(temperature=0.7, seed=6, min_p=0.05, max_tokens=32, **PEN)
    c = Sutro(verbose=False, cache_dir=str(tmp_path / "cache"))
    c.register_engine("m", eng)
    jid = c.infer(rows, model="m", system_prompt=SYS, sampling_params=sp, stay_attached=False)
    sdk_out = list(c.get_job_results(jid)["inference_result"])
    one = eng.infer_one_call(rows, system_prompt=SYS, max_new_tokens=32, temperature=0.7, seed=6,
                             min_p=0.05, **PEN)
    assert sdk_out == one.outputs
    # sb200_model_infer through ctypes, on a bundle of the same model
    bundle = export_bundle(eng, str(tmp_path / "bundle"))
    h = C.c_void_p()
    L.check(L.lib().sb200_model_open(bundle.encode(), 0, 8, 512, 512, C.byref(h)))
    try:
        job = JobC()
        job.truncate_rows, job.temperature, job.seed, job.min_p = 1, 0.7, 6, 0.05
        for k, val in PEN.items():
            setattr(job, k, val)
        blob = b"".join(r.encode("utf-8") for r in rows)
        off = np.zeros(len(rows) + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(r.encode("utf-8")) for r in rows])
        buf = np.frombuffer(blob, np.uint8).copy()
        res, st = C.POINTER(ResultC)(), JobStatsC()
        L.check(L.lib().sb200_model_infer(h, SYS.encode("utf-8"), None, 0, None, 32,
                                          C.byref(job), buf.ctypes.data, off.ctypes.data,
                                          len(rows), 0, C.byref(res), C.byref(st)))
        try:
            r = res.contents
            boff = np.ctypeslib.as_array(r.offsets, shape=(len(rows) + 1,)).copy()
            data = (bytes(np.ctypeslib.as_array(r.bytes, shape=(int(boff[-1]),)))
                    if boff[-1] else b"")
            c_out = [data[boff[i]:boff[i + 1]].decode("utf-8", "replace")
                     for i in range(len(rows))]
        finally:
            L.lib().sb200_result_free(res)
    finally:
        L.lib().sb200_model_close(h)
    assert c_out == one.outputs
    # and the penalties did change the job
    plain = eng.infer_one_call(rows, system_prompt=SYS, max_new_tokens=32, temperature=0.7,
                               seed=6)
    assert plain.outputs != one.outputs
