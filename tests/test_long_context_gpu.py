"""Long contexts: split-KV decode attention, dense prefill attention at 32,768 tokens, and the
engine serving rows longer than the 4,096-token split.

1. Decode kernel (sb200_attn_decode).  Rows longer than 4,096 tokens are attended in splits of
   4,096 tokens at absolute positions and merged in split order.  Outputs must meet the fp64 bound
   of test_attention_exact_gpu.py; slots past a row's context (inside its last page) hold large
   finite decoys and every page-table entry past its last page points at a NaN page, so a leak,
   at a split boundary or elsewhere, shows.  A row's output must not depend on the launch: short
   rows are bit-identical with and without long rows beside them, long rows alone, in a shuffled
   batch and beside a longer row with a wider page table (more splits in the launch).
2. Dense prefill attention at 8k, 16k and 32,768 own tokens, with and without a shared prefix,
   against fp64 on a sample of query rows that includes the last.
3. The engine with 16,384-token windows on the tiny models: rows of ~5k, 9k and 15k tokens among
   short ones, bit-identical to the one-row replay (tests/engine_replay.py) greedy, sampled and
   under a schema with jump-forward; rows that cross a split boundary during decode (4,096 ->
   4,097 and 8,192 -> 8,193 tokens of context) while the number of split rows and of splits grows
   within a job and from job to job; a system prompt longer than 4,096 tokens (every row split);
   greedy tokens against the CPU oracle; truncation past the window.
4. Real size: qwen-3-4b (~30k-token row) and llama-3.1-8b (~20k) against the replay, and
   `Sutro.infer` with default engine options serving a 20k-token row untruncated.
"""
import dataclasses
import random

import numpy as np
from typing import Literal

import pytest
import torch
from pydantic import BaseModel

import kv_layout as KV
import test_attention_exact_gpu as AX
from engine_replay import Replay
from oracle.bpe_ref import RefTokenizer
from sutro_b200 import modelspec as MS
from sutro_b200 import synth, vocab as VB

pytestmark = pytest.mark.gpu

DEV = "cuda"
HD, PAGE = KV.HD, KV.PAGE
SPLIT = 4096
LONG = [4097, 4111, 8192, 8193, 12289, 32767, 32768]
SHORT = [1, 17, 300, 4095, 4096]


# --------------------------------------------------------------------------- 1. decode kernel
def paged_rows(lens, hkv, seed):
    """Per-row K/V [L, hkv, 128] in a pool of shuffled pages.  Slots past a row's end inside its
    last page hold finite decoys (keys 30 along every dim, values +-1000); the page-table entries
    past a row's last page point at a page of NaN.  -> (pool, page table [n, max_pages], ks, vs)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    n_pages = [(n + PAGE - 1) // PAGE for n in lens]
    total = sum(n_pages) + 1
    perm = torch.randperm(total, generator=torch.Generator().manual_seed(seed))
    nan_page = int(perm[-1])
    pt = torch.full((len(lens), max(n_pages) + 2), nan_page, dtype=torch.int32)
    logical = torch.empty(total, hkv, 2, PAGE, HD, dtype=torch.bfloat16, device=DEV)
    logical[:, :, 0] = 30.0
    logical[:, :, 1] = AX.bf(1000 * torch.where(
        torch.rand(total, hkv, PAGE, HD, device=DEV, generator=g) < 0.5, -1.0, 1.0))
    logical[nan_page] = float("nan")
    ks, vs, at = [], [], 0
    for i, n in enumerate(lens):
        pages = perm[at:at + n_pages[i]]
        at += n_pages[i]
        pt[i, :n_pages[i]] = pages.to(torch.int32)
        k = AX.bf(torch.randn(n, hkv, HD, device=DEV, generator=g))
        v = AX.bf(torch.randn(n, hkv, HD, device=DEV, generator=g))
        pos = torch.arange(n, device=DEV)
        pg, r = pages.to(DEV)[pos // PAGE], pos % PAGE
        logical[pg, :, 0, r] = k
        logical[pg, :, 1, r] = v
        ks.append(k)
        vs.append(v)
    return KV.pack_tile(logical), pt, ks, vs


def decode(qkv, pool, pt, rows, lens, hq, hkv, width=None):
    """sb200_attn_decode of batch rows `rows` (indices into the page table) with contexts lens.
    `width` sets the page table's width, which bounds the contexts and so the launch's splits:
    columns are cut, or padded with the NaN page."""
    if width is not None and width > pt.shape[1]:
        pad = pt[:, -1:].expand(-1, width - pt.shape[1])
        pt = torch.cat([pt, pad], 1)
    elif width is not None:
        pt = pt[:, :width].contiguous()
    return AX.run_decode(qkv, pool, pt, rows, [lens[r] for r in rows], hq, hkv)


@pytest.mark.parametrize("hq,hkv", AX.HEADS, ids=AX.HEAD_IDS)
def test_split_decode_within_fp64_bound_and_no_leaks(hq, hkv):
    lens = LONG + SHORT
    pool, pt, ks, vs = paged_rows(lens, hkv, seed=hq + hkv)
    rows = list(range(len(lens)))
    torch.manual_seed(hq)
    qkv = AX.bf(torch.randn(len(rows), (hq + 2 * hkv) * HD, device=DEV))
    out = decode(qkv, pool, pt, rows, lens, hq, hkv)
    refs = [AX.attn_ref64(qkv[b:b + 1, :hq * HD].view(1, hq, HD), ks[b], vs[b], [lens[b]], hkv)
            for b in rows]
    for b in rows:
        AX.assert_within_bound(out[b:b + 1], refs[b][0], refs[b][1],
                               f"split decode G{hq // hkv} ctx {lens[b]}")


@pytest.mark.parametrize("hq,hkv", AX.HEADS, ids=AX.HEAD_IDS)
def test_split_decode_is_batch_invariant(hq, hkv):
    lens = LONG + SHORT
    pool, pt, ks, vs = paged_rows(lens, hkv, seed=7 + hq)
    n = len(lens)
    torch.manual_seed(100 + hq)
    q = AX.bf(torch.randn(n, (hq + 2 * hkv) * HD, device=DEV))
    short = [lens.index(x) for x in SHORT]
    # the batch's q rows follow `rows`; results are compared per page-table row
    def run(rows, width=None):
        return decode(q[rows].contiguous(), pool, pt, rows, lens, hq, hkv, width)

    full = run(list(range(n)))
    # short rows alone (no split in the launch) and beside the long rows
    alone_short = run(short, width=SPLIT // PAGE)
    for j, r in enumerate(short):
        assert torch.equal(alone_short[j], full[r]), ("short row changed by long rows", lens[r])
    rng = random.Random(hq)
    shuffled = list(range(n))
    rng.shuffle(shuffled)
    shuf = run(shuffled)
    for j, r in enumerate(shuffled):
        assert torch.equal(shuf[j], full[r]), ("shuffled batch", lens[r])
    for r, length in enumerate(lens):
        if length <= SPLIT:
            continue
        alone = run([r], width=(length + PAGE - 1) // PAGE)
        assert torch.equal(alone[0], full[r]), ("long row alone", length)
    # beside the 32,768-token row with a wider page table: more splits in the launch
    longest = lens.index(32768)
    for r in (lens.index(4097), lens.index(12289)):
        pair = run([longest, r], width=pt.shape[1] + 300)
        assert torch.equal(pair[1], full[r]), ("beside a longer row", lens[r])


def test_split_decode_many_short_rows_beside_one_long():
    """The mixed batch of a long job: one 32,768-token row among 2,000 short rows; the short rows
    match a launch without the long row bit for bit."""
    hq, hkv = 32, 8
    lens = [32768] + [1 + (37 * i) % 200 for i in range(2000)]
    pool, pt, ks, vs = paged_rows(lens, hkv, seed=3)
    torch.manual_seed(3)
    q = AX.bf(torch.randn(len(lens), (hq + 2 * hkv) * HD, device=DEV))
    rows = list(range(len(lens)))
    full = decode(q, pool, pt, rows, lens, hq, hkv)
    short = decode(q[1:].contiguous(), pool, pt, rows[1:], lens, hq, hkv, width=SPLIT // PAGE)
    assert torch.equal(full[1:], short)
    ref, mag = AX.attn_ref64(q[:1, :hq * HD].view(1, hq, HD), ks[0], vs[0], [lens[0]], hkv)
    AX.assert_within_bound(full[:1], ref, mag, "32k row among 2000 short rows")


# --------------------------------------------------------------------------- 2. dense prefill
@pytest.mark.parametrize("own,past", [(8192, 0), (8192, 1000), (16384, 0), (16384, 1000),
                                      (32768, 0), (32768, 777)])
@pytest.mark.parametrize("hq,hkv", AX.HEADS, ids=AX.HEAD_IDS)
def test_dense_prefill_long_rows_within_fp64_bound(hq, hkv, own, past):
    G, n_layers, layer = hq // hkv, 2, 1
    torch.manual_seed(own + past + G)
    qkv = AX.bf(torch.randn(own + 32, (hq + 2 * hkv) * HD, device=DEV))
    qkv[own:] = 0          # rows past the sequence, as the engine leaves them
    pre = None
    if past:
        pre = AX.bf(torch.randn(n_layers, past, 2 * hkv * HD, device=DEV))
    out = AX.run_dense(qkv, pre, past, n_layers, layer, [(past, own)], hq, hkv)
    k_own = qkv[:own, hq * HD:(hq + hkv) * HD].view(own, hkv, HD)
    v_own = qkv[:own, (hq + hkv) * HD:].view(own, hkv, HD)
    if past:
        k = torch.cat([pre[layer, :, :hkv * HD].view(past, hkv, HD), k_own])
        v = torch.cat([pre[layer, :, hkv * HD:].view(past, hkv, HD), v_own])
    else:
        k, v = k_own, v_own
    sample = sorted(set(torch.randint(0, own, (40,)).tolist()) | {0, own // 2, own - 1})
    idx = torch.tensor(sample, device=DEV)
    q = qkv[idx, :hq * HD].view(-1, hq, HD)
    ref, mag = AX.attn_ref64(q, k, v, (past + 1 + idx).tolist(), hkv)
    AX.assert_within_bound(out[idx], ref, mag, f"dense prefill G{G} own {own} past {past}")


# --------------------------------------------------------------------------- 3. engine (tiny)
class Sentiment(BaseModel):
    sentiment: Literal["positive", "neutral", "negative"]


def long_text(ref, n_tokens, seed):
    """About n_tokens tokens of synthetic prose."""
    words = " ".join(synth.documents(max(2, n_tokens // 250), seed=seed, words=400)).split()
    while len(words) < 2 * n_tokens:
        words = words + words
    k = n_tokens
    for _ in range(3):
        got = len(ref.encode(" ".join(words[:k])))
        k = max(1, int(k * n_tokens / max(got, 1)))
    return " ".join(words[:k])


def tiny_engine(name, window=16384, **kw):
    from sutro_b200.engine import LocalEngine
    spec = dataclasses.replace(MS.get_spec(name), max_position=window)
    w = MS.make_weights(spec, seed=0, std=0.05)
    v = VB.build_vocab(spec.family, spec.vocab_size, seed=0, n_trained=600)
    kw.setdefault("kv_pages", 4096)
    kw.setdefault("max_slots", 16)
    return LocalEngine(spec, MS.pack_for_engine(spec, w, DEV), v, device=0, **kw), w


def bits(t):
    t = t if torch.is_tensor(t) else torch.from_numpy(np.asarray(t, dtype=np.float32))
    return t.to(torch.float32).contiguous().view(torch.int32)


def compare(eng, rows, label, rep=None, **kw):
    """Every row of the engine job bit-identical to its one-row replay."""
    rep = rep or Replay(eng)
    res = eng.generate(rows, return_tokens=True, return_first_logits=True, return_logprobs=True,
                       **kw)
    reps = rep.job(rows, **kw)
    for i, r in enumerate(reps):
        assert res.out_tokens[i] == r.tokens, (label, i, res.out_tokens[i], r.tokens)
        assert torch.equal(bits(res.first_logits[i]), bits(r.first_logits)), (label, i)
        assert bits(res.cum_logprobs[i]).item() == bits(r.cum_logprob).item(), (label, i)
    print("LONG_PARITY", label, [r.prompt_len for r in reps], res.stats["rows_truncated"],
          res.stats["decode_steps"])
    assert res.stats["rows_truncated"] == 0, label
    return res, reps


@pytest.mark.parametrize("name", ["tiny-qwen3-g4", "tiny-llama"])
def test_engine_long_rows_match_replay(name):
    eng, _ = tiny_engine(name)
    try:
        ref = RefTokenizer(eng.vocab)
        longs = [long_text(ref, n, seed=40 + i) for i, n in enumerate((5000, 9000, 15000))]
        shorts = synth.product_reviews(5, seed=11)
        rows = [shorts[0], longs[0], shorts[1], longs[1], shorts[2], longs[2], shorts[3]]
        rep = Replay(eng)
        _, reps = compare(eng, rows, f"{name} greedy", rep, max_new_tokens=12, ignore_eos=True)
        assert max(r.prompt_len for r in reps) > 3 * SPLIT
        compare(eng, rows, f"{name} sampled", rep, max_new_tokens=12, temperature=0.8, top_p=0.9,
                seed=5)
        compare(eng, rows, f"{name} schema", rep, system_prompt=synth.README_SYSTEM_PROMPT,
                json_schema=Sentiment.model_json_schema(), max_new_tokens=16)
    finally:
        eng.close()


def exact_row(ref, tpl, n_prompt, seed):
    """A row of prose whose rendered prompt (prefix | row | suffix) is exactly n_prompt tokens."""
    n_body = n_prompt - len(ref.encode_pieces(tpl.prefix)) - len(ref.encode_pieces(tpl.suffix))
    text = long_text(ref, n_body + 300, seed)
    assert len(ref.encode(text)) > n_body
    lo, hi = 0, len(text)
    while lo < hi:                          # the shortest cut with at least n_body tokens
        mid = (lo + hi) // 2
        if len(ref.encode(text[:mid])) >= n_body:
            hi = mid
        else:
            lo = mid + 1
    for c in range(max(0, lo - 8), lo + 64):
        if len(ref.encode(text[:c])) == n_body:
            assert len(ref.render(tpl, text[:c])) == n_prompt
            return text[:c]
    raise AssertionError(f"no cut of the text renders to {n_prompt} tokens")


def split_schedule(reps):
    """Per decode step, (rows attended in splits, most splits of a row), when every row decodes
    from its first step on; a row's context in decode step t is prompt + 1 + t."""
    out = []
    for t in range(max(r.decode_steps for r in reps)):
        ctx = [r.prompt_len + 1 + t for r in reps if t < r.decode_steps]
        n = [-(-c // SPLIT) for c in ctx]
        out.append((sum(k > 1 for k in n), max(n)))
    return out


def test_engine_rows_cross_a_split_during_decode():
    """Rows whose context crosses 4,096 -> 4,097 in their first, second or ninth decode step, and
    8,192 -> 8,193, beside short rows, greedy and sampled; then, on the same engine, a job with
    fewer split rows (the grown split workspace reused) and one with more rows and splits (grown
    again).  Every row bit-identical to its replay."""
    eng, _ = tiny_engine("tiny-qwen3-g4")
    try:
        ref = RefTokenizer(eng.vocab)
        tpl = VB.chat_template(eng.spec.family, None)
        shorts = synth.product_reviews(3, seed=14)
        sizes = [4095, 4096, 4088, 8190]
        rows = [exact_row(ref, tpl, n, seed=100 + i) for i, n in enumerate(sizes)]
        rows = [shorts[0], rows[0], rows[1], shorts[1], rows[2], rows[3]]
        rep = Replay(eng)
        kw = dict(max_new_tokens=16, ignore_eos=True)
        _, reps = compare(eng, rows, "split crossing greedy", rep, **kw)
        assert [reps[i].prompt_len for i in (1, 2, 4, 5)] == sizes
        for i, bound in ((1, SPLIT), (2, SPLIT), (4, SPLIT), (5, 2 * SPLIT)):
            P, steps = reps[i].prompt_len, reps[i].decode_steps
            assert P <= bound < P + steps, (P, steps, bound)   # crossed in decode
        sched = split_schedule(reps)
        assert sched[0] == (2, 2) and sched[-1] == (4, 3), sched   # rows and splits both rise
        compare(eng, rows, "split crossing sampled", rep, temperature=0.8, top_p=0.9, seed=7, **kw)
        # fewer split rows: the workspace the first job grew is reused
        few = [shorts[2], exact_row(ref, tpl, 4100, seed=110)]
        _, reps = compare(eng, few, "fewer split rows", rep, **kw)
        assert max(n for n, _ in split_schedule(reps)) == 1
        # more split rows and more splits than the first job: it grows again
        more = [exact_row(ref, tpl, n, seed=120 + i)
                for i, n in enumerate((4090, 5000, 6000, 8185, 9000, 12286))] + [shorts[0]]
        _, reps = compare(eng, more, "more split rows", rep, temperature=0.7, seed=3, **kw)
        sched = split_schedule(reps)
        assert sched[0] == (5, 3) and sched[-1] == (6, 4), sched
    finally:
        eng.close()


def test_engine_system_prompt_longer_than_a_split():
    """A 5k-token system prompt: every row is split, the shared prefix is cached once."""
    eng, _ = tiny_engine("tiny-qwen3-g4")
    try:
        ref = RefTokenizer(eng.vocab)
        sp = long_text(ref, 5000, seed=60)
        rows = synth.product_reviews(6, seed=12) + [long_text(ref, 3000, seed=61)]
        res, reps = compare(eng, rows, "long system prompt", system_prompt=sp, max_new_tokens=10,
                            ignore_eos=True)
        assert res.stats["prefix_cached_tokens"] > SPLIT
        assert min(r.prompt_len for r in reps) > SPLIT
    finally:
        eng.close()


def test_engine_long_row_greedy_matches_cpu_oracle():
    from oracle.model_ref import RefModel
    eng, w = tiny_engine("tiny-qwen3-g4")
    try:
        ref = RefTokenizer(eng.vocab)
        row = long_text(ref, 8000, seed=70)
        res = eng.generate([row], max_new_tokens=8, return_tokens=True)
        assert res.stats["rows_truncated"] == 0
        tpl = VB.chat_template(eng.spec.family, None)
        prompt = ref.render(tpl, row)
        assert len(prompt) > 7000
        r = RefModel(eng.spec, w).generate(prompt, 8, eng.vocab.eos_id)
        cut = next((p for p, m in zip(r.decision_pos, r.margins) if m < 0.06), len(r.tokens))
        print("LONG_ORACLE", len(prompt), cut, res.out_tokens[0], r.tokens)
        assert res.out_tokens[0][:cut] == r.tokens[:cut]
    finally:
        eng.close()


def test_engine_row_past_the_window_is_truncated_or_refused():
    eng, _ = tiny_engine("tiny-qwen3-g4", window=8192)
    try:
        ref = RefTokenizer(eng.vocab)
        rows = [long_text(ref, 9000, seed=80), "short row"]
        res = eng.generate(rows, max_new_tokens=8, return_tokens=True)
        assert res.stats["rows_truncated"] == 1
        with pytest.raises(Exception, match="truncate_rows=False"):
            eng.generate(rows, max_new_tokens=8, truncate_rows=False)
    finally:
        eng.close()


# --------------------------------------------------------------------------- 4. real size
@pytest.mark.parametrize("name,n_long", [("qwen-3-4b", 30000), ("llama-3.1-8b", 20000)])
def test_real_size_long_row_matches_replay(name, n_long):
    from sutro_b200.engine import LocalEngine
    spec = MS.get_spec(name)
    assert spec.max_position == 32768
    w = MS.make_engine_weights_on_device(spec, 0, DEV)
    v = VB.build_vocab(spec.family, spec.vocab_size, seed=0)
    eng = LocalEngine(spec, w, v, device=0, kv_pages=2560, max_slots=8)
    try:
        ref = RefTokenizer(v)
        rows = [synth.README_REVIEWS[0], long_text(ref, n_long, seed=90), "ok",
                synth.README_REVIEWS[1]]
        _, reps = compare(eng, rows, f"{name} long row", max_new_tokens=8, ignore_eos=True)
        assert reps[1].prompt_len > n_long * 0.9
        assert all(r.decode_steps == 7 for r in reps)
    finally:
        eng.close()
        del eng, w
        torch.cuda.empty_cache()


def test_sdk_default_engine_serves_a_20k_row_untruncated(tmp_path):
    """Default engine options: the prefill budget holds a full-window row."""
    import pandas as pd
    from sutro_b200.interfaces import JobStatus
    from sutro_b200.sdk import Sutro
    so = Sutro(verbose=False, cache_dir=str(tmp_path))
    eng = so._engine("qwen-3-4b")
    try:
        assert eng.max_prefill_tokens == 32768
        row = long_text(RefTokenizer(eng.vocab), 20000, seed=95)
        df = pd.DataFrame({"text": [row, "fine"]})
        job_id = so.infer(df, model="qwen-3-4b", column="text",
                          sampling_params={"max_new_tokens": 4})
        st = so._job(job_id).stats
        print("SDK_LONG", st["input_tokens"], st["rows_truncated"])
        assert so.get_job_status(job_id) == JobStatus.SUCCEEDED
        assert st["rows_truncated"] == 0 and st["input_tokens"] > 18000
    finally:
        eng.close()
