"""Rows longer than the prefill budget, prefilled in chunks, on tiny models whose windows are
raised past their registered ones (YaRN for the Qwen3 ones).  Every row must be bit-identical to
the one-row replay (tests/engine_replay.py), which prefills each row in one step: the chunk
boundaries are multiples of the attention's history granularity, so the chunked prefill makes
exactly the same arithmetic as an unchunked one.  The same rows through an engine whose budget
holds a whole row must match the replay too."""
import random

import pytest
import torch

import test_engine_replay_gpu as ER
import test_long_context_gpu as LC
from engine_replay import Replay
from oracle.bpe_ref import RefTokenizer
from sutro_b200 import _lib as L
from sutro_b200 import modelspec as MS
from sutro_b200 import synth, vocab as VB

pytestmark = pytest.mark.gpu

# model -> (window, chunked budget): rows of up to ~window tokens chunk 2-10 times
MODELS = {"tiny-qwen3": (2048, 256), "tiny-qwen3-g4": (4096, 512),
          "tiny-qwen3-g5": (4096, 3200), "tiny-llama": (2048, 256),
          "tiny-qwen3-embedding": (2048, 384)}
_ENGINES = {}
_WEIGHTS = {}


def engine(name, budget=None, **kw):
    window, chunked_budget = MODELS[name]
    key = (name, budget, tuple(sorted(kw.items())))
    if key not in _ENGINES:
        from sutro_b200.engine import LocalEngine
        spec = MS.with_window(MS.get_spec(name), window)
        w = MS.make_weights(spec, seed=0, std=0.05)
        v = VB.build_vocab(spec.family, spec.vocab_size, seed=0, n_trained=600)
        kw.setdefault("kv_pages", 4096)
        kw.setdefault("max_slots", 8)
        eng = LocalEngine(spec, MS.pack_for_engine(spec, w, "cuda"), v, device=0,
                          max_prefill_tokens=budget or chunked_budget, **kw)
        _ENGINES[key] = (eng, Replay(eng))
        _WEIGHTS[key] = w
    return _ENGINES[key]


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for eng, _ in _ENGINES.values():
        eng.close()
    _ENGINES.clear()
    _WEIGHTS.clear()
    torch.cuda.empty_cache()


def long_rows(eng, sizes, seed):
    ref = RefTokenizer(eng.vocab)
    return [LC.long_text(ref, n, seed=seed + i) for i, n in enumerate(sizes)]


def mixed_rows(eng, seed=0):
    """Short rows around long ones: the long rows chunk 2-10 times at the chunked budget."""
    window = eng.spec.max_position
    longs = long_rows(eng, (int(window * 0.9), window // 2), seed=60 + seed)
    shorts = synth.product_reviews(5, seed=20 + seed)
    return [shorts[0], longs[0], shorts[1], shorts[2], longs[1], shorts[3], shorts[4]]


def chunk_count(eng, rep, row):
    n = len(rep.ref.render(rep.template(None), row))
    align = L.lib().sb200_attn_prefill_hist_align(eng.spec.n_q_heads, eng.spec.n_kv_heads)
    c = eng.max_prefill_tokens // align * align
    return n, -(-n // c) if n > eng.max_prefill_tokens else 1


@pytest.mark.parametrize("name", sorted(MODELS))
def test_chunked_rows_match_the_replay(name):
    eng, rep = engine(name)
    rows = mixed_rows(eng)
    counts = [chunk_count(eng, rep, r)[1] for r in rows]
    assert 2 <= max(counts) <= 10, counts
    emb = eng.spec.embedding_model
    kw = {} if emb else dict(max_new_tokens=12, ignore_eos=True)
    rec = ER.compare(eng, rows, f"{name} chunked greedy", rep=rep, **kw)
    assert rec["truncated"] == 0
    if emb:
        return
    ER.compare(eng, rows, f"{name} chunked sampled", rep=rep, max_new_tokens=12, temperature=0.8,
               top_p=0.9, seed=5, seed_per_row=True)
    # a budget that holds the whole row: the same engine path without chunks
    whole, wrep = engine(name, budget=eng.spec.max_position)
    ER.compare(whole, rows, f"{name} whole-row greedy", rep=wrep, **kw)


@pytest.mark.parametrize("share", [True, False])
@pytest.mark.parametrize("n_prefix", [15, 16, 17, 46])
def test_prefix_lengths_with_chunked_rows(n_prefix, share):
    eng, rep = engine("tiny-qwen3-g4")
    sp = ER.prompt_with_prefix(rep, n_prefix)
    rows = mixed_rows(eng, seed=n_prefix)
    rec = ER.compare(eng, rows, f"chunked prefix[{n_prefix},share={share}]", rep=rep,
                     system_prompt=sp, max_new_tokens=10, ignore_eos=True, share_prefix=share)
    assert (rec["tail_copy_rows"] > 0) == (share and n_prefix % 16 != 0 and n_prefix > 16)


@pytest.mark.parametrize("jump", [True, False])
def test_schema_jobs_with_chunked_rows(jump):
    eng, rep = engine("tiny-qwen3")
    rows = mixed_rows(eng, seed=3)
    rec = ER.compare(eng, rows, f"chunked schema[jump={jump}]", rep=rep, system_prompt=ER.SYS,
                     json_schema=ER.SentimentEnum.model_json_schema(), fsm_limits=ER.LIM,
                     max_new_tokens=32, jump_forward=jump)
    assert (rec["forced_prefix_tokens"] > 0) == jump, rec


@pytest.mark.parametrize("slots", [1, 3, 8])
def test_slot_counts_with_chunked_rows(slots):
    eng, rep = engine("tiny-qwen3-g4", max_slots=slots)
    rows = mixed_rows(eng, seed=slots)
    ER.compare(eng, rows, f"chunked slots={slots}", rep=rep, max_new_tokens=20, temperature=0.7,
               seed=9)


def test_kv_pool_holding_two_rows():
    """The pool holds two full-window rows: admission waits for pages between chunked rows."""
    window = MODELS["tiny-qwen3-g4"][0]
    eng, rep = engine("tiny-qwen3-g4", kv_pages=2 * (window // 16 + 2), max_slots=4)
    rows = long_rows(eng, (3500, 3000, 3700), seed=90) + synth.product_reviews(2, seed=4)
    rec = ER.compare(eng, rows, "chunked two-row pool", rep=rep, max_new_tokens=16,
                     ignore_eos=True)
    assert rec["prefill_steps"] > 6, rec


def test_chunks_interleave_with_decoding_rows():
    """Short rows decode while a long row is prefilled chunk by chunk.  The shorts take the
    first step and the long row's first chunk the next; every later chunk follows one decode step
    of the shorts, and the long row then needs its own 39 decode steps.  So the job takes
    (chunks - 1) + 39 decode steps; chunks run back to back would take 39."""
    eng, rep = engine("tiny-qwen3-g4", max_slots=8)
    shorts = synth.product_reviews(3, seed=8)
    rows = shorts + long_rows(eng, (3900,), seed=77)
    res = eng.generate(rows, max_new_tokens=40, ignore_eos=True, return_tokens=True)
    n, chunks = chunk_count(eng, rep, rows[-1])
    assert chunks >= 7
    # the shorts fill the first step (with the first chunk they would exceed the budget)
    assert res.stats["prefill_steps"] == chunks + 1
    assert res.stats["decode_steps"] == (chunks - 1) + 39, (res.stats["decode_steps"], chunks)
    ER.compare(eng, rows, "chunked interleave", rep=rep, max_new_tokens=40, ignore_eos=True)


def test_shuffled_batch_changes_nothing():
    eng, _ = engine("tiny-qwen3-g5")
    rows = mixed_rows(eng, seed=11)
    kw = dict(max_new_tokens=10, temperature=0.9, seed=3, seed_per_row=True)
    a = eng.generate(rows, return_tokens=True, return_first_logits=True, **kw)
    perm = list(range(len(rows)))
    random.Random(2).shuffle(perm)
    b = eng.generate([rows[i] for i in perm], row_ids=perm, return_tokens=True,
                     return_first_logits=True, **kw)
    for j, i in enumerate(perm):
        assert b.out_tokens[j] == a.out_tokens[i]
        assert torch.equal(ER.bits(b.first_logits[j]), ER.bits(a.first_logits[i]))


def test_row_past_the_window_is_truncated_or_refused():
    eng, _ = engine("tiny-qwen3")
    row = long_rows(eng, (2300,), seed=5)[0]
    res = eng.generate([row], max_new_tokens=8, ignore_eos=True)
    assert res.stats["rows_truncated"] == 1
    with pytest.raises(L.Sb200Error, match="fit the context window"):
        eng.generate([row], max_new_tokens=8, truncate_rows=False)


def test_greedy_on_the_tiny_yarn_model_matches_the_oracle():
    """tiny-qwen3 at 2,048 positions (YaRN x4 over 512), a ~1,900-token row prefilled in 8
    chunks: greedy tokens equal RefModel's up to its first decision with a top-2 margin under
    0.06 (the bar of test_engine_gpu.py)."""
    from oracle.model_ref import RefModel
    eng, rep = engine("tiny-qwen3")
    w = _WEIGHTS[("tiny-qwen3", None, ())]
    row = long_rows(eng, (1850,), seed=31)[0]
    n, chunks = chunk_count(eng, rep, row)
    assert chunks >= 7 and n > 1800
    res = eng.generate([row], max_new_tokens=8, return_tokens=True)
    prompt = rep.ref.render(rep.template(None), row)
    r = RefModel(eng.spec, w).generate(prompt, 8, eng.vocab.eos_id)
    cut = next((p for p, m in zip(r.decision_pos, r.margins) if m < 0.06), len(r.tokens))
    print("YARN_ORACLE", len(prompt), cut, res.out_tokens[0], r.tokens)
    assert cut > 0
    assert res.out_tokens[0][:cut] == r.tokens[:cut]
