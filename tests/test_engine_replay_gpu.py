"""Every row of an engine job, in every scheduling geometry, against a one-row replay of the
verified kernels (tests/engine_replay.py): tokens equal, first-decision fp32 logits and fp32
cumulative log-probabilities bit-identical (compared as int32 views), embeddings bit-identical.

No tolerance is involved: the kernels are individually verified and batch-invariant, so any
difference is a scheduler mistake (a wrong position, ctx_len, page, prefix tail, slot or chunk)
or a replay that misreads the engine's contract.  The cumulative log-probability sums every
decode step's log-softmax, so one changed bit in any step's logits changes it.

Each test prints one PARITY line: rows compared, decode steps replayed, and the nonzero
counters of the paths the case is meant to reach (`tail_copy`, `page_wait`, `chunked`, `forced`,
EOS stops, truncated rows, prefill steps).  Every counter comes from the engine's own
job statistics: `tail_copy_rows` from the prefix it cached (a prefix that does not end on a page
boundary is tail-copied into every row), `chunked_head_launches` from the sampler launches beyond
one per prefill or decode step, `page_wait_admissions` from the prefill steps beyond the first
when neither the slots nor the prefill budget can split the admission, `forced_prefix_tokens`
from the jump-forward plan.  The case asserts that its own counters are nonzero, so no case
passes vacuously.

Not covered: the branch of the engine's admission where a prompt ends inside the shared prefix.
Chat templates always end in a non-empty suffix, so no public call reaches it.
"""
from typing import List, Literal

import numpy as np
import pytest
import torch
from pydantic import BaseModel, Field

from engine_replay import PAGE, Replay
from oracle.bpe_ref import RefTokenizer
from sutro_b200 import modelspec as MS
from sutro_b200 import synth, vocab as VB
from sutro_b200.schema_fsm import FsmLimits

pytestmark = pytest.mark.gpu

SYS = synth.README_SYSTEM_PROMPT
LIM = FsmLimits(max_string_chars=8, max_array_items=2)


class SentimentEnum(BaseModel):
    sentiment: Literal["positive", "neutral", "negative"]


class Extract(BaseModel):
    name: str = Field(max_length=8)
    qty: int = Field(ge=0, le=20)
    tags: List[Literal["a", "b"]] = Field(max_length=2)


# ---------------------------------------------------------------------------- set-up helpers
def build(name, eos_alias=None, **kw):
    """A tiny model with the weights test_engine_gpu.py uses.  `eos_alias=t`: the EOS row of the
    LM head becomes 1.05 x the row of token t, so greedy decoding stops exactly where it would
    have emitted t (rows that never reach t run to max_new_tokens)."""
    from sutro_b200.engine import LocalEngine
    spec = MS.get_spec(name)
    w = MS.make_weights(spec, seed=0, std=0.05)
    v = VB.build_vocab(spec.family, spec.vocab_size, seed=0, n_trained=600)
    if eos_alias is not None:
        key = "model.embed_tokens.weight" if spec.tied_embeddings else "lm_head.weight"
        w[key] = w[key].clone()
        w[key][v.eos_id] = w[key][eos_alias].float().mul(1.05).to(w[key].dtype)
    kw.setdefault("kv_pages", 512)
    return LocalEngine(spec, MS.pack_for_engine(spec, w, "cuda"), v, device=0, **kw)


def residue_rows(ref: RefTokenizer, seed=5):
    """16 rows whose token counts cover every residue mod 16 (so do the prompt lengths)."""
    words = " ".join(synth.documents(2, seed=seed, words=200)).split()
    got = {}
    for k in range(1, len(words)):
        row = " ".join(words[k % 7:k % 7 + k])
        got.setdefault(len(ref.encode(row)) % PAGE, row)
        if len(got) == PAGE:
            return [got[i] for i in range(PAGE)]
    raise AssertionError("no row for some residue")


def prompt_with_prefix(rep, n_prefix):
    """A system prompt whose rendered template prefix is exactly n_prefix tokens long."""
    words = " ".join(synth.product_reviews(3, seed=31)).split()
    for tail in ("", ".", " ok", "!", " x y"):
        for k in range(0, 40):
            sp = " ".join(words[:k]) + tail
            if sp and len(rep.framing(sp)[0]) == n_prefix:
                return sp
    raise AssertionError(f"no system prompt renders to a {n_prefix}-token prefix")


def bits(t):
    """fp32 values as their int32 bit patterns (bitwise comparison; NaN != NaN is avoided)."""
    t = t if torch.is_tensor(t) else torch.from_numpy(np.asarray(t, dtype=np.float32))
    return t.to(torch.float32).contiguous().view(torch.int32)


def compare(eng, rows, label, one_call=False, rep=None, **kw):
    """Run the job on the engine and replay every row; returns the counters of the PARITY line."""
    rep = rep or Replay(eng)
    emb = eng.spec.embedding_model
    if one_call:
        res = eng.infer_one_call(rows, return_logprobs=not emb, **kw)
    else:
        res = eng.generate(rows, return_tokens=True, return_first_logits=not emb,
                           return_logprobs=not emb, **kw)
    reps = rep.job(rows, **kw)
    st = res.stats
    for i, r in enumerate(reps):
        if emb:
            assert torch.equal(bits(res.embeddings[i]), bits(r.embedding)), (label, i)
            continue
        assert res.out_tokens[i] == r.tokens, (label, i, res.out_tokens[i], r.tokens)
        if not one_call:
            got = res.first_logits[i]
            diff = (bits(got) != bits(r.first_logits)).sum().item()
            assert diff == 0, (label, i, "first logits differ", diff,
                               (got - r.first_logits).abs().max().item())
        assert bits(res.cum_logprobs[i]).item() == bits(r.cum_logprob).item(), \
            (label, i, float(res.cum_logprobs[i]), float(r.cum_logprob))
    n_prefix = len(rep.framing(kw.get("system_prompt"))[0])
    share = kw.get("share_prefix", True)
    cached = n_prefix if (share and n_prefix >= PAGE and not emb) else 0
    assert st["prefix_cached_tokens"] == cached, (label, st["prefix_cached_tokens"], cached)
    max_new = kw.get("max_new_tokens", 64)
    # the engine copies the prefix's partial last page into every row iff it caches a prefix
    # that does not end on a page boundary
    tail_copy = len(rows) if st["prefix_cached_tokens"] % PAGE else 0
    # every head_and_sample call launches one sampler per chunk of logit_chunk_rows rows
    heads = st["prefill_steps"] + st["decode_steps"]
    chunked = 0 if one_call or emb else st["kernel_launches"]["sample"] - heads
    # when neither the slots nor the prefill budget bind, the first admission takes every row
    # unless the KV pool runs out: each further prefill step is an admission that waited for pages
    new_tokens = sum(r.prompt_len - cached for r in reps)
    unbound = eng.max_slots >= len(rows) and new_tokens <= eng.max_prefill_tokens
    page_wait = st["prefill_steps"] - 1 if unbound and not emb else 0
    rec = {"rows": len(rows), "steps": sum(r.decode_steps for r in reps),
           "tail_copy_rows": tail_copy, "page_wait_admissions": page_wait,
           "chunked_head_launches": chunked,
           "forced_prefix_tokens": st.get("forced_prefix_tokens", 0),
           # without a schema a row ends before max_new_tokens only on EOS
           "eos_stops": sum(len(r.tokens) < max_new for r in reps)
           if not emb and kw.get("json_schema") is None else 0,
           "max_new_stops": sum(len(r.tokens) == max_new for r in reps) if not emb else 0,
           "truncated": st["rows_truncated"], "prefill_steps": st["prefill_steps"]}
    short = {"rows": "rows", "steps": "steps", "tail_copy_rows": "tail_copy",
             "page_wait_admissions": "page_wait", "chunked_head_launches": "chunked",
             "forced_prefix_tokens": "forced", "eos_stops": "eos", "truncated": "truncated",
             "prefill_steps": "prefills"}
    print("PARITY", label, " ".join(f"{short[k]}={rec[k]}" for k in short
                                    if rec[k] or k in ("rows", "steps")))
    return rec


_ENGINES = {}


def engine(name, **kw):
    """Engines are reused across the tests of this file: later jobs then run on recycled pages
    and slots, as a long-lived engine does."""
    key = (name, tuple(sorted(kw.items())))
    if key not in _ENGINES:
        eng = build(name, **kw)
        _ENGINES[key] = (eng, Replay(eng))
    return _ENGINES[key]


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for eng, _ in _ENGINES.values():
        eng.close()
    _ENGINES.clear()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------- the cases
@pytest.mark.parametrize("name", ["tiny-qwen3", "tiny-qwen3-g4", "tiny-llama"])
def test_models_match_the_replay(name):
    """q/k-norm (qwen3), GQA 4 (g4), llama-3.1 RoPE scaling; greedy, every prompt residue,
    decode across at least two page boundaries."""
    eng, rep = engine(name, max_slots=8, max_prefill_tokens=512)
    rows = residue_rows(rep.ref)
    rec = compare(eng, rows, f"models[{name}]", rep=rep, system_prompt=SYS, max_new_tokens=40,
                  ignore_eos=True)
    assert rec["steps"] == len(rows) * 39


@pytest.mark.parametrize("share", [True, False])
@pytest.mark.parametrize("n_prefix", [15, 16, 17, 31, 32, 33])
def test_prefix_lengths_around_page_boundaries(n_prefix, share):
    """15: no sharing; 16, 32: whole pages shared, no tail copy; 17, 31, 33: the partial last
    page of the prefix is copied into every row's first own page."""
    eng, rep = engine("tiny-qwen3", max_slots=8, max_prefill_tokens=512)
    sp = prompt_with_prefix(rep, n_prefix)
    rows = residue_rows(rep.ref, seed=n_prefix)
    rec = compare(eng, rows, f"prefix[{n_prefix},share={share}]", rep=rep, system_prompt=sp,
                  max_new_tokens=36, ignore_eos=True, share_prefix=share)
    assert (rec["tail_copy_rows"] > 0) == (share and n_prefix % PAGE != 0 and n_prefix > PAGE)


GEOMETRIES = {
    "slots1": dict(max_slots=1, max_prefill_tokens=512),
    "slots3": dict(max_slots=3, max_prefill_tokens=512),
    "slots8_admit1": dict(max_slots=8, max_prefill_tokens=512, min_admit_rows=1),
    "tight_prefill": dict(max_slots=8, max_prefill_tokens=96),
    "chunk1": dict(max_slots=8, max_prefill_tokens=512, logit_chunk_rows=1),
    "chunk3_admit1": dict(max_slots=8, max_prefill_tokens=512, logit_chunk_rows=3,
                          min_admit_rows=1),
    "page_pressure": dict(max_slots=16, max_prefill_tokens=1024, kv_pages="two rows"),
}


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_scheduling_geometry_matches_the_replay(geometry):
    """The same rows (sampled decoding, per-row Philox streams) under slot counts, prefill
    budgets, admission thresholds, LM-head chunks and a KV pool that holds about two rows."""
    kw = dict(GEOMETRIES[geometry])
    max_new = 40
    _, prep = engine("tiny-qwen3-g4", max_slots=8, max_prefill_tokens=512)
    sp = prompt_with_prefix(prep, 37)          # 2 shared pages + a 5-token tail copy
    job = dict(system_prompt=sp, max_new_tokens=max_new, ignore_eos=True, temperature=0.9,
               top_k=50, top_p=0.95, seed=17, seed_per_row=True)
    if kw.get("kv_pages") == "two rows":
        rows = residue_rows(prep.ref, seed=3)
        pre, _ = prep.framing(sp)
        tpl = prep.template(sp)
        own = max((len(prep.ref.render(tpl, r)) + max_new + PAGE - 1) // PAGE - len(pre) // PAGE
                  for r in rows)
        kw["kv_pages"] = max(8, (len(pre) + PAGE - 1) // PAGE + 2 * own + 1)
    eng, rep = engine("tiny-qwen3-g4", **kw)
    rows = residue_rows(rep.ref, seed=3)
    rec = compare(eng, rows, f"geometry[{geometry}]", rep=rep, **job)
    if geometry == "page_pressure":
        assert rec["page_wait_admissions"] > 0, rec
    if geometry.startswith("chunk"):
        assert rec["chunked_head_launches"] > 0, rec
    if geometry == "tight_prefill":
        assert rec["prefill_steps"] > (len(rows) + 7) // 8, rec
    assert rec["tail_copy_rows"] > 0, rec


def test_recycled_pages_with_stale_kv():
    """A different job first, so the test job runs on pages and slots that hold its K/V."""
    eng = build("tiny-qwen3", max_slots=4, max_prefill_tokens=512, kv_pages=64)
    rep = Replay(eng)
    try:
        eng.generate(synth.product_reviews(10, seed=40), system_prompt="Summarise the review.",
                     max_new_tokens=48, ignore_eos=True)
        rows = residue_rows(rep.ref, seed=41)
        rec = compare(eng, rows, "stale_pages", rep=rep, system_prompt=SYS, max_new_tokens=40,
                      ignore_eos=True)
        assert rec["tail_copy_rows"] > 0
    finally:
        eng.close()


EDGE_ROWS = ["word " * 600, "", None]      # truncated to the context window, empty, null


@pytest.mark.parametrize("jump", [True, False])
@pytest.mark.parametrize("schema_model", [SentimentEnum, Extract])
def test_schema_jobs_match_the_replay(schema_model, jump):
    eng, rep = engine("tiny-qwen3", max_slots=8, max_prefill_tokens=512)
    rows = synth.README_REVIEWS + synth.product_reviews(9, seed=7) + EDGE_ROWS[1:]
    rec = compare(eng, rows, f"schema[{schema_model.__name__},jump={jump}]", rep=rep,
                  system_prompt=SYS, json_schema=schema_model.model_json_schema(),
                  fsm_limits=LIM, max_new_tokens=64, jump_forward=jump)
    assert rec["steps"] > 0
    # jump=True must really run with a forced output prefix, or it repeats the jump=False case
    assert (rec["forced_prefix_tokens"] > 0) == jump, rec


# EOS aliased onto a token the seeded tiny-qwen3 emits in some rows' greedy continuations
EOS_ALIAS = 156


@pytest.mark.parametrize("ignore_eos", [False, True])
def test_greedy_eos_and_max_new_tokens(ignore_eos):
    eng, rep = engine("tiny-qwen3", eos_alias=EOS_ALIAS, max_slots=8, max_prefill_tokens=512)
    rows = synth.product_reviews(12, seed=7) + EDGE_ROWS
    rec = compare(eng, rows, f"greedy[ignore_eos={ignore_eos}]", rep=rep, system_prompt=SYS,
                  max_new_tokens=40, ignore_eos=ignore_eos)
    assert rec["truncated"] == 1
    assert rec["max_new_stops"] > 0
    assert (rec["eos_stops"] > 0) != ignore_eos, rec


def test_sampled_rows_with_explicit_row_ids():
    eng, rep = engine("tiny-qwen3", max_slots=8, max_prefill_tokens=512, logit_chunk_rows=3)
    rows = residue_rows(rep.ref, seed=9) + EDGE_ROWS
    ids = [1000 + 7 * i for i in range(len(rows))]
    rec = compare(eng, rows, "sampled_row_ids", rep=rep, system_prompt=SYS, max_new_tokens=36,
                  temperature=0.8, top_k=30, top_p=0.9, seed=5, seed_per_row=True, row_ids=ids)
    assert rec["truncated"] == 1 and rec["chunked_head_launches"] > 0


@pytest.mark.parametrize("kind", ["schema_jump", "sampled", "greedy"])
def test_one_call_entry_point_matches_the_replay(kind):
    """sb200_infer_text compacts and detokenises on its own path; its tokens and cumulative
    log-probabilities must equal the replay too."""
    eng, rep = engine("tiny-qwen3", max_slots=4, max_prefill_tokens=512)
    rows = synth.product_reviews(9, seed=6) + EDGE_ROWS
    kw = {"schema_jump": dict(system_prompt=SYS, json_schema=SentimentEnum.model_json_schema(),
                              max_new_tokens=32),
          "sampled": dict(max_new_tokens=20, temperature=0.8, top_k=30, seed=4, seed_per_row=True),
          "greedy": dict(system_prompt=SYS, max_new_tokens=34, ignore_eos=True)}[kind]
    rec = compare(eng, rows, f"one_call[{kind}]", one_call=True, rep=rep, **kw)
    assert rec["truncated"] == 1 and rec["steps"] > 0
    assert (rec["forced_prefix_tokens"] > 0) == (kind == "schema_jump"), rec
    assert (rec["tail_copy_rows"] > 0) == (kind != "sampled"), rec


def test_embedding_model_matches_the_replay():
    eng, rep = engine("tiny-qwen3-embedding", max_slots=4, max_prefill_tokens=1024)
    rows = residue_rows(rep.ref, seed=12) + EDGE_ROWS
    rec = compare(eng, rows, "embedding", rep=rep)
    assert rec["truncated"] == 1


@pytest.mark.parametrize("name", ["qwen-3-4b", "llama-3.1-8b"])
def test_real_size_models_match_the_replay(name):
    from sutro_b200.engine import LocalEngine
    spec = MS.get_spec(name)
    w = MS.make_engine_weights_on_device(spec, 0, "cuda")
    v = VB.build_vocab(spec.family, spec.vocab_size, seed=0)
    eng = LocalEngine(spec, w, v, device=0, kv_pages=256, max_slots=4, max_prefill_tokens=1024,
                      logit_chunk_rows=3)
    try:
        rows = [synth.README_REVIEWS[0], synth.product_reviews(3, seed=21)[1], "ok", ""]
        rec = compare(eng, rows, f"real_size[{name}]", system_prompt=SYS, max_new_tokens=9,
                      ignore_eos=True)
        # the first token comes from the prefill, then 8 decode steps per row
        assert rec["steps"] == 4 * 8 and rec["chunked_head_launches"] > 0
    finally:
        eng.close()
        del eng, w
        torch.cuda.empty_cache()
