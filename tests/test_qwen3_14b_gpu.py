"""The engine at a GQA group of 5: the tiny G = 5 model (`tiny-qwen3-g5`, 10 query heads over 2
KV heads) against the one-row replay and the CPU oracle, and qwen-3-14b (40 over 8) at real size
on seeded weights, through the engine and through `Sutro.infer`.

The replay (tests/engine_replay.py) runs each row alone through the same kernels, so every job
here must match it bit for bit: greedy, sampled and schema jobs, shared prefixes around page
boundaries, 1, 3 and 16 slots, a tight prefill budget and rows whose context crosses the
4,096-token decode split.  Against the oracle the bars are those of test_engine_gpu.py (tiny)
and test_zy_real_size_parity_gpu.py (real size)."""
import json
import os
import random
import resource

import pytest
import torch

import test_engine_gpu as EG
import test_engine_replay_gpu as ER
import test_long_context_gpu as LC
import test_zy_real_size_parity_gpu as ZY
from engine_replay import Replay
from oracle.model_ref import RefModel
from oracle.bpe_ref import RefTokenizer
from sutro_b200 import modelspec as MS
from sutro_b200 import synth, vocab as VB

pytestmark = pytest.mark.gpu

TINY = "tiny-qwen3-g5"
_ENGINES = {}


def engine(**kw):
    key = tuple(sorted(kw.items()))
    if key not in _ENGINES:
        eng = ER.build(TINY, **kw)
        _ENGINES[key] = (eng, Replay(eng))
    return _ENGINES[key]


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for eng, _ in _ENGINES.values():
        eng.close()
    _ENGINES.clear()
    torch.cuda.empty_cache()


# --------------------------------------------------------------------------- tiny G = 5 model
def test_greedy_matches_the_replay():
    eng, rep = engine(max_slots=8, max_prefill_tokens=512)
    rows = ER.residue_rows(rep.ref)
    rec = ER.compare(eng, rows, "g5 greedy", rep=rep, system_prompt=ER.SYS, max_new_tokens=40,
                     ignore_eos=True)
    assert rec["steps"] == len(rows) * 39


@pytest.mark.parametrize("geometry", ["slots1", "slots3", "slots16", "tight_prefill"])
def test_sampled_jobs_match_the_replay(geometry):
    kw = {"slots1": dict(max_slots=1, max_prefill_tokens=512),
          "slots3": dict(max_slots=3, max_prefill_tokens=512),
          "slots16": dict(max_slots=16, max_prefill_tokens=1024),
          "tight_prefill": dict(max_slots=8, max_prefill_tokens=96)}[geometry]
    eng, rep = engine(**kw)
    sp = ER.prompt_with_prefix(rep, 37)
    rows = ER.residue_rows(rep.ref, seed=3)
    rec = ER.compare(eng, rows, f"g5 sampled[{geometry}]", rep=rep, system_prompt=sp,
                     max_new_tokens=40, ignore_eos=True, temperature=0.9, top_k=50, top_p=0.95,
                     seed=17, seed_per_row=True)
    if geometry == "tight_prefill":
        assert rec["prefill_steps"] > (len(rows) + 7) // 8, rec


@pytest.mark.parametrize("share", [True, False])
@pytest.mark.parametrize("n_prefix", [15, 16, 17, 46])
def test_prefix_lengths_match_the_replay(n_prefix, share):
    eng, rep = engine(max_slots=8, max_prefill_tokens=512)
    sp = ER.prompt_with_prefix(rep, n_prefix)
    rows = ER.residue_rows(rep.ref, seed=n_prefix)
    rec = ER.compare(eng, rows, f"g5 prefix[{n_prefix},share={share}]", rep=rep, system_prompt=sp,
                     max_new_tokens=36, ignore_eos=True, share_prefix=share)
    assert (rec["tail_copy_rows"] > 0) == (share and n_prefix % 16 != 0 and n_prefix > 16)


@pytest.mark.parametrize("jump", [True, False])
@pytest.mark.parametrize("schema_model", [ER.SentimentEnum, ER.Extract])
def test_schema_jobs_match_the_replay(schema_model, jump):
    eng, rep = engine(max_slots=8, max_prefill_tokens=512)
    rows = synth.README_REVIEWS + synth.product_reviews(9, seed=7) + ER.EDGE_ROWS[1:]
    rec = ER.compare(eng, rows, f"g5 schema[{schema_model.__name__},jump={jump}]", rep=rep,
                     system_prompt=ER.SYS, json_schema=schema_model.model_json_schema(),
                     fsm_limits=ER.LIM, max_new_tokens=64, jump_forward=jump)
    # with jump-forward the enum's label can be decided by the prefill's token alone
    assert rec["steps"] > 0 or jump, rec
    assert (rec["forced_prefix_tokens"] > 0) == jump, rec


def test_rows_cross_a_split_during_decode():
    """An 8,192-token window: rows of 4,095 and 4,096 prompt tokens cross 4,096 -> 4,097 during
    decode, beside short rows, greedy and sampled."""
    eng, _ = LC.tiny_engine(TINY, window=8192)
    try:
        ref = RefTokenizer(eng.vocab)
        tpl = VB.chat_template(eng.spec.family, None)
        shorts = synth.product_reviews(2, seed=14)
        longs = [LC.exact_row(ref, tpl, n, seed=100 + i) for i, n in enumerate((4095, 4096))]
        rows = [shorts[0], longs[0], shorts[1], longs[1]]
        rep = Replay(eng)
        kw = dict(max_new_tokens=12, ignore_eos=True)
        _, reps = LC.compare(eng, rows, "g5 split crossing greedy", rep, **kw)
        for i in (1, 3):
            P, steps = reps[i].prompt_len, reps[i].decode_steps
            assert P <= LC.SPLIT < P + steps, (P, steps)
        LC.compare(eng, rows, "g5 split crossing sampled", rep, temperature=0.8, top_p=0.9,
                   seed=7, **kw)
    finally:
        eng.close()


def test_greedy_matches_the_oracle():
    EG.test_unconstrained_greedy_matches_oracle(TINY)


def test_teacher_forced_logits_within_tolerance():
    EG.test_teacher_forced_logits_within_tolerance(TINY)


def test_rows_are_batch_invariant_under_shuffling():
    eng, _ = engine(max_slots=8, max_prefill_tokens=512)
    rows = synth.product_reviews(24, seed=19)
    kw = dict(system_prompt=ER.SYS, max_new_tokens=16, ignore_eos=True, return_tokens=True)
    base = eng.generate(rows, **kw).out_tokens
    order = list(range(len(rows)))
    random.Random(5).shuffle(order)
    shuf = eng.generate([rows[i] for i in order], **kw).out_tokens
    assert [shuf[order.index(i)] for i in range(len(rows))] == base


# --------------------------------------------------------------------------- qwen-3-14b
def test_qwen3_14b_matches_the_replay():
    """4 rows x 8 decode steps on seeded weights."""
    ER.test_real_size_models_match_the_replay("qwen-3-14b")


def test_qwen3_14b_first_decision_logits_match_the_oracle():
    """The bars of test_zy_real_size_parity_gpu.py.  The oracle runs with fast=False, so the host
    holds one bf16 copy of the weights (~30 GB) instead of an fp32 one."""
    name = "qwen-3-14b"
    torch.set_num_threads(min(64, os.cpu_count() or 1))
    spec, w, v, eng = ZY._build(name)
    rows = ZY.ROWS[:2]
    try:
        res = eng.generate(rows, system_prompt=ZY.SYS, max_new_tokens=1, ignore_eos=True,
                           return_tokens=True, return_first_logits=True)
        eng.close()
        model, tok = RefModel(spec, MS.unpack_to_hf(spec, w), fast=False), RefTokenizer(v)
        tpl = VB.chat_template(spec.family, ZY.SYS)
        worst_rms = worst_max = 0.0
        noise_eng, noise_orc = [], []
        for i, row in enumerate(rows):
            prompt = tok.render(tpl, row)
            want = model.logits(prompt)[-1]
            exact = model.logits(prompt, exact=True)[-1]
            got = res.first_logits[i]
            sd = want.std().item()
            d = (got - want).abs()
            worst_rms = max(worst_rms, d.pow(2).mean().sqrt().item() / sd)
            worst_max = max(worst_max, d.max().item() / sd)
            noise_eng.append((got - exact).pow(2).mean().sqrt().item() / sd)
            noise_orc.append((want - exact).pow(2).mean().sqrt().item() / sd)
            top2 = torch.topk(want, 2).values
            assert int(got.argmax()) == int(want.argmax()) or (top2[0] - top2[1]).item() < 0.06
        peak_gb = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
        ZY._record({"model": name, "rows": len(rows), "logit_rms_over_sigma": worst_rms,
                    "logit_max_over_sigma": worst_max, "rms_engine_vs_exact": noise_eng,
                    "rms_bf16_oracle_vs_exact": noise_orc, "peak_host_gb": round(peak_gb, 1)})
        assert worst_rms < ZY.RMS_TOL and worst_max < ZY.MAX_TOL, (worst_rms, worst_max)
        for e, o in zip(noise_eng, noise_orc):
            assert e <= ZY.NOISE_FACTOR * o + ZY.NOISE_SLACK, (e, o)
    finally:
        eng.close()
        del eng, w
        torch.cuda.empty_cache()


def test_qwen3_14b_through_sutro_infer(tmp_path):
    """`Sutro.infer(model="qwen-3-14b", output_schema=...)` gives valid JSON per row, and the
    -thinking name gives {content, reasoning_content} on the same weights."""
    import sutro_b200 as so
    client = so.configure(engine_options=dict(kv_pages=512, max_slots=8, max_prefill_tokens=512),
                          verbose=False, cache_dir=str(tmp_path))
    try:
        rows = synth.README_REVIEWS + synth.product_reviews(3, seed=8)
        job = so.infer(rows, model="qwen-3-14b", system_prompt=synth.README_SYSTEM_PROMPT,
                       output_schema=ER.SentimentEnum, stay_attached=False)
        raw = so.get_job_results(job, unpack_json=False)["inference_result"]
        assert len(raw) == len(rows)
        for text in raw:
            ER.SentimentEnum.model_validate(json.loads(text))
        job = so.infer(rows, model="qwen-3-14b-thinking",
                       system_prompt=synth.README_SYSTEM_PROMPT, output_schema=ER.SentimentEnum,
                       sampling_params={"max_thinking_chars": 24}, stay_attached=False)
        for text in so.get_job_results(job, unpack_json=False)["inference_result"]:
            obj = json.loads(text)
            assert sorted(obj) == ["content", "reasoning_content"]
            ER.SentimentEnum.model_validate(obj["content"])
        assert len(client._engines) == 1           # one set of weights for both names
    finally:
        for e in client._engines.values():
            e.close()
        client._engines.clear()
        torch.cuda.empty_cache()
