"""The job options of the three Python entry points (`JobOptions`): the keywords each method
accepts and their defaults, and the sb200_job fields `_job_options` fills from them.  No GPU:
the methods are called on an engine object that was never constructed, so any device work
would fail with an AttributeError before it started."""
import dataclasses
import inspect

import numpy as np
import pytest

from sutro_b200 import engine as E
from sutro_b200 import modelspec as MS

REQUIRED = inspect.Parameter.empty

# the job knobs every entry point takes, with their defaults
JOB = {"system_prompt": None, "json_schema": None, "max_new_tokens": 64, "ignore_eos": False,
       "truncate_rows": True, "share_prefix": True, "fsm_limits": None, "jump_forward": True,
       "temperature": 0.0, "top_k": 0, "top_p": 1.0, "seed": 0, "seed_per_row": False,
       "thinking_chars": None, "presence_penalty": 0.0, "frequency_penalty": 0.0,
       "repetition_penalty": 1.0, "min_p": 0.0}

# what each method accepts by keyword, with its default
KEYWORDS = {
    "generate": {"rows": REQUIRED, **JOB, "progress": None, "return_tokens": False,
                 "return_text": True, "profile": False, "return_first_logits": False,
                 "return_logprobs": False, "row_ids": None},
    "run_blob_dev": {"d_text": REQUIRED, "d_off": REQUIRED, "n_rows": REQUIRED,
                     "n_bytes": REQUIRED, **JOB, "progress": None, "return_text": True,
                     "profile": False, "return_first_logits": False, "return_logprobs": False,
                     "row_ids": None},
    "infer_one_call": {"rows": REQUIRED, **JOB, "progress": None, "return_tokens": True,
                       "profile": False, "return_logprobs": False},
}
ARGS = {"generate": {"rows": ["a"]}, "infer_one_call": {"rows": ["a"]},
        "run_blob_dev": {"d_text": None, "d_off": None, "n_rows": 1, "n_bytes": 1}}


def accepted_keywords(fn):
    """name -> default of every keyword `fn` binds; `**options` stands for JobOptions' fields."""
    out = {}
    for p in inspect.signature(fn).parameters.values():
        if p.kind is p.VAR_KEYWORD:
            out.update({f.name: f.default for f in dataclasses.fields(E.JobOptions)})
        elif p.kind in (p.POSITIONAL_OR_KEYWORD, p.KEYWORD_ONLY) and p.name != "self":
            out[p.name] = p.default
    return out


def bare_engine():
    return E.LocalEngine.__new__(E.LocalEngine)


def test_job_options_declares_the_job_knobs_and_their_defaults():
    assert {f.name: f.default for f in dataclasses.fields(E.JobOptions)} == JOB


@pytest.mark.parametrize("method", sorted(KEYWORDS))
def test_entry_point_keywords_and_defaults(method):
    want = KEYWORDS[method]
    assert accepted_keywords(getattr(E.LocalEngine, method)) == want
    # every keyword binds: the call gets past its arguments to the engine's missing attributes
    for name, default in want.items():
        if default is REQUIRED:
            continue
        with pytest.raises(AttributeError):
            getattr(bare_engine(), method)(**ARGS[method], **{name: default})


@pytest.mark.parametrize("method", sorted(KEYWORDS))
@pytest.mark.parametrize("keyword", ["not_an_option", "stop", "balance"])
def test_unknown_keyword_raises_type_error_before_device_work(method, keyword):
    with pytest.raises(TypeError, match=keyword):
        getattr(bare_engine(), method)(**ARGS[method], **{keyword: 1})


@pytest.mark.parametrize("method,keyword", [
    ("infer_one_call", "row_ids"), ("infer_one_call", "return_first_logits"),
    ("infer_one_call", "return_text"), ("run_blob_dev", "return_tokens")])
def test_call_keywords_stay_with_their_method(method, keyword):
    with pytest.raises(TypeError, match=keyword):
        getattr(bare_engine(), method)(**ARGS[method], **{keyword: None})


JOBC_FIELDS = ("n_prefix", "n_suffix", "share_prefix", "max_new_tokens", "ignore_eos",
               "truncate_rows", "fsm_states", "fsm_start", "n_forced_prefix", "temperature",
               "top_k", "top_p", "seed", "seed_per_row", "presence_penalty", "frequency_penalty",
               "repetition_penalty", "min_p")


@pytest.mark.parametrize("options,template_args,want", [
    ({}, (None, False),
     (3, 2, 1, 64, 0, 1, 0, 0, 0, 0.0, 0, 1.0, 0, 0, 0.0, 0.0, 1.0, 0.0)),
    (dict(system_prompt="sys", max_new_tokens=17, ignore_eos=True, truncate_rows=False,
          share_prefix=False, temperature=0.7, top_k=40, top_p=0.9, seed=-1, seed_per_row=True,
          presence_penalty=0.5, frequency_penalty=-0.25, repetition_penalty=1.5, min_p=0.05),
     ("sys", False),
     (3, 2, 0, 17, 1, 0, 0, 0, 0, 0.699999988079071, 40, 0.8999999761581421,
      18446744073709551615, 1, 0.5, -0.25, 1.5, 0.05000000074505806)),
])
def test_job_options_fill_the_job_struct(options, template_args, want):
    eng = bare_engine()
    eng.spec = MS.get_spec("tiny-qwen3")
    asked = []
    pre, suf = np.array([5, 6, 7], np.int32), np.array([8, 9], np.int32)
    eng._template_tokens = lambda system_prompt, thinking: asked.append(
        (system_prompt, thinking)) or (pre, suf)
    job = E.JobC()
    dfa, plan, keep = eng._job_options(job, E.JobOptions(**options))
    assert (dfa, plan) == (None, None) and asked == [template_args]
    assert tuple(getattr(job, f) for f in JOBC_FIELDS) == want
    assert list(job.prefix_tokens[:3]) == [5, 6, 7] and list(job.suffix_tokens[:2]) == [8, 9]


def test_out_of_range_penalty_is_refused_when_the_job_is_filled():
    eng = bare_engine()
    eng.spec = MS.get_spec("tiny-qwen3")
    eng._template_tokens = lambda system_prompt, thinking: (np.zeros(1, np.int32),) * 2
    with pytest.raises(ValueError, match="repetition_penalty"):
        eng._job_options(E.JobC(), E.JobOptions(repetition_penalty=0.0))
