"""BASELINE.json configs[1] at FULL size (20,000 rows, qwen-3-4b architecture, bf16) through
size-independent properties (the file name sorts it last: it is the heaviest test) — the CPU oracle cannot run this size, so the checks are the ones
the domain offers:

* every output parses as JSON and validates against the schema (constrained decoding is exact);
* results are positional AND batch-invariant: planted duplicate rows get the same output
  wherever they sit in the frame, and a shuffled 2,000-row subset run on its own reproduces the
  full run's outputs — exactly, every row.  Which kernel variant / tile shape runs never depends
  on the batch composition (decode attention: one kernel; prefill attention: KV blocks by the
  row's own positions; GEMMs: the K loop order is the same in every tile shape), so a row's
  greedy tokens do not depend on its neighbours.  The measured agreement is printed
  (a PARITY line in the test output);
* counters add up (rows done, emitted tokens).
"""
import json
from typing import Literal

import numpy as np
import pytest
import torch
from pydantic import BaseModel

pytestmark = pytest.mark.gpu

N_ROWS = 20000
SYSTEM_PROMPT = ("Classify the sentiment of the product review as positive, neutral or negative. "
                 "Answer with JSON.")


class Sentiment(BaseModel):
    sentiment: Literal["positive", "neutral", "negative"]


def make_engine():
    from sutro_b200.engine import LocalEngine
    return LocalEngine.from_seed("qwen-3-4b", seed=0, device=0, max_slots=3584,
                                 max_prefill_tokens=32768)


def planted_rows(n, n_pairs, seed):
    from sutro_b200 import synth
    rows = synth.product_reviews(n, seed=seed)
    rng = np.random.RandomState(seed)
    src = rng.choice(n // 2, size=n_pairs, replace=False)
    dst = n // 2 + rng.choice(n - n // 2, size=n_pairs, replace=False)
    for a, b in zip(src, dst):
        rows[b] = rows[a]
    return rows, list(zip(src.tolist(), dst.tolist()))


def check_full_size_properties(eng, n_rows=N_ROWS, n_pairs=500, n_subset=2000):
    rows, pairs = planted_rows(n_rows, n_pairs, seed=0)
    kw = dict(system_prompt=SYSTEM_PROMPT, json_schema=Sentiment.model_json_schema(),
              max_new_tokens=24, return_tokens=True)
    full = eng.generate(rows, **kw)
    assert len(full.outputs) == n_rows and full.stats["rows_done"] == n_rows
    for text in full.outputs:                                   # exact: by construction
        Sentiment.model_validate(json.loads(text))
    assert full.stats["output_tokens"] == sum(len(t) for t in full.out_tokens)
    assert all(0 < len(t) <= 24 for t in full.out_tokens)
    same = sum(full.outputs[a] == full.outputs[b] for a, b in pairs)
    idx = np.random.RandomState(1).permutation(n_rows)[:n_subset]
    part = eng.generate([rows[i] for i in idx], **kw)
    agree = sum(part.out_tokens[k] == full.out_tokens[i] for k, i in enumerate(idx))
    rec = {"test": "full_size_batch_invariance", "rows": n_rows, "duplicate_pairs_equal":
           f"{same}/{len(pairs)}", "subset_rows_equal": f"{agree}/{n_subset}"}
    print("PARITY", json.dumps(rec))
    assert same == len(pairs), (same, len(pairs))
    assert agree == n_subset, (agree, n_subset)
    labels = {json.loads(t)["sentiment"] for t in full.outputs}
    assert labels <= {"positive", "neutral", "negative"} and len(labels) >= 2
    return same, agree


def test_configs1_full_size_properties():
    eng = make_engine()
    try:
        check_full_size_properties(eng)
    finally:
        eng.close()
        del eng
        torch.cuda.empty_cache()
