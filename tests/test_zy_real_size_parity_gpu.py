"""Parity at the REAL model sizes BASELINE.json names (qwen-3-4b, llama-3.1-8b,
qwen-3-embedding-0.6b; seeded random weights drawn on the GPU, the CPU oracle runs on a host
copy of the very same tensors): first-decision logits of a few rows against oracle/model_ref.py.
The file name sorts it near the end of the suite (it is heavy: the oracle multiplies 4-8 B
parameter models on the host cores).

A 32-36 layer bf16 network rounds ~10 times per layer; two correct bf16 implementations that
only differ in fp32 summation order therefore do not agree to the 0.03 sigma the two-layer test
models reach (tests/test_engine_gpu.py).  The yardstick here is the rounding noise itself: the
oracle is run twice per row, once with its bf16 rounding points (the engine's contract) and
once in fp32 throughout on the same bf16-valued weights (`exact`), and the engine must sit as
close to the exact logits as the bf16 oracle does.

Tolerances, in units of the row's logit standard deviation sigma (written once, used below):
  rms(engine - exact)   <= 1.5 x rms(bf16 oracle - exact) + 0.005     (noise-floor criterion)
  rms(engine - bf16 oracle) over the vocabulary  < 0.08 sigma, worst single logit < 0.40 sigma
  a different arg-max only inside the near-tie band (oracle margin < 0.06)
  embedding cosine      > 0.999
Measured values are printed (PARITY_REAL_SIZE lines in the test output)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle.bpe_ref import RefTokenizer
from oracle.model_ref import RefModel
from sutro_b200 import modelspec as MS
from sutro_b200 import synth, vocab as VB

pytestmark = pytest.mark.gpu

RMS_TOL, MAX_TOL, COS_TOL = 0.08, 0.40, 0.999
NOISE_FACTOR, NOISE_SLACK = 1.5, 0.005
SYS = synth.README_SYSTEM_PROMPT
ROWS = [synth.README_REVIEWS[0], synth.product_reviews(3, seed=21)[1],
        synth.product_reviews(3, seed=22)[2], "ok"]


def _record(rec):
    print("PARITY_REAL_SIZE", json.dumps(rec))


def _build(name, **kw):
    from sutro_b200.engine import LocalEngine
    spec = MS.get_spec(name)
    w = MS.make_engine_weights_on_device(spec, 0, "cuda")
    v = VB.build_vocab(spec.family, spec.vocab_size, seed=0)
    eng = LocalEngine(spec, w, v, device=0, kv_pages=2048, max_slots=16, max_prefill_tokens=4096,
                      **kw)
    return spec, w, v, eng


@pytest.mark.parametrize("name", ["qwen-3-4b", "llama-3.1-8b"])
def test_first_decision_logits_match_the_oracle_at_real_size(name):
    torch.set_num_threads(min(64, os.cpu_count() or 1))
    spec, w, v, eng = _build(name)
    try:
        res = eng.generate(ROWS, system_prompt=SYS, max_new_tokens=1, ignore_eos=True,
                           return_tokens=True, return_first_logits=True)
        model, tok = RefModel(spec, MS.unpack_to_hf(spec, w), fast=True), RefTokenizer(v)
        tpl = VB.chat_template(spec.family, SYS)
        worst_rms = worst_max = 0.0
        agree = 0
        noise_eng, noise_orc = [], []
        for i, row in enumerate(ROWS):
            prompt = tok.render(tpl, row)
            assert eng.tokenizer.encode([row])[0] == tok.encode(row)
            want = model.logits(prompt)[-1]
            got = res.first_logits[i]
            sd = want.std().item()
            d = (got - want).abs()
            rms, mx = d.pow(2).mean().sqrt().item() / sd, d.max().item() / sd
            worst_rms, worst_max = max(worst_rms, rms), max(worst_max, mx)
            if i < 2:      # the unrounded pass costs as much as the rounded one: two rows
                exact = model.logits(prompt, exact=True)[-1]
                noise_eng.append((got - exact).pow(2).mean().sqrt().item() / sd)
                noise_orc.append((want - exact).pow(2).mean().sqrt().item() / sd)
            top2 = torch.topk(want, 2).values
            margin = (top2[0] - top2[1]).item()
            same = int(got.argmax()) == int(want.argmax())
            agree += same
            # a different arg-max is only acceptable inside the near-tie band
            assert same or margin < 0.06, (name, i, margin)
            assert res.out_tokens[i][0] == int(got.argmax())
        _record({"model": name, "rows": len(ROWS), "logit_rms_over_sigma": worst_rms,
                 "logit_max_over_sigma": worst_max, "argmax_equal": f"{agree}/{len(ROWS)}",
                 "rms_engine_vs_exact": noise_eng, "rms_bf16_oracle_vs_exact": noise_orc})
        assert worst_rms < RMS_TOL and worst_max < MAX_TOL, (worst_rms, worst_max)
        for e, o in zip(noise_eng, noise_orc):
            assert e <= NOISE_FACTOR * o + NOISE_SLACK, (e, o)
    finally:
        eng.close()
        del eng, w
        torch.cuda.empty_cache()


def test_embeddings_match_the_oracle_at_real_size():
    torch.set_num_threads(min(64, os.cpu_count() or 1))
    spec, w, v, eng = _build("qwen-3-embedding-0.6b")
    try:
        rows = synth.short_texts(6, seed=2)
        res = eng.generate(rows)
        model, tok = RefModel(spec, MS.unpack_to_hf(spec, w), fast=True), RefTokenizer(v)
        tpl = VB.embedding_template(spec.family)
        cos = []
        for i, row in enumerate(rows):
            want = model.embed(tok.render(tpl, row)).numpy()
            cos.append(float(res.embeddings[i] @ want))
            assert abs(np.linalg.norm(res.embeddings[i]) - 1.0) < 1e-3
        _record({"model": spec.name, "rows": len(rows), "min_cosine": min(cos)})
        assert min(cos) > COS_TOL, cos
    finally:
        eng.close()
        del eng, w
        torch.cuda.empty_cache()
