"""131,072-token windows at real size, on seeded weights: qwen-3-4b with YaRN and llama-3.1-8b,
each with a row of 131,064 prompt tokens, so that its eighth and last decode step attends to all
131,072 positions (32 splits of 4,096) over K/V that four prefill chunks wrote to the pool.
Every row must match the one-row replay bit for bit; the replay prefills each row in one step, so
the engine is closed first to give it the memory.  Then the public paths: `Sutro.infer` with
`engine_options={"max_position": 131072}`, and the C host serving a bundle written by
`python -m sutro_b200.bundle --max-position`."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_c_host_gpu as CH
import test_engine_replay_gpu as ER
from engine_replay import Replay
from sutro_b200 import _lib as L
from sutro_b200 import modelspec as MS
from sutro_b200 import synth, vocab as VB

pytestmark = pytest.mark.gpu
DEV = "cuda"
WINDOW = 131072
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def n_tok(eng, text):
    return len(eng.tokenizer.encode([text])[0])


def text_of(eng, n_body, seed):
    """A row of synthetic prose that the GPU tokenizer (exact against `tokenizers`) encodes to
    exactly n_body tokens."""
    words = " ".join(synth.documents(max(2, n_body // 300), seed=seed, words=500)).split()
    while n_tok(eng, " ".join(words)) < n_body + 64:
        words = words + words
    lo, hi = 1, len(words)
    while lo < hi:                              # fewest words with at least n_body tokens
        mid = (lo + hi) // 2
        if n_tok(eng, " ".join(words[:mid])) >= n_body:
            hi = mid
        else:
            lo = mid + 1
    text = " ".join(words[:lo])
    for cut in range(len(text), max(0, len(text) - 200), -1):
        if n_tok(eng, text[:cut]) == n_body:
            return text[:cut]
    raise AssertionError(f"no cut renders to {n_body} tokens")


def exact_prompt_row(eng, n_prompt, seed):
    pre, suf = eng._template_tokens(None)
    return text_of(eng, n_prompt - len(pre) - len(suf), seed)


def run_then_replay(eng, rows, label, **kw):
    res = eng.generate(rows, return_tokens=True, return_first_logits=True, return_logprobs=True,
                       **kw)
    rep = Replay(eng)
    eng.close()
    torch.cuda.empty_cache()
    reps = rep.job(rows, **kw)
    for i, r in enumerate(reps):
        assert res.out_tokens[i] == r.tokens, (label, i)
        assert torch.equal(ER.bits(res.first_logits[i]), ER.bits(r.first_logits)), (label, i)
        assert ER.bits(res.cum_logprobs[i]).item() == ER.bits(r.cum_logprob).item(), (label, i)
    print("REAL_LONG", label, [r.prompt_len for r in reps], res.stats["prefill_steps"],
          res.stats["decode_steps"], res.stats["rows_truncated"])
    assert res.stats["rows_truncated"] == 0
    return res, reps


def real_engine(name, kv_tokens):
    from sutro_b200.engine import LocalEngine
    spec = MS.with_window(MS.get_spec(name), WINDOW)
    w = MS.make_engine_weights_on_device(spec, 0, DEV)
    v = VB.build_vocab(spec.family, spec.vocab_size, seed=0)
    eng = LocalEngine(spec, w, v, device=0, kv_pages=kv_tokens // 16 + 256, max_slots=4)
    assert eng.max_prefill_tokens == 32768
    return eng, w


def test_qwen3_4b_yarn_131072_rows_match_replay():
    eng, w = real_engine("qwen-3-4b", WINDOW + 70100)
    assert eng.spec.rope_scaling["rope_type"] == "yarn"
    rows = [synth.README_REVIEWS[0], exact_prompt_row(eng, WINDOW - 8, seed=1), "ok",
            exact_prompt_row(eng, 70000, seed=2), synth.README_REVIEWS[1]]
    res, reps = run_then_replay(eng, rows, "qwen-3-4b yarn", max_new_tokens=8, ignore_eos=True)
    assert reps[1].prompt_len == WINDOW - 8 and reps[3].prompt_len == 70000
    assert all(r.decode_steps == 7 for r in reps)
    # the last decode step of the longest row attends to 131,072 positions in 32 splits
    assert -(-(reps[1].prompt_len + reps[1].decode_steps) // 4096) == 32
    # four chunks for the long row, three for the 70k row
    assert res.stats["prefill_steps"] >= 7
    del w
    torch.cuda.empty_cache()


def test_llama_131072_row_matches_replay():
    eng, w = real_engine("llama-3.1-8b", WINDOW + 1000)
    rows = [exact_prompt_row(eng, WINDOW - 8, seed=3), "ok"]
    _, reps = run_then_replay(eng, rows, "llama-3.1-8b", max_new_tokens=8, ignore_eos=True)
    assert reps[0].prompt_len == WINDOW - 8 and reps[0].decode_steps == 7
    del w
    torch.cuda.empty_cache()


def test_row_longer_than_the_window_is_truncated_or_refused():
    eng, w = real_engine("qwen-3-4b", WINDOW + 1000)
    try:
        rows = [exact_prompt_row(eng, WINDOW - 8 + 40, seed=4)]      # 40 tokens too many
        res = eng.generate(rows, max_new_tokens=8, ignore_eos=True)
        assert res.stats["rows_truncated"] == 1
        with pytest.raises(L.Sb200Error, match="truncate_rows=False"):
            eng.generate(rows, max_new_tokens=8, truncate_rows=False)
    finally:
        eng.close()
        del w
        torch.cuda.empty_cache()


def test_sutro_infer_with_a_131072_window_serves_a_100k_row(tmp_path):
    import pandas as pd
    from sutro_b200.interfaces import JobStatus
    from sutro_b200.sdk import Sutro
    so = Sutro(verbose=False, cache_dir=str(tmp_path), engine_options={"max_position": WINDOW})
    eng = so._engine("qwen-3-4b")
    try:
        assert eng.spec.max_position == WINDOW and eng.max_prefill_tokens == 32768
        df = pd.DataFrame({"text": [text_of(eng, 100000, seed=5), "fine"]})
        job_id = so.infer(df, model="qwen-3-4b", column="text",
                          sampling_params={"max_new_tokens": 4})
        st = so._job(job_id).stats
        print("SDK_131K", st["input_tokens"], st["rows_truncated"], st["prefill_steps"])
        assert so.get_job_status(job_id) == JobStatus.SUCCEEDED
        assert st["rows_truncated"] == 0 and st["input_tokens"] > 100000
        assert st["prefill_steps"] >= 4
    finally:
        eng.close()
        torch.cuda.empty_cache()


def test_c_host_serves_a_bundle_written_with_max_position(tmp_path):
    """`python -m sutro_b200.bundle --max-position` writes the raised window and its YaRN tables;
    the C host serves the bundle and prints what the Python host produces for the same model.
    tiny-qwen3 at 2,048 (YaRN x4) keeps the bundle small.  The C host opens it with a 512-token
    prefill budget, so its 900-token row (past the registered 512-token window) is prefilled in
    two chunks, while the Python engine's default budget holds the row whole; its default output
    budget is half the window, 1,024 tokens, which the Python call is given too."""
    from sutro_b200.engine import LocalEngine
    exe = CH._compile(tmp_path)
    bundle = str(tmp_path / "bundle")
    subprocess.run([sys.executable, "-m", "sutro_b200.bundle", "--model", "tiny-qwen3",
                    "--max-position", "2048", "--out", bundle], check=True, cwd=ROOT)
    manifest = json.load(open(os.path.join(bundle, "manifest.json")))
    assert manifest["spec"]["max_position"] == 2048
    eng = LocalEngine.from_seed("tiny-qwen3", seed=0, device=0, kv_pages=512, max_slots=8,
                                max_position=2048)
    try:
        off = manifest["tensors"]["rope_cos"]
        data = np.fromfile(os.path.join(bundle, "data.bin"), dtype=np.uint8,
                           count=off["bytes"], offset=off["offset"])
        assert np.array_equal(data, eng.cos.cpu().view(torch.uint8).numpy().reshape(-1))
        rows = [text_of(eng, 900, seed=6), synth.README_REVIEWS[0]]
        res = eng.generate(rows, system_prompt=None, max_new_tokens=1024)
        assert res.stats["rows_truncated"] == 0
        want = res.outputs
    finally:
        eng.close()
    out = subprocess.run([exe, bundle, "", "-"] + rows, capture_output=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    got = out.stdout.decode("utf-8", errors="replace").split("\n")
    assert got[0] == want[0].split("\n")[0]
