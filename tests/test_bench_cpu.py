"""bench.py runs unattended: check on CPU that it imports, parses its command line, and that
its host-only helpers work (the GPU arms need an H100)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bench_imports_and_prints_usage():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--help"],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    for flag in ("--gpus", "--steps", "--warmup", "--impl", "--rows", "--workload",
                 "--no-secondary", "--dump-outputs"):
        assert flag in out.stdout


def test_host_helpers(tmp_path):
    sys.path.insert(0, ROOT)
    import numpy as np
    import bench
    from sutro_b200 import synth
    rows = synth.product_reviews(500, seed=0)
    p = bench.plumbing_cost("qwen-3-4b", rows, ['{"sentiment":"positive"}'] * len(rows))
    assert p["rows"] == 500 and p["rows_per_s"] > 0 and p["payload_bytes"] > 500
    # --dump-outputs: what the caller received, as float arrays that round-trip exactly
    outs = ['{"sentiment":"positive"}', '{"sentiment":"négatif"}', ""]

    class Job:
        cum_logprobs = np.array([-0.5, -1.25, 0.0], dtype=np.float32)
        confidence = np.exp(cum_logprobs.astype(np.float64))
    bench.dump_outputs(str(tmp_path), outs, Job)
    text = np.load(tmp_path / "outputs_utf8.npy")
    n = np.load(tmp_path / "output_bytes.npy")
    assert text.dtype == np.float32 and n.dtype == np.float64
    assert [bytes(text[i, :int(n[i])].astype(np.uint8)).decode() for i in range(3)] == outs
    assert np.array_equal(np.load(tmp_path / "cum_logprobs.npy"), Job.cum_logprobs)
    assert np.load(tmp_path / "confidence.npy").dtype == np.float64
    assert not (tmp_path / "sample_rows.npy").exists()
    pk = bench.peaks()
    assert pk["hbm_gbs"] > 1000 and pk["bf16_tflops_sustained"] > 100
    json.dumps(bench.SCHEMA)
    assert len(bench.make_rows(7, seed=1)) == 7
    # the nested configs[4] schema compiles, and the frame shape SURVEY.md §8d names is met:
    # synthetic reviews average ~96 tokens under the synthetic vocabulary
    from sutro_b200.schema_fsm import FsmLimits, compile_schema
    d = compile_schema(bench.ORDER_SCHEMA, FsmLimits(max_string_chars=12, max_array_items=3))
    assert d.matches(b'{"customer":"x","items":[{"name":"a","quantity":3,"kind":"b","price":null}],'
                     b'"paid":true}')
    kw = bench.infer_kwargs("qwen-3-4b")
    assert kw["output_schema"] == bench.SCHEMA and kw["column"] == bench.COLUMN


def test_synthetic_review_length_matches_the_survey_shape():
    sys.path.insert(0, ROOT)
    import numpy as np
    from oracle.bpe_ref import RefTokenizer
    from sutro_b200 import modelspec as MS
    from sutro_b200 import synth, vocab as VB
    spec = MS.get_spec("qwen-3-4b")
    tok = RefTokenizer(VB.build_vocab(spec.family, spec.vocab_size, seed=0))
    n = [len(tok.encode(r)) for r in synth.product_reviews(400, seed=5)]
    assert 80 <= np.mean(n) <= 110 and min(n) >= 12 and max(n) <= 300, (np.mean(n), min(n), max(n))
    assert tok.decode(tok.encode("round trip, 100% exact")) == "round trip, 100% exact"


def test_smoke_and_build_entry_points_exist():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    assert callable(g.build) and callable(g.smoke)
