"""The CPU mask reference (tests/mask_ref.py) against xgrammar at full vocabulary size.

tests/test_constrained_exact_gpu.py requires the GPU masks to equal mask_ref bit for bit; this
file pins mask_ref itself to xgrammar, on the qwen3 (151,936) and llama (128,256) synthetic
vocabularies, for the Python and the native automaton of every corpus schema xgrammar can
express (tests/schema_corpus.py).  Along seeded walks that prefer long tokens (a multi-byte
token is where a schema's structure gets split), at every step:

* finite languages: the allowed set equals xgrammar's, the end-of-sequence token included;
* open languages: ours is a subset of xgrammar's (our caps: FsmLimits, numbers without an
  exponent, no raw control characters in strings), and xgrammar accepts every token chosen.
  xgrammar gets the schema without `maxLength` (as in test_fsm_vs_xgrammar.py) and without the
  bounds of a `number` with fractional bounds: xgrammar 0.2.x refuses to end {"x":12} under
  0.5 <= x <= 12.25.  Those bounds are checked by validating what the automaton accepts
  (tests/test_schema_features.py).
"""
import copy
import json

import numpy as np
import pytest

import mask_ref as M
from schema_corpus import ENTRIES
from sutro_b200 import vocab as VB
from test_fsm_vs_xgrammar import strip_max_length

xgr = pytest.importorskip("xgrammar")

FULL = {"qwen3": 151936, "llama": 128256}
CASES = [(fam, e.name, compiler) for fam in FULL for e in ENTRIES if e.xgr is not None
         for compiler in ("python", "native") if compiler == "python" or e.native]
WALKS = 2


def loosen(schema):
    """The copy of an open schema given to xgrammar (see the module docstring)."""
    def drop_fractional_bounds(s):
        if isinstance(s, list):
            return [drop_fractional_bounds(x) for x in s]
        if not isinstance(s, dict):
            return s
        frac = s.get("type") == "number" and any(
            isinstance(s.get(k), float) and not float(s[k]).is_integer()
            for k in ("minimum", "maximum", "exclusiveMinimum", "exclusiveMaximum"))
        return {k: drop_fractional_bounds(x) for k, x in s.items()
                if not (frac and k in ("minimum", "maximum", "exclusiveMinimum",
                                       "exclusiveMaximum"))}
    return drop_fractional_bounds(strip_max_length(copy.deepcopy(schema)))


@pytest.fixture(scope="module")
def worlds():
    cache = {}

    def get(fam):
        if fam not in cache:
            v = VB.build_vocab(fam, FULL[fam], seed=0)
            info = xgr.TokenizerInfo([bytes(b) for b in v.token_bytes], vocab_type=xgr.VocabType.RAW,
                                     vocab_size=v.vocab_size, stop_token_ids=[v.eos_id])
            cache[fam] = (v, M.VocabTrie(v.token_bytes), xgr.GrammarCompiler(info))
        return cache[fam]
    return get


def walk(v, trie, compiled, dfa, seed, exact, rows, max_steps=400):
    matcher = xgr.GrammarMatcher(compiled)
    bitmask = xgr.allocate_token_bitmask(1, v.vocab_size)
    rng = np.random.default_rng(seed)
    state, text, steps, multi = dfa.start, b"", 0, 0
    for _ in range(max_steps):
        if state not in rows:
            rows[state] = M.allowed(dfa.trans, dfa.accept, trie, v.eos_id, [state])[0]
        mine = rows[state]
        matcher.fill_next_token_bitmask(bitmask)
        theirs = np.unpackbits(bitmask.numpy().view(np.uint8),
                               bitorder="little")[:v.vocab_size].astype(bool)
        extra = np.nonzero(mine & ~theirs)[0]
        assert len(extra) == 0, (text, [v.token_bytes[i] for i in extra[:5]])
        if exact:
            missing = np.nonzero(theirs & ~mine)[0]
            assert len(missing) == 0, (text, [v.token_bytes[i] for i in missing[:5]])
        ids = np.nonzero(mine)[0]
        assert len(ids) > 0, text                      # no dead end before a final state
        steps += 1
        words = ids[ids != v.eos_id]
        if len(words) == 0 or (mine[v.eos_id] and rng.random() < 0.25):
            assert matcher.accept_token(v.eos_id) and matcher.is_terminated(), text
            return text, steps, multi
        w = trie.lens[words].astype(np.float64) ** 3   # prefer long tokens
        tok = int(rng.choice(words, p=w / w.sum()))
        assert matcher.accept_token(tok), (text, v.token_bytes[tok])
        text += v.token_bytes[tok]
        multi += len(v.token_bytes[tok]) > 1
        for b in v.token_bytes[tok]:
            state = int(dfa.trans[state, b])
        assert state >= 0, text
    pytest.fail(f"walk did not terminate: {text!r}")


@pytest.mark.parametrize("fam,name,compiler", CASES)
def test_mask_reference_equals_xgrammar(worlds, fam, name, compiler):
    e = next(x for x in ENTRIES if x.name == name)
    v, trie, gc = worlds(fam)
    dfa = e.compile() if compiler == "python" else e.compile_native()
    exact = e.xgr == "finite"
    theirs = e.schema if exact else loosen(e.schema)
    compiled = gc.compile_json_schema(json.dumps(theirs), any_whitespace=False,
                                      separators=(",", ":"), strict_mode=True)
    rows, steps, multi = {}, 0, 0
    for seed in range(WALKS):
        text, n, m = walk(v, trie, compiled, dfa, seed, exact, rows)
        steps, multi = steps + n, multi + m
        json.loads(text)
    print("PARITY", f"xgrammar[{fam},{name},{compiler}]", f"states={len(rows)}/{dfa.n_states}",
          f"tokens={v.vocab_size}", f"steps={steps}", f"multibyte={multi}", "exact" if exact else "subset")
