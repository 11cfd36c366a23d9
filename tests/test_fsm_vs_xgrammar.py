"""The schema automaton and the oracle's token masks against xgrammar (the constrained-
decoding library SURVEY.md §8(c) names as the mask oracle; installed version: 0.2.x).

Both sides get the same synthetic vocabulary as raw bytes and the same schema with compact
separators.  Along random walks through OUR automaton, at every step:

* schemas with a finite language (enums, bounded integers, booleans, fixed arrays, anyOf of
  those): the allowed-token set is IDENTICAL to xgrammar's, the end-of-sequence token
  included;
* open schemas (free strings, numbers, optional fields, nested models): ours is a SUBSET of
  xgrammar's — we cap string lengths and array sizes (FsmLimits), write numbers without an
  exponent and refuse raw control characters inside strings — and xgrammar accepts every
  token we pick.  `maxLength` is removed from the copy given to xgrammar: its bounded-string
  pattern has no escape sequences, which is narrower than JSON Schema (a length-1 string may
  be spelled "\\n").
"""
import copy
import json
from typing import List, Literal, Optional

import numpy as np
import pytest
from pydantic import BaseModel, Field

from oracle.fsm_ref import TokenFSM
from sutro_b200 import modelspec as MS, vocab as VB
from sutro_b200.schema_fsm import FsmLimits, compile_schema

# FINITE and OPEN are also the start of tests/schema_corpus.py, which GPU tests import on
# machines without xgrammar: skip the tests, not the import
try:
    import xgrammar as xgr
except ImportError:
    xgr = None
pytestmark = pytest.mark.skipif(xgr is None, reason="xgrammar not installed")


class Item(BaseModel):
    name: str = Field(max_length=6)
    qty: int = Field(ge=0, le=20)
    kind: Literal["a", "b", "c"]
    price: Optional[float] = None


class Order(BaseModel):
    items: List[Item] = Field(max_length=2)
    ok: bool


def obj(**props):
    return {"type": "object", "properties": props, "required": list(props)}


FINITE = {
    "enum": obj(sentiment={"type": "string", "enum": ["positive", "neutral", "negative"]}),
    "int_0_10": obj(score={"type": "integer", "minimum": 0, "maximum": 10}),
    "int_neg_120": obj(score={"type": "integer", "minimum": -5, "maximum": 120}),
    "bool_null": obj(a={"type": "boolean"}, b={"type": "null"}),
    "fixed_array": obj(r={"type": "array", "items": {"type": "string", "enum": ["A", "B", "C"]},
                          "minItems": 3, "maxItems": 3}),
    "mixed_literals": {"type": "array", "items": {"enum": [1, 2, "x"]}, "minItems": 0,
                       "maxItems": 2},
    "anyof": {"anyOf": [{"type": "integer", "minimum": 1, "maximum": 3},
                        {"type": "string", "enum": ["none"]}]},
    "const": obj(k={"const": "v"}, flag={"type": "boolean"}),
}
OPEN = {
    "free_string": obj(t={"type": "string"}),
    "bounded_string": obj(t={"type": "string", "maxLength": 5}),
    "number": obj(n={"type": "number"}),
    "nested_model": Order.model_json_schema(),
    "string_array": obj(tags={"type": "array", "items": {"type": "string"}}),
    "wide_integer": obj(n={"type": "integer", "minimum": -3000, "maximum": 70000}),
    "one_sided_integer": obj(n={"type": "integer", "minimum": 17}),
    "decimal_range": obj(x={"type": "number", "minimum": 0.5, "maximum": 12.25}),
    "pattern": obj(code={"type": "string", "pattern": "^[a-z]{2,4}-[0-9]+$"}),
    "date": obj(day={"type": "string", "format": "date"}),
    "uuid": obj(id={"type": "string", "format": "uuid"}),
    "tuple": obj(t={"type": "array", "prefixItems": [{"type": "integer"}, {"type": "boolean"}],
                    "items": False, "minItems": 2, "maxItems": 2}),
    "mapping": obj(d={"type": "object", "additionalProperties": {"type": "boolean"}}),
}


@pytest.fixture(scope="module")
def world():
    spec = MS.get_spec("tiny-qwen3")
    v = VB.build_vocab(spec.family, spec.vocab_size, seed=0, n_trained=600)
    enc = [bytes(b) for b in v.token_bytes]
    info = xgr.TokenizerInfo(enc, vocab_type=xgr.VocabType.RAW, vocab_size=v.vocab_size,
                             stop_token_ids=[v.eos_id])
    return v, xgr.GrammarCompiler(info)


def strip_max_length(s):
    if isinstance(s, dict):
        return {k: strip_max_length(x) for k, x in s.items() if k != "maxLength"}
    if isinstance(s, list):
        return [strip_max_length(x) for x in s]
    return s


def walk(v, compiler, schema, seed, exact, max_steps=160):
    theirs_schema = schema if exact else strip_max_length(copy.deepcopy(schema))
    cg = compiler.compile_json_schema(json.dumps(theirs_schema), any_whitespace=False,
                                      separators=(",", ":"), strict_mode=True)
    fsm = TokenFSM(compile_schema(schema, FsmLimits(max_string_chars=12, max_array_items=3)), v)
    matcher = xgr.GrammarMatcher(cg)
    bitmask = xgr.allocate_token_bitmask(1, v.vocab_size)
    rng = np.random.default_rng(seed)
    state, text = fsm.start, b""
    for _ in range(max_steps):
        mine = fsm.allowed(state).numpy()
        matcher.fill_next_token_bitmask(bitmask)
        theirs = np.unpackbits(bitmask.numpy().view(np.uint8),
                               bitorder="little")[:v.vocab_size].astype(bool)
        extra = np.nonzero(mine & ~theirs)[0]
        assert len(extra) == 0, (text, [v.token_bytes[i] for i in extra[:5]])
        if exact:
            missing = np.nonzero(theirs & ~mine)[0]
            assert len(missing) == 0, (text, [v.token_bytes[i] for i in missing[:5]])
        allowed = np.nonzero(mine)[0]
        assert len(allowed) > 0, text                    # no dead ends before a final state
        tok = int(rng.choice(allowed))
        if tok == v.eos_id:
            assert matcher.accept_token(tok) and matcher.is_terminated()
            return text
        assert matcher.accept_token(tok), (text, v.token_bytes[tok])
        text += bytes(v.token_bytes[tok])
        state = fsm.step(state, tok)
        if fsm.is_final(state) and not fsm.allowed(state).numpy().any():
            return text
    pytest.fail(f"walk did not terminate: {text!r}")


@pytest.mark.parametrize("name", sorted(FINITE))
def test_masks_equal_xgrammar_on_finite_schemas(world, name):
    v, compiler = world
    for seed in range(6):
        out = walk(v, compiler, FINITE[name], seed, exact=True)
        json.loads(out)


@pytest.mark.parametrize("name", sorted(OPEN))
def test_masks_are_a_subset_of_xgrammar_on_open_schemas(world, name):
    v, compiler = world
    for seed in range(6):
        out = walk(v, compiler, OPEN[name], seed, exact=False)
        json.loads(out)
