"""The schemas the constrained-decoding tests share: every automaton they check, at the limits it
is decoded with.

Each entry says which compilers accept it (`native`: the C++ compiler behind
`sb200_schema_compile` accepts it too; the Python compiler accepts every entry) and how xgrammar
relates to it (`xgr`): "finite" — the language is finite, so the allowed-token sets must be
identical; "open" — we cap lengths and counts (FsmLimits), so ours must be a subset; None —
xgrammar has no JSON-Schema form for it (the thinking turn).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Dict, Optional

import bench
from sutro_b200.schema_fsm import ByteDFA, FsmLimits, compile_schema, compile_thinking
from test_engine_replay_gpu import LIM as REPLAY_LIMITS
from test_engine_replay_gpu import Extract, SentimentEnum
from test_fsm_vs_xgrammar import FINITE, OPEN

# the limits test_fsm_vs_xgrammar.walk and bench.py (configs[1] and [4]) compile with
WALK_LIMITS = FsmLimits(max_string_chars=12, max_array_items=3)
BENCH_LIMITS = FsmLimits(max_string_chars=12, max_array_items=3)


@dataclass(frozen=True)
class Entry:
    name: str
    schema: Optional[Dict[str, Any]]
    limits: FsmLimits
    native: bool                        # the C++ compiler accepts it as well
    xgr: Optional[str]                  # "finite", "open" or None
    thinking_chars: Optional[int] = None
    max_new: int = 64                   # max_new_tokens of the end-to-end runs
    non_ascii: bool = False             # forced strings split multi-byte characters

    def compile(self) -> ByteDFA:
        if self.thinking_chars is not None:
            return compile_thinking(self.schema, self.limits, self.thinking_chars)
        return compile_schema(self.schema, self.limits)

    def compile_native(self) -> ByteDFA:
        from sutro_b200.engine import native_compile_schema
        assert self.native, self.name
        return native_compile_schema(self.schema, self.limits)


def _obj(**props):
    return {"type": "object", "properties": props, "required": list(props)}


FORCED_PREFIX = _obj(greeting={"const": "hello from a forced prefix"}, ok={"type": "boolean"})

ENTRIES = (
    [Entry(f"finite.{k}", s, WALK_LIMITS, True, "finite") for k, s in sorted(FINITE.items())]
    + [Entry(f"open.{k}", s, WALK_LIMITS, k != "pattern", "open") for k, s in sorted(OPEN.items())]
    + [
        Entry("bench.SCHEMA", bench.SCHEMA, BENCH_LIMITS, True, "finite", max_new=bench.MAX_NEW),
        Entry("bench.ORDER_SCHEMA", bench.ORDER_SCHEMA, BENCH_LIMITS, True, "open", max_new=96),
        Entry("replay.SentimentEnum", SentimentEnum.model_json_schema(), REPLAY_LIMITS, True,
              "finite"),
        Entry("replay.Extract", Extract.model_json_schema(), REPLAY_LIMITS, True, "open"),
        Entry("non_ascii.enum", _obj(city={"type": "string", "enum": ["café", "東京", "Zürich"]}),
              WALK_LIMITS, True, "finite", non_ascii=True),
        # two-byte characters only: every split tail starts with exactly one continuation byte
        Entry("non_ascii.latin", _obj(word={"type": "string", "enum": ["café", "naïve"]}),
              WALK_LIMITS, True, "finite", non_ascii=True),
        Entry("non_ascii.const", _obj(city={"const": "東京"}, n={"type": "integer", "minimum": 0,
                                                                  "maximum": 9}),
              WALK_LIMITS, True, "finite"),     # forced whole, inside the prefix: no split
        # the forced prefix {"greeting":"hello from a forced prefix","ok": is longer than the
        # output budget in tokens: the plan is dropped and the model writes it itself
        Entry("forced_prefix", FORCED_PREFIX, WALK_LIMITS, True, "finite", max_new=8),
        # an accepting state with exactly one continuation ("1" may stop or go on to "12")
        Entry("accepting_prefix", {"enum": [1, 12, 123]}, WALK_LIMITS, True, "finite"),
        Entry("thinking", bench.SCHEMA, BENCH_LIMITS, False, None, thinking_chars=16, max_new=48),
        Entry("large", _obj(n={"type": "integer", "minimum": -3000, "maximum": 70000},
                            a={"type": "string", "maxLength": 200},
                            b={"type": "string", "maxLength": 200}),
              WALK_LIMITS, True, "open", max_new=32),
    ])
BY_NAME = {e.name: e for e in ENTRIES}
